// The job queue and result store of a proof stream (dph_zkml_stream_*): tickets, capacity, timed waits and cancellation.  It knows
// nothing of the device or the prover: a job is a callable that the serving threads run, so the queue's logic is tested on the CPU
// with a fake job (tests/stream_queue_io.cpp).
#pragma once
#include <chrono>
#include <condition_variable>
#include <cstdint>
#include <deque>
#include <exception>
#include <functional>
#include <mutex>
#include <string>
#include <vector>
#include "../../include/deepprove_b200.h"

namespace dp {

struct QueueResult {
    uint64_t ticket = 0;
    int32_t status = 0;             // 0, or the job's error code
    std::string error;              // the job's message when status != 0
    std::vector<uint64_t> proof;    // empty when status != 0
    std::vector<int64_t> output;    // empty when status != 0
};

class ProofQueue {
public:
    // Runs one job: input points at input_len elements; backlog is the number of jobs that were waiting when this one was taken,
    // itself included.  A failure sets r.status and r.error (an escaping exception counts as status 1).
    using Job = std::function<void(const int64_t *input, uint64_t backlog, QueueResult &r)>;

    ProofQueue(size_t input_len, uint64_t capacity) : input_len_(input_len), capacity_(capacity) {}

    // Copies n inputs and gives them the tickets *first_ticket ...; all or nothing.  Waits up to timeout_ms (0: no wait, < 0: for
    // ever) for room: submitted jobs not yet collected never exceed the capacity.
    int submit(const int64_t *inputs, uint64_t n, int64_t timeout_ms, uint64_t *first_ticket, std::string &err) {
        if (!inputs || !first_ticket) return fail(err, DP_ERR_INVALID, "dph_zkml_stream_submit: null argument");
        if (n == 0) return fail(err, DP_ERR_INVALID, "dph_zkml_stream_submit: no inputs");
        if (n > capacity_) return fail(err, DP_ERR_INVALID, "dph_zkml_stream_submit: more inputs than the stream's capacity");
        std::deque<Pending> jobs;
        for (uint64_t j = 0; j < n; j++) jobs.push_back(Pending{0, std::vector<int64_t>(inputs + j * input_len_, inputs + (j + 1) * input_len_)});
        std::unique_lock<std::mutex> lk(mu_);
        if (closed_) return fail(err, DP_ERR_STATE, "dph_zkml_stream_submit: the stream is closed");
        callers_++;
        const bool room = wait(lk, space_cv_, timeout_ms, [&] { return closed_ || outstanding() + n <= capacity_; });
        if (leave()) return fail(err, DP_ERR_STATE, "dph_zkml_stream_submit: the stream was closed");
        if (!room) return fail(err, DP_ERR_TIMEOUT, "dph_zkml_stream_submit: no room in the stream before the timeout");
        *first_ticket = next_ticket_;
        for (auto &p : jobs) { p.ticket = next_ticket_++; queued_.push_back(std::move(p)); }
        if (n == 1) work_cv_.notify_one(); else work_cv_.notify_all();
        return DP_OK;
    }

    // One finished job, in completion order, moved to the caller (so each result goes to exactly one caller).  DP_ERR_STATE at once
    // when nothing is queued, running or waiting to be collected; DP_ERR_TIMEOUT after timeout_ms (0: no wait, < 0: for ever).
    int next(int64_t timeout_ms, QueueResult &r, std::string &err) {
        std::unique_lock<std::mutex> lk(mu_);
        if (closed_) return fail(err, DP_ERR_STATE, "dph_zkml_stream_next: the stream is closed");
        callers_++;
        const bool ready = wait(lk, done_cv_, timeout_ms, [&] { return closed_ || !done_.empty() || (queued_.empty() && running_ == 0); });
        if (leave()) return fail(err, DP_ERR_STATE, "dph_zkml_stream_next: the stream was closed");
        if (!done_.empty()) {
            r = std::move(done_.front()); done_.pop_front();
            space_cv_.notify_all();
            return DP_OK;
        }
        if (!ready) return fail(err, DP_ERR_TIMEOUT, "dph_zkml_stream_next: no job finished before the timeout");
        return fail(err, DP_ERR_STATE, "dph_zkml_stream_next: nothing submitted is left to collect");
    }

    // Runs jobs on the calling thread until the queue is closed; any number of threads may serve one queue.
    void serve(const Job &job) {
        for (;;) {
            Pending p; uint64_t backlog;
            {
                std::unique_lock<std::mutex> lk(mu_);
                work_cv_.wait(lk, [&] { return closed_ || !queued_.empty(); });
                if (queued_.empty()) return;
                backlog = queued_.size();
                p = std::move(queued_.front()); queued_.pop_front();
                running_++;
            }
            QueueResult r; r.ticket = p.ticket;
            try { job(p.input.data(), backlog, r); }
            catch (const std::exception &e) { if (!r.status) r.status = 1; r.error = e.what(); }
            if (r.status) { r.proof.clear(); r.output.clear(); }
            std::lock_guard<std::mutex> lk(mu_);
            running_--;
            done_.push_back(std::move(r));
            done_cv_.notify_all();
        }
    }

    // Cancels the queued jobs (returns their count), wakes every waiting submit and next (they return DP_ERR_STATE), waits for the
    // running jobs and for those callers to leave, and drops the uncollected results.  The serving threads then return.
    uint64_t close() {
        std::unique_lock<std::mutex> lk(mu_);
        closed_ = true;
        const uint64_t cancelled = queued_.size();
        queued_.clear();
        work_cv_.notify_all(); space_cv_.notify_all(); done_cv_.notify_all();
        done_cv_.wait(lk, [&] { return running_ == 0 && callers_ == 0; });
        done_.clear();
        return cancelled;
    }

private:
    struct Pending { uint64_t ticket; std::vector<int64_t> input; };
    static int fail(std::string &err, int code, const char *msg) { err = msg; return code; }
    uint64_t outstanding() const { return queued_.size() + running_ + done_.size(); }
    template <class Pred>
    static bool wait(std::unique_lock<std::mutex> &lk, std::condition_variable &cv, int64_t timeout_ms, Pred pred) {
        if (timeout_ms < 0) { cv.wait(lk, pred); return true; }
        return cv.wait_for(lk, std::chrono::milliseconds(timeout_ms), pred);
    }
    // a waiting submit or next leaves: true when the queue was closed meanwhile (close waits for every such caller to leave)
    bool leave() { callers_--; if (closed_) done_cv_.notify_all(); return closed_; }

    const size_t input_len_;
    const uint64_t capacity_;
    std::mutex mu_;
    std::condition_variable work_cv_, space_cv_, done_cv_;
    std::deque<Pending> queued_;
    std::deque<QueueResult> done_;
    uint64_t running_ = 0, next_ticket_ = 0;
    uint32_t callers_ = 0;
    bool closed_ = false;
};

}  // namespace dp
