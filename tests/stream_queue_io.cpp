// TEST INFRASTRUCTURE ONLY.  The proof stream's queue (deep-prove_b200/host/proof_queue.hpp) served by host threads that run a fake
// job instead of a proof, so its tickets, capacity, timed waits, cancellation and concurrent delivery are tested without a device.
// Built next to this file as libdp_stream_queue_io.so; driven by tests/test_prove_stream_abi.py.
//
// The fake job on input x (input_len >= 2 elements): sleeps x[1] milliseconds, then fails with DP_ERR_INVALID when x[0] < 0, else
// returns the proof {x[0], backlog} and the output 2 * x.
#include "../deep-prove_b200/host/proof_queue.hpp"
#include <atomic>
#include <cstring>
#include <thread>

namespace {
thread_local std::string g_err;
struct FakeStream {
    dp::ProofQueue q;
    std::vector<std::thread> servers;
    std::atomic<uint64_t> started{0};
    FakeStream(uint64_t input_len, uint64_t capacity) : q(input_len, capacity) {}
};
}

extern "C" {

const char *dpq_last_error() { return g_err.c_str(); }

void *dpq_open(uint64_t input_len, uint64_t capacity, uint32_t n_servers) {
    auto *s = new FakeStream(input_len, capacity);
    for (uint32_t i = 0; i < n_servers; i++)
        s->servers.emplace_back([s, input_len] {
            s->q.serve([s, input_len](const int64_t *x, uint64_t backlog, dp::QueueResult &r) {
                s->started++;
                std::this_thread::sleep_for(std::chrono::milliseconds(x[1]));
                if (x[0] < 0) { r.status = DP_ERR_INVALID; r.error = "fake job: negative input"; return; }
                r.proof = {(uint64_t)x[0], backlog};
                for (uint64_t i = 0; i < input_len; i++) r.output.push_back(2 * x[i]);
            });
        });
    return s;
}

uint64_t dpq_started(void *s) { return ((FakeStream *)s)->started.load(); }

int dpq_submit(void *s, const int64_t *inputs, uint64_t n, int64_t timeout_ms, uint64_t *first_ticket) {
    return ((FakeStream *)s)->q.submit(inputs, n, timeout_ms, first_ticket, g_err);
}

// proof: 2 words; output: input_len elements; msg: msg_cap bytes, NUL-terminated
int dpq_next(void *s, int64_t timeout_ms, uint64_t *ticket, uint64_t *proof, uint64_t *proof_len, int64_t *output, int32_t *status,
             char *msg, uint64_t msg_cap) {
    dp::QueueResult r;
    const int rc = ((FakeStream *)s)->q.next(timeout_ms, r, g_err);
    if (rc) return rc;
    *ticket = r.ticket; *status = r.status; *proof_len = r.proof.size();
    memcpy(proof, r.proof.data(), 8 * r.proof.size());
    memcpy(output, r.output.data(), 8 * r.output.size());
    snprintf(msg, msg_cap, "%s", r.error.c_str());
    return 0;
}

// closes the queue, joins its servers and frees the stream: *cancelled = the jobs no server had started
void dpq_close(void *s, uint64_t *cancelled) {
    FakeStream *fs = (FakeStream *)s;
    *cancelled = fs->q.close();
    for (auto &t : fs->servers) t.join();
    delete fs;
}

}  // extern "C"
