// C entry points over the host mirror (for the Python tests / bench; a Rust caller would use its own
// crates above include/deepprove_b200.h instead).  Nothing here touches oracle/.
#include "sumcheck.hpp"

using namespace dp;
static thread_local std::string g_herr;
#define DPH_TRY try {
#define DPH_CATCH } catch (const Error &e) { g_herr = e.what(); return e.code ? e.code : 1; } catch (const std::exception &e) { g_herr = e.what(); return 1; }

// A caller's device MLE as a DeviceMle (a view, no copy); with T > 1, its slice t of T (the t-th contiguous part)
static DeviceMle view(const dp_mle *m, uint32_t t = 0, uint32_t T = 1) {
    uint64_t len; int ext; check(dp_mle_info(m, &len, &ext, nullptr));
    const uint64_t sl = len / T;
    return DeviceMle::wrap_device((char *)dp_mle_device_ptr(m) + (size_t)t * sl * (ext ? 16 : 8), sl, ext != 0);
}
// n extension elements given as [c0, c1] word pairs (a point, claimed evaluations)
static ExtVec exts(const u64 *w, size_t n) {
    ExtVec v;
    for (size_t i = 0; i < n; i++) v.push_back(Ext(w[2 * i], w[2 * i + 1]));
    return v;
}
// The flat-output rule: *out_len = the words the output needs; a null `out` only asks for that length, a `cap` below it is refused.
template <class W>
static int put_flat(const char *entry, const std::vector<W> &words, W *out, uint64_t cap, uint64_t *out_len) {
    *out_len = words.size();
    if (!out) return 0;
    if (words.size() > cap) throw Error(DP_ERR_INVALID, std::string(entry) + ": output buffer too small");
    memcpy(out, words.data(), sizeof(W) * words.size());
    return 0;
}

extern "C" {

const char *dph_last_error() { return g_herr.c_str(); }

void dph_poseidon2_permute(uint64_t *state) { Poseidon2::permute(state); }
// fast (weak-form) permutation against the canonical formulation on n seeded states, every third one drawn from edge values;
// returns the number of mismatching or non-canonical output words (0 expected)
uint64_t dph_poseidon2_selfcheck(uint64_t n, uint64_t seed) {
    auto sm = [&]() { uint64_t z = (seed += 0x9E3779B97F4A7C15ULL); z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL; z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL; return z ^ (z >> 31); };
    const uint64_t edge[] = {0, 1, 2, P - 1, P - 2, EPS, EPS + 1, 1ULL << 32, 1ULL << 63, (P - 1) / 2, 0xFFFFFFFEFFFFFFFFULL, 7};
    const int ne = sizeof(edge) / 8; uint64_t bad = 0, a[8], b[8], ca[8] = {0}, cb[8] = {0};
    for (uint64_t it = 0; it < n; it++) {
        for (int i = 0; i < 8; i++) a[i] = b[i] = (it % 3 == 0) ? edge[sm() % ne] : canon(sm());
        Poseidon2::permute(a); Poseidon2::permute_canonical(b);
        for (int i = 0; i < 8; i++) if (a[i] != b[i] || a[i] >= P) bad++;
        ca[it & 3] = cb[it & 3] = canon(sm());                       // and a chained (sponge-like) sequence
        Poseidon2::permute(ca); Poseidon2::permute_canonical(cb);
        for (int i = 0; i < 8; i++) if (ca[i] != cb[i]) bad++;
    }
    return bad;
}

// Hasher pair of everything proved from now on: 0 = PoseidonHasher + BasicTranscript (default), 1 = BlakeHasher + BlakeTranscript
// (the reference's cargo feature `blake`: mpcs/src/lib.rs:339-342, zkml/src/bin/bench.rs:29-44).  Process-wide; set it between proofs.
int dph_set_hasher(int kind) { if (kind != 0 && kind != 1) { g_herr = "dph_set_hasher: 0 or 1"; return 1; } if (dp_set_merkle_hasher(kind) != DP_OK) { g_herr = dp_last_error(); return 1; } dp::hasher_mode() = kind; return 0; }
void *dph_transcript_new(const char *label) { return new DynTranscript(label); }
void dph_transcript_free(void *t) { delete (DynTranscript *)t; }
void dph_transcript_append_f(void *t, const uint64_t *f, uint64_t n) { for (uint64_t i = 0; i < n; i++) ((DynTranscript *)t)->append_field_element(f[i]); }
void dph_transcript_append_msg(void *t, const uint8_t *m, uint64_t n) { ((DynTranscript *)t)->append_message(m, n); }
void dph_transcript_append_e(void *t, const uint64_t *e, uint64_t n) { for (uint64_t i = 0; i < n; i++) ((DynTranscript *)t)->append_field_element_ext(Ext(e[2 * i], e[2 * i + 1])); }
void dph_transcript_challenge(void *t, const char *label, uint64_t *out) { Ext c = ((DynTranscript *)t)->get_and_append_challenge(label); out[0] = c.c0; out[1] = c.c1; }
// The transcript's device state (what a prover hands to dp_sc_run_tail_fs[_blake] / dp_logup_run_layers_fs[_blake]): *kind = 0 none,
// 1 the 14-word Poseidon2 sponge, 2 the DP_B3T_WORDS BLAKE3 hasher image; words: DP_B3T_WORDS.  Load takes the same kind back (1 on
// a mismatch or an invalid image).
void dph_transcript_save_state(void *t, int *kind, uint64_t *words) { *kind = ((DynTranscript *)t)->save_sponge(words); }
int dph_transcript_load_state(void *t, int kind, const uint64_t *words) {
    DPH_TRY
    if (kind != ((DynTranscript *)t)->state_kind()) throw Error(DP_ERR_INVALID, "dph_transcript_load_state: not this transcript's kind of state");
    ((DynTranscript *)t)->load_sponge(words);
    return 0;
    DPH_CATCH
}

// VirtualPolynomial numbers MLEs by FIRST USE in the products (virtual_poly.rs:168-177), and get_mle_final_evaluations()
// returns them in that order; the C entry points below report final evaluations in the CALLER's `mles` order instead.
// remap[i] = position of caller MLE i in first-use order, UINT32_MAX when no product references it (its slot is zeroed).
static std::vector<uint32_t> first_use_remap(const dp_sc_product *products, uint32_t n_products, uint32_t n_mles) {
    std::vector<uint32_t> remap(n_mles, UINT32_MAX); uint32_t next = 0;
    for (uint32_t p = 0; p < n_products; p++) for (uint32_t j = 0; j < products[p].n_idx; j++) { uint32_t i = products[p].idx[j]; if (i < n_mles && remap[i] == UINT32_MAX) remap[i] = next++; }
    return remap;
}
// The caller's products over views of its device MLEs (no copies); with T > 1, over slice t of T (the t-th contiguous part of every MLE)
static VirtualPolynomial make_poly(dp_mle *const *mles, uint32_t n_mles, const dp_sc_product *products, uint32_t n_products, size_t max_nv,
                                   uint32_t t = 0, uint32_t T = 1) {
    VirtualPolynomial vp(max_nv);
    std::vector<DeviceMle> views;
    for (uint32_t i = 0; i < n_mles; i++) views.push_back(view(mles[i], t, T));
    for (uint32_t p = 0; p < n_products; p++) {
        std::vector<DeviceMle> l;
        for (uint32_t j = 0; j < products[p].n_idx; j++) l.push_back(views.at(products[p].idx[j]));
        vp.add_mle_list(l, Ext(products[p].coef[0], products[p].coef[1]));
    }
    return vp;
}
// out_point: nv x E; out_msgs: nv x (max_deg+1) x E; out_final: n_mles x E in the caller's `mles` order
static void write_proof(const std::pair<IOPProof, IOPProverState> &res, const dp_sc_product *products, uint32_t n_products, uint32_t n_mles,
                        uint64_t *out_point, uint64_t *out_msgs, uint64_t *out_final) {
    for (size_t i = 0; i < res.first.point.size(); i++) { out_point[2 * i] = res.first.point[i].c0; out_point[2 * i + 1] = res.first.point[i].c1; }
    size_t k = 0;
    for (auto &m : res.first.proofs) for (auto &e : m.evaluations) { out_msgs[2 * k] = e.c0; out_msgs[2 * k + 1] = e.c1; k++; }
    const ExtVec &fin = res.second.get_mle_final_evaluations();
    const std::vector<uint32_t> remap = first_use_remap(products, n_products, n_mles);
    for (size_t i = 0; i < remap.size(); i++) {
        Ext v = (remap[i] != UINT32_MAX && remap[i] < fin.size()) ? fin[remap[i]] : Ext::zero();
        out_final[2 * i] = v.c0; out_final[2 * i + 1] = v.c1;
    }
}

// IOPProverState::prove_parallel over device MLE handles with DynTranscript::new(label) (or an
// existing transcript when `transcript` is non-null).  out_msgs: nv x (max_deg+1) x E.
int dph_sumcheck_prove_parallel(dp_mle *const *mles, uint32_t n_mles, const dp_sc_product *products, uint32_t n_products,
                                uint32_t max_nv, const char *label, void *transcript, uint64_t *out_point, uint64_t *out_msgs,
                                uint64_t *out_final, uint32_t *out_max_deg) {
    DPH_TRY
    VirtualPolynomial vp = make_poly(mles, n_mles, products, n_products, max_nv);
    DynTranscript local(label ? label : "");
    DynTranscript &t = transcript ? *(DynTranscript *)transcript : local;
    auto res = IOPProverState::prove_parallel(std::move(vp), t);
    size_t deg = res.first.proofs.empty() ? 0 : res.first.proofs[0].evaluations.size() - 1;
    *out_max_deg = (uint32_t)deg;
    write_proof(res, products, n_products, n_mles, out_point, out_msgs, out_final);
    return 0;
    DPH_CATCH
}

}  // extern "C"

// ---- mpcs (host/mpcs.hpp) ----
#include "mpcs.hpp"
extern "C" {

// Basefold::commit + Basefold::open with BasefoldProof flattened (BasefoldProof::flatten layout)
int dph_pcs_open(dp_mle *poly, uint32_t full_log, const uint64_t *point, const char *label, uint64_t *out, uint64_t cap, uint64_t *out_len, uint64_t *out_root) {
    DPH_TRY
    DeviceMle m = view(poly);
    BasefoldProverParams pp; pp.full_message_size_log = full_log;
    auto comm = Basefold::commit(pp, m);
    if (out_root) memcpy(out_root, comm.root.v, 32);
    DynTranscript t(label);
    BasefoldProof pr = Basefold::open(pp, m, comm, exts(point, m.num_vars()), t);
    return put_flat("dph_pcs_open", pr.flatten(), out, cap, out_len);
    DPH_CATCH
}

}  // extern "C"

// ---- zkml MLP prover (host/zkml.hpp) ----
#include "zkml.hpp"
#include <chrono>
namespace {
struct ZkHandle {   // the stored trace lives in HBM; the batch-inference plan is built by the first dph_zkml_infer_batch
    dp::zkml::Model model; dp::zkml::Context ctx; dp::zkml::DeviceTrace trace; std::vector<dp::zkml::Element> trace_input;
    std::unique_ptr<dp::zkml::InferPlan> plan;
};
}
extern "C" {

extern "C" void dph_zkml_pool_free(void *handle);
void dph_zkml_context_free(void *h) { dph_zkml_pool_free(h); delete (ZkHandle *)h; }

// mode 0: inference + Prover::prove + flatten (end to end from the host input buffer)
// mode 1: run inference only and keep the trace in the handle (not proving)
// mode 2: Prover::prove on the stored trace (what zkml/src/bin/bench.rs times), flatten only if out != NULL
int dph_zkml_prove(void *handle, const int64_t *input, int mode, const char *label, uint64_t *out, uint64_t cap, uint64_t *out_len) {
    DPH_TRY
    using namespace dp::zkml;
    ZkHandle *h = (ZkHandle *)handle;
    size_t w = h->model.input_len;
    if (mode == 0 || mode == 1) { h->trace_input.assign(input, input + w); h->trace = run_device(h->ctx, h->trace_input); check(dp_synchronize()); if (mode == 1) return 0; }
    DynTranscript t(label);
    Prover<DynTranscript> prover(h->ctx, t);
    Proof p = prover.prove(h->trace);
    return out ? put_flat("dph_zkml_prove", p.flatten(h->model.nodes.size()), out, cap, out_len) : 0;
    DPH_CATCH
}

// The number of elements in the model's output: the last node's output tensor in the padded layout
int dph_zkml_output_len(void *handle, uint64_t *len) {
    DPH_TRY
    if (!handle || !len) throw Error(DP_ERR_INVALID, "dph_zkml_output_len: null argument");
    *len = ((ZkHandle *)handle)->model.output_len();
    return 0;
    DPH_CATCH
}

// The model output of the stored trace (dph_zkml_prove mode 0 or 1) as signed elements, by the flat-output rule
int dph_zkml_trace_output(void *handle, int64_t *out, uint64_t cap, uint64_t *out_len) {
    DPH_TRY
    if (!handle || !out_len) throw Error(DP_ERR_INVALID, "dph_zkml_trace_output: null argument");
    ZkHandle *h = (ZkHandle *)handle;
    if (!h->trace.valid()) throw Error(DP_ERR_STATE, "dph_zkml_trace_output: no stored trace (run dph_zkml_prove mode 0 or 1 first)");
    return put_flat("dph_zkml_trace_output", dp::zkml::to_elements(h->trace.outs.back()), out, cap, out_len);
    DPH_CATCH
}

}  // extern "C"

// ---- concurrent proving: a persistent pool of host threads, each with its own library context (stream + device
// arena) on `device`, proves the stored trace, the stored input or a batch of caller inputs; the GPU runs the threads' small
// latency-bound kernels side by side.  One call at a time per pool: a call on a busy pool is refused.
#include <thread>
#include <mutex>
#include <atomic>
#include <condition_variable>
#include "proof_queue.hpp"
namespace {
// Input x of the handle's model end to end, as one job of a batch or of a stream: inference, Prover::prove, the flat proof and the
// model output in host memory
void prove_input(ZkHandle *h, dp::zkml::Prover<dp::DynTranscript> &prover, const int64_t *x, std::vector<uint64_t> &flat,
                 std::vector<dp::zkml::Element> &y) {
    const size_t w = h->model.input_len;
    dp::zkml::DeviceTrace tr = dp::zkml::run_device(h->ctx, std::vector<dp::zkml::Element>(x, x + w));
    flat = prover.prove(tr).flatten(h->model.nodes.size());
    y = dp::zkml::to_elements(tr.outs.back());
    if (y.size() != h->model.output_len()) throw dp::Error(DP_ERR_STATE, "zkml prover: model output of unexpected length");
}
struct ZkStream;
struct ZkPool {
    std::vector<std::thread> th; std::mutex mu; std::condition_variable cv, done_cv;
    ZkHandle *h = nullptr; int device = 0; bool stop = false, busy = false; uint64_t pending = 0, inflight = 0; std::string label, err; bool failed = false; bool e2e = false;
    uint64_t *out = nullptr, out_cap = 0, *out_len = nullptr;   // when set: the flat proof of the call's last job is copied here
    // when set: every job's flat proof goes to all_out + job * all_stride, its length to all_lens[job], its worker to all_worker[job]
    uint64_t *all_out = nullptr, all_stride = 0, *all_lens = nullptr; uint32_t *all_worker = nullptr; uint64_t next_job = 0;
    // when set (dph_zkml_prove_batch): job j proves the caller's input j, in + j * input_len, end to end; its model output goes to
    // outputs + j * output_len.  A failing job does not fail the call: it gets status[j] != 0, proof length 0 and job_err[j].
    const int64_t *in = nullptr; int64_t *outputs = nullptr; int32_t *status = nullptr; std::vector<std::string> job_err;
    // Identical proofs started together stay in lockstep: all of them sit in the latency-bound layer sumchecks (GPU nearly idle)
    // and then all of them queue their GPU-filling opening kernels behind each other (CUPTI timeline).  So the
    // workers of one call start `stagger_s` apart (one proof duration spread over the workers; the duration is an average over the
    // proofs this pool has already run -- the first call of a pool is not staggered): latency-bound and GPU-bound phases of
    // different proofs then overlap.  The ramp-up and ramp-down this costs are inside the caller's timed region.
    uint32_t active = 0; uint64_t call_gen = 0; double stagger_s = 0.0, avg_proof_s = 0.0; uint64_t n_timed = 0;
    // The open stream (dph_zkml_stream_open), which the first `active` threads serve until it closes; stream_gen counts streams,
    // so each thread joins each stream once
    ZkStream *stream = nullptr; bool stream_closing = false; uint64_t stream_gen = 0;
    void serve_stream(uint32_t idx, ZkStream &s, bool &inited);
    void time_proof(double sec) { std::lock_guard<std::mutex> lk(mu); n_timed++; avg_proof_s += (sec - avg_proof_s) / (double)std::min<uint64_t>(n_timed, 64); }
    void worker(uint32_t idx) {
        bool inited = false; uint64_t seen_gen = 0, seen_stream = 0;
        for (;;) {
            uint64_t gen, job; double delay = 0.0; bool keep = false, all = false, batch = false; ZkStream *joined = nullptr;
            { std::unique_lock<std::mutex> lk(mu);
              cv.wait(lk, [&] { return stop || (pending > 0 && idx < active) || (stream && !stream_closing && idx < active && stream_gen != seen_stream); });
              if (stop) break;
              if (pending == 0) { joined = stream; seen_stream = stream_gen; inflight++; }
              else { pending--; inflight++; keep = pending == 0 && out; all = all_out != nullptr; batch = in != nullptr; job = next_job++; gen = call_gen; if (gen != seen_gen) { seen_gen = gen; delay = stagger_s * idx; } } }
            if (joined) {
                serve_stream(idx, *joined, inited);
                std::lock_guard<std::mutex> lk(mu); inflight--; if (inflight == 0) done_cv.notify_all();
                continue;
            }
            try {
                const bool first_ever = !inited;     // grows this thread's device arena: not a representative duration
                if (!inited) { dp::check(dp_init(device)); inited = true; }
                if (delay > 0.0) std::this_thread::sleep_for(std::chrono::duration<double>(delay));
                auto t0 = std::chrono::steady_clock::now();
                dp::DynTranscript t(label);
                dp::zkml::Prover<dp::DynTranscript> prover(h->ctx, t);
                std::vector<uint64_t> flat;
                if (batch) {   // the caller's input `job`: inference, prove, serialised proof and model output in host memory
                    const size_t ol = h->model.output_len();
                    std::vector<dp::zkml::Element> y;
                    prove_input(h, prover, in + job * h->model.input_len, flat, y);
                    if (flat.size() > all_stride) { std::lock_guard<std::mutex> lk(mu); failed = true; err = "dph_zkml_prove_batch: proof longer than the stride"; throw dp::Error(DP_ERR_INVALID, err); }
                    memcpy(outputs + job * ol, y.data(), 8 * ol);
                } else if (e2e) {   // from the host input vector: inference, prove, serialised proof in host memory
                    dp::zkml::Proof p = prover.prove(h->trace_input);
                    flat = p.flatten(h->model.nodes.size());
                    if (flat.empty()) throw dp::Error(DP_ERR_STATE, "empty proof");
                } else { dp::zkml::Proof p = prover.prove(h->trace); if (keep || all) flat = p.flatten(h->model.nodes.size()); }
                if (keep) {
                    std::lock_guard<std::mutex> lk(mu);
                    if (flat.size() > out_cap) throw dp::Error(DP_ERR_INVALID, "dph_zkml_prove_concurrent: output buffer too small");
                    memcpy(out, flat.data(), 8 * flat.size()); *out_len = flat.size();
                }
                if (all) {   // each job owns its slot: no lock
                    all_lens[job] = flat.size(); if (all_worker) all_worker[job] = idx;
                    if (flat.size() > all_stride) throw dp::Error(DP_ERR_INVALID, "dph_zkml_prove_concurrent_all: proof longer than the stride");
                    memcpy(all_out + job * all_stride, flat.data(), 8 * flat.size());
                }
                const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
                if (!first_ever) time_proof(sec);
            } catch (const std::exception &e) {
                std::lock_guard<std::mutex> lk(mu);
                if (batch) {   // this job's failure only
                    const dp::Error *de = dynamic_cast<const dp::Error *>(&e);
                    status[job] = de && de->code ? de->code : 1; all_lens[job] = 0; job_err[job] = e.what();
                } else { failed = true; err = e.what(); }
            }
            dp_profile_flush();   // per-kernel timing of the concurrent region (no-op unless dp_profile_enable(1))
            { std::lock_guard<std::mutex> lk(mu); inflight--; if (pending == 0 && inflight == 0) done_cv.notify_all(); }
        }
        if (inited) { dp_synchronize(); dp_shutdown(); }
    }
    ~ZkPool() { { std::lock_guard<std::mutex> lk(mu); stop = true; } cv.notify_all(); for (auto &t : th) t.join(); }
};
struct ZkStream {
    ZkPool *pool; uint32_t n_workers; uint64_t stride; std::string label; dp::ProofQueue q;
    ZkStream(ZkPool *p, uint32_t nw, uint64_t st, const char *lb, uint64_t capacity)
        : pool(p), n_workers(nw), stride(st), label(lb), q(p->h->model.input_len, capacity) {}
};
// One worker thread serving the stream: each job is one dph_zkml_prove_batch job (prove_input), except that a proof longer than the
// stride fails that job alone.  Stagger rule: a thread delays only its first job of the stream, by the batch rule's stagger_s * idx,
// and only when that job was taken from a backlog of at least 3 jobs per worker (the batch rule's bound); so a lone job on an idle
// stream starts at once, and a large submit spreads the workers' phases as a large batch does.
void ZkPool::serve_stream(uint32_t idx, ZkStream &s, bool &inited) {
    bool first = true;
    s.q.serve([&](const int64_t *x, uint64_t backlog, dp::QueueResult &r) {
        try {
            const bool first_ever = !inited;
            if (!inited) { dp::check(dp_init(device)); inited = true; }
            double delay = 0.0;
            if (first && s.n_workers > 1 && backlog >= 3ull * s.n_workers) { std::lock_guard<std::mutex> lk(mu); if (n_timed > 0) delay = avg_proof_s / s.n_workers * idx; }
            first = false;
            if (delay > 0.0) std::this_thread::sleep_for(std::chrono::duration<double>(delay));
            auto t0 = std::chrono::steady_clock::now();
            dp::DynTranscript t(s.label);
            dp::zkml::Prover<dp::DynTranscript> prover(h->ctx, t);
            prove_input(h, prover, x, r.proof, r.output);
            if (r.proof.size() > s.stride) throw dp::Error(DP_ERR_INVALID, "dph_zkml_stream_next: proof longer than the stream's stride");
            if (!first_ever) time_proof(std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count());
        } catch (const std::exception &e) {
            const dp::Error *de = dynamic_cast<const dp::Error *>(&e);
            r.status = de && de->code ? de->code : 1; r.error = e.what();
        }
        dp_profile_flush();
    });
}
// Closes a stream: cancels its queued jobs (returns their count), waits for the running ones and for the threads to leave it, and
// releases the pool
uint64_t close_stream(ZkStream *s) {
    ZkPool *p = s->pool;
    { std::lock_guard<std::mutex> lk(p->mu); p->stream_closing = true; }
    const uint64_t cancelled = s->q.close();
    { std::unique_lock<std::mutex> lk(p->mu); p->done_cv.wait(lk, [&] { return p->inflight == 0; }); p->stream = nullptr; p->stream_closing = false; p->busy = false; }
    delete s;
    return cancelled;
}
std::mutex g_pools_mu; std::map<void *, std::unique_ptr<ZkPool>> g_pools;
}
// Frees the handle's pool, closing its open stream first
extern "C" void dph_zkml_pool_free(void *handle) {
    std::unique_ptr<ZkPool> p;
    { std::lock_guard<std::mutex> lk(g_pools_mu); auto it = g_pools.find(handle); if (it == g_pools.end()) return; p = std::move(it->second); g_pools.erase(it); }
    ZkStream *s; { std::lock_guard<std::mutex> lk(p->mu); s = p->stream_closing ? nullptr : p->stream; }
    if (s) close_stream(s);
}
namespace {
// The handle's pool (made on first use, without threads), marked busy for the caller; refused when another call holds it
ZkPool *acquire_pool(void *handle) {
    ZkPool *pool;
    { std::lock_guard<std::mutex> lk(g_pools_mu); auto &pp = g_pools[handle]; if (!pp) { pp = std::make_unique<ZkPool>(); pp->h = (ZkHandle *)handle; } pool = pp.get(); }
    std::lock_guard<std::mutex> lk(pool->mu);
    if (pool->busy) throw dp::Error(DP_ERR_STATE, "the handle's worker pool is busy with another call");
    pool->busy = true;
    return pool;
}
struct AllOut { uint64_t *out; uint64_t stride; uint64_t *lens; uint32_t *worker; };
struct BatchIo { const int64_t *in; int64_t *outputs; int32_t *status; };
int prove_concurrent(void *handle, int device, uint32_t n_workers, uint32_t n_proofs, int e2e, const char *label, double *out_seconds,
                     uint64_t *out, uint64_t cap, uint64_t *out_len, const AllOut &all, const BatchIo &batch) {
    DPH_TRY
    ZkHandle *h = (ZkHandle *)handle;
    if (!batch.in && !h->trace.valid()) throw dp::Error(DP_ERR_STATE, "dph_zkml_prove_concurrent: run inference first (mode 1)");
    ZkPool *pool;
    pool = acquire_pool(handle);
    { std::lock_guard<std::mutex> lk(pool->mu); if (pool->th.empty()) pool->device = device; }
    while (pool->th.size() < n_workers) { const uint32_t idx = (uint32_t)pool->th.size(); pool->th.emplace_back([pool, idx] { pool->worker(idx); }); }
    auto t0 = std::chrono::steady_clock::now();
    {
        std::lock_guard<std::mutex> lk(pool->mu);
        pool->label = label; pool->failed = false; pool->e2e = e2e != 0; pool->pending = n_proofs; pool->active = n_workers; pool->call_gen++;
        pool->out = out; pool->out_cap = cap; pool->out_len = out_len; if (out_len) *out_len = 0;
        pool->all_out = all.out; pool->all_stride = all.stride; pool->all_lens = all.lens; pool->all_worker = all.worker; pool->next_job = 0;
        pool->in = batch.in; pool->outputs = batch.outputs; pool->status = batch.status;
        if (batch.in) pool->job_err.assign(n_proofs, std::string());
        // stagger only when every worker gets several proofs (otherwise the ramps cost more than the overlap gains)
        pool->stagger_s = (n_workers > 1 && n_proofs >= 3 * n_workers && pool->n_timed > 0) ? pool->avg_proof_s / n_workers : 0.0;
    }
    // only the first n_workers threads are woken usefully: notify_all, extra threads just compete for the same jobs
    pool->cv.notify_all();
    bool failed;
    { std::unique_lock<std::mutex> lk(pool->mu); pool->done_cv.wait(lk, [&] { return pool->pending == 0 && pool->inflight == 0; }); failed = pool->failed; if (failed) g_herr = pool->err; pool->busy = false; }
    if (out_seconds) *out_seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    return failed ? 1 : 0;
    DPH_CATCH
}
}
// out (optional, cap words): receives the flat proof of the last job handed out, *out_len its length in words.
extern "C" int dph_zkml_prove_concurrent(void *handle, int device, uint32_t n_workers, uint32_t n_proofs, int e2e, const char *label, double *out_seconds,
                                         uint64_t *out, uint64_t cap, uint64_t *out_len) {
    return prove_concurrent(handle, device, n_workers, n_proofs, e2e, label, out_seconds, out, cap, out_len, AllOut{nullptr, 0, nullptr, nullptr}, BatchIo{nullptr, nullptr, nullptr});
}
// The same call, but every job's flat proof is kept: job j's proof is written to out + j * stride (n_proofs x stride words),
// its length in words to out_lens[j] and, when out_worker is given, the index of the worker thread that proved it to out_worker[j].
// Jobs are numbered in the order workers take them.  Flattening every proof costs host time that dph_zkml_prove_concurrent does
// not spend on the stored-trace path.
extern "C" int dph_zkml_prove_concurrent_all(void *handle, int device, uint32_t n_workers, uint32_t n_proofs, int e2e, const char *label, double *out_seconds,
                                             uint64_t *out, uint64_t stride, uint64_t *out_lens, uint32_t *out_worker) {
    if (!out || !out_lens) { g_herr = "dph_zkml_prove_concurrent_all: out and out_lens are required"; return 1; }
    for (uint32_t j = 0; j < n_proofs; j++) out_lens[j] = 0;
    return prove_concurrent(handle, device, n_workers, n_proofs, e2e, label, out_seconds, nullptr, 0, nullptr, AllOut{out, stride, out_lens, out_worker},
                            BatchIo{nullptr, nullptr, nullptr});
}
// n distinct inputs (inputs: n x input_len), each proved end to end on the handle's worker pool (n_workers threads on `device`):
// input j's flat proof goes to proofs + j * stride, its length in words to proof_lens[j], its model output (output_len elements,
// dph_zkml_output_len) to outputs + j * output_len and its status to status[j].  Slots are indexed by input.  An input that fails
// (a value outside its lookup table, say) fails alone: status[j] != 0, proof_lens[j] = 0, and dph_zkml_job_error(handle, j) holds
// its message until the next batch or infer call on the handle.  Non-zero only for call-level errors: an argument refused, no device, a
// busy pool (DP_ERR_STATE), or a proof longer than `stride` (DP_ERR_INVALID, after the batch).  The stored trace is not touched.
extern "C" int dph_zkml_prove_batch(void *handle, int device, uint32_t n_workers, const int64_t *inputs, uint32_t n, const char *label,
                                    uint64_t *proofs, uint64_t stride, uint64_t *proof_lens, int64_t *outputs, int32_t *status, double *out_seconds) {
    DPH_TRY
    if (n == 0 || n_workers == 0) throw Error(DP_ERR_INVALID, "dph_zkml_prove_batch: no inputs or no workers");
    if (!inputs || !label || !proofs || !proof_lens || !outputs || !status) throw Error(DP_ERR_INVALID, "dph_zkml_prove_batch: null argument");
    const int n_dev = dp_device_count();
    if (n_dev <= 0) throw Error(DP_ERR_NO_DEVICE, "dph_zkml_prove_batch: no CUDA device visible (no CPU fallback)");
    if (device < 0 || device >= n_dev) throw Error(DP_ERR_INVALID, "dph_zkml_prove_batch: device index out of range");
    if (!handle) throw Error(DP_ERR_INVALID, "dph_zkml_prove_batch: null handle");
    for (uint32_t j = 0; j < n; j++) { proof_lens[j] = 0; status[j] = 0; }
    return prove_concurrent(handle, device, n_workers, n, 0, label, out_seconds, nullptr, 0, nullptr, AllOut{proofs, stride, proof_lens, nullptr},
                            BatchIo{inputs, outputs, status});
    DPH_CATCH
}
// n inputs (inputs: n x input_len) through the model without proving (csrc/infer.cu): input j's model output goes to outputs + j *
// output_len (dph_zkml_output_len), in the same padded layout and with the same values as the stored trace's, and its status to
// status[j].  The calling thread's device context runs it; the plan is built on the first call and kept until the context is freed.
// An input fails alone with the status and message dph_zkml_prove_batch gives it (dph_zkml_job_error(handle, j), until the next
// batch or infer call on the handle), and so does an input with a value outside [-128, 127]: the batch inference takes 8-bit inputs.
// Non-zero for call-level errors: an argument refused, no device, a busy pool (DP_ERR_STATE), a model the plan refuses
// (DP_ERR_INVALID, naming the node).  *out_seconds (optional): the inference's wall time, plan building excluded.  The stored trace
// is not touched.
extern "C" int dph_zkml_infer_batch(void *handle, const int64_t *inputs, uint32_t n, int64_t *outputs, int32_t *status, double *out_seconds) {
    DPH_TRY
    if (n == 0) throw Error(DP_ERR_INVALID, "dph_zkml_infer_batch: no inputs");
    if (!inputs || !outputs || !status) throw Error(DP_ERR_INVALID, "dph_zkml_infer_batch: null argument");
    if (dp_device_count() <= 0) throw Error(DP_ERR_NO_DEVICE, "dph_zkml_infer_batch: no CUDA device visible (no CPU fallback)");
    if (!handle) throw Error(DP_ERR_INVALID, "dph_zkml_infer_batch: null handle");
    ZkHandle *h = (ZkHandle *)handle;
    ZkPool *pool = acquire_pool(handle);
    struct Release { ZkPool *p; ~Release() { std::lock_guard<std::mutex> lk(p->mu); p->busy = false; } } release{pool};
    { std::lock_guard<std::mutex> lk(pool->mu); pool->job_err.assign(n, std::string()); }
    if (!h->plan) h->plan = std::make_unique<dp::zkml::InferPlan>(h->model);
    std::vector<uint32_t> bits(n);
    auto t0 = std::chrono::steady_clock::now();
    check(dp_infer_run(h->plan->get(), inputs, n, outputs, bits.data()));
    if (out_seconds) *out_seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    std::lock_guard<std::mutex> lk(pool->mu);
    for (uint32_t j = 0; j < n; j++) {
        status[j] = bits[j] ? DP_ERR_INVALID : 0;
        if (bits[j] & 16) pool->job_err[j] = "dph_zkml_infer_batch: an input value lies outside [-128, 127] (the batch inference takes 8-bit inputs)";
        else if (bits[j]) pool->job_err[j] = dp::zkml::lookup_error_message(bits[j]);
    }
    return 0;
    DPH_CATCH
}

// The message of job j of the handle's last batch or infer call, or NULL when job j succeeded (or there is no such job)
extern "C" const char *dph_zkml_job_error(void *handle, uint32_t j) {
    std::lock_guard<std::mutex> lk(g_pools_mu);
    auto it = g_pools.find(handle);
    if (it == g_pools.end()) return nullptr;
    std::lock_guard<std::mutex> pl(it->second->mu);
    const std::vector<std::string> &e = it->second->job_err;
    return j < e.size() && !e[j].empty() ? e[j].c_str() : nullptr;
}

// ---- proof stream: inputs submitted while proofs run, each result collected when its proof finishes (proof_queue.hpp) ----
// Opens a stream on the handle's worker pool (n_workers threads on `device`), which it holds until dph_zkml_stream_close: meanwhile
// dph_zkml_prove_batch, dph_zkml_prove_concurrent[_all] and dph_zkml_infer_batch on the handle are refused (DP_ERR_STATE), as for a
// busy pool.  Every job proves one input as dph_zkml_prove_batch does, under `label`.  `capacity` bounds the jobs submitted and not
// yet collected; `stride` is the longest proof a job may return.  Refused: a null argument, n_workers or capacity 0, no device
// (DP_ERR_NO_DEVICE), a device index out of range, a busy pool (DP_ERR_STATE).
extern "C" int dph_zkml_stream_open(void *handle, int device, uint32_t n_workers, const char *label, uint64_t stride, uint32_t capacity,
                                    void **stream) {
    DPH_TRY
    if (!label || !stream) throw Error(DP_ERR_INVALID, "dph_zkml_stream_open: null argument");
    if (n_workers == 0 || capacity == 0) throw Error(DP_ERR_INVALID, "dph_zkml_stream_open: no workers or no capacity");
    const int n_dev = dp_device_count();
    if (n_dev <= 0) throw Error(DP_ERR_NO_DEVICE, "dph_zkml_stream_open: no CUDA device visible (no CPU fallback)");
    if (device < 0 || device >= n_dev) throw Error(DP_ERR_INVALID, "dph_zkml_stream_open: device index out of range");
    if (!handle) throw Error(DP_ERR_INVALID, "dph_zkml_stream_open: null handle");
    ZkPool *pool = acquire_pool(handle);
    ZkStream *s;
    try {
        s = new ZkStream(pool, n_workers, stride, label, capacity);
        { std::lock_guard<std::mutex> lk(pool->mu); if (pool->th.empty()) pool->device = device; }
        while (pool->th.size() < n_workers) { const uint32_t idx = (uint32_t)pool->th.size(); pool->th.emplace_back([pool, idx] { pool->worker(idx); }); }
    } catch (...) { std::lock_guard<std::mutex> lk(pool->mu); pool->busy = false; throw; }
    { std::lock_guard<std::mutex> lk(pool->mu); pool->stream = s; pool->active = n_workers; pool->stream_gen++; }
    pool->cv.notify_all();
    *stream = s;
    return 0;
    DPH_CATCH
}
// Copies n inputs (n x input_len int64; the caller may reuse its buffer at once) and queues them with the consecutive tickets
// *first_ticket, ... (tickets count up from 0 in submission order across the stream's calls).  All or nothing: when the capacity has
// no room for all n, waits up to timeout_ms (0: no wait, < 0: for ever), then DP_ERR_TIMEOUT with nothing submitted.
// n > capacity is DP_ERR_INVALID.
extern "C" int dph_zkml_stream_submit(void *stream, const int64_t *inputs, uint32_t n, int64_t timeout_ms, uint64_t *first_ticket) {
    if (!stream) { g_herr = "dph_zkml_stream_submit: null stream"; return DP_ERR_INVALID; }
    return ((ZkStream *)stream)->q.submit(inputs, n, timeout_ms, first_ticket, g_herr);
}
// One finished job, in completion order: its ticket, its flat proof (at most stride words) and length, its model output (output_len
// elements, dph_zkml_output_len) and its status.  A job fails alone, as in dph_zkml_prove_batch: status != 0, proof_len 0, output
// zeros, and msg (msg_cap bytes, NUL-terminated, optional) holds the message dph_zkml_prove_batch gives that input; msg is empty for a
// proved job.  Unlike dph_zkml_prove_batch, a proof longer than the stride fails only its own job (DP_ERR_INVALID).  The call returns
// DP_ERR_STATE at once when nothing is queued, running or waiting to be collected, and DP_ERR_TIMEOUT after timeout_ms (0: no wait,
// < 0: for ever).  Several threads may call it, and submit, at once: each result goes to exactly one caller.
extern "C" int dph_zkml_stream_next(void *stream, int64_t timeout_ms, uint64_t *ticket, uint64_t *proof, uint64_t *proof_len, int64_t *output,
                                    int32_t *status, char *msg, uint64_t msg_cap) {
    DPH_TRY
    if (!stream || !ticket || !proof || !proof_len || !output || !status) throw Error(DP_ERR_INVALID, "dph_zkml_stream_next: null argument");
    ZkStream *s = (ZkStream *)stream;
    dp::QueueResult r;
    if (const int rc = s->q.next(timeout_ms, r, g_herr)) return rc;
    const size_t ol = s->pool->h->model.output_len();
    *ticket = r.ticket; *status = r.status; *proof_len = r.proof.size();
    memcpy(proof, r.proof.data(), 8 * r.proof.size());
    if (r.status) memset(output, 0, 8 * ol); else memcpy(output, r.output.data(), 8 * ol);
    if (msg && msg_cap) snprintf(msg, msg_cap, "%s", r.error.c_str());
    return 0;
    DPH_CATCH
}
// Closes the stream: the jobs no worker has started are cancelled, never proved, and counted in *n_cancelled (optional); the running
// jobs are waited for, uncollected results dropped, and the pool released.  A submit or next waiting on the stream returns
// DP_ERR_STATE before close returns; no call may use the stream pointer after it.  dph_zkml_context_free on the handle closes an
// open stream first, and the stream pointer is then invalid.
extern "C" int dph_zkml_stream_close(void *stream, uint64_t *n_cancelled) {
    if (!stream) { g_herr = "dph_zkml_stream_close: null stream"; return DP_ERR_INVALID; }
    const uint64_t n = close_stream((ZkStream *)stream);
    if (n_cancelled) *n_cancelled = n;
    return 0;
}

// One proof sharded over `world` ranks: `mles` are THIS rank's slices (nv_total - log2(world) variables each).
// Exchange: shm_region != NULL -> same-node shared-memory mailbox (sizeof = dph_shm_mailbox_bytes(), zero-initialised,
// mapped by every rank; `*shm_seq` carries the mailbox sequence number across calls); else `cb(user, send, n, recv)`.
extern "C" uint64_t dph_shm_mailbox_bytes() { return sizeof(ShmMailbox); }
// one raw all-gather through the mailbox (host-only; used by the CPU tests of the exchange itself)
extern "C" int dph_shm_allgather(void *shm_region, uint32_t world, uint32_t rank, uint64_t *shm_seq, const uint64_t *send, uint64_t n_words, uint64_t *recv) {
    DPH_TRY
    ShmExchange ex(shm_region, world, rank); ex.seq = *shm_seq;
    ex.allgather((const u64 *)send, n_words, (u64 *)recv);
    *shm_seq = ex.seq;
    return 0;
    DPH_CATCH
}
// Runs fn(ex) over this rank's exchange: the shared-memory mailbox when shm_region is given (its sequence number carried in and out
// through shm_seq; when fn throws the mailbox is poisoned, so peers fail fast instead of spinning on this rank's slot), else the callback.
template <class Fn>
static auto with_exchange(void *shm_region, uint64_t *shm_seq, CallbackExchange::Fn cb, void *user, uint32_t world, uint32_t rank, const char *entry, Fn fn) {
    if (shm_region) {
        ShmExchange ex(shm_region, world, rank); if (shm_seq) ex.seq = *shm_seq;
        try { auto r = fn(ex); if (shm_seq) *shm_seq = ex.seq; return r; }
        catch (...) { ex.poison(); if (shm_seq) *shm_seq = ex.seq; throw; }
    }
    if (!cb && world > 1) throw Error(DP_ERR_INVALID, std::string(entry) + ": no exchange given");
    CallbackExchange ex(cb, user, world, rank);
    return fn(ex);
}
extern "C" int dph_sumcheck_prove_sharded(uint32_t world, uint32_t rank, dp_mle *const *mles, uint32_t n_mles, const dp_sc_product *products, uint32_t n_products,
                                          uint32_t nv_total, const char *label, void *shm_region, uint64_t *shm_seq, CallbackExchange::Fn cb, void *user,
                                          uint64_t *out_point, uint64_t *out_msgs, uint64_t *out_final) {
    DPH_TRY
    uint32_t logG = 0; while ((1u << logG) < world) logG++;
    VirtualPolynomial vp = make_poly(mles, n_mles, products, n_products, nv_total - logG);
    DynTranscript tr(label);
    auto res = with_exchange(shm_region, shm_seq, cb, user, world, rank, "prove_sharded",
                             [&](Exchange &ex) { return IOPProverState::prove_sharded(std::move(vp), nv_total, ex, tr); });
    write_proof(res, products, n_products, n_mles, out_point, out_msgs, out_final);
    return 0;
    DPH_CATCH
}

// Basefold commit + open of ONE polynomial sharded over `world` ranks (every rank passes the whole polynomial, resident on its
// GPU).  Exchange as in dph_sumcheck_prove_sharded.  out = the flat proof image of dph_pcs_open (identical on every rank and
// identical to the unsharded proof), out_root = the commitment root.  `times_ms` (optional, 2 doubles): commit / open wall time.
extern "C" int dph_pcs_open_sharded(uint32_t world, uint32_t rank, dp_mle *poly, uint32_t full_log, const uint64_t *point, const char *label,
                                    void *shm_region, uint64_t *shm_seq, CallbackExchange::Fn cb, void *user,
                                    uint64_t *out, uint64_t cap, uint64_t *out_len, uint64_t *out_root, double *times_ms) {
    DPH_TRY
    DeviceMle m = view(poly);
    BasefoldProverParams pp; pp.full_message_size_log = full_log;
    const ExtVec pt = exts(point, m.num_vars());
    DynTranscript t(label);
    auto run = [&](Exchange &ex) {
        auto t0 = std::chrono::steady_clock::now();
        auto comm = Basefold::commit_sharded(pp, m, ex);
        auto t1 = std::chrono::steady_clock::now();
        if (out_root) memcpy(out_root, comm.root.v, 32);
        BasefoldProof pr = Basefold::open_sharded(pp, comm, pt, t, ex);
        auto t2 = std::chrono::steady_clock::now();
        if (times_ms) { times_ms[0] = std::chrono::duration<double, std::milli>(t1 - t0).count(); times_ms[1] = std::chrono::duration<double, std::milli>(t2 - t1).count(); }
        return pr.flatten();
    };
    return put_flat("dph_pcs_open_sharded", with_exchange(shm_region, shm_seq, cb, user, world, rank, "dph_pcs_open_sharded", run), out, cap, out_len);
    DPH_CATCH
}

// prove_batch_polys over T contiguous slices of the caller's device MLEs (views, no copies)
extern "C" int dph_sumcheck_prove_batch_polys(uint32_t T, dp_mle *const *mles, uint32_t n_mles, const dp_sc_product *products, uint32_t n_products,
                                              uint32_t max_nv, const char *label, uint64_t *out_point, uint64_t *out_msgs, uint64_t *out_final) {
    DPH_TRY
    uint32_t logT = 0; while ((1u << logT) < T) logT++;
    std::vector<VirtualPolynomial> polys;
    for (uint32_t t = 0; t < T; t++) polys.push_back(make_poly(mles, n_mles, products, n_products, max_nv - logT, t, T));
    DynTranscript tr(label);
    auto res = IOPProverState::prove_batch_polys(T, std::move(polys), tr);
    write_proof(res, products, n_products, n_mles, out_point, out_msgs, out_final);
    return 0;
    DPH_CATCH
}

// ---- FFT-convolution layer in isolation (host/conv.hpp): inference + layer proof ----------------------------------
// The output claim is drawn as Prover::prove draws the model-output claim (iop/prover.rs:423-436): point from the
// transcript, eval = MLE(cleared output)(point).  Flat layout: host/zkml.hpp flatten_conv_proof.
extern "C" int dph_conv_prove(uint32_t kw, uint32_t kx, uint32_t n_x, uint32_t real_nw, const int64_t *filter, const int64_t *bias, const uint32_t *unpadded_out,
                              const int64_t *input, const char *label, int64_t *out_after_bias, int64_t *out_cleared, uint64_t *out, uint64_t cap, uint64_t *out_len) {
    DPH_TRY
    using namespace dp::zkml;
    Convolution c; c.kw = kw; c.kx = kx; c.nw = n_x; c.real_nw = real_nw;
    c.filter.assign(filter, filter + (size_t)kw * kx * real_nw * real_nw); c.bias.assign(bias, bias + kw);
    for (int i = 0; i < 3; i++) c.unpadded_out[i] = unpadded_out[i];
    c.load();
    std::vector<Element> x(input, input + (size_t)kx * n_x * n_x);
    ConvData pd;
    DeviceMle cleared = c.op(DeviceMle::from_evaluations_vec(to_base(x)), pd);
    if (out_after_bias) { std::vector<Element> a = to_elements(pd.output_as_element); memcpy(out_after_bias, a.data(), 8 * a.size()); }
    if (out_cleared) { std::vector<Element> a = to_elements(cleared); memcpy(out_cleared, a.data(), 8 * a.size()); }
    if (!out_len) return 0;
    DynTranscript t(label);
    Claim cl; for (size_t i = 0; i < ceil_log2(cleared.len()); i++) cl.point.push_back(t.read_challenge());
    cl.eval = cleared.evaluate(cl.point);
    ConvProof pr; Claim in_claim = c.prove_convolution_step(t, cl, pd, pr);
    ProofImage w; flatten_conv_proof(w, pr, in_claim);
    return put_flat("dph_conv_prove", w.words, out, cap, out_len);
    DPH_CATCH
}

// General model builder: `desc` holds 9 int64 per node {kind, 8 shape words} and `data` the weights in node order
// (kind 5 MatMul {rows, inner, cols, transposed, has_bias}: the constant right matrix then the bias; kind 0 Dense {nrows, ncols}: weights then bias; 1 Requant {right_shift, fp_scale, multiplier, intermediate_bits};
//  2 ReLU; 3 Conv {kw, kx, nw, real_nw, unpadded_out[3]}: filter then bias; 4 Maxpool {C, H, W}).  Builds the Context: uploads
// weights, bias and tables and commits them (CommitmentContext::new) -- setup, not proving.  dph_zkml_prove /
// dph_zkml_prove_concurrent / dph_zkml_prove_batch / dph_zkml_context_free take the handle.
extern "C" int dph_model_context_new(const int64_t *desc, uint32_t n_nodes, const int64_t *data, uint64_t input_len, void **out) {
    DPH_TRY
    using namespace dp::zkml;
    auto h = std::make_unique<ZkHandle>();
    h->model.input_len = input_len;
    const int64_t *w = data;
    for (uint32_t i = 0; i < n_nodes; i++) {
        const int64_t *d = desc + 9 * (size_t)i; Node n;
        switch (d[0]) {
        case 0: n.op = Op::Dense; n.nrows = d[1]; n.ncols = d[2]; n.weights.assign(w, w + n.nrows * n.ncols); w += n.nrows * n.ncols; n.bias.assign(w, w + n.nrows); w += n.nrows; break;
        case 1: n.op = Op::Requant; n.rq.right_shift = d[1]; n.rq.fp_scale = d[2]; n.rq.fixed_point_multiplier = d[3]; n.rq.intermediate_bit_size = d[4]; break;
        case 2: n.op = Op::Relu; break;
        case 3: { n.op = Op::Conv; n.kw = d[1]; n.kx = d[2]; n.nw = d[3]; n.real_nw = d[4]; for (int k = 0; k < 3; k++) n.unpadded_out[k] = d[5 + k];
                  size_t fl = n.kw * n.kx * n.real_nw * n.real_nw; n.weights.assign(w, w + fl); w += fl; n.bias.assign(w, w + n.kw); w += n.kw; break; }
        case 4: n.op = Op::Pool; n.pool_c = d[1]; n.pool_h = d[2]; n.pool_w = d[3]; break;
        case 5: n.op = Op::MatMul; n.mm_r = d[1]; n.mm_k = d[2]; n.mm_c = d[3]; n.mm_t = d[4] != 0; n.mm_bias = d[5] != 0; n.weights.assign(w, w + n.mm_k * n.mm_c); w += n.mm_k * n.mm_c;
                if (n.mm_bias) { n.bias.assign(w, w + n.mm_c); w += n.mm_c; } break;
        default: throw Error(DP_ERR_INVALID, "dph_model_context_new: unknown node kind");
        }
        h->model.nodes.push_back(std::move(n));
    }
    h->ctx = Context::generate(h->model);
    check(dp_synchronize());
    *out = h.release();
    return 0;
    DPH_CATCH
}

// batch_commit (+ simple_batch_open at `point` when given): polys are caller-owned device MLEs of equal size / field
extern "C" int dph_pcs_simple_batch(dp_mle *const *polys, uint32_t n, uint32_t full_log, const uint64_t *point, uint32_t nv, const uint64_t *evals, const char *label,
                                    uint64_t *out_root, uint64_t *out, uint64_t cap, uint64_t *out_len) {
    DPH_TRY
    BasefoldProverParams pp; pp.full_message_size_log = full_log;
    std::vector<DeviceMle> ps;
    for (uint32_t i = 0; i < n; i++) ps.push_back(view(polys[i]));
    BasefoldCommitmentWithWitness comm = Basefold::batch_commit(pp, ps);
    memcpy(out_root, comm.root.v, 32);
    if (!point) return 0;
    DynTranscript t(label);
    SimpleBatchProof sp = Basefold::simple_batch_open(pp, comm, exts(point, nv), exts(evals, n), t);
    return put_flat("dph_pcs_simple_batch", sp.flatten(), out, cap, out_len);
    DPH_CATCH
}

// batch_open with an explicit evaluation list: `points` = n_points points concatenated (point k has point_nv[k] elements),
// evaluation j claims polys[eval_poly[j]] at points[eval_point[j]] (the value is computed here)
extern "C" int dph_pcs_batch_open_evals(dp_mle *const *polys, uint32_t n, uint32_t full_log, const uint64_t *points, const uint32_t *point_nv, uint32_t n_points,
                                        const uint32_t *eval_poly, const uint32_t *eval_point, uint32_t n_evals, const char *label, uint64_t *out, uint64_t cap, uint64_t *out_len) {
    DPH_TRY
    BasefoldProverParams pp; pp.full_message_size_log = full_log;
    std::vector<DeviceMle> ms; std::vector<BasefoldCommitmentWithWitness> comms; std::vector<ExtVec> pts; std::vector<Evaluation> evals;
    for (uint32_t i = 0; i < n; i++) { ms.push_back(view(polys[i])); comms.push_back(Basefold::commit(pp, ms.back())); }
    size_t o = 0;
    for (uint32_t k = 0; k < n_points; k++) { pts.push_back(exts(points + 2 * o, point_nv[k])); o += point_nv[k]; }
    for (uint32_t j = 0; j < n_evals; j++) { Evaluation ev; ev.poly = eval_poly[j]; ev.point = eval_point[j]; ev.value = ms.at(ev.poly).evaluate(pts.at(ev.point)); evals.push_back(ev); }
    DynTranscript t(label);
    BasefoldProof pr = Basefold::batch_open(pp, ms, comms, pts, evals, t);
    return put_flat("dph_pcs_batch_open_evals", pr.flatten(), out, cap, out_len);
    DPH_CATCH
}

// logup_gkr::prover::batch_prove (zkml.hpp logup_batch_prove) over device columns with DynTranscript::new(label): `table` (then mult is
// the multiplicities column) or lookup instances of columns_per_instance columns.  out: the proof as [n_proofs, then per proof its
// rounds, (deg+1) x E per round and its point], [n_evals per layer, evals], the final point and claims, then one challenge drawn from
// the transcript afterwards (its state); *out_len words.
extern "C" int dph_logup_prove(dp_mle *const *cols, uint32_t n_cols, dp_mle *mult, uint32_t columns_per_instance, const uint64_t cc[2], const uint64_t sc[2],
                    const char *label, uint64_t *out, uint64_t cap, uint64_t *out_len) {
    DPH_TRY
    zkml::LogUpInput in;
    in.table = mult != nullptr;
    for (uint32_t i = 0; i < n_cols; i++) in.column_evals.push_back(view(cols[i]));
    if (mult) in.multiplicities = view(mult);
    in.constant_challenge = Ext(cc[0], cc[1]); in.column_separation_challenge = Ext(sc[0], sc[1]); in.columns_per_instance = columns_per_instance;
    DynTranscript t(label ? label : "");
    zkml::LogUpProof pr = zkml::logup_batch_prove(in, t);
    ProofImage w;
    w.put(pr.sumcheck_proofs.size());
    for (auto &p : pr.sumcheck_proofs) { w.put(p.proofs.size()); for (auto &m : p.proofs) w.exts(m.evaluations); for (auto &e : p.point) w.ext(e); }
    for (auto &ev : pr.round_evaluations) w.exts(ev);
    for (auto &c : pr.output_claims) { for (auto &e : c.point) w.ext(e); w.ext(c.eval); }
    w.ext(t.get_and_append_challenge("after"));
    return put_flat("dph_logup_prove", w.words, out, cap, out_len);
    DPH_CATCH
}

