// Library-internal context: one per host thread, with its own stream and device arena.  A context belongs to the thread that
// made it and is only ever touched from that thread, so it needs no lock; a device block may still be released on another thread,
// through the arena's foreign-free path (dp_dev_free), which takes the slab registry's lock.
#pragma once
#include "gl.cuh"
#include "../../include/deepprove_b200.h"
#include <memory>
#include <string>
#include <utility>
#include <vector>
#include <cstdio>
#include <cstring>

struct DpCtx {
    bool ready = false;
    int device = -1;
    int sm_count = 132;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    u64 *sync_flag = nullptr; u64 sync_seq = 0;   // dp_stream_sync: this thread's pinned completion word
    std::vector<void *> zero_blocks;               // 256-byte device blocks known to hold zeros (dp_zero_block_get/put)
};
DpCtx &dp_ctx();
int dp_fail(int code, const std::string &s);

#define DP_CUDA(x)                                                                                          \
    do {                                                                                                    \
        cudaError_t e_ = (x);                                                                               \
        if (e_ != cudaSuccess) return dp_fail(DP_ERR_CUDA, std::string(#x) + ": " + cudaGetErrorString(e_)); \
    } while (0)
#define DP_CHECK(cond, code, msg) \
    do { if (!(cond)) return dp_fail((code), (msg)); } while (0)
#define DP_REQUIRE_CTX() DP_CHECK(dp_ctx().ready, DP_ERR_NO_DEVICE, "dp_init() has not succeeded: no CUDA device context")

// ---- launching kernels -------------------------------------------------------------------------------------------------
// Every kernel of the library is launched by one of these two: they count the launch (dp_kernel_launches) and return its error,
// for the caller's DP_CUDA.
void dp_count_launch();
template <class... P, class... A>
cudaError_t dp_launch(void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A &&...args) {
    kernel<<<grid, block, smem, st>>>(std::forward<A>(args)...);
    dp_count_launch();
    return cudaGetLastError();
}
// ... and as one thread-block cluster of ncta CTAs (the resident sumcheck kernels)
template <class... P, class... A>
cudaError_t dp_launch_cluster(void (*kernel)(P...), unsigned ncta, dim3 block, cudaStream_t st, A &&...args) {
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = ncta; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cudaLaunchConfig_t lc{};
    lc.gridDim = dim3(ncta); lc.blockDim = block; lc.dynamicSmemBytes = 0; lc.stream = st;
    lc.attrs = at; lc.numAttrs = 1;
    const cudaError_t e = cudaLaunchKernelEx(&lc, kernel, std::forward<A>(args)...);
    dp_count_launch();
    const cudaError_t last = cudaGetLastError();   // also clears the error a refused launch leaves there
    return e != cudaSuccess ? e : last;
}

// optional per-kernel timing with CUDA events on the launch stream (bench.py's roofline leg)
int dp_prof_begin(const char *name, u64 algorithmic_bytes, u64 units = 0);   // returns a token (or -1 when disabled); units: permutations / field ops
void dp_prof_end(int token);
struct DpProfScope {
    int tok;
    DpProfScope(const char *name, u64 bytes, u64 units = 0) : tok(dp_prof_begin(name, bytes, units)) {}
    ~DpProfScope() { dp_prof_end(tok); }
};

// ---- waiting for the device -------------------------------------------------------------------------------------------
// Every round of the prover ends with the host waiting for a word the GPU writes into mapped pinned memory.  Two modes:
//   DP_WAIT_SPIN  (default): the calling thread spins on the word -- lowest latency, one busy core per proof in flight.
//   DP_WAIT_BLOCK: the thread registers (word, expected value) with ONE process-wide poller thread and sleeps on a futex; the
//     poller sweeps all registered words and wakes the owner.  ~5 us more per wait, but a waiting proof costs no CPU, so the
//     number of proofs in flight per GPU is no longer capped by the host's cores (the measurement boxes give a GPU 16 CPUs).
// dp_wait_flag returns the value seen: `want`, or `fail` (if has_fail), or ~0 - 2 on timeout.
enum : int { DP_WAIT_SPIN = 0, DP_WAIT_BLOCK = 1 };
static constexpr u64 DP_WAIT_TIMEOUT = ~0ULL - 2;
int dp_wait_mode();
u64 dp_wait_flag(volatile u64 *flag, u64 want, bool has_fail, u64 fail, double timeout_s);
// cudaStreamSynchronize for the hot path: in DP_WAIT_BLOCK mode a one-thread kernel raises this thread's pinned word at the
// end of the stream's queued work and the thread sleeps on it (cudaStreamSynchronize itself spins in the driver).
cudaError_t dp_stream_sync(cudaStream_t st);
// A completion word: a kernel publishes `v` with dp_publish after its results, and the host waits for it with dp_await.  When the
// word does not come within timeout_s, dp_await drains the context's stream, looks once more and refuses with `refusal`.
__device__ __forceinline__ void dp_publish(volatile u64 *word, u64 v) { __threadfence_system(); *word = v; }
int dp_await(volatile u64 *word, u64 want, double timeout_s, const std::string &refusal);

// Device -> caller's (pageable) host memory, then wait: staged through pinned memory so that the copy call returns at once
// and the wait goes through the wait service.  (cudaMemcpyAsync into pageable memory blocks INSIDE the driver, spinning, until
// every kernel queued before it has finished: 182 such calls per Dense-4M proof were 7 ms of a 44 ms proof and, with 32
// proofs in flight, 6 of the 16 CPUs a GPU gets.)  Several pieces may be gathered before one wait: dp_d2h_begin / _add / _finish.
int dp_d2h(void *host_dst, const void *dev_src, size_t bytes, cudaStream_t st);
struct DpD2H {
    struct Piece { void *dst; size_t off, bytes; };
    void *pin = nullptr; size_t cap = 0, used = 0; std::vector<Piece> pieces; cudaStream_t st;
    explicit DpD2H(cudaStream_t s, size_t reserve_bytes);
    int add(void *host_dst, const void *dev_src, size_t bytes);
    int finish();          // wait for the stream, then scatter into the destinations
    ~DpD2H();
};

// 256-byte device blocks that hold zeros: ticket counters of the multi-block reductions.  The kernels leave them zero again, so a
// block is cleared once when it is first carved out of the arena and then recycled (a memset node per sumcheck -- 151 per
// Dense-4M proof -- was pure driver-call overhead).  Only put back blocks whose kernels have all completed normally.
int dp_zero_block_get(void **p);
void dp_zero_block_put(void *p);

// device blocks from this thread's arena
int dp_dev_alloc(void **p, size_t bytes);
int dp_dev_free(void *p);
void dp_arena_defer(bool on);   // hold releases back while several streams are in flight (dp_pcs_commit_many)
// pinned host staging buffers, cached per context (cudaHostAlloc/cudaFreeHost cost ~ms and synchronise)
int dp_pinned_alloc(void **p, size_t bytes);
void dp_pinned_free(void *p);

struct dp_mle {
    void *data = nullptr;   // u64[len] or gle[len]
    u64 len = 0;
    bool is_ext = false;
    bool owned = true;
    u32 num_vars() const { u32 l = 0; while ((1ULL << l) < len) l++; return l; }
    size_t bytes() const { return (size_t)len * (is_ext ? 16 : 8); }
};

// LogUp-GKR circuit (logup.cu); its small layers are also proved by the resident sumcheck kernel (sumcheck.cu)
struct dp_logup {
    bool table = false; u32 nv = 0;            // layer 0 has 2^nv entries
    std::vector<gle *> num, den;               // per layer; num[0] == nullptr for a lookup circuit
    gle *block = nullptr;
    u64 *h_out = nullptr;                      // mapped pinned: outputs + completion word written by k_logup_tail
};

// Owning handles for objects under construction: an error return releases whatever has been built so far.
template <auto Free> struct FreeWith { template <typename P> void operator()(P *p) const { Free(p); } };
using MlePtr = std::unique_ptr<dp_mle, FreeWith<dp_mle_free>>;
using DevPtr = std::unique_ptr<void, FreeWith<dp_dev_free>>;
using PinnedPtr = std::unique_ptr<void, FreeWith<dp_pinned_free>>;

// A table of `len` elements that the MLE owns, allocated in the arena (contents undefined)
static inline int dp_mle_alloc(u64 len, bool ext, MlePtr &out) {
    MlePtr m(new dp_mle());
    m->len = len; m->is_ext = ext;
    if (int e = dp_dev_alloc(&m->data, m->bytes())) return e;
    out = std::move(m);
    return DP_OK;
}
// A view of `len` elements at `data`, which stay the owner's
static inline dp_mle *dp_mle_view(void *data, u64 len, bool ext) {
    dp_mle *v = new dp_mle();
    v->data = data; v->len = len; v->is_ext = ext; v->owned = false;
    return v;
}

static inline int dp_grid_for(u64 work_items, int threads, int max_ctas_per_sm) {
    u64 g = (work_items + threads - 1) / threads;
    u64 cap = (u64)dp_ctx().sm_count * max_ctas_per_sm;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

// ---- kernel launchers shared between translation units (mle.cu) ----
int dpk_fold_low(const void *src, bool src_ext, u64 len, gle r, gle *out_dev);      // K2 (stand-alone)
