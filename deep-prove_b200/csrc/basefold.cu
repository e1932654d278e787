// Basefold multilinear PCS on device: commit (K7 hypercube interpolation, K8 RS/NTT encode, K9 Merkle tree:
// merkle.cu), open / batch_open commit phase (K10 FRI fold, K11 coefficient-form sumcheck via the sumcheck
// engine, K12 batch prelude) and query gathering (K13: merkle.cu).
// Reference: mpcs/src/basefold.rs:86-154,304-354,466-770; basefold/{commit_phase.rs,sumcheck.rs,
// encoding/rs.rs,query_phase.rs:31-138,373-534}; util/{arithmetic.rs:120-132,arithmetic/hypercube.rs}.
//
// Data layout in HBM (per commitment of a 2^nu polynomial): bh_evals = bit-reversed evaluations (8 or
// 16 B/elt), codeword = bit-reversed RS codeword of 2^(nu+1) elements, the Merkle tree over the codeword
// (merkle.cuh).  Everything stays resident until the opening: roots and round messages are the only D2H traffic.
//
// Linear-algebra shortcuts (exact arithmetic, identical field elements):
//  * interpolate_over_boolean_hypercube commutes with the bit-reversal permutation, so the coefficient
//    vector the reference encodes, bitrev(interp(evals)), is interp(bh_evals): one permutation serves both.
//  * a decimation-in-frequency NTT of the natural-order input yields the spectrum in bit-reversed order,
//    which IS the stored codeword (basefold.rs:151 bit-reverses the DIT output) -- no final permutation.
//  * the zero-padded upper half makes the first DIF level a pure copy-and-scale (k_expand).
#include "common.cuh"
#include "powtab.cuh"
#include "merkle.cuh"
#include <algorithm>
#include <atomic>
#include <map>
#include <memory>
#include <mutex>

static constexpr u32 BF_RATE_LOG = 1;            // RSCodeDefaultSpec (rs.rs:192-214)
static constexpr u32 BF_BASECODE_LOG = 7;
static constexpr u64 GL_ROOT32 = 1753635133440165772ULL;  // p3 Goldilocks two-adic generator, order 2^32

// ---- root-of-unity / coset power tables: x^e = T0[e & 2047] * T1[(e >> 11) & 2047] * T2[e >> 22] ----
__global__ void k_pow_table(u64 base, u64 *t /* 3 x 2048 */) {
    u32 k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= 3 * 2048) return;
    u32 part = k >> 11, idx = k & 2047;
    u64 e = (u64)idx << (11 * part);
    t[k] = gl_pow(base, e);
}
static PowTab powtab_at(const u64 *t) { PowTab p; p.t0 = t; p.t1 = t + 2048; p.t2 = t + 4096; return p; }
// a table that lives for the rest of the process, complete before it is returned: other host threads' streams may read it as soon
// as the caller publishes the pointer
static int pow_table_build(u64 base, const u64 **out) {
    u64 *tab = nullptr;
    DP_CUDA(cudaMalloc((void **)&tab, sizeof(u64) * 3 * 2048));
    DP_CUDA(dp_launch(k_pow_table, 24, 256, 0, dp_ctx().stream, base, tab));
    DP_CUDA(dp_stream_sync(dp_ctx().stream));
    *out = tab;
    return DP_OK;
}
static std::atomic<const u64 *> g_root_tab{nullptr};   // process-wide, read-only once built (shared by every host thread's context)
static std::mutex g_bf_mu;
static int bf_prepare() {
    if (g_root_tab.load()) return DP_OK;
    std::lock_guard<std::mutex> lk(g_bf_mu);
    if (!g_root_tab.load()) {
        const u64 *tab = nullptr;
        if (int e = pow_table_build(GL_ROOT32, &tab)) return e;
        g_root_tab.store(tab);
    }
    return DP_OK;
}
static PowTab root_tab() { return powtab_at(g_root_tab.load()); }
int dp_root_powtab(PowTab *out) { if (int e = bf_prepare()) return e; *out = root_tab(); return DP_OK; }
// shift^j tables, one per coset shift (i.e. per full_log - nv), built on first use and kept
static int shift_powtab(u64 shift, PowTab *out) {
    static std::map<u64, const u64 *> tabs;
    std::lock_guard<std::mutex> lk(g_bf_mu);
    auto it = tabs.find(shift);
    if (it == tabs.end()) {
        const u64 *tab = nullptr;
        if (int e = pow_table_build(shift, &tab)) return e;
        it = tabs.emplace(shift, tab).first;
    }
    *out = powtab_at(it->second);
    return DP_OK;
}
// coset shift of a 2^nv polynomial committed under full_log: 7^(2^(full_log - nv))  (rs.rs:481-488)
static u64 coset_shift(u32 full_log, u32 nv) { u64 shift = 7; for (u32 i = 0; i < full_log - nv; i++) shift = gl_sqr(shift); return shift; }

// ---- bit reversal (out of place) ----
template <typename T>
__global__ void k_bitrev(const T *__restrict__ in, T *__restrict__ out, u32 lg) {
    u64 n = 1ULL << lg, i = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    for (; i < n; i += stride) { u64 j = lg ? (__brevll(i) >> (64 - lg)) : 0; out[j] = in[i]; }
}

// ---- generic tiled butterfly pass over levels [a, b) of an n_log-sized array, in place ----
// level l pairs (i, i + (N >> (l+1))).  MODE 0: Moebius (hi -= lo).  MODE 1: DIF NTT (lo = u+v, hi = (u-v) w).
__device__ __forceinline__ u64 t_add(u64 a, u64 b) { return gl_add(a, b); }
__device__ __forceinline__ gle t_add(gle a, gle b) { return e_add(a, b); }
__device__ __forceinline__ u64 t_sub(u64 a, u64 b) { return gl_sub(a, b); }
__device__ __forceinline__ gle t_sub(gle a, gle b) { return e_sub(a, b); }
__device__ __forceinline__ u64 t_mulb(u64 a, u64 w) { return gl_mul(a, w); }
__device__ __forceinline__ gle t_mulb(gle a, u64 w) { return e_mul_base(a, w); }

template <typename T, int MODE>
__global__ void k_tile_pass(T *__restrict__ data, u32 n_log, u32 a, u32 b, u32 c_log, PowTab tab) {
    extern __shared__ unsigned char smem_raw[];
    T *sm = reinterpret_cast<T *>(smem_raw);
    const u32 lv = b - a, rows = 1u << lv, C = 1u << c_log;
    const u64 stride = 1ULL << (n_log - b);             // distance between tile rows
    const u64 ncolgroups = stride >> c_log;
    const u64 tile = blockIdx.x;                         // (hi, colgroup)
    const u64 hi = tile / ncolgroups, cg = tile % ncolgroups;
    const u64 base = hi * (1ULL << (n_log - a)) + cg * C;
    const u32 elems = rows * C;
    for (u32 k = threadIdx.x; k < elems; k += blockDim.x) { u32 t = k >> c_log, c = k & (C - 1); sm[k] = data[base + (u64)t * stride + c]; }
    __syncthreads();
    for (u32 s = 0; s < lv; s++) {
        const u32 l = a + s, hrows = rows >> (s + 1);    // pair distance in rows
        const u32 npairs = (rows >> 1) * C;
        for (u32 q = threadIdx.x; q < npairs; q += blockDim.x) {
            u32 c = q & (C - 1), pr = q >> c_log;
            u32 t = ((pr / hrows) * 2 * hrows) + (pr % hrows);
            u32 i0 = t * C + c, i1 = (t + hrows) * C + c;
            T u = sm[i0], v = sm[i1];
            if (MODE == 0) sm[i1] = t_sub(v, u);
            else {
                u64 gi = base + (u64)t * stride + c;                 // global index of the pair's first element
                u64 half = 1ULL << (n_log - l - 1);
                u64 e = (gi & (half - 1)) << l;                      // exponent of w_N
                u64 w = tab_pow(tab, e << (32 - n_log));
                sm[i0] = t_add(u, v); sm[i1] = t_mulb(t_sub(u, v), w);
            }
        }
        __syncthreads();
    }
    for (u32 k = threadIdx.x; k < elems; k += blockDim.x) { u32 t = k >> c_log, c = k & (C - 1); data[base + (u64)t * stride + c] = sm[k]; }
}

template <typename T, int MODE>
static int run_levels(T *data, u32 n_log, u32 from, u32 to) {
    // levels [from, to): the last chunk is contiguous (C = 1, up to 11 levels), earlier chunks use 16 columns x <= 7 levels
    DpCtx &c = dp_ctx();
    PowTab tab = root_tab();
    u32 b = to;
    std::vector<std::pair<u32, u32>> chunks;  // processed in increasing level order (required for DIF)
    if (to == n_log) { u32 lv = std::min<u32>(to - from, sizeof(T) == 8 ? 11 : 10); chunks.push_back({to - lv, to}); b = to - lv; }
    while (b > from) { u32 lv = std::min<u32>(b - from, 7); chunks.push_back({b - lv, b}); b -= lv; }
    std::sort(chunks.begin(), chunks.end());
    for (auto &ch : chunks) {
        u32 lv = ch.second - ch.first;
        u32 c_log = (ch.second == n_log) ? 0 : std::min<u32>(4, n_log - ch.second);
        u64 tiles = 1ULL << (n_log - lv - c_log);
        size_t smem = sizeof(T) << (lv + c_log);
        if (smem > 48 * 1024) DP_CUDA(cudaFuncSetAttribute(k_tile_pass<T, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        DpProfScope prof(MODE ? "k_tile_pass(ntt)" : "k_tile_pass(moebius)", (sizeof(T) << n_log) * 2);
        DP_CUDA(dp_launch(k_tile_pass<T, MODE>, (unsigned)tiles, 256, smem, c.stream, data, n_log, ch.first, ch.second, c_log, tab));
    }
    return DP_OK;
}

// zero-pad x2 + coset scale + first DIF level: out[j] = x, out[j + m] = x * w_N^j, x = c[j] * shift^j
template <typename T>
__global__ void k_expand(const T *__restrict__ c, T *__restrict__ out, u32 lg_m, PowTab shift_tab, PowTab tab) {
    u64 m = 1ULL << lg_m, j = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    for (; j < m; j += stride) {
        T x = t_mulb(c[j], tab_pow(shift_tab, j));
        out[j] = x;
        out[j + m] = t_mulb(x, tab_pow(tab, j << (32 - (lg_m + 1))));
    }
}

// One polynomial's codeword sharded over G = 2^logG GPUs (SURVEY.md 8e, BASELINE configs[3]): rank g owns the contiguous slice
// [g S, (g+1) S), S = N / G, of the BIT-REVERSED codeword.  In a decimation-in-frequency NTT that slice is an independent
// size-S transform of   y_r[t] = w_N^(t r) * sum_k x[t + k S] * w_G^(k r),   r = bitrev_logG(g),  x[j] = c[j] shift^j (zero for j >= N/2):
// the first logG levels collapse into this one pass over the coefficients (every rank reads all of them once, no inter-GPU
// butterfly exchange), the remaining levels are the ordinary tiled passes on the local slice.
template <typename T>
__global__ void k_shard_expand(const T *__restrict__ c, T *__restrict__ out, u32 lg_m, u32 logG, u32 r, PowTab shift_tab, PowTab tab) {
    const u32 n_log = lg_m + 1;
    const u64 S = 1ULL << (n_log - logG), terms = 1ULL << (logG - 1);      // x[t + k S] is zero for k >= G/2 (the zero-padded half)
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    for (; t < S; t += stride) {
        T acc = t_mulb(c[t], tab_pow(shift_tab, t));
        for (u64 k = 1; k < terms; k++) {
            const u64 j = t + k * S;
            const u64 w = gl_mul(tab_pow(shift_tab, j), tab_pow(tab, (u64)((k * r) & ((1ULL << logG) - 1)) << (32 - logG)));
            acc = t_add(acc, t_mulb(c[j], w));
        }
        out[t] = t_mulb(acc, tab_pow(tab, (t * r) << (32 - n_log)));
    }
}

// ---- small polynomials: bit reversal, hypercube interpolation, zero-pad + coset scale, and the whole DIF NTT in ONE block ----
// (k_bitrev -> k_tile_pass<T,0> -> k_expand -> k_tile_pass<T,1> on a codeword that fits in shared memory: a 2^10 witness column
//  costs one launch instead of six; same butterflies, same twiddles, same order -> identical codeword)
template <typename T>
__global__ void __launch_bounds__(512) k_encode_small(const T *__restrict__ in, T *__restrict__ bh, T *__restrict__ cw, u32 nv, u64 shift, PowTab tab) {
    extern __shared__ unsigned char smem_raw[];
    T *sm = reinterpret_cast<T *>(smem_raw);
    __shared__ u64 sq[16];                                  // shift^(2^k)
    const u32 m = 1u << nv, n_log = nv + 1, N = 2u << nv;
    if (threadIdx.x == 0) { u64 x = shift; for (u32 k = 0; k < nv; k++) { sq[k] = x; x = gl_sqr(x); } }
    for (u32 j = threadIdx.x; j < m; j += blockDim.x) { T v = in[__brev(j) >> (32 - nv)]; bh[j] = v; sm[j] = v; }
    __syncthreads();
    for (u32 l = 0; l < nv; l++) {                          // interpolate_over_boolean_hypercube on the bit-reversed evaluations
        const u32 half = m >> (l + 1);
        for (u32 q = threadIdx.x; q < (m >> 1); q += blockDim.x) { u32 i0 = (q / half) * 2 * half + (q % half); sm[i0 + half] = t_sub(sm[i0 + half], sm[i0]); }
        __syncthreads();
    }
    for (u32 j = threadIdx.x; j < m; j += blockDim.x) {    // k_expand: x = c[j] shift^j ; out[j] = x ; out[j+m] = x w_N^j  (first DIF level of the zero-padded input)
        u64 sp = 1; for (u32 k = 0; k < nv; k++) if (j >> k & 1) sp = gl_mul(sp, sq[k]);
        T x = t_mulb(sm[j], sp);
        sm[j] = x; sm[j + m] = t_mulb(x, tab_pow(tab, (u64)j << (32 - n_log)));
    }
    __syncthreads();
    for (u32 l = 1; l < n_log; l++) {                       // remaining DIF levels
        const u32 half = N >> (l + 1);
        for (u32 q = threadIdx.x; q < (N >> 1); q += blockDim.x) {
            u32 i0 = (q / half) * 2 * half + (q % half), i1 = i0 + half;
            u64 e = (u64)(i0 & (half - 1)) << l;
            u64 w = tab_pow(tab, e << (32 - n_log));
            T u = sm[i0], v = sm[i1];
            sm[i0] = t_add(u, v); sm[i1] = t_mulb(t_sub(u, v), w);
        }
        __syncthreads();
    }
    for (u32 k = threadIdx.x; k < N; k += blockDim.x) cw[k] = sm[k];
}

// ---- K10 FRI fold (commit_phase.rs:511-526, rs.rs:377-410, arithmetic.rs:120-132) ----
// out[i] = y0 + (r - x0) * (y1 - y0) * w,  x0 = w_{2^(level+1)}^{rev(i, level)} * gamma_lvl,  w = -1/(2 x0)
// (`n` outputs starting at global index `off`: a rank of a sharded opening folds its own contiguous slice)
__global__ void k_fri_fold(const gle *__restrict__ in, gle *__restrict__ out, u32 level, u64 n, u64 off, gle r, u64 gamma_lvl, u64 neg_half_gamma_inv, PowTab tab) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        u64 e = level ? (__brevll(i + off) >> (64 - level)) : 0;       // rev(i, level), exponent of w_{2^(level+1)}
        u64 L = 1ULL << (level + 1);
        u64 x0 = gl_mul(tab_pow(tab, e << (32 - (level + 1))), gamma_lvl);
        u64 x0inv_root = tab_pow(tab, ((L - e) & (L - 1)) << (32 - (level + 1)));   // w^{-e}
        u64 w = gl_mul(x0inv_root, neg_half_gamma_inv);                  // -1/(2 x0)
        gle y0 = ld_e(in + 2 * i), y1 = ld_e(in + 2 * i + 1);
        gle t = e_mul_base(e_sub(r, e_from_base(x0)), w);
        st_e(out + i, e_add(y0, e_mul(t, e_sub(y1, y0))));
    }
}

// ---- K12 batch prelude (commit_phase.rs:205-236,271-282): out[i] = (base[i]) + sum_k coef_k * src_k[i >> rep_k] ----
// ONE pass for all sources: the reference (and the first version here) adds one polynomial at a time, i.e. a read-modify-write of
// the whole running oracle per commitment -- 47 passes over a 16 MB table in a Dense-4M opening.  Each thread owns one output
// element, walks the source table (kernel parameters, <= LC_MAX entries per launch) and accumulates the raw 128-bit products in
// 192-bit sums that are reduced once (field addition is exact, so the order is free and the element is identical).
static constexpr u32 LC_MAX = 96;
struct LcSrc { const void *p; u64 c0, c1; u32 ext, rep_log; };
struct LcArgs { LcSrc s[LC_MAX]; u32 n; u32 pad; };
template <bool HAS_BASE>
__global__ void __launch_bounds__(256) k_lincomb_bcast(gle *__restrict__ out, const gle *__restrict__ base, const __grid_constant__ LcArgs a, u64 n) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        gl_acc s0 = {0, 0, 0}, s1 = {0, 0, 0};
        for (u32 k = 0; k < a.n; k++) {
            const LcSrc &q = a.s[k];
            const u64 j = i >> q.rep_log;
            if (q.ext) {   // (c0 + c1 X)(x0 + x1 X) = c0 x0 + 7 c1 x1 + (c0 x1 + c1 x0) X
                const gle x = ld_e((const gle *)q.p + j);
                gl_acc_mac(s1, q.c0, x.c1); gl_acc_mac(s1, q.c1, x.c0);
                gl_acc_mac(s0, q.c0, x.c0); gl_acc_mac(s0, gl_reduce128_weak(q.c1 * x.c1, __umul64hi(q.c1, x.c1)), 7ULL);
            } else {
                const u64 x = ((const u64 *)q.p)[j];
                gl_acc_mac(s0, q.c0, x); gl_acc_mac(s1, q.c1, x);
            }
        }
        gle v = e_make(gl_acc_reduce(s0), gl_acc_reduce(s1));
        if (HAS_BASE) v = e_add(v, ld_e(base + i));
        st_e(out + i, v);
    }
}
struct LcTerm { const void *p; gle coef; bool ext; u32 rep_log; };
// out = (base ? base : 0) + sum terms; out may alias base.  Zero terms and no base: out = 0.
static int lincomb_bcast(gle *out, const gle *base, const std::vector<LcTerm> &terms, u64 n) {
    DpCtx &c = dp_ctx();
    if (terms.empty()) {
        if (!base) DP_CUDA(cudaMemsetAsync(out, 0, sizeof(gle) * n, c.stream));
        else if (base != out) DP_CUDA(cudaMemcpyAsync(out, base, sizeof(gle) * n, cudaMemcpyDeviceToDevice, c.stream));
        return DP_OK;
    }
    const int g = dp_grid_for(n, 256, 8);
    for (size_t o = 0; o < terms.size(); o += LC_MAX) {
        LcArgs a; memset(&a, 0, sizeof a);
        a.n = (u32)std::min<size_t>(LC_MAX, terms.size() - o);
        u64 src_bytes = 0;
        for (u32 k = 0; k < a.n; k++) { const LcTerm &t = terms[o + k]; a.s[k].p = t.p; a.s[k].c0 = t.coef.c0; a.s[k].c1 = t.coef.c1; a.s[k].ext = t.ext ? 1 : 0; a.s[k].rep_log = t.rep_log; src_bytes += (n >> t.rep_log) * (t.ext ? 16 : 8); }
        const gle *b = o == 0 ? base : out;
        DpProfScope p("k_lincomb_bcast", src_bytes + n * (b ? 32 : 16));
        DP_CUDA(dp_launch(b ? k_lincomb_bcast<true> : k_lincomb_bcast<false>, g, 256, 0, c.stream, out, b, a, n));
    }
    return DP_OK;
}
__global__ void k_lift(const u64 *__restrict__ src, gle *__restrict__ out, u64 n) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    for (; i < n; i += stride) st_e(out + i, e_from_base(src[i]));
}

// =====================================================================================================
struct dp_pcs_comm {
    u32 num_vars = 0, full_log = 0; bool is_base = true, trivial = false;
    void *bh_evals = nullptr;   // bit-reversed evals (raw evals when trivial)
    void *codeword = nullptr;   // bit-reversed codeword (== bh_evals when trivial)
    u64 cw_len = 0;
    DevTree tree;                       // over `codeword`; empty for the parts of a batch commitment
    const DevTree *batch_tree = nullptr;   // a part of a batch commitment: the batch's tree, over all the parts' codewords
    uint64_t root[4] = {0, 0, 0, 0};
    std::vector<dp_pcs_comm *> parts;   // batch_commit: one (encode-only) commitment per polynomial
    // dp_pcs_commit_shard: `codeword` / `bh_evals` / `tree` are this rank's contiguous slice (cw_len = local length); `top` is the
    // replicated tree over the world's subtree roots (dp_pcs_comm_set_shard_roots), `root` the global root once it is set
    u32 shard_rank = 0, shard_log = 0; DevTree top; uint64_t local_root[4] = {0, 0, 0, 0};
};

struct OpenRound { gle *oracle = nullptr; DevTree tree; DevTree top; };   // tree over `oracle`; top: sharded openings
struct dp_pcs_open {
    u32 num_vars = 0, full_log = 0, num_rounds = 0, round = 0;
    std::vector<const dp_pcs_comm *> comms; std::vector<gle> coeffs; bool batch = false;
    gle *oracle0 = nullptr; u64 n0 = 0;        // running oracle of the current round (E)
    bool oracle0_owned = true;
    std::vector<OpenRound> rounds;             // trees over the folded oracles (pre-addition copies)
    dp_mle *eq = nullptr, *evals = nullptr; bool evals_owned = false;
    dp_sc *sc = nullptr;
    gle final_msg[1 << BF_BASECODE_LOG]; bool have_final = false;
    gle *scratch_sum_evals = nullptr;
    u64 *h_root = nullptr; u64 root_seq = 0;     // mapped pinned: [0..3] root of the round's tree, [8] completion word
    u32 shard_rank = 0, shard_log = 0;           // sharded opening (one commitment from dp_pcs_commit_shard): everything above is the local slice
};

static void msg_to_coeffs(const uint64_t *ev /* p(0),p(1),p(2) */, uint64_t *out /* c0,c1,c2 */) {
    gle p0 = e_make(ev[0], ev[1]), p1 = e_make(ev[2], ev[3]), p2 = e_make(ev[4], ev[5]);
    const u64 inv2 = 0x7FFFFFFF80000001ULL;  // (p+1)/2
    gle c2 = e_mul_base(e_add(e_sub(p2, e_dbl(p1)), p0), inv2);
    gle c1 = e_sub(e_sub(p1, p0), c2);
    out[0] = p0.c0; out[1] = p0.c1; out[2] = c1.c0; out[3] = c1.c1; out[4] = c2.c0; out[5] = c2.c1;
}

// Owning handles (common.cuh) for the commitments and openings under construction
using CommPtr = std::unique_ptr<dp_pcs_comm, FreeWith<dp_pcs_comm_free>>;
using OpenPtr = std::unique_ptr<dp_pcs_open, FreeWith<dp_pcs_open_free>>;

// Encode of a 2^nv polynomial whose whole codeword fits in one block's shared memory: one launch
template <typename T>
static int encode_small(const void *evals, void *bh_evals, void *codeword, u32 nv, u64 shift) {
    const u64 m = 1ULL << nv;
    const size_t smem = sizeof(T) << (nv + BF_RATE_LOG);
    DpProfScope p("k_encode_small(bitrev+moebius+expand+ntt)", sizeof(T) * m * 2 + smem);
    if (smem > 48 * 1024) DP_CUDA(cudaFuncSetAttribute(k_encode_small<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    DP_CUDA(dp_launch(k_encode_small<T>, 1, 512, smem, dp_ctx().stream, (const T *)evals, (T *)bh_evals, (T *)codeword, nv, shift, root_tab()));
    return DP_OK;
}

// Tiled encode of a 2^nv polynomial: bit reversal, Moebius levels (K7), then zero-pad + coset scale + the DIF levels (K8).
// logG = 0: bh_evals and codeword are whole; k_expand does the first DIF level, tiled passes do levels [1, n_log).
// logG > 0: they are rank `rank`'s slices (2^(nv - logG) evaluations, 2^(n_log - logG) codeword entries); k_shard_expand does the
// first logG levels for this slice, tiled passes do levels [0, n_log - logG) on it.
template <typename T>
static int encode_tiled(const void *evals, void *bh_evals, void *codeword, u32 nv, u64 shift, u32 logG, u32 rank) {
    DpCtx &c = dp_ctx();
    const size_t esz = sizeof(T);
    const u32 n_log = nv + BF_RATE_LOG;
    const u64 m = 1ULL << nv, Ml = m >> logG, S = (1ULL << n_log) >> logG;
    T *bh = (T *)bh_evals, *cw = (T *)codeword, *coef = nullptr;
    if (int e = dp_dev_alloc((void **)&coef, esz * m)) return e;
    DevPtr coef_owner(coef);
    PowTab st; if (int e = shift_powtab(shift, &st)) return e;
    const int g = dp_grid_for(m, 256, 8);
    { DpProfScope p("k_bitrev", esz * m * 2); DP_CUDA(dp_launch(k_bitrev<T>, g, 256, 0, c.stream, (const T *)evals, logG ? coef : bh, nv)); }
    if (!logG) DP_CUDA(cudaMemcpyAsync(coef, bh, esz * m, cudaMemcpyDeviceToDevice, c.stream));
    else if (cudaMemcpyAsync(bh, coef + Ml * rank, esz * Ml, cudaMemcpyDeviceToDevice, c.stream) != cudaSuccess)
        return dp_fail(DP_ERR_CUDA, "dp_pcs_commit_shard: copy of the evaluation slice failed");
    if (int e = run_levels<T, 0>(coef, nv, 0, nv)) return e;
    if (!logG) { DpProfScope p("k_expand", esz * m * 3); DP_CUDA(dp_launch(k_expand<T>, g, 256, 0, c.stream, coef, cw, nv, st, root_tab())); }
    else {
        u32 rev_rank = 0; for (u32 b = 0; b < logG; b++) if (rank >> b & 1) rev_rank |= 1u << (logG - 1 - b);
        DpProfScope p("k_shard_expand", esz * (m + S));
        DP_CUDA(dp_launch(k_shard_expand<T>, dp_grid_for(S, 256, 8), 256, 0, c.stream, coef, cw, nv, logG, rev_rank, st, root_tab()));
    }
    return run_levels<T, 1>(cw, n_log - logG, logG ? 0 : 1, n_log - logG);
}

extern "C" {

// enqueue every kernel of one commitment on the context's CURRENT stream; the root lands in `root_pinned` (null: no tree, a batch part)
static int commit_enqueue(const dp_mle *poly, uint32_t full_log, dp_pcs_comm **out, u64 *root_pinned) {
    u32 nv = poly->num_vars();
    DP_CHECK(nv <= full_log, DP_ERR_INVALID, "PolynomialTooLarge");                 // basefold.rs:97-99
    DP_CHECK(nv >= 1, DP_ERR_INVALID, "dp_pcs_commit: need at least one variable");
    if (int e = bf_prepare()) return e;
    DpCtx &c = dp_ctx();
    CommPtr cm(new dp_pcs_comm());
    cm->num_vars = nv; cm->full_log = full_log; cm->is_base = !poly->is_ext;
    size_t esz = poly->is_ext ? 16 : 8;
    u64 m = poly->len;
    if (int e = dp_dev_alloc(&cm->bh_evals, esz * m)) return e;
    if (nv <= BF_BASECODE_LOG) {   // TooSmall: Merkle tree over the raw evaluations (basefold.rs:102-104)
        cm->trivial = true;
        DP_CUDA(cudaMemcpyAsync(cm->bh_evals, poly->data, esz * m, cudaMemcpyDeviceToDevice, c.stream));
        cm->codeword = cm->bh_evals; cm->cw_len = m;
    } else {
        cm->cw_len = m << BF_RATE_LOG;
        if (int e = dp_dev_alloc(&cm->codeword, esz * cm->cw_len)) return e;
        const u64 shift = coset_shift(full_log, nv);
        int rc;
        if (esz * cm->cw_len <= 64 * 1024 && nv <= 15)   // the whole codeword fits in one block's shared memory
            rc = poly->is_ext ? encode_small<gle>(poly->data, cm->bh_evals, cm->codeword, nv, shift) : encode_small<u64>(poly->data, cm->bh_evals, cm->codeword, nv, shift);
        else rc = poly->is_ext ? encode_tiled<gle>(poly->data, cm->bh_evals, cm->codeword, nv, shift, 0, 0) : encode_tiled<u64>(poly->data, cm->bh_evals, cm->codeword, nv, shift, 0, 0);
        if (rc) return rc;
    }
    if (root_pinned) {
        RootOut ro{root_pinned, nullptr, 0};
        if (int e = tree_build(cm->tree, {cm->codeword}, poly->is_ext, cm->cw_len, &ro)) return e;   // K9
        if (!cm->tree.root_published) DP_CUDA(cudaMemcpyAsync(root_pinned, cm->tree.root_dev, 32, cudaMemcpyDeviceToHost, c.stream));
    }
    *out = cm.release();
    return DP_OK;
}

int dp_pcs_commit(const dp_mle *poly, uint32_t full_log, dp_pcs_comm **out) {
    DP_REQUIRE_CTX();
    DP_CHECK(poly && out, DP_ERR_INVALID, "dp_pcs_commit: null argument");
    u64 *pin = nullptr;
    if (int e = dp_pinned_alloc((void **)&pin, 32)) return e;
    int rc = commit_enqueue(poly, full_log, out, pin);
    if (rc == DP_OK) { DP_CUDA(dp_stream_sync(dp_ctx().stream)); memcpy((*out)->root, pin, 32); }
    dp_pinned_free(pin);
    return rc;
}


// Basefold::commit of ONE polynomial sharded over `world` = 2^k ranks (one process per GPU).  Every rank passes the whole
// polynomial (resident on its GPU) and keeps only its contiguous slice of the bit-reversed evaluations, of the bit-reversed
// codeword and the Merkle subtree over that slice; (*out)'s root is the SUBTREE root until dp_pcs_comm_set_shard_roots has been
// given all ranks' subtree roots (one all-gather of 32 bytes per rank -- the only exchange of the commit).
int dp_pcs_commit_shard(const dp_mle *poly, uint32_t full_log, uint32_t rank, uint32_t world, dp_pcs_comm **out) {
    DP_REQUIRE_CTX();
    DP_CHECK(poly && out, DP_ERR_INVALID, "dp_pcs_commit_shard: null argument");
    u32 logG = 0; while ((1u << logG) < world) logG++;
    DP_CHECK(world >= 2 && (1u << logG) == world && rank < world, DP_ERR_INVALID, "dp_pcs_commit_shard: world must be a power of two >= 2 and rank < world");
    DP_CHECK(!mk_blake3(), DP_ERR_UNSUPPORTED, "dp_pcs_commit_shard: Poseidon2 trees only");
    const u32 nv = poly->num_vars();
    DP_CHECK(nv <= full_log, DP_ERR_INVALID, "PolynomialTooLarge");
    DP_CHECK(logG <= 6 && nv >= BF_BASECODE_LOG + 4 && nv > logG + 11, DP_ERR_INVALID, "dp_pcs_commit_shard: polynomial too small to shard over this many ranks");
    if (int e = bf_prepare()) return e;
    DpCtx &c = dp_ctx();
    CommPtr cm(new dp_pcs_comm());
    cm->num_vars = nv; cm->full_log = full_log; cm->is_base = !poly->is_ext; cm->shard_rank = rank; cm->shard_log = logG;
    const size_t esz = poly->is_ext ? 16 : 8;
    cm->cw_len = (poly->len << BF_RATE_LOG) >> logG;
    if (int e = dp_dev_alloc(&cm->bh_evals, esz * (poly->len >> logG))) return e;
    if (int e = dp_dev_alloc(&cm->codeword, esz * cm->cw_len)) return e;
    const u64 shift = coset_shift(full_log, nv);
    if (int e = poly->is_ext ? encode_tiled<gle>(poly->data, cm->bh_evals, cm->codeword, nv, shift, logG, rank)
                             : encode_tiled<u64>(poly->data, cm->bh_evals, cm->codeword, nv, shift, logG, rank)) return e;
    if (int e = tree_build(cm->tree, {cm->codeword}, poly->is_ext, cm->cw_len)) return e;
    if (int e = dp_d2h(cm->local_root, cm->tree.root_dev, 32, c.stream)) return e;
    memcpy(cm->root, cm->local_root, 32);
    *out = cm.release();
    return DP_OK;
}
// `roots`: world x 4 words, rank-major (the all-gathered subtree roots).  Builds the replicated top of the tree; afterwards
// dp_pcs_comm_info returns the root of the whole 2^(nv+1)-leaf tree (identical to dp_pcs_commit's).
int dp_pcs_comm_set_shard_roots(dp_pcs_comm *cm, const uint64_t *roots, uint64_t out_root[4]) {
    DP_REQUIRE_CTX();
    DP_CHECK(cm && roots && cm->shard_log > 0, DP_ERR_INVALID, "dp_pcs_comm_set_shard_roots: not a sharded commitment");
    DP_CHECK(!cm->top.level0, DP_ERR_STATE, "dp_pcs_comm_set_shard_roots: roots already set");
    for (int k = 0; k < 4; k++) DP_CHECK(gl_canon(roots[4 * cm->shard_rank + k]) == cm->local_root[k], DP_ERR_INVALID, "dp_pcs_comm_set_shard_roots: this rank's entry is not its own subtree root");
    if (int e = top_tree_build(cm->top, roots, cm->shard_log, cm->root)) return e;
    if (out_root) memcpy(out_root, cm->root, 32);
    return DP_OK;
}
int dp_pcs_comm_shard_info(const dp_pcs_comm *cm, uint32_t *rank, uint32_t *world, uint64_t local_root[4]) {
    DP_CHECK(cm, DP_ERR_INVALID, "dp_pcs_comm_shard_info: null");
    if (rank) *rank = cm->shard_rank;
    if (world) *world = 1u << cm->shard_log;
    if (local_root) memcpy(local_root, cm->shard_log ? cm->local_root : cm->root, 32);
    return DP_OK;
}

// Basefold::batch_commit (basefold.rs:356-452): n polynomials of the same size and field under ONE Merkle tree whose leaves
// are the batches of values (merkle_tree.rs:68-74,286-312).  Encoding is the per-polynomial pipeline; the leaf level hashes
// all polynomials' values at an index pair; the levels above are the ordinary tree.
int dp_pcs_batch_commit(const dp_mle *const *polys, uint32_t n, uint32_t full_log, dp_pcs_comm **out) {
    DP_REQUIRE_CTX();
    DP_CHECK(polys && out && n >= 1, DP_ERR_INVALID, "cannot batch commit to zero polynomials");      // basefold.rs:367-371
    DP_CHECK(n <= MK_BATCH_MAX, DP_ERR_UNSUPPORTED, "dp_pcs_batch_commit: at most 64 polynomials per batch");
    for (u32 i = 0; i < n; i++) DP_CHECK(polys[i] && polys[i]->len == polys[0]->len && polys[i]->is_ext == polys[0]->is_ext, DP_ERR_INVALID,
                                         "cannot batch commit to polynomials with different number of variables");   // :379-386
    if (mk_blake3()) DP_CHECK((polys[0]->is_ext ? 2 * n : n) <= MK_B3_BATCH_WORDS, DP_ERR_UNSUPPORTED, "dp_pcs_batch_commit: BLAKE3 batch leaves are limited to one 1024-byte chunk (128 base / 64 extension polynomials)");
    if (int e = bf_prepare()) return e;
    DpCtx &c = dp_ctx();
    CommPtr b(new dp_pcs_comm());
    b->num_vars = polys[0]->num_vars(); b->full_log = full_log; b->is_base = !polys[0]->is_ext;
    if (n == 1) {   // merkelize with one value vector is the plain tree (merkle_tree.rs:274-285): the batch holds an ordinary commitment
        dp_pcs_comm *part = nullptr;
        if (int e = dp_pcs_commit(polys[0], full_log, &part)) return e;
        b->parts.push_back(part); b->trivial = part->trivial; b->cw_len = part->cw_len; memcpy(b->root, part->root, 32);
        *out = b.release();
        return DP_OK;
    }
    std::vector<const void *> codewords;
    for (u32 i = 0; i < n; i++) {
        dp_pcs_comm *part = nullptr;
        if (int e = commit_enqueue(polys[i], full_log, &part, nullptr)) return e;
        b->parts.push_back(part); codewords.push_back(part->codeword);
    }
    b->trivial = b->parts[0]->trivial; b->cw_len = b->parts[0]->cw_len;
    if (int e = tree_build(b->tree, codewords, !b->is_base, b->cw_len)) return e;
    for (auto *part : b->parts) part->batch_tree = &b->tree;
    if (int e = dp_d2h(b->root, b->tree.root_dev, 32, c.stream)) return e;
    for (auto *part : b->parts) memcpy(part->root, b->root, 32);
    *out = b.release();
    return DP_OK;
}
// number of polynomials under a commitment (1 for dp_pcs_commit) and the i-th per-polynomial view of a batch commitment
// (borrowed: valid until the batch commitment is freed) -- the handles dp_pcs_open_begin / dp_pcs_open_query take
uint32_t dp_pcs_comm_num_polys(const dp_pcs_comm *cm) { return cm ? (cm->parts.empty() ? 1u : (uint32_t)cm->parts.size()) : 0u; }
int dp_pcs_comm_part(const dp_pcs_comm *cm, uint32_t i, const dp_pcs_comm **out) {
    DP_CHECK(cm && out && i < cm->parts.size(), DP_ERR_INVALID, "dp_pcs_comm_part: not a batch commitment or index out of range");
    *out = cm->parts[i];
    return DP_OK;
}

// Independent commitments (the reference commits witness columns from rayon workers: activation.rs:293,
// requant.rs:298/315, lookup/context.rs:677) are enqueued round-robin on a pool of streams so their
// latency chains (tree depth x Poseidon2 latency) overlap; one synchronisation at the end.
// A host thread's streams for independent commits, recycled across (short-lived) host threads: creating streams and events is slow
// and synchronising.  The thread's set goes back to g_free_sets when the thread exits.
struct StreamSet { std::vector<cudaStream_t> s; std::vector<cudaEvent_t> e; cudaEvent_t main_ev = nullptr; };
static std::vector<StreamSet> g_free_sets; static std::mutex g_sets_mu;
static thread_local struct ThreadStreamSet : StreamSet {
    ~ThreadStreamSet() { if (!s.empty()) { std::lock_guard<std::mutex> lk(g_sets_mu); g_free_sets.push_back(std::move(*this)); } }
} t_streams;
int dp_pcs_commit_many(const dp_mle *const *polys, uint32_t n, uint32_t full_log, dp_pcs_comm **out) {
    DP_REQUIRE_CTX();
    DP_CHECK(polys && out && n > 0, DP_ERR_INVALID, "dp_pcs_commit_many: null argument");
    for (u32 i = 0; i < n; i++) DP_CHECK(polys[i] != nullptr, DP_ERR_INVALID, "dp_pcs_commit_many: null polynomial");
    if (int e = bf_prepare()) return e;
    DpCtx &c = dp_ctx();
    // streams per host thread for independent commits: 8 are created; a lone proof uses all of them (its 38 witness trees are a pure
    // latency chain each), with many proofs in flight 4 are enough and keep the number of live streams near the 32 hardware queues
    static const u32 SMAX = 8;
    const u32 S = dp_wait_mode() == DP_WAIT_BLOCK ? 4u : 8u;
    StreamSet &ss = t_streams;
    if (ss.s.empty()) {
        std::lock_guard<std::mutex> lk(g_sets_mu);
        if (!g_free_sets.empty()) { ss = std::move(g_free_sets.back()); g_free_sets.pop_back(); }
    }
    if (ss.s.empty()) {
        ss.s.resize(SMAX); ss.e.resize(SMAX);
        for (u32 s = 0; s < SMAX; s++) { DP_CUDA(cudaStreamCreateWithFlags(&ss.s[s], cudaStreamNonBlocking)); DP_CUDA(cudaEventCreateWithFlags(&ss.e[s], cudaEventDisableTiming)); }
        DP_CUDA(cudaEventCreateWithFlags(&ss.main_ev, cudaEventDisableTiming));
    }
    u64 *pin = nullptr;
    if (int e = dp_pinned_alloc((void **)&pin, 32 * (size_t)n)) return e;
    cudaStream_t main = c.stream;
    DP_CUDA(cudaEventRecord(ss.main_ev, main));
    u32 used = n < S ? n : S;
    for (u32 s = 0; s < used; s++) DP_CUDA(cudaStreamWaitEvent(ss.s[s], ss.main_ev, 0));
    int rc = DP_OK;
    dp_arena_defer(true);    // temporaries released by one commit must not be handed to another stream's commit
    for (u32 i = 0; i < n && rc == DP_OK; i++) { c.stream = ss.s[i % S]; rc = commit_enqueue(polys[i], full_log, &out[i], pin + 4 * i); }
    c.stream = main;
    for (u32 s = 0; s < used; s++) { cudaEventRecord(ss.e[s], ss.s[s]); cudaStreamWaitEvent(main, ss.e[s], 0); }
    cudaError_t se = dp_stream_sync(main);
    dp_arena_defer(false);
    if (se != cudaSuccess) return dp_fail(DP_ERR_CUDA, std::string("dp_pcs_commit_many: ") + cudaGetErrorString(se));
    if (rc == DP_OK) for (u32 i = 0; i < n; i++) memcpy(out[i]->root, pin + 4 * i, 32);
    dp_pinned_free(pin);
    return rc;
}

int dp_pcs_comm_info(const dp_pcs_comm *cm, uint32_t *num_vars, int *is_base, int *is_trivial, uint64_t root[4]) {
    if (!cm) return dp_fail(DP_ERR_INVALID, "dp_pcs_comm_info: null");
    if (num_vars) *num_vars = cm->num_vars;
    if (is_base) *is_base = cm->is_base;
    if (is_trivial) *is_trivial = cm->trivial;
    if (root) memcpy(root, cm->root, 32);
    return DP_OK;
}
int dp_pcs_comm_codeword(const dp_pcs_comm *cm, dp_mle **view) {
    DP_REQUIRE_CTX();
    DP_CHECK(cm && view, DP_ERR_INVALID, "dp_pcs_comm_codeword: null");
    *view = dp_mle_view(cm->codeword, cm->cw_len, !cm->is_base);
    return DP_OK;
}
int dp_pcs_comm_bh_evals(const dp_pcs_comm *cm, dp_mle **view) {
    DP_REQUIRE_CTX();
    DP_CHECK(cm && view, DP_ERR_INVALID, "dp_pcs_comm_bh_evals: null");
    *view = dp_mle_view(cm->bh_evals, 1ULL << cm->num_vars, !cm->is_base);
    return DP_OK;
}
int dp_pcs_comm_free(dp_pcs_comm *cm) {
    if (!cm) return DP_OK;
    if (dp_ctx().ready) { tree_free(cm->tree); if (!cm->trivial) dp_dev_free(cm->codeword); dp_dev_free(cm->bh_evals); tree_free(cm->top); }
    for (auto *p : cm->parts) dp_pcs_comm_free(p);
    delete cm;
    return DP_OK;
}

// oracle0 of the opening of one commitment (or of this rank's slice of it): its codeword, in the extension field
static int open_oracle_from_codeword(dp_pcs_open *o, const dp_pcs_comm *cm) {
    DpCtx &c = dp_ctx();
    o->n0 = cm->cw_len;
    if (int e = dp_dev_alloc((void **)&o->oracle0, sizeof(gle) * o->n0)) return e;
    if (cm->is_base) DP_CUDA(dp_launch(k_lift, dp_grid_for(o->n0, 256, 8), 256, 0, c.stream, (const u64 *)cm->codeword, o->oracle0, o->n0));
    else DP_CUDA(cudaMemcpyAsync(o->oracle0, cm->codeword, sizeof(gle) * o->n0, cudaMemcpyDeviceToDevice, c.stream));
    return DP_OK;
}

// commit_phase / batch_commit_phase up to and including the first sumcheck message
int dp_pcs_open_begin(const dp_pcs_comm *const *comms, const uint64_t *coeffs, uint32_t n_comms, const uint64_t *point, uint32_t num_vars,
                      dp_pcs_open **out, uint64_t first_msg[6]) {
    DP_REQUIRE_CTX();
    DP_CHECK(comms && n_comms >= 1 && point && out && first_msg, DP_ERR_INVALID, "dp_pcs_open_begin: null argument");
    if (int e = bf_prepare()) return e;
    DpCtx &c = dp_ctx();
    const dp_pcs_comm *cm = comms[0];
    const u32 full_log = cm ? cm->full_log : 0;
    for (u32 i = 0; i < n_comms; i++) {
        DP_CHECK(comms[i] && !comms[i]->trivial, DP_ERR_INVALID, "dp_pcs_open_begin: trivial commitment (open it on the host)");   // basefold.rs:481-483, 562-565
        DP_CHECK(comms[i]->num_vars <= num_vars && comms[i]->full_log == full_log, DP_ERR_INVALID, "dp_pcs_open_begin: commitment larger than the opening");
    }
    DP_CHECK(num_vars > BF_BASECODE_LOG, DP_ERR_INVALID, "minimum number of variables must be greater than basecode_msg_size_log");
    for (u32 i = 0; i < n_comms; i++) DP_CHECK(comms[i]->shard_log == 0 || (n_comms == 1 && !coeffs), DP_ERR_UNSUPPORTED, "dp_pcs_open_begin: a sharded commitment is opened alone");
    if (cm->shard_log) DP_CHECK(cm->num_vars == num_vars && cm->top.level0, DP_ERR_STATE, "dp_pcs_open_begin: sharded commitment needs num_vars variables and its shard roots set");
    else if (!coeffs) DP_CHECK(n_comms == 1 && cm->num_vars == num_vars, DP_ERR_INVALID, "dp_pcs_open_begin: single open needs one commitment of num_vars variables");

    OpenPtr o(new dp_pcs_open());
    o->num_vars = num_vars; o->batch = coeffs != nullptr; o->full_log = full_log;
    o->num_rounds = num_vars - BF_BASECODE_LOG;
    o->comms.assign(comms, comms + n_comms);
    if (coeffs) for (u32 i = 0; i < n_comms; i++) o->coeffs.push_back(e_from_host(coeffs + 2 * i));
    // eq = bitrev(build_eq_x_r_vec(point)) == build_eq_x_r_vec(reversed point)  (commit_phase.rs:61-64)
    std::vector<uint64_t> rp(2 * num_vars);
    for (u32 i = 0; i < num_vars; i++) { rp[2 * i] = point[2 * (num_vars - 1 - i)]; rp[2 * i + 1] = point[2 * (num_vars - 1 - i) + 1]; }
    u32 sc_vars = num_vars;
    if (cm->shard_log) {
        // Sharded opening: everything below works on this rank's contiguous slices; the messages it returns are PARTIAL sums (the
        // coefficient form is linear in the evaluations), the roots SUBTREE roots -- the caller all-gathers and adds / combines them.
        const u32 logG = cm->shard_log, nvl = num_vars - logG;
        const u64 Ml = 1ULL << nvl;
        o->shard_rank = cm->shard_rank; o->shard_log = logG;
        if (int e = open_oracle_from_codeword(o.get(), cm)) return e;
        o->evals = dp_mle_view(cm->bh_evals, Ml, !cm->is_base);
        // eq slice: the table over the low nvl variables of the reversed point, times the eq factor of this rank's top bits
        dp_mle *eq_low = nullptr;
        if (int e = dp_eq_build(rp.data(), nvl, &eq_low)) return e;
        MlePtr eq_low_owner(eq_low);
        gle scal = e_one();
        for (u32 j = 0; j < logG; j++) {
            gle x = e_from_host(&rp[2 * (nvl + j)]);
            scal = e_mul(scal, ((cm->shard_rank >> j) & 1) ? x : e_sub(e_one(), x));
        }
        MlePtr eq;
        if (int e = dp_mle_alloc(Ml, true, eq)) return e;
        o->eq = eq.release();
        if (int e = lincomb_bcast((gle *)o->eq->data, nullptr, {LcTerm{eq_low->data, scal, true, 0}}, Ml)) return e;
        sc_vars = nvl;
    } else {
        const u64 N = 1ULL << (num_vars + BF_RATE_LOG), M = 1ULL << num_vars;
        if (!o->batch) {
            if (int e = open_oracle_from_codeword(o.get(), cm)) return e;
            o->evals = dp_mle_view(cm->bh_evals, M, !cm->is_base);     // running_evals = bh_evals (commit_phase.rs:50)
        } else {
            // running_oracle = sum of coeff * codeword over the full-size commitments (commit_phase.rs:205-223)
            o->n0 = N;
            if (int e = dp_dev_alloc((void **)&o->oracle0, sizeof(gle) * N)) return e;
            std::vector<LcTerm> terms;
            for (u32 i = 0; i < n_comms; i++) if (comms[i]->cw_len == N) terms.push_back({comms[i]->codeword, o->coeffs[i], !comms[i]->is_base, 0});
            if (int e = lincomb_bcast(o->oracle0, nullptr, terms, N)) return e;
            // sum_of_all_evals_for_sumcheck: smaller polynomials are broadcast over chunks (commit_phase.rs:225-236)
            if (int e = dp_dev_alloc((void **)&o->scratch_sum_evals, sizeof(gle) * M)) return e;
            terms.clear();
            for (u32 i = 0; i < n_comms; i++) terms.push_back({comms[i]->bh_evals, o->coeffs[i], !comms[i]->is_base, num_vars - comms[i]->num_vars});
            if (int e = lincomb_bcast(o->scratch_sum_evals, nullptr, terms, M)) return e;
            o->evals = dp_mle_view(o->scratch_sum_evals, M, true);
        }
        if (int e = dp_eq_build(rp.data(), num_vars, &o->eq)) return e;
    }
    // the Basefold-internal sumcheck (basefold/sumcheck.rs) is a degree-2 LSB-first sumcheck of eq * evals on
    // the bit-reversed tables; its coefficient-form message is recovered from p(0), p(1), p(2)
    dp_mle *ms[2] = {o->eq, o->evals};
    dp_sc_product pr; memset(&pr, 0, sizeof pr); pr.coef[0] = 1; pr.n_idx = 2; pr.idx[0] = 0; pr.idx[1] = 1;
    if (int e = dp_sc_create(ms, 2, &pr, 1, sc_vars, 2, &o->sc)) return e;
    uint64_t ev3[6];
    if (int e = dp_sc_round(o->sc, nullptr, ev3)) return e;
    msg_to_coeffs(ev3, first_msg);
    *out = o.release();
    return DP_OK;
}

// One commit-phase round (commit_phase.rs:85-171 / :253-352): fold the oracle by `challenge`; unless this is
// the last round return the next sumcheck message and the root of the folded oracle's tree.
int dp_pcs_open_round(dp_pcs_open *o, const uint64_t challenge[2], uint64_t next_msg[6], uint64_t root[4], int *is_last) {
    DP_REQUIRE_CTX();
    DP_CHECK(o && challenge && is_last, DP_ERR_INVALID, "dp_pcs_open_round: null argument");
    DP_CHECK(o->round < o->num_rounds, DP_ERR_STATE, "dp_pcs_open_round: commit phase already finished");
    DpCtx &c = dp_ctx();
    gle r = e_from_host(challenge);
    u32 i = o->round;
    if (i > 0 && o->batch) {
        // merge the commitments whose codeword size matches the running oracle (commit_phase.rs:271-282); the
        // tree built last round keeps the pre-addition copy
        u64 len = o->n0; bool any = false;
        for (auto cm : o->comms) if (cm->cw_len == len) any = true;
        if (any) {
            gle *merged = nullptr;
            if (int e = dp_dev_alloc((void **)&merged, sizeof(gle) * len)) return e;
            std::vector<LcTerm> terms;
            for (size_t k = 0; k < o->comms.size(); k++) if (o->comms[k]->cw_len == len) terms.push_back({o->comms[k]->codeword, o->coeffs[k], !o->comms[k]->is_base, 0});
            if (int e = lincomb_bcast(merged, o->oracle0, terms, len)) return e;
            o->oracle0 = merged; o->oracle0_owned = true;   // the previous buffer stays owned by rounds.back()
        }
    }
    // K10: fold the running oracle
    u64 len = o->n0; u32 level = 0; while ((2ULL << level) < (len << o->shard_log)) level++;   // log2(global len) - 1
    gle *folded = nullptr;
    if (int e = dp_dev_alloc((void **)&folded, sizeof(gle) * (len >> 1))) return e;
    {
        u32 gexp = o->full_log + BF_RATE_LOG - level - 1;
        u64 gamma = 7; for (u32 k = 0; k < gexp; k++) gamma = gl_sqr(gamma);
        u64 nhgi = gl_neg(gl_mul(gl_inv(gamma), 0x7FFFFFFF80000001ULL));   // -(1/gamma_lvl)/2
        DpProfScope p("k_fri_fold", len * 16 + (len >> 1) * 16);
        DP_CUDA(dp_launch(k_fri_fold, dp_grid_for(len >> 1, 256, 8), 256, 0, c.stream, o->oracle0, folded, level, len >> 1, (u64)o->shard_rank * (len >> 1), r, gamma,
                          nhgi, root_tab()));
    }
    // the oracle just consumed is either round i-1's tree leaves (kept) or the initial / merged buffer (freed)
    bool consumed_is_tree_leaves = !o->rounds.empty() && o->rounds.back().oracle == o->oracle0;
    if (!consumed_is_tree_leaves) dp_dev_free(o->oracle0);
    o->oracle0 = folded; o->n0 = len >> 1;
    uint64_t ch[2] = {r.c0, r.c1};
    uint64_t ev3[6];
    if (i + 1 < o->num_rounds) {
        if (int e = dp_sc_round(o->sc, ch, ev3)) return e;       // sum_check_challenge_round
        msg_to_coeffs(ev3, next_msg);
        OpenRound rd; rd.oracle = folded;
        if (!o->h_root) { void *hp = nullptr; if (int e = dp_pinned_alloc(&hp, 128)) return e; o->h_root = (u64 *)hp; o->h_root[8] = 0; o->root_seq = 0; }
        RootOut ro{o->h_root, o->h_root + 8, ++o->root_seq};
        if (int e = tree_build(rd.tree, {folded}, true, len >> 1, &ro)) return e;   // compute_inner_ext
        if (rd.tree.root_published) {   // the tree's last launch stores the root and then the sequence number in mapped memory
            if (int e = dp_await(o->h_root + 8, o->root_seq, 30.0, "dp_pcs_open_round: tree kernel finished without publishing its root")) return e;
            memcpy(root, o->h_root, 32);
        } else if (int e = dp_d2h(root, rd.tree.root_dev, 32, c.stream)) return e;
        o->rounds.push_back(rd);
        *is_last = 0;
    } else {
        // sum_check_last_round: fold once more, then un-bit-reverse the 2^7 evaluations (commit_phase.rs:132-146)
        if (int e = dp_sc_round(o->sc, ch, ev3)) return e;       // fold (the message it also computes is unused)
        dp_mle *view = nullptr;
        if (int e = dp_sc_current_mle(o->sc, 1, &view)) return e;
        DP_CHECK(view->len == ((1ULL << BF_BASECODE_LOG) >> o->shard_log) && view->is_ext, DP_ERR_STATE, "dp_pcs_open_round: unexpected final message size");
        gle tmp[1 << BF_BASECODE_LOG];
        if (int e = dp_d2h(tmp, view->data, sizeof(gle) * view->len, c.stream)) return e;
        dp_mle_free(view);
        if (o->shard_log) {   // this rank's slice of the bit-reversed final message: the caller concatenates the ranks' slices and un-bit-reverses
            for (u32 k = 0; k < ((1u << BF_BASECODE_LOG) >> o->shard_log); k++) o->final_msg[k] = tmp[k];
        } else
        for (u32 k = 0; k < (1u << BF_BASECODE_LOG); k++) { u32 j = 0; for (u32 b = 0; b < BF_BASECODE_LOG; b++) if (k >> b & 1) j |= 1u << (BF_BASECODE_LOG - 1 - b); o->final_msg[j] = tmp[k]; }
        o->have_final = true;
        *is_last = 1;
    }
    o->round++;
    return DP_OK;
}

// Sharded openings: after a round that returned a subtree root, the caller all-gathers the ranks' subtree roots and hands them back;
// this builds the replicated top of that round's tree (needed for the query paths) and returns the root of the whole oracle tree.
int dp_pcs_open_set_shard_roots(dp_pcs_open *o, const uint64_t *roots, uint64_t out_root[4]) {
    DP_REQUIRE_CTX();
    DP_CHECK(o && roots && out_root && o->shard_log > 0 && !o->rounds.empty(), DP_ERR_INVALID, "dp_pcs_open_set_shard_roots: not a sharded opening with a pending round");
    OpenRound &rd = o->rounds.back();
    DP_CHECK(!rd.top.level0, DP_ERR_STATE, "dp_pcs_open_set_shard_roots: roots of this round already set");
    return top_tree_build(rd.top, roots, o->shard_log, out_root);
}

// (sharded opening: this rank's (2^7 >> log world) entries of the BIT-REVERSED final message -- concatenate by rank, then un-bit-reverse)
int dp_pcs_open_final_message(dp_pcs_open *o, uint64_t *out) {
    DP_CHECK(o && out, DP_ERR_INVALID, "dp_pcs_open_final_message: null argument");
    DP_CHECK(o->have_final, DP_ERR_STATE, "dp_pcs_open_final_message: commit phase not finished");
    for (u32 k = 0; k < ((1u << BF_BASECODE_LOG) >> o->shard_log); k++) { out[2 * k] = o->final_msg[k].c0; out[2 * k + 1] = o->final_msg[k].c1; }
    return DP_OK;
}

// the trees a query opens, in the order of dp_pcs_open_query's output: every commitment's, then every round oracle's
static std::vector<MkPath> query_paths(const dp_pcs_open *o) {
    std::vector<MkPath> paths;   // a commitment of nv variables is queried at x >> (num_vars - nv)
    for (auto cm : o->comms) paths.push_back({cm->batch_tree ? cm->batch_tree : &cm->tree, cm->codeword, o->num_vars - cm->num_vars, &cm->top});
    for (size_t i = 0; i < o->rounds.size(); i++) paths.push_back({&o->rounds[i].tree, o->rounds[i].oracle, (u32)i + 1, &o->rounds[i].top});
    return paths;
}

// u64 words one query occupies in dp_pcs_open_query's output
uint64_t dp_pcs_open_query_words(const dp_pcs_open *o) { return o ? mk_query_words(query_paths(o), o->shard_log) : 0; }

// K13 (query_phase.rs:373-474): for every x index, for every commitment then every round oracle:
// [p0.c0 p0.c1 p1.c0 p1.c1] + Merkle path without leaf sibling or root (merkle_tree.rs:139-152).
int dp_pcs_open_query(dp_pcs_open *o, const uint64_t *x_indices, uint32_t n, uint64_t *out) {
    DP_REQUIRE_CTX();
    DP_CHECK(o && x_indices && out && n > 0, DP_ERR_INVALID, "dp_pcs_open_query: null argument");
    DP_CHECK(o->have_final, DP_ERR_STATE, "dp_pcs_open_query: commit phase not finished");
    if (o->shard_log) for (auto &rd : o->rounds) DP_CHECK(rd.top.level0 != nullptr, DP_ERR_STATE, "dp_pcs_open_query: a round's shard roots were never set");
    return mk_query_gather(query_paths(o), o->shard_log, o->shard_rank, x_indices, n, out);
}

int dp_pcs_open_free(dp_pcs_open *o) {
    if (!o) return DP_OK;
    if (dp_ctx().ready) {
        if (o->sc) dp_sc_destroy(o->sc);
        bool oracle_in_rounds = false;
        for (auto &rd : o->rounds) { if (rd.oracle == o->oracle0) oracle_in_rounds = true; tree_free(rd.tree); dp_dev_free(rd.oracle); tree_free(rd.top); }
        if (!oracle_in_rounds) dp_dev_free(o->oracle0);
        dp_dev_free(o->scratch_sum_evals);
    }
    if (o->h_root && o->h_root[8] != o->root_seq && dp_ctx().ready) dp_stream_sync(dp_ctx().stream);   // a tree kernel still owns the pinned block
    dp_pinned_free(o->h_root);
    if (o->eq) dp_mle_free(o->eq);
    if (o->evals) dp_mle_free(o->evals);
    delete o;
    return DP_OK;
}

}  // extern "C"
