// Basefold multilinear PCS on device: commit (K7 hypercube interpolation, K8 RS/NTT encode, K9 Poseidon2
// Merkle), open / batch_open commit phase (K10 FRI fold, K11 coefficient-form sumcheck via the sumcheck
// engine, K12 batch prelude) and query gathering (K13).
// Reference: mpcs/src/basefold.rs:86-154,304-354,466-770; basefold/{commit_phase.rs,sumcheck.rs,
// encoding/rs.rs,query_phase.rs:31-138,373-534}; util/{merkle_tree.rs,hash.rs,arithmetic.rs:120-132,
// arithmetic/hypercube.rs}.
//
// Data layout in HBM (per commitment of a 2^nu polynomial): bh_evals = bit-reversed evaluations (8 or
// 16 B/elt), codeword = bit-reversed RS codeword of 2^(nu+1) elements, digests = Merkle levels >= 1
// (4 x u64 each; level 0 of the reference is a zero-padded copy of the leaf pair -- hash_or_noop of <= 4
// elements, poseidon_hash.rs:22-28 -- so it is recomputed from the leaves on demand, never stored).
// Everything stays resident until the opening: roots and round messages are the only D2H traffic.
//
// Linear-algebra shortcuts (exact arithmetic, identical field elements):
//  * interpolate_over_boolean_hypercube commutes with the bit-reversal permutation, so the coefficient
//    vector the reference encodes, bitrev(interp(evals)), is interp(bh_evals): one permutation serves both.
//  * a decimation-in-frequency NTT of the natural-order input yields the spectrum in bit-reversed order,
//    which IS the stored codeword (basefold.rs:151 bit-reverses the DIT output) -- no final permutation.
//  * the zero-padded upper half makes the first DIF level a pure copy-and-scale (k_expand).
#include "common.cuh"
#include "powtab.cuh"
#include "poseidon2.cuh"
#include "blake3.cuh"
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
struct BfGlobals { std::atomic<const u64 *> root_tab{nullptr}; std::atomic<bool> p2_ready{false}; };
static BfGlobals g_bf;          // process-wide, read-only once built (shared by every host thread's context)
static std::mutex g_bf_mu;
static int bf_prepare() {
    if (g_bf.p2_ready.load() && g_bf.root_tab.load()) return DP_OK;
    std::lock_guard<std::mutex> lk(g_bf_mu);
    if (!g_bf.p2_ready.load()) {
        DP_CUDA(p2_upload_constants((const u64 *)&DP_P2_EXT_RC[0][0][0], (const u64 *)DP_P2_INT_RC, (const u64 *)DP_P2_DIAG));
        g_bf.p2_ready.store(true);
    }
    if (!g_bf.root_tab.load()) {
        const u64 *tab = nullptr;
        if (int e = pow_table_build(GL_ROOT32, &tab)) return e;
        g_bf.root_tab.store(tab);
    }
    return DP_OK;
}
static PowTab root_tab() { return powtab_at(g_bf.root_tab.load()); }
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

// ---- K9 Merkle ----
template <bool EXT> __device__ __forceinline__ void leaf_pair_digest(const void *leaves, u64 pair, u64 d[4]) {
    if (EXT) { const gle *l = (const gle *)leaves + 2 * pair; gle a = ld_e(l), b = ld_e(l + 1); d[0] = a.c0; d[1] = a.c1; d[2] = b.c0; d[3] = b.c1; }
    else { ulonglong2 v = ld_b2((const u64 *)leaves + 2 * pair); d[0] = v.x; d[1] = v.y; d[2] = 0; d[3] = 0; }
}
// the two children of hash i on the first level of a single-polynomial tree: leaf pairs 2i and 2i + 1
template <bool EXT> __device__ __forceinline__ void mk_leaf_children(const void *leaves, u64 i, u64 x[4], u64 y[4]) {
    leaf_pair_digest<EXT>(leaves, 2 * i, x); leaf_pair_digest<EXT>(leaves, 2 * i + 1, y);
}
// the two children of a hash on a higher level: the 8 digest words at `in`
__device__ __forceinline__ void mk_node_children(const u64 *in, u64 x[4], u64 y[4]) {
    ulonglong2 a = *reinterpret_cast<const ulonglong2 *>(in), b = *reinterpret_cast<const ulonglong2 *>(in + 2);
    ulonglong2 c = *reinterpret_cast<const ulonglong2 *>(in + 4), d = *reinterpret_cast<const ulonglong2 *>(in + 6);
    x[0] = a.x; x[1] = a.y; x[2] = b.x; x[3] = b.y; y[0] = c.x; y[1] = c.y; y[2] = d.x; y[3] = d.y;
}
__device__ __forceinline__ void mk_store(u64 *out, u64 i, const u64 d[4]) {
    *reinterpret_cast<ulonglong2 *>(out + 4 * i) = make_ulonglong2(d[0], d[1]);
    *reinterpret_cast<ulonglong2 *>(out + 4 * i + 2) = make_ulonglong2(d[2], d[3]);
}
template <bool EXT>
__global__ void k_merkle_l1(const void *__restrict__ leaves, u64 n_out, u64 *__restrict__ out) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    for (; i < n_out; i += stride) {
        u64 x[4], y[4], o[4];
        mk_leaf_children<EXT>(leaves, i, x, y);
        p2_compress(x, y, o);
        mk_store(out, i, o);
    }
}
__global__ void k_merkle_up(const u64 *__restrict__ in, u64 n_out, u64 *__restrict__ out) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    for (; i < n_out; i += stride) {
        u64 x[4], y[4], o[4];
        mk_node_children(in + 8 * i, x, y);
        p2_compress(x, y, o);
        mk_store(out, i, o);
    }
}
template <bool EXT, bool FROM_LEAVES>
__global__ void __launch_bounds__(64) k_merkle_mid(const void *__restrict__ src, u64 n_out, u64 *__restrict__ out) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_out) return;
    u64 x[4], y[4], o[4];
    if (FROM_LEAVES) mk_leaf_children<EXT>(src, i, x, y);
    else mk_node_children((const u64 *)src + 8 * i, x, y);
    p2_compress_lat(x, y, o);
    mk_store(out, i, o);
}
// 8 lanes per hash (poseidon2.cuh): word w of the leaf-pair digest `pair`
template <bool EXT> __device__ __forceinline__ u64 leaf_pair_word(const void *leaves, u64 pair, int w) {
    if (EXT) return ((const u64 *)leaves)[4 * pair + w];
    return w < 2 ? ((const u64 *)leaves)[2 * pair + w] : 0ULL;
}
// Every remaining level of a tree whose current level has <= MK_SMALL hashes, in ONE launch.  Each block owns MK_SUB hashes of the
// first level and walks that subtree up to its root with a block barrier per level; the last block to finish (ticket) folds the
// <= 8 subtree roots.  A level with >= 64 hashes per block runs one THREAD per hash (latency-optimised permutation): the same
// ~40 us per level as a single-warp chain costs anyway, at 1/5 of the issue slots of the lane-parallel form -- with dozens of proofs
// in flight these small trees were as much GPU work as all the wide Merkle levels together (8 lanes x ~4.5 k instructions per
// permutation against 12.8 k for one thread).  Levels with <= 32 hashes per block use 8 lanes per hash (shorter dependent chain,
// ~27 us per level); 88 % of a 2048-hash tree's permutations are in the thread-per-hash levels.
struct LvlOff { u64 off[36]; };
static constexpr u32 MK_SUB = 256;
static constexpr u64 MK_SMALL = 2048;
// `rt`: optional hand-over of the root to the host with the kernel's own stores (mapped pinned memory): root words, then a system
// fence, then the sequence number the host waits for -- no D2H copy node and no separate signal launch per tree.
struct RootOut { u64 *root_host; u64 *flag; u64 seq; };
__device__ __forceinline__ void mk_publish_root(const RootOut &rt, const u64 *root_dev) {   // one thread, after the barrier that follows the root's stores
    if (!rt.root_host) return;
#pragma unroll
    for (int k = 0; k < 4; k++) rt.root_host[k] = __ldcg(root_dev + k);
    if (rt.flag) dp_publish(rt.flag, rt.seq);
}
template <bool EXT, bool FROM_LEAVES>
__global__ void __launch_bounds__(256) k_merkle_small(const void *src, u32 first_level, u32 lg, u64 nl_first, u64 *levels, LvlOff lo, u32 *ticket, RootOut rt, u32 sub_max, u32 tph_min) {
    // (sub_max, tph_min) = (256, 64) with many proofs in flight (see above); (32, never) for a single proof: 64 blocks x one 8-lane pass
    // per level is the shortest chain (~20 us per level against ~40 us for a thread per hash) and nothing else wants the issue slots
    const int lane8 = threadIdx.x & 7; const u32 grp = threadIdx.x >> 3;
    const u32 sub = (u32)(nl_first < sub_max ? nl_first : sub_max);
    u32 l = first_level;
    for (u32 k = 0; (sub >> k) >= 1 && l < lg; k++, l++) {
        const u32 cnt = sub >> k; const u64 base = (u64)blockIdx.x * cnt;
        u64 *out = levels + 4 * lo.off[l];
        const u64 *prev = k == 0 ? (const u64 *)src : levels + 4 * lo.off[l - 1];
        if (cnt >= tph_min) {                              // one thread per hash
            if (threadIdx.x < cnt) {
                const u64 i = base + threadIdx.x;
                u64 x[4], y[4], o[4];
                if (k == 0 && FROM_LEAVES) mk_leaf_children<EXT>(src, i, x, y);
                else {   // the 8 words inline: through mk_node_children this kernel's instruction order changes
                    const u64 *in = prev + 8 * i;
                    ulonglong2 a = *reinterpret_cast<const ulonglong2 *>(in), b = *reinterpret_cast<const ulonglong2 *>(in + 2);
                    ulonglong2 c = *reinterpret_cast<const ulonglong2 *>(in + 4), d = *reinterpret_cast<const ulonglong2 *>(in + 6);
                    x[0] = a.x; x[1] = a.y; x[2] = b.x; x[3] = b.y; y[0] = c.x; y[1] = c.y; y[2] = d.x; y[3] = d.y;
                }
                p2_compress_lat(x, y, o);
                mk_store(out, i, o);
            }
        } else for (u32 b = 0; b < cnt; b += 32) {         // 8 lanes per hash, 32 hashes per pass
            if (b + (grp & ~3u) >= cnt) continue;          // warp-uniform (a warp holds 4 lane groups): idle warps skip the permutations
            const bool live = b + grp < cnt; const u64 i = base + b + grp;
            u64 xw = 0, yw = 0;
            if (live && lane8 < 4) {
                if (k == 0 && FROM_LEAVES) { xw = leaf_pair_word<EXT>(src, 2 * i, lane8); yw = leaf_pair_word<EXT>(src, 2 * i + 1, lane8); }
                else { const u64 *in = prev + 8 * i; xw = in[lane8]; yw = in[4 + lane8]; }
            }
            const u64 sres = p2x8_compress(xw, yw, lane8);
            if (live && lane8 < 4) out[4 * i + (3 - lane8)] = sres;
        }
        __syncthreads();
    }
    if (gridDim.x == 1) { if (threadIdx.x == 0) mk_publish_root(rt, levels + 4 * lo.off[lg - 1]); return; }
    __shared__ bool last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) { const u32 t = atomicAdd(ticket, 1u); last = (t == gridDim.x - 1); if (last) *ticket = 0; }
    __syncthreads();
    if (!last) return;
    __threadfence();
    for (u32 cnt = gridDim.x >> 1; cnt >= 1 && l < lg; cnt >>= 1, l++) {
        u64 *out = levels + 4 * lo.off[l];
        const u64 *in0 = levels + 4 * lo.off[l - 1];
        for (u32 b = 0; b < cnt; b += 32) {
            if (b + (grp & ~3u) >= cnt) continue;
            const u32 j = b + grp; const bool live = j < cnt;
            u64 xw = 0, yw = 0;
            if (live && lane8 < 4) { xw = __ldcg(in0 + 8 * (u64)j + lane8); yw = __ldcg(in0 + 8 * (u64)j + 4 + lane8); }   // written by other blocks / an earlier pass
            const u64 sres = p2x8_compress(xw, yw, lane8);
            if (live && lane8 < 4) out[4 * (u64)j + (3 - lane8)] = sres;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) mk_publish_root(rt, levels + 4 * lo.off[lg - 1]);
}
// process-wide pool of zeroed ticket counters (each k_merkle_small launch takes the next one and leaves it zero again)
static std::atomic<u32 *> g_mk_tickets{nullptr}; static std::atomic<u32> g_mk_next{0}; static constexpr u32 MK_TICKETS = 4096;
static int mk_ticket(u32 **out) {
    u32 *tickets = g_mk_tickets.load();
    if (!tickets) {
        std::lock_guard<std::mutex> lk(g_bf_mu);
        tickets = g_mk_tickets.load();
        if (!tickets) {
            DP_CUDA(cudaMalloc((void **)&tickets, sizeof(u32) * MK_TICKETS));
            DP_CUDA(cudaMemset(tickets, 0, sizeof(u32) * MK_TICKETS));
            g_mk_tickets.store(tickets);
        }
    }
    *out = tickets + (g_mk_next.fetch_add(1, std::memory_order_relaxed) % MK_TICKETS);
    return DP_OK;
}

// batch_commit leaf level (merkle_tree.rs:286-312, util/hash.rs:30-41): digest_i = compress(hash(values of all m polynomials at
// index 2i), hash(... at 2i+1)), hash = hash_or_noop over the base-field limbs
struct BatchPtrs { const void *p[64]; };
template <bool EXT>
__global__ void k_merkle_batch_l0(BatchPtrs bp, u32 m, u64 n_out, u64 *__restrict__ out) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_out) return;
    u64 x[4], y[4], o[4];
    const int n = EXT ? 2 * (int)m : (int)m;
    auto ga = [&](int k) -> u64 { return EXT ? ((const u64 *)bp.p[k >> 1])[2 * (2 * i) + (k & 1)] : ((const u64 *)bp.p[k])[2 * i]; };
    auto gb = [&](int k) -> u64 { return EXT ? ((const u64 *)bp.p[k >> 1])[2 * (2 * i + 1) + (k & 1)] : ((const u64 *)bp.p[k])[2 * i + 1]; };
    p2_hash_or_noop(ga, n, x); p2_hash_or_noop(gb, n, y);
    p2_compress(x, y, o);
    mk_store(out, i, o);
}
template <bool EXT> __global__ void k_leafpair_root(const void *leaves, u64 *out) { u64 d[4]; leaf_pair_digest<EXT>(leaves, 0, d); for (int i = 0; i < 4; i++) out[i] = d[i]; }

// ---- the `blake` MerkleHasher (mpcs/src/util/hash.rs:79-95): leaf pair -> BLAKE3(LE bytes), inner node -> BLAKE3(left || right) ----
// Selected process-wide with dp_set_merkle_hasher (the reference selects at compile time: feature `blake`, mpcs/src/lib.rs:339-342).
static std::atomic<int> g_hasher{0};          // 0 Poseidon2 (default), 1 BLAKE3
static inline bool blake_on() { return g_hasher.load(std::memory_order_relaxed) == 1; }
template <bool EXT> __device__ __forceinline__ void b3_leaf_pair(const void *leaves, u64 pair, u64 d[4]) {
    u64 w[4];
    if (EXT) { const gle *l = (const gle *)leaves + 2 * pair; gle a = ld_e(l), b = ld_e(l + 1); w[0] = a.c0; w[1] = a.c1; w[2] = b.c0; w[3] = b.c1; b3::hash_words(w, 4, d); }
    else { ulonglong2 v = ld_b2((const u64 *)leaves + 2 * pair); w[0] = v.x; w[1] = v.y; b3::hash_words(w, 2, d); }
}
// level 0 (hash_two_leaves) of a single-polynomial tree: one digest per leaf pair.  Stored (unlike the Poseidon variant, whose
// level 0 is a zero-padded copy of the pair and is recomputed on demand).
template <bool EXT> __global__ void k_b3_leaves(const void *__restrict__ leaves, u64 n_out, u64 *__restrict__ out) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_out) return;
    u64 d[4]; b3_leaf_pair<EXT>(leaves, i, d);
    mk_store(out, i, d);
}
__global__ void k_b3_up(const u64 *__restrict__ in, u64 n_out, u64 *__restrict__ out) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_out) return;
    u64 w[8];
#pragma unroll
    for (int k = 0; k < 8; k += 2) { ulonglong2 v = *reinterpret_cast<const ulonglong2 *>(in + 8 * i + k); w[k] = v.x; w[k + 1] = v.y; }
    u64 d[4]; b3::hash_words(w, 8, d);
    mk_store(out, i, d);
}
// every remaining level (<= 1024 hashes at the first one) in one single-block launch
__global__ void __launch_bounds__(1024) k_b3_tail(const u64 *__restrict__ in0, u32 first_level, u32 lg, u64 nl_first, u64 *levels, LvlOff lo) {
    const u64 *in = in0; u64 nl = nl_first;
    for (u32 l = first_level; l < lg; l++, nl >>= 1) {
        u64 *out = levels + 4 * lo.off[l];
        if (threadIdx.x < nl) {
            u64 w[8];
#pragma unroll
            for (int k = 0; k < 8; k++) w[k] = in[8 * (u64)threadIdx.x + k];
            u64 d[4]; b3::hash_words(w, 8, d);
#pragma unroll
            for (int k = 0; k < 4; k++) out[4 * (u64)threadIdx.x + k] = d[k];
        }
        __syncthreads();
        in = out;
    }
}

// batch_commit leaf level under BLAKE3: digest_i = H( H(values of all polynomials at 2i) || H(... at 2i+1) )  (hash_two_leaves_batch_*)
template <bool EXT>
__global__ void k_b3_batch_l0(BatchPtrs bp, u32 m, u64 n_out, u64 *__restrict__ out) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_out) return;
    const int n = EXT ? 2 * (int)m : (int)m;
    auto ga = [&](int k) -> u64 { return EXT ? ((const u64 *)bp.p[k >> 1])[2 * (2 * i) + (k & 1)] : ((const u64 *)bp.p[k])[2 * i]; };
    auto gb = [&](int k) -> u64 { return EXT ? ((const u64 *)bp.p[k >> 1])[2 * (2 * i + 1) + (k & 1)] : ((const u64 *)bp.p[k])[2 * i + 1]; };
    u64 w[8], d[4];
    b3::hash_stream(ga, n, w); b3::hash_stream(gb, n, w + 4);
    b3::hash_words(w, 8, d);
#pragma unroll
    for (int k = 0; k < 4; k++) out[4 * i + k] = d[k];
}

// A Merkle tree over `n` leaves living in HBM: levels >= 1 packed back to back.
struct DevTree {
    const void *leaves = nullptr; bool ext = false; u64 n = 0; u32 lg = 0;
    u64 *levels = nullptr;            // level l (1-based) at offset lvl_off[l] (in digests)
    std::vector<u64> lvl_off;         // lvl_off[l] for l = 1..lg-1
    u64 *root_dev = nullptr;          // 4 limbs
    const u64 *level0 = nullptr;      // batch trees only: stored digests of the leaf pairs (single-polynomial trees recompute them)
    bool own_levels = true;           // false for the per-polynomial views of a batch commitment
    bool own_level0 = false;          // BLAKE3 trees of one polynomial store their leaf-pair digests (Poseidon2 recomputes them: zero-padded copies)
};
// `lvl0` != NULL: a batch tree -- the digests of the leaf pairs are given (k_merkle_batch_l0) instead of being packed from `leaves`
// `rt` (optional): the launch that produces the root also stores it (and then rt->flag = rt->seq) in mapped host memory; *rt_done
// tells the caller whether that happened (single-level and BLAKE3 trees do not: the caller copies the root as before)
static int tree_build(DevTree &t, const void *leaves, bool ext, u64 n, const u64 *lvl0 = nullptr, const RootOut *rt = nullptr, bool *rt_done = nullptr) {
    if (rt_done) *rt_done = false;
    DpCtx &c = dp_ctx();
    t.level0 = lvl0;
    t.leaves = leaves; t.ext = ext; t.n = n; t.lg = 0; while ((1ULL << t.lg) < n) t.lg++;
    DP_CHECK(t.lg >= 1, DP_ERR_INVALID, "merkle tree needs at least two leaves");
    t.lvl_off.assign(t.lg + 1, 0);
    u64 total = 0;
    for (u32 l = 1; l < t.lg; l++) { t.lvl_off[l] = total; total += n >> (l + 1); }
    if (int e = dp_dev_alloc((void **)&t.levels, sizeof(u64) * 4 * (total + 1))) return e;
    LvlOff lo_all; memset(&lo_all, 0, sizeof lo_all);
    for (u32 k = 1; k < t.lg && k < 36; k++) lo_all.off[k] = t.lvl_off[k];
    if (blake_on()) {
        const u64 *l0 = lvl0;
        if (!l0) {
            u64 *own = nullptr; if (int e = dp_dev_alloc((void **)&own, sizeof(u64) * 4 * (n >> 1))) return e;
            DpProfScope prof("k_b3_leaves(blake3)", n * (ext ? 16 : 8) + (n >> 1) * 32);
            t.level0 = l0 = own; t.own_level0 = true;
            DP_CUDA(dp_launch(ext ? k_b3_leaves<true> : k_b3_leaves<false>, (unsigned)(((n >> 1) + 255) / 256), 256, 0, c.stream, leaves, n >> 1, own));
        }
        if (t.lg == 1) { t.root_dev = const_cast<u64 *>(l0); return DP_OK; }
        for (u32 l = 1; l < t.lg; l++) {
            const u64 nl = n >> (l + 1);
            const u64 *in = l == 1 ? l0 : t.levels + 4 * t.lvl_off[l - 1];
            if (nl <= 1024 && t.lg < 36) { DpProfScope prof("k_b3_tail(blake3)", nl * 96); DP_CUDA(dp_launch(k_b3_tail, 1, 1024, 0, c.stream, in, l, t.lg, nl, t.levels, lo_all)); break; }
            DpProfScope prof("k_b3_up(blake3)", nl * 96);
            DP_CUDA(dp_launch(k_b3_up, (unsigned)((nl + 255) / 256), 256, 0, c.stream, in, nl, t.levels + 4 * t.lvl_off[l]));
        }
        t.root_dev = t.levels + 4 * t.lvl_off[t.lg - 1];
        return DP_OK;
    }
    if (t.lg == 1 && lvl0) { t.root_dev = const_cast<u64 *>(lvl0); }
    else if (t.lg == 1) {
        DP_CUDA(dp_launch(ext ? k_leafpair_root<true> : k_leafpair_root<false>, 1, 1, 0, c.stream, leaves, t.levels));
        t.root_dev = t.levels;
    } else {
        for (u32 l = 1; l < t.lg; l++) {
            const u64 nl = n >> (l + 1);
            const bool from_leaves = (l == 1 && !lvl0);
            const u64 in_bytes = from_leaves ? nl * (ext ? 64 : 32) : nl * 64;
            const void *src = l == 1 ? (lvl0 ? (const void *)lvl0 : leaves) : (const void *)(t.levels + 4 * t.lvl_off[l - 1]);
            u64 *out = t.levels + 4 * t.lvl_off[l];
            if (nl <= MK_SMALL && t.lg < 36) {   // this and every remaining level in one launch
                DpProfScope prof("k_merkle_small(poseidon2 compress, all remaining levels)", in_bytes + (2 * nl - 1) * 32 * 2, 2 * (2 * nl - 1));
                const bool many = dp_wait_mode() == DP_WAIT_BLOCK;     // the throughput configuration (many proofs in flight)
                const u32 sub_max = many ? MK_SUB : 32, tph_min = many ? 64 : 0xFFFFFFFFu;
                const unsigned g = (unsigned)((nl + sub_max - 1) / sub_max);
                u32 *ticket = nullptr; if (int e = mk_ticket(&ticket)) return e;
                RootOut ro = rt ? *rt : RootOut{nullptr, nullptr, 0};
                const auto kern = from_leaves ? (ext ? k_merkle_small<true, true> : k_merkle_small<false, true>) : k_merkle_small<false, false>;
                DP_CUDA(dp_launch(kern, g, 256, 0, c.stream, src, l, t.lg, nl, t.levels, lo_all, ticket, ro, sub_max, tph_min));
                if (rt && rt_done) *rt_done = true;
                break;
            }
            if (nl <= 32768) {
                // Mid levels (2 k .. 32 k hashes): one thread per hash in 64-thread blocks, with the latency-optimised permutation.  A
                // level is one wave of single-warp chains either way (46 us per compress per warp, 39 us in this formulation vs 52 us
                // for the 8-lanes-per-hash kernel used before), but it now holds 1/8 of the thread slots and issues ~1/5 of the
                // instructions, so the mid levels of many proofs' trees overlap instead of queueing behind each other.
                DpProfScope prof("k_merkle_mid(poseidon2 compress, thread per hash)", in_bytes + nl * 32, 2 * nl);
                const auto kern = from_leaves ? (ext ? k_merkle_mid<true, true> : k_merkle_mid<false, true>) : k_merkle_mid<false, false>;
                DP_CUDA(dp_launch(kern, (unsigned)((nl + 63) / 64), 64, 0, c.stream, src, nl, out));
                continue;
            }
            DpProfScope prof("k_merkle(poseidon2 compress)", in_bytes + nl * 32, 2 * nl);
            const unsigned mgrid = (unsigned)std::min<u64>((nl + 127) / 128, 1u << 22);
            // one hash per thread, many SHORT blocks (no persistent grid-stride blocks): with 16 proofs in flight the block
            // scheduler can interleave other streams' latency-critical single-block kernels every few microseconds
            if (from_leaves) DP_CUDA(dp_launch(ext ? k_merkle_l1<true> : k_merkle_l1<false>, mgrid, 128, 0, c.stream, src, nl, out));
            else DP_CUDA(dp_launch(k_merkle_up, mgrid, 128, 0, c.stream, (const u64 *)src, nl, out));
        }
        t.root_dev = t.levels + 4 * t.lvl_off[t.lg - 1];
    }
    return DP_OK;
}
static void tree_free(DevTree &t) { if (t.own_levels) dp_dev_free(t.levels); t.levels = nullptr; if (t.own_level0) { dp_dev_free(const_cast<u64 *>(t.level0)); t.level0 = nullptr; t.own_level0 = false; } t.leaves = nullptr; }
// the same tree, owning nothing (the per-polynomial views of a batch commitment)
static DevTree tree_view(const DevTree &t) { DevTree v = t; v.own_levels = false; v.own_level0 = false; return v; }

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

// ---- K13 query gather: per (query, tree): [p0.c0 p0.c1 p1.c0 p1.c1][path digests x (lg-1)] ----
// Sharded trees (logG > 0): `leaves` / `levels` are this rank's subtree over 2^lg_local leaves, `top_*` the replicated tree over the G
// subtree roots; a query whose leaf pair another rank owns leaves its row untouched (zero) -- the ranks' rows are summed afterwards.
struct QTree { const void *leaves; const u64 *levels; const u64 *level0; u64 off[34]; u32 lg; u32 ext; u32 shift; u32 logG;
               u32 lg_local; u32 rank; const u64 *top_lvl0; const u64 *top_levels; u64 top_off[9]; };
__global__ void k_query_gather(const QTree *__restrict__ trees, u32 n_trees, const u64 *__restrict__ xs, const u64 *__restrict__ out_off, u64 per_query, u64 *__restrict__ out) {
    u32 q = blockIdx.x, ti = blockIdx.y;
    QTree t = trees[ti];
    u64 idx = xs[q] >> t.shift;
    u64 p0 = (idx | 1) - 1;
    u64 *o = out + (u64)q * per_query + out_off[ti];
    u64 owner = 0;
    if (t.logG) { owner = p0 >> t.lg_local; if (owner != t.rank) return; p0 &= (1ULL << t.lg_local) - 1; }
    const u32 lgl = t.logG ? t.lg_local : t.lg;
    for (u32 k = threadIdx.x; k < t.lg; k += blockDim.x) {
        if (k == 0) {
            if (t.ext) { gle a = ld_e((const gle *)t.leaves + p0), b = ld_e((const gle *)t.leaves + p0 + 1); o[0] = a.c0; o[1] = a.c1; o[2] = b.c0; o[3] = b.c1; }
            else { const u64 *l = (const u64 *)t.leaves; o[0] = l[p0]; o[1] = 0; o[2] = l[p0 + 1]; o[3] = 0; }
        }
        if (k + 1 < t.lg && k + 1 >= lgl) {   // above this rank's subtree: the sibling subtree root, then the replicated top levels
            const u32 kk = k + 1 - lgl;
            const u64 *sd = kk == 0 ? t.top_lvl0 + 4 * (owner ^ 1) : t.top_levels + 4 * (t.top_off[kk] + ((owner >> kk) ^ 1));
            u64 *d = o + 4 + 4 * k;
            d[0] = sd[0]; d[1] = sd[1]; d[2] = sd[2]; d[3] = sd[3];
        } else
        if (k + 1 < t.lg) {   // path entry k = inner[k][(p0 >> (k+1)) ^ 1]
            u64 node = (p0 >> (k + 1)) ^ 1;
            u64 *d = o + 4 + 4 * k;
            if (k == 0 && t.level0) { const u64 *sd = t.level0 + 4 * node; d[0] = sd[0]; d[1] = sd[1]; d[2] = sd[2]; d[3] = sd[3]; }
            else if (k == 0) {
                if (t.ext) { const gle *l = (const gle *)t.leaves + 2 * node; gle a = ld_e(l), b = ld_e(l + 1); d[0] = a.c0; d[1] = a.c1; d[2] = b.c0; d[3] = b.c1; }
                else { const u64 *l = (const u64 *)t.leaves + 2 * node; d[0] = l[0]; d[1] = l[1]; d[2] = 0; d[3] = 0; }
            } else {
                const u64 *s = t.levels + 4 * (t.off[k] + node);
                d[0] = s[0]; d[1] = s[1]; d[2] = s[2]; d[3] = s[3];
            }
        }
    }
}

// =====================================================================================================
struct dp_pcs_comm {
    u32 num_vars = 0, full_log = 0; bool is_base = true, trivial = false;
    void *bh_evals = nullptr;   // bit-reversed evals (raw evals when trivial)
    void *codeword = nullptr;   // bit-reversed codeword (== bh_evals when trivial)
    u64 cw_len = 0;
    DevTree tree;
    u64 root[4] = {0, 0, 0, 0};
    std::vector<dp_pcs_comm *> parts;   // batch_commit: one (encode-only) commitment per polynomial; their trees are views of `tree`
    u64 *level0 = nullptr;              // batch_commit: digests of the leaf pairs
    // dp_pcs_commit_shard: `codeword` / `bh_evals` / `tree` are this rank's contiguous slice (cw_len = local length); `top` is the
    // replicated tree over the world's subtree roots (dp_pcs_comm_set_shard_roots), `root` the global root once it is set
    u32 shard_rank = 0, shard_log = 0; DevTree top; u64 *top_lvl0 = nullptr; u64 local_root[4] = {0, 0, 0, 0};
};

struct OpenRound { gle *oracle = nullptr; u64 len = 0; DevTree tree; DevTree top; u64 *top_lvl0 = nullptr; };
struct dp_pcs_open {
    u32 num_vars = 0, full_log = 0, num_rounds = 0, round = 0;
    std::vector<const dp_pcs_comm *> comms; std::vector<gle> coeffs; bool batch = false;
    gle *oracle0 = nullptr; u64 n0 = 0;        // running oracle of the current round (E)
    bool oracle0_owned = true;
    std::vector<OpenRound> rounds;             // trees over the folded oracles (pre-addition copies)
    gle *pending = nullptr; u64 pending_len = 0;  // folded oracle awaiting its tree/addition
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

int dp_set_merkle_hasher(int kind) {
    DP_CHECK(kind == 0 || kind == 1, DP_ERR_INVALID, "dp_set_merkle_hasher: 0 = Poseidon2 (PoseidonHasher), 1 = BLAKE3 (BlakeHasher)");
    g_hasher.store(kind);
    return DP_OK;
}
int dp_get_merkle_hasher(void) { return g_hasher.load(); }

int dp_poseidon2_init(const uint64_t *ext_rc /*2x4x8*/, const uint64_t *int_rc /*22*/, const uint64_t *diag /*8*/) {
    DP_REQUIRE_CTX();
    DP_CHECK(ext_rc && int_rc && diag, DP_ERR_INVALID, "dp_poseidon2_init: null argument");
    u64 a[64], b[22], d[8];
    for (int i = 0; i < 64; i++) a[i] = gl_canon(ext_rc[i]);
    for (int i = 0; i < 22; i++) b[i] = gl_canon(int_rc[i]);
    for (int i = 0; i < 8; i++) d[i] = gl_canon(diag[i]);
    DP_CUDA(dp_stream_sync(dp_ctx().stream));
    DP_CUDA(p2_upload_constants(a, b, d));
    g_bf.p2_ready.store(true);
    return DP_OK;
}

// enqueue every kernel of one commitment on the context's CURRENT stream; the root lands in `root_pinned`
static int commit_enqueue(const dp_mle *poly, uint32_t full_log, dp_pcs_comm **out, u64 *root_pinned, bool with_tree = true) {
    u32 nv = poly->num_vars();
    DP_CHECK(nv <= full_log, DP_ERR_INVALID, "PolynomialTooLarge");                 // basefold.rs:97-99
    DP_CHECK(nv >= 1, DP_ERR_INVALID, "dp_pcs_commit: need at least one variable");
    if (int e = bf_prepare()) return e;
    DpCtx &c = dp_ctx();
    if (!root_pinned && with_tree) return dp_fail(DP_ERR_INVALID, "commit_enqueue: no root buffer");
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
    if (with_tree) {
        RootOut ro{root_pinned, nullptr, 0}; bool published = false;
        if (int e = tree_build(cm->tree, cm->codeword, poly->is_ext, cm->cw_len, nullptr, &ro, &published)) return e;   // K9
        if (!published) DP_CUDA(cudaMemcpyAsync(root_pinned, cm->tree.root_dev, 32, cudaMemcpyDeviceToHost, c.stream));
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


// the replicated tree over the world's subtree roots: level "0" = the G roots, then log G levels of compress
static int top_tree_build(DevTree &top, u64 **top_lvl0, const uint64_t *roots, u32 logG, u64 out_root[4]) {
    DpCtx &c = dp_ctx();
    const u64 G = 1ULL << logG;
    if (int e = dp_dev_alloc((void **)top_lvl0, 32 * G)) return e;
    u64 *pin = nullptr;
    if (int e = dp_pinned_alloc((void **)&pin, 32 * G + 64)) return e;
    for (u64 k = 0; k < 4 * G; k++) pin[k] = gl_canon(roots[k]);
    DP_CUDA(cudaMemcpyAsync(*top_lvl0, pin, 32 * G, cudaMemcpyHostToDevice, c.stream));
    int rc = tree_build(top, nullptr, false, 2 * G, *top_lvl0);
    if (rc == DP_OK) rc = dp_d2h(out_root, top.root_dev, 32, c.stream);
    else cudaStreamSynchronize(c.stream);
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
    DP_CHECK(!blake_on(), DP_ERR_UNSUPPORTED, "dp_pcs_commit_shard: Poseidon2 trees only");
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
    if (int e = tree_build(cm->tree, cm->codeword, poly->is_ext, cm->cw_len)) return e;
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
    DP_CHECK(!cm->top_lvl0, DP_ERR_STATE, "dp_pcs_comm_set_shard_roots: roots already set");
    for (int k = 0; k < 4; k++) DP_CHECK(gl_canon(roots[4 * cm->shard_rank + k]) == cm->local_root[k], DP_ERR_INVALID, "dp_pcs_comm_set_shard_roots: this rank's entry is not its own subtree root");
    if (int e = top_tree_build(cm->top, &cm->top_lvl0, roots, cm->shard_log, cm->root)) return e;
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
    DP_CHECK(n <= 64, DP_ERR_UNSUPPORTED, "dp_pcs_batch_commit: at most 64 polynomials per batch");
    for (u32 i = 0; i < n; i++) DP_CHECK(polys[i] && polys[i]->len == polys[0]->len && polys[i]->is_ext == polys[0]->is_ext, DP_ERR_INVALID,
                                         "cannot batch commit to polynomials with different number of variables");   // :379-386
    if (int e = bf_prepare()) return e;
    DpCtx &c = dp_ctx();
    CommPtr b(new dp_pcs_comm());
    b->num_vars = polys[0]->num_vars(); b->full_log = full_log; b->is_base = !polys[0]->is_ext;
    if (n == 1) {   // merkelize with one value vector is the plain tree (merkle_tree.rs:274-285): the batch is a view of an ordinary commitment
        dp_pcs_comm *part = nullptr; u64 *pin1 = nullptr;
        if (int e = dp_pinned_alloc((void **)&pin1, 32)) return e;
        int rc = commit_enqueue(polys[0], full_log, &part, pin1, true);
        if (rc == DP_OK) { dp_stream_sync(c.stream); memcpy(part->root, pin1, 32); memcpy(b->root, pin1, 32); }
        dp_pinned_free(pin1);
        if (rc != DP_OK) return rc;
        b->parts.push_back(part); b->trivial = part->trivial; b->cw_len = part->cw_len;
        b->tree = tree_view(part->tree);
        *out = b.release();
        return DP_OK;
    }
    BatchPtrs bp; memset(&bp, 0, sizeof bp);
    for (u32 i = 0; i < n; i++) {
        dp_pcs_comm *part = nullptr;
        if (int e = commit_enqueue(polys[i], full_log, &part, nullptr, false)) return e;
        b->parts.push_back(part); bp.p[i] = part->codeword;
    }
    b->trivial = b->parts[0]->trivial; b->cw_len = b->parts[0]->cw_len;
    u64 N = b->cw_len, n0 = N >> 1;
    if (int e = dp_dev_alloc((void **)&b->level0, 32 * n0)) return e;
    {
        DpProfScope prof("k_merkle_batch_l0(poseidon2 sponge + compress)", (u64)n * N * (b->is_base ? 8 : 16) + 32 * n0);
        const bool blake = blake_on();
        if (blake) DP_CHECK((b->is_base ? n : 2 * n) <= 128, DP_ERR_UNSUPPORTED, "dp_pcs_batch_commit: BLAKE3 batch leaves are limited to one 1024-byte chunk (128 base / 64 extension polynomials)");
        const auto kern = blake ? (b->is_base ? k_b3_batch_l0<false> : k_b3_batch_l0<true>) : (b->is_base ? k_merkle_batch_l0<false> : k_merkle_batch_l0<true>);
        DP_CUDA(dp_launch(kern, (unsigned)((n0 + 127) / 128), 128, 0, c.stream, bp, n, n0, b->level0));
    }
    if (int e = tree_build(b->tree, b->parts[0]->codeword, !b->is_base, N, b->level0)) return e;
    for (auto *part : b->parts) { part->tree = tree_view(b->tree); part->tree.leaves = part->codeword; }   // own leaves, the batch tree's digests
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
    if (dp_ctx().ready) { tree_free(cm->tree); if (!cm->trivial) dp_dev_free(cm->codeword); dp_dev_free(cm->bh_evals); dp_dev_free(cm->level0); tree_free(cm->top); dp_dev_free(cm->top_lvl0); }
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
    if (cm->shard_log) DP_CHECK(cm->num_vars == num_vars && cm->top_lvl0, DP_ERR_STATE, "dp_pcs_open_begin: sharded commitment needs num_vars variables and its shard roots set");
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
        OpenRound rd; rd.oracle = folded; rd.len = len >> 1;
        if (!o->h_root) { void *hp = nullptr; if (int e = dp_pinned_alloc(&hp, 128)) return e; o->h_root = (u64 *)hp; o->h_root[8] = 0; o->root_seq = 0; }
        RootOut ro{o->h_root, o->h_root + 8, ++o->root_seq}; bool published = false;
        if (int e = tree_build(rd.tree, folded, true, rd.len, nullptr, &ro, &published)) return e;   // compute_inner_ext
        if (published) {   // the tree's last launch stores the root and then the sequence number in mapped memory
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
    DP_CHECK(!rd.top_lvl0, DP_ERR_STATE, "dp_pcs_open_set_shard_roots: roots of this round already set");
    u64 rt[4];
    if (int e = top_tree_build(rd.top, &rd.top_lvl0, roots, o->shard_log, rt)) return e;
    for (int k = 0; k < 4; k++) out_root[k] = rt[k];
    return DP_OK;
}

// (sharded opening: this rank's (2^7 >> log world) entries of the BIT-REVERSED final message -- concatenate by rank, then un-bit-reverse)
int dp_pcs_open_final_message(dp_pcs_open *o, uint64_t *out) {
    DP_CHECK(o && out, DP_ERR_INVALID, "dp_pcs_open_final_message: null argument");
    DP_CHECK(o->have_final, DP_ERR_STATE, "dp_pcs_open_final_message: commit phase not finished");
    for (u32 k = 0; k < ((1u << BF_BASECODE_LOG) >> o->shard_log); k++) { out[2 * k] = o->final_msg[k].c0; out[2 * k + 1] = o->final_msg[k].c1; }
    return DP_OK;
}

// u64 words one query occupies in dp_pcs_open_query's output
uint64_t dp_pcs_open_query_words(const dp_pcs_open *o) {
    if (!o) return 0;
    u64 w = 0;
    for (auto cm : o->comms) { u32 lg = 0; while ((1ULL << lg) < cm->cw_len) lg++; lg += o->shard_log; w += 4 + 4 * (u64)(lg - 1); }
    for (auto &rd : o->rounds) w += 4 + 4 * (u64)(rd.tree.lg + o->shard_log - 1);
    return w;
}

// K13 (query_phase.rs:373-474): for every x index, for every commitment then every round oracle:
// [p0.c0 p0.c1 p1.c0 p1.c1] + Merkle path without leaf sibling or root (merkle_tree.rs:139-152).
int dp_pcs_open_query(dp_pcs_open *o, const uint64_t *x_indices, uint32_t n, uint64_t *out) {
    DP_REQUIRE_CTX();
    DP_CHECK(o && x_indices && out && n > 0, DP_ERR_INVALID, "dp_pcs_open_query: null argument");
    DP_CHECK(o->have_final, DP_ERR_STATE, "dp_pcs_open_query: commit phase not finished");
    DpCtx &c = dp_ctx();
    u32 nt = (u32)(o->comms.size() + o->rounds.size());
    std::vector<QTree> qt(nt); std::vector<u64> off(nt);
    u32 lgN = o->num_vars + BF_RATE_LOG; u64 w = 0; u32 k = 0;
    const u32 logG = o->shard_log;
    auto fill = [&](const DevTree &t, u32 shift, const DevTree *top, const u64 *top_lvl0) {
        QTree &q = qt[k]; memset(&q, 0, sizeof q);
        q.leaves = t.leaves; q.levels = t.levels; q.level0 = t.level0; q.lg = t.lg + logG; q.ext = t.ext; q.shift = shift;
        for (u32 l = 1; l < t.lg && l < 34; l++) q.off[l] = t.lvl_off[l];
        q.logG = logG; q.lg_local = t.lg; q.rank = o->shard_rank;
        if (logG) { q.top_lvl0 = top_lvl0; q.top_levels = top->levels; for (u32 l = 1; l < top->lg && l < 9; l++) q.top_off[l] = top->lvl_off[l]; }
        off[k] = w; w += 4 + 4 * (u64)(q.lg - 1); k++;
    };
    if (logG) for (auto &rd : o->rounds) DP_CHECK(rd.top_lvl0 != nullptr, DP_ERR_STATE, "dp_pcs_open_query: a round's shard roots were never set");
    for (auto cm : o->comms) fill(cm->tree, lgN - (cm->tree.lg + logG), &cm->top, cm->top_lvl0);
    for (size_t i = 0; i < o->rounds.size(); i++) fill(o->rounds[i].tree, (u32)i + 1, &o->rounds[i].top, o->rounds[i].top_lvl0);
    QTree *dq = nullptr; u64 *doff = nullptr, *dx = nullptr, *dout = nullptr;
    if (int e = dp_dev_alloc((void **)&dq, sizeof(QTree) * nt)) return e;
    if (int e = dp_dev_alloc((void **)&doff, 8 * nt)) return e;
    if (int e = dp_dev_alloc((void **)&dx, 8 * (size_t)n)) return e;
    if (int e = dp_dev_alloc((void **)&dout, 8 * w * n)) return e;
    DP_CUDA(cudaMemcpyAsync(dq, qt.data(), sizeof(QTree) * nt, cudaMemcpyHostToDevice, c.stream));
    DP_CUDA(cudaMemcpyAsync(doff, off.data(), 8 * nt, cudaMemcpyHostToDevice, c.stream));
    DP_CUDA(cudaMemcpyAsync(dx, x_indices, 8 * (size_t)n, cudaMemcpyHostToDevice, c.stream));
    DP_CUDA(dp_stream_sync(c.stream));   // qt/off are stack-owned host buffers
    if (logG) DP_CUDA(cudaMemsetAsync(dout, 0, 8 * w * n, c.stream));   // rows of queries other ranks own stay zero
    DP_CUDA(dp_launch(k_query_gather, dim3(n, nt), 32, 0, c.stream, dq, nt, dx, doff, w, dout));
    if (int e = dp_d2h(out, dout, 8 * w * n, c.stream)) return e;
    dp_dev_free(dq); dp_dev_free(doff); dp_dev_free(dx); dp_dev_free(dout);
    return DP_OK;
}

int dp_pcs_open_free(dp_pcs_open *o) {
    if (!o) return DP_OK;
    if (dp_ctx().ready) {
        if (o->sc) dp_sc_destroy(o->sc);
        bool oracle_in_rounds = false;
        for (auto &rd : o->rounds) { if (rd.oracle == o->oracle0) oracle_in_rounds = true; tree_free(rd.tree); dp_dev_free(rd.oracle); tree_free(rd.top); dp_dev_free(rd.top_lvl0); }
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
