// K9 Merkle trees and K13 query paths of the Basefold PCS, under the process-wide hasher: Poseidon2 (PoseidonHasher) or BLAKE3
// (BlakeHasher).  Reference: mpcs/src/util/{merkle_tree.rs,hash.rs}, basefold/query_phase.rs:373-474.  Tree layout: merkle.cuh.
#include "merkle.cuh"
#include "poseidon2.cuh"
#include "blake3.cuh"
#include <algorithm>
#include <atomic>
#include <mutex>

// Selected process-wide with dp_set_merkle_hasher (the reference selects at compile time: feature `blake`, mpcs/src/lib.rs:339-342).
static std::atomic<int> g_hasher{0};          // 0 Poseidon2 (default), 1 BLAKE3
bool mk_blake3() { return g_hasher.load(std::memory_order_relaxed) == 1; }

// Level l >= 1 of a tree over n leaves starts (n >> 1) - (n >> l) digests into the packed levels (level l has n >> (l + 1)).
__host__ __device__ __forceinline__ u64 level_off(u64 n, u32 l) { return (n >> 1) - (n >> l); }
static constexpr u32 MK_LEVELS = 36;              // levels a tree may have: 2^36 leaves are far more than HBM holds
struct LvlOff { u64 off[MK_LEVELS]; };            // level_off of every level, for the kernels that build several levels

// the digest of leaf pair `pair` (elements 2 pair and 2 pair + 1): the Ext pair's four limbs, or the Base pair zero-padded
template <bool EXT> __device__ __forceinline__ void leaf_pair_digest(const void *leaves, u64 pair, u64 d[4]) {
    if (EXT) { const gle *l = (const gle *)leaves + 2 * pair; gle a = ld_e(l), b = ld_e(l + 1); d[0] = a.c0; d[1] = a.c1; d[2] = b.c0; d[3] = b.c1; }
    else { ulonglong2 v = ld_b2((const u64 *)leaves + 2 * pair); d[0] = v.x; d[1] = v.y; d[2] = 0; d[3] = 0; }
}
// ... word w of it, for 8 lanes per hash (poseidon2.cuh): a lane loads only its own word
template <bool EXT> __device__ __forceinline__ u64 leaf_pair_word(const void *leaves, u64 pair, int w) {
    if (EXT) return ((const u64 *)leaves)[4 * pair + w];
    return w < 2 ? ((const u64 *)leaves)[2 * pair + w] : 0ULL;
}
// batch_commit leaves (merkle_tree.rs:286-312, util/hash.rs:30-41): word k of the values of all m polynomials at index `leaf`,
// base-field limbs in polynomial order
struct BatchPtrs { const void *p[MK_BATCH_MAX]; };
template <bool EXT> __device__ __forceinline__ u64 batch_word(const BatchPtrs &bp, u64 leaf, int k) {
    return EXT ? ((const u64 *)bp.p[k >> 1])[2 * leaf + (k & 1)] : ((const u64 *)bp.p[k])[leaf];
}

// ---- Poseidon2 levels ----
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
// one hash per thread, many short blocks (levels of more than 32 k hashes)
template <bool EXT, bool FROM_LEAVES>
__global__ void k_merkle_wide(const void *__restrict__ src, u64 n_out, u64 *__restrict__ out) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    for (; i < n_out; i += stride) {
        u64 x[4], y[4], o[4];
        if (FROM_LEAVES) mk_leaf_children<EXT>(src, i, x, y);
        else mk_node_children((const u64 *)src + 8 * i, x, y);
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
// Every remaining level of a tree whose current level has <= MK_SMALL hashes, in ONE launch.  Each block owns MK_SUB hashes of the
// first level and walks that subtree up to its root with a block barrier per level; the last block to finish (ticket) folds the
// <= 8 subtree roots.  A level with >= 64 hashes per block runs one THREAD per hash (latency-optimised permutation): the same
// ~40 us per level as a single-warp chain costs anyway, at 1/5 of the issue slots of the lane-parallel form -- with dozens of proofs
// in flight these small trees were as much GPU work as all the wide Merkle levels together (8 lanes x ~4.5 k instructions per
// permutation against 12.8 k for one thread).  Levels with <= 32 hashes per block use 8 lanes per hash (shorter dependent chain,
// ~27 us per level); 88 % of a 2048-hash tree's permutations are in the thread-per-hash levels.
static constexpr u32 MK_SUB = 256;
static constexpr u64 MK_SMALL = 2048;
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
static std::mutex g_mk_mu;
// once per process, before the first tree or dp_poseidon2_init: the ticket pool and the built-in Poseidon2 constants
static int mk_prepare() {
    if (g_mk_tickets.load()) return DP_OK;
    std::lock_guard<std::mutex> lk(g_mk_mu);
    if (g_mk_tickets.load()) return DP_OK;
    DP_CUDA(p2_upload_constants((const u64 *)&DP_P2_EXT_RC[0][0][0], (const u64 *)DP_P2_INT_RC, (const u64 *)DP_P2_DIAG));
    u32 *tickets = nullptr;
    DP_CUDA(cudaMalloc((void **)&tickets, sizeof(u32) * MK_TICKETS));
    DP_CUDA(cudaMemset(tickets, 0, sizeof(u32) * MK_TICKETS));
    g_mk_tickets.store(tickets);
    return DP_OK;
}

// batch_commit leaf level: digest_i = compress(hash(values of all m polynomials at index 2i), hash(... at 2i+1)), hash = hash_or_noop
template <bool EXT>
__global__ void k_merkle_batch_l0(BatchPtrs bp, u32 m, u64 n_out, u64 *__restrict__ out) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_out) return;
    u64 x[4], y[4], o[4];
    const int n = EXT ? 2 * (int)m : (int)m;
    auto ga = [&](int k) -> u64 { return batch_word<EXT>(bp, 2 * i, k); };
    auto gb = [&](int k) -> u64 { return batch_word<EXT>(bp, 2 * i + 1, k); };
    p2_hash_or_noop(ga, n, x); p2_hash_or_noop(gb, n, y);
    p2_compress(x, y, o);
    mk_store(out, i, o);
}
template <bool EXT> __global__ void k_leafpair_root(const void *leaves, u64 *out) { u64 d[4]; leaf_pair_digest<EXT>(leaves, 0, d); for (int i = 0; i < 4; i++) out[i] = d[i]; }

// ---- BLAKE3 levels (mpcs/src/util/hash.rs:79-95): leaf pair -> BLAKE3(LE bytes), inner node -> BLAKE3(left || right) ----
// level 0 (hash_two_leaves) of a single-polynomial tree: one digest per leaf pair, stored (a hash, unlike Poseidon2's level 0)
template <bool EXT> __global__ void k_b3_leaves(const void *__restrict__ leaves, u64 n_out, u64 *__restrict__ out) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_out) return;
    u64 w[4], d[4];
    leaf_pair_digest<EXT>(leaves, i, w);
    b3::hash_words(w, EXT ? 4 : 2, d);
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
    auto ga = [&](int k) -> u64 { return batch_word<EXT>(bp, 2 * i, k); };
    auto gb = [&](int k) -> u64 { return batch_word<EXT>(bp, 2 * i + 1, k); };
    u64 w[8], d[4];
    b3::hash_stream(ga, n, w); b3::hash_stream(gb, n, w + 4);
    b3::hash_words(w, 8, d);
#pragma unroll
    for (int k = 0; k < 4; k++) out[4 * i + k] = d[k];
}

// ---- building a tree ----
// A t.level0 the caller set (a sharded top tree) is level 0.  Level 1 reads the stored level 0 if there is one, otherwise the leaves.
int tree_build(DevTree &t, const std::vector<const void *> &leaves, bool ext, u64 n, const RootOut *rt) {
    DpCtx &c = dp_ctx();
    t.ext = ext; t.lg = 0; while ((1ULL << t.lg) < n) t.lg++;
    DP_CHECK(n == 1ULL << t.lg && t.lg >= 1 && t.lg <= MK_LEVELS, DP_ERR_INVALID, "merkle tree needs 2^1 .. 2^36 leaves (a power of two)");
    DP_CHECK(!leaves.empty() && leaves.size() <= MK_BATCH_MAX, DP_ERR_INVALID, "merkle tree needs 1 .. 64 leaf vectors");
    if (int e = mk_prepare()) return e;
    const bool blake = mk_blake3();
    const u64 n0 = n >> 1;
    if (!t.level0 && (leaves.size() > 1 || blake)) {   // a stored level 0 of leaf-pair digests, made here
        if (int e = dp_dev_alloc((void **)&t.level0, 32 * n0)) return e;
        if (leaves.size() > 1) {
            BatchPtrs bp; memset(&bp, 0, sizeof bp);
            std::copy(leaves.begin(), leaves.end(), bp.p);
            const u32 m = (u32)leaves.size();
            DpProfScope prof("k_merkle_batch_l0(poseidon2 sponge + compress)", (u64)m * n * (ext ? 16 : 8) + 32 * n0);
            const auto kern = blake ? (ext ? k_b3_batch_l0<true> : k_b3_batch_l0<false>) : (ext ? k_merkle_batch_l0<true> : k_merkle_batch_l0<false>);
            DP_CUDA(dp_launch(kern, (unsigned)((n0 + 127) / 128), 128, 0, c.stream, bp, m, n0, t.level0));
        } else {
            DpProfScope prof("k_b3_leaves(blake3)", n * (ext ? 16 : 8) + n0 * 32);
            DP_CUDA(dp_launch(ext ? k_b3_leaves<true> : k_b3_leaves<false>, (unsigned)((n0 + 255) / 256), 256, 0, c.stream, leaves[0], n0, t.level0));
        }
    }
    LvlOff lo; memset(&lo, 0, sizeof lo);
    for (u32 l = 1; l < t.lg; l++) lo.off[l] = level_off(n, l);
    if (int e = dp_dev_alloc((void **)&t.levels, sizeof(u64) * 4 * (level_off(n, t.lg) + 1))) return e;
    if (t.lg == 1) {   // the root is level 0
        if (!t.level0) DP_CUDA(dp_launch(t.ext ? k_leafpair_root<true> : k_leafpair_root<false>, 1, 1, 0, c.stream, leaves[0], t.levels));
        t.root_dev = t.level0 ? t.level0 : t.levels;
        return DP_OK;
    }
    for (u32 l = 1; l < t.lg; l++) {
        const u64 nl = n >> (l + 1);
        const bool from_leaves = l == 1 && !t.level0;
        const void *src = l > 1 ? (const void *)(t.levels + 4 * lo.off[l - 1]) : t.level0 ? (const void *)t.level0 : leaves[0];
        u64 *out = t.levels + 4 * lo.off[l];
        if (blake) {
            if (nl <= 1024) { DpProfScope prof("k_b3_tail(blake3)", nl * 96); DP_CUDA(dp_launch(k_b3_tail, 1, 1024, 0, c.stream, (const u64 *)src, l, t.lg, nl, t.levels, lo)); break; }
            DpProfScope prof("k_b3_up(blake3)", nl * 96);
            DP_CUDA(dp_launch(k_b3_up, (unsigned)((nl + 255) / 256), 256, 0, c.stream, (const u64 *)src, nl, out));
            continue;
        }
        const u64 in_bytes = from_leaves ? nl * (t.ext ? 64 : 32) : nl * 64;
        if (nl <= MK_SMALL) {   // this and every remaining level in one launch
            DpProfScope prof("k_merkle_small(poseidon2 compress, all remaining levels)", in_bytes + (2 * nl - 1) * 32 * 2, 2 * (2 * nl - 1));
            const bool many = dp_wait_mode() == DP_WAIT_BLOCK;     // the throughput configuration (many proofs in flight)
            const u32 sub_max = many ? MK_SUB : 32, tph_min = many ? 64 : 0xFFFFFFFFu;
            const unsigned g = (unsigned)((nl + sub_max - 1) / sub_max);
            u32 *ticket = g_mk_tickets.load() + (g_mk_next.fetch_add(1, std::memory_order_relaxed) % MK_TICKETS);
            RootOut ro = rt ? *rt : RootOut{nullptr, nullptr, 0};
            const auto kern = from_leaves ? (t.ext ? k_merkle_small<true, true> : k_merkle_small<false, true>) : k_merkle_small<false, false>;
            DP_CUDA(dp_launch(kern, g, 256, 0, c.stream, src, l, t.lg, nl, t.levels, lo, ticket, ro, sub_max, tph_min));
            t.root_published = rt != nullptr;
            break;
        }
        if (nl <= 32768) {
            // Mid levels (2 k .. 32 k hashes): one thread per hash in 64-thread blocks, with the latency-optimised permutation.  A
            // level is one wave of single-warp chains either way (46 us per compress per warp, 39 us in this formulation vs 52 us
            // for the 8-lanes-per-hash kernel used before), but it now holds 1/8 of the thread slots and issues ~1/5 of the
            // instructions, so the mid levels of many proofs' trees overlap instead of queueing behind each other.
            DpProfScope prof("k_merkle_mid(poseidon2 compress, thread per hash)", in_bytes + nl * 32, 2 * nl);
            const auto kern = from_leaves ? (t.ext ? k_merkle_mid<true, true> : k_merkle_mid<false, true>) : k_merkle_mid<false, false>;
            DP_CUDA(dp_launch(kern, (unsigned)((nl + 63) / 64), 64, 0, c.stream, src, nl, out));
            continue;
        }
        DpProfScope prof("k_merkle(poseidon2 compress)", in_bytes + nl * 32, 2 * nl);
        const unsigned mgrid = (unsigned)std::min<u64>((nl + 127) / 128, 1u << 22);
        // one hash per thread, many SHORT blocks (no persistent grid-stride blocks): with 16 proofs in flight the block
        // scheduler can interleave other streams' latency-critical single-block kernels every few microseconds
        const auto kern = from_leaves ? (t.ext ? k_merkle_wide<true, true> : k_merkle_wide<false, true>) : k_merkle_wide<false, false>;
        DP_CUDA(dp_launch(kern, mgrid, 128, 0, c.stream, src, nl, out));
    }
    t.root_dev = t.levels + 4 * lo.off[t.lg - 1];
    return DP_OK;
}

// level 0 is the G subtree roots, then log G levels
int top_tree_build(DevTree &top, const uint64_t *roots, u32 logG, uint64_t out_root[4]) {
    DpCtx &c = dp_ctx();
    const u64 G = 1ULL << logG;
    if (int e = dp_dev_alloc((void **)&top.level0, 32 * G)) return e;
    u64 *pin = nullptr;
    if (int e = dp_pinned_alloc((void **)&pin, 32 * G + 64)) return e;
    for (u64 k = 0; k < 4 * G; k++) pin[k] = gl_canon(roots[k]);
    DP_CUDA(cudaMemcpyAsync(top.level0, pin, 32 * G, cudaMemcpyHostToDevice, c.stream));
    int rc = tree_build(top, {nullptr}, false, 2 * G);
    if (rc == DP_OK) rc = dp_d2h(out_root, top.root_dev, 32, c.stream);
    else cudaStreamSynchronize(c.stream);
    dp_pinned_free(pin);
    return rc;
}

void tree_free(DevTree &t) { dp_dev_free(t.level0); dp_dev_free(t.levels); t = DevTree(); }

// ---- K13 query gather: per (query, tree): [p0.c0 p0.c1 p1.c0 p1.c1][path digests x (lg-1)] at out_off of the query's row ----
// Sharded trees (logG > 0): `level0` / `levels` are this rank's subtree over 2^lg_local leaves, `top_*` the replicated tree over
// the G subtree roots; a query whose leaf pair another rank owns leaves its row untouched (zero) -- the ranks' rows are summed afterwards.
struct QTree { const u64 *level0, *levels, *top_level0, *top_levels; const void *leaves; u64 out_off; u32 lg, ext, shift, logG, lg_local, rank; };
// entry k of a path in a tree over n leaves, the digest of `node` on level k: stored level 0 if there is one, otherwise the leaf
// pair; above level 0, the packed level
__device__ void path_entry(const u64 *level0, const u64 *levels, u64 n, const void *leaves, bool ext, u32 k, u64 node, u64 d[4]) {
    const u64 *s;
    if (k > 0) s = levels + 4 * (level_off(n, k) + node);
    else if (level0) s = level0 + 4 * node;
    else { if (ext) leaf_pair_digest<true>(leaves, node, d); else leaf_pair_digest<false>(leaves, node, d); return; }
    d[0] = s[0]; d[1] = s[1]; d[2] = s[2]; d[3] = s[3];
}
__global__ void k_query_gather(const QTree *__restrict__ trees, const u64 *__restrict__ xs, u64 per_query, u64 *__restrict__ out) {
    const QTree &t = trees[blockIdx.y];
    u64 p0 = ((xs[blockIdx.x] >> t.shift) | 1) - 1;
    u64 *o = out + (u64)blockIdx.x * per_query + t.out_off;
    u64 owner = 0;
    if (t.logG) { owner = p0 >> t.lg_local; if (owner != t.rank) return; p0 &= (1ULL << t.lg_local) - 1; }
    for (u32 k = threadIdx.x; k < t.lg; k += blockDim.x) {
        if (k == 0) {   // the queried pair read as a leaf-pair digest; Base leaves lifted to the extension: (a, b, 0, 0) -> (a, 0, b, 0)
            path_entry(nullptr, nullptr, 0, t.leaves, t.ext, 0, p0 >> 1, o);
            if (!t.ext) { o[2] = o[1]; o[1] = 0; }
        }
        if (k + 1 >= t.lg) continue;
        if (k + 1 >= t.lg_local) {   // above this rank's subtree: the sibling subtree root, then the replicated top levels
            const u32 kk = k + 1 - t.lg_local;
            path_entry(t.top_level0, t.top_levels, 2ULL << t.logG, nullptr, false, kk, (owner >> kk) ^ 1, o + 4 + 4 * k);
        } else path_entry(t.level0, t.levels, 1ULL << t.lg_local, t.leaves, t.ext, k, (p0 >> (k + 1)) ^ 1, o + 4 + 4 * k);
    }
}

u64 mk_query_words(const std::vector<MkPath> &paths, u32 logG, std::vector<u64> *row_off) {
    u64 w = 0;
    for (auto &p : paths) { if (row_off) row_off->push_back(w); w += 4 * (u64)(p.tree->lg + logG); }
    return w;
}

int mk_query_gather(const std::vector<MkPath> &paths, u32 logG, u32 rank, const uint64_t *x_indices, u32 n, uint64_t *out) {
    DpCtx &c = dp_ctx();
    const u32 nt = (u32)paths.size();
    std::vector<QTree> qt(nt); std::vector<u64> off;
    const u64 w = mk_query_words(paths, logG, &off);
    for (u32 k = 0; k < nt; k++) {
        const DevTree &t = *paths[k].tree;
        qt[k] = QTree{t.level0, t.levels, paths[k].top->level0, paths[k].top->levels, paths[k].leaves, off[k], t.lg + logG, t.ext, paths[k].shift, logG, t.lg, rank};
    }
    QTree *dq = nullptr; u64 *dx = nullptr, *dout = nullptr;
    if (int e = dp_dev_alloc((void **)&dq, sizeof(QTree) * nt)) return e;
    if (int e = dp_dev_alloc((void **)&dx, 8 * (size_t)n)) return e;
    if (int e = dp_dev_alloc((void **)&dout, 8 * w * n)) return e;
    DP_CUDA(cudaMemcpyAsync(dq, qt.data(), sizeof(QTree) * nt, cudaMemcpyHostToDevice, c.stream));
    DP_CUDA(cudaMemcpyAsync(dx, x_indices, 8 * (size_t)n, cudaMemcpyHostToDevice, c.stream));
    DP_CUDA(dp_stream_sync(c.stream));   // qt is a host vector
    if (logG) DP_CUDA(cudaMemsetAsync(dout, 0, 8 * w * n, c.stream));   // rows of queries other ranks own stay zero
    DP_CUDA(dp_launch(k_query_gather, dim3(n, nt), 32, 0, c.stream, dq, dx, w, dout));
    if (int e = dp_d2h(out, dout, 8 * w * n, c.stream)) return e;
    dp_dev_free(dq); dp_dev_free(dx); dp_dev_free(dout);
    return DP_OK;
}

extern "C" {

int dp_set_merkle_hasher(int kind) {
    DP_CHECK(kind == 0 || kind == 1, DP_ERR_INVALID, "dp_set_merkle_hasher: 0 = Poseidon2 (PoseidonHasher), 1 = BLAKE3 (BlakeHasher)");
    g_hasher.store(kind);
    return DP_OK;
}
int dp_get_merkle_hasher(void) { return g_hasher.load(); }

// the Merkle kernels' Poseidon2 constants (the transcript's copy in sumcheck.cu keeps the built-in ones)
int dp_poseidon2_init(const uint64_t *ext_rc /*2x4x8*/, const uint64_t *int_rc /*22*/, const uint64_t *diag /*8*/) {
    DP_REQUIRE_CTX();
    DP_CHECK(ext_rc && int_rc && diag, DP_ERR_INVALID, "dp_poseidon2_init: null argument");
    u64 a[64], b[22], d[8];
    for (int i = 0; i < 64; i++) a[i] = gl_canon(ext_rc[i]);
    for (int i = 0; i < 22; i++) b[i] = gl_canon(int_rc[i]);
    for (int i = 0; i < 8; i++) d[i] = gl_canon(diag[i]);
    if (int e = mk_prepare()) return e;   // the built-in constants are never uploaded after these
    DP_CUDA(dp_stream_sync(dp_ctx().stream));
    DP_CUDA(p2_upload_constants(a, b, d));
    return DP_OK;
}

}  // extern "C"
