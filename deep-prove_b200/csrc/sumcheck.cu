// Sumcheck prover rounds on device (K1 + K2 fused).
// Reference: sumcheck/src/prover.rs:498-741 (prove_parallel / prove_round_and_update_state_parallel),
// sumcheck_macro/src/lib.rs:46-326 (the per-pair arithmetic), multilinear_extensions/src/mle.rs:631-712
// (fix_variables_parallel).
//
// Design: ONE launch per round for the whole VirtualPolynomial.  grid.y = product index, grid.x
// tiles the pairs; each operand is streamed once with 16-byte loads.  From round 2 on the fold by the
// previous challenge is fused into the same pass: a thread reads 4 consecutive elements of the old
// table, folds them to one adjacent pair, the owning product writes the pair to the (half-size)
// ping-pong table, and every product using the operand feeds the pair straight into the round
// polynomial accumulators.  Accumulators live in registers, are combined with warp shuffles, then per
// block through shared memory, and the last block of each product (ticket counter) reduces the block
// partials -- field addition is exact, so the summation order is free and the result is bit-identical
// to the reference's rayon fold.  The (deg+1) sums per product go back through a pinned buffer; the
// O(deg^2) glue (2^k multiplicity, coefficient, barycentric extrapolation -- prover.rs:713-724,
// util.rs:101-136) is one rule, sc_glue_product: the host applies it inside dp_sc_round, and CTA 0 of
// the resident kernel applies it when the kernel runs the transcript itself.
#include "common.cuh"
#include "poseidon2.cuh"
#include "blake3.cuh"
#include "../../include/dp_blake3.h"
#include <mutex>
#include <algorithm>

enum : u32 { OPM_B = 0, OPM_E = 1, OPM_BF = 2, OPM_EF = 3 };
struct ScOp { const void *src; gle *dst; u32 mode; u32 pad; };
struct ScProd { ScOp op[5]; u64 npairs; u32 d; u32 allbase; u32 konst; u32 pad; };
static constexpr int SC_NACC = 6;
static constexpr int SC_THREADS = 256;

__device__ __forceinline__ gle fold_b(u64 a, u64 b, gle r) { return e_add(e_mul_base(r, gl_sub(b, a)), e_from_base(a)); }
__device__ __forceinline__ gle fold_e(gle a, gle b, gle r) { return e_add(a, e_mul(e_sub(b, a), r)); }
// CG: L1-bypassing loads (ld.global.cg) -- the resident cluster kernel reads tables other CTAs of the cluster wrote a round earlier
template <bool CG> __device__ __forceinline__ gle ldx_e(const gle *p) {
    if (CG) { ulonglong2 v = __ldcg(reinterpret_cast<const ulonglong2 *>(p)); return e_make(v.x, v.y); }
    return ld_e(p);
}
template <bool CG> __device__ __forceinline__ ulonglong2 ldx_b2(const u64 *p) { return CG ? __ldcg(reinterpret_cast<const ulonglong2 *>(p)) : ld_b2(p); }
template <bool CG> __device__ __forceinline__ u64 ldx_b(const u64 *p) { return CG ? __ldcg(p) : *p; }

// length-1 operands (sumcheck_macro/src/lib.rs:236-241): value at every evaluation point
template <bool CG = false>
__device__ __forceinline__ gle sc_load_const(const ScOp &op, gle r) {
    switch (op.mode) {
    case OPM_B: return e_from_base(ldx_b<CG>((const u64 *)op.src));
    case OPM_E: return ldx_e<CG>((const gle *)op.src);
    case OPM_BF: { ulonglong2 v = ldx_b2<CG>((const u64 *)op.src); gle x = fold_b(v.x, v.y, r); if (op.dst) st_e(op.dst, x); return x; }
    default: { const gle *s = (const gle *)op.src; gle x = fold_e(ldx_e<CG>(s), ldx_e<CG>(s + 1), r); if (op.dst) st_e(op.dst, x); return x; }
    }
}

// Out-of-line copies for the latency-bound kernels (general rounds, resident rounds).  Their cost is instruction FETCH, not issue:
// with every E x E (122 instructions) and every operand's 4-way mode switch inlined, k_sc_res<3> was 6.9 k instructions (110 KB) and
// k_sc_round<3> 5.5 k -- more than the SM's instruction cache holds -- so a round of a few hundred pairs spent most of its ~15 us
// refetching its own code from L2.  One shared copy of each costs a call (~20 cycles) per use and keeps the round loop resident.
__device__ __noinline__ gle e_mul_ni(gle a, gle b) { return e_mul(a, b); }
struct gle2 { gle lo, hi; };
template <bool CG>
__device__ __noinline__ gle2 sc_load_pair_ni(const ScOp *op, u64 i, gle r, bool store = true) {
    gle2 o;
    switch (op->mode) {
    case OPM_B: { ulonglong2 v = ldx_b2<CG>((const u64 *)op->src + 2 * i); o.lo = e_from_base(v.x); o.hi = e_from_base(v.y); } break;
    case OPM_E: { const gle *s = (const gle *)op->src + 2 * i; o.lo = ldx_e<CG>(s); o.hi = ldx_e<CG>(s + 1); } break;
    case OPM_BF: {
        const u64 *s = (const u64 *)op->src + 4 * i;
        ulonglong2 v0 = ldx_b2<CG>(s), v1 = ldx_b2<CG>(s + 2);
        o.lo = fold_b(v0.x, v0.y, r); o.hi = fold_b(v1.x, v1.y, r);
        if (store && op->dst) { st_e(op->dst + 2 * i, o.lo); st_e(op->dst + 2 * i + 1, o.hi); }
    } break;
    default: {
        const gle *s = (const gle *)op->src + 4 * i;
        gle f0 = ldx_e<CG>(s), f1 = ldx_e<CG>(s + 1), f2 = ldx_e<CG>(s + 2), f3 = ldx_e<CG>(s + 3);
        o.lo = e_add(f0, e_mul_ni(e_sub(f1, f0), r)); o.hi = e_add(f2, e_mul_ni(e_sub(f3, f2), r));
        if (store && op->dst) { st_e(op->dst + 2 * i, o.lo); st_e(op->dst + 2 * i + 1, o.hi); }
    } break;
    }
    return o;
}

// a[t] += p with a runtime t but register-resident a[] (predicated select, no local memory)
template <int N> __device__ __forceinline__ void acc_add_dyn(u64 (&a)[N], int t, u64 p) {
#pragma unroll
    for (int k = 0; k < N; k++) if (k == t) a[k] = gl_add(a[k], p);
}
template <int N> __device__ __forceinline__ void acc_add_dyn_e(gle (&a)[N], int t, gle p) {
#pragma unroll
    for (int k = 0; k < N; k++) if (k == t) a[k] = e_add(a[k], p);
}

// General body: any mix of operand modes, decided at run time per operand (mixed Base/Ext products, shared MLEs, constants).
// The uniform-mode rounds that carry the bandwidth (all operands Base / all folding) take the lean kernels below instead.
template <int D, bool CG = false>
__device__ __forceinline__ void sc_body(const ScProd &pd, gle r, gle acc[SC_NACC], const u64 tid, const u64 stride) {
    if (pd.konst) {
        if (tid == 0) {
            gle p = sc_load_const<CG>(pd.op[0], r);
#pragma unroll
            for (int j = 1; j < D; j++) p = e_mul_ni(p, sc_load_const<CG>(pd.op[j], r));
#pragma unroll
            for (int t = 0; t <= D; t++) acc[t] = p;
        }
        return;
    }
    if (pd.allbase) {
        // all operands Base and unfolded: stay in F (sumcheck_macro/src/lib.rs:294-299 lifts at the end)
        u64 a[D + 1];
#pragma unroll
        for (int t = 0; t <= D; t++) a[t] = 0;
        for (u64 i = tid; i < pd.npairs; i += stride) {
            u64 cur[D], st[D];
#pragma unroll
            for (int j = 0; j < D; j++) {
                ulonglong2 v = ldx_b2<CG>((const u64 *)pd.op[j].src + 2 * i);
                cur[j] = v.x; st[j] = gl_sub(v.y, v.x);
            }
#pragma unroll 1
            for (int t = 0; t <= D; t++) {
                u64 p = cur[0];
#pragma unroll
                for (int j = 1; j < D; j++) p = gl_mul(p, cur[j]);
                acc_add_dyn<D + 1>(a, t, p);
                if (t < D) {
#pragma unroll
                    for (int j = 0; j < D; j++) cur[j] = gl_add(cur[j], st[j]);
                }
            }
        }
#pragma unroll
        for (int t = 0; t <= D; t++) acc[t] = e_from_base(a[t]);
        return;
    }
    gle a[D + 1];
#pragma unroll
    for (int t = 0; t <= D; t++) a[t] = e_zero();
    for (u64 i = tid; i < pd.npairs; i += stride) {
        gle cur[D], st[D];
#pragma unroll
        for (int j = 0; j < D; j++) {
            const gle2 v = sc_load_pair_ni<CG>(&pd.op[j], i, r);
            cur[j] = v.lo; st[j] = e_sub(v.hi, v.lo);
        }
#pragma unroll 1
        for (int t = 0; t <= D; t++) {
            gle p = cur[0];
#pragma unroll
            for (int j = 1; j < D; j++) p = (pd.op[j].mode == OPM_B) ? e_mul_base(p, cur[j].c0) : e_mul_ni(p, cur[j]);
            acc_add_dyn_e<D + 1>(a, t, p);
            if (t < D) {
#pragma unroll
                for (int j = 0; j < D; j++) cur[j] = e_add(cur[j], st[j]);
            }
        }
    }
#pragma unroll
    for (int t = 0; t <= D; t++) acc[t] = a[t];
}

// Small resident rounds (fewer pairs than a quarter of the lanes a product owns): one (pair, evaluation point) per LANE instead of one
// pair per lane.  The 2^tpl lanes of a pair load and fold it redundantly (same instructions, no extra time), then each computes the
// product at ITS point only -- the dependent chain per lane drops from D folds x 2 + (D+1)(D-1) extension multiplications to
// D x 2 + (D-1) (8 instead of 14 for D = 3), which is most of a small round's device time (phase clocks: 6.2 us of "work" for <= 64
// pairs).  Lane t == 0 of a pair writes the folded table; the other lanes' accumulators stay zero, so the ordinary reduction applies.
template <int D, bool CG>
__device__ __forceinline__ void sc_body_split(const ScProd &pd, gle r, gle acc[SC_NACC], const u64 L, const u32 tpl) {
    const u64 i = L >> tpl; const u32 t = (u32)L & ((1u << tpl) - 1);
    if (i >= pd.npairs || t > (u32)D) return;
    gle cur[D];
#pragma unroll
    for (int j = 0; j < D; j++) {
        const gle2 v = sc_load_pair_ni<CG>(&pd.op[j], i, r, t == 0);
        const gle st = e_sub(v.hi, v.lo);
        gle c = v.lo;
        for (u32 q = 0; q < t; q++) c = e_add(c, st);
        cur[j] = c;
    }
    gle p = cur[0];
#pragma unroll
    for (int j = 1; j < D; j++) p = (pd.op[j].mode == OPM_B) ? e_mul_base(p, cur[j].c0) : e_mul_ni(p, cur[j]);
#pragma unroll
    for (int tt = 0; tt <= D; tt++) if (tt == (int)t) acc[tt] = p;
}

// Degree dispatch of the bodies: DSEL = 1..5 is the degree of every product; DSEL = 0 takes the product's own degree
template <int DSEL, bool CG>
__device__ __forceinline__ void sc_body_dsel(const ScProd &pd, gle r, gle acc[SC_NACC], const u64 tid, const u64 stride) {
    if constexpr (DSEL != 0) sc_body<DSEL, CG>(pd, r, acc, tid, stride);
    else switch (pd.d) {
    case 1: sc_body<1, CG>(pd, r, acc, tid, stride); break;
    case 2: sc_body<2, CG>(pd, r, acc, tid, stride); break;
    case 3: sc_body<3, CG>(pd, r, acc, tid, stride); break;
    case 4: sc_body<4, CG>(pd, r, acc, tid, stride); break;
    default: sc_body<5, CG>(pd, r, acc, tid, stride); break;
    }
}
template <int DSEL, bool CG>
__device__ __forceinline__ void sc_body_split_dsel(const ScProd &pd, gle r, gle acc[SC_NACC], const u64 L, const u32 tpl) {
    if constexpr (DSEL != 0) sc_body_split<DSEL, CG>(pd, r, acc, L, tpl);
    else switch (pd.d) {
    case 1: sc_body_split<1, CG>(pd, r, acc, L, tpl); break;
    case 2: sc_body_split<2, CG>(pd, r, acc, L, tpl); break;
    case 3: sc_body_split<3, CG>(pd, r, acc, L, tpl); break;
    case 4: sc_body_split<4, CG>(pd, r, acc, L, tpl); break;
    default: sc_body_split<5, CG>(pd, r, acc, L, tpl); break;
    }
}

// completion signal: `out` and `flag` live in mapped pinned host memory, so the round message reaches the host
// with the kernel's own stores -- no D2H copy node, and the host spins on the flag instead of a stream sync.
// Called by ONE thread after a block barrier that follows the message stores of its block mates: its system-scope fence
// orders those stores (observed through the barrier) before the flag.
__device__ __forceinline__ void sc_signal(u64 seq, u64 *flag, u32 *done) {
    if (gridDim.y == 1) { dp_publish(flag, seq); return; }
    __threadfence_system();
    u32 t = atomicAdd(done, 1u);
    if (t == gridDim.y - 1) { *done = 0; dp_publish(flag, seq); }
}

// Block + grid reduction of the per-thread accumulators of one product (blockIdx.y) and hand-over to the host:
// registers -> warp shuffles -> shared memory -> one partial per block; the last block to finish (ticket) adds the block
// partials.  Field addition is exact, so the summation order is free and the message is bit-identical to the reference's fold.
// The sums are LAZY: canonical limbs are added as plain 96-bit integers (add.cc / addc: 2 instructions and one carry of latency per
// step instead of a 9-instruction modular add) and reduced once per stage -- the reduction tree is the serial part of every round.
struct wsum96 { u64 lo; u32 hi; };
__device__ __forceinline__ void ws_add(wsum96 &a, u64 lo, u32 hi) { asm("{\n\tadd.cc.u64 %0, %0, %2;\n\taddc.u32 %1, %1, %3;\n\t}" : "+l"(a.lo), "+r"(a.hi) : "l"(lo), "r"(hi)); }
__device__ __forceinline__ u64 ws_reduce(const wsum96 &a) { return gl_reduce128(a.lo, (u64)a.hi); }
__device__ __forceinline__ void ws_warp_reduce(wsum96 &a) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) { u64 l = __shfl_down_sync(0xffffffffu, a.lo, d); u32 h = __shfl_down_sync(0xffffffffu, a.hi, d); ws_add(a, l, h); }
}
template <int BLOCK>
__device__ __forceinline__ void sc_epilogue(const gle (&acc)[SC_NACC], const int nacc, gle *__restrict__ partials, u32 *__restrict__ counters,
                                            gle *__restrict__ out, u64 seq, u64 *flag, u32 *done) {
    __shared__ u64 wlo[BLOCK / 32][SC_NACC][2];
    __shared__ u32 whi[BLOCK / 32][SC_NACC][2];
    __shared__ bool is_last;
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int t = 0; t < SC_NACC; t++) if (t < nacc) {
        wsum96 v0 = {acc[t].c0, 0}, v1 = {acc[t].c1, 0};
        ws_warp_reduce(v0); ws_warp_reduce(v1);
        if (lane == 0) { wlo[warp][t][0] = v0.lo; whi[warp][t][0] = v0.hi; wlo[warp][t][1] = v1.lo; whi[warp][t][1] = v1.hi; }
    }
    __syncthreads();
    if (threadIdx.x < 2 * nacc) {                     // thread (t, limb) adds the warps' sums and reduces once
        const u32 t = threadIdx.x >> 1, limb = threadIdx.x & 1;
        wsum96 v = {0, 0};
#pragma unroll
        for (int w = 0; w < BLOCK / 32; w++) ws_add(v, wlo[w][t][limb], whi[w][t][limb]);
        const u64 r = ws_reduce(v);
        u64 *dst = gridDim.x == 1 ? (u64 *)(out + (u64)blockIdx.y * SC_NACC + t) : (u64 *)(partials + ((u64)blockIdx.y * gridDim.x + blockIdx.x) * SC_NACC + t);
        dst[limb] = r;
    }
    if (gridDim.x == 1) { __syncthreads(); if (threadIdx.x == 0) sc_signal(seq, flag, done); return; }   // no cross-block stage
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        u32 ticket = atomicAdd(counters + blockIdx.y, 1u);
        is_last = (ticket == gridDim.x - 1);
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    // last block of this product: all threads add the block partials (independent L2 loads in flight), then the same tree
    wsum96 v[SC_NACC][2];
#pragma unroll
    for (int t = 0; t < SC_NACC; t++) { v[t][0] = {0, 0}; v[t][1] = {0, 0}; }
    for (u32 x = threadIdx.x; x < gridDim.x; x += BLOCK) {
        const gle *pp = partials + ((u64)blockIdx.y * gridDim.x + x) * SC_NACC;
#pragma unroll
        for (int t = 0; t < SC_NACC; t++) if (t < nacc) {
            ulonglong2 q = __ldcg(reinterpret_cast<const ulonglong2 *>(pp + t));
            ws_add(v[t][0], q.x, 0); ws_add(v[t][1], q.y, 0);
        }
    }
    __syncthreads();
#pragma unroll
    for (int t = 0; t < SC_NACC; t++) if (t < nacc) {
        ws_warp_reduce(v[t][0]); ws_warp_reduce(v[t][1]);
        if (lane == 0) { wlo[warp][t][0] = v[t][0].lo; whi[warp][t][0] = v[t][0].hi; wlo[warp][t][1] = v[t][1].lo; whi[warp][t][1] = v[t][1].hi; }
    }
    __syncthreads();
    if (threadIdx.x < 2 * nacc) {
        const u32 t = threadIdx.x >> 1, limb = threadIdx.x & 1;
        wsum96 w = {0, 0};
#pragma unroll
        for (int k = 0; k < BLOCK / 32; k++) ws_add(w, wlo[k][t][limb], whi[k][t][limb]);
        ((u64 *)(out + (u64)blockIdx.y * SC_NACC + t))[limb] = ws_reduce(w);
    }
    __syncthreads();
    if (threadIdx.x == 0) { counters[blockIdx.y] = 0; sc_signal(seq, flag, done); }
}

template <int DSEL>   // DSEL = 0: any degree (mixed-degree polynomials); 1..5: every product has this degree
__global__ void __launch_bounds__(SC_THREADS)
k_sc_round(const ScProd *__restrict__ descs, const __grid_constant__ ScProd desc0, gle r, gle *__restrict__ partials, u32 *__restrict__ counters,
           gle *__restrict__ out, u64 seq, u64 *flag, u32 *done) {
    __shared__ ScProd pd;
    {
        // single-product polynomials carry their descriptor in the kernel parameters; otherwise `descs` is mapped host
        // memory for small grids (no copy node) and a device copy for large ones (hundreds of CTAs each fetching 216 B
        // over PCIe was the dominant cost of large rounds: ncu r01b showed 44 % of stall cycles at this barrier)
        const u64 *s = descs ? (const u64 *)(descs + blockIdx.y) : (const u64 *)&desc0;
        u64 *d = (u64 *)&pd;
        for (int k = threadIdx.x; k < (int)(sizeof(ScProd) / 8); k += blockDim.x) d[k] = s[k];
    }
    __syncthreads();
    gle acc[SC_NACC];
#pragma unroll
    for (int t = 0; t < SC_NACC; t++) acc[t] = e_zero();
    const u64 gtid = (u64)blockIdx.x * blockDim.x + threadIdx.x, gstride = (u64)gridDim.x * blockDim.x;
    sc_body_dsel<DSEL, false>(pd, r, acc, gtid, gstride);
    sc_epilogue<SC_THREADS>(acc, DSEL != 0 ? DSEL + 1 : (int)pd.d + 1, partials, counters, out, seq, flag, done);
}

// ---- lean kernels for the rounds that move the bytes ---------------------------------------------------------------------
// Every operand of every product is in the SAME storage mode this round (all Base: the first round of a Base polynomial; all
// folding Base->Ext: its second round; all folding Ext->Ext: every later round; all Ext: the first round of an Ext polynomial)
// and every product has the same degree D in {2, 3}.  The mode and the degree are compile-time, so the body is a straight line
// of loads and multiply chains (no per-operand switch, 64-118 registers instead of 122 for everything), the products of the
// last multiplication are accumulated UNREDUCED in 160-bit (Base) / 2 x 160-bit (Ext) sums and reduced once per thread and
// evaluation point, and the block shape follows the measurements in tools/kbench.cu: Base rounds 256 threads x 2 pairs in
// flight (HBM-bound: 1.9 TB/s at nu = 20), folding rounds 128 threads x 1 pair (issue-bound: 122 instructions per E x E).
struct eacc { gl_acc c0, c1; };
__device__ __forceinline__ void eacc_mac(eacc &a, gle x, gle y) {   // a += x * y   (c1 = x0 y1 + x1 y0; c0 = x0 y0 + 7 w, w = weak(x1 y1))
    gl_acc_mac(a.c1, x.c0, y.c1); gl_acc_mac(a.c1, x.c1, y.c0);
    u64 w = gl_reduce128_weak(x.c1 * y.c1, __umul64hi(x.c1, y.c1));
    gl_acc_mac(a.c0, x.c0, y.c0); gl_acc_mac(a.c0, w, 7ULL);
}
template <int MODE> struct ScLeanShape { static constexpr int BLOCK = MODE == OPM_B ? 256 : 128, MINB = 4, PPT = MODE == OPM_B ? 2 : 1; };

template <int D, int MODE>
__global__ void __launch_bounds__(ScLeanShape<MODE>::BLOCK, ScLeanShape<MODE>::MINB)
k_sc_lean(const ScProd *__restrict__ descs, const __grid_constant__ ScProd desc0, gle r, gle *__restrict__ partials, u32 *__restrict__ counters,
          gle *__restrict__ out, u64 seq, u64 *flag, u32 *done) {
    constexpr int BLOCK = ScLeanShape<MODE>::BLOCK, PPT = ScLeanShape<MODE>::PPT;
    __shared__ ScProd pd;
    {
        const u64 *s = descs ? (const u64 *)(descs + blockIdx.y) : (const u64 *)&desc0;
        u64 *d = (u64 *)&pd;
        for (int k = threadIdx.x; k < (int)(sizeof(ScProd) / 8); k += BLOCK) d[k] = s[k];
    }
    __syncthreads();
    const u64 npairs = pd.npairs, T = (u64)gridDim.x * BLOCK;
    gle acc[SC_NACC];
#pragma unroll
    for (int t = 0; t < SC_NACC; t++) acc[t] = e_zero();
    if (MODE == OPM_B) {
        gl_acc a[D + 1];
#pragma unroll
        for (int t = 0; t <= D; t++) { a[t].lo = 0; a[t].hi = 0; a[t].top = 0; }
        const u64 *src[D];
#pragma unroll
        for (int j = 0; j < D; j++) src[j] = (const u64 *)pd.op[j].src;
        for (u64 i0 = (u64)blockIdx.x * BLOCK + threadIdx.x; i0 < npairs; i0 += PPT * T) {
            ulonglong2 v[PPT][D];
#pragma unroll
            for (int p = 0; p < PPT; p++) {
                u64 i = i0 + p * T; const bool ok = i < npairs; if (!ok) i = i0;
#pragma unroll
                for (int j = 0; j < D; j++) v[p][j] = ld_b2(src[j] + 2 * i);
                if (!ok) v[p][0] = make_ulonglong2(0, 0);          // a zero factor contributes nothing at every point
            }
#pragma unroll
            for (int p = 0; p < PPT; p++) {
                u64 c[D], s[D];
#pragma unroll
                for (int j = 0; j < D; j++) { c[j] = v[p][j].x; s[j] = gl_sub(v[p][j].y, v[p][j].x); }
#pragma unroll
                for (int t = 0; t <= D; t++) {
                    u64 q = c[0];
#pragma unroll
                    for (int j = 1; j < D - 1; j++) q = gl_mul_weak(q, c[j]);
                    gl_acc_mac(a[t], q, c[D - 1]);
                    if (t < D) {
#pragma unroll
                        for (int j = 0; j < D; j++) c[j] = gl_add(c[j], s[j]);
                    }
                }
            }
        }
#pragma unroll
        for (int t = 0; t <= D; t++) acc[t] = e_from_base(gl_acc_reduce(a[t]));
    } else {
        eacc a[D + 1];
#pragma unroll
        for (int t = 0; t <= D; t++) { a[t].c0 = {0, 0, 0}; a[t].c1 = {0, 0, 0}; }
        for (u64 i = (u64)blockIdx.x * BLOCK + threadIdx.x; i < npairs; i += T) {
            gle c[D], s[D];
#pragma unroll
            for (int j = 0; j < D; j++) {
                gle lo, hi;
                if (MODE == OPM_BF) {
                    const u64 *q = (const u64 *)pd.op[j].src + 4 * i;
                    ulonglong2 v0 = ld_b2(q), v1 = ld_b2(q + 2);
                    lo = fold_b(v0.x, v0.y, r); hi = fold_b(v1.x, v1.y, r);
                    if (pd.op[j].dst) { st_e(pd.op[j].dst + 2 * i, lo); st_e(pd.op[j].dst + 2 * i + 1, hi); }
                } else if (MODE == OPM_EF) {
                    const gle *q = (const gle *)pd.op[j].src + 4 * i;
                    gle f0 = ld_e(q), f1 = ld_e(q + 1), f2 = ld_e(q + 2), f3 = ld_e(q + 3);
                    lo = fold_e(f0, f1, r); hi = fold_e(f2, f3, r);
                    if (pd.op[j].dst) { st_e(pd.op[j].dst + 2 * i, lo); st_e(pd.op[j].dst + 2 * i + 1, hi); }
                } else {
                    const gle *q = (const gle *)pd.op[j].src + 2 * i;
                    lo = ld_e(q); hi = ld_e(q + 1);
                }
                c[j] = lo; s[j] = e_sub(hi, lo);
            }
#pragma unroll
            for (int t = 0; t <= D; t++) {
                gle q = c[0];
#pragma unroll
                for (int j = 1; j < D - 1; j++) q = e_mul(q, c[j]);
                eacc_mac(a[t], q, c[D - 1]);
                if (t < D) {
#pragma unroll
                    for (int j = 0; j < D; j++) c[j] = e_add(c[j], s[j]);
                }
            }
        }
#pragma unroll
        for (int t = 0; t <= D; t++) acc[t] = e_make(gl_acc_reduce(a[t].c0), gl_acc_reduce(a[t].c1));
    }
    sc_epilogue<BLOCK>(acc, D + 1, partials, counters, out, seq, flag, done);
}


// ---- resident rounds: every remaining round of a small sumcheck in ONE launch of a thread-block CLUSTER --------------------
// Once the tables are small a round is pure latency: launch + two-stage reduction + the host's Fiat-Shamir.  This kernel stays
// resident instead: up to 8 CTAs (one cluster: co-scheduled by the hardware, hardware barrier between them) split the pairs of
// every product by warp, the warp partials meet in a small global scratch, CTA 0 adds them, writes the round message to mapped
// host memory, raises the flag and polls a mapped mailbox for the next challenge (one thread, one PCIe read in flight); the
// challenge reaches the other CTAs through the cluster barrier.  A round costs the compute of its widest product spread over
// <= 2048 threads + two cluster barriers (~0.2 us each) + two PCIe hops + the host sponge -- no launch, no cross-block ticket
// stage, no cold instruction cache.  The folded tables ping-pong in HBM/L2 (the cluster barrier orders the stores; readers use
// L1-bypassing loads).  The per-round bookkeeping the host does for k_sc_round (operand order, fold destinations, ping-pong
// buffers) runs in every CTA's shared memory through the same functions (sc_desc, sc_commit_fold).  The kernel cannot hang: the poll gives up after
// SC_RES_TIMEOUT cycles or when the host posts the abort value, and the other CTAs only ever wait on the cluster barrier.
// Opt-in per handle (dp_sc_set_resident_tail): the caller promises not to wait on other work in the same stream between rounds.
static constexpr u32 SC_RES_MAXM = 96, SC_RES_MAXP = 48, SC_RES_MAXCTA = 8;
static constexpr u64 SC_RES_WORK = 2048;                     // resident once sum over products of (pairs this round) <= this (larger rounds are faster in the multi-block kernels; 2048 measured best of 1024 / 2048 / 4096 on H100)
static constexpr long long SC_RES_TIMEOUT = 6000000000LL;   // ~3 s at 1.9 GHz
static constexpr u64 SC_TAIL_ABORT = ~0ULL, SC_TAIL_FAILED = ~0ULL - 1;
static constexpr u32 SC_NO_WRITER = ~0u;

// Round state of one MLE, kept by the host for the per-round kernels and by every CTA of the resident kernel
struct ScMle {
    const void *cur; gle *work;   // work: [len0/2 + len0/4] E: ping (offset 0) / pong (offset len0/2)
    u64 len, len0;
    u32 is_ext, where;            // where: 0 = caller's input, 1 = ping, 2 = pong (3 = owned by the resident kernel)
};
__host__ __device__ inline gle *sc_fold_dst(const ScMle &m) { return m.where == 1 ? m.work + (m.len0 >> 1) : m.work; }
__host__ __device__ inline void sc_commit_fold(ScMle &m, gle *dst) { m.cur = dst; m.where = dst == m.work ? 1 : 2; m.len >>= 1; m.is_ext = 1; }

// Descriptor of product p this round.  fold[i] / dst[i]: MLE i halves this round into dst[i]; writer[i]: the product that stores
// the folded table (the first one referencing MLE i; its first operand on MLE i does the store).  The macro sorts Ext operands first
// (sumcheck_macro/src/lib.rs:87-140); multiplication commutes, so only operand 0 must be an Ext one when the product is mixed (the
// bodies multiply INTO it).
__host__ __device__ inline void sc_desc(ScProd &pd, u32 p, const u32 *idx, u32 n_idx, const ScMle *mles, const unsigned char *fold,
                                        gle *const *dst, const u32 *writer) {
    u32 order[5], c = 0;
    for (u32 j = 0; j < n_idx; j++) if (mles[idx[j]].is_ext || fold[idx[j]]) order[c++] = j;
    for (u32 j = 0; j < n_idx; j++) if (!(mles[idx[j]].is_ext || fold[idx[j]])) order[c++] = j;
    bool allbase = true; u64 newlen = 0;
    for (u32 jj = 0; jj < n_idx; jj++) {
        const u32 mi = idx[order[jj]]; const ScMle &m = mles[mi]; ScOp &op = pd.op[jj];
        op.src = m.cur; op.dst = nullptr;
        if (fold[mi]) {
            op.mode = m.is_ext ? OPM_EF : OPM_BF;
            bool first = writer[mi] == p;
            for (u32 q = 0; q < jj; q++) if (idx[order[q]] == mi) first = false;
            if (first) op.dst = dst[mi];
            newlen = m.len >> 1; allbase = false;
        } else { op.mode = m.is_ext ? OPM_E : OPM_B; newlen = m.len; if (m.is_ext) allbase = false; }
    }
    pd.d = n_idx; pd.allbase = allbase; pd.konst = newlen == 1; pd.npairs = newlen >> 1;
}

struct TProd { u32 n_idx; u32 idx[5]; };
// bary[d - 1][i][j]: weight of point j when a degree-d product's values at 0 .. d are extrapolated to point d + 1 + i (sc_bary)
typedef u64 ScBary[4][4][5];

// The glue of one product (prover.rs:694-724, sumcheck_macro/src/lib.rs:242): its d + 1 sums v[0..d] times the multiplicity
// 2^(max_nv - (l2 + R - 1)) of its MLEs' `len` entries in round R (l2 >= 1), times the coefficient, then extrapolated to v[0..max_deg].
// False: a negative multiplicity, which the host refuses (on the device dp_sc_create's num_vars bound rules it out).  The host's rounds
// (sc_glue) and the device transcript's (sc_res_fs_round) share it; on the device the multiply stays out of line (see e_mul_ni).
__host__ __device__ inline gle sc_glue_mul(gle a, gle b) {
#ifdef __CUDA_ARCH__
    return e_mul_ni(a, b);
#else
    return e_mul(a, b);
#endif
}
__host__ __device__ inline bool sc_glue_product(gle *v, u32 d, u64 len, u32 max_nv, u32 R, gle coef, u32 max_deg, const ScBary &bary) {
    u32 l2 = 1; while ((1ULL << l2) < len) l2++;
    const int mult = (int)max_nv - (int)(l2 + R - 1);
    const u64 scale = gl_canon(1ULL << (mult > 0 ? mult : 0));
    for (u32 t = 0; t <= d; t++) { gle x = v[t]; if (mult > 0) x = e_mul_base(x, scale); v[t] = sc_glue_mul(x, coef); }
    for (u32 i = 0; d + 1 + i <= max_deg; i++) {
        gle x = e_zero();
        for (u32 j = 0; j <= d; j++) x = e_add(x, e_mul_base(v[j], bary[d - 1][i][j]));
        v[d + 1 + i] = x;
    }
    return mult >= 0;
}

// Fiat-Shamir in the resident kernels (dp_sc_run_tail_fs[_blake], dp_logup_run_layers_fs[_blake]): what the glue and the transcript need
static constexpr u32 SC_MAX_ROUNDS = 40;
// sponge: the transcript's state, the larger of the two images (TrP2: P2S_WORDS, TrB3: DP_B3T_WORDS)
static constexpr int SC_FS_WORDS = DP_B3T_WORDS;
static_assert(P2S_WORDS <= SC_FS_WORDS && DP_B3T_WORDS == (int)dpb3::IMAGE_WORDS && DP_B3T_STACK == (int)dpb3::IMAGE_STACK &&
              DP_B3T_STACK == (int)b3::T_STACK_MAX && DP_B3T_WORDS == TrB3::WORDS, "one BLAKE3 state image");
struct ScTailFs { u32 max_deg, max_nv, round0, pad; u64 label[2]; u64 coef[SC_RES_MAXP][2]; ScBary bary; u64 sponge[SC_FS_WORDS]; };
struct ScTailFsOut { gle msg[SC_MAX_ROUNDS][SC_NACC]; gle chal[SC_MAX_ROUNDS]; u64 sponge[SC_FS_WORDS]; };
struct ScTail { u32 n_mles, n_products, n_rounds, first_has_challenge; ScMle m[SC_RES_MAXM]; u32 writer[SC_RES_MAXM]; TProd p[SC_RES_MAXP]; ScTailFs fs; };

__device__ __forceinline__ u32 cl_rank() { u32 r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ u32 cl_size() { u32 r; asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r)); return r; }
// all threads of all CTAs of the cluster; release/acquire at cluster scope (global stores before it are visible after it)
__device__ __forceinline__ void cl_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// Round k of the device-transcript tail, in CTA 0 once the product sums are in sprod and this round's folds are committed to sm:
// the glue (one thread per product, on the lengths the host's bookkeeping has after the fold), the sum over products, then the
// transcript TR (TrP2 or TrB3) -- append_field_element_exts(message), get_and_append_challenge("Internal round") -- and the challenge
// goes to xctl for the cluster.  Out of line: the round loop keeps its registers (transcript state in shared memory between rounds).
template <class TR>
__device__ __noinline__ void sc_res_fs_round(ScTailFs &f, gle (*sprod)[SC_NACC], const TProd *sp, const ScMle *sm, u32 np, u32 k, bool last,
                                             ScTailFsOut *fsout, u64 *xctl) {
    const u32 R = f.round0 + k + 1, max_deg = f.max_deg;
    for (u32 p = threadIdx.x; p < np; p += blockDim.x)
        sc_glue_product(sprod[p], sp[p].n_idx, sm[sp[p].idx[0]].len, f.max_nv, R, e_make(f.coef[p][0], f.coef[p][1]), max_deg, f.bary);
    __syncthreads();
    for (u32 t = threadIdx.x; t <= max_deg; t += blockDim.x) {
        gle v = e_zero();
        for (u32 p = 0; p < np; p++) v = e_add(v, sprod[p][t]);
        sprod[0][t] = v;                                         // column t is read and written by this thread only
        st_e(&fsout->msg[k][t], v);
    }
    __syncthreads();
    if (TR::runs()) {
        TR t(f.sponge);
        for (u32 i = 0; i <= max_deg; i++) t.ext(sprod[0][i]);
        t.label(f.label);
        const gle c = t.challenge();
        t.store(f.sponge, last ? fsout->sponge : nullptr);
        if (threadIdx.x == 0) { __stcg(xctl + 1, c.c0); __stcg(xctl + 2, c.c1); __stcg(xctl, 0ULL); st_e(&fsout->chal[k], c); }
    }
}

// Shared-memory round state of the resident kernels (every CTA keeps its own copy of the bookkeeping)
struct ScResSmem {
    ScMle sm[SC_RES_MAXM]; TProd sp[SC_RES_MAXP]; ScProd spd[SC_RES_MAXP]; gle *sdst[SC_RES_MAXM]; u32 swriter[SC_RES_MAXM];
    unsigned char sfold[SC_RES_MAXM];
    gle sprod[SC_RES_MAXP][SC_NACC];                                   // device transcript: each product's sums
    ScTailFs sfs;
};

// The rounds of one sumcheck on the cluster, from the bookkeeping in S (nm MLEs, np products, nr rounds; first_fold: round 0 folds
// by r first).  Returns early when the host aborted the tail or a challenge never came.  After the last round the tables' pairs go to
// `pairs` and the flag is raised -- unless CHAIN (one of several sumchecks in a launch, device transcript): then every CTA records
// the challenges of rounds 0 .. nr - 2 in schal (shared) and the caller does what follows the last round.
template <int DSEL, bool CHAIN, class TR>
__device__ __forceinline__ void sc_res_rounds(ScResSmem &S, const u32 nm, const u32 np, const u32 nr, const bool first_fold, gle r,
                                              gle *out, gle *pairs, volatile u64 *flag, volatile u64 *chal, u64 seq0, gle *xpart, u64 *xctl,
                                              ScTailFsOut *fsout, gle *schal) {
    const bool fs = fsout != nullptr;
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = SC_THREADS / 32;
    const u32 rank = cl_rank(), ncta = cl_size();
    const u32 W = ncta * nwarps, gw = rank * nwarps + warp;              // warps of the cluster, this warp's index
    // pairs of a product are split over G warps (G a power of two, np * G <= W); with more products than warps a warp takes several
    u32 G = 1; while (np * (G << 1) <= W) G <<= 1;
    // The descriptors of a round depend on the fold bookkeeping only, never on the challenge VALUE: they are rebuilt right after a
    // round's message has been signalled, i.e. in the shadow of the host's Fiat-Shamir, which keeps ~2.2 us per round off the path
    // from the challenge's arrival to the first load.
    auto build_descs = [&](const bool fold) {
        for (u32 i = threadIdx.x; i < nm; i += blockDim.x) {
            bool f = fold && S.sm[i].len > 1;
            S.sfold[i] = f;
            S.sdst[i] = f ? sc_fold_dst(S.sm[i]) : nullptr;
        }
        __syncthreads();
        for (u32 p = threadIdx.x; p < np; p += blockDim.x) sc_desc(S.spd[p], p, S.sp[p].idx, S.sp[p].n_idx, S.sm, S.sfold, S.sdst, S.swriter);
        __syncthreads();
    };
    build_descs(first_fold);
    for (u32 k = 0; k < nr; k++) {
        const u64 seq = seq0 + k;
        if (k > 0) {   // wait for the host's challenge for this round (device transcript: CTA 0 posted it to xctl last round)
            if (rank == 0 && threadIdx.x == 0 && !fs) {
                long long t0 = clock64(); u64 v, status = 0;
                while ((v = chal[0]) != seq) {
                    if (v == SC_TAIL_ABORT) { status = 1; break; }
                    if (clock64() - t0 > SC_RES_TIMEOUT) { status = 2; break; }
                }
                u64 c0 = 0, c1 = 0;
                if (!status) { __threadfence_system(); c0 = chal[1]; c1 = chal[2]; }
                __stcg(xctl + 1, c0); __stcg(xctl + 2, c1); __stcg(xctl, status);
            }
            cl_sync();
            const u64 status = __ldcg(xctl);
            if (status) { if (rank == 0 && threadIdx.x == 0 && status == 2) dp_publish(flag, SC_TAIL_FAILED); return; }   // uniform over the cluster
            r = e_make(__ldcg(xctl + 1), __ldcg(xctl + 2));
            if (CHAIN && threadIdx.x == 0) schal[k - 1] = r;
        }
        // work: slot (p, s) = sub-slice s of product p's pairs; warp gw owns slots gw, gw + W, ...
        for (u32 slot = gw; slot < np * G; slot += W) {
            const u32 p = slot / G, s = slot % G;
            const ScProd &pd = S.spd[p];
            gle acc[SC_NACC];
#pragma unroll
            for (int t = 0; t < SC_NACC; t++) acc[t] = e_zero();
            const u64 first = (u64)s * 32 + lane, stride = (u64)G * 32;
            const u32 tpl = pd.d <= 3 ? 2 : 3;
            const bool split = !pd.konst && !pd.allbase && (pd.npairs << tpl) <= stride;     // uniform over the warps of this product
            if (split) sc_body_split_dsel<DSEL, true>(pd, r, acc, first, tpl);
            else sc_body_dsel<DSEL, true>(pd, r, acc, first, stride);
            const int nacc = DSEL != 0 ? DSEL + 1 : (int)pd.d + 1;
#pragma unroll
            for (int t = 0; t < SC_NACC; t++) if (t < nacc) {     // lazy 96-bit warp sums, one reduction per limb (see sc_epilogue)
                wsum96 v0 = {acc[t].c0, 0}, v1 = {acc[t].c1, 0};
                ws_warp_reduce(v0); ws_warp_reduce(v1);
                if (lane == 0) __stcg(reinterpret_cast<ulonglong2 *>(xpart + (u64)slot * SC_NACC + t), make_ulonglong2(ws_reduce(v0), ws_reduce(v1)));
            }
        }
        cl_sync();                                             // warp partials and folded tables of every CTA are visible
        if (rank == 0) {                                       // the message first: it is what the host is waiting for
            gle *const mout = fs ? &S.sprod[0][0] : out;
            // few partials per (product, point): one THREAD each (many products run side by side); many (a single product spread over
            // >= 32 warps): one WARP each, its lanes gather the partials with independent L2 loads -- faster for a single wide product,
            // while the warp form slows the 6-product LogUp shape
            if (G < 32) {
                for (u32 x = threadIdx.x; x < np * SC_NACC; x += blockDim.x) {
                    const u32 p = x / SC_NACC, t = x % SC_NACC;
                    if (t > S.spd[p].d) continue;
                    gle v = e_zero();
                    for (u32 s = 0; s < G; s++) { ulonglong2 q = __ldcg(reinterpret_cast<const ulonglong2 *>(xpart + ((u64)p * G + s) * SC_NACC + t)); v = e_add(v, e_make(q.x, q.y)); }
                    st_e(mout + (u64)p * SC_NACC + t, v);
                }
            } else
            for (u32 x = warp; x < np * SC_NACC; x += nwarps) {
                const u32 p = x / SC_NACC, t = x % SC_NACC;
                if (t > S.spd[p].d) continue;                  // warp-uniform
                wsum96 v0 = {0, 0}, v1 = {0, 0};
                for (u32 s = lane; s < G; s += 32) { ulonglong2 q = __ldcg(reinterpret_cast<const ulonglong2 *>(xpart + ((u64)p * G + s) * SC_NACC + t)); ws_add(v0, q.x, 0); ws_add(v1, q.y, 0); }
                ws_warp_reduce(v0); ws_warp_reduce(v1);
                if (lane == 0) st_e(mout + (u64)p * SC_NACC + t, e_make(ws_reduce(v0), ws_reduce(v1)));
            }
        }
        for (u32 i = threadIdx.x; i < nm; i += blockDim.x) if (S.sfold[i]) sc_commit_fold(S.sm[i], S.sdst[i]);   // every CTA keeps its own copy
        __syncthreads();
        if (rank == 0 && fs) sc_res_fs_round<TR>(S.sfs, S.sprod, S.sp, S.sm, np, k, k == nr - 1, fsout, xctl);
        if (rank == 0 && !CHAIN) {
            if (k == nr - 1) {   // last round: hand the (<= 2)-entry tables over with the message (k_sc_gather's job)
                for (u32 i = threadIdx.x; i < nm; i += blockDim.x) {
                    const ScMle &m = S.sm[i]; gle a, b;
                    if (m.is_ext) { a = ldx_e<true>((const gle *)m.cur); b = m.len > 1 ? ldx_e<true>((const gle *)m.cur + 1) : a; }
                    else { a = e_from_base(ldx_b<true>((const u64 *)m.cur)); b = m.len > 1 ? e_from_base(ldx_b<true>((const u64 *)m.cur + 1)) : a; }
                    st_e(pairs + 2 * i, a); st_e(pairs + 2 * i + 1, b);
                }
                __syncthreads();
            }
            if (threadIdx.x == 0 && (!fs || k == nr - 1)) dp_publish(flag, seq);   // device transcript: once, at the end
        }
        if (k + 1 < nr) build_descs(true);                     // next round's descriptors while the host hashes
        // CTAs other than 0 run ahead to the next cluster barrier; xpart is not rewritten before it (the work phase follows it)
    }
}

template <int DSEL, class TR>   // TR: the device transcript when fsout is not null (TrP2 serves the host-transcript launches too)
__global__ void __launch_bounds__(SC_THREADS)
k_sc_res(const ScTail *__restrict__ cfg, gle r0, gle *out /* mapped */, gle *pairs /* mapped */, volatile u64 *flag /* mapped */,
         volatile u64 *chal /* mapped: [seq, c0, c1] */, u64 seq0, gle *xpart /* device: warp partials */, u64 *xctl /* device: [status, c0, c1] */,
         ScTailFsOut *fsout /* mapped; null: the host runs the transcript between rounds */) {
    __shared__ ScResSmem S;
    const u32 nm = cfg->n_mles, np = cfg->n_products, nr = cfg->n_rounds;
    const u32 rank = cl_rank();
    for (u32 i = threadIdx.x; i < nm; i += blockDim.x) { S.sm[i] = cfg->m[i]; S.swriter[i] = cfg->writer[i]; }
    for (u32 i = threadIdx.x; i < np; i += blockDim.x) S.sp[i] = cfg->p[i];
    if (fsout && rank == 0)
        for (u32 i = threadIdx.x; i < sizeof(ScTailFs) / 8; i += blockDim.x) ((u64 *)&S.sfs)[i] = ((const u64 *)&cfg->fs)[i];
    __syncthreads();
    sc_res_rounds<DSEL, false, TR>(S, nm, np, nr, cfg->first_has_challenge != 0, r0, out, pairs, flag, chal, seq0, xpart, xctl, fsout, nullptr);
}

// ---- the small layers of a LogUp-GKR batch, back to back in ONE resident launch (dp_logup_run_layers_fs) --------------------------
// logup_gkr::prover::batch_prove (prover.rs:24-237) layer by layer, with the transcript TR on the device: per layer CTA 0 absorbs the
// claim, num_vars and the degree (prove_parallel), every CTA builds its slice of the layer's eq table from the point and the layer's
// bookkeeping (the products of zkml.hpp's logup_batch_prove), the rounds run through sc_res_rounds, and CTA 0 folds the final
// evaluations, squeezes logup_batching / logup_alpha / logup_lambda and forms the next claim and point.  The host sleeps once per call
// instead of once per layer, and no eq table, sumcheck handle or launch is made per layer.
static constexpr u32 LG_MAXC = 16, LG_MAXL = 12;
struct LgCfg {
    u32 n_circuits, first, n_layers, pad;
    gle claim, alpha, lambda;
    gle point[SC_MAX_ROUNDS + 1];                                  // layer `first`'s point (its last entry is the batching challenge)
    const gle *num[LG_MAXL][LG_MAXC], *den[LG_MAXL][LG_MAXC];     // layer first + l of circuit c: [lo | hi]; num null: numerators all -1
    gle *eq, *work; u64 work_stride;                               // device scratch: the eq table, each MLE's ping-pong tables
    u64 label[3][2];                                               // "logup_batching", "logup_alpha", "logup_lambda"
    ScTailFs fs;                                                   // the rounds' transcript; coef and max_nv are set per layer
};
struct LgLayerOut { ScTailFsOut fs; gle evals[SC_RES_MAXM]; };
struct LgOut { LgLayerOut layer[LG_MAXL]; gle point[SC_MAX_ROUNDS + 1]; gle claim, alpha, lambda; u64 sponge[SC_FS_WORDS]; u64 flag; };

// state of the layer loop in shared memory: kept out of registers across the rounds, which need all of theirs
struct LgSmem { gle pt[SC_MAX_ROUNDS + 1], fe[SC_RES_MAXM], claim, alpha, lambda, batching; u32 v, nm, per, two; };

// layer l's start: its transcript prefix and coefficients (CTA 0), eq table slice and bookkeeping (every CTA)
template <class TR>
__device__ __noinline__ void lg_layer_begin(const LgCfg *cfg, ScResSmem &S, LgSmem &L, const u32 l, const gle *xpoint) {
    const u32 rank = cl_rank(), ncta = cl_size(), nc = cfg->n_circuits, np = 3 * nc;
    const u32 v = cfg->first + l;
    const u64 half = 1ULL << v;
    const bool two = cfg->num[l][0] == nullptr;                    // the lookup circuit's first layer: views [den_lo, den_hi]
    const u32 per = two ? 2 : 4, nm = 1 + per * nc;
    for (u32 i = threadIdx.x; i < v; i += blockDim.x) L.pt[i] = l == 0 ? cfg->point[i] : ldx_e<true>(xpoint + i);
    if (rank == 0) {
        for (u32 p = threadIdx.x; p < np; p += blockDim.x) {       // coefficients: alpha^c x (1, 1, lambda), or (-1, -1, lambda)
            gle cur = e_one();
            for (u32 c = 0; c < p / 3; c++) cur = e_mul_ni(cur, L.alpha);
            const gle cf = p % 3 == 2 ? e_mul_ni(cur, L.lambda) : two ? e_neg(cur) : cur;
            S.sfs.coef[p][0] = cf.c0; S.sfs.coef[p][1] = cf.c1;
        }
        if (TR::runs()) {                                          // t.append_field_element_ext(claim); append_usize(nv); append_usize(deg)
            TR t(S.sfs.sponge);
            t.ext(L.claim); t.usize(v); t.usize(3);
            t.store(S.sfs.sponge, nullptr);
        }
        if (threadIdx.x == 0) S.sfs.max_nv = v;
    }
    if (threadIdx.x == 0) { L.v = v; L.nm = nm; L.per = per; L.two = two; }
    __syncthreads();
    for (u64 x = (u64)rank * blockDim.x + threadIdx.x; x < half; x += (u64)ncta * blockDim.x) {   // build_eq_x_r(point)
        gle p = e_one();
        for (u32 b = 0; b < v; b++) p = e_mul_ni(p, ((x >> b) & 1) ? L.pt[b] : e_sub(e_one(), L.pt[b]));
        __stcg(reinterpret_cast<ulonglong2 *>(cfg->eq + x), make_ulonglong2(p.c0, p.c1));
    }
    // MLE order of VirtualPolynomial::add_mle_list: eq, then per circuit its views in first use, [num_lo, den_hi, num_hi, den_lo]
    // ([den_hi, den_lo] with two views); writer = the first product using the MLE
    for (u32 i = threadIdx.x; i < nm; i += blockDim.x) {
        ScMle m; m.len = m.len0 = half; m.is_ext = 1; m.where = 0; m.work = cfg->work + i * cfg->work_stride;
        u32 w = 0;
        if (i == 0) m.cur = cfg->eq;
        else {
            const u32 c = (i - 1) / per, j = (i - 1) % per;
            const gle *nu = cfg->num[l][c], *de = cfg->den[l][c];
            if (two) { m.cur = j == 0 ? de + half : de; w = 3 * c + j; }
            else { m.cur = j == 0 ? nu : j == 1 ? de + half : j == 2 ? nu + half : de; w = 3 * c + (j < 2 ? 0 : 1); }
        }
        S.sm[i] = m; S.swriter[i] = w;
    }
    for (u32 p = threadIdx.x; p < np; p += blockDim.x) {
        const u32 b = 1 + per * (p / 3), q = p % 3;
        TProd t = {};
        if (two) { t.n_idx = q == 2 ? 3 : 2; t.idx[0] = 0; t.idx[1] = q == 0 ? b : b + 1; t.idx[2] = b; }
        else { t.n_idx = 3; t.idx[0] = 0; t.idx[1] = q == 0 ? b : q == 1 ? b + 2 : b + 3; t.idx[2] = q == 0 ? b + 1 : q == 1 ? b + 3 : b + 1; }
        S.sp[p] = t;
    }
    __syncthreads();
}

// layer l's end in CTA 0: get_mle_final_evaluations, logup_batching / logup_alpha / logup_lambda, the next claim and point (zkml.hpp)
template <class TR>
__device__ __noinline__ void lg_layer_end(const LgCfg *cfg, LgOut *out, ScResSmem &S, LgSmem &L, const u32 l, const u64 *xctl, gle *xpoint) {
    const u32 v = L.v, nm = L.nm, per = L.per, nc = cfg->n_circuits;
    const bool two = L.two;
    const gle rl = e_make(__ldcg(xctl + 1), __ldcg(xctl + 2));    // the last round's challenge
    for (u32 i = 1 + threadIdx.x; i < nm; i += blockDim.x) {
        const gle *t = (const gle *)S.sm[i].cur, a = ldx_e<true>(t), b = ldx_e<true>(t + 1);
        const gle f = e_add(a, e_mul_ni(e_sub(b, a), rl));
        L.fe[i] = f; st_e(&out->layer[l].evals[i - 1], f);
    }
    __syncthreads();
    if (TR::runs()) {
        TR t(S.sfs.sponge);
        gle ch[3];
        for (int q = 0; q < 3; q++) { t.label(cfg->label[q]); ch[q] = t.challenge(); }
        t.store(S.sfs.sponge, nullptr);
        if (threadIdx.x == 0) {
            const gle bt = ch[0], al = ch[1], lm = ch[2];
            gle acc = e_zero(), a = e_one();
            for (u32 c = 0; c < nc; c++) {
                const gle *e = &L.fe[1 + per * c];
                const gle term = two ? e_add(e_mul_ni(bt, e_sub(e[0], e[1])), e[1])
                                     : e_add(e_add(e_mul_ni(bt, e_sub(e[2], e[0])), e[0]), e_mul_ni(lm, e_add(e_mul_ni(bt, e_sub(e[1], e[3])), e[3])));
                acc = e_add(acc, e_mul_ni(a, term)); a = e_mul_ni(a, al);
            }
            L.claim = acc; L.batching = bt; L.alpha = al; L.lambda = lm;
            L.pt[v - 1] = rl;                                      // rounds 0 .. v - 2 recorded theirs
        }
    }
    __syncthreads();
    const bool last = l + 1 == cfg->n_layers;
    for (u32 i = threadIdx.x; i <= v; i += blockDim.x) {           // point = sumcheck challenges || batching
        const gle x = i < v ? L.pt[i] : L.batching;
        __stcg(reinterpret_cast<ulonglong2 *>(xpoint + i), make_ulonglong2(x.c0, x.c1));
        if (last) st_e(&out->point[i], x);
    }
    if (last) {
        for (u32 i = threadIdx.x; i < TR::WORDS; i += blockDim.x) out->sponge[i] = S.sfs.sponge[i];
        if (threadIdx.x == 0) { st_e(&out->claim, L.claim); st_e(&out->alpha, L.alpha); st_e(&out->lambda, L.lambda); }
        __syncthreads();
        if (threadIdx.x == 0) dp_publish(&out->flag, 1);
    }
}

template <class TR>
__global__ void __launch_bounds__(SC_THREADS)
k_logup_res(const LgCfg *__restrict__ cfg, LgOut *out /* mapped */, gle *xpart, u64 *xctl, gle *xpoint /* device */) {
    __shared__ ScResSmem S;
    __shared__ LgSmem L;
    if (cl_rank() == 0) {
        if (threadIdx.x == 0) { L.alpha = cfg->alpha; L.lambda = cfg->lambda; L.claim = cfg->claim; }
        for (u32 i = threadIdx.x; i < sizeof(ScTailFs) / 8; i += blockDim.x) ((u64 *)&S.sfs)[i] = ((const u64 *)&cfg->fs)[i];
    }
    __syncthreads();                                               // the copied state is complete before lg_layer_begin reads and writes it
    for (u32 l = 0; l < cfg->n_layers; l++) {
        lg_layer_begin<TR>(cfg, S, L, l, xpoint);
        cl_sync();                                                 // the eq table of every CTA is visible
        sc_res_rounds<0, true, TR>(S, L.nm, 3 * cfg->n_circuits, L.v, false, e_zero(), nullptr, nullptr, nullptr, nullptr, 0, xpart, xctl, &out->layer[l].fs, L.pt);
        if (cl_rank() == 0) { __syncthreads(); lg_layer_end<TR>(cfg, out, S, L, l, xctl, xpoint); }
        cl_sync();                                                 // the next point is visible; every read of this layer's tables is done
    }
}

struct ScFin { const void *src; u32 mode; u32 len; };
// after the LAST round every MLE has <= 2 entries: copy them out with the round message so the closing fold
// (prover.rs:544-568) needs no further device round trip
__global__ void k_sc_gather(const ScFin *__restrict__ f, u32 n, gle *__restrict__ out /* 2 per MLE */) {
    u32 m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= n) return;
    ScFin d = f[m];
    gle a, b = e_zero();
    if (d.mode == OPM_E) { const gle *s = (const gle *)d.src; a = ld_e(s); if (d.len > 1) b = ld_e(s + 1); }
    else { const u64 *s = (const u64 *)d.src; a = e_from_base(s[0]); if (d.len > 1) b = e_from_base(s[1]); }
    st_e(out + 2 * m, a); st_e(out + 2 * m + 1, b);
}

// ---------------------------------------------------------------------------------------------------
struct dp_sc {
    u32 n_mles = 0, n_products = 0, max_nv = 0, max_deg = 0, round = 0;
    bool finished = false;
    std::vector<ScMle> mles;
    std::vector<u32> writer;                              // per MLE: the product that stores its folded tables (SC_NO_WRITER: none)
    std::vector<dp_sc_product> products;
    ScProd *d_descs = nullptr, *h_descs = nullptr;
    gle *d_partials = nullptr, *d_out = nullptr, *h_out = nullptr;
    u32 *d_counters = nullptr; bool counters_pooled = false, round_in_flight = false;
    ScFin *d_fin = nullptr, *h_fin = nullptr;
    gle *h_pairs = nullptr; bool have_pairs = false;
    u64 seq = 0; u64 *h_flag = nullptr; u32 *d_done = nullptr;
    int gx = 1;
    bool tail_enabled = false, tail_active = false;
    ScTail *h_tail = nullptr; u64 *h_chal = nullptr; ScTailFsOut *h_fs = nullptr;
    gle *d_xpart = nullptr; u64 *d_xctl = nullptr;        // resident cluster kernel: warp partials, [status, c0, c1]
    std::vector<gle> challenges;
};

// The weights of ScBary for every degree up to 5 (dp_sc_create's bound): barycentric extrapolation, sumcheck/src/util.rs:19-136 (exact
// arithmetic, so plain Lagrange gives the same element).  Built once per process.
static const ScBary &sc_bary() {
    static const struct Tab {
        ScBary w = {};
        Tab() {
            for (u32 d = 1; d <= 4; d++)
                for (u32 i = 0; d + 1 + i <= 5; i++)
                    for (u32 j = 0; j <= d; j++) {
                        u64 num = 1, den = 1;
                        for (u32 q = 0; q <= d; q++) if (q != j) { num = gl_mul(num, gl_sub(d + 1 + i, q)); den = gl_mul(den, gl_sub(j, q)); }
                        w[d - 1][i][j] = gl_mul(num, gl_inv(den));
                    }
        }
    } tab;
    return tab.w;
}

static int sc_free_all(dp_sc *s) {
    for (auto &m : s->mles) if (m.work) { dp_dev_free(m.work); m.work = nullptr; }
    dp_dev_free(s->d_descs); dp_dev_free(s->d_partials); dp_dev_free(s->d_out); dp_dev_free(s->d_fin);
    if (s->counters_pooled && !s->round_in_flight) dp_zero_block_put(s->d_counters); else dp_dev_free(s->d_counters);   // a round that never signalled may have left tickets behind
    dp_dev_free(s->d_xpart); dp_dev_free(s->d_xctl);
    dp_pinned_free(s->h_flag);
    dp_pinned_free(s->h_descs); dp_pinned_free(s->h_out); dp_pinned_free(s->h_fin); dp_pinned_free(s->h_pairs);
    dp_pinned_free(s->h_tail); dp_pinned_free(s->h_chal); dp_pinned_free(s->h_fs);
    return DP_OK;
}

// host glue: every product's sums through sc_glue_product, summed over products (prover.rs:694-733)
static int sc_glue(dp_sc *s, uint64_t *out_evals) {
    gle msg[SC_NACC];
    for (u32 t = 0; t <= s->max_deg; t++) msg[t] = e_zero();
    for (u32 p = 0; p < s->n_products; p++) {
        const dp_sc_product &pr = s->products[p];
        gle v[SC_NACC];
        for (u32 t = 0; t <= pr.n_idx; t++) v[t] = s->h_out[p * SC_NACC + t];
        DP_CHECK(sc_glue_product(v, pr.n_idx, s->mles[pr.idx[0]].len, s->max_nv, s->round, e_make(pr.coef[0], pr.coef[1]), s->max_deg, sc_bary()),
                 DP_ERR_INVALID, "dp_sc_round: negative num_vars multiplicity");
        for (u32 t = 0; t <= s->max_deg; t++) msg[t] = e_add(msg[t], v[t]);
    }
    for (u32 t = 0; t <= s->max_deg; t++) { out_evals[2 * t] = msg[t].c0; out_evals[2 * t + 1] = msg[t].c1; }
    return DP_OK;
}

// Can a resident kernel talk to the host while it runs?  Not under tools that serialise launches (Nsight Compute blocks the
// launching thread until the profiled kernel has finished, so the kernel would wait for a challenge its host cannot post).
// Checked once per process: known injection environments are refused outright, otherwise a one-thread probe kernel waits
// (<= ~50 ms) for a word the host posts right after the launch call returns.
__global__ void k_tail_probe(volatile u64 *mailbox, volatile u64 *result, long long limit_cycles) {
    long long t0 = clock64(); u64 ok = 2;
    while (clock64() - t0 < limit_cycles) { if (mailbox[0] == 1) { ok = 1; break; } }
    dp_publish(result, ok);
}
static bool sc_tail_supported() {
    static std::once_flag once; static bool supported = false;
    std::call_once(once, [] {
        if (getenv("CUDA_INJECTION64_PATH") || getenv("CUDA_INJECTION32_PATH") || getenv("NV_NSIGHT_INJECTION_TRANSPORT_TYPE") ||
            getenv("NV_NSIGHT_INJECTION_PORT_BASE") || getenv("NV_COMPUTE_PROFILER_PERFWORKS_DIR")) return;
        u64 *pin = nullptr;
        if (dp_pinned_alloc((void **)&pin, 128) != DP_OK) return;
        pin[0] = 0; pin[8] = 0;
        cudaStream_t st = dp_ctx().stream;
        if (dp_launch(k_tail_probe, 1, 1, 0, st, pin, pin + 8, 100000000LL) == cudaSuccess) {
            __atomic_store_n(&pin[0], (u64)1, __ATOMIC_RELEASE);      // reached at once unless the launch call itself waits for the kernel
            if (dp_stream_sync(st) == cudaSuccess) supported = (pin[8] == 1);
        }
        dp_pinned_free(pin);
    });
    return supported;
}

// ---- resident rounds, host side ----
// total pair-items of the round that would start the resident kernel (every product's pairs after this round's fold)
static u64 sc_round_work(const dp_sc *s, bool fold) {
    u64 work = 0;
    for (auto &pr : s->products) { const ScMle &m = s->mles[pr.idx[0]]; u64 nl = (fold && m.len > 1) ? m.len >> 1 : m.len; work += std::max<u64>(nl >> 1, 1); }
    return work;
}
static bool sc_tail_eligible(const dp_sc *s, bool fold) {
    if (!s->tail_enabled || s->n_mles > SC_RES_MAXM || s->n_products > SC_RES_MAXP || s->max_nv - s->round < 2) return false;
    for (u32 i = 0; i < s->n_mles; i++) if (s->writer[i] == SC_NO_WRITER && s->mles[i].len > 1) return false;
    return sc_round_work(s, fold) <= SC_RES_WORK;
}
// the kernels by DSEL (0: mixed degrees, 1..5: every product has this degree) and the lean ones by [MODE][D - 2]
// [blake][DSEL]: k_sc_res with BasicTranscript (also every host-transcript launch) or BlakeTranscript on the device
static decltype(&k_sc_res<0, TrP2>) const k_sc_res_dsel[2][6] = {
    {k_sc_res<0, TrP2>, k_sc_res<1, TrP2>, k_sc_res<2, TrP2>, k_sc_res<3, TrP2>, k_sc_res<4, TrP2>, k_sc_res<5, TrP2>},
    {k_sc_res<0, TrB3>, k_sc_res<1, TrB3>, k_sc_res<2, TrB3>, k_sc_res<3, TrB3>, k_sc_res<4, TrB3>, k_sc_res<5, TrB3>}};
static decltype(&k_sc_round<0>) const k_sc_round_dsel[6] = {k_sc_round<0>, k_sc_round<1>, k_sc_round<2>, k_sc_round<3>, k_sc_round<4>, k_sc_round<5>};
static decltype(&k_sc_round<0>) const k_sc_lean_md[4][2] = {{k_sc_lean<2, OPM_B>, k_sc_lean<3, OPM_B>}, {k_sc_lean<2, OPM_E>, k_sc_lean<3, OPM_E>},
                                                              {k_sc_lean<2, OPM_BF>, k_sc_lean<3, OPM_BF>}, {k_sc_lean<2, OPM_EF>, k_sc_lean<3, OPM_EF>}};
static constexpr int SC_LEAN_BLOCK[4] = {ScLeanShape<OPM_B>::BLOCK, ScLeanShape<OPM_E>::BLOCK, ScLeanShape<OPM_BF>::BLOCK, ScLeanShape<OPM_EF>::BLOCK};

// The cluster of a resident launch whose first round has `work` pair-items over np products: ~512 pair-items per CTA, a power of two
// <= SC_RES_MAXCTA (portable cluster size); and the warp-partial slots of its xpart scratch (one per warp, at least one per product).
struct ScResShape { u32 ncta, slots; };
static ScResShape sc_res_shape(u64 work, u32 np) {
    u32 ncta = 1; while (ncta < SC_RES_MAXCTA && (u64)ncta * 512 < work) ncta <<= 1;
    return {ncta, std::max<u32>(ncta * (SC_THREADS / 32), np)};
}

// The previous round's challenge (prover.rs:655-669): none before round 0, one after it; recorded, and the first one refuses constant
// MLEs.  r: the challenge (zero in round 0); returns whether this round folds by it.
static int sc_take_challenge(dp_sc *s, const uint64_t *challenge, gle &r, bool &fold) {
    r = e_zero(); fold = s->round > 0;
    if (!fold) { DP_CHECK(challenge == nullptr, DP_ERR_STATE, "first round should be prover first."); return DP_OK; }   // prover.rs:655
    DP_CHECK(challenge != nullptr, DP_ERR_STATE, "verifier message is empty");  // prover.rs:657
    r = e_from_host(challenge);
    s->challenges.push_back(r);
    if (s->challenges.size() == 1)
        for (auto &m : s->mles) DP_CHECK(m.len > 1, DP_ERR_INVALID, "calling sumcheck on constant");  // prover.rs:667-669
    return DP_OK;
}
// one round's fold done by the resident kernel: the tables now live in its bookkeeping
static void sc_fold_in_kernel(dp_sc *s) {
    for (auto &m : s->mles) if (m.len > 1) { m.len >>= 1; m.is_ext = true; m.cur = nullptr; m.where = 3; }
}
// wait for the resident kernel's flag with tag s->seq; when it does not come, release the kernel and refuse with `msg`
static int sc_tail_wait(dp_sc *s, const std::string &msg) {
    if (dp_wait_flag(s->h_flag, s->seq, true, SC_TAIL_FAILED, 8.0) == s->seq) return DP_OK;
    s->h_chal[0] = SC_TAIL_ABORT; dp_stream_sync(dp_ctx().stream);
    return dp_fail(DP_ERR_CUDA, msg);
}

// start the resident kernel for all remaining rounds; the first one's message is tagged s->seq.  fs: the kernel runs the transcript
// (BlakeTranscript when blake, else BasicTranscript) from this state and writes messages, challenges and the final state to s->h_fs
// (null: the host posts every challenge).
static int sc_tail_launch(dp_sc *s, gle r, bool fold, const ScTailFs *fs, bool blake = false) {
    int e = 0;
    if (!s->h_tail && (e = dp_pinned_alloc((void **)&s->h_tail, sizeof(ScTail)))) return e;
    if (!s->h_chal && (e = dp_pinned_alloc((void **)&s->h_chal, 64))) return e;
    if (fs && !s->h_fs && (e = dp_pinned_alloc((void **)&s->h_fs, sizeof(ScTailFsOut)))) return e;
    ScTail &t = *s->h_tail;
    t.n_mles = s->n_mles; t.n_products = s->n_products; t.n_rounds = s->max_nv - s->round; t.first_has_challenge = fold ? 1 : 0;
    if (fs) t.fs = *fs;
    for (u32 i = 0; i < s->n_mles; i++) {
        ScMle &m = s->mles[i];
        if (m.len > 1 && !m.work) { if ((e = dp_dev_alloc((void **)&m.work, sizeof(gle) * ((m.len0 >> 1) + (m.len0 >> 2) + 1)))) return e; }
        t.m[i] = m; t.writer[i] = s->writer[i];
    }
    for (u32 p = 0; p < s->n_products; p++) { t.p[p].n_idx = s->products[p].n_idx; for (u32 j = 0; j < 5; j++) t.p[p].idx[j] = s->products[p].idx[j]; }
    s->h_chal[0] = 0;
    const ScResShape sh = sc_res_shape(sc_round_work(s, fold), s->n_products);
    if (!s->d_xpart && (e = dp_dev_alloc((void **)&s->d_xpart, sizeof(gle) * SC_NACC * sh.slots))) return e;
    if (!s->d_xctl && (e = dp_dev_alloc((void **)&s->d_xctl, 64))) return e;
    u32 dsel = s->products[0].n_idx;
    for (auto &pr : s->products) if (pr.n_idx != dsel) dsel = 0;
    {
        DpProfScope prof(!fs ? "k_sc_res(resident cluster rounds; time includes the host's Fiat-Shamir between rounds)"
                         : blake ? "k_sc_res(resident cluster rounds, BLAKE3 device transcript)"
                                 : "k_sc_res(resident cluster rounds with the device transcript)", 0);
        DP_CUDA(dp_launch_cluster(k_sc_res_dsel[fs && blake][dsel], sh.ncta, SC_THREADS, dp_ctx().stream, (const ScTail *)s->h_tail, r, s->h_out, s->h_pairs,
                                  s->h_flag, s->h_chal, s->seq, s->d_xpart, s->d_xctl, fs ? s->h_fs : nullptr));
    }
    s->tail_active = true;
    return DP_OK;
}

// one round served by the resident kernel (started here on its first round)
static int sc_tail_round(dp_sc *s, gle r, bool fold, uint64_t *out_evals) {
    s->seq++;
    if (!s->tail_active) {
        if (int e = sc_tail_launch(s, r, fold, nullptr)) return e;
    } else {   // post the challenge: value first, then the sequence number the kernel polls
        s->h_chal[1] = r.c0; s->h_chal[2] = r.c1;
        __atomic_store_n(&s->h_chal[0], s->seq, __ATOMIC_RELEASE);
    }
    if (fold) sc_fold_in_kernel(s);
    s->round += 1;
    if (int e = sc_tail_wait(s, "dp_sc_round: resident kernel timed out waiting for a challenge (other work queued in the same stream?)")) return e;
    if (s->round == s->max_nv) s->have_pairs = true;   // written to mapped memory before the flag
    return sc_glue(s, out_evals);
}

// the Poseidon2 constants of this module's copy of the permutation: the transcript's, never those of dp_poseidon2_init
static cudaError_t sc_fs_constants() {
    static std::once_flag once; static cudaError_t ce = cudaSuccess;
    std::call_once(once, [] {
        cudaStream_t st = dp_ctx().stream;
        if ((ce = cudaMemcpyToSymbolAsync(c_p2_ext, &DP_P2_EXT_RC[0][0][0], sizeof(u64) * 64, 0, cudaMemcpyHostToDevice, st)) == cudaSuccess &&
            (ce = cudaMemcpyToSymbolAsync(c_p2_int, DP_P2_INT_RC, sizeof(u64) * 22, 0, cudaMemcpyHostToDevice, st)) == cudaSuccess &&
            (ce = cudaMemcpyToSymbolAsync(c_p2_diag, DP_P2_DIAG, sizeof(u64) * 8, 0, cudaMemcpyHostToDevice, st)) == cudaSuccess)
            ce = dp_stream_sync(st);
    });
    return ce;
}

// The transcript state an entry point takes: BasicTranscript's 14-word sponge (canonical words, counts in range), or a valid image of
// BlakeTranscript's hasher (dpb3::image_ok), copied into the kernel's SC_FS_WORDS buffer.  False: out of range.
static bool fs_state_in(const uint64_t *in, bool blake, u64 *dst) {
    if (blake) { if (!dpb3::image_ok(in)) return false; for (int w = 0; w < DP_B3T_WORDS; w++) dst[w] = in[w]; return true; }
    if (!(in[12] < 4 && in[13] <= 4)) return false;
    for (int w = 0; w < P2S_WORDS; w++) dst[w] = w < 12 ? gl_canon(in[w]) : in[w];
    return true;
}
// ... and the state the kernel returns, in dpb3::Hasher::save's form (the stack words past stack_len, which merges leave behind in
// the kernel, are zero).  False: the BLAKE3 hasher needed more than DP_B3T_STACK stack entries (more than 2^17 chunks).
static bool fs_state_out(const u64 *src, bool blake, uint64_t *out) {
    if (blake && (src[b3::T_SLEN] & b3::T_OVERFLOW)) return false;
    const int n = blake ? b3::T_STACK + 4 * (int)src[b3::T_SLEN] : P2S_WORDS;
    for (int w = 0; w < (blake ? DP_B3T_WORDS : P2S_WORDS); w++) out[w] = w < n ? src[w] : 0;
    return true;
}
// The transcript part of a device-transcript launch's ScTailFs (fn: the entry point, for the refusal): the caller's state, refused out
// of range; the Poseidon2 constants unless BLAKE3; the "Internal round" label (Transcript::append_message: 8-byte little-endian words);
// the extrapolation weights.
static int sc_fs_setup(ScTailFs &fs, const uint64_t *state_in, bool blake, const char *fn) {
    DP_CHECK(fs_state_in(state_in, blake, fs.sponge), DP_ERR_INVALID, std::string(fn) + (blake ? ": not a BLAKE3 hasher state" : ": sponge state out of range"));
    if (!blake) DP_CUDA(sc_fs_constants());
    static const char label[16] = "Internal round";
    memcpy(fs.label, label, sizeof label);
    memcpy(fs.bary, sc_bary(), sizeof(ScBary));
    return DP_OK;
}

static int sc_run_tail_fs(dp_sc *s, const uint64_t *prev_challenge, const uint64_t *sponge_in, uint64_t *msgs_out, uint64_t *challenges_out,
                          uint64_t *sponge_out, bool blake) {
    const char *const fn = blake ? "dp_sc_run_tail_fs_blake" : "dp_sc_run_tail_fs";
    DP_CHECK(s && sponge_in && msgs_out && challenges_out && sponge_out, DP_ERR_INVALID, std::string(fn) + ": null argument");
    DP_CHECK(!s->finished && s->round < s->max_nv && !s->tail_active, DP_ERR_STATE, "Prover is not active");
    ScTailFs fs{};
    if (int e = sc_fs_setup(fs, sponge_in, blake, fn)) return e;
    DP_CHECK(sc_tail_eligible(s, s->round > 0), DP_ERR_STATE, std::string(fn) + ": the next round does not start the resident tail");
    gle r; bool fold;
    if (int e = sc_take_challenge(s, prev_challenge, r, fold)) return e;
    fs.max_deg = s->max_deg; fs.max_nv = s->max_nv; fs.round0 = s->round;
    for (u32 p = 0; p < s->n_products; p++) { fs.coef[p][0] = s->products[p].coef[0]; fs.coef[p][1] = s->products[p].coef[1]; }
    const u32 nr = s->max_nv - s->round;
    s->seq++;
    if (int e = sc_tail_launch(s, r, fold, &fs, blake)) return e;
    s->seq += nr - 1;                                              // the kernel raises the flag once, with the last round's tag
    for (u32 k = 0; k < nr; k++) if (k > 0 || fold) sc_fold_in_kernel(s);
    s->round = s->max_nv;
    if (int e = sc_tail_wait(s, std::string(fn) + ": the resident kernel did not finish")) return e;
    s->have_pairs = true;
    const ScTailFsOut &o = *s->h_fs;
    const u32 w = s->max_deg + 1;
    for (u32 k = 0; k < nr; k++) {
        for (u32 t = 0; t < w; t++) { msgs_out[2 * (k * w + t)] = o.msg[k][t].c0; msgs_out[2 * (k * w + t) + 1] = o.msg[k][t].c1; }
        challenges_out[2 * k] = o.chal[k].c0; challenges_out[2 * k + 1] = o.chal[k].c1;
        if (k + 1 < nr) s->challenges.push_back(o.chal[k]);     // the last one is dp_sc_finish's
    }
    DP_CHECK(fs_state_out(o.sponge, blake, sponge_out), DP_ERR_STATE, std::string(fn) + ": the transcript outgrew the BLAKE3 state image");
    return DP_OK;
}

// How many layers from `first` on dp_logup_run_layers_fs takes: blocking waits, a launch that can run resident, at most LG_MAXC equal
// circuits, and layers whose first round is resident-sized (the same SC_RES_WORK bound as the tail of a single sumcheck).
static u32 lg_fs_layers(dp_logup *const *c, u32 n, u32 first) {
    if (dp_wait_mode() != DP_WAIT_BLOCK || !c || n == 0 || n > LG_MAXC || first == 0) return 0;
    for (u32 i = 0; i < n; i++) if (!c[i] || c[i]->nv != c[0]->nv) return 0;
    static_assert(1 + 4 * LG_MAXC <= SC_RES_MAXM && 3 * LG_MAXC <= SC_RES_MAXP, "a batch of LG_MAXC circuits fits the resident kernel");
    const u32 total = c[0]->nv - 1;
    u32 k = 0;
    while (first + k <= total && k < LG_MAXL && first + k < SC_MAX_ROUNDS && (u64)3 * n * (1ULL << (first + k - 1)) <= SC_RES_WORK) k++;
    return k && sc_tail_supported() ? k : 0;
}

static int lg_run_layers_fs(dp_logup *const *circuits, uint32_t n_circuits, uint32_t first_layer, uint32_t last_layer, uint64_t *claim,
                            uint64_t *point, uint64_t *alpha, uint64_t *lambda, uint64_t *sponge, uint64_t *msgs_out, uint64_t *challenges_out,
                            uint64_t *evals_out, bool blake) {
    const char *const fn = blake ? "dp_logup_run_layers_fs_blake" : "dp_logup_run_layers_fs";
    DP_CHECK(circuits && claim && point && alpha && lambda && sponge && msgs_out && challenges_out && evals_out, DP_ERR_INVALID,
             std::string(fn) + ": null argument");
    DP_CHECK(first_layer >= 1 && last_layer >= first_layer && last_layer - first_layer < lg_fs_layers(circuits, n_circuits, first_layer), DP_ERR_STATE,
             std::string(fn) + ": these layers do not run resident (wait mode, circuit count or layer size)");
    ScTailFs fs{};
    if (int e = sc_fs_setup(fs, sponge, blake, fn)) return e;
    const u32 nl = last_layer - first_layer + 1, n = n_circuits, np = 3 * n, nm_max = 1 + 4 * n;
    const u64 len_max = 1ULL << last_layer, stride = (len_max >> 1) + (len_max >> 2) + 1;
    const ScResShape sh = sc_res_shape((u64)np * (len_max >> 1), np);   // sized by the largest layer
    LgCfg *cfg = nullptr; LgOut *out = nullptr; char *scratch = nullptr;
    if (int e = dp_pinned_alloc((void **)&cfg, sizeof(LgCfg))) return e;
    PinnedPtr cfg_owner(cfg);
    if (int e = dp_pinned_alloc((void **)&out, sizeof(LgOut))) return e;
    PinnedPtr out_owner(out);
    const size_t off_point = 64, off_part = off_point + sizeof(gle) * (SC_MAX_ROUNDS + 1), off_eq = off_part + sizeof(gle) * SC_NACC * sh.slots,
                 off_work = off_eq + sizeof(gle) * len_max, bytes = off_work + sizeof(gle) * stride * nm_max;
    if (int e = dp_dev_alloc((void **)&scratch, bytes)) return e;
    DevPtr scratch_owner(scratch);
    memset(cfg, 0, sizeof(LgCfg));
    cfg->n_circuits = n; cfg->first = first_layer; cfg->n_layers = nl;
    cfg->claim = e_from_host(claim); cfg->alpha = e_from_host(alpha); cfg->lambda = e_from_host(lambda);
    for (u32 i = 0; i < first_layer; i++) cfg->point[i] = e_from_host(point + 2 * i);
    for (u32 l = 0; l < nl; l++) {
        const u32 k = circuits[0]->nv - 1 - (first_layer + l);    // circuit layer with 2^(v+1) entries (dp_logup_layer_mles)
        for (u32 c = 0; c < n; c++) { cfg->num[l][c] = circuits[c]->num[k]; cfg->den[l][c] = circuits[c]->den[k]; }
    }
    cfg->eq = (gle *)(scratch + off_eq); cfg->work = (gle *)(scratch + off_work); cfg->work_stride = stride;
    static const char lbl[3][16] = {"logup_batching", "logup_alpha", "logup_lambda"};   // BasicTranscript::append_message words
    memcpy(cfg->label, lbl, sizeof lbl);
    cfg->fs = fs; cfg->fs.max_deg = 3;
    out->flag = 0;
    {
        DpProfScope prof(blake ? "k_logup_res(resident LogUp-GKR layers, BLAKE3 transcript)" : "k_logup_res(resident LogUp-GKR layers, device transcript)", 0);
        DP_CUDA(dp_launch_cluster(blake ? k_logup_res<TrB3> : k_logup_res<TrP2>, sh.ncta, SC_THREADS, dp_ctx().stream, (const LgCfg *)cfg, out,
                                  (gle *)(scratch + off_part), (u64 *)scratch, (gle *)(scratch + off_point)));
    }
    if (int e = dp_await(&out->flag, 1, 8.0, std::string(fn) + ": the resident kernel did not finish")) return e;
    size_t om = 0, oc = 0, oe = 0;
    for (u32 l = 0; l < nl; l++) {
        const u32 v = first_layer + l, per = cfg->num[l][0] ? 4 : 2;
        const LgLayerOut &o = out->layer[l];
        for (u32 k = 0; k < v; k++) {
            for (u32 t = 0; t < 4; t++) { msgs_out[om++] = o.fs.msg[k][t].c0; msgs_out[om++] = o.fs.msg[k][t].c1; }
            challenges_out[oc++] = o.fs.chal[k].c0; challenges_out[oc++] = o.fs.chal[k].c1;
        }
        for (u32 i = 0; i < per * n; i++) { evals_out[oe++] = o.evals[i].c0; evals_out[oe++] = o.evals[i].c1; }
    }
    for (u32 i = 0; i <= last_layer; i++) { point[2 * i] = out->point[i].c0; point[2 * i + 1] = out->point[i].c1; }
    claim[0] = out->claim.c0; claim[1] = out->claim.c1; alpha[0] = out->alpha.c0; alpha[1] = out->alpha.c1; lambda[0] = out->lambda.c0; lambda[1] = out->lambda.c1;
    DP_CHECK(fs_state_out(out->sponge, blake, sponge), DP_ERR_STATE, std::string(fn) + ": the transcript outgrew the BLAKE3 state image");
    return DP_OK;
}

extern "C" {

int dp_sc_create(dp_mle *const *mles, uint32_t n_mles, const dp_sc_product *products, uint32_t n_products,
                 uint32_t max_nv, uint32_t max_deg, dp_sc **out) {
    DP_REQUIRE_CTX();
    DP_CHECK(mles && products && out && n_mles > 0 && n_products > 0, DP_ERR_INVALID, "dp_sc_create: null/empty argument");
    DP_CHECK(max_nv != 0, DP_ERR_INVALID, "Attempt to prove a constant.");  // prover.rs:590-593
    DP_CHECK(max_nv <= 40, DP_ERR_INVALID, "dp_sc_create: max_num_variables too large");
    for (u32 i = 0; i < n_mles; i++) DP_CHECK(mles[i] != nullptr, DP_ERR_INVALID, "dp_sc_create: null MLE");   // every entry is dereferenced below, referenced by a product or not
    u32 seen_deg = 0;
    for (u32 p = 0; p < n_products; p++) {
        const dp_sc_product &pr = products[p];
        DP_CHECK(pr.n_idx >= 1, DP_ERR_INVALID, "input mle_list is empty");  // virtual_poly.rs:143
        DP_CHECK(pr.n_idx <= 5, DP_ERR_UNSUPPORTED, "do not support degree > 5");  // prover.rs:710
        for (u32 j = 0; j < pr.n_idx; j++) {
            DP_CHECK(pr.idx[j] < n_mles, DP_ERR_INVALID, "dp_sc_create: product index out of range");
            const dp_mle *m = mles[pr.idx[j]];
            DP_CHECK(m != nullptr, DP_ERR_INVALID, "dp_sc_create: null MLE");
            DP_CHECK(m->num_vars() <= max_nv, DP_ERR_INVALID, "invalid max num vars");  // virtual_poly.rs:151-154
            DP_CHECK(m->len == mles[pr.idx[0]]->len, DP_ERR_INVALID, "mle in mle_list must be in same num_vars() in same product");
        }
        seen_deg = std::max(seen_deg, pr.n_idx);
    }
    DP_CHECK(seen_deg <= max_deg, DP_ERR_INVALID, "dp_sc_create: max_degree smaller than a product's degree");
    DP_CHECK(max_deg <= 5, DP_ERR_UNSUPPORTED, "do not support degree > 5");  // prover.rs:710; sc_glue's message arrays hold degree 5
    dp_sc *s = new dp_sc();
    s->n_mles = n_mles; s->n_products = n_products; s->max_nv = max_nv; s->max_deg = max_deg;
    s->mles.resize(n_mles);
    u64 max_pairs = 1;
    for (u32 i = 0; i < n_mles; i++) {
        ScMle &m = s->mles[i];
        m.cur = mles[i]->data; m.len = m.len0 = mles[i]->len; m.is_ext = mles[i]->is_ext; m.where = 0;
        max_pairs = std::max<u64>(max_pairs, m.len >> 1);
    }
    s->writer.assign(n_mles, SC_NO_WRITER);
    for (u32 p = n_products; p-- > 0;) for (u32 j = 0; j < products[p].n_idx; j++) s->writer[products[p].idx[j]] = p;
    s->products.assign(products, products + n_products);
    for (auto &pr : s->products) { pr.coef[0] = gl_canon(pr.coef[0]); pr.coef[1] = gl_canon(pr.coef[1]); }
    s->gx = (int)std::min<u64>((max_pairs + 127) / 128 + 1, (u64)dp_ctx().sm_count * 16);   // upper bound of any round's grid (partials buffer): lean folding rounds use 128-thread blocks, one pair per thread
    // any failure below releases what was already allocated (dp_sc_destroy tolerates the partially built handle)
    auto build = [&]() -> int {
        int e = 0;
        if ((e = dp_dev_alloc((void **)&s->d_descs, sizeof(ScProd) * n_products))) return e;
        if ((e = dp_dev_alloc((void **)&s->d_partials, sizeof(gle) * SC_NACC * (size_t)s->gx * n_products))) return e;
        if ((e = dp_dev_alloc((void **)&s->d_out, sizeof(gle) * SC_NACC * n_products))) return e;
        if (sizeof(u32) * (n_products + 1) <= 256) { if ((e = dp_zero_block_get((void **)&s->d_counters))) return e; s->counters_pooled = true; }
        else { if ((e = dp_dev_alloc((void **)&s->d_counters, sizeof(u32) * (n_products + 1)))) return e; DP_CUDA(cudaMemsetAsync(s->d_counters, 0, sizeof(u32) * (n_products + 1), dp_ctx().stream)); }
        s->d_done = s->d_counters + n_products;
        if ((e = dp_pinned_alloc((void **)&s->h_flag, 64))) return e;
        *s->h_flag = 0;
        if ((e = dp_dev_alloc((void **)&s->d_fin, sizeof(ScFin) * n_mles + sizeof(gle) * 2 * n_mles))) return e;
        if ((e = dp_pinned_alloc((void **)&s->h_descs, sizeof(ScProd) * n_products))) return e;
        if ((e = dp_pinned_alloc((void **)&s->h_out, sizeof(gle) * SC_NACC * n_products))) return e;
        if ((e = dp_pinned_alloc((void **)&s->h_fin, sizeof(ScFin) * n_mles))) return e;
        if ((e = dp_pinned_alloc((void **)&s->h_pairs, sizeof(gle) * 2 * n_mles))) return e;
        return DP_OK;
    };
    if (int e = build()) { sc_free_all(s); delete s; return e; }
    *out = s;
    return DP_OK;
}

int dp_sc_round(dp_sc *s, const uint64_t *challenge, uint64_t *out_evals) {
    DP_REQUIRE_CTX();
    DP_CHECK(s && out_evals, DP_ERR_INVALID, "dp_sc_round: null argument");
    DP_CHECK(!s->finished && s->round < s->max_nv, DP_ERR_STATE, "Prover is not active");  // prover.rs:636-639
    gle r; bool fold;
    if (int e = sc_take_challenge(s, challenge, r, fold)) return e;
    if (s->tail_active || sc_tail_eligible(s, fold)) return sc_tail_round(s, r, fold, out_evals);
    // plan this round's folds: every MLE with >= 1 variable halves (prover.rs:659-684)
    std::vector<gle *> dst(s->n_mles, nullptr);
    std::vector<unsigned char> folds(s->n_mles, 0);
    u64 bytes = 0, round_pairs = 1;                       // bytes: operand reads + folded-table writes, for the profile
    if (fold) {
        for (u32 i = 0; i < s->n_mles; i++) {
            ScMle &m = s->mles[i];
            if (m.len <= 1) continue;
            if (!m.work) { if (int e = dp_dev_alloc((void **)&m.work, sizeof(gle) * ((m.len0 >> 1) + (m.len0 >> 2) + 1))) return e; }
            folds[i] = 1;
            dst[i] = sc_fold_dst(m);
            if (s->writer[i] != SC_NO_WRITER) bytes += (m.len >> 1) * 16;
        }
    }
    for (u32 p = 0; p < s->n_products; p++) {
        const dp_sc_product &pr = s->products[p];
        ScProd &d = s->h_descs[p];
        memset(&d, 0, sizeof d);
        sc_desc(d, p, pr.idx, pr.n_idx, s->mles.data(), folds.data(), dst.data(), s->writer.data());
        for (u32 j = 0; j < pr.n_idx; j++) { const ScMle &m = s->mles[pr.idx[j]]; bytes += m.len * (m.is_ext ? 16 : 8); }
        round_pairs = std::max<u64>(round_pairs, d.npairs);
    }
    // uniform rounds take the lean kernels: every operand of every product in the same mode, one degree in {2, 3}, no constants
    u32 dsel = s->products[0].n_idx;
    for (auto &pr : s->products) if (pr.n_idx != dsel) dsel = 0;
    int lean_mode = -1;
    if ((dsel == 2 || dsel == 3) && round_pairs > 2048) {
        lean_mode = (int)s->h_descs[0].op[0].mode;
        for (u32 p = 0; p < s->n_products && lean_mode >= 0; p++) {
            const ScProd &d = s->h_descs[p];
            if (d.konst) lean_mode = -1;
            for (u32 j = 0; j < d.d && lean_mode >= 0; j++) if ((int)d.op[j].mode != lean_mode) lean_mode = -1;
        }
    }
    // field operations of this round in the operand field (SURVEY.md 8(d)): (d-1)(d+1) mul + (5d+4) add per pair, + (1 mul + 2 add) for
    // each of the 2 elements a folding operand contributes to a pair
    u64 ops = 0;
    for (u32 p = 0; p < s->n_products; p++) { const ScProd &d = s->h_descs[p]; u64 nf = 0; for (u32 j = 0; j < d.d; j++) if (d.op[j].mode >= OPM_BF) nf++; ops += d.npairs * ((u64)(d.d - 1) * (d.d + 1) + 5 * d.d + 4 + 6 * nf); }
    // grid sized for THIS round.  lean: Base rounds 256 threads x 2 pairs in flight, folding rounds 128 threads x 1 pair (tools/kbench.cu);
    // general kernel: 2 pairs per thread minimum so small rounds run in a single block
    int gx;
    if (lean_mode == (int)OPM_B) gx = (int)std::min<u64>((round_pairs + 511) / 512, (u64)dp_ctx().sm_count * 4);
    else if (lean_mode >= 0) gx = (int)std::min<u64>((round_pairs + 127) / 128, (u64)s->gx);
    else gx = round_pairs > 8192 ? std::min(s->gx, dp_grid_for(round_pairs, SC_THREADS, 6))
                                 : std::min(s->gx, dp_grid_for(round_pairs <= 256 ? round_pairs : (round_pairs + 1) / 2, SC_THREADS, 4));
    cudaStream_t st = dp_ctx().stream;
    // MLEs no product references still have to be folded (cannot happen through add_mle_list, kept for safety)
    for (u32 i = 0; i < s->n_mles; i++) if (folds[i] && s->writer[i] == SC_NO_WRITER) {
        ScMle &m = s->mles[i];
        if (int e = dpk_fold_low(m.cur, m.is_ext, m.len, r, dst[i])) return e;
    }
    dim3 grid((unsigned)gx, s->n_products);
    {
        DpProfScope prof(lean_mode == (int)OPM_B ? "k_sc_lean(msg, Base)" : lean_mode == (int)OPM_E ? "k_sc_lean(msg, Ext)" : lean_mode == (int)OPM_BF ? "k_sc_lean(fold Base->Ext + msg)"
                         : lean_mode == (int)OPM_EF ? "k_sc_lean(fold Ext + msg)" : fold ? "k_sc_round(fold+msg)" : "k_sc_round(msg)", bytes, ops);
        s->seq++; s->round_in_flight = true;
        const ScProd *descs_arg = s->h_descs;                 // mapped pinned memory: no copy node on the latency path
        if (s->n_products == 1) descs_arg = nullptr;          // descriptor travels in the kernel parameters
        else if ((u64)gx * s->n_products > 32) { DP_CUDA(cudaMemcpyAsync(s->d_descs, s->h_descs, sizeof(ScProd) * s->n_products, cudaMemcpyHostToDevice, st)); descs_arg = s->d_descs; }
        // one small kernel per uniform degree keeps the instruction footprint low
        const auto kern = lean_mode >= 0 ? k_sc_lean_md[lean_mode][dsel - 2] : k_sc_round_dsel[dsel];
        const int block = lean_mode >= 0 ? SC_LEAN_BLOCK[lean_mode] : SC_THREADS;
        DP_CUDA(dp_launch(kern, grid, block, 0, st, descs_arg, s->h_descs[0], r, s->d_partials, s->d_counters, s->h_out, s->seq, s->h_flag, s->d_done));
    }
    // commit the folds to the bookkeeping while the GPU works
    for (u32 i = 0; i < s->n_mles; i++) if (folds[i]) sc_commit_fold(s->mles[i], dst[i]);
    s->round += 1;
    if (s->round == s->max_nv) {   // last round: bring the (<= 2)-entry tables back together with the message
        bool ok = true;
        for (u32 i = 0; i < s->n_mles; i++) { const ScMle &m = s->mles[i]; if (m.len > 2) ok = false; s->h_fin[i].src = m.cur; s->h_fin[i].mode = m.is_ext ? OPM_E : OPM_B; s->h_fin[i].len = (u32)m.len; }
        if (ok) {
            gle *d_pairs = (gle *)((char *)s->d_fin + sizeof(ScFin) * s->n_mles);
            DP_CUDA(cudaMemcpyAsync(s->d_fin, s->h_fin, sizeof(ScFin) * s->n_mles, cudaMemcpyHostToDevice, st));
            DP_CUDA(dp_launch(k_sc_gather, (s->n_mles + 127) / 128, 128, 0, st, s->d_fin, s->n_mles, d_pairs));
            DP_CUDA(cudaMemcpyAsync(s->h_pairs, d_pairs, sizeof(gle) * 2 * s->n_mles, cudaMemcpyDeviceToHost, st));
            s->have_pairs = true;
        }
    }
    if (s->have_pairs) { DP_CUDA(dp_stream_sync(st)); s->round_in_flight = false; }      // last round: the gathered pairs follow the kernel
    else {
        if (int e = dp_await(s->h_flag, s->seq, 2.0, "dp_sc_round: kernel finished without signalling")) return e;
        s->round_in_flight = false;
    }
    return sc_glue(s, out_evals);
}

int dp_sc_finish(dp_sc *s, const uint64_t *last_challenge, uint64_t *out_final) {
    DP_REQUIRE_CTX();
    DP_CHECK(s && last_challenge && out_final, DP_ERR_INVALID, "dp_sc_finish: null argument");
    DP_CHECK(!s->finished && s->round == s->max_nv, DP_ERR_STATE, "dp_sc_finish: rounds not complete");
    gle r = e_from_host(last_challenge);
    s->challenges.push_back(r);
    // the last round fetched the pairs unless an MLE still had more than 2 entries; get_mle_final_evaluations asserts
    // len == 1 after the last fix (prover.rs:479-483)
    DP_CHECK(s->have_pairs, DP_ERR_STATE, "mle.evaluations.len() != 1, must be called after prove_round_and_update_state");
    for (u32 i = 0; i < s->n_mles; i++) {   // O(#MLEs) host glue on the pairs fetched with the last message
        gle a = s->h_pairs[2 * i], b = s->h_pairs[2 * i + 1];
        gle v = s->mles[i].len > 1 ? e_add(a, e_mul(e_sub(b, a), r)) : a;
        out_final[2 * i] = v.c0; out_final[2 * i + 1] = v.c1;
    }
    s->finished = true;
    return DP_OK;
}

int dp_sc_destroy(dp_sc *s) {
    if (!s) return DP_OK;
    if (dp_ctx().ready) {
        if (s->tail_active && s->round < s->max_nv) { s->h_chal[0] = SC_TAIL_ABORT; dp_stream_sync(dp_ctx().stream); }   // release the waiting kernel
        sc_free_all(s);
    }
    delete s;
    return DP_OK;
}

int dp_sc_set_resident_tail(dp_sc *s, int enable) {
    DP_REQUIRE_CTX();
    DP_CHECK(s && !s->tail_active, DP_ERR_STATE, "dp_sc_set_resident_tail: null handle or tail already running");
    s->tail_enabled = enable != 0 && sc_tail_supported();
    return DP_OK;
}

// The device transcript pays where a proving thread would otherwise sleep through every round trip: in blocking wait mode, many
// proofs in flight.  In spin mode the host's round trip is a few microseconds, less than the kernel's hash chain per round (3
// dependent Poseidon2 permutations on one warp, or a few BLAKE3 compressions on one thread: DESIGN.md section 5.2), so a lone proof
// keeps the host transcript with either hasher.
int dp_sc_tail_fs_next(dp_sc *s, int *out) {
    DP_REQUIRE_CTX();
    DP_CHECK(s && out, DP_ERR_INVALID, "dp_sc_tail_fs_next: null argument");
    *out = !s->finished && s->round < s->max_nv && !s->tail_active && dp_wait_mode() == DP_WAIT_BLOCK && sc_tail_eligible(s, s->round > 0);
    return DP_OK;
}

int dp_sc_run_tail_fs(dp_sc *s, const uint64_t *prev_challenge, const uint64_t *sponge_in, uint64_t *msgs_out, uint64_t *challenges_out,
                      uint64_t *sponge_out) {
    DP_REQUIRE_CTX();
    return sc_run_tail_fs(s, prev_challenge, sponge_in, msgs_out, challenges_out, sponge_out, false);
}
int dp_sc_run_tail_fs_blake(dp_sc *s, const uint64_t *prev_challenge, const uint64_t *state_in, uint64_t *msgs_out, uint64_t *challenges_out,
                            uint64_t *state_out) {
    DP_REQUIRE_CTX();
    return sc_run_tail_fs(s, prev_challenge, state_in, msgs_out, challenges_out, state_out, true);
}

int dp_sc_current_mle(dp_sc *s, uint32_t idx, dp_mle **out) {
    DP_REQUIRE_CTX();
    DP_CHECK(s && out && idx < s->n_mles, DP_ERR_INVALID, "dp_sc_current_mle: bad argument");
    const ScMle &m = s->mles[idx];
    DP_CHECK(!s->tail_active, DP_ERR_STATE, "dp_sc_current_mle: tables are owned by the resident tail kernel");
    *out = dp_mle_view(const_cast<void *>(m.cur), m.len, m.is_ext);
    return DP_OK;
}

int dp_logup_layers_fs_next(dp_logup *const *circuits, uint32_t n_circuits, uint32_t first_layer, uint32_t *n_layers) {
    DP_REQUIRE_CTX();
    DP_CHECK(circuits && n_layers, DP_ERR_INVALID, "dp_logup_layers_fs_next: null argument");
    *n_layers = lg_fs_layers(circuits, n_circuits, first_layer);
    return DP_OK;
}
int dp_logup_run_layers_fs(dp_logup *const *circuits, uint32_t n_circuits, uint32_t first_layer, uint32_t last_layer, uint64_t *claim,
                           uint64_t *point, uint64_t *alpha, uint64_t *lambda, uint64_t *sponge, uint64_t *msgs_out, uint64_t *challenges_out,
                           uint64_t *evals_out) {
    DP_REQUIRE_CTX();
    return lg_run_layers_fs(circuits, n_circuits, first_layer, last_layer, claim, point, alpha, lambda, sponge, msgs_out, challenges_out, evals_out, false);
}
int dp_logup_run_layers_fs_blake(dp_logup *const *circuits, uint32_t n_circuits, uint32_t first_layer, uint32_t last_layer, uint64_t *claim,
                                 uint64_t *point, uint64_t *alpha, uint64_t *lambda, uint64_t *state, uint64_t *msgs_out, uint64_t *challenges_out,
                                 uint64_t *evals_out) {
    DP_REQUIRE_CTX();
    return lg_run_layers_fs(circuits, n_circuits, first_layer, last_layer, claim, point, alpha, lambda, state, msgs_out, challenges_out, evals_out, true);
}

}  // extern "C"
