// Kernel micro-benchmarks (development tool, round 2): candidate formulations of the hot kernels timed with CUDA events on a
// real H100 before they replace the library versions.  Every candidate is checked against the library formulation first.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Iinclude -o deep-prove_b200/kbench_bin tools/kbench.cu
//   gpurun -- ./deep-prove_b200/kbench_bin [section ...]      sections: perm lat sc
#include <cstdio>
#include <cstring>
#include <vector>
#include <string>
#include <algorithm>
#include <chrono>
#include <thread>
#include <atomic>
#include "../deep-prove_b200/csrc/poseidon2.cuh"
#include "../deep-prove_b200/csrc/blake3.cuh"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1); } } while (0)
static u64 sm64(u64 &st) { u64 z = (st += 0x9E3779B97F4A7C15ULL); z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL; z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL; return z ^ (z >> 31); }

template <class F> static float time_ms(F f, int reps = 5, int warm = 2) {
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    for (int i = 0; i < warm; i++) f();
    float best = 1e30f;
    for (int i = 0; i < reps; i++) { cudaEventRecord(a); f(); cudaEventRecord(b); cudaEventSynchronize(b); float ms; cudaEventElapsedTime(&ms, a, b); best = std::min(best, ms); }
    CK(cudaGetLastError());
    return best;
}
static u64 checksum(const u64 *d, size_t n) { std::vector<u64> h(n); cudaMemcpy(h.data(), d, n * 8, cudaMemcpyDeviceToHost); u64 s = 0; for (size_t i = 0; i < n; i++) s = s * 0x100000001B3ULL + h[i]; return s; }

// =====================================================================================================================
// Poseidon2 candidates
// =====================================================================================================================
// (a) NH interleaved hashes per thread, (b) internal rounds restructured so the S-box chain of round r+1 only waits for the
// s0 update of round r (the other seven multiply-adds and the running sum of lanes 1..7 sit in its shadow), unrolled by UI.
template <int NH, int UI>
__device__ __forceinline__ void p2_permute_v(u64 (&s)[NH][8]) {
#pragma unroll
    for (int h = 0; h < NH; h++) p2_mds_light(s[h]);
#pragma unroll 1
    for (int r = 0; r < 4; r++) {
#pragma unroll
        for (int h = 0; h < NH; h++) {
#pragma unroll
            for (int i = 0; i < 8; i++) s[h][i] = p2_pow7(w_add_canon(s[h][i], c_p2_ext[0][r][i]));
        }
#pragma unroll
        for (int h = 0; h < NH; h++) p2_mds_light(s[h]);
    }
    p2w R[NH];
#pragma unroll
    for (int h = 0; h < NH; h++) { R[h] = ww(s[h][1]); for (int i = 2; i < 8; i++) R[h] = ww_addu(R[h], s[h][i]); }
#pragma unroll 1
    for (int r = 0; r < 22; r += UI) {
#pragma unroll
        for (int u = 0; u < UI; u++) {
#pragma unroll
            for (int h = 0; h < NH; h++) {
                u64 t = p2_pow7(w_add_canon(s[h][0], c_p2_int[r + u]));
                p2w sum = ww_addu(R[h], t);
                s[h][0] = w_mul_add(t, c_p2_diag[0], sum);
                p2w nr = ww(0);
#pragma unroll
                for (int i = 1; i < 8; i++) { s[h][i] = w_mul_add(s[h][i], c_p2_diag[i], sum); nr = ww_addu(nr, s[h][i]); }
                R[h] = nr;
            }
        }
    }
#pragma unroll 1
    for (int r = 0; r < 4; r++) {
#pragma unroll
        for (int h = 0; h < NH; h++) {
#pragma unroll
            for (int i = 0; i < 8; i++) s[h][i] = p2_pow7(w_add_canon(s[h][i], c_p2_ext[1][r][i]));
        }
#pragma unroll
        for (int h = 0; h < NH; h++) p2_mds_light(s[h]);
    }
}
template <int NH, int UI>
__device__ __forceinline__ void p2_compress_v(const u64 (&x)[NH][4], const u64 (&y)[NH][4], u64 (&o)[NH][4]) {
    u64 s[NH][8];
#pragma unroll
    for (int h = 0; h < NH; h++) { for (int k = 0; k < 4; k++) { s[h][k] = x[h][k]; s[h][4 + k] = 0; } }
    p2_permute_v<NH, UI>(s);
#pragma unroll
    for (int h = 0; h < NH; h++) for (int k = 0; k < 4; k++) s[h][k] = y[h][k];
    p2_permute_v<NH, UI>(s);
#pragma unroll
    for (int h = 0; h < NH; h++) for (int k = 0; k < 4; k++) o[h][k] = gl_canon_weak(s[h][3 - k]);
}

// library formulation (k_merkle_up)
__global__ void k_up_lib(const u64 *__restrict__ in, u64 n_out, u64 *__restrict__ out) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    for (; i < n_out; i += stride) {
        u64 x[4], y[4], o[4];
        ulonglong2 a = *reinterpret_cast<const ulonglong2 *>(in + 8 * i), b = *reinterpret_cast<const ulonglong2 *>(in + 8 * i + 2);
        ulonglong2 c = *reinterpret_cast<const ulonglong2 *>(in + 8 * i + 4), d = *reinterpret_cast<const ulonglong2 *>(in + 8 * i + 6);
        x[0] = a.x; x[1] = a.y; x[2] = b.x; x[3] = b.y; y[0] = c.x; y[1] = c.y; y[2] = d.x; y[3] = d.y;
        p2_compress(x, y, o);
        *reinterpret_cast<ulonglong2 *>(out + 4 * i) = make_ulonglong2(o[0], o[1]);
        *reinterpret_cast<ulonglong2 *>(out + 4 * i + 2) = make_ulonglong2(o[2], o[3]);
    }
}
template <int NH, int UI, int BLOCK, int MINB>
__global__ void __launch_bounds__(BLOCK, MINB) k_up_v(const u64 *__restrict__ in, u64 n_out, u64 *__restrict__ out) {
    // thread t of the grid owns hashes t, t + T, ... (T = threads): consecutive lanes read consecutive 64-byte blocks
    const u64 T = (u64)gridDim.x * BLOCK;
    for (u64 i0 = (u64)blockIdx.x * BLOCK + threadIdx.x; i0 < n_out; i0 += NH * T) {
        u64 x[NH][4], y[NH][4], o[NH][4];
#pragma unroll
        for (int h = 0; h < NH; h++) {
            u64 i = i0 + h * T; if (i >= n_out) i = i0;
            ulonglong2 a = *reinterpret_cast<const ulonglong2 *>(in + 8 * i), b = *reinterpret_cast<const ulonglong2 *>(in + 8 * i + 2);
            ulonglong2 c = *reinterpret_cast<const ulonglong2 *>(in + 8 * i + 4), d = *reinterpret_cast<const ulonglong2 *>(in + 8 * i + 6);
            x[h][0] = a.x; x[h][1] = a.y; x[h][2] = b.x; x[h][3] = b.y; y[h][0] = c.x; y[h][1] = c.y; y[h][2] = d.x; y[h][3] = d.y;
        }
        p2_compress_v<NH, UI>(x, y, o);
#pragma unroll
        for (int h = 0; h < NH; h++) {
            u64 i = i0 + h * T; if (i >= n_out) continue;
            *reinterpret_cast<ulonglong2 *>(out + 4 * i) = make_ulonglong2(o[h][0], o[h][1]);
            *reinterpret_cast<ulonglong2 *>(out + 4 * i + 2) = make_ulonglong2(o[h][2], o[h][3]);
        }
    }
}

// latency: every thread runs a chain of `len` dependent compresses (x <- compress(x, y))
template <int UI>
__global__ void k_chain_tph(u64 *io, int len) {
    u64 x[1][4], y[1][4], o[1][4];
    for (int k = 0; k < 4; k++) { x[0][k] = io[8 * threadIdx.x + k]; y[0][k] = io[8 * threadIdx.x + 4 + k]; }
    for (int it = 0; it < len; it++) { p2_compress_v<1, UI>(x, y, o); for (int k = 0; k < 4; k++) x[0][k] = o[0][k]; }
    for (int k = 0; k < 4; k++) io[8 * threadIdx.x + k] = x[0][k];
}
__global__ void k_chain_lib(u64 *io, int len) {
    u64 x[4], y[4], o[4];
    for (int k = 0; k < 4; k++) { x[k] = io[8 * threadIdx.x + k]; y[k] = io[8 * threadIdx.x + 4 + k]; }
    for (int it = 0; it < len; it++) { p2_compress(x, y, o); for (int k = 0; k < 4; k++) x[k] = o[k]; }
    for (int k = 0; k < 4; k++) io[8 * threadIdx.x + k] = x[k];
}
__global__ void k_chain_latopt(u64 *io, int len) {
    u64 x[4], y[4], o[4];
    for (int k = 0; k < 4; k++) { x[k] = io[8 * threadIdx.x + k]; y[k] = io[8 * threadIdx.x + 4 + k]; }
    for (int it = 0; it < len; it++) { p2_compress_lat(x, y, o); for (int k = 0; k < 4; k++) x[k] = o[k]; }
    for (int k = 0; k < 4; k++) io[8 * threadIdx.x + k] = x[k];
}
__global__ void k_chain_x8(u64 *io, int len) {   // 8 lanes per hash: hash h = thread / 8
    const int lane8 = threadIdx.x & 7, h = threadIdx.x >> 3;
    u64 xw = lane8 < 4 ? io[8 * h + lane8] : 0, yw = lane8 < 4 ? io[8 * h + 4 + lane8] : 0;
    for (int it = 0; it < len; it++) {
        u64 s = p2x8_compress(xw, yw, lane8);      // lane k < 4 holds digest word 3 - k
        u64 w = __shfl_sync(0xffffffffu, s, 3 - (lane8 & 3), 8);
        if (lane8 < 4) xw = w;
    }
    if (lane8 < 4) io[8 * h + lane8] = xw;
}

// =====================================================================================================================
// Sumcheck round candidates (degree 3, one product of three MLEs)
// =====================================================================================================================
// gl_acc (gl.cuh): one reduction per thread per evaluation point instead of one per product

// all-Base first round: message only.  PPT pairs in flight per thread (3 * PPT independent 16-byte loads).
template <int PPT, int BLOCK, int MINB>
__global__ void __launch_bounds__(BLOCK, MINB) k_scb3(const u64 *__restrict__ f0, const u64 *__restrict__ f1, const u64 *__restrict__ f2, u64 npairs, u64 *__restrict__ partials) {
    gl_acc a[4];
#pragma unroll
    for (int t = 0; t < 4; t++) { a[t].lo = 0; a[t].hi = 0; a[t].top = 0; }
    const u64 T = (u64)gridDim.x * BLOCK;
    for (u64 i0 = (u64)blockIdx.x * BLOCK + threadIdx.x; i0 < npairs; i0 += PPT * T) {
        ulonglong2 v[PPT][3];
#pragma unroll
        for (int p = 0; p < PPT; p++) {
            u64 i = i0 + p * T; const bool ok = i < npairs; if (!ok) i = i0;
            v[p][0] = ld_b2(f0 + 2 * i); v[p][1] = ld_b2(f1 + 2 * i); v[p][2] = ld_b2(f2 + 2 * i);
            if (!ok) { v[p][0] = make_ulonglong2(0, 0); }     // a zero factor contributes nothing at every point
        }
#pragma unroll
        for (int p = 0; p < PPT; p++) {
            u64 c0 = v[p][0].x, c1 = v[p][1].x, c2 = v[p][2].x;
            const u64 s0 = gl_sub(v[p][0].y, c0), s1 = gl_sub(v[p][1].y, c1), s2 = gl_sub(v[p][2].y, c2);
#pragma unroll
            for (int t = 0; t < 4; t++) {
                gl_acc_mac(a[t], w_mul(c0, c1), c2);
                if (t < 3) { c0 = gl_add(c0, s0); c1 = gl_add(c1, s1); c2 = gl_add(c2, s2); }
            }
        }
    }
    __shared__ u64 ws[BLOCK / 32][4];
#pragma unroll
    for (int t = 0; t < 4; t++) {
        u64 v = gl_acc_reduce(a[t]);
        for (int d = 16; d > 0; d >>= 1) v = gl_add(v, __shfl_down_sync(0xffffffffu, v, d));
        if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5][t] = v;
    }
    __syncthreads();
    if (threadIdx.x < 4) { u64 v = ws[0][threadIdx.x]; for (int w = 1; w < BLOCK / 32; w++) v = gl_add(v, ws[w][threadIdx.x]); partials[4 * blockIdx.x + threadIdx.x] = v; }
}
// library-style body for comparison (canonical accumulation, two pairs in flight) -- the shape of sc_body<3, BIG> all-Base
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_scb3_lib(const u64 *__restrict__ f0, const u64 *__restrict__ f1, const u64 *__restrict__ f2, u64 npairs, u64 *__restrict__ partials) {
    u64 a[4] = {0, 0, 0, 0};
    const u64 stride = (u64)gridDim.x * BLOCK;
    const u64 *src[3] = {f0, f1, f2};
    for (u64 i = (u64)blockIdx.x * BLOCK + threadIdx.x; i < npairs; i += 2 * stride) {
        const u64 i2 = i + stride; const bool two = i2 < npairs;
        u64 c0[3], s0[3], c1[3], s1[3];
#pragma unroll
        for (int j = 0; j < 3; j++) {
            ulonglong2 v = ld_b2(src[j] + 2 * i);
            ulonglong2 w = two ? ld_b2(src[j] + 2 * i2) : make_ulonglong2(0, 0);
            c0[j] = v.x; s0[j] = gl_sub(v.y, v.x); c1[j] = w.x; s1[j] = gl_sub(w.y, w.x);
        }
#pragma unroll
        for (int t = 0; t < 4; t++) {
            u64 p = c0[0], q = c1[0];
#pragma unroll
            for (int j = 1; j < 3; j++) { p = gl_mul(p, c0[j]); q = gl_mul(q, c1[j]); }
            a[t] = gl_add(a[t], gl_add(p, q));
            if (t < 3) {
#pragma unroll
                for (int j = 0; j < 3; j++) { c0[j] = gl_add(c0[j], s0[j]); c1[j] = gl_add(c1[j], s1[j]); }
            }
        }
    }
    __shared__ u64 ws[BLOCK / 32][4];
#pragma unroll
    for (int t = 0; t < 4; t++) {
        u64 v = a[t];
        for (int d = 16; d > 0; d >>= 1) v = gl_add(v, __shfl_down_sync(0xffffffffu, v, d));
        if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5][t] = v;
    }
    __syncthreads();
    if (threadIdx.x < 4) { u64 v = ws[0][threadIdx.x]; for (int w = 1; w < BLOCK / 32; w++) v = gl_add(v, ws[w][threadIdx.x]); partials[4 * blockIdx.x + threadIdx.x] = v; }
}

// ---- the same message kernel with the operand tiles staged in shared memory by bulk-async copies (cp.async.bulk + mbarrier,
// UBLKCP in SASS): one elected thread keeps STAGES tiles of every operand in flight, the block consumes tile by tile -------------
__device__ __forceinline__ u32 smem_u32(const void *p) { return (u32)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(u64 *bar, u32 count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)); }
__device__ __forceinline__ void mbar_expect_tx(u64 *bar, u32 bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_arrive(u64 *bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory"); }
__device__ __forceinline__ void mbar_wait(u64 *bar, u32 parity) {
    asm volatile("{\n\t.reg .pred p;\n\tWAIT_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, u32 bytes, u64 *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
template <int TILE /* pairs per tile */, int STAGES, int BLOCK, int MINB>
__global__ void __launch_bounds__(BLOCK, MINB) k_scb3_tma(const u64 *__restrict__ f0, const u64 *__restrict__ f1, const u64 *__restrict__ f2, u64 npairs, u64 *__restrict__ partials) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    u64 *tiles = (u64 *)smem_raw;                                   // [STAGES][3][2 * TILE]
    __shared__ __align__(8) u64 full[STAGES], empty[STAGES];
    const u64 ntiles = (npairs + TILE - 1) / TILE;
    const u64 *src[3] = {f0, f1, f2};
    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], BLOCK / 32); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    gl_acc a[4];
#pragma unroll
    for (int t = 0; t < 4; t++) { a[t].lo = 0; a[t].hi = 0; a[t].top = 0; }
    // tiles of this block: blockIdx.x, blockIdx.x + gridDim.x, ...
    u64 my = (ntiles > blockIdx.x) ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    auto issue = [&](u64 k) {   // thread 0: fill stage k % STAGES with this block's k-th tile
        const int s = (int)(k % STAGES);
        const u64 tile = blockIdx.x + k * gridDim.x, first = tile * TILE;
        const u32 pairs = (u32)((npairs - first) < (u64)TILE ? (npairs - first) : (u64)TILE), bytes = pairs * 16;
        mbar_expect_tx(&full[s], 3 * bytes);
        for (int j = 0; j < 3; j++) bulk_g2s(tiles + ((size_t)s * 3 + j) * 2 * TILE, src[j] + 2 * first, bytes, &full[s]);
    };
    if (threadIdx.x == 0) for (u64 k = 0; k < my && k < STAGES; k++) issue(k);
    for (u64 k = 0; k < my; k++) {
        const int s = (int)(k % STAGES); const u32 par = (u32)((k / STAGES) & 1);
        mbar_wait(&full[s], par);
        const u64 tile = blockIdx.x + k * gridDim.x, first = tile * TILE;
        const u32 pairs = (u32)((npairs - first) < (u64)TILE ? (npairs - first) : (u64)TILE);
        const u64 *t0 = tiles + ((size_t)s * 3 + 0) * 2 * TILE, *t1 = t0 + 2 * TILE, *t2 = t1 + 2 * TILE;
#pragma unroll 2
        for (u32 i = threadIdx.x; i < pairs; i += BLOCK) {
            ulonglong2 v0 = *reinterpret_cast<const ulonglong2 *>(t0 + 2 * i), v1 = *reinterpret_cast<const ulonglong2 *>(t1 + 2 * i), v2 = *reinterpret_cast<const ulonglong2 *>(t2 + 2 * i);
            u64 c0 = v0.x, c1 = v1.x, c2 = v2.x;
            const u64 s0 = gl_sub(v0.y, c0), s1 = gl_sub(v1.y, c1), s2 = gl_sub(v2.y, c2);
#pragma unroll
            for (int t = 0; t < 4; t++) {
                gl_acc_mac(a[t], w_mul(c0, c1), c2);
                if (t < 3) { c0 = gl_add(c0, s0); c1 = gl_add(c1, s1); c2 = gl_add(c2, s2); }
            }
        }
        __syncwarp();
        if ((threadIdx.x & 31) == 0) mbar_arrive(&empty[s]);          // this warp is done with the stage
        if (threadIdx.x == 0 && k + STAGES < my) { mbar_wait(&empty[s], par); issue(k + STAGES); }
    }
    __shared__ u64 ws[BLOCK / 32][4];
#pragma unroll
    for (int t = 0; t < 4; t++) {
        u64 v = gl_acc_reduce(a[t]);
        for (int d = 16; d > 0; d >>= 1) v = gl_add(v, __shfl_down_sync(0xffffffffu, v, d));
        if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5][t] = v;
    }
    __syncthreads();
    if (threadIdx.x < 4) { u64 v = ws[0][threadIdx.x]; for (int w = 1; w < BLOCK / 32; w++) v = gl_add(v, ws[w][threadIdx.x]); partials[4 * blockIdx.x + threadIdx.x] = v; }
}

// ---- round 2 of a Base polynomial: fold by r (Base -> Ext), write the half-size Ext tables, message from the folded pairs ----
__device__ __forceinline__ gle kfold_b(u64 a, u64 b, gle r) { return e_add(e_mul_base(r, gl_sub(b, a)), e_from_base(a)); }
// Ext lazy accumulation: both limbs of a product as 160-bit sums (c1 = a0 b1 + a1 b0; c0 = a0 b0 + 7 w, w = weak(a1 b1))
struct eacc { gl_acc c0, c1; };
__device__ __forceinline__ void eacc_mac(eacc &a, gle x, gle y) {
    gl_acc_mac(a.c1, x.c0, y.c1); gl_acc_mac(a.c1, x.c1, y.c0);
    u64 w = gl_reduce128_weak(x.c1 * y.c1, __umul64hi(x.c1, y.c1));
    gl_acc_mac(a.c0, x.c0, y.c0); gl_acc_mac(a.c0, w, 7ULL);
}
template <int PPT, int BLOCK, int MINB, bool LAZY>
__global__ void __launch_bounds__(BLOCK, MINB) k_scf3(const u64 *__restrict__ f0, const u64 *__restrict__ f1, const u64 *__restrict__ f2, gle r,
                                                    gle *__restrict__ g0, gle *__restrict__ g1, gle *__restrict__ g2, u64 npairs /* of the folded tables */, gle *__restrict__ partials) {
    eacc la[4]; gle ca[4];
#pragma unroll
    for (int t = 0; t < 4; t++) { la[t].c0 = {0, 0, 0}; la[t].c1 = {0, 0, 0}; ca[t] = e_zero(); }
    const u64 T = (u64)gridDim.x * BLOCK;
    const u64 *src[3] = {f0, f1, f2}; gle *dst[3] = {g0, g1, g2};
    for (u64 i0 = (u64)blockIdx.x * BLOCK + threadIdx.x; i0 < npairs; i0 += PPT * T) {
        ulonglong2 v[PPT][3][2];
#pragma unroll
        for (int p = 0; p < PPT; p++) {
            u64 i = i0 + p * T; if (i >= npairs) i = i0;
#pragma unroll
            for (int j = 0; j < 3; j++) { v[p][j][0] = ld_b2(src[j] + 4 * i); v[p][j][1] = ld_b2(src[j] + 4 * i + 2); }
        }
#pragma unroll
        for (int p = 0; p < PPT; p++) {
            const u64 i = i0 + p * T; const bool ok = i < npairs;
            gle c[3], s[3];
#pragma unroll
            for (int j = 0; j < 3; j++) {
                gle lo = kfold_b(v[p][j][0].x, v[p][j][0].y, r), hi = kfold_b(v[p][j][1].x, v[p][j][1].y, r);
                if (ok) { st_e(dst[j] + 2 * i, lo); st_e(dst[j] + 2 * i + 1, hi); }
                c[j] = lo; s[j] = e_sub(hi, lo);
            }
            if (!ok) c[0] = e_zero(), s[0] = e_zero();
#pragma unroll
            for (int t = 0; t < 4; t++) {
                gle pq = e_mul(c[0], c[1]);
                if (LAZY) eacc_mac(la[t], pq, c[2]); else ca[t] = e_add(ca[t], e_mul(pq, c[2]));
                if (t < 3) { c[0] = e_add(c[0], s[0]); c[1] = e_add(c[1], s[1]); c[2] = e_add(c[2], s[2]); }
            }
        }
    }
    __shared__ gle ws[BLOCK / 32][4];
#pragma unroll
    for (int t = 0; t < 4; t++) {
        gle v = LAZY ? e_make(gl_acc_reduce(la[t].c0), gl_acc_reduce(la[t].c1)) : ca[t];
        for (int d = 16; d > 0; d >>= 1) v = e_add(v, shfl_down_e(v, d));
        if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5][t] = v;
    }
    __syncthreads();
    if (threadIdx.x < 4) { gle v = ws[0][threadIdx.x]; for (int w = 1; w < BLOCK / 32; w++) v = e_add(v, ws[w][threadIdx.x]); partials[4 * blockIdx.x + threadIdx.x] = v; }
}
// later rounds: Ext tables folded by r (4 Ext in -> 2 Ext out per operand) + message
template <int PPT, int BLOCK, int MINB, bool LAZY>
__global__ void __launch_bounds__(BLOCK, MINB) k_sce3(const gle *__restrict__ f0, const gle *__restrict__ f1, const gle *__restrict__ f2, gle r,
                                                    gle *__restrict__ g0, gle *__restrict__ g1, gle *__restrict__ g2, u64 npairs, gle *__restrict__ partials) {
    eacc la[4]; gle ca[4];
#pragma unroll
    for (int t = 0; t < 4; t++) { la[t].c0 = {0, 0, 0}; la[t].c1 = {0, 0, 0}; ca[t] = e_zero(); }
    const u64 T = (u64)gridDim.x * BLOCK;
    const gle *src[3] = {f0, f1, f2}; gle *dst[3] = {g0, g1, g2};
    for (u64 i0 = (u64)blockIdx.x * BLOCK + threadIdx.x; i0 < npairs; i0 += PPT * T) {
#pragma unroll
        for (int p = 0; p < PPT; p++) {
            const u64 i = i0 + p * T; if (i >= npairs) break;
            gle c[3], s[3];
#pragma unroll
            for (int j = 0; j < 3; j++) {
                const gle *q = src[j] + 4 * i;
                gle a0 = ld_e(q), a1 = ld_e(q + 1), a2 = ld_e(q + 2), a3 = ld_e(q + 3);
                gle lo = e_add(a0, e_mul(e_sub(a1, a0), r)), hi = e_add(a2, e_mul(e_sub(a3, a2), r));
                st_e(dst[j] + 2 * i, lo); st_e(dst[j] + 2 * i + 1, hi);
                c[j] = lo; s[j] = e_sub(hi, lo);
            }
#pragma unroll
            for (int t = 0; t < 4; t++) {
                gle pq = e_mul(c[0], c[1]);
                if (LAZY) eacc_mac(la[t], pq, c[2]); else ca[t] = e_add(ca[t], e_mul(pq, c[2]));
                if (t < 3) { c[0] = e_add(c[0], s[0]); c[1] = e_add(c[1], s[1]); c[2] = e_add(c[2], s[2]); }
            }
        }
    }
    __shared__ gle ws[BLOCK / 32][4];
#pragma unroll
    for (int t = 0; t < 4; t++) {
        gle v = LAZY ? e_make(gl_acc_reduce(la[t].c0), gl_acc_reduce(la[t].c1)) : ca[t];
        for (int d = 16; d > 0; d >>= 1) v = e_add(v, shfl_down_e(v, d));
        if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5][t] = v;
    }
    __syncthreads();
    if (threadIdx.x < 4) { gle v = ws[0][threadIdx.x]; for (int w = 1; w < BLOCK / 32; w++) v = e_add(v, ws[w][threadIdx.x]); partials[4 * blockIdx.x + threadIdx.x] = v; }
}

// ---- host <-> resident-kernel round trip (the per-round floor of the resident sumcheck kernel) ----
__device__ __forceinline__ u64 ld_relaxed_sys(const u64 *p) { u64 v; asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ u64 ld_acquire_sys(const u64 *p) { u64 v; asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ void st_release_sys(u64 *p, u64 v) { asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ void st_relaxed_sys(u64 *p, u64 v) { asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
// variant bits: 1 poll with ld.relaxed.sys (else volatile), 2 flag with st.release.sys (else __threadfence_system + volatile store),
// 4 dirty 64 KB of device memory before signalling (as a folding round does), 8 no fence at all (PCIe posted-write order only)
__global__ void k_pingpong(u64 *mailbox, u64 *flag, u64 *out_mapped, u64 *scratch, int n, int variant) {
    for (int k = 1; k <= n; k++) {
        if (threadIdx.x == 0) {
            if (variant & 1) { while (ld_relaxed_sys(mailbox) != (u64)k) {} } else { while (*(volatile u64 *)mailbox != (u64)k) {} }
        }
        __syncthreads();
        if (variant & 4) for (int i = threadIdx.x; i < 8192; i += blockDim.x) scratch[i] = k + i;
        if (threadIdx.x < 8) out_mapped[threadIdx.x] = (u64)k + threadIdx.x;
        __syncthreads();
        if (threadIdx.x == 0) {
            if (variant & 8) st_relaxed_sys(flag, (u64)k);
            else if (variant & 2) st_release_sys(flag, (u64)k);
            else { __threadfence_system(); *(volatile u64 *)flag = (u64)k; }
        }
    }
}
__global__ void k_tiny(u64 *flag, u64 *out_mapped, u64 k) { if (threadIdx.x < 8) out_mapped[threadIdx.x] = k + threadIdx.x; __syncthreads(); if (threadIdx.x == 0) { __threadfence_system(); *(volatile u64 *)flag = k; } }

// sum of the block partials on the host (field addition is exact: any order gives the same element)
static void host_sum_f(const u64 *d, int blocks, u64 out[4]) {
    std::vector<u64> h(4 * blocks); cudaMemcpy(h.data(), d, 32 * blocks, cudaMemcpyDeviceToHost);
    for (int t = 0; t < 4; t++) { u64 s = 0; for (int b = 0; b < blocks; b++) s = gl_add(s, h[4 * b + t]); out[t] = s; }
}
static void host_sum_e(const gle *d, int blocks, gle out[4]) {
    std::vector<gle> h(4 * blocks); cudaMemcpy(h.data(), d, 64 * blocks, cudaMemcpyDeviceToHost);
    for (int t = 0; t < 4; t++) { gle s = e_zero(); for (int b = 0; b < blocks; b++) s = e_add(s, h[4 * b + t]); out[t] = s; }
}

// ---- fs: one round of the resident tail's device transcript (TrP2 in poseidon2.cuh, TrB3 in blake3.cuh) alone, `rounds` rounds back
// to back in a 1-block kernel, with the state image in shared memory and the message loop rolled as in the kernel (whose degree is a
// run-time value): absorb a degree-D message (D + 1 extension elements) and the "Internal round" label, draw the challenge.  The
// message of round r is derived from the previous challenge, so the rounds form one dependent chain as in the kernel.
template <class TR, int D> __global__ void k_fs(u64 *w, int rounds) {
    __shared__ u64 img[TrB3::WORDS];
    for (int i = threadIdx.x; i < TrB3::WORDS; i += blockDim.x) img[i] = w[i];
    __syncthreads();
    if (TR::runs()) {
        const u64 label[2] = {b3::le_word("Internal", 8), b3::le_word(" round", 6)};
        TR t(img);
        u64 c = 1;
        for (int r = 0; r < rounds; r++) {
#pragma unroll 1
            for (int k = 0; k <= D; k++) t.ext(e_make(gl_canon(c * (2 * k + 3)), gl_canon(c * (2 * k + 4))));
            t.label(label);
            const gle ch = t.challenge();
            c = ch.c0 ^ ch.c1;
        }
        t.store(img, nullptr);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < TrB3::WORDS; i += blockDim.x) w[i] = img[i];
}

// =====================================================================================================================
int main(int argc, char **argv) {
    auto want = [&](const char *s) { if (argc <= 1) return true; for (int i = 1; i < argc; i++) if (!strcmp(argv[i], s)) return true; return false; };
    CK(cudaSetDevice(0));
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
    const int SM = prop.multiProcessorCount;
    printf("device %s, %d SMs, clock %.0f MHz\n", prop.name, SM, prop.clockRate / 1e3);
    CK(p2_upload_constants((const u64 *)&DP_P2_EXT_RC[0][0][0], (const u64 *)DP_P2_INT_RC, (const u64 *)DP_P2_DIAG));
    u64 st = 7;
    char *flush = nullptr; CK(cudaMalloc(&flush, 256u << 20));

    if (want("fs")) {
        const int rounds = 2000;
        u64 *w; CK(cudaMalloc(&w, 80 * 8)); CK(cudaMemset(w, 0, 80 * 8));
        printf("[fs] device transcript step alone, one 1-block kernel of %d dependent rounds (256 threads)\n", rounds);
        auto run = [&](const char *name, auto kern) {
            const float ms = time_ms([&] { CK(cudaMemset(w, 0, 80 * 8)); kern<<<1, 256>>>(w, rounds); });
            printf("  %-40s %8.2f us per round\n", name, 1e3 * ms / rounds);
        };
        run("Poseidon2 sponge (warp 0), degree 2", k_fs<TrP2, 2>); run("Poseidon2 sponge (warp 0), degree 3", k_fs<TrP2, 3>);
        run("BLAKE3 hasher (thread 0), degree 2", k_fs<TrB3, 2>); run("BLAKE3 hasher (thread 0), degree 3", k_fs<TrB3, 3>);
        cudaFree(w);
    }

    if (want("perm")) {
        const u64 n_out = 1ULL << 22;     // 2^22 compressions = 2^23 permutations; 256 MB in, 128 MB out (> L2)
        u64 *in, *out, *ref; CK(cudaMalloc(&in, n_out * 64)); CK(cudaMalloc(&out, n_out * 32)); CK(cudaMalloc(&ref, n_out * 32));
        { std::vector<u64> h(n_out * 8); for (auto &v : h) v = gl_canon(sm64(st)); CK(cudaMemcpy(in, h.data(), n_out * 64, cudaMemcpyHostToDevice)); }
        k_up_lib<<<(unsigned)(n_out / 128), 128>>>(in, n_out, ref); CK(cudaDeviceSynchronize());
        const u64 want_sum = checksum(ref, 1 << 16);
        auto report = [&](const char *name, float ms, u64 *o) {
            u64 cs = checksum(o, 1 << 16);
            printf("  %-44s %8.3f ms  %6.2f G perm/s  %s\n", name, ms, 2.0 * n_out / (ms * 1e-3) / 1e9, cs == want_sum ? "ok" : "MISMATCH");
        };
        printf("[perm] %llu compressions per launch (thread-per-hash level kernel)\n", n_out);
        report("lib k_merkle_up<<<n/128,128>>>", time_ms([&] { k_up_lib<<<(unsigned)(n_out / 128), 128>>>(in, n_out, out); }), out);
        report("lib, grid SMx8 persistent, 128", time_ms([&] { k_up_lib<<<SM * 8, 128>>>(in, n_out, out); }), out);
#define RUN_UP(NH, UI, BLOCK, MINB, GRIDMUL) report("v NH=" #NH " UI=" #UI " block=" #BLOCK " minb=" #MINB " grid=SMx" #GRIDMUL, \
            time_ms([&] { k_up_v<NH, UI, BLOCK, MINB><<<SM * GRIDMUL, BLOCK>>>(in, n_out, out); }), out)
        RUN_UP(1, 1, 128, 1, 16); RUN_UP(1, 2, 128, 1, 16); RUN_UP(1, 2, 128, 6, 16); RUN_UP(1, 2, 256, 3, 8); RUN_UP(1, 2, 64, 12, 32);
        RUN_UP(2, 1, 128, 1, 8);  RUN_UP(2, 2, 128, 1, 8);  RUN_UP(2, 2, 128, 4, 8);  RUN_UP(2, 2, 256, 2, 4);  RUN_UP(2, 2, 64, 8, 16);
        RUN_UP(1, 11, 128, 1, 16); RUN_UP(2, 11, 128, 1, 8);
        cudaFree(in); cudaFree(out); cudaFree(ref);
    }

    if (want("lat")) {
        u64 *io; CK(cudaMalloc(&io, 1024 * 64));
        std::vector<u64> h(1024 * 8); for (auto &v : h) v = gl_canon(sm64(st));
        const int LEN = 64;
        printf("[lat] chain of %d dependent compresses (2 permutations each); us per compress\n", LEN);
        auto run = [&](const char *name, auto launch, int threads, int hashes) {
            CK(cudaMemcpy(io, h.data(), 1024 * 64, cudaMemcpyHostToDevice));
            launch(threads); CK(cudaDeviceSynchronize());
            u64 cs = checksum(io, 4);   // hash 0's digest after LEN steps
            CK(cudaMemcpy(io, h.data(), 1024 * 64, cudaMemcpyHostToDevice));
            float ms = time_ms([&] { launch(threads); }, 3, 1);
            printf("  %-52s %3d hashes  %7.2f us/compress   digest0 %016llx\n", name, hashes, 1e3 * ms / LEN, cs);
        };
        // NB: time_ms re-runs the chain on its own output; the digest printed is from the first clean run
        for (int th : {32, 64, 128, 256}) {
            run("thread-per-hash lib p2_compress", [&](int t) { k_chain_lib<<<1, t>>>(io, LEN); }, th, th);
            run("thread-per-hash lat-opt (3-deep internal rounds)", [&](int t) { k_chain_latopt<<<1, t>>>(io, LEN); }, th, th);
            run("thread-per-hash v UI=1", [&](int t) { k_chain_tph<1><<<1, t>>>(io, LEN); }, th, th);
            run("thread-per-hash v UI=2", [&](int t) { k_chain_tph<2><<<1, t>>>(io, LEN); }, th, th);
            run("thread-per-hash v UI=11", [&](int t) { k_chain_tph<11><<<1, t>>>(io, LEN); }, th, th);
        }
        for (int th : {32, 256}) run("8 lanes per hash (lib p2x8_compress)", [&](int t) { k_chain_x8<<<1, t>>>(io, LEN); }, th, th / 8);
        cudaFree(io);
    }

    if (want("sc")) {
        const int NV = 20; const u64 n = 1ULL << NV, npairs = n / 2;
        u64 *f[3]; for (int j = 0; j < 3; j++) { CK(cudaMalloc(&f[j], n * 8)); std::vector<u64> h(n); u64 s2 = j + 1; for (auto &v : h) v = sm64(s2) % GL_P; CK(cudaMemcpy(f[j], h.data(), n * 8, cudaMemcpyHostToDevice)); }
        u64 *part; CK(cudaMalloc(&part, 32 * 65536));
        printf("[sc] round 1, nu=%d, three Base MLEs, degree 3: 25.2 MB algorithmic read\n", NV);
        u64 refm[4];
        k_scb3_lib<256><<<888, 256>>>(f[0], f[1], f[2], npairs, part); CK(cudaDeviceSynchronize()); host_sum_f(part, 888, refm);
        auto rep1 = [&](const char *name, int blocks, float ms) {
            u64 m[4]; host_sum_f(part, blocks, m);
            bool ok = !memcmp(m, refm, 32);
            printf("  %-56s %7.2f us  %7.1f GB/s  %s\n", name, 1e3 * ms, 3.0 * n * 8 / (ms * 1e-3) / 1e9, ok ? "ok" : "MISMATCH");
        };
        auto fl = [&] { cudaMemsetAsync(flush, 1, 256u << 20); };
        // every timed launch is preceded (outside the events? no: inside would count) -- so time pairs and subtract the flush
        float t_flush = time_ms([&] { fl(); });
        auto timed = [&](auto k) { return time_ms([&] { fl(); k(); }) - t_flush; };
        rep1("lib body (2 in flight, canonical acc) 888x256", 888, timed([&] { k_scb3_lib<256><<<888, 256>>>(f[0], f[1], f[2], npairs, part); }));
#define RUN_B(PPT, BLOCK, MINB, GRID) rep1("lean PPT=" #PPT " block=" #BLOCK " minb=" #MINB " grid=" #GRID, GRID, timed([&] { k_scb3<PPT, BLOCK, MINB><<<GRID, BLOCK>>>(f[0], f[1], f[2], npairs, part); }))
        RUN_B(1, 256, 1, 2048); RUN_B(2, 256, 1, 1024); RUN_B(4, 256, 1, 512); RUN_B(2, 256, 4, 528); RUN_B(4, 256, 4, 528); RUN_B(4, 256, 3, 396); RUN_B(2, 128, 8, 1056); RUN_B(4, 128, 8, 1056); RUN_B(8, 128, 4, 528);
        RUN_B(4, 512, 2, 264);
        {
#define RUN_T(TILE, STAGES, BLOCK, MINB, GRID) do { size_t sm_ = (size_t)STAGES * 3 * 2 * TILE * 8; \
            CK(cudaFuncSetAttribute(k_scb3_tma<TILE, STAGES, BLOCK, MINB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_)); \
            rep1("bulk-async TILE=" #TILE " STAGES=" #STAGES " block=" #BLOCK " minb=" #MINB " grid=" #GRID, GRID, \
                 timed([&] { k_scb3_tma<TILE, STAGES, BLOCK, MINB><<<GRID, BLOCK, sm_>>>(f[0], f[1], f[2], npairs, part); })); } while (0)
            RUN_T(512, 3, 256, 2, 264); RUN_T(512, 4, 256, 2, 264); RUN_T(256, 4, 256, 4, 528); RUN_T(1024, 3, 512, 1, 132); RUN_T(512, 2, 256, 3, 396); RUN_T(256, 3, 128, 6, 792);
        }
        // round 2: fold Base -> Ext + message over 2^18 pairs (50.3 MB algorithmic: 25.2 read + 25.2 written)
        gle r = e_make(0x123456789abcdefULL % GL_P, 0xfedcba987654321ULL % GL_P);
        gle *g[3], *g2[3], *parte; for (int j = 0; j < 3; j++) { CK(cudaMalloc(&g[j], n / 2 * 16)); CK(cudaMalloc(&g2[j], n / 4 * 16)); } CK(cudaMalloc(&parte, 64 * 65536));
        printf("[sc] round 2: fold Base->Ext + message, 2^%d pairs: 50.3 MB algorithmic\n", NV - 2);
        gle refe[4];
        k_scf3<1, 256, 1, false><<<1024, 256>>>(f[0], f[1], f[2], r, g[0], g[1], g[2], npairs / 2, parte); CK(cudaDeviceSynchronize()); host_sum_e(parte, 1024, refe);
        const u64 gsum = checksum((u64 *)g[1], 1 << 16);
        auto rep2 = [&](const char *name, int blocks, float ms, double mb, const gle *refx, gle *tab, u64 tabsum) {
            gle m[4]; host_sum_e(parte, blocks, m);
            bool ok = !memcmp(m, refx, 64) && checksum((u64 *)tab, 1 << 16) == tabsum;
            printf("  %-56s %7.2f us  %7.1f GB/s  %s\n", name, 1e3 * ms, mb * 1e6 / (ms * 1e-3) / 1e9, ok ? "ok" : "MISMATCH");
        };
#define RUN_F(PPT, BLOCK, MINB, LAZY, GRID) rep2("fold-b PPT=" #PPT " block=" #BLOCK " minb=" #MINB " lazy=" #LAZY " grid=" #GRID, GRID, \
            timed([&] { k_scf3<PPT, BLOCK, MINB, LAZY><<<GRID, BLOCK>>>(f[0], f[1], f[2], r, g[0], g[1], g[2], npairs / 2, parte); }), 50.33, refe, g[1], gsum)
        RUN_F(1, 256, 1, false, 1024); RUN_F(1, 256, 1, true, 1024); RUN_F(2, 256, 1, false, 512); RUN_F(2, 256, 1, true, 512); RUN_F(1, 256, 3, true, 1024); RUN_F(2, 256, 2, true, 512);
        RUN_F(1, 128, 4, true, 2048); RUN_F(2, 128, 4, true, 1024); RUN_F(1, 128, 6, true, 2048);
        // round 3: fold Ext -> Ext + message over 2^17 pairs (25.2 MB read + 12.6 MB written)
        printf("[sc] round 3: fold Ext->Ext + message, 2^%d pairs: 37.7 MB algorithmic\n", NV - 3);
        gle refe3[4];
        k_sce3<1, 256, 1, false><<<512, 256>>>(g[0], g[1], g[2], r, g2[0], g2[1], g2[2], npairs / 4, parte); CK(cudaDeviceSynchronize()); host_sum_e(parte, 512, refe3);
        const u64 g2sum = checksum((u64 *)g2[1], 1 << 16);
#define RUN_E(PPT, BLOCK, MINB, LAZY, GRID) rep2("fold-e PPT=" #PPT " block=" #BLOCK " minb=" #MINB " lazy=" #LAZY " grid=" #GRID, GRID, \
            timed([&] { k_sce3<PPT, BLOCK, MINB, LAZY><<<GRID, BLOCK>>>(g[0], g[1], g[2], r, g2[0], g2[1], g2[2], npairs / 4, parte); }), 37.75, refe3, g2[1], g2sum)
        RUN_E(1, 256, 1, false, 512); RUN_E(1, 256, 1, true, 512); RUN_E(1, 256, 3, true, 512); RUN_E(1, 128, 4, true, 1024); RUN_E(1, 128, 6, true, 1024); RUN_E(2, 128, 4, true, 512); RUN_E(1, 64, 8, true, 2048);
    }
    if (want("pp")) {
        u64 *pin; CK(cudaHostAlloc((void **)&pin, 4096 * 3, cudaHostAllocMapped));
        volatile u64 *mailbox = pin, *flag = pin + 512, *outm = pin + 1024;
        u64 *scratch; CK(cudaMalloc(&scratch, 8192 * 8));
        const int N = 2000;
        printf("[pp] host <-> resident kernel round trip, %d iterations (host: store mailbox, spin on flag)\n", N);
        for (int variant : {0, 1, 2, 3, 4, 6, 8, 9, 12}) {
            mailbox[0] = 0; flag[0] = 0;
            k_pingpong<<<1, 256>>>((u64 *)mailbox, (u64 *)flag, (u64 *)outm, scratch, N, variant);
            auto t0 = std::chrono::steady_clock::now();
            for (int k = 1; k <= N; k++) {
                __atomic_store_n(&mailbox[0], (u64)k, __ATOMIC_RELEASE);
                while (__atomic_load_n(&flag[0], __ATOMIC_ACQUIRE) != (u64)k) {}
            }
            double us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count();
            CK(cudaDeviceSynchronize());
            printf("  variant %2d (%s poll, %s%s): %6.2f us per round trip (payload word0 %llu)\n", variant, (variant & 1) ? "ld.relaxed.sys" : "volatile", (variant & 8) ? "st.relaxed.sys, no fence" : (variant & 2) ? "st.release.sys" : "membar.sys + volatile st",
                   (variant & 4) ? ", 64 KB device writes first" : "", us / N, (unsigned long long)outm[0]);
        }
        {   // reference: one tiny launch per round
            flag[0] = 0;
            auto t0 = std::chrono::steady_clock::now();
            for (int k = 1; k <= N; k++) { k_tiny<<<1, 256>>>((u64 *)flag, (u64 *)outm, (u64)k); while (__atomic_load_n(&flag[0], __ATOMIC_ACQUIRE) != (u64)k) {} }
            double us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count();
            CK(cudaDeviceSynchronize());
            printf("  one launch per round (tiny kernel + membar.sys + flag): %6.2f us per round\n", us / N);
        }
    }
    if (want("launch")) {
        // How many kernel launches per second does one process sustain from T host threads, each on its own stream?  (a) fire and
        // forget: T threads x N tiny launches, one sync at the end; (b) round trips: launch, spin on the flag the kernel raises
        // (the prover's per-round pattern); (c) like (a) with a burst of 4 launches between flag waits (the prover's mix).
        printf("[launch] tiny-kernel launches from T threads on T streams (one process, one context)\n");
        for (int T : {1, 2, 4, 8, 16, 24, 32}) {
            const int N = 20000 / (T > 4 ? 2 : 1);
            std::vector<cudaStream_t> st(T); std::vector<u64 *> pins(T);
            for (int t = 0; t < T; t++) { CK(cudaStreamCreateWithFlags(&st[t], cudaStreamNonBlocking)); CK(cudaHostAlloc((void **)&pins[t], 4096, cudaHostAllocMapped)); pins[t][0] = 0; }
            for (int mode = 0; mode < 3; mode++) {
                std::atomic<int> go{0};
                std::vector<std::thread> th;
                std::vector<double> call_us(T, 0.0);
                for (int t = 0; t < T; t++) th.emplace_back([&, t] {
                    cudaSetDevice(0);
                    volatile u64 *flag = pins[t]; u64 *outm = pins[t] + 64;
                    while (!go.load()) {}
                    double acc = 0;
                    for (int k = 1; k <= N; k++) {
                        auto c0 = std::chrono::steady_clock::now();
                        k_tiny<<<1, 256, 0, st[t]>>>((u64 *)flag, outm, (u64)k + (u64)mode * 1000000);
                        if (mode == 2) for (int q = 0; q < 3; q++) k_tiny<<<1, 256, 0, st[t]>>>((u64 *)flag, outm, (u64)k + (u64)mode * 1000000);
                        acc += std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - c0).count();
                        if (mode >= 1) while (__atomic_load_n(&flag[0], __ATOMIC_ACQUIRE) != (u64)k + (u64)mode * 1000000) {}
                    }
                    cudaStreamSynchronize(st[t]);
                    call_us[t] = acc / N;
                });
                auto t0 = std::chrono::steady_clock::now();
                go.store(1);
                for (auto &x : th) x.join();
                double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
                double per = 0; for (double v : call_us) per += v; per /= T;
                const double launches = (double)T * N * (mode == 2 ? 4 : 1);
                printf("  T=%2d %-28s %8.1f k launches/s   %6.2f us per loop iteration per thread, %5.2f us inside the launch call(s)\n", T,
                       mode == 0 ? "fire-and-forget" : mode == 1 ? "launch + spin on flag" : "4 launches + spin on flag", launches / sec / 1e3, 1e6 * sec / N, per);
            }
            for (int t = 0; t < T; t++) { cudaStreamDestroy(st[t]); cudaFreeHost(pins[t]); }
        }
    }
    printf("done (%s)\n", cudaGetErrorString(cudaDeviceSynchronize()));
    return 0;
}
