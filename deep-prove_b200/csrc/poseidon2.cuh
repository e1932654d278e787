// Poseidon2 (Goldilocks, width 8, x^7, 4+22+4 rounds) with the state held in registers, and the two
// Merkle hash shapes built on it.  Reference: ff_ext/src/lib.rs:177-235 (NoAllocPoseidon),
// poseidon/src/poseidon_hash.rs:17-71 over p3 DuplexChallenger<_,_,8,4> (overwrite-mode absorb,
// outputs popped from the end of the rate).  Constants: include/dp_poseidon2_constants.h (provenance and
// pinning status are documented in the generator script that emits that header).
#pragma once
#include "gl.cuh"
#include "../../include/dp_poseidon2_constants.h"

__constant__ u64 c_p2_ext[2][4][8];
__constant__ u64 c_p2_int[22];
__constant__ u64 c_p2_diag[8];

static inline cudaError_t p2_upload_constants(const u64 *ext /*64*/, const u64 *internal /*22*/, const u64 *diag /*8*/) {
    cudaError_t e;
    if ((e = cudaMemcpyToSymbol(c_p2_ext, ext, sizeof(u64) * 64)) != cudaSuccess) return e;
    if ((e = cudaMemcpyToSymbol(c_p2_int, internal, sizeof(u64) * 22)) != cudaSuccess) return e;
    return cudaMemcpyToSymbol(c_p2_diag, diag, sizeof(u64) * 8);
}

// ---- "weak" arithmetic: state words live in [0, 2^64) (not reduced below p) between operations ----------------
// The permutation is ALU-bound, so it is written to minimise instructions: products are reduced to a weak 64-bit
// value (11 instructions instead of 16 + canonicalisation), the linear layers accumulate in 64+32-bit "wide"
// sums that are folded once per output, and the internal-layer multiply-add is one 128-bit accumulate + one
// reduction.  Only the four digest words are canonicalised at the end.  Every step is exact modular arithmetic,
// so the digests are bit-identical to the canonical formulation.
struct p2w { u64 lo; u32 hi; };                                                   // value = lo + hi * 2^64
__device__ __forceinline__ u64 w_red(u64 lo, u64 hi) { return gl_reduce128_weak(lo, hi); }
__device__ __forceinline__ u64 w_mul(u64 a, u64 b) { u64 lo, hi; gl_mul128(a, b, lo, hi); return w_red(lo, hi); }
__device__ __forceinline__ u64 w_add_canon(u64 a, u64 c) {                        // a weak, c < p  ->  weak
    u64 r; asm("{\n\t.reg .u32 c;\n\t.reg .u64 t;\n\tadd.cc.u64 t, %1, %2;\n\taddc.u32 c, 0, 0;\n\tmad.wide.u32 %0, c, 0xFFFFFFFF, t;\n\t}" : "=l"(r) : "l"(a), "l"(c));
    return r;
}
__device__ __forceinline__ u64 w_add(u64 a, u64 b) {                              // weak + weak -> weak (two possible wraps)
    u64 r; asm("{\n\t.reg .u32 c;\n\t.reg .u64 t, e;\n\tadd.cc.u64 t, %1, %2;\n\taddc.u32 c, 0, 0;\n\tmul.wide.u32 e, c, 0xFFFFFFFF;\n\t"
               "add.cc.u64 t, t, e;\n\taddc.u32 c, 0, 0;\n\tmad.wide.u32 %0, c, 0xFFFFFFFF, t;\n\t}" : "=l"(r) : "l"(a), "l"(b));
    return r;
}
__device__ __forceinline__ p2w ww(u64 a) { p2w r; r.lo = a; r.hi = 0; return r; }
__device__ __forceinline__ p2w ww_add(p2w a, p2w b) { asm("{\n\tadd.cc.u64 %0, %0, %2;\n\taddc.u32 %1, %1, %3;\n\t}" : "+l"(a.lo), "+r"(a.hi) : "l"(b.lo), "r"(b.hi)); return a; }
__device__ __forceinline__ p2w ww_addu(p2w a, u64 b) { asm("{\n\tadd.cc.u64 %0, %0, %2;\n\taddc.u32 %1, %1, 0;\n\t}" : "+l"(a.lo), "+r"(a.hi) : "l"(b)); return a; }
__device__ __forceinline__ u64 ww_fold(p2w a) {                                   // hi <= a few dozen: hi * 2^64 == hi * EPS
    u64 r; asm("{\n\t.reg .u64 t;\n\t.reg .u32 c;\n\tmul.wide.u32 t, %2, 0xFFFFFFFF;\n\tadd.cc.u64 t, %1, t;\n\taddc.u32 c, 0, 0;\n\tmad.wide.u32 %0, c, 0xFFFFFFFF, t;\n\t}" : "=l"(r) : "l"(a.lo), "r"(a.hi));
    return r;
}
// a * c + (sum as wide) -> weak, one reduction  (internal layer: s[i] * diag[i] + sum)
__device__ __forceinline__ u64 w_mul_add(u64 a, u64 c, p2w sum) {
    u64 lo, hi; gl_mul128(a, c, lo, hi);
    asm("{\n\t.reg .u64 h64;\n\tcvt.u64.u32 h64, %3;\n\tadd.cc.u64 %0, %0, %2;\n\taddc.u64 %1, %1, h64;\n\t}" : "+l"(lo), "+l"(hi) : "l"(sum.lo), "r"(sum.hi));
    return w_red(lo, hi);
}
__device__ __forceinline__ u64 p2_pow7(u64 x) { u64 x2 = w_mul(x, x), x4 = w_mul(x2, x2); return w_mul(w_mul(x2, x), x4); }
// p3 MDSMat4 = circ(2,3,1,1) on each half, then state[i] += column sums: out[i] = 2 n[i] + n[i ^ 4]
__device__ __forceinline__ void p2_mat4w(u64 x0, u64 x1, u64 x2, u64 x3, p2w &n0, p2w &n1, p2w &n2, p2w &n3) {
    p2w t01 = ww_addu(ww(x0), x1), t23 = ww_addu(ww(x2), x3), all = ww_add(t01, t23);
    p2w a1 = ww_addu(all, x1), a3 = ww_addu(all, x3);
    n0 = ww_add(a1, t01);                       // 2x0 + 3x1 + x2 + x3
    n1 = ww_addu(ww_addu(a1, x2), x2);          // x0 + 2x1 + 3x2 + x3
    n2 = ww_add(a3, t23);                       // x0 + x1 + 2x2 + 3x3
    n3 = ww_addu(ww_addu(a3, x0), x0);          // 3x0 + x1 + x2 + 2x3
}
__device__ __forceinline__ void p2_mds_light(u64 (&s)[8]) {
    p2w n[8];
    p2_mat4w(s[0], s[1], s[2], s[3], n[0], n[1], n[2], n[3]);
    p2_mat4w(s[4], s[5], s[6], s[7], n[4], n[5], n[6], n[7]);
#pragma unroll
    for (int i = 0; i < 8; i++) s[i] = ww_fold(ww_add(ww_add(n[i], n[i]), n[i ^ 4]));
}
// One loop over the 30 rounds with a warp-uniform branch between the two round shapes: ONE copy of the external-round body
// (8 S-boxes + linear layer, ~900 instructions) instead of two, so the whole permutation is ~1.3 k instructions of code.  The
// level kernels were stalled on instruction fetch more than on anything else (ncu r02b: no_instruction 3.7 stall cycles per
// issued instruction with the ~4 k-instruction version: two permutations x three round loops inlined back to back).
__device__ __forceinline__ void p2_permute(u64 (&s)[8]) {      // weak in, weak out
    p2_mds_light(s);
#pragma unroll 1
    for (int r = 0; r < 30; r++) {
        if (r < 4 || r >= 26) {
            const u64 *rc = r < 4 ? c_p2_ext[0][r] : c_p2_ext[1][r - 26];
#pragma unroll
            for (int i = 0; i < 8; i++) s[i] = p2_pow7(w_add_canon(s[i], rc[i]));
            p2_mds_light(s);
        } else {
            s[0] = p2_pow7(w_add_canon(s[0], c_p2_int[r - 4]));
            p2w sum = ww(s[0]);
#pragma unroll
            for (int i = 1; i < 8; i++) sum = ww_addu(sum, s[i]);
#pragma unroll
            for (int i = 0; i < 8; i++) s[i] = w_mul_add(s[i], c_p2_diag[i], sum);
        }
    }
}

// Latency-optimised formulation for the tree tops (one thread per hash, few hashes): the only serial dependency of the internal
// rounds is the S-box lane, x' = (d0 + 1) y + R with y = (x + c)^7 and R = the sum of the other seven words, so the chain per round
// is three multiplications deep -- [t^2 | u = (d0+1) t] -> [t^4 | u t^2] -> (u t^2) t^4 + R -- instead of five (S-box, then the
// multiply-add); y itself and the seven multiply-adds of the other words sit in the shadow of the next round's chain.  Two extra
// multiplications per round, exact arithmetic, same digest.
__device__ __forceinline__ u64 w_mul_addu(u64 a, u64 b, u64 c) {                  // a * b + c -> weak (a, b, c any u64)
    u64 lo, hi; gl_mul128(a, b, lo, hi);
    asm("{\n\tadd.cc.u64 %0, %0, %2;\n\taddc.u64 %1, %1, 0;\n\t}" : "+l"(lo), "+l"(hi) : "l"(c));
    return w_red(lo, hi);
}
__device__ __forceinline__ void p2_permute_lat(u64 (&s)[8]) {  // weak in, weak out
    p2_mds_light(s);
#pragma unroll 1
    for (int r = 0; r < 4; r++) {
#pragma unroll
        for (int i = 0; i < 8; i++) s[i] = p2_pow7(w_add_canon(s[i], c_p2_ext[0][r][i]));
        p2_mds_light(s);
    }
    const u64 d0p1 = c_p2_diag[0] + 1;                          // diag is canonical (< p), so this fits; weak is fine for w_mul
    p2w R = ww(s[1]);
#pragma unroll
    for (int i = 2; i < 8; i++) R = ww_addu(R, s[i]);
#pragma unroll 2
    for (int r = 0; r < 22; r++) {
        const u64 t = w_add_canon(s[0], c_p2_int[r]);
        const u64 t2 = w_mul(t, t), u = w_mul(t, d0p1);
        const u64 t4 = w_mul(t2, t2), u3 = w_mul(u, t2), t3 = w_mul(t, t2);
        s[0] = w_mul_addu(u3, t4, ww_fold(R));
        const p2w sum = ww_addu(R, w_mul(t3, t4));
        p2w nr; nr.lo = 0; nr.hi = 0;
#pragma unroll
        for (int i = 1; i < 8; i++) { s[i] = w_mul_add(s[i], c_p2_diag[i], sum); nr = ww_addu(nr, s[i]); }
        R = nr;
    }
#pragma unroll 1
    for (int r = 0; r < 4; r++) {
#pragma unroll
        for (int i = 0; i < 8; i++) s[i] = p2_pow7(w_add_canon(s[i], c_p2_ext[1][r][i]));
        p2_mds_light(s);
    }
}
__device__ __forceinline__ void p2_compress_lat(const u64 x[4], const u64 y[4], u64 out[4]) {
    u64 s[8] = {x[0], x[1], x[2], x[3], 0, 0, 0, 0};
#pragma unroll 1
    for (int half = 0; half < 2; half++) {
        if (half) { s[0] = y[0]; s[1] = y[1]; s[2] = y[2]; s[3] = y[3]; }
        p2_permute_lat(s);
    }
    out[0] = gl_canon_weak(s[3]); out[1] = gl_canon_weak(s[2]); out[2] = gl_canon_weak(s[1]); out[3] = gl_canon_weak(s[0]);
}

// ---- lane-parallel variant: 8 consecutive lanes hold the 8 state words of ONE permutation ----------------
// Used where a level has too few hashes to fill the GPU with one thread per hash (tree tops, witness-sized
// trees): the dependent-instruction chain per permutation drops ~3x (every lane does one S-box in the full
// rounds; the linear layers are warp shuffles inside the 8-lane group).
__device__ __forceinline__ u64 shfl8(u64 v, int src) { return __shfl_sync(0xffffffffu, v, src, 8); }
__device__ __forceinline__ u64 shfl8_xor(u64 v, int m) { return __shfl_xor_sync(0xffffffffu, v, m, 8); }
__device__ __forceinline__ u64 p2x8_mds_light(u64 s, int lane8) {
    int g = lane8 & 4, r = lane8 & 3;
    u64 a = shfl8(s, g + ((r + 1) & 3)), b = shfl8(s, g + ((r + 2) & 3)), c = shfl8(s, g + ((r + 3) & 3));
    // row r of circ(2,3,1,1): 2 x_r + 3 x_{r+1} + x_{r+2} + x_{r+3}
    p2w o = ww_addu(ww_addu(ww_addu(ww_addu(ww_addu(ww_addu(ww(s), s), a), a), a), b), c);
    u64 of = ww_fold(o);
    u64 partner = shfl8_xor(of, 4);
    return ww_fold(ww_addu(ww_addu(ww(of), of), partner));     // state[i] += out[i] + out[i ^ 4]
}
// sum over the 8 lanes of a group (every lane gets it)
__device__ __forceinline__ u64 p2x8_allsum(u64 v) { v = w_add(v, shfl8_xor(v, 1)); v = w_add(v, shfl8_xor(v, 2)); return w_add(v, shfl8_xor(v, 4)); }
__device__ __forceinline__ u64 p2x8_permute(u64 s, int lane8) {
    s = p2x8_mds_light(s, lane8);
#pragma unroll 1
    for (int r = 0; r < 4; r++) { s = p2_pow7(w_add_canon(s, c_p2_ext[0][r][lane8])); s = p2x8_mds_light(s, lane8); }
    // Internal rounds: S-box on lane 0, then an 8-lane all-reduce, then the multiply-add.  (A variant that keeps the sum of words 1..7
    // on every lane and refreshes it in the shadow of the next S-box was measured slower per compress with
    // tools/kbench.cu `lat`: the extra shuffles it issues ahead of the S-box cost more than the all-reduce latency they hide.)
    const u64 dg = c_p2_diag[lane8];
#pragma unroll 1
    for (int r = 0; r < 22; r++) {
        if (lane8 == 0) s = p2_pow7(w_add_canon(s, c_p2_int[r]));
        const u64 sum = p2x8_allsum(s);
        s = w_mul_add(s, dg, ww(sum));
    }
#pragma unroll 1
    for (int r = 0; r < 4; r++) { s = p2_pow7(w_add_canon(s, c_p2_ext[1][r][lane8])); s = p2x8_mds_light(s, lane8); }
    return s;
}
// lanes 0..3 pass x[lane] / y[lane] (lanes 4..7 pass anything); returns on lane k < 4 the digest word 3 - k
__device__ __forceinline__ u64 p2x8_compress(u64 xw, u64 yw, int lane8) {
    u64 s = lane8 < 4 ? xw : 0ULL;
    s = p2x8_permute(s, lane8);
    if (lane8 < 4) s = yw;
    s = p2x8_permute(s, lane8);
    return gl_canon_weak(s);    // lane k holds state[k]; digest = [s3, s2, s1, s0]
}

// DuplexChallenger<F, Poseidon2, WIDTH = 8, RATE = 4> (host/transcript.hpp Sponge) on the 8 lanes of a group: lane k holds state
// word k (canonical) and, for k < 4, input word k; nin / nout are uniform.  The output buffer is not stored: a duplex copies the
// first four state words into it and nothing else changes the state before the next duplex, so out[k] == state[k] while nout > 0.
// Every lane of the warp must call these together (the permutation shuffles over the full mask).
// Exchange format with the host (Sponge::save / load): [state[0..7], in[0..3], nin, nout].
static constexpr int P2S_WORDS = 14;
struct P2Sponge { u64 st, in; u32 nin, nout; };
__device__ __forceinline__ void p2s_load(P2Sponge &s, const u64 *w, int lane8) {
    s.st = w[lane8]; s.in = lane8 < 4 ? w[8 + lane8] : 0; s.nin = (u32)w[12]; s.nout = (u32)w[13];
}
__device__ __forceinline__ void p2s_store(const P2Sponge &s, u64 *w, int lane8) {
    w[lane8] = s.st;
    if (lane8 < 4) w[8 + lane8] = s.in;
    if (lane8 == 0) { w[12] = s.nin; w[13] = s.nout; }
}
__device__ __forceinline__ void p2s_duplex(P2Sponge &s, int lane8) {
    if (lane8 < (int)s.nin) s.st = s.in;
    s.nin = 0;
    s.st = gl_canon_weak(p2x8_permute(s.st, lane8));
    s.nout = 4;
}
__device__ __forceinline__ void p2s_observe(P2Sponge &s, u64 v, int lane8) {
    s.nout = 0;
    if (lane8 == (int)s.nin) s.in = v;
    if (++s.nin == 4) p2s_duplex(s, lane8);
}
__device__ __forceinline__ u64 p2s_sample(P2Sponge &s, int lane8) {
    if (s.nin || !s.nout) p2s_duplex(s, lane8);
    return shfl8(s.st, (int)--s.nout);
}

// The transcripts of the resident sumcheck kernels are compile-time policies (TrP2 here, TrB3 in blake3.cuh).  The threads of a block
// for which runs() holds build one and call its members together; the state image lives in shared memory between calls and the
// challenges are valid in thread 0.  TrP2: BasicTranscript, the sponge above on the 8-lane groups of warp 0.
struct TrP2 {
    static constexpr int WORDS = P2S_WORDS;
    __device__ static bool runs() { return threadIdx.x < 32; }
    P2Sponge s; int l8;
    __device__ explicit TrP2(const u64 *w) : l8(threadIdx.x & 7) { p2s_load(s, w, l8); }
    __device__ void ext(gle e) { p2s_observe(s, e.c0, l8); p2s_observe(s, e.c1, l8); }                 // append_field_element_ext
    __device__ void usize(u64 v) { p2s_observe(s, v, l8); }                                             // append_usize
    __device__ void label(const u64 (&w)[2]) { p2s_observe(s, w[0], l8); p2s_observe(s, w[1], l8); }   // append_message, 9..16 bytes
    __device__ gle challenge() { const u64 c0 = p2s_sample(s, l8), c1 = p2s_sample(s, l8); return e_make(c0, c1); }
    __device__ void store(u64 *w, u64 *also /* or null */) { __syncwarp(); if (threadIdx.x < 8) { p2s_store(s, w, l8); if (also) p2s_store(s, also, l8); } }
};

// compress(x, y): absorb x -> permute -> overwrite rate with y -> permute -> [s3, s2, s1, s0]  (one copy of the permutation: see above)
__device__ __forceinline__ void p2_compress(const u64 x[4], const u64 y[4], u64 out[4]) {
    u64 s[8] = {x[0], x[1], x[2], x[3], 0, 0, 0, 0};
#pragma unroll 1
    for (int half = 0; half < 2; half++) {
        if (half) { s[0] = y[0]; s[1] = y[1]; s[2] = y[2]; s[3] = y[3]; }
        p2_permute(s);
    }
    out[0] = gl_canon_weak(s[3]); out[1] = gl_canon_weak(s[2]); out[2] = gl_canon_weak(s[1]); out[3] = gl_canon_weak(s[0]);
}

// PoseidonHash::hash_or_noop (poseidon/src/poseidon_hash.rs:22-28) for n elements fetched through `get(i)`:
// n <= 4: zero-padded copy, no permutation; else the duplex sponge (rate 4, overwrite-mode absorb, a trailing partial
// block overwrites only its own words) and the digest is popped from the end of the rate: [s3, s2, s1, s0].
template <class F>
__device__ __forceinline__ void p2_hash_or_noop(F get, int n, u64 out[4]) {
    if (n <= 4) { for (int i = 0; i < 4; i++) out[i] = i < n ? get(i) : 0ULL; return; }
    u64 s[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < n; i += 4) {
#pragma unroll
        for (int k = 0; k < 4; k++) if (i + k < n) s[k] = get(i + k);
        p2_permute(s);
    }
    out[0] = gl_canon_weak(s[3]); out[1] = gl_canon_weak(s[2]); out[2] = gl_canon_weak(s[1]); out[3] = gl_canon_weak(s[0]);
}
