// Goldilocks F = Z/(2^64 - 2^32 + 1) and E = F[X]/(X^2 - 7) for sm_90a device code (and host code
// inside the library, for the O(degree)-sized per-round glue).
// Reference semantics: ff_ext/src/lib.rs:7,13 (p3 Goldilocks / BinomialExtensionField<_,2>, W = 7).
// All values are canonical (< p) in memory and in registers between operations; E is AoS {c0,c1} so a
// 16-byte vector load brings one element, exactly the reference's Vec<E> layout.
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>

#define GL_HD __host__ __device__ __forceinline__

typedef unsigned long long u64;
typedef unsigned int u32;

static constexpr u64 GL_P = 0xFFFFFFFF00000001ULL;
static constexpr u64 GL_EPS = 0xFFFFFFFFULL;  // 2^64 mod p

GL_HD u64 gl_canon(u64 a) { return a >= GL_P ? a - GL_P : a; }

// hi*2^64 + lo  ->  "weak" representative in [0, 2^64) (not necessarily < p)
__device__ __forceinline__ u64 gl_reduce128_weak(u64 lo, u64 hi) {
    u64 r;
    asm("{\n\t.reg .u64 t0, t1, m64;\n\t.reg .u32 hl, hh, m;\n\t"
        "mov.b64 {hl, hh}, %2;\n\t"
        "cvt.u64.u32 m64, hh;\n\t"
        "sub.cc.u64 t0, %1, m64;\n\t"                          // lo - hi_hi          (2^96 == -1)
        "subc.u32 m, 0, 0;\n\t"
        "cvt.u64.u32 m64, m;\n\t"
        "sub.u64 t0, t0, m64;\n\t"                             // borrow: - EPS, cannot underflow
        "mul.wide.u32 t1, hl, 0xFFFFFFFF;\n\t"                 // hi_lo * (2^32 - 1)   (2^64 == 2^32 - 1)
        "add.cc.u64 t0, t0, t1;\n\t"
        "addc.u32 m, 0, 0;\n\t"                               // NB: subc after add.cc does NOT give -carry (borrow = !carry in hardware)
        "mad.wide.u32 %0, m, 0xFFFFFFFF, t0;\n\t}"            // carry: + EPS, cannot carry again
        : "=l"(r) : "l"(lo), "l"(hi));
    return r;
}
// 64 x 64 -> 128 bits
__device__ __forceinline__ void gl_mul128(u64 a, u64 b, u64 &lo, u64 &hi) { lo = a * b; hi = __umul64hi(a, b); }
__device__ __forceinline__ u64 gl_canon_weak(u64 r) {          // [0, 2^64) -> [0, p)
    u64 t; u32 c;
    asm("{\n\tadd.cc.u64 %0, %2, 0xFFFFFFFF;\n\taddc.u32 %1, 0, 0;\n\t}" : "=l"(t), "=r"(c) : "l"(r));
    return c ? t : r;
}
#ifdef __CUDA_ARCH__
// Device fast paths: explicit carry chains (add.cc / addc / sub.cc / subc).  The compiler's lowering of the
// compare-and-select formulation spends ~2x the instructions, almost all on the half-rate ALU pipe, and the
// Poseidon2 / Ext-multiply kernels are ALU-bound (ncu: ALU pipe 73 % active, DRAM 0.2 %).
// After add.cc, `addc c, 0, 0` yields the carry (0/1); after sub.cc, `subc m, 0, 0` yields 0 - borrow
// (0 or 0xFFFFFFFF == 2^64 mod p).
// after sub.cc it yields 0 - borrow.  The two flags are NOT interchangeable: use addc after add.cc, subc after sub.cc.
__device__ __forceinline__ u64 gl_add(u64 a, u64 b) {          // a, b < p  ->  < p
    u64 s, t; u32 c;
    asm("{\n\t.reg .u32 c1;\n\t"
        "add.cc.u64 %0, %3, %4;\n\t"
        "addc.u32 c1, 0, 0;\n\t"
        "add.cc.u64 %1, %0, 0xFFFFFFFF;\n\t"                  // s + EPS == s - p (mod 2^64); carries iff s >= p
        "addc.u32 %2, c1, 0;\n\t}" : "=l"(s), "=l"(t), "=r"(c) : "l"(a), "l"(b));
    return c ? t : s;                                          // a + b >= p  <=>  either addition carried
}
__device__ __forceinline__ u64 gl_sub(u64 a, u64 b) {          // a, b < p  ->  < p
    u64 d; u32 m;
    asm("{\n\tsub.cc.u64 %0, %2, %3;\n\tsubc.u32 %1, 0, 0;\n\t}" : "=l"(d), "=r"(m) : "l"(a), "l"(b));
    return d - (u64)m;                                         // borrow: + p == - EPS (mod 2^64)
}
__device__ __forceinline__ u64 gl_reduce128(u64 lo, u64 hi) { return gl_canon_weak(gl_reduce128_weak(lo, hi)); }
__device__ __forceinline__ u64 gl_mul_weak(u64 a, u64 b) { u64 lo, hi; gl_mul128(a, b, lo, hi); return gl_reduce128_weak(lo, hi); }   // any u64 inputs -> [0, 2^64)
__device__ __forceinline__ void gl_mul_wide(u64 a, u64 b, u64 &lo, u64 &hi) { lo = a * b; hi = __umul64hi(a, b); }
GL_HD u64 gl_neg(u64 a) { return a ? GL_P - a : 0ULL; }
GL_HD u64 gl_dbl(u64 a) { return gl_add(a, a); }
#else
GL_HD u64 gl_add(u64 a, u64 b) {
    u64 s = a + b;
    // a,b < p: on wrap the true sum is s + 2^64, and (s + 2^64) - p == s - p (mod 2^64)
    return (s < a || s >= GL_P) ? s - GL_P : s;
}
GL_HD u64 gl_sub(u64 a, u64 b) { u64 d = a - b; return a < b ? d + GL_P : d; }
GL_HD u64 gl_neg(u64 a) { return a ? GL_P - a : 0ULL; }
GL_HD u64 gl_dbl(u64 a) { return gl_add(a, a); }

GL_HD void gl_mul_wide(u64 a, u64 b, u64 &lo, u64 &hi) {
    unsigned __int128 t = (unsigned __int128)a * b; lo = (u64)t; hi = (u64)(t >> 64);
}
// reduce hi*2^64 + lo (any 128-bit value) to canonical form: 2^64 = 2^32 - 1, 2^96 = -1 (mod p)
GL_HD u64 gl_reduce128(u64 lo, u64 hi) {
    u64 hi_hi = hi >> 32, hi_lo = hi & GL_EPS;
    u64 t0 = lo - hi_hi;
    if (lo < hi_hi) t0 -= GL_EPS;            // borrow: + p == - EPS (mod 2^64), cannot underflow
    u64 t1 = hi_lo * GL_EPS;                 // < 2^64
    u64 r = t0 + t1;
    if (r < t1) r += GL_EPS;                 // carry: 2^64 == EPS (mod p), cannot overflow again
    return r >= GL_P ? r - GL_P : r;
}
#endif
GL_HD u64 gl_mul(u64 a, u64 b) { u64 lo, hi; gl_mul_wide(a, b, lo, hi); return gl_reduce128(lo, hi); }
GL_HD u64 gl_sqr(u64 a) { return gl_mul(a, a); }
GL_HD u64 gl_mul7(u64 a) { u64 lo, hi; gl_mul_wide(a, 7ULL, lo, hi); return gl_reduce128(lo, hi); }
GL_HD u64 gl_pow(u64 a, u64 e) { u64 r = 1; while (e) { if (e & 1) r = gl_mul(r, a); a = gl_sqr(a); e >>= 1; } return r; }
GL_HD u64 gl_inv(u64 a) { return gl_pow(a, GL_P - 2); }

struct __align__(16) gle {  // one E element
    u64 c0, c1;
};
GL_HD gle e_make(u64 a, u64 b) { gle r; r.c0 = a; r.c1 = b; return r; }
GL_HD gle e_from_host(const uint64_t *p) { return e_make(gl_canon(p[0]), gl_canon(p[1])); }   // an element as the C ABI passes it: {c0, c1}, any u64
GL_HD gle e_zero() { return e_make(0, 0); }
GL_HD gle e_one() { return e_make(1, 0); }
GL_HD gle e_from_base(u64 a) { return e_make(a, 0); }
GL_HD gle e_add(gle a, gle b) { return e_make(gl_add(a.c0, b.c0), gl_add(a.c1, b.c1)); }
GL_HD gle e_sub(gle a, gle b) { return e_make(gl_sub(a.c0, b.c0), gl_sub(a.c1, b.c1)); }
GL_HD gle e_neg(gle a) { return e_make(gl_neg(a.c0), gl_neg(a.c1)); }
GL_HD gle e_dbl(gle a) { return e_add(a, a); }
GL_HD bool e_eq(gle a, gle b) { return a.c0 == b.c0 && a.c1 == b.c1; }
#ifdef __CUDA_ARCH__
// top*2^128 + hi*2^64 + lo with top < 2^31.  2^128 = (2^32-1)^2 = -2^32 (mod p)  =>  subtract top << 32.
__device__ __forceinline__ u64 gl_reduce160(u64 lo, u64 hi, u32 top) {
    u64 r = gl_reduce128_weak(lo, hi), d; u32 m;
    u64 x = (u64)top << 32;
    asm("{\n\tsub.cc.u64 %0, %2, %3;\n\tsubc.u32 %1, 0, 0;\n\t}" : "=l"(d), "=r"(m) : "l"(r), "l"(x));
    return gl_canon_weak(d - (u64)m);                          // borrow: - EPS; r < x < 2^63 here, so no second borrow
}
#else
GL_HD u64 gl_reduce160(u64 lo, u64 hi, u64 top) {  // top*2^128 + hi*2^64 + lo, top < 2^32
    // 2^128 = (2^32-1)^2 mod p = 2^64 - 2^33 + 1 = -2^32 (mod p)  => top*2^128 = -(top << 32)
    u64 r = gl_reduce128(lo, hi);
    return gl_sub(r, gl_canon(top << 32));
}
#endif
// Lazy sum of raw 128-bit products, lo + hi 2^64 + top 2^128: one reduction for the whole sum instead of one per term.
// top < #terms must stay below 2^31 (gl_reduce160).
struct gl_acc { u64 lo, hi; u32 top; };
__device__ __forceinline__ void gl_acc_mac(gl_acc &a, u64 x, u64 y) {   // a += x * y
    u64 pl = x * y, ph = __umul64hi(x, y);
    asm("{\n\tadd.cc.u64 %0, %0, %3;\n\taddc.cc.u64 %1, %1, %4;\n\taddc.u32 %2, %2, 0;\n\t}" : "+l"(a.lo), "+l"(a.hi), "+r"(a.top) : "l"(pl), "l"(ph));
}
__device__ __forceinline__ u64 gl_acc_reduce(const gl_acc &a) { return gl_reduce160(a.lo, a.hi, a.top); }
// (a0 + a1 X)(b0 + b1 X) = (a0 b0 + 7 a1 b1) + (a0 b1 + a1 b0) X.
// The two limbs are each ONE reduction of a <=131-bit sum of raw 128-bit products (fewer reductions
// than 4 reduced multiplies; same canonical result because the arithmetic is exact).
#ifdef __CUDA_ARCH__
__device__ __forceinline__ gle e_mul(gle a, gle b) {
    // c1 = a0 b1 + a1 b0 : one reduction of the 129-bit sum
    gl_acc s = {a.c0 * b.c1, __umul64hi(a.c0, b.c1), 0};
    gl_acc_mac(s, a.c1, b.c0);
    u64 c1 = gl_acc_reduce(s);
    // c0 = a0 b0 + 7 (a1 b1) : reduce a1 b1 to 64 bits (weak), times 7 is a 67-bit addend
    u64 w = gl_reduce128_weak(a.c1 * b.c1, __umul64hi(a.c1, b.c1));
    s = {a.c0 * b.c0, __umul64hi(a.c0, b.c0), 0};
    gl_acc_mac(s, w, 7ULL);
    u64 c0 = gl_acc_reduce(s);
    return e_make(c0, c1);
}
#else
GL_HD gle e_mul(gle a, gle b) {
    u64 l0, h0, l1, h1;
    // c1 = a0 b1 + a1 b0  (129 bits)
    gl_mul_wide(a.c0, b.c1, l0, h0); gl_mul_wide(a.c1, b.c0, l1, h1);
    u64 lo = l0 + l1; u64 c = lo < l0; u64 hi = h0 + h1; u64 top = hi < h0; hi += c; top += (hi < c);
    u64 c1 = gl_reduce160(lo, hi, top);
    // c0 = a0 b0 + 7 a1 b1  (131 bits)
    gl_mul_wide(a.c0, b.c0, l0, h0); gl_mul_wide(a.c1, b.c1, l1, h1);
    // 7 * (h1:l1) as 192-bit
    u64 m_lo, m_c; gl_mul_wide(l1, 7ULL, m_lo, m_c);
    u64 m_hi, m_top; gl_mul_wide(h1, 7ULL, m_hi, m_top);
    m_hi += m_c; m_top += (m_hi < m_c);
    lo = l0 + m_lo; c = lo < l0; hi = h0 + m_hi; top = m_top + (hi < h0); hi += c; top += (hi < c);
    u64 c0 = gl_reduce160(lo, hi, top);
    return e_make(c0, c1);
}
#endif
GL_HD gle e_mul_base(gle a, u64 b) { return e_make(gl_mul(a.c0, b), gl_mul(a.c1, b)); }
GL_HD gle e_sqr(gle a) { return e_mul(a, a); }
GL_HD gle e_inv(gle a) {
    u64 n = gl_sub(gl_sqr(a.c0), gl_mul7(gl_sqr(a.c1)));
    u64 ni = gl_inv(n);
    return e_make(gl_mul(a.c0, ni), gl_mul(gl_neg(a.c1), ni));
}
GL_HD gle e_from_u64(u64 v) { return e_make(gl_canon(v), 0); }

#ifdef __CUDACC__
// 16-byte vector loads/stores of E and of a Base pair
__device__ __forceinline__ gle ld_e(const gle *p) { ulonglong2 v = *reinterpret_cast<const ulonglong2 *>(p); return e_make(v.x, v.y); }
__device__ __forceinline__ void st_e(gle *p, gle v) { *reinterpret_cast<ulonglong2 *>(p) = make_ulonglong2(v.c0, v.c1); }
__device__ __forceinline__ ulonglong2 ld_b2(const u64 *p) { return *reinterpret_cast<const ulonglong2 *>(p); }
__device__ __forceinline__ gle shfl_down_e(gle v, int d) {
    gle r; r.c0 = __shfl_down_sync(0xffffffffu, v.c0, d); r.c1 = __shfl_down_sync(0xffffffffu, v.c1, d); return r;
}
__device__ __forceinline__ gle shfl_xor_e(gle v, int d) {
    gle r; r.c0 = __shfl_xor_sync(0xffffffffu, v.c0, d); r.c1 = __shfl_xor_sync(0xffffffffu, v.c1, d); return r;
}
#endif
