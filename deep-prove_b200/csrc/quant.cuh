// The scalar rules of the quantised layers, shared by the witness kernels (witness.cu) and the batch-inference epilogues
// (infer.cu), so that both compute the same values and raise the same error bits:
//   1 a requant input with |v| > 2^intermediate_bit_size, 2 a clamping-table miss, 4 a relu-table miss, 8 a pooling difference
//   outside the range table (dp_wit_finish, dp_infer_run).
#pragma once
#include "common.cuh"

static constexpr long long WQMIN = -127, WQMAX = 127;     // quantization/mod.rs:28-29

struct RqRule {
    u32 shift, clamp_size;     // fp_scale + right_shift; the clamping table's bits
    long long fpm, lim;        // fixed_point_multiplier; 2^intermediate_bit_size
};
struct RqVal { long long tmp, cl, out; };
// Requant (layers/requant.rs:208-330): tmp = v * m + 2^(shift-1); cl = tmp >> shift is the clamping table's input, which must lie in
// [-2^(size-1), 2^(size-1)); the output is cl clamped to [-127, 127]
__device__ __forceinline__ RqVal rq_rule(long long v, const RqRule &r, u32 &err) {
    RqVal q;
    if (v > r.lim || v < -r.lim) err |= 1u;                  // "Could not apply requantisation, tensor element had absolute value too large"
    q.tmp = v * r.fpm + (1LL << (r.shift - 1));
    q.cl = q.tmp >> r.shift;
    q.out = q.cl < WQMIN ? WQMIN : (q.cl > WQMAX ? WQMAX : q.cl);
    const long long idx = q.cl + (1LL << (r.clamp_size - 1));
    if (idx < 0 || idx >= (1LL << r.clamp_size)) err |= 2u;
    return q;
}
// Relu (layers/activation.rs:238-323): the table's rows are v = QMIN-1 .. QMAX
__device__ __forceinline__ long long relu_rule(long long v, u32 &err) {
    if (v < WQMIN - 1 || v > WQMAX) err |= 4u;
    return v < 0 ? 0 : v;
}
// Maxpool2D (layers/pooling.rs:686-771): each (output - input) difference is looked up in the 8-bit range table
__device__ __forceinline__ void pool_rule(long long d, u32 &err) {
    if (d > 255) err |= 8u;
}
