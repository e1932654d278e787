// Quantised inference and lookup-witness generation on the device (SURVEY.md 8f.3).
// Reference (all host code there): Dense::op (zkml/src/layers/dense.rs), Requant::op + gen_lookup_witness
// (layers/requant.rs:208-330), Activation (Relu) gen_lookup_witness (layers/activation.rs:238-323), Maxpool2D::op +
// compute_polys (layers/pooling.rs:210-271,667-771), table multiplicities (lookup/context.rs:675-737 -- HashMap counts there).
//
// Tensors are Base MLEs holding canonical field elements of SIGNED integers (v < 0  <->  p - |v|), i.e. exactly what the
// reference's Tensor<Element> -> to_field conversion produces, so a trace tensor IS a witness column and nothing is copied.
// Every node is ONE streaming kernel that writes the node's output tensor, its lookup columns, and adds its lookups to the
// per-proof multiplicity histograms (u32 atomics in HBM/L2; the tables have 2^8 .. 2^17 entries); dp_wit_finish turns the
// histograms into the multiplicity polynomials.  Per proof only the model input crosses PCIe.
// Values outside a table (a broken model/trace) raise an error flag that dp_wit_finish reports -- the reference panics there.
#include "common.cuh"

static constexpr long long WQMIN = -127, WQMAX = 127;     // quantization/mod.rs:28-29
static constexpr u32 W_BIT_LEN = 8;
__device__ __forceinline__ long long f2i(u64 f) { return f > (GL_P >> 1) ? -(long long)(GL_P - f) : (long long)f; }
__device__ __forceinline__ u64 i2f(long long v) { return v < 0 ? GL_P - (u64)(-v) : (u64)v; }

struct dp_wit {
    u32 n_tables = 0;
    u32 kind[8] = {0}, size[8] = {0};      // TableType: 0 relu, 2 range, 3 clamping(size)
    u32 *counts = nullptr;                 // all tables' histograms back to back, then the error word
    u64 off[9] = {0};
    u32 *err_pinned = nullptr;
};
static u32 wit_vars(u32 kind, u32 size) { return kind == 3 ? size : W_BIT_LEN; }   // multiplicity_poly_vars (lookup/context.rs:482-493)

// ---- Dense::op: out[r] = bias[r] + sum_c w[r][c] x[c]  (signed 64-bit integers; one warp per row) ----
__global__ void k_wit_dense(const u64 *__restrict__ w, const u64 *__restrict__ bias, const u64 *__restrict__ x, u32 nrows, u32 ncols, u64 *__restrict__ out) {
    const u32 row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (row >= nrows) return;
    const u64 *wr = w + (u64)row * ncols;
    long long acc = 0;
    for (u32 c = 2 * lane; c < ncols; c += 64) {
        ulonglong2 a = ld_b2(wr + c), b = ld_b2(x + c);
        acc += f2i(a.x) * f2i(b.x) + f2i(a.y) * f2i(b.y);
    }
    for (int d = 16; d > 0; d >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, d);
    if (lane == 0) out[row] = i2f(acc + f2i(bias[row]));
}
__global__ void k_wit_dense_small(const u64 *__restrict__ w, const u64 *__restrict__ bias, const u64 *__restrict__ x, u32 nrows, u32 ncols, u64 *__restrict__ out) {
    const u32 row = blockIdx.x * blockDim.x + threadIdx.x;      // ncols < 2: scalar rows
    if (row >= nrows) return;
    long long acc = f2i(bias[row]);
    for (u32 c = 0; c < ncols; c++) acc += f2i(w[(u64)row * ncols + c]) * f2i(x[c]);
    out[row] = i2f(acc);
}

// ---- MatMul::op (layers/matrix_mul.rs:230-311): out[r][c] = bias[c] + sum_k left[r][k] * right(k, c); right stored [K][C], or [C][K] with TransposeB ----
// one thread per output element; the K-loop reads the left row (broadcast within the threads of a row) and a right column / row
__global__ void k_wit_matmul(const u64 *__restrict__ left, const u64 *__restrict__ right, const u64 *__restrict__ bias, u32 R, u32 K, u32 C, int transposed, u64 *__restrict__ out) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (u64)R * C) return;
    const u32 r = (u32)(i / C), c = (u32)(i % C);
    long long acc = bias ? f2i(bias[c]) : 0;
    const u64 *lr = left + (u64)r * K;
    if (transposed) { const u64 *rr = right + (u64)c * K; for (u32 k = 0; k < K; k++) acc += f2i(lr[k]) * f2i(rr[k]); }
    else for (u32 k = 0; k < K; k++) acc += f2i(lr[k]) * f2i(right[(u64)k * C + c]);
    out[i] = i2f(acc);
}

// ---- Requant: tmp = v * m + 2^(shift-1); cin = tmp >> shift; cout = clamp(cin); chunks = bytes of (tmp & (2^shift - 1)) ----
struct RqCols { u64 *cin, *cout, *chunk[8]; u32 n_chunks; };
__global__ void k_wit_requant(const u64 *__restrict__ x, u64 n, u32 shift, long long fpm, long long lim, RqCols c, u32 *clamp_counts, u32 clamp_size, u32 *range_counts, u32 *err) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long v = f2i(x[i]);
    if (v > lim || v < -lim) atomicOr(err, 1u);              // "Could not apply requantisation, tensor element had absolute value too large"
    const long long tmp = v * fpm + (1LL << (shift - 1)), cl = tmp >> shift;
    const long long co = cl < WQMIN ? WQMIN : (cl > WQMAX ? WQMAX : cl);
    const u64 sh = (u64)tmp & ((1ULL << shift) - 1);
    c.cin[i] = i2f(cl); c.cout[i] = i2f(co);
    const long long idx = cl + (1LL << (clamp_size - 1));
    if (idx < 0 || idx >= (1LL << clamp_size)) atomicOr(err, 2u); else atomicAdd(clamp_counts + idx, 1u);
    for (u32 j = 0; j < c.n_chunks; j++) { const u32 b = (u32)(sh >> (j * W_BIT_LEN)) & 255u; c.chunk[j][i] = b; atomicAdd(range_counts + b, 1u); }
}
// ---- Relu: out = max(v, 0); table rows are v = QMIN-1 .. QMAX ----
__global__ void k_wit_relu(const u64 *__restrict__ x, u64 n, u64 *__restrict__ out, u32 *relu_counts, u32 *err) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long v = f2i(x[i]);
    out[i] = v < 0 ? 0ULL : (u64)v;
    const long long idx = v - (WQMIN - 1);
    if (idx < 0 || idx > WQMAX - (WQMIN - 1)) atomicOr(err, 4u); else atomicAdd(relu_counts + idx, 1u);
}
// ---- Maxpool2D (kernel = stride = 2) on [C][H][W]: out = max of the 2x2 window; columns out - in(2r+dr, 2c+dc), (dr,dc) = (0,0),(1,0),(0,1),(1,1) ----
struct PoolCols { u64 *out, *diff[4]; };
__global__ void k_wit_pool(const u64 *__restrict__ x, u32 C, u32 H, u32 W, PoolCols p, u32 *range_counts, u32 *err) {
    const u64 oi = (u64)blockIdx.x * blockDim.x + threadIdx.x, n = (u64)C * (H / 2) * (W / 2);
    if (oi >= n) return;
    const u32 cc = (u32)(oi % (W / 2)), r = (u32)((oi / (W / 2)) % (H / 2)), c = (u32)(oi / ((u64)(W / 2) * (H / 2)));
    long long v[4]; const u32 DR[4] = {0, 1, 0, 1}, DC[4] = {0, 0, 1, 1};
    long long mx = 0;
    for (int k = 0; k < 4; k++) { v[k] = f2i(x[((u64)c * H + 2 * r + DR[k]) * W + 2 * cc + DC[k]]); mx = k == 0 ? v[0] : (v[k] > mx ? v[k] : mx); }
    p.out[oi] = i2f(mx);
    for (int k = 0; k < 4; k++) {
        const long long d = mx - v[k];
        p.diff[k][oi] = (u64)d;
        if (d > 255) atomicOr(err, 8u); else atomicAdd(range_counts + d, 1u);
    }
}
// ---- multiplicity polynomials: every table row is distinct in these tables (table_count == 1), so m[i] = count[i] ----
struct MultOut { u64 *m[8]; u64 off[9]; u32 n; };
__global__ void k_wit_mult(const u32 *__restrict__ counts, MultOut o) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= o.off[o.n]) return;
    u32 t = 0; while (i >= o.off[t + 1]) t++;
    o.m[t][i - o.off[t]] = (u64)counts[i];
}

static int wit_new_base(u64 len, dp_mle **out) {
    dp_mle *m = new dp_mle(); m->len = len; m->is_ext = false; m->owned = true;
    if (int e = dp_dev_alloc(&m->data, m->bytes())) { delete m; return e; }
    *out = m; return DP_OK;
}
// n fresh columns of `len`, or none: on a failed allocation the ones already made are freed
static int wit_new_cols(u64 len, u32 n, dp_mle **cols) {
    for (u32 k = 0; k < n; k++) {
        if (int e = wit_new_base(len, &cols[k])) {
            for (u32 q = 0; q < k; q++) { dp_mle_free(cols[q]); cols[q] = nullptr; }
            return e;
        }
    }
    return DP_OK;
}

extern "C" {

int dp_wit_begin(uint32_t n_tables, const uint32_t *kinds, const uint32_t *sizes, dp_wit **out) {
    DP_REQUIRE_CTX();
    DP_CHECK(out && kinds && sizes && n_tables >= 1 && n_tables <= 8, DP_ERR_INVALID, "dp_wit_begin: 1..8 tables");
    for (u32 t = 0; t < n_tables; t++)
        DP_CHECK(kinds[t] == 0 || kinds[t] == 2 || (kinds[t] == 3 && sizes[t] >= 1 && sizes[t] <= 24), DP_ERR_INVALID, "dp_wit_begin: unknown table type");
    dp_wit *w = new dp_wit(); w->n_tables = n_tables;
    for (u32 t = 0; t < n_tables; t++) {
        w->kind[t] = kinds[t]; w->size[t] = sizes[t]; w->off[t + 1] = w->off[t] + (1ULL << wit_vars(kinds[t], sizes[t]));
    }
    int e;
    if ((e = dp_dev_alloc((void **)&w->counts, sizeof(u32) * (w->off[n_tables] + 4)))) { delete w; return e; }
    if ((e = dp_pinned_alloc((void **)&w->err_pinned, 64))) { dp_dev_free(w->counts); delete w; return e; }
    DP_CUDA(cudaMemsetAsync(w->counts, 0, sizeof(u32) * (w->off[n_tables] + 4), dp_ctx().stream));
    *out = w;
    return DP_OK;
}

int dp_wit_dense(const dp_mle *weights, const dp_mle *bias, const dp_mle *x, uint32_t nrows, uint32_t ncols, dp_mle **out) {
    DP_REQUIRE_CTX();
    DP_CHECK(weights && bias && x && out, DP_ERR_INVALID, "dp_wit_dense: null argument");
    DP_CHECK(!weights->is_ext && !bias->is_ext && !x->is_ext, DP_ERR_INVALID, "dp_wit_dense: tensors are Base");
    DP_CHECK(weights->len == (u64)nrows * ncols && bias->len == nrows && x->len == ncols, DP_ERR_INVALID, "dp_wit_dense: shape mismatch");
    dp_mle *o; if (int e = wit_new_base(nrows, &o)) return e;
    DpProfScope prof("k_wit_dense", weights->bytes() + x->bytes() + 16ull * nrows);
    if (ncols >= 2) k_wit_dense<<<(nrows * 32 + 255) / 256, 256, 0, dp_ctx().stream>>>((const u64 *)weights->data, (const u64 *)bias->data, (const u64 *)x->data, nrows, ncols, (u64 *)o->data);
    else k_wit_dense_small<<<(nrows + 255) / 256, 256, 0, dp_ctx().stream>>>((const u64 *)weights->data, (const u64 *)bias->data, (const u64 *)x->data, nrows, ncols, (u64 *)o->data);
    DP_LAUNCHED(); DP_CUDA(cudaGetLastError());
    *out = o;
    return DP_OK;
}

int dp_wit_matmul(const dp_mle *left, const dp_mle *right, const dp_mle *bias, uint32_t R, uint32_t K, uint32_t C, int transposed, dp_mle **out) {
    DP_REQUIRE_CTX();
    DP_CHECK(left && right && out, DP_ERR_INVALID, "dp_wit_matmul: null argument");
    DP_CHECK(!left->is_ext && !right->is_ext && (!bias || !bias->is_ext), DP_ERR_INVALID, "dp_wit_matmul: tensors are Base");
    DP_CHECK(left->len == (u64)R * K && right->len == (u64)K * C && (!bias || bias->len == C), DP_ERR_INVALID, "Incompatible shape found for input matrix");   // matrix_mul.rs:277-283
    dp_mle *o; if (int e = wit_new_base((u64)R * C, &o)) return e;
    DpProfScope prof("k_wit_matmul", left->bytes() + right->bytes() + 8ull * R * C);
    k_wit_matmul<<<(unsigned)(((u64)R * C + 255) / 256), 256, 0, dp_ctx().stream>>>((const u64 *)left->data, (const u64 *)right->data, bias ? (const u64 *)bias->data : nullptr, R, K, C, transposed, (u64 *)o->data);
    DP_LAUNCHED(); DP_CUDA(cudaGetLastError());
    *out = o;
    return DP_OK;
}

static int wit_table(const dp_wit *w, uint32_t t, u32 kind, const char *what) {
    if (!(w && t < w->n_tables && w->kind[t] == kind)) return dp_fail(DP_ERR_INVALID, std::string(what) + ": wrong table index/type");
    return DP_OK;
}

// cols[0] = clamping input, cols[1] = clamping output (= the node's output tensor), cols[2..] = the shift/8 byte chunks
int dp_wit_requant(dp_wit *w, const dp_mle *x, uint32_t shift, int64_t fixed_point_multiplier, uint32_t intermediate_bit_size,
                   uint32_t clamp_table, uint32_t range_table, dp_mle **cols, uint32_t n_cols) {
    DP_REQUIRE_CTX();
    DP_CHECK(w && x && cols && !x->is_ext, DP_ERR_INVALID, "dp_wit_requant: bad argument");
    DP_CHECK(shift >= 1 && shift <= 62 && shift % W_BIT_LEN == 0 && shift / W_BIT_LEN <= 8 && n_cols == 2 + shift / W_BIT_LEN, DP_ERR_INVALID, "dp_wit_requant: shift must be a multiple of BIT_LEN (<= 64 bits) and n_cols = 2 + shift / BIT_LEN");
    if (int e = wit_table(w, clamp_table, 3, "dp_wit_requant")) return e;
    // 1 << intermediate_bit_size bounds |x|; the reference asserts intermediate_bit_size + fp_scale <= 63 (requant.rs:423-427)
    DP_CHECK(intermediate_bit_size <= 62, DP_ERR_INVALID, "dp_wit_requant: intermediate_bit_size must be at most 62");
    if (int e = wit_table(w, range_table, 2, "dp_wit_requant")) return e;
    RqCols c; c.n_chunks = shift / W_BIT_LEN;
    if (int e = wit_new_cols(x->len, n_cols, cols)) return e;
    c.cin = (u64 *)cols[0]->data; c.cout = (u64 *)cols[1]->data;
    for (u32 j = 0; j < c.n_chunks; j++) c.chunk[j] = (u64 *)cols[2 + j]->data;
    DpProfScope prof("k_wit_requant", x->bytes() * (1 + n_cols));
    k_wit_requant<<<(unsigned)((x->len + 255) / 256), 256, 0, dp_ctx().stream>>>((const u64 *)x->data, x->len, shift, (long long)fixed_point_multiplier, 1LL << intermediate_bit_size, c,
                                                                               w->counts + w->off[clamp_table], w->size[clamp_table], w->counts + w->off[range_table], w->counts + w->off[w->n_tables]);
    DP_LAUNCHED(); DP_CUDA(cudaGetLastError());
    return DP_OK;
}

int dp_wit_relu(dp_wit *w, const dp_mle *x, uint32_t relu_table, dp_mle **out) {
    DP_REQUIRE_CTX();
    DP_CHECK(w && x && out && !x->is_ext, DP_ERR_INVALID, "dp_wit_relu: bad argument");
    if (int e = wit_table(w, relu_table, 0, "dp_wit_relu")) return e;
    dp_mle *o; if (int e = wit_new_base(x->len, &o)) return e;
    DpProfScope prof("k_wit_relu", x->bytes() * 2);
    k_wit_relu<<<(unsigned)((x->len + 255) / 256), 256, 0, dp_ctx().stream>>>((const u64 *)x->data, x->len, (u64 *)o->data, w->counts + w->off[relu_table], w->counts + w->off[w->n_tables]);
    DP_LAUNCHED(); DP_CUDA(cudaGetLastError());
    *out = o;
    return DP_OK;
}

// cols[0..3] = out - in(2r+dr, 2c+dc); cols[4] = the output tensor
int dp_wit_pool(dp_wit *w, const dp_mle *x, uint32_t C, uint32_t H, uint32_t Wd, uint32_t range_table, dp_mle **cols) {
    DP_REQUIRE_CTX();
    DP_CHECK(w && x && cols && !x->is_ext && x->len == (u64)C * H * Wd && H % 2 == 0 && Wd % 2 == 0, DP_ERR_INVALID, "dp_wit_pool: bad argument");
    if (int e = wit_table(w, range_table, 2, "dp_wit_pool")) return e;
    const u64 n = (u64)C * (H / 2) * (Wd / 2);
    DP_CHECK((n & (n - 1)) == 0, DP_ERR_INVALID, "dp_wit_pool: output length must be a power of two");
    PoolCols p;
    if (int e = wit_new_cols(n, 5, cols)) return e;
    for (u32 k = 0; k < 4; k++) p.diff[k] = (u64 *)cols[k]->data;
    p.out = (u64 *)cols[4]->data;
    DpProfScope prof("k_wit_pool", x->bytes() + 5 * n * 8);
    k_wit_pool<<<(unsigned)((n + 255) / 256), 256, 0, dp_ctx().stream>>>((const u64 *)x->data, C, H, Wd, p, w->counts + w->off[range_table], w->counts + w->off[w->n_tables]);
    DP_LAUNCHED(); DP_CUDA(cudaGetLastError());
    return DP_OK;
}

// multiplicity polynomials of every table (in dp_wit_begin order) + the error word of all node kernels so far
int dp_wit_finish(dp_wit *w, dp_mle **mults, uint32_t *error_bits) {
    DP_REQUIRE_CTX();
    DP_CHECK(w && mults && error_bits, DP_ERR_INVALID, "dp_wit_finish: null argument");
    MultOut o; o.n = w->n_tables;
    for (u32 t = 0; t < w->n_tables; t++) { if (int e = wit_new_base(w->off[t + 1] - w->off[t], &mults[t])) return e; o.m[t] = (u64 *)mults[t]->data; }
    for (u32 t = 0; t <= w->n_tables; t++) o.off[t] = w->off[t];
    cudaStream_t st = dp_ctx().stream;
    k_wit_mult<<<(unsigned)((w->off[w->n_tables] + 255) / 256), 256, 0, st>>>(w->counts, o); DP_LAUNCHED();
    DP_CUDA(cudaMemcpyAsync(w->err_pinned, w->counts + w->off[w->n_tables], 4, cudaMemcpyDeviceToHost, st));
    DP_CUDA(dp_stream_sync(st));
    *error_bits = *w->err_pinned;
    return DP_OK;
}

int dp_wit_free(dp_wit *w) {
    if (!w) return DP_OK;
    std::lock_guard<std::recursive_mutex> lk(dp_ctx().mu);
    if (dp_ctx().ready) { dp_dev_free(w->counts); dp_pinned_free(w->err_pinned); }
    delete w;
    return DP_OK;
}

}  // extern "C"
