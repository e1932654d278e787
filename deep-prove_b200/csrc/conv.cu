// FFT-convolution layer: witness tensors and the helper tables of its proof, on the device.
// Reference: zkml/src/tensor.rs:220-323 (get_root_of_unity, index_w, index_u, fft), :458-523 (fft_conv);
// zkml/src/layers/convolution.rs:152-162 (add_bias), :870 (beta_acc), :1535-1550 (index_wf);
// zkml/src/iop/prover.rs:164-289 (delegate_matrix_evaluation's phi vectors, phi_pow_init, phi_g_init).
// Rows of 2*n_x^2 <= 2^13 Ext values (n_x <= 64) are transformed one block per row in shared memory; longer rows, up to
// 2^21 (n_x <= 1024, e.g. a 224x224 image padded to 256), by a two-pass four-step FFT.  The kernels exist so that the
// tensors a conv proof needs (input_fft, prod, the FFT-matrix tables, the layer output) are produced where the sumchecks
// consume them -- no host round trips.
#include "common.cuh"
#include "powtab.cuh"
#include "../../include/deepprove_b200.h"
#include <algorithm>

// ---- fft(v, flag) on rows (tensor.rs:261-323): natural order in/out, w = get_root_of_unity(log n) (inverse when flag) ----
constexpr u32 FFT_ROWS_MAX_LOG = 13;
__global__ void __launch_bounds__(256) k_fft_rows(gle *data, u32 lg, int inverse, PowTab tab) {
    extern __shared__ unsigned char smem_raw[];
    gle *sm = reinterpret_cast<gle *>(smem_raw);
    const u32 n = 1u << lg;
    gle *row = data + (u64)blockIdx.x * n;
    for (u32 i = threadIdx.x; i < n; i += blockDim.x) sm[lg ? (__brev(i) >> (32 - lg)) : 0] = row[i];
    __syncthreads();
    for (u32 s = 1; s <= lg; s++) {
        const u32 half = 1u << (s - 1);
        for (u32 q = threadIdx.x; q < (n >> 1); q += blockDim.x) {
            u32 k = q & (half - 1), c = (q >> (s - 1)) << s;
            u32 e = (n >> s) * k;                                       // w[n / i * k], i = 2^s
            if (inverse && e) e = n - e;
            u64 w = tab_pow(tab, (u64)e << (32 - lg));
            gle u = sm[c + k], l = e_mul_base(sm[c + k + half], w);
            sm[c + k] = e_add(u, l); sm[c + k + half] = e_sub(u, l);
        }
        __syncthreads();
    }
    u64 ilen = inverse ? gl_inv((u64)n) : 1ULL;
    for (u32 i = threadIdx.x; i < n; i += blockDim.x) row[i] = inverse ? e_mul_base(sm[i], ilen) : sm[i];
}
extern "C" int dp_fft_rows(dp_mle *m, uint32_t log_n, int inverse) {
    DP_REQUIRE_CTX();
    DP_CHECK(m && m->is_ext, DP_ERR_INVALID, "dp_fft_rows: need an Ext MLE");
    DP_CHECK(log_n >= 1 && log_n <= FFT_ROWS_MAX_LOG && (m->len >> log_n) >= 1 && (m->len & ((1ULL << log_n) - 1)) == 0, DP_ERR_INVALID,
             "dp_fft_rows: row length must be 2^1..2^13 and divide the MLE length");
    PowTab tab; if (int e = dp_root_powtab(&tab)) return e;
    size_t smem = sizeof(gle) << log_n;
    // the largest request of any row length (2^13 values, 128 KB), never the call's own: proving threads transform rows of 2^12 and
    // 2^13 concurrently, and lowering the function's limit under another thread's launch would refuse that launch
    const int smem_max = (int)(sizeof(gle) << FFT_ROWS_MAX_LOG);
    if (smem > 48 * 1024) DP_CUDA(cudaFuncSetAttribute(k_fft_rows, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max));
    DpProfScope prof("k_fft_rows", m->bytes() * 2);
    DP_CUDA(dp_launch(k_fft_rows, (unsigned)(m->len >> log_n), 256, smem, dp_ctx().stream, (gle *)m->data, log_n, inverse, tab));
    return DP_OK;
}

// ---- the same transform on rows of 2^14..2^21: four-step FFT, N = N1 N2, n = N2 n1 + n2, k = k1 + N1 k2 ----
//   X[k1 + N1 k2] = sum_n2 W_N2^(n2 k2) W_N^(n2 k1) sum_n1 x[N2 n1 + n2] W_N1^(n1 k1),  W_M = get_root_of_unity(log M)
// pass 1 (k_fft_long_cols): the N1-point transforms down the columns n2, times W_N^(n2 k1), into tmp[N2 k1 + n2];
// pass 2 (k_fft_long_rows): the N2-point transforms along tmp's rows, written transposed to X[k1 + N1 k2].
// Two reads and two writes of the tensor in all.  Every root is a power of the same 2^32-th root, so W_N^N2 == W_N1 and the
// result is the reference's fft exactly (field arithmetic has no rounding).  A block transforms FFT_G adjacent columns
// (rows) at once, so every global access moves FFT_G * 16 = 64 contiguous bytes.
constexpr u32 FFT_G = 4, FFT_LONG_MIN = 14, FFT_LONG_MAX = 21;
// FFT_G interleaved 2^lg-point transforms in shared memory, sm[j * FFT_G + g], entered in bit-reversed order
__device__ __forceinline__ void smem_fft_g(gle *sm, u32 lg, int inverse, const PowTab &tab) {
    const u32 n = 1u << lg;
    for (u32 s = 1; s <= lg; s++) {
        const u32 half = 1u << (s - 1);
        for (u32 q = threadIdx.x; q < (n >> 1) * FFT_G; q += blockDim.x) {
            u32 g = q % FFT_G, p = q / FFT_G, k = p & (half - 1), c = (p >> (s - 1)) << s;
            u32 e = (n >> s) * k;
            if (inverse && e) e = n - e;
            u64 w = tab_pow(tab, (u64)e << (32 - lg));
            gle *a = sm + (c + k) * FFT_G + g, *b = a + half * FFT_G;
            gle u = *a, l = e_mul_base(*b, w);
            *a = e_add(u, l); *b = e_sub(u, l);
        }
        __syncthreads();
    }
}
__global__ void __launch_bounds__(512) k_fft_long_cols(const gle *__restrict__ data, gle *__restrict__ tmp, u32 lg1, u32 lg2, int inverse, PowTab tab) {
    extern __shared__ unsigned char smem_raw[];
    gle *sm = reinterpret_cast<gle *>(smem_raw);
    const u32 n1 = 1u << lg1, n2 = 1u << lg2, lg = lg1 + lg2, groups = n2 / FFT_G;
    const u64 row = (u64)(blockIdx.x / groups) << lg;
    const u32 col0 = (blockIdx.x % groups) * FFT_G;
    for (u32 i = threadIdx.x; i < n1 * FFT_G; i += blockDim.x) {
        u32 j = i / FFT_G, g = i % FFT_G;
        sm[(__brev(j) >> (32 - lg1)) * FFT_G + g] = data[row + (u64)j * n2 + col0 + g];
    }
    __syncthreads();
    smem_fft_g(sm, lg1, inverse, tab);
    for (u32 i = threadIdx.x; i < n1 * FFT_G; i += blockDim.x) {
        u32 k1 = i / FFT_G, g = i % FFT_G, e = k1 * (col0 + g);                // < N: no reduction needed
        if (inverse && e) e = (1u << lg) - e;
        tmp[row + (u64)k1 * n2 + col0 + g] = e_mul_base(sm[i], tab_pow(tab, (u64)e << (32 - lg)));
    }
}
__global__ void __launch_bounds__(512) k_fft_long_rows(const gle *__restrict__ tmp, gle *__restrict__ data, u32 lg1, u32 lg2, int inverse, u64 ilen, PowTab tab) {
    extern __shared__ unsigned char smem_raw[];
    gle *sm = reinterpret_cast<gle *>(smem_raw);
    const u32 n1 = 1u << lg1, n2 = 1u << lg2, lg = lg1 + lg2, groups = n1 / FFT_G;
    const u64 row = (u64)(blockIdx.x / groups) << lg;
    const u32 k10 = (blockIdx.x % groups) * FFT_G;
    for (u32 i = threadIdx.x; i < n2 * FFT_G; i += blockDim.x) {
        u32 g = i >> lg2, j = i & (n2 - 1);
        sm[(__brev(j) >> (32 - lg2)) * FFT_G + g] = tmp[row + (u64)(k10 + g) * n2 + j];
    }
    __syncthreads();
    smem_fft_g(sm, lg2, inverse, tab);
    for (u32 i = threadIdx.x; i < n2 * FFT_G; i += blockDim.x) {
        u32 k2 = i / FFT_G, g = i % FFT_G;
        data[row + k10 + g + (u64)k2 * n1] = inverse ? e_mul_base(sm[i], ilen) : sm[i];
    }
}
extern "C" int dp_fft_rows_long(dp_mle *m, uint32_t log_n, int inverse) {
    DP_REQUIRE_CTX();
    DP_CHECK(m && m->is_ext, DP_ERR_INVALID, "dp_fft_rows_long: need an Ext MLE");
    DP_CHECK(log_n >= FFT_LONG_MIN && log_n <= FFT_LONG_MAX && (m->len >> log_n) >= 1 && (m->len & ((1ULL << log_n) - 1)) == 0, DP_ERR_INVALID,
             "dp_fft_rows_long: row length must be 2^14..2^21 and divide the MLE length");
    PowTab tab; if (int e = dp_root_powtab(&tab)) return e;
    const u32 lg1 = log_n / 2, lg2 = log_n - lg1;
    const u64 rows = m->len >> log_n;
    DP_CHECK(rows * ((1ULL << lg2) / FFT_G) < (1ULL << 31), DP_ERR_INVALID, "dp_fft_rows_long: too many rows");
    void *tmp = nullptr;
    if (int e = dp_dev_alloc(&tmp, m->bytes())) return e;
    DevPtr tmp_owner(tmp);
    const size_t smem1 = (sizeof(gle) * FFT_G) << lg1, smem2 = (sizeof(gle) * FFT_G) << lg2;
    // the largest request of any row length (128 KB), never the call's own: proving threads launch other row lengths concurrently,
    // and lowering the function's limit under another thread's launch would refuse that launch
    const int smem_max = (int)((sizeof(gle) * FFT_G) << (FFT_LONG_MAX - FFT_LONG_MAX / 2));
    DP_CUDA(cudaFuncSetAttribute(k_fft_long_cols, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max));
    DP_CUDA(cudaFuncSetAttribute(k_fft_long_rows, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max));
    cudaStream_t st = dp_ctx().stream;
    DpProfScope prof("k_fft_long", m->bytes() * 4);
    DP_CUDA(dp_launch(k_fft_long_cols, (unsigned)((rows << lg2) / FFT_G), 512, smem1, st, (const gle *)m->data, (gle *)tmp, lg1, lg2, inverse, tab));
    DP_CUDA(dp_launch(k_fft_long_rows, (unsigned)((rows << lg1) / FFT_G), 512, smem2, st, (const gle *)tmp, (gle *)m->data, lg1, lg2, inverse,
                      inverse ? gl_inv(1ULL << log_n) : 1ULL, tab));
    return DP_OK;
}

// ---- index_w / index_wf: an n_real x n_real block placed top-left in an n x n grid, row padded with zeros to out_len ----
template <bool EXT>
__global__ void k_pad_rows(const void *src, u64 rows, u32 n_real, u32 n, u64 out_len, gle *out) {
    u64 total = rows * out_len, t = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    for (; t < total; t += stride) {
        u64 r = t / out_len, idx = t % out_len, i = idx / n, j = idx % n;
        gle v = e_zero();
        if (i < n_real && j < n_real) { u64 s = r * n_real * n_real + i * n_real + j; v = EXT ? ((const gle *)src)[s] : e_from_base(((const u64 *)src)[s]); }
        out[t] = v;
    }
}
extern "C" int dp_pad_rows(const dp_mle *src, uint64_t rows, uint32_t n_real, uint32_t n, uint64_t out_len, dp_mle **out) {
    DP_REQUIRE_CTX();
    DP_CHECK(src && out && rows && n_real && n_real <= n, DP_ERR_INVALID, "dp_pad_rows: bad arguments");
    DP_CHECK(src->len == rows * n_real * n_real, DP_ERR_INVALID, "dp_pad_rows: source length != rows * n_real^2");
    u64 total = rows * out_len;
    DP_CHECK(total && (total & (total - 1)) == 0, DP_ERR_INVALID, "dp_pad_rows: rows * out_len must be a power of two");
    MlePtr m; if (int e = dp_mle_alloc(total, true, m)) return e;
    DP_CUDA(dp_launch(src->is_ext ? k_pad_rows<true> : k_pad_rows<false>, dp_grid_for(total, 256, 8), 256, 0, dp_ctx().stream, src->data, rows, n_real, n,
                      out_len, (gle *)m->data));
    *out = m.release(); return DP_OK;
}

// ---- fft_conv accumulation (tensor.rs:489-509): out[i][k] = sum_j x_fft[j][k] * w_fft[i][j][k] ----
__global__ void k_conv_prod(const gle *__restrict__ x, const gle *__restrict__ w, u32 kw, u32 kx, u64 n, gle *__restrict__ out) {
    u64 total = (u64)kw * n, t = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    for (; t < total; t += stride) {
        u64 i = t / n, k = t % n;
        gle acc = e_zero();
        for (u32 j = 0; j < kx; j++) acc = e_add(acc, e_mul(x[(u64)j * n + k], w[(i * kx + j) * n + k]));
        out[t] = acc;
    }
}
extern "C" int dp_conv_prod(const dp_mle *x_fft, const dp_mle *w_fft, uint32_t kw, uint32_t kx, uint64_t row_len, dp_mle **out) {
    DP_REQUIRE_CTX();
    DP_CHECK(x_fft && w_fft && out && x_fft->is_ext && w_fft->is_ext, DP_ERR_INVALID, "dp_conv_prod: need Ext operands");
    DP_CHECK(x_fft->len == (u64)kx * row_len && w_fft->len == (u64)kw * kx * row_len, DP_ERR_INVALID, "dp_conv_prod: operand shapes do not match [kx, n] / [kw, kx, n]");
    MlePtr m; if (int e = dp_mle_alloc((u64)kw * row_len, true, m)) return e;
    DpProfScope prof("k_conv_prod", (w_fft->bytes() + x_fft->bytes() + m->bytes()));
    DP_CUDA(dp_launch(k_conv_prod, dp_grid_for((u64)kw * row_len, 128, 8), 128, 0, dp_ctx().stream, (const gle *)x_fft->data, (const gle *)w_fft->data, kw, kx,
                      row_len, (gle *)m->data));
    *out = m.release(); return DP_OK;
}

// ---- index_u + to_element + add_bias: out[i][t] = to_element(rows[i][n_x^2 - 1 - t]) + bias[i] ----
__global__ void k_conv_out_elems(const gle *rows, u32 kw, u32 nx2, const long long *bias, long long *out) {
    u64 total = (u64)kw * nx2, t = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    for (; t < total; t += stride) {
        u64 i = t / nx2, k = t % nx2;
        u64 c = rows[i * 2 * nx2 + (nx2 - 1 - k)].c0;
        long long v = c <= (GL_P >> 1) ? (long long)c : -(long long)(GL_P - c);     // quantization/mod.rs:225-242
        out[t] = v + bias[i];
    }
}
extern "C" int dp_conv_output_elements(const dp_mle *out_rows, uint32_t kw, uint32_t n_x, const int64_t *bias, int64_t *out_host) {
    DP_REQUIRE_CTX();
    u64 nx2 = (u64)n_x * n_x;
    DP_CHECK(out_rows && out_rows->is_ext && bias && out_host && out_rows->len == 2 * nx2 * kw, DP_ERR_INVALID, "dp_conv_output_elements: need [kw, 2 n_x^2] Ext rows");
    long long *d = nullptr, *db = nullptr;
    if (int e = dp_dev_alloc((void **)&d, 8 * nx2 * kw)) return e;
    DevPtr d_owner(d);
    if (int e = dp_dev_alloc((void **)&db, 8 * (size_t)kw)) return e;
    DevPtr db_owner(db);
    cudaStream_t st = dp_ctx().stream;
    DP_CUDA(cudaMemcpyAsync(db, bias, 8 * (size_t)kw, cudaMemcpyHostToDevice, st));
    DP_CUDA(dp_launch(k_conv_out_elems, dp_grid_for(nx2 * kw, 256, 8), 256, 0, st, (const gle *)out_rows->data, kw, (u32)nx2, db, d));
    return dp_d2h(out_host, d, 8 * nx2 * kw, st);
}
// The same tensor as a device Base MLE of canonical field elements (Tensor::to_field of the Element tensor: from_i64(to_element(c) + b)
// == c + b), plus the cleared output (the product with the layer's 0/1 clearing mask, convolution.rs:1484-1530), in one pass
__global__ void k_conv_output(const gle *rows, u32 kw, u32 nx2, const u64 *bias, const u64 *mask, u64 *after, u64 *cleared) {
    u64 total = (u64)kw * nx2, t = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    for (; t < total; t += stride) {
        u64 i = t / nx2, k = t % nx2;
        u64 v = gl_add(gl_canon(rows[i * 2 * nx2 + (nx2 - 1 - k)].c0), bias[i]);
        after[t] = v; cleared[t] = mask[t] ? v : 0;
    }
}
extern "C" int dp_conv_output(const dp_mle *out_rows, uint32_t kw, uint32_t n_x, const dp_mle *bias, const dp_mle *mask, dp_mle **after, dp_mle **cleared) {
    DP_REQUIRE_CTX();
    u64 nx2 = (u64)n_x * n_x;
    DP_CHECK(out_rows && out_rows->is_ext && out_rows->len == 2 * nx2 * kw && after && cleared, DP_ERR_INVALID, "dp_conv_output: need [kw, 2 n_x^2] Ext rows");
    DP_CHECK(bias && !bias->is_ext && bias->len == kw && mask && !mask->is_ext && mask->len == nx2 * kw, DP_ERR_INVALID, "dp_conv_output: need a Base bias [kw] and a Base mask [kw, n_x, n_x]");
    MlePtr a, c;
    if (int e = dp_mle_alloc(nx2 * kw, false, a)) return e;
    if (int e = dp_mle_alloc(nx2 * kw, false, c)) return e;
    DP_CUDA(dp_launch(k_conv_output, dp_grid_for(nx2 * kw, 256, 8), 256, 0, dp_ctx().stream, (const gle *)out_rows->data, kw, (u32)nx2, (const u64 *)bias->data,
                      (const u64 *)mask->data, (u64 *)a->data, (u64 *)c->data));
    *after = a.release(); *cleared = c.release(); return DP_OK;
}

// ---- index_x (tensor.rs:343-361, ConvData::new): every row of a Base MLE reversed, out[r][i] = src[r][row_len - 1 - i] ----
__global__ void k_reverse_rows(const u64 *src, u64 total, u64 row_len, u64 *out) {
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    for (; t < total; t += stride) { u64 i = t % row_len; out[t] = src[t - i + row_len - 1 - i]; }
}
extern "C" int dp_reverse_rows(const dp_mle *src, uint64_t row_len, dp_mle **out) {
    DP_REQUIRE_CTX();
    DP_CHECK(src && out && !src->is_ext && row_len && src->len % row_len == 0, DP_ERR_INVALID, "dp_reverse_rows: need a Base MLE of whole rows");
    MlePtr m; if (int e = dp_mle_alloc(src->len, false, m)) return e;
    DP_CUDA(dp_launch(k_reverse_rows, dp_grid_for(src->len, 256, 8), 256, 0, dp_ctx().stream, (const u64 *)src->data, src->len, row_len, (u64 *)m->data));
    *out = m.release(); return DP_OK;
}

// ---- phi_g_init (iop/prover.rs:231-289): the FFT / iFFT matrix row W(rx, .) and its per-level prefixes ----
// Level i doubles the table: 2^(i-1) butterflies, each reading phi_g[b] and writing phi_g[b] and phi_g[b + 2^(i-1)]; mid[i - 1] is
// the table's first 2^i entries after level i.  Up to 2^14 (dp_phi_g_init) every level runs in one block; above that
// (dp_phi_g_init_long) the first PHI_HEAD_LEVELS levels do, then one grid launch per level (at most 10, each latency-bound),
// then the iFFT case's closing scale.
constexpr u32 PHI_MAX_N = 21, PHI_HEAD_LEVELS = 11;
struct PhiArgs { gle rx[PHI_MAX_N]; gle scale; gle *mid[PHI_MAX_N - 1]; };
__device__ __forceinline__ void phi_butterfly(gle *phi_g, gle rxm, u32 n, u32 m, u32 b, u32 cnt, int is_fft, const PowTab &tab, gle *mid) {
    u32 e = b << m;                                                     // phi_mul[b << m]: root (inverse when is_fft) of order 2^n
    if (is_fft && e) e = (1u << n) - e;
    u64 w = tab_pow(tab, (u64)e << (32 - n));
    gle tmp1 = e_sub(e_one(), rxm), tmp2 = e_mul_base(rxm, w), pl = phi_g[b];
    gle r = e_mul(pl, e_sub(tmp1, tmp2)), l = e_mul(pl, e_add(tmp1, tmp2));
    phi_g[b ^ cnt] = r; phi_g[b] = l;
    if (mid) { mid[b ^ cnt] = r; mid[b] = l; }
}
__device__ __forceinline__ void phi_scale(gle *phi_g, gle rx0, u32 n, u32 b, const PowTab &tab) {   // the iFFT case's last factor
    u64 w = tab_pow(tab, (u64)b << (32 - n));
    phi_g[b] = e_mul(phi_g[b], e_add(e_sub(e_one(), rx0), e_mul_base(rx0, w)));
}
// levels 1..upto in one block; the closing scale too when upto is the last level
__global__ void __launch_bounds__(1024) k_phi_g_init(gle *phi_g, PhiArgs a, u32 n, u32 upto, int is_fft, PowTab tab) {
    const u32 tid = threadIdx.x;
    if (tid == 0) { phi_g[0] = a.scale; if (is_fft) phi_g[1] = a.scale; }
    __syncthreads();
    for (u32 i = 1; i <= upto; i++) {
        const u32 cnt = 1u << (i - 1);
        for (u32 b = tid; b < cnt; b += blockDim.x) phi_butterfly(phi_g, a.rx[n - i], n, n - i, b, cnt, is_fft, tab, i < n ? a.mid[i - 1] : nullptr);
        __syncthreads();
    }
    if (!is_fft && upto == n - 1) for (u32 b = tid; b < (1u << (n - 1)); b += blockDim.x) phi_scale(phi_g, a.rx[0], n, b, tab);
}
__global__ void k_phi_g_level(gle *phi_g, gle rxm, u32 n, u32 i, int is_fft, gle *mid, PowTab tab) {
    const u32 cnt = 1u << (i - 1), b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < cnt) phi_butterfly(phi_g, rxm, n, n - i, b, cnt, is_fft, tab, mid);
}
__global__ void k_phi_g_scale(gle *phi_g, gle rx0, u32 n, PowTab tab) {
    const u32 b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < (1u << (n - 1))) phi_scale(phi_g, rx0, n, b, tab);
}
static int phi_g_init_run(const uint64_t *rx, uint32_t n, const uint64_t *scale, int is_fft, u32 max_head, dp_mle **w_red, dp_mle **mid) {
    PowTab tab; if (int e = dp_root_powtab(&tab)) return e;
    PhiArgs a; memset(&a, 0, sizeof a);
    for (u32 i = 0; i < n; i++) a.rx[i] = e_from_host(rx + 2 * i);
    a.scale = e_from_host(scale);
    std::fill(mid, mid + n - 1, nullptr);   // a failed call leaves no dangling entries
    MlePtr w; if (int e = dp_mle_alloc(1ULL << n, true, w)) return e;
    cudaStream_t st = dp_ctx().stream;
    DP_CUDA(cudaMemsetAsync(w->data, 0, w->bytes(), st));                // the reference's vec![E::ZERO; ..]: the FFT case leaves the top half zero
    std::vector<MlePtr> own(n - 1);
    for (u32 i = 0; i + 1 < n; i++) { if (int e = dp_mle_alloc(2ULL << i, true, own[i])) return e; a.mid[i] = (gle *)own[i]->data; }
    const u32 last = is_fft ? n : n - 1, head = std::min(last, max_head);
    gle *phi = (gle *)w->data;
    DP_CUDA(dp_launch(k_phi_g_init, 1, 1024, 0, st, phi, a, n, head, is_fft, tab));
    for (u32 i = head + 1; i <= last; i++)
        DP_CUDA(dp_launch(k_phi_g_level, ((1u << (i - 1)) + 255) / 256, 256, 0, st, phi, a.rx[n - i], n, i, is_fft, i < n ? a.mid[i - 1] : nullptr, tab));
    if (!is_fft && head < last) DP_CUDA(dp_launch(k_phi_g_scale, ((1u << (n - 1)) + 255) / 256, 256, 0, st, phi, a.rx[0], n, tab));
    for (u32 i = 0; i + 1 < n; i++) mid[i] = own[i].release();
    *w_red = w.release(); return DP_OK;
}
extern "C" int dp_phi_g_init(const uint64_t *rx, uint32_t n, const uint64_t *scale, int is_fft, dp_mle **w_red, dp_mle **mid) {
    DP_REQUIRE_CTX();
    DP_CHECK(rx && scale && w_red && mid && n >= 2 && n <= 14, DP_ERR_INVALID, "dp_phi_g_init: need 2 <= n <= 14");
    return phi_g_init_run(rx, n, scale, is_fft, n, w_red, mid);
}
extern "C" int dp_phi_g_init_long(const uint64_t *rx, uint32_t n, const uint64_t *scale, int is_fft, dp_mle **w_red, dp_mle **mid) {
    DP_REQUIRE_CTX();
    DP_CHECK(rx && scale && w_red && mid && n >= 15 && n <= PHI_MAX_N, DP_ERR_INVALID, "dp_phi_g_init_long: need 15 <= n <= 21");
    return phi_g_init_run(rx, n, scale, is_fft, PHI_HEAD_LEVELS, w_red, mid);
}

// ---- one level of delegate_matrix_evaluation (prover.rs:182-195): phi[i] = A + B * omega^(i << shift), omega of order 2^n_total ----
__global__ void k_phi_level(gle *out, u32 len, u32 n_total, u32 shift, gle A, gle B, int inverse, PowTab tab) {
    u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= len) return;
    u32 e = (i << shift) & ((1u << n_total) - 1);
    if (inverse && e) e = (1u << n_total) - e;
    out[i] = e_add(A, e_mul_base(B, tab_pow(tab, (u64)e << (32 - n_total))));
}
extern "C" int dp_phi_level(uint32_t len_log, uint32_t n_total, uint32_t shift, const uint64_t *A, const uint64_t *B, int inverse, dp_mle **out) {
    DP_REQUIRE_CTX();
    DP_CHECK(A && B && out && n_total >= 1 && n_total <= 32 && len_log + shift <= n_total, DP_ERR_INVALID, "dp_phi_level: bad arguments");
    PowTab tab; if (int e = dp_root_powtab(&tab)) return e;
    MlePtr m; if (int e = dp_mle_alloc(1ULL << len_log, true, m)) return e;
    u32 len = 1u << len_log;
    DP_CUDA(dp_launch(k_phi_level, (len + 255) / 256, 256, 0, dp_ctx().stream, (gle *)m->data, len, n_total, shift, e_from_host(A), e_from_host(B), inverse, tab));
    *out = m.release(); return DP_OK;
}

// ---- out = src repeated `times` times (beta_acc = vec![beta2; kx].concat(), convolution.rs:870) ----
__global__ void k_repeat(const gle *src, u64 len, u64 total, gle *out) {
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    for (; t < total; t += stride) out[t] = src[t & (len - 1)];
}
extern "C" int dp_mle_repeat(const dp_mle *src, uint32_t times, dp_mle **out) {
    DP_REQUIRE_CTX();
    DP_CHECK(src && out && src->is_ext && times && (times & (times - 1)) == 0, DP_ERR_INVALID, "dp_mle_repeat: need an Ext MLE and a power-of-two count");
    MlePtr m; if (int e = dp_mle_alloc(src->len * times, true, m)) return e;
    DP_CUDA(dp_launch(k_repeat, dp_grid_for(m->len, 256, 8), 256, 0, dp_ctx().stream, (const gle *)src->data, src->len, m->len, (gle *)m->data));
    *out = m.release(); return DP_OK;
}
