// multilinear_extensions on device: upload/canonicalise, eq table (K5), MSB fold (K3), LSB fold (K2),
// evaluate (K4).  Reference: multilinear_extensions/src/mle.rs:454-712, virtual_poly.rs:346-453,
// zkml/src/commit/mod.rs:10-28.  All kernels are HBM-streaming integer kernels: 16-byte vector loads,
// coalesced along the fastest index, lazy (160-bit) accumulation so a dot product costs one modular
// reduction per output instead of one per term.
#include "common.cuh"
#include <algorithm>

struct PointArg { gle r[32]; };

__global__ void k_canonicalize(u64 *v, u64 n) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    for (; i < n; i += stride) { u64 x = v[i]; v[i] = x >= GL_P ? x - GL_P : x; }
}

// ---- K5: eq / beta table --------------------------------------------------------------------------
// table[x] = prod_b (x_b ? r[off+b] : 1 - r[off+b]),  x < 2^nbits
__global__ void k_eq_small(PointArg pt, u32 off, u32 nbits, gle *table) {
    u32 x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= (1u << nbits)) return;
    gle p = e_one();
    for (u32 b = 0; b < nbits; b++) {
        gle r = pt.r[off + b];
        p = e_mul(p, ((x >> b) & 1) ? r : e_sub(e_one(), r));
    }
    st_e(table + x, p);
}
// out[x] = hi[x >> L] * lo[x & (2^L-1)]
__global__ void k_eq_expand(const gle *__restrict__ lo, const gle *__restrict__ hi, u32 L, u64 n, gle *__restrict__ out) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    u64 mask = (1ULL << L) - 1;
    for (; i < n; i += stride) st_e(out + i, e_mul(ld_e(hi + (i >> L)), ld_e(lo + (i & mask))));
}

static int dpk_eq_build(const gle *point, u32 nv, gle *out) {
    DpCtx &c = dp_ctx();
    DP_CHECK(nv <= 32, DP_ERR_INVALID, "eq_build: num_vars > 32");
    PointArg pa; memset(&pa, 0, sizeof pa);
    for (u32 i = 0; i < nv; i++) pa.r[i] = point[i];
    const u32 L = 10;
    if (nv <= L + 2) {
        u32 n = 1u << nv;
        DP_CUDA(dp_launch(k_eq_small, (n + 127) / 128, 128, 0, c.stream, pa, 0, nv, out));
        return DP_OK;
    }
    u32 H = nv - L;
    gle *lo = nullptr, *hi = nullptr;
    if (int e = dp_dev_alloc((void **)&lo, sizeof(gle) << L)) return e;
    DevPtr lo_owner(lo);
    if (int e = dp_dev_alloc((void **)&hi, sizeof(gle) << H)) return e;
    DevPtr hi_owner(hi);
    DP_CUDA(dp_launch(k_eq_small, ((1u << L) + 127) / 128, 128, 0, c.stream, pa, 0, L, lo));
    if (H <= 14) DP_CUDA(dp_launch(k_eq_small, ((1u << H) + 127) / 128, 128, 0, c.stream, pa, L, H, hi));
    else {  // recurse once for very large tables
        gle sub[32];
        for (u32 i = 0; i < H; i++) sub[i] = point[L + i];
        if (int e = dpk_eq_build(sub, H, hi)) return e;
    }
    u64 n = 1ULL << nv;
    DP_CUDA(dp_launch(k_eq_expand, dp_grid_for(n, 256, 8), 256, 0, c.stream, lo, hi, L, n, out));
    return DP_OK;
}

// ---- K2: LSB fold, stand-alone ---------------------------------------------------------------------
template <bool EXT>
__global__ void k_fold_low(const void *__restrict__ src, u64 half, gle r, gle *__restrict__ out) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    for (; i < half; i += stride) {
        if (EXT) {
            const gle *s = (const gle *)src;
            gle a = ld_e(s + 2 * i), b = ld_e(s + 2 * i + 1);
            st_e(out + i, e_add(a, e_mul(e_sub(b, a), r)));
        } else {
            ulonglong2 v = ld_b2((const u64 *)src + 2 * i);
            st_e(out + i, e_add(e_mul_base(r, gl_sub(v.y, v.x)), e_from_base(v.x)));
        }
    }
}
int dpk_fold_low(const void *src, bool src_ext, u64 len, gle r, gle *out) {
    DpCtx &c = dp_ctx();
    u64 half = len >> 1;
    DP_CUDA(dp_launch(src_ext ? k_fold_low<true> : k_fold_low<false>, dp_grid_for(half, 256, 8), 256, 0, c.stream, src, half, r, out));
    return DP_OK;
}

// ---- K3: MSB fold of k variables in ONE pass --------------------------------------------------------
// fix_high_variables_in_place folds one variable per pass (mle.rs:562-603, ~48n bytes).  The map is
// linear, so out[i] = sum_j eq(point)[j] * f[j*S + i] is the same field element: one pass, 16n(1+2^-k)
// bytes (SURVEY.md 8d).  Grid: x tiles the S outputs (coalesced), y splits the J = 2^k rows.
template <bool EXT>
__global__ void k_fixhigh_cols(const void *__restrict__ src, const gle *__restrict__ w, u64 S, u64 J, u64 rows_per_y,
                               gle *__restrict__ part /* [gridDim.y][S] */) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= S) return;
    u64 j0 = (u64)blockIdx.y * rows_per_y, j1 = j0 + rows_per_y; if (j1 > J) j1 = J;
    if (EXT) {
        const gle *f = (const gle *)src;
        gl_acc s00 = {0, 0, 0}, s11 = {0, 0, 0}, s01 = {0, 0, 0};
#pragma unroll 4
        for (u64 j = j0; j < j1; j++) {
            gle a = ld_e(w + j), b = ld_e(f + j * S + i);
            gl_acc_mac(s00, a.c0, b.c0); gl_acc_mac(s11, a.c1, b.c1); gl_acc_mac(s01, a.c0, b.c1); gl_acc_mac(s01, a.c1, b.c0);
        }
        st_e(part + (u64)blockIdx.y * S + i, e_make(gl_add(gl_acc_reduce(s00), gl_mul7(gl_acc_reduce(s11))), gl_acc_reduce(s01)));
    } else {
        const u64 *f = (const u64 *)src;
        gl_acc s0 = {0, 0, 0}, s1 = {0, 0, 0};
#pragma unroll 4
        for (u64 j = j0; j < j1; j++) {
            gle a = ld_e(w + j); u64 b = f[j * S + i];
            gl_acc_mac(s0, a.c0, b); gl_acc_mac(s1, a.c1, b);
        }
        st_e(part + (u64)blockIdx.y * S + i, e_make(gl_acc_reduce(s0), gl_acc_reduce(s1)));
    }
}
__global__ void k_sum_parts(const gle *__restrict__ part, u64 S, u32 ny, gle *__restrict__ out) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= S) return;
    gle a = e_zero();
    for (u32 y = 0; y < ny; y++) a = e_add(a, ld_e(part + (u64)y * S + i));
    st_e(out + i, a);
}
// the sum of every thread's `acc` (blockDim.x a multiple of 32), stored to *dst by thread 0
__device__ __forceinline__ void block_sum_store(gle acc, gle *dst) {
    __shared__ gle sm[32];
    for (int d = 16; d > 0; d >>= 1) acc = e_add(acc, shfl_down_e(acc, d));
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x < 32) {
        acc = threadIdx.x < (blockDim.x >> 5) ? sm[threadIdx.x] : e_zero();
        for (int d = 16; d > 0; d >>= 1) acc = e_add(acc, shfl_down_e(acc, d));
        if (threadIdx.x == 0) st_e(dst, acc);
    }
}
// few outputs (S < 32): one block per output, threads stride over the J rows, block reduction
template <bool EXT>
__global__ void k_fixhigh_dot(const void *__restrict__ src, const gle *__restrict__ w, u64 S, u64 J, gle *__restrict__ out) {
    u64 i = blockIdx.x;
    gle acc = e_zero();
    for (u64 j = threadIdx.x; j < J; j += blockDim.x) {
        gle a = ld_e(w + j);
        if (EXT) acc = e_add(acc, e_mul(a, ld_e((const gle *)src + j * S + i)));
        else acc = e_add(acc, e_mul_base(a, ((const u64 *)src)[j * S + i]));
    }
    block_sum_store(acc, out + i);
}

// several MLEs of equal size evaluated at ONE point: the eq table is built once, one launch, one copy back
struct EvalArg { const void *src[16]; u32 ext[16]; };
__global__ void k_eval_many(EvalArg a, const gle *__restrict__ w, u64 J, gle *__restrict__ out) {
    const u32 y = blockIdx.x;
    gle acc = e_zero();
    for (u64 j = threadIdx.x; j < J; j += blockDim.x) {
        gle wj = ld_e(w + j);
        if (a.ext[y]) acc = e_add(acc, e_mul(wj, ld_e((const gle *)a.src[y] + j)));
        else acc = e_add(acc, e_mul_base(wj, ((const u64 *)a.src[y])[j]));
    }
    block_sum_store(acc, out + y);
}

static int dpk_fix_high(const void *src, bool src_ext, u64 len, const gle *point, u32 k, gle *out) {
    DpCtx &c = dp_ctx();
    u64 J = 1ULL << k, S = len >> k;
    gle *w = nullptr;
    if (int e = dp_dev_alloc((void **)&w, sizeof(gle) * J)) return e;
    DevPtr w_owner(w);
    if (int e = dpk_eq_build(point, k, w)) return e;
    DpProfScope prof(S < 32 ? "k_fixhigh_dot" : "k_fixhigh_cols", len * (src_ext ? 16 : 8) + S * 16);
    if (S < 32) {
        DP_CUDA(dp_launch(src_ext ? k_fixhigh_dot<true> : k_fixhigh_dot<false>, (unsigned)S, 256, 0, c.stream, src, w, S, J, out));
    } else {
        const int T = 128;
        u64 gx = (S + T - 1) / T;
        u64 want = (u64)c.sm_count * 8;
        u64 ny = gx >= want ? 1 : (want + gx - 1) / gx;
        if (ny > J) ny = J;
        if (ny > 1024) ny = 1024;
        u64 rows = (J + ny - 1) / ny; ny = (J + rows - 1) / rows;
        gle *part = out;
        DevPtr part_owner;
        if (ny > 1) { if (int e = dp_dev_alloc((void **)&part, sizeof(gle) * S * ny)) return e; part_owner.reset(part); }
        DP_CUDA(dp_launch(src_ext ? k_fixhigh_cols<true> : k_fixhigh_cols<false>, dim3((unsigned)gx, (unsigned)ny), T, 0, c.stream, src, w, S, J, rows, part));
        if (ny > 1) DP_CUDA(dp_launch(k_sum_parts, (unsigned)((S + 255) / 256), 256, 0, c.stream, part, S, (u32)ny, out));
    }
    return DP_OK;
}

static void point_from_host(const uint64_t *point, u32 k, gle *out) {
    for (u32 i = 0; i < k; i++) out[i] = e_from_host(point + 2 * i);
}

// fix_high_variables (mle.rs:529-603): `m` with its top k >= 1 variables fixed at `point`, as a new Ext MLE
static int fix_high(const dp_mle *m, const uint64_t *point, u32 k, MlePtr &out) {
    gle pt[32]; point_from_host(point, k, pt);
    MlePtr r;
    if (int e = dp_mle_alloc(m->len >> k, true, r)) return e;
    if (int e = dpk_fix_high(m->data, m->is_ext, m->len, pt, k, (gle *)r->data)) return e;
    out = std::move(r);
    return DP_OK;
}

// =====================================================================================================
extern "C" {

int dp_mle_upload(const uint64_t *evals, uint64_t len, int is_ext, dp_mle **out) {
    DP_REQUIRE_CTX();
    DP_CHECK(out && evals, DP_ERR_INVALID, "dp_mle_upload: null argument");
    DP_CHECK(len > 0 && (len & (len - 1)) == 0, DP_ERR_INVALID, "dp_mle_upload: len must be a power of two");
    MlePtr m;
    if (int e = dp_mle_alloc(len, is_ext != 0, m)) return e;
    DP_CUDA(cudaMemcpyAsync(m->data, evals, m->bytes(), cudaMemcpyHostToDevice, dp_ctx().stream));
    u64 n = len * (is_ext ? 2 : 1);
    DP_CUDA(dp_launch(k_canonicalize, dp_grid_for(n, 256, 8), 256, 0, dp_ctx().stream, (u64 *)m->data, n));
    *out = m.release();
    return DP_OK;
}

int dp_mle_wrap_device(void *dev_ptr, uint64_t len, int is_ext, dp_mle **out) {
    DP_REQUIRE_CTX();
    DP_CHECK(out && dev_ptr, DP_ERR_INVALID, "dp_mle_wrap_device: null argument");
    DP_CHECK(len > 0 && (len & (len - 1)) == 0, DP_ERR_INVALID, "dp_mle_wrap_device: len must be a power of two");
    DP_CHECK(((uintptr_t)dev_ptr & 15) == 0, DP_ERR_INVALID, "dp_mle_wrap_device: pointer must be 16-byte aligned");
    *out = dp_mle_view(dev_ptr, len, is_ext != 0);
    return DP_OK;
}

int dp_mle_clone(const dp_mle *src, dp_mle **out) {
    DP_REQUIRE_CTX();
    DP_CHECK(src && out, DP_ERR_INVALID, "dp_mle_clone: null argument");
    MlePtr m;
    if (int e = dp_mle_alloc(src->len, src->is_ext, m)) return e;
    DP_CUDA(cudaMemcpyAsync(m->data, src->data, m->bytes(), cudaMemcpyDeviceToDevice, dp_ctx().stream));
    *out = m.release();
    return DP_OK;
}

int dp_mle_download(const dp_mle *m, uint64_t *out_evals) {
    DP_REQUIRE_CTX();
    DP_CHECK(m && out_evals, DP_ERR_INVALID, "dp_mle_download: null argument");
    return dp_d2h(out_evals, m->data, m->bytes(), dp_ctx().stream);
}

int dp_mle_info(const dp_mle *m, uint64_t *len, int *is_ext, uint32_t *num_vars) {
    if (!m) return dp_fail(DP_ERR_INVALID, "dp_mle_info: null");
    if (len) *len = m->len;
    if (is_ext) *is_ext = m->is_ext;
    if (num_vars) *num_vars = m->num_vars();
    return DP_OK;
}
void *dp_mle_device_ptr(const dp_mle *m) { return m ? m->data : nullptr; }

int dp_mle_free(dp_mle *m) {
    if (!m) return DP_OK;
    if (m->owned && dp_ctx().ready) dp_dev_free(m->data);
    delete m;
    return DP_OK;
}

int dp_mle_fix_high(dp_mle *m, const uint64_t *point, uint32_t k) {
    DP_REQUIRE_CTX();
    DP_CHECK(m && (point || k == 0), DP_ERR_INVALID, "dp_mle_fix_high: null argument");
    DP_CHECK(k <= m->num_vars(), DP_ERR_INVALID, "invalid size of partial point");  // mle.rs:564-567
    if (k == 0) return DP_OK;  // reference leaves a Base MLE untouched when the point is empty
    MlePtr r;
    if (int e = fix_high(m, point, k, r)) return e;
    std::swap(*m, *r);         // m takes the folded table; its old one leaves with r
    return DP_OK;
}

// fix_high_variables (mle.rs:529-560): same as above but returns a new MLE and leaves `m` untouched
int dp_mle_fix_high_new(const dp_mle *m, const uint64_t *point, uint32_t k, dp_mle **outp) {
    DP_REQUIRE_CTX();
    DP_CHECK(m && outp && (point || k == 0), DP_ERR_INVALID, "dp_mle_fix_high_new: null argument");
    DP_CHECK(k <= m->num_vars(), DP_ERR_INVALID, "invalid size of partial point");
    if (k == 0) return dp_mle_clone(m, outp);
    MlePtr r;
    if (int e = fix_high(m, point, k, r)) return e;
    *outp = r.release();
    return DP_OK;
}

int dp_mle_fix_low(const dp_mle *m, const uint64_t *point, uint32_t k, dp_mle **outp) {
    DP_REQUIRE_CTX();
    DP_CHECK(m && outp && (point || k == 0), DP_ERR_INVALID, "dp_mle_fix_low: null argument");
    DP_CHECK(k <= m->num_vars(), DP_ERR_INVALID, "invalid size of partial point");  // mle.rs:457-460
    if (k == 0) return dp_mle_clone(m, outp);
    gle pt[32]; point_from_host(point, k, pt);
    MlePtr cur(dp_mle_view(m->data, m->len, m->is_ext));    // each fold reads the previous table and frees it once done
    for (u32 i = 0; i < k; i++) {
        MlePtr nxt;
        if (int e = dp_mle_alloc(cur->len >> 1, true, nxt)) return e;
        if (int e = dpk_fold_low(cur->data, cur->is_ext, cur->len, pt[i], (gle *)nxt->data)) return e;
        cur = std::move(nxt);
    }
    *outp = cur.release();
    return DP_OK;
}

int dp_mle_evaluate(const dp_mle *m, const uint64_t *point, uint32_t num_vars, uint64_t out[2]) {
    DP_REQUIRE_CTX();
    DP_CHECK(m && out, DP_ERR_INVALID, "dp_mle_evaluate: null argument");
    DP_CHECK(num_vars == m->num_vars(), DP_ERR_INVALID, "MLE size does not match the point");  // mle.rs:609-613
    gle *res = nullptr;
    if (int e = dp_dev_alloc((void **)&res, sizeof(gle))) return e;
    DevPtr res_owner(res);
    if (num_vars == 0) {
        if (m->is_ext) DP_CUDA(cudaMemcpyAsync(res, m->data, 16, cudaMemcpyDeviceToDevice, dp_ctx().stream));
        else { DP_CUDA(cudaMemsetAsync(res, 0, 16, dp_ctx().stream)); DP_CUDA(cudaMemcpyAsync(res, m->data, 8, cudaMemcpyDeviceToDevice, dp_ctx().stream)); }
    } else {
        gle pt[32]; point_from_host(point, num_vars, pt);
        // evaluate == fold every variable; as a linear map it is sum_x eq(point)[x] f[x].  Two MSB passes:
        // the top (nv-10) variables stream f once, the remaining 2^10 values finish in one block.
        const u32 LOW = 10;
        if (num_vars <= LOW + 2) {
            if (int e = dpk_fix_high(m->data, m->is_ext, m->len, pt, num_vars, res)) return e;
        } else {
            gle *mid = nullptr;
            if (int e = dp_dev_alloc((void **)&mid, sizeof(gle) << LOW)) return e;
            DevPtr mid_owner(mid);
            if (int e = dpk_fix_high(m->data, m->is_ext, m->len, pt + LOW, num_vars - LOW, mid)) return e;
            if (int e = dpk_fix_high(mid, true, 1ULL << LOW, pt, LOW, res)) return e;
        }
    }
    return dp_d2h(out, res, 16, dp_ctx().stream);
}

// evaluate (mle.rs:607-623) for n MLEs with the same num_vars at the same point (e.g. the LogUp output claims,
// logup_gkr/prover.rs:172-183): out = n x [c0,c1]
int dp_mle_evaluate_many(const dp_mle *const *mles, uint32_t n, const uint64_t *point, uint32_t num_vars, uint64_t *out) {
    DP_REQUIRE_CTX();
    DP_CHECK(mles && out && n > 0 && (point || num_vars == 0), DP_ERR_INVALID, "dp_mle_evaluate_many: null argument");
    for (u32 i = 0; i < n; i++) DP_CHECK(mles[i] && mles[i]->num_vars() == num_vars, DP_ERR_INVALID, "MLE size does not match the point");
    if (num_vars == 0 || num_vars > 16) {   // rare shapes: one by one
        for (u32 i = 0; i < n; i++) if (int e = dp_mle_evaluate(mles[i], point, num_vars, out + 2 * i)) return e;
        return DP_OK;
    }
    gle pt[32]; point_from_host(point, num_vars, pt);
    u64 J = 1ULL << num_vars;
    gle *w = nullptr, *res = nullptr, *hres = nullptr;
    if (int e = dp_dev_alloc((void **)&w, sizeof(gle) * J)) return e;
    DevPtr w_owner(w);
    if (int e = dp_dev_alloc((void **)&res, sizeof(gle) * n)) return e;
    DevPtr res_owner(res);
    if (int e = dp_pinned_alloc((void **)&hres, sizeof(gle) * n)) return e;
    PinnedPtr hres_owner(hres);
    if (int e = dpk_eq_build(pt, num_vars, w)) return e;
    for (u32 base = 0; base < n; base += 16) {
        EvalArg a; memset(&a, 0, sizeof a);
        u32 cnt = std::min<u32>(16, n - base);
        for (u32 i = 0; i < cnt; i++) { a.src[i] = mles[base + i]->data; a.ext[i] = mles[base + i]->is_ext; }
        DP_CUDA(dp_launch(k_eval_many, cnt, 256, 0, dp_ctx().stream, a, w, J, res + base));
    }
    DP_CUDA(cudaMemcpyAsync(hres, res, sizeof(gle) * n, cudaMemcpyDeviceToHost, dp_ctx().stream));
    DP_CUDA(dp_stream_sync(dp_ctx().stream));
    for (u32 i = 0; i < n; i++) { out[2 * i] = hres[i].c0; out[2 * i + 1] = hres[i].c1; }
    return DP_OK;
}

int dp_eq_build(const uint64_t *point, uint32_t num_vars, dp_mle **outp) {
    DP_REQUIRE_CTX();
    DP_CHECK(outp && (point || num_vars == 0), DP_ERR_INVALID, "dp_eq_build: null argument");
    DP_CHECK(num_vars <= 32, DP_ERR_INVALID, "dp_eq_build: num_vars > 32");
    gle pt[32]; point_from_host(point, num_vars, pt);
    MlePtr r;
    if (int e = dp_mle_alloc(1ULL << num_vars, true, r)) return e;
    if (int e = dpk_eq_build(pt, num_vars, (gle *)r->data)) return e;
    *outp = r.release();
    return DP_OK;
}

}  // extern "C"
