// LogUp-GKR fractional-sum circuit on device (K6) + linear combinations of MLEs.
// Reference: zkml/src/lookup/logup_gkr/circuit.rs:49-287 (LogUpLayer::next_layer, LogUpCircuit::{new,
// new_lookup_circuit,new_table_circuit}), structs.rs:45-56 (Fraction add), zkml/src/commit/same_poly.rs:88-110
// (final_beta = sum_i a_i * beta(r_i)).
//
// The reference builds every layer with sequential iterators; here each layer is one streaming kernel
// over HBM (read 2 x 32 B, write 32 B per output fraction) and all layers stay resident because each is
// the input of one sumcheck of batch_prove (prover.rs:24-198) -- the (low, high) halves the sumcheck needs
// (circuit.rs:137-180 copies them) are just pointer offsets into the layer arrays.
#include "common.cuh"

// den[i] = c + sum_k gamma^k * col_k[i]   (circuit.rs:213-222 / :247-256)
struct ColsArg { const u64 *col[16]; gle pw[16]; u32 n; };
__global__ void k_logup_den(ColsArg a, gle c, u64 len, gle *__restrict__ den) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    for (; i < len; i += stride) {
        gle acc = c;
        for (u32 k = 0; k < a.n; k++) acc = e_add(acc, e_mul_base(a.pw[k], a.col[k][i]));
        st_e(den + i, acc);
    }
}
__global__ void k_lift_b2e(const u64 *__restrict__ src, gle *__restrict__ out, u64 n) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    for (; i < n; i += stride) st_e(out + i, e_from_base(src[i]));
}
// (n1/d1) + (n2/d2) = (n1 d2 + d1 n2) / (d1 d2), pairing i with i + half   (circuit.rs:66-78, structs.rs:45-56)
template <bool INIT_LOOKUP>
__global__ void k_logup_layer(const gle *__restrict__ num, const gle *__restrict__ den, u64 half, gle *__restrict__ onum, gle *__restrict__ oden) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    for (; i < half; i += stride) {
        gle d1 = ld_e(den + i), d2 = ld_e(den + i + half);
        gle n;
        if (INIT_LOOKUP) n = e_neg(e_add(d2, d1));   // numerators are all -1 (circuit.rs:85-91): (-1) d2 + d1 (-1)
        else { gle n1 = ld_e(num + i), n2 = ld_e(num + i + half); n = e_add(e_mul(n1, d2), e_mul(d1, n2)); }
        st_e(onum + i, n);
        st_e(oden + i, e_mul(d1, d2));
    }
}
// all remaining (small) layers in one single-block launch
struct LayerPtrs { gle *num[40]; gle *den[40]; };
// `out_host` (mapped pinned, 9 words): the circuit's outputs [n0, n1, d0, d1] and then the completion word, stored by the kernel itself
__global__ void __launch_bounds__(256) k_logup_tail(LayerPtrs lp, u32 from_layer, u32 n_layers, u64 len0, bool first_is_lookup, u64 *out_host, u64 seq) {
    for (u32 k = from_layer; k + 1 < n_layers; k++) {
        u64 half = len0 >> (k + 1);
        const gle *num = lp.num[k], *den = lp.den[k];
        for (u64 i = threadIdx.x; i < half; i += blockDim.x) {
            gle d1 = den[i], d2 = den[i + half], n;
            if (k == 0 && first_is_lookup) n = e_neg(e_add(d2, d1));
            else { gle n1 = num[i], n2 = num[i + half]; n = e_add(e_mul(n1, d2), e_mul(d1, n2)); }
            lp.num[k + 1][i] = n; lp.den[k + 1][i] = e_mul(d1, d2);
        }
        __syncthreads();
    }
    if (out_host && threadIdx.x == 0) {
        const gle *num = lp.num[n_layers - 1], *den = lp.den[n_layers - 1];
        const gle a = num[0], b = num[1], c = den[0], d = den[1];
        out_host[0] = a.c0; out_host[1] = a.c1; out_host[2] = b.c0; out_host[3] = b.c1; out_host[4] = c.c0; out_host[5] = c.c1; out_host[6] = d.c0; out_host[7] = d.c1;
        dp_publish(out_host + 8, seq);
    }
}
// out[i] = sum_k coef_k * m_k[i]
struct LinArg { const gle *m[16]; gle coef[16]; u32 n; };
__global__ void k_lincomb(LinArg a, u64 len, gle *__restrict__ out) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
    for (; i < len; i += stride) {
        gle acc = e_zero();
        for (u32 k = 0; k < a.n; k++) acc = e_add(acc, e_mul(a.coef[k], ld_e(a.m[k] + i)));
        st_e(out + i, acc);
    }
}

extern "C" {

// LogUpCircuit::new_lookup_circuit (multiplicities == NULL) / new_table_circuit
int dp_logup_build(dp_mle *const *columns, uint32_t n_columns, const dp_mle *multiplicities, const uint64_t constant_challenge[2],
                   const uint64_t column_separation_challenge[2], dp_logup **out) {
    DP_REQUIRE_CTX();
    DP_CHECK(columns && n_columns >= 1 && n_columns <= 16 && out && constant_challenge && column_separation_challenge, DP_ERR_INVALID, "dp_logup_build: bad argument");
    for (u32 k = 0; k < n_columns; k++) DP_CHECK(columns[k], DP_ERR_INVALID, "dp_logup_build: null column");
    u64 len = columns[0]->len;
    for (u32 k = 0; k < n_columns; k++) DP_CHECK(!columns[k]->is_ext && columns[k]->len == len, DP_ERR_INVALID, "All sets of evaluations should be the same length");   // structs.rs:168-176
    DP_CHECK(len >= 4, DP_ERR_INVALID, "dp_logup_build: need at least 4 evaluations");
    if (multiplicities) DP_CHECK(!multiplicities->is_ext && multiplicities->len == len, DP_ERR_INVALID, "Multiplicities length was not equal to column evaluations length");
    DpCtx &c = dp_ctx();
    std::unique_ptr<dp_logup, FreeWith<dp_logup_free>> L(new dp_logup());
    L->table = multiplicities != nullptr;
    L->nv = 0; while ((1ULL << L->nv) < len) L->nv++;
    // one allocation: layer k has 2^(nv-k) entries, k = 0..nv-1; (num, den) each
    u64 total = 0;
    for (u32 k = 0; k < L->nv; k++) total += 2 * (len >> k);
    if (int e = dp_dev_alloc((void **)&L->block, sizeof(gle) * total)) return e;
    gle *p = L->block;
    for (u32 k = 0; k < L->nv; k++) { L->num.push_back(p); p += len >> k; L->den.push_back(p); p += len >> k; }
    ColsArg ca; memset(&ca, 0, sizeof ca); ca.n = n_columns;
    gle sep = e_from_host(column_separation_challenge);
    gle pw = e_one();
    for (u32 k = 0; k < n_columns; k++) { ca.col[k] = (const u64 *)columns[k]->data; ca.pw[k] = pw; pw = e_mul(pw, sep); }
    gle cc = e_from_host(constant_challenge);
    int g = dp_grid_for(len, 256, 8);
    { DpProfScope prof("k_logup_den", len * (8 * n_columns + 16)); DP_CUDA(dp_launch(k_logup_den, g, 256, 0, c.stream, ca, cc, len, L->den[0])); }
    if (L->table) DP_CUDA(dp_launch(k_lift_b2e, g, 256, 0, c.stream, (const u64 *)multiplicities->data, L->num[0], len));
    u32 k = 0;
    for (; k + 1 < L->nv && (len >> (k + 1)) > 1024; k++) {
        u64 half = len >> (k + 1);
        const bool init_lookup = k == 0 && !L->table;       // a lookup circuit's first numerators are all -1: L->num[0] holds none
        DpProfScope prof("k_logup_layer", half * 96);
        DP_CUDA(dp_launch(init_lookup ? k_logup_layer<true> : k_logup_layer<false>, dp_grid_for(half, 256, 8), 256, 0, c.stream,
                          init_lookup ? nullptr : L->num[k], L->den[k], half, L->num[k + 1], L->den[k + 1]));
    }
    if (k + 1 < L->nv) {
        LayerPtrs lp; memset(&lp, 0, sizeof lp);
        for (u32 q = 0; q < L->nv && q < 40; q++) { lp.num[q] = L->num[q]; lp.den[q] = L->den[q]; }
        DpProfScope prof("k_logup_tail", (len >> k) * 96);
        void *hp = nullptr;
        if (L->nv - 1 > k && dp_pinned_alloc(&hp, 128) == DP_OK) { L->h_out = (u64 *)hp; L->h_out[8] = 0; }
        DP_CUDA(dp_launch(k_logup_tail, 1, 256, 0, c.stream, lp, k, L->nv, len, !L->table, L->h_out, 1));
    }
    if (!L->table) L->num[0] = nullptr;
    *out = L.release();
    return DP_OK;
}

int dp_logup_num_vars(const dp_logup *L, uint32_t *input_num_vars) {
    if (!L || !input_num_vars) return dp_fail(DP_ERR_INVALID, "dp_logup_num_vars: null");
    *input_num_vars = L->nv - 1;   // LogUpLayer::num_vars of the input layer (circuit.rs:35-42)
    return DP_OK;
}

// LogUpCircuit::outputs (circuit.rs:273-275): [n0, n1, d0, d1] of the last layer
int dp_logup_outputs(const dp_logup *L, uint64_t out[8]) {
    DP_REQUIRE_CTX();
    DP_CHECK(L && out, DP_ERR_INVALID, "dp_logup_outputs: null");
    u32 last = L->nv - 1;
    DP_CHECK(L->num[last] != nullptr, DP_ERR_INVALID, "dp_logup_outputs: circuit too small");
    if (L->h_out) {   // stored by the tail kernel itself
        if (int e = dp_await(L->h_out + 8, 1, 30.0, "dp_logup_outputs: the tail kernel did not publish the outputs")) return e;
        memcpy(out, L->h_out, 64);
        return DP_OK;
    }
    DpD2H x(dp_ctx().stream, 64);
    if (int e = x.add(out, L->num[last], 32)) return e;
    if (int e = x.add(out + 4, L->den[last], 32)) return e;
    return x.finish();
}

// LogUpLayer::get_mles (circuit.rs:137-180) of the layer whose halves have `layer_vars` variables:
// views [num_low, num_high, den_low, den_high], or [den_low, den_high] for the initial lookup layer.
int dp_logup_layer_mles(const dp_logup *L, uint32_t layer_vars, dp_mle **out_views, uint32_t *n_views) {
    DP_REQUIRE_CTX();
    DP_CHECK(L && out_views && n_views, DP_ERR_INVALID, "dp_logup_layer_mles: null");
    DP_CHECK(layer_vars + 1 <= L->nv, DP_ERR_INVALID, "One of the circuits was not the same size as the others");   // prover.rs:103-105
    u32 k = L->nv - 1 - layer_vars;          // layer index: 2^(layer_vars+1) entries
    u64 half = 1ULL << layer_vars;
    u32 n = 0;
    if (L->num[k]) { out_views[n++] = dp_mle_view(L->num[k], half, true); out_views[n++] = dp_mle_view(L->num[k] + half, half, true); }
    out_views[n++] = dp_mle_view(L->den[k], half, true); out_views[n++] = dp_mle_view(L->den[k] + half, half, true);
    *n_views = n;
    return DP_OK;
}

int dp_logup_free(dp_logup *L) {
    if (!L) return DP_OK;
    if (dp_ctx().ready) {
        if (L->h_out && L->h_out[8] != 1) dp_stream_sync(dp_ctx().stream);   // the tail kernel still owns the pinned block
        dp_dev_free(L->block);
    }
    dp_pinned_free(L->h_out);
    delete L;
    return DP_OK;
}

// out = sum_k coefs[k] * mles[k]  (all Ext, same length) -- same_poly's final_beta (same_poly.rs:91-110)
int dp_mle_linear_combination(dp_mle *const *mles, const uint64_t *coefs, uint32_t n, dp_mle **out) {
    DP_REQUIRE_CTX();
    DP_CHECK(mles && coefs && out && n >= 1 && n <= 16, DP_ERR_INVALID, "dp_mle_linear_combination: bad argument");
    for (u32 k = 0; k < n; k++) DP_CHECK(mles[k], DP_ERR_INVALID, "dp_mle_linear_combination: null operand");
    LinArg a; memset(&a, 0, sizeof a); a.n = n;
    u64 len = mles[0]->len;
    for (u32 k = 0; k < n; k++) {
        DP_CHECK(mles[k]->is_ext && mles[k]->len == len, DP_ERR_INVALID, "dp_mle_linear_combination: operands must be Ext MLEs of equal length");
        a.m[k] = (const gle *)mles[k]->data; a.coef[k] = e_from_host(coefs + 2 * k);
    }
    MlePtr r;
    if (int e = dp_mle_alloc(len, true, r)) return e;
    DP_CUDA(dp_launch(k_lincomb, dp_grid_for(len, 256, 8), 256, 0, dp_ctx().stream, a, len, (gle *)r->data));
    *out = r.release();
    return DP_OK;
}

}  // extern "C"
