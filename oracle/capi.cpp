// ORACLE -- TEST INFRASTRUCTURE ONLY.  C entry points (ctypes) over the CPU restatement.
// Loaded only by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg.
#include "sumcheck.hpp"
#include <thread>
#include <string>

using namespace dpo;

static std::shared_ptr<MLE> mk_mle(const u64 *data, u64 len, int is_ext) {
    auto m = std::make_shared<MLE>();
    m->is_ext = is_ext != 0; m->num_vars = ceil_log2(len);
    if (is_ext) { m->ext.resize(len); for (u64 i = 0; i < len; i++) m->ext[i] = E(f_from_u64(data[2 * i]), f_from_u64(data[2 * i + 1])); }
    else { m->base.resize(len); for (u64 i = 0; i < len; i++) m->base[i] = f_from_u64(data[i]); }
    return m;
}
static std::vector<E> mk_point(const u64 *p, u32 k) { std::vector<E> v(k); for (u32 i = 0; i < k; i++) v[i] = E(f_from_u64(p[2 * i]), f_from_u64(p[2 * i + 1])); return v; }
static void put_e(u64 *out, size_t i, E e) { out[2 * i] = e.c0; out[2 * i + 1] = e.c1; }
static thread_local std::string g_err;

extern "C" {

const char *dpo_last_error() { return g_err.c_str(); }
int dpo_num_threads() { return (int)std::thread::hardware_concurrency(); }   // hardware threads of the host
int dpo_get_threads() { return (int)dpo_threads(); }                           // threads a par_for may use right now
void dpo_set_threads(int n) { dpo_threads_var().store(n > 0 ? (unsigned)n : 1u); }

// ---- field (vectorised, for the device-arithmetic tests) ----
void dpo_f_binop(int op, const u64 *a, const u64 *b, u64 n, u64 *out) {
    for (u64 i = 0; i < n; i++) {
        u64 x = f_from_u64(a[i]), y = f_from_u64(b[i]);
        out[i] = op == 0 ? f_add(x, y) : op == 1 ? f_sub(x, y) : f_mul(x, y);
    }
}
void dpo_e_binop(int op, const u64 *a, const u64 *b, u64 n, u64 *out) {
    for (u64 i = 0; i < n; i++) {
        E x(f_from_u64(a[2 * i]), f_from_u64(a[2 * i + 1])), y(f_from_u64(b[2 * i]), f_from_u64(b[2 * i + 1]));
        put_e(out, i, op == 0 ? e_add(x, y) : op == 1 ? e_sub(x, y) : e_mul(x, y));
    }
}
void dpo_e_inv(const u64 *a, u64 n, u64 *out) { for (u64 i = 0; i < n; i++) put_e(out, i, e_inv(E(a[2 * i], a[2 * i + 1]))); }
void dpo_splitmix_f(u64 seed, u64 n, u64 *out) { SplitMix64 g(seed); for (u64 i = 0; i < n; i++) out[i] = g.next_f(); }

// ---- MLE ----
int dpo_fix_high(const u64 *evals, u64 len, int is_ext, const u64 *point, u32 k, u64 *out) {
    try { MLE r = mle_fix_high_variables(*mk_mle(evals, len, is_ext), mk_point(point, k)); for (size_t i = 0; i < r.len(); i++) put_e(out, i, r.get(i)); return 0; }
    catch (std::exception &e) { g_err = e.what(); return 1; }
}
int dpo_fix_low(const u64 *evals, u64 len, int is_ext, const u64 *point, u32 k, u64 *out) {
    try { MLE r = mle_fix_variables(*mk_mle(evals, len, is_ext), mk_point(point, k)); for (size_t i = 0; i < r.len(); i++) put_e(out, i, r.get(i)); return 0; }
    catch (std::exception &e) { g_err = e.what(); return 1; }
}
int dpo_evaluate(const u64 *evals, u64 len, int is_ext, const u64 *point, u32 nv, u64 *out) {
    try { put_e(out, 0, mle_evaluate(*mk_mle(evals, len, is_ext), mk_point(point, nv))); return 0; }
    catch (std::exception &e) { g_err = e.what(); return 1; }
}
void dpo_build_eq(const u64 *point, u32 nv, u64 *out) { auto v = build_eq_x_r_vec(mk_point(point, nv)); for (size_t i = 0; i < v.size(); i++) put_e(out, i, v[i]); }
void dpo_eq_eval(const u64 *x, const u64 *y, u32 n, u64 *out) { put_e(out, 0, eq_eval(mk_point(x, n), mk_point(y, n))); }

// ---- hasher selection + BLAKE3 (include/dp_blake3.h) ----
void dpo_set_hash_mode(int m) { hash_mode_var().store(m == 1 ? 1 : 0); }      // 0 Poseidon2 + BasicTranscript, 1 BLAKE3 + BlakeTranscript
int dpo_get_hash_mode() { return hash_mode_var().load(); }
// hash `n` bytes fed in pieces of `piece` bytes (0 = all at once); when `mid` > 0 a finalize is taken after `mid` bytes first (the
// running hasher must not be disturbed by it); `out_len` bytes of extendable output
void dpo_blake3(const uint8_t *data, u64 n, u64 piece, u64 mid, uint8_t *out, u64 out_len) {
    dpb3::Hasher h; u64 off = 0; uint8_t tmp[64];
    if (piece == 0) piece = n ? n : 1;
    while (off < n) { u64 take = std::min<u64>(piece, n - off); if (mid > off && mid < off + take) take = mid - off; h.update(data + off, take); off += take; if (off == mid) h.finalize(tmp, 64); }
    h.finalize(out, out_len);
}
void dpo_hash_bases(const u64 *in, u64 n, u64 *out) { Digest d = hash_or_noop(in, n); memcpy(out, d.v, 32); }
void dpo_hash_two_digests(const u64 *a, const u64 *b, u64 *out) { Digest x, y; memcpy(x.v, a, 32); memcpy(y.v, b, 32); Digest d = compress(x, y); memcpy(out, d.v, 32); }

// ---- Poseidon2 / challenger / transcript ----
void dpo_poseidon2_permute(u64 *state) { poseidon2_permute(state); }
void dpo_hash_or_noop(const u64 *in, u64 n, u64 *out) { Digest d = hash_or_noop(in, n); memcpy(out, d.v, 32); }
void dpo_compress(const u64 *x, const u64 *y, u64 *out) { Digest a, b; memcpy(a.v, x, 32); memcpy(b.v, y, 32); Digest d = compress(a, b); memcpy(out, d.v, 32); }
void *dpo_transcript_new(const char *label) { return new Transcript(label); }
void dpo_transcript_free(void *t) { delete (Transcript *)t; }
void dpo_transcript_append_f(void *t, const u64 *f, u64 n) { ((Transcript *)t)->append_field_elements(f, n); }
void dpo_transcript_append_msg(void *t, const uint8_t *m, u64 n) { ((Transcript *)t)->append_message(m, n); }
void dpo_transcript_append_e(void *t, const u64 *e, u64 n) { for (u64 i = 0; i < n; i++) ((Transcript *)t)->append_field_element_ext(E(e[2 * i], e[2 * i + 1])); }
void dpo_transcript_challenge(void *t, const char *label, u64 *out) { put_e(out, 0, ((Transcript *)t)->get_and_append_challenge(label)); }
void dpo_transcript_read_challenge(void *t, u64 *out) { put_e(out, 0, ((Transcript *)t)->read_challenge()); }

// ---- sumcheck ----
static VirtualPolynomial mk_vp(u32 n_mles, const u64 *const *data, const u64 *lens, const int *is_ext, u32 n_products,
                               const u64 *coefs, const u32 *deg, const u32 *idx, u32 max_nv) {
    VirtualPolynomial vp(max_nv);
    std::vector<std::shared_ptr<MLE>> ms;
    for (u32 i = 0; i < n_mles; i++) ms.push_back(mk_mle(data[i], lens[i], is_ext[i]));
    // keep the caller's MLE numbering: register every MLE in order first
    for (auto &m : ms) vp.add_mle(m);
    size_t o = 0;
    for (u32 p = 0; p < n_products; p++) {
        std::vector<std::shared_ptr<MLE>> l;
        for (u32 j = 0; j < deg[p]; j++) l.push_back(ms[idx[o + j]]);
        o += deg[p];
        vp.add_mle_list(l, E(f_from_u64(coefs[2 * p]), f_from_u64(coefs[2 * p + 1])));
    }
    return vp;
}

// prove_parallel with BasicTranscript::new(label).  out_point: nv x E; out_msgs: nv x (max_deg+1) x E;
// out_final: n_mles x E.  Returns max_degree via *out_max_deg.
int dpo_sumcheck_prove(u32 n_mles, const u64 *const *data, const u64 *lens, const int *is_ext, u32 n_products, const u64 *coefs,
                       const u32 *deg, const u32 *idx, u32 max_nv, const char *label, u64 *out_point, u64 *out_msgs, u64 *out_final,
                       u32 *out_max_deg) {
    try {
        VirtualPolynomial vp = mk_vp(n_mles, data, lens, is_ext, n_products, coefs, deg, idx, max_nv);
        Transcript t(label);
        auto res = sumcheck_prove(vp, t);
        *out_max_deg = (u32)vp.max_degree;
        for (size_t i = 0; i < res.first.point.size(); i++) put_e(out_point, i, res.first.point[i]);
        size_t k = 0;
        for (auto &m : res.first.proofs) for (E e : m) put_e(out_msgs, k++, e);
        for (size_t i = 0; i < res.second.size(); i++) put_e(out_final, i, res.second[i]);
        return 0;
    } catch (std::exception &e) { g_err = e.what(); return 1; }
}

// Round-by-round with INJECTED challenges (challenges: max_nv x E; the i-th is used after round i).
int dpo_sumcheck_rounds_fixed(u32 n_mles, const u64 *const *data, const u64 *lens, const int *is_ext, u32 n_products, const u64 *coefs,
                              const u32 *deg, const u32 *idx, u32 max_nv, const u64 *challenges, u64 *out_msgs, u64 *out_final) {
    try {
        VirtualPolynomial vp = mk_vp(n_mles, data, lens, is_ext, n_products, coefs, deg, idx, max_nv);
        IOPProverState st(vp);
        size_t k = 0;
        for (u32 i = 0; i < max_nv; i++) {
            E c = i ? E(challenges[2 * (i - 1)], challenges[2 * (i - 1) + 1]) : E();
            auto msg = st.prove_round(i ? &c : nullptr);
            for (E e : msg) put_e(out_msgs, k++, e);
        }
        st.finish(E(challenges[2 * (max_nv - 1)], challenges[2 * (max_nv - 1) + 1]));
        auto fin = st.final_evaluations();
        for (size_t i = 0; i < fin.size(); i++) put_e(out_final, i, fin[i]);
        return 0;
    } catch (std::exception &e) { g_err = e.what(); return 1; }
}

// verify a proof produced with BasicTranscript::new(label); returns 0 and the subclaim on success
int dpo_sumcheck_verify(const u64 *claimed_sum, u32 nv, u32 max_deg, const u64 *msgs, const char *label, u64 *out_point, u64 *out_expected) {
    try {
        IOPProof pr;
        for (u32 i = 0; i < nv; i++) { std::vector<E> m; for (u32 t = 0; t <= max_deg; t++) { size_t k = (size_t)i * (max_deg + 1) + t; m.push_back(E(msgs[2 * k], msgs[2 * k + 1])); } pr.proofs.push_back(m); }
        Transcript t(label);
        auto sc = sumcheck_verify(E(claimed_sum[0], claimed_sum[1]), pr, nv, max_deg, t);
        for (size_t i = 0; i < sc.point.size(); i++) put_e(out_point, i, sc.point[i]);
        put_e(out_expected, 0, sc.expected_evaluation);
        return 0;
    } catch (std::exception &e) { g_err = e.what(); return 1; }
}

}  // extern "C"

// ---- Basefold (oracle/basefold.hpp) ----
#include "basefold.hpp"
static FVec mk_fvec(const u64 *data, u64 len, int is_ext) {
    FVec v; v.is_ext = is_ext != 0;
    if (is_ext) { v.e.resize(len); for (u64 i = 0; i < len; i++) v.e[i] = E(f_from_u64(data[2 * i]), f_from_u64(data[2 * i + 1])); }
    else { v.b.resize(len); for (u64 i = 0; i < len; i++) v.b[i] = f_from_u64(data[i]); }
    return v;
}
static void put_fvec(const FVec &v, u64 *out) { if (v.is_ext) for (size_t i = 0; i < v.e.size(); i++) put_e(out, i, v.e[i]); else for (size_t i = 0; i < v.b.size(); i++) out[i] = v.b[i]; }

extern "C" {

// RS encode of an already-prepared coefficient vector (rs.rs encode_internal): out has 2*len elements
void dpo_rs_encode(const u64 *coeffs, u64 len, int is_ext, u32 full_log, u64 *out) { put_fvec(rs_encode(mk_fvec(coeffs, len, is_ext), full_log), out); }
void dpo_interpolate_hc(const u64 *evals, u64 len, int is_ext, u64 *out) {
    FVec v = mk_fvec(evals, len, is_ext);
    if (is_ext) interpolate_hc<E>(v.e, e_sub); else interpolate_hc<u64>(v.b, f_sub);
    put_fvec(v, out);
}
void dpo_merkle_root(const u64 *leaves, u64 len, int is_ext, u64 *out_root) { auto t = merkelize(mk_fvec(leaves, len, is_ext)); memcpy(out_root, t.back()[0].v, 32); }
void dpo_folding_coeffs(u32 full_log, u32 level, u64 index, u64 *x0, u64 *w) { folding_coeffs(full_log, level, index, *x0, *w); }
void dpo_fri_fold(const u64 *vals, u64 len, u32 full_log, const u64 *r, u64 *out) {
    std::vector<E> v(len); for (u64 i = 0; i < len; i++) v[i] = E(vals[2 * i], vals[2 * i + 1]);
    auto o = fri_fold(v, full_log, E(r[0], r[1]));
    for (size_t i = 0; i < o.size(); i++) put_e(out, i, o[i]);
}
// commit: root + (optionally) codeword and bh_evals, all bit-reversed as stored by the reference
int dpo_pcs_commit(const u64 *evals, u64 len, int is_ext, u32 full_log, u64 *out_root, u64 *out_codeword, u64 *out_bh) {
    try {
        Commitment c = basefold_commit(mk_fvec(evals, len, is_ext), full_log);
        memcpy(out_root, c.root().v, 32);
        if (out_codeword) put_fvec(c.codeword_tree.leaves, out_codeword);
        if (out_bh) put_fvec(c.bh_evals, out_bh);
        return 0;
    } catch (std::exception &e) { g_err = e.what(); return 1; }
}
int dpo_pcs_open(const u64 *evals, u64 len, int is_ext, u32 full_log, const u64 *point, const char *label, u64 *out, u64 cap, u64 *out_len) {
    try {
        Commitment c = basefold_commit(mk_fvec(evals, len, is_ext), full_log);
        Transcript t(label);
        BasefoldProof p = basefold_open(full_log, c, mk_point(point, (u32)c.num_vars), t);
        std::vector<u64> f = flatten_proof(p);
        *out_len = f.size();
        if (f.size() > cap) { g_err = "dpo_pcs_open: output buffer too small"; return 2; }
        memcpy(out, f.data(), 8 * f.size());
        return 0;
    } catch (std::exception &e) { g_err = e.what(); return 1; }
}
// batch_open with Evaluation::new(i, i, poly_i(point_i)); points are concatenated (poly i has nv_i elements)
int dpo_pcs_batch_open(u32 n, const u64 *const *data, const u64 *lens, const int *is_ext, u32 full_log, const u64 *points, const char *label,
                       u64 *out, u64 cap, u64 *out_len) {
    try {
        std::vector<FVec> polys; std::vector<Commitment> comms; std::vector<std::vector<E>> pts; std::vector<Evaluation> evals;
        size_t o = 0;
        for (u32 i = 0; i < n; i++) {
            polys.push_back(mk_fvec(data[i], lens[i], is_ext[i]));
            comms.push_back(basefold_commit(polys.back(), full_log));
            u32 nv = (u32)ceil_log2(lens[i]);
            pts.push_back(mk_point(points + 2 * o, nv)); o += nv;
            MLE m; m.is_ext = polys.back().is_ext; m.num_vars = nv; m.base = polys.back().b; m.ext = polys.back().e;
            evals.push_back({i, i, mle_evaluate(m, pts.back())});
        }
        std::vector<const Commitment *> cp; for (auto &c : comms) cp.push_back(&c);
        Transcript t(label);
        BasefoldProof p = basefold_batch_open(full_log, polys, cp, pts, evals, t);
        std::vector<u64> f = flatten_proof(p);
        *out_len = f.size();
        if (f.size() > cap) { g_err = "dpo_pcs_batch_open: output buffer too small"; return 2; }
        memcpy(out, f.data(), 8 * f.size());
        return 0;
    } catch (std::exception &e) { g_err = e.what(); return 1; }
}

}  // extern "C"

// ---- zkml MLP prover (oracle/zkml.hpp) ----
#include "zkml.hpp"
#include <chrono>
extern "C" {
// Synthetic MLP (SURVEY.md 8d Cfg 2): context generation (weight commits) + Prover::prove.  Returns the flat proof.
// out_ms[0] = context (setup) time, out_ms[1] = prove time.
int dpo_zkml_prove(u32 n_layers, u32 width, u64 seed_model, u64 seed_input, const char *label, u64 *out, u64 cap, u64 *out_len, double *out_ms) {
    try {
        Model m = synthetic_mlp(n_layers, width, seed_model);
        std::vector<Element> input = synthetic_input(width, seed_input);
        auto t0 = std::chrono::steady_clock::now();
        ZkContext ctx = zk_context(m);
        auto t1 = std::chrono::steady_clock::now();
        Transcript t(label);
        ModelProof p = zk_prove(ctx, input, t);
        auto t2 = std::chrono::steady_clock::now();
        if (out_ms) { out_ms[0] = std::chrono::duration<double, std::milli>(t1 - t0).count(); out_ms[1] = std::chrono::duration<double, std::milli>(t2 - t1).count(); }
        std::vector<u64> f = flatten_model_proof(p, m.nodes.size());
        *out_len = f.size();
        if (out) { if (f.size() > cap) { g_err = "dpo_zkml_prove: output buffer too small"; return 2; } memcpy(out, f.data(), 8 * f.size()); }
        return 0;
    } catch (std::exception &e) { g_err = e.what(); return 1; }
}
// model / input generators exposed so the product's host side gets the SAME synthetic tensors without touching oracle code paths
void dpo_synthetic_mlp(u32 n_layers, u32 width, u64 seed, int64_t *weights /* n_layers*width*width */, int64_t *bias /* n_layers*width */, int64_t *rq /* n_layers*4 */) {
    Model m = synthetic_mlp(n_layers, width, seed);
    size_t l = 0;
    for (auto &n : m.nodes) {
        if (n.kind == OP_DENSE) { memcpy(weights + l * width * width, n.weights.data(), 8 * n.weights.size()); memcpy(bias + l * width, n.bias.data(), 8 * n.bias.size()); }
        if (n.kind == OP_REQUANT) { rq[4 * l] = n.rq.right_shift; rq[4 * l + 1] = n.rq.fp_scale; rq[4 * l + 2] = n.rq.fixed_point_multiplier; rq[4 * l + 3] = n.rq.intermediate_bit_size; l++; }
    }
}
void dpo_synthetic_input(u32 width, u64 seed, int64_t *out) { auto v = synthetic_input(width, seed); memcpy(out, v.data(), 8 * v.size()); }
// LogUpCircuit::new_lookup_circuit (mult == NULL) / new_table_circuit: every layer, bottom to top.  Layer k (k = 0 .. log2(len) - 1)
// has len >> k fractions; `out` holds, layer after layer, its numerators and then its denominators ([c0, c1] each).  The numerators
// of an initial lookup layer (all -1, never stored) are written as zeros.
void dpo_logup_circuit(const u64 *const *cols, u32 n_cols, u64 len, const u64 *mult, const u64 c[2], const u64 gamma[2], u64 *out) {
    std::vector<std::vector<u64>> cv(n_cols);
    std::vector<const std::vector<u64> *> cp;
    for (u32 k = 0; k < n_cols; k++) { cv[k].assign(cols[k], cols[k] + len); cp.push_back(&cv[k]); }
    std::vector<u64> mv; if (mult) mv.assign(mult, mult + len);
    LogUpCircuit C = logup_circuit(cp, mult ? &mv : nullptr, E(f_from_u64(c[0]), f_from_u64(c[1])), E(f_from_u64(gamma[0]), f_from_u64(gamma[1])));
    size_t o = 0;
    for (const LogUpLayer &l : C.layers) {
        for (size_t i = 0; i < l.den.size(); i++) put_e(out, o + i, l.has_num ? l.num[i] : E());
        o += l.den.size();
        for (size_t i = 0; i < l.den.size(); i++) put_e(out, o + i, l.den[i]);
        o += l.den.size();
    }
}
}

// prove_batch_polys: the caller passes the FULL MLEs; they are split into T contiguous slices here
extern "C" int dpo_sumcheck_prove_batch(u32 T, u32 n_mles, const u64 *const *data, const u64 *lens, const int *is_ext, u32 n_products, const u64 *coefs,
                                         const u32 *deg, const u32 *idx, u32 max_nv, const char *label, u64 *out_point, u64 *out_msgs, u64 *out_final) {
    try {
        u32 logT = (u32)ceil_log2(T);
        std::vector<VirtualPolynomial> polys;
        for (u32 t = 0; t < T; t++) {
            std::vector<const u64 *> d(n_mles); std::vector<u64> l(n_mles);
            for (u32 i = 0; i < n_mles; i++) { l[i] = lens[i] / T; d[i] = data[i] + (size_t)t * l[i] * (is_ext[i] ? 2 : 1); }
            polys.push_back(mk_vp(n_mles, d.data(), l.data(), is_ext, n_products, coefs, deg, idx, max_nv - logT));
        }
        Transcript t(label);
        auto res = sumcheck_prove_batch_polys(polys, t);
        for (size_t i = 0; i < res.first.point.size(); i++) put_e(out_point, i, res.first.point[i]);
        size_t k = 0;
        for (auto &m : res.first.proofs) for (E e : m) put_e(out_msgs, k++, e);
        for (size_t i = 0; i < res.second.size(); i++) put_e(out_final, i, res.second[i]);
        return 0;
    } catch (std::exception &e) { g_err = e.what(); return 1; }
}

// ---- FFT convolution layer (conv.hpp): inference + isolated layer proof on a synthetic layer ----
extern "C" {
// synthetic padded layer: filter [kw][kx][real_nw][real_nw], bias [kw], input [kx][n_x][n_x]  (all int64)
void dpo_synthetic_conv(u32 kw, u32 kx, u32 n_x, u32 real_nw, u32 kw_u, u32 k_u, u32 kx_u, u32 n_x_u, u64 seed_model, u64 seed_input,
                        int64_t *filter, int64_t *bias, int64_t *input) {
    ConvLayer f = synthetic_conv(kw, kx, n_x, real_nw, kw_u, k_u, n_x_u, seed_model);
    memcpy(filter, f.filter.data(), 8 * f.filter.size()); memcpy(bias, f.bias.data(), 8 * f.bias.size());
    auto x = synthetic_conv_input(kx, n_x, kx_u, n_x_u, seed_input); memcpy(input, x.data(), 8 * x.size());
}
// Convolution::op: out_after_bias / out_cleared are [kw][n_x][n_x]
int dpo_conv_op(u32 kw, u32 kx, u32 n_x, u32 real_nw, const int64_t *filter, const int64_t *bias, const u32 *unpadded_out, const int64_t *input,
                int64_t *out_after_bias, int64_t *out_cleared) {
    try {
        ConvLayer f; f.kw = kw; f.kx = kx; f.nw = n_x; f.real_nw = real_nw; f.filter.assign(filter, filter + (size_t)kw * kx * real_nw * real_nw); f.bias.assign(bias, bias + kw);
        for (int i = 0; i < 3; i++) f.unpadded_out[i] = unpadded_out[i];
        std::vector<Element> x(input, input + (size_t)kx * n_x * n_x); ConvData cd;
        auto cleared = conv_op(f, x, n_x, cd);
        if (out_after_bias) memcpy(out_after_bias, cd.output_as_element.data(), 8 * cd.output_as_element.size());
        if (out_cleared) memcpy(out_cleared, cleared.data(), 8 * cleared.size());
        return 0;
    } catch (std::exception &e) { g_err = e.what(); return 1; }
}
// the layer proof in isolation: output claim = (point drawn from the transcript, MLE(cleared output)(point)) as Prover::prove
// does for the model output (iop/prover.rs:423-436); flat layout: conv.hpp flatten_conv_proof
int dpo_conv_prove(u32 kw, u32 kx, u32 n_x, u32 real_nw, const int64_t *filter, const int64_t *bias, const u32 *unpadded_out, const int64_t *input,
                   const char *label, u64 *out, u64 cap, u64 *out_len) {
    try {
        ConvLayer f; f.kw = kw; f.kx = kx; f.nw = n_x; f.real_nw = real_nw; f.filter.assign(filter, filter + (size_t)kw * kx * real_nw * real_nw); f.bias.assign(bias, bias + kw);
        for (int i = 0; i < 3; i++) f.unpadded_out[i] = unpadded_out[i];
        std::vector<Element> x(input, input + (size_t)kx * n_x * n_x); ConvData cd;
        auto cleared = conv_op(f, x, n_x, cd);
        Transcript t(label);
        Claim c; c.point = t.sample_vec(ceil_log2(cleared.size()));
        auto ce = elems_to_ext(cleared); c.eval = mle_evaluate(*ext_mle(ce.data(), ce.size()), c.point);
        ConvProof pr; Claim in_claim = prove_convolution_step(f, t, c, cd, pr);
        auto xe = elems_to_ext(x);
        if (!(mle_evaluate(*ext_mle(xe.data(), xe.size()), in_claim.point) == in_claim.eval)) throw std::runtime_error("conv: returned claim is not an evaluation of the input tensor");
        std::vector<u64> fl = flatten_conv_proof(pr, in_claim);
        *out_len = fl.size();
        if (out) { if (fl.size() > cap) { g_err = "dpo_conv_prove: output buffer too small"; return 2; } memcpy(out, fl.data(), 8 * fl.size()); }
        return 0;
    } catch (std::exception &e) { g_err = e.what(); return 1; }
}
// tensor.rs:261 fft on [rows][n] Ext values in place (flag 0: FFT, 1: iFFT)
void dpo_fft_ext(u64 *data, u64 rows, u64 n, int inverse) {
    for (u64 r = 0; r < rows; r++) { std::vector<E> v(n); for (u64 i = 0; i < n; i++) v[i] = E(data[2 * (r * n + i)], data[2 * (r * n + i) + 1]); fft_ext(v, inverse != 0); for (u64 i = 0; i < n; i++) { data[2 * (r * n + i)] = v[i].c0; data[2 * (r * n + i) + 1] = v[i].c1; } }
}
}

// ---- synthetic CNN (conv -> requant -> relu -> maxpool x2, then 3 dense layers): full Prover::prove ----
extern "C" {
int dpo_cnn_prove(int small, u64 seed_model, u64 seed_input, const char *label, u64 *out, u64 cap, u64 *out_len, double *out_ms) {
    try {
        Model m = synthetic_cnn(small, seed_model);
        std::vector<Element> input = synthetic_cnn_input(small, seed_input);
        auto t0 = std::chrono::steady_clock::now();
        ZkContext ctx = zk_context(m);
        auto t1 = std::chrono::steady_clock::now();
        Transcript t(label);
        ModelProof p = zk_prove(ctx, input, t);
        auto t2 = std::chrono::steady_clock::now();
        if (out_ms) { out_ms[0] = std::chrono::duration<double, std::milli>(t1 - t0).count(); out_ms[1] = std::chrono::duration<double, std::milli>(t2 - t1).count(); }
        std::vector<u64> f = flatten_model_proof(p, m.nodes.size());
        *out_len = f.size();
        if (out) { if (f.size() > cap) { g_err = "dpo_cnn_prove: output buffer too small"; return 2; } memcpy(out, f.data(), 8 * f.size()); }
        return 0;
    } catch (std::exception &e) { g_err = e.what(); return 1; }
}
// the model description for the product's host side (same synthetic tensors, no oracle code on the product path):
// per node: kind, then 8 shape words; weights/bias/filter data are appended to `data` in node order
int dpo_synthetic_cnn(int small, u64 seed_model, u64 seed_input, int64_t *desc, u64 desc_cap, u64 *desc_len, int64_t *data, u64 data_cap, u64 *data_len, int64_t *input, u64 *input_len) {
    try {
        Model m = synthetic_cnn(small, seed_model);
        std::vector<int64_t> d, w;
        for (auto &n : m.nodes) {
            d.push_back(n.kind);
            if (n.kind == OP_DENSE) { d.insert(d.end(), {(int64_t)n.nrows, (int64_t)n.ncols, 0, 0, 0, 0, 0, 0}); w.insert(w.end(), n.weights.begin(), n.weights.end()); w.insert(w.end(), n.bias.begin(), n.bias.end()); }
            else if (n.kind == OP_REQUANT) d.insert(d.end(), {(int64_t)n.rq.right_shift, (int64_t)n.rq.fp_scale, (int64_t)n.rq.fixed_point_multiplier, (int64_t)n.rq.intermediate_bit_size, 0, 0, 0, 0});
            else if (n.kind == OP_CONV) { auto &c = *n.conv; d.insert(d.end(), {(int64_t)c.kw, (int64_t)c.kx, (int64_t)c.nw, (int64_t)c.real_nw, (int64_t)c.unpadded_out[0], (int64_t)c.unpadded_out[1], (int64_t)c.unpadded_out[2], 0}); w.insert(w.end(), c.filter.begin(), c.filter.end()); w.insert(w.end(), c.bias.begin(), c.bias.end()); }
            else if (n.kind == OP_POOL) d.insert(d.end(), {(int64_t)n.pool_c, (int64_t)n.pool_h, (int64_t)n.pool_w, 0, 0, 0, 0, 0});
            else d.insert(d.end(), {0, 0, 0, 0, 0, 0, 0, 0});
        }
        std::vector<Element> in = synthetic_cnn_input(small, seed_input);
        *desc_len = d.size(); *data_len = w.size(); *input_len = in.size();
        if (desc && d.size() <= desc_cap) memcpy(desc, d.data(), 8 * d.size());
        if (data && w.size() <= data_cap) memcpy(data, w.data(), 8 * w.size());
        if (input) memcpy(input, in.data(), 8 * in.size());
        return 0;
    } catch (std::exception &e) { g_err = e.what(); return 1; }
}
}

// Prover::prove of a model given as the layer descriptor the product's model builder takes (deep-prove_b200/models.py):
// 9 int64 per node {kind, 8 shape words}, weights in node order.
extern "C" int dpo_model_prove(const int64_t *desc, u32 n_nodes, const int64_t *data, const int64_t *input, u64 input_len, const char *label,
                               u64 *out, u64 cap, u64 *out_len, double *out_ms) {
    try {
        Model m; m.input_len = input_len; const int64_t *w = data;
        for (u32 i = 0; i < n_nodes; i++) {
            const int64_t *d = desc + 9 * (size_t)i; Node n;
            switch (d[0]) {
            case 0: n.kind = OP_DENSE; n.nrows = d[1]; n.ncols = d[2]; n.weights.assign(w, w + n.nrows * n.ncols); w += n.nrows * n.ncols; n.bias.assign(w, w + n.nrows); w += n.nrows; break;
            case 1: n.kind = OP_REQUANT; n.rq.right_shift = d[1]; n.rq.fp_scale = d[2]; n.rq.fixed_point_multiplier = d[3]; n.rq.intermediate_bit_size = d[4]; break;
            case 2: n.kind = OP_RELU; break;
            case 3: { n.kind = OP_CONV; auto c = std::make_shared<ConvLayer>(); c->kw = d[1]; c->kx = d[2]; c->nw = d[3]; c->real_nw = d[4]; for (int k = 0; k < 3; k++) c->unpadded_out[k] = d[5 + k];
                      size_t fl = c->kw * c->kx * c->real_nw * c->real_nw; c->filter.assign(w, w + fl); w += fl; c->bias.assign(w, w + c->kw); w += c->kw; n.conv = c; break; }
            case 4: n.kind = OP_POOL; n.pool_c = d[1]; n.pool_h = d[2]; n.pool_w = d[3]; break;
            case 5: n.kind = OP_MATMUL; n.mm_r = d[1]; n.mm_k = d[2]; n.mm_c = d[3]; n.mm_t = d[4] != 0; n.mm_bias = d[5] != 0; n.weights.assign(w, w + n.mm_k * n.mm_c); w += n.mm_k * n.mm_c; if (n.mm_bias) { n.bias.assign(w, w + n.mm_c); w += n.mm_c; } break;
            default: throw std::runtime_error("dpo_model_prove: unknown node kind");
            }
            m.nodes.push_back(n);
        }
        std::vector<Element> in(input, input + input_len);
        auto t0 = std::chrono::steady_clock::now();
        ZkContext ctx = zk_context(m);
        auto t1 = std::chrono::steady_clock::now();
        Transcript t(label);
        ModelProof p = zk_prove(ctx, in, t);
        auto t2 = std::chrono::steady_clock::now();
        if (out_ms) { out_ms[0] = std::chrono::duration<double, std::milli>(t1 - t0).count(); out_ms[1] = std::chrono::duration<double, std::milli>(t2 - t1).count(); }
        std::vector<u64> f = flatten_model_proof(p, m.nodes.size());
        if (out_len) *out_len = f.size();
        if (out) { if (f.size() > cap) { g_err = "dpo_model_prove: output buffer too small"; return 2; } memcpy(out, f.data(), 8 * f.size()); }
        return 0;
    } catch (std::exception &e) { g_err = e.what(); return 1; }
}

// ---- Basefold verifier (verify.hpp) on a flat proof image (from this library or from the device) ----
#include "verify.hpp"
extern "C" {
// Basefold::verify: 0 = accepted; 1 = rejected (dpo_last_error says why)
int dpo_pcs_verify(const u64 *flat, u64 n, const u64 *root, u32 num_vars, int is_base, u32 full_log, const u64 *point, const u64 *eval, const char *label) {
    try {
        BasefoldProof pr = unflatten_proof(flat, n);
        PureCommitment c; for (int i = 0; i < 4; i++) c.root.v[i] = root[i]; c.num_vars = num_vars; c.is_base = is_base != 0;
        Transcript t(label);
        basefold_verify(full_log, c, mk_point(point, num_vars), E(eval[0], eval[1]), pr, t);
        return 0;
    } catch (std::exception &e) { g_err = e.what(); return 1; }
}
// Basefold::batch_verify with Evaluation::new(i, i, evals[i]); points concatenated (poly i has num_vars[i] elements)
int dpo_pcs_batch_verify(const u64 *flat, u64 n, u32 n_polys, const u64 *roots, const u32 *num_vars, const int *is_base, u32 full_log, const u64 *points, const u64 *evals, const char *label) {
    try {
        BasefoldProof pr = unflatten_proof(flat, n);
        std::vector<PureCommitment> comms; std::vector<std::vector<E>> pts; std::vector<Evaluation> ev; size_t o = 0;
        for (u32 i = 0; i < n_polys; i++) {
            PureCommitment c; for (int k = 0; k < 4; k++) c.root.v[k] = roots[4 * i + k]; c.num_vars = num_vars[i]; c.is_base = is_base[i] != 0; comms.push_back(c);
            pts.push_back(mk_point(points + 2 * o, num_vars[i])); o += num_vars[i];
            ev.push_back({i, i, E(evals[2 * i], evals[2 * i + 1])});
        }
        Transcript t(label);
        basefold_batch_verify(full_log, comms, pts, ev, pr, t);
        return 0;
    } catch (std::exception &e) { g_err = e.what(); return 1; }
}
}

// ---- model verifier (zk_verify.hpp): prove on the checker, then verify on a FRESH transcript as deep-prove's verifier would ----
#include "zk_verify.hpp"
extern "C" int dpo_zkml_prove_verify(u32 n_layers, u32 width, u64 seed_model, u64 seed_input, const char *label, int tamper) {
    try {
        Model m = synthetic_mlp(n_layers, width, seed_model);
        std::vector<Element> input = synthetic_input(width, seed_input);
        ZkContext ctx = zk_context(m);
        Transcript tp(label);
        ModelProof p = zk_prove(ctx, input, tp);
        std::vector<Element> output = zk_run(m, input).back();
        if (tamper == 1) output[0] += 1;                                          // wrong public output
        if (tamper == 2) p.dense.begin()->second.individual_claims[1].c0 ^= 1;    // a forged claim
        if (tamper == 3) p.table_proofs[0].lookup.circuit_outputs[0][0].c0 ^= 1;  // a forged lookup fraction
        Transcript tv(label);
        zk_verify(ctx, input, output, p, tv);
        return 0;
    } catch (std::exception &e) { g_err = e.what(); return 1; }
}

// prove + verify for a model given as a layer descriptor (same format as dpo_model_prove)
extern "C" int dpo_model_prove_verify(const int64_t *desc, u32 n_nodes, const int64_t *data, const int64_t *input, u64 input_len, const char *label, int tamper) {
    try {
        Model m; m.input_len = input_len; const int64_t *w = data;
        for (u32 i = 0; i < n_nodes; i++) {
            const int64_t *d = desc + 9 * (size_t)i; Node n;
            switch (d[0]) {
            case 0: n.kind = OP_DENSE; n.nrows = d[1]; n.ncols = d[2]; n.weights.assign(w, w + n.nrows * n.ncols); w += n.nrows * n.ncols; n.bias.assign(w, w + n.nrows); w += n.nrows; break;
            case 1: n.kind = OP_REQUANT; n.rq.right_shift = d[1]; n.rq.fp_scale = d[2]; n.rq.fixed_point_multiplier = d[3]; n.rq.intermediate_bit_size = d[4]; break;
            case 2: n.kind = OP_RELU; break;
            case 3: { n.kind = OP_CONV; auto c = std::make_shared<ConvLayer>(); c->kw = d[1]; c->kx = d[2]; c->nw = d[3]; c->real_nw = d[4]; for (int k = 0; k < 3; k++) c->unpadded_out[k] = d[5 + k];
                      size_t fl = c->kw * c->kx * c->real_nw * c->real_nw; c->filter.assign(w, w + fl); w += fl; c->bias.assign(w, w + c->kw); w += c->kw; n.conv = c; break; }
            case 4: n.kind = OP_POOL; n.pool_c = d[1]; n.pool_h = d[2]; n.pool_w = d[3]; break;
            case 5: n.kind = OP_MATMUL; n.mm_r = d[1]; n.mm_k = d[2]; n.mm_c = d[3]; n.mm_t = d[4] != 0; n.mm_bias = d[5] != 0; n.weights.assign(w, w + n.mm_k * n.mm_c); w += n.mm_k * n.mm_c; if (n.mm_bias) { n.bias.assign(w, w + n.mm_c); w += n.mm_c; } break;
            default: throw std::runtime_error("dpo_model_prove_verify: unknown node kind");
            }
            m.nodes.push_back(n);
        }
        std::vector<Element> in(input, input + input_len);
        ZkContext ctx = zk_context(m);
        Transcript tp(label);
        ModelProof p = zk_prove(ctx, in, tp);
        std::vector<Element> output = zk_run(m, in).back();
        if (tamper == 1) output[0] += 1;
        if (tamper == 2 && !p.conv.empty()) p.conv.begin()->second.partial_evals[0].c0 ^= 1;
        if (tamper == 3 && !p.pooling.empty()) p.pooling.begin()->second.zerocheck_evals[1].c1 ^= 1;
        if (tamper == 4 && !p.dense.empty()) p.dense.begin()->second.individual_claims[0].c0 ^= 1;      // Dense / MatMul: a forged final evaluation
        if (tamper == 5 && !p.dense.empty()) p.dense.begin()->second.bias_eval.c0 ^= 1;                 // ... a forged bias evaluation
        Transcript tv(label);
        zk_verify(ctx, in, output, p, tv);
        return 0;
    } catch (std::exception &e) { g_err = e.what(); return 1; }
}

// ---- batch_commit + simple_batch_open (+ verify) ----
extern "C" {
// polys: n_polys arrays of len elements (same size, same field); returns root and, optionally, the flat proof of
// simple_batch_open at `point` with evals = each polynomial's evaluation there (computed here)
int dpo_pcs_simple_batch(u32 n_polys, const u64 *const *data, u64 len, int is_ext, u32 full_log, const u64 *point, const char *label,
                         u64 *out_root, u64 *out_evals, u64 *out, u64 cap, u64 *out_len) {
    try {
        std::vector<FVec> polys; for (u32 i = 0; i < n_polys; i++) polys.push_back(mk_fvec(data[i], len, is_ext));
        BatchCommitment c = basefold_batch_commit(polys, full_log);
        for (int i = 0; i < 4; i++) out_root[i] = c.root().v[i];
        if (!point) return 0;
        std::vector<E> pt = mk_point(point, (u32)c.num_vars), evals;
        for (auto &p : polys) { MLE m; m.is_ext = p.is_ext; m.num_vars = c.num_vars; m.base = p.b; m.ext = p.e; evals.push_back(mle_evaluate(m, pt)); }
        for (u32 i = 0; i < n_polys; i++) { out_evals[2 * i] = evals[i].c0; out_evals[2 * i + 1] = evals[i].c1; }
        Transcript t(label);
        SimpleBatchProof p = basefold_simple_batch_open(full_log, c, pt, evals, t);
        std::vector<u64> f = flatten_simple_batch_proof(p);
        *out_len = f.size();
        if (f.size() > cap) { g_err = "dpo_pcs_simple_batch: output buffer too small"; return 2; }
        memcpy(out, f.data(), 8 * f.size());
        return 0;
    } catch (std::exception &e) { g_err = e.what(); return 1; }
}
int dpo_pcs_simple_batch_verify(const u64 *flat, u64 n, const u64 *root, u32 num_vars, int is_base, u32 n_polys, u32 full_log, const u64 *point, const u64 *evals, const char *label) {
    try {
        SimpleBatchProof pr = unflatten_simple_batch_proof(flat, n);
        PureCommitment c; for (int i = 0; i < 4; i++) c.root.v[i] = root[i]; c.num_vars = num_vars; c.is_base = is_base != 0;
        std::vector<E> ev; for (u32 i = 0; i < n_polys; i++) ev.push_back(E(evals[2 * i], evals[2 * i + 1]));
        Transcript t(label);
        basefold_simple_batch_verify(full_log, c, n_polys, mk_point(point, num_vars), ev, pr, t);
        return 0;
    } catch (std::exception &e) { g_err = e.what(); return 1; }
}
}

// batch_open / batch_verify with an explicit evaluation list (several polynomials may share a point)
extern "C" int dpo_pcs_batch_open_evals(u32 n, const u64 *const *data, const u64 *lens, const int *is_ext, u32 full_log, const u64 *points, const u32 *point_nv, u32 n_points,
                                        const u32 *eval_poly, const u32 *eval_point, u32 n_evals, const char *label, u64 *out_roots, u64 *out_values, u64 *out, u64 cap, u64 *out_len, int verify) {
    try {
        std::vector<FVec> polys; std::vector<Commitment> comms; std::vector<std::vector<E>> pts; std::vector<Evaluation> evals;
        for (u32 i = 0; i < n; i++) { polys.push_back(mk_fvec(data[i], lens[i], is_ext[i])); comms.push_back(basefold_commit(polys.back(), full_log)); for (int k = 0; k < 4; k++) out_roots[4 * i + k] = comms.back().root().v[k]; }
        size_t o = 0;
        for (u32 k = 0; k < n_points; k++) { pts.push_back(mk_point(points + 2 * o, point_nv[k])); o += point_nv[k]; }
        for (u32 j = 0; j < n_evals; j++) {
            const FVec &p = polys.at(eval_poly[j]); MLE m; m.is_ext = p.is_ext; m.num_vars = ceil_log2(p.len()); m.base = p.b; m.ext = p.e;
            E v = mle_evaluate(m, pts.at(eval_point[j])); evals.push_back({eval_poly[j], eval_point[j], v}); out_values[2 * j] = v.c0; out_values[2 * j + 1] = v.c1;
        }
        std::vector<const Commitment *> cp; for (auto &c : comms) cp.push_back(&c);
        Transcript t(label);
        BasefoldProof p = basefold_batch_open(full_log, polys, cp, pts, evals, t);
        if (verify) {
            std::vector<PureCommitment> pcs; for (auto &c : comms) { PureCommitment q; q.root = c.root(); q.num_vars = c.num_vars; q.is_base = c.is_base; pcs.push_back(q); }
            Transcript tv(label);
            basefold_batch_verify(full_log, pcs, pts, evals, p, tv);
        }
        std::vector<u64> f = flatten_proof(p);
        *out_len = f.size();
        if (f.size() > cap) { g_err = "dpo_pcs_batch_open_evals: output buffer too small"; return 2; }
        memcpy(out, f.data(), 8 * f.size());
        return 0;
    } catch (std::exception &e) { g_err = e.what(); return 1; }
}

// fast permutation vs the plain restatement on n seeded states (edge values every third state): number of mismatching words
extern "C" u64 dpo_poseidon2_selfcheck(u64 n, u64 seed) {
    SplitMix64 g(seed);
    const u64 edge[] = {0, 1, 2, GL_P - 1, GL_P - 2, 0xFFFFFFFFULL, 0x100000000ULL, 1ULL << 63, (GL_P - 1) / 2, 0xFFFFFFFEFFFFFFFFULL, 7};
    const int ne = sizeof(edge) / 8; u64 bad = 0, a[8], b[8];
    for (u64 it = 0; it < n; it++) {
        for (int i = 0; i < 8; i++) a[i] = b[i] = (it % 3 == 0) ? edge[g.next() % ne] : g.next_f();
        poseidon2_permute(a); poseidon2_permute_plain(b);
        for (int i = 0; i < 8; i++) if (a[i] != b[i] || a[i] >= GL_P) bad++;
    }
    return bad;
}
