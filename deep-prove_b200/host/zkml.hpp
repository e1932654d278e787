// Host mirror of the zkml prover for the MLP path (Dense -> Requant -> ReLU chains) over the C ABI.
//   zkml::{Context::generate, Prover::new/.prove} (zkml/src/iop/context.rs:110-215, iop/prover.rs:401-486),
//   prove_tables (:110-157), layers/{dense.rs:423-551, requant.rs:208-330,531-680, activation.rs:238-460},
//   lookup/{context.rs:158-296,464-480,631-781, witness.rs, logup_gkr/prover.rs:24-237},
//   commit/{context.rs:59-190,290-418, same_poly.rs:88-126}.
// Orchestration, Fiat-Shamir, claims bookkeeping and the (tiny) quantised witness columns stay on the host as
// in the reference; every polynomial lives in HBM and every O(n) loop goes through include/deepprove_b200.h.
#pragma once
#include "mpcs.hpp"
#include <unordered_map>
#include <cstdlib>
#include <cstdio>

namespace dp {
namespace zkml {

typedef int64_t Element;                                    // zkml/src/lib.rs:40
constexpr size_t BIT_LEN = 8;                               // quantization/mod.rs:20-26
constexpr Element QMIN = -127, QMAX = 127;                  // quantization/mod.rs:28-29
constexpr Element COLUMN_SEPARATOR = (Element)1 << 32;      // lookup/context.rs:622
inline size_t ceil_log2(size_t x) { size_t l = 0; while (((size_t)1 << l) < x) l++; return l; }

struct Claim { ExtVec point; Ext eval; };

struct Requant {                                            // layers/requant.rs:52-70
    size_t right_shift = 0, fp_scale = 0, intermediate_bit_size = 0; Element fixed_point_multiplier = 0;
    size_t shift() const { return fp_scale + right_shift; }
    size_t clamping_size() const { return intermediate_bit_size + ceil_log2((size_t)fixed_point_multiplier) - shift(); }
    Element apply(Element e) const {
        Element rounding = (Element)1 << (shift() - 1);
        Element unclamped = (rounding + e * fixed_point_multiplier) >> shift();
        Element sign = unclamped >= 0 ? 1 : -1, a = unclamped < 0 ? -unclamped : unclamped;
        return a >= QMAX ? QMAX * sign : unclamped;
    }
    Ext recombine_claims(Ext clamping_claim, const ExtVec &shifted) const {   // requant.rs:483-515
        Ext full = Ext::from_base(canon(1ULL << shift())) * clamping_claim, p2 = Ext::one();
        for (auto &v : shifted) { full += v * p2; p2 *= Ext::from_base(1ULL << BIT_LEN); }
        return (full - Ext::from_base(canon(1ULL << (shift() - 1)))) * Ext::from_base(from_i64(fixed_point_multiplier)).inverse();
    }
};

enum class Op { Dense, Requant, Relu, Conv, Pool, MatMul };
struct Node {
    Op op; size_t nrows = 0, ncols = 0; std::vector<Element> weights, bias; Requant rq;
    size_t kw = 0, kx = 0, nw = 0, real_nw = 0, unpadded_out[3] = {0, 0, 0};     // Conv: padded layer, `weights` = filter [kw][kx][real_nw][real_nw], `bias` [kw]
    size_t pool_c = 0, pool_h = 0, pool_w = 0;                                   // Pool: padded input shape [C][H][W] (Maxpool2D, kernel = stride = 2)
    // MatMul (layers/matrix_mul.rs), OperandMatrix::Input x OperandMatrix::Weight: the node's input is the left matrix [mm_r][mm_k], `weights` the
    // constant right matrix [mm_k][mm_c] ([mm_c][mm_k] with Config::TransposeB), `bias` (optional) one value per output column
    size_t mm_r = 0, mm_k = 0, mm_c = 0; bool mm_t = false, mm_bias = false;
};
struct Model { std::vector<Node> nodes; size_t input_len = 0; };

// TableType with the enum's derive(Ord) order (lookup/context.rs:53-63): Relu < Range < Clamping(size)
struct TableType {
    int kind; size_t size;
    bool operator<(const TableType &o) const { return kind != o.kind ? kind < o.kind : size < o.size; }
    static TableType relu() { return {0, 0}; }
    static TableType range() { return {2, 0}; }
    static TableType clamping(size_t s) { return {3, s}; }
    size_t multiplicity_poly_vars() const { return kind == 3 ? size : BIT_LEN; }   // :482-493
};
inline Element relu(Element e) { return e < 0 ? 0 : e; }
inline std::vector<u64> to_base(const std::vector<Element> &v) { std::vector<u64> o(v.size()); for (size_t i = 0; i < v.size(); i++) o[i] = from_i64(v[i]); return o; }
inline std::vector<Element> to_elements(const DeviceMle &m) { std::vector<u64> f = m.download(); std::vector<Element> o(f.size()); for (size_t i = 0; i < f.size(); i++) o[i] = f[i] > (P >> 1) ? -(Element)(P - f[i]) : (Element)f[i]; return o; }

// (PCS::CommitmentWithWitness, DenseMultilinearExtension) -- lookup/context.rs:38-41
struct ProverCommitment { BasefoldCommitmentWithWitness comm; DeviceMle poly; };

struct TableData { std::vector<Element> merged; std::map<Element, u64> table_count; std::vector<DeviceMle> columns; };

struct LogUpProof {
    std::vector<IOPProof> sumcheck_proofs; std::vector<ExtVec> round_evaluations; std::vector<Claim> output_claims; std::vector<ExtVec> circuit_outputs; bool table = false;
};
struct LogUpInput {   // logup_gkr/structs.rs:134-148 with the columns resident in HBM
    bool table = false; std::vector<DeviceMle> column_evals; DeviceMle multiplicities; Ext constant_challenge, column_separation_challenge; size_t columns_per_instance = 1;
};

struct LogUpHandle { dp_logup *h = nullptr; ~LogUpHandle() { if (h) dp_logup_free(h); } };

// logup_gkr::prover::batch_prove (prover.rs:24-237)
template <class T>
LogUpProof logup_batch_prove(const LogUpInput &in, T &t) {
    std::vector<std::unique_ptr<LogUpHandle>> circuits;
    u64 cc[2] = {in.constant_challenge.c0, in.constant_challenge.c1}, sc[2] = {in.column_separation_challenge.c0, in.column_separation_challenge.c1};
    auto build = [&](size_t from, size_t n, const DeviceMle *mult) {
        std::vector<dp_mle *> cols; for (size_t k = 0; k < n; k++) cols.push_back(in.column_evals[from + k].handle());
        auto L = std::make_unique<LogUpHandle>();
        check(dp_logup_build(cols.data(), (uint32_t)n, mult ? mult->handle() : nullptr, cc, sc, &L->h));
        circuits.push_back(std::move(L));
    };
    if (in.table) build(0, in.column_evals.size(), &in.multiplicities);
    else for (size_t i = 0; i < in.column_evals.size(); i += in.columns_per_instance) build(i, in.columns_per_instance, nullptr);
    LogUpProof pr; pr.table = in.table;
    size_t total_layers = 0;
    for (auto &c : circuits) {
        uint32_t nv; check(dp_logup_num_vars(c->h, &nv)); total_layers = std::max<size_t>(total_layers, nv);
        u64 o[8]; check(dp_logup_outputs(c->h, o));
        pr.circuit_outputs.push_back({Ext(o[0], o[1]), Ext(o[2], o[3]), Ext(o[4], o[5]), Ext(o[6], o[7])});
    }
    t.append_field_element(canon(circuits.size()));
    for (auto &o : pr.circuit_outputs) t.append_field_element_exts(o);
    Ext batching = t.get_and_append_challenge("initial_batching"), alpha = t.get_and_append_challenge("initial_alpha"), lambda = t.get_and_append_challenge("initial_lambda");
    Ext claim = Ext::zero(), ac = Ext::one();
    for (auto &e : pr.circuit_outputs) { claim += ac * (batching * (e[1] - e[0]) + e[0] + lambda * (batching * (e[3] - e[2]) + e[2])); ac *= alpha; }
    ExtVec point = {batching};
    size_t v = 1;
    // the leading small layers in one resident launch that runs the transcript on the device, when the library takes them (blocking
    // waits) and the transcript's state can go there (BasicTranscript's sponge, or BlakeTranscript's hasher up to 2^16 chunks)
    std::vector<dp_logup *> hs; for (auto &c : circuits) hs.push_back(c->h);
    uint32_t n_dev = 0;
    check(dp_logup_layers_fs_next(hs.data(), (uint32_t)hs.size(), 1, &n_dev));
    const size_t last = n_dev, n_rounds = last * (last + 1) / 2;
    auto views = [&](size_t layer) -> size_t { return !in.table && layer == total_layers ? 2 : 4; };   // dp_logup_layer_mles
    size_t n_evals = 0; for (size_t l = 1; l <= last; l++) n_evals += views(l) * circuits.size();
    std::vector<u64> pt(2 * (last + 1)), msgs(2 * 4 * n_rounds), ch(2 * n_rounds), ev(2 * n_evals);
    pt[0] = batching.c0; pt[1] = batching.c1;
    u64 cl[2] = {claim.c0, claim.c1}, al[2] = {alpha.c0, alpha.c1}, lm[2] = {lambda.c0, lambda.c1};
    if (n_dev > 0 && run_device_transcript(t, dp_logup_run_layers_fs, dp_logup_run_layers_fs_blake, [&](auto run, u64 *sp) {
            return run(hs.data(), (uint32_t)hs.size(), 1, (uint32_t)last, cl, pt.data(), al, lm, sp, msgs.data(), ch.data(), ev.data()); })) {
        size_t oe = 0;
        for (size_t l = 1, k = 0; l <= last; k += l, l++) {    // k: rounds before layer l
            IOPProof p;
            append_device_rounds(p, p.point, l, 3, msgs.data() + 2 * 4 * k, ch.data() + 2 * k);
            pr.sumcheck_proofs.push_back(std::move(p));
            ExtVec evals; for (size_t i = 0; i < views(l) * circuits.size(); i++, oe += 2) evals.push_back(Ext(ev[oe], ev[oe + 1]));
            pr.round_evaluations.push_back(std::move(evals));
        }
        point.clear(); for (size_t i = 0; i <= last; i++) point.push_back(Ext(pt[2 * i], pt[2 * i + 1]));
        claim = Ext(cl[0], cl[1]); alpha = Ext(al[0], al[1]); lambda = Ext(lm[0], lm[1]);
        v = last + 1;
    }
    for (; v <= total_layers; v++) {
        t.append_field_element_ext(claim);
        DeviceMle eq = DeviceMle::build_eq_x_r(point);           // compute_betas_eval(&sumcheck_point)
        VirtualPolynomial vp(v);
        Ext cur = Ext::one();
        for (auto &c : circuits) {
            dp_mle *views[4]; uint32_t n = 0;
            check(dp_logup_layer_mles(c->h, (uint32_t)v, views, &n));
            std::vector<DeviceMle> m; for (uint32_t k = 0; k < n; k++) m.push_back(DeviceMle(views[k]));
            if (n == 4) { vp.add_mle_list({eq, m[0], m[3]}, cur); vp.add_mle_list({eq, m[1], m[2]}, cur); vp.add_mle_list({eq, m[2], m[3]}, cur * lambda); }
            else { vp.add_mle_list({eq, m[1]}, -cur); vp.add_mle_list({eq, m[0]}, -cur); vp.add_mle_list({eq, m[0], m[1]}, cur * lambda); }
            cur *= alpha;
        }
        auto res = IOPProverState::prove_parallel(std::move(vp), t);
        point = res.first.point;
        const ExtVec &fe = res.second.get_mle_final_evaluations();
        ExtVec evals(fe.begin() + 1, fe.end());
        batching = t.get_and_append_challenge("logup_batching"); alpha = t.get_and_append_challenge("logup_alpha"); lambda = t.get_and_append_challenge("logup_lambda");
        point.push_back(batching);
        pr.sumcheck_proofs.push_back(res.first);
        Ext acc = Ext::zero(), al = Ext::one();
        if (v != total_layers || in.table) for (size_t i = 0; i + 3 < evals.size(); i += 4) { const Ext *e = &evals[i]; acc += al * (batching * (e[2] - e[0]) + e[0] + lambda * (batching * (e[1] - e[3]) + e[3])); al *= alpha; }
        else for (size_t i = 0; i + 1 < evals.size(); i += 2) { const Ext *e = &evals[i]; acc += al * (batching * (e[0] - e[1]) + e[1]); al *= alpha; }   // final_round_claim, Lookup
        claim = acc;
        pr.round_evaluations.push_back(evals);
    }
    // output claims about the base columns (prover.rs:172-183)
    std::vector<DeviceMle> base; if (in.table) base.push_back(in.multiplicities);
    for (auto &c : in.column_evals) base.push_back(c);
    ExtVec be = DeviceMle::evaluate_many(base, point);
    for (auto &e : be) pr.output_claims.push_back({point, e});
    return pr;
}

// same_poly::Prover (commit/same_poly.rs:58-126)
struct SamePolyProof { IOPProof sumcheck; ExtVec evals; Claim extract_claim() const { return {sumcheck.point, evals.at(1)}; } };
template <class T>
SamePolyProof same_poly_prove(const DeviceMle &poly, const std::vector<Claim> &claims, T &t) {
    ExtVec ch; for (size_t i = 0; i < claims.size(); i++) { if (claims[i].point.size() != poly.num_vars()) throw Error(DP_ERR_INVALID, "Invalid claim length"); ch.push_back(t.read_challenge()); }
    std::vector<DeviceMle> betas; for (auto &c : claims) betas.push_back(DeviceMle::build_eq_x_r(c.point));
    DeviceMle final_beta = DeviceMle::linear_combination(betas, ch);
    VirtualPolynomial vp(poly.num_vars());
    vp.add_mle_list({final_beta, poly}, Ext::one());
    auto res = IOPProverState::prove_parallel(std::move(vp), t);
    return {res.first, res.second.get_mle_final_evaluations()};
}

}  // namespace zkml
}  // namespace dp
#include "conv.hpp"   // FFT-convolution layer (uses the definitions above; the Prover below uses it)
namespace dp {
namespace zkml {

struct DenseProof { IOPProof sumcheck; Ext bias_eval; ExtVec individual_claims; };
struct PoolingProof { IOPProof sumcheck; LogUpProof lookup; ExtVec zerocheck_evals; size_t variable_gap = 0; std::vector<Digest> commitments; };   // layers/pooling.rs:60-75
struct RequantProof { IOPProof io_accumulation; ExtVec accumulation_evals; LogUpProof clamping_lookup, shifted_lookup; std::vector<Digest> commitments; };
struct ActivationProof { SamePolyProof io_accumulation; LogUpProof lookup; std::vector<Digest> commits; };
struct TableProof { Digest multiplicity_commit; LogUpProof lookup; };
struct Proof {   // zkml/src/iop/mod.rs:21-31 + commit::context::ModelOpeningProof
    std::map<size_t, DenseProof> dense; std::map<size_t, RequantProof> requant; std::map<size_t, ActivationProof> activation;
    std::map<size_t, ConvProof> conv; std::map<size_t, PoolingProof> pooling;
    std::vector<TableProof> table_proofs; BasefoldProof batch_proof; std::vector<BasefoldProof> trivial_proofs;
    std::vector<u64> flatten(size_t n_nodes) const;
};

// Context (iop/context.rs:38-47): step info + CommitmentContext (weights/bias committed at setup) + lookup tables
class Context {
  public:
    static Context generate(const Model &m) {
        Context c; c.model = &m;
        size_t max_len = m.input_len; std::map<TableType, int> tabs;
        for (auto &n : m.nodes) {
            if (n.op == Op::Dense) max_len = std::max(max_len, std::max(n.nrows * n.ncols, n.nrows));
            if (n.op == Op::MatMul) max_len = std::max(max_len, std::max(n.mm_k * n.mm_c, n.mm_c));
            if (n.op == Op::Requant) { tabs[TableType::range()] = 1; tabs[TableType::clamping(n.rq.clamping_size())] = 1; }
            if (n.op == Op::Relu) tabs[TableType::relu()] = 1;
            if (n.op == Op::Conv) max_len = std::max(max_len, std::max(n.weights.size(), n.kw * n.nw * n.nw));
            if (n.op == Op::Pool) { tabs[TableType::range()] = 1; max_len = std::max(max_len, n.pool_c * n.pool_h * n.pool_w); }   // pooling.rs:130-170
        }
        for (auto &kv : tabs) max_len = std::max(max_len, (size_t)1 << kv.first.multiplicity_poly_vars());   // context.rs:171-175
        size_t p2 = 1; while (p2 < max_len) p2 <<= 1;
        c.pp = Basefold::setup_and_trim(p2);
        for (size_t id = 0; id < m.nodes.size(); id++) if (m.nodes[id].op == Op::Dense) {   // CommitmentContext::new (commit/context.rs:59-103)
            for (auto &kv : std::map<std::string, const std::vector<Element> *>{{"DenseBias", &m.nodes[id].bias}, {"DenseWeight", &m.nodes[id].weights}}) {
                DeviceMle poly = DeviceMle::from_evaluations_vec(to_base(*kv.second));
                c.model_comms[id][kv.first] = {Basefold::commit(c.pp, poly), poly};
            }
        } else if (m.nodes[id].op == Op::MatMul) {   // MatMul::ctx (matrix_mul.rs:951-963): the constant matrix and the bias are model polynomials
            const Node &n = m.nodes[id];
            if (n.mm_bias) { DeviceMle poly = DeviceMle::from_evaluations_vec(to_base(n.bias)); c.model_comms[id]["MatMulBias"] = {Basefold::commit(c.pp, poly), poly}; }
            DeviceMle poly = DeviceMle::from_evaluations_vec(to_base(n.weights));
            c.model_comms[id]["MatMulWeight"] = {Basefold::commit(c.pp, poly), poly};
        } else if (m.nodes[id].op == Op::Conv) {   // convolution.rs:532-540: ConvBias, ConvFilter (BTreeMap order)
            const Node &n = m.nodes[id];
            Convolution cv; cv.kw = n.kw; cv.kx = n.kx; cv.nw = n.nw; cv.real_nw = n.real_nw; cv.filter = n.weights; cv.bias = n.bias;
            for (int i = 0; i < 3; i++) cv.unpadded_out[i] = n.unpadded_out[i];
            cv.load();
            DeviceMle bias_poly = DeviceMle::from_evaluations_vec(to_base(n.bias));
            c.model_comms[id]["ConvBias"] = {Basefold::commit(c.pp, bias_poly), bias_poly};
            c.model_comms[id]["ConvFilter"] = {Basefold::commit(c.pp, cv.filter_mle), cv.filter_mle};
            c.convs[id] = std::move(cv);
        }
        for (auto &kv : tabs) {   // get_merged_table_column (lookup/context.rs:158-296), resident for every proof
            TableData td; std::vector<std::vector<u64>> cols;
            const TableType &tt = kv.first;
            if (tt.kind == 0) { cols.resize(2); for (Element i = QMIN - 1; i <= QMAX; i++) { Element o = relu(i); td.merged.push_back(i + o * COLUMN_SEPARATOR); cols[0].push_back(from_i64(i)); cols[1].push_back(from_i64(o)); } }
            else if (tt.kind == 2) { cols.resize(1); for (Element i = 0; i < ((Element)1 << BIT_LEN); i++) { td.merged.push_back(i); cols[0].push_back(from_i64(i)); } }
            else { cols.resize(2); Element mx = (Element)1 << (tt.size - 1); for (Element i = -mx; i < mx; i++) { Element o = i < QMIN ? QMIN : (i > QMAX ? QMAX : i); td.merged.push_back(i + o * COLUMN_SEPARATOR); cols[0].push_back(from_i64(i)); cols[1].push_back(from_i64(o)); } }
            for (Element e : td.merged) td.table_count[e]++;
            for (auto &col : cols) td.columns.push_back(DeviceMle::from_evaluations_vec(col));
            c.tables[tt] = std::move(td);
        }
        return c;
    }
    template <class T> void write_to_transcript(T &t) const { for (auto &nk : model_comms) for (auto &pk : nk.second) Basefold::write_commitment(pk.second.comm.root, t); }   // commit/context.rs:181-190
    const Model *model = nullptr; BasefoldProverParams pp;
    std::map<size_t, std::map<std::string, ProverCommitment>> model_comms;
    std::map<TableType, TableData> tables;
    std::map<size_t, Convolution> convs;                      // resident conv layers (weights, FFT'd filters)
};

struct LogUpWitness { bool table = false; std::vector<ProverCommitment> commits; std::vector<DeviceMle> column_evals; DeviceMle multiplicity_evals; size_t columns_per_instance = 1; TableType tt{0, 0}; };

// quantised inference (model run): outputs[i] = output tensor of node i
// Maxpool2D::op (pooling.rs:667-677) on a padded [C][H][W] tensor
inline std::vector<Element> maxpool2d(const std::vector<Element> &x, size_t C, size_t H, size_t W) {
    std::vector<Element> o(C * (H / 2) * (W / 2));
    for (size_t c = 0; c < C; c++) for (size_t r = 0; r < H / 2; r++) for (size_t cc = 0; cc < W / 2; cc++) {
        Element mx = x[(c * H + 2 * r) * W + 2 * cc];
        for (size_t a = 0; a < 2; a++) for (size_t b = 0; b < 2; b++) mx = std::max(mx, x[(c * H + 2 * r + a) * W + 2 * cc + b]);
        o[(c * (H / 2) + r) * (W / 2) + cc] = mx;
    }
    return o;
}
inline std::vector<std::vector<Element>> run(const Model &m, const std::vector<Element> &input, const Context *ctx = nullptr, std::map<size_t, ConvData> *conv_data = nullptr) {
    std::vector<std::vector<Element>> outs; std::vector<Element> cur = input;
    for (auto &n : m.nodes) {
        std::vector<Element> o;
        if (n.op == Op::Dense) { o.resize(n.nrows); for (size_t r = 0; r < n.nrows; r++) { Element a = n.bias[r]; const Element *w = &n.weights[r * n.ncols]; for (size_t c = 0; c < n.ncols; c++) a += w[c] * cur[c]; o[r] = a; } }
        else if (n.op == Op::Requant) { Element lim = (Element)1 << n.rq.intermediate_bit_size; for (Element e : cur) { if (e > lim || e < -lim) throw Error(DP_ERR_INVALID, "Could not apply requantisation, tensor element had absolute value too large"); o.push_back(n.rq.apply(e)); } }
        else if (n.op == Op::Relu) for (Element e : cur) o.push_back(relu(e));
        else if (n.op == Op::Pool) o = maxpool2d(cur, n.pool_c, n.pool_h, n.pool_w);
        else if (n.op == Op::MatMul) {
            if (cur.size() != n.mm_r * n.mm_k) throw Error(DP_ERR_INVALID, "Incompatible shape found for input matrix");
            o.assign(n.mm_r * n.mm_c, 0);
            for (size_t r = 0; r < n.mm_r; r++) for (size_t c = 0; c < n.mm_c; c++) {
                Element a = n.mm_bias ? n.bias[c] : 0;
                for (size_t k = 0; k < n.mm_k; k++) a += cur[r * n.mm_k + k] * (n.mm_t ? n.weights[c * n.mm_k + k] : n.weights[k * n.mm_c + c]);
                o[r * n.mm_c + c] = a;
            }
        }
        else {
            if (!ctx || !conv_data) throw Error(DP_ERR_INVALID, "run: a convolution needs the Context (resident FFT'd filters)");
            ConvData cd; o = ctx->convs.at(outs.size()).op(cur, cd); (*conv_data)[outs.size()] = std::move(cd);
        }
        outs.push_back(o); cur = o;
    }
    return outs;
}
inline std::vector<std::vector<Element>> run(const Context &ctx, const std::vector<Element> &input, std::map<size_t, ConvData> *conv_data) { return run(*ctx.model, input, &ctx, conv_data); }

// The inference trace ON THE DEVICE: every tensor is a Base MLE of canonical field elements of signed integers (Tensor::to_field),
// so a trace tensor doubles as a lookup column.  Built by run_device (quantised inference on the device: only the model input
// crosses PCIe) or by uploading a host trace once (upload_trace); read-only afterwards, shared by concurrent provers.
struct DeviceTrace { DeviceMle input; std::vector<DeviceMle> outs; std::map<size_t, ConvData> conv; bool valid() const { return input.valid(); } };
struct WitHandle { dp_wit *w = nullptr; ~WitHandle() { if (w) dp_wit_free(w); } };
// the tables of a Context in TableType order (the reference's BTreeMap order) as the dp_wit_begin arguments
inline void wit_tables(const Context &ctx, std::vector<uint32_t> &kinds, std::vector<uint32_t> &sizes, std::map<TableType, uint32_t> &index) {
    for (auto &kv : ctx.tables) { index[kv.first] = (uint32_t)kinds.size(); kinds.push_back((uint32_t)kv.first.kind); sizes.push_back((uint32_t)kv.first.size); }
}
inline DeviceMle wit_own(dp_mle *h) { return DeviceMle(h); }
inline std::vector<DeviceMle> wit_requant(dp_wit *w, const DeviceMle &x, const Requant &rq, const std::map<TableType, uint32_t> &ti) {
    size_t nc = 2 + rq.shift() / BIT_LEN; std::vector<dp_mle *> raw(nc, nullptr);
    check(dp_wit_requant(w, x.handle(), (uint32_t)rq.shift(), rq.fixed_point_multiplier, (uint32_t)rq.intermediate_bit_size,
                         ti.at(TableType::clamping(rq.clamping_size())), ti.at(TableType::range()), raw.data(), (uint32_t)nc));
    std::vector<DeviceMle> cols; for (dp_mle *h : raw) cols.push_back(wit_own(h));
    return cols;
}
inline std::vector<DeviceMle> wit_pool(dp_wit *w, const DeviceMle &x, const Node &n, const std::map<TableType, uint32_t> &ti) {
    dp_mle *raw[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    check(dp_wit_pool(w, x.handle(), (uint32_t)n.pool_c, (uint32_t)n.pool_h, (uint32_t)n.pool_w, ti.at(TableType::range()), raw));
    std::vector<DeviceMle> cols; for (dp_mle *h : raw) cols.push_back(wit_own(h));
    return cols;
}
inline void wit_check(uint32_t bits) {
    if (bits & 1) throw Error(DP_ERR_INVALID, "Could not apply requantisation, tensor element had absolute value too large");
    if (bits) throw Error(DP_ERR_INVALID, "lookup witness: a value is not in its table (clamping / relu / pooling range)");
}
// Model::run on the device (Dense / Requant / Relu / Maxpool2D kernels of csrc/witness.cu, the FFT convolution of csrc/conv.cu):
// only the model input crosses PCIe
inline DeviceTrace run_device(const Context &ctx, const std::vector<Element> &input) {
    const Model &m = *ctx.model;
    DeviceTrace tr; tr.input = DeviceMle::from_evaluations_vec(to_base(input));
    std::vector<uint32_t> kinds, sizes; std::map<TableType, uint32_t> ti; wit_tables(ctx, kinds, sizes, ti);
    WitHandle wh; if (!kinds.empty()) check(dp_wit_begin((uint32_t)kinds.size(), kinds.data(), sizes.data(), &wh.w));
    DeviceMle cur = tr.input;
    for (size_t id = 0; id < m.nodes.size(); id++) {
        const Node &n = m.nodes[id]; DeviceMle o;
        if (n.op == Op::Dense) { const auto &c = ctx.model_comms.at(id); dp_mle *h; check(dp_wit_dense(c.at("DenseWeight").poly.handle(), c.at("DenseBias").poly.handle(), cur.handle(), (uint32_t)n.nrows, (uint32_t)n.ncols, &h)); o = wit_own(h); }
        else if (n.op == Op::Requant) o = wit_requant(wh.w, cur, n.rq, ti)[1];
        else if (n.op == Op::Relu) { dp_mle *h; check(dp_wit_relu(wh.w, cur.handle(), ti.at(TableType::relu()), &h)); o = wit_own(h); }
        else if (n.op == Op::Pool) o = wit_pool(wh.w, cur, n, ti)[4];
        else if (n.op == Op::MatMul) { const auto &c = ctx.model_comms.at(id); dp_mle *h; check(dp_wit_matmul(cur.handle(), c.at("MatMulWeight").poly.handle(), n.mm_bias ? c.at("MatMulBias").poly.handle() : nullptr, (uint32_t)n.mm_r, (uint32_t)n.mm_k, (uint32_t)n.mm_c, n.mm_t ? 1 : 0, &h)); o = wit_own(h); }
        else { ConvData cd; o = ctx.convs.at(id).op(cur, cd); tr.conv[id] = std::move(cd); }
        tr.outs.push_back(o); cur = o;
    }
    if (wh.w) { std::vector<dp_mle *> mu(kinds.size(), nullptr); uint32_t bits = 0; check(dp_wit_finish(wh.w, mu.data(), &bits)); for (dp_mle *h : mu) wit_own(h); wit_check(bits); }
    return tr;
}
inline DeviceTrace upload_trace(const std::vector<Element> &input, const std::vector<std::vector<Element>> &outs, const std::map<size_t, ConvData> *conv_data) {
    DeviceTrace tr; tr.input = DeviceMle::from_evaluations_vec(to_base(input));
    for (auto &o : outs) tr.outs.push_back(DeviceMle::from_evaluations_vec(to_base(o)));
    if (conv_data) tr.conv = *conv_data;
    return tr;
}

// Prover<'a, E, T, PCS> (iop/prover.rs:40-60)
template <class T>
class Prover {
  public:
    Prover(const Context &ctx, T &transcript) : ctx_(ctx), t_(transcript) {}

    // end to end from the host input vector: inference on the device, then prove
    Proof prove(const std::vector<Element> &input) { DeviceTrace tr = run_device(ctx_, input); return prove(tr); }
    // a host trace (the reference's InferenceTrace): uploaded once, tensor by tensor
    Proof prove(const std::vector<Element> &input, const std::vector<std::vector<Element>> &outs, const std::map<size_t, ConvData> *conv_data = nullptr) {
        DeviceTrace tr = upload_trace(input, outs, conv_data); return prove(tr);
    }
    // Prover::prove(full_trace): the inference trace is an INPUT of proving (zkml/src/bin/bench.rs:390-408 times only this)
    Proof prove(const DeviceTrace &tr) {
        const Model &m = *ctx_.model;
        if (tr.outs.size() != m.nodes.size()) throw Error(DP_ERR_INVALID, "prove: the trace does not match the model");
        const std::map<size_t, ConvData> *conv_data = &tr.conv;
        auto node_input = [&](size_t id) -> const DeviceMle & { return id == 0 ? tr.input : tr.outs[id - 1]; };
        ctx_.write_to_transcript(t_);
        instantiate_witness_ctx(m, tr);
        // output claim (prover.rs:423-436)
        const DeviceMle &fo = tr.outs.back();
        Claim last; for (size_t i = 0, nv = fo.num_vars(); i < nv; i++) last.point.push_back(t_.read_challenge());
        last.eval = fo.evaluate(last.point);
        for (size_t id = m.nodes.size(); id-- > 0;) {
            const Node &n = m.nodes[id];
            if (n.op == Op::Dense) last = prove_dense(id, n, last, node_input(id));
            else if (n.op == Op::Requant) last = prove_requant(id, n, last);
            else if (n.op == Op::Relu) last = prove_activation(id, last);
            else if (n.op == Op::Pool) last = prove_pooling(id, n, last);
            else if (n.op == Op::MatMul) last = prove_matmul(id, n, last, node_input(id));
            else {
                if (!conv_data || !conv_data->count(id)) throw Error(DP_ERR_INVALID, "prove: no convolution proving data in the trace");
                last = prove_convolution(id, last, conv_data->at(id));
            }
        }
        prove_tables();
        commit_prove();
        return std::move(proof_);
    }

  private:
    void add_witness_claim(const ProverCommitment &pc, const Claim &c) { (pc.poly.num_vars() <= Basefold::trivial_num_vars() ? trivial_claims_ : claims_).push_back({pc, c}); }   // commit/context.rs:290-310
    ProverCommitment commit_column(const std::vector<u64> &ev) { DeviceMle p = DeviceMle::from_evaluations_vec(ev); return {Basefold::commit(ctx_.pp, p), p}; }

    // generate_lookup_witnesses (lookup/context.rs:631-756) + initialise_from_table_set (:758-781).
    // The reference commits every witness column from rayon workers before any challenge is drawn; here all
    // columns are gathered first and committed with ONE Basefold::commit_many call (concurrent on the device).
    void instantiate_witness_ctx(const Model &m, const DeviceTrace &tr) {
        auto node_input = [&](size_t id) -> const DeviceMle & { return id == 0 ? tr.input : tr.outs[id - 1]; };
        std::vector<DeviceMle> polys;                            // every column to commit, in creation order (all device-resident)
        struct Slot { size_t node; size_t witness; bool table; bool column = true; };  // where commitment k goes (column: also a lookup column)
        std::vector<Slot> slots;
        std::vector<uint32_t> kinds, sizes; std::map<TableType, uint32_t> ti; wit_tables(ctx_, kinds, sizes, ti);
        WitHandle wh; if (!kinds.empty()) check(dp_wit_begin((uint32_t)kinds.size(), kinds.data(), sizes.data(), &wh.w));
        std::map<TableType, bool> used;
        for (size_t id = 0; id < m.nodes.size(); id++) {
            const Node &n = m.nodes[id];
            if (n.op == Op::Requant) {   // requant.rs:208-330: clamping (input, output) columns + the byte chunks of the shifted-out bits
                TableType tc = TableType::clamping(n.rq.clamping_size()), trg = TableType::range();
                used[tc] = used[trg] = true;
                std::vector<DeviceMle> c = wit_requant(wh.w, node_input(id), n.rq, ti);
                LogUpWitness wc; wc.tt = tc; wc.columns_per_instance = 2;
                LogUpWitness ws; ws.tt = trg; ws.columns_per_instance = 1;
                lookup_witness_[id] = {wc, ws};
                for (size_t k = 0; k < c.size(); k++) { polys.push_back(c[k]); slots.push_back({id, k < 2 ? (size_t)0 : (size_t)1, false}); }
            } else if (n.op == Op::Relu) {   // activation.rs:238-323: the node's input and output tensors ARE the two columns
                TableType tt = TableType::relu(); LogUpWitness w; w.tt = tt; w.columns_per_instance = 2; used[tt] = true;
                dp_mle *h; check(dp_wit_relu(wh.w, node_input(id).handle(), ti.at(tt), &h)); DeviceMle out = wit_own(h);
                lookup_witness_[id] = {w};
                polys.push_back(node_input(id)); slots.push_back({id, 0, false});
                polys.push_back(out); slots.push_back({id, 0, false});
            } else if (n.op == Op::Pool) {   // pooling.rs:210-271 + compute_polys (:686-771)
                TableType trg = TableType::range(); LogUpWitness w; w.tt = trg; w.columns_per_instance = 1; used[trg] = true;
                std::vector<DeviceMle> c = wit_pool(wh.w, node_input(id), n, ti);
                lookup_witness_[id] = {w};
                for (size_t k = 0; k < 4; k++) { polys.push_back(c[k]); slots.push_back({id, 0, false}); }
                polys.push_back(c[4]); slots.push_back({id, 0, false, false});   // the output poly: committed, not a lookup column
            }
        }
        std::vector<TableType> table_order;
        if (wh.w) {   // table multiplicities (lookup/context.rs:675-737): histograms the node kernels filled, every table row distinct
            std::vector<dp_mle *> mu(kinds.size(), nullptr); uint32_t bits = 0;
            check(dp_wit_finish(wh.w, mu.data(), &bits));
            std::vector<DeviceMle> mults; for (dp_mle *h : mu) mults.push_back(wit_own(h));
            wit_check(bits);
            for (auto &kv : ctx_.tables) {
                if (!used.count(kv.first)) continue;
                for (auto &tc : kv.second.table_count) if (tc.second != 1) throw Error(DP_ERR_UNSUPPORTED, "device multiplicities need distinct table rows");
                LogUpWitness w; w.table = true; w.tt = kv.first; w.column_evals = kv.second.columns;
                table_witness_.push_back(w); table_order.push_back(kv.first);
                polys.push_back(mults[ti.at(kv.first)]); slots.push_back({0, table_witness_.size() - 1, true});
            }
        }
        std::vector<BasefoldCommitmentWithWitness> comms = Basefold::commit_many(ctx_.pp, polys);
        for (size_t k = 0; k < slots.size(); k++) {
            ProverCommitment pc{comms[k], polys[k]};
            if (slots[k].table) { LogUpWitness &w = table_witness_[slots[k].witness]; w.commits.push_back(pc); w.multiplicity_evals = polys[k]; }
            else { LogUpWitness &w = lookup_witness_[slots[k].node][slots[k].witness]; w.commits.push_back(pc); if (slots[k].column) w.column_evals.push_back(polys[k]); }
        }
        constant_challenge_ = t_.get_and_append_challenge("table_constant");
        for (auto &tt : table_order) challenge_map_[tt] = tt.kind == 0 ? t_.get_and_append_challenge("Relu") : (tt.kind == 3 ? t_.get_and_append_challenge("Clamping") : Ext::one());
    }
    LogUpInput get_logup_input(const LogUpWitness &w) const {   // lookup/witness.rs:96-140
        LogUpInput in; in.table = w.table; in.column_evals = w.column_evals; in.multiplicities = w.multiplicity_evals;
        in.constant_challenge = constant_challenge_; in.column_separation_challenge = challenge_map_.at(w.tt); in.columns_per_instance = w.columns_per_instance;
        return in;
    }

    // Dense::prove_step (layers/dense.rs:423-551)
    Claim prove_dense(size_t id, const Node &n, const Claim &last_claim, const DeviceMle &input) {
        const auto &comms = ctx_.model_comms.at(id);
        const DeviceMle &weights = comms.at("DenseWeight").poly, &bias = comms.at("DenseBias").poly;
        if (ceil_log2(n.nrows) != last_claim.point.size()) throw Error(DP_ERR_INVALID, "something's wrong with the randomness");
        Ext bias_eval = bias.evaluate(last_claim.point);
        DeviceMle mat = weights.fix_high_variables(last_claim.point);      // rows are the HIGH variables (dense.rs:471-475)
        const DeviceMle &in = input;                                        // the trace tensor itself (a sumcheck borrows its inputs)
        VirtualPolynomial vp(in.num_vars());
        vp.add_mle_list({mat, in}, Ext::one());
        auto res = IOPProverState::prove_parallel(std::move(vp), t_);
        const ExtVec &fe = res.second.get_mle_final_evaluations();
        ExtVec wp = res.first.point; wp.insert(wp.end(), last_claim.point.begin(), last_claim.point.end());
        add_witness_claim(comms.at("DenseBias"), {last_claim.point, bias_eval});   // BTreeMap order of PolyId
        add_witness_claim(comms.at("DenseWeight"), {wp, fe[0]});
        proof_.dense[id] = {res.first, bias_eval, fe};
        return {res.first.point, fe[1]};
    }

    // MatMul::prove_step (layers/matrix_mul.rs:701-874) for Input x Weight: the output claim splits into the row part (fixes the HIGH variables of
    // the left = input matrix) and the column part (fixes the LOW variables of the constant matrix, or its HIGH ones when it is stored
    // transposed); one degree-2 sumcheck over the shared inner dimension; the left evaluation is the claim handed to the previous node
    Claim prove_matmul(size_t id, const Node &n, const Claim &last_claim, const DeviceMle &input) {
        const auto &comms = ctx_.model_comms.at(id);
        const size_t vr = ceil_log2(n.mm_r), vc = ceil_log2(n.mm_c), vk = ceil_log2(n.mm_k);
        if (last_claim.point.size() != vr + vc) throw Error(DP_ERR_INVALID, "Wrong length of last claim point");
        const ExtVec p_right(last_claim.point.begin(), last_claim.point.begin() + vc), p_left(last_claim.point.begin() + vc, last_claim.point.end());   // split_claim
        Ext bias_eval = Ext::zero();
        if (n.mm_bias) bias_eval = comms.at("MatMulBias").poly.evaluate(p_right);
        DeviceMle left = input.fix_high_variables(p_left);
        const DeviceMle &w = comms.at("MatMulWeight").poly;
        DeviceMle right = n.mm_t ? w.fix_high_variables(p_right) : w.fix_variables(p_right);
        if (left.num_vars() != vk || right.num_vars() != vk) throw Error(DP_ERR_INVALID, "matmul: free variables of the two matrices differ");
        VirtualPolynomial vp(vk);
        vp.add_mle_list({left, right}, Ext::one());
        auto res = IOPProverState::prove_parallel(std::move(vp), t_);
        const ExtVec &fe = res.second.get_mle_final_evaluations();
        ExtVec pl = res.first.point; pl.insert(pl.end(), p_left.begin(), p_left.end());                      // full_points
        ExtVec pr;
        if (n.mm_t) { pr = res.first.point; pr.insert(pr.end(), p_right.begin(), p_right.end()); } else { pr = p_right; pr.insert(pr.end(), res.first.point.begin(), res.first.point.end()); }
        if (n.mm_bias) add_witness_claim(comms.at("MatMulBias"), {p_right, bias_eval});                       // BTreeMap order of PolyId
        add_witness_claim(comms.at("MatMulWeight"), {pr, fe[1]});
        proof_.dense[id] = {res.first, bias_eval, fe};                                                         // MatMulProof has DenseProof's shape
        return {pl, fe[0]};
    }

    // Requant::prove_step (layers/requant.rs:531-680)
    Claim prove_requant(size_t id, const Node &n, const Claim &last_claim) {
        std::vector<LogUpWitness> ws = lookup_witness_.at(id);
        if (ws.size() != 2) throw Error(DP_ERR_INVALID, "There should be two lookup witnesses during requantisation");
        LogUpInput cin = get_logup_input(ws[0]), sin = get_logup_input(ws[1]);
        LogUpProof cp = logup_batch_prove(cin, t_), sp = logup_batch_prove(sin, t_);
        size_t nv = cin.column_evals[0].num_vars();
        DeviceMle cbeta = DeviceMle::build_eq_x_r(cp.output_claims[0].point), lbeta = DeviceMle::build_eq_x_r(last_claim.point), sbeta = DeviceMle::build_eq_x_r(sp.output_claims[0].point);
        Ext bc = t_.get_and_append_challenge("requant_batching");
        VirtualPolynomial vp(nv);
        vp.add_mle_list({cin.column_evals[1], lbeta}, Ext::one());
        vp.add_mle_list({cin.column_evals[1], cbeta}, bc);
        Ext comb = bc * bc; vp.add_mle_list({cin.column_evals[0], cbeta}, comb);
        comb *= bc;
        for (auto &col : sin.column_evals) { vp.add_mle_list({sbeta, col}, comb); comb *= bc; }
        auto res = IOPProverState::prove_parallel(std::move(vp), t_);
        const ExtVec &fe = res.second.get_mle_final_evaluations(); ExtVec point = res.first.point;
        Ext cout_eval = fe[0], cin_eval = fe[3]; ExtVec sh(fe.begin() + 5, fe.end());
        Ext combined = n.rq.recombine_claims(cin_eval, sh);
        RequantProof rp; rp.io_accumulation = res.first; rp.clamping_lookup = cp; rp.shifted_lookup = sp;
        ExtVec evs = {cin_eval, cout_eval}; evs.insert(evs.end(), sh.begin(), sh.end());
        std::vector<ProverCommitment> cw = ws[0].commits; cw.insert(cw.end(), ws[1].commits.begin(), ws[1].commits.end());
        for (size_t i = 0; i < evs.size(); i++) { add_witness_claim(cw[i], {point, evs[i]}); rp.accumulation_evals.push_back(evs[i]); rp.commitments.push_back(cw[i].comm.root); }
        proof_.requant[id] = rp;
        return {point, combined};
    }

    // Activation::prove_step (layers/activation.rs:385-460)
    Claim prove_activation(size_t id, const Claim &last_claim) {
        std::vector<LogUpWitness> ws = lookup_witness_.at(id);
        if (ws.size() != 1) throw Error(DP_ERR_INVALID, "Activation only requires a lookup into one table type");
        LogUpProof lp = logup_batch_prove(get_logup_input(ws[0]), t_);
        // the output tensor as an MLE; col_two of the lookup holds the same values (activation.rs:281-283), reuse it
        SamePolyProof acc = same_poly_prove(ws[0].column_evals[1], {last_claim, lp.output_claims[1]}, t_);
        Claim input_claim = lp.output_claims[0];
        ActivationProof ap; ap.io_accumulation = acc; ap.lookup = lp;
        std::vector<Claim> cc = {input_claim, acc.extract_claim()};
        for (size_t i = 0; i < 2; i++) { add_witness_claim(ws[0].commits[i], cc[i]); ap.commits.push_back(ws[0].commits[i].comm.root); }
        proof_.activation[id] = ap;
        return input_claim;
    }

    // Convolution::prove (convolution.rs:609-636) -> prove_convolution_step, then add_common_claims (:1003-1010)
    Claim prove_convolution(size_t id, const Claim &last_claim, const ConvData &pd) {
        ConvProof cp; Claim in_claim = ctx_.convs.at(id).prove_convolution_step(t_, last_claim, pd, cp);
        const auto &comms = ctx_.model_comms.at(id);
        add_witness_claim(comms.at("ConvBias"), cp.bias_poly_claim);                  // BTreeMap order of PolyId
        add_witness_claim(comms.at("ConvFilter"), cp.filter_claim);
        proof_.conv[id] = cp;
        return in_claim;
    }
    // Pooling::prove_pooling (layers/pooling.rs:342-519)
    Claim prove_pooling(size_t id, const Node &n, const Claim &last_claim) {
        std::vector<LogUpWitness> ws = lookup_witness_.at(id);
        if (ws.size() != 1) throw Error(DP_ERR_INVALID, "Pooling only requires a lookup into one table type");
        LogUpInput in = get_logup_input(ws[0]);
        LogUpProof lp = logup_batch_prove(in, t_);
        const ExtVec &lookup_point = lp.output_claims[0].point;
        size_t nv = lookup_point.size(), ks = 4;
        Ext bc = t_.get_and_append_challenge("batch_pooling");
        DeviceMle beta_poly = DeviceMle::build_eq_x_r(lookup_point), last_beta = DeviceMle::build_eq_x_r(last_claim.point);
        std::vector<DeviceMle> diffs = in.column_evals;
        VirtualPolynomial vp(nv);
        { std::vector<DeviceMle> all = diffs; all.push_back(beta_poly); vp.add_mle_list(all, Ext::one()); }   // zerocheck: prod_k (out - in_k) = 0
        Ext comb = bc; for (auto &d : diffs) { vp.add_mle_list({d, beta_poly}, comb); comb *= bc; }
        DeviceMle out_mle = ws[0].commits[ks].poly;
        vp.add_mle_list({out_mle, last_beta}, comb);
        auto res = IOPProverState::prove_parallel(std::move(vp), t_);
        const ExtVec &fe = res.second.get_mle_final_evaluations(); const ExtVec &zc = res.first.point;
        Ext output_eval = fe[ks + 1];
        PoolingProof pp; pp.sumcheck = res.first; pp.lookup = lp;
        for (size_t i = 0; i <= ks; i++) { Ext ev = i < ks ? fe[i] : output_eval; add_witness_claim(ws[0].commits[i], {zc, ev}); pp.commitments.push_back(ws[0].commits[i].comm.root); pp.zerocheck_evals.push_back(ev); }
        size_t lw = ceil_log2(n.pool_w);
        Ext r1 = t_.get_and_append_challenge("input_batching"), r2 = r1;            // `[challenge; 2]` is ONE challenge, copied (pooling.rs:453-456)
        Ext m1 = Ext::one() - r1, m2 = Ext::one() - r2;
        Ext mult[4] = {m1 * m2, m1 * r2, r1 * m2, r1 * r2};
        Ext zc_in = Ext::zero(); for (size_t k = 0; k < ks; k++) zc_in += mult[k] * (output_eval - fe[k]);
        Claim next; next.point.push_back(r1); next.point.insert(next.point.end(), zc.begin(), zc.begin() + (lw - 1));
        next.point.push_back(r2); next.point.insert(next.point.end(), zc.begin() + (lw - 1), zc.end());
        next.eval = zc_in; pp.variable_gap = lw - 1;
        proof_.pooling[id] = pp;
        return next;
    }

    // prove_tables (iop/prover.rs:110-157)
    void prove_tables() {
        for (auto &w : table_witness_) {
            LogUpProof tp = logup_batch_prove(get_logup_input(w), t_);
            add_witness_claim(w.commits[0], tp.output_claims.front());
            proof_.table_proofs.push_back({w.commits[0].comm.root, tp});   // Relu/Range/Clamping have no committed table columns (lookup/context.rs:495-546)
        }
    }

    // CommitmentProver::prove (commit/context.rs:355-418)
    void commit_prove() {
        for (auto &c : trivial_claims_) proof_.trivial_proofs.push_back(Basefold::open(ctx_.pp, c.first.poly, c.first.comm, c.second.point, t_));
        std::vector<DeviceMle> polys; std::vector<BasefoldCommitmentWithWitness> comms; std::vector<ExtVec> points; std::vector<Evaluation> evals;
        for (size_t i = 0; i < claims_.size(); i++) { polys.push_back(claims_[i].first.poly); comms.push_back(claims_[i].first.comm); points.push_back(claims_[i].second.point); Evaluation e; e.poly = i; e.point = i; e.value = claims_[i].second.eval; evals.push_back(e); }
        proof_.batch_proof = Basefold::batch_open(ctx_.pp, polys, comms, points, evals, t_);
    }

    const Context &ctx_; T &t_; Proof proof_;
    std::map<size_t, std::vector<LogUpWitness>> lookup_witness_; std::vector<LogUpWitness> table_witness_;
    Ext constant_challenge_; std::map<TableType, Ext> challenge_map_;
    std::vector<std::pair<ProverCommitment, Claim>> claims_, trivial_claims_;
};

// flat u64 image for the parity tests (layout documented in tests/test_gpu_zkml.py)
inline void flat_e(std::vector<u64> &o, const Ext &e) { o.push_back(e.c0); o.push_back(e.c1); }
inline void flat_iop(std::vector<u64> &o, const IOPProof &p) { o.push_back(p.point.size()); for (auto &e : p.point) flat_e(o, e); o.push_back(p.proofs.size()); for (auto &m : p.proofs) { o.push_back(m.evaluations.size()); for (auto &e : m.evaluations) flat_e(o, e); } }
inline void flat_logup(std::vector<u64> &o, const LogUpProof &p) {
    o.push_back(p.sumcheck_proofs.size()); for (auto &s : p.sumcheck_proofs) flat_iop(o, s);
    o.push_back(p.round_evaluations.size()); for (auto &r : p.round_evaluations) { o.push_back(r.size()); for (auto &e : r) flat_e(o, e); }
    o.push_back(p.output_claims.size()); for (auto &c : p.output_claims) { o.push_back(c.point.size()); for (auto &e : c.point) flat_e(o, e); flat_e(o, c.eval); }
    o.push_back(p.circuit_outputs.size()); for (auto &r : p.circuit_outputs) { o.push_back(r.size()); for (auto &e : r) flat_e(o, e); }
    o.push_back(p.table ? 1 : 0);
}
inline void flat_evec(std::vector<u64> &o, const ExtVec &v) { o.push_back(v.size()); for (auto &e : v) flat_e(o, e); }
// same layout as the CPU checker's flattening: ConvProof field order (convolution.rs:97-121), the two commitment claims, the input claim
inline std::vector<u64> flatten_conv_proof(const ConvProof &p, const Claim &input_claim) {
    std::vector<u64> o;
    flat_iop(o, p.fft_proof); flat_evec(o, p.fft_claims); flat_iop(o, p.fft_proof_weights); flat_iop(o, p.ifft_proof);
    o.push_back(p.fft_delegation.proofs.size()); for (auto &q : p.fft_delegation.proofs) flat_iop(o, q);
    o.push_back(p.fft_delegation_weights.proofs.size()); for (auto &q : p.fft_delegation_weights.proofs) flat_iop(o, q);
    o.push_back(p.ifft_delegation.proofs.size()); for (auto &q : p.ifft_delegation.proofs) flat_iop(o, q);
    flat_iop(o, p.hadamard_proof); flat_evec(o, p.ifft_claims); flat_evec(o, p.fft_weight_claims);
    o.push_back(p.fft_delegation.claims.size()); for (auto &c : p.fft_delegation.claims) flat_evec(o, c);
    o.push_back(p.fft_delegation_weights.claims.size()); for (auto &c : p.fft_delegation_weights.claims) flat_evec(o, c);
    o.push_back(p.ifft_delegation.claims.size()); for (auto &c : p.ifft_delegation.claims) flat_evec(o, c);
    flat_evec(o, p.hadamard_claims); flat_e(o, p.bias_claim); flat_evec(o, p.partial_evals);
    flat_iop(o, p.clearing_proof.sumcheck); flat_evec(o, p.clearing_proof.individual_claim);
    flat_evec(o, p.filter_claim.point); flat_e(o, p.filter_claim.eval); flat_evec(o, p.bias_poly_claim.point); flat_e(o, p.bias_poly_claim.eval);
    flat_evec(o, input_claim.point); flat_e(o, input_claim.eval);
    return o;
}

inline std::vector<u64> Proof::flatten(size_t n_nodes) const {
    std::vector<u64> o;
    auto fd = [&](const Digest &d) { for (int i = 0; i < 4; i++) o.push_back(d.v[i]); };
    for (size_t id = 0; id < n_nodes; id++) {
        if (dense.count(id)) { const auto &d = dense.at(id); o.push_back(100 + id); flat_iop(o, d.sumcheck); flat_e(o, d.bias_eval); o.push_back(d.individual_claims.size()); for (auto &e : d.individual_claims) flat_e(o, e); }
        if (requant.count(id)) { const auto &r = requant.at(id); o.push_back(200 + id); flat_iop(o, r.io_accumulation); o.push_back(r.accumulation_evals.size()); for (auto &e : r.accumulation_evals) flat_e(o, e); flat_logup(o, r.clamping_lookup); flat_logup(o, r.shifted_lookup); o.push_back(r.commitments.size()); for (auto &d : r.commitments) fd(d); }
        if (activation.count(id)) { const auto &a = activation.at(id); o.push_back(300 + id); flat_iop(o, a.io_accumulation.sumcheck); o.push_back(a.io_accumulation.evals.size()); for (auto &e : a.io_accumulation.evals) flat_e(o, e); flat_logup(o, a.lookup); o.push_back(a.commits.size()); for (auto &d : a.commits) fd(d); }
        if (conv.count(id)) { o.push_back(400 + id); std::vector<u64> c = flatten_conv_proof(conv.at(id), Claim()); o.insert(o.end(), c.begin(), c.end()); }
        if (pooling.count(id)) { const auto &q = pooling.at(id); o.push_back(500 + id); flat_iop(o, q.sumcheck); flat_logup(o, q.lookup); flat_evec(o, q.zerocheck_evals); o.push_back(q.variable_gap); o.push_back(q.commitments.size()); for (auto &d : q.commitments) fd(d); }
    }
    o.push_back(table_proofs.size()); for (auto &t : table_proofs) { fd(t.multiplicity_commit); flat_logup(o, t.lookup); }
    o.push_back(trivial_proofs.size());
    std::vector<u64> b = batch_proof.flatten(); o.push_back(b.size()); o.insert(o.end(), b.begin(), b.end());
    return o;
}

}  // namespace zkml
}  // namespace dp
