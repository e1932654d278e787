// Host mirror of the zkml prover for the MLP path (Dense -> Requant -> ReLU chains) over the C ABI.
//   zkml::{Context::generate, Prover::new/.prove} (zkml/src/iop/context.rs:110-215, iop/prover.rs:401-486),
//   prove_tables (:110-157), layers/{dense.rs:423-551, requant.rs:208-330,531-680, activation.rs:238-460},
//   lookup/{context.rs:158-296,464-480,631-781, witness.rs, logup_gkr/prover.rs:24-237},
//   commit/{context.rs:59-190,290-418, same_poly.rs:88-126}.
// Orchestration, Fiat-Shamir, claims bookkeeping and the (tiny) quantised witness columns stay on the host as
// in the reference; every polynomial lives in HBM and every O(n) loop goes through include/deepprove_b200.h.
#pragma once
#include "mpcs.hpp"
#include <optional>
#include <set>
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
struct Model {
    std::vector<Node> nodes; size_t input_len = 0;
    // elements of the last node's output tensor in the padded layout (DeviceTrace::outs.back() of run_device)
    size_t output_len() const {
        size_t len = input_len;
        for (auto &n : nodes) {
            if (n.op == Op::Dense) len = n.nrows;
            else if (n.op == Op::MatMul) len = n.mm_r * n.mm_c;
            else if (n.op == Op::Conv) len = n.kw * n.nw * n.nw;
            else if (n.op == Op::Pool) len = n.pool_c * (n.pool_h / 2) * (n.pool_w / 2);
        }
        return len;
    }
};

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
// A Dense / MatMul / Conv node's model polynomials, committed at setup: `weight` is the dense weight matrix, the MatMul constant
// matrix or the conv filter; `bias` is absent for a MatMul without bias.  Bias goes before weight in the transcript and in the
// claims: the reference keys them by PolyId in a BTreeMap (commit/context.rs:59-103).
struct ModelCommitment { std::optional<ProverCommitment> bias; ProverCommitment weight; };

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
        // CommitmentContext::new (commit/context.rs:59-103); a braced list evaluates in order, so the bias is committed first
        auto commit = [&](const DeviceMle &poly) { return ProverCommitment{Basefold::commit(c.pp, poly), poly}; };
        auto upload = [](const std::vector<Element> &v) { return DeviceMle::from_evaluations_vec(to_base(v)); };
        for (size_t id = 0; id < m.nodes.size(); id++) {
            const Node &n = m.nodes[id];
            if (n.op == Op::Dense) c.model_comms[id] = {commit(upload(n.bias)), commit(upload(n.weights))};
            else if (n.op == Op::MatMul) {   // MatMul::ctx (matrix_mul.rs:951-963): the constant matrix and the bias are model polynomials
                ModelCommitment &mc = c.model_comms[id];
                if (n.mm_bias) mc.bias = commit(upload(n.bias));
                mc.weight = commit(upload(n.weights));
            } else if (n.op == Op::Conv) {   // convolution.rs:532-540
                Convolution cv; cv.kw = n.kw; cv.kx = n.kx; cv.nw = n.nw; cv.real_nw = n.real_nw; cv.filter = n.weights; cv.bias = n.bias;
                for (int i = 0; i < 3; i++) cv.unpadded_out[i] = n.unpadded_out[i];
                cv.load();
                c.model_comms[id] = {commit(upload(n.bias)), commit(cv.filter_mle)};
                c.convs[id] = std::move(cv);
            }
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
    template <class T> void write_to_transcript(T &t) const {   // commit/context.rs:181-190
        for (auto &kv : model_comms) { if (kv.second.bias) Basefold::write_commitment(kv.second.bias->comm.root, t); Basefold::write_commitment(kv.second.weight.comm.root, t); }
    }
    const Model *model = nullptr; BasefoldProverParams pp;
    std::map<size_t, ModelCommitment> model_comms;
    std::map<TableType, TableData> tables;
    std::map<size_t, Convolution> convs;                      // resident conv layers (weights, FFT'd filters)
};

struct LogUpWitness { bool table = false; std::vector<ProverCommitment> commits; std::vector<DeviceMle> column_evals; DeviceMle multiplicity_evals; size_t columns_per_instance = 1; TableType tt{0, 0}; };

// The inference trace on the device: every tensor is a Base MLE of canonical field elements of signed integers (Tensor::to_field),
// so a trace tensor doubles as a lookup column.  Built by run_device only (quantised inference on the device: only the model input
// crosses PCIe); read-only afterwards, shared by concurrent provers.
struct DeviceTrace {
    DeviceMle input; std::vector<DeviceMle> outs; std::map<size_t, ConvData> conv;
    bool valid() const { return input.valid(); }
    const DeviceMle &node_input(size_t id) const { return id == 0 ? input : outs[id - 1]; }
};

// The message of a non-zero lookup error word (dp_wit_finish, dp_infer_run)
inline const char *lookup_error_message(uint32_t bits) {
    return bits & 1 ? "Could not apply requantisation, tensor element had absolute value too large"
                    : "lookup witness: a value is not in its table (clamping / relu / pooling range)";
}

// One lookup-witness pass (csrc/witness.cu): a dp_wit over the Context's tables in TableType order (the reference's BTreeMap
// order), whose histograms the node kernels fill; finish() turns them into the multiplicity polynomials.
class LookupPass {
  public:
    explicit LookupPass(const Context &ctx) {
        std::vector<uint32_t> kinds, sizes;
        for (auto &kv : ctx.tables) { index_[kv.first] = (uint32_t)kinds.size(); kinds.push_back((uint32_t)kv.first.kind); sizes.push_back((uint32_t)kv.first.size); }
        if (!kinds.empty()) check(dp_wit_begin((uint32_t)kinds.size(), kinds.data(), sizes.data(), &w_));
    }
    ~LookupPass() { if (w_) dp_wit_free(w_); }
    LookupPass(const LookupPass &) = delete;
    LookupPass &operator=(const LookupPass &) = delete;

    // The lookup columns of a Requant / ReLU / Maxpool2D node over its input x, in commit order; the node's output is column 1
    // (Requant, ReLU) or 4 (Maxpool2D).
    //   Requant (requant.rs:208-330): the clamping (input, output) pair, then the byte chunks of the shifted-out bits
    //   ReLU (activation.rs:238-323): the node's input and output tensors
    //   Maxpool2D (pooling.rs:210-271, compute_polys :686-771): the four (output - input) differences, then the output
    std::vector<DeviceMle> columns(const Node &n, const DeviceMle &x) {
        if (n.op == Op::Relu) { dp_mle *h; check(dp_wit_relu(w_, x.handle(), table(TableType::relu()), &h)); return {x, DeviceMle(h)}; }
        const Requant &rq = n.rq;
        std::vector<dp_mle *> raw(n.op == Op::Pool ? 5 : 2 + rq.shift() / BIT_LEN, nullptr);
        if (n.op == Op::Requant) check(dp_wit_requant(w_, x.handle(), (uint32_t)rq.shift(), rq.fixed_point_multiplier, (uint32_t)rq.intermediate_bit_size,
                                                      table(TableType::clamping(rq.clamping_size())), table(TableType::range()), raw.data(), (uint32_t)raw.size()));
        else if (n.op == Op::Pool) check(dp_wit_pool(w_, x.handle(), (uint32_t)n.pool_c, (uint32_t)n.pool_h, (uint32_t)n.pool_w, table(TableType::range()), raw.data()));
        else throw Error(DP_ERR_INVALID, "lookup witness: the node has no lookup columns");
        std::vector<DeviceMle> cols; for (dp_mle *h : raw) cols.push_back(DeviceMle(h));
        return cols;
    }
    // the multiplicity polynomial of every table; refuses a trace with a value outside its table
    std::map<TableType, DeviceMle> finish() {
        if (!w_) return {};
        std::vector<dp_mle *> raw(index_.size(), nullptr); uint32_t bits = 0;
        check(dp_wit_finish(w_, raw.data(), &bits));
        std::map<TableType, DeviceMle> mults; for (auto &kv : index_) mults[kv.first] = DeviceMle(raw[kv.second]);
        if (bits) throw Error(DP_ERR_INVALID, lookup_error_message(bits));
        return mults;
    }
  private:
    uint32_t table(const TableType &tt) const { return index_.at(tt); }
    dp_wit *w_ = nullptr; std::map<TableType, uint32_t> index_;
};

// Model::run on the device (Dense / Requant / Relu / Maxpool2D kernels of csrc/witness.cu, the FFT convolution of csrc/conv.cu):
// only the model input crosses PCIe
inline DeviceTrace run_device(const Context &ctx, const std::vector<Element> &input) {
    const Model &m = *ctx.model;
    DeviceTrace tr; tr.input = DeviceMle::from_evaluations_vec(to_base(input));
    LookupPass wit(ctx);
    DeviceMle cur = tr.input;
    for (size_t id = 0; id < m.nodes.size(); id++) {
        const Node &n = m.nodes[id]; DeviceMle o;
        if (n.op == Op::Dense) { const ModelCommitment &c = ctx.model_comms.at(id); dp_mle *h; check(dp_wit_dense(c.weight.poly.handle(), c.bias->poly.handle(), cur.handle(), (uint32_t)n.nrows, (uint32_t)n.ncols, &h)); o = DeviceMle(h); }
        else if (n.op == Op::MatMul) { const ModelCommitment &c = ctx.model_comms.at(id); dp_mle *h; check(dp_wit_matmul(cur.handle(), c.weight.poly.handle(), c.bias ? c.bias->poly.handle() : nullptr, (uint32_t)n.mm_r, (uint32_t)n.mm_k, (uint32_t)n.mm_c, n.mm_t ? 1 : 0, &h)); o = DeviceMle(h); }
        else if (n.op == Op::Conv) { ConvData cd; o = ctx.convs.at(id).op(cur, cd); tr.conv[id] = std::move(cd); }
        else o = wit.columns(n, cur)[n.op == Op::Pool ? 4 : 1];
        tr.outs.push_back(o); cur = o;
    }
    wit.finish();
    return tr;
}

// The model's batch-inference plan (csrc/infer.cu): the nodes as dp_infer_node, handed over once; the device keeps what it needs
class InferPlan {
  public:
    explicit InferPlan(const Model &m) {
        std::vector<dp_infer_node> v(m.nodes.size());
        for (size_t i = 0; i < m.nodes.size(); i++) {
            const Node &n = m.nodes[i]; dp_infer_node &d = v[i];
            d = dp_infer_node{}; d.kind = (uint32_t)n.op;    // Op follows the layer-descriptor kinds
            auto dims = [&](std::initializer_list<size_t> l) { uint32_t k = 0; for (size_t x : l) d.dims[k++] = (uint32_t)x; };
            if (n.op == Op::Dense) dims({n.nrows, n.ncols});
            else if (n.op == Op::Conv) dims({n.kw, n.kx, n.nw, n.real_nw, n.unpadded_out[0], n.unpadded_out[1], n.unpadded_out[2]});
            else if (n.op == Op::Pool) dims({n.pool_c, n.pool_h, n.pool_w});
            else if (n.op == Op::MatMul) dims({n.mm_r, n.mm_k, n.mm_c, n.mm_t ? 1u : 0u});
            else if (n.op == Op::Requant) {
                d.shift = (uint32_t)n.rq.shift(); d.clamp_size = (uint32_t)n.rq.clamping_size();
                d.intermediate_bits = (uint32_t)n.rq.intermediate_bit_size; d.multiplier = n.rq.fixed_point_multiplier;
            }
            d.weights = n.weights.empty() ? nullptr : n.weights.data();
            d.bias = n.bias.empty() ? nullptr : n.bias.data();
        }
        check(dp_infer_plan(v.data(), (uint32_t)v.size(), m.input_len, &p_));
    }
    ~InferPlan() { if (p_) dp_infer_free(p_); }
    InferPlan(const InferPlan &) = delete;
    InferPlan &operator=(const InferPlan &) = delete;
    dp_infer *get() const { return p_; }
  private:
    dp_infer *p_ = nullptr;
};

// Prover<'a, E, T, PCS> (iop/prover.rs:40-60)
template <class T>
class Prover {
  public:
    Prover(const Context &ctx, T &transcript) : ctx_(ctx), t_(transcript) {}

    // end to end from the host input vector: inference on the device, then prove
    Proof prove(const std::vector<Element> &input) { DeviceTrace tr = run_device(ctx_, input); return prove(tr); }
    // Prover::prove(full_trace): the inference trace is an INPUT of proving (zkml/src/bin/bench.rs:390-408 times only this)
    Proof prove(const DeviceTrace &tr) {
        const Model &m = *ctx_.model;
        if (tr.outs.size() != m.nodes.size()) throw Error(DP_ERR_INVALID, "prove: the trace does not match the model");
        ctx_.write_to_transcript(t_);
        instantiate_witness_ctx(m, tr);
        // output claim (prover.rs:423-436)
        const DeviceMle &fo = tr.outs.back();
        Claim last; for (size_t i = 0, nv = fo.num_vars(); i < nv; i++) last.point.push_back(t_.read_challenge());
        last.eval = fo.evaluate(last.point);
        for (size_t id = m.nodes.size(); id-- > 0;) {
            const Node &n = m.nodes[id];
            if (n.op == Op::Dense) last = prove_dense(id, n, last, tr.node_input(id));
            else if (n.op == Op::Requant) last = prove_requant(id, n, last);
            else if (n.op == Op::Relu) last = prove_activation(id, last);
            else if (n.op == Op::Pool) last = prove_pooling(id, n, last);
            else if (n.op == Op::MatMul) last = prove_matmul(id, n, last, tr.node_input(id));
            else last = prove_convolution(id, last, tr.conv.at(id));
        }
        prove_tables();
        commit_prove();
        return std::move(proof_);
    }

  private:
    void add_witness_claim(const ProverCommitment &pc, const Claim &c) { (pc.poly.num_vars() <= Basefold::trivial_num_vars() ? trivial_claims_ : claims_).push_back({pc, c}); }   // commit/context.rs:290-310
    // a node's model-polynomial claims, bias first (ModelCommitment); a MatMul without bias has no bias claim
    void add_model_claims(size_t id, const Claim &bias, const Claim &weight) {
        const ModelCommitment &mc = ctx_.model_comms.at(id);
        if (mc.bias) add_witness_claim(*mc.bias, bias);
        add_witness_claim(mc.weight, weight);
    }

    // generate_lookup_witnesses (lookup/context.rs:631-756) + initialise_from_table_set (:758-781).
    // The reference commits every witness column from rayon workers before any challenge is drawn; here all
    // columns are gathered first and committed with ONE Basefold::commit_many call (concurrent on the device).
    void instantiate_witness_ctx(const Model &m, const DeviceTrace &tr) {
        std::vector<DeviceMle> polys;                            // every column to commit, in creation order (all device-resident)
        struct Slot { size_t node; size_t witness; bool table; bool column = true; };  // where commitment k goes (column: also a lookup column)
        std::vector<Slot> slots;
        LookupPass wit(ctx_);
        std::set<TableType> used;
        auto witness = [&](TableType tt, size_t columns_per_instance) { LogUpWitness w; w.tt = tt; w.columns_per_instance = columns_per_instance; used.insert(tt); return w; };
        for (size_t id = 0; id < m.nodes.size(); id++) {
            const Node &n = m.nodes[id];
            if (n.op != Op::Requant && n.op != Op::Relu && n.op != Op::Pool) continue;
            const std::vector<DeviceMle> c = wit.columns(n, tr.node_input(id));
            auto add = [&](size_t k, size_t which, bool column = true) { polys.push_back(c[k]); slots.push_back({id, which, false, column}); };
            if (n.op == Op::Requant) {   // the clamping (input, output) pair goes to the clamping table, the byte chunks to the range table
                lookup_witness_[id] = {witness(TableType::clamping(n.rq.clamping_size()), 2), witness(TableType::range(), 1)};
                for (size_t k = 0; k < c.size(); k++) add(k, k < 2 ? 0 : 1);
            } else if (n.op == Op::Relu) {
                lookup_witness_[id] = {witness(TableType::relu(), 2)};
                add(0, 0); add(1, 0);
            } else {
                lookup_witness_[id] = {witness(TableType::range(), 1)};
                for (size_t k = 0; k < 4; k++) add(k, 0);
                add(4, 0, false);   // the output poly: committed, not a lookup column
            }
        }
        // table multiplicities (lookup/context.rs:675-737): histograms the node kernels filled, every table row distinct
        std::map<TableType, DeviceMle> mults = wit.finish();
        std::vector<TableType> table_order;
        for (auto &kv : ctx_.tables) {
            if (!used.count(kv.first)) continue;
            for (auto &tc : kv.second.table_count) if (tc.second != 1) throw Error(DP_ERR_UNSUPPORTED, "device multiplicities need distinct table rows");
            LogUpWitness w; w.table = true; w.tt = kv.first; w.column_evals = kv.second.columns;
            table_witness_.push_back(w); table_order.push_back(kv.first);
            polys.push_back(mults.at(kv.first)); slots.push_back({0, table_witness_.size() - 1, true});
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
        const ModelCommitment &mc = ctx_.model_comms.at(id);
        const DeviceMle &weights = mc.weight.poly, &bias = mc.bias->poly;
        if (ceil_log2(n.nrows) != last_claim.point.size()) throw Error(DP_ERR_INVALID, "something's wrong with the randomness");
        Ext bias_eval = bias.evaluate(last_claim.point);
        DeviceMle mat = weights.fix_high_variables(last_claim.point);      // rows are the HIGH variables (dense.rs:471-475)
        const DeviceMle &in = input;                                        // the trace tensor itself (a sumcheck borrows its inputs)
        VirtualPolynomial vp(in.num_vars());
        vp.add_mle_list({mat, in}, Ext::one());
        auto res = IOPProverState::prove_parallel(std::move(vp), t_);
        const ExtVec &fe = res.second.get_mle_final_evaluations();
        ExtVec wp = res.first.point; wp.insert(wp.end(), last_claim.point.begin(), last_claim.point.end());
        add_model_claims(id, {last_claim.point, bias_eval}, {wp, fe[0]});
        proof_.dense[id] = {res.first, bias_eval, fe};
        return {res.first.point, fe[1]};
    }

    // MatMul::prove_step (layers/matrix_mul.rs:701-874) for Input x Weight: the output claim splits into the row part (fixes the HIGH variables of
    // the left = input matrix) and the column part (fixes the LOW variables of the constant matrix, or its HIGH ones when it is stored
    // transposed); one degree-2 sumcheck over the shared inner dimension; the left evaluation is the claim handed to the previous node
    Claim prove_matmul(size_t id, const Node &n, const Claim &last_claim, const DeviceMle &input) {
        const ModelCommitment &mc = ctx_.model_comms.at(id);
        const size_t vr = ceil_log2(n.mm_r), vc = ceil_log2(n.mm_c), vk = ceil_log2(n.mm_k);
        if (last_claim.point.size() != vr + vc) throw Error(DP_ERR_INVALID, "Wrong length of last claim point");
        const ExtVec p_right(last_claim.point.begin(), last_claim.point.begin() + vc), p_left(last_claim.point.begin() + vc, last_claim.point.end());   // split_claim
        Ext bias_eval = Ext::zero();
        if (mc.bias) bias_eval = mc.bias->poly.evaluate(p_right);
        DeviceMle left = input.fix_high_variables(p_left);
        const DeviceMle &w = mc.weight.poly;
        DeviceMle right = n.mm_t ? w.fix_high_variables(p_right) : w.fix_variables(p_right);
        if (left.num_vars() != vk || right.num_vars() != vk) throw Error(DP_ERR_INVALID, "matmul: free variables of the two matrices differ");
        VirtualPolynomial vp(vk);
        vp.add_mle_list({left, right}, Ext::one());
        auto res = IOPProverState::prove_parallel(std::move(vp), t_);
        const ExtVec &fe = res.second.get_mle_final_evaluations();
        ExtVec pl = res.first.point; pl.insert(pl.end(), p_left.begin(), p_left.end());                      // full_points
        ExtVec pr;
        if (n.mm_t) { pr = res.first.point; pr.insert(pr.end(), p_right.begin(), p_right.end()); } else { pr = p_right; pr.insert(pr.end(), res.first.point.begin(), res.first.point.end()); }
        add_model_claims(id, {p_right, bias_eval}, {pr, fe[1]});
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
        add_model_claims(id, cp.bias_poly_claim, cp.filter_claim);
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

// flat u64 images for the parity tests, word for word the CPU checker's
inline void flat_logup(ProofImage &w, const LogUpProof &p) {
    w.put(p.sumcheck_proofs.size()); for (auto &s : p.sumcheck_proofs) w.iop(s);
    w.put(p.round_evaluations.size()); for (auto &r : p.round_evaluations) w.exts(r);
    w.put(p.output_claims.size()); for (auto &c : p.output_claims) { w.exts(c.point); w.ext(c.eval); }
    w.put(p.circuit_outputs.size()); for (auto &r : p.circuit_outputs) w.exts(r);
    w.put(p.table ? 1 : 0);
}
// ConvProof field order (convolution.rs:97-121), the two commitment claims, the input claim
inline void flatten_conv_proof(ProofImage &w, const ConvProof &p, const Claim &input_claim) {
    const MatrixEvalProof *delegations[3] = {&p.fft_delegation, &p.fft_delegation_weights, &p.ifft_delegation};
    w.iop(p.fft_proof); w.exts(p.fft_claims); w.iop(p.fft_proof_weights); w.iop(p.ifft_proof);
    for (auto *d : delegations) { w.put(d->proofs.size()); for (auto &q : d->proofs) w.iop(q); }
    w.iop(p.hadamard_proof); w.exts(p.ifft_claims); w.exts(p.fft_weight_claims);
    for (auto *d : delegations) { w.put(d->claims.size()); for (auto &c : d->claims) w.exts(c); }
    w.exts(p.hadamard_claims); w.ext(p.bias_claim); w.exts(p.partial_evals);
    w.iop(p.clearing_proof.sumcheck); w.exts(p.clearing_proof.individual_claim);
    w.exts(p.filter_claim.point); w.ext(p.filter_claim.eval); w.exts(p.bias_poly_claim.point); w.ext(p.bias_poly_claim.eval);
    w.exts(input_claim.point); w.ext(input_claim.eval);
}

inline std::vector<u64> Proof::flatten(size_t n_nodes) const {
    ProofImage w;
    for (size_t id = 0; id < n_nodes; id++) {
        if (dense.count(id)) { const auto &d = dense.at(id); w.put(100 + id); w.iop(d.sumcheck); w.ext(d.bias_eval); w.exts(d.individual_claims); }
        if (requant.count(id)) { const auto &r = requant.at(id); w.put(200 + id); w.iop(r.io_accumulation); w.exts(r.accumulation_evals); flat_logup(w, r.clamping_lookup); flat_logup(w, r.shifted_lookup); w.put(r.commitments.size()); for (auto &d : r.commitments) w.digest(d); }
        if (activation.count(id)) { const auto &a = activation.at(id); w.put(300 + id); w.iop(a.io_accumulation.sumcheck); w.exts(a.io_accumulation.evals); flat_logup(w, a.lookup); w.put(a.commits.size()); for (auto &d : a.commits) w.digest(d); }
        if (conv.count(id)) { w.put(400 + id); flatten_conv_proof(w, conv.at(id), Claim()); }
        if (pooling.count(id)) { const auto &q = pooling.at(id); w.put(500 + id); w.iop(q.sumcheck); flat_logup(w, q.lookup); w.exts(q.zerocheck_evals); w.put(q.variable_gap); w.put(q.commitments.size()); for (auto &d : q.commitments) w.digest(d); }
    }
    w.put(table_proofs.size()); for (auto &t : table_proofs) { w.digest(t.multiplicity_commit); flat_logup(w, t.lookup); }
    w.put(trivial_proofs.size());
    std::vector<u64> b = batch_proof.flatten(); w.put(b.size()); w.words.insert(w.words.end(), b.begin(), b.end());
    return w.words;
}

}  // namespace zkml
}  // namespace dp
