// Host mirror of the reference's `mpcs` crate for the configured scheme
//   Basefold<GoldilocksExt2, BasefoldRSParams<PoseidonHasher>>   (zkml/src/bin/bench.rs:25)
// over the C ABI: trait PolynomialCommitmentScheme<E> {setup, trim, commit, write_commitment,
// get_pure_commitment, trivial_num_vars, open, batch_open} (mpcs/src/lib.rs:111-226).  Fiat-Shamir and the
// proof structs live here on the host; every O(n) loop (interpolation, RS encode, Merkle, FRI fold,
// sumchecks, query gather) runs on the device.  Errors mirror mpcs::Error (lib.rs:306-328) as dp::Error.
#pragma once
#include "sumcheck.hpp"

namespace dp {

struct Digest { u64 v[4] = {0, 0, 0, 0}; bool operator==(const Digest &o) const { return !memcmp(v, o.v, 32); } };

constexpr uint32_t RS_NUM_QUERIES = 200, RS_RATE_LOG = 1, RS_BASECODE_MSG_SIZE_LOG = 7;  // encoding/rs.rs:204-214

// BasefoldParams / ProverParams: only the trimmed maximum message size matters to the prover (rs.rs:222-227)
struct BasefoldProverParams { uint32_t full_message_size_log = 0; };
inline uint32_t log2_strict(u64 n) { uint32_t l = 0; while ((1ULL << l) < n) l++; if ((1ULL << l) != n) throw Error(DP_ERR_INVALID, "log2_strict: not a power of two"); return l; }

class BasefoldCommitmentWithWitness {
  public:
    BasefoldCommitmentWithWitness() {}
    explicit BasefoldCommitmentWithWitness(dp_pcs_comm *h) : h_(h, [](dp_pcs_comm *p) { dp_pcs_comm_free(p); }) {
        int b, t; check(dp_pcs_comm_info(h, &num_vars, &b, &t, root.v)); is_base = b; trivial = t;
    }
    dp_pcs_comm *handle() const { return h_.get(); }
    uint32_t num_vars = 0; bool is_base = true, trivial = false; Digest root;
    uint32_t num_polys() const { return dp_pcs_comm_num_polys(h_.get()); }
    u64 codeword_size() const { return trivial ? (1ULL << num_vars) : (1ULL << (num_vars + RS_RATE_LOG)); }
  private:
    std::shared_ptr<dp_pcs_comm> h_;
};

struct CodewordQuery { Ext p0, p1; u64 index = 0; bool is_base = false; std::vector<Digest> merkle_path; };
struct SingleQueryResult { u64 x_index = 0; CodewordQuery commitment_query; std::vector<CodewordQuery> oracle_query; };
struct BatchedQueryResult { u64 x_index = 0; std::vector<CodewordQuery> oracle_query, commitments_query; };

// Writer of the flat u64 proof images the parity tests compare word for word with the CPU checker's flatteners
struct ProofImage {
    std::vector<u64> words;
    void put(u64 w) { words.push_back(w); }
    void ext(const Ext &e) { put(e.c0); put(e.c1); }
    void exts(const ExtVec &v) { put(v.size()); for (auto &e : v) ext(e); }        // length, then the elements
    void digest(const Digest &d) { for (u64 w : d.v) put(w); }
    void query(const CodewordQuery &q) {                                            // a base-field leaf pair as one word per leaf
        put(q.index); put(q.is_base ? 1 : 0);
        if (q.is_base) { put(q.p0.c0); put(q.p1.c0); } else { ext(q.p0); ext(q.p1); }
        put(q.merkle_path.size()); for (auto &d : q.merkle_path) digest(d);
    }
    void iop(const IOPProof &p) { exts(p.point); put(p.proofs.size()); for (auto &m : p.proofs) exts(m.evaluations); }
};

// BasefoldProof (structure.rs:329-345)
struct BasefoldProof {
    std::vector<ExtVec> sumcheck_messages;
    std::vector<Digest> roots;
    ExtVec final_message;
    std::vector<SingleQueryResult> single_queries;      // ProofQueriesResultWithMerklePath::Single
    std::vector<BatchedQueryResult> batched_queries;    // ::Batched
    std::vector<ExtVec> sumcheck_proof;                 // Option<SumcheckProof<Coefficients>>: 3 coefficients per round
    bool is_trivial = false; std::vector<u64> trivial_proof; bool trivial_is_ext = false;
    // flat u64 image used by the parity tests (layout documented in tests/test_oracle_basefold.py parse_flat)
    std::vector<u64> flatten() const {
        ProofImage w;
        w.put(sumcheck_proof.size()); for (auto &m : sumcheck_proof) for (auto &e : m) w.ext(e);
        w.put(sumcheck_messages.size()); for (auto &m : sumcheck_messages) for (auto &e : m) w.ext(e);
        w.put(roots.size()); for (auto &d : roots) w.digest(d);
        w.exts(final_message);
        w.put(single_queries.size());
        for (auto &q : single_queries) { w.put(q.x_index); w.query(q.commitment_query); w.put(q.oracle_query.size()); for (auto &x : q.oracle_query) w.query(x); }
        w.put(batched_queries.size());
        for (auto &q : batched_queries) { w.put(q.x_index); w.put(q.oracle_query.size()); for (auto &x : q.oracle_query) w.query(x); w.put(q.commitments_query.size()); for (auto &x : q.commitments_query) w.query(x); }
        return w.words;
    }
};

// ProofQueriesResultWithMerklePath::SimpleBatched (query_phase.rs:1420-1560): every committed polynomial's leaf pair + ONE path
struct SimpleBatchQueryResult { u64 x_index = 0, index = 0; bool is_base = false; ExtVec left, right; std::vector<Digest> merkle_path; std::vector<CodewordQuery> oracle_query; };
struct SimpleBatchProof {
    std::vector<ExtVec> sumcheck_messages; std::vector<Digest> roots; ExtVec final_message; std::vector<SimpleBatchQueryResult> queries;
    bool is_trivial = false;
    std::vector<u64> flatten() const {   // same image as the CPU checker's flatten_simple_batch_proof
        ProofImage w;
        w.put(sumcheck_messages.size()); for (auto &m : sumcheck_messages) for (auto &e : m) w.ext(e);
        w.put(roots.size()); for (auto &d : roots) w.digest(d);
        w.exts(final_message);
        w.put(queries.size());
        for (auto &q : queries) {
            w.put(q.x_index); w.put(q.index); w.put(q.is_base ? 1 : 0); w.put(q.left.size());
            for (size_t k = 0; k < q.left.size(); k++) { if (q.is_base) { w.put(q.left[k].c0); w.put(q.right[k].c0); } else { w.ext(q.left[k]); w.ext(q.right[k]); } }
            w.put(q.merkle_path.size()); for (auto &d : q.merkle_path) w.digest(d);
            w.put(q.oracle_query.size()); for (auto &x : q.oracle_query) w.query(x);
        }
        return w.words;
    }
};

struct Evaluation { size_t poly = 0, point = 0; Ext value; };

inline Ext eq_xy_eval(const ExtVec &x, const ExtVec &y) {
    Ext r = Ext::one();
    for (size_t i = 0; i < x.size(); i++) { Ext xy = x[i] * y[i]; r *= xy + xy + Ext::one() - x[i] - y[i]; }
    return r;
}
inline ExtVec build_eq_x_r_vec_host(const ExtVec &r) {   // small tables only (batch coefficients)
    ExtVec buf(1ULL << r.size()); buf[0] = Ext::one();
    size_t i = 0;
    for (size_t k = r.size(); k-- > 0; i++) for (size_t idx = (1ULL << (i + 1)); idx >= 2; idx -= 2) { Ext prev = buf[(idx - 2) >> 1], t = r[k] * prev; buf[idx - 1] = t; buf[idx - 2] = prev - t; }
    return buf;
}

class Basefold {
  public:
    // setup + trim (basefold.rs:279-301): the RS tables are recomputed on the device, only the size is kept
    static BasefoldProverParams setup_and_trim(u64 poly_size) { BasefoldProverParams p; p.full_message_size_log = log2_strict(poly_size); return p; }
    static uint32_t trivial_num_vars() { return RS_BASECODE_MSG_SIZE_LOG; }

    static BasefoldCommitmentWithWitness commit(const BasefoldProverParams &pp, const DeviceMle &poly) {
        dp_pcs_comm *h; check(dp_pcs_commit(poly.handle(), pp.full_message_size_log, &h));
        return BasefoldCommitmentWithWitness(h);
    }
    static std::vector<BasefoldCommitmentWithWitness> commit_many(const BasefoldProverParams &pp, const std::vector<DeviceMle> &polys) {
        std::vector<dp_mle *> hs; for (auto &p : polys) hs.push_back(p.handle());
        std::vector<dp_pcs_comm *> cs(polys.size(), nullptr);
        if (!polys.empty()) check(dp_pcs_commit_many(hs.data(), (uint32_t)hs.size(), pp.full_message_size_log, cs.data()));
        std::vector<BasefoldCommitmentWithWitness> out; for (auto *c : cs) out.push_back(BasefoldCommitmentWithWitness(c));
        return out;
    }
    template <class T> static void write_commitment(const Digest &root, T &t) { for (int i = 0; i < 4; i++) t.append_field_element(root.v[i]); }

    // Basefold::commit of one polynomial sharded over the ranks of `ex` (every rank holds the polynomial; csrc/basefold.cu
    // dp_pcs_commit_shard): the one exchange is the all-gather of the 32-byte subtree roots.  Same root as commit().
    static BasefoldCommitmentWithWitness commit_sharded(const BasefoldProverParams &pp, const DeviceMle &poly, Exchange &ex) {
        dp_pcs_comm *h; check(dp_pcs_commit_shard(poly.handle(), pp.full_message_size_log, (uint32_t)ex.rank, (uint32_t)ex.world, &h));
        BasefoldCommitmentWithWitness c(h);      // c.root = this rank's subtree root for now
        std::vector<u64> all(4 * ex.world);
        ex.allgather(c.root.v, 4, all.data());
        check(dp_pcs_comm_set_shard_roots(h, all.data(), c.root.v));
        return c;
    }
    // Basefold::open of a sharded commitment: the proof of open() on the unsharded polynomial, identical on every rank
    template <class T>
    static BasefoldProof open_sharded(const BasefoldProverParams &pp, const BasefoldCommitmentWithWitness &comm, const ExtVec &point, T &transcript, Exchange &ex) {
        (void)pp;
        BasefoldProof pr;
        dp_pcs_comm *cs[1] = {comm.handle()};
        run_commit_phase(cs, nullptr, 1, point, comm.num_vars, transcript, pr, /*batch=*/false, {comm.codeword_size()}, {comm.is_base}, &ex);
        return pr;
    }

    // Basefold::open (basefold.rs:466-539)
    template <class T>
    static BasefoldProof open(const BasefoldProverParams &pp, const DeviceMle &poly, const BasefoldCommitmentWithWitness &comm, const ExtVec &point, T &transcript) {
        BasefoldProof pr;
        if (comm.trivial) { pr.is_trivial = true; pr.trivial_proof = poly.download(); pr.trivial_is_ext = poly.is_ext(); return pr; }   // Proof::trivial(evals)
        (void)pp;
        dp_pcs_comm *cs[1] = {comm.handle()};
        run_commit_phase(cs, nullptr, 1, point, comm.num_vars, transcript, pr, /*batch=*/false, {comm.codeword_size()}, {comm.is_base});
        return pr;
    }

    // Basefold::batch_open (basefold.rs:546-770)
    template <class T>
    static BasefoldProof batch_open(const BasefoldProverParams &pp, const std::vector<DeviceMle> &polys, const std::vector<BasefoldCommitmentWithWitness> &comms,
                                    const std::vector<ExtVec> &points, const std::vector<Evaluation> &evals, T &transcript) {
        BasefoldProof pr;
        if (polys.empty() && comms.empty() && points.empty() && evals.empty()) { pr.is_trivial = true; return pr; }
        uint32_t num_vars = 0, min_nv = UINT32_MAX;
        for (auto &p : polys) { num_vars = std::max(num_vars, p.num_vars()); min_nv = std::min(min_nv, p.num_vars()); }
        if (min_nv <= RS_BASECODE_MSG_SIZE_LOG) throw Error(DP_ERR_INVALID, "minimum number of variables must be greater than basecode_msg_size_log");
        for (auto &c : comms) if (c.trivial) throw Error(DP_ERR_INVALID, "batch_open: trivial commitment");
        if (num_vars > pp.full_message_size_log) throw Error(DP_ERR_INVALID, "batch open: polynomial larger than the parameters");
        size_t bsl = 0; while ((1ULL << bsl) < evals.size()) bsl++;
        ExtVec t; for (size_t i = 0; i < bsl; i++) t.push_back(transcript.get_and_append_challenge("batch coeffs"));
        ExtVec eq_xt = build_eq_x_r_vec_host(t);
        Ext target = Ext::zero();
        for (size_t i = 0; i < evals.size(); i++) target += evals[i].value * Ext::from_base(canon(1ULL << (num_vars - points[evals[i].point].size()))) * eq_xt[i];
        // merged polynomials (basefold.rs:617-640): the reference forms sum_i eq_xt[i] * poly_i per point.  The sumcheck message
        // is linear in the polynomial, so one product (eq(point_k), poly_i) with coefficient eq_xt[i] PER EVALUATION gives the
        // identical messages without materialising the merge; the point's eq table is shared (folded once) by all its products.
        // ClassicSumCheck<CoefficientsProver>::prove (sum_check/classic.rs:230-285, classic/coeff.rs:196-345):
        // LSB-first, 3 coefficients per round with c1 from the running sum
        VirtualPolynomial vp(num_vars);
        std::vector<DeviceMle> eqs;
        for (size_t k = 0; k < points.size(); k++) eqs.push_back(DeviceMle::build_eq_x_r(points[k]));
        std::vector<bool> used(points.size(), false);
        for (size_t i = 0; i < evals.size(); i++) {
            if (evals[i].point >= points.size() || evals[i].poly >= polys.size()) throw Error(DP_ERR_INVALID, "batch_open: evaluation refers to a missing polynomial / point");
            if (polys[evals[i].poly].num_vars() != points[evals[i].point].size()) throw Error(DP_ERR_INVALID, "batch_open: point length != polynomial num_vars");   // basefold.rs:575-580
            vp.add_mle_list({eqs[evals[i].point], polys[evals[i].poly]}, eq_xt[i]);
            used[evals[i].point] = true;
        }
        for (bool u : used) if (!u) throw Error(DP_ERR_INVALID, "batch_open: point without evaluation");
        std::vector<dp_mle *> hs; for (auto &m : vp.flattened_ml_extensions) hs.push_back(m.handle());
        dp_sc *sc = nullptr;
        check(dp_sc_create(hs.data(), (uint32_t)hs.size(), vp.products.data(), (uint32_t)vp.products.size(), num_vars, 2, &sc));
        std::shared_ptr<dp_sc> guard(sc, [](dp_sc *p) { dp_sc_destroy(p); });
        check(dp_sc_set_resident_tail(sc, 1));
        Ext sum = target, ch; bool have = false; ExtVec challenges;
        const u64 inv2 = 0x7FFFFFFF80000001ULL;
        for (uint32_t round = 0; round < num_vars; round++) {
            u64 ev[6], c[2] = {ch.c0, ch.c1};
            check(dp_sc_round(sc, have ? c : nullptr, ev));
            Ext p0(ev[0], ev[1]), p1(ev[2], ev[3]), p2(ev[4], ev[5]);
            Ext c0 = p0, c2 = (p2 - (p1 + p1) + p0) * inv2;
            Ext c1 = sum - (c0 + c0) - c2;                                   // coeff.rs:218
            ExtVec msg = {c0, c1, c2};
            transcript.append_field_element_exts(msg);
            pr.sumcheck_proof.push_back(msg);
            ch = transcript.get_and_append_challenge("sumcheck round"); have = true;
            challenges.push_back(ch);
            sum = c0 + ch * (c1 + ch * c2);                                  // horner (Coefficients::evaluate)
        }
        guard.reset();
        // coeffs[poly] = sum_i eq_xy(point_i, challenges[..|point_i|]) * eq_xt[i]   (basefold.rs:690-701)
        ExtVec coeffs(comms.size(), Ext::zero());
        for (size_t i = 0; i < evals.size(); i++) {
            const ExtVec &pt = points[evals[i].point];
            coeffs[evals[i].poly] += eq_xy_eval(ExtVec(challenges.begin(), challenges.begin() + pt.size()), pt) * eq_xt[i];
        }
        std::vector<dp_pcs_comm *> cs; std::vector<u64> cw; std::vector<bool> isb;
        for (auto &c : comms) { cs.push_back(c.handle()); cw.push_back(c.codeword_size()); isb.push_back(c.is_base); }
        run_commit_phase(cs.data(), &coeffs, (uint32_t)cs.size(), challenges, num_vars, transcript, pr, /*batch=*/true, cw, isb);
        return pr;
    }

    // Basefold::batch_commit (basefold.rs:356-452)
    static BasefoldCommitmentWithWitness batch_commit(const BasefoldProverParams &pp, const std::vector<DeviceMle> &polys) {
        std::vector<dp_mle *> hs; for (auto &p : polys) hs.push_back(p.handle());
        dp_pcs_comm *h; check(dp_pcs_batch_commit(hs.data(), (uint32_t)hs.size(), pp.full_message_size_log, &h));
        return BasefoldCommitmentWithWitness(h);
    }
    // Basefold::simple_batch_open (basefold.rs:777-861): all polynomials of one batch commitment at ONE point.  The commit phase is
    // the batch commit phase over the per-polynomial views with coefficients eq(t) (simple_batch_commit_phase, commit_phase.rs:363-510)
    template <class T>
    static SimpleBatchProof simple_batch_open(const BasefoldProverParams &pp, const BasefoldCommitmentWithWitness &comm, const ExtVec &point, const ExtVec &evals, T &transcript) {
        (void)pp;
        SimpleBatchProof sp;
        if (comm.trivial) { sp.is_trivial = true; return sp; }                       // Proof::trivial(bh_evals): the caller holds the evaluations
        uint32_t n = comm.num_polys();
        if (n != evals.size() || point.size() != comm.num_vars) throw Error(DP_ERR_INVALID, "simple_batch_open: one evaluation per committed polynomial at a num_vars-long point");
        size_t bsl = 0; while ((1ULL << bsl) < evals.size()) bsl++;
        ExtVec t; for (size_t i = 0; i < bsl; i++) t.push_back(transcript.get_and_append_challenge("batch coeffs"));
        ExtVec eq_xt = build_eq_x_r_vec_host(t); eq_xt.resize(evals.size());
        std::vector<dp_pcs_comm *> cs; std::vector<u64> cw; std::vector<bool> isb;
        for (uint32_t i = 0; i < n; i++) { const dp_pcs_comm *part; check(dp_pcs_comm_part(comm.handle(), i, &part)); cs.push_back(const_cast<dp_pcs_comm *>(part)); cw.push_back(comm.codeword_size()); isb.push_back(comm.is_base); }
        BasefoldProof pr;
        run_commit_phase(cs.data(), &eq_xt, n, point, comm.num_vars, transcript, pr, /*batch=*/true, cw, isb);
        sp.sumcheck_messages = pr.sumcheck_messages; sp.roots = pr.roots; sp.final_message = pr.final_message;
        for (auto &b : pr.batched_queries) {
            SimpleBatchQueryResult q; q.x_index = b.x_index; q.index = b.commitments_query[0].index; q.is_base = comm.is_base;
            for (auto &c : b.commitments_query) { q.left.push_back(c.p0); q.right.push_back(c.p1); }
            q.merkle_path = b.commitments_query[0].merkle_path;                        // one tree: every view authenticates with the same path
            q.oracle_query = b.oracle_query;
            sp.queries.push_back(q);
        }
        return sp;
    }

  private:
    template <class T>
    // `ex` != null (sharded opening, one commitment from dp_pcs_commit_shard per rank): the device calls return this rank's partial
    // messages / subtree roots / query rows; every rank combines them through `ex` and runs the same transcript, so all ranks end
    // with the identical proof -- the proof of the unsharded polynomial.
    static void run_commit_phase(dp_pcs_comm *const *cs, const ExtVec *coeffs, uint32_t n, const ExtVec &point, uint32_t num_vars, T &transcript,
                                 BasefoldProof &pr, bool batch, const std::vector<u64> &cw_sizes, const std::vector<bool> &is_base, Exchange *ex = nullptr) {
        if (point.size() != num_vars) throw Error(DP_ERR_INVALID, "open: point length does not match num_vars");
        auto pf = flatten(point);
        std::vector<u64> cf; if (coeffs) cf = flatten(*coeffs);
        dp_pcs_open *o = nullptr; u64 m[6];
        check(dp_pcs_open_begin(cs, coeffs ? cf.data() : nullptr, n, pf.data(), num_vars, &o, m));
        std::shared_ptr<dp_pcs_open> guard(o, [](dp_pcs_open *p) { dp_pcs_open_free(p); });
        uint32_t num_rounds = num_vars - RS_BASECODE_MSG_SIZE_LOG;
        const size_t W = ex ? ex->world : 1;
        auto sum_msgs = [&](const std::vector<u64> &all, size_t stride, u64 *out6) {     // add the ranks' coefficient triples mod p
            for (int k = 0; k < 3; k++) { Ext s = Ext::zero(); for (size_t g = 0; g < W; g++) s += Ext(all[g * stride + 2 * k], all[g * stride + 2 * k + 1]); out6[2 * k] = s.c0; out6[2 * k + 1] = s.c1; }
        };
        if (ex) { std::vector<u64> all(6 * W); ex->allgather(m, 6, all.data()); sum_msgs(all, 6, m); }
        ExtVec last = {Ext(m[0], m[1]), Ext(m[2], m[3]), Ext(m[4], m[5])};
        for (uint32_t i = 0; i < num_rounds; i++) {
            transcript.append_field_element_exts(last);
            pr.sumcheck_messages.push_back(last);
            Ext ch = transcript.get_and_append_challenge("commit round");
            u64 c[2] = {ch.c0, ch.c1}, nm[6]; Digest root; int is_last = 0;
            check(dp_pcs_open_round(o, c, nm, root.v, &is_last));
            if (ex && !is_last) {   // partial message + subtree root of every rank -> the message and the oracle's root
                u64 send[10]; memcpy(send, nm, 48); memcpy(send + 6, root.v, 32);
                std::vector<u64> all(10 * W); ex->allgather(send, 10, all.data());
                sum_msgs(all, 10, nm);
                std::vector<u64> roots(4 * W); for (size_t g = 0; g < W; g++) memcpy(&roots[4 * g], &all[10 * g + 6], 32);
                check(dp_pcs_open_set_shard_roots(o, roots.data(), root.v));
            }
            if (!is_last) {
                last = {Ext(nm[0], nm[1]), Ext(nm[2], nm[3]), Ext(nm[4], nm[5])};
                for (int k = 0; k < 4; k++) transcript.append_field_element(root.v[k]);    // digest_to_transcript
                pr.roots.push_back(root);
            } else {
                std::vector<u64> fm(2ULL << RS_BASECODE_MSG_SIZE_LOG);
                check(dp_pcs_open_final_message(o, fm.data()));
                if (ex) {   // the ranks' slices of the bit-reversed message, rank-major, then un-bit-reverse (commit_phase.rs:132-146)
                    const size_t per = fm.size() / W;
                    std::vector<u64> all(fm.size()); ex->allgather(fm.data(), per, all.data());
                    for (u64 k = 0; k < (1ULL << RS_BASECODE_MSG_SIZE_LOG); k++) { u64 j = 0; for (uint32_t b = 0; b < RS_BASECODE_MSG_SIZE_LOG; b++) if (k >> b & 1) j |= 1ULL << (RS_BASECODE_MSG_SIZE_LOG - 1 - b); fm[2 * j] = all[2 * k]; fm[2 * j + 1] = all[2 * k + 1]; }
                }
                for (size_t k = 0; k < fm.size() / 2; k++) pr.final_message.push_back(Ext(fm[2 * k], fm[2 * k + 1]));
                transcript.append_field_element_exts(pr.final_message);
            }
        }
        // query phase (query_phase.rs:31-101): indices from the transcript, gather on the device
        u64 codeword_size = 1ULL << (num_vars + RS_RATE_LOG);
        std::vector<u64> xs;
        for (uint32_t q = 0; q < RS_NUM_QUERIES; q++) xs.push_back(transcript.get_and_append_challenge("query indices").c0 % codeword_size);
        u64 words = dp_pcs_open_query_words(o);
        std::vector<u64> buf(words * xs.size());
        check(dp_pcs_open_query(o, xs.data(), (uint32_t)xs.size(), buf.data()));
        if (ex) {   // every row is filled by the one rank that owns its leaf pair: the word-wise sum of the ranks' buffers is the full gather
            std::vector<u64> all(buf.size() * W); ex->allgather(buf.data(), buf.size(), all.data());
            for (size_t i = 0; i < buf.size(); i++) { u64 s = 0; for (size_t g = 0; g < W; g++) s += all[g * buf.size() + i]; buf[i] = s; }
        }
        uint32_t lgN = num_vars + RS_RATE_LOG;
        for (size_t q = 0; q < xs.size(); q++) {
            const u64 *p = buf.data() + q * words;
            auto take = [&](u64 idx, uint32_t lg, bool base) {
                CodewordQuery cq; cq.index = (idx | 1) - 1; cq.is_base = base;
                cq.p0 = Ext(p[0], p[1]); cq.p1 = Ext(p[2], p[3]); p += 4;
                for (uint32_t k = 0; k + 1 < lg; k++) { Digest d; memcpy(d.v, p, 32); p += 4; cq.merkle_path.push_back(d); }
                return cq;
            };
            std::vector<CodewordQuery> cqs, oqs;
            for (uint32_t k = 0; k < n; k++) { uint32_t lg = log2_strict(cw_sizes[k]); cqs.push_back(take(xs[q] >> (lgN - lg), lg, is_base[k])); }
            for (uint32_t i = 0; i + 1 < num_rounds; i++) oqs.push_back(take(xs[q] >> (i + 1), lgN - i - 1, false));
            if (batch) { BatchedQueryResult r; r.x_index = xs[q]; r.oracle_query = oqs; r.commitments_query = cqs; pr.batched_queries.push_back(r); }
            else { SingleQueryResult r; r.x_index = xs[q]; r.commitment_query = cqs[0]; r.oracle_query = oqs; pr.single_queries.push_back(r); }
        }
    }
};

}  // namespace dp
