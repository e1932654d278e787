// Host mirror of the reference's `multilinear_extensions` + `sumcheck` public API over the C ABI.
//   DeviceMle            <-> DenseMultilinearExtension      (multilinear_extensions/src/mle.rs:130-181)
//   VirtualPolynomial    <-> VirtualPolynomial               (virtual_poly.rs:50-180)
//   IOPProverState::prove_parallel, IOPProof, get_mle_final_evaluations (sumcheck/src/prover.rs:498-585,
//   :474-490; structs.rs:15-34)
// Same names, argument meaning and error behaviour: where the reference asserts/panics this throws
// dp::Error carrying the reference's message.
#pragma once
#include "field.hpp"
#include "transcript.hpp"
#include "../../include/deepprove_b200.h"
#include <memory>
#include <algorithm>
#include <map>
#include <chrono>

namespace dp {

struct Error : std::runtime_error { int code; Error(int c, const std::string &m) : std::runtime_error(m), code(c) {} };
inline void check(int rc) { if (rc != DP_OK) throw Error(rc, dp_last_error()); }

class DeviceMle {
  public:
    DeviceMle() {}
    explicit DeviceMle(dp_mle *h) : h_(h, [](dp_mle *p) { dp_mle_free(p); }) {}
    static DeviceMle from_evaluations_vec(const std::vector<u64> &base) { dp_mle *h; check(dp_mle_upload(base.data(), base.size(), 0, &h)); return DeviceMle(h); }
    static DeviceMle from_evaluations_ext_vec(const ExtVec &ext) { auto f = flatten(ext); dp_mle *h; check(dp_mle_upload(f.data(), ext.size(), 1, &h)); return DeviceMle(h); }
    static DeviceMle from_raw(const u64 *data, u64 len, bool is_ext) { dp_mle *h; check(dp_mle_upload(data, len, is_ext, &h)); return DeviceMle(h); }
    static DeviceMle wrap_device(void *ptr, u64 len, bool is_ext) { dp_mle *h; check(dp_mle_wrap_device(ptr, len, is_ext, &h)); return DeviceMle(h); }
    static DeviceMle build_eq_x_r(const ExtVec &r) { auto f = flatten(r); dp_mle *h; check(dp_eq_build(f.data(), (uint32_t)r.size(), &h)); return DeviceMle(h); }
    dp_mle *handle() const { return h_.get(); }
    bool valid() const { return (bool)h_; }
    u64 len() const { u64 l; check(dp_mle_info(h_.get(), &l, nullptr, nullptr)); return l; }
    bool is_ext() const { int e; check(dp_mle_info(h_.get(), nullptr, &e, nullptr)); return e != 0; }
    uint32_t num_vars() const { uint32_t n; check(dp_mle_info(h_.get(), nullptr, nullptr, &n)); return n; }
    Ext evaluate(const ExtVec &point) const { auto f = flatten(point); u64 o[2]; check(dp_mle_evaluate(h_.get(), f.data(), (uint32_t)point.size(), o)); return Ext(o[0], o[1]); }
    static ExtVec evaluate_many(const std::vector<DeviceMle> &ms, const ExtVec &point) {
        std::vector<dp_mle *> hs; for (auto &m : ms) hs.push_back(m.handle());
        auto f = flatten(point); std::vector<u64> o(2 * ms.size());
        if (!ms.empty()) check(dp_mle_evaluate_many(hs.data(), (uint32_t)hs.size(), f.data(), (uint32_t)point.size(), o.data()));
        ExtVec r; for (size_t i = 0; i < ms.size(); i++) r.push_back(Ext(o[2 * i], o[2 * i + 1]));
        return r;
    }
    void fix_high_variables_in_place(const ExtVec &point) { auto f = flatten(point); check(dp_mle_fix_high(h_.get(), f.data(), (uint32_t)point.size())); }
    DeviceMle fix_high_variables(const ExtVec &point) const { auto f = flatten(point); dp_mle *o; check(dp_mle_fix_high_new(h_.get(), f.data(), (uint32_t)point.size(), &o)); return DeviceMle(o); }
    static DeviceMle linear_combination(const std::vector<DeviceMle> &ms, const ExtVec &coefs) {
        std::vector<dp_mle *> hs; for (auto &m : ms) hs.push_back(m.handle());
        auto f = flatten(coefs); dp_mle *o; check(dp_mle_linear_combination(hs.data(), f.data(), (uint32_t)hs.size(), &o)); return DeviceMle(o);
    }
    DeviceMle fix_variables(const ExtVec &point) const { auto f = flatten(point); dp_mle *o; check(dp_mle_fix_low(h_.get(), f.data(), (uint32_t)point.size(), &o)); return DeviceMle(o); }
    DeviceMle clone() const { dp_mle *o; check(dp_mle_clone(h_.get(), &o)); return DeviceMle(o); }
    std::vector<u64> download() const { std::vector<u64> v(len() * (is_ext() ? 2 : 1)); check(dp_mle_download(h_.get(), v.data())); return v; }
  private:
    std::shared_ptr<dp_mle> h_;
};

// Inter-rank exchange used by IOPProverState::prove_sharded: an all-gather of a few u64 words per rank.
struct Exchange {
    size_t world = 1, rank = 0;
    virtual ~Exchange() {}
    virtual void allgather(const u64 *send, size_t n_words, u64 *recv /* world * n_words, rank-major */) = 0;
};
// Same-node exchange through a shared-memory mailbox (all ranks of one box map the same zero-initialised region).
// The per-round message has to reach the host anyway (Fiat-Shamir runs there), so host-to-host shared memory is the
// shortest path: ~1 us per exchange instead of a device collective's launch + copy-back.  Slots are double-buffered
// by sequence parity; a slot is rewritten only two exchanges later, which every reader has passed by then.
struct ShmMailbox {
    static constexpr size_t MAX_WORLD = 16, PAYLOAD = 2046;     // 16 KB slots: round messages use a few words, the sharded Basefold query rows ~2 MB in ~120 exchanges
    struct alignas(64) Slot { volatile u64 seq; u64 n; u64 payload[PAYLOAD]; };
    Slot slots[MAX_WORLD][2];
};
struct ShmExchange : Exchange {
    ShmMailbox *mb; u64 seq = 0;
    static constexpr u64 POISON = ~0ULL; static constexpr int TIMEOUT_S = 60;
    // called by a rank that is abandoning the proof (exception path): wakes every peer with an error instead of a hang
    void poison() { for (int b = 0; b < 2; b++) __atomic_store_n(&mb->slots[rank][b].seq, POISON, __ATOMIC_RELEASE); }
    ShmExchange(void *region, size_t w, size_t r) : mb((ShmMailbox *)region) { world = w; rank = r; if (w > ShmMailbox::MAX_WORLD) throw std::runtime_error("ShmExchange: world too large"); }
    void allgather(const u64 *send, size_t n, u64 *recv) override {
        for (size_t off = 0; off < n || off == 0; off += ShmMailbox::PAYLOAD) {
            size_t m = std::min(n - off, ShmMailbox::PAYLOAD);
            seq++;
            const auto t_start = std::chrono::steady_clock::now();
            ShmMailbox::Slot &mine = mb->slots[rank][seq & 1];
            for (size_t i = 0; i < m; i++) mine.payload[i] = send[off + i];
            mine.n = m;
            __atomic_store_n(&mine.seq, seq, __ATOMIC_RELEASE);
            for (size_t g = 0; g < world; g++) {
                ShmMailbox::Slot &sl = mb->slots[g][seq & 1];
                // bounded: a rank that died or threw mid-proof must not hang its peers forever (a failing rank posts POISON)
                for (u64 spins = 0;; spins++) {
                    u64 v = __atomic_load_n(&sl.seq, __ATOMIC_ACQUIRE);
                    if (v == seq) break;
                    if (v == POISON) throw std::runtime_error("ShmExchange: a peer rank aborted the exchange");
                    if ((spins & 0xFFFF) == 0xFFFF && std::chrono::steady_clock::now() - t_start > std::chrono::seconds(TIMEOUT_S)) throw std::runtime_error("ShmExchange: timed out waiting for a peer rank");
                    __builtin_ia32_pause();
                }
                for (size_t i = 0; i < m; i++) recv[g * n + off + i] = sl.payload[i];
            }
            if (n == 0) break;
        }
    }
};
// Exchange through a caller-supplied function (e.g. a torch.distributed all-gather over NCCL or gloo)
struct CallbackExchange : Exchange {
    typedef int (*Fn)(void *user, const uint64_t *send, uint64_t n_words, uint64_t *recv);
    Fn fn; void *user;
    CallbackExchange(Fn f, void *u, size_t w, size_t r) : fn(f), user(u) { world = w; rank = r; }
    void allgather(const u64 *send, size_t n, u64 *recv) override {
        if (!fn) { if (world != 1) throw std::runtime_error("exchange callback missing"); for (size_t i = 0; i < n; i++) recv[i] = send[i]; return; }   // a world of one needs no exchange
        if (fn(user, send, n, recv)) throw std::runtime_error("exchange callback failed");
    }
};

struct VPAuxInfo { size_t max_degree = 0, max_num_variables = 0; };

class VirtualPolynomial {
  public:
    explicit VirtualPolynomial(size_t max_num_variables = 0) { aux_info.max_num_variables = max_num_variables; }
    // add_mle_list: MLE identity is the device handle, as the reference's is the Arc pointer
    void add_mle_list(const std::vector<DeviceMle> &list, Ext coefficient) {
        if (list.empty()) throw Error(DP_ERR_INVALID, "input mle_list is empty");
        dp_sc_product pr{};
        pr.coef[0] = coefficient.c0; pr.coef[1] = coefficient.c1;
        if (list.size() > 5) throw Error(DP_ERR_UNSUPPORTED, "do not support degree > 5");
        for (auto &m : list) {
            if (m.num_vars() > aux_info.max_num_variables) throw Error(DP_ERR_INVALID, "invalid max num vars");
            if (m.num_vars() != list[0].num_vars()) throw Error(DP_ERR_INVALID, "mle in mle_list must be in same num_vars() in same product");
            auto it = index_.find(m.handle());
            uint32_t id;
            if (it == index_.end()) { id = (uint32_t)flattened_ml_extensions.size(); flattened_ml_extensions.push_back(m); index_[m.handle()] = id; }
            else id = it->second;
            pr.idx[pr.n_idx++] = id;
        }
        if (list.size() > aux_info.max_degree) aux_info.max_degree = list.size();
        products.push_back(pr);
    }
    VPAuxInfo aux_info;
    std::vector<dp_sc_product> products;
    std::vector<DeviceMle> flattened_ml_extensions;
  private:
    std::map<dp_mle *, uint32_t> index_;
};

struct IOPProverMessage { ExtVec evaluations; };
struct IOPProof {
    ExtVec point;
    std::vector<IOPProverMessage> proofs;
    Ext extract_sum() const { return proofs.at(0).evaluations.at(0) + proofs.at(0).evaluations.at(1); }
};

// The hand-off to a device-transcript entry point: the transcript's state goes, through call(entry, state), to the Poseidon2 form
// (p2) or the BLAKE3 form (b3) of the entry point as the state's kind says, and the state the entry point returns is loaded back.
// False, with nothing called, when the transcript has no device state (DS_NONE).
template <class T, class F, class C>
inline bool run_device_transcript(T &transcript, F p2, F b3, C &&call) {
    u64 sp[DEVICE_STATE_WORDS];
    const int kind = transcript.save_sponge(sp);
    if (kind == DS_NONE) return false;
    check(call(kind == DS_BLAKE3 ? b3 : p2, sp));
    transcript.load_sponge(sp);
    return true;
}
// n rounds of a device-transcript entry point's flat output appended to proof and challenges: msgs, n messages of deg + 1 elements;
// ch, n challenges; [c0, c1] words per element
inline void append_device_rounds(IOPProof &proof, ExtVec &challenges, size_t n, size_t deg, const u64 *msgs, const u64 *ch) {
    for (size_t k = 0; k < n; k++) {
        IOPProverMessage msg;
        for (size_t t = 0; t <= deg; t++, msgs += 2) msg.evaluations.push_back(Ext(msgs[0], msgs[1]));
        proof.proofs.push_back(std::move(msg));
        challenges.push_back(Ext(ch[2 * k], ch[2 * k + 1]));
    }
}

class IOPProverState {
  public:
    ~IOPProverState() { if (sc_) dp_sc_destroy(sc_); }
    IOPProverState() {}
    IOPProverState(IOPProverState &&o) noexcept { *this = std::move(o); }
    IOPProverState &operator=(IOPProverState &&o) noexcept { std::swap(sc_, o.sc_); challenges = std::move(o.challenges); finals_ = std::move(o.finals_); poly_ = std::move(o.poly_); return *this; }
    ExtVec challenges;
    const ExtVec &get_mle_final_evaluations() const { return finals_; }

    // IOPProverState::prove_parallel(poly, transcript) -> (IOPProof, IOPProverState)
    template <class T>
    static std::pair<IOPProof, IOPProverState> prove_parallel(VirtualPolynomial poly, T &transcript) {
        IOPProof proof; IOPProverState st;
        size_t nv = poly.aux_info.max_num_variables, deg = poly.aux_info.max_degree;
        if (nv == 0) return {std::move(proof), std::move(st)};  // constant polynomial: IOPProof::default()
        transcript.append_usize(nv);
        transcript.append_usize(deg);
        std::vector<dp_mle *> hs;
        for (auto &m : poly.flattened_ml_extensions) hs.push_back(m.handle());
        check(dp_sc_create(hs.data(), (uint32_t)hs.size(), poly.products.data(), (uint32_t)poly.products.size(), (uint32_t)nv, (uint32_t)deg, &st.sc_));
        check(dp_sc_set_resident_tail(st.sc_, 1));   // this loop only runs the transcript between rounds: small rounds stay resident on the device
        std::vector<u64> buf(2 * (deg + 1));
        run_rounds(nv, deg, transcript, proof, st, [&](const u64 *c, ExtVec &ev) {
            check(dp_sc_round(st.sc_, c, buf.data()));
            for (size_t t = 0; t <= deg; t++) ev[t] = Ext(buf[2 * t], buf[2 * t + 1]);
        }, st.sc_);
        u64 c[2] = {st.challenges.back().c0, st.challenges.back().c1};
        std::vector<u64> fin(2 * hs.size());
        check(dp_sc_finish(st.sc_, c, fin.data()));
        for (size_t i = 0; i < hs.size(); i++) st.finals_.push_back(Ext(fin[2 * i], fin[2 * i + 1]));
        proof.point = st.challenges;
        st.poly_ = std::move(poly);
        return {std::move(proof), std::move(st)};
    }
    // IOPProverState::prove_batch_polys(max_thread_id, polys, transcript) (sumcheck/src/prover.rs:37-321): the devirgo
    // split with one device sumcheck per slice.  Same proof as prove_parallel on the un-split polynomial.
    template <class T>
    static std::pair<IOPProof, IOPProverState> prove_batch_polys(size_t max_thread_id, std::vector<VirtualPolynomial> polys, T &transcript) {
        if (polys.empty() || polys.size() != max_thread_id || (max_thread_id & (max_thread_id - 1))) throw Error(DP_ERR_INVALID, "prove_batch_polys: polys.len() must equal a power-of-two max_thread_id");
        size_t nv = polys[0].aux_info.max_num_variables, deg = polys[0].aux_info.max_degree, logT = 0;
        while (((size_t)1 << logT) < max_thread_id) logT++;
        for (auto &p : polys) if (p.aux_info.max_num_variables != nv || p.aux_info.max_degree != deg) throw Error(DP_ERR_INVALID, "prove_batch_polys: polys differ in (max_num_variables, max_degree)");
        IOPProof proof; IOPProverState st;
        if (nv == 0) return {std::move(proof), std::move(st)};
        transcript.append_usize(nv + logT);
        transcript.append_usize(deg);
        struct H { dp_sc *h = nullptr; ~H() { if (h) dp_sc_destroy(h); } };
        std::vector<H> hs(polys.size());
        std::vector<std::vector<dp_mle *>> mh(polys.size());
        for (size_t t = 0; t < polys.size(); t++) {
            for (auto &m : polys[t].flattened_ml_extensions) mh[t].push_back(m.handle());
            check(dp_sc_create(mh[t].data(), (uint32_t)mh[t].size(), polys[t].products.data(), (uint32_t)polys[t].products.size(), (uint32_t)nv, (uint32_t)deg, &hs[t].h));
        }
        std::vector<u64> buf(2 * (deg + 1));
        run_rounds(nv, deg, transcript, proof, st, [&](const u64 *c, ExtVec &ev) {
            for (auto &h : hs) { check(dp_sc_round(h.h, c, buf.data())); for (size_t k = 0; k <= deg; k++) ev[k] += Ext(buf[2 * k], buf[2 * k + 1]); }
        });
        size_t n_mles = mh[0].size();
        std::vector<ExtVec> residual(n_mles);                 // merge_sumcheck_polys (util.rs:215-243)
        u64 c[2] = {st.challenges.back().c0, st.challenges.back().c1};
        for (auto &h : hs) { std::vector<u64> fin(2 * n_mles); check(dp_sc_finish(h.h, c, fin.data())); for (size_t i = 0; i < n_mles; i++) residual[i].push_back(Ext(fin[2 * i], fin[2 * i + 1])); }
        if (logT == 0) { for (size_t i = 0; i < n_mles; i++) st.finals_.push_back(residual[i][0]); proof.point = st.challenges; return {std::move(proof), std::move(st)}; }
        finish_merged(residual, polys[0].products, deg, logT, transcript, proof, st);
        return {std::move(proof), std::move(st)};
    }

    // One proof sharded over `ex.world` ranks (one process per GPU): rank g holds the slice [g n/G, (g+1) n/G) of
    // every MLE as `poly` (nv_total - log G variables).  Same protocol as prove_batch_polys with max_thread_id = G
    // (prover.rs:37-321): per round ONE all-gather of the (deg+1)-element partial message replaces the reference's
    // per-thread channels (prover.rs:150-170); every rank adds the partials and runs the same transcript, so no
    // challenge broadcast exists.  The proof is identical on every rank and to prove_parallel on the unsplit poly.
    template <class T>
    static std::pair<IOPProof, IOPProverState> prove_sharded(VirtualPolynomial poly, size_t nv_total, Exchange &ex, T &transcript) {
        size_t G = ex.world, logG = 0; while (((size_t)1 << logG) < G) logG++;
        if (G == 0 || (G & (G - 1))) throw Error(DP_ERR_INVALID, "prove_sharded: world size must be a power of two");
        size_t nv = poly.aux_info.max_num_variables, deg = poly.aux_info.max_degree;
        if (nv + logG != nv_total || nv == 0) throw Error(DP_ERR_INVALID, "prove_sharded: slice must have nv_total - log2(world) >= 1 variables");
        IOPProof proof; IOPProverState st;
        transcript.append_usize(nv_total);
        transcript.append_usize(deg);
        struct H { dp_sc *h = nullptr; ~H() { if (h) dp_sc_destroy(h); } } hs;
        std::vector<dp_mle *> mh; for (auto &m : poly.flattened_ml_extensions) mh.push_back(m.handle());
        check(dp_sc_create(mh.data(), (uint32_t)mh.size(), poly.products.data(), (uint32_t)poly.products.size(), (uint32_t)nv, (uint32_t)deg, &hs.h));
        size_t W = 2 * (deg + 1);
        std::vector<u64> buf(W), all(W * G);
        run_rounds(nv, deg, transcript, proof, st, [&](const u64 *c, ExtVec &ev) {
            check(dp_sc_round(hs.h, c, buf.data()));
            ex.allgather(buf.data(), W, all.data());
            for (size_t g = 0; g < G; g++) for (size_t k = 0; k <= deg; k++) ev[k] += Ext(all[g * W + 2 * k], all[g * W + 2 * k + 1]);
        });
        size_t n_mles = mh.size();
        u64 c[2] = {st.challenges.back().c0, st.challenges.back().c1};
        std::vector<u64> fin(2 * n_mles), fall(2 * n_mles * G);
        check(dp_sc_finish(hs.h, c, fin.data()));
        if (G == 1) { for (size_t i = 0; i < n_mles; i++) st.finals_.push_back(Ext(fin[2 * i], fin[2 * i + 1])); proof.point = st.challenges; return {std::move(proof), std::move(st)}; }
        ex.allgather(fin.data(), 2 * n_mles, fall.data());
        std::vector<ExtVec> residual(n_mles);                 // merge_sumcheck_polys (util.rs:215-243), slice order = rank order
        for (size_t g = 0; g < G; g++) for (size_t i = 0; i < n_mles; i++) residual[i].push_back(Ext(fall[g * 2 * n_mles + 2 * i], fall[g * 2 * n_mles + 2 * i + 1]));
        finish_merged(residual, poly.products, deg, logG, transcript, proof, st);   // last log G rounds, replicated on every rank
        return {std::move(proof), std::move(st)};
    }
  private:
    // The rounds of one sumcheck: round(c, evals) fills the (deg + 1) zeroed evaluations of the next message from the previous
    // round's challenge c ([c0, c1]; null in round 0).  Each message goes to the transcript, which draws the next challenge.
    // sc: the single device handle behind `round`, if there is one; when the library says its resident tail runs the transcript
    // on the device from the next round on (dp_sc_tail_fs_next) and the transcript's state can go there, the remaining rounds
    // are one dp_sc_run_tail_fs (BasicTranscript) or dp_sc_run_tail_fs_blake (BlakeTranscript) call.
    template <class T, class F>
    static void run_rounds(size_t nv, size_t deg, T &transcript, IOPProof &proof, IOPProverState &st, F &&round, dp_sc *sc = nullptr) {
        for (size_t i = 0; i < nv; i++) {
            u64 c[2] = {0, 0};
            if (i > 0) { c[0] = st.challenges.back().c0; c[1] = st.challenges.back().c1; }
            int dev = 0;
            if (sc) check(dp_sc_tail_fs_next(sc, &dev));
            if (dev) {
                const size_t n = nv - i;
                std::vector<u64> msgs(2 * n * (deg + 1)), ch(2 * n);
                if (run_device_transcript(transcript, dp_sc_run_tail_fs, dp_sc_run_tail_fs_blake, [&](auto run, u64 *sp) {
                        return run(sc, i > 0 ? c : nullptr, sp, msgs.data(), ch.data(), sp); })) {
                    append_device_rounds(proof, st.challenges, n, deg, msgs.data(), ch.data());
                    return;
                }
            }
            IOPProverMessage msg; msg.evaluations.assign(deg + 1, Ext::zero());
            round(i > 0 ? c : nullptr, msg.evaluations);
            transcript.append_field_element_exts(msg.evaluations);
            proof.proofs.push_back(std::move(msg));
            st.challenges.push_back(transcript.get_and_append_challenge("Internal round"));
        }
    }
    // stage 2 of the devirgo split: the last log T rounds over the T residual values of every MLE
    template <class T>
    static void finish_merged(const std::vector<ExtVec> &residual, const std::vector<dp_sc_product> &products, size_t deg, size_t logT, T &transcript, IOPProof &proof, IOPProverState &st) {
        size_t n_mles = residual.size();
        struct H { dp_sc *h = nullptr; ~H() { if (h) dp_sc_destroy(h); } };
        std::vector<u64> buf(2 * (deg + 1));
        VirtualPolynomial merged(logT);
        std::vector<DeviceMle> mm; for (auto &r : residual) mm.push_back(DeviceMle::from_evaluations_ext_vec(r));
        for (auto &pr : products) { std::vector<DeviceMle> l; for (uint32_t j = 0; j < pr.n_idx; j++) l.push_back(mm[pr.idx[j]]); merged.add_mle_list(l, Ext(pr.coef[0], pr.coef[1])); }
        merged.aux_info.max_degree = deg;
        // MLE numbering of `merged` follows first use in the products; map back for the final evaluations
        std::vector<dp_mle *> h2; for (auto &m : merged.flattened_ml_extensions) h2.push_back(m.handle());
        dp_sc *s2 = nullptr;
        check(dp_sc_create(h2.data(), (uint32_t)h2.size(), merged.products.data(), (uint32_t)merged.products.size(), (uint32_t)logT, (uint32_t)deg, &s2));
        H g2; g2.h = s2;
        run_rounds(logT, deg, transcript, proof, st, [&](const u64 *c, ExtVec &ev) {
            check(dp_sc_round(s2, c, buf.data()));
            for (size_t k = 0; k <= deg; k++) ev[k] = Ext(buf[2 * k], buf[2 * k + 1]);
        });
        u64 cc[2] = {st.challenges.back().c0, st.challenges.back().c1};
        std::vector<u64> fin(2 * h2.size()); check(dp_sc_finish(s2, cc, fin.data()));
        ExtVec f2; for (size_t i = 0; i < h2.size(); i++) f2.push_back(Ext(fin[2 * i], fin[2 * i + 1]));
        for (size_t i = 0; i < n_mles; i++) { Ext v; for (size_t k = 0; k < h2.size(); k++) if (h2[k] == mm[i].handle()) v = f2[k]; st.finals_.push_back(v); }
        proof.point = st.challenges;
    }
    dp_sc *sc_ = nullptr;
    ExtVec finals_;
    VirtualPolynomial poly_;
};

}  // namespace dp
