// Host mirror of the FFT-convolution layer over the C ABI:
//   Convolution<Element>::{op, prove_convolution_step, prove_batch_fft_weights} (zkml/src/layers/convolution.rs:320-350,
//   :368-458, :697-1077), hadamard::prove (layers/hadamard.rs:83-126), Prover::{prove_batch_fft, prove_batch_ifft,
//   delegate_matrix_evaluation} (iop/prover.rs:164-212,295-399), Tensor::fft_conv (tensor.rs:458-523).
// Same structure and names as the reference; every tensor lives in HBM (include/deepprove_b200.h), the host keeps the
// transcript, the O(log n) scalars and the claims.  dp_sc_* borrows its operands and never modifies them, so resident
// tensors (filters, the inference trace) are shared by any number of proofs.
#pragma once
// included from the middle of zkml.hpp (needs Claim, Element, to_base; Prover below needs this file)

namespace dp {
namespace zkml {

// rows up to 2^13 one block per row, longer rows (images wider than 64) through the two-pass kernel
inline DeviceMle fft_rows(DeviceMle m, uint32_t log_n, bool inverse) { check((log_n <= 13 ? dp_fft_rows : dp_fft_rows_long)(m.handle(), log_n, inverse ? 1 : 0)); return m; }
inline DeviceMle pad_rows(const DeviceMle &src, u64 rows, uint32_t n_real, uint32_t n, u64 out_len) { dp_mle *o; check(dp_pad_rows(src.handle(), rows, n_real, n, out_len, &o)); return DeviceMle(o); }
inline DeviceMle repeat(const DeviceMle &src, uint32_t times) { dp_mle *o; check(dp_mle_repeat(src.handle(), times, &o)); return DeviceMle(o); }
inline ExtVec download_ext(const DeviceMle &m) {
    std::vector<u64> raw = m.download(); ExtVec v;
    if (m.is_ext()) for (size_t i = 0; i + 1 < raw.size(); i += 2) v.push_back(Ext(raw[i], raw[i + 1]));
    else for (u64 x : raw) v.push_back(Ext::from_base(x));
    return v;
}
inline Ext mle_eval_host(ExtVec v, const ExtVec &point) {          // evaluate (mle.rs:607-623) for O(1)-sized vectors
    for (const Ext &r : point) { ExtVec n(v.size() / 2); for (size_t i = 0; i < n.size(); i++) n[i] = v[2 * i] + r * (v[2 * i + 1] - v[2 * i]); v.swap(n); }
    return v[0];
}

struct HadamardProof { IOPProof sumcheck; ExtVec individual_claim; };
// hadamard::prove (hadamard.rs:83-126) on two resident tensors
template <class T>
HadamardProof hadamard_prove(T &t, const Claim &output_claim, const DeviceMle &a, const DeviceMle &b) {
    const u64 n = a.len();
    if (n != b.len() || (n & (n - 1)) || output_claim.point.size() != ceil_log2(n)) throw Error(DP_ERR_INVALID, "hadamard: shapes / claim point do not match");
    DeviceMle beta = DeviceMle::build_eq_x_r(output_claim.point);
    VirtualPolynomial vp(output_claim.point.size());
    vp.add_mle_list({a, b, beta}, Ext::one());
    auto res = IOPProverState::prove_parallel(std::move(vp), t);
    const ExtVec &fe = res.second.get_mle_final_evaluations();
    return {res.first, {fe[0], fe[1]}};
}

struct MatrixEvalProof { std::vector<IOPProof> proofs; std::vector<ExtVec> claims; };
struct PhiTables { DeviceMle w_red; std::vector<DeviceMle> mid; };
// Prover::phi_g_init (iop/prover.rs:231-289)
inline PhiTables phi_g_init(const ExtVec &rx, Ext scale, size_t n, bool is_fft) {
    auto f = flatten(rx); u64 sc[2] = {scale.c0, scale.c1};
    dp_mle *w = nullptr; std::vector<dp_mle *> mid(n - 1, nullptr);
    check((n <= 14 ? dp_phi_g_init : dp_phi_g_init_long)(f.data(), (uint32_t)n, sc, is_fft ? 1 : 0, &w, mid.data()));
    PhiTables p; p.w_red = DeviceMle(w); for (auto *m : mid) p.mid.push_back(DeviceMle(m));
    return p;
}
// Prover::delegate_matrix_evaluation (iop/prover.rs:164-212)
template <class T>
MatrixEvalProof delegate_matrix_evaluation(T &t, std::vector<DeviceMle> &f_middle, const ExtVec &r1, ExtVec r2, bool is_fft) {
    MatrixEvalProof out; Ext one = Ext::one(), two = Ext::from_base(2);
    size_t fm = f_middle.size();
    for (size_t l = r1.size() - 1; l-- > 0;) {
        Ext rl = r1[(fm - 1) - l], last = r2.back(), A, B;
        if (!is_fft && l == fm - 1) { A = (one - last) * (one - rl); B = (one - last) * rl; }
        else { A = one - rl; B = (one - two * last) * rl; }
        u64 a[2] = {A.c0, A.c1}, b[2] = {B.c0, B.c1};
        dp_mle *ph; check(dp_phi_level((uint32_t)(l + 1), (uint32_t)r1.size(), (uint32_t)((fm - 1) - l), a, b, is_fft ? 1 : 0, &ph));
        DeviceMle phi(ph), beta = DeviceMle::build_eq_x_r(ExtVec(r2.begin(), r2.end() - 1));
        VirtualPolynomial vp(l + 1);
        vp.add_mle_list({beta, phi, f_middle[l]}, Ext::one());
        auto res = IOPProverState::prove_parallel(std::move(vp), t);
        r2 = res.first.point;
        out.proofs.push_back(res.first); out.claims.push_back(res.second.get_mle_final_evaluations());
    }
    return out;
}
struct BatchFFTProof { IOPProof proof; ExtVec claims; MatrixEvalProof matrix_eval; };
// shared tail of prove_batch_fft / prove_batch_ifft: `rows` is [n_rows][row_len] resident; y = sum_i W(r1, i) X(i, r2)
template <class T>
BatchFFTProof prove_batch_matrix(T &t, const ExtVec &r, const DeviceMle &rows, size_t n_rows, size_t row_len, Ext scale, bool is_fft) {
    size_t l1 = ceil_log2(row_len), l2 = ceil_log2(n_rows);
    ExtVec r1(r.begin(), r.begin() + l1), r2(r.begin() + l1, r.begin() + l1 + l2);
    if (is_fft && !(r1.back() == Ext::zero())) throw Error(DP_ERR_INVALID, "Error in randomness init batch ifft");
    PhiTables ph = phi_g_init(r1, scale, l1, is_fft);
    DeviceMle f_m = rows.fix_high_variables(r2);                     // X(., r2): the row index is the HIGH variable block
    VirtualPolynomial vp(l1);
    vp.add_mle_list({f_m, ph.w_red}, Ext::one());
    auto res = IOPProverState::prove_parallel(std::move(vp), t);
    BatchFFTProof o; o.proof = res.first; o.claims = res.second.get_mle_final_evaluations();
    o.matrix_eval = delegate_matrix_evaluation(t, ph.mid, r1, res.first.point, is_fft);
    return o;
}

struct ConvData {                                                   // tensor.rs:326-337, the parts the prover reads
    DeviceMle input;                                                // [kx][n_x^2] Base: index_x(real_input) = each channel reversed
    DeviceMle input_fft, prod;                                      // [kx][2 n_x^2], [kw][2 n_w^2] Ext
    DeviceMle output_as_element;                                    // conv output after bias, before clearing, [kw][n_x][n_x] Base
};
struct BatchFFTWeightsProof { IOPProof proof; ExtVec claims, partial_evals; MatrixEvalProof matrix_evaluation; };
struct ConvProof {                                                  // convolution.rs:97-121
    IOPProof fft_proof, fft_proof_weights, ifft_proof, hadamard_proof;
    MatrixEvalProof fft_delegation, fft_delegation_weights, ifft_delegation;
    ExtVec fft_claims, ifft_claims, fft_weight_claims, hadamard_claims, partial_evals;
    Ext bias_claim;
    HadamardProof clearing_proof;
    Claim filter_claim, bias_poly_claim;                            // for CommitmentProver::add_common_claims (:1003-1010)
};

// Convolution<Element> after into_padded_and_ffted (convolution.rs:309-318): filter shape [kw, kx, nw, nw] with the
// power-of-two padded weights [kw][kx][real_nw][real_nw] as data
struct Convolution {
    size_t kw = 0, kx = 0, nw = 0, real_nw = 0;
    std::vector<Element> filter, bias;
    size_t unpadded_out[3] = {0, 0, 0};
    DeviceMle filter_mle, bias_mle, w_fft, mask;                    // resident: weights (Base), bias (Base), FFT(index_w(filter)) [kw][kx][2 nw^2],
                                                                    // clearing tensor (Base 0/1) [kw][nw][nw]
    size_t filter_size() const { return nw * nw; }
    size_t row_len() const { return 2 * nw * nw; }
    void load() {
        if (filter.size() != kw * kx * real_nw * real_nw || bias.size() != kw) throw Error(DP_ERR_INVALID, "Convolution: filter/bias shape mismatch");
        filter_mle = DeviceMle::from_evaluations_vec(to_base(filter));
        bias_mle = DeviceMle::from_evaluations_vec(to_base(bias));
        w_fft = fft_rows(pad_rows(filter_mle, kw * kx, (uint32_t)real_nw, (uint32_t)nw, row_len()), (uint32_t)ceil_log2(row_len()), false);   // tensor.rs:492-503, hoisted out of the inference
        mask = DeviceMle::from_evaluations_vec(to_base(clearing_tensor()));
    }
    std::vector<Element> clearing_tensor() const {                  // new_clearing_tensor (convolution.rs:1508-1530)
        std::vector<Element> d(kw * nw * nw, 0);
        for (size_t i = 0; i < kw; i++) for (size_t j = 0; j < nw; j++) for (size_t k = 0; k < nw; k++)
            if (i < unpadded_out[0] && j < unpadded_out[1] && k < unpadded_out[2]) d[(i * nw + j) * nw + k] = 1;
        return d;
    }
    // Convolution::op (convolution.rs:320-350) over Tensor::fft_conv (tensor.rs:458-523) on a resident input tensor (Base,
    // canonical field elements): returns the cleared output, resident too
    DeviceMle op(const DeviceMle &x, ConvData &pd) const {
        size_t n_x = nw, chunk = n_x * n_x;
        if (x.is_ext() || x.len() != kx * chunk) throw Error(DP_ERR_INVALID, "Convolution::op: input is not [kx, n_x, n_x]");
        dp_mle *rev; check(dp_reverse_rows(x.handle(), chunk, &rev));
        pd.input = DeviceMle(rev);
        pd.input_fft = fft_rows(pad_rows(pd.input, kx, (uint32_t)n_x, (uint32_t)n_x, 2 * chunk), (uint32_t)ceil_log2(2 * chunk), false);
        dp_mle *pr; check(dp_conv_prod(pd.input_fft.handle(), w_fft.handle(), (uint32_t)kw, (uint32_t)kx, row_len(), &pr));
        pd.prod = DeviceMle(pr);
        DeviceMle out = fft_rows(pd.prod.clone(), (uint32_t)ceil_log2(row_len()), true);
        dp_mle *after, *cleared;
        check(dp_conv_output(out.handle(), (uint32_t)kw, (uint32_t)n_x, bias_mle.handle(), mask.handle(), &after, &cleared));
        pd.output_as_element = DeviceMle(after);
        return DeviceMle(cleared);
    }
    // Convolution::prove_batch_fft_weights (convolution.rs:368-458)
    template <class T>
    BatchFFTWeightsProof prove_batch_fft_weights(T &t, const ExtVec &r) const {
        size_t padded_rows = row_len(), l1 = ceil_log2(padded_rows);
        ExtVec r1(r.begin(), r.begin() + l1), r2(r.begin() + l1, r.end());
        PhiTables ph = phi_g_init(r1, Ext::one(), l1, false);
        DeviceMle w1 = filter_mle.fix_high_variables(r2);            // w1_reduced[k] = sum_{i,j} beta(r2)[i kx + j] filter[i][j][k]
        BatchFFTWeightsProof o; o.partial_evals = download_ext(w1);
        DeviceMle f_m = pad_rows(w1, 1, (uint32_t)real_nw, (uint32_t)nw, padded_rows);
        VirtualPolynomial vp(l1);
        vp.add_mle_list({f_m, ph.w_red}, Ext::one());
        auto res = IOPProverState::prove_parallel(std::move(vp), t);
        o.proof = res.first; o.claims = res.second.get_mle_final_evaluations();
        o.matrix_evaluation = delegate_matrix_evaluation(t, ph.mid, r1, res.first.point, false);
        return o;
    }
    // Convolution::prove_convolution_step (convolution.rs:697-1077)
    template <class T>
    Claim prove_convolution_step(T &t, const Claim &last_claim_in, const ConvData &pd, ConvProof &out) const {
        size_t lfs = ceil_log2(filter_size()), lkw = ceil_log2(kw), lrow = ceil_log2(row_len());
        out.clearing_proof = hadamard_prove(t, last_claim_in, pd.output_as_element, mask);
        Claim last_claim{out.clearing_proof.sumcheck.point, out.clearing_proof.individual_claim[0]};
        if (lfs + lkw != last_claim.point.size()) throw Error(DP_ERR_INVALID, "Inconsistent random point size");
        ExtVec r(last_claim.point.size() + 1, Ext::zero()), bias_point(lkw, Ext::zero());
        for (size_t i = 0; i < lfs; i++) r[i] = Ext::one() - last_claim.point[i];
        for (size_t i = 0; i < lkw; i++) { r[i + lfs + 1] = last_claim.point[i + lfs]; bias_point[i] = last_claim.point[i + lfs]; }
        Ext bias_eval = Ext::zero();
        if (!bias_point.empty()) bias_eval = bias_mle.evaluate(bias_point);
        else if (bias.size() == 1) bias_eval = Ext::from_base(from_i64(bias[0]));

        Ext scale = Ext::from_base(canon((u64)row_len())).inverse();
        BatchFFTProof ifft = prove_batch_matrix(t, r, pd.prod, kw, row_len(), scale, true);     // prove_batch_ifft (prover.rs:351-399)
        if (ifft.proof.point.size() != lfs + 1) throw Error(DP_ERR_INVALID, "Error in ifft sumceck");
        ExtVec r_ifft = ifft.proof.point;
        for (size_t i = lrow; i < r.size(); i++) r_ifft.push_back(r[i]);
        ExtVec r1(r_ifft.begin() + lrow, r_ifft.end()), r2(r_ifft.begin(), r_ifft.begin() + lrow);
        // aggregated_filter[i] = fft(index_wf(sum_j beta1[j] filter[j][i][.]))  (:872-896): the kw block is the HIGH variable block
        DeviceMle agg = filter_mle.fix_high_variables(r1);
        DeviceMle f1 = fft_rows(pad_rows(agg, kx, (uint32_t)real_nw, (uint32_t)nw, row_len()), (uint32_t)lrow, false);
        DeviceMle f3 = repeat(DeviceMle::build_eq_x_r(r2), (uint32_t)kx);                       // beta_acc (:870)
        VirtualPolynomial vp(lrow + ceil_log2(kx));
        vp.add_mle_list({f1, pd.input_fft, f3}, Ext::one());
        auto had = IOPProverState::prove_parallel(std::move(vp), t);
        out.hadamard_proof = had.first; out.hadamard_claims = had.second.get_mle_final_evaluations();
        ExtVec point = had.first.point; point.insert(point.end(), r1.begin(), r1.end());

        size_t n_x = nw;                                                                         // prove_batch_fft (prover.rs:295-349)
        DeviceMle x = pad_rows(pd.input, kx, (uint32_t)n_x, (uint32_t)n_x, 2 * n_x * n_x);
        BatchFFTProof fftp = prove_batch_matrix(t, had.first.point, x, kx, 2 * n_x * n_x, Ext::one(), false);
        BatchFFTWeightsProof fw = prove_batch_fft_weights(t, point);
        size_t lw = ceil_log2(real_nw * real_nw);
        ExtVec weights_rand; for (size_t i = 0; i < lw; i++) weights_rand.push_back(t.read_challenge());   // read_challenges (:929-931)

        out.bias_poly_claim = Claim{bias_point, bias_eval};
        ExtVec fp = weights_rand; fp.insert(fp.end(), point.begin() + lrow, point.end());
        out.filter_claim = Claim{fp, mle_eval_host(fw.partial_evals, weights_rand)};
        out.fft_proof = fftp.proof; out.fft_claims = fftp.claims; out.fft_delegation = fftp.matrix_eval;
        out.fft_proof_weights = fw.proof; out.fft_weight_claims = fw.claims; out.fft_delegation_weights = fw.matrix_evaluation; out.partial_evals = fw.partial_evals;
        out.ifft_proof = ifft.proof; out.ifft_claims = ifft.claims; out.ifft_delegation = ifft.matrix_eval;
        out.bias_claim = bias_eval;

        ExtVec input_point = fftp.proof.point;
        Ext v = (Ext::one() - input_point.back()).inverse(); input_point.pop_back();
        for (auto &ip : input_point) ip = Ext::one() - ip;
        Claim fin; fin.point = input_point; fin.point.insert(fin.point.end(), had.first.point.begin() + lrow, had.first.point.end());
        fin.eval = fftp.claims[0] * v;
        return fin;
    }
};

}  // namespace zkml
}  // namespace dp
