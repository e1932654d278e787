/* deepprove_b200 -- C ABI of the H100-native (sm_90a) prover hot path.
 *
 * This is the drop-in boundary of SURVEY.md section 8(b): the entry points a Rust `-sys` crate would
 * bind so that deep-prove's `sumcheck`, `multilinear_extensions` and `mpcs` crates keep their public
 * API while their O(n) loops run on the GPU.  Fiat-Shamir (transcript), proof structs and the verifier
 * stay on the host, so the API is ROUND-GRANULAR: the host appends each prover message to its
 * transcript and hands the squeezed challenge back.
 *
 * Conventions
 *   - F = Goldilocks (p = 2^64 - 2^32 + 1) as one little-endian uint64 limb, canonical (< p) on output;
 *     inputs may be any u64 (they are canonicalised on upload).
 *   - E = GoldilocksExt2 = F[X]/(X^2-7) as two limbs [c0, c1]  (ff_ext/src/lib.rs:13).
 *   - MLE evaluations: little-endian hypercube index, Base = len x u64, Ext = len x [c0,c1] (AoS),
 *     exactly `DenseMultilinearExtension.evaluations` (multilinear_extensions/src/mle.rs:130-181).
 *   - Every function returns an int status (DP_OK = 0) and never unwinds across the FFI; the Rust shim
 *     maps non-zero to `panic!`/`Err` to keep the reference behaviour.  dp_last_error() gives the text.
 *   - A handle is used by one host thread at a time; the library serialises access to the device
 *     context internally (PCS::commit is called from rayon workers in the reference).
 *   - No CPU fallback exists: without a CUDA device every compute entry point returns DP_ERR_NO_DEVICE.
 */
#ifndef DEEPPROVE_B200_H
#define DEEPPROVE_B200_H
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DP_OK 0
#define DP_ERR_INVALID 1      /* bad argument (the reference would assert!/panic) */
#define DP_ERR_CUDA 2         /* CUDA runtime error */
#define DP_ERR_NO_DEVICE 3    /* no usable GPU / dp_init not called */
#define DP_ERR_STATE 4        /* call out of protocol order ("Prover is not active", ...) */
#define DP_ERR_UNSUPPORTED 5  /* e.g. product degree > 5 (sumcheck/src/prover.rs:710) */
#define DP_ERR_TIMEOUT 6      /* a timed wait ran out (dph_zkml_stream_submit / dph_zkml_stream_next) */

typedef struct dp_mle dp_mle; /* device-resident DenseMultilinearExtension */
typedef struct dp_sc dp_sc;   /* IOPProverState (sumcheck/src/structs.rs:37-48) on device */

/* ---- context -------------------------------------------------------------------------------- */
int dp_init(int device);                 /* select GPU `device`, create stream + memory pool */
int dp_shutdown(void);
int dp_device_count(void);               /* 0 when no GPU is visible; never fails */
const char *dp_last_error(void);
const char *dp_version(void);
int dp_set_stream(void *cuda_stream);    /* run on a caller-owned cudaStream_t (e.g. torch's current stream) */
int dp_synchronize(void);
uint64_t dp_kernel_launches(void);       /* number of kernels this library launched so far */
uint64_t dp_host_waits(void);            /* number of times a host thread of this library waited for the device so far */
/* How a host thread waits for the device at the end of a round (process-wide).  0 (default) = spin on the completion word:
 * lowest latency, one busy core per proof in flight.  1 = sleep on a futex that ONE poller thread of the library signals:
 * ~5 us more per wait, but waiting proofs cost no CPU, so many more proofs than cores can be in flight per GPU (the
 * reference gets the same effect from rayon's sleeping workers). */
int dp_set_wait_mode(int mode);
int dp_get_wait_mode(void);
/* Per-kernel timing with CUDA events recorded on the launch stream around each hot kernel (off by
 * default).  dp_profile_read_ex fills parallel arrays (kernel name, launches, summed ms, summed algorithmic
 * bytes per SURVEY.md 8(d), and, when `units` is not NULL, each kernel's own work unit summed over launches: Poseidon2
 * permutations for the Merkle kernels, field operations for the sumcheck rounds, 0 elsewhere) and returns the number of
 * distinct kernels.  The table is process-wide: proving threads fold their launches in with dp_profile_flush(), so a
 * batch of concurrent proofs is profiled as it runs. */
int dp_profile_enable(int on);
int dp_profile_reset(void);
int dp_profile_read_ex(char (*names)[64], uint64_t *counts, double *total_ms, uint64_t *bytes, uint64_t *units, int cap);
int dp_profile_flush(void);

/* ---- multilinear_extensions ------------------------------------------------------------------ */
/* DenseMultilinearExtension::from_evaluations_vec / _ext_vec (mle.rs:183-260): copy host -> HBM. */
int dp_mle_upload(const uint64_t *evals, uint64_t len, int is_ext, dp_mle **out);
/* Non-owning view of `len` elements already resident in HBM (must be canonical). */
int dp_mle_wrap_device(void *dev_ptr, uint64_t len, int is_ext, dp_mle **out);
int dp_mle_clone(const dp_mle *m, dp_mle **out);
int dp_mle_download(const dp_mle *m, uint64_t *out_evals);
int dp_mle_info(const dp_mle *m, uint64_t *len, int *is_ext, uint32_t *num_vars);
void *dp_mle_device_ptr(const dp_mle *m);
int dp_mle_free(dp_mle *m);
/* fix_high_variables_in_place (mle.rs:562-603): fixes the TOP k variables at `point` (k x [c0,c1]),
 * i.e. for r in point.rev(): lo[i] += (hi[i]-lo[i])*r.  The MLE becomes Ext with num_vars - k. */
int dp_mle_fix_high(dp_mle *m, const uint64_t *point, uint32_t k);
/* fix_high_variables (mle.rs:529-560): non-mutating variant, returns a new Ext MLE. */
int dp_mle_fix_high_new(const dp_mle *m, const uint64_t *point, uint32_t k, dp_mle **out);
/* fix_variables (mle.rs:454-484): fixes the LOW k variables (adjacent pairs), returns a new MLE. */
int dp_mle_fix_low(const dp_mle *m, const uint64_t *point, uint32_t k, dp_mle **out);
/* evaluate (mle.rs:607-623): point has num_vars elements; out = [c0,c1]. */
int dp_mle_evaluate(const dp_mle *m, const uint64_t *point, uint32_t num_vars, uint64_t out[2]);
/* n MLEs with the same num_vars evaluated at one point (one eq table, one launch): out = n x [c0,c1]. */
int dp_mle_evaluate_many(const dp_mle *const *mles, uint32_t n, const uint64_t *point, uint32_t num_vars, uint64_t *out);
/* build_eq_x_r_vec (virtual_poly.rs:414-453) == compute_betas_eval (zkml/src/commit/mod.rs:10-28). */
int dp_eq_build(const uint64_t *point, uint32_t num_vars, dp_mle **out);

/* ---- sumcheck -------------------------------------------------------------------------------- */
/* One term  coef * prod_j mles[idx[j]]  of a VirtualPolynomial (virtual_poly.rs:50-60). */
typedef struct dp_sc_product {
    uint64_t coef[2];
    uint32_t n_idx;   /* 1..5 */
    uint32_t idx[5];
} dp_sc_product;

/* IOPProverState::prover_init_parallel (sumcheck/src/prover.rs:588-612).  Input MLEs are BORROWED and
 * never modified (the reference clones on the first fold, prover.rs:659-670); they must stay alive
 * until dp_sc_destroy.  All MLEs of one product must have equal length (virtual_poly.rs:148-160).
 * max_degree must lie between the highest product degree and 5; above 5 it is DP_ERR_UNSUPPORTED (prover.rs:710). */
int dp_sc_create(dp_mle *const *mles, uint32_t n_mles, const dp_sc_product *products, uint32_t n_products,
                 uint32_t max_num_variables, uint32_t max_degree, dp_sc **out);
/* prove_round_and_update_state_parallel (prover.rs:625-741): `challenge` is NULL in round 0 and the
 * previous round's challenge [c0,c1] afterwards.  out_evals receives (max_degree+1) x [c0,c1]:
 * the round polynomial at 0..max_degree, products already scaled, extrapolated and summed. */
int dp_sc_round(dp_sc *s, const uint64_t *challenge, uint64_t *out_evals);
/* Opt in to the resident tail: once a round's pairs, summed over the products, number <= 2048, ALL remaining rounds are served
 * by one kernel that stays on the device: a thread-block cluster of up to 8 CTAs (~512 pairs each) that posts each round
 * message to mapped host memory and polls a mapped mailbox for the next challenge (no launch per round).  Handles with more
 * than 96 MLEs or 48 products keep the per-round kernels.  Contract: between consecutive dp_sc_round calls on this
 * handle the calling thread must not WAIT on other work submitted to the same stream (it would queue behind the
 * resident kernel).  The kernel gives up by itself after ~3 s without a challenge and dp_sc_round reports the error;
 * dp_sc_destroy releases it.  Results are identical with and without it.  It disables itself under tools that serialise
 * kernel launches (Nsight Compute, compute-sanitizer): a one-time probe checks that a running kernel can see a word the
 * host posts after the launch call returned. */
int dp_sc_set_resident_tail(dp_sc *s, int enable);
/* *out = 1 when the library runs the next round and all later ones with the transcript on the device (dp_sc_run_tail_fs, or
 * dp_sc_run_tail_fs_blake for a BlakeTranscript): the next round starts the resident tail and the wait mode is blocking
 * (dp_set_wait_mode(1)).  In spin mode a host round trip is cheaper than the kernel's own hash chain, so callers keep calling
 * dp_sc_round there. */
int dp_sc_tail_fs_next(dp_sc *s, int *out);
/* Every remaining round in the resident tail, with BasicTranscript's Fiat-Shamir run by the kernel: each round message is absorbed
 * (append_field_element_exts), then the label "Internal round", and the challenge (c0, c1) is sampled.  prev_challenge: the
 * challenge of the previous round (NULL in round 0).  sponge_in / sponge_out: the Poseidon2 duplex state before and after, 14
 * words [state[0..7], input[0..3], n_input, n_output] (may be the same buffer).  With n = max_num_variables - rounds done:
 * msgs_out receives n x (max_degree+1) x [c0,c1] (what dp_sc_round returns), challenges_out n x [c0,c1]; the last challenge goes
 * to dp_sc_finish.  DP_ERR_STATE unless the next round would start the resident tail (dp_sc_set_resident_tail enabled, small
 * enough rounds). */
int dp_sc_run_tail_fs(dp_sc *s, const uint64_t *prev_challenge, const uint64_t *sponge_in, uint64_t *msgs_out, uint64_t *challenges_out,
                      uint64_t *sponge_out);
/* The state of a BlakeTranscript (transcript/src/blake.rs: one running unkeyed BLAKE3 hasher) as DP_B3T_WORDS u64 words, the image
 * of its blake3::Hasher: [0..3] the chunk chaining value (8 x u32, little-endian pairs), [4] chunk_counter, [5..12] the 64-byte block
 * buffer (zero past block_len), [13] block_len, [14] blocks_compressed, [15] stack_len, [16 + 4i .. 19 + 4i] chaining-value stack
 * entry i (8 x u32).  The hasher is lazy: a full block is compressed, and a full chunk pushed, only when more input arrives.  A
 * valid image has block_len <= 64, blocks_compressed <= 15 (and block_len > 0 when blocks_compressed > 0), zero bytes past
 * block_len and stack_len == popcount(chunk_counter) <= DP_B3T_STACK; a transcript of more than 2^16 chunks (64 MiB) has no image. */
#define DP_B3T_STACK 16
#define DP_B3T_WORDS 80
/* dp_sc_run_tail_fs with BlakeTranscript's Fiat-Shamir on the device: per round the message (append_field_element_exts), the label
 * "Internal round" (two 8-byte words, each appended as a field element), then read_challenge.  state_in / state_out: DP_B3T_WORDS
 * images (may be the same buffer).  Arguments, outputs and DP_ERR_STATE as dp_sc_run_tail_fs; DP_ERR_INVALID for an invalid image. */
int dp_sc_run_tail_fs_blake(dp_sc *s, const uint64_t *prev_challenge, const uint64_t *state_in, uint64_t *msgs_out, uint64_t *challenges_out,
                            uint64_t *state_out);
/* Tail of prove_parallel (prover.rs:544-568) + get_mle_final_evaluations (:474-490): fixes the last
 * challenge and writes n_mles x [c0,c1]. */
int dp_sc_finish(dp_sc *s, const uint64_t *last_challenge, uint64_t *out_final_evals);
int dp_sc_destroy(dp_sc *s);
/* Non-owning view of MLE `idx` as folded so far (valid until the next dp_sc_round / dp_sc_destroy):
 * the state's `poly.flattened_ml_extensions[idx]` after the rounds run so far. */
int dp_sc_current_mle(dp_sc *s, uint32_t idx, dp_mle **out_view);

/* ---- zkml lookup: LogUp-GKR fractional-sum circuit (zkml/src/lookup/logup_gkr/circuit.rs) --------------- */
typedef struct dp_logup dp_logup;
/* LogUpCircuit::new_lookup_circuit (multiplicities == NULL; numerators are -1) or new_table_circuit.
 * columns: Base MLEs of equal power-of-two length; denominators are c + sum_k gamma^k col_k[i]. */
int dp_logup_build(dp_mle *const *columns, uint32_t n_columns, const dp_mle *multiplicities, const uint64_t constant_challenge[2],
                   const uint64_t column_separation_challenge[2], dp_logup **out);
int dp_logup_num_vars(const dp_logup *l, uint32_t *input_layer_num_vars);   /* LogUpCircuit::num_vars */
int dp_logup_outputs(const dp_logup *l, uint64_t out[8]);                    /* [n0, n1, d0, d1] x [c0,c1] */
/* LogUpLayer::get_mles of the layer whose halves have `layer_vars` variables: non-owning views
 * [num_low, num_high, den_low, den_high] (or [den_low, den_high] for the initial lookup layer). */
int dp_logup_layer_mles(const dp_logup *l, uint32_t layer_vars, dp_mle **out_views, uint32_t *n_views);
int dp_logup_free(dp_logup *l);
/* *n_layers = how many layers, from the layer whose halves have first_layer variables upwards, dp_logup_run_layers_fs (or, for a
 * BlakeTranscript, dp_logup_run_layers_fs_blake) proves for this
 * batch of circuits (0: none, the caller proves each layer with the sumcheck entry points).  Nonzero only in the blocking wait mode
 * (dp_set_wait_mode(1)), for at most 16 circuits of one size and layers whose first sumcheck round is small enough to run resident. */
int dp_logup_layers_fs_next(dp_logup *const *circuits, uint32_t n_circuits, uint32_t first_layer, uint32_t *n_layers);
/* Layers first_layer..last_layer of logup_gkr::prover::batch_prove (prover.rs:62-170) in one resident launch with BasicTranscript's
 * Fiat-Shamir on the device.  Per layer v: append the claim, append_usize(v), append_usize(3), prove_parallel on the layer's
 * VirtualPolynomial (eq(point) times each circuit's views, coefficients alpha^c (1, 1, lambda), or (-1, -1, lambda) for the two-view
 * first layer of a lookup circuit), take the final evaluations, draw logup_batching, logup_alpha and logup_lambda and form the next
 * claim and point.  In/out: claim [c0,c1]; point (in: first_layer elements, the last one the batching challenge; out: last_layer + 1);
 * alpha, lambda [c0,c1]; sponge, the 14-word Poseidon2 duplex state of dp_sc_run_tail_fs.  Out, layer after layer: msgs_out
 * v x 4 x [c0,c1] (the round messages), challenges_out v x [c0,c1] (the sumcheck point), evals_out n_views x n_circuits x [c0,c1]
 * (the final evaluations without eq's, in add_mle_list order: [num_lo, den_hi, num_hi, den_lo] per circuit, [den_hi, den_lo] with
 * two views).  DP_ERR_STATE unless dp_logup_layers_fs_next(first_layer) covers last_layer. */
int dp_logup_run_layers_fs(dp_logup *const *circuits, uint32_t n_circuits, uint32_t first_layer, uint32_t last_layer, uint64_t *claim,
                           uint64_t *point, uint64_t *alpha, uint64_t *lambda, uint64_t *sponge, uint64_t *msgs_out, uint64_t *challenges_out,
                           uint64_t *evals_out);
/* dp_logup_run_layers_fs with BlakeTranscript's Fiat-Shamir on the device; state: a DP_B3T_WORDS image, in and out.  Arguments,
 * outputs and DP_ERR_STATE as dp_logup_run_layers_fs; DP_ERR_INVALID for an invalid image. */
int dp_logup_run_layers_fs_blake(dp_logup *const *circuits, uint32_t n_circuits, uint32_t first_layer, uint32_t last_layer, uint64_t *claim,
                                 uint64_t *point, uint64_t *alpha, uint64_t *lambda, uint64_t *state, uint64_t *msgs_out, uint64_t *challenges_out,
                                 uint64_t *evals_out);
/* out = sum_k coefs[k] * mles[k] over Ext MLEs of equal length (same_poly.rs:91-110 final_beta). */
int dp_mle_linear_combination(dp_mle *const *mles, const uint64_t *coefs, uint32_t n, dp_mle **out);

/* ---- FFT-convolution layer (zkml/src/layers/convolution.rs, zkml/src/tensor.rs:220-523, zkml/src/iop/prover.rs:164-399) --
 * The tensors a convolution proof consumes (FFT of the reversed input, the product tensor, the reduced FFT-matrix rows
 * W(r, .) with their per-level prefixes) are built on the device next to the sumchecks that read them. */
/* tensor.rs:261-323 `fft(v, flag)` applied to every row of an Ext MLE viewed as [len >> log_n][2^log_n], in place;
 * natural order in and out, root = get_root_of_unity(log_n) (tensor.rs:220), inverse includes the 1/n scaling. */
int dp_fft_rows(dp_mle *m, uint32_t log_n, int inverse);
/* dp_fft_rows for rows of 2^14..2^21 (padded image widths 128..1024): the same transform, contract and root table, as a
 * four-step FFT in two passes over HBM with a scratch tensor the size of the MLE.  The caller picks by the row length. */
int dp_fft_rows_long(dp_mle *m, uint32_t log_n, int inverse);
/* index_w / index_wf (tensor.rs:236-253, convolution.rs:1535-1550): every source row holds an n_real x n_real block that is
 * placed top-left in an n x n grid and zero-padded to out_len; the result is Ext, rows * out_len long. */
int dp_pad_rows(const dp_mle *src, uint64_t rows, uint32_t n_real, uint32_t n, uint64_t out_len, dp_mle **out);
/* fft_conv accumulation (tensor.rs:489-509): out[i][k] = sum_j x_fft[j][k] * w_fft[i][j][k]; x_fft [kx][row_len], w_fft [kw][kx][row_len]. */
int dp_conv_prod(const dp_mle *x_fft, const dp_mle *w_fft, uint32_t kw, uint32_t kx, uint64_t row_len, dp_mle **out);
/* index_u + to_element + add_bias (tensor.rs:255-259,343-361; convolution.rs:152-162): out_host[i][t] =
 * to_element(out_rows[i][n_x^2 - 1 - t]) + bias[i], out_rows = iFFT(prod) as [kw][2 n_x^2]; bias and out_host are HOST arrays. */
int dp_conv_output_elements(const dp_mle *out_rows, uint32_t kw, uint32_t n_x, const int64_t *bias, int64_t *out_host);
/* the same tensor kept on the device: *after = to_field(index_u + to_element + add_bias) as a Base MLE [kw][n_x^2], and
 * *cleared = after * mask, the layer's clearing tensor (convolution.rs:1484-1530); bias [kw] and mask [kw][n_x^2] are Base MLEs
 * of canonical field elements. */
int dp_conv_output(const dp_mle *out_rows, uint32_t kw, uint32_t n_x, const dp_mle *bias, const dp_mle *mask, dp_mle **after, dp_mle **cleared);
/* index_x (tensor.rs:343-361): every row of `row_len` values of a Base MLE reversed, into a new MLE. */
int dp_reverse_rows(const dp_mle *src, uint64_t row_len, dp_mle **out);
/* Prover::phi_g_init (iop/prover.rs:231-289): w_red = W(rx, .) of the FFT (is_fft = 0) or iFFT (is_fft = 1, the reference's
 * flag value in prove_batch_ifft) matrix scaled by `scale`, length 2^n, plus the n - 1 intermediate tables mid[i] (2^(i+1) values). */
int dp_phi_g_init(const uint64_t *rx, uint32_t n, const uint64_t scale[2], int is_fft, dp_mle **w_red, dp_mle **mid);
/* dp_phi_g_init for 15 <= n <= 21 (the FFT rows of dp_fft_rows_long): same arguments and outputs; the levels wider than one
 * block run as one grid launch each. */
int dp_phi_g_init_long(const uint64_t *rx, uint32_t n, const uint64_t scale[2], int is_fft, dp_mle **w_red, dp_mle **mid);
/* one level of delegate_matrix_evaluation (iop/prover.rs:182-195): out[i] = A + B * omega^(i << shift), omega =
 * get_root_of_unity(n_total) (its inverse when `inverse`), i < 2^len_log; A, B are Ext scalars the host derives from r1, r2. */
int dp_phi_level(uint32_t len_log, uint32_t n_total, uint32_t shift, const uint64_t A[2], const uint64_t B[2], int inverse, dp_mle **out);
/* out = src repeated `times` times back to back (beta_acc, convolution.rs:870). */
int dp_mle_repeat(const dp_mle *src, uint32_t times, dp_mle **out);

/* ---- mpcs: Basefold over RS code (rate 1/2, 200 queries, basecode 2^7) + Poseidon2 Merkle trees ------ */
typedef struct dp_pcs_comm dp_pcs_comm;  /* BasefoldCommitmentWithWitness (mpcs/src/basefold/structure.rs:63-72) */
typedef struct dp_pcs_open dp_pcs_open;  /* prover state of one commit phase (oracles + their trees) */

/* MerkleHasher of every commitment built from now on (process-wide): 0 = PoseidonHasher (default), 1 = BlakeHasher
 * (mpcs/src/util/hash.rs:44-98; the reference selects with the cargo feature `blake`, mpcs/src/lib.rs:339-342).  Digests are
 * 4 x u64 in both cases (BLAKE3: the 32 digest bytes as little-endian words).  Do not mix hashers within one proof. */
int dp_set_merkle_hasher(int kind);
int dp_get_merkle_hasher(void);
/* Optional: replace the built-in Poseidon2 constants (HL Goldilocks width-8 instance) with the ones the
 * Rust host reads from p3-goldilocks: ext_rc[2][4][8], int_rc[22], diag[8]  (ff_ext/src/lib.rs:179-194). */
int dp_poseidon2_init(const uint64_t *ext_rc, const uint64_t *int_rc, const uint64_t *diag);
/* Basefold::commit (basefold.rs:304-354).  `full_message_size_log` is the trimmed parameter size
 * (RSCodeProverParameters.full_message_size_log, rs.rs:222-227): it fixes the coset shift.  Polynomials
 * with <= 7 variables get a Merkle tree over their raw evaluations ("TooSmall", basefold.rs:102-104). */
int dp_pcs_commit(const dp_mle *poly, uint32_t full_message_size_log, dp_pcs_comm **out);
/* n independent commitments issued concurrently (what the reference does from rayon workers:
 * activation.rs:293, requant.rs:298/315, lookup/context.rs:677); same results as n dp_pcs_commit calls. */
int dp_pcs_commit_many(const dp_mle *const *polys, uint32_t n, uint32_t full_message_size_log, dp_pcs_comm **out);
/* Basefold::batch_commit (mpcs/src/basefold.rs:356-452): n polynomials of equal size and field type under ONE Merkle tree with
 * batch leaves (merkle_tree.rs:68-74,286-312; hash_two_leaves_batch_*, util/hash.rs:30-41).  dp_pcs_comm_info gives the root.
 * dp_pcs_comm_part(i) is a borrowed per-polynomial view (own codeword, the batch tree's digests): simple_batch_open
 * (basefold.rs:777-861) is dp_pcs_open_begin over the n views with coeffs = eq(t)[0..n] followed by the usual rounds, and
 * dp_pcs_open_query returns for view i its leaf pair and the (shared) batch path -- see host/mpcs.hpp::simple_batch_open. */
int dp_pcs_batch_commit(const dp_mle *const *polys, uint32_t n, uint32_t full_log, dp_pcs_comm **out);
uint32_t dp_pcs_comm_num_polys(const dp_pcs_comm *c);
int dp_pcs_comm_part(const dp_pcs_comm *c, uint32_t i, const dp_pcs_comm **out);
int dp_pcs_comm_info(const dp_pcs_comm *c, uint32_t *num_vars, int *is_base, int *is_trivial, uint64_t root[4]);
int dp_pcs_comm_codeword(const dp_pcs_comm *c, dp_mle **out_view);   /* bit-reversed codeword (view) */
int dp_pcs_comm_bh_evals(const dp_pcs_comm *c, dp_mle **out_view);   /* bit-reversed evaluations (view) */
int dp_pcs_comm_free(dp_pcs_comm *c);
/* commit_phase (commit_phase.rs:30-183) when coeffs == NULL (one commitment, num_vars == its size), else
 * batch_commit_phase (:187-358) with one E coefficient per commitment.  Returns the first sumcheck
 * message as 3 coefficients [c0,c1,c2] x [limb0,limb1].  The host appends it to the transcript, squeezes
 * "commit round" and calls dp_pcs_open_round. */
int dp_pcs_open_begin(const dp_pcs_comm *const *comms, const uint64_t *coeffs, uint32_t n_comms, const uint64_t *point,
                      uint32_t num_vars, dp_pcs_open **out, uint64_t first_msg[6]);
/* Fold by `challenge`.  If *is_last == 0: next_msg (3 coefficients) and the root of the folded oracle's
 * Merkle tree are returned (the host appends msg later and the root now).  If *is_last == 1 the final
 * message is ready (dp_pcs_open_final_message) and next_msg/root are untouched. */
int dp_pcs_open_round(dp_pcs_open *o, const uint64_t challenge[2], uint64_t next_msg[6], uint64_t root[4], int *is_last);
int dp_pcs_open_final_message(dp_pcs_open *o, uint64_t *out /* 2^7 x [c0,c1] */);
/* Query phase gather (query_phase.rs:373-474).  For each x index, for every commitment (codeword index
 * x >> (log N - log |codeword|)) and then every round oracle i (index x >> (i+1)):
 *   [p0.c0 p0.c1 p1.c0 p1.c1] (Base values have c1 = 0) followed by the Merkle path without leaf sibling
 *   or root (log|leaves| - 1 digests of 4 limbs).  dp_pcs_open_query_words() = words per x index. */
uint64_t dp_pcs_open_query_words(const dp_pcs_open *o);
int dp_pcs_open_query(dp_pcs_open *o, const uint64_t *x_indices, uint32_t n, uint64_t *out);
int dp_pcs_open_free(dp_pcs_open *o);

/* ---- ONE polynomial sharded over the GPUs of a node (SURVEY.md 8e, BASELINE configs[3]; one process per GPU) ------------------
 * The reference has no counterpart (it is single-host, rayon-parallel); the split follows its data layout: rank g of world = 2^k
 * owns the contiguous slice [g L/world, (g+1) L/world) of every bit-reversed table of length L (evaluations, codeword, the folded
 * oracles), so the folds (adjacent pairs), the Basefold-internal sumcheck (LSB-first) and the Merkle subtrees are local, and the
 * per-round exchange is one all-gather of a partial 3-coefficient message plus a 32-byte subtree root.  The proof is bit-identical
 * to the unsharded one.  Orchestration: deep-prove_b200/multigpu.py (basefold_commit_open_sharded). */
/* every rank passes the whole polynomial; the handle keeps this rank's slices; root (dp_pcs_comm_shard_info) = SUBTREE root */
int dp_pcs_commit_shard(const dp_mle *poly, uint32_t full_message_size_log, uint32_t rank, uint32_t world, dp_pcs_comm **out);
int dp_pcs_comm_shard_info(const dp_pcs_comm *c, uint32_t *rank, uint32_t *world, uint64_t local_root[4]);
/* roots: world x 4 words rank-major (all-gathered subtree roots) -> the root of the whole tree (== dp_pcs_commit's) */
int dp_pcs_comm_set_shard_roots(dp_pcs_comm *c, const uint64_t *roots, uint64_t out_root[4]);
/* dp_pcs_open_begin / dp_pcs_open_round on a sharded commitment return PARTIAL messages (add the ranks' coefficient triples
 * mod p) and SUBTREE roots; after each round that returned a root, hand the all-gathered roots back with this call to obtain the
 * oracle's root.  dp_pcs_open_final_message returns this rank's (2^7 / world) entries of the bit-reversed final message;
 * dp_pcs_open_query fills the rows of the queries whose leaf pair this rank owns and zeroes the rest (sum the ranks' buffers). */
int dp_pcs_open_set_shard_roots(dp_pcs_open *o, const uint64_t *roots, uint64_t out_root[4]);

/* ---- quantised inference + lookup-witness generation on the device (SURVEY.md 8f.3) ---------------------------------
 * Replaces the host loops of Dense::op (zkml/src/layers/dense.rs), Requant::op / gen_lookup_witness
 * (layers/requant.rs:208-330), Activation::gen_lookup_witness (layers/activation.rs:238-323), Maxpool2D::op + compute_polys
 * (layers/pooling.rs:210-271,667-771) and the multiplicity counting of generate_lookup_witnesses (lookup/context.rs:675-737).
 * Tensors are Base MLEs of canonical field elements of signed integers (exactly Tensor<Element>::to_field), so a trace
 * tensor is itself a witness column.  One dp_wit per proof holds the tables' multiplicity histograms; the node calls add
 * their lookups to them.  Table types as in lookup/context.rs:53-63: kind 0 Relu, 2 Range, 3 Clamping(size). */
typedef struct dp_wit dp_wit;
int dp_wit_begin(uint32_t n_tables, const uint32_t *kinds, const uint32_t *sizes, dp_wit **out);
int dp_wit_dense(const dp_mle *weights /* [nrows][ncols] */, const dp_mle *bias, const dp_mle *x, uint32_t nrows, uint32_t ncols, dp_mle **out);
/* MatMul::op (layers/matrix_mul.rs:230-311): left [R][K] x right ([K][C], or [C][K] when `transposed`: Config::TransposeB) + bias[C] on every
 * row (bias may be NULL) -> [R][C] */
int dp_wit_matmul(const dp_mle *left, const dp_mle *right, const dp_mle *bias, uint32_t R, uint32_t K, uint32_t C, int transposed, dp_mle **out);
/* cols[0] clamping input, cols[1] clamping output (= the node's output tensor), cols[2 ..] the shift / BIT_LEN byte chunks.
 * Inputs with |x| > 2^intermediate_bit_size set error bit 1; intermediate_bit_size must be at most 62 (the reference requires
 * intermediate_bit_size + fp_scale <= 63, requant.rs:423-427), larger values are refused with DP_ERR_INVALID. */
int dp_wit_requant(dp_wit *w, const dp_mle *x, uint32_t shift, int64_t fixed_point_multiplier, uint32_t intermediate_bit_size,
                   uint32_t clamp_table, uint32_t range_table, dp_mle **cols, uint32_t n_cols);
int dp_wit_relu(dp_wit *w, const dp_mle *x, uint32_t relu_table, dp_mle **out);
/* cols[0..3] = out - in(2r+dr, 2c+dc) for (dr,dc) = (0,0),(1,0),(0,1),(1,1); cols[4] = the pooled output [C][H/2][W/2] */
int dp_wit_pool(dp_wit *w, const dp_mle *x, uint32_t C, uint32_t H, uint32_t W, uint32_t range_table, dp_mle **cols);
/* multiplicity polynomial of every table (dp_wit_begin order).  error_bits != 0: a value fell outside its table (1 requant
 * input too large, 2 clamping, 4 relu, 8 pooling) -- the reference panics there. */
int dp_wit_finish(dp_wit *w, dp_mle **mults, uint32_t *error_bits);
int dp_wit_free(dp_wit *w);

/* ---- batch inference without proving (csrc/infer.cu) ------------------------------------------------------------------
 * The model's integer outputs for many inputs at once, exactly as the witness path computes them (same values, same error bits),
 * with every Dense / MatMul / Convolution on the int8 tensor cores (int32 accumulation).  A plan is built once per model from its
 * nodes; each run takes host inputs and writes host outputs in the padded layout of the last node's output tensor.
 * The plan refuses (DP_ERR_INVALID, naming the node): a weight outside [-128, 127], a bias outside int32, a Dense / MatMul /
 * Convolution whose input is not 8-bit (not the model input nor a Requant output, optionally through Relu and/or Maxpool), an
 * output row or channel with 128 * sum|w| + |b| > 2^31 - 1 (int32 accumulation would not be exact), a Convolution filter wider than
 * its padded image (real_nw > nw: the prover refuses it too), and shapes that do not chain. */
typedef struct dp_infer dp_infer;
typedef struct dp_infer_node {
    uint32_t kind;        /* the layer-descriptor kinds: 0 Dense, 1 Requant, 2 Relu, 3 Convolution, 4 Maxpool (2x2, stride 2), 5 MatMul */
    uint32_t dims[7];     /* Dense {nrows, ncols}; Convolution {kw, kx, nw, real_nw, unpadded_out[3]}; Maxpool {C, H, W};
                             MatMul {R, K, C, transposed} */
    uint32_t shift, clamp_size, intermediate_bits;   /* Requant: fp_scale + right_shift, the clamping table's bits, log2 of the input bound */
    int64_t multiplier;                              /* Requant: fixed_point_multiplier */
    const int64_t *weights, *bias;   /* Dense [nrows][ncols] + [nrows]; Convolution [kw][kx][real_nw][real_nw] + [kw];
                                        MatMul [K][C] ([C][K] when transposed) + [C] or NULL; read during dp_infer_plan only */
} dp_infer_node;
/* Inputs per device pass: a run processes its batch in chunks of at most this many inputs, fewer when free device memory is short. */
#define DP_INFER_MAX_CHUNK 4096
int dp_infer_plan(const dp_infer_node *nodes, uint32_t n_nodes, uint64_t input_len, dp_infer **out);
/* inputs: n x input_len; outputs: n x (the last node's output length); err_bits[j]: input j's lookup error bits as dp_wit_finish
 * reports them (1 requant input too large, 2 clamping, 4 relu, 8 pooling), plus 16 when one of its values lies outside [-128, 127]
 * (such an input is computed as zeros).  Runs on the calling thread's context and stream; returns when the outputs are written. */
int dp_infer_run(dp_infer *p, const int64_t *inputs, uint32_t n, int64_t *outputs, uint32_t *err_bits);
int dp_infer_free(dp_infer *p);

#ifdef __cplusplus
}
#endif
#endif /* DEEPPROVE_B200_H */
