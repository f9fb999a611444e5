/*
 * snarkvm_b200 — C ABI of the H100 (sm_90a) proving backend for snarkVM's two hot paths:
 *   VariableBase::msm over BLS12-377 G1 and the radix-2 EvaluationDomain NTT over Fr.
 *
 * PART 1 is the drop-in boundary: the three symbols the reference's Rust FFI binds
 * (declared at /root/reference/algorithms/cuda/src/lib.rs:42-69, defined by the reference at
 * algorithms/cuda/cuda/snarkvm_api.cu:52-84).  Same names, argument order, data layouts and
 * error convention, so `snarkvm-algorithms-cuda` links against this library unchanged
 * (see INTEGRATION.md).
 *
 * PART 2 is the extended, device-resident API (pointers already in HBM) used by the
 * host mirror, bench.py and multi-GPU sharding.
 *
 * Data layouts (identical to the reference's in-memory Rust types):
 *   Fr element   : 32 B, 4 x u64 little-endian limbs, Montgomery form  (fields/src/fp_256.rs:52)
 *   MSM scalar   : 32 B, canonical integer < r, NOT Montgomery         (BigInteger256; snarkvm.cu:275 mont=false)
 *   G1 affine    : x[48] y[48] (Montgomery Fq) infinity[1] pad -> 104-byte stride
 *                  (curves/src/templates/short_weierstrass_jacobian/affine.rs:41-46; lib.rs:161)
 *   G1 projective: X[48] Y[48] Z[48] Jacobian, infinity <=> Z == 0     (projective.rs:36-60)
 */
#ifndef SNARKVM_B200_H
#define SNARKVM_B200_H

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define SNARKVM_API __attribute__((visibility("default")))
#else
#define SNARKVM_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------
 * PART 1 — drop-in replacements for the reference FFI
 * ---------------------------------------------------------------------------------------- */

/* #[repr(C)] enums of algorithms/cuda/src/lib.rs:22-40 */
typedef enum { SNARKVM_NTT_NN = 0, SNARKVM_NTT_NR = 1, SNARKVM_NTT_RN = 2, SNARKVM_NTT_RR = 3 } snarkvm_ntt_order_t;
typedef enum { SNARKVM_NTT_FORWARD = 0, SNARKVM_NTT_INVERSE = 1 } snarkvm_ntt_direction_t;
typedef enum { SNARKVM_NTT_STANDARD = 0, SNARKVM_NTT_COSET = 1 } snarkvm_ntt_type_t;

/* `cuda::Error` of sppark::cuda_error!() (lib.rs:19), returned BY VALUE.  The Rust side reads
 * .code (lib.rs:93,141,164; 0 = success, otherwise a cudaError_t) and frees .message, which is
 * therefore malloc()ed or NULL (shape evidenced at algorithms/cuda/cuda/snarkvm.cu:279). */
typedef struct {
    int code;
    char* message;
} snarkvm_error_t;

/* Replaces `snarkvm_ntt` (lib.rs:43-49 ; snarkvm_api.cu:53-62 ; called from
 * algorithms/src/fft/domain.rs:375-388, 404-417, 425-438).  In-place transform of 2^lg_domain_size
 * Fr elements in HOST memory.  NN (the only order any reference caller passes) is native; NR / RN / RR
 * add explicit bit-reversal passes (R = bit-reversed index order on that side).  On failure `inout` is
 * left untouched and a non-zero cudaError_t is returned, which makes the Rust caller fall back to CPU. */
SNARKVM_API snarkvm_error_t snarkvm_ntt(void* inout, uint32_t lg_domain_size, snarkvm_ntt_order_t ntt_order,
                            snarkvm_ntt_direction_t ntt_direction, snarkvm_ntt_type_t ntt_type);

/* Replaces `snarkvm_polymul` (lib.rs:51-60 ; snarkvm_api.cu:64-75 ; called from
 * algorithms/src/fft/polynomial/multiplier.rs:79-95).  out[2^lg] = iNTT( prod NTT(pad(poly_i)) * prod eval_j ).
 * polynomials: const Fr* [pcount] with lengths plens[] (<= 2^lg); evaluations: const Fr* [ecount] in natural
 * order with elens[] == 2^lg.  0 operands: success, out untouched. */
SNARKVM_API snarkvm_error_t snarkvm_polymul(void* out, size_t pcount, const void* polynomials, const void* plens, size_t ecount,
                                const void* evaluations, const void* elens, uint32_t lg_domain_size);

/* Replaces `snarkvm_msm` (lib.rs:62-68 ; snarkvm_api.cu:77-83 ; called from
 * algorithms/src/msm/variable_base/mod.rs:33-42).  out (144 B) = sum scalars[i] * points[i], i < npoints.
 * The result is written NORMALISED (Z = Montgomery one, or (0, R, 0) for infinity), i.e. the bytes of
 * `reference_result.to_affine().to_projective()`. */
SNARKVM_API snarkvm_error_t snarkvm_msm(void* out, const void* points_with_infinity, size_t npoints, const void* scalars,
                            size_t ffi_affine_sz);

/* ------------------------------------------------------------------------------------------
 * PART 2 — extended API.  `d_` pointers are device pointers on the CURRENT device; `stream` is a
 * cudaStream_t (NULL = legacy default stream).  All functions return 0 or a cudaError_t.
 * ---------------------------------------------------------------------------------------- */

SNARKVM_API const char* snarkvm_b200_version(void);
/* number of CUDA kernels this library has launched in this process (bench.py's gpu_launches) */
SNARKVM_API uint64_t snarkvm_b200_launch_count(void);

/* In-place transform of 2^lg Fr elements resident in HBM (any of the four orders).  d_scratch: 2^lg elements or NULL. */
SNARKVM_API int snarkvm_b200_ntt_device(void* d_inout, uint32_t lg, int ntt_order, int ntt_direction, int ntt_type,
                            void* d_scratch, void* stream);

/* Device-resident polymul: d_out[2^lg]; polys/evals are HOST arrays of device pointers. */
SNARKVM_API int snarkvm_b200_polymul_device(void* d_out, size_t pcount, const void* const* d_polys, const size_t* plens,
                                size_t ecount, const void* const* d_evals, const size_t* elens, uint32_t lg,
                                void* stream);

/* Window/bucket plan the MSM will use for npoints (signed c-bit digits). */
SNARKVM_API int snarkvm_b200_msm_plan(size_t npoints, int* c, int* nwin, uint32_t* cap);
/* batched-affine pair levels the plan for `npoints` runs before the XYZZ accumulation (0 = gather + XYZZ only) */
SNARKVM_API int snarkvm_b200_msm_plan_levels(size_t npoints);

/* Full MSM with bases and scalars resident in HBM; out144 is HOST memory (normalised projective). */
SNARKVM_API int snarkvm_b200_msm_device(void* out144, const void* d_points, size_t npoints, const void* d_scalars,
                            size_t stride, void* stream);

/* `count` MSMs over the SAME resident bases in ONE pass (all commitments of a prover round share powers_of_beta_g,
 * polycommit/sonic_pc/mod.rs:177-257): one digit/sort keyed by (vector, window, bucket), one set of pair levels, one D2H and one
 * synchronisation.  d_scalars / nscalars: HOST arrays of device pointers / lengths (canonical 32-byte integers);
 * out144s: count * 144 B of HOST memory.  Vector i uses the first nscalars[i] bases. */
SNARKVM_API int snarkvm_b200_msm_batch_device(void* out144s, const void* d_points, size_t stride, const void* const* d_scalars,
                                              const size_t* nscalars, size_t count, void* stream);

/* MSM pieces for multi-GPU sharding: per-window sums as XYZZ points (192 B each) in HBM ... */
SNARKVM_API int snarkvm_b200_msm_window_sums_device(void* d_window_sums /* nwin * 192 B */, const void* d_points, size_t npoints,
                                        const void* d_scalars, size_t stride, void* stream);
/* ... under the plan of `plan_npoints` >= npoints: every rank of a sharded MSM passes the size of the LARGEST shard, so all ranks
 * use the same window size and window count whatever their own shard length (snarkvm_b200_msm_plan(plan_npoints) gives nwin and c);
 * an empty shard (npoints = 0) contributes infinity sums.  d_flags: device u32 that receives bit 0 = "a scalar has bits 253..255
 * set" (the sums are then meaningless), or NULL to ignore. */
SNARKVM_API int snarkvm_b200_msm_window_sums_plan_device(void* d_window_sums, uint32_t* d_flags, size_t plan_npoints, const void* d_points,
                                                         size_t npoints, const void* d_scalars, size_t stride, void* stream);
/* ... the same from HOST buffers: uploads the shard (point ranges overlapped with the kernels of the previous range, pageable sources
 * staged through pinned buffers) and leaves its window sums in HBM without synchronising, so a collective can follow at once. */
SNARKVM_API int snarkvm_b200_msm_window_sums_host(void* d_window_sums, uint32_t* d_flags, size_t plan_npoints, const void* h_points,
                                                  size_t npoints, const void* h_scalars, size_t stride, void* stream);
/* ... summed across ranks after an all-gather: d_out[i] = sum_r d_in[r][i] ... */
SNARKVM_API int snarkvm_b200_xyzz_sum_ranks_device(void* d_out, const void* d_in, int nranks, int count, void* stream);
/* ... and folded on the host: out144 = sum_w 2^(c*w) * window_sums[w]  (h_window_sums in HOST memory). */
SNARKVM_API int snarkvm_b200_msm_finish(void* out144, const void* h_window_sums, int nwin, int c);

/* KZG10::commit core (algorithms/src/polycommit/kzg10/mod.rs:98-156): Montgomery coefficients ->
 * canonical (to_bigint, :455-474) -> MSM against resident powers.  out144 is HOST memory. */
SNARKVM_API int snarkvm_b200_kzg_commit_device(void* out144, const void* d_powers, size_t stride, const void* d_coeffs_mont,
                                   size_t ncoeffs, void* stream);

/* Fixed base sets (an SRS kept in HBM across many commitments): precompute the tables 2^(c*w) * P_i, w < nwin, once; every MSM
 * over those bases then uses ONE bucket set for all windows (c = 22, 12 windows at 2^24 points instead of 17 / 15).  The handle owns
 * npoints * nwin * 128 bytes of HBM (25.8 GB at 2^24).  nscalars <= npoints selects the prefix P_0..P_{nscalars-1}
 * (`&powers_of_beta_g[..len]`, polycommit/kzg10/mod.rs:121-135).  Results are the same group elements as snarkvm_b200_msm_device. */
SNARKVM_API int snarkvm_b200_msm_precompute_device(void** handle_out, const void* d_points, size_t npoints, size_t stride, void* stream);
SNARKVM_API int snarkvm_b200_msm_precomputed_free(void* handle);
SNARKVM_API int snarkvm_b200_msm_precomputed_info(const void* handle, size_t* npoints, int* c, int* nwin, size_t* table_bytes);
SNARKVM_API int snarkvm_b200_msm_precomputed_device(void* out144, const void* handle, const void* d_scalars, size_t nscalars, void* stream);
SNARKVM_API int snarkvm_b200_kzg_commit_precomputed_device(void* out144, const void* handle, const void* d_coeffs_mont, size_t ncoeffs,
                                                           void* stream);

/* KZG10::commit with hiding_bound = Some(_) (polycommit/kzg10/mod.rs:98-156): MSM(powers_of_beta_g, coeffs) +
 * MSM(powers_of_beta_times_gamma_g, blinding coefficients).  The caller samples the blinding polynomial; all coefficient arrays are
 * Montgomery Fr in HBM; nblinding = 0 gives the plain commitment. */
SNARKVM_API int snarkvm_b200_kzg_commit_hiding_device(void* out144, const void* d_powers, size_t stride, const void* d_coeffs_mont,
                                                      size_t ncoeffs, const void* d_gamma_powers, const void* d_blinding_mont,
                                                      size_t nblinding, void* stream);
/* `count` commitments against the same resident powers in ONE pass (one prover round, polycommit/sonic_pc/mod.rs:177-257).
 * d_coeffs_mont / ncoeffs: HOST arrays of device pointers / lengths; out144s: count * 144 B of HOST memory. */
SNARKVM_API int snarkvm_b200_kzg_commit_batch_device(void* out144s, const void* d_powers, size_t stride, const void* const* d_coeffs_mont,
                                                     const size_t* ncoeffs, size_t count, void* stream);
/* ... with hiding bounds: polynomial i also gets sum_j blinding_i[j] * gamma_powers[j] (nblinding[i] = 0: plain commitment);
 * the blinding terms ride in the same pass as a second scalar segment of the same sum. */
SNARKVM_API int snarkvm_b200_kzg_commit_batch_hiding_device(void* out144s, const void* d_powers, size_t stride,
                                                            const void* const* d_coeffs_mont, const size_t* ncoeffs,
                                                            const void* d_gamma_powers, const void* const* d_blinding_mont,
                                                            const size_t* nblinding, size_t count, void* stream);
/* ... over the precomputed tables of the resident powers (one bucket set per polynomial). */
SNARKVM_API int snarkvm_b200_kzg_commit_batch_precomputed_device(void* out144s, const void* handle, const void* const* d_coeffs_mont,
                                                                 const size_t* ncoeffs, size_t count, void* stream);

/* SonicKZG10::commit for all polynomials of a round (polycommit/sonic_pc/mod.rs:177-257) in one pass: polynomial i is committed
 * against d_bases[i] — the powers (ck.powers()), the powers advanced by max_degree - degree_bound points
 * (ck.shifted_powers_of_beta_g(degree_bound), sonic_pc/data_structures.rs:310-331) or a Lagrange basis (mod.rs:215-227) — plus, when
 * nblinding[i] > 0, sum_j blinding_i[j] * d_gamma_bases[i][j] (hiding_bound = Some(_), kzg10/mod.rs:129-150).  Base slices may
 * overlap (they are merged); all arrays share `stride`.  d_gamma_bases / d_blinding_mont / nblinding may be NULL (no hiding). */
SNARKVM_API int snarkvm_b200_sonic_commit_batch_device(void* out144s, size_t stride, const void* const* d_bases,
                                                       const void* const* d_coeffs_mont, const size_t* ncoeffs,
                                                       const void* const* d_gamma_bases, const void* const* d_blinding_mont,
                                                       const size_t* nblinding, size_t count, void* stream);

/* MSM scratch budget of the current device (bytes): the limit concurrent calls share (60 % of the device unless
 * SNARKVM_B200_SCRATCH_LIMIT_GB is set; callers that do not fit wait instead of failing), what is in flight, and the high-water mark. */
SNARKVM_API int snarkvm_b200_msm_scratch_stats(size_t* limit_bytes, size_t* in_use_bytes, size_t* peak_bytes);
/* change the limit at run time (also resets the high-water mark) */
SNARKVM_API int snarkvm_b200_msm_set_scratch_limit(size_t limit_bytes);

/* FFT over G1 points (EvaluationDomain::{fft,ifft} with T = G1Projective, fft/domain.rs:169-221): 2^lg affine points in, affine
 * points out, natural order.  direction 1 = inverse, which is UniversalParams::lagrange_basis
 * (polycommit/kzg10/data_structures.rs:68-72): the commitment key for commit_lagrange (kzg10/mod.rs:159-206). */
SNARKVM_API int snarkvm_b200_g1_ntt_device(void* d_out, size_t out_stride, const void* d_in, size_t in_stride, uint32_t lg, int direction,
                                           void* stream);

/* batch_inversion_and_mul (fields/src/lib.rs:78-129): v_i <- coeff * v_i^{-1} in place, zeros stay zero.  coeff: 32 B HOST. */
SNARKVM_API int snarkvm_b200_fr_batch_inversion_and_mul_device(void* d_v, size_t n, const void* coeff_mont_host, void* stream);
/* DensePolynomial::divide_by_vanishing_poly (fft/polynomial/dense.rs:162-169): p (m coefficients) = q * (x^n - 1) + r;
 * d_q receives max(m - n, 0) coefficients, d_r receives min(m, n) (neither trimmed). */
SNARKVM_API int snarkvm_b200_poly_divide_by_vanishing_device(void* d_q, void* d_r, const void* d_p, size_t m, size_t n, void* stream);
/* KZG10::compute_witness_polynomial (polycommit/kzg10/mod.rs:220-241): quotient of p (m coefficients) / (x - point); d_q receives
 * m - 1 coefficients; the remainder p(point) is dropped as in the reference.  point: 32 B Montgomery, HOST. */
SNARKVM_API int snarkvm_b200_poly_divide_by_linear_device(void* d_q, const void* d_p, size_t m, const void* point_mont_host, void* stream);
/* z_M = M * (public || private) for a sparse R1CS matrix (inner_product, snark/varuna/ahp/prover/round_functions/mod.rs:169-189,
 * called per row of A, B, C at :128-152).  CSR in HBM: row_ptr = nrows + 1 u32, cols = u32 indices into d_x (nvars Montgomery Fr),
 * vals = Montgomery Fr.  A column >= nvars makes the call return cudaErrorInvalidValue. */
SNARKVM_API int snarkvm_b200_sparse_matvec_device(void* d_out, const void* d_row_ptr, const void* d_cols, const void* d_vals, size_t nrows,
                                                  const void* d_x, size_t nvars, void* stream);
/* Elementwise Fr arithmetic on HBM vectors (the zip loops between transforms, e.g. polycommit/kzg10/mod.rs:292-297,
 * fft/evaluations.rs:49-74): op 0 = a + b, 1 = a - b, 2 = a * b; out may alias an input; the scalar form takes a 32-byte HOST scalar. */
SNARKVM_API int snarkvm_b200_fr_vec_op_device(void* d_out, const void* d_a, const void* d_b, size_t n, int op, void* stream);
SNARKVM_API int snarkvm_b200_fr_vec_scalar_op_device(void* d_out, const void* d_a, const void* scalar_mont_host, size_t n, int op, void* stream);
/* EvaluationDomain::elements (fft/domain.rs:307-309): d_out[i] = group_gen^i, i < 2^lg, Montgomery. */
SNARKVM_API int snarkvm_b200_domain_elements_device(void* d_out, uint32_t lg, void* stream);
/* Varuna's matrix_evals (snark/varuna/ahp/matrices.rs:138-195, called by index_helper, ahp/indexer/indexer.rs:186-203) for one CSR
 * matrix in HBM: row_ptr = nrows + 1 u32, cols = nnz u32 variable indices (public first), vals = nnz Montgomery Fr.  Entry e gets
 * row = w_R^(its row), col = w_C^(reindex_by_subdomain(col), fft/domain.rs:322-344) and row_col_val = val * row * col; entries
 * nnz .. 2^lg_non_zero - 1 get (1, 1, 0).  d_row, d_col, d_row_col_val receive 2^lg_non_zero Montgomery Fr each.  input_size is the
 * (power-of-two) input domain; 2^lg_variable <= input_size (where reindex_by_subdomain errors), nrows > 2^lg_constraint,
 * nnz > 2^lg_non_zero or nvars > 2^lg_variable return cudaErrorInvalidValue before any launch; a column >= nvars returns
 * cudaErrorInvalidValue after the pass.  Synchronises the stream. */
SNARKVM_API int snarkvm_b200_varuna_matrix_evals_device(void* d_row, void* d_col, void* d_row_col_val, const void* d_row_ptr, size_t nrows,
                                                        const void* d_cols, const void* d_vals, size_t nnz, size_t nvars, size_t input_size,
                                                        uint32_t lg_constraint, uint32_t lg_variable, uint32_t lg_non_zero, void* stream);
/* Varuna's transpose (snark/varuna/ahp/matrices.rs:249-270) of the same CSR matrix over the variable domain: transposed row
 * reindex_by_subdomain(col) holds (val, row) for every entry of that column.  d_t_row_ptr receives 2^lg_variable + 1 u32, d_t_cols nnz
 * u32 row indices, d_t_vals nnz Montgomery Fr; the order of the entries inside a transposed row is unspecified (equal to the
 * reference's as a matrix).  Same argument checks and errors as snarkvm_b200_varuna_matrix_evals_device.  Synchronises the stream. */
SNARKVM_API int snarkvm_b200_csr_transpose_device(void* d_t_row_ptr, void* d_t_cols, void* d_t_vals, const void* d_row_ptr, size_t nrows,
                                                  const void* d_cols, const void* d_vals, size_t nnz, size_t nvars, size_t input_size,
                                                  uint32_t lg_variable, void* stream);
/* DensePolynomial::evaluate (fft/polynomial/dense.rs:98-114): out = sum c_i * point^i; out and point are 32-byte HOST buffers. */
SNARKVM_API int snarkvm_b200_poly_evaluate_device(void* out_mont_host, const void* d_coeffs, size_t m, const void* point_mont_host,
                                                  void* stream);
/* The circuit id's byte stream of one CSR matrix (Circuit::hash, snark/varuna/ahp/indexer/circuit.rs:109-121, which feeds it to
 * Blake2s): serialize_uncompressed of Vec<Vec<(Fr, usize)>> — [u64 nrows] then per row [u64 len][len x (32 B canonical LE value,
 * u64 LE column)] — written to d_out (out_bytes = 8 + 8 * nrows + 40 * nnz, 8-byte aligned).  Same CSR layout as
 * snarkvm_b200_varuna_matrix_evals_device.  A wrong out_bytes, nnz > 0 with no rows or a misaligned d_out return cudaErrorInvalidValue
 * before any launch; a row_ptr that is not non-decreasing from 0 to nnz returns cudaErrorInvalidValue after the pass.  Synchronises. */
SNARKVM_API int snarkvm_b200_csr_serialize_device(void* d_out, size_t out_bytes, const void* d_row_ptr, size_t nrows, const void* d_cols,
                                                  const void* d_vals, size_t nnz, void* stream);
/* d_out (n Montgomery Fr) = sum_j c_j * p_j over nterms <= 12 polynomials of different lengths, in one pass (the `+= (c, &p)` sequence
 * of LinearCombination polynomials, bit for bit).  d_polys, lens and coeffs_mont_host (nterms x 32 B) are HOST arrays; lens[j] <= n.
 * nterms > 12 or lens[j] > n return cudaErrorInvalidValue before any launch. */
SNARKVM_API int snarkvm_b200_fr_lincomb_device(void* d_out, size_t n, const void* const* d_polys, const size_t* lens, const void* coeffs_mont_host,
                                               uint32_t nterms, void* stream);
/* MatrixEvals::evaluate (snark/varuna/ahp/matrices.rs:114-126): out_mont_host (4 x 32 B HOST) = sum l*row, sum l*col, sum l*row*col,
 * sum l*row_col_val over n Montgomery Fr in HBM, l being the Lagrange coefficients of K at a point.  Synchronises the stream. */
SNARKVM_API int snarkvm_b200_matrix_evals_dot_device(void* out_mont_host, const void* d_row, const void* d_col, const void* d_row_col_val,
                                                     const void* d_lagrange, size_t n, void* stream);

/* Many circuits per call (VarunaSNARK::batch_circuit_setup, varuna.rs:72-134; a deployment's setup and certificates, one circuit
 * per function).  Each entry point below does in ONE pass what the one-matrix entry point above does per matrix; the results are
 * bit-identical to a loop of those calls.  Segment tables are HOST arrays; the device pointers in them follow the layouts above. */

/* In-place transforms, transform i of 2^lgs[i] Fr at d_data[i] (HOST array of device pointers), natural order, one direction and
 * type for all.  Each result equals snarkvm_b200_ntt_device's.  Transforms of equal size share their launches (one launch per pass
 * for all of them); the sizes may be mixed, from 2^0 up. */
SNARKVM_API int snarkvm_b200_ntt_batch_device(void* const* d_data, const uint32_t* lgs, size_t count, int ntt_direction, int ntt_type,
                                              void* stream);

/* One CSR matrix of a segmented indexer call (the arguments of snarkvm_b200_varuna_matrix_evals_device).  d_out: row, col and
 * row_col_val (2^lg_non_zero Fr each) for matrix_evals; d_out[0] alone receives the 8 + 8 * nrows + 40 * nnz bytes (8-byte
 * aligned) of the byte stream for csr_serialize, which reads only the CSR arrays, nrows and nnz. */
typedef struct {
    const void* d_row_ptr;
    const void* d_cols;
    const void* d_vals;
    uint64_t nrows, nnz, nvars, input_size;
    uint32_t lg_constraint, lg_variable, lg_non_zero, reserved;
    void* d_out[3];
} snarkvm_b200_csr_segment_t;
/* matrix_evals of every segment in one launch and one synchronisation.  Argument errors return cudaErrorInvalidValue before any
 * launch.  A bad column or row_ptr in any segment returns cudaErrorInvalidValue after the pass, and *bad_segment (HOST, may be
 * NULL) receives the index of the first such segment (-1 otherwise); outputs are then unspecified. */
SNARKVM_API int snarkvm_b200_varuna_matrix_evals_batch_device(const snarkvm_b200_csr_segment_t* segs, size_t count, int64_t* bad_segment,
                                                              void* stream);
/* The circuit id's byte stream of every segment in one launch and one synchronisation; errors as above. */
SNARKVM_API int snarkvm_b200_csr_serialize_batch_device(const snarkvm_b200_csr_segment_t* segs, size_t count, int64_t* bad_segment,
                                                        void* stream);

/* One output of a segmented linear combination: d_out (n Fr) = sum_j coeffs_mont[j] * d_polys[j], lens[j] <= n, nterms <= 12. */
typedef struct {
    void* d_out;
    uint64_t n;
    const void* d_polys[12];
    uint64_t lens[12];
    uint8_t coeffs_mont[12][32];
    uint32_t nterms, reserved;
} snarkvm_b200_lincomb_segment_t;
/* every segment's combination in one launch (snarkvm_b200_fr_lincomb_device per segment, bit for bit) */
SNARKVM_API int snarkvm_b200_fr_lincomb_batch_device(const snarkvm_b200_lincomb_segment_t* segs, size_t count, void* stream);

/* One matrix of a segmented MatrixEvals::evaluate: its row, col and row_col_val on K (n = |K| Fr each, n a power of two) and the
 * point (32 B Montgomery). */
typedef struct {
    const void* d_row;
    const void* d_col;
    const void* d_row_col_val;
    uint64_t n;
    uint8_t point_mont[32];
} snarkvm_b200_evals_segment_t;
/* For every segment: the Lagrange coefficients of its K at its point (fft/domain.rs:258-292, a point inside K included) and the four
 * inner products of snarkvm_b200_matrix_evals_dot_device with them.  All denominators share one batch inversion; one
 * synchronisation.  out_mont_host: count x 4 x 32 B HOST. */
SNARKVM_API int snarkvm_b200_matrix_evals_at_points_device(void* out_mont_host, const snarkvm_b200_evals_segment_t* segs, size_t count,
                                                           void* stream);

/* The batched Varuna prover (VarunaSNARK::prove_batch, varuna.rs:336-620, over many circuits and instances).  Segment tables are
 * HOST arrays, as above.  Argument errors return cudaErrorInvalidValue before any launch. */

/* One term of an uncapped linear combination: a view of len Fr at d_poly, added times coeff_mont at output positions offset +
 * k * period + u (u < len) for k < reps.  reps = 1 is one plain term (period is then ignored); reps > 1 needs period >= len.  The
 * last copy must end inside its output. */
typedef struct {
    const void* d_poly;
    uint64_t len, offset, period, reps;
    uint8_t coeff_mont[32];
} snarkvm_b200_lincomb_term_t;
/* One output: d_out (n Fr) = the sum of terms [first_term, first_term + nterms) of the term table; positions no term covers are 0. */
typedef struct {
    void* d_out;
    uint64_t n, first_term, nterms;
} snarkvm_b200_lincomb_output_t;
/* every output in one launch, bit-identical to the sequence of scaled, shifted additions it stands for; no cap on the number of
 * terms.  snarkvm_b200_fr_lincomb_batch_device and snarkvm_b200_fr_lincomb_device are calls of this kernel. */
SNARKVM_API int snarkvm_b200_fr_lincomb_terms_device(const snarkvm_b200_lincomb_output_t* outs, size_t nouts,
                                                     const snarkvm_b200_lincomb_term_t* terms, size_t nterms, void* stream);

/* One CSR sparse mat-vec of a segmented call: d_out (nrows Fr) = M * d_x (nvars Fr), with nnz = row_ptr[nrows]. */
typedef struct {
    const void* d_row_ptr;
    const void* d_cols;
    const void* d_vals;
    uint64_t nrows, nnz;
    const void* d_x;
    uint64_t nvars;
    void* d_out;
} snarkvm_b200_spmv_segment_t;
/* every segment's product in one pass of three launches (rows over 256 entries of any segment share one work list) and one
 * synchronisation.  A column >= nvars, or a row_ptr that is not non-decreasing up to nnz, returns cudaErrorInvalidValue after the
 * pass with *bad_segment (HOST, may be NULL) = the first such segment (-1 otherwise).  snarkvm_b200_sparse_matvec_device is a
 * one-segment call. */
SNARKVM_API int snarkvm_b200_sparse_matvec_batch_device(const snarkvm_b200_spmv_segment_t* segs, size_t count, int64_t* bad_segment,
                                                        void* stream);

/* One product of a batched PolyMultiplier: d_out (2^lg Fr) = d_a (len_a Fr) * d_b (len_b Fr) with len_a + len_b - 1 <= 2^lg. */
typedef struct {
    void* d_out;
    const void* d_a;
    const void* d_b;
    uint64_t len_a, len_b;
    uint32_t lg, reserved;
} snarkvm_b200_polymul_job_t;
/* every product in one pass: one load launch, the forward transforms of both operands through snarkvm_b200_ntt_batch_device
 * (equal sizes share launches), one pointwise launch, the inverse transforms the same way.  Each result equals
 * snarkvm_b200_polymul_device of the two operands at the same lg. */
SNARKVM_API int snarkvm_b200_polymul_batch_device(const snarkvm_b200_polymul_job_t* jobs, size_t count, void* stream);

/* One matrix of Varuna's fourth round (fourth.rs:151-245): its row, col, row_col_val on K (n = |K| Fr) and its circuit's constants,
 * all 32 B Montgomery: v_rc = v_R(alpha) * v_C(beta), rc = |R| * |C|, f_scale = v_rc / (|R| * |C|).  Writes, on K:
 * d_a = v_rc * row_col_val, d_b = rc * (row - alpha)(col - beta) and d_f = f_scale * row_col_val / ((row - alpha)(col - beta))
 * (0 where the denominator is 0, as batch_inversion_and_mul leaves it). */
typedef struct {
    const void* d_row;
    const void* d_col;
    const void* d_row_col_val;
    uint64_t n;
    uint8_t v_rc_mont[32], rc_mont[32], f_scale_mont[32];
    void* d_a;
    void* d_b;
    void* d_f;
} snarkvm_b200_round4_segment_t;
/* every segment in one launch, one batch inversion over the concatenation of all denominators and one launch for f; alpha / beta:
 * 32 B Montgomery HOST.  No synchronisation. */
SNARKVM_API int snarkvm_b200_varuna_round4_evals_device(const snarkvm_b200_round4_segment_t* segs, size_t count, const void* alpha_mont,
                                                        const void* beta_mont, void* stream);
/* A fourth-round segment with its own challenges (many proofs in one call): the members of snarkvm_b200_round4_segment_t, then
 * alpha and beta (32 B Montgomery each). */
typedef struct {
    const void* d_row;
    const void* d_col;
    const void* d_row_col_val;
    uint64_t n;
    uint8_t v_rc_mont[32], rc_mont[32], f_scale_mont[32];
    void* d_a;
    void* d_b;
    void* d_f;
    uint8_t alpha_mont[32], beta_mont[32];
} snarkvm_b200_round4_batch_segment_t;
/* snarkvm_b200_varuna_round4_evals_device with each segment's own alpha and beta, in the same three launches; the entry point above
 * is a call of this kernel with its alpha and beta in every segment.  No synchronisation. */
SNARKVM_API int snarkvm_b200_varuna_round4_evals_batch_device(const snarkvm_b200_round4_batch_segment_t* segs, size_t count, void* stream);

/* One polynomial of a segmented evaluation: m Montgomery Fr coefficients at d_coeffs (low degree first) and the point. */
typedef struct {
    const void* d_coeffs;
    uint64_t m;
    uint8_t point_mont[32];
} snarkvm_b200_poly_eval_segment_t;
/* DensePolynomial::evaluate of every segment in one pass: one partial-sum launch over all segments (a long polynomial spreads over
 * many CTAs), one launch that adds each segment's partials, one D2H copy and one synchronisation.  out_mont_host: count x 32 B
 * Montgomery HOST; a segment of length 0 evaluates to 0.  snarkvm_b200_poly_evaluate_device is a one-segment call. */
SNARKVM_API int snarkvm_b200_poly_evaluate_batch_device(void* out_mont_host, const snarkvm_b200_poly_eval_segment_t* segs, size_t count,
                                                        void* stream);
/* One quotient of a segmented division by (x - point): d_q receives m - 1 coefficients of d_p (m coefficients) / (x - point). */
typedef struct {
    void* d_q;
    const void* d_p;
    uint64_t m;
    uint8_t point_mont[32];
} snarkvm_b200_poly_divide_segment_t;
/* KZG10::compute_witness_polynomial of every segment in three launches (local chunk values, one carry CTA per segment, final scan);
 * segments of length 0 and 1 have empty quotients.  No synchronisation.  snarkvm_b200_poly_divide_by_linear_device is a one-segment
 * call. */
SNARKVM_API int snarkvm_b200_poly_divide_by_linear_batch_device(const snarkvm_b200_poly_divide_segment_t* segs, size_t count, void* stream);

/* Fr Montgomery <-> canonical, n elements in HBM (to_bigint / from_bigint, fields/src/fp_256.rs:362-413). */
SNARKVM_API int snarkvm_b200_fr_from_mont_device(void* d_out, const void* d_in, size_t n, void* stream);
SNARKVM_API int snarkvm_b200_fr_to_mont_device(void* d_out, const void* d_in, size_t n, void* stream);

/* SRS ingest: npoints uncompressed canonical G1 points as stored in a `.usrs` file after its 8-byte count (x LE 48 B, y LE 48 B,
 * bit 6 of the last byte = infinity; parameters/src/mainnet/powers.rs, utilities/src/serialize/flags.rs:72-98) -> the reference's
 * Affine images (Montgomery, `stride` bytes apart) in HBM.  *d_invalid (device u32) receives the number of points that are
 * out of range, off the curve y^2 = x^3 + 1 or badly flagged.  d_in96 must be 4-byte aligned. */
SNARKVM_API int snarkvm_b200_srs_decode_device(void* d_out, size_t stride, const void* d_in96, size_t npoints, uint32_t* d_invalid, void* stream);

/* Resident bases for the drop-in snarkvm_msm: upload `host_points` (npoints x stride bytes) to the current device once;
 * later snarkvm_msm calls whose `points_with_infinity` is this same pointer (same stride, npoints <= registered) skip the
 * upload.  The SRS powers of a proving key are constant (polycommit/sonic_pc/data_structures.rs:41-63) and the reference
 * passes the same slice to every commitment.  The caller must not mutate the slice while it is registered. */
SNARKVM_API int snarkvm_b200_register_bases(const void* host_points, size_t npoints, size_t stride);
SNARKVM_API int snarkvm_b200_unregister_bases(const void* host_points);
/* As snarkvm_b200_register_bases, and also builds the fixed-base tables (snarkvm_b200_msm_precompute_device) of the uploaded copy:
 * snarkvm_msm calls on this slice then run over the tables (npoints * nwin * 128 B of HBM, seconds of one-off set-up). */
SNARKVM_API int snarkvm_b200_register_bases_precomputed(const void* host_points, size_t npoints, size_t stride);

/* Per-kernel CUDA-event timing on the launching stream (off by default).  kind: 0 = MSM bucket sort
 * (digit histogram + scatter), 1 = MSM bucket accumulation, 2 = MSM bucket reduction, 3 = NTT passes.
 * collect() waits for the recorded launches of that kind, returns their summed milliseconds and count, and
 * clears them. */
SNARKVM_API int snarkvm_b200_profile_enable(int on);
SNARKVM_API int snarkvm_b200_profile_collect(int kind, double* total_ms, uint64_t* count);

/* Device self-test of the warp-cooperative Fq multiplication / inversion used by the CTA-shared inversions: nwarps pseudo-random cases
 * (plus 0, 1, q - 1 and a long-carry value) checked against the per-thread multiplier; *mismatches (HOST) = failing cases. */
SNARKVM_API int snarkvm_b200_selftest_coop(uint32_t nwarps, uint64_t seed, uint32_t* mismatches, void* stream);
/* host-only self-test of the pageable-memory staging copies (copy-thread pool, non-temporal stores); needs no GPU */
SNARKVM_API int snarkvm_b200_selftest_host_copy(size_t max_bytes, uint64_t seed, uint32_t* mismatches);

/* Element-wise test entry points of the field and group arithmetic, for comparison with big integers.  Operands come from the
 * caller; elements are little-endian 32-bit limbs (Fr 8, Fq 12, Fq2 24 = c0 then c1), Montgomery images unless stated.
 *
 * snarkvm_b200_test_field_op_device: d_out[i] = op(d_a[i], d_b[i]) for i < n, all device pointers.  ctx picks the translation unit
 * the test kernel is compiled in: MSM = msm.cu, where MUL / SQR call the out-of-line mul_call / sqr_call that msm.cu's kernels call
 * as well; NTT = ntt.cu, where they are inlined into the test kernel (a copy of its own, not the one in the NTT butterflies);
 * PAIRING = pairing.cu, which also calls out-of-line mul_call / sqr_call, but its own copies (the library is not built with
 * relocatable device code, so each translation unit compiles its own): the ones every Fq6 / Fq12 product of the pairing calls.
 * Fr and Fq take ops ADD … FROM_MONT and the warp-cooperative COOP_MUL / COOP_INVERSE (one warp per element; a COOP_MUL
 * whose lanes >= N do not return 0 is written as all-ones limbs); Fq2 takes ADD, SUB, NEG, DBL, MUL, SQR, INVERSE; TIMES5 is
 * Fq2::times5 on plain Fq elements (field = FQ).  TO_MONT / FROM_MONT take any value < p. */
enum {
    SNARKVM_B200_TEST_CTX_MSM = 0, SNARKVM_B200_TEST_CTX_NTT = 1, SNARKVM_B200_TEST_CTX_PAIRING = 2,
    SNARKVM_B200_FIELD_FR = 0, SNARKVM_B200_FIELD_FQ = 1, SNARKVM_B200_FIELD_FQ2 = 2,
    SNARKVM_B200_GROUP_G1 = 0, SNARKVM_B200_GROUP_G2 = 1
};
enum {
    SNARKVM_B200_OP_ADD = 0, SNARKVM_B200_OP_SUB = 1, SNARKVM_B200_OP_NEG = 2, SNARKVM_B200_OP_DBL = 3, SNARKVM_B200_OP_HALF = 4,
    SNARKVM_B200_OP_MUL = 5, SNARKVM_B200_OP_MUL_INLINE = 6, SNARKVM_B200_OP_MUL_CALL = 7, SNARKVM_B200_OP_MUL_KARATSUBA = 8,
    SNARKVM_B200_OP_SQR = 9, SNARKVM_B200_OP_SQR_INLINE = 10, SNARKVM_B200_OP_SQR_CALL = 11, SNARKVM_B200_OP_INVERSE = 12,
    SNARKVM_B200_OP_TO_MONT = 13, SNARKVM_B200_OP_FROM_MONT = 14, SNARKVM_B200_OP_TIMES5 = 15,
    SNARKVM_B200_OP_COOP_MUL = 16, SNARKVM_B200_OP_COOP_INVERSE = 17,
    /* group ops: XYZZ points X Y ZZ ZZZ over Fq (G1, 48 words) or Fq2 (G2, 96 words), infinity <=> ZZ == 0 */
    SNARKVM_B200_OP_XYZZ_ADD = 32, SNARKVM_B200_OP_XYZZ_ADD_AFFINE = 33, SNARKVM_B200_OP_XYZZ_DBL = 34,
    SNARKVM_B200_OP_XYZZ_MUL_U32 = 35, SNARKVM_B200_OP_XYZZ_TO_AFFINE = 36,
    SNARKVM_B200_OP_QUAD_ADD = 37, SNARKVM_B200_OP_QUAD_DBL = 38, SNARKVM_B200_OP_QUAD_ADD_AFFINE = 39
};
SNARKVM_API int snarkvm_b200_test_field_op_device(int ctx, int field, int op, void* d_out, const void* d_a, const void* d_b, size_t n,
                                                  void* stream);
/* d_out[i] = op(d_a[i], d_b[i], d_k[i]) over XYZZ points of the group (msm.cu's arithmetic).  ADD: a + b.  ADD_AFFINE: a + (±b) with b
 * read as the affine point (b.X, b.Y), infinity when b.ZZ == 0, negated when d_k[i] != 0.  DBL: 2a.  MUL_U32: d_k[i]·a.
 * TO_AFFINE: X = x, Y = y, ZZ word 0 = the infinity flag, all other words 0.  QUAD_ADD / QUAD_DBL / QUAD_ADD_AFFINE (G1 only): the
 * same operations by four lanes (quad.cuh); a result whose four lanes disagree is written as all-ones words. */
SNARKVM_API int snarkvm_b200_test_curve_op_device(int group, int op, void* d_out, const void* d_a, const void* d_b, const uint32_t* d_k,
                                                  size_t n, void* stream);
/* The host arithmetic that finishes every MSM (host_ec.hpp), on HOST buffers; needs no GPU.  field FQ: ADD, SUB, MUL, SQR, INVERSE;
 * field FQ2: ADD, SUB, MUL, SQR, INVERSE; XYZZ_ADD / XYZZ_DBL on XYZZ points over the field (G1 for FQ, G2 for FQ2). */
SNARKVM_API int snarkvm_b200_test_field_op_host(int field, int op, void* out, const void* a, const void* b, size_t n);
/* The extension tower and the G2 line steps of the pairing (tower.cuh, pairing.cu), element-wise and compiled in pairing.cu, where
 * the pairing kernels call them: d_out[i] = op(d_a[i], d_b[i], d_c[i]) for i < n, all device pointers.  An Fq6 is c0 c1 c2 of Fq2
 * (72 words), an Fq12 is c0 c1 of Fq6 (144 words, the GT image order); a line-step state is X Y Z of Fq2 (72 words).
 *   FQ6_MUL a·b, FQ6_SQR a², FQ6_MUL_BY_NONRESIDUE a·v, FQ6_INVERSE a⁻¹ (zero ↦ zero), FQ6_FROBENIUS a^(q^k), k < 6: Fq6 in and out.
 *   FQ6_MUL_BY_01: a·(b0 + b1·v), d_b = b0 b1 (48 words).
 *   FQ12_MUL a·b, FQ12_SQR a², FQ12_INVERSE a⁻¹ (zero ↦ zero), FQ12_CONJUGATE, FQ12_FROBENIUS a^(q^k), k < 12: Fq12 in and out.
 *   FQ12_CYCLOTOMIC_SQUARE (Granger–Scott) and FQ12_EXP_BY_X (a^X, X = 0x8508c00000000001): a must lie in the cyclotomic subgroup.
 *   FQ12_FINAL_EXPONENTIATION: the pairing's final exponentiation, zero ↦ zero.  FQ12_IS_ONE: one word per element, 1 when a is
 *   the Montgomery image of one, else 0.
 *   FQ12_MUL_BY_034: a·((c0, 0, 0) + (c3, c4, 0)·w), d_b = c0 c3 c4 (72 words).  FQ12_ELL: the Miller loop's line evaluation
 *   a·mul_by_034(c0·p.y, c1·p.x, c2), d_b = a prepared coefficient triple c0 c1 c2 (72 words), d_c = the G1 point p.x p.y (24 words).
 *   G2_DOUBLING_STEP (d_a = X Y Z) and G2_ADDITION_STEP (d_a = X Y Z, d_b = the affine Q: x y, 48 words) of G2 preparation:
 *   the new X Y Z, then the coefficient triple (144 words).  The steps are polynomial formulas: any Fq2 operands are valid.
 * k is the Frobenius power and must be 0 for every other op; an unknown op or a k out of range returns cudaErrorInvalidValue. */
enum {
    SNARKVM_B200_OP_FQ6_MUL = 48, SNARKVM_B200_OP_FQ6_SQR = 49, SNARKVM_B200_OP_FQ6_MUL_BY_01 = 50,
    SNARKVM_B200_OP_FQ6_MUL_BY_NONRESIDUE = 51, SNARKVM_B200_OP_FQ6_INVERSE = 52, SNARKVM_B200_OP_FQ6_FROBENIUS = 53,
    SNARKVM_B200_OP_FQ12_MUL = 54, SNARKVM_B200_OP_FQ12_SQR = 55, SNARKVM_B200_OP_FQ12_MUL_BY_034 = 56,
    SNARKVM_B200_OP_FQ12_CYCLOTOMIC_SQUARE = 57, SNARKVM_B200_OP_FQ12_INVERSE = 58, SNARKVM_B200_OP_FQ12_CONJUGATE = 59,
    SNARKVM_B200_OP_FQ12_FROBENIUS = 60, SNARKVM_B200_OP_FQ12_IS_ONE = 61, SNARKVM_B200_OP_FQ12_EXP_BY_X = 62,
    SNARKVM_B200_OP_FQ12_FINAL_EXPONENTIATION = 63, SNARKVM_B200_OP_FQ12_ELL = 64,
    SNARKVM_B200_OP_G2_DOUBLING_STEP = 65, SNARKVM_B200_OP_G2_ADDITION_STEP = 66
};
SNARKVM_API int snarkvm_b200_test_tower_op_device(int op, int k, void* d_out, const void* d_a, const void* d_b, const void* d_c, size_t n,
                                                  void* stream);
/* The square roots of the point decoders (verify.cu), element-wise and compiled there: the same out-of-line fq_sqrt (Tonelli–Shanks)
 * and fq2_sqrt (by the norm) that k_g1_deserialize and k_g2_deserialize call.  field FQ: d_in and d_out hold n Fq (12 words), field
 * FQ2: n Fq2 (24 words, c0 then c1); Montgomery images below q, d_in and d_out 16-byte aligned.  d_ok[i] (int32, 4-byte aligned)
 * is 1 when d_in[i] is a square and d_out[i] then holds the root the decoders would use (either sign), else 0 with d_out[i] zero.
 * Another field returns cudaErrorInvalidValue.  One launch, one thread per element, no synchronisation. */
SNARKVM_API int snarkvm_b200_test_sqrt_device(int field, void* d_out, int32_t* d_ok, const void* d_in, size_t n, void* stream);

/* Deterministic synthetic bases P_i = h(seed, i) * G written in the reference affine layout. */
/* ---- G2 (points over Fq2) ----------------------------------------------------------------------------------------------
 * VariableBase::msm for Affine<G2> — the type the reference dispatches to standard::msm
 * (algorithms/src/msm/variable_base/mod.rs:44-47, standard.rs:79-118).  Point layout: x.c0 x.c1 y.c0 y.c1 (4 × 48 B Montgomery
 * Fq), infinity flag, padding: stride ≥ 200 (curves/src/templates/short_weierstrass_jacobian/affine.rs:41-46 over Fq2);
 * scalars: canonical 32-byte integers.  Result: 288 bytes, Projective<G2> X Y Z over Fq2, normalised (Z = 1, or (0, 1, 0)). */
SNARKVM_API snarkvm_error_t snarkvm_b200_msm_g2(void* out288, const void* points, size_t npoints, const void* scalars, size_t ffi_affine_sz);
SNARKVM_API int snarkvm_b200_msm_g2_device(void* out288, const void* d_points, size_t npoints, const void* d_scalars, size_t stride, void* stream);
/* test / bench input: P_i = h(seed, i)·G2 with the multipliers of snarkvm_b200_generate_bases_device */
SNARKVM_API int snarkvm_b200_generate_bases_g2_device(void* d_points, size_t npoints, size_t stride, uint64_t seed, void* stream);

SNARKVM_API int snarkvm_b200_generate_bases_device(void* d_points, size_t npoints, size_t stride, uint64_t seed, void* stream);
/* P_i = s_i * G for npoints canonical scalars (32 B each) in HBM, written in the reference Affine layout: s_i = beta^i gives the
 * powers_of_beta_g of a universal setup with a KNOWN trapdoor (kzg10/data_structures.rs UniversalParams) for tests and benches. */
SNARKVM_API int snarkvm_b200_generator_mul_device(void* d_points, size_t stride, const void* d_scalars, size_t npoints, void* stream);

/* BLS12-377 pairing (curves/src/templates/bls12/{bls12.rs, g2.rs}).
 * A prepared G2 point (G2Prepared::from_affine) is SNARKVM_B200_G2_PREPARED_BYTES bytes: 69 coefficient triples of three Fq2
 * (c0.c0 c0.c1 c1.c0 … c2.c1, Montgomery: 288 B per triple), then its infinity flag as a u32 and 28 zero bytes.  The point at
 * infinity has no coefficients (zeros) and contributes nothing to a Miller loop.
 * A GT value is the reference's Fp12 image: twelve Montgomery Fq in the order c0.c0.c0, c0.c0.c1, c0.c1.c0, … c1.c2.c1, 576 B. */
#define SNARKVM_B200_G2_PREPARED_BYTES 19904
#define SNARKVM_B200_GT_BYTES 576
/* Prepares npoints G2 Affine images (x.c0 x.c1 y.c0 y.c1 infinity, stride ≥ 200, a multiple of 8, as snarkvm_b200_msm_g2_device
 * takes them) into d_prepared (npoints × SNARKVM_B200_G2_PREPARED_BYTES, 16-byte aligned).  One launch, one synchronisation.  A
 * coordinate whose image is not below q returns cudaErrorInvalidValue and *bad_point (HOST, may be NULL) receives the lowest such
 * point's index (-1 otherwise); d_prepared is then unspecified. */
SNARKVM_API int snarkvm_b200_g2_prepare_device(void* d_prepared, const void* d_points, size_t npoints, size_t stride, int64_t* bad_point,
                                               void* stream);
/* Products of pairings over a table of checks (PairingEngine::product_of_pairings per check).  Pair i is (G1 Affine image at
 * d_g1 + i·g1_stride, prepared G2 number d_g2_index[i] of d_prepared); check c owns pairs [d_check_start[c], d_check_start[c + 1]),
 * so d_check_start (device, nchecks + 1 u32) starts at 0, never decreases and ends at npairs.  Writes each check's GT value
 * (d_gt: nchecks × 576 B, 16-byte aligned) and d_is_one[c] = 1 when it is one (device u32).  d_miller (may be NULL) receives each
 * pair's Miller loop value (npairs × 576 B); the pairs of a check are multiplied and the final exponentiation runs once per check.
 * A pair at infinity on either side contributes one; a check with no other pairs gives one.  One synchronisation per call.  A
 * coordinate not below q, a G2 index ≥ nprepared or a malformed d_check_start returns cudaErrorInvalidValue, and *bad_check (HOST,
 * may be NULL) receives the lowest check concerned (-1 otherwise); the outputs are then unspecified. */
SNARKVM_API int snarkvm_b200_pairing_products_device(void* d_gt, uint32_t* d_is_one, void* d_miller, const void* d_g1, size_t g1_stride,
                                                     const uint32_t* d_g2_index, size_t npairs, const void* d_prepared, size_t nprepared,
                                                     const uint32_t* d_check_start, size_t nchecks, int64_t* bad_check, void* stream);

/* Poseidon duplex sponge transcripts (PoseidonSponge<F, 2, 1>, algorithms/src/crypto_hash/poseidon.rs; snarkVM's Fiat–Shamir
 * sponge is field = FQ), one thread per transcript.  d_params: the sponge's 39 × 3 round keys then its 3 × 3 MDS matrix, Montgomery
 * F (snarkvm_b200/poseidon.py builds them).  Transcript t runs operations [d_op_start[t], d_op_start[t + 1]) of d_ops, each three
 * u32 (kind, n, offset), on a sponge of its own:
 *   ABSORB                    absorb_native_field_elements of d_in[offset … offset + n)  (Montgomery F, each below p)
 *   SQUEEZE                   squeeze_native_field_elements(n) → d_out[offset …]         (Montgomery F)
 *   SQUEEZE_NONNATIVE         squeeze_nonnative_field_elements::<Fr>(n) → d_out_fr[offset …]  (Montgomery Fr, 32 B)
 *   SQUEEZE_SHORT_NONNATIVE   squeeze_short_nonnative_field_elements::<Fr>(n) (168-bit) → d_out_fr[offset …]
 * Elements are 32 B (Fr) or 48 B (Fq); d_params, d_in, d_out and d_out_fr are 16-byte aligned.  n = 0 is no operation.  Two launches
 * and one synchronisation per call.  An unknown kind, a range outside nin / nout / nout_fr, an absorbed element not below p or a
 * d_op_start entry out of order or beyond nops returns cudaErrorInvalidValue, *bad_transcript (HOST, may be NULL) receives the
 * lowest transcript concerned (-1 otherwise), and no output is written. */
enum {
    SNARKVM_B200_POSEIDON_ABSORB = 0, SNARKVM_B200_POSEIDON_SQUEEZE = 1, SNARKVM_B200_POSEIDON_SQUEEZE_NONNATIVE = 2,
    SNARKVM_B200_POSEIDON_SQUEEZE_SHORT_NONNATIVE = 3
};
SNARKVM_API int snarkvm_b200_poseidon_transcripts_device(int field, const void* d_params, const uint32_t* d_ops, const uint32_t* d_op_start,
                                                         size_t ntranscripts, size_t nops, const void* d_in, size_t nin, void* d_out,
                                                         size_t nout, void* d_out_fr, size_t nout_fr, int64_t* bad_transcript, void* stream);

/* The same transcripts resumed from, and saved back to, d_state: one record per transcript, 16-byte aligned, of 3·(F's words) + 4
 * u32 (Fr 28, Fq 40): the three state elements (Montgomery F, the capacity element first), then DuplexSpongeMode (0 absorbing,
 * 1 squeezing), then next_absorb_index / next_squeeze_index (0 … 2), then two words written as zero.  A fresh sponge is all zeros.
 * The record is read before the first operation and written after the last.  Besides the errors above, a record with an element
 * not below p, an unknown mode or an index above 2 is reported in the same way (lowest transcript concerned), and then neither the
 * outputs nor any record is written.  d_state may be NULL only when ntranscripts = 0. */
SNARKVM_API int snarkvm_b200_poseidon_transcripts_resume_device(int field, const void* d_params, const uint32_t* d_ops,
                                                                const uint32_t* d_op_start, size_t ntranscripts, size_t nops,
                                                                const void* d_in, size_t nin, void* d_out, size_t nout, void* d_out_fr,
                                                                size_t nout_fr, void* d_state, int64_t* bad_transcript, void* stream);

/* Validation of G1 points taken from outside (Affine::check of the reference: curves/src/bls12_377/g1.rs:98-106).  d_points holds n
 * Affine<G1> images (x, y Montgomery Fq, infinity flag; stride ≥ 104, a multiple of 8, 8-byte aligned); d_status[i] (device int32)
 * receives point i's status: VALID (the point at infinity included), NOT_CANONICAL (a coordinate image not below q), NOT_ON_CURVE
 * (y² ≠ x³ + 1) or NOT_IN_SUBGROUP ([x²]·φ(P) + P ≠ O, x the BLS parameter, φ(x, y) = (PHI·x, y)), the first test that fails.  One
 * launch, one thread per point, no synchronisation. */
enum {
    SNARKVM_B200_G1_VALID = 0, SNARKVM_B200_G1_NOT_CANONICAL = 1, SNARKVM_B200_G1_NOT_ON_CURVE = 2, SNARKVM_B200_G1_NOT_IN_SUBGROUP = 3,
    SNARKVM_B200_G1_BAD_FLAGS = 4
};
SNARKVM_API int snarkvm_b200_g1_validate_device(int32_t* d_status, const void* d_points, size_t n, size_t stride, void* stream);

/* The byte forms of a G1 point: `form` of the two entry points below. */
enum { SNARKVM_B200_G1_FORM_UNCOMPRESSED = 0, SNARKVM_B200_G1_FORM_COMPRESSED = 1, SNARKVM_B200_G1_FORM_TO_BYTES = 2 };

/* G1 points from their byte forms (CanonicalDeserialize of Affine<G1>: curves/src/templates/macros.rs:118-144, SWFlags of
 * utilities/src/serialize/flags.rs; FromBytes of Affine, short_weierstrass_jacobian/affine.rs:302-313).  d_bytes holds n points
 * of 48 bytes (FORM_COMPRESSED: x little-endian, bit 7 of the last byte PositiveY, bit 6 Infinity), 96 bytes (FORM_UNCOMPRESSED: x,
 * then y with the flags; x carries none) or 97 bytes (FORM_TO_BYTES: canonical x, canonical y, an infinity byte), no alignment
 * needed.  d_points (8-byte aligned, 104-byte stride) receives each point's Affine<G1> image and d_status[i] (device int32, 4-byte
 * aligned) its status: BAD_FLAGS (both flag bits set, or bit 7 of an uncompressed x; ToBytes: an infinity byte other than 0 or 1,
 * or y = 1 with the infinity byte disagreeing with x = 0), NOT_CANONICAL (a coordinate not below q after the flags are masked),
 * NOT_ON_CURVE (compressed: x³ + 1 has no square root in Fq), the first that applies; otherwise VALID, and with `validate` the
 * status of Affine::check as snarkvm_b200_g1_validate_device reports it.  A compressed or uncompressed infinity decodes to
 * Affine::zero() (0, 1, infinity) whatever the coordinates below q were; a ToBytes point keeps the x and y it was read with, so it
 * writes back to the same bytes.  A compressed point's y is the root of x³ + 1 that is the larger of y, −y (canonical integers)
 * when PositiveY is set, the smaller otherwise.  An uncompressed or ToBytes point is not tested against the curve unless
 * `validate`.  Bytes that decode to no point leave an all-zero image.  Another form returns cudaErrorInvalidValue.  One launch,
 * one thread per point, no synchronisation. */
SNARKVM_API int snarkvm_b200_g1_deserialize_device(void* d_points, int32_t* d_status, const void* d_bytes, size_t n, int form,
                                                   int validate, void* stream);
/* G1 points to their byte forms (CanonicalSerialize of Affine<G1>, macros.rs:67-97; ToBytes of Affine, affine.rs:293-300).  For
 * FORM_COMPRESSED and FORM_UNCOMPRESSED, d_points holds n normalised projective images (X, Y, Z Montgomery Fq, 144 bytes each,
 * 8-byte aligned; Z = one, or Z = 0 for infinity); d_bytes receives 48 bytes per point (compressed: canonical x, PositiveY iff
 * y > −y; infinity: x = 0 with the Infinity bit) or 96 (uncompressed: canonical x and y, no sign flag; infinity: x = 0, y = 1 with
 * the Infinity bit).  For FORM_TO_BYTES, d_points holds n Affine<G1> images (104-byte stride, 8-byte aligned) and d_bytes receives
 * 97 bytes per point: canonical x and y as the image holds them, then the infinity byte.  One launch, one thread per point, no
 * synchronisation. */
SNARKVM_API int snarkvm_b200_g1_serialize_device(void* d_bytes, const void* d_points, size_t n, int form, void* stream);

/* G2 points taken from outside.  These three entry points report the SNARKVM_B200_G1_* status values above: the values are shared
 * by both groups, and there is no G2 enum.
 *
 * Validation (Valid for Affine<G2> of the reference: is_on_curve and [r]·P = O, curves/src/bls12_377/g2.rs:120-124).  d_points
 * holds n Affine<G2> images (x.c0, x.c1, y.c0, y.c1 Montgomery Fq, infinity flag; stride ≥ 200, a multiple of 8, 8-byte aligned);
 * d_status[i] (device int32) receives point i's status: VALID (the point at infinity included), NOT_CANONICAL (a coordinate image
 * not below q), NOT_ON_CURVE (y² ≠ x³ + B', B' = (0, −1/5)) or NOT_IN_SUBGROUP ([r]·P ≠ O, r the order of G1 and G2), the first
 * test that fails.  One launch, one thread per point, no synchronisation. */
SNARKVM_API int snarkvm_b200_g2_validate_device(int32_t* d_status, const void* d_points, size_t n, size_t stride, void* stream);
/* G2 points from their byte forms (CanonicalDeserialize of Affine<G2>: curves/src/templates/macros.rs:118-144, Fp2 of
 * fields/src/fp2.rs:450-457).  d_bytes holds n points of 96 bytes (compressed != 0: x.c0, x.c1, 48 bytes little-endian each, bit 7
 * of the last byte PositiveY, bit 6 Infinity) or 192 bytes (compressed = 0: x.c0, x.c1, y.c0, y.c1, the flags on y.c1), no
 * alignment needed.  d_points (8-byte aligned, 200-byte stride) receives each point's Affine<G2> image and d_status[i] (device
 * int32, 4-byte aligned) its status.  The coordinates are read in order: bit 7 of the last byte of a coordinate other than the
 * last gives BAD_FLAGS (EmptyFlags), as do both flag bits of the last one; then a value not below q (flags masked) gives
 * NOT_CANONICAL.  A compressed x whose x³ + B' has no square root in Fq2 gives NOT_ON_CURVE.  Otherwise VALID, and with `validate`
 * the status of Affine::check as snarkvm_b200_g2_validate_device reports it.  An infinity decodes to Affine::zero() (0, 1,
 * infinity) whatever the coordinates below q were.  A compressed point's y is the root of x³ + B' that is the larger of y, −y in
 * the reference's order on Fp2 (c1 compared first, then c0, as canonical integers) when PositiveY is set, the smaller otherwise.
 * An uncompressed point is not tested against the curve unless `validate`.  Bytes that decode to no point leave an all-zero image.
 * One launch, one thread per point, no synchronisation. */
SNARKVM_API int snarkvm_b200_g2_deserialize_device(void* d_points, int32_t* d_status, const void* d_bytes, size_t n, int compressed,
                                                   int validate, void* stream);
/* G2 points to their byte forms (CanonicalSerialize of Affine<G2>, macros.rs:67-97).  d_points holds n Affine<G2> images
 * (200-byte stride, 8-byte aligned); d_bytes receives 96 bytes per point (compressed != 0: canonical x, PositiveY iff y > −y in the
 * order above; infinity: x = 0 with the Infinity bit) or 192 (uncompressed: canonical x and y, no sign flag; infinity: x = 0, y = 1
 * with the Infinity bit).  One launch, one thread per point, no synchronisation. */
SNARKVM_API int snarkvm_b200_g2_serialize_device(void* d_bytes, const void* d_points, size_t n, int compressed, void* stream);

/* One run of Fr records in a proving key's bytes (CanonicalSerialize of Circuit: snark/varuna/ahp/indexer/circuit.rs:158-237).
 * stride 32: `count` canonical Fr at d_blob + offset, 32 bytes apart (an Evaluations vector).  stride 40: matrix entries, each a
 * canonical Fr and a u64 column; with d_row_ptr (int32 [nrows + 1], device) `offset` is the matrix section (its u64 row count) and
 * entry e of row i sits at offset + 16 + 8·i + 40·e.  d_out (16-byte aligned) receives count Montgomery Fr; for stride 40, d_cols
 * (4-byte aligned) receives the columns as int32, each of which must be below num_cols (≤ 2^31). */
typedef struct {
    uint64_t offset, count;
    uint32_t stride, reserved;
    const void* d_row_ptr;
    uint64_t nrows;
    void* d_out;
    void* d_cols;
    uint64_t num_cols;
} snarkvm_b200_fr_records_segment_t;
enum { SNARKVM_B200_FR_RECORD_NOT_CANONICAL = 1, SNARKVM_B200_FR_RECORD_BAD_COLUMN = 2 };
/* Every record of every segment (HOST table) decoded from d_blob (blob_bytes bytes in HBM, no alignment) in one launch and one
 * synchronisation.  bad_record (HOST, count entries) receives per segment UINT64_MAX, or (e << 2) | reason for its first bad
 * record e: NOT_CANONICAL (an Fr not below r; checked first) or BAD_COLUMN (a column ≥ num_cols).  The outputs of a bad record are
 * unspecified.  A stride other than 32 or 40, a segment whose bytes leave the blob or a misaligned output returns
 * cudaErrorInvalidValue before any launch. */
SNARKVM_API int snarkvm_b200_fr_records_decode_device(const void* d_blob, size_t blob_bytes, const snarkvm_b200_fr_records_segment_t* segs,
                                                      size_t count, uint64_t* bad_record, void* stream);
/* A HOST function: the row headers of one matrix section (CanonicalSerialize of Vec<Vec<(Fr, u64)>>), after its u64 row count.
 * `rows` holds `bytes` bytes (HOST); row i is a u64 length and that many 40-byte entries.  row_ptr (HOST, nrows + 1 int32)
 * receives the CSR row starts.  A row whose header or entries overrun `bytes`, or whose length carries the count past nnz, returns
 * cudaErrorInvalidValue with *bad_row = i; a total below nnz, with *bad_row = nrows; nnz ≥ 2^31, with *bad_row = −1. */
SNARKVM_API int snarkvm_b200_matrix_row_walk(const void* rows, size_t bytes, uint64_t nrows, uint64_t nnz, int32_t* row_ptr,
                                             int64_t* bad_row);

#ifdef __cplusplus
}
#endif
#endif /* SNARKVM_B200_H */
