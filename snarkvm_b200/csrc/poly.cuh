// Device-resident polynomial / field-vector helpers (see poly.cu for the reference map).
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/snarkvm_b200.h"   // the segment tables of the batched entry points

namespace b200 {

// v_i ← coeff · v_i^{-1} in place on n Montgomery Fr elements in HBM; zeros stay zero.  coeff: 32 B Montgomery, HOST memory.
int fr_batch_inversion_and_mul_device(void* d_v, size_t n, const void* coeff_mont_host, cudaStream_t stream);

// p (m coefficients) = q·(x^n − 1) + r:  d_q gets max(m − n, 0) coefficients, d_r gets min(m, n).
int poly_divide_by_vanishing_device(void* d_q, void* d_r, const void* d_p, size_t m, size_t n, cudaStream_t stream);

// quotient of p (m coefficients) / (x − point): d_q gets m − 1 coefficients (the KZG witness polynomial, kzg10/mod.rs:220-241)
int poly_divide_by_linear_device(void* d_q, const void* d_p, size_t m, const void* point_mont_host, cudaStream_t stream);

// out = Σ c_i·point^i (Montgomery in and out; out and point are 32-byte HOST buffers; synchronises the stream)
int poly_evaluate_device(void* out_mont_host, const void* d_coeffs, size_t m, const void* point_mont_host, cudaStream_t stream);

// out[r] = Σ_e vals[e]·x[cols[e]] over e ∈ [row_ptr[r], row_ptr[r+1]) — CSR sparse matrix × vector over Fr (Montgomery);
// row_ptr: nrows + 1 u32, cols: u32.  A column ≥ nvars returns cudaErrorInvalidValue.  Synchronises the stream.
int sparse_matvec_device(void* d_out, const void* d_row_ptr, const void* d_cols, const void* d_vals, size_t nrows, const void* d_x,
                         size_t nvars, cudaStream_t stream);

// elementwise on n Montgomery Fr in HBM: op 0 = a + b, 1 = a − b, 2 = a·b; the scalar form takes a 32-byte HOST scalar
int fr_vec_op_device(void* d_out, const void* d_a, const void* d_b, size_t n, int op, cudaStream_t stream);
int fr_vec_scalar_op_device(void* d_out, const void* d_a, const void* scalar_mont_host, size_t n, int op, cudaStream_t stream);
// out[i] = ω_n^i, i < n = 2^lg (EvaluationDomain::elements, fft/domain.rs:307-309)
int domain_elements_device(void* d_out, uint32_t lg, cudaStream_t stream);

// Varuna indexer over a CSR matrix (row_ptr nrows + 1 u32, cols nnz u32 < nvars, vals Montgomery Fr); input_size = |I| (a power of
// two), the domains are R = 2^lg_constraint ≥ nrows, C = 2^lg_variable > |I| with C ≥ nvars, K = 2^lg_non_zero ≥ nnz.  A column
// ≥ nvars or a row_ptr not running from 0 to nnz returns cudaErrorInvalidValue.  Both synchronise the stream.
// matrix_evals (ahp/matrices.rs:138-195): row / col / row_col_val evaluations on K, 2^lg_non_zero Montgomery Fr each.
int varuna_matrix_evals_device(void* d_row, void* d_col, void* d_row_col_val, const void* d_row_ptr, size_t nrows, const void* d_cols,
                               const void* d_vals, size_t nnz, size_t nvars, size_t input_size, uint32_t lg_constraint,
                               uint32_t lg_variable, uint32_t lg_non_zero, cudaStream_t stream);
// transpose (ahp/matrices.rs:249-270) as CSR over the reindexed variable domain: t_row_ptr 2^lg_variable + 1 u32, t_cols nnz u32
// (row indices of the input), t_vals nnz Montgomery Fr; the order of the entries inside a transposed row is unspecified.
int csr_transpose_device(void* d_t_row_ptr, void* d_t_cols, void* d_t_vals, const void* d_row_ptr, size_t nrows, const void* d_cols,
                         const void* d_vals, size_t nnz, size_t nvars, size_t input_size, uint32_t lg_variable, cudaStream_t stream);

// The circuit id's byte stream of a CSR matrix (Circuit::hash, ahp/indexer/circuit.rs:109-121): serialize_uncompressed of
// Vec<Vec<(Fr, usize)>> — [u64 nrows], per row [u64 len][len × (32 B canonical value, u64 column)] — into out_bytes = 8 + 8·nrows +
// 40·nnz bytes of HBM (8-byte aligned).  A row_ptr not non-decreasing from 0 to nnz returns cudaErrorInvalidValue.  Synchronises.
int csr_serialize_device(void* d_out, size_t out_bytes, const void* d_row_ptr, size_t nrows, const void* d_cols, const void* d_vals, size_t nnz,
                         cudaStream_t stream);
// out (n Montgomery Fr) = Σ_j c_j·p_j for nterms ≤ 12 polynomials: d_polys / lens / coeffs are HOST arrays (device pointers,
// lengths ≤ n, 32-byte Montgomery coefficients); coefficients past a polynomial's length count as zero
int fr_lincomb_device(void* d_out, size_t n, const void* const* d_polys, const size_t* lens, const void* coeffs_mont_host, uint32_t nterms,
                      cudaStream_t stream);
// MatrixEvals::evaluate (ahp/matrices.rs:114-126): out (4 × 32 B Montgomery, HOST) = Σ l·row, Σ l·col, Σ l·row·col, Σ l·row_col_val
// over n elements; synchronises the stream
int matrix_evals_dot_device(void* out_mont_host, const void* d_row, const void* d_col, const void* d_row_col_val, const void* d_lagrange,
                            size_t n, cudaStream_t stream);

// The segmented forms (one launch per job for many matrices; see include/snarkvm_b200.h).  The one-matrix entry points above are
// one-segment calls of these.
int varuna_matrix_evals_batch_device(const snarkvm_b200_csr_segment_t* segs, size_t count, int64_t* bad_segment, cudaStream_t stream);
int csr_serialize_batch_device(const snarkvm_b200_csr_segment_t* segs, size_t count, int64_t* bad_segment, cudaStream_t stream);
int fr_lincomb_batch_device(const snarkvm_b200_lincomb_segment_t* segs, size_t count, cudaStream_t stream);
int matrix_evals_at_points_device(void* out_mont_host, const snarkvm_b200_evals_segment_t* segs, size_t count, cudaStream_t stream);

// The batched Varuna prover's pieces (include/snarkvm_b200.h).  fr_lincomb_batch_device / fr_lincomb_device are calls of
// fr_lincomb_terms_device, sparse_matvec_device a one-segment call of sparse_matvec_batch_device.
int fr_lincomb_terms_device(const snarkvm_b200_lincomb_output_t* outs, size_t nouts, const snarkvm_b200_lincomb_term_t* terms, size_t nterms,
                            cudaStream_t stream);
int sparse_matvec_batch_device(const snarkvm_b200_spmv_segment_t* segs, size_t count, int64_t* bad_segment, cudaStream_t stream);
int polymul_batch_device(const snarkvm_b200_polymul_job_t* jobs, size_t count, cudaStream_t stream);
int varuna_round4_evals_device(const snarkvm_b200_round4_segment_t* segs, size_t count, const void* alpha_mont, const void* beta_mont,
                               cudaStream_t stream);
// Many proofs per call: round 4 with per-segment challenges, and the segmented forms of poly_evaluate_device and
// poly_divide_by_linear_device (both of which are one-segment calls of these).
int varuna_round4_evals_batch_device(const snarkvm_b200_round4_batch_segment_t* segs, size_t count, cudaStream_t stream);
int poly_evaluate_batch_device(void* out_mont_host, const snarkvm_b200_poly_eval_segment_t* segs, size_t count, cudaStream_t stream);
int poly_divide_by_linear_batch_device(const snarkvm_b200_poly_divide_segment_t* segs, size_t count, cudaStream_t stream);

// Group FFT over G1 (DomainCoeff = G1Projective, fft/domain.rs:169-221 generic path): n = 2^lg affine points in, affine points
// out (natural order both sides).  direction 1 = inverse (includes n^{-1}): UniversalParams::lagrange_basis
// (polycommit/kzg10/data_structures.rs:68-72).
int g1_ntt_device(void* d_out, size_t out_stride, const void* d_in, size_t in_stride, uint32_t lg, int direction, cudaStream_t stream);

// ntt.cu: the cached table ω_N^j (j < N/2, Montgomery), N = 2^lgN ≥ 2^lg
int ntt_get_twiddles(int lg, const void** tw, int* lgN);

}  // namespace b200
