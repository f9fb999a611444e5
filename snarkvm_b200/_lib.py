"""ctypes binding of snarkvm_b200/libsnarkvm_b200.so (the C ABI in include/snarkvm_b200.h).

The library is the product: there is NO CPU fallback.  If the shared object is missing or a
symbol is absent, importing fails loudly; if a call returns a non-zero cudaError_t, CudaError
is raised (the Rust reference would fall back to its CPU path at this point —
algorithms/src/msm/variable_base/mod.rs:39-43 — this package never does).
"""
from __future__ import annotations

import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SNARKVM_B200_LIB") or os.path.join(_HERE, "libsnarkvm_b200.so")   # override: A/B builds

# every symbol include/snarkvm_b200.h declares
SYMBOLS = (
    "snarkvm_ntt", "snarkvm_polymul", "snarkvm_msm",
    "snarkvm_b200_version", "snarkvm_b200_launch_count", "snarkvm_b200_ntt_device",
    "snarkvm_b200_polymul_device", "snarkvm_b200_msm_plan", "snarkvm_b200_msm_device",
    "snarkvm_b200_msm_window_sums_device", "snarkvm_b200_xyzz_sum_ranks_device", "snarkvm_b200_msm_finish",
    "snarkvm_b200_kzg_commit_device", "snarkvm_b200_fr_from_mont_device", "snarkvm_b200_fr_to_mont_device",
    "snarkvm_b200_srs_decode_device", "snarkvm_b200_register_bases", "snarkvm_b200_unregister_bases", "snarkvm_b200_profile_enable", "snarkvm_b200_profile_collect", "snarkvm_b200_generate_bases_device",
    "snarkvm_b200_msm_precompute_device", "snarkvm_b200_msm_precomputed_free", "snarkvm_b200_msm_precomputed_info",
    "snarkvm_b200_msm_precomputed_device", "snarkvm_b200_kzg_commit_precomputed_device",
    "snarkvm_b200_kzg_commit_hiding_device", "snarkvm_b200_kzg_commit_batch_device", "snarkvm_b200_g1_ntt_device",
    "snarkvm_b200_fr_batch_inversion_and_mul_device", "snarkvm_b200_poly_divide_by_vanishing_device", "snarkvm_b200_poly_evaluate_device",
    "snarkvm_b200_poly_divide_by_linear_device", "snarkvm_b200_sparse_matvec_device",
    "snarkvm_b200_fr_vec_op_device", "snarkvm_b200_fr_vec_scalar_op_device", "snarkvm_b200_domain_elements_device",
    "snarkvm_b200_register_bases_precomputed",
    "snarkvm_b200_msm_batch_device", "snarkvm_b200_msm_window_sums_plan_device", "snarkvm_b200_kzg_commit_batch_hiding_device",
    "snarkvm_b200_kzg_commit_batch_precomputed_device", "snarkvm_b200_msm_scratch_stats", "snarkvm_b200_msm_set_scratch_limit", "snarkvm_b200_msm_window_sums_host", "snarkvm_b200_selftest_coop", "snarkvm_b200_msm_plan_levels", "snarkvm_b200_msm_g2", "snarkvm_b200_msm_g2_device", "snarkvm_b200_generate_bases_g2_device",
    "snarkvm_b200_sonic_commit_batch_device", "snarkvm_b200_generator_mul_device", "snarkvm_b200_selftest_host_copy",
    "snarkvm_b200_test_field_op_device", "snarkvm_b200_test_curve_op_device", "snarkvm_b200_test_field_op_host",
    "snarkvm_b200_varuna_matrix_evals_device", "snarkvm_b200_csr_transpose_device",
    "snarkvm_b200_csr_serialize_device", "snarkvm_b200_fr_lincomb_device", "snarkvm_b200_matrix_evals_dot_device",
    "snarkvm_b200_ntt_batch_device", "snarkvm_b200_varuna_matrix_evals_batch_device", "snarkvm_b200_csr_serialize_batch_device",
    "snarkvm_b200_fr_lincomb_batch_device", "snarkvm_b200_matrix_evals_at_points_device",
    "snarkvm_b200_fr_lincomb_terms_device", "snarkvm_b200_sparse_matvec_batch_device", "snarkvm_b200_polymul_batch_device",
    "snarkvm_b200_varuna_round4_evals_device", "snarkvm_b200_g2_prepare_device", "snarkvm_b200_pairing_products_device",
    "snarkvm_b200_test_tower_op_device", "snarkvm_b200_poseidon_transcripts_device",
    "snarkvm_b200_poseidon_transcripts_resume_device", "snarkvm_b200_g1_validate_device",
    "snarkvm_b200_g1_deserialize_device", "snarkvm_b200_g1_serialize_device", "snarkvm_b200_fr_records_decode_device",
    "snarkvm_b200_matrix_row_walk", "snarkvm_b200_varuna_round4_evals_batch_device", "snarkvm_b200_poly_evaluate_batch_device",
    "snarkvm_b200_poly_divide_by_linear_batch_device", "snarkvm_b200_g2_validate_device", "snarkvm_b200_g2_deserialize_device",
    "snarkvm_b200_g2_serialize_device", "snarkvm_b200_test_sqrt_device",
)


class CsrSegment(ctypes.Structure):
    """snarkvm_b200_csr_segment_t"""
    _fields_ = [("d_row_ptr", ctypes.c_void_p), ("d_cols", ctypes.c_void_p), ("d_vals", ctypes.c_void_p),
                ("nrows", ctypes.c_uint64), ("nnz", ctypes.c_uint64), ("nvars", ctypes.c_uint64), ("input_size", ctypes.c_uint64),
                ("lg_constraint", ctypes.c_uint32), ("lg_variable", ctypes.c_uint32), ("lg_non_zero", ctypes.c_uint32),
                ("reserved", ctypes.c_uint32), ("d_out", ctypes.c_void_p * 3)]


class LincombSegment(ctypes.Structure):
    """snarkvm_b200_lincomb_segment_t"""
    _fields_ = [("d_out", ctypes.c_void_p), ("n", ctypes.c_uint64), ("d_polys", ctypes.c_void_p * 12), ("lens", ctypes.c_uint64 * 12),
                ("coeffs_mont", (ctypes.c_uint8 * 32) * 12), ("nterms", ctypes.c_uint32), ("reserved", ctypes.c_uint32)]


class EvalsSegment(ctypes.Structure):
    """snarkvm_b200_evals_segment_t"""
    _fields_ = [("d_row", ctypes.c_void_p), ("d_col", ctypes.c_void_p), ("d_row_col_val", ctypes.c_void_p), ("n", ctypes.c_uint64),
                ("point_mont", ctypes.c_uint8 * 32)]


class LincombTerm(ctypes.Structure):
    """snarkvm_b200_lincomb_term_t"""
    _fields_ = [("d_poly", ctypes.c_void_p), ("len", ctypes.c_uint64), ("offset", ctypes.c_uint64), ("period", ctypes.c_uint64),
                ("reps", ctypes.c_uint64), ("coeff_mont", ctypes.c_uint8 * 32)]


class LincombOutput(ctypes.Structure):
    """snarkvm_b200_lincomb_output_t"""
    _fields_ = [("d_out", ctypes.c_void_p), ("n", ctypes.c_uint64), ("first_term", ctypes.c_uint64), ("nterms", ctypes.c_uint64)]


class SpmvSegment(ctypes.Structure):
    """snarkvm_b200_spmv_segment_t"""
    _fields_ = [("d_row_ptr", ctypes.c_void_p), ("d_cols", ctypes.c_void_p), ("d_vals", ctypes.c_void_p), ("nrows", ctypes.c_uint64),
                ("nnz", ctypes.c_uint64), ("d_x", ctypes.c_void_p), ("nvars", ctypes.c_uint64), ("d_out", ctypes.c_void_p)]


class PolymulJob(ctypes.Structure):
    """snarkvm_b200_polymul_job_t"""
    _fields_ = [("d_out", ctypes.c_void_p), ("d_a", ctypes.c_void_p), ("d_b", ctypes.c_void_p), ("len_a", ctypes.c_uint64),
                ("len_b", ctypes.c_uint64), ("lg", ctypes.c_uint32), ("reserved", ctypes.c_uint32)]


class Round4Segment(ctypes.Structure):
    """snarkvm_b200_round4_segment_t"""
    _fields_ = [("d_row", ctypes.c_void_p), ("d_col", ctypes.c_void_p), ("d_row_col_val", ctypes.c_void_p), ("n", ctypes.c_uint64),
                ("v_rc_mont", ctypes.c_uint8 * 32), ("rc_mont", ctypes.c_uint8 * 32), ("f_scale_mont", ctypes.c_uint8 * 32),
                ("d_a", ctypes.c_void_p), ("d_b", ctypes.c_void_p), ("d_f", ctypes.c_void_p)]


class Round4BatchSegment(ctypes.Structure):
    """snarkvm_b200_round4_batch_segment_t"""
    _fields_ = Round4Segment._fields_ + [("alpha_mont", ctypes.c_uint8 * 32), ("beta_mont", ctypes.c_uint8 * 32)]


class PolyEvalSegment(ctypes.Structure):
    """snarkvm_b200_poly_eval_segment_t"""
    _fields_ = [("d_coeffs", ctypes.c_void_p), ("m", ctypes.c_uint64), ("point_mont", ctypes.c_uint8 * 32)]


class PolyDivideSegment(ctypes.Structure):
    """snarkvm_b200_poly_divide_segment_t"""
    _fields_ = [("d_q", ctypes.c_void_p), ("d_p", ctypes.c_void_p), ("m", ctypes.c_uint64), ("point_mont", ctypes.c_uint8 * 32)]


class FrRecordsSegment(ctypes.Structure):
    """snarkvm_b200_fr_records_segment_t"""
    _fields_ = [("offset", ctypes.c_uint64), ("count", ctypes.c_uint64), ("stride", ctypes.c_uint32), ("reserved", ctypes.c_uint32),
                ("d_row_ptr", ctypes.c_void_p), ("nrows", ctypes.c_uint64), ("d_out", ctypes.c_void_p), ("d_cols", ctypes.c_void_p),
                ("num_cols", ctypes.c_uint64)]


class CudaError(RuntimeError):
    """Mirror of `cuda::Error` (algorithms/cuda/src/lib.rs:19): .code is the cudaError_t."""

    def __init__(self, code: int, message: str = ""):
        super().__init__(f"cuda error {code}: {message}")
        self.code = code
        self.message = message


class _RustError(ctypes.Structure):
    _fields_ = [("code", ctypes.c_int), ("message", ctypes.c_void_p)]


_lib = None
_libc = None


def lib():
    global _lib, _libc
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing — build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(snarkvm_b200 has no CPU fallback)")
    L = ctypes.CDLL(LIB_PATH)
    for s in SYMBOLS:
        if not hasattr(L, s):
            raise ImportError(f"{LIB_PATH} does not export {s}")
    vp, sz, u32, i32, u64 = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_uint32, ctypes.c_int, ctypes.c_uint64
    L.snarkvm_ntt.restype = _RustError
    L.snarkvm_ntt.argtypes = [vp, u32, i32, i32, i32]
    L.snarkvm_polymul.restype = _RustError
    L.snarkvm_polymul.argtypes = [vp, sz, vp, vp, sz, vp, vp, u32]
    L.snarkvm_msm.restype = _RustError
    L.snarkvm_msm.argtypes = [vp, vp, sz, vp, sz]
    L.snarkvm_b200_version.restype = ctypes.c_char_p
    L.snarkvm_b200_launch_count.restype = u64
    L.snarkvm_b200_ntt_device.argtypes = [vp, u32, i32, i32, i32, vp, vp]
    L.snarkvm_b200_polymul_device.argtypes = [vp, sz, vp, vp, sz, vp, vp, u32, vp]
    L.snarkvm_b200_msm_plan.argtypes = [sz, ctypes.POINTER(i32), ctypes.POINTER(i32), ctypes.POINTER(u32)]
    L.snarkvm_b200_msm_device.argtypes = [vp, vp, sz, vp, sz, vp]
    L.snarkvm_b200_msm_window_sums_device.argtypes = [vp, vp, sz, vp, sz, vp]
    L.snarkvm_b200_xyzz_sum_ranks_device.argtypes = [vp, vp, i32, i32, vp]
    L.snarkvm_b200_msm_finish.argtypes = [vp, vp, i32, i32]
    L.snarkvm_b200_kzg_commit_device.argtypes = [vp, vp, sz, vp, sz, vp]
    L.snarkvm_b200_fr_from_mont_device.argtypes = [vp, vp, sz, vp]
    L.snarkvm_b200_fr_to_mont_device.argtypes = [vp, vp, sz, vp]
    L.snarkvm_b200_srs_decode_device.argtypes = [vp, sz, vp, sz, vp, vp]
    L.snarkvm_b200_register_bases.argtypes = [vp, sz, sz]
    L.snarkvm_b200_unregister_bases.argtypes = [vp]
    L.snarkvm_b200_register_bases_precomputed.argtypes = [vp, sz, sz]
    L.snarkvm_b200_profile_enable.argtypes = [i32]
    L.snarkvm_b200_profile_collect.argtypes = [i32, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(u64)]
    L.snarkvm_b200_generate_bases_device.argtypes = [vp, sz, sz, u64, vp]
    L.snarkvm_b200_generate_bases_g2_device.argtypes = [vp, sz, sz, u64, vp]
    L.snarkvm_b200_msm_plan_levels.argtypes = [sz]
    L.snarkvm_b200_msm_g2_device.argtypes = [vp, vp, sz, vp, sz, vp]
    L.snarkvm_b200_msm_g2.argtypes = [vp, vp, sz, vp, sz]
    L.snarkvm_b200_msm_precompute_device.argtypes = [ctypes.POINTER(vp), vp, sz, sz, vp]
    L.snarkvm_b200_msm_precomputed_free.argtypes = [vp]
    L.snarkvm_b200_msm_precomputed_info.argtypes = [vp, ctypes.POINTER(sz), ctypes.POINTER(i32), ctypes.POINTER(i32), ctypes.POINTER(sz)]
    L.snarkvm_b200_msm_precomputed_device.argtypes = [vp, vp, vp, sz, vp]
    L.snarkvm_b200_kzg_commit_precomputed_device.argtypes = [vp, vp, vp, sz, vp]
    L.snarkvm_b200_kzg_commit_hiding_device.argtypes = [vp, vp, sz, vp, sz, vp, vp, sz, vp]
    L.snarkvm_b200_kzg_commit_batch_device.argtypes = [vp, vp, sz, vp, vp, sz, vp]
    L.snarkvm_b200_g1_ntt_device.argtypes = [vp, sz, vp, sz, u32, i32, vp]
    L.snarkvm_b200_fr_batch_inversion_and_mul_device.argtypes = [vp, sz, vp, vp]
    L.snarkvm_b200_poly_divide_by_vanishing_device.argtypes = [vp, vp, vp, sz, sz, vp]
    L.snarkvm_b200_poly_evaluate_device.argtypes = [vp, vp, sz, vp, vp]
    L.snarkvm_b200_poly_divide_by_linear_device.argtypes = [vp, vp, sz, vp, vp]
    L.snarkvm_b200_sparse_matvec_device.argtypes = [vp, vp, vp, vp, sz, vp, sz, vp]
    L.snarkvm_b200_fr_vec_op_device.argtypes = [vp, vp, vp, sz, i32, vp]
    L.snarkvm_b200_fr_vec_scalar_op_device.argtypes = [vp, vp, vp, sz, i32, vp]
    L.snarkvm_b200_domain_elements_device.argtypes = [vp, u32, vp]
    L.snarkvm_b200_varuna_matrix_evals_device.argtypes = [vp, vp, vp, vp, sz, vp, vp, sz, sz, sz, u32, u32, u32, vp]
    L.snarkvm_b200_csr_transpose_device.argtypes = [vp, vp, vp, vp, sz, vp, vp, sz, sz, sz, u32, vp]
    L.snarkvm_b200_csr_serialize_device.argtypes = [vp, sz, vp, sz, vp, vp, sz, vp]
    L.snarkvm_b200_fr_lincomb_device.argtypes = [vp, sz, vp, vp, vp, u32, vp]
    L.snarkvm_b200_matrix_evals_dot_device.argtypes = [vp, vp, vp, vp, vp, sz, vp]
    L.snarkvm_b200_ntt_batch_device.argtypes = [vp, vp, sz, i32, i32, vp]
    L.snarkvm_b200_varuna_matrix_evals_batch_device.argtypes = [ctypes.POINTER(CsrSegment), sz, ctypes.POINTER(ctypes.c_int64), vp]
    L.snarkvm_b200_csr_serialize_batch_device.argtypes = [ctypes.POINTER(CsrSegment), sz, ctypes.POINTER(ctypes.c_int64), vp]
    L.snarkvm_b200_fr_lincomb_batch_device.argtypes = [ctypes.POINTER(LincombSegment), sz, vp]
    L.snarkvm_b200_matrix_evals_at_points_device.argtypes = [vp, ctypes.POINTER(EvalsSegment), sz, vp]
    L.snarkvm_b200_fr_lincomb_terms_device.argtypes = [ctypes.POINTER(LincombOutput), sz, ctypes.POINTER(LincombTerm), sz, vp]
    L.snarkvm_b200_sparse_matvec_batch_device.argtypes = [ctypes.POINTER(SpmvSegment), sz, ctypes.POINTER(ctypes.c_int64), vp]
    L.snarkvm_b200_polymul_batch_device.argtypes = [ctypes.POINTER(PolymulJob), sz, vp]
    L.snarkvm_b200_varuna_round4_evals_device.argtypes = [ctypes.POINTER(Round4Segment), sz, vp, vp, vp]
    L.snarkvm_b200_varuna_round4_evals_batch_device.argtypes = [ctypes.POINTER(Round4BatchSegment), sz, vp]
    L.snarkvm_b200_poly_evaluate_batch_device.argtypes = [vp, ctypes.POINTER(PolyEvalSegment), sz, vp]
    L.snarkvm_b200_poly_divide_by_linear_batch_device.argtypes = [ctypes.POINTER(PolyDivideSegment), sz, vp]
    L.snarkvm_b200_g2_prepare_device.argtypes = [vp, vp, sz, sz, ctypes.POINTER(ctypes.c_int64), vp]
    L.snarkvm_b200_pairing_products_device.argtypes = [vp, vp, vp, vp, sz, vp, sz, vp, sz, vp, sz, ctypes.POINTER(ctypes.c_int64), vp]
    L.snarkvm_b200_poseidon_transcripts_device.argtypes = [i32, vp, vp, vp, sz, sz, vp, sz, vp, sz, vp, sz, ctypes.POINTER(ctypes.c_int64), vp]
    L.snarkvm_b200_poseidon_transcripts_resume_device.argtypes = [i32, vp, vp, vp, sz, sz, vp, sz, vp, sz, vp, sz, vp,
                                                                  ctypes.POINTER(ctypes.c_int64), vp]
    L.snarkvm_b200_g1_validate_device.argtypes = [vp, vp, sz, sz, vp]
    L.snarkvm_b200_g1_deserialize_device.argtypes = [vp, vp, vp, sz, i32, i32, vp]
    L.snarkvm_b200_g1_serialize_device.argtypes = [vp, vp, sz, i32, vp]
    L.snarkvm_b200_g2_validate_device.argtypes = [vp, vp, sz, sz, vp]
    L.snarkvm_b200_g2_deserialize_device.argtypes = [vp, vp, vp, sz, i32, i32, vp]
    L.snarkvm_b200_g2_serialize_device.argtypes = [vp, vp, sz, i32, vp]
    L.snarkvm_b200_fr_records_decode_device.argtypes = [vp, sz, ctypes.POINTER(FrRecordsSegment), sz, ctypes.POINTER(u64), vp]
    L.snarkvm_b200_matrix_row_walk.argtypes = [vp, sz, u64, u64, vp, ctypes.POINTER(ctypes.c_int64)]
    L.snarkvm_b200_msm_batch_device.argtypes = [vp, vp, sz, vp, vp, sz, vp]
    L.snarkvm_b200_msm_window_sums_plan_device.argtypes = [vp, vp, sz, vp, sz, vp, sz, vp]
    L.snarkvm_b200_kzg_commit_batch_hiding_device.argtypes = [vp, vp, sz, vp, vp, vp, vp, vp, sz, vp]
    L.snarkvm_b200_kzg_commit_batch_precomputed_device.argtypes = [vp, vp, vp, vp, sz, vp]
    L.snarkvm_b200_sonic_commit_batch_device.argtypes = [vp, sz, vp, vp, vp, vp, vp, vp, sz, vp]
    L.snarkvm_b200_generator_mul_device.argtypes = [vp, sz, vp, sz, vp]
    L.snarkvm_b200_msm_scratch_stats.argtypes = [ctypes.POINTER(sz), ctypes.POINTER(sz), ctypes.POINTER(sz)]
    L.snarkvm_b200_msm_set_scratch_limit.argtypes = [sz]
    L.snarkvm_b200_selftest_coop.argtypes = [u32, u64, ctypes.POINTER(u32), vp]
    L.snarkvm_b200_selftest_host_copy.argtypes = [sz, u64, ctypes.POINTER(u32)]
    L.snarkvm_b200_test_field_op_device.argtypes = [i32, i32, i32, vp, vp, vp, sz, vp]
    L.snarkvm_b200_test_curve_op_device.argtypes = [i32, i32, vp, vp, vp, vp, sz, vp]
    L.snarkvm_b200_test_field_op_host.argtypes = [i32, i32, vp, vp, vp, sz]
    L.snarkvm_b200_test_tower_op_device.argtypes = [i32, i32, vp, vp, vp, vp, sz, vp]
    L.snarkvm_b200_test_sqrt_device.argtypes = [i32, vp, vp, vp, sz, vp]
    L.snarkvm_b200_msm_window_sums_host.argtypes = [vp, vp, sz, vp, sz, vp, sz, vp]
    for s in SYMBOLS[5:]:
        getattr(L, s).restype = i32
    L.snarkvm_b200_launch_count.restype = u64
    L.snarkvm_b200_msm_g2.restype = _RustError
    _libc = ctypes.CDLL(None)
    _libc.free.argtypes = [ctypes.c_void_p]
    _lib = L
    return L


def check_rust_error(err: _RustError) -> None:
    """`if err.code != 0 { return Err(err) }` (lib.rs:93-96); frees the malloc'd message."""
    if err.code != 0:
        msg = ""
        if err.message:
            msg = ctypes.string_at(err.message).decode(errors="replace")
            _libc.free(err.message)
        raise CudaError(err.code, msg)


def check(code: int) -> None:
    if code != 0:
        raise CudaError(code, "see cudaError_t")


def launch_count() -> int:
    return int(lib().snarkvm_b200_launch_count())


PROF_MSM_SORT, PROF_MSM_ACCUMULATE, PROF_MSM_REDUCE, PROF_NTT_PASS = 0, 1, 2, 3


def profile_enable(on: bool) -> None:
    check(lib().snarkvm_b200_profile_enable(1 if on else 0))


def profile_collect(kind: int):
    """(total_ms, launches) of the recorded kernels of `kind` since the last collect."""
    ms, cnt = ctypes.c_double(), ctypes.c_uint64()
    check(lib().snarkvm_b200_profile_collect(kind, ctypes.byref(ms), ctypes.byref(cnt)))
    return ms.value, cnt.value
