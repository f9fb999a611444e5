"""Device-resident entry points (PART 2 of include/snarkvm_b200.h) on torch CUDA tensors.

PyTorch is plumbing only: it owns the HBM allocations and the stream; every kernel that runs
is one of this repository's hand-written sm_90a kernels inside libsnarkvm_b200.so.
Tensor conventions: any dtype, contiguous, interpreted as raw bytes in the reference layouts
(Fr: 32 B/elt; scalar: 32 B; affine: `stride` B/point, stride ≥ 104 and a multiple of 8).
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _lib, poseidon
from .cuda import NTTDirection, NTTInputOutputOrder, NTTType

XYZZ_BYTES = 192
AFFINE_STRIDE = 104


def _check(t: torch.Tensor, name: str) -> int:
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.is_contiguous()):
        raise TypeError(f"{name} must be a contiguous CUDA tensor")
    return t.data_ptr()


def _nbytes(t: torch.Tensor) -> int:
    return t.numel() * t.element_size()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def ntt_(x: torch.Tensor, direction: NTTDirection = NTTDirection.Forward, ntt_type: NTTType = NTTType.Standard,
         scratch: torch.Tensor | None = None) -> torch.Tensor:
    """In-place natural-order NTT of the 2^lg Fr elements in `x` (32 B each)."""
    n = _nbytes(x) // 32
    if n <= 0 or n & (n - 1) or n * 32 != _nbytes(x):
        raise ValueError("domain_size is not power of 2")
    lg = n.bit_length() - 1
    sp = 0
    if scratch is not None:
        if _nbytes(scratch) < _nbytes(x):
            raise ValueError("scratch too small")
        sp = _check(scratch, "scratch")
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().snarkvm_b200_ntt_device(_check(x, "x"), lg, int(NTTInputOutputOrder.NN), int(direction),
                                                       int(ntt_type), sp, _stream()))
    return x


def polymul(polys: list, evals: list, lg: int) -> torch.Tensor:
    dev = (polys + evals)[0].device
    n = 1 << lg
    out = torch.zeros((n, 4), dtype=torch.int64, device=dev)
    pp = (ctypes.c_void_p * max(1, len(polys)))(*[_check(p, "poly") for p in polys])
    pl = (ctypes.c_size_t * max(1, len(polys)))(*[_nbytes(p) // 32 for p in polys])
    ep = (ctypes.c_void_p * max(1, len(evals)))(*[_check(e, "eval") for e in evals])
    el = (ctypes.c_size_t * max(1, len(evals)))(*[_nbytes(e) // 32 for e in evals])
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().snarkvm_b200_polymul_device(out.data_ptr(), len(polys), ctypes.cast(pp, ctypes.c_void_p),
                                                           ctypes.cast(pl, ctypes.c_void_p), len(evals),
                                                           ctypes.cast(ep, ctypes.c_void_p), ctypes.cast(el, ctypes.c_void_p),
                                                           lg, _stream()))
    return out


def msm_plan(npoints: int) -> dict:
    c, nwin, cap = ctypes.c_int(), ctypes.c_int(), ctypes.c_uint32()
    _lib.check(_lib.lib().snarkvm_b200_msm_plan(npoints, ctypes.byref(c), ctypes.byref(nwin), ctypes.byref(cap)))
    return {"c": c.value, "nwin": nwin.value, "cap": cap.value, "levels": int(_lib.lib().snarkvm_b200_msm_plan_levels(npoints))}


def _msm_args(bases: torch.Tensor, scalars: torch.Tensor, stride: int):
    npoints = _nbytes(scalars) // 32
    if npoints * 32 != _nbytes(scalars):
        raise ValueError("scalars must be a whole number of 32-byte integers")
    if npoints * stride > _nbytes(bases):
        raise ValueError(f"length mismatch {_nbytes(bases) // stride} points < {npoints} scalars")
    return npoints


def msm(bases: torch.Tensor, scalars: torch.Tensor, stride: int = AFFINE_STRIDE) -> np.ndarray:
    """VariableBase::msm with bases and scalars resident in HBM → normalised projective uint64[18]."""
    npoints = _msm_args(bases, scalars, stride)
    out = np.zeros(18, dtype=np.uint64)
    with torch.cuda.device(bases.device):
        _lib.check(_lib.lib().snarkvm_b200_msm_device(out.ctypes.data, _check(bases, "bases"), npoints,
                                                       _check(scalars, "scalars"), stride, _stream()))
    return out


G2_AFFINE_STRIDE = 200       # Affine<G2>: x.c0 x.c1 y.c0 y.c1 (4 × 48 B) infinity pad


def msm_g2(bases: torch.Tensor, scalars: torch.Tensor, stride: int = G2_AFFINE_STRIDE) -> np.ndarray:
    """VariableBase::msm over G2 (standard::msm semantics) with bases and scalars resident in HBM → normalised Projective<G2>
    image uint64[36] (X, Y, Z over Fq2)."""
    npoints = _msm_args(bases, scalars, stride)
    out = np.zeros(36, dtype=np.uint64)
    with torch.cuda.device(bases.device):
        _lib.check(_lib.lib().snarkvm_b200_msm_g2_device(out.ctypes.data, _check(bases, "bases"), npoints,
                                                          _check(scalars, "scalars"), stride, _stream()))
    return out


def generate_bases_g2(npoints: int, seed: int, device="cuda", stride: int = G2_AFFINE_STRIDE) -> torch.Tensor:
    """Synthetic G2 bases P_i = h(seed, i)·G2 in the reference Affine<G2> layout, generated in HBM."""
    t = torch.empty((npoints, stride), dtype=torch.uint8, device=device)
    with torch.cuda.device(t.device):
        _lib.check(_lib.lib().snarkvm_b200_generate_bases_g2_device(t.data_ptr(), npoints, stride, seed & (2**64 - 1), _stream()))
    return t


G2_PREPARED_BYTES = 19904    # 69 coefficient triples of three Fq2, infinity flag (u32), padding
GT_BYTES = 576               # Fp12: twelve Montgomery Fq


def g2_prepare(points: torch.Tensor, stride: int = G2_AFFINE_STRIDE) -> torch.Tensor:
    """G2Prepared::from_affine of every Affine<G2> image in HBM → prepared points [n, G2_PREPARED_BYTES] (uint8, HBM).  A
    coordinate image ≥ q raises CudaError naming the lowest such point (.point)."""
    n = _nbytes(points) // stride
    out = torch.empty((n, G2_PREPARED_BYTES), dtype=torch.uint8, device=points.device)
    bad = ctypes.c_int64(-1)
    with torch.cuda.device(points.device):
        code = _lib.lib().snarkvm_b200_g2_prepare_device(out.data_ptr(), _check(points, "points") if n else None, n, stride,
                                                         ctypes.byref(bad), _stream())
    if code != 0:
        err = _lib.CudaError(code, f"G2 point {bad.value}" if bad.value >= 0 else "see cudaError_t")
        err.point = bad.value if bad.value >= 0 else None
        raise err
    return out


def pairing_products(g1: torch.Tensor, g2_index: torch.Tensor, prepared: torch.Tensor, check_start: torch.Tensor,
                     g1_stride: int = AFFINE_STRIDE, miller: bool = False):
    """PairingEngine::product_of_pairings for every check in one call.  Pair i is (G1 Affine image g1[i], prepared point
    prepared[g2_index[i]]); check c owns pairs check_start[c] .. check_start[c + 1] − 1 (check_start: int32, nchecks + 1 entries,
    from 0 to the number of pairs).  → (GT values [nchecks, GT_BYTES] uint8 in HBM, is_one: bool tensor [nchecks] in HBM), and with
    `miller` the pairs' Miller values [npairs, GT_BYTES] as a third item.  A coordinate image ≥ q, a G2 index out of range or a
    malformed check_start raises CudaError naming the lowest check concerned (.check)."""
    dev = check_start.device
    nchecks = check_start.numel() - 1
    if nchecks < 0 or check_start.dtype != torch.int32:
        raise ValueError("check_start: int32, one entry more than there are checks")
    npairs = _nbytes(g1) // g1_stride
    if g2_index.numel() != npairs or (npairs and g2_index.dtype != torch.int32):
        raise ValueError("one int32 G2 index per G1 point")
    gt = torch.empty((max(nchecks, 0), GT_BYTES), dtype=torch.uint8, device=dev)
    is_one = torch.zeros(max(nchecks, 0), dtype=torch.int32, device=dev)
    mv = torch.empty((npairs, GT_BYTES), dtype=torch.uint8, device=dev) if miller else None
    bad = ctypes.c_int64(-1)
    with torch.cuda.device(dev):
        code = _lib.lib().snarkvm_b200_pairing_products_device(
            gt.data_ptr(), is_one.data_ptr(), mv.data_ptr() if miller and npairs else None,
            _check(g1, "g1") if npairs else None, g1_stride, _check(g2_index, "g2_index") if npairs else None, npairs,
            _check(prepared, "prepared") if prepared.numel() else None, _nbytes(prepared) // G2_PREPARED_BYTES,
            _check(check_start, "check_start"), nchecks, ctypes.byref(bad), _stream())
    if code != 0:
        err = _lib.CudaError(code, f"check {bad.value}" if bad.value >= 0 else "see cudaError_t")
        err.check = bad.value if bad.value >= 0 else None
        raise err
    return (gt, is_one.bool(), mv) if miller else (gt, is_one.bool())


G1_VALID, G1_NOT_CANONICAL, G1_NOT_ON_CURVE, G1_NOT_IN_SUBGROUP, G1_BAD_FLAGS = 0, 1, 2, 3, 4
G1_COMPRESSED_BYTES, G1_UNCOMPRESSED_BYTES, G1_TO_BYTES_BYTES = 48, 96, 97
# the byte forms of a G1 point (SNARKVM_B200_G1_FORM_*): False / True name the first two, as `compressed` flags
G1_UNCOMPRESSED, G1_COMPRESSED, G1_TO_BYTES = 0, 1, 2
_G1_FORM_BYTES = {G1_UNCOMPRESSED: G1_UNCOMPRESSED_BYTES, G1_COMPRESSED: G1_COMPRESSED_BYTES, G1_TO_BYTES: G1_TO_BYTES_BYTES}


def _g1_form(compressed) -> int:
    form = int(compressed)
    if form not in _G1_FORM_BYTES:
        raise ValueError(f"unknown G1 byte form {compressed!r}")
    return form


def g1_validate(points: torch.Tensor, stride: int = AFFINE_STRIDE) -> torch.Tensor:
    """Affine::check of every Affine<G1> image in HBM (snarkvm_b200_g1_validate_device) → int32 status per point in HBM: G1_VALID
    (infinity included), G1_NOT_CANONICAL (a coordinate image ≥ q), G1_NOT_ON_CURVE or G1_NOT_IN_SUBGROUP, the first test failed."""
    n = _nbytes(points) // stride
    status = torch.empty(n, dtype=torch.int32, device=points.device)
    if n:
        with torch.cuda.device(points.device):
            _lib.check(_lib.lib().snarkvm_b200_g1_validate_device(status.data_ptr(), _check(points, "points"), n, stride, _stream()))
    return status


def g1_deserialize(bytes_u8: torch.Tensor, compressed=True, validate: bool = True):
    """G1 points from their byte forms (snarkvm_b200_g1_deserialize_device): `bytes_u8` a uint8 CUDA tensor of n × 48 compressed,
    n × 96 uncompressed or (compressed = G1_TO_BYTES) n × 97 ToBytes bytes → (Affine<G1> images uint8 [n, 104], int32 status [n]),
    both in HBM.  Status G1_BAD_FLAGS (both flag bits set, or bit 7 of an uncompressed x; ToBytes: an infinity byte above 1, or
    y = 1 with the infinity byte disagreeing with x = 0), G1_NOT_CANONICAL (a coordinate ≥ q), G1_NOT_ON_CURVE (compressed: x³ + 1
    has no square root), else G1_VALID or, with `validate`, g1_validate's status.  Bytes that decode to no point leave an all-zero
    image; a ToBytes infinity keeps the coordinates it was read with."""
    form = _g1_form(compressed)
    size = _G1_FORM_BYTES[form]
    if bytes_u8.dtype != torch.uint8 or _nbytes(bytes_u8) % size:
        raise ValueError(f"g1_deserialize takes uint8 bytes, {size} per point")
    n = _nbytes(bytes_u8) // size
    images = torch.empty((n, AFFINE_STRIDE), dtype=torch.uint8, device=bytes_u8.device)
    status = torch.empty(n, dtype=torch.int32, device=bytes_u8.device)
    if n:
        with torch.cuda.device(bytes_u8.device):
            _lib.check(_lib.lib().snarkvm_b200_g1_deserialize_device(images.data_ptr(), status.data_ptr(), _check(bytes_u8, "bytes_u8"),
                                                                     n, form, int(bool(validate)), _stream()))
    return images, status


def g1_serialize(projective: torch.Tensor, compressed=True) -> torch.Tensor:
    """G1 points to their byte forms (snarkvm_b200_g1_serialize_device): `projective` a CUDA tensor of n normalised projective
    images (X, Y, Z Montgomery Fq, 144 bytes each; Z = one, or zero for infinity) → uint8 [n, 48] compressed or [n, 96]
    uncompressed, in HBM.  With compressed = G1_TO_BYTES, `projective` holds Affine<G1> images (104 bytes each) instead → uint8
    [n, 97], their ToBytes form."""
    form = _g1_form(compressed)
    image = AFFINE_STRIDE if form == G1_TO_BYTES else 144
    if _nbytes(projective) % image:
        raise ValueError(f"g1_serialize takes {image}-byte images in this form")
    n = _nbytes(projective) // image
    size = _G1_FORM_BYTES[form]
    out = torch.empty((n, size), dtype=torch.uint8, device=projective.device)
    if n:
        with torch.cuda.device(projective.device):
            _lib.check(_lib.lib().snarkvm_b200_g1_serialize_device(out.data_ptr(), _check(projective, "projective"), n,
                                                                   form, _stream()))
    return out


G2_COMPRESSED_BYTES, G2_UNCOMPRESSED_BYTES = 96, 192


def g2_validate(points: torch.Tensor, stride: int = G2_AFFINE_STRIDE) -> torch.Tensor:
    """Valid for Affine<G2> of every Affine<G2> image in HBM (snarkvm_b200_g2_validate_device) → int32 status per point in HBM,
    the G1_* values: G1_VALID (infinity included), G1_NOT_CANONICAL (a coordinate image ≥ q), G1_NOT_ON_CURVE or
    G1_NOT_IN_SUBGROUP ([r]·P ≠ O), the first test failed."""
    n = _nbytes(points) // stride
    status = torch.empty(n, dtype=torch.int32, device=points.device)
    if n:
        with torch.cuda.device(points.device):
            _lib.check(_lib.lib().snarkvm_b200_g2_validate_device(status.data_ptr(), _check(points, "points"), n, stride, _stream()))
    return status


def g2_deserialize(bytes_u8: torch.Tensor, compressed: bool = True, validate: bool = True):
    """G2 points from their byte forms (snarkvm_b200_g2_deserialize_device): `bytes_u8` a uint8 CUDA tensor of n × 96 compressed
    or n × 192 uncompressed bytes → (Affine<G2> images uint8 [n, 200], int32 status [n]), both in HBM.  Status G1_BAD_FLAGS (both
    flag bits set, or bit 7 of a coordinate that carries no flags), G1_NOT_CANONICAL (a coordinate ≥ q), G1_NOT_ON_CURVE
    (compressed: x³ + B' has no square root in Fq2), else G1_VALID or, with `validate`, g2_validate's status.  Bytes that decode to
    no point leave an all-zero image."""
    size = G2_COMPRESSED_BYTES if compressed else G2_UNCOMPRESSED_BYTES
    if bytes_u8.dtype != torch.uint8 or _nbytes(bytes_u8) % size:
        raise ValueError(f"g2_deserialize takes uint8 bytes, {size} per point")
    n = _nbytes(bytes_u8) // size
    images = torch.empty((n, G2_AFFINE_STRIDE), dtype=torch.uint8, device=bytes_u8.device)
    status = torch.empty(n, dtype=torch.int32, device=bytes_u8.device)
    if n:
        with torch.cuda.device(bytes_u8.device):
            _lib.check(_lib.lib().snarkvm_b200_g2_deserialize_device(images.data_ptr(), status.data_ptr(), _check(bytes_u8, "bytes_u8"),
                                                                     n, int(bool(compressed)), int(bool(validate)), _stream()))
    return images, status


def g2_serialize(images: torch.Tensor, compressed: bool = True) -> torch.Tensor:
    """G2 points to their byte forms (snarkvm_b200_g2_serialize_device): `images` a CUDA tensor of n Affine<G2> images (200 bytes
    each) → uint8 [n, 96] compressed or [n, 192] uncompressed, in HBM"""
    if _nbytes(images) % G2_AFFINE_STRIDE:
        raise ValueError(f"g2_serialize takes {G2_AFFINE_STRIDE}-byte Affine<G2> images")
    n = _nbytes(images) // G2_AFFINE_STRIDE
    out = torch.empty((n, G2_COMPRESSED_BYTES if compressed else G2_UNCOMPRESSED_BYTES), dtype=torch.uint8, device=images.device)
    if n:
        with torch.cuda.device(images.device):
            _lib.check(_lib.lib().snarkvm_b200_g2_serialize_device(out.data_ptr(), _check(images, "images"), n, int(bool(compressed)),
                                                                   _stream()))
    return out


FR_RECORD_NOT_CANONICAL, FR_RECORD_BAD_COLUMN = 1, 2


def fr_records_decode(blob: torch.Tensor, segments: list) -> list:
    """Fr records of a byte blob in HBM (snarkvm_b200_fr_records_decode_device), every segment in one launch and one
    synchronisation.  A segment is (offset, count, stride, out, cols, num_cols, row_ptr): `count` canonical Fr 32 bytes apart
    (stride 32) or Fr-and-u64-column entries (stride 40), written to `out` ([count, 4] int64 CUDA tensor, Montgomery) and, for
    stride 40, the columns to `cols` (int32 [count]), each checked below num_cols.  With `row_ptr` (int32 [nrows + 1] CUDA tensor)
    the segment is a matrix section at `offset` whose entry e of row i sits at offset + 16 + 8·i + 40·e.  → per segment None, or
    (index, FR_RECORD_NOT_CANONICAL or FR_RECORD_BAD_COLUMN) of its first bad record."""
    if blob.dtype != torch.uint8:
        raise TypeError("blob must be a uint8 tensor")
    if not segments:
        return []
    segs = (_lib.FrRecordsSegment * len(segments))()
    for k, (offset, count, stride, out, cols, num_cols, row_ptr) in enumerate(segments):
        if _nbytes(out) != 32 * count or (cols is not None and (cols.dtype != torch.int32 or cols.numel() != count)):
            raise ValueError(f"segment {k}: one 32-byte output and one int32 column per record")
        s = segs[k]
        s.offset, s.count, s.stride = offset, count, stride
        s.d_out = _check(out, "out") if count else None
        s.d_cols = _check(cols, "cols") if cols is not None and count else None
        s.num_cols = num_cols
        if row_ptr is not None:
            if row_ptr.dtype != torch.int32:
                raise TypeError("row_ptr must be an int32 tensor")
            s.d_row_ptr, s.nrows = _check(row_ptr, "row_ptr"), row_ptr.numel() - 1
    bad = (ctypes.c_uint64 * len(segments))()
    with torch.cuda.device(blob.device):
        _lib.check(_lib.lib().snarkvm_b200_fr_records_decode_device(_check(blob, "blob"), _nbytes(blob), segs, len(segments), bad,
                                                                    _stream()))
    return [None if v == 2**64 - 1 else (v >> 2, v & 3) for v in bad]


def matrix_row_walk(blob, offset: int, nrows: int, nnz: int):
    """the row headers of one matrix section of a HOST buffer (snarkvm_b200_matrix_row_walk): its rows start at byte `offset` of
    `blob` (anything with the buffer protocol; no copy) → (int32 row_ptr [nrows + 1] as a numpy array, None), or (None, the first
    row that overruns the buffer or carries the count past nnz; nrows when the rows hold fewer than nnz entries)"""
    buf = np.frombuffer(blob, dtype=np.uint8)
    if not 0 <= offset <= buf.size:
        raise ValueError("offset outside the buffer")
    if nnz >= 2**31:
        return None, -1
    row_ptr = np.empty(nrows + 1, dtype=np.int32)
    bad = ctypes.c_int64(-1)
    code = _lib.lib().snarkvm_b200_matrix_row_walk(buf.ctypes.data + offset if nrows else None, buf.size - offset, nrows, nnz,
                                                   row_ptr.ctypes.data, ctypes.byref(bad))
    if code != 0:
        return None, bad.value
    return row_ptr, None


POSEIDON_ABSORB, POSEIDON_SQUEEZE, POSEIDON_SQUEEZE_NONNATIVE, POSEIDON_SQUEEZE_SHORT_NONNATIVE = 0, 1, 2, 3


def poseidon_transcripts(field: int, ops: torch.Tensor, op_start: torch.Tensor, inputs: torch.Tensor, nout: int, nout_fr: int,
                         state: torch.Tensor | None = None):
    """PoseidonSponge<F, 2, 1> transcripts, one per thread (snarkvm_b200_poseidon_transcripts_device): transcript t runs the
    operations ops[op_start[t] : op_start[t + 1]] (int32 [nops, 3]: kind POSEIDON_*, n, offset) on a sponge of its own.  field:
    poseidon.FIELD_FQ (snarkVM's Fiat–Shamir sponge) or FIELD_FR.  inputs: Montgomery F elements as int64 [nin, 6] (Fq) or
    [nin, 4] (Fr).  → (native squeezes int64 [nout, limbs] Montgomery F, nonnative squeezes int64 [nout_fr, 4] Montgomery Fr), both in
    HBM.  A malformed operation or an absorbed element ≥ p raises CudaError naming the lowest such transcript (.transcript), and no
    output is written.
    `state`: None starts every transcript from a fresh sponge.  Otherwise one state record per transcript (int64 CUDA tensor
    [ntranscripts, poseidon.state_words(field) // 2], poseidon.fresh_states makes fresh ones): each transcript resumes from its
    record and the record is updated in place (snarkvm_b200_poseidon_transcripts_resume_device).  A malformed record raises like a
    malformed operation, and then no record is written either."""
    if field not in poseidon.FIELDS:
        raise ValueError(f"unknown field {field}")
    words = poseidon.FIELDS[field][2]
    dev = op_start.device
    if op_start.dtype != torch.int32 or op_start.dim() != 1 or op_start.numel() < 1:
        raise ValueError("op_start: int32, one entry more than there are transcripts")
    if ops.dtype != torch.int32 or ops.dim() != 2 or ops.shape[1] != 3:
        raise ValueError("ops: int32 [nops, 3]")
    if inputs.dtype != torch.int64 or inputs.dim() != 2 or inputs.shape[1] != words // 2:
        raise ValueError(f"inputs: int64 [nin, {words // 2}]")
    ntranscripts, nops, nin = op_start.numel() - 1, ops.shape[0], inputs.shape[0]
    out = torch.empty((nout, words // 2), dtype=torch.int64, device=dev)
    out_fr = torch.empty((nout_fr, 4), dtype=torch.int64, device=dev)
    if state is not None and (state.dtype != torch.int64 or state.shape != (ntranscripts, poseidon.state_words(field) // 2)):
        raise ValueError(f"state: int64 [{ntranscripts}, {poseidon.state_words(field) // 2}], one record per transcript")
    params = poseidon.device_parameters(field, dev)
    bad = ctypes.c_int64(-1)
    args = (field, _check(params, "params"), _check(ops, "ops") if nops else None, _check(op_start, "op_start"), ntranscripts, nops,
            _check(inputs, "inputs") if nin else None, nin, out.data_ptr() if nout else None, nout,
            out_fr.data_ptr() if nout_fr else None, nout_fr)
    with torch.cuda.device(dev):
        if state is None:
            code = _lib.lib().snarkvm_b200_poseidon_transcripts_device(*args, ctypes.byref(bad), _stream())
        else:
            code = _lib.lib().snarkvm_b200_poseidon_transcripts_resume_device(*args, _check(state, "state") if ntranscripts else None,
                                                                              ctypes.byref(bad), _stream())
    if code != 0:
        err = _lib.CudaError(code, f"transcript {bad.value}" if bad.value >= 0 else "see cudaError_t")
        err.transcript = bad.value if bad.value >= 0 else None
        raise err
    return out, out_fr


def msm_window_sums(bases: torch.Tensor, scalars: torch.Tensor, stride: int = AFFINE_STRIDE, plan_npoints: int | None = None,
                    flags: torch.Tensor | None = None, out: torch.Tensor | None = None) -> torch.Tensor:
    """Per-window XYZZ sums [nwin, 24] (int64 view of 192-byte points), left in HBM.  `plan_npoints` (≥ the number of
    scalars) fixes the window plan — all ranks of a sharded MSM pass the largest shard size; an empty shard gives infinity
    sums.  `flags`: optional int32 CUDA tensor [1] that receives bit 0 = "a scalar ≥ 2^253 was seen"."""
    npoints = _msm_args(bases, scalars, stride)
    pn = npoints if plan_npoints is None else int(plan_npoints)
    if pn < max(npoints, 1):
        raise ValueError("plan_npoints must be at least the shard size and positive")
    plan = msm_plan(pn)
    dev = bases.device if bases.is_cuda else scalars.device
    sums = torch.empty((plan["nwin"], XYZZ_BYTES // 8), dtype=torch.int64, device=dev) if out is None else out
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().snarkvm_b200_msm_window_sums_plan_device(
            _check(sums, "out"), flags.data_ptr() if flags is not None else None, pn, _check(bases, "bases") if npoints else None, npoints,
            _check(scalars, "scalars") if npoints else None, stride, _stream()))
    return sums


def msm_window_sums_host(out: torch.Tensor, flags: torch.Tensor | None, plan_npoints: int, points: np.ndarray, scalars: np.ndarray,
                         stride: int = AFFINE_STRIDE) -> torch.Tensor:
    """msm_window_sums from HOST buffers (numpy uint8 [n, stride] points, uint64 [n, 4] canonical scalars): the library uploads
    them (ranges overlapped with the kernels, pageable memory staged through pinned buffers) and leaves the sums in `out`
    (CUDA, [nwin, 24] int64) without synchronising.  Pageable inputs may be reused once the call returns; pinned inputs are
    read by DMA after it returns, so the caller keeps them unchanged until the stream has passed the call."""
    if not (isinstance(points, np.ndarray) and points.dtype == np.uint8 and points.ndim == 2 and points.flags["C_CONTIGUOUS"]):
        raise TypeError(f"points must be a C-contiguous uint8 array [n, {stride}]")
    if points.shape[1] != stride:
        raise ValueError(f"points rows are {points.shape[1]} bytes, the stride is {stride}")
    if not (isinstance(scalars, np.ndarray) and scalars.dtype == np.uint64 and scalars.ndim == 2 and scalars.shape[1] == 4
            and scalars.flags["C_CONTIGUOUS"]):
        raise TypeError("scalars must be a C-contiguous uint64 array [n, 4]")
    npoints = scalars.shape[0]
    if npoints > points.shape[0]:
        raise ValueError(f"length mismatch {points.shape[0]} points < {npoints} scalars")
    with torch.cuda.device(out.device):
        _lib.check(_lib.lib().snarkvm_b200_msm_window_sums_host(
            _check(out, "out"), flags.data_ptr() if flags is not None else None, int(plan_npoints), points.ctypes.data if npoints else None,
            npoints, scalars.ctypes.data if npoints else None, stride, _stream()))
    return out


def msm_batch(bases: torch.Tensor, scalar_vectors: list, stride: int = AFFINE_STRIDE) -> np.ndarray:
    """`len(scalar_vectors)` MSMs over the same resident bases in ONE pass → [count, 18] u64 (normalised projective each)."""
    count = len(scalar_vectors)
    out = np.zeros((count, 18), dtype=np.uint64)
    if count == 0:
        return out
    lens = [_msm_args(bases, v, stride) for v in scalar_vectors]
    ptrs = (ctypes.c_void_p * count)(*[(_check(v, "scalars") if n else None) for v, n in zip(scalar_vectors, lens)])
    szs = (ctypes.c_size_t * count)(*lens)
    with torch.cuda.device(bases.device):
        _lib.check(_lib.lib().snarkvm_b200_msm_batch_device(out.ctypes.data, _check(bases, "bases"), stride, ptrs, szs, count, _stream()))
    return out


def msm_set_scratch_limit(nbytes: int) -> None:
    """bytes of MSM scratch concurrent calls on the current device may hold together (callers beyond it wait)"""
    _lib.check(_lib.lib().snarkvm_b200_msm_set_scratch_limit(int(nbytes)))


def msm_scratch_stats() -> dict:
    """MSM scratch budget of the current device: {'limit', 'in_use', 'peak'} in bytes."""
    a, b, c = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t()
    _lib.check(_lib.lib().snarkvm_b200_msm_scratch_stats(ctypes.byref(a), ctypes.byref(b), ctypes.byref(c)))
    return {"limit": a.value, "in_use": b.value, "peak": c.value}


def xyzz_sum_ranks(gathered: torch.Tensor, nranks: int, count: int) -> torch.Tensor:
    out = torch.empty((count, XYZZ_BYTES // 8), dtype=torch.int64, device=gathered.device)
    with torch.cuda.device(gathered.device):
        _lib.check(_lib.lib().snarkvm_b200_xyzz_sum_ranks_device(out.data_ptr(), _check(gathered, "gathered"), nranks, count,
                                                                  _stream()))
    return out


def msm_finish(window_sums_host: np.ndarray, c: int) -> np.ndarray:
    """Host fold Σ_w 2^{c·w}·S_w of XYZZ window sums (c = 0: plain sum) → normalised projective."""
    ws = np.ascontiguousarray(window_sums_host).view(np.uint8).reshape(-1, XYZZ_BYTES)
    out = np.zeros(18, dtype=np.uint64)
    _lib.check(_lib.lib().snarkvm_b200_msm_finish(out.ctypes.data, ws.ctypes.data, ws.shape[0], c))
    return out


def kzg_commit(powers: torch.Tensor, coeffs_mont: torch.Tensor, stride: int = AFFINE_STRIDE) -> np.ndarray:
    """KZG10::commit core: Σ to_bigint(coeff_i)·powers_i (kzg10/mod.rs:98-156), all operands in HBM."""
    n = _msm_args(powers, coeffs_mont, stride)
    out = np.zeros(18, dtype=np.uint64)
    with torch.cuda.device(powers.device):
        _lib.check(_lib.lib().snarkvm_b200_kzg_commit_device(out.ctypes.data, _check(powers, "powers"), stride,
                                                              _check(coeffs_mont, "coeffs"), n, _stream()))
    return out


def kzg_commit_hiding(powers: torch.Tensor, coeffs_mont: torch.Tensor, gamma_powers: torch.Tensor, blinding_mont: torch.Tensor,
                      stride: int = AFFINE_STRIDE) -> np.ndarray:
    """KZG10::commit with hiding_bound = Some(_) (kzg10/mod.rs:98-156): Σ to_bigint(c_i)·powers_i + Σ to_bigint(b_j)·gamma_powers_j;
    the caller samples the blinding polynomial b (KZGRandomness::rand)."""
    n = _msm_args(powers, coeffs_mont, stride)
    nb = _nbytes(blinding_mont) // 32
    if nb > _nbytes(gamma_powers) // stride:
        raise ValueError("hiding bound exceeds powers_of_beta_times_gamma_g")      # check_hiding_bound, mod.rs:134-137
    out = np.zeros(18, dtype=np.uint64)
    with torch.cuda.device(powers.device):
        _lib.check(_lib.lib().snarkvm_b200_kzg_commit_hiding_device(
            out.ctypes.data, _check(powers, "powers"), stride, _check(coeffs_mont, "coeffs"), n,
            _check(gamma_powers, "gamma_powers"), _check(blinding_mont, "blinding"), nb, _stream()))
    return out


def kzg_commit_batch(powers: torch.Tensor, polys_mont: list, stride: int = AFFINE_STRIDE, gamma_powers: torch.Tensor | None = None,
                     blindings_mont: list | None = None) -> np.ndarray:
    """All commitments of a round against the same resident powers in ONE pass (sonic_pc/mod.rs:177-257) → [count, 18] u64.
    With `gamma_powers` and `blindings_mont` (one Montgomery coefficient tensor or None per polynomial) the hiding terms
    Σ_j blinding_i[j]·gamma_powers[j] (kzg10/mod.rs:129-150) ride in the same pass."""
    count = len(polys_mont)
    out = np.zeros((count, 18), dtype=np.uint64)
    if count == 0:
        return out
    nb = _nbytes(powers) // stride
    lens = [_nbytes(p) // 32 for p in polys_mont]
    if max(lens) > nb:
        raise ValueError("polynomial degree exceeds the number of powers")         # check_degree_is_too_large, mod.rs:105
    ptrs = (ctypes.c_void_p * count)(*[(_check(p, "poly") if n else None) for p, n in zip(polys_mont, lens)])
    szs = (ctypes.c_size_t * count)(*lens)
    with torch.cuda.device(powers.device):
        if blindings_mont is None:
            _lib.check(_lib.lib().snarkvm_b200_kzg_commit_batch_device(out.ctypes.data, _check(powers, "powers"), stride, ptrs, szs, count, _stream()))
        else:
            if len(blindings_mont) != count:
                raise ValueError("one blinding polynomial (or None) per polynomial")
            blens = [0 if b is None else _nbytes(b) // 32 for b in blindings_mont]
            if max(blens) > _nbytes(gamma_powers) // stride:
                raise ValueError("hiding bound exceeds powers_of_beta_times_gamma_g")          # check_hiding_bound, mod.rs:134-137
            bptrs = (ctypes.c_void_p * count)(*[(_check(b, "blinding") if n else None) for b, n in zip(blindings_mont, blens)])
            bszs = (ctypes.c_size_t * count)(*blens)
            _lib.check(_lib.lib().snarkvm_b200_kzg_commit_batch_hiding_device(
                out.ctypes.data, _check(powers, "powers"), stride, ptrs, szs, _check(gamma_powers, "gamma_powers"), bptrs, bszs, count, _stream()))
    return out


def generator_mul(scalars: torch.Tensor, stride: int = AFFINE_STRIDE) -> torch.Tensor:
    """P_i = s_i·G for canonical scalars [n, 4] in HBM → affine points [n, stride] (set-up helper, not a hot path)"""
    n = _nbytes(scalars) // 32
    out = torch.empty((n, stride), dtype=torch.uint8, device=scalars.device)
    with torch.cuda.device(scalars.device):
        _lib.check(_lib.lib().snarkvm_b200_generator_mul_device(out.data_ptr(), stride, _check(scalars, "scalars") if n else None, n, _stream()))
    return out


def generate_powers(n: int, beta: int, scale: int = 1, device="cuda", stride: int = AFFINE_STRIDE) -> torch.Tensor:
    """scale·β^i·G for i < n: powers_of_beta_g (scale = 1) or powers_of_beta_times_gamma_g (scale = γ) of a universal setup whose
    trapdoor the caller knows.  The scalars are built by doubling (v[m:2m] = β^m·v[0:m]), then one fixed-base pass."""
    from .algorithms import _fr_int_to_mont, _R_MOD
    s = torch.zeros((n, 4), dtype=torch.int64, device=device)
    if n == 0:
        return torch.empty((0, stride), dtype=torch.uint8, device=device)
    s[0] = torch.from_numpy(_fr_int_to_mont(scale % _R_MOD).view(np.int64)).to(s.device)
    m = 1
    while m < n:
        k = min(m, n - m)
        fr_vec_op(s[:k], _fr_int_to_mont(pow(beta, m, _R_MOD)), FR_MUL, out=s[m:m + k])
        m *= 2
    return generator_mul(fr_from_mont(s), stride)


def sonic_commit_batch(bases: list, polys_mont: list, gamma_bases: list | None = None, blindings_mont: list | None = None,
                       stride: int = AFFINE_STRIDE) -> np.ndarray:
    """SonicKZG10::commit of a round in ONE pass (sonic_pc/mod.rs:177-257) → [count, 18] u64.  `bases[i]` is the CUDA tensor (or a
    row slice of one: shifted powers are suffixes of the SRS) polynomial i is committed against; `gamma_bases[i]` / `blindings_mont[i]`
    (or None) its hiding terms (kzg10/mod.rs:129-150)."""
    count = len(polys_mont)
    out = np.zeros((count, 18), dtype=np.uint64)
    if count == 0:
        return out
    if len(bases) != count:
        raise ValueError("one base array per polynomial")
    lens = [_nbytes(p) // 32 for p in polys_mont]
    for b, n in zip(bases, lens):
        if n > _nbytes(b) // stride:
            raise ValueError("polynomial degree exceeds the number of powers")             # check_degree_is_too_large, kzg10/mod.rs:105
    bptr = (ctypes.c_void_p * count)(*[(_check(b, "bases") if n else None) for b, n in zip(bases, lens)])
    cptr = (ctypes.c_void_p * count)(*[(_check(p, "poly") if n else None) for p, n in zip(polys_mont, lens)])
    szs = (ctypes.c_size_t * count)(*lens)
    gptr = rptr = rszs = None
    if blindings_mont is not None:
        if gamma_bases is None or len(blindings_mont) != count or len(gamma_bases) != count:
            raise ValueError("one (gamma powers, blinding polynomial) pair (or None) per polynomial")
        blens = [0 if r is None else _nbytes(r) // 32 for r in blindings_mont]
        for g, n in zip(gamma_bases, blens):
            if n and (g is None or n > _nbytes(g) // stride):
                raise ValueError("hiding bound exceeds powers_of_beta_times_gamma_g")      # check_hiding_bound, kzg10/mod.rs:134-137
        gptr = (ctypes.c_void_p * count)(*[(_check(g, "gamma") if n else None) for g, n in zip(gamma_bases, blens)])
        rptr = (ctypes.c_void_p * count)(*[(_check(r, "blinding") if n else None) for r, n in zip(blindings_mont, blens)])
        rszs = (ctypes.c_size_t * count)(*blens)
    dev = next(b.device for b in bases if b is not None)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().snarkvm_b200_sonic_commit_batch_device(out.ctypes.data, stride, bptr, cptr, szs, gptr, rptr, rszs, count, _stream()))
    return out


def g1_ntt(points: torch.Tensor, inverse: bool, stride: int = AFFINE_STRIDE) -> torch.Tensor:
    """FFT / iFFT over 2^k G1 points (EvaluationDomain with T = G1Projective, fft/domain.rs:169-221) → affine points, same stride."""
    n = _nbytes(points) // stride
    if n == 0 or n & (n - 1):
        raise ValueError("domain size must be a power of two")
    out = torch.empty_like(points)
    with torch.cuda.device(points.device):
        _lib.check(_lib.lib().snarkvm_b200_g1_ntt_device(out.data_ptr(), stride, _check(points, "points"), stride, n.bit_length() - 1,
                                                          1 if inverse else 0, _stream()))
    return out


def lagrange_basis(powers_of_beta_g: torch.Tensor, stride: int = AFFINE_STRIDE) -> torch.Tensor:
    """UniversalParams::lagrange_basis (kzg10/data_structures.rs:68-72): ifft of the first n powers, normalised to affine."""
    return g1_ntt(powers_of_beta_g, True, stride)


def _fr_host(x) -> np.ndarray:
    a = np.ascontiguousarray(x, dtype=np.uint64).reshape(4)
    return a


def fr_batch_inversion_and_mul(v: torch.Tensor, coeff_mont) -> torch.Tensor:
    """fields/src/lib.rs:78-129, in place on a CUDA tensor of Montgomery Fr: v_i ← coeff·v_i^{-1}; zeros stay zero."""
    c = _fr_host(coeff_mont)
    with torch.cuda.device(v.device):
        _lib.check(_lib.lib().snarkvm_b200_fr_batch_inversion_and_mul_device(_check(v, "v"), _nbytes(v) // 32, c.ctypes.data, _stream()))
    return v


def poly_divide_by_vanishing(p: torch.Tensor, domain_size: int):
    """DensePolynomial::divide_by_vanishing_poly (fft/polynomial/dense.rs:162-169) → (quotient, remainder) CUDA tensors [.., 4] i64,
    max(m − n, 0) and min(m, n) coefficients, not trimmed."""
    m = _nbytes(p) // 32
    q = torch.empty((max(m - domain_size, 0), 4), dtype=torch.int64, device=p.device)
    r = torch.empty((min(m, domain_size), 4), dtype=torch.int64, device=p.device)
    if m:
        with torch.cuda.device(p.device):
            _lib.check(_lib.lib().snarkvm_b200_poly_divide_by_vanishing_device(q.data_ptr() if q.numel() else None, r.data_ptr(),
                                                                                _check(p, "p"), m, domain_size, _stream()))
    return q, r


FR_ADD, FR_SUB, FR_MUL = 0, 1, 2


def fr_vec_op(a: torch.Tensor, b, op: int, out: torch.Tensor | None = None) -> torch.Tensor:
    """Elementwise a (op) b on Montgomery Fr vectors in HBM; b is a tensor of the same length or one 32-byte host scalar."""
    out = torch.empty_like(a) if out is None else out
    n = _nbytes(a) // 32
    with torch.cuda.device(a.device):
        if isinstance(b, torch.Tensor):
            if _nbytes(b) != _nbytes(a):
                raise ValueError("length mismatch")
            _lib.check(_lib.lib().snarkvm_b200_fr_vec_op_device(out.data_ptr(), _check(a, "a"), _check(b, "b"), n, op, _stream()))
        else:
            s = _fr_host(b)
            _lib.check(_lib.lib().snarkvm_b200_fr_vec_scalar_op_device(out.data_ptr(), _check(a, "a"), s.ctypes.data, n, op, _stream()))
    return out


def domain_elements(lg: int, device="cuda") -> torch.Tensor:
    """EvaluationDomain::elements (fft/domain.rs:307-309): [2^lg, 4] i64, element i = group_gen^i (Montgomery)."""
    out = torch.empty((1 << lg, 4), dtype=torch.int64, device=device)
    with torch.cuda.device(out.device):
        _lib.check(_lib.lib().snarkvm_b200_domain_elements_device(out.data_ptr(), lg, _stream()))
    return out


def sparse_matvec(row_ptr: torch.Tensor, cols: torch.Tensor, vals: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """z_M = M·x for a CSR matrix over Fr (inner_product per row, varuna/ahp/prover/round_functions/mod.rs:130-189).
    row_ptr: int32 [nrows + 1], cols: int32 [nnz], vals: [nnz, 4] i64 Montgomery, x: [nvars, 4] i64 Montgomery → [nrows, 4] i64."""
    if row_ptr.dtype != torch.int32 or cols.dtype != torch.int32:
        raise TypeError("row_ptr and cols must be int32 tensors")
    nrows = row_ptr.numel() - 1
    out = torch.empty((max(nrows, 0), 4), dtype=torch.int64, device=x.device)
    if nrows > 0:
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().snarkvm_b200_sparse_matvec_device(out.data_ptr(), _check(row_ptr, "row_ptr"),
                                                                     _check(cols, "cols") if cols.numel() else None,
                                                                     _check(vals, "vals") if vals.numel() else None, nrows, _check(x, "x"),
                                                                     _nbytes(x) // 32, _stream()))
    return out


def _csr_args(row_ptr: torch.Tensor, cols: torch.Tensor, vals: torch.Tensor):
    if row_ptr.dtype != torch.int32 or cols.dtype != torch.int32:
        raise TypeError("row_ptr and cols must be int32 tensors")
    nnz = cols.numel()
    if _nbytes(vals) != nnz * 32:
        raise ValueError("one 32-byte value per column index")
    return (_check(row_ptr, "row_ptr"), row_ptr.numel() - 1, _check(cols, "cols") if nnz else None, _check(vals, "vals") if nnz else None,
            nnz)


def varuna_matrix_evals(row_ptr: torch.Tensor, cols: torch.Tensor, vals: torch.Tensor, nvars: int, input_size: int, lg_constraint: int,
                        lg_variable: int, lg_non_zero: int):
    """matrix_evals (snark/varuna/ahp/matrices.rs:138-195) of a CSR matrix (row_ptr int32 [nrows + 1], cols int32 [nnz], vals [nnz, 4]
    i64 Montgomery) → (row, col, row_col_val), [2^lg_non_zero, 4] i64 Montgomery each, padded with (1, 1, 0).  A column ≥ nvars
    raises CudaError."""
    rp, nrows, cp, vp, nnz = _csr_args(row_ptr, cols, vals)
    K = 1 << lg_non_zero
    row, col, rcv = (torch.empty((K, 4), dtype=torch.int64, device=row_ptr.device) for _ in range(3))
    with torch.cuda.device(row_ptr.device):
        _lib.check(_lib.lib().snarkvm_b200_varuna_matrix_evals_device(row.data_ptr(), col.data_ptr(), rcv.data_ptr(), rp, nrows, cp, vp, nnz,
                                                                       nvars, input_size, lg_constraint, lg_variable, lg_non_zero, _stream()))
    return row, col, rcv


def csr_transpose(row_ptr: torch.Tensor, cols: torch.Tensor, vals: torch.Tensor, nvars: int, input_size: int, lg_variable: int):
    """transpose (snark/varuna/ahp/matrices.rs:249-270) over the variable domain → (t_row_ptr int32 [2^lg_variable + 1], t_cols int32
    [nnz] row indices, t_vals [nnz, 4] i64); entries inside a transposed row come in no fixed order.  A column ≥ nvars raises
    CudaError."""
    rp, nrows, cp, vp, nnz = _csr_args(row_ptr, cols, vals)
    dev = row_ptr.device
    t_row_ptr = torch.empty((1 << lg_variable) + 1, dtype=torch.int32, device=dev)
    t_cols = torch.empty(nnz, dtype=torch.int32, device=dev)
    t_vals = torch.empty((nnz, 4), dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().snarkvm_b200_csr_transpose_device(t_row_ptr.data_ptr(), t_cols.data_ptr() if nnz else None,
                                                                 t_vals.data_ptr() if nnz else None, rp, nrows, cp, vp, nnz, nvars,
                                                                 input_size, lg_variable, _stream()))
    return t_row_ptr, t_cols, t_vals


def csr_serialize(row_ptr: torch.Tensor, cols: torch.Tensor, vals: torch.Tensor) -> torch.Tensor:
    """The circuit id's byte stream of one CSR matrix (Circuit::hash, snark/varuna/ahp/indexer/circuit.rs:109-121):
    serialize_uncompressed of Vec<Vec<(Fr, usize)>> → CUDA uint8 tensor of 8 + 8·nrows + 40·nnz bytes.  A row_ptr that is not
    non-decreasing from 0 to nnz raises CudaError."""
    rp, nrows, cp, vp, nnz = _csr_args(row_ptr, cols, vals)
    nbytes = 8 + 8 * nrows + 40 * nnz
    out = torch.empty(nbytes // 8, dtype=torch.int64, device=row_ptr.device)          # int64 storage: 8-byte aligned
    with torch.cuda.device(row_ptr.device):
        _lib.check(_lib.lib().snarkvm_b200_csr_serialize_device(out.data_ptr(), nbytes, rp, nrows, cp, vp, nnz, _stream()))
    return out.view(torch.uint8)


LINCOMB_MAX_TERMS = 12


def fr_lincomb(polys: list, coeffs_mont: list) -> torch.Tensor:
    """Σ_j coeffs_j·polys_j in one pass over up to 12 Montgomery coefficient tensors of different lengths → CUDA tensor
    [max length, 4] i64, bit-identical to the `poly_axpy` sequence (sonic_pc.py)"""
    if len(polys) != len(coeffs_mont) or not polys:
        raise ValueError("one coefficient per polynomial, at least one polynomial")
    if len(polys) > LINCOMB_MAX_TERMS:
        raise ValueError(f"at most {LINCOMB_MAX_TERMS} polynomials")
    lens = [_nbytes(p) // 32 for p in polys]
    n = max(lens)
    dev = polys[0].device
    out = torch.empty((n, 4), dtype=torch.int64, device=dev)
    k = len(polys)
    ptrs = (ctypes.c_void_p * k)(*[(_check(p, "poly") if m else None) for p, m in zip(polys, lens)])
    szs = (ctypes.c_size_t * k)(*lens)
    cs = np.ascontiguousarray(np.stack([_fr_host(c) for c in coeffs_mont]))
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().snarkvm_b200_fr_lincomb_device(out.data_ptr() if n else None, n, ctypes.cast(ptrs, ctypes.c_void_p),
                                                              ctypes.cast(szs, ctypes.c_void_p), cs.ctypes.data, k, _stream()))
    return out


def matrix_evals_dot(row: torch.Tensor, col: torch.Tensor, row_col_val: torch.Tensor, lagrange: torch.Tensor) -> np.ndarray:
    """MatrixEvals::evaluate (snark/varuna/ahp/matrices.rs:114-126): Σ l·row, Σ l·col, Σ l·row·col, Σ l·row_col_val over K →
    uint64[4, 4] Montgomery on the host"""
    n = _nbytes(lagrange) // 32
    for t in (row, col, row_col_val):
        if _nbytes(t) != n * 32:
            raise ValueError("length mismatch")
    out = np.zeros((4, 4), dtype=np.uint64)
    with torch.cuda.device(lagrange.device):
        args = [_check(t, name) if n else None for t, name in ((row, "row"), (col, "col"), (row_col_val, "row_col_val"), (lagrange, "lagrange"))]
        _lib.check(_lib.lib().snarkvm_b200_matrix_evals_dot_device(out.ctypes.data, *args, n, _stream()))
    return out


def ntt_batch_(xs: list, direction: NTTDirection = NTTDirection.Forward, ntt_type: NTTType = NTTType.Standard) -> list:
    """ntt_ of every tensor in `xs` (2^lg_i Fr each, sizes may differ, all on one device) in place, transforms of equal size sharing
    their launches → xs"""
    if not xs:
        return xs
    lgs = []
    for x in xs:
        n = _nbytes(x) // 32
        if n <= 0 or n & (n - 1) or n * 32 != _nbytes(x):
            raise ValueError("domain_size is not power of 2")
        lgs.append(n.bit_length() - 1)
    dev = xs[0].device
    ptrs = (ctypes.c_void_p * len(xs))(*[_check(x, "x") for x in xs])
    lg_arr = (ctypes.c_uint32 * len(xs))(*lgs)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().snarkvm_b200_ntt_batch_device(ptrs, lg_arr, len(xs), int(direction), int(ntt_type), _stream()))
    return xs


def _check_segments(code: int, bad: ctypes.c_int64) -> None:
    if code != 0:
        err = _lib.CudaError(code, f"segment {bad.value}" if bad.value >= 0 else "see cudaError_t")
        err.segment = bad.value if bad.value >= 0 else None
        raise err


def _csr_segment(row_ptr: torch.Tensor, cols: torch.Tensor, vals: torch.Tensor, outs) -> "_lib.CsrSegment":
    rp, nrows, cp, vp, nnz = _csr_args(row_ptr, cols, vals)
    s = _lib.CsrSegment()
    s.d_row_ptr, s.d_cols, s.d_vals, s.nrows, s.nnz = rp, cp, vp, nrows, nnz
    for k, o in enumerate(outs):
        s.d_out[k] = o
    return s


def varuna_matrix_evals_batch(specs: list) -> list:
    """varuna_matrix_evals of every (row_ptr, cols, vals, nvars, input_size, lg_constraint, lg_variable, lg_non_zero) in `specs` in one
    launch and one synchronisation → [(row, col, row_col_val)], views of one buffer.  A bad matrix raises CudaError whose `segment`
    is the index of the first bad spec."""
    if not specs:
        return []
    dev = specs[0][0].device
    sizes = [1 << s[7] for s in specs]
    buf = torch.empty((3 * sum(sizes), 4), dtype=torch.int64, device=dev)
    segs = (_lib.CsrSegment * len(specs))()
    outs, off = [], 0
    for k, (spec, K) in enumerate(zip(specs, sizes)):
        row_ptr, cols, vals, nvars, input_size, lg_r, lg_c, lg_k = spec
        trio = (buf[off: off + K], buf[off + K: off + 2 * K], buf[off + 2 * K: off + 3 * K])
        off += 3 * K
        s = _csr_segment(row_ptr, cols, vals, [t.data_ptr() for t in trio])
        s.nvars, s.input_size, s.lg_constraint, s.lg_variable, s.lg_non_zero = nvars, input_size, lg_r, lg_c, lg_k
        segs[k] = s
        outs.append(trio)
    bad = ctypes.c_int64(-1)
    with torch.cuda.device(dev):
        _check_segments(_lib.lib().snarkvm_b200_varuna_matrix_evals_batch_device(segs, len(specs), ctypes.byref(bad), _stream()), bad)
    return outs


def csr_serialize_batch(mats: list) -> tuple:
    """csr_serialize of every (row_ptr, cols, vals) in `mats` in one launch and one synchronisation → (CUDA uint8 buffer, byte offsets
    [len(mats) + 1]): stream k is buffer[offsets[k]:offsets[k + 1]].  Errors as varuna_matrix_evals_batch."""
    if not mats:
        return torch.empty(0, dtype=torch.uint8), [0]
    dev = mats[0][0].device
    offsets = [0]
    for row_ptr, cols, _vals in mats:
        offsets.append(offsets[-1] + 8 + 8 * (row_ptr.numel() - 1) + 40 * cols.numel())
    buf = torch.empty(offsets[-1] // 8, dtype=torch.int64, device=dev)          # int64 storage: every stream 8-byte aligned
    segs = (_lib.CsrSegment * len(mats))()
    for k, m in enumerate(mats):
        segs[k] = _csr_segment(*m, [buf.data_ptr() + offsets[k]])
    bad = ctypes.c_int64(-1)
    with torch.cuda.device(dev):
        _check_segments(_lib.lib().snarkvm_b200_csr_serialize_batch_device(segs, len(mats), ctypes.byref(bad), _stream()), bad)
    return buf.view(torch.uint8), offsets


def fr_lincomb_batch(jobs: list) -> list:
    """fr_lincomb of every (polys, coeffs_mont) in `jobs` in one launch → one CUDA tensor per job, bit-identical to fr_lincomb"""
    if not jobs:
        return []
    dev = jobs[0][0][0].device
    segs = (_lib.LincombSegment * len(jobs))()
    outs = []
    for k, (polys, coeffs_mont) in enumerate(jobs):
        if len(polys) != len(coeffs_mont) or not polys:
            raise ValueError("one coefficient per polynomial, at least one polynomial")
        if len(polys) > LINCOMB_MAX_TERMS:
            raise ValueError(f"at most {LINCOMB_MAX_TERMS} polynomials")
        lens = [_nbytes(p) // 32 for p in polys]
        out = torch.empty((max(lens), 4), dtype=torch.int64, device=dev)
        s = segs[k]
        s.d_out, s.n, s.nterms = out.data_ptr() if out.numel() else None, out.shape[0], len(polys)
        for j, (p, m, c) in enumerate(zip(polys, lens, coeffs_mont)):
            s.d_polys[j] = _check(p, "poly") if m else None
            s.lens[j] = m
            ctypes.memmove(s.coeffs_mont[j], _fr_host(c).ctypes.data, 32)
        outs.append(out)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().snarkvm_b200_fr_lincomb_batch_device(segs, len(jobs), _stream()))
    return outs


def matrix_evals_at_points(jobs: list) -> np.ndarray:
    """For every (row, col, row_col_val, point_mont) in `jobs` (evaluations on a K of 2^k elements, the point a Montgomery Fr): the
    Lagrange coefficients of K at the point and matrix_evals_dot's four inner products with them, all in one pass → uint64[count, 4, 4]
    Montgomery on the host"""
    out = np.zeros((len(jobs), 4, 4), dtype=np.uint64)
    if not jobs:
        return out
    segs = (_lib.EvalsSegment * len(jobs))()
    for k, (row, col, rcv, point) in enumerate(jobs):
        n = _nbytes(row) // 32
        if _nbytes(col) != n * 32 or _nbytes(rcv) != n * 32:
            raise ValueError("length mismatch")
        s = segs[k]
        s.d_row, s.d_col, s.d_row_col_val, s.n = _check(row, "row"), _check(col, "col"), _check(rcv, "row_col_val"), n
        ctypes.memmove(s.point_mont, _fr_host(point).ctypes.data, 32)
    with torch.cuda.device(jobs[0][0].device):
        _lib.check(_lib.lib().snarkvm_b200_matrix_evals_at_points_device(out.ctypes.data, segs, len(jobs), _stream()))
    return out


def fr_lincomb_terms(jobs: list, outs: list | None = None) -> list:
    """Uncapped linear combinations in one launch: job k is (n, terms) with every term (poly, coeff_mont, offset, period, reps) or
    (poly, coeff_mont, offset) or (poly, coeff_mont): out_k (n Fr) = Σ coeff·poly placed at offset + i·period for i < reps (reps = 1
    by default).  Terms are contiguous CUDA views (a row slice of a polynomial is one).  `outs[k]`, when given, is the CUDA tensor that
    receives job k (n rows); otherwise each output is allocated → [out_k], bit-identical to the sequence of additions"""
    if not jobs:
        return []
    if outs is not None and len(outs) != len(jobs):
        raise ValueError("one output per job")
    nterms = sum(len(t) for _n, t in jobs)
    outputs = (_lib.LincombOutput * len(jobs))()
    terms = (_lib.LincombTerm * max(1, nterms))()
    dev, result, k = None, [], 0
    for j, (n, tlist) in enumerate(jobs):
        for t in tlist:
            poly, coeff = t[0], t[1]
            offset, period, reps = (tuple(t[2:]) + (0, 0, 1)[len(t) - 2:])[:3]
            m = _nbytes(poly) // 32
            dev = dev or poly.device
            s = terms[k]
            s.d_poly, s.len, s.offset, s.period, s.reps = _check(poly, "poly") if m else None, m, offset, period, reps
            ctypes.memmove(s.coeff_mont, _fr_host(coeff).ctypes.data, 32)
            k += 1
        out = outs[j] if outs is not None else None
        if out is None:
            out = torch.empty((n, 4), dtype=torch.int64, device=dev or "cuda")
        elif _nbytes(out) != n * 32:
            raise ValueError("an output must hold n Fr")
        outputs[j].d_out, outputs[j].n = _check(out, "out") if n else None, n
        outputs[j].first_term, outputs[j].nterms = k - len(tlist), len(tlist)
        result.append(out)
    with torch.cuda.device(result[0].device):
        _lib.check(_lib.lib().snarkvm_b200_fr_lincomb_terms_device(outputs, len(jobs), terms, nterms, _stream()))
    return result


def sparse_matvec_batch(jobs: list, outs: list | None = None) -> list:
    """sparse_matvec of every (row_ptr, cols, vals, x) in one pass (three launches, one synchronisation) → one CUDA tensor [nrows, 4]
    per job (or into `outs[k]`).  A bad column or row_ptr raises CudaError whose `segment` is the first bad job."""
    if not jobs:
        return []
    segs = (_lib.SpmvSegment * len(jobs))()
    result = []
    for k, (row_ptr, cols, vals, x) in enumerate(jobs):
        rp, nrows, cp, vp, nnz = _csr_args(row_ptr, cols, vals)
        out = outs[k] if outs is not None else torch.empty((max(nrows, 0), 4), dtype=torch.int64, device=x.device)
        if _nbytes(out) != nrows * 32:
            raise ValueError("an output must hold nrows Fr")
        s = segs[k]
        s.d_row_ptr, s.d_cols, s.d_vals, s.nrows, s.nnz = rp, cp, vp, nrows, nnz
        s.d_x, s.nvars, s.d_out = _check(x, "x"), _nbytes(x) // 32, _check(out, "out") if nrows else None
        result.append(out)
    bad = ctypes.c_int64(-1)
    with torch.cuda.device(jobs[0][3].device):
        _check_segments(_lib.lib().snarkvm_b200_sparse_matvec_batch_device(segs, len(jobs), ctypes.byref(bad), _stream()), bad)
    return result


def polymul_batch(pairs: list) -> list:
    """PolyMultiplier::multiply of every (a, b) in one pass (one load launch, the forward transforms through ntt_batch_, one pointwise
    launch, the inverse transforms) → one CUDA tensor [2^lg, 4] per pair, lg = log2 of next_pow2(len a + len b − 1), each equal to
    polymul(a, b); an empty operand gives an empty product"""
    outs = []
    jobs = (_lib.PolymulJob * max(1, len(pairs)))()
    count = 0
    for a, b in pairs:
        la, lb = _nbytes(a) // 32, _nbytes(b) // 32
        if la == 0 or lb == 0:
            outs.append(torch.zeros((0, 4), dtype=torch.int64, device=a.device))
            continue
        lg = (la + lb - 2).bit_length()
        out = torch.empty((1 << lg, 4), dtype=torch.int64, device=a.device)
        j = jobs[count]
        j.d_out, j.d_a, j.d_b, j.len_a, j.len_b, j.lg = out.data_ptr(), _check(a, "a"), _check(b, "b"), la, lb, lg
        outs.append(out)
        count += 1
    if count:
        with torch.cuda.device(pairs[0][0].device):
            _lib.check(_lib.lib().snarkvm_b200_polymul_batch_device(jobs, count, _stream()))
    return outs


def varuna_round4_evals(jobs: list, alpha_mont, beta_mont) -> list:
    """Varuna's fourth-round evaluations on K for every (row, col, row_col_val, v_rc_mont, rc_mont, f_scale_mont): three launches for all
    of them → [(a, b, f)], views of one buffer: a = v_rc·row_col_val, b = rc·(row − α)(col − β), f = f_scale·row_col_val /
    ((row − α)(col − β)), zero where the denominator is zero"""
    return varuna_round4_evals_batch([tuple(j) + (alpha_mont, beta_mont) for j in jobs])


def varuna_round4_evals_batch(jobs: list) -> list:
    """varuna_round4_evals with each job's own challenges, for many proofs in one pass: every (row, col, row_col_val, v_rc_mont, rc_mont,
    f_scale_mont, alpha_mont, beta_mont) in the same three launches → [(a, b, f)], views of one buffer"""
    if not jobs:
        return []
    dev = jobs[0][0].device
    sizes = [_nbytes(j[0]) // 32 for j in jobs]
    buf = torch.empty((3 * sum(sizes), 4), dtype=torch.int64, device=dev)
    segs = (_lib.Round4BatchSegment * len(jobs))()
    outs, off = [], 0
    for k, ((row, col, rcv, v_rc, rc, scale, alpha, beta), n) in enumerate(zip(jobs, sizes)):
        if _nbytes(col) != n * 32 or _nbytes(rcv) != n * 32:
            raise ValueError("length mismatch")
        trio = (buf[off: off + n], buf[off + n: off + 2 * n], buf[off + 2 * n: off + 3 * n])
        off += 3 * n
        s = segs[k]
        s.d_row, s.d_col, s.d_row_col_val, s.n = _check(row, "row"), _check(col, "col"), _check(rcv, "row_col_val"), n
        for name, v in (("v_rc_mont", v_rc), ("rc_mont", rc), ("f_scale_mont", scale), ("alpha_mont", alpha), ("beta_mont", beta)):
            ctypes.memmove(getattr(s, name), _fr_host(v).ctypes.data, 32)
        s.d_a, s.d_b, s.d_f = (t.data_ptr() for t in trio)
        outs.append(trio)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().snarkvm_b200_varuna_round4_evals_batch_device(segs, len(jobs), _stream()))
    return outs


def poly_divide_by_linear(p: torch.Tensor, point_mont) -> torch.Tensor:
    """Quotient of p / (x − point), the KZG witness polynomial (kzg10/mod.rs:220-241) → CUDA tensor [m − 1, 4] i64, not trimmed."""
    z = _fr_host(point_mont)
    m = _nbytes(p) // 32
    q = torch.empty((max(m - 1, 0), 4), dtype=torch.int64, device=p.device)
    if m > 1:
        with torch.cuda.device(p.device):
            _lib.check(_lib.lib().snarkvm_b200_poly_divide_by_linear_device(q.data_ptr(), _check(p, "p"), m, z.ctypes.data, _stream()))
    return q


def poly_evaluate(coeffs: torch.Tensor, point_mont) -> np.ndarray:
    """DensePolynomial::evaluate (fft/polynomial/dense.rs:98-114) → Montgomery Fr as uint64[4] on the host."""
    z = _fr_host(point_mont)
    out = np.zeros(4, dtype=np.uint64)
    m = _nbytes(coeffs) // 32
    with torch.cuda.device(coeffs.device):
        _lib.check(_lib.lib().snarkvm_b200_poly_evaluate_device(out.ctypes.data, _check(coeffs, "coeffs") if m else None, m, z.ctypes.data, _stream()))
    return out


def poly_divide_by_linear_batch(jobs: list) -> list:
    """poly_divide_by_linear of every (p, point_mont) in one pass of three launches → one CUDA tensor [m − 1, 4] per job (empty for m ≤ 1),
    each equal to poly_divide_by_linear(p, point_mont)"""
    if not jobs:
        return []
    segs = (_lib.PolyDivideSegment * len(jobs))()
    outs = []
    for k, (p, point) in enumerate(jobs):
        m = _nbytes(p) // 32
        q = torch.empty((max(m - 1, 0), 4), dtype=torch.int64, device=p.device)
        s = segs[k]
        s.d_q, s.d_p, s.m = (q.data_ptr(), _check(p, "p"), m) if m > 1 else (None, None, m)
        ctypes.memmove(s.point_mont, _fr_host(point).ctypes.data, 32)
        outs.append(q)
    with torch.cuda.device(jobs[0][0].device):
        _lib.check(_lib.lib().snarkvm_b200_poly_divide_by_linear_batch_device(segs, len(jobs), _stream()))
    return outs


def poly_evaluate_batch(jobs: list) -> np.ndarray:
    """poly_evaluate of every (coeffs, point_mont) in one pass and one synchronisation → Montgomery Fr uint64[count, 4] on the host, row
    k equal to poly_evaluate of job k (zero for an empty polynomial)"""
    out = np.zeros((len(jobs), 4), dtype=np.uint64)
    if not jobs:
        return out
    segs = (_lib.PolyEvalSegment * len(jobs))()
    for k, (c, point) in enumerate(jobs):
        m = _nbytes(c) // 32
        segs[k].d_coeffs, segs[k].m = (_check(c, "coeffs") if m else None), m
        ctypes.memmove(segs[k].point_mont, _fr_host(point).ctypes.data, 32)
    with torch.cuda.device(jobs[0][0].device):
        _lib.check(_lib.lib().snarkvm_b200_poly_evaluate_batch_device(out.ctypes.data, segs, len(jobs), _stream()))
    return out


class PrecomputedBases:
    """A fixed base set with its tables 2^{c·w}·P_i resident in HBM (snarkvm_b200_msm_precompute_device): MSMs over it use one
    bucket set for all windows.  `msm(scalars)` / `kzg_commit(coeffs_mont)` take the first len(scalars) bases, like
    `&powers_of_beta_g[..len]` in KZG10::commit (kzg10/mod.rs:121-135)."""

    def __init__(self, bases: torch.Tensor, stride: int = AFFINE_STRIDE):
        npoints = _nbytes(bases) // stride
        self.device = bases.device
        h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().snarkvm_b200_msm_precompute_device(ctypes.byref(h), _check(bases, "bases"), npoints, stride, _stream()))
        self._h = h
        n, c, nwin, tb = ctypes.c_size_t(), ctypes.c_int(), ctypes.c_int(), ctypes.c_size_t()
        _lib.check(_lib.lib().snarkvm_b200_msm_precomputed_info(h, ctypes.byref(n), ctypes.byref(c), ctypes.byref(nwin), ctypes.byref(tb)))
        self.npoints, self.c, self.nwin, self.table_bytes = n.value, c.value, nwin.value, tb.value

    def _run(self, fn, scalars: torch.Tensor) -> np.ndarray:
        if self._h is None:
            raise ValueError("PrecomputedBases was freed")
        n = _nbytes(scalars) // 32
        if n > self.npoints:
            raise ValueError("more scalars than bases")
        out = np.zeros(18, dtype=np.uint64)
        with torch.cuda.device(self.device):
            _lib.check(fn(out.ctypes.data, self._h, _check(scalars, "scalars") if n else None, n, _stream()))
        return out

    def msm(self, scalars: torch.Tensor) -> np.ndarray:
        return self._run(_lib.lib().snarkvm_b200_msm_precomputed_device, scalars)

    def kzg_commit(self, coeffs_mont: torch.Tensor) -> np.ndarray:
        return self._run(_lib.lib().snarkvm_b200_kzg_commit_precomputed_device, coeffs_mont)

    def kzg_commit_batch(self, polys_mont: list) -> np.ndarray:
        """all commitments of a round over the tables, one pass → [count, 18] u64"""
        if self._h is None:
            raise ValueError("PrecomputedBases was freed")
        count = len(polys_mont)
        out = np.zeros((count, 18), dtype=np.uint64)
        if count == 0:
            return out
        lens = [_nbytes(p) // 32 for p in polys_mont]
        if max(lens) > self.npoints:
            raise ValueError("more coefficients than bases")
        ptrs = (ctypes.c_void_p * count)(*[(_check(p, "poly") if n else None) for p, n in zip(polys_mont, lens)])
        szs = (ctypes.c_size_t * count)(*lens)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().snarkvm_b200_kzg_commit_batch_precomputed_device(out.ctypes.data, self._h, ptrs, szs, count, _stream()))
        return out

    def free(self) -> None:
        if self._h is not None:
            _lib.check(_lib.lib().snarkvm_b200_msm_precomputed_free(self._h))
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def fr_from_mont(x: torch.Tensor) -> torch.Tensor:
    out = torch.empty_like(x)
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().snarkvm_b200_fr_from_mont_device(out.data_ptr(), _check(x, "x"), _nbytes(x) // 32, _stream()))
    return out


def fr_to_mont(x: torch.Tensor) -> torch.Tensor:
    out = torch.empty_like(x)
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().snarkvm_b200_fr_to_mont_device(out.data_ptr(), _check(x, "x"), _nbytes(x) // 32, _stream()))
    return out


def generate_bases(npoints: int, seed: int, device="cuda", stride: int = AFFINE_STRIDE) -> torch.Tensor:
    """Synthetic G1 bases P_i = h(seed, i)·G in the reference affine layout, generated in HBM."""
    t = torch.empty((npoints, stride), dtype=torch.uint8, device=device)
    with torch.cuda.device(t.device):
        _lib.check(_lib.lib().snarkvm_b200_generate_bases_device(t.data_ptr(), npoints, stride, seed & (2**64 - 1), _stream()))
    return t


def srs_decode(usrs_points: torch.Tensor, stride: int = AFFINE_STRIDE):
    """`.usrs` payload in HBM (uint8, 96 B per uncompressed canonical point, count header already stripped) →
    (bases in the reference affine layout, number of invalid points).  parameters/src/mainnet/powers.rs."""
    nbytes = _nbytes(usrs_points)
    if nbytes % 96:
        raise ValueError("payload must be a whole number of 96-byte points")
    n = nbytes // 96
    out = torch.empty((n, stride), dtype=torch.uint8, device=usrs_points.device)
    invalid = torch.zeros(1, dtype=torch.int32, device=usrs_points.device)
    with torch.cuda.device(usrs_points.device):
        _lib.check(_lib.lib().snarkvm_b200_srs_decode_device(out.data_ptr(), stride, _check(usrs_points, "usrs_points"), n,
                                                              invalid.data_ptr(), _stream()))
    return out, int(invalid.item())
