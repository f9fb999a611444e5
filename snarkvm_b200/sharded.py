"""Multi-GPU MSM: shard (bases, scalars) by contiguous point ranges, one process per GPU.

Replaces the reference's multi-GPU split (algorithms/cuda/cuda/snarkvm.cu:254-295: even split over
ngpus(), partial Jacobian points copied to the host and added there with point_t::dadd).  Here each
rank leaves its per-window XYZZ sums in HBM, the only exchange is one all-gather of nwin × 192 B per
rank over NCCL/NVLink, a device kernel adds the ranks window by window, and the ≤ 24 window sums are
folded on the host (Horner).  MSM is a sum, so no other collective exists on the path.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.distributed as dist

from . import device


def shard_range(npoints: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous ⌈n/G⌉ split, the reference's own (snarkvm.cu:254-269)."""
    per = (npoints + world - 1) // world
    lo = min(npoints, rank * per)
    return lo, min(npoints, lo + per)


def combine_partials_host(partials: np.ndarray) -> np.ndarray:
    """Σ of per-rank partial results given as XYZZ points [world, 192 B] on the host."""
    return device.msm_finish(partials, 0)


class PendingMsm:
    """A sharded MSM whose device work (shard MSM → all-gather → rank sum → D2H of the window sums) has been enqueued;
    `result()` waits for it and folds the ≤ 24 window sums on the host.  Issuing several before collecting any keeps the
    GPUs busy back to back instead of idling every step behind a blocking read."""

    def __init__(self, host_sums, host_flags, event, c):
        self._sums, self._flags, self._event, self._c = host_sums, host_flags, event, c

    def result(self) -> np.ndarray:
        self._event.synchronize()
        if bool((self._flags != 0).any()):
            from ._lib import CudaError
            raise CudaError(1, "a scalar has bits 253..255 set (not a canonical Fr)")
        return device.msm_finish(self._sums.numpy(), self._c)


def msm_sharded_async(bases_shard, scalars_shard, group=None, stride: int = device.AFFINE_STRIDE,
                      plan_npoints: int | None = None, dev=None) -> PendingMsm:
    """Every rank passes ITS shard (any length, also empty — `shard_range` gives ⌈n/G⌉ splits whose last shards are shorter).
    All ranks run under the window plan of the LARGEST shard — pass it as `plan_npoints` when known, else it is found with one
    all-reduce(MAX) (a host round trip) — so the gathered window sums share one radix; an empty shard contributes infinity.
    CUDA tensors are used where they are; numpy arrays (HOST buffers: uint8 [n, stride] points, uint64 [n, 4] scalars) are
    uploaded by the library with the upload overlapped with the shard's kernels.  Pinned numpy inputs are read by DMA after
    this call returns, so the caller keeps them unchanged until `result()`; pageable ones may be reused at once."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    host = isinstance(scalars_shard, np.ndarray)
    if host:
        npoints = scalars_shard.shape[0]
        dev = torch.device("cuda", torch.cuda.current_device()) if dev is None else torch.device(dev)
    else:
        npoints = (scalars_shard.numel() * scalars_shard.element_size()) // 32
        dev = scalars_shard.device
    plan_n = plan_npoints
    if plan_n is None:
        plan_n = npoints
        if world > 1:
            t = torch.tensor([npoints], dtype=torch.int64, device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
            plan_n = int(t.item())
    if plan_n == 0:
        ev = torch.cuda.Event(); ev.record()
        return PendingMsm(torch.zeros((1, device.XYZZ_BYTES), dtype=torch.uint8), torch.zeros(1, dtype=torch.int32), ev, 0)
    plan = device.msm_plan(plan_n)
    nwin = plan["nwin"]
    # record layout: nwin window sums + one 192-byte record whose first word is the overflow flag
    mine = torch.zeros((nwin + 1, device.XYZZ_BYTES // 8), dtype=torch.int64, device=dev)
    flags = mine[nwin].view(torch.int32)[:1]
    if host:
        device.msm_window_sums_host(mine[:nwin], flags, plan_n, bases_shard, scalars_shard, stride)
    else:
        device.msm_window_sums(bases_shard, scalars_shard, stride, plan_npoints=plan_n, flags=flags, out=mine[:nwin])
    with torch.cuda.device(dev):
        if world > 1:
            gathered = torch.empty((world,) + tuple(mine.shape), dtype=mine.dtype, device=dev)
            dist.all_gather_into_tensor(gathered, mine, group=group)
            sums = device.xyzz_sum_ranks(gathered[:, :nwin].contiguous(), world, nwin)
            fl = gathered[:, nwin, 0].to(torch.int32)
        else:
            sums, fl = mine[:nwin], flags
        h_sums = torch.empty(sums.shape, dtype=sums.dtype, pin_memory=True)
        h_flags = torch.empty(fl.shape, dtype=fl.dtype, pin_memory=True)
        h_sums.copy_(sums, non_blocking=True)
        h_flags.copy_(fl, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
    return PendingMsm(h_sums, h_flags, ev, plan["c"])


def msm_sharded(bases_shard, scalars_shard, group=None, stride: int = device.AFFINE_STRIDE,
                plan_npoints: int | None = None) -> np.ndarray:
    """msm_sharded_async(...).result(): every rank returns the full sum."""
    return msm_sharded_async(bases_shard, scalars_shard, group, stride, plan_npoints).result()
