"""View-sharded data parallelism (SURVEY.md §8e): one process per GPU, Gaussians
replicated, camera views sharded, ONE all-reduce of a flat gradient bucket per step.

The reference is single-process/single-GPU (no collective anywhere); this is the only
cross-GPU exchange the path needs.  `GradBucket` is backend-agnostic (NCCL on GPUs,
gloo in the CPU tests).  `SymmetricGradBucket` is the NVLink-native version: the fused backward
writes its gradients straight into a symmetric-memory bucket and one kernel of ours
(csrc/collective.cu: NVSwitch multimem reduction, or peer loads/stores) sums it in place;
`make_grad_bucket` picks it when the process group supports it, else `GradBucket`.
"""
from __future__ import annotations

import os
from typing import Iterable, List, Sequence

import torch
import torch.distributed as dist
from torch._utils import _flatten_dense_tensors, _unflatten_dense_tensors


def view_for_rank(step: int, rank: int, world: int, n_views: int) -> int:
    """Round-robin: at step s rank r renders view (s*world + r) mod n_views, so a step covers
    `world` distinct consecutive views and an epoch covers all of them."""
    return (step * world + rank) % n_views


def shard_views(n_views: int, rank: int, world: int) -> List[int]:
    """Static partition used by render-only sweeps (C5): views rank, rank+world, ..."""
    return list(range(rank, n_views, world))


class GradBucket:
    """Flat fp32 bucket over the gradients of `params` (order fixed at construction).
    `allreduce()` sums (or averages) the bucket across ranks with a single collective and
    scatters the result back into each `.grad` in place."""

    def __init__(self, params: Sequence[torch.Tensor], average: bool = False, group=None):
        self.params = list(params)
        self.average = average
        self.group = group

    def nbytes(self) -> int:
        return sum(p.numel() for p in self.params) * 4

    def allreduce(self, async_op: bool = False):
        if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(self.group) == 1:
            return None
        grads = [p.grad if p.grad is not None else torch.zeros_like(p) for p in self.params]
        flat = _as_one_buffer(grads)          # zero-copy when the grads are views of one flat buffer
        in_place = flat is not None
        if not in_place:
            flat = _flatten_dense_tensors(grads)
        work = dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=self.group, async_op=async_op)

        def finish():
            if self.average:
                flat.div_(dist.get_world_size(self.group))
            if in_place:
                return
            for p, g, f in zip(self.params, grads, _unflatten_dense_tensors(flat, grads)):
                if p.grad is None:
                    p.grad = f.clone()
                else:
                    g.copy_(f)

        if async_op:
            return work, finish
        finish()
        return None


class SymmetricGradBucket:
    """Gradient exchange fused with the backward's output buffer, over NVLink peer memory.

    The flat bucket the fused backward writes (renderer._flat_grads) is ONE persistent
    symmetric-memory allocation mapped into every rank; `allreduce()` is
    barrier -> one exchange kernel (csrc/collective.cu) -> barrier, stream-ordered on the current
    stream, in place, no staging copies and no NCCL kernel.  Rank r owns slice r of the bucket:

      mode "multimem": `multimem.ld_reduce` sums the W copies of the slice inside the NVSwitch and
                       `multimem.st` multicasts the sum back (NVLink SHARP); moves (1 + 1/W) bucket
                       sizes per direction - the least for W >= 4.
      mode "p2p":      system-scope loads of the slice from every peer, stores of the sum to every
                       peer; moves 2 (W-1)/W bucket sizes per direction - the least for W = 2.
      mode "push":     the exchange starts INSIDE the backward: `fused_project_bwd_kernel` stores every
                       gradient float that belongs to another rank's slice straight into that owner's
                       staging slot over NVLink (gs_grad_push), so the reduce half overlaps the
                       kernel; after the barrier the owner sums its slice with W-1 local staging
                       slots and stores the sum to every bucket (gs_allreduce_push_finish_f32).
                       (W-1)/W bucket sizes per direction hidden under the backward + the same
                       again exposed.  The bucket is only complete after `allreduce()`.
      mode "auto":     push (W = 2, 4, 8; GS_DP_PUSH_MC=1 sends its broadcast half through the NVSwitch with
                       multimem.st), else multimem / p2p.

    The exchange timings of these modes have not been measured on H100; `tests/test_exchange_gpu.py`
    checks every mode against NCCL on 2 GPUs.

    `allocator` must be installed with `renderer.set_flat_grad_allocator` (make_grad_bucket does
    it).  A change of the bucket size (densification changes N on every rank at the same step)
    re-allocates and re-rendezvouses collectively.
    """

    def __init__(self, params: Sequence[torch.Tensor], average: bool = False, group=None, mode: str = "auto"):
        import gaussian
        import torch.distributed._symmetric_memory as symm_mem
        self._gaussian, self._symm = gaussian, symm_mem
        self.params = list(params)
        self.average = average
        self.group = group if group is not None else dist.group.WORLD
        self.world = dist.get_world_size(self.group)
        self.rank = dist.get_rank(self.group)
        assert mode in ("auto", "multimem", "p2p", "push")
        self.mode = mode
        self.buf = None
        self.hdl = None
        self.staging = None
        self.staging_hdl = None
        self.per = 0
        self._probe()

    def _alloc(self, numel, device):
        buf = self._symm.empty(numel, dtype=torch.float32, device=device)
        hdl = self._symm.rendezvous(buf, group=self.group.group_name)
        return buf, hdl

    def _probe(self):
        """Resolve the mode and check the sum on a tiny buffer; raises at construction (so that
        the caller can fall back to NCCL) when the group cannot do it."""
        dev = self.params[0].device
        buf, hdl = self._alloc(1024, dev)
        has_mc = bool(getattr(hdl, "multicast_ptr", 0))
        p2p_ok = self.world in (2, 4, 8)
        push = self.mode == "push"
        if push:
            self.mode = "p2p"                  # the self-check below runs the plain p2p kernel
        if self.mode == "auto":
            push = p2p_ok
            self.mode = "p2p" if (p2p_ok or not has_mc) else "multimem"
        # broadcast half of the pushed exchange: plain peer stores by default; GS_DP_PUSH_MC=1 sends it through
        # the NVSwitch instead (one multimem.st per 16 bytes: each GPU sends its slice once, but the switch also
        # loops the slice back to its owner); the simpler peer stores are the default
        self.push_mc = has_mc and os.environ.get("GS_DP_PUSH_MC") == "1"
        if self.mode == "multimem" and not has_mc:
            raise RuntimeError("symmetric memory has no multicast mapping (NVLS unavailable)")
        if self.mode == "p2p" and not p2p_ok:
            raise RuntimeError("p2p exchange supports 2, 4 or 8 ranks")
        buf.fill_(float(self.rank + 1))
        self._reduce(buf, hdl, 1024)
        want = self.world * (self.world + 1) / 2
        if not bool((buf == want).all()):
            raise RuntimeError("peer-memory all-reduce self-check failed")
        if push:
            self.mode = "push"

    def _reduce(self, buf, hdl, numel):
        hdl.barrier(channel=0)                  # every rank's bucket is written (push: and every pushed slice)
        if self.mode == "push":
            if self.push_mc:
                self._gaussian.allreduce_push_finish_mc(int(hdl.multicast_ptr), int(buf.data_ptr()),
                                                        int(self.staging.data_ptr()), int(numel), int(self.per),
                                                        self.rank, self.world, buf.device.index)
            else:
                self._gaussian.allreduce_push_finish([int(p) for p in hdl.buffer_ptrs], int(self.staging.data_ptr()),
                                                     int(numel), int(self.per), self.rank, self.world,
                                                     buf.device.index)
        elif self.mode == "multimem":
            self._gaussian.allreduce_multimem(int(hdl.multicast_ptr), int(numel), self.rank, self.world,
                                              buf.device.index)
        else:
            self._gaussian.allreduce_p2p([int(p) for p in hdl.buffer_ptrs], int(numel), self.rank, self.world,
                                         buf.device.index)
        hdl.barrier(channel=1)                  # every slice has reached every rank

    def allocator(self, numel: int, device) -> torch.Tensor:
        numel = (numel + 3) // 4 * 4
        # The bucket is ONE persistent buffer and `.grad` tensors are views of it: a second backward
        # while a `.grad` still aliases it would overwrite that gradient and autograd would then add
        # the buffer to itself (silently 2 x the last gradient).  Gradient accumulation therefore
        # needs zero_grad(set_to_none=True) between backwards - refuse anything else.
        if self.buf is not None:
            lo, hi = self.buf.data_ptr(), self.buf.data_ptr() + self.buf.numel() * 4
            for p in self.params:
                if p.grad is not None and lo <= p.grad.data_ptr() < hi:
                    raise RuntimeError("SymmetricGradBucket: a parameter's .grad still aliases the symmetric bucket "
                                       "while a new backward wants to write it; clear gradients with "
                                       "zero_grad(set_to_none=True) / p.grad = None before every backward "
                                       "(gradient accumulation over several backwards is not supported in this mode)")
        if self.buf is None or self.buf.numel() != numel or self.buf.device != device:
            self.buf, self.hdl = self._alloc(numel, device)
            if self.mode == "push":
                self.per = (numel // 4 + self.world - 1) // self.world * 4
                self.staging, self.staging_hdl = self._alloc(self.world * self.per, device)
                self.staging.zero_()                    # pad floats are never pushed: keep them finite
                self.hdl.barrier(channel=0)             # nobody pushes into a buffer that is still being zeroed
        if self.mode == "push":
            return self.buf, (int(self.buf.data_ptr()), [int(p) for p in self.staging_hdl.buffer_ptrs], int(self.per),
                              self.rank)
        return self.buf

    def nbytes(self) -> int:
        return sum(p.numel() for p in self.params) * 4

    def allreduce(self, async_op: bool = False):
        assert not async_op, "the peer-memory exchange is stream-ordered; there is nothing to wait on"
        grads = [p.grad for p in self.params]
        flat = None if any(g is None for g in grads) else _as_one_buffer(grads)
        if (flat is None or self.buf is None or flat.data_ptr() != self.buf.data_ptr()
                or flat.numel() > self.buf.numel()):
            raise RuntimeError("gradients are not views of the symmetric bucket "
                               "(install SymmetricGradBucket.allocator with renderer.set_flat_grad_allocator "
                               "and clear .grad with set_to_none=True)")
        self._reduce(self.buf, self.hdl, self.buf.numel())
        if self.average:
            flat.div_(self.world)
        return None


def make_grad_bucket(params: Sequence[torch.Tensor], average: bool = False, group=None, exchange: str = "auto"):
    """The gradient exchange for `params`: `exchange` (env GS_DP_EXCHANGE overrides) is
    "nccl" (portable `GradBucket`), "multimem" / "p2p" / "push" (required `SymmetricGradBucket` mode) or
    "auto": a push-mode `SymmetricGradBucket` (installed as the backward's bucket allocator) when
    the group is NCCL with 2, 4 or 8 ranks on CUDA and symmetric memory works (each validated against
    NCCL's sum by tests/test_exchange_gpu.py and, on every multi-GPU bench run, by bench.py's
    `exchange_check`) - else `GradBucket`."""
    import os
    import sys
    exchange = os.environ.get("GS_DP_EXCHANGE", exchange)
    assert exchange in ("auto", "nccl", "multimem", "p2p", "push"), exchange
    params = list(params)
    usable = (dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1
              and len(params) > 0 and params[0].is_cuda and dist.get_backend(group) == "nccl")
    if exchange == "auto" and usable and dist.get_world_size(group) not in (2, 4, 8):
        exchange = "nccl"
    if exchange != "nccl" and usable:
        try:
            import renderer
            bucket = SymmetricGradBucket(params, average=average, group=group, mode=exchange)
            renderer.set_flat_grad_allocator(bucket.allocator)
            return bucket
        except Exception as e:          # setup-time only: every rank fails or succeeds together
            if exchange != "auto":
                raise
            print(f"[dp] peer-memory gradient exchange unavailable ({e}); using NCCL all-reduce", file=sys.stderr)
    elif exchange in ("multimem", "p2p", "push") and dist.is_initialized() and dist.get_world_size(group) > 1:
        raise RuntimeError("peer-memory gradient exchange needs an initialised NCCL group on CUDA")
    return GradBucket(params, average=average, group=group)


def _as_one_buffer(grads):
    """If the gradient tensors are contiguous views laid out in order in ONE storage with at most
    3 pad elements between them (the fused backward allocates them that way,
    renderer._RenderFrame.backward), return the flat 1-D view spanning them so the collective
    runs in place; else None."""
    try:
        g0 = grads[0]
        base = g0.untyped_storage().data_ptr()
        off = g0.storage_offset()
        end = off
        for g in grads:
            gap = g.storage_offset() - end
            if (g.dtype != g0.dtype or not g.is_contiguous() or g.untyped_storage().data_ptr() != base
                    or gap < 0 or gap > 3):
                return None
            end = g.storage_offset() + g.numel()
        return torch.empty(0, dtype=g0.dtype, device=g0.device).set_(g0.untyped_storage(), off, (end - off,))
    except Exception:
        return None


def allreduce_stats(tensors: Iterable[torch.Tensor], group=None):
    """Densification statistics that are per-view in the reference (train.py:148-150:
    |grad_pos| accumulation and culling_mask counts) must be summed over ranks so that every
    replica takes the same clone/split/prune decisions."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return
    for t in tensors:
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)


def all_reduce_visible(mask: torch.Tensor, group=None) -> torch.Tensor:
    """Union over the ranks of the visibility masks (`Splatter.visible_mask()`, uint8 [n]) for a visible-only
    optimizer step (`FlatAdam.step(visible=...)`), in place.  The gradients are summed over the ranks, so the rows to
    update are those any rank saw, and the replicas stay bit-identical only if every rank steps the same rows.
    n bytes per step."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(mask, op=dist.ReduceOp.MAX, group=group)
    return mask
