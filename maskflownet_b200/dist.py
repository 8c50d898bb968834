"""Data-parallel plumbing for the hot path: one process per GPU, batch sharded along N, no data-path collective in the
forward (replicas), and ONE flattened fp32 gradient all-reduce per training step.

Mirrors what the reference does implicitly with gluon: `split_and_load` over ctx (network/pipeline.py:95,173,206) and
`trainer.step(batch_size)` (:114), whose kvstore('device') sums each parameter's gradient across GPUs and rescales by
1/batch_size.  Here: torch.distributed (NCCL over NVLink on the GPU box, gloo in CPU tests) on a single bucket
(MaskFlownet-S: 10,514,256 floats = 42 MB), small enough for one all-reduce per step -- so it is
neither fused into a kernel nor split into per-layer buckets (SURVEY.md section 5).
"""
from __future__ import annotations

import os
from typing import Iterable, List, Sequence, Tuple

import torch
import torch.distributed as dist


def init_from_env(backend: str | None = None) -> Tuple[int, int, int]:
    """Initialise torch.distributed from torchrun's env (RANK / LOCAL_RANK / WORLD_SIZE / MASTER_*).
    Returns (rank, local_rank, world_size); world_size == 1 without the env means single-process."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local)
        dist.init_process_group(backend=backend, rank=rank, world_size=world)
    return rank, local, world


def shard_batch(n_total: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous batch shard [begin, end) of this rank; like the reference, the batch must divide evenly
    (`assert batch_size % len(ctx) == 0`, main.py:371)."""
    if n_total % world:
        raise ValueError(f"batch {n_total} is not divisible by {world} devices")
    per = n_total // world
    return rank * per, (rank + 1) * per


class GradBucket:
    """Flat fp32 view over the gradients of `params` for a single all-reduce per step."""

    def __init__(self, params: Iterable[torch.nn.Parameter]):
        self.params: List[torch.nn.Parameter] = [p for p in params if p.requires_grad]
        if not self.params:
            raise ValueError("no trainable parameters")
        dev = self.params[0].device
        if any(p.device != dev or p.dtype != torch.float32 for p in self.params):
            raise ValueError("GradBucket: all parameters must be float32 on one device")
        self.numel = sum(p.numel() for p in self.params)
        self.flat = torch.zeros(self.numel, dtype=torch.float32, device=dev)
        off = 0
        for p in self.params:  # gradients become views into the bucket: no pack/unpack copies
            p.grad = self.flat[off:off + p.numel()].view_as(p)
            off += p.numel()

        self._views = [p.grad for p in self.params]

    def zero_(self):
        """The ONLY supported way to clear the gradients: `optimizer.zero_grad()` / `model.zero_grad()` default to
        set_to_none=True, which would drop the views into the bucket."""
        self.flat.zero_()

    def rebind_(self):
        """Re-attach the gradient views (after an accidental zero_grad(set_to_none=True)); gradients accumulated into
        detached tensors in the meantime are copied into the bucket."""
        for p, v in zip(self.params, self._views):
            if p.grad is None:
                p.grad = v
            elif p.grad.data_ptr() != v.data_ptr():
                v.copy_(p.grad)
                p.grad = v

    def _check_aliasing(self):
        for p, v in zip(self.params, self._views):
            if p.grad is None or p.grad.data_ptr() != v.data_ptr():
                raise RuntimeError("GradBucket: a parameter's .grad no longer aliases the bucket (zero_grad(set_to_none=True)?); "
                                   "use bucket.zero_() to clear gradients, or bucket.rebind_() to re-attach")

    class _Handle:
        """async all-reduce in flight: wait() completes it AND applies the 1/global_batch scale."""

        def __init__(self, work, flat, scale):
            self.work, self.flat, self.scale = work, flat, scale

        def wait(self):
            if self.work is not None:
                self.work.wait()
                self.work = None
                self.flat.mul_(self.scale)

    def allreduce_(self, global_batch: int, async_op: bool = False):
        """Sum over ranks, then scale by 1/global_batch (MXNet Trainer.step(batch_size) semantics: per-sample losses are
        summed, the optimizer rescales by 1/batch_size).  async_op=True returns a handle whose wait() finishes the
        reduction and applies the scale."""
        self._check_aliasing()
        scale = 1.0 / float(global_batch)
        if dist.is_initialized() and dist.get_world_size() > 1:
            work = dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, async_op=async_op)
            if async_op:
                return GradBucket._Handle(work, self.flat, scale)
        self.flat.mul_(scale)
        return None


def max_over_ranks(value: float, device) -> float:
    """max over ranks of a scalar (device-timed milliseconds in bench.py)."""
    if not (dist.is_initialized() and dist.get_world_size() > 1):
        return float(value)
    t = torch.tensor([value], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())
