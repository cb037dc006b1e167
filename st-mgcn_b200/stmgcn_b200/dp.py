"""Batch-sharded data parallelism: one process per GPU, one gradient all-reduce per step.

The reference has no multi-device path (``Main.py:22-23`` picks one device).  Every window of a batch is
independent (no cross-sample op anywhere in ``STMGCN.py``), supports and the ~1.2 MB of weights are
replicated, so the only exchange is the sum of the parameter gradients: ONE ``all_reduce`` over ONE flat
fp32 bucket (302 777 floats at K=3, T=12) on the compute stream, then a scale by ``1/world`` -- with equal
shards and ``MSELoss(reduction='mean')`` this reproduces the single-GPU gradient (SURVEY.md section 8(e)).
At this size the collective is latency-bound; bucketing/overlap would only add launches.
"""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.distributed as dist


class GradBucket:
    """All parameter gradients of one or more modules as views into one flat contiguous buffer: ``GradBucket(model)``,
    or ``GradBucket(model, *adjacencies)`` to reduce learnable graphs (``LearnableAdjacency``, held outside the model so
    its ``state_dict`` keys stay the reference's) in the same single collective.  A parameter shared by two modules is
    taken once."""

    def __init__(self, module: torch.nn.Module, *more: torch.nn.Module):
        self.params, seen = [], set()
        for mod in (module,) + more:
            for p in mod.parameters():
                if p.requires_grad and id(p) not in seen:
                    seen.add(id(p))
                    self.params.append(p)
        kinds = {(p.dtype, p.device) for p in self.params}
        if len(kinds) > 1:
            raise ValueError(f"GradBucket: the parameters must share one dtype and device, got {sorted(map(str, kinds))}")
        total = sum(p.numel() for p in self.params)
        ref = self.params[0]
        self.flat = torch.zeros(total, dtype=ref.dtype, device=ref.device)
        off = 0
        for p in self.params:
            p.grad = self.flat[off:off + p.numel()].view_as(p)      # autograd accumulates in place
            off += p.numel()

        self._offsets = []
        off = 0
        for p in self.params:
            self._offsets.append(off)
            off += p.numel()

    def zero_(self) -> None:
        self.flat.zero_()

    def rebind_(self) -> int:
        """Make sure every ``p.grad`` still IS its view into the flat buffer.  ``optimizer.zero_grad()`` defaults to
        ``set_to_none=True`` (and so does ``Model_Trainer.py:40``'s call): it drops the views, autograd then allocates fresh
        ``.grad`` tensors and an all-reduce of the flat buffer would silently average zeros.  Gradients found outside the
        buffer are copied in and re-aliased.  Returns the number of parameters that had to be re-bound."""
        fixed = 0
        base = self.flat.data_ptr()
        esz = self.flat.element_size()
        for p, off in zip(self.params, self._offsets):
            view = self.flat[off:off + p.numel()].view_as(p)
            g = p.grad
            if g is None:
                view.zero_()
                p.grad = view
                fixed += 1
            elif g.data_ptr() != base + off * esz or not g.is_contiguous():
                view.copy_(g)
                p.grad = view
                fixed += 1
        return fixed

    def all_reduce_mean_(self, group=None) -> None:
        """ONE collective over the flat bucket.  NCCL averages inside the collective (``ReduceOp.AVG``): the step has a
        single post-backward kernel; gloo (CPU tests) has no AVG, so SUM + scale."""
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
            self.rebind_()
            if dist.get_backend(group) == "nccl":
                dist.all_reduce(self.flat, op=dist.ReduceOp.AVG, group=group)
            else:
                dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=group)
                self.flat.mul_(1.0 / dist.get_world_size(group))


def init_from_env(backend: Optional[str] = None):
    """``torch.distributed`` rendezvous from torchrun's environment. Returns (rank, world, local_rank)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        kwargs = {}
        if backend == "nccl":
            torch.cuda.set_device(local_rank)
            kwargs["device_id"] = torch.device("cuda", local_rank)
        dist.init_process_group(backend=backend, rank=rank, world_size=world, **kwargs)
    return rank, world, local_rank


def shard_batch(x: torch.Tensor, rank: int, world: int) -> torch.Tensor:
    """Rank r takes windows [r*B/W, (r+1)*B/W) of the global batch (equal shards required)."""
    b = x.shape[0]
    if b % world:
        raise ValueError(f"global batch {b} is not divisible by world size {world}")
    per = b // world
    return x[rank * per:(rank + 1) * per]
