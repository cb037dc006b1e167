"""CUDA-graph capture of one training step (forward + loss + backward [+ gradient all-reduce]).

A step of the hot path is ~300 kernel launches of 3-2000 us each plus a few dozen tiny torch kernels; launched
eagerly from Python the GPU idles ~15 % of the time between them.  All shapes are static for a fixed batch size
(the reference's DataLoader yields one short last batch: use the eager path for it), so the whole step is captured
once into a CUDA graph and replayed: ``GraphedStep(model, criterion, x, y, supports)`` then ``loss = step(x, y)``.

The kernels launched through the C ABI take the stream from ``torch.cuda.current_stream()``, so they are captured
like any torch op; every buffer they touch comes from torch's allocator and therefore from the graph's private pool.
Gradients are accumulated into ``GradBucket`` views (static addresses).  The optimizer step stays outside the graph.

The supports are baked in too: the graph reads the CSR tensors of the support sets converted at capture.  The step holds
those sets (so their memory stays valid whatever happens to the conversion cache) and the supports' versions
(``graph.support_version``); a call after any support was edited raises instead of replaying the old supports.
Learnable supports (a ``SparseSupports`` whose values require grad, or a dense stack that requires grad) are refused at
construction: their values are read again at every forward, which a replayed graph cannot do.

A ``LearnableAdjacency`` is accepted: its normalisation (``ops.AdjNorm``) is captured with the step and reads ``weight``
at its own address, so each replay runs at the weights the optimizer left there (fused optimizers included).  Its
``support_version`` is the version of its pattern tensors.  The default bucket covers the model and these modules; an
explicit ``bucket`` must hold their parameters (else ``ValueError``: their gradients would land outside the reduced
buffer).
"""
from __future__ import annotations

from typing import Callable, Optional, Sequence

import torch

from .dp import GradBucket
from .graph import LearnableAdjacency, SparseSupports, support_version, supports_from_dense


class GraphedStep:
    def __init__(self, model: torch.nn.Module, criterion: Callable, x: torch.Tensor, y: torch.Tensor,
                 supports: Sequence, bucket: Optional[GradBucket] = None, all_reduce: bool = False,
                 warmup: int = 3):
        learnable = [m for m, s in enumerate(supports) if isinstance(s, SparseSupports) and s.requires_grad]
        if learnable:
            raise ValueError(f"GraphedStep: supports {learnable} have values that require grad; a captured step replays "
                             f"the values of capture time, so learnable supports run eagerly")
        dense = [m for m, s in enumerate(supports) if isinstance(s, torch.Tensor) and s.requires_grad]
        if dense:
            raise ValueError(f"GraphedStep: the dense support stacks {dense} require grad; a captured step replays the "
                             f"conversion of capture time, so stacks that require grad run eagerly")
        self.model, self.criterion, self.supports = model, criterion, list(supports)
        adjs = []
        for s in self.supports:
            if isinstance(s, LearnableAdjacency) and all(s is not a for a in adjs):
                adjs.append(s)
        if bucket is not None:
            held = {id(p) for p in bucket.params}
            lacking = [m for m, s in enumerate(self.supports) if isinstance(s, LearnableAdjacency)
                       and any(p.requires_grad and id(p) not in held for p in s.parameters())]
            if lacking:
                raise ValueError(f"GraphedStep: the bucket lacks the parameters of the learnable adjacencies {lacking}; "
                                 f"build it as GradBucket(model, *adjacencies)")
        self.bucket = bucket if bucket is not None else GradBucket(model, *adjs)
        self.all_reduce = all_reduce
        self.x = torch.empty_like(x)
        self.y = torch.empty_like(y)
        self.x.copy_(x)
        self.y.copy_(y)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):                 # warm-up on a side stream (allocator + lazy inits)
            for _ in range(warmup):
                self._eager()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        # the conversions the warm-up cached, which the capture below reads (a learnable adjacency holds its own structure
        # and is normalised inside the capture)
        self.support_sets = [s if isinstance(s, LearnableAdjacency) else supports_from_dense(s) for s in self.supports]
        self.support_versions = [support_version(s) for s in self.supports]
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.loss = self._eager()

    def _eager(self) -> torch.Tensor:
        self.bucket.zero_()
        out = self.model(obs_seq=self.x, sta_adj_list=self.supports)
        loss = self.criterion(out, self.y)
        loss.backward()
        if self.all_reduce:
            self.bucket.all_reduce_mean_()
        self.out = out.detach()         # after capture: the static buffer of the replayed step's prediction
        return loss

    def __call__(self, x: Optional[torch.Tensor] = None, y: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Copy the batch into the static buffers (host or device source) and replay. Returns the loss tensor
        (static buffer: read it before the next call).  Raises ``RuntimeError`` if a support was edited since the
        capture (build a new ``GraphedStep`` then)."""
        changed = [m for m, s in enumerate(self.supports) if support_version(s) != self.support_versions[m]]
        if changed:
            raise RuntimeError(f"GraphedStep: supports {changed} were edited after the step was captured; the captured "
                               f"graph would replay the supports of capture time: capture a new GraphedStep")
        if x is not None and tuple(x.shape) != tuple(self.x.shape):
            # a batch of another size (the reference's DataLoader yields one short last batch, Data_Container.py:122):
            # shapes are baked into the captured graph, so this batch runs eagerly
            self.bucket.zero_()
            out = self.model(obs_seq=x.to(self.x.device, non_blocking=True), sta_adj_list=self.supports)
            loss = self.criterion(out, y.to(self.y.device, non_blocking=True))
            loss.backward()
            if self.all_reduce:
                self.bucket.all_reduce_mean_()
            self.out = out.detach()
            return loss
        if x is not None:
            self.x.copy_(x, non_blocking=True)
        if y is not None:
            self.y.copy_(y, non_blocking=True)
        self.graph.replay()
        return self.loss
