"""Synthetic region x timestep workloads (SURVEY.md section 8(d)).

The reference ships no dataset (``Main.py:9`` points at ``./data/data_dict.npz`` which is not in the
repository), so every parity test and every bench line in this repo runs on inputs produced here.

Graph ``m``: ``g = torch.Generator().manual_seed(1000 + m)``; ``A = rand(N, N) < density / 2``;
``A = (A + A^T) > 0``; zero diagonal; ring edges ``(i, (i + 1) mod N)`` in both directions (an isolated
region would make the reference's ``symmetric_normalize`` emit NaN, ``GCN.py:109``); float32 0/1.
Inputs: ``torch.manual_seed(seed)``; ``x = randn(B, T, N, C)``, ``y = randn(B, N, C)``.

This module is product-side host code (it is what ``bench.py`` feeds the hot path with); it never imports
anything from ``oracle/``.
"""
from __future__ import annotations

import dataclasses
from typing import List, Tuple

import torch


@dataclasses.dataclass(frozen=True)
class Workload:
    """One row of the BASELINE.json ``configs`` list (SURVEY.md section 8(d) table)."""
    name: str
    n_regions: int      # N
    n_graphs: int       # M
    cheb_order: int     # K  (supports = K + 1)
    seq_len: int        # T
    batch: int          # B per GPU
    density: float
    dtype: str          # arithmetic type the config is quoted in
    input_dim: int = 1          # C   (Main.py:62)
    lstm_hidden: int = 64       # H   (Main.py:62)
    lstm_layers: int = 3        # L   (Main.py:62)
    gcn_hidden: int = 64        # G   (Main.py:63)

    @property
    def n_supports(self) -> int:
        return self.cheb_order + 1

    @property
    def region_timesteps(self) -> int:
        return self.batch * self.n_regions * self.seq_len


WORKLOADS = {
    "cfg1": Workload("cfg1", 64, 1, 2, 4, 8, 0.10, "f32"),
    "cfg2": Workload("cfg2", 1024, 3, 3, 12, 32, 0.01, "bf16"),
    "cfg3": Workload("cfg3", 4096, 3, 3, 12, 64, 0.01, "f32"),
    "cfg4": Workload("cfg4", 4096, 3, 3, 12, 64, 0.01, "bf16"),     # 512 global on 8 GPUs
    "cfg5": Workload("cfg5", 16384, 3, 5, 24, 32, 0.01, "bf16"),    # 256 global on 8 GPUs
}


def make_adjacency(n: int, m: int, density: float) -> torch.Tensor:
    """Dense 0/1 float32 adjacency of graph ``m`` (symmetric Erdos-Renyi + ring), CPU."""
    g = torch.Generator().manual_seed(1000 + m)
    a = torch.rand(n, n, generator=g) < (density / 2.0)
    a = (a | a.t())
    a.fill_diagonal_(False)
    idx = torch.arange(n)
    a[idx, (idx + 1) % n] = True
    a[(idx + 1) % n, idx] = True
    if n <= 2:                                   # degenerate ring: keep it loop-free
        a.fill_diagonal_(False)
    return a.to(torch.float32)


def make_directed_adjacency(n: int, m: int, density: float) -> torch.Tensor:
    """Dense 0/1 float32 DIRECTED adjacency of graph ``m`` (the ``random_walk_diffusion`` workloads), CPU:
    ``g = torch.Generator().manual_seed(2000 + m)``; arcs ``rand(N, N) < density``, no self-loops, and a one-way ring
    ``i -> (i + 1) mod N``, so every region has an out-arc and an in-arc (the Chebyshev normalisation of the same graph,
    by row sums, stays finite too)."""
    g = torch.Generator().manual_seed(2000 + m)
    a = torch.rand(n, n, generator=g) < density
    idx = torch.arange(n)
    a[idx, (idx + 1) % n] = True
    a.fill_diagonal_(False)
    return a.to(torch.float32)


def make_similarity_adjacency(n: int, m: int, dim: int = 16, width: float = 1.0) -> torch.Tensor:
    """Dense float32 similarity adjacency of graph ``m``, CPU, every off-diagonal entry non-zero (a functional-similarity
    or Gaussian-kernel distance graph nobody thresholded): ``g = torch.Generator().manual_seed(3000 + m)``; region
    vectors ``v = rand(N, dim)``; ``A_ij = exp(-|v_i - v_j|^2 / (width * dim / 6))`` (``dim / 6`` is the mean squared
    distance of two such vectors), zero diagonal."""
    g = torch.Generator().manual_seed(3000 + m)
    v = torch.rand(n, dim, generator=g, dtype=torch.float64)
    a = torch.exp(-torch.cdist(v, v).square() / (width * dim / 6.0))
    a.fill_diagonal_(0.0)
    return a.to(torch.float32)


def make_adjacency_list(w: Workload) -> List[torch.Tensor]:
    return [make_adjacency(w.n_regions, m, w.density) for m in range(w.n_graphs)]


def make_inputs(w: Workload, seed: int = 0, batch: int | None = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(x, y)`` with ``x:(B,T,N,C)``, ``y:(B,N,C)`` standard normal, CPU float32."""
    b = w.batch if batch is None else batch
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, w.seq_len, w.n_regions, w.input_dim, generator=g)
    y = torch.randn(b, w.n_regions, w.input_dim, generator=g)
    return x, y


def model_kwargs(w: Workload) -> dict:
    """Keyword arguments of ``STMGCN.ST_MGCN`` for this workload (names from ``Main.py:62-63``)."""
    from torch import nn
    return dict(M=w.n_graphs, seq_len=w.seq_len, n_nodes=w.n_regions, input_dim=w.input_dim,
                lstm_hidden_dim=w.lstm_hidden, lstm_num_layers=w.lstm_layers,
                gcn_hidden_dim=w.gcn_hidden,
                sta_kernel_config={"kernel_type": "chebyshev", "K": w.cheb_order},
                gconv_use_bias=True, gconv_activation=nn.ReLU)
