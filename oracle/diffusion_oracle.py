"""CPU oracle for ``kernel_type='random_walk_diffusion'``.  TEST INFRASTRUCTURE ONLY (same rules as
``stmgcn_oracle.py``: only ``tests/``, ``bench_diffusion.py`` and the fixture script under ``oracle/`` import it).

* **dense supports** (torch): the bidirectional ``2K+1`` stack ``[I, T_1(P_f^T) .. T_K(P_f^T), T_1(P_b^T) ..
  T_K(P_b^T)]``, ``P_f = D_out^-1 A``, ``P_b = D_in^-1 A^T`` (the reference's commented-out block ``GCN.py:82-90``;
  ``random_walk_normalize`` ``GCN.py:100-104``; ``T_k`` the recurrence of ``GCN.py:125-135``).  With it the dense
  restatement of ``stmgcn_oracle`` (``dense_st_mgcn``, ``dense_loss_and_grads``) runs the diffusion model unchanged.
* **ChainOracle** (numpy + scipy): ``stmgcn_oracle.SparseOracle`` with one or more recurrence chains per graph that
  share ``T_0 = I`` -- chain ``c`` gives supports ``1 + cK .. (c+1)K`` = ``T_1(X_c) .. T_K(X_c)`` -- and the
  hand-written backward extended to match: one adjoint Clenshaw per chain, all adding into ``dX``.
* **golden fixture** helpers of ``tests/golden/diffusion_ref.npz`` (``oracle/make_diffusion_golden.py``): its
  parameters and the weights of its ``CG_LSTM`` probe are not stored but drawn from the seed in the fixture
  (``stmgcn_oracle.init_params``, a seeded ``torch.Generator``), which keeps the fixture small.
"""
from __future__ import annotations

import os

import numpy as np
import torch

import stmgcn_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                      "diffusion_ref.npz")


def random_walk_normalize_dense(adj: torch.Tensor) -> torch.Tensor:
    """``P = D^-1 A`` with ``D`` the row sums, ``d_inv = 0`` for a zero row (``GCN.py:100-104``)."""
    d_inv = adj.sum(dim=1).pow(-1)
    d_inv = torch.where(torch.isinf(d_inv), torch.zeros_like(d_inv), d_inv)
    return d_inv[:, None] * adj


def diffusion_supports_dense(adj: torch.Tensor, order: int) -> torch.Tensor:
    """``(2K+1, N, N)`` bidirectional random-walk diffusion stack (see the module docstring)."""
    eye = torch.eye(adj.shape[0], dtype=adj.dtype)
    series = []
    for p in (random_walk_normalize_dense(adj), random_walk_normalize_dense(adj.t())):
        x = p.t()
        polys = [eye, x]
        for _ in range(2, order + 1):
            polys.append(2.0 * (x @ polys[-1]) - polys[-2])
        series += polys[1:order + 1]
    return torch.stack([eye] + series, dim=0)


def diffusion_chains_csr(adj: torch.Tensor):
    """scipy CSR of the two chains' matrices ``[P_f^T, P_b^T]``: a graph's entry of :class:`ChainOracle`'s ``chains``."""
    import scipy.sparse as sp
    return [sp.csr_matrix(random_walk_normalize_dense(a).t().numpy()) for a in (adj, adj.t())]


class ChainOracle(O.SparseOracle):
    """:class:`stmgcn_oracle.SparseOracle` whose graphs carry recurrence chains: ``chains[m]`` is a list of scipy
    matrices ``X_c`` (one matrix: the Chebyshev stack of ``L~``; ``[P_f^T, P_b^T]``: bidirectional diffusion), with
    ``n_supports = 1 + len(chains[m]) * K``.  Other arguments as for ``SparseOracle``."""

    def __init__(self, params, chains, n_supports: int, relu: bool = True, dtype=np.float64, relu_masks=None):
        super().__init__(params, [], n_supports, relu, dtype, relu_masks)
        self.lap = [[c.astype(self.dt).tocsr() for c in ch] for ch in chains]
        self.lap_t = [[c.T.tocsr() for c in ch] for ch in self.lap]
        self.m = len(self.lap)
        assert all(ch and (n_supports - 1) % len(ch) == 0 for ch in self.lap)

    def _cheb_stack(self, chains, x):
        """x:(N,B,p) -> S:(Ks,N,B,p): S_0 = x, then per chain X: T_1 = X x, T_k = 2 X T_{k-1} - T_{k-2}."""
        n = x.shape[0]
        flat = x.reshape(n, -1)
        out = [flat]
        for lap in chains:
            terms = [flat]
            for k in range(1, (self.ks - 1) // len(chains) + 1):
                terms.append(lap @ flat if k == 1 else 2.0 * (lap @ terms[-1]) - terms[-2])
            out += terms[1:]
        return np.stack(out).reshape((self.ks,) + x.shape)

    def _gcn_bwd(self, chains_t, s, out, d_out, w, need_dx: bool, mask=None):
        """``SparseOracle._gcn_bwd`` with one adjoint Clenshaw per chain, each adding into ``dX``."""
        p = s.shape[-1]
        if self.relu:
            dz = d_out * (mask if mask is not None else (out > 0))
        else:
            dz = d_out
        db = dz.reshape(-1, dz.shape[-1]).sum(0)
        dw = np.concatenate([np.tensordot(s[k], dz, axes=([0, 1], [0, 1])) for k in range(self.ks)], 0)
        dx = None
        if need_dx:
            n = s.shape[1]
            u = [(dz @ w[k * p:(k + 1) * p].T).reshape(n, -1) for k in range(self.ks)]
            k_ord = (self.ks - 1) // len(chains_t)
            dx = u[0]
            for c, lap_t in enumerate(chains_t if k_ord > 0 else []):
                b2 = np.zeros_like(u[0])        # b_{k+2}
                b1 = np.zeros_like(u[0])        # b_{k+1}
                for k in range(k_ord, 0, -1):
                    bk = u[c * k_ord + k] + 2.0 * (lap_t @ b1) - b2
                    b2, b1 = b1, bk
                dx = dx + lap_t @ b1 - b2
            dx = dx.reshape(s.shape[1:])
        return dw, db, dx


def load_golden(path: str = GOLDEN):
    """``(meta, params, grads, supports, adjs, blob)`` of the diffusion fixture; ``params`` (torch, the reference's
    ``state_dict`` names) are drawn from the fixture's seed, as the fixture script drew them."""
    blob = np.load(path)
    n, m, k, t, b, c, hid, layers, gcn_hid, seed = [int(v) for v in blob["meta"]]
    meta = dict(n=n, m=m, k=k, t=t, b=b, c=c, hid=hid, layers=layers, gcn_hid=gcn_hid, seed=seed)
    params = golden_params(meta)
    grads = {key[len("grad."):]: blob[key] for key in blob.files if key.startswith("grad.")}
    supports = [torch.from_numpy(blob[f"supports.{g}"]) for g in range(m)]
    adjs = [torch.from_numpy(blob[f"adj.{g}"]) for g in range(m)]
    return meta, params, grads, supports, adjs, blob


def golden_params(meta) -> dict:
    """The fixture's parameters: ``stmgcn_oracle.init_params`` (the reference's names, shapes and init distributions)
    drawn from the fixture's seed."""
    return O.init_params(meta["m"], meta["t"], meta["c"], meta["hid"], meta["layers"], meta["gcn_hid"],
                         2 * meta["k"] + 1, seed=meta["seed"])


def golden_probe(meta) -> torch.Tensor:
    """``cg_w`` (B, N, H): the weights of the fixture's scalar probe ``sum(cg_out * cg_w)`` of ``CG_LSTM``."""
    gen = torch.Generator().manual_seed(meta["seed"] + 1)
    return torch.randn(meta["b"], meta["n"], meta["hid"], generator=gen)
