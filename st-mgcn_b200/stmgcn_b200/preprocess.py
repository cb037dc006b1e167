"""Support construction: drop-in for ``GCN.Adj_Preprocessor`` (reference ``GCN.py:50-135``) plus the
sparse-native path of SURVEY.md section 8(f)-1.

``process(adj)`` returns the same dense ``(K+1, N, N)`` stack the reference returns (so ``Main.py:49-55``
runs unchanged); ``process_sparse(adj)`` returns a :class:`~stmgcn_b200.graph.SparseSupports` holding only
the matrices the kernels multiply by, as CSR (for ``chebyshev`` the rescaled Laplacian, for
``random_walk_diffusion`` the forward and backward transition matrices) -- no ``N x N`` polynomial is ever built
(the reference needs K dense ``N^3`` products and 19 GB of supports at 16384 regions).

``lambda_max``: the reference calls ``torch.eig`` (``GCN.py:117``), which no longer exists in torch >= 1.13;
its bare ``except`` then uses 2 (``GCN.py:119-121``).  ``lambda_max="reference"`` (default) reproduces that
behaviour, a float fixes the value, ``"power"`` estimates the largest eigenvalue by power iteration.
"""
from __future__ import annotations

from typing import Union

import torch

from .graph import ChebSupports, LearnableAdjacency, SparseSupports, _stored_entries, csr_from_coo


class Adj_Preprocessor(object):
    def __init__(self, kernel_type: str, K: int, lambda_max: Union[str, float] = "reference"):
        if kernel_type not in ("chebyshev", "localpool", "random_walk_diffusion"):
            raise ValueError('Invalid kernel_type. Must be one of [chebyshev, localpool, random_walk_diffusion].')
        self.kernel_type = kernel_type
        self.K = K if kernel_type != "localpool" else 1      # GCN.py:54
        self.lambda_max = lambda_max

    # ---- normalisations (GCN.py:99-111), written with broadcasting instead of diag/mm -------------------
    @staticmethod
    def symmetric_normalize(A: torch.Tensor) -> torch.Tensor:
        d = A.sum(dim=1).pow(-0.5)
        return d.unsqueeze(1) * A * d.unsqueeze(0)

    @staticmethod
    def random_walk_normalize(A: torch.Tensor) -> torch.Tensor:
        d = A.sum(dim=1).pow(-1)
        d = torch.where(torch.isinf(d), torch.zeros_like(d), d)
        return d.unsqueeze(1) * A

    def _lambda(self, lap: torch.Tensor) -> float:
        if isinstance(self.lambda_max, (int, float)):
            return float(self.lambda_max)
        if self.lambda_max == "reference":
            return 2.0
        if self.lambda_max == "power":
            v = torch.ones(lap.shape[0], dtype=lap.dtype, device=lap.device)
            lam = 2.0
            for _ in range(200):
                w = lap @ v
                nrm = float(w.norm())
                if nrm == 0.0:
                    break
                lam, v = nrm / max(float(v.norm()), 1e-30), w / nrm
            return lam
        raise ValueError(f"lambda_max={self.lambda_max!r}")

    def rescale_laplacian(self, L: torch.Tensor) -> torch.Tensor:
        eye = torch.eye(L.shape[0], dtype=L.dtype, device=L.device)
        return (2.0 / self._lambda(L)) * L - eye

    def _polynomials(self, x: torch.Tensor):
        """``T_0 .. T_K`` of the matrix ``x`` (GCN.py:125-135)."""
        polys = [torch.eye(x.shape[0], dtype=x.dtype, device=x.device)]
        if self.K >= 1:
            polys.append(x)
        while len(polys) < self.K + 1:
            polys.append(2 * (x @ polys[-1]) - polys[-2])
        return polys

    def process(self, adj: torch.Tensor) -> torch.Tensor:
        """(N,N) adjacency -> (K_supports, N, N) dense stack, as ``GCN.py:57-97``."""
        if self.kernel_type == "localpool":
            a_norm = self.symmetric_normalize(adj)
            kernels = [torch.eye(adj.shape[0], dtype=adj.dtype, device=adj.device) + a_norm]
        elif self.kernel_type == "chebyshev":
            a_norm = self.symmetric_normalize(adj)
            lap = torch.eye(adj.shape[0], dtype=adj.dtype, device=adj.device) - a_norm
            kernels = self._polynomials(self.rescale_laplacian(lap))
        else:   # random_walk_diffusion: K+1 polynomials of P^T (the reference's forward-only variant)
            kernels = self._polynomials(self.random_walk_normalize(adj).T)
        return torch.stack(kernels, dim=0)

    def process_sparse(self, adj: torch.Tensor) -> SparseSupports:
        """The supports of :meth:`process` without dense polynomials or dense ``N x N`` products: only the matrices the
        kernels multiply into the features are formed, as CSR.

        * ``chebyshev``: ``L~`` (a :class:`ChebSupports`, ``K+1`` supports, one recurrence chain);
        * ``random_walk_diffusion``: ``P_f^T`` and ``P_b^T``, ``P_f = D_out^-1 A``, ``P_b = D_in^-1 A^T`` (a zero
          degree gives ``d_inv = 0``, ``GCN.py:100-104``): the ``2K+1`` bidirectional supports
          ``[I, T_1(P_f^T) .. T_K(P_f^T), T_1(P_b^T) .. T_K(P_b^T)]`` of the reference's commented-out block
          (``GCN.py:82-90``), two recurrence chains sharing ``T_0 = I``.  ``A`` may be directed.  At most
          8 supports (``K <= 3``): the projection kernels take up to 8;
        * ``localpool``: ``I + D^-1/2 A D^-1/2`` as one generic support.

        When ``adj`` (dense) or its values (sparse COO) require grad, the handle's stored values keep the autograd graph
        back to them: rebuilt every step, the supports carry the loss's gradient to the adjacency's entries through the
        normalisations (``lambda_max`` is a constant).  The gradient lives on the stored pattern: an absent edge, or an
        entry dropped as an exact zero, gets none (a dense ``process()`` stack would give one there).
        ``adj`` may be dense ``(N,N)`` or a sparse COO/CSR tensor.  The result is accepted wherever the
        dense stack is (``GCN.forward``, ``ST_MGCN.forward``'s ``sta_adj_list``)."""
        coo = adj.to_sparse_coo().coalesce() if adj.layout != torch.sparse_coo else adj.coalesce()
        n = coo.shape[0]
        row, col = coo.indices()
        val = coo.values().to(torch.float32)
        dev = val.device
        if self.kernel_type == "random_walk_diffusion":
            ks = 2 * self.K + 1
            if ks > 8:
                raise ValueError(f"process_sparse: random_walk_diffusion with K={self.K} needs {ks} supports; the "
                                 f"projection kernels take at most 8 supports (K <= 3)")

            def inv(deg):
                d = deg.pow(-1)
                return torch.where(torch.isinf(d), torch.zeros_like(d), d)
            d_out = inv(torch.zeros(n, dtype=torch.float32, device=dev).index_add_(0, row, val))
            d_in = inv(torch.zeros(n, dtype=torch.float32, device=dev).index_add_(0, col, val))
            # P_f^T[j, i] = A[i, j] / out_deg(i);  P_b^T[i, j] = A[i, j] / in_deg(j)
            mats = [_csr(n, col, row, val * d_out[row]), _csr(n, row, col, val * d_in[col])]
            return SparseSupports("cheb", n, ks, mats)
        deg = torch.zeros(n, dtype=torch.float32, device=dev).index_add_(0, row, val)
        d = deg.pow(-0.5)
        a_norm = d[row] * val * d[col]
        ar = torch.arange(n, device=dev)
        if self.kernel_type == "localpool":
            ones = torch.ones(n, dtype=torch.float32, device=dev)
            return SparseSupports("generic", n, 1, [_csr(n, torch.cat([row, ar]), torch.cat([col, ar]),
                                                         torch.cat([a_norm, ones]))])
        if self.lambda_max == "reference":
            lam = 2.0
        elif isinstance(self.lambda_max, (int, float)):
            lam = float(self.lambda_max)
        else:
            lam = self._lambda_sparse(n, row, col, a_norm.detach())      # a constant: no gradient through it
        scale = 2.0 / lam
        # L~ = scale * (I - A_norm) - I  => off-diagonal -scale*A_norm, diagonal (scale - 1) - scale*A_norm_ii
        diag_val = scale - 1.0
        idx_r, idx_c, vals = row, col, -scale * a_norm
        if diag_val != 0.0:
            idx_r, idx_c = torch.cat([idx_r, ar]), torch.cat([idx_c, ar])
            vals = torch.cat([vals, torch.full((n,), diag_val, dtype=torch.float32, device=dev)])
        return ChebSupports(n, self.K + 1, *_csr(n, idx_r, idx_c, vals))

    def process_learnable(self, adj: torch.Tensor) -> LearnableAdjacency:
        """A learnable graph on the fixed pattern of ``adj``: a :class:`~stmgcn_b200.graph.LearnableAdjacency` whose only
        parameter ``weight`` holds one value per stored edge (initialised to ``adj``'s values; a dense ``adj``'s non-zero
        entries, a sparse one's stored entries, stored zeros included).  Every forward normalises the weights on the
        device into the supports :meth:`process_sparse` would build from them (``lambda_max`` is evaluated once, here, and
        held constant).  It stands in for the supports wherever they go; train it by giving ``module.parameters()`` to
        the optimizer (and to ``dp.GradBucket`` / ``GraphedStep``'s bucket under data parallelism)."""
        lam = 2.0
        if self.kernel_type == "chebyshev":
            if self.lambda_max == "reference":
                lam = 2.0
            elif isinstance(self.lambda_max, (int, float)):
                lam = float(self.lambda_max)
            else:
                n, row, col, val = _stored_entries(adj)
                d = torch.zeros(n, dtype=torch.float32, device=val.device).index_add_(0, row, val).pow(-0.5)
                lam = self._lambda_sparse(n, row, col, d[row] * val * d[col])
        return LearnableAdjacency(self.kernel_type, self.K, adj, scale=2.0 / lam, lambda_max=lam)

    @staticmethod
    def _lambda_sparse(n, row, col, a_norm) -> float:
        v = torch.ones(n, dtype=torch.float32, device=a_norm.device)
        lam = 2.0
        for _ in range(200):
            w = v - torch.zeros_like(v).index_add_(0, row, a_norm * v[col])      # (I - A_norm) v
            nrm = float(w.norm())
            if nrm == 0.0:
                break
            lam, v = nrm / max(float(v.norm()), 1e-30), w / nrm
        return lam


def _csr(n: int, rows: torch.Tensor, cols: torch.Tensor, vals: torch.Tensor):
    """CSR of the ``n x n`` matrix with entries ``(rows, cols, vals)`` in any order (repeats summed, exact zeros dropped).
    With ``vals`` requiring grad the CSR's values are the differentiable values (the indices are copies)."""
    m = torch.sparse_coo_tensor(torch.stack([rows, cols]), vals, (n, n)).coalesce()
    keep = m.values() != 0
    rowptr, colidx, v = csr_from_coo(n, m.indices()[0][keep], m.indices()[1][keep], m.values()[keep])
    if vals.requires_grad:
        v = m.values()[keep].to(torch.float32)
    return rowptr, colidx, v
