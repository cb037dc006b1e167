"""Support ingestion: the constant operand of the hot path.

The reference hands ``GCN.forward`` a dense ``(K+1, N, N)`` stack built once by
``Adj_Preprocessor.process`` (``GCN.py:57-97``; stacked ``:95``) and multiplies each slice into the
features (``GCN.py:34-36``).  Here the stack is inspected ONCE per tensor (cached on identity + version):

* if it is a Chebyshev stack -- ``A[0] = I`` and ``A[k] = 2 A[1] A[k-1] - A[k-2]`` (``GCN.py:125-135``),
  checked with a random probe -- only ``L~ = A[1]`` is kept, as CSR + CSR^T on the device, and the forward
  runs the recurrence on the features (``SupportSet.mode == "cheb"``, one chain);
* otherwise (``localpool``, hand-made supports) every slice is sparsified on its own and applied
  directly (``mode == "generic"``) -- same kernels, same results as the reference's einsum.

``SparseSupports`` is the sparse-native handle ``GCN.Adj_Preprocessor.process_sparse`` returns (``ChebSupports``
for ``chebyshev``): it quacks like the reference's tensor where ``Main.py`` touches it (``.to(device)``, ``len``,
``.shape``) but never materialises ``N x N`` polynomials (SURVEY.md section 8(f)-1).  Its ``"cheb"`` stacks are one or
more recurrence chains that share ``T_0 = I``: one for ``chebyshev`` (``L~``), two for ``random_walk_diffusion``
(``P_f^T`` and ``P_b^T``, DCRNN's dual random-walk diffusion).
"""
from __future__ import annotations

import copy
from collections import OrderedDict
from typing import List, Optional

import torch


def csr_from_coo(n: int, rows: torch.Tensor, cols: torch.Tensor, vals: torch.Tensor):
    """int32 CSR ``(rowptr, colidx, vals)`` of the ``n x n`` matrix whose entries ``(rows, cols, vals)`` are sorted
    row-major (by row, then column).  The result shares no memory with the arguments."""
    nnz = rows.numel()
    if not 0 < n < 2 ** 30 or nnz >= 2 ** 31:
        raise ValueError(f"CSR: n={n} must be in [1, 2^30) and nnz={nnz} below 2^31 (int32 indices)")
    rowptr = torch.zeros(n + 1, dtype=torch.int32, device=rows.device)
    rowptr[1:] = torch.cumsum(torch.bincount(rows, minlength=n), 0)
    return rowptr, cols.to(torch.int32, copy=True), vals.detach().to(torch.float32, copy=True).contiguous()


def check_csr(n: int, rowptr: torch.Tensor, colidx: torch.Tensor, vals: torch.Tensor) -> None:
    """Raise ``ValueError`` naming the first fault of an ``n x n`` CSR matrix: dtypes, devices, sizes, ``rowptr``
    starting at 0, never decreasing and ending at ``nnz``, every column index in ``[0, n)``.  One host sync."""
    if rowptr.dtype != torch.int32 or colidx.dtype != torch.int32 or vals.dtype != torch.float32:
        raise ValueError(f"CSR: rowptr / colidx must be int32 and vals float32, got {rowptr.dtype} / {colidx.dtype} / "
                         f"{vals.dtype}")
    devices = {str(t.device) for t in (rowptr, colidx, vals)}
    if len(devices) != 1:
        raise ValueError(f"CSR: rowptr, colidx and vals are on mixed devices {sorted(devices)}")
    if rowptr.dim() != 1 or colidx.dim() != 1 or vals.dim() != 1:
        raise ValueError("CSR: rowptr, colidx and vals must be 1-D")
    if rowptr.numel() != n + 1:
        raise ValueError(f"CSR: rowptr has {rowptr.numel()} entries, n + 1 = {n + 1} expected")
    nnz = colidx.numel()
    if vals.numel() != nnz:
        raise ValueError(f"CSR: vals has {vals.numel()} entries, colidx {nnz}")
    faults = torch.stack([rowptr[0] != 0, (rowptr[1:] < rowptr[:-1]).any(), rowptr[-1] != nnz,
                          ((colidx < 0) | (colidx >= n)).any()]).tolist()
    names = ["rowptr[0] is not 0", "rowptr decreases", f"rowptr[-1] is not nnz = {nnz}",
             f"a column index is outside [0, {n})"]
    for fault, name in zip(faults, names):
        if fault:
            raise ValueError(f"CSR: {name}")


class GraphHandle:
    """CSR and CSR^T of one ``n x n`` support matrix: int32 ``rowptr`` / ``colidx`` and fp32 ``vals`` tensors.

    The handle owns its tensors (copies of what it was built from), so the CSR and the CSR^T are one snapshot of the
    matrix: an edit of the source after the build reaches neither."""

    def __init__(self, n: int, rows: torch.Tensor, cols: torch.Tensor, vals: torch.Tensor):
        """From the matrix's entries, sorted row-major; ``rows`` and ``cols`` are int64."""
        self.n, self.nnz, self.device = n, rows.numel(), rows.device
        # CSR^T: the entries in column-major order (stable: repeated (row, col) entries keep their order)
        order = torch.argsort(cols * n + rows, stable=True)
        self._csr = (csr_from_coo(n, rows, cols, vals), csr_from_coo(n, cols[order], rows[order], vals[order]))
        self._order = order

    def with_values(self, vals: torch.Tensor) -> "GraphHandle":
        """The same structure (shared index tensors) with the values ``vals``, given in this handle's CSR entry order
        (a CSR source's storage order), copied -- the matrix a learnable support has at one forward."""
        new = copy.copy(self)
        v = vals.detach().to(torch.float32, copy=True).contiguous()
        (rp, ci, _), (rpt, cit, _) = self._csr
        new._csr = ((rp, ci, v), (rpt, cit, v[self._order]))
        return new

    @classmethod
    def from_dense(cls, mat: torch.Tensor) -> "GraphHandle":
        """Exact zeros (-0.0 included) are dropped, every other entry (NaN included) is kept verbatim: supports[1] of
        ``Adj_Preprocessor.process`` (``GCN.py:57-97``) becomes the sparse rescaled Laplacian."""
        assert mat.dtype == torch.float32 and mat.dim() == 2 and mat.shape[0] == mat.shape[1]
        rows, cols = (mat != 0).nonzero(as_tuple=True)           # row-major order
        return cls(mat.shape[0], rows, cols, mat[rows, cols])

    @classmethod
    def from_csr(cls, n: int, rowptr: torch.Tensor, colidx: torch.Tensor, vals: torch.Tensor) -> "GraphHandle":
        """From a CSR matrix (checked by :func:`check_csr`).  Columns may be unsorted within a row, entries repeated
        (each one is applied: repeats add up) and stored zeros kept."""
        check_csr(n, rowptr, colidx, vals)
        rows = torch.repeat_interleave(torch.arange(n, device=rowptr.device), (rowptr[1:] - rowptr[:-1]).long(),
                                       output_size=colidx.numel())
        return cls(n, rows, colidx.long(), vals)

    def export(self, transpose: bool = False):
        """``(rowptr, colidx, vals)`` of the matrix, or with ``transpose`` of its transpose."""
        return self._csr[int(transpose)]


class SupportSet:
    """What the kernels need to know about one ``(Ks, N, N)`` support stack.

    ``"cheb"``: ``graphs`` are the recurrence matrices ``X_c`` of chains that share ``T_0 = I``; chain ``c`` owns the
    segments ``1 + cK .. (c+1)K``, ``T_k(X_c)`` with ``K = (Ks - 1) / len(graphs)`` (no graph when ``Ks == 1``).
    ``"generic"``: ``graphs[k]`` is ``A_k``.

    ``values`` (optional): the source tensors of the graphs' stored values, one per graph in CSR entry order, when some
    of them require grad (a learnable :class:`SparseSupports`).  The graphs hold detached copies; the graph
    convolutions take these tensors as inputs, so their gradients reach them.
    """

    def __init__(self, mode: str, n: int, ks: int, graphs: List[GraphHandle], device: torch.device,
                 values: Optional[List[torch.Tensor]] = None):
        assert mode in ("cheb", "generic")
        assert len(graphs) == ks if mode == "generic" else (ks - 1) % max(len(graphs), 1) == 0 and (ks == 1) == (not graphs)
        assert values is None or len(values) == len(graphs)
        self.mode, self.n, self.ks, self.graphs, self.device = mode, n, ks, graphs, device
        self.values = values

    def grad_values(self) -> tuple:
        """The value tensors the graph convolutions take as inputs: ``values`` when one of them requires grad, else ()."""
        if self.values is not None and any(v.requires_grad for v in self.values):
            return tuple(self.values)
        return ()

    @property
    def order(self) -> int:
        """``K`` of each chain (``"cheb"`` only)."""
        return (self.ks - 1) // len(self.graphs) if self.graphs else 0

    def chain_segments(self, c: int) -> List[int]:
        """Stack indices of chain ``c``'s terms ``T_0 .. T_K`` (``T_0 = I`` is segment 0 for every chain)."""
        k = self.order
        return [0] + list(range(1 + c * k, 1 + (c + 1) * k))

    @property
    def nnz(self) -> int:
        return sum(g.nnz for g in self.graphs)


def _is_chebyshev_stack(a: torch.Tensor, tol: float = 5e-5) -> bool:
    """Probe ``A[0] v = v`` and ``A[k] v = 2 A[1] (A[k-1] v) - A[k-2] v`` with a fixed random ``v``."""
    ks, n, _ = a.shape
    g = torch.Generator(device="cpu").manual_seed(1234)
    v = torch.randn(n, 4, generator=g).to(a.device)

    def close(x, y):
        scale = max(float(y.abs().max()), 1e-20)
        return bool(torch.isfinite(x).all()) and float((x - y).abs().max()) <= tol * scale

    if not close(a[0] @ v, v):
        return False
    if ks == 1:
        return True
    prev2, prev1 = v, a[1] @ v
    for k in range(2, ks):
        want = a[k] @ v
        if not close(2.0 * (a[1] @ prev1) - prev2, want):
            return False
        prev2, prev1 = prev1, want
    return True


_CACHE: "OrderedDict[tuple, tuple]" = OrderedDict()
_CACHE_MAX = 32


def support_version(a) -> tuple:
    """What a support stack's conversion is keyed on: identity and in-place version of its tensors.  Any edit of the
    stack through a torch op changes it."""
    if isinstance(a, SparseSupports):
        return a.version()
    return (a.data_ptr(), a._version, tuple(a.shape), tuple(a.stride()), str(a.device), a.dtype)


def supports_from_dense(a: torch.Tensor) -> SupportSet:
    """Cached conversion of a dense support stack (keyed on tensor identity + in-place version)."""
    if isinstance(a, SparseSupports):
        return a.support_set()
    if not isinstance(a, torch.Tensor) or a.dim() != 3 or a.shape[1] != a.shape[2]:
        raise ValueError(f"supports must be a (K, N, N) tensor, got {type(a)} {getattr(a, 'shape', None)}")
    if not a.is_cuda:
        raise RuntimeError("stmgcn_b200 has no CPU path: supports must live on a CUDA device "
                           "(the reference moves them there at Main.py:54)")
    key = support_version(a)
    hit = _CACHE.get(key)
    if hit is not None:
        _CACHE.move_to_end(key)
        return hit[1]
    af = a.detach()
    if af.dtype != torch.float32:
        af = af.float()
    ks, n, _ = af.shape
    with torch.cuda.device(a.device):
        if _is_chebyshev_stack(af):
            graphs = [GraphHandle.from_dense(af[1])] if ks > 1 else []
            sset = SupportSet("cheb", n, ks, graphs, a.device)
        else:
            sset = SupportSet("generic", n, ks, [GraphHandle.from_dense(af[k]) for k in range(ks)], a.device)
    _CACHE[key] = (a, sset)          # keep `a` alive so the data_ptr cannot be recycled under the key
    while len(_CACHE) > _CACHE_MAX:
        _CACHE.popitem(last=False)
    return sset


def clear_cache() -> None:
    _CACHE.clear()


class SparseSupports:
    """Sparse-native ``(Ks, N, N)`` support stack: the matrices of a :class:`SupportSet` as CSR, nothing ``N x N``.

    ``mode == "cheb"``: ``mats`` are the recurrence matrices of the chains (see :class:`SupportSet`);
    ``mode == "generic"``: ``mats[k]`` is ``A_k``.  Each matrix is an int32 ``rowptr`` / ``colidx``, fp32 ``vals`` triple.

    Stands in for the dense tensor of the reference where its callers touch it: ``.to(device)`` (``Main.py:54``),
    ``len()`` / ``.shape[0]`` (``GCN.py:31``), ``.device``, ``.is_cuda``.
    """

    def __init__(self, mode: str, n: int, ks: int, mats):
        assert mode in ("cheb", "generic") and len(mats) >= 1
        self.mode, self.n, self.ks = mode, int(n), int(ks)
        self.mats = [(rp.to(torch.int32), ci.to(torch.int32), v.float()) for rp, ci, v in mats]
        self._sset: Optional[SupportSet] = None
        self._sset_version: tuple = ()
        self._structure: Optional[List[GraphHandle]] = None
        self._structure_key: tuple = ()

    @property
    def shape(self):
        return torch.Size((self.ks, self.n, self.n))

    @property
    def device(self):
        return self.mats[0][0].device

    @property
    def is_cuda(self):
        return self.mats[0][0].is_cuda

    def __len__(self):
        return self.ks

    def to(self, device, *_, **__):
        device = torch.device(device)
        if device == self.device:
            return self
        moved = copy.copy(self)
        moved.mats = [tuple(t.to(device) for t in m) for m in self.mats]
        moved._sset = None
        moved._structure = None
        return moved

    def cuda(self, device=None):
        return self.to(torch.device("cuda", torch.cuda.current_device() if device is None else device))

    def version(self) -> tuple:
        """Identity and in-place version of every stored tensor: changes with any edit through a torch op."""
        return tuple((t.data_ptr(), t._version) for m in self.mats for t in m)

    @property
    def requires_grad(self) -> bool:
        """Whether some stored values require grad (learnable edge weights on the fixed sparsity pattern)."""
        return any(v.requires_grad for _, _, v in self.mats)

    def support_set(self) -> SupportSet:
        """The kernels' copy of the stored matrices, built again whenever :meth:`version` has changed since the last
        build (as :func:`supports_from_dense` does for a dense stack).

        With values that require grad the structure (CSR and CSR^T indices, the transpose's permutation) is cached on the
        index tensors only, and the values are copied again on every call: an optimizer may change them without a
        version bump (fused optimizers, ``.data`` writes), and each forward must multiply by the values it differentiates
        at.  The returned set carries the value tensors (:attr:`SupportSet.values`)."""
        if self.requires_grad:
            return self._learnable_support_set()
        version = self.version()
        if self._sset is None or self._sset_version != version:
            if not self.is_cuda:
                raise RuntimeError(f"{type(self).__name__} must be moved to a CUDA device before use (.to(device))")
            mats = self.mats if self.mode == "generic" or self.ks > 1 else []
            graphs = [GraphHandle.from_csr(self.n, *m) for m in mats]
            self._sset = SupportSet(self.mode, self.n, self.ks, graphs, self.device)
            self._sset_version = version
        return self._sset

    def _learnable_support_set(self) -> SupportSet:
        if not self.is_cuda:
            raise RuntimeError(f"{type(self).__name__} must be moved to a CUDA device before use (.to(device))")
        # a one-support Chebyshev stack ([I], K = 0) multiplies by no matrix: its values are not an input of any
        # convolution and their .grad stays None, as for any tensor the loss does not use
        mats = self.mats if self.mode == "generic" or self.ks > 1 else []
        key = tuple((rp.data_ptr(), rp._version, ci.data_ptr(), ci._version, v.numel()) for rp, ci, v in mats)
        if self._structure is None or self._structure_key != key:
            self._structure = [GraphHandle.from_csr(self.n, rp, ci, v.detach()) for rp, ci, v in mats]
            self._structure_key = key
        graphs = [h.with_values(v) for h, (_, _, v) in zip(self._structure, mats)]
        return SupportSet(self.mode, self.n, self.ks, graphs, self.device, values=[v for _, _, v in mats])

    def matrices_dense(self) -> List[torch.Tensor]:
        """The stored matrices as dense ``(N, N)`` tensors (tests / small graphs only)."""
        return [torch.sparse_csr_tensor(rp.long(), ci.long(), v.detach(), size=(self.n, self.n)).to_dense()
                for rp, ci, v in self.mats]


class ChebSupports(SparseSupports):
    """Sparse-native Chebyshev supports: ``L~`` as CSR plus the number of supports ``Ks`` (one chain)."""

    def __init__(self, n: int, ks: int, rowptr: torch.Tensor, colidx: torch.Tensor, vals: torch.Tensor):
        super().__init__("cheb", n, ks, [(rowptr, colidx, vals)])

    @property
    def rowptr(self):
        return self.mats[0][0]

    @property
    def colidx(self):
        return self.mats[0][1]

    @property
    def vals(self):
        return self.mats[0][2]

    def laplacian_dense(self) -> torch.Tensor:
        """Dense ``L~`` (tests / small graphs only)."""
        return self.matrices_dense()[0]
