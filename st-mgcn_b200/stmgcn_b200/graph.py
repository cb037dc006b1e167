"""Support ingestion: the constant operand of the hot path.

The reference hands ``GCN.forward`` a dense ``(K+1, N, N)`` stack built once by
``Adj_Preprocessor.process`` (``GCN.py:57-97``; stacked ``:95``) and multiplies each slice into the
features (``GCN.py:34-36``).  Here the stack is inspected ONCE per tensor (cached on identity + version; a stack that
requires grad at every forward, and its set carries it so the graph convolutions give it its gradient):

* if it is a Chebyshev stack -- ``A[0] = I`` and ``A[k] = 2 A[1] A[k-1] - A[k-2]`` (``GCN.py:125-135``),
  checked with a random probe -- only ``L~ = A[1]`` is kept, as CSR + CSR^T on the device, and the forward
  runs the recurrence on the features (``SupportSet.mode == "cheb"``, one chain);
* otherwise (``localpool``, hand-made supports) every slice is sparsified on its own and applied
  directly (``mode == "generic"``) -- same kernels, same results as the reference's einsum.

Each matrix kept (``L~``, or a generic slice) is held as CSR, or, when it is too dense to gather, as a dense snapshot
(:class:`DenseGraph`) that the kernels multiply on the tensor cores: :func:`dense_rule` under the ``"auto"`` mode of
``ops.dense_supports()`` (``STMGCN_DENSE_SUPPORTS``), always under ``"on"``, never under ``"off"``.

``SparseSupports`` is the sparse-native handle ``GCN.Adj_Preprocessor.process_sparse`` returns (``ChebSupports``
for ``chebyshev``): it quacks like the reference's tensor where ``Main.py`` touches it (``.to(device)``, ``len``,
``.shape``) but never materialises ``N x N`` polynomials (SURVEY.md section 8(f)-1).  Its ``"cheb"`` stacks are one or
more recurrence chains that share ``T_0 = I``: one for ``chebyshev`` (``L~``), two for ``random_walk_diffusion``
(``P_f^T`` and ``P_b^T``, DCRNN's dual random-walk diffusion).

``LearnableAdjacency`` (``Adj_Preprocessor.process_learnable``) is a learnable graph on a fixed pattern: an ``nn.Module``
whose edge weights are normalised into such a handle's values on the device at every forward.
"""
from __future__ import annotations

import copy
from collections import OrderedDict
from typing import List, Optional

import torch
from torch import nn


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
    def from_dense(cls, mat: torch.Tensor, nnz: Optional[int] = None) -> "GraphHandle":
        """Exact zeros (-0.0 included) are dropped, every other entry (NaN included) is kept verbatim: supports[1] of
        ``Adj_Preprocessor.process`` (``GCN.py:57-97``) becomes the sparse rescaled Laplacian.  ``nnz``: the matrix's
        non-zero count when the caller has it already (then no host sync here)."""
        assert mat.dtype == torch.float32 and mat.dim() == 2 and mat.shape[0] == mat.shape[1]
        if nnz is None:
            rows, cols = (mat != 0).nonzero(as_tuple=True)           # row-major order
        else:
            rows, cols = torch.nonzero_static(mat != 0, size=nnz).unbind(1)
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


class DenseGraph:
    """One ``n x n`` support matrix held dense, for a matrix too dense to gather: the graph convolutions multiply it on
    the tensor cores (``ops.spmm_step`` dispatches on the handle type; stmgcn_dense_mm_step), as the reference's einsum.

    ``mat`` is an fp32 contiguous snapshot (a copy of what it was built from), so the forward and the backward of a step
    multiply by one matrix and an edit of the source after the build reaches neither.  ``copy=False`` holds ``mat``
    itself (detached), for a caller that builds a fresh fp32 contiguous matrix at every forward and never edits it: a
    :class:`LearnableAdjacency` multiplied dense, whose matrix is the output of its scatter.  ``nnz`` is the number of
    stored entries, ``n * n``."""

    def __init__(self, mat: torch.Tensor, copy: bool = True):
        assert mat.dim() == 2 and mat.shape[0] == mat.shape[1]
        self.n, self.nnz, self.device = mat.shape[0], mat.shape[0] * mat.shape[0], mat.device
        if copy:
            self.mat = mat.detach().to(torch.float32, copy=True).contiguous()
        else:
            assert mat.dtype == torch.float32 and mat.is_contiguous()
            self.mat = mat.detach()


# When a dense support matrix is multiplied dense (DenseGraph) instead of gathered from CSR (GraphHandle): from this
# fraction of non-zero entries on, at n >= DENSE_MIN_N.  bench_dense_supports.py (H100, DESIGN.md K1e) puts the crossover
# at 10-10.4 % for N = 512 .. 4096 at F = 4096 and at 10 % (N = 4096) to 16.5 % (N = 512) at F = 768: 17 % is past it
# at every measured size and width.  Below N = 512 a step takes at most 26 us on either path, and CSR stays.
DENSE_MIN_DENSITY = 0.17
DENSE_MIN_N = 512


def dense_rule(n: int, nnz: int) -> bool:
    """Whether an ``n x n`` matrix with ``nnz`` non-zero entries is multiplied dense under the ``"auto"`` mode."""
    return n >= DENSE_MIN_N and nnz >= DENSE_MIN_DENSITY * n * n


class SupportSet:
    """What the kernels need to know about one ``(Ks, N, N)`` support stack.

    ``"cheb"``: ``graphs`` are the recurrence matrices ``X_c`` of chains that share ``T_0 = I``; chain ``c`` owns the
    segments ``1 + cK .. (c+1)K``, ``T_k(X_c)`` with ``K = (Ks - 1) / len(graphs)`` (no graph when ``Ks == 1``).
    ``"generic"``: ``graphs[k]`` is ``A_k``.  A graph is a :class:`GraphHandle` (CSR) or a :class:`DenseGraph`.

    ``values`` (optional): the source tensors of the graphs' stored values, one per graph, when some of them require
    grad: in CSR entry order for a CSR graph (a learnable :class:`SparseSupports`), the ``(N, N)`` matrix itself for a
    :class:`DenseGraph` (a :class:`LearnableAdjacency` multiplied dense).  The graphs hold detached copies (a dense
    matrix: the same storage, built fresh at each forward); the graph convolutions take these tensors as inputs, so their
    gradients reach them -- the SDDMM's at the stored entries, or the whole matrix's (``ops.dense_chain_grad``, or
    ``ops.dense_support_grad`` for a generic slice).

    ``dense`` (optional): the dense ``(Ks, N, N)`` stack the set was converted from, when it requires grad.  The graphs
    hold a snapshot of its slices; the graph convolutions take the stack as their one extra input and give it
    ``dA_k = U_k x^T`` for every slice (``ops.dense_support_grad``), however the forward multiplied by it.
    """

    def __init__(self, mode: str, n: int, ks: int, graphs: List[GraphHandle], device: torch.device,
                 values: Optional[List[torch.Tensor]] = None, dense: Optional[torch.Tensor] = None):
        assert mode in ("cheb", "generic")
        assert len(graphs) == ks if mode == "generic" else (ks - 1) % max(len(graphs), 1) == 0 and (ks == 1) == (not graphs)
        assert values is None or len(values) == len(graphs)
        assert values is None or dense is None
        self.mode, self.n, self.ks, self.graphs, self.device = mode, n, ks, graphs, device
        self.values, self.dense = values, dense

    def grad_values(self) -> tuple:
        """The tensors the graph convolutions take as inputs so that gradients reach them: ``values`` when one of them
        requires grad, ``(dense,)`` when the dense stack requires grad, else ()."""
        if self.dense is not None and self.dense.requires_grad:
            return (self.dense,)
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
    if isinstance(a, (SparseSupports, LearnableAdjacency)):
        return a.version()
    return (a.data_ptr(), a._version, tuple(a.shape), tuple(a.stride()), str(a.device), a.dtype)


def supports_from_dense(a: torch.Tensor) -> SupportSet:
    """Cached conversion of a dense support stack (keyed on tensor identity + in-place version).

    A stack that requires grad is converted at every call and never cached: an optimizer may change it without a version
    bump (fused optimizers, ``.data`` writes), and each forward must multiply by the values it differentiates at.  Its
    set carries the stack (:attr:`SupportSet.dense`), so the graph convolutions give it its gradient."""
    if isinstance(a, (SparseSupports, LearnableAdjacency)):
        return a.support_set()
    if not isinstance(a, torch.Tensor) or a.dim() != 3 or a.shape[1] != a.shape[2]:
        raise ValueError(f"supports must be a (K, N, N) tensor, got {type(a)} {getattr(a, 'shape', None)}")
    if not a.is_cuda:
        raise RuntimeError("stmgcn_b200 has no CPU path: supports must live on a CUDA device "
                           "(the reference moves them there at Main.py:54)")
    if a.requires_grad:
        return _convert_dense(a, dense=a)
    key = _cache_key(a)
    hit = _CACHE.get(key)
    if hit is not None:
        _CACHE.move_to_end(key)
        return hit[1]
    sset = _convert_dense(a)
    _CACHE[key] = (a.detach(), sset)     # keep the storage alive so the data_ptr cannot be recycled under the key
    while len(_CACHE) > _CACHE_MAX:
        _CACHE.popitem(last=False)
    return sset


def _cache_key(a: torch.Tensor) -> tuple:
    """The conversion cache's key of a dense stack: its :func:`support_version` and the dense-supports mode it was
    converted under (a switch of the mode converts it again)."""
    from . import ops
    return support_version(a) + (ops.dense_supports(),)


def _graph_from_dense(mat: torch.Tensor):
    """The handle the kernels multiply ``mat`` through: a :class:`DenseGraph` when the dense-supports mode says so,
    else CSR (:class:`GraphHandle`).  ``"auto"`` decides by :func:`dense_rule` on the non-zero count, the one host sync
    of the conversion (the CSR build then takes the count and does not synchronise again)."""
    from . import ops
    mode = ops.dense_supports()
    if mode == "off":
        return GraphHandle.from_dense(mat)
    if mode == "on":
        return DenseGraph(mat)
    nnz = int((mat != 0).sum())
    return DenseGraph(mat) if dense_rule(mat.shape[0], nnz) else GraphHandle.from_dense(mat, nnz)


def _convert_dense(a: torch.Tensor, dense: Optional[torch.Tensor] = None) -> SupportSet:
    af = a.detach()
    if af.dtype != torch.float32:
        af = af.float()
    ks, n, _ = af.shape
    with torch.cuda.device(a.device):
        if _is_chebyshev_stack(af):
            graphs = [_graph_from_dense(af[1])] if ks > 1 else []
            return SupportSet("cheb", n, ks, graphs, a.device, dense=dense)
        return SupportSet("generic", n, ks, [_graph_from_dense(af[k]) for k in range(ks)], a.device, dense=dense)


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
        return self.support_set_with([v for _, _, v in self.mats])

    def support_set_with(self, values) -> SupportSet:
        """The kernels' set for this handle's index structure with the stored values ``values`` (one tensor per matrix,
        in its CSR entry order) copied in; the set carries ``values`` as the convolutions' inputs, so their gradients
        reach them.  The structure (CSR and CSR^T indices, the transpose's permutation) is cached on the index tensors:
        only the first call converts it (one host sync); the later ones copy values and never synchronise."""
        if not self.is_cuda:
            raise RuntimeError(f"{type(self).__name__} must be moved to a CUDA device before use (.to(device))")
        # a one-support Chebyshev stack ([I], K = 0) multiplies by no matrix: its values are not an input of any
        # convolution and their .grad stays None, as for any tensor the loss does not use
        mats = self.mats if self.mode == "generic" or self.ks > 1 else []
        values = list(values)[:len(mats)]
        key = tuple((rp.data_ptr(), rp._version, ci.data_ptr(), ci._version, v.numel())
                    for (rp, ci, _), v in zip(mats, values))
        if self._structure is None or self._structure_key != key:
            self._structure = [GraphHandle.from_csr(self.n, rp, ci, v.detach().float()) for (rp, ci, _), v in zip(mats, values)]
            self._structure_key = key
        graphs = [h.with_values(v) for h, v in zip(self._structure, values)]
        return SupportSet(self.mode, self.n, self.ks, graphs, self.device, values=values)

    def matrices_dense(self) -> List[torch.Tensor]:
        """The stored matrices as dense ``(N, N)`` tensors (tests / small graphs only)."""
        return [torch.sparse_csr_tensor(rp.long(), ci.long(), v.detach(), size=(self.n, self.n)).to_dense()
                for rp, ci, v in self.mats]


def _stored_entries(adj: torch.Tensor):
    """``(n, rows, cols, vals)`` of a square adjacency, row-major: a dense one's non-zero entries, a sparse (COO / CSR)
    one's stored entries, stored zeros included (repeats summed)."""
    if adj.dim() != 2 or adj.shape[0] != adj.shape[1]:
        raise ValueError(f"the adjacency must be (N, N), got {tuple(adj.shape)}")
    if adj.layout == torch.strided:
        rows, cols = (adj != 0).nonzero(as_tuple=True)
        vals = adj[rows, cols]
    else:
        coo = adj.coalesce() if adj.layout == torch.sparse_coo else adj.to_sparse_coo().coalesce()
        (rows, cols), vals = coo.indices(), coo.values()
    return adj.shape[0], rows, cols, vals.detach().to(torch.float32)


class LearnableAdjacency(nn.Module):
    """A learnable adjacency on a fixed sparsity pattern: ``weight`` (one per stored edge) is its only parameter, and each
    forward normalises it on the device into the supports ``Adj_Preprocessor.process_sparse`` would build from it
    (``ops.AdjNorm``: no host synchronisation, fixed-order sums), so a step that learns the graph can be captured
    (``GraphedStep``) and its edge weights reduced with the model's gradients (``GradBucket(model, adjacency)``).

    Each forward hands the kernels the supports' matrices as CSR, or dense when ``ops.dense_supports()`` says so for the
    pattern (``"auto"``: :func:`dense_rule` on ``N`` and the pattern's entry count, known without a host sync; ``"on"``:
    always; ``"off"``: never).  Dense, the normalised values are scattered into fresh ``(N, N)`` matrices
    (``ops.PatternToDense``) that the graph convolutions multiply on the tensor cores and differentiate whole
    (``ops.dense_chain_grad``); the matrices' gradients are read back at the pattern's entries into ``AdjNorm``'s
    backward.  No ``N^3`` product and no polynomial stack is formed, and the forward still never synchronises.
    Non-finite values: a dense product forms ``0 * x`` for every entry off the pattern too, as the reference's dense
    einsum, so a NaN or Inf in the features reaches every output row (CSR: only rows with an entry in its column).

    Built by ``Adj_Preprocessor.process_learnable``.  The pattern -- the stored entries plus a diagonal slot in every row
    that lacks one when the kind has a diagonal term (``localpool``; ``chebyshev`` with ``2 / lambda_max != 1``) -- is
    built once, as CSR and CSR^T on the module's buffers; ``lambda_max`` is a constant.  Stands in for the support stack
    wherever one goes (``ST_MGCN.forward``'s ``sta_adj_list``, ``GCN.forward``, ``CG_LSTM.forward``): ``.shape ==
    (Ks, N, N)``, ``len``, ``.device``, and ``nn.Module.to``.  The supports are fed to the kernels through a
    :class:`SparseSupports` handle on the module's own index tensors, so the structure is converted once and every
    forward only copies the new values in."""

    def __init__(self, kind: str, order: int, adj: torch.Tensor, scale: float = 1.0, lambda_max: float = 2.0):
        super().__init__()
        if kind not in ("chebyshev", "localpool", "random_walk_diffusion"):
            raise ValueError(f"kind={kind!r}")
        n, rows, cols, vals = _stored_entries(adj)
        nnz_w = rows.numel()
        self.kind, self.order, self.n = kind, int(order), int(n)
        self.ks = {"chebyshev": self.order + 1, "localpool": 1, "random_walk_diffusion": 2 * self.order + 1}[kind]
        if kind == "random_walk_diffusion" and self.ks > 8:
            raise ValueError(f"LearnableAdjacency: random_walk_diffusion with K={self.order} needs {self.ks} supports; the "
                             f"projection kernels take at most 8 supports (K <= 3)")
        self.scale, self.lambda_max = float(scale), float(lambda_max)
        dev = rows.device
        prow, pcol, src = rows, cols, None
        if kind == "localpool" or (kind == "chebyshev" and self.scale != 1.0):
            has = torch.zeros(n, dtype=torch.bool, device=dev)
            has[rows[rows == cols]] = True
            extra = (~has).nonzero().flatten()
            if extra.numel():
                order_ = torch.argsort(torch.cat([rows, extra]) * n + torch.cat([cols, extra]))
                prow, pcol = torch.cat([rows, extra])[order_], torch.cat([cols, extra])[order_]
                src = torch.cat([torch.arange(nnz_w, device=dev), torch.full_like(extra, -1)])[order_]
        nnz = prow.numel()
        if not 0 < n < 2 ** 30 or nnz >= 2 ** 31:
            raise ValueError(f"LearnableAdjacency: n={n} must be in [1, 2^30) and nnz={nnz} below 2^31 (int32 indices)")
        rowptr = torch.zeros(n + 1, dtype=torch.int32, device=dev)
        rowptr[1:] = torch.cumsum(torch.bincount(prow, minlength=n), 0)
        tord = torch.argsort(pcol * n + prow)
        rowptr_t = torch.zeros(n + 1, dtype=torch.int32, device=dev)
        rowptr_t[1:] = torch.cumsum(torch.bincount(pcol, minlength=n), 0)
        self.register_buffer("rowptr", rowptr)
        self.register_buffer("colidx", pcol.to(torch.int32))
        self.register_buffer("rowptr_t", rowptr_t)
        self.register_buffer("colidx_t", prow[tord].to(torch.int32))
        self.register_buffer("perm_t", tord.to(torch.int32))
        self.register_buffer("widx", None if src is None else src.to(torch.int32))
        self.weight = nn.Parameter(vals.clone())
        self._handle: Optional[SparseSupports] = None
        self._handle_key: tuple = ()

    def extra_repr(self) -> str:
        return f"{self.kind}, Ks={self.ks}, N={self.n}, edges={self.weight.numel()}, lambda_max={self.lambda_max:g}"

    @property
    def shape(self):
        return torch.Size((self.ks, self.n, self.n))

    @property
    def device(self):
        return self.weight.device

    @property
    def is_cuda(self):
        return self.weight.is_cuda

    def __len__(self):
        return self.ks

    def pattern(self) -> tuple:
        """``(rowptr, colidx, rowptr_t, colidx_t, perm_t, widx)``: the pattern the normalisation runs on (widx: each
        pattern entry's index in ``weight``, -1 for an added diagonal slot; None when there is no such slot)."""
        return self.rowptr, self.colidx, self.rowptr_t, self.colidx_t, self.perm_t, self.widx

    def version(self) -> tuple:
        """Identity and in-place version of the pattern's tensors (not of ``weight``: its values are read at every
        forward)."""
        return tuple((t.data_ptr(), t._version) for t in self.pattern() if t is not None)

    def edges(self):
        """int64 ``(rows, cols)`` of the stored edges, in ``weight``'s order (row-major), read off the pattern."""
        rows = torch.repeat_interleave(torch.arange(self.n, device=self.rowptr.device),
                                       (self.rowptr[1:] - self.rowptr[:-1]).long(), output_size=self.colidx.numel())
        cols = self.colidx.long()
        if self.widx is not None:            # the stored entries keep their row-major order among the added slots
            keep = self.widx >= 0
            rows, cols = rows[keep], cols[keep]
        return rows, cols

    def learned_adjacency(self) -> torch.Tensor:
        """The current edge weights as a sparse COO ``(N, N)`` tensor on the stored pattern (a detached copy)."""
        return torch.sparse_coo_tensor(torch.stack(self.edges()), self.weight.detach().clone(), (self.n, self.n),
                                       is_coalesced=True)

    def _supports_handle(self) -> SparseSupports:
        key = self.version()
        if self._handle is None or self._handle_key != key:
            blank = torch.empty(self.colidx.numel(), device=self.device)
            if self.kind == "random_walk_diffusion":
                self._handle = SparseSupports("cheb", self.n, self.ks, [(self.rowptr_t, self.colidx_t, blank),
                                                                         (self.rowptr, self.colidx, blank)])
            elif self.kind == "chebyshev":
                self._handle = ChebSupports(self.n, self.ks, self.rowptr, self.colidx, blank)
            else:
                self._handle = SparseSupports("generic", self.n, 1, [(self.rowptr, self.colidx, blank)])
            self._handle_key = key
        return self._handle

    def _values(self):
        """The stored values of the supports' matrices at the current weights, in the handle's matrix order."""
        from . import ops
        vals = ops.AdjNorm.apply(self.weight, self.kind, self.scale, *self.pattern())
        return list(vals) if isinstance(vals, tuple) else [vals]

    def dense(self) -> bool:
        """Whether the forward multiplies the supports' matrices dense under the current ``ops.dense_supports()`` mode
        (``"auto"``: :func:`dense_rule` on the pattern's entry count)."""
        from . import ops
        mode = ops.dense_supports()
        return mode == "on" or (mode == "auto" and dense_rule(self.n, self.colidx.numel()))

    def forward(self) -> SupportSet:
        """The kernels' support set at the current weights: one normalisation launch pair, then the values copied into
        the cached structure (:meth:`SparseSupports.support_set_with`), or, multiplied dense (:meth:`dense`), scattered
        into one fresh ``(N, N)`` matrix per chain (or slice): a set of :class:`DenseGraph`s whose ``values`` are those
        matrices."""
        if not self.is_cuda:
            raise RuntimeError("LearnableAdjacency must be moved to a CUDA device before use (.to(device))")
        handle = self._supports_handle()
        if not self.dense():
            return handle.support_set_with(self._values())
        from . import ops
        mats = handle.mats if handle.mode == "generic" or handle.ks > 1 else []
        dense = [ops.PatternToDense.apply(v, rp, ci) for (rp, ci, _), v in zip(mats, self._values())]
        return SupportSet(handle.mode, self.n, self.ks, [DenseGraph(d, copy=False) for d in dense], self.device,
                          values=dense)

    def supports(self) -> SparseSupports:
        """The supports at the current weights as a fixed handle (detached copies of the values): what
        ``process_sparse`` would return for the learned graph."""
        with torch.no_grad():
            vals = self._values()
        h = self._supports_handle()
        return SparseSupports(h.mode, h.n, h.ks, [(rp, ci, v) for (rp, ci, _), v in zip(h.mats, vals)])

    support_set = forward


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
