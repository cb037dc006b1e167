"""fp64 references of the support-value gradient (the gradient of a support's stored CSR values) and the graphs its
suites run on.  Shared by the host and the GPU suites.

Two independent restatements:
* ``dvals_formula``: the sparse formula the kernels implement -- the total adjoints G_k of a Chebyshev chain by the
  adjoint Clenshaw recurrence, then d vals[e] = sum_k c_k <G_k[i], T_{k-1}[j]> (c_1 = 1, c_k = 2);
* ``dense_matrix``: the dense (N, N) matrix of a CSR built from a leaf of its values (repeats added), so autograd through
  any dense computation gives d vals at every stored entry.
"""
import torch

import stmgcn_oracle as O
from kernel_cases import handmade_csr


def coo_of(rowptr, colidx):
    """int64 (rows, cols) of a CSR's entries, in storage order."""
    rowptr = rowptr.long()
    rows = torch.repeat_interleave(torch.arange(rowptr.numel() - 1, device=rowptr.device), rowptr[1:] - rowptr[:-1])
    return rows, colidx.long()


def spmm(rows, cols, vals, x, transpose=False):
    """``X x`` (or ``X^T x``) of the matrix with entries (rows, cols, vals); differentiable in ``vals`` and ``x``."""
    if transpose:
        rows, cols = cols, rows
    flat = x.reshape(x.shape[0], -1)
    out = torch.zeros_like(flat).index_add(0, rows, vals[:, None].to(flat.dtype) * flat[cols])
    return out.reshape(x.shape)


def chain_terms(rows, cols, vals, x, order):
    """``[T_0 x .. T_order x]`` of the chain matrix."""
    t = [x]
    if order >= 1:
        t.append(spmm(rows, cols, vals, x))
    for _ in range(2, order + 1):
        t.append(2.0 * spmm(rows, cols, vals, t[-1]) - t[-2])
    return t


def chain_adjoints(rows, cols, vals, u):
    """Total adjoints ``[G_1 .. G_K]`` of a chain given the direct adjoints ``u = [U_0 .. U_K]`` (Clenshaw)."""
    k_ord = len(u) - 1
    g = [None] * (k_ord + 2)
    g[k_ord + 1] = torch.zeros_like(u[0])
    for k in range(k_ord, 0, -1):
        g[k] = u[k].clone()
        if k + 1 <= k_ord:
            g[k] = g[k] + 2.0 * spmm(rows, cols, vals, g[k + 1], transpose=True)
        if k + 2 <= k_ord:
            g[k] = g[k] - g[k + 2]
    return g[1:k_ord + 1]


def dvals_formula(rows, cols, vals, x, u, coefs=None, pattern=None):
    """d vals of a chain (terms T_k x, direct adjoints ``u[k]``) by the sparse formula.  ``coefs``: c_1 .. c_K (default
    1, 2, 2, ..); ``pattern``: (rows, cols) the formula reads at (default the chain's own; the transposed pattern is a
    negative control)."""
    k_ord = len(u) - 1
    t = chain_terms(rows, cols, vals, x, k_ord)
    g = chain_adjoints(rows, cols, vals, u)
    coefs = coefs or [1.0] + [2.0] * (k_ord - 1)
    pr, pc = pattern or (rows, cols)
    out = torch.zeros(rows.numel(), dtype=x.dtype)
    for k in range(1, k_ord + 1):
        out = out + coefs[k - 1] * (g[k - 1].reshape(x.shape[0], -1)[pr] * t[k - 1].reshape(x.shape[0], -1)[pc]).sum(1)
    return out


def dense_matrix(n, rows, cols, vals):
    """Dense (N, N) matrix of the entries, repeats added; differentiable in ``vals``."""
    return torch.zeros(n, n, dtype=vals.dtype, device=vals.device).index_put((rows, cols), vals, accumulate=True)


def dense_chain(mat, order):
    """``[I, T_1(X) .. T_K(X)]`` dense."""
    eye = torch.eye(mat.shape[0], dtype=mat.dtype, device=mat.device)
    polys = [eye]
    if order >= 1:
        polys.append(mat)
    for _ in range(2, order + 1):
        polys.append(2.0 * (mat @ polys[-1]) - polys[-2])
    return polys


def directed_graph(n, seed, density=0.2):
    """fp64 weighted directed adjacency with a sink (row 0), a source (column 1) and an isolated region (2)."""
    gen = torch.Generator().manual_seed(seed)
    a = (torch.rand(n, n, generator=gen) < density).double() * (0.5 + torch.rand(n, n, generator=gen, dtype=torch.float64))
    a.fill_diagonal_(0.0)
    a[0, :] = 0.0
    a[:, 1] = 0.0
    a[2, :] = 0.0
    a[:, 2] = 0.0
    return a


def handmade(n, seed):
    """Hand-made CSR (repeats, unsorted columns, stored zeros, empty rows) of :func:`kernel_cases.handmade_csr`."""
    return handmade_csr(n, seed)


# ---- model-level fp64 reference -------------------------------------------------------------------------------------
def handle_stack(handle, leaves, device):
    """Dense fp64 (Ks, N, N) stack of a SparseSupports handle whose stored values are ``leaves`` (one per matrix)."""
    n = handle.n
    mats = [dense_matrix(n, *[t.to(device) for t in coo_of(rp, ci)], leaf) for (rp, ci, _), leaf in zip(handle.mats, leaves)]
    if handle.mode == "generic":
        return torch.stack(mats)
    order = (handle.ks - 1) // len(mats)
    out = [torch.eye(n, dtype=torch.float64, device=device)]
    for m in mats:
        out += dense_chain(m, order)[1:]
    return torch.stack(out)


def model_reference(params, obs, y, handles, branch_handle, relu=True, device="cpu", window_chunk=None, masks=None):
    """fp64 loss, parameter gradients, d obs and d vals (per handle, per matrix) of ``ST_MGCN`` on the learnable handles
    ``handles``; branch m reads ``handles[branch_handle[m]]`` (one handle may feed several branches).  The MSE is the mean
    over the whole batch; ``window_chunk`` evaluates it in chunks of windows (the windows are independent), summing the
    gradients.  ``masks`` (ReLU only): the ReLU masks of the GPU's own forward, boolean (N, B, q) per GCN in the order
    temporal 0, spatial 0, temporal 1, ... (:func:`record_relu_masks`), so a pre-activation within rounding distance of
    the kink takes the same branch here as in the kernels."""
    import stmgcn_oracle as O
    leaves = {k: v.detach().to(device, torch.float64).clone().requires_grad_(True) for k, v in params.items()}
    vleaves = [[v.detach().to(device, torch.float64).clone().requires_grad_(True) for _, _, v in h.mats] for h in handles]
    obs = obs.detach().to(device, torch.float64)
    y = y.detach().to(device, torch.float64)
    d_obs, loss = torch.zeros_like(obs), 0.0
    b = obs.shape[0]
    chunk = window_chunk or b
    for w0 in range(0, b, chunk):
        o_leaf = obs[w0:w0 + chunk].clone().requires_grad_(True)
        stacks = [handle_stack(h, vl, device) for h, vl in zip(handles, vleaves)]
        mk = None if masks is None else [m_[:, w0:w0 + chunk].to(device) for m_ in masks]
        out = O.dense_st_mgcn(leaves, o_leaf, [stacks[i] for i in branch_handle], relu, masks=mk)
        part = ((out - y[w0:w0 + chunk]) ** 2).sum() / y.numel()
        part.backward()
        d_obs[w0:w0 + chunk] = o_leaf.grad
        loss += float(part)
    grads = {k: v.grad for k, v in leaves.items()}
    return loss, grads, d_obs, [[v.grad for v in vl] for vl in vleaves]


class record_relu_masks:
    """Context manager: the ReLU mask (``out > 0``, boolean (N, B, q)) of every graph convolution the kernels run inside
    it, in launch order (``ST_MGCN``: temporal 0, spatial 0, temporal 1, ...)."""

    def __enter__(self):
        from stmgcn_b200 import ops
        self.ops, self.real, self.masks = ops, ops._proj_fwd, []

        def proj_fwd(*a, **k):
            out = self.real(*a, **k)
            self.masks.append(out > 0)
            return out
        ops._proj_fwd = proj_fwd
        return self

    def __exit__(self, *exc):
        self.ops._proj_fwd = self.real


class ForcedValueReference(O.BF16ModeReference):
    """:class:`O.BF16ModeReference` (rounding, ReLU masks and tapes as there) whose support values are autograd leaves:
    every chain product is an ``index_add`` over the handle's stored entries (:func:`spmm`), so the backward also gives
    d vals.  Chebyshev-chain handles only; branch m reads ``handles[branch_handle[m]]``.  :meth:`value_grads` returns the
    parameter gradients, d obs and d vals."""

    def __init__(self, params, handles, branch_handle, relu=True, rounding=True, relu_masks=None, device="cpu",
                 dtype=torch.float64):
        import scipy.sparse as sp
        assert all(h.mode == "cheb" and h.ks > 1 for h in handles)
        chains = []
        for i in branch_handle:             # the parent's chains: only for its bookkeeping, the products are ours
            h = handles[i]
            chains.append([sp.csr_matrix((v.detach().double().cpu().numpy(), ci.cpu().numpy(), rp.cpu().numpy()),
                                         shape=(h.n, h.n)) for rp, ci, v in h.mats])
        super().__init__(params, chains, handles[0].ks, relu, rounding, relu_masks, device, dtype)
        self.branch_handle = list(branch_handle)
        self.coo = [[tuple(t.to(self.dev) for t in coo_of(rp, ci)) for rp, ci, _ in h.mats] for h in handles]
        self.vleaves = [[v.detach().to(self.dev, dtype).clone().requires_grad_(True) for _, _, v in h.mats]
                        for h in handles]

    def _stack(self, m, x, spatial, tape_s=None):
        n = x.shape[0]
        flat = x.reshape(n, -1)
        rnd = self._rnd if spatial else (lambda v: v)

        def forced(k, computed):
            if tape_s is None:
                return computed
            return tape_s[k].reshape(n, -1) + (computed - computed.detach())
        used, comp = [forced(0, flat)] + [None] * (self.ks - 1), [flat] + [None] * (self.ks - 1)
        h = self.branch_handle[m]
        k_ord = (self.ks - 1) // len(self.coo[h])
        for c, ((rows, cols), vals) in enumerate(zip(self.coo[h], self.vleaves[h])):
            seg = [0] + list(range(1 + c * k_ord, 1 + (c + 1) * k_ord))
            for j in range(1, len(seg)):
                y = spmm(rows, cols, vals, rnd(used[seg[j - 1]]))
                if j > 1:
                    y = 2.0 * y - used[seg[j - 2]]
                comp[seg[j]], used[seg[j]] = y, forced(seg[j], y)
        return used, comp

    def value_grads(self, obs, y, tapes=None):
        """(loss, parameter gradients, d obs, d vals per handle and matrix) of the MSE over the whole batch."""
        p = self.leaves()
        obs = torch.as_tensor(obs).to(self.dev, self.dt).detach().clone().requires_grad_(True)
        out = self.forward(p, obs, tapes)
        loss = torch.mean((out - torch.as_tensor(y).to(self.dev, self.dt)) ** 2)
        flat = [v for vl in self.vleaves for v in vl]
        keys = list(p)
        res = torch.autograd.grad(loss, [p[k] for k in keys] + [obs] + flat)
        grads = dict(zip(keys, res[:len(keys)]))
        it = iter(res[len(keys) + 1:])
        return float(loss), grads, res[len(keys)], [[next(it) for _ in vl] for vl in self.vleaves]
