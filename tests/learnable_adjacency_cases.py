"""fp64 restatement of a learnable adjacency's normalisation (``LearnableAdjacency`` / ``stmgcn_adj_norm_*``), the
graphs its suites run on, and the dense stacks the model-level references take.  Shared by the host and the GPU suites.

``normalise64`` restates the formulas the kernels implement on the module's own pattern, as torch autograd in fp64: the
degrees are ``index_add`` sums of the stored weights, ``D^-1/2`` is ``pow(-0.5)`` and the random walk's inverse degree
``pow(-1)`` with infinities set to 0 (``GCN.py:99-104``), so its gradient, NaN and Inf included, is torch's.
"""
import torch

import stmgcn_oracle as O

KINDS = ("chebyshev", "localpool", "random_walk_diffusion")


def pattern_of(adj):
    """``(prow, pcol, widx, perm_t)`` int64 on the CPU: a ``LearnableAdjacency``'s pattern in CSR order, each entry's
    index in ``weight`` (-1: an added diagonal slot) and the CSR^T -> CSR permutation."""
    rp = adj.rowptr.long().cpu()
    prow = torch.repeat_interleave(torch.arange(adj.n), rp[1:] - rp[:-1])
    pcol = adj.colidx.long().cpu()
    widx = torch.arange(pcol.numel()) if adj.widx is None else adj.widx.long().cpu()
    return prow, pcol, widx, adj.perm_t.long().cpu()


def normalise64(kind, n, prow, pcol, widx, perm_t, w, scale):
    """The stored values on the pattern: a tensor in CSR order (symmetric kinds) or ``(P_f^T in CSR^T order, P_b^T in
    CSR order)`` (diffusion).  Differentiable in ``w`` (one per stored entry)."""
    stored = widx >= 0
    e_st = stored.nonzero().flatten()
    r, c, ws = prow[e_st], pcol[e_st], w[widx[e_st]]
    nnz = prow.numel()
    if kind == "random_walk_diffusion":
        def inv(deg):
            d = deg.pow(-1)
            return torch.where(torch.isinf(d), torch.zeros_like(d), d)
        d_out = inv(torch.zeros(n, dtype=w.dtype).index_add(0, r, ws))
        d_in = inv(torch.zeros(n, dtype=w.dtype).index_add(0, c, ws))
        vb = torch.zeros(nnz, dtype=w.dtype).index_put((e_st,), ws * d_in[c])
        vf = torch.zeros(nnz, dtype=w.dtype).index_put((e_st,), ws * d_out[r])
        return vf[perm_t], vb
    a = torch.zeros(n, dtype=w.dtype).index_add(0, r, ws).pow(-0.5)
    coef, diag = (-scale, scale - 1.0) if kind == "chebyshev" else (1.0, 1.0)
    vals = torch.zeros(nnz, dtype=w.dtype).index_put((e_st,), coef * ((a[r] * ws) * a[c]))
    if diag != 0.0:
        vals = vals + diag * (prow == pcol).to(w.dtype)
    return vals


def module_values64(adj, w):
    """:func:`normalise64` on a module's pattern at the weights ``w``."""
    prow, pcol, widx, perm_t = pattern_of(adj)
    return normalise64(adj.kind, adj.n, prow, pcol, widx, perm_t, w, adj.scale)


def dense_of(n, rows, cols, vals):
    return torch.zeros(n, n, dtype=vals.dtype, device=vals.device).index_put((rows, cols), vals, accumulate=True)


def module_stack64(adj, w):
    """Dense fp64 ``(Ks, N, N)`` stack of the module's supports at the weights ``w`` (differentiable in ``w``): the
    Chebyshev polynomials of ``L~``, ``[I + D^-1/2 A D^-1/2]``, or the bidirectional diffusion stack."""
    prow, pcol, _, perm_t = pattern_of(adj)
    v = module_values64(adj, w)
    if adj.kind == "random_walk_diffusion":
        vf, vb = v
        pf = dense_of(adj.n, pcol[perm_t], prow[perm_t], vf)
        pb = dense_of(adj.n, prow, pcol, vb)
        return O.chain_stack_dense([pf, pb], adj.order)
    m = dense_of(adj.n, prow, pcol, v)
    if adj.kind == "localpool":
        return m.unsqueeze(0)
    return O.chain_stack_dense([m], adj.order)


def dense_reference_stack(kind, order, a, lam=2.0):
    """The dense fp64 stack of the adjacency ``a`` by the dense preprocessing: ``Adj_Preprocessor.process`` for the
    symmetric kinds, ``O.chain_stack_dense`` of the dense ``P_f^T``, ``P_b^T`` for diffusion (``process`` builds only
    the forward-only ``K+1`` stack)."""
    import GCN
    pre = GCN.Adj_Preprocessor(kind, order, lambda_max=lam)
    if kind != "random_walk_diffusion":
        return pre.process(a)
    return O.chain_stack_dense([pre.random_walk_normalize(a).T, pre.random_walk_normalize(a.T).T], order)


def graph(n, seed, directed=False, loops=True, isolated=True, hub=True, density=0.25):
    """fp64 weighted adjacency: random edges in (0.5, 1.5), some self-loops, an isolated region (row and column 2, when
    ``isolated``) and a hub (row and column 0 full, when ``hub``); symmetric unless ``directed`` (then, with
    ``isolated``, also a sink: row 1 empty)."""
    gen = torch.Generator().manual_seed(seed)
    a = (torch.rand(n, n, generator=gen) < density).double() * (0.5 + torch.rand(n, n, generator=gen, dtype=torch.float64))
    if not directed:
        a = torch.triu(a, 1)
        a = a + a.T
    else:
        a.fill_diagonal_(0.0)
    if loops:
        idx = torch.arange(3, n, 4)
        a[idx, idx] = 0.5 + torch.rand(idx.numel(), generator=gen, dtype=torch.float64)
    if hub:
        a[0, 3:] = 0.7
        if not directed:
            a[3:, 0] = 0.7
    if isolated:
        a[2, :] = 0.0
        a[:, 2] = 0.0
    if directed and isolated:
        a[1, :] = 0.0
    return a


def zero_sum_graph():
    """A directed sparse COO adjacency whose column 2 and row 4 hold only stored zeros (zero in- and out-degrees with
    stored entries), beside ordinary edges."""
    idx = torch.tensor([[0, 0, 1, 1, 3, 4, 4, 5], [1, 2, 2, 3, 0, 0, 5, 3]])
    vals = torch.tensor([1.0, 0.0, 0.0, 0.7, 1.3, 0.0, 0.0, 0.4])
    return torch.sparse_coo_tensor(idx, vals, (6, 6)).coalesce()
