"""Shared inputs and row sizes of the kernel-level suites: projection cases, graphs with empty rows and columns,
hand-made and malformed CSR."""
import numpy as np
import scipy.sparse as sp
import torch

from helpers import sm_count


ACTS = [(True, True), (True, False), (False, True), (False, False)]      # (ReLU, bias)


def proj_inputs(ks, p, q, rows, relu, bias, seed):
    """Seeded CPU inputs of one projection case: every fifth row of the stack is zero, and so is every third bias entry,
    so those pre-activations are exactly 0 (ReLU output 0: dZ must be 0 there)."""
    gen = torch.Generator().manual_seed(seed)
    s = torch.randn(ks, rows, p, generator=gen)
    s[:, 4::5] = 0.0
    w = torch.randn(ks * p, q, generator=gen) / p ** 0.5
    bv = torch.randn(q, generator=gen) * 0.3
    bv[::3] = 0.0
    d_out = torch.randn(rows, q, generator=gen)
    return s, w, (bv if bias else None), d_out


def round_tf32(v):
    """``v`` rounded to tf32 (10 mantissa bits, to nearest), as fp64."""
    i = v.float().contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32).double()


def proj_ref_out(s64, w64, b64, relu):
    ks, rows, p = s64.shape
    z = torch.einsum("krp,kpq->rq", s64, w64.reshape(ks, p, -1))
    if b64 is not None:
        z = z + b64
    return z.clamp_min(0) if relu else z


def proj_rows(rows_id):
    """Rows of an exact-fp32 projection case."""
    if rows_id == "waves":      # the 512-row tiles of the TN = 64 tall GEMM fill every SM more than twice, ragged
        return 512 * (2 * sm_count() + 1) + 77
    return rows_id


def fuse_rows(rows_id):
    """(N, B) of a fusion case."""
    if rows_id == "waves":      # more rows than the forward's 64 * SMs per grid pass, twice over, ragged
        return (2 * 64 * sm_count() + 5) // 3 + 1, 3
    return 7, 3


def isolated_matrix(n, seed, kind="isolated", density=0.1):
    """Random n x n float32 matrix.  ``isolated``: about a tenth of the rows empty, a tenth of the columns empty and a
    tenth of the indices with both empty (isolated regions); ``zero``: no entries at all."""
    rng = np.random.default_rng(seed)
    if kind == "zero":
        return np.zeros((n, n), np.float32)
    if n == 1:
        return np.full((1, 1), 0.7, np.float32)
    a = (rng.random((n, n)) < density) * rng.standard_normal((n, n))
    idx = rng.permutation(n)
    k = max(1, n // 10)
    a[idx[:k], :] = 0.0
    a[:, idx[k:2 * k]] = 0.0
    a[idx[2 * k:3 * k], :] = 0.0
    a[:, idx[2 * k:3 * k]] = 0.0
    return a.astype(np.float32)


def tc_shape(rows_id):
    """(N, B) with N * B rows for the tensor-core projection."""
    if rows_id == "waves":
        return (128 * (2 * sm_count() + 1) + 77) // 7 + 1, 7
    return {1: (1, 1), 31: (31, 1), 33: (11, 3), 129: (43, 3)}[rows_id]


def handmade_csr(n, seed, hub_row=0, hub_col=1, scale=True):
    """int32 / float32 CSR ``(rowptr, colidx, vals)`` of an ``n x n`` matrix as a caller might hand-make it: row ``i`` has
    ``i % 10`` entries (every tail length of the SpMM's 4-way unroll, empty rows included), row ``hub_row`` has ``n - 1``
    and column ``hub_col`` is in almost every row; columns are shuffled within each row, every third non-empty row
    repeats one of its entries, and some stored values are ``0.0`` and ``-0.0``.  With ``scale`` each value is divided by
    the larger of its row's and its column's absolute sum (entries counted one by one), so the matrix's 1- and inf-norms,
    and with them its spectral radius, are at most 1."""
    rng = np.random.default_rng(seed)
    rows = []
    for i in range(n):
        deg = n - 1 if i == hub_row else i % 10
        cols = list(rng.choice(n, size=min(deg, n), replace=False))
        if i != hub_row and hub_col not in cols and i % 10 > 1:
            cols[0] = hub_col
        if cols and i % 3 == 0:
            cols.append(cols[int(rng.integers(len(cols)))])             # a repeated (i, j) entry
        cols = list(rng.permutation(cols))
        rows.append(cols)
    vals = [rng.standard_normal(len(c)) for c in rows]
    for i, v in enumerate(vals):
        if len(v) >= 3 and i % 4 == 1:
            v[1] = 0.0
        if len(v) >= 3 and i % 4 == 3:
            v[2] = -0.0
    rowptr = np.concatenate([[0], np.cumsum([len(c) for c in rows])]).astype(np.int32)
    colidx = np.concatenate([np.asarray(c, np.int64) for c in rows]).astype(np.int32)
    data = np.concatenate(vals)
    if scale:
        a, row_of = np.abs(data), np.repeat(np.arange(n), np.diff(rowptr))
        r = np.bincount(row_of, weights=a, minlength=n)
        c = np.bincount(colidx, weights=a, minlength=n)
        data = data / np.maximum(np.maximum(r[row_of], c[colidx]), 1e-30)
    return torch.from_numpy(rowptr), torch.from_numpy(colidx), torch.from_numpy(data.astype(np.float32))


def scipy_of(rowptr, colidx, vals, n):
    """fp64 scipy CSR of a CSR triple, entries verbatim (repeats are summed by every product scipy computes)."""
    return sp.csr_matrix((vals.double().cpu().numpy(), colidx.cpu().numpy(), rowptr.cpu().numpy()), shape=(n, n))


def valid_csr(n=40):
    return handmade_csr(n, 7)


def malformed(case):
    """(n, rowptr, colidx, vals, message) of one malformed CSR, made from a valid one."""
    n = 40
    rp, ci, v = (t.clone() for t in valid_csr(n))
    if case == "rowptr_start":
        rp[0] = 1
        return n, rp, ci, v, "rowptr\\[0\\] is not 0"
    if case == "rowptr_decreasing":
        rp[20] = rp[21] + 1
        return n, rp, ci, v, "rowptr decreases"
    if case == "rowptr_end":
        return n, rp, ci[:-1].clone(), v[:-1].clone(), "rowptr\\[-1\\] is not nnz"
    if case == "short_vals":
        return n, rp, ci, v[:-2].clone(), "vals has .* entries, colidx"
    if case == "col_negative":
        ci[5] = -1
        return n, rp, ci, v, "column index is outside \\[0, 40\\)"
    if case == "col_n":
        ci[-1] = n
        return n, rp, ci, v, "column index is outside \\[0, 40\\)"
    if case == "rowptr_length":
        return n, rp[:-1].clone(), ci, v, "rowptr has 40 entries, n \\+ 1 = 41"
    if case == "dtype":
        return n, rp, ci, v.double(), "must be int32 and vals float32"
    raise KeyError(case)


MALFORMED = ["rowptr_start", "rowptr_decreasing", "rowptr_end", "short_vals", "col_negative", "col_n", "rowptr_length",
             "dtype"]
