"""``torch.autograd.Function`` wrappers around the C ABI -- host plumbing only.

Every tensor the kernels touch is allocated here through torch's caching allocator on the current stream
(the library never allocates, SURVEY.md section 8(b) "ownership").  All feature tensors are fp32
"node-major": ``(N, B, p)`` contiguous, rows ``r = n*B + b``.

Functions (reference lines they replace):
  ObsToNodeMajor   STMGCN.py:36,39 (sum over C, permute) and :47 (row order of the shared LSTM); only when obs requires grad
  ChebGCN          GCN.py:24-43 on a sparse L~ (recurrence on features) -> out (N,B,q)
  TemporalPool     STMGCN.py:40-42: GCN over time-as-features + residual + sum over regions -> (B,T)
  ContextGate      STMGCN.py:42-43: /N, fc, relu, fc (same weights), sigmoid -> s (B,T)
  SharedLSTM       STMGCN.py:44,47-50: modulate + 3-layer shared LSTM (lstm16.cu / lstm.cu: one call each way)
  FuseOut          STMGCN.py:116-118: sum over graphs + output FC -> (B,N,C)
  AdjNorm          GCN.py:99-111 on a fixed pattern: a learnable adjacency's weights -> its supports' stored values
  PatternToDense   a learnable adjacency's stored values -> the dense matrix they form, when it is multiplied dense
"""
from __future__ import annotations

import math
import os
from typing import List, Optional, Sequence

import torch

from . import _lib
from .graph import DenseGraph, SupportSet

L = _lib.lib


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


_LSTM_PATH = os.environ.get("STMGCN_LSTM_PATH", "tc")


def lstm_path() -> str:
    """"tc": tensor-core (wgmma) kernels where shapes allow (LSTM: H = 64, C <= 4; projection: p = q = 64); "fma": exact-fp32 FFMA kernels."""
    return _LSTM_PATH


def set_lstm_path(path: str) -> None:
    global _LSTM_PATH
    if path not in ("tc", "fma"):
        raise ValueError(path)
    _LSTM_PATH = path


_DENSE_SUPPORTS = os.environ.get("STMGCN_DENSE_SUPPORTS", "auto")


def dense_supports() -> str:
    """How a dense support stack's matrices are multiplied: "auto" (dense on the tensor cores when ``graph.dense_rule``
    says so, CSR gathers otherwise), "on" (always dense), "off" (always CSR).  Sparse handles always stay CSR."""
    return _DENSE_SUPPORTS


def set_dense_supports(mode: str) -> None:
    global _DENSE_SUPPORTS
    if mode not in ("auto", "on", "off"):
        raise ValueError(f"dense supports mode {mode!r}: 'auto', 'on' or 'off'")
    _DENSE_SUPPORTS = mode


if _DENSE_SUPPORTS not in ("auto", "on", "off"):
    raise ValueError(f"STMGCN_DENSE_SUPPORTS={_DENSE_SUPPORTS!r}: 'auto', 'on' or 'off'")


# The module-level limits of the kernels, the numbers the C entry points enforce (include/stmgcn_b200.h).  The modules
# check them before a step's first launch (check_limits), so a configuration beyond one raises at once, naming the limit,
# instead of failing after some kernels ran or, worse, only in its backward.
LIMITS = {
    "M": 8,                 # graph branches fused by stmgcn_fuse_out_*
    "supports": 8,          # supports per GCN (the projections' segments)
    "C": 4,                 # input_dim of the shared LSTM (both kernel families)
    "L": 8,                 # LSTM layers (both kernel families)
    "H": 128,               # lstm_hidden_dim, a multiple of 4 (exact-fp32 LSTM; the tensor cores take H = 64)
    "T": 2048,              # seq_len: the context gate (stmgcn_gate_*)
    "q": 8192,              # output width of a GCN projection (stmgcn_proj_*)
    "C*G+C": 12288,         # the output layer's weights and bias in the fusion backward's 48 KB of shared memory
}


def check_limits(m: Optional[int] = None, ks: Optional[int] = None, c_in: Optional[int] = None,
                 n_layers: Optional[int] = None, hid: Optional[int] = None, t_len: Optional[int] = None,
                 gcn_hid: Optional[int] = None) -> None:
    """Raise ``ValueError`` naming every limit of :data:`LIMITS` the given sizes exceed (None: not checked).  ``gcn_hid``
    with ``c_in`` also checks the fusion's ``C*G + C``.  Launches nothing."""
    faults = []
    if m is not None and not 1 <= m <= LIMITS["M"]:
        faults.append(f"M={m} graphs (at most {LIMITS['M']})")
    if ks is not None and not 1 <= ks <= LIMITS["supports"]:
        faults.append(f"{ks} supports per GCN (at most {LIMITS['supports']})")
    if c_in is not None and not 1 <= c_in <= LIMITS["C"]:
        faults.append(f"input_dim C={c_in} (at most {LIMITS['C']})")
    if n_layers is not None and not 1 <= n_layers <= LIMITS["L"]:
        faults.append(f"lstm_num_layers L={n_layers} (at most {LIMITS['L']})")
    if hid is not None and not (hid > 0 and hid % 4 == 0 and hid <= LIMITS["H"]):
        faults.append(f"lstm_hidden_dim H={hid} (a multiple of 4, at most {LIMITS['H']})")
    if t_len is not None and not 1 <= t_len <= LIMITS["T"]:
        faults.append(f"seq_len T={t_len} (at most {LIMITS['T']})")
    if gcn_hid is not None and not 1 <= gcn_hid <= LIMITS["q"]:
        faults.append(f"GCN hidden_dim {gcn_hid} (at most {LIMITS['q']})")
    if gcn_hid is not None and c_in is not None and c_in * gcn_hid + c_in > LIMITS["C*G+C"]:
        faults.append(f"output layer C*G + C = {c_in * gcn_hid + c_in} floats (at most {LIMITS['C*G+C']})")
    if faults:
        raise ValueError("stmgcn_b200: configuration beyond the kernels' limits: " + "; ".join(faults))


def _p(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _f32c(t: torch.Tensor) -> torch.Tensor:
    if t.dtype != torch.float32:
        t = t.float()
    return t if t.is_contiguous() else t.contiguous()


def _require_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("stmgcn_b200 kernels need CUDA tensors (there is no CPU fallback)")


# --------------------------------------------------------------------------------------------------
# raw helpers (no autograd)
# --------------------------------------------------------------------------------------------------
def spmm_step(g, transpose: bool, alpha: float, x: torch.Tensor, beta: float, z: Optional[torch.Tensor],
              gamma: float, u: Optional[torch.Tensor], y: torch.Tensor) -> None:
    """``y = alpha * op(A) x + beta * z + gamma * u`` on ``(N, F)`` views; op(A) = A, or A^T with ``transpose``.  A
    :class:`DenseGraph` is multiplied dense on the tensor cores, a CSR handle by the row gather."""
    n = g.n
    f_total = x.numel() // n
    if isinstance(g, DenseGraph):
        _lib.check(L.stmgcn_dense_mm_step(n, g.mat.data_ptr(), n, int(transpose), alpha, x.data_ptr(), beta, _p(z), gamma,
                                          _p(u), y.data_ptr(), f_total, _stream()), "dense_mm_step")
        return
    rowptr, colidx, vals = g.export(transpose)
    _lib.check(L.stmgcn_cheb_spmm_step(n, rowptr.data_ptr(), colidx.data_ptr(), vals.data_ptr(), alpha, x.data_ptr(),
                                       beta, _p(z), gamma, _p(u), y.data_ptr(), f_total, _stream()), "cheb_spmm_step")


def spmm_step16(g, transpose: bool, alpha: float, x16: torch.Tensor, beta: float, z: Optional[torch.Tensor],
                gamma: float, u: Optional[torch.Tensor], y: torch.Tensor, y16: Optional[torch.Tensor]) -> None:
    """:func:`spmm_step` with the gathered operand read from its bf16 copy ``x16``; writes the bf16 copy of ``y`` to ``y16``."""
    f_total = y.numel() // g.n
    if isinstance(g, DenseGraph):
        _lib.check(L.stmgcn_dense_mm_step16(g.n, g.mat.data_ptr(), g.n, int(transpose), alpha, x16.data_ptr(), beta, _p(z),
                                            gamma, _p(u), y.data_ptr(), _p(y16), f_total, _stream()), "dense_mm_step16")
        return
    rowptr, colidx, vals = g.export(transpose)
    _lib.check(L.stmgcn_cheb_spmm_step16(g.n, rowptr.data_ptr(), colidx.data_ptr(), vals.data_ptr(), alpha,
                                         x16.data_ptr(), beta, _p(z), gamma, _p(u), y.data_ptr(), _p(y16), f_total,
                                         _stream()), "cheb_spmm_step16")


def to_bf16(x: torch.Tensor) -> torch.Tensor:
    y = torch.empty(x.shape, device=x.device, dtype=torch.bfloat16)
    _lib.check(L.stmgcn_to_bf16(x.data_ptr(), y.data_ptr(), x.numel(), _stream()), "to_bf16")
    return y


def _gather16(sset: SupportSet, x: torch.Tensor) -> bool:
    """bf16 gather copies: only in the single-plane (bf16 arithmetic) mode, for the recurrence chains of a "cheb" stack."""
    return lstm_planes() == 1 and sset.mode == "cheb" and (x.numel() // sset.graphs[0].n) % 8 == 0 and x.numel() % 8 == 0


def cheb_stack_(sset: SupportSet, s: torch.Tensor, gather16: bool = False) -> None:
    """Fill ``s[1:]`` from ``s[0]``;  s: (Ks, N, B, p).  ``gather16``: allow bf16 gather copies (bf16-arithmetic mode only).

    One recurrence per chain of the support set (SupportSet), each over its own segments of ``s``."""
    if sset.mode != "cheb":
        raise AssertionError("generic supports are stacked by cheb_stack_generic")
    for c, g in enumerate(sset.graphs):
        _cheb_chain_(g, [s[i] for i in sset.chain_segments(c)], gather16 and _gather16(sset, s[0]))


def _cheb_chain_(g, t: List[torch.Tensor], gather16: bool) -> None:
    """``t[k] = T_k(X) t[0]`` for k >= 1, X the matrix of ``g``: T_1 = X t_0, T_k = 2 X T_{k-1} - T_{k-2}."""
    ks = len(t)
    if gather16:
        # bf16 mode: every step gathers from the bf16 copy of the previous term (half the gather volume)
        src = to_bf16(t[0])
        nxt = torch.empty_like(src) if ks > 2 else None
        for k in range(1, ks):
            out16 = nxt if k < ks - 1 else None
            spmm_step16(g, False, 1.0 if k == 1 else 2.0, src, 0.0 if k == 1 else -1.0, None if k == 1 else t[k - 2],
                        0.0, None, t[k], out16)
            src, nxt = out16, src
        return
    spmm_step(g, False, 1.0, t[0], 0.0, None, 0.0, None, t[1])
    for k in range(2, ks):
        spmm_step(g, False, 2.0, t[k - 1], -1.0, t[k - 2], 0.0, None, t[k])


def cheb_stack_generic(sset: SupportSet, x: torch.Tensor) -> torch.Tensor:
    """Generic supports: S_k = A_k x for every k (including k = 0)."""
    s = torch.empty((sset.ks,) + tuple(x.shape), device=x.device, dtype=torch.float32)
    for k in range(sset.ks):
        spmm_step(sset.graphs[k], False, 1.0, x, 0.0, None, 0.0, None, s[k])
    return s


def build_stack(sset: SupportSet, x: torch.Tensor, gather16: bool = False) -> torch.Tensor:
    if sset.mode == "cheb":
        s = torch.empty((sset.ks,) + tuple(x.shape), device=x.device, dtype=torch.float32)
        s[0].copy_(x)
        cheb_stack_(sset, s, gather16)
        return s
    return cheb_stack_generic(sset, x)


def adjoint_stack_(sset: SupportSet, u: torch.Tensor, need_dx: bool = True) -> Optional[torch.Tensor]:
    """Given U_k = dZ W_k^T stacked in ``u`` (Ks, N, B, p) return dX (N, B, p); ``u`` is clobbered.

    cheb: one adjoint Clenshaw per chain with X_c^T (SURVEY.md section 8(a)), each adding its part into U_0 (T_0 = I is
    shared); generic: sum_k A_k^T U_k.  Afterwards ``u[k]`` holds, for every segment k >= 1 of a chain, the total adjoint
    G_k = dL/dT_k that :func:`support_value_grads` needs.  ``need_dx=False``: only that (cheb: each chain's last step
    into U_0 is skipped; generic: nothing to do); returns None.
    """
    if sset.mode == "cheb":
        for c, g in enumerate(sset.graphs):
            segs = [u[i] for i in sset.chain_segments(c)]
            if need_dx:
                _adjoint_chain_(g, segs)
            else:
                _adjoint_chain_(g, segs, False)
        return u[0] if need_dx else None
    if not need_dx:
        return None
    out = torch.empty_like(u[0])
    acc = None
    for k in range(sset.ks):
        tgt = out if (k % 2 == 0) else torch.empty_like(out)
        spmm_step(sset.graphs[k], True, 1.0, u[k], 0.0, None, 1.0 if acc is not None else 0.0, acc, tgt)
        acc = tgt
    return acc


def _adjoint_chain_(g, u: List[torch.Tensor], into_u0: bool = True) -> None:
    """Adjoint of :func:`_cheb_chain_`: ``u[0] += sum_{k>=1} T_k(X)^T u[k]``; ``u[1:]`` is overwritten with the Clenshaw
    b_k, which is G_k = dL/dT_k.  ``into_u0=False`` stops there (``u[0]`` untouched)."""
    k_ord = len(u) - 1
    # b_K = U_K (in place).  b_k = U_k + 2 X^T b_{k+1} - b_{k+2}  written over U_k.
    # (always fp32 gathers here, also in the bf16-arithmetic mode: rounding b_{k+1} to bf16 before every gather puts
    # ~1.5e-2 into dX on the golden case -- the Clenshaw sum cancels -- and pushed one LSTM weight gradient to 2.2e-2,
    # past the 2e-2 bar of that mode; measured.  The forward stack keeps its bf16 gather copies.)
    for k in range(k_ord - 1, 0, -1):
        z = u[k + 2] if k + 2 <= k_ord else None
        spmm_step(g, True, 2.0, u[k + 1], -1.0 if z is not None else 0.0, z, 1.0, u[k], u[k])
    if not into_u0:
        return
    z = u[2] if k_ord >= 2 else None
    spmm_step(g, True, 1.0, u[1], -1.0 if z is not None else 0.0, z, 1.0, u[0], u[0])


def sddmm_tiles(f_total: int) -> int:
    """Column tiles of :func:`csr_sddmm_` (include/stmgcn_b200.h, stmgcn_csr_sddmm): float4 lanes when f_total % 4 == 0."""
    width = 128 if f_total % 4 == 0 else 32
    return (f_total + width - 1) // width


def csr_sddmm_(g, terms, dvals: torch.Tensor, round_b16: bool = False) -> None:
    """``dvals[e] += sum_t coef_t <A_t[i, :], B_t[j, :]>`` over the stored entries e = (i, j) of ``g``'s CSR, in its
    entry order; ``terms``: (A_t, B_t, coef_t) with A_t, B_t (N, ...) fp32 contiguous.  ``round_b16``: B rounded to bf16.
    Sparse handles only: a dense stack's gradient is ``dense_support_grad``'s, and a sparse handle is never densified."""
    if isinstance(g, DenseGraph):
        raise AssertionError("csr_sddmm_ takes CSR handles only: a DenseGraph's gradient is dense_support_grad's")
    rowptr, colidx, _ = g.export(False)
    f_total = terms[0][0].numel() // g.n
    tiles = sddmm_tiles(f_total)
    work = torch.empty(tiles * g.nnz, device=dvals.device, dtype=torch.float32) if tiles > 1 and g.nnz else None
    a = _lib.ptr_array([t[0].data_ptr() for t in terms])
    b = _lib.ptr_array([t[1].data_ptr() for t in terms])
    coef = _lib.float_array([float(t[2]) for t in terms])
    _lib.check(L.stmgcn_csr_sddmm(g.n, rowptr.data_ptr(), colidx.data_ptr(), g.nnz, len(terms), a, b, coef,
                                  int(round_b16), f_total, _p(work), 0 if work is None else work.numel(),
                                  dvals.data_ptr(), _stream()), "csr_sddmm")


def support_value_grads(sset: SupportSet, s: torch.Tensor, u: torch.Tensor, x: Optional[torch.Tensor],
                        round_b16: bool, need: Sequence[bool]) -> List[Optional[torch.Tensor]]:
    """The gradient of each graph's stored values, None where ``need`` is False: CSR entry order for a CSR handle, the
    whole ``(N, N)`` matrix for a :class:`DenseGraph`.  ``u`` after :func:`adjoint_stack_`; ``s`` the forward stack;
    ``x`` the input (generic supports only).

    cheb, chain X with terms T_0 .. T_K:  dX = sum_k c_k G_k T_{k-1}^T, c_1 = 1, c_k = 2 (k >= 2): at the stored entries,
    one SDDMM launch per chain over its own segments, or everywhere, one :func:`dense_chain_grad` launch (``round_b16``:
    the bf16 copies the forward multiplied); generic S_k = A_k x:  dA_k = U_k x^T, at the stored entries or everywhere
    (:func:`dense_support_grad`)."""
    grads: List[Optional[torch.Tensor]] = []
    for c, g in enumerate(sset.graphs):
        if not need[c]:
            grads.append(None)
            continue
        if sset.mode == "cheb":
            seg = sset.chain_segments(c)
            terms = [(u[seg[k]], s[seg[k - 1]], 1.0 if k == 1 else 2.0) for k in range(1, len(seg))]
        else:
            terms = [(u[c], x, 1.0)]
        if isinstance(g, DenseGraph):
            grads.append(dense_chain_grad(terms, round_b16) if sset.mode == "cheb"
                         else dense_support_grad(u[c:c + 1], x)[0])
            continue
        dv = torch.zeros(g.nnz, device=u.device, dtype=torch.float32)
        csr_sddmm_(g, terms, dv, round_b16 and sset.mode == "cheb")
        grads.append(dv)
    return grads


def dense_chain_grad(terms, round_b16: bool = False) -> torch.Tensor:
    """``sum_t coef_t A_t B_t^T`` (stmgcn_dense_chain_grad), the ``(N, N)`` gradient of a dense recurrence matrix;
    ``terms``: (A_t, B_t, coef_t) with A_t, B_t (N, ...) fp32 contiguous.  ``round_b16``: B rounded to bf16."""
    n = terms[0][0].shape[0]
    out = torch.empty((n, n), device=terms[0][0].device, dtype=torch.float32)
    a = _lib.ptr_array([t[0].data_ptr() for t in terms])
    b = _lib.ptr_array([t[1].data_ptr() for t in terms])
    coef = _lib.float_array([float(t[2]) for t in terms])
    _lib.check(L.stmgcn_dense_chain_grad(n, terms[0][0].numel() // n, len(terms), a, b, coef, int(round_b16),
                                         out.data_ptr(), _stream()), "dense_chain_grad")
    return out


def dense_support_grad(u: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """``dA_k = U_k x^T`` for every slice k (stmgcn_dense_support_grad): ``u`` (Ks, N, ...) the projection backward's U
    before the adjoint Clenshaw, ``x`` (N, ...) the features the slices multiplied; both fp32 contiguous.  (Ks, N, N)."""
    ks, n = u.shape[0], u.shape[1]
    da = torch.empty((ks, n, n), device=u.device, dtype=torch.float32)
    _lib.check(L.stmgcn_dense_support_grad(n, x.numel() // n, ks, u.data_ptr(), u[0].numel(), x.data_ptr(),
                                           da.data_ptr(), _stream()), "dense_support_grad")
    return da


def _support_grads(ctx, s: torch.Tensor, u: Optional[torch.Tensor], x: Optional[torch.Tensor], need_dx: bool,
                   round16: bool):
    """The graph convolutions' shared backward tail: (dX or None, the gradients of their extra inputs).  ``u`` from the
    projection backward (None when nothing needs it); a dense stack's gradient is taken from it before the adjoint
    Clenshaw overwrites it, a sparse set's value gradients after."""
    sset, need_v = ctx.sset, ctx.needs_input_grad[5:]
    extra = [None] * len(need_v)
    dense = sset.dense is not None and any(need_v)
    if dense:
        extra[0] = dense_support_grad(u, s[0] if x is None else x).to(sset.dense.dtype)
    dx = None
    if need_dx:
        dx = adjoint_stack_(sset, u)
    elif any(need_v) and not dense:
        adjoint_stack_(sset, u, False)          # G_k into u for the value gradients only
    if any(need_v) and not dense:
        extra = support_value_grads(sset, s, u, x, round16, need_v)
    return dx, extra


NORM_KINDS = {"chebyshev": 0, "localpool": 1, "random_walk_diffusion": 2}      # STMGCN_NORM_* of the C ABI


def _norm_args(kind: str, pattern, w: torch.Tensor, scale: float):
    """The pattern and weight arguments stmgcn_adj_norm_fwd / _bwd share: ``pattern`` is (rowptr, colidx, rowptr_t,
    colidx_t, perm_t, widx or None) int32 on the device."""
    rowptr, colidx, rowptr_t, colidx_t, perm_t, widx = pattern
    return (NORM_KINDS[kind], rowptr.numel() - 1, rowptr.data_ptr(), colidx.data_ptr(), rowptr_t.data_ptr(),
            colidx_t.data_ptr(), perm_t.data_ptr(), colidx.numel(), _p(widx), w.data_ptr(), w.numel(), scale)


class AdjNorm(torch.autograd.Function):
    """The stored values of a learnable adjacency's supports from its edge weights, on its fixed pattern
    (stmgcn_adj_norm_fwd / _bwd): ``L~`` (chebyshev) or ``I + D^-1/2 A D^-1/2`` (localpool) in CSR order, or
    ``(P_f^T in CSR^T order, P_b^T in CSR order)`` (random_walk_diffusion).  Backward: d weight, the direct and the
    degree terms, in a fixed order.  Allocates through torch and never synchronises, so it is captured by a CUDA graph;
    the kernels read ``weight`` at its own address, so a replay sees in-place optimizer updates."""

    @staticmethod
    def forward(ctx, weight, kind: str, scale: float, *pattern):
        _require_cuda(weight, pattern[0])
        w = _f32c(weight.detach())
        n, nnz = pattern[0].numel() - 1, pattern[1].numel()
        diff = kind == "random_walk_diffusion"
        work = torch.empty(2 * n, device=w.device, dtype=torch.float32)
        vals = torch.empty(nnz, device=w.device, dtype=torch.float32)
        vals_t = torch.empty(nnz, device=w.device, dtype=torch.float32) if diff else None
        _lib.check(L.stmgcn_adj_norm_fwd(*_norm_args(kind, pattern, w, scale), work.data_ptr(), work.numel(),
                                         vals.data_ptr(), _p(vals_t), _stream()), "adj_norm_fwd")
        ctx.kind, ctx.scale, ctx.pattern = kind, scale, pattern
        ctx.save_for_backward(w)
        return (vals_t, vals) if diff else vals

    @staticmethod
    def backward(ctx, *grads):
        (w,) = ctx.saved_tensors
        pattern = ctx.pattern
        n, nnz = pattern[0].numel() - 1, pattern[1].numel()
        g_t, g = (_f32c(grads[0]), _f32c(grads[1])) if ctx.kind == "random_walk_diffusion" else (None, _f32c(grads[0]))
        work = torch.empty(3 * n + nnz, device=w.device, dtype=torch.float32)
        dw = torch.empty_like(w)
        _lib.check(L.stmgcn_adj_norm_bwd(*_norm_args(ctx.kind, pattern, w, ctx.scale), g.data_ptr(), _p(g_t),
                                         work.data_ptr(), work.numel(), dw.data_ptr(), _stream()), "adj_norm_bwd")
        return (dw, None, None) + (None,) * len(pattern)


def pattern_scatter(vals: torch.Tensor, rowptr: torch.Tensor, colidx: torch.Tensor) -> torch.Tensor:
    """The ``(N, N)`` matrix of a CSR pattern's values (stmgcn_pattern_scatter): zeros off the pattern, repeated entries
    added in entry order; ``vals`` fp32 contiguous in the order of ``(rowptr, colidx)``."""
    n = rowptr.numel() - 1
    dense = torch.empty((n, n), device=vals.device, dtype=torch.float32)
    _lib.check(L.stmgcn_pattern_scatter(n, rowptr.data_ptr(), colidx.data_ptr(), colidx.numel(), vals.data_ptr(),
                                        dense.data_ptr(), _stream()), "pattern_scatter")
    return dense


def pattern_gather(dense: torch.Tensor, rowptr: torch.Tensor, colidx: torch.Tensor) -> torch.Tensor:
    """``dense[i, j]`` at every entry ``(i, j)`` of a CSR pattern, in its order (stmgcn_pattern_gather)."""
    dv = torch.empty(colidx.numel(), device=dense.device, dtype=torch.float32)
    _lib.check(L.stmgcn_pattern_gather(rowptr.numel() - 1, rowptr.data_ptr(), colidx.data_ptr(), colidx.numel(),
                                       dense.data_ptr(), dv.data_ptr(), _stream()), "pattern_gather")
    return dv


class PatternToDense(torch.autograd.Function):
    """The ``(N, N)`` matrix a pattern's stored values form (:func:`pattern_scatter`): ``vals`` in the order of the CSR
    ``(rowptr, colidx)``.  Backward: the matrix's gradient read back at the entries (:func:`pattern_gather`).  A fresh
    matrix at every call; no host synchronisation."""

    @staticmethod
    def forward(ctx, vals, rowptr, colidx):
        _require_cuda(vals, rowptr)
        ctx.pattern = (rowptr, colidx)
        return pattern_scatter(_f32c(vals.detach()), rowptr, colidx)

    @staticmethod
    def backward(ctx, d_dense):
        return pattern_gather(_f32c(d_dense), *ctx.pattern), None, None


def _proj_images(w: torch.Tensor, ks: int, p: int, need_bwd: bool):
    """Tensor-core operand images (forward, backward or None) of the projection weights (p = q = 64, ks <= 8), or
    (None, None) when the tensor-core path does not apply.  Packed from ``w`` as it is now, on every call."""
    if lstm_path() != "tc" or p != 64 or w.shape[1] != 64 or ks > 8:
        return None, None
    img_f = torch.empty(ks * 64 * 64 * 2, device=w.device, dtype=torch.float32)
    img_b = torch.zeros((2 if ks > 4 else 1) * 2 * 2 * 256 * 32, device=w.device, dtype=torch.float32) if need_bwd else None
    _lib.check(L.stmgcn_proj_pack_tc(w.data_ptr(), ks, img_f.data_ptr(), _p(img_b), _stream()), "proj_pack_tc")
    return img_f, img_b


def _proj_fwd(s: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], act: int, pool: Optional[torch.Tensor],
              b_inner: int, wimg: Optional[torch.Tensor] = None) -> torch.Tensor:
    ks, n, b, p = s.shape
    q = w.shape[1]
    out = torch.empty((n, b, q), device=s.device, dtype=torch.float32)
    _lib.check(L.stmgcn_proj_fwd(s.data_ptr(), n * b * p, ks, n * b, p, w.data_ptr(), _p(bias), q, act,
                                 out.data_ptr(), _p(pool), b_inner, _p(wimg), _stream()), "proj_fwd")
    return out


def _proj_bwd(s: torch.Tensor, w: torch.Tensor, act: int, out: torch.Tensor, d_out: Optional[torch.Tensor],
              d_bcast: Optional[torch.Tensor], scale: float, b_inner: int, need_bias: bool, need_u: bool,
              wimg_t: Optional[torch.Tensor] = None, need_w: bool = True):
    """(dw, db, u), each None unless asked for (need_w, need_bias, need_u): nothing is launched for a gradient not asked for."""
    ks, n, b, p = s.shape
    q = w.shape[1]
    dw = torch.zeros_like(w, dtype=torch.float32) if need_w else None
    db = torch.zeros(q, device=s.device, dtype=torch.float32) if need_bias else None
    dz = torch.empty((n * b, q), device=s.device, dtype=torch.float32)
    u = torch.empty_like(s) if need_u else None
    wt = w.t().contiguous() if need_u else None
    _lib.check(L.stmgcn_proj_bwd(s.data_ptr(), n * b * p, ks, n * b, p, _p(wt), q, act, out.data_ptr(), _p(d_out),
                                 _p(d_bcast), scale, b_inner, dz.data_ptr(), _p(dw), _p(db), _p(u),
                                 n * b * p, _p(wimg_t), _stream()), "proj_bwd")
    return dw, db, u


# --------------------------------------------------------------------------------------------------
# autograd Functions
# --------------------------------------------------------------------------------------------------
def obs_to_node_major(obs: torch.Tensor):
    """obs (B,T,N,C) -> xo (N,B,T,C), xt (N,B,T).  With ``obs.requires_grad`` both carry gradients back to obs."""
    _require_cuda(obs)
    if obs.requires_grad:
        xt_or_both = ObsToNodeMajor.apply(obs)
        if obs.shape[3] > 1:
            return xt_or_both
        # C == 1: xo is a view of xt outside the Function, so autograd folds both gradients into d_xt
        xt = xt_or_both
        return xt.unsqueeze(3), xt
    return _obs_to_node_major(_f32c(obs.detach()))


def _obs_to_node_major(obs: torch.Tensor):
    b, t, n, c = obs.shape
    xt = torch.empty((n, b, t), device=obs.device, dtype=torch.float32)
    xo = torch.empty((n, b, t, c), device=obs.device, dtype=torch.float32) if c > 1 else None
    _lib.check(L.stmgcn_obs_to_node_major(obs.data_ptr(), _p(xo), xt.data_ptr(), b, t, n, c, _stream()),
               "obs_to_node_major")
    return (xo if xo is not None else xt.view(n, b, t, 1)), xt


class ObsToNodeMajor(torch.autograd.Function):
    """:func:`obs_to_node_major` for an obs that requires grad: returns (xo, xt), or xt alone when C == 1.
    Backward: d_obs[b,t,n,c] = d_xo[n,b,t,c] + d_xt[n,b,t] (stmgcn_obs_grad)."""

    @staticmethod
    def forward(ctx, obs):
        ctx.set_materialize_grads(False)
        ctx.shape, ctx.dtype = tuple(obs.shape), obs.dtype
        xo, xt = _obs_to_node_major(_f32c(obs.detach()))
        return (xo, xt) if obs.shape[3] > 1 else xt

    @staticmethod
    def backward(ctx, *grads):
        d_xo, d_xt = grads if len(grads) == 2 else (None, grads[0])
        if d_xo is None and d_xt is None:
            return None
        b, t, n, c = ctx.shape
        d_obs = torch.empty((b, t, n, c), device=(d_xt if d_xt is not None else d_xo).device, dtype=torch.float32)
        d_xo = _f32c(d_xo) if d_xo is not None else None
        d_xt = _f32c(d_xt) if d_xt is not None else None
        _lib.check(L.stmgcn_obs_grad(_p(d_xo), _p(d_xt), d_obs.data_ptr(), b, t, n, c, _stream()), "obs_grad")
        return d_obs.to(ctx.dtype)


class ChebGCN(torch.autograd.Function):
    """out (N,B,q) = act( sum_k (T_k x) W_k + b ),  x (N,B,p) node-major.

    ``vals``: ``sset.grad_values()``, the set's value tensors or its dense stack, inputs only so that their gradients
    reach them: the kernels read the set's own copies."""

    @staticmethod
    def forward(ctx, x, w, bias, sset: SupportSet, act: int, *vals):
        _require_cuda(x, w)
        x, w = _f32c(x), _f32c(w)
        bias_c = _f32c(bias) if bias is not None else None
        # bf16-arithmetic mode: the spatial recurrence (F = B*64 features per node: the step's large gather volume) reads its
        # gathered operand from bf16 copies.  Not the temporal GCN (TemporalPool): its output feeds a global mean and the
        # two-layer gate, whose parameter gradients are small differences of large sums -- with bf16 gathers there they
        # moved by 2-3.6e-2 on the golden case (measured), past that mode's 2e-2 bar -- and its F = B*T rows are cheap.
        s = build_stack(sset, x, gather16=True)
        need_grad = any(ctx.needs_input_grad)
        img_f, img_b = _proj_images(w, sset.ks, x.shape[2], need_grad)
        out = _proj_fwd(s, w, bias_c, act, None, x.shape[1], img_f)
        ctx.sset, ctx.act, ctx.has_bias = sset, act, bias is not None
        # the value gradients' B operand is what the recurrence gathered: bf16(T_{k-1}) where it read bf16 copies (asked
        # only when a value needs grad: such a set has a graph, and a set without values runs nothing new; a dense
        # stack's gradient takes the fp32 x, and its set may have no graph: [I])
        ctx.round16 = sset.dense is None and any(ctx.needs_input_grad[5:]) and _gather16(sset, x)
        if need_grad:
            # x (the value or dense-stack gradients of generic supports only) is saved last, and only then
            need_x = any(ctx.needs_input_grad[5:]) and sset.mode == "generic"
            ctx.save_for_backward(s, w, out, img_b, *([x] if need_x else []))
        return out

    @staticmethod
    def backward(ctx, d_out):
        s, w, out, img_b, *x = ctx.saved_tensors
        x = x[0] if x else None
        need_dx, need_dw, need_db = ctx.needs_input_grad[:3]
        d_out = _f32c(d_out)
        need_u = need_dx or any(ctx.needs_input_grad[5:])
        dw, db, u = _proj_bwd(s, w, ctx.act, out, d_out, None, 1.0, s.shape[2], ctx.has_bias and need_db, need_u, img_b,
                              need_w=need_dw)
        dx, extra = _support_grads(ctx, s, u, x, need_dx, ctx.round16)
        return (dx, dw, db, None, None, *extra)


class TemporalPool(torch.autograd.Function):
    """pool (B,T) = sum_n ( x + act(GCN_T(x)) )[n,b,:]  (STMGCN.py:40-42 before the division by N).  ``vals`` as for
    :class:`ChebGCN`."""

    @staticmethod
    def forward(ctx, x, w, bias, sset: SupportSet, act: int, *vals):
        _require_cuda(x, w)
        x, w = _f32c(x), _f32c(w)
        bias_c = _f32c(bias) if bias is not None else None
        n, b, t = x.shape
        if w.shape[1] != t:
            raise ValueError("temporal GCN must map seq_len -> seq_len")
        s = build_stack(sset, x)
        if sset.mode == "cheb":
            # s[0] IS x (T_0 = I): the kernel's fused pooling adds the residual from the stack's first segment
            pool = torch.zeros((b, t), device=x.device, dtype=torch.float32)
            out = _proj_fwd(s, w, bias_c, act, pool, b)
        else:
            # generic supports (localpool, hand-made stacks): s[0] = A_0 x is NOT the residual of STMGCN.py:41
            out = _proj_fwd(s, w, bias_c, act, None, b)
            pool = (x + out).sum(dim=0)
        ctx.act, ctx.has_bias, ctx.sset = act, bias is not None, sset
        if any(ctx.needs_input_grad):
            need_x = any(ctx.needs_input_grad[5:]) and sset.mode == "generic"
            ctx.save_for_backward(s, w, out, *([x] if need_x else []))
        return pool

    @staticmethod
    def backward(ctx, d_pool):
        s, w, out, *x = ctx.saved_tensors
        x = x[0] if x else None
        d_pool = _f32c(d_pool)
        need_dx, need_dw, need_db = ctx.needs_input_grad[:3]
        need_u = need_dx or any(ctx.needs_input_grad[5:])
        dw, db, u = _proj_bwd(s, w, ctx.act, out, None, d_pool, 1.0, s.shape[2], ctx.has_bias and need_db, need_u,
                              need_w=need_dw)
        dx, extra = _support_grads(ctx, s, u, x, need_dx, False)
        if dx is not None:
            # the GCN's dX (adjoint Clenshaw / sum_k A_k^T U_k) plus the residual's: d_pool broadcast over regions
            dx = dx + d_pool.unsqueeze(0)
        return (dx, dw, db, None, None, *extra)


class ContextGate(torch.autograd.Function):
    """s = sigmoid(fc(relu(fc(pool / N))))  -- the same fc twice (STMGCN.py:43)."""

    @staticmethod
    def forward(ctx, pool, fcw, fcb, n_regions: int):
        _require_cuda(pool, fcw, fcb)
        pool, fcw, fcb = _f32c(pool), _f32c(fcw), _f32c(fcb)
        b, t = pool.shape
        z, a1, s = (torch.empty_like(pool) for _ in range(3))
        _lib.check(L.stmgcn_gate_fwd(pool.data_ptr(), b, t, n_regions, fcw.data_ptr(), fcb.data_ptr(),
                                     z.data_ptr(), a1.data_ptr(), s.data_ptr(), _stream()), "gate_fwd")
        ctx.n_regions = n_regions
        ctx.save_for_backward(z, a1, s, fcw)
        return s

    @staticmethod
    def backward(ctx, d_s):
        z, a1, s, fcw = ctx.saved_tensors
        d_s = _f32c(d_s)
        b, t = s.shape
        # the fc gradients come together from the kernel: both, or neither when the fc is frozen
        need_fcw, need_fcb = ctx.needs_input_grad[1:3]
        need_fc = need_fcw or need_fcb
        d_fcw = torch.zeros_like(fcw) if need_fc else None
        d_fcb = torch.zeros(t, device=s.device, dtype=torch.float32) if need_fc else None
        d_z = torch.empty_like(s)
        _lib.check(L.stmgcn_gate_bwd(d_s.data_ptr(), z.data_ptr(), a1.data_ptr(), s.data_ptr(), b, t,
                                     fcw.data_ptr(), _p(d_fcw), _p(d_fcb), d_z.data_ptr(),
                                     _stream()), "gate_bwd")
        d_pool = d_z / float(ctx.n_regions) if ctx.needs_input_grad[0] else None
        return d_pool, d_fcw if need_fcw else None, d_fcb if need_fcb else None, None


def to_blocked(x: torch.Tensor) -> torch.Tensor:
    """(..., R, 64) row-major -> tile-blocked (..., ceil(R/128)*128, 64) flat layout [tile][unit/4][128][4]."""
    *lead, r, h = x.shape
    rp = ((r + 127) // 128) * 128
    if rp != r:
        pad = x.new_zeros(*lead, rp, h)
        pad[..., :r, :] = x
        x = pad
    return x.reshape(*lead, rp // 128, 128, 16, 4).transpose(-3, -2).contiguous().reshape(*lead, rp, h)


def from_blocked(x: torch.Tensor, rows: int) -> torch.Tensor:
    """Inverse of :func:`to_blocked`."""
    *lead, rp, h = x.shape
    return x.reshape(*lead, rp // 128, 16, 128, 4).transpose(-3, -2).reshape(*lead, rp, h)[..., :rows, :].contiguous()


def _pack_lstm(weights: Sequence[torch.Tensor], n_layers: int, hid: int):
    """nn.LSTM parameters -> packed operands (see include/stmgcn_b200.h): wx (C,4H); flat wp / wpt holding each layer's
    (kd_l,4H) / (4H,kd_l) block after the blocks of the layers below (kd_0 = H, kd_l = 2H); bp (L,4H)."""
    w_ih0 = weights[0]
    c_in = w_ih0.shape[1]
    wx = w_ih0.reshape(4, hid, c_in).permute(2, 1, 0).reshape(c_in, 4 * hid).contiguous()
    wp, bp, wpt = [], [], []
    for l in range(n_layers):
        w_ih, w_hh, b_ih, b_hh = weights[4 * l:4 * l + 4]
        cat = w_hh if l == 0 else torch.cat([w_ih, w_hh], dim=1)
        kd = cat.shape[1]
        packed = cat.reshape(4, hid, kd).permute(2, 1, 0).reshape(kd, 4 * hid)
        wp.append(packed.reshape(-1))
        wpt.append(packed.t().reshape(-1))
        bp.append((b_ih + b_hh).reshape(4, hid).t().reshape(4 * hid))
    return wx, torch.cat(wp), torch.stack(bp), torch.cat(wpt)


def _unpack_lstm_grads(dwx, dwp, dbp, n_layers: int, hid: int, c_in: int):
    grads = []
    kds = [hid] + [2 * hid] * (n_layers - 1)
    for l, (kd, blk) in enumerate(zip(kds, dwp.split([kd * 4 * hid for kd in kds]))):
        full = blk.reshape(kd, hid, 4).permute(2, 1, 0).reshape(4 * hid, kd)
        if l == 0:
            d_ih = dwx.reshape(c_in, hid, 4).permute(2, 1, 0).reshape(4 * hid, c_in).contiguous()
            d_hh = full.contiguous()
        else:
            d_ih, d_hh = full[:, :hid].contiguous(), full[:, hid:].contiguous()
        d_b = dbp[l].reshape(hid, 4).t().reshape(4 * hid).contiguous()
        grads += [d_ih, d_hh, d_b, d_b.clone()]
    return grads


# --------------------------------------------------------------------------------------------------
# bf16-plane LSTM path (H = 64): weight images packed on every forward
# --------------------------------------------------------------------------------------------------
_PLANES = int(os.environ.get("STMGCN_LSTM_PLANES", "2"))     # 2: 3xBF16 (fp32-grade); 1: single-pass bf16 arithmetic


def lstm_planes() -> int:
    return _PLANES


def set_lstm_planes(planes: int) -> None:
    """2 = hi + lo bf16 planes, three tensor-core passes (fp32-grade, the 1e-4 parity mode);
    1 = hi plane only, one pass (the arithmetic of the bf16-quoted BASELINE configs)."""
    global _PLANES
    if planes not in (1, 2):
        raise ValueError(planes)
    _PLANES = planes


def _lstm16_images(weights: Sequence[torch.Tensor], n_layers: int, c_in: int):
    """Operand images of the shared LSTM's parameters for the bf16-plane kernels (stmgcn_lstm16_pack): the flat wimg,
    bias (L, 256) and wih_t, packed from the weights as they are now, on every call."""
    dev = weights[0].device
    wimg = torch.empty(65536 * (2 * n_layers - 1), dtype=torch.uint8, device=dev)
    bias = torch.empty((n_layers, 256), dtype=torch.float32, device=dev)
    wih_t = torch.empty(c_in * 256, dtype=torch.float32, device=dev)
    st = _stream()
    for l in range(n_layers):
        w_ih, w_hh, b_ih, b_hh = weights[4 * l:4 * l + 4]
        _lib.check(L.stmgcn_lstm16_pack(w_ih.data_ptr(), w_hh.data_ptr(), b_ih.data_ptr(), b_hh.data_ptr(), l, c_in,
                                        wimg.data_ptr(), bias.data_ptr(), wih_t.data_ptr(), st), "lstm16_pack")
    return wimg, bias, wih_t


def to_planes(x: torch.Tensor, planes: int) -> torch.Tensor:
    """(..., R, 64) fp32 -> (..., planes, R, 64) bf16: hi = bf16(x), lo = bf16(x - hi)."""
    hi = x.to(torch.bfloat16)
    if planes == 1:
        return hi.unsqueeze(-3).contiguous()
    lo = (x - hi.float()).to(torch.bfloat16)
    return torch.stack([hi, lo], dim=-3).contiguous()


# the tensors of the bf16-plane path's tape, in the order SharedLSTM saves them
_TAPE16 = ("hp", "cs", "h0p", "c0b", "wimg", "bias", "wih_t")


def _lstm16_forward(xo, s_gate, h0c, c0c, n_layers, want_state, weights, planes, keep_tape):
    """Forward of the bf16-plane path, one library call after the weight packs.  Returns (h_top (N,B,64), h_n, c_n, tape
    dict or None): the tape holds the _TAPE16 tensors, the weight images among them."""
    n, b, t_len, c_in = xo.shape
    rows = n * b
    rows_pad = ((rows + 127) // 128) * 128
    wimg, bias, wih_t = _lstm16_images(weights, n_layers, c_in)
    hp = torch.empty((n_layers, t_len, planes, rows, 64), device=xo.device, dtype=torch.bfloat16)
    cs = xo.new_empty((n_layers, t_len, rows_pad, 64))
    h0p = to_planes(h0c, planes) if h0c is not None else None        # (L, P, R, 64)
    c0b = to_blocked(c0c) if c0c is not None else None
    h_n = xo.new_empty((n_layers, rows, 64)) if want_state else None
    h_top = h_n[n_layers - 1] if want_state else xo.new_empty((rows, 64))
    _lib.check(L.stmgcn_lstm16_fwd(t_len, n_layers, rows, c_in, b, planes, xo.data_ptr(), s_gate.data_ptr(), wimg.data_ptr(),
                                   bias.data_ptr(), wih_t.data_ptr(), _p(h0p), _p(c0b), hp.data_ptr(), cs.data_ptr(),
                                   h_top.data_ptr(), _p(h_n), _stream()), "lstm16_fwd")
    if want_state:
        c_n = from_blocked(cs[:, t_len - 1], rows)
    else:                       # ST_MGCN discards the final state (STMGCN.py:113)
        h_n = c_n = xo.new_empty(0)
    tape = dict(hp=hp, cs=cs, h0p=h0p, c0b=c0b, wimg=wimg, bias=bias, wih_t=wih_t) if keep_tape else None
    return h_top.view(n, b, 64), h_n, c_n, tape


def _zero_tile(dev: torch.device) -> torch.Tensor:
    """16 KB of zeros, the h_prev operand tile at t = 0 without an initial state, made on the current stream for each
    call.  (Not cached: a tile filled on one graph branch's stream would be read by the other branches' backward kernels
    with nothing ordering the read after the fill.)"""
    return torch.zeros(128 * 64, device=dev, dtype=torch.bfloat16)


def _lstm16_backward(xo, s_gate, tape, n_layers, planes, d_top):
    """BPTT of the bf16-plane path, one library call (per layer one fused launch over all timesteps and one weight-gradient
    reduction).  Returns (d_s, [native nn.LSTM gradients]): views of one flat buffer."""
    return _lstm16_backward_ex(xo, s_gate, tape, n_layers, planes, d_top)[:2]


def _lstm16_backward_ex(xo, s_gate, tape, n_layers, planes, d_top, dh_n=None, dc_n=None, want=(False, False, False),
                        wgrad=True):
    """:func:`_lstm16_backward` with the gradients at the inputs and the recurrent state: returns (d_s, grads, (d_xo, dh0,
    dc0)).  dh_n / dc_n (L, R, 64) or None seed the final state's gradients; ``want`` = which of d_xo, dh0, dc0 to compute
    (None otherwise).  Without any of them the plain entry point runs.  ``wgrad=False``: no weight gradients (grads is a
    list of None; the kernels' variant without the weight-gradient stage runs and no reduction is launched)."""
    hp, cs, h0p, c0b, wimg, bias, wih_t = (tape[k] for k in _TAPE16)
    n, b, t_len, c_in = xo.shape
    rows = n * b
    rows_pad = cs.shape[2]
    d_top = to_blocked(_f32c(d_top).view(rows, 64))
    # no workspace needs initialisation: stmgcn_lstm16_bwd zeroes dw_scratch and dbp itself (both only with wgrad)
    dh_rec = xo.new_empty((rows_pad, 64))
    dc = xo.new_empty((rows_pad, 64))
    dx_work = xo.new_empty((min(2, n_layers - 1), t_len, rows_pad, 64)) if n_layers > 1 else None
    d_s = xo.new_zeros((b, t_len))
    shapes = [s for l in range(n_layers) for s in ((256, c_in if l == 0 else 64), (256, 64), (256,), (256,))]
    if wgrad:
        dw_scratch = xo.new_empty((int(L.stmgcn_lstm16_grid(rows)), 128 * 256))
        dbp = xo.new_empty((n_layers, 256))
        grads = xo.new_empty(sum(math.prod(s) for s in shapes))
        w_grads = [g.view(s) for g, s in zip(grads.split([math.prod(s) for s in shapes]), shapes)]
    else:
        dw_scratch = dbp = grads = None
        w_grads = [None] * len(shapes)
    zero_tile = _zero_tile(xo.device)              # held until the launches below are enqueued
    args = (t_len, n_layers, rows, c_in, b, planes, xo.data_ptr(), s_gate.data_ptr(), wimg.data_ptr(), bias.data_ptr(),
            wih_t.data_ptr(), _p(h0p), _p(c0b), hp.data_ptr(), cs.data_ptr(), d_top.data_ptr(), dh_rec.data_ptr(),
            dc.data_ptr(), _p(dx_work), _p(dw_scratch), _p(dbp), zero_tile.data_ptr(),
            d_s.data_ptr(), _p(grads))
    if dh_n is None and dc_n is None and not any(want):
        _lib.check(L.stmgcn_lstm16_bwd(*args, _stream()), "lstm16_bwd")
        return d_s, w_grads, (None, None, None)
    # the state gradients are tile-blocked (L, R_pad, 64) at the C ABI
    dh_nb = to_blocked(_f32c(dh_n)) if dh_n is not None else None
    dc_nb = to_blocked(_f32c(dc_n)) if dc_n is not None else None
    d_xo = xo.new_empty(xo.shape) if want[0] else None
    dh0b = xo.new_empty((n_layers, rows_pad, 64)) if want[1] else None
    dc0b = xo.new_empty((n_layers, rows_pad, 64)) if want[2] else None
    _lib.check(L.stmgcn_lstm16_bwd_ex(*args, _p(dh_nb), _p(dc_nb), _p(dh0b), _p(dc0b), _p(d_xo), _stream()), "lstm16_bwd_ex")
    dh0 = from_blocked(dh0b, rows) if dh0b is not None else None
    dc0 = from_blocked(dc0b, rows) if dc0b is not None else None
    return d_s, w_grads, (d_xo, dh0, dc0)


def _exact_forward(xo, s_gate, h0c, c0c, n_layers, hid, want_state, weights, keep_tape):
    """Forward of the exact-fp32 path, one library call.  Returns (h_top (N,B,H), h_n, c_n, tape tuple or None)."""
    n, b, t_len, c_in = xo.shape
    rows = n * b
    wx, wp, bp, wpt = _pack_lstm(weights, n_layers, hid)
    hs = xo.new_empty((n_layers, t_len, rows, hid))
    cs = xo.new_empty((n_layers, t_len, rows, hid))
    gates = xo.new_empty((n_layers, t_len, rows, 4 * hid)) if keep_tape else None
    _lib.check(L.stmgcn_lstm_fwd(t_len, n_layers, rows, hid, c_in, b, xo.data_ptr(), s_gate.data_ptr(), wx.data_ptr(),
                                 wp.data_ptr(), bp.data_ptr(), _p(h0c), _p(c0c), hs.data_ptr(), cs.data_ptr(), _p(gates),
                                 _stream()), "lstm_fwd")
    h_top = hs[n_layers - 1, t_len - 1].view(n, b, hid)
    if want_state:
        h_n, c_n = hs[:, t_len - 1], cs[:, t_len - 1]
    else:                       # ST_MGCN discards the final state (STMGCN.py:113)
        h_n = c_n = hs.new_empty(0)
    return h_top, h_n, c_n, ((h0c, c0c, hs, cs, gates, wx, wpt) if keep_tape else None)


def _exact_backward(xo, s_gate, tape, n_layers, hid, d_top):
    """BPTT of the exact-fp32 path, one library call; it overwrites the gate tape with dA.  Returns (d_s, grads)."""
    return _exact_backward_ex(xo, s_gate, tape, n_layers, hid, d_top)[:2]


def _exact_backward_ex(xo, s_gate, tape, n_layers, hid, d_top, dh_n=None, dc_n=None, want=(False, False, False),
                       wgrad=True):
    """:func:`_exact_backward` with the extras and ``wgrad`` of :func:`_lstm16_backward_ex`: returns (d_s, grads, (d_xo,
    dh0, dc0))."""
    h0, c0, hs, cs, gates, wx, wpt = tape
    n, b, t_len, c_in = xo.shape
    rows = n * b
    d_top = _f32c(d_top).view(rows, hid)
    # dh_rec / dc need no initialisation: the step at t = T-1 treats them as zero (stmgcn_lstm_bwd)
    dh_rec = xo.new_empty((n_layers, rows, hid))
    dc = xo.new_empty((n_layers, rows, hid))
    dx_work = xo.new_empty((rows, hid))
    d_s = xo.new_zeros((b, t_len))
    dwx = torch.zeros_like(wx) if wgrad else None
    dwp = torch.zeros_like(wpt) if wgrad else None
    dbp = xo.new_zeros((n_layers, 4 * hid)) if wgrad else None
    args = (t_len, n_layers, rows, hid, c_in, b, xo.data_ptr(), s_gate.data_ptr(), wx.data_ptr(), wpt.data_ptr(), _p(h0),
            _p(c0), cs.data_ptr(), hs.data_ptr(), gates.data_ptr(), d_top.data_ptr(), dh_rec.data_ptr(), dc.data_ptr(),
            dx_work.data_ptr(), d_s.data_ptr(), _p(dwx), _p(dwp), _p(dbp))
    extras = (None, None, None)
    if dh_n is None and dc_n is None and not any(want):
        _lib.check(L.stmgcn_lstm_bwd(*args, _stream()), "lstm_bwd")
    else:
        dh_n = _f32c(dh_n) if dh_n is not None else None
        dc_n = _f32c(dc_n) if dc_n is not None else None
        extras = tuple(xo.new_empty(shape) if w else None
                       for w, shape in zip(want, (xo.shape, (n_layers, rows, hid), (n_layers, rows, hid))))
        _lib.check(L.stmgcn_lstm_bwd_ex(*args, _p(dh_n), _p(dc_n), _p(extras[1]), _p(extras[2]), _p(extras[0]),
                                        _stream()), "lstm_bwd_ex")
    w_grads = _unpack_lstm_grads(dwx, dwp, dbp, n_layers, hid, c_in) if wgrad else [None] * (4 * n_layers)
    return d_s, w_grads, extras


class SharedLSTM(torch.autograd.Function):
    """h_top (N,B,H) of the shared multi-layer LSTM over rows r = n*B + b; input ``xo * s[b,t]``.

    forward(xo (N,B,T,C), s (B,T), h0|None, c0|None (L,R,H), n_layers, hid, want_state, *lstm_weights) where
    lstm_weights = [w_ih_l0, w_hh_l0, b_ih_l0, b_hh_l0, w_ih_l1, ...] (nn.LSTM names/shapes).
    Returns (h_top, h_n (L,R,H), c_n (L,R,H)), three distinct tensors; h_n / c_n are differentiable with ``want_state``
    (empty and not differentiable without).  Gradients flow to xo, s, h0, c0 and the weights.

    Two kernel families (include/stmgcn_b200.h):
    * H = 64, C <= 4, T <= 64 (the reference's configuration, Main.py:62) and ``lstm_path() == "tc"``: the tensor-core bf16-plane
      kernels of lstm16.cu -- tape = hidden-state planes + cell state, no gate tape, fused recompute backward;
    * anything else, or ``lstm_path() == "fma"``: the exact-fp32 CUDA-core kernels of lstm.cu with their own tape
      (hs, cs, gates); their backward overwrites the gate tape in place, so it can run only once per forward.
    """

    @staticmethod
    def forward(ctx, xo, s_gate, h0, c0, n_layers: int, hid: int, want_state: bool, *weights):
        _require_cuda(xo, s_gate, *weights)
        xo, s_gate = _f32c(xo), _f32c(s_gate)
        weights = [_f32c(w) for w in weights]
        c_in, t_len = xo.shape[3], xo.shape[2]
        h0c = _f32c(h0) if h0 is not None else None
        c0c = _f32c(c0) if c0 is not None else None
        need_grad = any(ctx.needs_input_grad)
        ctx.dims = (n_layers, hid)
        ctx.planes16 = hid == 64 and lstm_path() == "tc" and c_in <= 4 and t_len <= 64
        if ctx.planes16:
            ctx.planes = lstm_planes()
            h_top, h_n, c_n, tape = _lstm16_forward(xo, s_gate, h0c, c0c, n_layers, want_state, weights, ctx.planes,
                                                    need_grad)
            if need_grad:
                tape = [tape[k] for k in _TAPE16]
        else:
            h_top, h_n, c_n, tape = _exact_forward(xo, s_gate, h0c, c0c, n_layers, hid, want_state, weights, need_grad)
        if need_grad:
            ctx.save_for_backward(xo, s_gate, *tape)
        ctx.set_materialize_grads(False)
        if want_state:
            # three distinct outputs: h_top is a view of h_n (tensor cores) or both are views of the tape (exact path)
            h_top = h_top.clone()
            if not ctx.planes16:
                h_n, c_n = h_n.clone(), c_n.clone()
        else:
            ctx.mark_non_differentiable(h_n, c_n)
        return h_top, h_n, c_n

    @staticmethod
    def backward(ctx, d_top, dh_n, dc_n):
        n_layers, hid = ctx.dims
        xo, s_gate, *tape = ctx.saved_tensors
        if d_top is None:
            d_top = xo.new_zeros((xo.shape[0], xo.shape[1], hid))
        want = (ctx.needs_input_grad[0], ctx.needs_input_grad[2], ctx.needs_input_grad[3])
        # the weight gradients of the whole stack, or none of them when no LSTM weight requires grad
        wgrad = any(ctx.needs_input_grad[7:])
        if ctx.planes16:
            tape16 = dict(zip(_TAPE16, tape))
            d_s, w_grads, extras = _lstm16_backward_ex(xo, s_gate, tape16, n_layers, ctx.planes, d_top, dh_n, dc_n, want,
                                                       wgrad)
        else:
            if getattr(ctx, "tape_consumed", False):
                raise RuntimeError("SharedLSTM (exact-fp32 kernels): the gate tape was overwritten in place by the first "
                                   "backward pass; a second backward over the same graph is not supported on this path")
            ctx.tape_consumed = True
            d_s, w_grads, extras = _exact_backward_ex(xo, s_gate, tape, n_layers, hid, d_top, dh_n, dc_n, want, wgrad)
        d_xo, dh0, dc0 = extras
        return (d_xo, d_s, dh0, dc0, None, None, None, *w_grads)


class FuseOut(torch.autograd.Function):
    """y (B,N,C) = fc( sum_m g_m ),  g_m (N,B,G) node-major  (STMGCN.py:116-118)."""

    @staticmethod
    def forward(ctx, fcw, fcb, *gs):
        _require_cuda(fcw, fcb, *gs)
        fcw, fcb = _f32c(fcw), _f32c(fcb)
        gs = [_f32c(g) for g in gs]
        n, b, gdim = gs[0].shape
        c = fcw.shape[0]
        feat = torch.empty_like(gs[0])
        y = torch.empty((b, n, c), device=feat.device, dtype=torch.float32)
        arr = _lib.ptr_array([g.data_ptr() for g in gs])
        _lib.check(L.stmgcn_fuse_out_fwd(arr, len(gs), n, b, gdim, c, fcw.data_ptr(), fcb.data_ptr(),
                                         feat.data_ptr(), y.data_ptr(), _stream()), "fuse_out_fwd")
        ctx.m = len(gs)
        ctx.save_for_backward(feat, fcw)
        return y

    @staticmethod
    def backward(ctx, d_y):
        feat, fcw = ctx.saved_tensors
        d_y = _f32c(d_y)
        n, b, gdim = feat.shape
        c = fcw.shape[0]
        d_feat = torch.empty_like(feat)
        need_fcw, need_fcb = ctx.needs_input_grad[:2]
        need_fc = need_fcw or need_fcb                  # both from the kernel, or neither
        d_fcw = torch.zeros_like(fcw) if need_fc else None
        d_fcb = torch.zeros(c, device=feat.device, dtype=torch.float32) if need_fc else None
        _lib.check(L.stmgcn_fuse_out_bwd(d_y.data_ptr(), feat.data_ptr(), n, b, gdim, c, fcw.data_ptr(),
                                         d_feat.data_ptr(), _p(d_fcw), _p(d_fcb), _stream()),
                   "fuse_out_bwd")
        return (d_fcw if need_fcw else None, d_fcb if need_fcb else None) + tuple(d_feat for _ in range(ctx.m))
