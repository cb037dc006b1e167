"""CPU oracle for the ST-MGCN hot path.  TEST INFRASTRUCTURE ONLY.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference``
legs may import this file.  Nothing under ``st-mgcn_b200/``, ``GCN.py`` or ``STMGCN.py`` does, and the
product path raises if the CUDA library is missing rather than falling back to anything in here.

Two independent restatements of the reference algorithm (all citations into the reference ST-MGCN sources):

* **dense** (``dense_*`` functions, torch CPU): the algorithm exactly as the reference executes it --
  K+1 dense ``N x N`` supports multiplied into the features one by one (``GCN.py:34-36``), concatenated
  (``GCN.py:37``), projected (``GCN.py:39-42``); context gate (``STMGCN.py:35-44``); shared LSTM with
  PyTorch gate order i,f,g,o and two biases (``STMGCN.py:47-50``); sum over graphs and output FC
  (``STMGCN.py:112-118``).  Gradients come from autograd.  The LSTM exists twice: ``lstm_explicit``
  (written out cell by cell) and ``lstm_library`` (``torch.nn.LSTM``, what the reference calls,
  ``STMGCN.py:21-22``); tests pin one against the other.
* **sparse** (``SparseOracle``, numpy + scipy CSR, fp32 or fp64): the algorithm the CUDA path runs --
  Chebyshev recurrence on the *features* with the sparse rescaled Laplacian ``L = supports[1]``
  (``T_k X = 2 L T_{k-1} X - T_{k-2} X``, the same polynomial ``GCN.py:125-135`` builds on matrices) --
  with the forward AND the hand-derived backward (adjoint Clenshaw with ``L^T``, BPTT, gate) written
  out.  It is validated against the dense restatement (and through it against the reference) in
  ``tests/test_oracle.py`` and is the oracle at sizes where dense supports are infeasible.

``BF16ModeReference`` (torch autograd, fp64) is the sparse model once more, in the bf16-arithmetic mode: it rounds where
the kernels of that mode round and can be forced with the kernels' own values at every rounding point.  With rounding
off it is pinned to ``SparseOracle`` in ``tests/test_oracle.py``.

Parity pin: the reference has no tests, golden vectors or fixtures of its own (SURVEY.md section 4) --
"parity unpinned" by the reference's own tests.  The pin used here is the reference code itself,
imported from a reference checkout (``oracle/make_golden.py`` ->
``tests/golden/*.npz``; ``tests/test_oracle.py::test_dense_matches_reference_modules``).
"""
from __future__ import annotations

import warnings
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

Params = Dict[str, torch.Tensor]


# --------------------------------------------------------------------------------------------------
# support construction (GCN.py:57-97, 107-135) -- constant operand of the hot path
# --------------------------------------------------------------------------------------------------
def rescaled_laplacian_dense(adj: torch.Tensor, lambda_max: float = 2.0) -> torch.Tensor:
    """``L~ = (2/lambda_max)(I - D^-1/2 A D^-1/2) - I`` (``GCN.py:107-111``, ``:73``, ``:113-123``).

    On torch >= 1.13 the reference's ``torch.eig`` call raises and its bare ``except`` uses
    ``lambda_max = 2`` (``GCN.py:117-121``); that is the default here.
    """
    d = adj.sum(dim=1).pow(-0.5)
    a_norm = d[:, None] * adj * d[None, :]
    eye = torch.eye(adj.shape[0], dtype=adj.dtype, device=adj.device)
    lap = eye - a_norm
    return (2.0 / lambda_max) * lap - eye


def chebyshev_supports_dense(adj: torch.Tensor, order: int, lambda_max: float = 2.0) -> torch.Tensor:
    """``(order+1, N, N)`` stack ``T_0..T_K`` of ``L~`` (``GCN.py:125-135``, stacked at ``:95``)."""
    lt = rescaled_laplacian_dense(adj, lambda_max)
    polys = [torch.eye(adj.shape[0], dtype=adj.dtype)]
    if order >= 1:
        polys.append(lt)
    for _ in range(2, order + 1):
        polys.append(2.0 * (lt @ polys[-1]) - polys[-2])
    return torch.stack(polys, dim=0)


def chain_stack_dense(mats: Sequence[torch.Tensor], order: int) -> torch.Tensor:
    """Dense stack of Chebyshev recurrence chains sharing ``T_0 = I``: ``[I, T_1(X_0)..T_K(X_0), T_1(X_1)..]`` for the
    chain matrices ``X_c`` of ``mats`` (in their dtype and on their device), ``K = order``: the stack a support set of
    chains stands for."""
    eye = torch.eye(mats[0].shape[0], dtype=mats[0].dtype, device=mats[0].device)
    out = [eye]
    for x in mats:
        polys = [eye, x]
        for _ in range(2, order + 1):
            polys.append(2.0 * (x @ polys[-1]) - polys[-2])
        out += polys[1:order + 1]
    return torch.stack(out)


# --------------------------------------------------------------------------------------------------
# dense restatement (torch CPU; autograd supplies the backward)
# --------------------------------------------------------------------------------------------------
def _activate(z: torch.Tensor, relu, mask: Optional[torch.Tensor]) -> torch.Tensor:
    """The GCN activation ``relu`` of the dense restatement on the pre-activation ``z`` (B, N, q): True = ReLU, False or
    None = none, anything else a callable applied to ``z`` (a torch module such as ``nn.Tanh()``, as the reference's
    ``self.activation``).  ``mask`` (ReLU only): a boolean ReLU mask in the kernels' node-major layout (N, B, q) used in
    place of ``z > 0``: ``out = z * mask``."""
    if relu is True:
        return torch.relu(z) if mask is None else z * mask.permute(1, 0, 2).to(z.dtype)
    if mask is not None:
        raise ValueError("a forced ReLU mask needs the ReLU activation")
    if relu is False or relu is None:
        return z
    return relu(z)


def dense_gcn(supports: torch.Tensor, x: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor],
              relu=True, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``GCN.forward`` (``GCN.py:24-43``): ``act(cat_k(A_k x) W + b)``; rows ``[k p,(k+1) p)`` of W
    pair with support k.  ``relu`` / ``mask``: the activation and an optional forced ReLU mask (:func:`_activate`).
    Runs on the device and in the dtype of its arguments (fp64 on the GPU for the model-level sweeps)."""
    n_sup = supports.shape[0]
    p = x.shape[-1]
    assert w.shape[0] == n_sup * p                      # GCN.py:31 in spirit
    out = None
    for k in range(n_sup):
        s_k = torch.matmul(supports[k], x)              # (B,N,p): sum_j A_k[i,j] x[b,j,:]
        term = torch.matmul(s_k, w[k * p:(k + 1) * p])
        out = term if out is None else out + term
    if b is not None:
        out = out + b
    return _activate(out, relu, mask)


def lstm_explicit(x: torch.Tensor, layers: Sequence[Tuple[torch.Tensor, ...]],
                  h0: Optional[torch.Tensor] = None, c0: Optional[torch.Tensor] = None):
    """Multi-layer LSTM, ``batch_first``, PyTorch semantics (gate order i,f,g,o; ``b_ih + b_hh``).

    ``x:(R,T,in)``; ``layers[l] = (w_ih (4H,in_l), w_hh (4H,H), b_ih (4H), b_hh (4H))``.
    Returns ``(top-layer outputs (R,T,H), (h_n, c_n) each (L,R,H))`` like ``nn.LSTM``.
    """
    r, t_len, _ = x.shape
    hid = layers[0][1].shape[1]
    seq = x
    h_n, c_n = [], []
    for l, (w_ih, w_hh, b_ih, b_hh) in enumerate(layers):
        h = x.new_zeros(r, hid) if h0 is None else h0[l]
        c = x.new_zeros(r, hid) if c0 is None else c0[l]
        outs = []
        for t in range(t_len):
            gates = seq[:, t] @ w_ih.t() + b_ih + h @ w_hh.t() + b_hh
            i, f, g, o = gates.split(hid, dim=1)
            i, f, g, o = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)
            c = f * c + i * g
            h = o * torch.tanh(c)
            outs.append(h)
        seq = torch.stack(outs, dim=1)
        h_n.append(h)
        c_n.append(c)
    return seq, (torch.stack(h_n), torch.stack(c_n))


def round_bf16(v: torch.Tensor) -> torch.Tensor:
    """``v`` rounded to bf16 (round-to-nearest-even, from its fp32 value) in ``v``'s dtype; the gradient passes straight
    through, like the kernels' bf16 stores."""
    return v + (v.float().to(torch.bfloat16).to(v.dtype) - v).detach()


def lstm_planes_reference(x: torch.Tensor, layers: Sequence[Tuple[torch.Tensor, ...]], planes: int = 2,
                          h0: Optional[torch.Tensor] = None, c0: Optional[torch.Tensor] = None,
                          tape: Optional[Dict[str, torch.Tensor]] = None):
    """The arithmetic of the bf16-plane tensor-core LSTM (``lstm16.cu``) in the dtype of ``x`` (fp64 for tests),
    differentiable by autograd.  Same contract as :func:`lstm_explicit`; ``x:(R,T,C)`` is the modulated input ``xo * s``.

    ``planes = 2`` (hi + lo operand planes): exact operands, i.e. :func:`lstm_explicit`.  ``planes = 1`` (one bf16 plane):
    the operands of the tensor-core products are rounded to bf16 -- the hidden states (h_below, h_prev, h0) and the MMA
    weights (``W_hh`` of every layer, ``W_ih`` of layers > 0).  Layer 0's input term ``x W_ih^T``, the biases and the
    cell state are not rounded (the kernels add them with fp32 FMAs).

    ``tape`` (optional): the kernel's own tape as values of ``x``'s dtype -- ``h (L,T,R,H)`` (the hidden-state planes
    summed), ``c (L,T,R,H)`` and, with an initial state, ``h0 (L,R,H)`` (its planes summed).  Every step then takes the
    VALUES of h_below, h_prev and c_prev from the tape but routes their GRADIENT through this function's own h and c
    (``operand = tape + (computed - computed.detach())``): the forward consumes what the kernel consumed, so a rounding
    boundary that fp32 and fp64 see on different sides cannot propagate, and the autograd backward has the kernel
    backward's semantics (gates recomputed from the tape, straight through the bf16 stores).

    Returns ``(top-layer outputs (R,T,H), (h_n, c_n), (hs, cs))``; ``hs[l][t]`` / ``cs[l][t]`` are the computed states
    of every layer-step (with a tape: step-local, i.e. one step of the recurrence from the kernel's own inputs).
    """
    if planes not in (1, 2):
        raise ValueError(planes)
    rnd = round_bf16 if planes == 1 else (lambda v: v)

    def forced(computed, l, t, key):
        if tape is None:
            return computed
        return (tape[key][l] if t is None else tape[key][l, t]) + (computed - computed.detach())

    r, t_len, _ = x.shape
    hid = layers[0][1].shape[1]
    seq = x
    h_n, c_n, hs_all, cs_all = [], [], [], []
    for l, (w_ih, w_hh, b_ih, b_hh) in enumerate(layers):
        w_in = w_ih if l == 0 else rnd(w_ih)
        w_rec = rnd(w_hh)
        h = x.new_zeros(r, hid) if h0 is None else h0[l]
        c = x.new_zeros(r, hid) if c0 is None else c0[l]
        if h0 is not None:
            h = forced(h, l, None, "h0")
        hs, cs = [], []
        for t in range(t_len):
            x_t = seq[t] if l > 0 else x[:, t]
            if l > 0:
                x_t = rnd(forced(x_t, l - 1, t, "h"))
            h_op = rnd(h if t == 0 else forced(h, l, t - 1, "h"))
            c_op = c if t == 0 else forced(c, l, t - 1, "c")
            gates = x_t @ w_in.t() + h_op @ w_rec.t() + (b_ih + b_hh)
            i, f, g, o = gates.split(hid, dim=1)
            i, f, g, o = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)
            c = f * c_op + i * g
            h = o * torch.tanh(c)
            hs.append(h)
            cs.append(c)
        seq = hs
        h_n.append(h)
        c_n.append(c)
        hs_all.append(hs)
        cs_all.append(cs)
    return torch.stack(seq, dim=1), (torch.stack(h_n), torch.stack(c_n)), (hs_all, cs_all)


def lstm_library(x: torch.Tensor, layers: Sequence[Tuple[torch.Tensor, ...]],
                 h0: Optional[torch.Tensor] = None, c0: Optional[torch.Tensor] = None):
    """Same contract as :func:`lstm_explicit` through ``torch.nn.LSTM`` -- the library call the
    reference makes (``STMGCN.py:21-22, :48``).  Used for the CPU baseline timing."""
    hid = layers[0][1].shape[1]
    mod = torch.nn.LSTM(input_size=x.shape[-1], hidden_size=hid, num_layers=len(layers),
                        batch_first=True).to(x.dtype)
    flat = {}
    for l, (w_ih, w_hh, b_ih, b_hh) in enumerate(layers):
        flat[f"weight_ih_l{l}"], flat[f"weight_hh_l{l}"] = w_ih, w_hh
        flat[f"bias_ih_l{l}"], flat[f"bias_hh_l{l}"] = b_ih, b_hh
    r = x.shape[0]
    if h0 is None:
        h0 = x.new_zeros(len(layers), r, hid)
    if c0 is None:
        c0 = x.new_zeros(len(layers), r, hid)
    return torch.func.functional_call(mod, flat, (x, (h0, c0)))


def _lstm_layers(params: Params, prefix: str, n_layers: int):
    return [(params[f"{prefix}weight_ih_l{l}"], params[f"{prefix}weight_hh_l{l}"],
             params[f"{prefix}bias_ih_l{l}"], params[f"{prefix}bias_hh_l{l}"]) for l in range(n_layers)]


def _count_lstm_layers(params: Params, prefix: str) -> int:
    n = 0
    while f"{prefix}weight_ih_l{n}" in params:
        n += 1
    return n


def _gcn(supports, x, w, b, relu, mask):
    """:func:`dense_gcn` as the model functions call it: through the module attribute, and with ``mask`` only when one
    is forced, so a caller that puts a graph convolution of the five-argument form ``(supports, x, w, b, relu)`` in
    place of ``dense_gcn`` still runs the model on it."""
    if mask is None:
        return dense_gcn(supports, x, w, b, relu)
    return dense_gcn(supports, x, w, b, relu, mask)


def dense_cg_lstm(supports: torch.Tensor, obs: torch.Tensor, params: Params, prefix: str,
                  relu=True, lstm=lstm_explicit, hidden=None, mask: Optional[torch.Tensor] = None):
    """``CG_LSTM.forward`` (``STMGCN.py:24-51``).  ``params`` uses the reference ``state_dict`` names
    under ``prefix`` (e.g. ``rnn_list.0.``).  ``relu`` / ``mask``: the temporal GCN's activation and forced ReLU mask
    (:func:`_activate`).  Returns ``(out (B,N,H), (h_n, c_n))``."""
    b_sz, t_len, n, c_in = obs.shape
    x_seq = obs.sum(dim=-1).permute(0, 2, 1)                                    # :36, :39  (B,N,T)
    gconv = _gcn(supports, x_seq, params[prefix + "gconv_temporal_feats.W"],
                 params.get(prefix + "gconv_temporal_feats.b"), relu, mask)       # :40
    x_hat = x_seq + gconv                                                        # :41
    z = x_hat.sum(dim=1) / n                                                     # :42  (B,T)
    fw, fb = params[prefix + "fc.weight"], params[prefix + "fc.bias"]
    s = torch.sigmoid(torch.relu(z @ fw.t() + fb) @ fw.t() + fb)                 # :43 (same fc twice)
    mod = obs * s[:, :, None, None]                                              # :44
    rows = mod.permute(0, 2, 1, 3).reshape(b_sz * n, t_len, c_in)                # :47
    layers = _lstm_layers(params, prefix + "lstm.", _count_lstm_layers(params, prefix + "lstm."))
    h0, c0 = (None, None) if hidden is None else hidden
    seq, hc = lstm(rows, layers, h0, c0)                                         # :48
    return seq[:, -1, :].reshape(b_sz, n, -1), hc                                # :50


def dense_st_mgcn(params: Params, obs: torch.Tensor, supports_list: Sequence[torch.Tensor],
                  relu=True, lstm=lstm_explicit, masks=None) -> torch.Tensor:
    """``ST_MGCN.forward`` (``STMGCN.py:100-119``) -> ``(B,N,C)``.  ``relu``: every GCN's activation (:func:`_activate`);
    ``masks`` (ReLU only, optional): the forced ReLU masks of the 2M GCNs, boolean (N, B, q) each, in the kernels' order
    temporal 0, spatial 0, temporal 1, ... (as :class:`SparseOracle` takes them)."""
    if masks is not None and len(masks) != 2 * len(supports_list):
        raise ValueError(f"{len(masks)} ReLU masks for {len(supports_list)} graphs (two GCNs each)")
    fused = None
    for m, sup in enumerate(supports_list):                                       # :112
        mt, ms = (None, None) if masks is None else masks[2 * m:2 * m + 2]
        cg, _ = dense_cg_lstm(sup, obs, params, f"rnn_list.{m}.", relu, lstm, mask=mt)  # :113
        g = _gcn(sup, cg, params[f"gcn_list.{m}.W"], params.get(f"gcn_list.{m}.b"), relu, ms)   # :114
        fused = g if fused is None else fused + g                                 # :116
    return fused @ params["fc.weight"].t() + params["fc.bias"]                   # :118


def dense_loss_and_grads(params: Params, obs: torch.Tensor, y: torch.Tensor,
                         supports_list: Sequence[torch.Tensor], relu=True, lstm=lstm_explicit, masks=None,
                         want_obs: bool = False):
    """MSE(mean) loss (``Main.py:66-67``, ``Model_Trainer.py:38``) + gradient of every parameter (and, with ``want_obs``,
    of ``obs`` under the key ``"obs"``).  ``relu`` / ``masks`` as for :func:`dense_st_mgcn`."""
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
    obs_leaf = obs.detach().clone().requires_grad_(want_obs)
    out = dense_st_mgcn(leaves, obs_leaf, supports_list, relu, lstm, masks)
    loss = torch.mean((out - y) ** 2)
    grads = torch.autograd.grad(loss, list(leaves.values()) + ([obs_leaf] if want_obs else []), allow_unused=True)
    res = {k: g for k, g in zip(list(leaves.keys()) + (["obs"] if want_obs else []), grads)}
    return out.detach(), loss.detach(), res


def init_params(n_graphs: int, seq_len: int, c_in: int, hid: int, n_layers: int, gcn_hid: int,
                n_sup: int, seed: int = 0, bias: bool = True) -> Params:
    """Random parameters with the reference's names, shapes and init *distributions*
    (``GCN.py:17-22`` xavier-normal/zeros, ``nn.Linear``/``nn.LSTM`` defaults) -- distributionally, not
    bit-for-bit, equal to constructing the reference model (tests that need the reference's exact
    init build the reference model instead)."""
    g = torch.Generator().manual_seed(seed)
    p: Params = {}

    def xavier(rows, cols):
        return torch.randn(rows, cols, generator=g) * (2.0 / (rows + cols)) ** 0.5

    def uni(shape, bound):
        return (torch.rand(*shape, generator=g) * 2 - 1) * bound

    for m in range(n_graphs):
        pre = f"rnn_list.{m}."
        p[pre + "gconv_temporal_feats.W"] = xavier(n_sup * seq_len, seq_len)
        if bias:
            p[pre + "gconv_temporal_feats.b"] = uni((seq_len,), 0.1)
        p[pre + "fc.weight"] = uni((seq_len, seq_len), seq_len ** -0.5)
        p[pre + "fc.bias"] = uni((seq_len,), seq_len ** -0.5)
        for l in range(n_layers):
            in_l = c_in if l == 0 else hid
            p[pre + f"lstm.weight_ih_l{l}"] = uni((4 * hid, in_l), hid ** -0.5)
            p[pre + f"lstm.weight_hh_l{l}"] = uni((4 * hid, hid), hid ** -0.5)
            p[pre + f"lstm.bias_ih_l{l}"] = uni((4 * hid,), hid ** -0.5)
            p[pre + f"lstm.bias_hh_l{l}"] = uni((4 * hid,), hid ** -0.5)
        p[f"gcn_list.{m}.W"] = xavier(n_sup * hid, gcn_hid)
        if bias:
            p[f"gcn_list.{m}.b"] = uni((gcn_hid,), 0.1)
    p["fc.weight"] = uni((c_in, gcn_hid), gcn_hid ** -0.5)
    p["fc.bias"] = uni((c_in,), gcn_hid ** -0.5)
    return p


# --------------------------------------------------------------------------------------------------
# sparse restatement with explicit backward (numpy + scipy.sparse)
# --------------------------------------------------------------------------------------------------
def _sigmoid(v):
    return 1.0 / (1.0 + np.exp(-v))


class SparseOracle:
    """Recurrence-on-features forward + hand-written backward, one numpy dtype throughout.

    ``laplacians`` are scipy CSR matrices ``L~_m`` (``supports[1]`` of the reference, taken verbatim
    so a non-unit ``lambda_max`` or an asymmetric graph is handled, SURVEY.md section 0.3).
    Internal layout mirrors the CUDA path: node-major ``(N, B, p)`` feature rows.

    ``relu_masks`` (optional, ReLU only): the ReLU masks to use instead of ``z > 0``, one boolean ``(N, B, q)`` array per
    GCN in the order temporal graph 0, spatial graph 0, temporal graph 1, ...  With the masks a GPU run took, the oracle
    follows the same branch of every ReLU, so a pre-activation within rounding distance of the kink cannot move the
    gradients.
    """

    def __init__(self, params: Dict[str, np.ndarray], laplacians, n_supports: int, relu: bool = True,
                 dtype=np.float64, relu_masks=None):
        self.dt = np.dtype(dtype)
        self.p = {k: np.asarray(v, dtype=self.dt) for k, v in params.items()}
        self.lap = [l.astype(self.dt).tocsr() for l in laplacians]
        self.lap_t = [l.T.tocsr() for l in self.lap]
        self.ks = n_supports
        self.relu = relu
        self.relu_masks = relu_masks
        self.m = len(self.lap)
        n = 0
        while f"rnn_list.0.lstm.weight_ih_l{n}" in self.p:
            n += 1
        self.n_layers = n

    # ---- Chebyshev GCN --------------------------------------------------------------------------
    def _cheb_stack(self, lap, x):
        """x:(N,B,p) -> S:(Ks,N,B,p) with S_0 = x, S_1 = L x, S_k = 2 L S_{k-1} - S_{k-2}."""
        n = x.shape[0]
        flat = x.reshape(n, -1)
        out = [flat]
        if self.ks > 1:
            out.append(lap @ flat)
        for _ in range(2, self.ks):
            out.append(2.0 * (lap @ out[-1]) - out[-2])
        return np.stack(out).reshape((self.ks,) + x.shape)

    def _gcn_pre(self, lap, x, w, b):
        """-> (pre-activation z, stack)."""
        s = self._cheb_stack(lap, x)
        p = x.shape[-1]
        z = sum(s[k] @ w[k * p:(k + 1) * p] for k in range(self.ks))
        if b is not None:
            z = z + b
        return z, s

    def _gcn_fwd(self, lap, x, w, b):
        z, s = self._gcn_pre(lap, x, w, b)
        return (np.maximum(z, 0) if self.relu else z), s

    def _gcn_fwd_masked(self, lap, x, w, b, mask):
        """:meth:`_gcn_fwd` with a given ReLU mask in place of ``z > 0``: ``out = z * mask``."""
        z, s = self._gcn_pre(lap, x, w, b)
        return z * mask, s

    def _gcn_bwd(self, lap_t, s, out, d_out, w, need_dx: bool, mask=None):
        """Spec in SURVEY.md section 8(a) "Backward".  ReLU mask: ``mask`` if given, else ``out > 0``."""
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
            k_ord = self.ks - 1
            if k_ord == 0:
                dx = u[0]
            else:
                b2 = np.zeros_like(u[0])        # b_{k+2}
                b1 = np.zeros_like(u[0])        # b_{k+1}
                for k in range(k_ord, 0, -1):
                    bk = u[k] + 2.0 * (lap_t @ b1) - b2
                    b2, b1 = b1, bk
                dx = u[0] + lap_t @ b1 - b2
            dx = dx.reshape(s.shape[1:])
        return dw, db, dx

    # ---- LSTM -----------------------------------------------------------------------------------
    def _lstm_fwd(self, x, pre):
        """x:(R,T,C) -> saved activations + top h_T."""
        r, t_len, _ = x.shape
        hid = self.p[pre + "weight_hh_l0"].shape[1]
        saved = []
        seq = x
        for l in range(self.n_layers):
            w_ih, w_hh = self.p[pre + f"weight_ih_l{l}"], self.p[pre + f"weight_hh_l{l}"]
            bias = self.p[pre + f"bias_ih_l{l}"] + self.p[pre + f"bias_hh_l{l}"]
            h = np.zeros((r, hid), self.dt)
            c = np.zeros((r, hid), self.dt)
            hs, cs, gs = [], [], []
            for t in range(t_len):
                a = seq[:, t] @ w_ih.T + h @ w_hh.T + bias
                i, f = _sigmoid(a[:, :hid]), _sigmoid(a[:, hid:2 * hid])
                g, o = np.tanh(a[:, 2 * hid:3 * hid]), _sigmoid(a[:, 3 * hid:])
                c = f * c + i * g
                h = o * np.tanh(c)
                hs.append(h), cs.append(c), gs.append((i, f, g, o))
            saved.append((seq, hs, cs, gs))
            seq = np.stack(hs, axis=1)
        return seq[:, -1], saved

    def _lstm_bwd(self, d_top, saved, pre, grads):
        """BPTT; ``d_top`` is the gradient of the top layer's last hidden state.  Returns dx:(R,T,C)."""
        t_len = len(saved[0][1])
        hid = d_top.shape[1]
        d_seq = [np.zeros_like(d_top) for _ in range(t_len)]
        d_seq[-1] = d_top
        for l in range(self.n_layers - 1, -1, -1):
            x_in, hs, cs, gs = saved[l]
            w_ih, w_hh = self.p[pre + f"weight_ih_l{l}"], self.p[pre + f"weight_hh_l{l}"]
            dw_ih, dw_hh = np.zeros_like(w_ih), np.zeros_like(w_hh)
            dbias = np.zeros(4 * hid, self.dt)
            dh_rec = np.zeros_like(d_top)
            dc = np.zeros_like(d_top)
            d_in = []
            for t in range(t_len - 1, -1, -1):
                i, f, g, o = gs[t]
                c_prev = cs[t - 1] if t > 0 else np.zeros_like(cs[0])
                h_prev = hs[t - 1] if t > 0 else np.zeros_like(hs[0])
                dh = d_seq[t] + dh_rec
                tc = np.tanh(cs[t])
                dc = dc + dh * o * (1 - tc * tc)
                da = np.concatenate([dc * g * i * (1 - i), dc * c_prev * f * (1 - f),
                                     dc * i * (1 - g * g), dh * tc * o * (1 - o)], axis=1)
                dw_ih += da.T @ x_in[:, t]
                dw_hh += da.T @ h_prev
                dbias += da.sum(0)
                dh_rec = da @ w_hh
                d_in.append(da @ w_ih)
                dc = dc * f
            d_seq = d_in[::-1]
            grads[pre + f"weight_ih_l{l}"] = dw_ih
            grads[pre + f"weight_hh_l{l}"] = dw_hh
            grads[pre + f"bias_ih_l{l}"] = dbias.copy()
            grads[pre + f"bias_hh_l{l}"] = dbias.copy()
        return np.stack(d_seq, axis=1)

    # ---- whole model ----------------------------------------------------------------------------
    def forward(self, obs: np.ndarray, keep: bool = False):
        """obs:(B,T,N,C) -> y:(B,N,C).  With ``keep`` the tape for :meth:`backward` is stored."""
        obs = np.asarray(obs, self.dt)
        b_sz, t_len, n, c_in = obs.shape
        xo = np.ascontiguousarray(obs.transpose(2, 0, 1, 3))         # (N,B,T,C) node-major
        xt = xo.sum(-1)                                               # (N,B,T)     STMGCN.py:36,39
        tape = []
        fused = None
        for m in range(self.m):
            pre = f"rnn_list.{m}."
            wt, bt = self.p[pre + "gconv_temporal_feats.W"], self.p.get(pre + "gconv_temporal_feats.b")
            mt, ms = self.relu_masks[2 * m:2 * m + 2] if self.relu and self.relu_masks is not None else (None, None)
            gt, st = (self._gcn_fwd(self.lap[m], xt, wt, bt) if mt is None            # STMGCN.py:40
                      else self._gcn_fwd_masked(self.lap[m], xt, wt, bt, mt))
            z = (xt + gt).sum(0) / n                                  # :41-42  (B,T)
            fw, fb = self.p[pre + "fc.weight"], self.p[pre + "fc.bias"]
            a1 = z @ fw.T + fb
            r1 = np.maximum(a1, 0)
            s = _sigmoid(r1 @ fw.T + fb)                              # :43
            rows = (xo * s[None, :, :, None]).reshape(n * b_sz, t_len, c_in)   # :44, :47 (row = n*B+b)
            h_top, saved = self._lstm_fwd(rows, pre + "lstm.")        # :48-50
            hm = h_top.reshape(n, b_sz, -1)
            ws, bs = self.p[f"gcn_list.{m}.W"], self.p.get(f"gcn_list.{m}.b")
            gs, ss = (self._gcn_fwd(self.lap[m], hm, ws, bs) if ms is None            # :114
                      else self._gcn_fwd_masked(self.lap[m], hm, ws, bs, ms))
            fused = gs if fused is None else fused + gs               # :116
            if keep:
                tape.append(dict(st=st, gt=gt, mt=mt, z=z, a1=a1, r1=r1, s=s, saved=saved, ss=ss, gs=gs, ms=ms))
        y = fused @ self.p["fc.weight"].T + self.p["fc.bias"]        # :118  (N,B,C)
        if keep:
            self._tape = dict(obs_nm=xo, fused=fused, per_graph=tape)
        return np.ascontiguousarray(y.transpose(1, 0, 2))

    def backward(self, d_y: np.ndarray) -> Dict[str, np.ndarray]:
        """d_y:(B,N,C) -> gradient of every parameter (reference ``state_dict`` names)."""
        tp = self._tape
        xo, fused = tp["obs_nm"], tp["fused"]
        n, b_sz, t_len, c_in = xo.shape
        dy = np.asarray(d_y, self.dt).transpose(1, 0, 2)               # (N,B,C)
        grads: Dict[str, np.ndarray] = {}
        grads["fc.weight"] = np.tensordot(dy, fused, axes=([0, 1], [0, 1]))
        grads["fc.bias"] = dy.reshape(-1, c_in).sum(0)
        d_fused = dy @ self.p["fc.weight"]                            # (N,B,G)
        for m in range(self.m):
            t = tp["per_graph"][m]
            pre = f"rnn_list.{m}."
            ws = self.p[f"gcn_list.{m}.W"]
            dws, dbs, d_h = self._gcn_bwd(self.lap_t[m], t["ss"], t["gs"], d_fused, ws, True, t["ms"])
            grads[f"gcn_list.{m}.W"] = dws
            if f"gcn_list.{m}.b" in self.p:
                grads[f"gcn_list.{m}.b"] = dbs
            d_rows = self._lstm_bwd(d_h.reshape(n * b_sz, -1), t["saved"], pre + "lstm.", grads)
            d_mod = d_rows.reshape(n, b_sz, t_len, c_in)
            d_s = (d_mod * xo).sum(axis=(0, 3))                       # (B,T)
            fw = self.p[pre + "fc.weight"]
            s = t["s"]
            d_a2 = d_s * s * (1 - s)
            d_fw = d_a2.T @ t["r1"]
            d_fb = d_a2.sum(0)
            d_a1 = (d_a2 @ fw) * (t["a1"] > 0)
            d_fw = d_fw + d_a1.T @ t["z"]
            d_fb = d_fb + d_a1.sum(0)
            grads[pre + "fc.weight"], grads[pre + "fc.bias"] = d_fw, d_fb
            d_z = d_a1 @ fw                                           # (B,T)
            d_gt = np.broadcast_to(d_z[None] / n, t["gt"].shape)
            wt = self.p[pre + "gconv_temporal_feats.W"]
            dwt, dbt, _ = self._gcn_bwd(self.lap_t[m], t["st"], t["gt"], d_gt, wt, False, t["mt"])
            grads[pre + "gconv_temporal_feats.W"] = dwt
            if pre + "gconv_temporal_feats.b" in self.p:
                grads[pre + "gconv_temporal_feats.b"] = dbt
        return grads

    def loss_and_grads(self, obs: np.ndarray, y_true: np.ndarray):
        out = self.forward(obs, keep=True)
        diff = out - np.asarray(y_true, self.dt)
        loss = float(np.mean(diff * diff))
        grads = self.backward(2.0 * diff / diff.size)
        return out, loss, grads


# --------------------------------------------------------------------------------------------------
# the bf16-arithmetic mode (STMGCN_LSTM_PLANES=1), torch fp64 autograd, optionally forced with the kernels' values
# --------------------------------------------------------------------------------------------------
class CsrMatmul(torch.autograd.Function):
    """``L @ X`` for a sparse CSR ``L`` held together with its transpose: the backward is ``L^T @ G`` (torch's own sparse
    autograd is not involved)."""

    @staticmethod
    def forward(ctx, x, lap, lap_t):
        ctx.lap_t = lap_t
        return lap @ x

    @staticmethod
    def backward(ctx, g):
        return ctx.lap_t @ g, None, None


def torch_csr_pair(mat, device="cpu", dtype=torch.float64):
    """``(L, L^T)`` as torch sparse CSR tensors from a scipy matrix, for :class:`CsrMatmul`."""
    def conv(m):
        m = m.tocsr()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")           # "sparse CSR support is in beta"
            return torch.sparse_csr_tensor(torch.from_numpy(m.indptr).long(), torch.from_numpy(m.indices).long(),
                                           torch.from_numpy(m.data).to(dtype), size=m.shape).to(device)
    return conv(mat), conv(mat.T)


class BF16ModeReference:
    """``ST_MGCN`` / ``CG_LSTM`` in the bf16-arithmetic mode (``ops.set_lstm_planes(1)``), as a torch autograd model in
    fp64 (or any dtype) on any device.

    The mode rounds at two places, and so does this model (``rounding=True``):

    * the shared LSTM keeps one bf16 hidden-state plane: :func:`lstm_planes_reference` with ``planes=1``;
    * the spatial GCN's Chebyshev recurrence gathers from bf16 copies, per chain of the support set (one chain ``L~`` for
      ``chebyshev``, two for ``random_walk_diffusion``, segments as ``SupportSet.chain_segments``):
      ``S_1 = X bf16(S_0)``, ``S_k = 2 X bf16(S_{k-1}) - S_{k-2}`` with ``S_{k-2}`` in full precision.

    The rounding is straight-through (:func:`round_bf16`), so the autograd backward is the exact adjoint the kernels run
    (fp32 gathers in the adjoint Clenshaw).  The temporal GCN, the context gate, the projections, the fusion and the
    output FC are not rounded.  ``rounding=False``: two planes and no bf16 gathers, i.e. the model of
    :class:`SparseOracle` (fp32-grade mode).

    ``chains[m]``: the recurrence matrices of graph ``m`` (scipy); ``n_supports = 1 + len(chains[m]) * K``.
    ``relu``: ReLU after both GCNs (else no activation); ``relu_masks`` as for :class:`SparseOracle` (boolean
    ``(N, B, q)`` arrays or tensors, order temporal 0, spatial 0, temporal 1, ...): ``out = z * mask``.

    ``tapes`` (optional, per graph): the kernels' values at every rounding point, in any precision, rows
    ``r = n*B + b`` of the windows this model is given -- ``h``, ``c`` (L, T, R, H) and ``h0`` (L, R, H) as
    :func:`lstm_planes_reference` takes them, and ``s`` (Ks, N, B, H): the spatial stack, ``s[0]`` the fp32 h_top.
    Every operand of the spatial recurrence, and every stack term the projection reads, then takes the tape's value with
    the gradient routed through this model's own value (``tape + (computed - computed.detach())``), so each layer-step
    and each ``S_k`` is one step from the kernels' own inputs and the gradients are the kernels' backward.
    """

    def __init__(self, params: Dict[str, torch.Tensor], chains, n_supports: int, relu: bool = True,
                 rounding: bool = True, relu_masks=None, device="cpu", dtype=torch.float64):
        self.dev, self.dt = torch.device(device), dtype
        self.p = {k: torch.as_tensor(v).to(self.dev, dtype) for k, v in params.items()}
        self.chains = [[torch_csr_pair(c, self.dev, dtype) for c in ch] for ch in chains]
        self.ks, self.relu, self.rounding = n_supports, relu, rounding
        self.masks = None if relu_masks is None else [torch.as_tensor(mk).to(self.dev) for mk in relu_masks]
        self.m = len(chains)
        self.n_layers = _count_lstm_layers(self.p, "rnn_list.0.lstm.")
        assert all(ch and (n_supports - 1) % len(ch) == 0 for ch in self.chains) or n_supports == 1

    def leaves(self) -> Dict[str, torch.Tensor]:
        """Fresh autograd leaves of the parameters (pass them to the methods below)."""
        return {k: v.detach().clone().requires_grad_(True) for k, v in self.p.items()}

    def _rnd(self, v):
        return round_bf16(v) if self.rounding else v

    def _stack(self, m, x, spatial: bool, tape_s=None):
        """x (N, B, p) -> (terms the projection reads, terms as computed): (Ks, N, B*p) each; ``spatial``: the recurrence
        gathers from bf16 copies (rounding on) and is forced with ``tape_s``."""
        n = x.shape[0]
        flat = x.reshape(n, -1)
        rnd = self._rnd if spatial else (lambda v: v)

        def forced(k, computed):
            if tape_s is None:
                return computed
            return tape_s[k].reshape(n, -1) + (computed - computed.detach())
        used, comp = [forced(0, flat)] + [None] * (self.ks - 1), [flat] + [None] * (self.ks - 1)
        chains = self.chains[m] if self.ks > 1 else []
        k_ord = (self.ks - 1) // max(len(chains), 1)
        for c, (lap, lap_t) in enumerate(chains):
            seg = [0] + list(range(1 + c * k_ord, 1 + (c + 1) * k_ord))
            for j in range(1, len(seg)):
                y = CsrMatmul.apply(rnd(used[seg[j - 1]]), lap, lap_t)
                if j > 1:
                    y = 2.0 * y - used[seg[j - 2]]
                comp[seg[j]], used[seg[j]] = y, forced(seg[j], y)
        return used, comp

    def _gcn(self, m, x, w, b, mask_i, spatial, tape_s=None, windows=None):
        """act(sum_k S_k W_k + b) on node-major x (N, B, p) -> (out (N, B, q), computed stack terms).  ``windows``: the
        slice of the masks' batch that x holds."""
        n, bsz, p = x.shape
        used, comp = self._stack(m, x, spatial, tape_s)
        z = sum(used[k].reshape(n, bsz, p) @ w[k * p:(k + 1) * p] for k in range(self.ks))
        if b is not None:
            z = z + b
        if self.relu and self.masks is not None:
            mask = self.masks[mask_i] if windows is None else self.masks[mask_i][:, windows]
            z = z * mask.to(z.dtype)
        elif self.relu:
            z = torch.relu(z)
        return z, comp

    def cg_lstm_node_major(self, p, m, xo, tape=None, h0=None, c0=None, windows=None):
        """Graph ``m``'s ``CG_LSTM`` on node-major xo (N, B, T, C) -> (h_top (N, B, H), h_n, c_n (L, R, H), (hs, cs)):
        ``hs`` / ``cs`` the computed states of every layer-step (see :func:`lstm_planes_reference`).  ``windows``: the
        slice of the masks' batch that xo holds (``tape`` is taken as given, already sliced)."""
        pre = f"rnn_list.{m}."
        n, bsz, t_len, c_in = xo.shape
        xt = xo.sum(-1)
        gt, _ = self._gcn(m, xt, p[pre + "gconv_temporal_feats.W"], p.get(pre + "gconv_temporal_feats.b"), 2 * m,
                          False, windows=windows)
        z = (xt + gt).sum(0) / n
        fw, fb = p[pre + "fc.weight"], p[pre + "fc.bias"]
        s = torch.sigmoid(torch.relu(z @ fw.t() + fb) @ fw.t() + fb)
        rows = (xo * s[None, :, :, None]).reshape(n * bsz, t_len, c_in)
        layers = _lstm_layers(p, pre + "lstm.", self.n_layers)
        lstm_tape = None if tape is None else {k: tape[k] for k in ("h", "c", "h0") if k in tape}
        _, (h_n, c_n), (hs, cs) = lstm_planes_reference(rows, layers, 1 if self.rounding else 2, h0, c0, lstm_tape)
        return hs[-1][-1].reshape(n, bsz, -1), h_n, c_n, (hs, cs)

    def cg_lstm(self, p, obs, hidden=None, tape=None, m=0):
        """``CG_LSTM.forward`` on graph ``m``: obs (B, T, N, C), ``hidden`` = (h0, c0) (L, B*N, H) with the module's rows
        ``b*N + n``, or None -> (out (B, N, H), (h_n, c_n)) in the module's layout.  ``tape`` rows are ``n*B + b``."""
        bsz, _, n, _ = obs.shape
        h0 = c0 = None
        if hidden is not None:
            lyr, _, hid = hidden[0].shape
            h0, c0 = (v.reshape(lyr, bsz, n, hid).permute(0, 2, 1, 3).reshape(lyr, n * bsz, hid) for v in hidden)
        h_top, h_n, c_n, _ = self.cg_lstm_node_major(p, m, obs.permute(2, 0, 1, 3), tape, h0, c0)
        to_module = lambda v: v.reshape(v.shape[0], n, bsz, -1).permute(0, 2, 1, 3).reshape(v.shape[0], bsz * n, -1)  # noqa: E731
        return h_top.permute(1, 0, 2), (to_module(h_n), to_module(c_n))

    def branch(self, p, m, xo, tape=None, windows=None):
        """Graph ``m``'s branch of ``ST_MGCN`` on node-major xo -> dict: ``out`` (N, B, G) and the computed values of
        every rounding point -- ``hs`` / ``cs`` (per layer, per step) and ``stack`` (spatial S_k, (N, B*H) each).

        ``windows`` (a slice, optional): xo holds only these windows of the batch that ``relu_masks`` and ``tape``
        describe; the masks and the tape are sliced to them.  The tape may be in any precision (the kernels' own: h in
        bf16, c and s in fp32): only the slice taken is cast to this model's dtype."""
        if tape is not None:
            tape = _tape_windows(tape, xo.shape[0], slice(None) if windows is None else windows, self.dt)
        h_top, _, _, (hs, cs) = self.cg_lstm_node_major(p, m, xo, tape, windows=windows)
        g, stack = self._gcn(m, h_top, p[f"gcn_list.{m}.W"], p.get(f"gcn_list.{m}.b"), 2 * m + 1, True,
                             None if tape is None else tape["s"], windows)
        return dict(out=g, hs=hs, cs=cs, stack=stack)

    def forward(self, p, obs, tapes=None):
        """``ST_MGCN.forward``: obs (B, T, N, C) -> y (B, N, C), all branches in one autograd graph."""
        xo = obs.permute(2, 0, 1, 3)
        fused = sum(self.branch(p, m, xo, None if tapes is None else tapes[m])["out"] for m in range(self.m))
        return (fused @ p["fc.weight"].t() + p["fc.bias"]).permute(1, 0, 2)

    def loss_and_grads(self, obs, y, tapes=None, want_obs: bool = False, on_branch=None, window_chunk=None):
        """MSE(mean) loss and the gradient of every parameter (and of obs with ``want_obs``), one graph branch in memory
        at a time: the branches' outputs first (no autograd), then the fusion's gradient, then each branch's backward.
        ``on_branch(m, branch dict)`` (optional) sees each branch's forward values, once per chunk with ``window_chunk``;
        ``branch["windows"]`` is the slice of the batch they belong to (all of it without chunks).  Returns (out, loss,
        grads).

        ``window_chunk`` (optional): each branch's forward and backward run on ``window_chunk`` windows at a time (the
        last chunk may be shorter), so the autograd tape held at once is that of one chunk of one branch.  Windows are
        independent (``STMGCN.py:47``: the only reductions are over the regions of one window and over graphs), so the
        fusion's gradient is taken on the whole batch and each chunk's backward, seeded with its windows' share of it,
        adds that chunk's exact contribution to the parameter gradients (and writes its windows' d obs)."""
        obs = torch.as_tensor(obs).to(self.dev, self.dt)
        y = torch.as_tensor(y).to(self.dev, self.dt)
        bsz = obs.shape[0]
        if window_chunk is None:
            wins = [None]
        else:
            if window_chunk < 1:
                raise ValueError(f"window_chunk must be at least 1, got {window_chunk}")
            wins = [slice(i, min(i + window_chunk, bsz)) for i in range(0, bsz, window_chunk)]
        p = self.leaves()
        xo = obs.permute(2, 0, 1, 3)
        with torch.no_grad():
            outs = []
            for m in range(self.m):
                parts = []
                for win in wins:
                    br = self.branch(p, m, xo if win is None else xo[:, win], None if tapes is None else tapes[m], win)
                    if on_branch is not None:
                        br["windows"] = slice(0, bsz) if win is None else win
                        on_branch(m, br)
                    parts.append(br["out"])
                    del br
                outs.append(parts[0] if len(parts) == 1 else torch.cat(parts, dim=1))
                del parts
        gs = [o.requires_grad_(True) for o in outs]
        out = (sum(gs) @ p["fc.weight"].t() + p["fc.bias"]).permute(1, 0, 2)
        loss = torch.mean((out - y) ** 2)
        top = torch.autograd.grad(loss, gs + [p["fc.weight"], p["fc.bias"]])
        grads = {"fc.weight": top[-2], "fc.bias": top[-1]}
        d_obs = torch.zeros_like(obs) if want_obs else None
        for m in range(self.m):
            keys = [k for k in p if k.startswith((f"rnn_list.{m}.", f"gcn_list.{m}."))]
            for win in wins:
                ob = (obs if win is None else obs[win]).detach().clone().requires_grad_(want_obs)
                g = self.branch(p, m, ob.permute(2, 0, 1, 3), None if tapes is None else tapes[m], win)["out"]
                res = torch.autograd.grad(g, [p[k] for k in keys] + ([ob] if want_obs else []),
                                          grad_outputs=top[m] if win is None else top[m][:, win])
                for k, r in zip(keys, res):
                    grads[k] = r if k not in grads else grads[k] + r
                if want_obs:
                    d_obs[slice(None) if win is None else win] += res[-1]
                del g, res
        if want_obs:
            grads["obs"] = d_obs
        return out.detach(), loss.detach(), grads


def _tape_windows(tape, n, windows, dtype=None):
    """A :class:`BF16ModeReference` tape (rows ``r = n*B + b``) cut to the windows ``windows`` (a slice of the B), in
    ``dtype`` (given): a tape kept in the kernels' precision is widened one slice at a time."""
    def rows(v, axis):                  # (..., N*B, ...) -> (..., N*len(windows), ...)
        shape = v.shape
        v = v.reshape(shape[:axis] + (n, shape[axis] // n) + shape[axis + 1:])
        v = v[(slice(None),) * (axis + 1) + (windows,)]
        return v.reshape(shape[:axis] + (-1,) + shape[axis + 1:])
    row_axis = {"h": 2, "c": 2, "h0": 1}          # h, c (L, T, R, H); h0 (L, R, H); s (Ks, N, B, H)
    cut = {k: v[:, :, windows] if k == "s" else rows(v, row_axis[k]) for k, v in tape.items()}
    return cut if dtype is None else {k: v.to(dtype) for k, v in cut.items()}


def laplacian_csr_from_supports(supports: torch.Tensor):
    """scipy CSR of ``supports[1]`` (the rescaled Laplacian), exact zeros dropped."""
    import scipy.sparse as sp
    if supports.shape[0] < 2:                       # order-0 stack: only T_0 = I, no Laplacian needed
        return sp.csr_matrix((supports.shape[1], supports.shape[1]), dtype=np.float32)
    return sp.csr_matrix(supports[1].detach().cpu().numpy())


def max_rel_err(new, ref) -> float:
    """Parity metric of SURVEY.md section 8(d): ``max|new - ref| / max|ref|``."""
    new = np.asarray(new, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    den = float(np.max(np.abs(ref)))
    return float(np.max(np.abs(new - ref)) / (den if den > 0 else 1.0))
