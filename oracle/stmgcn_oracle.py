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

Parity pin: the reference has no tests, golden vectors or fixtures of its own (SURVEY.md section 4) --
"parity unpinned" by the reference's own tests.  The pin used here is the reference code itself,
imported from a reference checkout (``oracle/make_golden.py`` ->
``tests/golden/*.npz``; ``tests/test_oracle.py::test_dense_matches_reference_modules``).
"""
from __future__ import annotations

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
    eye = torch.eye(adj.shape[0], dtype=adj.dtype)
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


# --------------------------------------------------------------------------------------------------
# dense restatement (torch CPU; autograd supplies the backward)
# --------------------------------------------------------------------------------------------------
def dense_gcn(supports: torch.Tensor, x: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor],
              relu: bool = True) -> torch.Tensor:
    """``GCN.forward`` (``GCN.py:24-43``): ``act(cat_k(A_k x) W + b)``; rows ``[k p,(k+1) p)`` of W
    pair with support k."""
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
    return torch.relu(out) if relu else out


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


def dense_cg_lstm(supports: torch.Tensor, obs: torch.Tensor, params: Params, prefix: str,
                  relu: bool = True, lstm=lstm_explicit, hidden=None):
    """``CG_LSTM.forward`` (``STMGCN.py:24-51``).  ``params`` uses the reference ``state_dict`` names
    under ``prefix`` (e.g. ``rnn_list.0.``).  Returns ``(out (B,N,H), (h_n, c_n))``."""
    b_sz, t_len, n, c_in = obs.shape
    x_seq = obs.sum(dim=-1).permute(0, 2, 1)                                    # :36, :39  (B,N,T)
    gconv = dense_gcn(supports, x_seq, params[prefix + "gconv_temporal_feats.W"],
                      params.get(prefix + "gconv_temporal_feats.b"), relu)        # :40
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
                  relu: bool = True, lstm=lstm_explicit) -> torch.Tensor:
    """``ST_MGCN.forward`` (``STMGCN.py:100-119``) -> ``(B,N,C)``."""
    fused = None
    for m, sup in enumerate(supports_list):                                       # :112
        cg, _ = dense_cg_lstm(sup, obs, params, f"rnn_list.{m}.", relu, lstm)      # :113
        g = dense_gcn(sup, cg, params[f"gcn_list.{m}.W"], params.get(f"gcn_list.{m}.b"), relu)  # :114
        fused = g if fused is None else fused + g                                 # :116
    return fused @ params["fc.weight"].t() + params["fc.bias"]                   # :118


def dense_loss_and_grads(params: Params, obs: torch.Tensor, y: torch.Tensor,
                         supports_list: Sequence[torch.Tensor], relu: bool = True, lstm=lstm_explicit):
    """MSE(mean) loss (``Main.py:66-67``, ``Model_Trainer.py:38``) + gradient of every parameter."""
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
    out = dense_st_mgcn(leaves, obs, supports_list, relu, lstm)
    loss = torch.mean((out - y) ** 2)
    grads = torch.autograd.grad(loss, list(leaves.values()), allow_unused=True)
    return out.detach(), loss.detach(), {k: g for k, g in zip(leaves.keys(), grads)}


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
    """

    def __init__(self, params: Dict[str, np.ndarray], laplacians, n_supports: int, relu: bool = True,
                 dtype=np.float64):
        self.dt = np.dtype(dtype)
        self.p = {k: np.asarray(v, dtype=self.dt) for k, v in params.items()}
        self.lap = [l.astype(self.dt).tocsr() for l in laplacians]
        self.lap_t = [l.T.tocsr() for l in self.lap]
        self.ks = n_supports
        self.relu = relu
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

    def _gcn_fwd(self, lap, x, w, b):
        s = self._cheb_stack(lap, x)
        p = x.shape[-1]
        z = sum(s[k] @ w[k * p:(k + 1) * p] for k in range(self.ks))
        if b is not None:
            z = z + b
        return (np.maximum(z, 0) if self.relu else z), s

    def _gcn_bwd(self, lap_t, s, out, d_out, w, need_dx: bool):
        """Spec in SURVEY.md section 8(a) "Backward"."""
        p = s.shape[-1]
        dz = d_out * (out > 0) if self.relu else d_out
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
            gt, st = self._gcn_fwd(self.lap[m], xt, wt, bt)           # STMGCN.py:40
            z = (xt + gt).sum(0) / n                                  # :41-42  (B,T)
            fw, fb = self.p[pre + "fc.weight"], self.p[pre + "fc.bias"]
            a1 = z @ fw.T + fb
            r1 = np.maximum(a1, 0)
            s = _sigmoid(r1 @ fw.T + fb)                              # :43
            rows = (xo * s[None, :, :, None]).reshape(n * b_sz, t_len, c_in)   # :44, :47 (row = n*B+b)
            h_top, saved = self._lstm_fwd(rows, pre + "lstm.")        # :48-50
            hm = h_top.reshape(n, b_sz, -1)
            ws, bs = self.p[f"gcn_list.{m}.W"], self.p.get(f"gcn_list.{m}.b")
            gs, ss = self._gcn_fwd(self.lap[m], hm, ws, bs)           # :114
            fused = gs if fused is None else fused + gs               # :116
            if keep:
                tape.append(dict(st=st, gt=gt, z=z, a1=a1, r1=r1, s=s, saved=saved, ss=ss, gs=gs))
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
            dws, dbs, d_h = self._gcn_bwd(self.lap_t[m], t["ss"], t["gs"], d_fused, ws, True)
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
            dwt, dbt, _ = self._gcn_bwd(self.lap_t[m], t["st"], t["gt"], d_gt, wt, False)
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
