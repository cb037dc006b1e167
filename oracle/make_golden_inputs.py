"""Generate ``tests/golden/inputgrad_ref.npz``: the gradients at the model's inputs and recurrent state, computed by the
UNMODIFIED reference ST-MGCN checkout on CPU fp32.

TEST INFRASTRUCTURE, kept apart from ``make_golden.py`` so that the four existing fixtures are never regenerated:

    python oracle/make_golden_inputs.py /path/to/reference

Two cases, keys prefixed ``st.`` / ``cg.``:

* ``st``: ``ST_MGCN`` (3 graphs, C = 2, weighted asymmetric adjacency, odd sizes) with ``obs_seq.requires_grad`` and an
  MSE loss.  Stores the supports, ``state_dict``, inputs, output, loss, ``grad_obs`` and every parameter gradient.
* ``cg``: ``CG_LSTM`` with ``obs_seq``, ``h0`` and ``c0`` requiring grad; loss ``mse(out, y) + <h_n, r1> + <c_n, r2>``.
  Stores ``grad_obs``, ``grad_h0``, ``grad_c0`` and every parameter gradient besides the inputs and outputs.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)


def _adjacencies(n, m, density):
    sys.path.insert(0, os.path.join(REPO, "st-mgcn_b200"))
    from stmgcn_b200 import synth
    adjs = [synth.make_adjacency(n, g, density) for g in range(m)]
    gen = torch.Generator().manual_seed(78)
    return [a * (0.25 + torch.rand(n, n, generator=gen)) for a in adjs]       # weighted, asymmetric => asymmetric L~


def st_case(ref_gcn, ref_stmgcn, blob):
    n, m, k, t, b, c, hid, layers, gcn_hid = 37, 3, 3, 5, 3, 2, 16, 2, 24
    adjs = _adjacencies(n, m, 0.15)
    sups = [ref_gcn.Adj_Preprocessor("chebyshev", k).process(a) for a in adjs]
    torch.manual_seed(11)
    model = ref_stmgcn.ST_MGCN(M=m, seq_len=t, n_nodes=n, input_dim=c, lstm_hidden_dim=hid, lstm_num_layers=layers,
                               gcn_hidden_dim=gcn_hid, sta_kernel_config={"kernel_type": "chebyshev", "K": k},
                               gconv_use_bias=True, gconv_activation=nn.ReLU)
    x = torch.randn(b, t, n, c).requires_grad_(True)
    y = torch.randn(b, n, c)
    out = model(obs_seq=x, sta_adj_list=sups)
    loss = nn.MSELoss(reduction="mean")(out, y)
    loss.backward()
    blob["st.meta"] = np.array([n, m, k, t, b, c, hid, layers, gcn_hid], dtype=np.int64)
    blob.update({"st.x": x.detach().numpy(), "st.y": y.numpy(), "st.out": out.detach().numpy(),
                 "st.loss": np.array(loss.item(), dtype=np.float64), "st.grad_obs": x.grad.numpy()})
    for g, s in enumerate(sups):
        blob[f"st.supports.{g}"] = s.numpy()
    for key, val in model.state_dict().items():
        blob["st.param." + key] = val.numpy()
    for key, val in model.named_parameters():
        blob["st.grad." + key] = val.grad.numpy()
    return f"st: loss {loss.item():.6f}, |d obs| {float(x.grad.abs().max()):.3g}"


def cg_case(ref_gcn, ref_stmgcn, blob):
    n, k, t, b, c, hid, layers = 29, 2, 6, 3, 3, 16, 2
    adj = _adjacencies(n, 1, 0.2)[0]
    sup = ref_gcn.Adj_Preprocessor("chebyshev", k).process(adj)
    torch.manual_seed(12)
    model = ref_stmgcn.CG_LSTM(seq_len=t, n_nodes=n, input_dim=c, lstm_hidden_dim=hid, lstm_num_layers=layers, K=k + 1,
                               gconv_use_bias=True, gconv_activation=nn.ReLU)
    x = torch.randn(b, t, n, c).requires_grad_(True)
    h0 = (0.3 * torch.randn(layers, b * n, hid)).requires_grad_(True)
    c0 = (0.5 * torch.randn(layers, b * n, hid)).requires_grad_(True)
    y = torch.randn(b, n, hid)
    r1, r2 = torch.randn(layers, b * n, hid), torch.randn(layers, b * n, hid)
    out, (h_n, c_n) = model(sup, x, (h0, c0))
    loss = nn.MSELoss(reduction="mean")(out, y) + (h_n * r1).sum() + (c_n * r2).sum()
    loss.backward()
    blob["cg.meta"] = np.array([n, k, t, b, c, hid, layers], dtype=np.int64)
    blob.update({"cg.supports": sup.numpy(), "cg.x": x.detach().numpy(), "cg.h0": h0.detach().numpy(),
                 "cg.c0": c0.detach().numpy(), "cg.y": y.numpy(), "cg.r1": r1.numpy(), "cg.r2": r2.numpy(),
                 "cg.out": out.detach().numpy(), "cg.h_n": h_n.detach().numpy(), "cg.c_n": c_n.detach().numpy(),
                 "cg.loss": np.array(loss.item(), dtype=np.float64), "cg.grad_obs": x.grad.numpy(),
                 "cg.grad_h0": h0.grad.numpy(), "cg.grad_c0": c0.grad.numpy()})
    for key, val in model.state_dict().items():
        blob["cg.param." + key] = val.numpy()
    for key, val in model.named_parameters():
        blob["cg.grad." + key] = val.grad.numpy()
    return f"cg: loss {loss.item():.6f}, |d h0| {float(h0.grad.abs().max()):.3g}"


if __name__ == "__main__":
    ref = os.path.abspath(sys.argv[1]) if len(sys.argv) > 1 else os.environ.get("STMGCN_REFERENCE_DIR", "")
    if not os.path.exists(os.path.join(ref, "STMGCN.py")):
        sys.exit("usage: python oracle/make_golden_inputs.py /path/to/reference  (the directory with GCN.py and STMGCN.py)")
    sys.path.insert(0, HERE)
    import make_golden
    make_golden.REF = ref
    torch.set_num_threads(1)
    ref_gcn, ref_stmgcn = make_golden.import_reference()
    blob = {}
    print(st_case(ref_gcn, ref_stmgcn, blob))
    print(cg_case(ref_gcn, ref_stmgcn, blob))
    path = os.path.join(REPO, "tests", "golden", "inputgrad_ref.npz")
    np.savez_compressed(path, **blob)
    print(f"-> {path} ({os.path.getsize(path) / 1024:.0f} KiB)")
