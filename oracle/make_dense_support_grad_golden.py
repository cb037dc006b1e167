"""Generate ``tests/golden/dense_support_grad_ref.npz``: the gradients the UNMODIFIED reference ST-MGCN gives its dense
support stacks (``GCN.py:34-36`` differentiated in ``A[k]``) and, through ``Adj_Preprocessor.process``, the adjacency
behind them; CPU fp32.

TEST INFRASTRUCTURE.  Needs a checkout of the reference (its ``GCN.py`` / ``STMGCN.py``); the fixture it writes is
committed, so the tests never need the reference itself:

    python oracle/make_dense_support_grad_golden.py /path/to/reference

Four cases, each stored under its own key prefix ``<case>.``:

* ``cheb_leaf``: ``ST_MGCN`` (M = 2, Chebyshev K = 2) whose two stacks ``process(adj_g)`` are autograd leaves: the MSE
  loss's ``stack_grad.<g>``;
* ``localpool_leaf``: the same with ``localpool`` stacks (one support, not ``I``);
* ``cheb_adj``: ``ST_MGCN`` (M = 2, Chebyshev K = 2) on ``process(adj_g)`` with ``adj_g`` requiring grad: ``adj_grad.<g>``;
* ``cglstm_adj``: the first ``CG_LSTM`` alone on ``process(adj_0)`` (Chebyshev K = 2), zero initial state, the scalar
  ``sum(out * probe)``: ``adj_grad.0``.

Stored per case: ``meta`` (``n, m, k, t, b, c, hid, layers, gcn_hid``), ``kernel_type``, ``adj.<g>``, ``supports.<g>``,
the reference model's parameters ``param.*`` (its ``state_dict`` after ``torch.manual_seed(seed)``), ``x``, ``y`` (or
``probe``), ``out``, ``loss``, every parameter gradient ``grad.*`` and the support or adjacency gradients above.  The
graphs are symmetric, weighted and connected (a ring under random edges): no region has a zero degree, whose
``pow(0, -0.5)`` would make the adjacency's gradient NaN.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import make_golden  # noqa: E402

N, M, T, B, C, HID, LAYERS, GCN_HID = 20, 2, 5, 3, 1, 16, 2, 8


def graph(n: int, seed: int) -> torch.Tensor:
    """Symmetric weighted adjacency: a ring plus random chords, no self-loops."""
    gen = torch.Generator().manual_seed(seed)
    a = (torch.rand(n, n, generator=gen) < 0.2).float() * (0.5 + torch.rand(n, n, generator=gen))
    ring = torch.zeros(n, n)
    idx = torch.arange(n)
    ring[idx, (idx + 1) % n] = 1.0
    a = a + ring
    a = 0.5 * (a + a.t())
    a.fill_diagonal_(0.0)
    return a


def case(blob: dict, name: str, kernel_type: str, k: int, leaf: bool, cg_only: bool, seed: int) -> None:
    ref_gcn, ref_stmgcn = make_golden.import_reference()
    adjs = [graph(N, 10 * seed + g) for g in range(M)]
    if not leaf:
        adjs = [a.clone().requires_grad_(True) for a in adjs]
    pre = ref_gcn.Adj_Preprocessor(kernel_type, k)
    sups = [pre.process(a) for a in adjs]
    if leaf:
        sups = [s.detach().clone().requires_grad_(True) for s in sups]
    torch.manual_seed(seed)
    model = ref_stmgcn.ST_MGCN(M=M, seq_len=T, n_nodes=N, input_dim=C, lstm_hidden_dim=HID, lstm_num_layers=LAYERS,
                               gcn_hidden_dim=GCN_HID, sta_kernel_config={"kernel_type": kernel_type, "K": k},
                               gconv_use_bias=True, gconv_activation=nn.ReLU)
    x = torch.randn(B, T, N, C)
    p = name + "."
    if cg_only:
        cg = model.rnn_list[0]
        out, _ = cg(sups[0], x, cg.init_hidden(B))
        probe = torch.randn(out.shape)
        loss = (out * probe).sum()
        blob[p + "probe"] = probe.numpy()
    else:
        y = torch.randn(B, N, C)
        out = model(obs_seq=x, sta_adj_list=sups)
        loss = nn.MSELoss(reduction="mean")(out, y)
        blob[p + "y"] = y.numpy()
    loss.backward()
    blob[p + "meta"] = np.array([N, M, k, T, B, C, HID, LAYERS, GCN_HID], dtype=np.int64)
    blob[p + "kernel_type"] = np.array(kernel_type)
    blob[p + "x"] = x.numpy()
    blob[p + "out"] = out.detach().numpy()
    blob[p + "loss"] = np.array(loss.item(), dtype=np.float64)
    for g, (a, s) in enumerate(zip(adjs, sups)):
        blob[p + f"adj.{g}"] = a.detach().numpy()
        blob[p + f"supports.{g}"] = s.detach().numpy()
        grad = s.grad if leaf else a.grad
        if grad is not None:
            blob[p + (f"stack_grad.{g}" if leaf else f"adj_grad.{g}")] = grad.numpy()
    for key, val in model.state_dict().items():
        blob[p + "param." + key] = val.numpy()
    for key, val in model.named_parameters():
        if val.grad is not None:
            blob[p + "grad." + key] = val.grad.numpy()


if __name__ == "__main__":
    ref = os.path.abspath(sys.argv[1]) if len(sys.argv) > 1 else make_golden.REF
    if not os.path.exists(os.path.join(ref, "STMGCN.py")):
        sys.exit("usage: python oracle/make_dense_support_grad_golden.py /path/to/reference")
    make_golden.REF = ref
    torch.set_num_threads(1)
    blob: dict = {}
    case(blob, "cheb_leaf", "chebyshev", 2, leaf=True, cg_only=False, seed=1)
    case(blob, "localpool_leaf", "localpool", 1, leaf=True, cg_only=False, seed=2)
    case(blob, "cheb_adj", "chebyshev", 2, leaf=False, cg_only=False, seed=3)
    case(blob, "cglstm_adj", "chebyshev", 2, leaf=False, cg_only=True, seed=4)
    path = os.path.join(REPO, "tests", "golden", "dense_support_grad_ref.npz")
    np.savez_compressed(path, **blob)
    print(f"{path}: {len(blob)} arrays ({os.path.getsize(path) / 1024:.0f} KiB)")
