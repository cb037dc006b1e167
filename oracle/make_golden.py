"""Generate ``tests/golden/*.npz`` by running the UNMODIFIED reference ST-MGCN checkout on CPU fp32.

TEST INFRASTRUCTURE.  Needs a checkout of the reference (its ``GCN.py`` / ``STMGCN.py``); the fixtures it writes are
committed, so the tests never need the reference itself:

    python oracle/make_golden.py /path/to/reference

Each fixture stores: the adjacency matrices, the reference's supports ``Adj_Preprocessor.process``
(``GCN.py:57-97``), the reference model's ``state_dict`` after ``torch.manual_seed(seed)`` construction,
inputs ``x, y``, the forward output of ``ST_MGCN.forward`` (``STMGCN.py:100-119``), the MSE loss and the
autograd gradient of every parameter.  Reference modules are imported under their own names from a
temporary ``sys.path`` entry and removed again so they can never shadow the repo's drop-in modules.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
REF = os.environ.get("STMGCN_REFERENCE_DIR", "")     # set from the command line, see __main__


def import_reference():
    """Import the reference ``GCN`` / ``STMGCN`` modules as private objects (not left in sys.modules)."""
    saved = {k: sys.modules.pop(k) for k in ("GCN", "STMGCN") if k in sys.modules}
    sys.path.insert(0, REF)
    try:
        import GCN as ref_gcn          # noqa: N811
        import STMGCN as ref_stmgcn    # noqa: N811
    finally:
        sys.path.remove(REF)
        for k in ("GCN", "STMGCN"):
            sys.modules.pop(k, None)
        sys.modules.update(saved)
    return ref_gcn, ref_stmgcn


def build_case(name, n, m, k, t, b, c, hid, layers, gcn_hid, density, seed, weighted=False):
    sys.path.insert(0, os.path.join(REPO, "st-mgcn_b200"))
    from stmgcn_b200 import synth
    ref_gcn, ref_stmgcn = import_reference()
    adjs = [synth.make_adjacency(n, g, density) for g in range(m)]
    if weighted:                                    # asymmetric, weighted => asymmetric L~
        gen = torch.Generator().manual_seed(77)
        adjs = [a * (0.25 + torch.rand(n, n, generator=gen)) for a in adjs]
    sups = [ref_gcn.Adj_Preprocessor("chebyshev", k).process(a) for a in adjs]
    torch.manual_seed(seed)
    model = ref_stmgcn.ST_MGCN(M=m, seq_len=t, n_nodes=n, input_dim=c, lstm_hidden_dim=hid,
                               lstm_num_layers=layers, gcn_hidden_dim=gcn_hid,
                               sta_kernel_config={"kernel_type": "chebyshev", "K": k},
                               gconv_use_bias=True, gconv_activation=nn.ReLU)
    x = torch.randn(b, t, n, c)
    y = torch.randn(b, n, c)
    out = model(obs_seq=x, sta_adj_list=sups)
    loss = nn.MSELoss(reduction="mean")(out, y)
    loss.backward()
    blob = {"meta": np.array([n, m, k, t, b, c, hid, layers, gcn_hid], dtype=np.int64),
            "x": x.numpy(), "y": y.numpy(), "out": out.detach().numpy(),
            "loss": np.array(loss.item(), dtype=np.float64)}
    for g, (a, s) in enumerate(zip(adjs, sups)):
        blob[f"adj.{g}"] = a.numpy()
        blob[f"supports.{g}"] = s.numpy()
    for key, val in model.state_dict().items():
        blob["param." + key] = val.numpy()
    for key, val in model.named_parameters():
        blob["grad." + key] = val.grad.numpy()
    path = os.path.join(REPO, "tests", "golden", name + ".npz")
    np.savez_compressed(path, **blob)
    print(f"{name}: out|max|={float(out.abs().max()):.4g} loss={loss.item():.6f} -> {path} "
          f"({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    REF = os.path.abspath(sys.argv[1]) if len(sys.argv) > 1 else REF
    if not os.path.exists(os.path.join(REF, "STMGCN.py")):
        sys.exit("usage: python oracle/make_golden.py /path/to/reference  (the directory with GCN.py and STMGCN.py)")
    torch.set_num_threads(1)
    # BASELINE.json configs[0]: 64 regions, 1 graph, K=2, seq_len=4, batch=8, H=G=64, L=3, C=1.
    build_case("cfg1_ref", 64, 1, 2, 4, 8, 1, 64, 3, 64, 0.10, seed=0)
    # ragged/small case: 3 graphs, weighted asymmetric adjacency, C=2, odd sizes.
    build_case("ragged_ref", 37, 3, 3, 5, 3, 2, 16, 2, 24, 0.15, seed=1, weighted=True)
    # BASELINE.json configs[1]/[2] hyper-parameters (3 graphs, K=3, seq_len=12, H=G=64, L=3, C=1) at a size the reference
    # finishes in seconds: 96 regions x batch 6 = 576 LSTM rows (4.5 tiles of 128: ragged last tile on the GPU).
    build_case("cfg3_small_ref", 96, 3, 3, 12, 6, 1, 64, 3, 64, 0.05, seed=2)
    # two graphs, two LSTM layers, narrow hidden sizes (H=16, G=8): pins the oracle's dense restatement to the reference
    # modules away from the H=64 shapes of the other fixtures.
    build_case("small_ref", 30, 2, 3, 5, 2, 1, 16, 2, 8, 0.2, seed=3)
