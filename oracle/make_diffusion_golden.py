"""Generate ``tests/golden/diffusion_ref.npz``: the UNMODIFIED reference ST-MGCN on bidirectional random-walk diffusion
supports, CPU fp32.

TEST INFRASTRUCTURE.  Needs a checkout of the reference (its ``GCN.py`` / ``STMGCN.py``); the fixture it writes is
committed, so the tests never need the reference itself:

    python oracle/make_diffusion_golden.py /path/to/reference

The reference's ``Adj_Preprocessor.process`` builds only the forward ``K+1`` diffusion stack, while its ``ST_MGCN``
sizes every GCN for ``2K+1`` supports (``STMGCN.py:87-88``), so ``kernel_type='random_walk_diffusion'`` does not run
there as shipped.  The ``2K+1`` stack is the bidirectional one of its commented-out block (``GCN.py:82-90``), built here
with the reference's own ``Adj_Preprocessor.random_walk_normalize`` and ``compute_chebyshev_polynomials``:
``[I, T_1(P_f^T) .. T_K(P_f^T), T_1(P_b^T) .. T_K(P_b^T)]``, ``P_f = D^-1 A``, ``P_b = D^-1 A^T``.  The unmodified
reference ``ST_MGCN`` (and its first ``CG_LSTM`` alone) then run on that stack.

The graphs are directed and weighted, each with a sink (no out-edge), a source (no in-edge) and an isolated region, so
both normalisations meet a zero degree (``d_inv = 0``, ``GCN.py:102``).

The model's parameters are drawn by ``stmgcn_oracle.init_params`` from the seed in ``meta`` (the reference's names,
shapes and init distributions) and loaded into the reference model; they are not stored
(``diffusion_oracle.golden_params`` draws them again).  Stored: ``meta`` (``n, m, k, t, b, c, hid, layers, gcn_hid,
seed``), ``adj.<g>``, ``supports.<g>`` (the dense ``2K+1`` stack), ``x, y``, the ``ST_MGCN`` forward ``out``, the MSE
``loss``, every parameter gradient (``grad.*``) and ``grad_x`` (``d loss / d obs_seq``); for ``rnn_list.0`` alone on
graph 0 with the zero initial state: ``cg_out``, ``cg_h_n``, ``cg_c_n`` and, for the scalar
``sum(cg_out * cg_w)`` with ``cg_w = diffusion_oracle.golden_probe(meta)``, the gradients ``cg_grad.*`` (the
``rnn_list.0.`` parameters) and ``cg_grad_x``.
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
import diffusion_oracle as D  # noqa: E402
import make_golden  # noqa: E402


def directed_adjacency(n: int, g: int, density: float) -> torch.Tensor:
    """Weighted directed graph ``g``: region 0 is a sink, region 1 a source, region 2 isolated."""
    gen = torch.Generator().manual_seed(500 + g)
    a = (torch.rand(n, n, generator=gen) < density).float() * (0.25 + torch.rand(n, n, generator=gen))
    idx = torch.arange(n)
    a[idx, (idx + 1) % n] = 1.0 + g                      # a one-way ring keeps most regions reachable
    a.fill_diagonal_(0.0)
    a[0, :] = 0.0                                         # sink: zero out-degree
    a[:, 1] = 0.0                                         # source: zero in-degree
    a[2, :] = 0.0
    a[:, 2] = 0.0                                         # isolated
    return a


def bidirectional_supports(ref_gcn, adj: torch.Tensor, k: int) -> torch.Tensor:
    pre = ref_gcn.Adj_Preprocessor("random_walk_diffusion", k)
    p_f = pre.random_walk_normalize(adj)
    p_b = pre.random_walk_normalize(adj.T)
    forward_series = pre.compute_chebyshev_polynomials(p_f.T, [])
    backward_series = pre.compute_chebyshev_polynomials(p_b.T, [])
    return torch.stack(forward_series + backward_series[1:], dim=0)


def build(name, n, m, k, t, b, c, hid, layers, gcn_hid, density, seed):
    ref_gcn, ref_stmgcn = make_golden.import_reference()
    adjs = [directed_adjacency(n, g, density) for g in range(m)]
    sups = [bidirectional_supports(ref_gcn, a, k) for a in adjs]
    assert all(torch.isfinite(s).all() for s in sups)
    cfg = {"kernel_type": "random_walk_diffusion", "K": k}
    meta = dict(n=n, m=m, k=k, t=t, b=b, c=c, hid=hid, layers=layers, gcn_hid=gcn_hid, seed=seed)
    torch.manual_seed(seed)
    model = ref_stmgcn.ST_MGCN(M=m, seq_len=t, n_nodes=n, input_dim=c, lstm_hidden_dim=hid, lstm_num_layers=layers,
                               gcn_hidden_dim=gcn_hid, sta_kernel_config=cfg, gconv_use_bias=True,
                               gconv_activation=nn.ReLU)
    assert model.sta_K == 2 * k + 1 == sups[0].shape[0]
    params = D.golden_params(meta)
    assert set(params) == set(model.state_dict())
    model.load_state_dict(params)
    x = torch.randn(b, t, n, c).requires_grad_(True)
    y = torch.randn(b, n, c)
    cg_w = D.golden_probe(meta)
    out = model(obs_seq=x, sta_adj_list=sups)
    loss = nn.MSELoss(reduction="mean")(out, y)
    loss.backward()
    blob = {"meta": np.array([n, m, k, t, b, c, hid, layers, gcn_hid, seed], dtype=np.int64),
            "x": x.detach().numpy(), "y": y.numpy(), "out": out.detach().numpy(),
            "loss": np.array(loss.item(), dtype=np.float64), "grad_x": x.grad.numpy().copy()}
    for g, (a, s) in enumerate(zip(adjs, sups)):
        blob[f"adj.{g}"] = a.numpy()
        blob[f"supports.{g}"] = s.numpy()
    for key, val in model.named_parameters():
        blob["grad." + key] = val.grad.numpy().copy()
    # the first CG_LSTM alone (STMGCN.py:24-51) on graph 0
    model.zero_grad()
    x.grad = None
    cg = model.rnn_list[0]
    cg_out, (h_n, c_n) = cg(sups[0], x, cg.init_hidden(b))
    cg_loss = (cg_out * cg_w).sum()
    cg_loss.backward()
    blob.update(cg_out=cg_out.detach().numpy(), cg_h_n=h_n.detach().numpy(), cg_c_n=c_n.detach().numpy(),
                cg_grad_x=x.grad.numpy().copy())
    for key, val in cg.named_parameters():
        blob["cg_grad." + key] = val.grad.numpy().copy()
    path = os.path.join(REPO, "tests", "golden", name + ".npz")
    np.savez_compressed(path, **blob)
    print(f"{name}: out|max|={float(out.abs().max()):.4g} loss={loss.item():.6f} -> {path} "
          f"({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    ref = os.path.abspath(sys.argv[1]) if len(sys.argv) > 1 else os.environ.get("STMGCN_REFERENCE_DIR", "")
    if not os.path.exists(os.path.join(ref, "STMGCN.py")):
        sys.exit("usage: python oracle/make_diffusion_golden.py /path/to/reference  (the directory with GCN.py and "
                 "STMGCN.py)")
    make_golden.REF = ref
    torch.set_num_threads(1)
    # the reference's K=2, H=G=64, C=1 (Main.py:62-63) -- the tensor-core shapes of the LSTM and the projection, 5 supports
    # (two projection groups) -- with one graph and one LSTM layer (the stored weight gradients dominate the fixture's
    # size; three graphs of three layers are pinned at cfg3 size against the fp64 oracle), 40 regions, batch 4 (160 LSTM
    # rows: a ragged second tile of 128 on the GPU), seq_len 6
    build("diffusion_ref", 40, 1, 2, 6, 4, 1, 64, 1, 64, 0.12, seed=4)
