"""The kernels' module-level limits (``ops.LIMITS``): checked by ``ST_MGCN`` / ``CG_LSTM`` / ``GCN.forward`` before the
first launch, the same numbers in both directions of every kernel, and the same numbers as the C entry points.

At each limit the model passes the fp64 check (``T`` at the gate's limit and ``C*G + C`` at the fusion's here; ``M = 8``,
``L = 8``, 8 supports, ``C = 4`` and ``H = 128`` are rows of ``test_gpu_config_sweep.py``); one past each limit it raises
a ``ValueError`` naming the limit without launching anything; and a direct C-ABI call one past each limit is refused.
"""
import pytest
import torch
from torch import nn

from helpers import DEV, TOL



def test_check_limits_names_each_limit_and_accepts_each_bound():
    from stmgcn_b200 import ops
    lim = ops.LIMITS
    ops.check_limits(m=lim["M"], ks=lim["supports"], c_in=lim["C"], n_layers=lim["L"], hid=lim["H"], t_len=lim["T"])
    ops.check_limits(c_in=4, gcn_hid=(lim["C*G+C"] - 4) // 4)
    ops.check_limits(c_in=1, gcn_hid=lim["q"])
    beyond = [(dict(m=lim["M"] + 1), "M=9 graphs"), (dict(ks=lim["supports"] + 1), "9 supports per GCN"),
              (dict(c_in=lim["C"] + 1), "input_dim C=5"), (dict(n_layers=lim["L"] + 1), "lstm_num_layers L=9"),
              (dict(hid=lim["H"] + 4), "lstm_hidden_dim H=132"), (dict(hid=66), "lstm_hidden_dim H=66"),
              (dict(t_len=lim["T"] + 1), "seq_len T=2049"), (dict(gcn_hid=lim["q"] + 1), "GCN hidden_dim 8193"),
              (dict(c_in=4, gcn_hid=3072), "C*G + C = 12292")]
    for kw, name in beyond:
        with pytest.raises(ValueError, match=name.replace("*", r"\*").replace("+", r"\+")):
            ops.check_limits(**kw)


def _model(m=1, t=4, c=1, h=8, g=8, lyr=1, k=1, act=nn.ReLU):
    import STMGCN
    torch.manual_seed(0)
    return STMGCN.ST_MGCN(M=m, seq_len=t, n_nodes=6, input_dim=c, lstm_hidden_dim=h, lstm_num_layers=lyr,
                          gcn_hidden_dim=g, sta_kernel_config={"kernel_type": "chebyshev", "K": k},
                          gconv_use_bias=True, gconv_activation=act).to(DEV)


def _sups(m, k, n=6):
    import GCN
    from stmgcn_b200 import synth
    return [GCN.Adj_Preprocessor("chebyshev", k).process(synth.make_adjacency(n, g, 0.4)).to(DEV) for g in range(m)]


BEYOND = [
    ("M=9", dict(m=9), "M=9 graphs"),
    ("K=8", dict(k=8), "9 supports per GCN"),
    ("C=5", dict(c=5), "input_dim C=5"),
    ("L=9", dict(lyr=9), "lstm_num_layers L=9"),
    ("H=132", dict(h=132), "lstm_hidden_dim H=132"),
    ("H=66", dict(h=66), "lstm_hidden_dim H=66"),
    ("T=2049", dict(t=2049), "seq_len T=2049"),
    ("G=8193", dict(g=8193), "GCN hidden_dim 8193"),
    ("C*G", dict(c=4, g=3072), r"C\*G \+ C = 12292"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("what,kw,name", BEYOND, ids=[b[0] for b in BEYOND])
def test_model_one_past_each_limit_raises_before_any_launch(what, kw, name):
    """ST_MGCN one past each limit: a ValueError naming it from the forward, and no kernel launched (before, M = 9 ran
    all nine branches and then failed in the fusion, and T = 2049 passed its forward and failed in the backward)."""
    from stmgcn_b200 import _lib
    model = _model(**kw)
    m, t, c = kw.get("m", 1), kw.get("t", 4), kw.get("c", 1)
    sups = _sups(m, kw.get("k", 1))
    x = torch.randn(2, t, 6, c, device=DEV)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    with pytest.raises(ValueError, match=name):
        out = model(obs_seq=x, sta_adj_list=sups)
        out.sum().backward()
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0, f"{what}: {_lib.launch_count() - n0} launches before the error"


@pytest.mark.gpu
def test_cg_lstm_and_gcn_check_their_limits_before_any_launch():
    import GCN
    import STMGCN
    from stmgcn_b200 import _lib
    sup = _sups(1, 8)[0]
    n0 = _lib.launch_count()
    cg = STMGCN.CG_LSTM(seq_len=4, n_nodes=6, input_dim=1, lstm_hidden_dim=8, lstm_num_layers=1, K=9,
                        gconv_use_bias=True).to(DEV)
    with pytest.raises(ValueError, match="9 supports per GCN"):
        cg(sup, torch.randn(2, 4, 6, 1, device=DEV), None)
    cg = STMGCN.CG_LSTM(seq_len=2049, n_nodes=6, input_dim=1, lstm_hidden_dim=8, lstm_num_layers=1, K=2,
                        gconv_use_bias=True).to(DEV)
    with pytest.raises(ValueError, match="seq_len T=2049"):
        cg(_sups(1, 1)[0], torch.randn(2, 2049, 6, 1, device=DEV), None)
    layer = GCN.GCN(K=9, input_dim=4, hidden_dim=8).to(DEV)
    with pytest.raises(ValueError, match="9 supports per GCN"):
        layer(sup, torch.randn(2, 6, 4, device=DEV))
    layer = GCN.GCN(K=2, input_dim=4, hidden_dim=8193).to(DEV)
    with pytest.raises(ValueError, match="GCN hidden_dim 8193"):
        layer(_sups(1, 1)[0], torch.randn(2, 6, 4, device=DEV))
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0


def _fp64_step(model, sups, x, y, relu):
    """One step of ``model`` against ``O.dense_loss_and_grads`` in fp64 on the GPU (the kernels' ReLU masks); returns the
    worst error."""
    import stmgcn_oracle as O
    from full_batch import _errors, gpu_step
    got = gpu_step(model, sups, x, y, False, keep_masks=relu)
    params = {k: v.detach().double() for k, v in model.state_dict().items()}
    out, loss, grads = O.dense_loss_and_grads(params, x.double().to(DEV), y.double().to(DEV),
                                              [s.double() for s in sups], relu=relu,
                                              masks=got["masks"] if relu else None)
    errs = _errors(got, dict(out=out, loss=float(loss), grads=grads), False)
    return errs


@pytest.mark.gpu
def test_model_at_the_gate_limit_matches_fp64(monkeypatch):
    """seq_len T = 2048 (the context gate's limit, both directions), a few LSTM rows on the exact-fp32 path: one step
    against fp64."""
    from stmgcn_b200 import ops
    t = ops.LIMITS["T"]
    monkeypatch.setattr(ops, "_LSTM_PATH", "fma")
    model = _model(t=t, h=8, g=8, act=None)
    gen = torch.Generator().manual_seed(3)
    x, y = torch.randn(2, t, 6, 1, generator=gen), torch.randn(2, 6, 1, generator=gen)
    errs = _fp64_step(model, _sups(1, 1), x, y, False)
    print(f"T={t}: worst {max(errs.values()):.2e} ({max(errs, key=errs.get)})")
    assert max(errs.values()) <= TOL, errs


@pytest.mark.gpu
def test_model_at_the_fusion_limit_matches_fp64():
    """C = 4 and G = 3071: C*G + C = 12 288 floats, the fusion backward's whole shared-memory accumulator."""
    from stmgcn_b200 import ops
    c, g = 4, (ops.LIMITS["C*G+C"] - 4) // 4
    model = _model(m=2, c=c, g=g, h=16, k=2)
    gen = torch.Generator().manual_seed(4)
    x, y = torch.randn(3, 4, 6, c, generator=gen), torch.randn(3, 6, c, generator=gen)
    errs = _fp64_step(model, _sups(2, 2), x, y, True)
    print(f"C={c} G={g}: worst {max(errs.values()):.2e} ({max(errs, key=errs.get)})")
    assert max(errs.values()) <= TOL, errs


def _abi_calls():
    """One direct C-ABI call one past each limit of ``ops.LIMITS`` (valid buffers otherwise)."""
    from stmgcn_b200 import ops
    lim = ops.LIMITS
    t1, q1, m1, l1, c1, h1, k1 = lim["T"] + 1, lim["q"] + 1, lim["M"] + 1, lim["L"] + 1, lim["C"] + 1, lim["H"] + 4, \
        lim["supports"] + 1
    cg = (4, (lim["C*G+C"] - 4) // 4 + 1)           # C = 4, G one past its bound
    return [
        ("M", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_fuse_out_fwd(pa([a] * m1), m1, 4, 2, 8, 2, b, c, d, e, st)),
        ("supports", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_proj_fwd(a, 768, k1, 64, 12, b, c, 12, 1, d, None, 4,
                                                                          None, st)),
        ("supports", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_proj_bwd(a, 768, k1, 64, 12, b, 12, 1, c, d, None, 1.0,
                                                                          4, e, f, None, None, 0, None, st)),
        ("C", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_lstm_fwd(3, 2, 8, 8, c1, 2, a, b, c, d, e, None, None, f, a, b,
                                                                   st)),
        ("C", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_lstm16_fwd(3, 2, 100, c1, 4, 2, a, b, c, d, e, None, None, f, a,
                                                                     b, None, st)),
        ("L", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_lstm_fwd(3, l1, 8, 8, 1, 2, a, b, c, d, e, None, None, f, a, b,
                                                                   st)),
        ("L", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_lstm16_fwd(3, l1, 100, 1, 4, 2, a, b, c, d, e, None, None, f, a,
                                                                     b, None, st)),
        ("H", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_lstm_fwd(3, 2, 8, h1, 1, 2, a, b, c, d, e, None, None, f, a, b,
                                                                   st)),
        ("T", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_gate_fwd(a, 2, t1, 10, b, c, d, e, f, st)),
        ("T", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_gate_bwd(a, b, c, d, 2, t1, e, f, a, b, st)),
        ("q", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_proj_fwd(a, 768, 1, 64, 12, b, c, q1, 1, d, None, 4, None,
                                                                   st)),
        ("q", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_proj_bwd(a, 768, 1, 64, 12, b, q1, 1, c, d, None, 1.0, 4, e, f,
                                                                   None, None, 0, None, st)),
        ("C*G+C", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_fuse_out_fwd(pa([a]), 1, 4, 2, cg[1], cg[0], b, c, d, e,
                                                                           st)),
        ("C*G+C", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_fuse_out_bwd(a, b, 4, 2, cg[1], cg[0], c, d, e, f, st)),
    ]


@pytest.mark.gpu
def test_c_abi_refuses_one_past_each_limit_of_the_python_table():
    """The Python table cannot drift above the C side: every entry point one past a limit of ``ops.LIMITS`` returns an
    error with a message and launches nothing (every limit has such a call, in each direction that has one)."""
    from stmgcn_b200 import _lib, ops
    calls = _abi_calls()
    assert {k for k, _ in calls} == set(ops.LIMITS)
    bufs = [torch.randn(1 << 16, device=DEV) for _ in range(6)]
    st = torch.cuda.current_stream().cuda_stream
    for key, call in calls:
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        rc = call(_lib.lib, _lib.ptr_array, st, *(b.data_ptr() for b in bufs))
        torch.cuda.synchronize()
        assert rc < 0 and _lib.lib.stmgcn_last_error(), f"{key}: rc={rc}"
        assert _lib.launch_count() == n0, key
        print(f"{key}: {_lib.lib.stmgcn_last_error().decode()}")
