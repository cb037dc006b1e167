"""The model across its configuration surface, against fp64: every constructor argument and dispatch boundary of
``ST_MGCN`` in pairwise combination.

Each user-visible call is dispatched by independent predicates (``ops`` / ``modules``):

* shared LSTM: the tensor-core kernels iff ``H == 64``, ``C <= 4``, ``T <= 64`` and the path is ``tc``; else exact fp32;
* spatial projection: the tensor-core kernels iff the path is ``tc``, ``H == G == 64`` and ``Ks <= 8``; else FFMA (a
  torch-applied activation sends the temporal GCN through the same choice with ``p = q = T``);
* supports: a ``cheb`` set with one recurrence chain (Chebyshev) or two (diffusion handle), or ``generic`` (localpool,
  a dense diffusion stack);
* activation: ReLU or none in the kernels, or a torch module applied outside them (``modules._act_code`` is None);
* graph branches: one CUDA stream per branch iff ``M > 1`` and ``STMGCN_GRAPH_STREAMS`` is not ``0``.

``CASES`` is a pairwise covering table over the factors of ``FACTORS``: every pair of levels of any two factors is in at
least one row (``test_case_table_covers_every_pair_of_levels``, a CPU test), and each row states which kernel families
and streams it exercises.  Each GPU case runs one training step with seeded parameters and inputs, records the ReLU
masks the kernels took, and compares every window's output (each held to its own maximum), the loss, every parameter
gradient and, where asked, d obs with the dense restatement (``O.dense_loss_and_grads``) in fp64 on the GPU, at the
project bar of 1e-4.  A dispatch witness wraps ``ops._lstm16_forward`` / ``ops._exact_forward`` / ``ops._proj_images``
and fails a case that did not run what its row claims.
"""
import itertools
import os
import subprocess
import sys
import textwrap
import time

import pytest
import torch
from torch import nn

import stmgcn_oracle as O
from helpers import DEV, TOL, sm_count


FACTORS = {
    "M": ["1", "2", "3", "8"],
    "supports": ["cheb0", "cheb1", "cheb3", "cheb7", "localpool", "rwd1", "rwd3"],   # chebyshev K / diffusion K
    "form": ["dense", "handle"],             # a dense (Ks, N, N) stack, or Adj_Preprocessor.process_sparse's handle
    "T": ["1", "12", "64", "65"],
    "C": ["1", "2", "4"],
    "H": ["64", "32", "68", "128"],
    "G": ["64", "20"],
    "L": ["1", "3", "8"],
    "bias": ["yes", "no"],                   # gconv_use_bias
    "act": ["relu", "none", "tanh"],         # nn.ReLU, None, nn.Tanh
    "rows": ["sub", "x128", "ragged", "wave"],   # LSTM rows N*B: see region_batch
    "path": ["tc", "fma"],                   # ops.set_lstm_path
    "streams": ["on", "off"],                # STMGCN_GRAPH_STREAMS
    "caller": ["default", "side"],           # the step runs on the default stream, or on a side stream
    "d_obs": ["no", "yes"],                  # obs_seq.requires_grad
}
CLAIMS = ("lstm", "proj", "branches")        # what ran: tc / exact, tc / fma, multi / one

# One row per case; the last three columns are the row's claims, checked against the predicates on the CPU and against
# what ran on the GPU.
CASES_TABLE = """
id   M  supports   form    T   C  H    G   L  bias act   rows    path streams caller  d_obs lstm  proj branches
c01  1  cheb0      dense   65  1  32   64  1  no   relu  wave    fma  on      default yes   exact fma  one
c02  1  cheb1      dense   64  4  32   64  1  yes  relu  sub     tc   off     side    no    exact fma  one
c03  1  cheb1      handle  65  4  128  20  8  no   tanh  ragged  tc   on      side    no    exact fma  one
c04  1  cheb3      handle  1   2  32   20  1  yes  none  wave    fma  on      default yes   exact fma  one
c05  1  cheb7      handle  64  4  68   64  3  no   none  ragged  tc   on      side    no    exact fma  one
c06  1  localpool  handle  64  1  64   64  1  no   relu  x128    tc   on      default yes   tc    tc   one
c07  1  rwd1       handle  64  2  32   20  3  no   none  sub     fma  on      default yes   exact fma  one
c08  1  rwd3       dense   12  2  64   20  8  yes  none  ragged  tc   on      default no    tc    fma  one
c09  1  rwd3       dense   64  1  32   20  1  no   tanh  wave    tc   off     default no    exact fma  one
c10  2  cheb0      dense   1   1  64   20  3  no   tanh  sub     fma  on      default no    exact fma  multi
c11  2  cheb1      dense   12  2  68   64  3  yes  none  x128    fma  on      default no    exact fma  multi
c12  2  cheb3      handle  64  1  128  64  8  yes  relu  sub     fma  off     default no    exact fma  one
c13  2  cheb7      dense   1   4  64   20  8  yes  tanh  x128    tc   on      side    yes   tc    fma  multi
c14  2  cheb7      handle  12  2  32   20  1  no   relu  wave    fma  off     default yes   exact fma  one
c15  2  localpool  handle  12  4  68   20  3  no   none  sub     tc   on      default yes   exact fma  multi
c16  2  rwd1       dense   12  1  64   64  1  yes  tanh  ragged  tc   on      default no    tc    tc   multi
c17  2  rwd3       handle  65  4  128  64  8  no   tanh  x128    fma  off     default no    exact fma  one
c18  3  cheb0      handle  12  1  68   64  1  yes  relu  ragged  fma  off     default no    exact fma  one
c19  3  cheb1      handle  1   1  64   64  1  yes  none  wave    tc   on      default yes   tc    tc   multi
c20  3  cheb3      dense   65  1  68   20  3  no   relu  ragged  tc   on      side    yes   exact fma  multi
c21  3  cheb7      handle  65  1  64   64  3  no   none  sub     tc   off     default no    exact tc   one
c22  3  localpool  dense   1   1  128  64  8  yes  relu  ragged  fma  on      side    no    exact fma  multi
c23  3  localpool  handle  65  2  32   20  1  yes  tanh  x128    fma  on      side    yes   exact fma  multi
c24  3  rwd1       dense   1   4  68   64  8  yes  relu  wave    tc   off     side    no    exact fma  one
c25  3  rwd3       dense   64  1  68   64  1  yes  relu  sub     fma  on      default no    exact fma  multi
c26  8  cheb0      dense   12  4  128  20  3  no   none  x128    fma  off     side    yes   exact fma  one
c27  8  cheb0      dense   64  2  68   64  8  no   tanh  sub     tc   on      side    yes   exact fma  multi
c28  8  cheb1      handle  1   1  64   64  3  yes  tanh  wave    fma  on      default yes   exact fma  multi
c29  8  cheb3      handle  12  4  64   64  8  no   tanh  x128    tc   off     side    no    tc    tc   one
c30  8  cheb7      handle  64  4  128  64  1  no   tanh  ragged  fma  off     side    no    exact fma  one
c31  8  localpool  dense   1   2  128  64  1  no   none  wave    tc   off     side    no    exact fma  one
c32  8  rwd1       dense   12  2  128  64  3  no   tanh  x128    tc   on      default no    exact fma  multi
c33  8  rwd1       dense   65  4  32   64  8  yes  relu  x128    fma  on      default no    exact fma  multi
c34  8  rwd3       dense   1   1  32   64  3  yes  relu  ragged  tc   on      side    yes   exact fma  multi
c35  2  cheb3      dense   12  1  64   64  1  yes  relu  wave    tc   on      default no    tc    tc   multi
c36  3  cheb3      handle  12  1  64   64  3  no   relu  ragged  tc   on      side    yes   tc    tc   multi
c37  2  rwd3       handle  64  2  64   64  3  no   tanh  x128    tc   on      default no    tc    tc   multi
c38  3  localpool  dense   12  1  64   64  3  no   tanh  ragged  tc   on      default yes   tc    tc   multi
c39  1  cheb7      dense   12  1  64   64  1  no   none  sub     tc   off     default no    tc    tc   one
c40  8  cheb1      dense   12  1  64   64  1  yes  relu  ragged  tc   on      default no    tc    tc   multi
"""

# Pairs no row can hold, with the reason.  (None so far: every pair of levels is a configuration the modules accept.)
IMPOSSIBLE = {}


def _parse(table):
    lines = [ln.split() for ln in table.strip().splitlines()]
    head = lines[0]
    return [dict(zip(head, ln)) for ln in lines[1:]]


CASES = _parse(CASES_TABLE)

N_SUPPORTS = {"cheb0": 1, "cheb1": 2, "cheb3": 4, "cheb7": 8, "localpool": 1, "rwd1": 3, "rwd3": 7}


def predicted(case):
    """What the dispatch predicates of ``ops`` / ``modules`` run for a row (the claims it must state)."""
    h, g, t, c, m = (int(case[k]) for k in ("H", "G", "T", "C", "M"))
    tc = case["path"] == "tc"
    return {"lstm": "tc" if (tc and h == 64 and c <= 4 and t <= 64) else "exact",
            "proj": "tc" if (tc and h == 64 and g == 64 and N_SUPPORTS[case["supports"]] <= 8) else "fma",
            "branches": "multi" if (m > 1 and case["streams"] == "on") else "one"}


def support_kind(case):
    """``cheb`` with its number of recurrence chains, or ``generic``: how the kernels see the row's supports."""
    sup, form = case["supports"], case["form"]
    if sup == "localpool" or (sup.startswith("rwd") and form == "dense"):
        return "generic"
    if sup.startswith("rwd"):
        return "cheb, 2 chains"
    return "cheb, 0 chains" if sup == "cheb0" else "cheb, 1 chain"


# ----------------------------------------------------------------------------------------------------------------------
# the table (CPU)
# ----------------------------------------------------------------------------------------------------------------------
def test_case_table_covers_every_pair_of_levels():
    """Every pair of levels of any two factors is in some row (or declared impossible, with a reason); every row uses
    only known levels and has a unique id."""
    assert len({c["id"] for c in CASES}) == len(CASES)
    for case in CASES:
        for f, levels in FACTORS.items():
            assert case[f] in levels, f"{case['id']}: {f}={case[f]} is not a level"
    missing = []
    for (fa, la), (fb, lb) in itertools.combinations(FACTORS.items(), 2):
        for va, vb in itertools.product(la, lb):
            if any(c[fa] == va and c[fb] == vb for c in CASES):
                continue
            if ((fa, va), (fb, vb)) in IMPOSSIBLE:
                continue
            missing.append(f"{fa}={va} with {fb}={vb}")
    assert not missing, f"{len(missing)} pairs of levels in no case: {missing[:20]}"
    for pair, reason in IMPOSSIBLE.items():
        assert reason and not any(all(c[f] == v for f, v in pair) for c in CASES), pair
    print(f"{len(CASES)} cases cover all {sum(len(a) * len(b) for a, b in itertools.combinations(FACTORS.values(), 2))} "
          f"pairs of levels of {len(FACTORS)} factors")


def test_case_table_claims_and_both_sides_of_every_dispatch():
    """Each row's claims are what the predicates give, and every predicate has cases on both sides (with the boundary
    values among them: H = 64 vs 68, T = 64 vs 65, G = 64 vs 20)."""
    for case in CASES:
        want = predicted(case)
        got = {k: case[k] for k in CLAIMS}
        assert got == want, f"{case['id']} claims {got}, the predicates give {want}"
    sides = {
        "LSTM family": {c["lstm"] for c in CASES},
        "projection family": {c["proj"] for c in CASES},
        "supports": {support_kind(c) for c in CASES},
        "activation": {c["act"] for c in CASES},
        "branch streams": {c["branches"] for c in CASES},
    }
    assert sides["LSTM family"] == {"tc", "exact"}
    assert sides["projection family"] == {"tc", "fma"}
    assert sides["supports"] == {"cheb, 0 chains", "cheb, 1 chain", "cheb, 2 chains", "generic"}
    assert sides["activation"] == {"relu", "none", "tanh"}
    assert sides["branch streams"] == {"multi", "one"}

    def has(**kv):
        return any(all(c[k] == v for k, v in kv.items()) for c in CASES)
    # the boundaries themselves, on the tensor-core path
    assert has(path="tc", H="64", T="64", lstm="tc") and has(path="tc", H="64", T="65", lstm="exact")
    assert has(path="tc", H="68", lstm="exact") and has(path="tc", H="64", G="20", lstm="tc", proj="fma")
    assert has(path="tc", T="65", H="64", G="64", lstm="exact", proj="tc")
    assert has(path="tc", C="4", lstm="tc") and has(M="8", branches="multi") and has(M="8", branches="one")
    # a torch-applied activation with T = 64 on the tensor-core path: the temporal GCN's projection on the tensor cores
    assert has(path="tc", act="tanh", T="64", H="64", G="64")


# ----------------------------------------------------------------------------------------------------------------------
# one case on the GPU
# ----------------------------------------------------------------------------------------------------------------------
def region_batch(rows_kind, sms):
    """(N, B) of a row's LSTM rows N*B: under one 128-row tile, an exact multiple of 128, a ragged multi-tile count, or
    more than one wave of tiles on this device (one 128-row tile per SM), ending in a partial tile."""
    if rows_kind == "sub":
        return 20, 3                         # 60 rows
    if rows_kind == "x128":
        return 64, 4                         # 256 rows
    if rows_kind == "ragged":
        return 70, 5                         # 350 rows: 2 tiles and 94 rows
    n = 200
    b = (128 * sms) // n + 1
    while (n * b) % 128 == 0:
        b += 1
    return n, b


def make_supports(case, n, m):
    """(supports the model takes, their dense fp64 stacks on the device) for each of the ``m`` graphs."""
    import GCN
    import diffusion_oracle as D
    from stmgcn_b200 import synth
    sup, form = case["supports"], case["form"]
    kind, k = ("localpool", 1) if sup == "localpool" else (
        ("random_walk_diffusion" if sup.startswith("rwd") else "chebyshev"), int(sup[-1]))
    dens = 4.0 / n + 0.02
    model_sups, ref_sups = [], []
    for g in range(m):
        if kind == "random_walk_diffusion":
            adj = synth.make_directed_adjacency(n, g, dens)
            adj = adj * (0.5 + torch.rand(n, n, generator=torch.Generator().manual_seed(50 + g)))
        else:
            adj = synth.make_adjacency(n, g, dens)
        pre = GCN.Adj_Preprocessor(kind, k)
        if form == "handle":
            h = pre.process_sparse(adj).to(DEV)
            mats = [v.double().cpu() for v in h.matrices_dense()]
            ref = mats[0][None] if kind == "localpool" else O.chain_stack_dense(mats if h.ks > 1 else [mats[0]], k)
            model_sups.append(h)
        elif kind == "random_walk_diffusion":     # the 2K+1 bidirectional stack, dense (the generic path)
            ref = D.diffusion_supports_dense(adj.double(), k)
            model_sups.append(ref.float().to(DEV))
        else:
            dense = pre.process(adj)
            model_sups.append(dense.to(DEV))
            ref = dense.double() if kind == "localpool" else O.chain_stack_dense([dense[1].double()], k) if k else dense.double()
        ref_sups.append(ref.to(DEV))
    return model_sups, ref_sups


ACTIVATIONS = {"relu": (nn.ReLU, True), "none": (None, False), "tanh": (nn.Tanh, nn.Tanh())}


def build_case(case, sms, seed):
    """The seeded model, supports, inputs and targets of a row.  The GCN biases are drawn at random (their init is
    zero), so a bias that goes astray shows."""
    import STMGCN
    m, t, c, h, g, lyr = (int(case[k]) for k in ("M", "T", "C", "H", "G", "L"))
    n, b = region_batch(case["rows"], sms)
    sup = case["supports"]
    cfg = {"kernel_type": "localpool", "K": 1} if sup == "localpool" else {
        "kernel_type": "random_walk_diffusion" if sup.startswith("rwd") else "chebyshev", "K": int(sup[-1])}
    torch.manual_seed(seed)
    model = STMGCN.ST_MGCN(M=m, seq_len=t, n_nodes=n, input_dim=c, lstm_hidden_dim=h, lstm_num_layers=lyr,
                           gcn_hidden_dim=g, sta_kernel_config=cfg, gconv_use_bias=case["bias"] == "yes",
                           gconv_activation=ACTIVATIONS[case["act"]][0])
    with torch.no_grad():
        for name, p in model.named_parameters():
            if name.endswith(".b"):
                p.uniform_(-0.2, 0.2)
    model = model.to(DEV)
    sups, ref_sups = make_supports(case, n, m)
    gen = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(b, t, n, c, generator=gen)
    y = torch.randn(b, n, c, generator=gen)
    return model, sups, ref_sups, x, y


class Witness:
    """Records which LSTM family and projection family ran, and on which streams (``torch.cuda.current_stream()``
    inside the wrapped calls)."""

    def __init__(self, monkeypatch):
        from stmgcn_b200 import ops
        self.lstm, self.proj, self.streams = [], [], set()
        real16, real_exact, real_img = ops._lstm16_forward, ops._exact_forward, ops._proj_images

        def lstm16(*a, **k):
            self.lstm.append("tc")
            self.streams.add(torch.cuda.current_stream().cuda_stream)
            return real16(*a, **k)

        def exact(*a, **k):
            self.lstm.append("exact")
            self.streams.add(torch.cuda.current_stream().cuda_stream)
            return real_exact(*a, **k)

        def images(w, ks, p, need_bwd):
            img = real_img(w, ks, p, need_bwd)
            self.proj.append((p, int(w.shape[1]), "tc" if img[0] is not None else "fma"))
            self.streams.add(torch.cuda.current_stream().cuda_stream)
            return img
        monkeypatch.setattr(ops, "_lstm16_forward", lstm16)
        monkeypatch.setattr(ops, "_exact_forward", exact)
        monkeypatch.setattr(ops, "_proj_images", images)


def run_step(case, model, sups, x, y, monkeypatch, want_obs):
    """One training step of the row (path, branch streams and caller stream as the row says) under the witness.
    Returns (``full_batch.gpu_step``'s result, witness, the caller's stream)."""
    from full_batch import gpu_step
    from stmgcn_b200 import ops
    monkeypatch.setenv("STMGCN_GRAPH_STREAMS", "1" if case["streams"] == "on" else "0")
    wit = Witness(monkeypatch)
    old = ops.lstm_path()
    ops.set_lstm_path(case["path"])
    try:
        if case["caller"] == "side":
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                got = gpu_step(model, sups, x, y, want_obs, keep_masks=case["act"] == "relu")
            torch.cuda.current_stream().wait_stream(side)
            caller = side.cuda_stream
        else:
            got = gpu_step(model, sups, x, y, want_obs, keep_masks=case["act"] == "relu")
            caller = torch.cuda.current_stream().cuda_stream
    finally:
        ops.set_lstm_path(old)
    return got, wit, caller


def reference(model, ref_sups, x, y, act, masks, want_obs, drop=None):
    """``O.dense_loss_and_grads`` in fp64 on the GPU at the model's parameters (``drop``: a GCN bias whose ``+ b`` the
    reference leaves out, i.e. takes as zero)."""
    params = {k: (torch.zeros_like(v) if k == drop else v).detach().double() for k, v in model.state_dict().items()}
    out, loss, grads = O.dense_loss_and_grads(params, x.double().to(DEV), y.double().to(DEV), ref_sups, relu=act,
                                              masks=masks, want_obs=want_obs)
    return dict(out=out, loss=float(loss), grads=grads)


def errors(got, ref, want_obs):
    from full_batch import _errors
    return _errors(got, ref, want_obs)


def check_witness(case, wit, caller):
    m = int(case["M"])
    assert wit.lstm == [case["lstm"]] * m, f"{case['id']}: LSTM families {wit.lstm}, the row claims {case['lstm']}"
    h, g = int(case["H"]), int(case["G"])
    spatial = [fam for p, q, fam in wit.proj if (p, q) == (h, g)]
    assert spatial and set(spatial) == {case["proj"]}, f"{case['id']}: projections {wit.proj}, claims {case['proj']}"
    for p, q, fam in wit.proj:               # every projection (the torch-activated temporal GCN's too) as predicted
        want = "tc" if (case["path"] == "tc" and p == 64 and q == 64) else "fma"
        assert fam == want, f"{case['id']}: projection p={p} q={q} ran {fam}, the predicate gives {want}"
    if case["branches"] == "multi":
        assert len(wit.streams) == m and caller not in wit.streams, f"{case['id']}: streams {wit.streams}"
    else:
        assert wit.streams == {caller}, f"{case['id']}: streams {wit.streams}, caller {caller}"


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_config_sweep_case_matches_fp64(case, monkeypatch):
    """One training step of the row against the fp64 dense restatement at the kernels' own ReLU masks: every window's
    output, the loss, every parameter gradient and (where the row asks) d obs, at 1e-4; and the row ran the kernel
    families and streams it claims."""
    sms = sm_count()
    seed = int(case["id"][1:])
    want_obs = case["d_obs"] == "yes"
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    model, sups, ref_sups, x, y = build_case(case, sms, seed)
    got, wit, caller = run_step(case, model, sups, x, y, monkeypatch, want_obs)
    t1 = time.perf_counter()
    relu = case["act"] == "relu"
    ref = reference(model, ref_sups, x, y, ACTIVATIONS[case["act"]][1], got["masks"] if relu else None, want_obs)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    errs = errors(got, ref, want_obs)
    worst = max(errs, key=errs.get)
    n, b = x.shape[2], x.shape[0]
    print(f"{case['id']} ({' '.join(f'{k}={case[k]}' for k in FACTORS)}; N={n} B={b}): worst {errs[worst]:.2e} "
          f"({worst}); GPU step {t1 - t0:.2f} s, fp64 reference {t2 - t1:.2f} s, peak "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    check_witness(case, wit, caller)
    bad = {k: v for k, v in errs.items() if not v <= TOL}
    assert not bad, f"{case['id']}: above {TOL:.0e}: {bad}"


# ----------------------------------------------------------------------------------------------------------------------
# negative controls: each must fail the bar
# ----------------------------------------------------------------------------------------------------------------------
def _case(cid):
    return next(c for c in CASES if c["id"] == cid)


@pytest.mark.gpu
def test_negative_control_reference_without_one_gcn_bias(monkeypatch):
    """The reference with one spatial GCN's bias dropped is far outside the bar: the bias reaches the comparison."""
    case = _case("c40")
    model, sups, ref_sups, x, y = build_case(case, 0, 40)
    got, _, _ = run_step(case, model, sups, x, y, monkeypatch, False)
    ok = errors(got, reference(model, ref_sups, x, y, True, got["masks"], False), False)
    assert max(ok.values()) <= TOL
    bad = errors(got, reference(model, ref_sups, x, y, True, got["masks"], False, drop="gcn_list.3.b"), False)
    print(f"without gcn_list.3.b: out {bad['out']:.2e}, loss {bad['loss']:.2e}")
    assert bad["out"] > 10 * TOL


@pytest.mark.gpu
@pytest.mark.parametrize("cid,swapped", [("c16", False), ("c11", nn.Tanh())])
def test_negative_control_reference_with_the_activation_swapped(cid, swapped, monkeypatch):
    """A Tanh model against the reference without activation, and a model without activation against a Tanh reference:
    both fail the bar."""
    case = _case(cid)
    model, sups, ref_sups, x, y = build_case(case, 0, int(cid[1:]))
    got, _, _ = run_step(case, model, sups, x, y, monkeypatch, False)
    errs = errors(got, reference(model, ref_sups, x, y, swapped, None, False), False)
    print(f"{cid} against the reference with activation {swapped}: worst {max(errs.values()):.2e}")
    assert max(errs.values()) > 10 * TOL


@pytest.mark.gpu
def test_negative_control_kernels_with_relu_forced_for_a_tanh_model(monkeypatch):
    """``modules._act_code`` forced to the kernels' ReLU for a Tanh model: the kernels then compute another model, and
    the comparison with the Tanh reference fails the bar."""
    from stmgcn_b200 import _lib, modules
    case = _case("c16")
    model, sups, ref_sups, x, y = build_case(case, 0, 16)
    monkeypatch.setattr(modules, "_act_code", lambda mod: _lib.ACT_RELU)
    got, _, _ = run_step(case, model, sups, x, y, monkeypatch, False)
    errs = errors(got, reference(model, ref_sups, x, y, nn.Tanh(), None, False), False)
    print(f"kernels with ReLU for a Tanh model: worst {max(errs.values()):.2e}")
    assert max(errs.values()) > 10 * TOL


# ----------------------------------------------------------------------------------------------------------------------
# the tensor-core LSTM backward's zero tile, on branch streams
# ----------------------------------------------------------------------------------------------------------------------
ZERO_TILE_SCRIPT = textwrap.dedent(r"""
    import sys
    import torch
    from torch import nn
    sys.path[:0] = [{repo!r}, {pkg!r}, {oracle!r}]
    import GCN, STMGCN
    import stmgcn_oracle as O
    from stmgcn_b200 import ops, synth

    dev = "cuda:0"
    n, b, t, m = 40, 4, 12, 3
    torch.manual_seed(0)
    model = STMGCN.ST_MGCN(M=m, seq_len=t, n_nodes=n, input_dim=1, lstm_hidden_dim=64, lstm_num_layers=2,
                           gcn_hidden_dim=64, sta_kernel_config={{"kernel_type": "chebyshev", "K": 2}},
                           gconv_use_bias=True, gconv_activation=None).to(dev)
    sups = [GCN.Adj_Preprocessor("chebyshev", 2).process(synth.make_adjacency(n, g, 0.1)) for g in range(m)]
    gen = torch.Generator().manual_seed(1)
    x, y = torch.randn(b, t, n, 1, generator=gen), torch.randn(b, n, 1, generator=gen)
    real = ops._zero_tile
    calls = []

    def poisoned_then_slow(device):
        # a freed NaN-filled block of every size the tile can take, in this stream's cache; the first call (the one that
        # makes the tile in a process-wide cache) then waits ~0.1 s on its own stream before the tile's fill is queued
        blocks = [torch.full((128 * 64,), float("nan"), device=device, dtype=torch.bfloat16) for _ in range(64)]
        del blocks
        if not calls:
            torch.cuda._sleep(200_000_000)
        calls.append(torch.cuda.current_stream().cuda_stream)
        return real(device)
    ops._zero_tile = poisoned_then_slow
    out = model(obs_seq=x.to(dev), sta_adj_list=[s.to(dev) for s in sups])
    loss = nn.MSELoss()(out, y.to(dev))
    loss.backward()
    torch.cuda.synchronize()
    assert len(set(calls)) == m, calls
    params = {{k: v.detach().double() for k, v in model.state_dict().items()}}
    _, _, ref = O.dense_loss_and_grads(params, x.double().to(dev), y.double().to(dev),
                                       [s.double().to(dev) for s in sups], relu=False)
    worst = 0.0
    for k, p in model.named_parameters():
        g = p.grad.double()
        if not bool(torch.isfinite(g).all()):
            print(f"NONFINITE {{k}}")
            sys.exit(3)
        worst = max(worst, float((g - ref[k]).abs().max() / ref[k].abs().max()))
    print(f"WORST {{worst:.3e}}")
    sys.exit(0 if worst <= {tol} else 4)
""")


@pytest.mark.gpu
def test_first_backward_on_branch_streams_reads_a_filled_zero_tile():
    """The first tensor-core LSTM backward of a process, on three branch streams.  Each stream's cache holds freed
    NaN-filled blocks and the stream that first asks for the zero tile (the h_prev operand at t = 0) is held back before
    the tile's fill: a tile shared across streams without ordering is then read as NaN by the other branches.  The
    gradients must be finite and at the bar.  Runs once, in a fresh process (the first backward of a process is the one
    that makes a process-wide tile), which exits before the test returns."""
    here = os.path.dirname(os.path.abspath(__file__))
    repo = os.path.dirname(here)
    script = ZERO_TILE_SCRIPT.format(repo=repo, pkg=os.path.join(repo, "st-mgcn_b200"), oracle=os.path.join(repo, "oracle"),
                                     tol=TOL)
    # eager module loading: the lazy load at a kernel's first launch can synchronise the device, which would order the
    # other branches after the fill by accident and hide a missing ordering
    env = dict(os.environ, STMGCN_GRAPH_STREAMS="1", STMGCN_LSTM_PATH="tc", CUDA_MODULE_LOADING="EAGER")
    res = subprocess.run([sys.executable, "-s", "-c", script], env=env, capture_output=True, text=True, timeout=600)
    print(res.stdout[-2000:], res.stderr[-2000:])
    assert res.returncode == 0, f"exit {res.returncode}: {res.stdout[-500:]} {res.stderr[-1500:]}"
