"""GPU tests of the device-side input pipeline (``stmgcn_b200.data``, ``stmgcn_window_gather``).

* Every batch of every mode is bit-identical to the reference ``DataLoader``'s (the unmodified ``Data_Container`` that
  ``__graft_entry__.build()`` stages into ``oracle/_ref/``; skipped without it) on float64 series holding NaN, +-0, +-Inf
  and values whose fp32 rounding is not the obvious one.
* The C entry point keeps the memory and stream contract of ``tests/abi_harness.py``.
* At N = 16384 the loader's device memory is the series plus the batches in flight.
* Two epochs of the reference trainer agree with either loader.
"""
import ctypes
import importlib.machinery
import importlib.util
import io
import os
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch
from torch import nn

from abi_harness import Buf, Call, bits, run_captured, run_contract
from helpers import DEV, lib, rel_err

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(REPO, "oracle", "_ref")


def _reference(name):
    path = os.path.join(REF, name + ".pyc")
    if not os.path.exists(path):
        pytest.skip(f"oracle/_ref/{name}.pyc not staged (run __graft_entry__.build() where a reference exists)")
    loader = importlib.machinery.SourcelessFileLoader("_ref_" + name, path)
    spec = importlib.util.spec_from_loader("_ref_" + name, loader)
    mod = importlib.util.module_from_spec(spec)
    loader.exec_module(mod)
    return mod


def _hostile_series(s_len, n, c, seed):
    """float64 (s_len, n, c): normals, plus NaN (two payloads), +-0, +-Inf, fp32 overflow and underflow, and ties and
    near-ties of the fp32 rounding."""
    rng = np.random.default_rng(seed)
    v = rng.normal(0, 3, (s_len, n, c))
    special = np.array([np.nan, -np.nan, np.frombuffer(np.uint64(0x7FF0000000000123).tobytes(), np.float64)[0], 0.0,
                        -0.0, np.inf, -np.inf, 1e39, -1e39, 1e-46, -1e-40, 1 + 2.0 ** -24, 1 + 3 * 2.0 ** -24,
                        1 + 2.0 ** -24 + 2.0 ** -50, 3.4028235677973366e38, 0.1])
    flat = v.reshape(-1)
    pick = rng.choice(flat.size, size=min(flat.size // 3, 40 * special.size), replace=False)
    flat[pick] = special[np.arange(pick.size) % special.size]
    return v


# (name, regions N, C, dt, cpt, dates, series rows)
CASES = [
    ("dropin", 58, 1, 1, (3, 1, 1), ["0101", "0107", "0108", "0109"], 24 * 16),     # row % 4 != 0: scalar kernel
    ("wrapped", 58, 1, 1, (2, 2, 2), ["0101", "0107", "0108", "0109"], 24 * 24),    # weekly rows from the series' end
    ("c2_dt2", 58, 2, 2, (3, 1, 1), ["0101", "0107", "0108", "0109"], 12 * 17),    # row = 116: float4 kernel
    ("row64", 64, 1, 1, (3, 1, 1), ["0102", "0106", "0107", "0107"], 24 * 14),       # row % 4 == 0: float4 kernel
]


@pytest.mark.parametrize("batch_size", [1, 7, 32, 500])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_every_batch_is_bit_identical_to_the_reference_loader(case, batch_size):
    from stmgcn_b200 import _lib
    from stmgcn_b200.data import DataGenerator
    dc = _reference("Data_Container")
    _, n, c, dt, cpt, dates, s_len = case
    data = {"taxi": _hostile_series(s_len, n, c, seed=s_len + n)}
    args = dict(dt=dt, obs_len=cpt, train_test_dates=dates, val_ratio=0.2)
    ref = dc.DataGenerator(**args).get_data_loader(data, batch_size=batch_size, device=DEV)
    ours = DataGenerator(**args).get_data_loader(data, batch_size=batch_size, device=DEV)
    for mode in ("train", "validate", "test"):
        assert len(ours[mode]) == len(ref[mode]), mode
        n0 = _lib.launch_count()
        got = list(ours[mode])
        assert _lib.launch_count() - n0 == len(got), "one launch per batch"
        want = list(ref[mode])
        assert len(got) == len(want), mode
        for i, ((xg, yg), (xw, yw)) in enumerate(zip(got, want)):
            assert xg.shape == xw.shape and yg.shape == yw.shape, (mode, i, xg.shape, xw.shape)
            assert xg.dtype == torch.float32 and xg.device == xw.device and xg.is_contiguous()
            assert torch.equal(bits(xg), bits(xw)), f"{mode} batch {i}: x differs"
            assert torch.equal(bits(yg), bits(yw)), f"{mode} batch {i}: y differs"


# ======================================================================================================================
# the C ABI contract
# ======================================================================================================================
def _gather_call(s_len, row, lags, first, b, seed):
    series = torch.from_numpy(_hostile_series(s_len, row, 1, seed)[..., 0]).float()
    t_len = len(lags)
    bufs = dict(series=Buf("in", series), obs=Buf("out", shape=(b, t_len, row), finite=False),
                y=Buf("out", shape=(b, row), finite=False))
    lv = (ctypes.c_int32 * t_len)(*lags)

    def ref(res):
        k = torch.arange(b)[:, None]
        src = first + k - torch.tensor(lags)[None, :]
        src = torch.where(src < 0, src + s_len, src)
        assert torch.equal(bits(res["obs"].cpu()), bits(series[src]))
        assert torch.equal(bits(res["y"].cpu()), bits(series[first:first + b]))

    return Call(f"window_gather(row={row})", bufs, lambda st: lib().stmgcn_window_gather(
        bufs["series"].p, s_len, row, lv, t_len, first, b, bufs["obs"].p, bufs["y"].p, st), ref, 1)


@pytest.mark.parametrize("row", [58, 116, 4096 + 4])
def test_window_gather_keeps_the_memory_contract_eager_and_captured(row):
    """Guard bands, poisoned outputs, untouched inputs, one launch; then eager on a side stream against a graph replay."""
    lags = [336, 168, 48, 24, 2, 1]                      # cpt (2, 2, 2)-like: window 0 wraps
    call = _gather_call(400, row, lags, first=170, b=37, seed=row)
    run_contract(call)
    run_captured(call)


def test_window_gather_falls_back_to_scalar_accesses_on_misaligned_pointers():
    s_len, row, lags, first, b = 90, 64, [60, 7, 1], 10, 9
    base = torch.randn(s_len * row + 1, device=DEV)
    series = base[1:].view(s_len, row)                   # 4-byte aligned only: row % 4 == 0 but no float4 access
    out = torch.empty(b * len(lags) * row + b * row + 1, device=DEV)
    obs = out[1:1 + b * len(lags) * row].view(b, len(lags), row)
    y = out[1 + b * len(lags) * row:].view(b, row)
    lv = (ctypes.c_int32 * len(lags))(*lags)
    assert lib().stmgcn_window_gather(series.data_ptr(), s_len, row, lv, len(lags), first, b, obs.data_ptr(),
                                      y.data_ptr(), torch.cuda.current_stream().cuda_stream) == 0
    src = first + torch.arange(b, device=DEV)[:, None] - torch.tensor(lags, device=DEV)[None, :]
    src = torch.where(src < 0, src + s_len, src)
    assert torch.equal(bits(obs), bits(series[src])) and torch.equal(bits(y), bits(series[first:first + b]))


# ======================================================================================================================
# memory at scale
# ======================================================================================================================
def test_memory_at_scale_is_the_series_plus_the_batches_in_flight():
    """N = 16384, C = 1, cpt (8, 4, 4): T = 16.  The weekly step is 4 weeks (Data_Container.py:142), so the first window
    (row 672) reaches back 16 weeks to row -2016: the series has 12 weeks, and the early weekly rows wrap to its end."""
    from stmgcn_b200.data import DataGenerator
    n, s_len, batch = 16384, 24 * 7 * 12, 64
    rng = np.random.default_rng(3)
    taxi = rng.standard_normal((s_len, n, 1), dtype=np.float32).astype(np.float64)
    gen = DataGenerator(dt=1, obs_len=(8, 4, 4), train_test_dates=["0101", "0120", "0121", "0131"], val_ratio=0.2)
    series = torch.from_numpy(taxi).float().to(DEV)                            # for the spot checks
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    loaders = gen.get_data_loader({"taxi": taxi}, batch_size=batch, device=DEV)
    series_bytes, batch_bytes = s_len * n * 4, batch * (16 + 1) * n * 4
    seen = 0
    checks = {("train", 0), ("train", 3), ("validate", 1), ("test", len(loaders["test"]) - 1)}
    for mode in ("train", "validate", "test"):
        # a plain loop: enumerate / zip keep the previous item in their reused result tuples, a third batch
        ranges, i = loaders[mode].batches(), 0
        for x, y in loaders[mode]:
            first, b = ranges[i]
            key, i = (mode, i), i + 1
            seen += x.shape[0]
            if key in checks:
                rows = first + torch.arange(b, device=DEV)[:, None] - torch.tensor(gen.lags(), device=DEV)[None, :]
                if key == ("train", 0):
                    assert int(rows.min()) < 0, "the first batch reads wrapped rows"
                rows = torch.where(rows < 0, rows + s_len, rows)
                for k in range(b):          # one window at a time: a batch-sized temporary would count as a third batch
                    assert torch.equal(bits(x[k]), bits(series[rows[k]])), key + (k,)
                assert torch.equal(bits(y), bits(series[first:first + b])), key
    torch.cuda.synchronize()
    growth = torch.cuda.max_memory_allocated() - base
    assert seen == sum(gen.mode_len.values())
    assert growth <= series_bytes + 2 * batch_bytes + 64 * 2 ** 20, (growth, series_bytes, batch_bytes)


# ======================================================================================================================
# training equivalence
# ======================================================================================================================
class _RecordingMSE(nn.Module):
    """MSELoss that keeps (grad enabled, loss * batch, batch) of every call: the trainer's running_loss terms."""

    def __init__(self):
        super().__init__()
        self.log = []

    def forward(self, pred, true):
        loss = nn.functional.mse_loss(pred, true)
        self.log.append((torch.is_grad_enabled(), float(loss.detach()) * true.shape[0], true.shape[0]))
        return loss


def test_two_epochs_of_the_reference_trainer_agree_with_either_loader(tmp_path):
    import GCN
    import STMGCN
    from stmgcn_b200.data import DataGenerator
    dc, mt = _reference("Data_Container"), _reference("Model_Trainer")
    n, s_len = 20, 24 * 12
    rng = np.random.default_rng(11)
    data = {"taxi": np.abs(rng.normal(0.5, 0.3, (s_len, n, 1)))}
    adjs = []
    for dens in (0.2, 0.35):
        a = (rng.random((n, n)) < dens).astype(np.float64)
        a = np.maximum(a, a.T)
        np.fill_diagonal(a, 0)
        idx = np.arange(n)
        a[idx, (idx + 1) % n] = a[(idx + 1) % n, idx] = 1
        adjs.append(GCN.Adj_Preprocessor("chebyshev", 2).process(torch.from_numpy(a).float()).to(DEV))
    args = dict(dt=1, obs_len=(3, 1, 1), train_test_dates=["0101", "0104", "0105", "0105"], val_ratio=0.2)
    runs = {}
    for name, gen in (("reference", dc.DataGenerator(**args)), ("device", DataGenerator(**args))):
        loaders = gen.get_data_loader(data, batch_size=16, device=DEV)
        torch.manual_seed(5)
        model = STMGCN.ST_MGCN(M=2, seq_len=5, n_nodes=n, input_dim=1, lstm_hidden_dim=64, lstm_num_layers=2,
                               gcn_hidden_dim=16, sta_kernel_config={"kernel_type": "chebyshev", "K": 2},
                               gconv_use_bias=True, gconv_activation=nn.ReLU).to(DEV)
        crit = _RecordingMSE()
        trainer = mt.ModelTrainer(model=model, loss=crit, optimizer=torch.optim.Adam, lr=2e-3, wd=1e-4, n_epochs=2)
        os.makedirs(tmp_path / name, exist_ok=True)
        with redirect_stdout(io.StringIO()):
            trainer.train(data_loader=loaders, sta_adj_list=adjs, modes=["train", "validate"],
                          model_dir=str(tmp_path / name))
        val = [(s, b) for grad, s, b in crit.log if not grad]
        per = len(loaders["validate"])
        assert len(val) == 2 * per
        losses = [sum(s for s, _ in val[e * per:(e + 1) * per]) / sum(b for _, b in val[e * per:(e + 1) * per])
                  for e in range(2)]
        runs[name] = (losses, {k: v.detach().clone() for k, v in model.state_dict().items()},
                      sum(1 for grad, _, _ in crit.log if grad))
    (l_ref, p_ref, steps_ref), (l_dev, p_dev, steps_dev) = runs["reference"], runs["device"]
    assert steps_ref == steps_dev == 2 * 5
    for a, b in zip(l_dev, l_ref):
        assert abs(a - b) <= 1e-5 * abs(b), (l_dev, l_ref)
    for k in p_ref:
        assert rel_err(p_dev[k], p_ref[k]) <= 1e-5, k
