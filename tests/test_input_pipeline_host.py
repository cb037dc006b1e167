"""CPU tests of the device-side input pipeline (``stmgcn_b200.data``): its window table against the reference's own
``DataGenerator``, the argument checks of ``stmgcn_window_gather``, and the loader's errors.

The reference comparison runs the unmodified ``Data_Container`` that ``__graft_entry__.build()`` byte-compiles into
``oracle/_ref/`` on a series whose row ``s`` holds the value ``s``: every value of a reference batch then names the series
row it came from, wrapped rows included.  It skips when that file has not been staged."""
import ctypes
import importlib.machinery
import importlib.util
import os

import numpy as np
import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DC = os.path.join(REPO, "oracle", "_ref", "Data_Container.pyc")

OBS_LENS = [(3, 1, 1), (0, 1, 1), (3, 0, 0), (2, 2, 2), (1, 0, 3)]
S_LEN = 1400            # > 1008: (1, 0, 3) at dt = 1 reads row 504 - 1512 = -1008, wrapped from the end


def _reference_data_container():
    if not os.path.exists(REF_DC):
        pytest.skip("oracle/_ref/Data_Container.pyc not staged (run __graft_entry__.build() where a reference exists)")
    pytest.importorskip("pandas")          # the reference's date arithmetic
    loader = importlib.machinery.SourcelessFileLoader("_ref_Data_Container", REF_DC)
    spec = importlib.util.spec_from_loader("_ref_Data_Container", loader)
    mod = importlib.util.module_from_spec(spec)
    loader.exec_module(mod)
    return mod


def _row_series(s_len):
    return np.arange(s_len, dtype=np.float64)[:, None, None] * np.ones((1, 1, 1))


@pytest.mark.parametrize("obs_len", OBS_LENS)
def test_window_table_and_batches_match_the_reference_data_generator(obs_len):
    from stmgcn_b200.data import DataGenerator, WindowLoader
    dc = _reference_data_container()
    data = {"taxi": _row_series(S_LEN)}
    checked = 0
    for dt in (1, 2, 3):
        for dates in (["0101", "0103", "0104", "0104"], ["0105", "0108", "0109", "0110"]):
            for val_ratio in (0.2, 0.35):
                args = dict(dt=dt, obs_len=obs_len, train_test_dates=dates, val_ratio=val_ratio)
                ref, gen = dc.DataGenerator(**args), DataGenerator(**args)
                assert (gen.start_idx, gen.mode_len) == (ref.start_idx, ref.mode_len), args
                ranges = gen.mode_ranges(S_LEN)
                lags = np.asarray(gen.lags())
                ref_loaders = ref.get_data_loader(data, batch_size=7, device="cpu")
                for mode, (first, n) in ranges.items():
                    # every window of the mode: its target row and the source row of every step
                    ds = ref_loaders[mode].dataset
                    x, y = ds.inputs["x_seq"].numpy(), ds.output.numpy()
                    assert len(ds) == n and x.shape[:2] == (n, len(lags)) and y.shape[0] == n, (args, mode)
                    want_y = first + np.arange(n)
                    want_x = want_y[:, None] - lags[None, :]
                    want_x = np.where(want_x < 0, want_x + S_LEN, want_x)
                    np.testing.assert_array_equal(y[:, 0, 0], want_y, err_msg=f"{args} {mode} targets")
                    np.testing.assert_array_equal(x[:, :, 0, 0], want_x, err_msg=f"{args} {mode} source rows")
                    # batch boundaries: first target row and size of every reference batch
                    got = WindowLoader(torch.zeros(S_LEN, 1, 1), gen.lags(), first, n, 7)
                    want = [(int(yb[0, 0, 0]), yb.shape[0]) for _, yb in ref_loaders[mode]]
                    assert got.batches() == want and len(got) == len(ref_loaders[mode]), (args, mode)
                    checked += n
    assert checked > 0


def test_wrapped_rows_are_exercised():
    from stmgcn_b200.data import DataGenerator
    for obs_len in ((2, 2, 2), (1, 0, 3)):
        gen = DataGenerator(dt=1, obs_len=obs_len, train_test_dates=["0101", "0103", "0104", "0104"], val_ratio=0.2)
        first, _ = gen.mode_ranges(S_LEN)["train"]
        assert first - max(gen.lags()) < 0


# ======================================================================================================================
# the C entry point's checks
# ======================================================================================================================
def test_window_gather_rejects_bad_arguments_before_any_launch():
    from stmgcn_b200 import _lib
    lib = _lib.lib
    p = ctypes.c_void_p
    fake = 0x100000          # never dereferenced: every call below fails its checks first
    s_len, row, t_len, first, b = 100, 8, 3, 20, 10
    # series @0 (3200 B), obs @65536 (960 B), y @131072 (320 B)
    at = dict(series=0, obs=65536, y=131072)

    def call(lags=(5, 2, 1), s_len=s_len, row=row, t_len=t_len, first=first, b=b, **over):
        ptr = {k: (None if over.get(k, 0) is None else fake + over.get(k, v)) for k, v in at.items()}
        lv = None if lags is None else (ctypes.c_int32 * max(len(lags), 1))(*lags)
        return lib.stmgcn_window_gather(p(ptr["series"]), s_len, row, lv, t_len, first, b, p(ptr["obs"]), p(ptr["y"]),
                                        None)

    before = _lib.launch_count()
    cases = [
        (dict(series=None), "null pointer"), (dict(obs=None), "null pointer"), (dict(y=None), "null pointer"),
        (dict(lags=None), "null pointer"),
        (dict(s_len=0), "bad shape"), (dict(row=0), "bad shape"), (dict(b=0), "bad shape"), (dict(t_len=0), "bad shape"),
        (dict(row=-4), "bad shape"), (dict(t_len=2049, lags=[1] * 2049), "T=2049"),
        (dict(first=-1), "run past the series"), (dict(first=91), "run past the series"),
        (dict(first=100, b=1), "run past the series"),
        (dict(lags=(5, -1, 1)), "lags[1]=-1 is negative"),
        (dict(first=0, lags=(101, 2, 1)), "before -s_len"), (dict(first=5, lags=(5, 106, 1)), "before -s_len"),
        (dict(obs=3200 - 4), "overlap the series"), (dict(y=-320 + 4), "overlap the series"),
        (dict(obs=1000), "overlap the series"), (dict(y=65536 + 960 - 4), "obs and y overlap"),
        (dict(row=1 << 40, s_len=1 << 20), "too large"),
    ]
    for over, msg in cases:
        rc = call(**over)
        assert rc < 0, (over, rc)
        assert msg in lib.stmgcn_last_error().decode(), (over, lib.stmgcn_last_error())
    assert _lib.launch_count() == before, "a rejected call launched a kernel"


def test_window_gather_is_bound():
    from stmgcn_b200 import _lib
    sig = {name: args for name, _, args in _lib.SIGNATURES}
    assert len(sig["stmgcn_window_gather"]) == 10 and _lib.ABI_VERSION == 8


# ======================================================================================================================
# the loader's errors
# ======================================================================================================================
def test_invalid_dates_raise_value_error_as_the_reference_does():
    from stmgcn_b200.data import DataGenerator
    for dates in (["0230", "0301", "0302", "0303"], ["0101", "0132", "0201", "0202"], ["0101", "0105", "011", "0107"],
                  ["0101", "0105", "0106", "1301"]):
        with pytest.raises(ValueError):
            DataGenerator(dt=1, obs_len=(3, 1, 1), train_test_dates=dates, val_ratio=0.2)
    gen = DataGenerator(dt=1, obs_len=(3, 1, 1), train_test_dates=["0101", "1231", "0101", "0101"], val_ratio=0.2)
    assert gen.mode_len["train"] + gen.mode_len["validate"] == 365 * 24
    leap = DataGenerator(dt=2, obs_len=(3, 1, 1), train_test_dates=["0229", "0229", "0301", "0301"], val_ratio=0.0,
                         year=2016)
    assert leap.start_idx == 59 and leap.mode_len == {"train": 12, "validate": 0, "test": 12}


def test_a_mode_running_past_the_series_raises_value_error_naming_it():
    from stmgcn_b200.data import DataGenerator
    gen = DataGenerator(dt=1, obs_len=(3, 1, 1), train_test_dates=["0101", "0107", "0108", "0109"], val_ratio=0.2)
    s_len = gen.first_window() + gen.mode_len["train"] + gen.mode_len["validate"] + gen.mode_len["test"]
    assert gen.mode_ranges(s_len)["test"] == (gen.first_window() + 168, 48)
    for short, mode in ((1, "'test'"), (49, "'validate'"), (49 + 34, "'train'")):
        with pytest.raises(ValueError, match=mode):
            gen.mode_ranges(s_len - short)
    with pytest.raises(ValueError, match="'test'"):
        gen.get_data_loader({"taxi": np.zeros((s_len - 1, 4, 1))}, batch_size=8, device="cuda:0")


def test_loader_refuses_the_cpu_and_bad_batch_sizes_and_reaching_before_the_series():
    from stmgcn_b200.data import DataGenerator
    gen = DataGenerator(dt=1, obs_len=(3, 1, 1), train_test_dates=["0101", "0107", "0108", "0109"], val_ratio=0.2)
    data = {"taxi": np.zeros((400, 4, 1))}
    with pytest.raises(RuntimeError, match="CUDA"):
        gen.get_data_loader(data, batch_size=8, device="cpu")
    for bad in (0, -3, 2.0):
        with pytest.raises(ValueError, match="batch_size"):
            gen.get_data_loader(data, batch_size=bad, device="cuda:0")
    # cpt (1, 0, 3): window 504 reads row 504 - 1512 = -1008; the reference's get_feats raises IndexError there
    far = DataGenerator(dt=1, obs_len=(1, 0, 3), train_test_dates=["0101", "0102", "0103", "0103"], val_ratio=0.2)
    with pytest.raises(IndexError):
        far.mode_ranges(1000)
    assert far.mode_ranges(1008)["train"][0] == 504
