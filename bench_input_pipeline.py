"""The input pipeline: the reference's ``Data_Container`` loader against ``stmgcn_b200.data``'s device gather.  Prints one
JSON line.

    python bench_input_pipeline.py [--rounds 5] [--launches 200]

Two shapes: cfg3's (4096 regions, C = 1, batch 64, cpt (8, 2, 2): T = 12) on five weeks of hourly data, and Main.py's
(58 regions, batch 32, cpt (3, 1, 1), its default dates) on one year.  Before any time is measured, every batch of the
first and last few of each mode is compared bit for bit with the reference loader's.  Then, per shape:

* ``ms_per_batch``: a full pass over the training mode between CUDA events, the device idle at the start and
  synchronised at the end (so the host's iteration is inside the window), divided by its batches, for each loader; the
  two alternate for ``--rounds`` rounds and the median round is reported;
* ``gather_us`` / ``gather_gbs_written``: one batch's ``stmgcn_window_gather`` alone, CUDA events over ``--launches``
  launches, and the bytes it writes (x and y) over that time;
* ``construction``: host peak RSS growth (sampled every ~1 ms) and device peak memory of ``get_data_loader`` for each
  loader, each measured in a fresh process.

The reference loader is the unmodified module ``__graft_entry__.build()`` stages into ``oracle/_ref/``; without it this
script fails.  Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

from benchlib import REPO, alternate, device_record, require_cuda, setup_paths, timed

REF_DC = os.path.join(REPO, "oracle", "_ref", "Data_Container.pyc")

# (name, regions, series rows, cpt, dates, batch)
SHAPES = {
    "cfg3": (4096, 24 * 7 * 5, (8, 2, 2), ["0101", "0115", "0116", "0121"], 64),
    "main": (58, 24 * 365, (3, 1, 1), ["0101", "0630", "0701", "0731"], 32),
}


def _reference_module():
    import importlib.machinery
    import importlib.util
    if not os.path.exists(REF_DC):
        raise SystemExit(f"{REF_DC} is missing: run __graft_entry__.build() where a reference checkout exists")
    loader = importlib.machinery.SourcelessFileLoader("_ref_Data_Container", REF_DC)
    spec = importlib.util.spec_from_loader("_ref_Data_Container", loader)
    mod = importlib.util.module_from_spec(spec)
    loader.exec_module(mod)
    return mod


def _setup(shape):
    import numpy as np
    n, s_len, cpt, dates, batch = SHAPES[shape]
    taxi = np.random.default_rng(0).normal(0, 1, (s_len, n, 1))
    args = dict(dt=1, obs_len=cpt, train_test_dates=dates, val_ratio=0.2)
    return {"taxi": taxi}, args, batch


def _loaders(kind, data, args, batch):
    from stmgcn_b200.data import DataGenerator
    gen = _reference_module().DataGenerator(**args) if kind == "reference" else DataGenerator(**args)
    return gen.get_data_loader(data, batch_size=batch, device="cuda:0")


def _rss_bytes() -> int:
    with open("/proc/self/statm") as f:
        return int(f.read().split()[1]) * os.sysconf("SC_PAGE_SIZE")


def construction_child(kind: str, shape: str) -> None:
    """One loader's construction in this (fresh) process: host peak RSS growth and device peak memory.  The process's
    own high-water mark would keep the peak of CUDA's initialisation, so the RSS is sampled by a thread every ~1 ms
    while the loaders are built."""
    import threading
    import torch
    data, args, batch = _setup(shape)
    torch.zeros(1, device="cuda:0").float().to("cuda:0")
    _reference_module()                                 # imports (pandas, ...) outside the measured window
    import stmgcn_b200.data  # noqa: F401
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    rss0, dev0 = _rss_bytes(), torch.cuda.memory_allocated()
    peak, done = [rss0], threading.Event()

    def sample():
        while not done.is_set():
            peak[0] = max(peak[0], _rss_bytes())
            time.sleep(0.001)
    sampler = threading.Thread(target=sample)
    sampler.start()
    _loaders(kind, data, args, batch)
    torch.cuda.synchronize()
    done.set()
    sampler.join()
    peak_rss = max(peak[0], _rss_bytes())
    print(json.dumps({"host_peak_rss_growth_mb": round(max(peak_rss - rss0, 0) / 2 ** 20, 1),
                      "device_peak_mb": round((torch.cuda.max_memory_allocated() - dev0) / 2 ** 20, 1)}))


def _check_bits(ref, ours, sample=3):
    import torch
    checked = 0
    for mode in ("train", "validate", "test"):
        assert len(ref[mode]) == len(ours[mode]), mode
        got, want = list(ours[mode]), list(ref[mode])
        idx = sorted(set(range(min(sample, len(got)))) | set(range(max(len(got) - sample, 0), len(got))))
        for i in idx:
            for a, b in zip(got[i], want[i]):
                if a.shape != b.shape or not torch.equal(a.view(torch.int32), b.view(torch.int32)):
                    raise SystemExit(f"{mode} batch {i}: the device gather differs from the reference loader")
            checked += 1
    return checked


def measure(shape: str, rounds: int, launches: int) -> dict:
    import torch
    from stmgcn_b200 import _lib
    data, args, batch = _setup(shape)
    loaders = {kind: _loaders(kind, data, args, batch) for kind in ("reference", "device")}
    checked = _check_bits(loaders["reference"], loaders["device"])

    def epoch(kind):
        for _x, _y in loaders[kind]["train"]:
            pass

    ms, _ = alternate({kind: lambda kind=kind: epoch(kind) for kind in loaders}, rounds, 1, 1)
    times = {kind: [t / len(loaders[kind]["train"]) for t in v] for kind, v in ms.items()}

    # one full batch's gather alone
    dev = loaders["device"]["train"]
    first, b = dev.batches()[0]
    series = dev.series
    row = series[0].numel()
    x = torch.empty((b, dev.t_len, row), device=series.device)
    y = torch.empty((b, row), device=series.device)
    st = torch.cuda.current_stream().cuda_stream

    def gather():
        _lib.check(_lib.lib.stmgcn_window_gather(series.data_ptr(), series.shape[0], row, dev.lags, dev.t_len, first,
                                                 b, x.data_ptr(), y.data_ptr(), st), "window_gather")
    us = timed(gather, launches, 10)[0] * 1e3
    written = (x.numel() + y.numel()) * 4

    construction = {}
    for kind in ("reference", "device"):
        out = subprocess.run([sys.executable, os.path.abspath(__file__), "--construction", kind, shape],
                             capture_output=True, text=True, check=True)
        construction[kind] = json.loads(out.stdout.strip().splitlines()[-1])
    n, s_len, cpt, dates, _ = SHAPES[shape]
    return {"regions": n, "series_rows": s_len, "cpt": list(cpt), "dates": dates, "batch": batch, "T": dev.t_len,
            "train_batches": len(dev), "batches_checked_bitwise": checked,
            "ms_per_batch": {k: round(statistics.median(v), 4) for k, v in times.items()},
            "ms_per_batch_rounds": {k: [round(t, 4) for t in v] for k, v in times.items()},
            "gather_us": round(us, 2), "gather_bytes_written": written,
            "gather_gbs_written": round(written / us / 1e3, 1), "construction": construction}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--construction", nargs=2, metavar=("KIND", "SHAPE"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    require_cuda("bench_input_pipeline.py")
    setup_paths()
    if args.construction:
        construction_child(*args.construction)
        return
    name, limit = device_record()
    result = {"device": name, "power_limit": limit, "nvidia_smi": f"{name}, {limit}"}
    for shape in SHAPES:
        result[shape] = measure(shape, args.rounds, args.launches)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
