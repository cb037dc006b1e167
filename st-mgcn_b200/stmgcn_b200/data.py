"""Training windows gathered on the device: a drop-in ``DataGenerator`` for the reference's ``Data_Container.py``.

The reference (``Data_Container.py:74-146``) builds every serial, daily and weekly window of the series on the host in
float64, concatenates them all again per mode and copies each mode to the device, so every series entry is stored about
``T`` times.  Here the series is converted once (``torch.from_numpy(...).float()``, the reference's own rounding) and
uploaded once; each batch is gathered straight out of it by one launch of ``stmgcn_window_gather``.  Nothing of size
windows x T exists on the host or on the device.

This module alone owns the reference's windowing policy; the kernel only copies rows.  The batches are bit-identical to
the reference's ``DataLoader`` batches, in the same order and with the same short last batch.  One deliberate
difference: a mode whose windows run past the end of the series raises ``ValueError`` naming the mode at
``get_data_loader``, where the reference fails part-way through an epoch with an ``IndexError``.
"""
from __future__ import annotations

import ctypes
import datetime
import math
from typing import Dict, List, Tuple

import numpy as np
import torch

from . import _lib

MODES = ("train", "validate", "test")
MAX_STEPS = 2048            # stmgcn_window_gather's t_len limit (ops.LIMITS["T"])


class DataGenerator(object):
    """The reference's ``DataGenerator`` (same constructor, attributes and ``get_data_loader``); the loaders it returns
    gather on the device."""

    def __init__(self, dt: int, obs_len: tuple, train_test_dates: list, val_ratio: float, year=2017):
        self.day_timesteps = 24 // dt
        self.serial_len, self.daily_len, self.weekly_len = obs_len
        self.train_test_dates = train_test_dates        # [train_start, train_end, test_start, test_end]
        self.val_ratio = val_ratio
        self.start_idx, self.mode_len = self.date2len(year=year)

    def date2len(self, year: int):
        """Data_Container.py:100-111 with ``datetime`` for pandas: an invalid date raises ``ValueError`` from
        ``list.index``, as there.  ``start_idx`` is the training start's DAY index (:104), used as a window index (below)."""
        first = datetime.date(year, 1, 1)
        days = (datetime.date(year + 1, 1, 1) - first).days
        date_range = [(first + datetime.timedelta(days=d)).strftime("%Y%m%d") for d in range(days)]
        train_s_idx, train_e_idx = date_range.index(str(year) + self.train_test_dates[0]), \
            date_range.index(str(year) + self.train_test_dates[1])
        train_len = (train_e_idx + 1 - train_s_idx) * self.day_timesteps
        validate_len = int(train_len * self.val_ratio)
        train_len -= validate_len
        test_s_idx, test_e_idx = date_range.index(str(year) + self.train_test_dates[2]), \
            date_range.index(str(year) + self.train_test_dates[3])
        test_len = (test_e_idx + 1 - test_s_idx) * self.day_timesteps
        return train_s_idx, {"train": train_len, "validate": validate_len, "test": test_len}

    # ---- the windowing policy ------------------------------------------------------------------------------------
    def first_window(self) -> int:
        """Series row of window 0's target (Data_Container.py:134): max(serial, daily * day_ts, weekly * day_ts * 7)."""
        return max(self.serial_len, self.daily_len * self.day_timesteps, self.weekly_len * self.day_timesteps * 7)

    def lags(self) -> List[int]:
        """How many rows before its target row each step of a window reads, in the order of the concatenation
        (Data_Container.py:84-86): weekly, daily, serial, each oldest first (the periodic parts reversed, :145)."""
        # the periodic step is daily_len * day_ts (:138), not day_ts, and weekly_len * day_ts * 7 (:142): with a length
        # >= 2 the early windows reach before row 0 and read the END of the series through numpy's negative index (:140)
        weekly = [self.weekly_len * self.day_timesteps * 7 * w for w in range(self.weekly_len, 0, -1)]
        daily = [self.daily_len * self.day_timesteps * d for d in range(self.daily_len, 0, -1)]
        serial = list(range(self.serial_len, 0, -1))                 # data[i - serial_len : i] (:136)
        return weekly + daily + serial

    def mode_ranges(self, s_len: int) -> Dict[str, Tuple[int, int]]:
        """``{mode: (series row of its first target, number of windows)}`` on a series of ``s_len`` rows.

        Mode offsets are ``start_idx`` plus the lengths of the earlier modes (Data_Container.py:75-80), in windows.
        Raises ``IndexError`` where the reference's ``get_feats`` does (a periodic step before row -s_len) and
        ``ValueError`` naming a mode whose windows run past the series (the deliberate difference)."""
        first, lags = self.first_window(), self.lags()
        if not lags:
            raise ValueError("DataGenerator: obs_len has no observation step")
        if len(lags) > MAX_STEPS:
            raise ValueError(f"DataGenerator: {len(lags)} observation steps (at most {MAX_STEPS})")
        if first < s_len and first - max(lags) < -s_len:
            raise IndexError(f"DataGenerator: window {first} reads row {first - max(lags)}, before the series' "
                             f"first row -{s_len}")
        windows = max(s_len - first, 0)
        out, start = {}, self.start_idx
        for mode in MODES:
            n = self.mode_len[mode]
            if n > 0 and start + n > windows:
                raise ValueError(f"DataGenerator: the {mode!r} windows [{start}, {start + n}) run past the {windows} "
                                 f"windows of a series of {s_len} rows")
            out[mode] = (first + start, n)
            start += n
        return out

    def get_data_loader(self, data: dict, batch_size: int, device: str):
        """``{'train', 'validate', 'test'}`` loaders over ``data['taxi']`` (S, N, C): each yields ``(x (B,T,N,C),
        y (B,N,C))`` float32 tensors on the CUDA ``device``, gathered from one resident copy of the series."""
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("stmgcn_b200 kernels need CUDA tensors (there is no CPU fallback)")
        if isinstance(batch_size, bool) or not isinstance(batch_size, int) or batch_size <= 0:
            raise ValueError(f"batch_size should be a positive integer value, but got batch_size={batch_size}")
        taxi = np.asarray(data["taxi"])
        if taxi.ndim < 2:
            raise ValueError(f"DataGenerator: data['taxi'] of shape {taxi.shape}: (S, N, ...) expected")
        ranges = self.mode_ranges(taxi.shape[0])
        series = torch.from_numpy(np.ascontiguousarray(taxi)).float().contiguous().to(device)
        lags = self.lags()
        return {mode: WindowLoader(series, lags, first, n, batch_size) for mode, (first, n) in ranges.items()}


class WindowLoader(object):
    """Batches of ``n`` consecutive windows whose targets start at series row ``first``: ``len()`` and iteration as a
    ``DataLoader(batch_size=batch_size, shuffle=False)``.  Each batch is gathered by one kernel launch on the current
    stream into fresh tensors."""

    def __init__(self, series: torch.Tensor, lags: List[int], first: int, n: int, batch_size: int):
        self.series, self.first, self.n, self.batch_size = series, first, n, batch_size
        self.lags = (ctypes.c_int32 * len(lags))(*lags)
        self.t_len = len(lags)

    def batches(self) -> List[Tuple[int, int]]:
        """``(series row of the batch's first target, batch size)`` of every batch, in order."""
        return [(self.first + s, min(self.batch_size, self.n - s)) for s in range(0, self.n, self.batch_size)]

    def __len__(self) -> int:
        return math.ceil(self.n / self.batch_size)

    def __iter__(self):
        s_len, feat = self.series.shape[0], self.series.shape[1:]
        row = self.series[0].numel()
        for first, b in self.batches():
            x = torch.empty((b, self.t_len) + feat, dtype=torch.float32, device=self.series.device)
            y = torch.empty((b,) + feat, dtype=torch.float32, device=self.series.device)
            with torch.cuda.device(self.series.device):
                _lib.check(_lib.lib.stmgcn_window_gather(self.series.data_ptr(), s_len, row, self.lags, self.t_len,
                                                         first, b, x.data_ptr(), y.data_ptr(),
                                                         torch.cuda.current_stream().cuda_stream), "window_gather")
            yield x, y
