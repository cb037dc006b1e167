"""What the side benchmarks (every ``bench_*.py`` but ``bench.py``) share: the import path, the refusal to run without a
CUDA device, the card's record, and CUDA-event timing, alone or of variants alternated round by round.

The record is read with one query; nothing here changes a device or host setting.
"""
from __future__ import annotations

import os
import subprocess
import sys

REPO = os.path.dirname(os.path.abspath(__file__))


def setup_paths() -> None:
    """Put the repository root, ``st-mgcn_b200/`` and ``oracle/`` on ``sys.path``."""
    for p in (REPO, os.path.join(REPO, "st-mgcn_b200"), os.path.join(REPO, "oracle")):
        if p not in sys.path:
            sys.path.insert(0, p)


def require_cuda(script: str) -> None:
    """Exit non-zero unless a CUDA device is visible: the benchmarks time the GPU and have no CPU fallback."""
    import torch
    if not torch.cuda.is_available():
        sys.exit(f"{script} needs a CUDA device (an H100); none is visible")


def device_record() -> tuple:
    """``(name, power limit)`` of the first visible device (``CUDA_VISIBLE_DEVICES`` honoured), from one read-only
    nvidia-smi query.  When the query fails the name comes from torch and the power limit is ``"unknown"``."""
    import torch
    idx = os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0].strip() or "0"
    try:
        q = subprocess.run(["nvidia-smi", "-i", idx, "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        fields = q.stdout.strip().splitlines()[0].split(",") if q.returncode == 0 and q.stdout.strip() else []
    except (OSError, subprocess.SubprocessError):
        fields = []
    if len(fields) != 2:
        return torch.cuda.get_device_name(0), "unknown"
    return fields[0].strip(), fields[1].strip()


def timed(fn, steps: int, warmup: int = 0) -> tuple:
    """Call ``fn`` ``warmup`` times, then time ``steps`` calls between CUDA events, the device synchronised before and
    after: ``(ms per call, library kernel launches per call)``."""
    import torch
    from stmgcn_b200 import _lib
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / steps, (_lib.launch_count() - n0) // steps


def alternate(variants: dict, rounds: int, steps: int, warmup: int) -> tuple:
    """Warm every variant of ``variants`` (name -> callable) up ``warmup`` times, then time ``steps`` calls of each in
    turn, round after round: ``({name: [ms per call, one per round]}, {name: launches per call})``."""
    for _ in range(warmup):
        for fn in variants.values():
            fn()
    ms = {name: [] for name in variants}
    launches = {}
    for _ in range(rounds):
        for name, fn in variants.items():
            t, launches[name] = timed(fn, steps)
            ms[name].append(t)
    return ms, launches
