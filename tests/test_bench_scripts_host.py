"""The side benchmarks (every ``bench_*.py`` but ``bench.py``) without a GPU: each answers ``--help``, each refuses to
run when no CUDA device is visible instead of falling back to the CPU, and none keeps its own card query or CUDA-event
timing loop beside ``benchlib.py``'s."""
import glob
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPTS = sorted(os.path.basename(p) for p in glob.glob(os.path.join(ROOT, "bench_*.py")))


def _run(script, *args):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")         # no device visible, on any machine
    return subprocess.run([sys.executable, os.path.join(ROOT, script), *args], cwd=ROOT, env=env, timeout=300,
                          capture_output=True, text=True)


def test_the_side_benchmarks_are_found():
    assert "bench_frozen.py" in SCRIPTS and "bench.py" not in SCRIPTS


@pytest.mark.parametrize("script", SCRIPTS)
def test_answers_help(script):
    res = _run(script, "--help")
    assert res.returncode == 0, res.stderr[-2000:]
    assert "usage:" in res.stdout


@pytest.mark.parametrize("script", SCRIPTS)
def test_refuses_to_run_without_cuda(script):
    res = _run(script)
    assert res.returncode != 0
    assert "CUDA" in res.stderr + res.stdout, res.stderr[-2000:]


@pytest.mark.parametrize("script", SCRIPTS)
def test_card_and_timing_helpers_live_in_benchlib(script):
    with open(os.path.join(ROOT, script)) as f:
        src = f.read()
    for helper in ("nvidia-smi", "Event(enable_timing"):
        assert helper not in src, f"{script} has its own {helper!r}: use benchlib.device_record / benchlib.timed"
