"""bench.py contract checks that need no GPU: the reference arm (the unmodified reference modules from oracle/_ref, or the oracle port, timed on host cores) prints one JSON
line with the keys the driver reads, non-zero ranks of a multi-process launch stay silent, and the product arm refuses
to run without a CUDA device instead of falling back to anything on the CPU."""
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(args, env_extra=None, timeout=600):
    env = dict(os.environ)
    env.update(env_extra or {})
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + args, cwd=ROOT, env=env, timeout=timeout,
                          capture_output=True, text=True)


def test_reference_arm_prints_the_contract_line():
    res = _run(["--impl", "reference", "--workload", "cfg1", "--steps", "2", "--warmup", "1"])
    assert res.returncode == 0, res.stderr[-2000:]
    lines = [l for l in res.stdout.strip().splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["higher_is_better"] is True and d["unit"] == "region-timesteps/s"
    for key in ("metric", "value", "n_gpus", "steps", "warmup", "ms_per_step", "scaling", "dtype", "data", "config",
                "cpu_baseline", "e2e"):
        assert key in d, key
    staged = os.path.exists(os.path.join(ROOT, "oracle", "_ref", "STMGCN.pyc"))
    assert d["value"] > 0 and d["cpu_baseline"]["cores"] >= 1
    # the unmodified reference (built by build()) when present, else the oracle port
    assert d["cpu_baseline"]["kind"] == ("reference" if staged else "port")
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert d["e2e"]["value"] == d["value"] == d["cpu_baseline"]["value"]
    assert "workload" in d["config"]


def test_reference_arm_non_zero_rank_is_silent():
    res = _run(["--impl", "reference", "--workload", "cfg1", "--gpus", "2", "--steps", "1", "--warmup", "0"],
               {"RANK": "1", "LOCAL_RANK": "1", "WORLD_SIZE": "2", "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": "29577"})
    assert res.returncode == 0, res.stderr[-2000:]
    assert res.stdout.strip() == ""


@pytest.mark.skipif(torch.cuda.is_available(), reason="only meaningful on a machine without a GPU")
def test_product_arm_refuses_to_run_without_cuda():
    res = _run(["--workload", "cfg1", "--steps", "1", "--warmup", "0", "--no-cpu-baseline"])
    assert res.returncode != 0
    assert "CUDA" in (res.stderr + res.stdout)
