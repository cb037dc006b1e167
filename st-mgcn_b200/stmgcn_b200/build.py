"""Build ``libstmgcn_b200.so`` in-tree with nvcc for sm_90a (H100; and nothing else).

``python -m stmgcn_b200.build`` (with ``st-mgcn_b200/`` on ``sys.path``) or ``__graft_entry__.build()``.
The shared object lands in ``st-mgcn_b200/lib/`` (git-ignored build output).
Objects are rebuilt only when a source or header is newer.
"""
from __future__ import annotations

import os
import re
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG_DIR)                      # st-mgcn_b200/
REPO = os.path.dirname(ROOT)
CSRC = os.path.join(ROOT, "csrc")
LIB_DIR = os.path.join(ROOT, "lib")
OBJ_DIR = os.path.join(ROOT, "build")
LIB_PATH = os.path.join(LIB_DIR, "libstmgcn_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",     # the long form: `-arch=sm_90a` drops the `a` features (wgmma)
    "-O3", "-lineinfo", "-std=c++17",               # no --use_fast_math: IEEE div / sqrt; the fast exp is explicit
    "-Xcompiler", "-fPIC", "-Xcompiler", "-O3",
    "-Xptxas", "-v",
]
# ptxas C7511 / C7512: every wgmma of the function then waits for the previous one to complete.  Only a warning, but it
# costs the tensor-core kernels most of their throughput, so the build refuses it.
_SERIALIZED_WGMMA = re.compile(r"wgmma\.mma_async instructions are serialized .*? function '([^']+)'")


def _nvcc() -> str:
    path = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(path):
        raise RuntimeError("nvcc not found: libstmgcn_b200.so cannot be built")
    return path


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _headers():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs.append(os.path.join(REPO, "include", "stmgcn_b200.h"))
    return hs


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(verbose: bool = False, force: bool = False) -> str:
    os.makedirs(LIB_DIR, exist_ok=True)
    os.makedirs(OBJ_DIR, exist_ok=True)
    nvcc = _nvcc()
    hdrs = _headers()
    objs, jobs = [], []
    for src in sources():
        obj = os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        if force or _stale(obj, [src] + hdrs):
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        cmd = [nvcc] + NVCC_FLAGS + ["-c", src, "-o", obj]
        res = subprocess.run(cmd, capture_output=True, text=True)
        log = res.stdout + res.stderr
        with open(obj + ".log", "w") as fh:
            fh.write(" ".join(cmd) + "\n" + log)
        if res.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{log}")
        serialized = sorted(set(_SERIALIZED_WGMMA.findall(log)))
        if serialized:
            os.remove(obj)              # not left behind as up to date
            raise RuntimeError(f"ptxas serialized the wgmma instructions of {', '.join(serialized)} in {src} "
                               f"(insufficient register resources):\n{log}")
        return src, log

    if jobs:
        with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as pool:
            for src, log in pool.map(compile_one, jobs):
                if verbose:
                    print(f"[build] {os.path.basename(src)}\n{log}")
    if force or jobs or _stale(LIB_PATH, objs):
        cmd = [nvcc, "-shared", "-o", LIB_PATH] + objs + ["-lcudart"]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("link failed:\n" + res.stdout + res.stderr)
    return LIB_PATH


if __name__ == "__main__":
    path = build(verbose="-v" in sys.argv, force="-f" in sys.argv)
    print(path)
