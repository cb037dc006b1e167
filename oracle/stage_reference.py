"""Build the reference artifacts under ``oracle/_ref/`` (git-ignored; called by ``__graft_entry__.build()``).

TEST INFRASTRUCTURE.  The reference (``underdoc-wang/ST-MGCN``) is pure Python, so its build product is byte code: each
of its modules is compiled, unmodified, to a sourceless ``oracle/_ref/<name>.pyc`` for the running interpreter (the one
the tests and ``bench.py`` use), next to the reference's ``LICENSE``.  Two consumers, both optional -- they skip or fall
back when the directory is absent:

* ``tests/test_gpu_dropin_main.py`` runs the reference's own ``Main.py`` / ``Model_Trainer.py`` / ``Data_Container.py``
  against this repository's ``GCN`` / ``STMGCN`` modules;
* ``bench.py``'s CPU baseline times the reference's own ``GCN`` / ``STMGCN`` modules (``kind: "reference"``).

Where the reference checkout is: ``$STMGCN_REFERENCE_DIR``, else a ``reference`` directory next to this repository's
root, else ``/root/reference``.  Without one nothing is built and an existing ``oracle/_ref/`` is left as it is.

    python oracle/stage_reference.py [/path/to/reference]
"""
from __future__ import annotations

import os
import py_compile
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
REF_DST = os.path.join(HERE, "_ref")
MODULES = ("GCN", "STMGCN", "Model_Trainer", "Main", "Data_Container")


def find_reference(explicit: str | None = None) -> str | None:
    for cand in (explicit, os.environ.get("STMGCN_REFERENCE_DIR"), os.path.join(os.path.dirname(REPO), "reference"),
                 "/root/reference"):
        if cand and all(os.path.exists(os.path.join(cand, m + ".py")) for m in MODULES):
            return os.path.abspath(cand)
    return None


def stage(explicit: str | None = None) -> bool:
    """Compile the reference modules into ``oracle/_ref/``; True when the directory holds a complete set afterwards."""
    src = find_reference(explicit)
    if src is not None:
        os.makedirs(REF_DST, exist_ok=True)
        for m in MODULES:
            py_compile.compile(os.path.join(src, m + ".py"), cfile=os.path.join(REF_DST, m + ".pyc"), doraise=True,
                               invalidation_mode=py_compile.PycInvalidationMode.UNCHECKED_HASH)
        if os.path.exists(os.path.join(src, "LICENSE")):
            shutil.copyfile(os.path.join(src, "LICENSE"), os.path.join(REF_DST, "LICENSE"))
        print(f"[build] reference modules compiled -> {REF_DST}")
    return staged()


def staged() -> bool:
    return all(os.path.exists(os.path.join(REF_DST, m + ".pyc")) for m in MODULES)


if __name__ == "__main__":
    ok = stage(sys.argv[1] if len(sys.argv) > 1 else None)
    sys.exit(0 if ok else 1)
