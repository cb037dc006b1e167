"""Drop-in replacement for the reference's top-level ``GCN`` module (import name fixed by ``Main.py:5``).

Exports ``GCN`` (reference ``GCN.py:7-46``) and ``Adj_Preprocessor`` (reference ``GCN.py:50-135``) with the
reference's signatures; the arithmetic runs in ``libstmgcn_b200.so`` (hand-written sm_90a CUDA, C ABI in
``include/stmgcn_b200.h``).  Implementation: ``st-mgcn_b200/stmgcn_b200/{modules,preprocess}.py``.
"""
import os as _os
import sys as _sys

_PKG_ROOT = _os.path.join(_os.path.dirname(_os.path.abspath(__file__)), "st-mgcn_b200")
if _PKG_ROOT not in _sys.path:
    _sys.path.insert(0, _PKG_ROOT)

from stmgcn_b200.modules import GCN                      # noqa: E402,F401
from stmgcn_b200.preprocess import Adj_Preprocessor      # noqa: E402,F401

__all__ = ["GCN", "Adj_Preprocessor"]
