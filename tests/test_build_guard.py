"""The build refuses objects in which ptxas serialised the wgmma instructions of a function (C7511 / C7512)."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "st-mgcn_b200"))

from stmgcn_b200 import build  # noqa: E402

_FN = "_ZN41_GLOBAL__N__f48d0a9f_9_lstm16_cu_ba2339df17lstm16_bwd_kernelILi2ELi0EEEvNS_11Bwd16ParamsE"


def test_serialised_wgmma_diagnostics_name_the_function():
    log = (
        "ptxas info    : (C7511) Potential Performance Loss: wgmma.mma_async instructions are serialized due to "
        f"insufficient register resources for the wgmma pipeline in the function '{_FN}'\n"
        "ptxas info    : (C7512) Potential Performance Loss: wgmma.mma_async instructions are serialized due to "
        "insufficient register resources for the function '_Z3foov'\n"
        f"ptxas info    : Compiling entry function '{_FN}' for 'sm_90a'\n"
        "ptxas info    : Used 168 registers, used 16 barriers\n"
    )
    assert build._SERIALIZED_WGMMA.findall(log) == [_FN, "_Z3foov"]


def test_clean_ptxas_log_passes():
    log = (
        f"ptxas info    : Compiling entry function '{_FN}' for 'sm_90a'\n"
        "ptxas info    : Function properties for x\n    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n"
    )
    assert build._SERIALIZED_WGMMA.findall(log) == []
