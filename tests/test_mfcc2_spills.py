"""Register budgets of the fused MFCC kernels compiled for sm_90a (CUDA 12.9, -Xptxas -v).  Runs wherever nvcc is
present; no GPU needed.
  * k_mfcc_fused2<2,3,5,8> (v2) stay at the 96-register cap of its 20 warps, with at most a few bytes of spills
    (per-tile values outside the transforms; the spills in the twiddle products and the power stores are gone).
  * k_mfcc_fused<2,3,5,8> (v1) use the 128 registers of its 16 warps and spill nothing."""
import os
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.realpath(__file__)))
KERNELS = os.path.join(ROOT, "audioflux_b200", "csrc", "kernels")
SRC = os.path.join(KERNELS, "mfcc_fused2.cu")
MAX_SPILL_BYTES = 16


def _nvcc():
    for p in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if p and os.path.exists(p):
            return p
    return None


def _report(src, kernel):
    import importlib.util
    spec = importlib.util.spec_from_file_location("mfcc_sass_budget", os.path.join(ROOT, "tools", "mfcc_sass_budget.py"))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    with tempfile.TemporaryDirectory() as tmp:
        _, log = tool.compile_cubin(src, _nvcc(), tmp)
    rep = tool.ptxas_report(log, kernel)
    assert sorted(rep) == [2, 3, 5, 8], log
    return rep


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not found")
def test_mfcc_fused2_registers_and_spills():
    for ct, (regs, st, ld) in _report(SRC, "k_mfcc_fused2").items():
        assert regs <= 96, (ct, regs)
        assert st <= MAX_SPILL_BYTES and ld <= MAX_SPILL_BYTES, (ct, st, ld)


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not found")
def test_mfcc_fused_registers_and_spills():
    for ct, (regs, st, ld) in _report(os.path.join(KERNELS, "mfcc_fused.cu"), "k_mfcc_fused").items():
        assert regs <= 128, (ct, regs)
        assert st == 0 and ld == 0, (ct, st, ld)
