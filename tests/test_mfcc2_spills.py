"""Register budget of the fused MFCC kernel: k_mfcc_fused2<2,3,5,8> compiled for sm_90a stay at the 96-register cap of
its 20 warps, with at most a few bytes of spills (per-tile values outside the transforms; the spills in the twiddle
products and the power stores are gone).  Runs wherever nvcc is present; no GPU needed."""
import os
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.realpath(__file__)))
SRC = os.path.join(ROOT, "audioflux_b200", "csrc", "kernels", "mfcc_fused2.cu")
MAX_SPILL_BYTES = 16


def _nvcc():
    for p in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if p and os.path.exists(p):
            return p
    return None


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not found")
def test_mfcc_fused2_registers_and_spills():
    import importlib.util
    spec = importlib.util.spec_from_file_location("mfcc_sass_budget", os.path.join(ROOT, "tools", "mfcc_sass_budget.py"))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    with tempfile.TemporaryDirectory() as tmp:
        _, log = tool.compile_cubin(SRC, _nvcc(), tmp)
    rep = tool.ptxas_report(log)
    assert sorted(rep) == [2, 3, 5, 8], log
    for ct, (regs, st, ld) in rep.items():
        assert regs <= 96, (ct, regs)
        assert st <= MAX_SPILL_BYTES and ld <= MAX_SPILL_BYTES, (ct, st, ld)
