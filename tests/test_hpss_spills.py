"""Register budget of the HPSS mask kernel: k_hpss_mask compiled for sm_90a as the Makefile compiles it (-fmad=false)
spills nothing.  Runs wherever nvcc is present; no GPU needed."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.realpath(__file__)))
SRC = os.path.join(ROOT, "audioflux_b200", "csrc", "kernels", "hpss.cu")


def _nvcc():
    for p in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if p and os.path.exists(p):
            return p
    return None


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not found")
def test_hpss_kernel_does_not_spill():
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false",
                            "-Xptxas", "-v", "-c", SRC, "-o", os.path.join(tmp, "hpss.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    seen = {}
    kernel = None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            kernel = m.group(1) if "k_hpss_mask" in m.group(1) else None
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and kernel:
            seen[kernel] = tuple(int(v) for v in m.groups())
    assert len(seen) == 1, r.stderr
    assert all(v == (0, 0, 0) for v in seen.values()), seen
