"""Register budget of the resampler kernel: both instantiations of k_resample (table in shared memory, table in global
memory) compiled for sm_90a as the Makefile compiles them (-fmad=false) spill nothing.  Runs wherever nvcc is present;
no GPU needed."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.realpath(__file__)))
SRC = os.path.join(ROOT, "audioflux_b200", "csrc", "kernels", "resample.cu")


def _nvcc():
    for p in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if p and os.path.exists(p):
            return p
    return None


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not found")
def test_resample_kernel_does_not_spill():
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false",
                            "-Xptxas", "-v", "-c", SRC, "-o", os.path.join(tmp, "resample.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    seen = {}
    kernel = None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            name = m.group(1)
            kernel = "smem" if "k_resampleILb1" in name else "global" if "k_resampleILb0" in name else None
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and kernel:
            seen[kernel] = (int(m.group(1)), int(m.group(2)))
    assert sorted(seen) == ["global", "smem"], r.stderr
    assert all(v == (0, 0) for v in seen.values()), seen
