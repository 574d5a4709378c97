"""Register and spill budgets of the kernels compiled for sm_90a exactly as audioflux_b200/csrc/Makefile compiles them
(its own nvcc line, per-file flags such as -fmad=false included, plus -Xptxas -v).  Runs wherever nvcc is present; no
GPU needed."""
import collections
import importlib.util
import os
import shlex
import shutil
import subprocess
import tempfile

import pytest

from conftest import ROOT

CSRC = os.path.join(ROOT, "audioflux_b200", "csrc")
Budget = collections.namedtuple("Budget", "source labels max_registers max_spill max_stack")

# labels: a piece of each instantiation's mangled name -> its label; every label must be compiled exactly once.
# max_spill bounds the spill stores and the spill loads, each in bytes.
BUDGETS = [
    Budget("cepstrogram.cu", {"k_cepstrogramILb0": "clips", "k_cepstrogramILb1": "planes"}, None, 0, None),
    Budget("hpss.cu", {"k_hpss_mask": "mask"}, None, 0, 0),
    Budget("nsgt.cu", {"k_nsgt_bluestein": "bluestein", "k_nsgt_direct": "direct"}, None, 0, None),
    Budget("resample.cu", {"k_resampleILb1": "smem", "k_resampleILb0": "global"}, None, 0, None),
    Budget("st.cu", {"k_st_rowsILb0": "rows", "k_st_rowsILb1": "rows_inplace", "k_fst_segments": "segments",
                     "k_fst_expand": "expand"}, None, 0, None),
    # v2 at the 96-register cap of its 20 warps, with at most a few bytes of spills (per-tile values outside the
    # transforms); v1 uses the 128 registers of its 16 warps and spills nothing
    Budget("mfcc_fused2.cu", {f"k_mfcc_fused2ILi{ct}E": ct for ct in (2, 3, 5, 8)}, 96, 16, None),
    Budget("mfcc_fused.cu", {f"k_mfcc_fusedILi{ct}E": ct for ct in (2, 3, 5, 8)}, 128, 0, None),
]


def _ptxas_entries():
    path = os.path.join(ROOT, "tools", "mfcc_sass_budget.py")
    spec = importlib.util.spec_from_file_location("mfcc_sass_budget", path)
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    return tool.ptxas_entries


def makefile_nvcc_line(source):
    """the Makefile's nvcc command for kernels/<source>, as a list of arguments (run it in audioflux_b200/csrc)"""
    out = subprocess.run(["make", "-n", "-B", "--no-print-directory", "-C", CSRC, f"build/{source}.o"],
                         capture_output=True, text=True, check=True).stdout
    lines = [ln for ln in out.splitlines() if f"-c kernels/{source}" in ln]
    assert len(lines) == 1, out
    return shlex.split(lines[0])


@pytest.mark.parametrize("budget", BUDGETS, ids=[b.source for b in BUDGETS])
def test_kernel_budget(budget):
    cmd = makefile_nvcc_line(budget.source)
    nvcc = shutil.which(cmd[0])
    if nvcc is None:
        pytest.skip(f"nvcc not found: {cmd[0]}")
    cmd[0] = nvcc
    with tempfile.TemporaryDirectory() as tmp:
        o = cmd.index("-o")
        cmd[o + 1] = os.path.join(tmp, budget.source + ".o")
        r = subprocess.run(cmd + ["-Xptxas", "-v"], cwd=CSRC, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    seen = collections.defaultdict(list)
    for entry, figures in _ptxas_entries()(r.stderr).items():
        for piece, label in budget.labels.items():
            if piece in entry:
                seen[label].append(figures)
    assert sorted(seen, key=str) == sorted(set(budget.labels.values()), key=str), r.stderr
    for label, figures in seen.items():
        assert len(figures) == 1, (label, figures)
        regs, stack, st, ld = figures[0]
        if budget.max_registers is not None:
            assert regs <= budget.max_registers, (label, regs)
        assert st <= budget.max_spill and ld <= budget.max_spill, (label, st, ld)
        if budget.max_stack is not None:
            assert stack <= budget.max_stack, (label, stack)
