"""Register and spill budgets of the kernels compiled for sm_90a exactly as audioflux_b200/csrc/Makefile compiles them
(its own nvcc line, per-file flags such as -fmad=false included, plus -Xptxas -v), and the flags that line must carry.
Runs wherever nvcc is present; no GPU needed."""
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
Budget = collections.namedtuple("Budget", "source labels max_registers max_spill max_stack flags", defaults=((),))

# labels: a piece of each instantiation's mangled name -> its label; every label must be compiled exactly once.  Where
# one kernel's name is a prefix of another's, the piece carries the name's length prefix (7k_xcorr, not k_xcorr_pad).
# max_registers: one cap for every label, or {label: cap} for each of them.  max_spill bounds the spill stores and the
# spill loads, each in bytes.  flags: arguments the Makefile's nvcc line for the source must carry.
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
    Budget("onset.cu", {k: k for k in ("k_onset_maxfilter", "k_onset_pick")}, None, 0, 0),
    # CTAs of 1024 threads, and two of k_harmonic_ratio's per SM
    Budget("harmonic_ratio.cu", {"16k_harmonic_ratio": "k_harmonic_ratio",
                                 "22k_harmonic_ratio_carry": "k_harmonic_ratio_carry"},
           {"k_harmonic_ratio": 32, "k_harmonic_ratio_carry": 64}, 0, 0, ("-fmad=false",)),
    Budget("wavelet.cu", {k: k for k in ("k_wavelet_level", "k_wavelet_expand", "k_swt_level")}, 64, 0, 0),
    # 256-thread CTAs: two per SM at least
    Budget("nmf.cu", {k: k for k in ("k_nmf_d", "k_nmf_h", "k_nmf_w", "k_nmf_norm")}, 96, 0, 0, ("-fmad=false",)),
    # the one-CTA-per-row kernels fit 1024 threads
    Budget("xcorr.cu", {"7k_xcorr": "k_xcorr", "k_xcorr_pad": "k_xcorr_pad", "k_xcorr_cross": "k_xcorr_cross",
                        "k_xcorr_finish": "k_xcorr_finish", "k_xcorr_argmax": "k_xcorr_argmax"}, 64, 0, 0,
           ("-fmad=false",)),
    Budget("czt.cu", {"5k_czt": "k_czt", "k_czt_filter": "k_czt_filter"}, 64, 0, 0, ("-fmad=false",)),
    # CTAs of up to 1024 threads, two per SM at n = 2^12: at most 32 registers
    Budget("pitch_pef.cu", {"k_pitch_pef": "k_pitch_pef"}, 32, 0, 0, ("-fmad=false",)),
    # CTAs of up to 1024 threads; the launcher sizes them for 1536 threads per SM (65 536 registers / 40, rounded down)
    Budget("pitch_yin.cu", {"k_pitch_yin": "k_pitch_yin"}, 40, 0, 0, ("-fmad=false",)),
    # CTAs of up to 1024 threads; the launcher sizes them for 2048 threads per SM (65 536 registers / 32)
    Budget("pitch_ncf_cep.cu", {"k_pitch_ncf": "k_pitch_ncf", "k_pitch_cep": "k_pitch_cep"}, 32, 0, 0, ("-fmad=false",)),
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
    missing = [f for f in budget.flags if f not in cmd]
    assert not missing, (budget.source, "the Makefile's nvcc line lacks", missing)
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
        cap = budget.max_registers[label] if isinstance(budget.max_registers, dict) else budget.max_registers
        if cap is not None:
            assert regs <= cap, (label, regs)
        assert st <= budget.max_spill and ld <= budget.max_spill, (label, st, ld)
        if budget.max_stack is not None:
            assert stack <= budget.max_stack, (label, stack)
