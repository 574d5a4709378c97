#!/usr/bin/env python3
"""Static instruction budget of k_mfcc_fused2 per warp role, from the compiler output (no GPU needed).

Cross-compiles kernels/mfcc_fused2.cu for sm_90a with line info, disassembles it (nvdisasm -gi) and attributes every
SASS instruction to the line of mfcc_fused2.cu it was inlined into.  The roles are the kernel's own sections (producer,
bank warps, DCT warps, frame warps); the frame warps' `Mag` branch (|X| instead of |X|^2) is counted apart, so
"frame power path" is what a frame of the default power spectrum executes.  Also prints ptxas' register / spill report.
These are static counts of the fully unrolled code, not measurements on a device.

    python3 tools/mfcc_sass_budget.py [--ct 5] [--src path/to/mfcc_fused2.cu]
"""
import argparse
import collections
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.realpath(__file__)))
SRC = os.path.join(ROOT, "audioflux_b200", "csrc", "kernels", "mfcc_fused2.cu")
CLASSES = ("FADD", "FMUL", "FFMA", "LDS", "STS", "LDL", "STL")


def nvcc_path():
    for p in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if p and os.path.exists(p):
            return p
    return None


def compile_cubin(src, nvcc, out_dir):
    cubin = os.path.join(out_dir, os.path.splitext(os.path.basename(src))[0] + ".cubin")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-cubin",
                        "-Xptxas", "-v", "-o", cubin, src], capture_output=True, text=True, check=True)
    return cubin, r.stderr


def ptxas_entries(log):
    """{entry function: (registers, stack frame bytes, spill store bytes, spill load bytes)} from a -Xptxas -v log."""
    rep, entry, props = {}, None, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            entry = m.group(1)
            rep[entry] = [0, 0, 0, 0]
            continue
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            props = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and props in rep:
            rep[props][1:] = [int(v) for v in m.groups()]
        m = re.search(r"Used (\d+) registers", line)
        if m and entry is not None:
            rep[entry][0] = int(m.group(1))
    return {k: tuple(v) for k, v in rep.items()}


def ptxas_report(log, kernel="k_mfcc_fused2"):
    """{CT: (registers, spill store bytes, spill load bytes)} of kernel<CT> from the -Xptxas -v log."""
    rep = {}
    for name, (regs, _, st, ld) in ptxas_entries(log).items():
        m = re.search(kernel + r"ILi(\d+)E", name)
        if m:
            rep[int(m.group(1))] = (regs, st, ld)
    return rep


def role_ranges(src):
    """Source line ranges (1-based, inclusive) of the kernel's sections, found by their banner comments."""
    lines = open(src).read().splitlines()

    def find(pat, start=0):
        for i in range(start, len(lines)):
            if pat in lines[i]:
                return i + 1
        raise SystemExit(f"marker {pat!r} not found in {src}")

    prod = find("================= producer")
    bank = find("================= bank warps")
    dct = find("================= DCT warps")
    frame = find("================= frame warps")
    end = find("void free_plan", frame)
    mag0 = find("p.dataType == SpectralData_Mag", frame)
    mag1 = find("} else {", mag0)
    return [("prologue", 1, prod - 1), ("producer", prod, bank - 1), ("bank", bank, dct - 1), ("dct", dct, frame - 1),
            ("frame Mag branch", mag0 + 1, mag1 - 1), ("frame power path", frame, end - 1)]


def count(sass, ranges, ct):
    """Per role: Counter of instruction classes (+ 'FP32' and 'total') of the instantiation k_mfcc_fused2<ct>."""
    base = os.path.basename(SRC)
    cur_kernel, line = None, None
    per = collections.defaultdict(collections.Counter)
    block = []
    for raw in sass.splitlines():
        s = raw.strip()
        if s.startswith(".text."):
            m = re.search(r"k_mfcc_fused2ILi(\d+)E", s)
            cur_kernel = int(m.group(1)) if m else None
            line = None
            continue
        if s.startswith("//##"):
            block.append(s)
            continue
        if block:
            hits = re.findall(re.escape(base) + r'", line (\d+)', " ".join(block))
            line = int(hits[-1]) if hits else line
            block = []
        m = re.match(r"/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_]*)(\.[A-Z0-9_.]+)?", s)
        if not m or cur_kernel != ct or line is None:
            continue
        op = m.group(1)
        role = None
        for name, a, b in ranges:      # the Mag branch lies inside the frame section: checked first
            if a <= line <= b:
                role = name
                break
        if role is None:
            continue
        c = per[role]
        c["total"] += 1
        if op in CLASSES:
            c[op] += 1
        if op in ("FADD", "FMUL", "FFMA"):
            c["FP32"] += 1
    return per


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--ct", type=int, default=5, help="instantiation k_mfcc_fused2<CT> (bench: 5)")
    ap.add_argument("--src", default=SRC)
    args = ap.parse_args()
    nvcc = nvcc_path()
    if not nvcc:
        sys.exit("nvcc not found")
    nvdisasm = os.path.join(os.path.dirname(nvcc), "nvdisasm")
    with tempfile.TemporaryDirectory() as tmp:
        cubin, log = compile_cubin(os.path.abspath(args.src), nvcc, tmp)
        sass = subprocess.run([nvdisasm, "-gi", "-c", cubin], capture_output=True, text=True, check=True).stdout
    per = count(sass, role_ranges(args.src), args.ct)
    cols = ("total", "FP32") + CLASSES
    print(f"k_mfcc_fused2<{args.ct}> static SASS instructions by role (fully unrolled loop bodies)")
    print("| role | " + " | ".join(cols) + " |")
    print("|---|" + "---|" * len(cols))
    for name, _, _ in role_ranges(args.src):
        print(f"| {name} | " + " | ".join(str(per[name][c]) for c in cols) + " |")
    print()
    for ct, (regs, st, ld) in sorted(ptxas_report(log).items()):
        print(f"k_mfcc_fused2<{ct}>: {regs} registers, {st} B spill stores, {ld} B spill loads")


if __name__ == "__main__":
    main()
