"""ST / FST throughput on the device (device-resident clips, CUDA-event timing, median of the timed calls after warm-up):

  st12   ST  at 2^12, rows 1 .. 2047, 128 clips   (8.6 GB of output planes per call)
  fst12  FST at 2^12, rows 1 .. 2047, 128 clips   (the same output: a pure store stream after two small kernels)
  st14   ST  at 2^14, rows 1000 .. 1063, 128 clips (the in-place shared-memory path)

Per workload: ms per call, the kernels' own times (torch.profiler, a separate run), compulsory bytes (clips in, planes
out) and their share of 3.35 TB/s, for ST the FP32 rate of the inverse FFTs (5 N log2 N per row), a parity gate on
clip 0 against the float64 oracle, the card's name, power limit and max SM clock, and where oracle/_ref exists the
reference build's time per clip on one CPU core.  Prints one JSON line per workload.

    python tools/bench_st.py [--steps 20] [--warmup 3] [--workloads st12,fst12,st14] [--out results.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.realpath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import audioflux_b200 as af  # noqa: E402
import _st_oracle as SO  # noqa: E402

HBM = 3.35e12
WORKLOADS = {
    "st12": dict(kind="st", radix2_exp=12, lo=1, hi=2047, batch=128),
    "fst12": dict(kind="fst", radix2_exp=12, lo=1, hi=2047, batch=128),
    "st14": dict(kind="st", radix2_exp=14, lo=1000, hi=1063, batch=128),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name()


def kernel_times(fn, xd, calls=3):
    """device ms per call of each kernel, from torch.profiler"""
    from torch.profiler import profile, ProfilerActivity
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn(xd)
        torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if us <= 0 or e.key.startswith(("Memcpy", "Memset", "cuda")):
            continue
        key = next((k for k in ("k_st_rows", "k_fst_segments", "k_fst_expand", "k_stft_generic") if k in e.key), e.key[:60])
        per[key] = per.get(key, 0) + us / 1e3 / calls
    return per


def reference_ms_per_clip(w, x, clips=2):
    from oracle import ref_lib as R
    if not R.available():
        return None
    lib = R.get_ref_lib()
    t0 = time.perf_counter()
    for i in range(clips):
        kw = dict(radix2_exp=w["radix2_exp"], min_index=w["lo"], max_index=w["hi"])
        (SO.c_st_case if w["kind"] == "st" else SO.c_fst_case)(lib, kw, x[i])   # construction included, as a user pays it
    return (time.perf_counter() - t0) * 1e3 / clips


def run(name, steps, warmup):
    w = WORKLOADS[name]
    r, B = w["radix2_exp"], w["batch"]
    n, rows = 1 << r, w["hi"] - w["lo"] + 1
    if w["kind"] == "st":
        obj = af.ST(radix2_exp=r, min_index=w["lo"], max_index=w["hi"])
        fn = obj.st_batch
    else:
        obj = af.FST(radix2_exp=r, min_index=w["lo"], max_index=w["hi"])
        fn = obj.fst_batch
    rng = np.random.default_rng(0)
    x = (0.1 * rng.standard_normal((B, n))).astype(np.float32)
    x[0] = SO.case_signal(1, n)
    xd = torch.from_numpy(x).cuda()
    for _ in range(warmup):
        out = fn(xd)
    del out
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(steps):
        e0.record()
        re, im = fn(xd)
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
        if len(times) < steps:
            del re, im
    ms = float(np.median(times))
    want = SO.st(x[0], list(range(w["lo"], w["hi"] + 1))) if w["kind"] == "st" else SO.fst(x[0], w["lo"], w["hi"])
    err, _ = SO.row_errors(re[0].cpu().numpy(), im[0].cpu().numpy(), want)
    del re, im
    per = kernel_times(fn, xd)
    nbytes = B * n * 4 + B * rows * n * 8
    res = dict(workload=name, kind=w["kind"], clips=B, samples=n, rows=rows,
               ms_per_call=round(ms, 4), ms_min=round(float(np.min(times)), 4), ms_max=round(float(np.max(times)), 4),
               kernels_ms={k: round(v, 4) for k, v in per.items()},
               compulsory_bytes=nbytes, hbm_share=round(nbytes / (ms * 1e-3) / HBM, 4),
               parity_worst_row_clip0=float(err.max()), parity_ok=bool(err.max() <= 1e-4), card=card())
    if w["kind"] == "st":
        flop = 5.0 * n * r * rows * B
        res["fft_tflops"] = round(flop / (ms * 1e-3) / 1e12, 3)
        k = per.get("k_st_rows")
        if k:
            res["k_st_rows_hbm_share"] = round(B * rows * n * 8 / (k * 1e-3) / HBM, 4)
            res["k_st_rows_tflops"] = round(flop / (k * 1e-3) / 1e12, 3)
    else:
        k = per.get("k_fst_expand")
        if k:
            res["k_fst_expand_hbm_share"] = round(B * rows * n * 8 / (k * 1e-3) / HBM, 4)
    res["reference_ms_per_clip_1core"] = reference_ms_per_clip(w, x)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workloads", default="st12,fst12,st14")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_st needs a CUDA device")
    results = []
    for wname in a.workloads.split(","):
        results.append(run(wname, a.steps, a.warmup))
        print(json.dumps(results[-1]), flush=True)
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)
    if not all(r["parity_ok"] for r in results):
        sys.exit("parity gate failed")


if __name__ == "__main__":
    main()
