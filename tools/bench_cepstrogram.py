"""Cepstrogram throughput on the device (device-resident clips, CUDA-event timing, median of the timed calls after
warm-up):

  c12   N = 2^12, 1024 clips x 160 000 samples (5 s at 32 kHz), slide 1024, cepNum 4, all three outputs
  c10   N = 2^10, 1024 clips x  80 000 samples (5 s at 16 kHz), slide  256, cepNum 20, all three outputs
  c14   N = 2^14,  256 clips x 441 000 samples,                 slide 4096, cepNum 128, all three outputs

Per workload: ms per call, the kernel's own time (torch.profiler, a separate run), compulsory bytes (clips in, requested
planes out) and their share of 3.35 TB/s, the FP32 rate counting 2.5 N log2 N flops per real N-point transform (four
per frame: forward, cepstrum, envelope, details), a parity gate on clip 0 against the float64 oracle, the card's name,
power limit and max SM clock, and where oracle/_ref exists the reference build's time per clip on one CPU core.
Prints one JSON line per workload.

    python tools/bench_cepstrogram.py [--steps 20] [--warmup 3] [--workloads c12,c10,c14] [--out results.json]"""
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
import _cepstrogram_oracle as CO  # noqa: E402

HBM = 3.35e12
WORKLOADS = {
    "c12": dict(radix2_exp=12, clips=1024, length=160000, slide=1024, cep_num=4),
    "c10": dict(radix2_exp=10, clips=1024, length=80000, slide=256, cep_num=20),
    "c14": dict(radix2_exp=14, clips=256, length=441000, slide=4096, cep_num=128),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name()


def kernel_times(fn, calls=3):
    """device ms per call of each kernel, from torch.profiler"""
    from torch.profiler import profile, ProfilerActivity
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if us <= 0 or e.key.startswith(("Memcpy", "Memset", "cuda")):
            continue
        key = "k_cepstrogram" if "k_cepstrogram" in e.key else e.key[:60]
        per[key] = per.get(key, 0) + us / 1e3 / calls
    return per


def reference_ms_per_clip(w, x, clips=2):
    from oracle import ref_lib as R
    if not R.available():
        return None
    lib = R.get_ref_lib()
    kw = dict(radix2_exp=w["radix2_exp"], window_type=CO.W_RECT, slide=w["slide"], cep_num=w["cep_num"])
    t0 = time.perf_counter()
    for i in range(clips):
        CO.c_case(lib, kw, x[i])          # construction included, as a user pays it
    return (time.perf_counter() - t0) * 1e3 / clips


def run(name, steps, warmup):
    w = WORKLOADS[name]
    r, B, length, c = w["radix2_exp"], w["clips"], w["length"], w["cep_num"]
    n = 1 << r
    obj = af.Cepstrogram(radix2_exp=r, slide_length=w["slide"])
    T = obj.cal_time_length(length)
    rng = np.random.default_rng(0)
    x = (0.1 * rng.standard_normal((B, length))).astype(np.float32)
    x[0] = CO.signal(1, length)
    xd = torch.from_numpy(x).cuda()

    def fn():
        return obj.cepstrogram_batch(xd, c)
    for _ in range(warmup):
        out = fn()
    del out
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(steps):
        e0.record()
        out = fn()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
        if len(times) < steps:
            del out
    ms = float(np.median(times))
    *want, logs = CO.cepstrogram(x[0], n, w["slide"], CO.W_RECT, c)
    err = max(float(CO.frame_errors(o[0].cpu().numpy(), wt, logs).max()) for o, wt in zip(out, want))
    del out
    per = kernel_times(fn)
    nbytes = B * length * 4 + 3 * B * T * (n // 2 + 1) * 4
    flop = 4 * 2.5 * n * r * T * B
    res = dict(workload=name, clips=B, samples=length, fft_length=n, slide=w["slide"], cep_num=c, frames=T * B,
               ms_per_call=round(ms, 4), ms_min=round(float(np.min(times)), 4), ms_max=round(float(np.max(times)), 4),
               kernels_ms={k: round(v, 4) for k, v in per.items()},
               compulsory_bytes=nbytes, hbm_share=round(nbytes / (ms * 1e-3) / HBM, 4),
               fft_tflops=round(flop / (ms * 1e-3) / 1e12, 3),
               parity_worst_frame_clip0=err, parity_ok=bool(err <= 1e-4), card=card())
    k = per.get("k_cepstrogram")
    if k:
        res["k_cepstrogram_hbm_share"] = round(nbytes / (k * 1e-3) / HBM, 4)
        res["k_cepstrogram_tflops"] = round(flop / (k * 1e-3) / 1e12, 3)
    res["reference_ms_per_clip_1core"] = reference_ms_per_clip(w, x)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workloads", default="c12,c10,c14")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_cepstrogram needs a CUDA device")
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
