"""NSGT throughput on the device, two workloads (device-resident clips, CUDA-event timing after warm-up):

  (a) 1024 clips x 2^15 samples at 32 kHz, Octave 84, 12 bins per octave, Slaney, BandWidth (the reference class's
      defaults at the length of its docs example)
  (b) 64 clips x 2^19 samples at 44.1 kHz, Octave 84 (widest band 5587 points: the direct path runs)

Per workload: ms per call, split into the forward FFT and the band kernels (torch.profiler, a separate run), compulsory
bytes (clips in, matrix out) and their share of 3.35 TB/s, a parity gate against the oracle on clip 0, and for (a) the
reference build's time per clip on one CPU core when oracle/_ref exists.  Prints one JSON line per workload.

    python tools/bench_nsgt.py [--steps 20] [--warmup 3] [--out results.json]"""
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
import _nsgt_oracle as NO  # noqa: E402
from oracle import af_oracle as O  # noqa: E402

HBM = 3.35e12
WORKLOADS = {
    "a": dict(batch=1024, radix2_exp=15, samplate=32000),
    "b": dict(batch=64, radix2_exp=19, samplate=44100),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name()


def split_times(t, xd, calls=3):
    """device time per call of the forward FFT kernels and of the band kernels (k_nsgt_*), from torch.profiler"""
    from torch.profiler import profile, ProfilerActivity
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            t.nsgt_batch(xd)
        torch.cuda.synchronize()
    fwd = band = 0.0
    per = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if us <= 0 or e.key.startswith(("Memcpy", "Memset", "cuda")):
            continue
        per[e.key] = per.get(e.key, 0) + us / 1e3 / calls
        if "k_nsgt_" in e.key:
            band += us / 1e3 / calls
        else:
            fwd += us / 1e3 / calls
    return fwd, band, per


def reference_ms_per_clip(kw, x, clips=5):
    from oracle import ref_lib as R
    if not R.available():
        return None
    lib = R.get_ref_lib()
    st, obj = NO.c_new(lib, **kw)
    if st != 0:
        return None
    NO.c_nsgt(lib, obj, x[0], kw["num"])          # builds nothing new, but touches the matrices once
    t0 = time.perf_counter()
    for i in range(clips):
        NO.c_nsgt(lib, obj, x[i % len(x)], kw["num"])
    ms = (time.perf_counter() - t0) * 1e3 / clips
    lib.nsgtObj_free(obj)
    return ms


def run(name, steps, warmup):
    w = WORKLOADS[name]
    kw = dict(num=84, radix2_exp=w["radix2_exp"], samplate=w["samplate"], low_fre=32.703196, bin_per_octave=12,
              scale_type=O.SCALE_OCTAVE, style_type=O.STYLE_SLANEY, normal_type=O.NORM_BANDWIDTH)
    t = af.NSGT(num=84, radix2_exp=w["radix2_exp"], samplate=w["samplate"], bin_per_octave=12)
    n, B = 1 << w["radix2_exp"], w["batch"]
    rng = np.random.default_rng(0)
    x = (0.1 * rng.standard_normal((B, n))).astype(np.float32)
    x[0] = NO.case_signal(1, n, w["samplate"])
    xd = torch.from_numpy(x).cuda()
    for _ in range(warmup):
        t.nsgt_batch(xd)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(steps):
        e0.record()
        re, im = t.nsgt_batch(xd)
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    ms = float(np.median(times))
    _, p = NO.params(**kw)
    _, m = NO.transform(x[0], p)
    r0, i0 = re[0].cpu().numpy(), im[0].cpu().numpy()
    err = max(np.abs(r0 - m.real).max() / np.abs(m.real).max(), np.abs(i0 - m.imag).max() / np.abs(m.imag).max())
    fwd, band, per = split_times(t, xd)
    T = t.get_max_time_length()
    nbytes = B * n * 4 + B * 84 * T * 8
    res = dict(workload=name, clips=B, samples=n, samplate=w["samplate"], max_len=T,
               total_len=t.get_total_time_length(), widest=int(t.get_time_length_arr().max()),
               ms_per_call=round(ms, 4), ms_min=round(float(np.min(times)), 4), ms_max=round(float(np.max(times)), 4),
               ms_forward_fft=round(fwd, 4), ms_band_kernels=round(band, 4),
               kernels_ms={k: round(v, 4) for k, v in per.items()},
               compulsory_bytes=nbytes, hbm_share=round(nbytes / (ms * 1e-3) / HBM, 4),
               parity_rel_err_clip0=float(err), parity_ok=bool(err <= 1e-4), card=card())
    if name == "a":
        res["reference_ms_per_clip_1core"] = reference_ms_per_clip(kw, x)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workloads", default="ab")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_nsgt needs a CUDA device")
    results = [run(w, a.steps, a.warmup) for w in a.workloads]
    for r in results:
        print(json.dumps(r))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)
    if not all(r["parity_ok"] for r in results):
        sys.exit("parity gate failed")


if __name__ == "__main__":
    main()
