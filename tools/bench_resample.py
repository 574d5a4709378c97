"""Resampler throughput on the device (device-resident seeded clips of 5 s at the source rate, 1024 per call,
CUDA-event timing, median of the timed calls after warm-up):

  best_48k_16k   Best quality, 48 000 -> 16 000
  mid_48k_16k    Mid quality,  48 000 -> 16 000
  fast_48k_16k   Fast quality, 48 000 -> 16 000
  best_44k_16k   Best quality, 44 100 -> 16 000
  best_16k_48k   Best quality, 16 000 -> 48 000

Per workload: ms per call, the kernel's own time (torch.profiler, a separate run), output samples and taps per second
(taps counted with the reference's tap-count rule), the compulsory HBM bytes (clips in, outputs out) over kernel time and
their share of 3.35 TB/s, a parity gate on clip 0 against the float64 oracle, the card's name, power limit and max SM
clock, and where oracle/_ref exists the reference build's time per clip on one CPU core.  Prints one JSON line per
workload.

    python tools/bench_resample.py [--steps 20] [--warmup 3] [--workloads best_48k_16k,...] [--out results.json]"""
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
import _resample_oracle as RO  # noqa: E402

HBM = 3.35e12
CLIPS = 1024
WORKLOADS = {
    "best_48k_16k": dict(qual=0, src=48000, dst=16000),
    "mid_48k_16k": dict(qual=1, src=48000, dst=16000),
    "fast_48k_16k": dict(qual=2, src=48000, dst=16000),
    "best_44k_16k": dict(qual=0, src=44100, dst=16000),
    "best_16k_48k": dict(qual=0, src=16000, dst=48000),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name()


def kernel_times(fn, calls=3):
    """device ms per launch of each kernel, from torch.profiler (one launch per call)"""
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
        key = "k_resample" if "k_resample" in e.key else e.key[:60]
        per[key] = per.get(key, 0) + us / 1e3 / max(e.count, 1)      # per launch: the profiler may drop a call
    return per


def reference_ms_per_clip(w, x, clips=2):
    from oracle import ref_lib as R
    if not R.available():
        return None
    lib = R.get_ref_lib()
    t0 = time.perf_counter()
    for i in range(clips):                 # construction included, as a user pays it
        st, o = RO.c_new(lib, w["qual"])
        lib.resampleObj_setSamplate(o, w["src"], w["dst"])
        RO.c_resample(lib, o, x[i])
        lib.resampleObj_free(o)
    return (time.perf_counter() - t0) * 1e3 / clips


def run(name, steps, warmup):
    w = WORKLOADS[name]
    length = 5 * w["src"]
    obj = af.Resample(af.ResampleQualityType(w["qual"]))
    obj.set_samplate(w["src"], w["dst"])
    m = obj.cal_data_length(length)
    rng = np.random.default_rng(0)
    x = (0.1 * rng.standard_normal((CLIPS, length))).astype(np.float32)
    x[0] = RO.case_signal(name, dict(length=length))
    xd = torch.from_numpy(x).cuda()

    def fn():
        return obj.resample_batch(xd)
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
    o = RO.Resampler(w["qual"])
    o.set_samplate(w["src"], w["dst"])
    want = o.resample(x[0])
    got = out[0].cpu().numpy()
    err = float(np.abs(got - want).max() / np.abs(want).max())
    del out
    per = kernel_times(fn)
    taps = int(o.taps(length).sum()) * CLIPS
    nbytes = CLIPS * (length + m) * 4
    res = dict(workload=name, clips=CLIPS, samples=length, outputs=m, quality=w["qual"], rates=[w["src"], w["dst"]],
               ms_per_call=round(ms, 4), ms_min=round(float(np.min(times)), 4), ms_max=round(float(np.max(times)), 4),
               kernels_ms={k: round(v, 4) for k, v in per.items()},
               taps_per_output=round(taps / (CLIPS * m), 2),
               outputs_per_s=round(CLIPS * m / (ms * 1e-3), 1), taps_per_s=round(taps / (ms * 1e-3), 1),
               compulsory_bytes=nbytes, parity_clip0=err, parity_ok=bool(err <= 1e-4), card=card())
    k = per.get("k_resample")
    if k:
        res["k_resample_hbm_share"] = round(nbytes / (k * 1e-3) / HBM, 4)
        res["k_resample_taps_per_s"] = round(taps / (k * 1e-3), 1)
    res["reference_ms_per_clip_1core"] = reference_ms_per_clip(w, x)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_resample needs a CUDA device")
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
