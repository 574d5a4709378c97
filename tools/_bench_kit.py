"""What the object benchmarks (tools/bench_<object>.py) share: the card line, per-kernel device times from
torch.profiler, the CUDA-event loop, the reference build's time per clip on one CPU core, and the command-line driver.
Nothing here changes a device or host setting; the card is only read."""
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

HBM = 3.35e12                # bytes/s: the H100 SXM data sheet's HBM3 bandwidth


def card():
    """"name, power limit, max SM clock" of the current device as nvidia-smi reports them (else the name alone)"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name()


def kernel_times(fn, kernels, calls=3, per_launch=False):
    """device ms of each kernel per call of fn (per launch with per_launch), from torch.profiler over `calls` calls.
    A kernel whose name contains one of `kernels` is reported under that name, any other under its own; copies,
    memsets and runtime calls are left out."""
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
        key = next((k for k in kernels if k in e.key), e.key)
        per[key] = per.get(key, 0) + us / 1e3 / (max(e.count, 1) if per_launch else calls)
    return per


def event_times(fn, steps, warmup):
    """`warmup` untimed calls of fn, then `steps` calls each timed with CUDA events -> (ms of each, the last output).
    Each output is dropped before the next call, so that two never share the device."""
    out = None
    for _ in range(warmup):
        out = fn()
    out = None
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(steps):
        out = None
        e0.record()
        out = fn()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    return times, out


def ms_stats(times, digits):
    """ms_per_call (the median), ms_min and ms_max of event_times"""
    return dict(ms_per_call=round(float(np.median(times)), digits), ms_min=round(float(np.min(times)), digits),
                ms_max=round(float(np.max(times)), digits))


def reference_ms_per_clip(prepare, clips):
    """ms per clip of the reference build on one CPU core: prepare(lib) returns clip(i), which processes clip i and is
    timed over `clips` calls; None where the reference build is missing"""
    from oracle import ref_lib as R
    if not R.available():
        return None
    clip = prepare(R.get_ref_lib())
    t0 = time.perf_counter()
    for i in range(clips):
        clip(i)
    return (time.perf_counter() - t0) * 1e3 / clips


def main(run, workloads, steps, warmup, split=lambda s: s.split(",")):
    """--steps, --warmup, --workloads (split() of it names them), --out: runs run(name, steps, warmup) per workload and
    prints its result as one JSON line; --out also writes them all as one JSON list.  Exits non-zero when a workload's
    parity gate fails."""
    prog = os.path.splitext(os.path.basename(sys.argv[0]))[0]
    ap = argparse.ArgumentParser(prog=prog)
    ap.add_argument("--steps", type=int, default=steps)
    ap.add_argument("--warmup", type=int, default=warmup)
    ap.add_argument("--workloads", default=workloads)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit(f"{prog} needs a CUDA device")
    results = []
    for name in split(a.workloads):
        results.append(run(name, a.steps, a.warmup))
        print(json.dumps(results[-1]), flush=True)
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)
    if not all(r["parity_ok"] for r in results):
        sys.exit("parity gate failed")
