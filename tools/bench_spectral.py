"""Spectral-descriptor throughput: the C2 geometry (1024 clips x 465 frames x 1025 bins, a Linear power spectrogram,
1.95 GB) resident on the device.  Prints one JSON line: event-timed ms of every non-phase feature in ONE
spectralObj_spectralBatch call and of one call per feature, the compulsory bytes (input read once + outputs) over time
against the 3.35 TB/s H100 SXM data sheet, the reference build's single-thread CPU rate on the same input (when
oracle/_ref is built) and the GPU name and power limit read in the same run.

    python tools/bench_spectral.py [--clips 1024] [--steps 20] [--warmup 3]"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.realpath(__file__)))
import _bench_kit as K  # noqa: E402

import torch  # noqa: E402

import audioflux_b200 as af  # noqa: E402
from audioflux_b200 import spectral as SP  # noqa: E402


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(steps):
        fn()
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=1024)
    ap.add_argument("--frames", type=int, default=465)
    ap.add_argument("--num", type=int, default=1025)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ref-clips", type=int, default=2)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    B, T, N = a.clips, a.frames, a.num
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.rand((B, T, N), device="cuda", generator=g) ** 4          # power-like spread of levels
    fre = np.linspace(0, 24000, N).astype(np.float32)
    s = af.Spectral(N, fre)
    feats = [(n, {}) for n in SP.FEATURES if n not in SP.PHASE_FEATURES]
    planes = sum(2 if n in SP.TWO_PLANES else 1 for n, _ in feats)

    all_ms = timed(lambda: s.spectral_batch(x, feats), a.steps, a.warmup)
    per = {}
    for f in feats:
        per[f[0]] = timed(lambda f=f: s.spectral_batch(x, [f]), max(a.steps // 4, 2), 1)
    in_bytes = B * T * N * 4
    out_bytes = planes * B * T * 4
    res = {
        "workload": f"{B} clips x {T} frames x {N} bins float32 ({in_bytes / 1e9:.2f} GB), device-resident",
        "features_in_one_call": len(feats),
        "all_features_one_call_ms": round(all_ms, 3),
        "one_call_per_feature_total_ms": round(sum(per.values()), 3),
        "one_call_per_feature_ms": {k: round(v, 3) for k, v in per.items()},
        "compulsory_GB": round((in_bytes + out_bytes) / 1e9, 3),
        "all_features_TBps": round((in_bytes + out_bytes) / all_ms / 1e9, 3),
        "fraction_of_3.35TBps": round((in_bytes + out_bytes) / all_ms / 1e-3 / K.HBM, 3),
    }
    card = [v.strip() for v in K.card().split(",")]
    res["gpu"], res["power_limit"] = card[0], card[1] if len(card) > 1 else "unknown"

    if a.ref_clips > 0:
        import _spectral_cases as SC
        xs = x[:a.ref_clips].cpu().numpy()
        ms = K.reference_ms_per_clip(
            lambda lib: lambda b: [SC.call_c(lib, n, xs[b], fre, "full", None, **kw) for n, kw in feats], a.ref_clips)
        if ms is not None:
            res["reference_cpu_ms_per_clip_all_features"] = round(ms, 2)
            res["reference_cpu_extrapolated_ms_for_workload"] = round(ms * B, 1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
