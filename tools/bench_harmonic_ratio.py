"""Harmonic ratio throughput on the device (device-resident clips, CUDA-event timing, median of the timed calls after
warm-up):

  h12    W = 2^12, 1024 clips x 160 000 samples (5 s at 32 kHz), slide 1024, lowFre C1 (maxLength 978), 156 672 frames
  h11    W = 2^11, 1024 clips x 220 500 samples (5 s at 44.1 kHz), slide 512, lowFre 50
  h13    W = 2^13,  256 clips x 441 000 samples (at 32 kHz), slide 2048, lowFre C1
  h12dc  h12 with a DC offset on every clip: no frame's autocorrelation crosses zero below maxLength, so every frame takes
         the carry pass (the worst case of the second launch)

Per workload: ms per call, the kernels' own times (torch.profiler, a separate run), compulsory bytes (clips in, values
out) and their share of 3.35 TB/s, the FP32 rate counting 2.5 N log2 N flops per real N-point transform (N = 2W, two per
frame, and two more per frame of the carry pass), a parity gate on clip 0 against the float64 oracle, the card's name,
power limit and max SM clock, and where oracle/_ref exists the reference build's time per clip on one CPU core.
Prints one JSON line per workload.

    python tools/bench_harmonic_ratio.py [--steps 20] [--warmup 3] [--workloads h12,h11,h13,h12dc] [--out results.json]"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.realpath(__file__)))
import _bench_kit as K  # noqa: E402

import torch  # noqa: E402

import audioflux_b200 as af  # noqa: E402
import _harmonic_ratio_oracle as HO  # noqa: E402

C1 = 32.703196
WORKLOADS = {
    "h12": dict(radix2_exp=12, clips=1024, length=160000, sr=32000, slide=1024, low_fre=C1, dc=0.0),
    "h11": dict(radix2_exp=11, clips=1024, length=220500, sr=44100, slide=512, low_fre=50.0, dc=0.0),
    "h13": dict(radix2_exp=13, clips=256, length=441000, sr=32000, slide=2048, low_fre=C1, dc=0.0),
    "h12dc": dict(radix2_exp=12, clips=1024, length=160000, sr=32000, slide=1024, low_fre=C1, dc=1.0),
}


def clips(w):
    """seeded noise with a harmonic tone per clip (f0 80 .. 600 Hz), plus the workload's DC offset"""
    rng = np.random.default_rng(0)
    B, n = w["clips"], w["length"]
    t = np.arange(n, dtype=np.float32) / np.float32(w["sr"])
    f0 = rng.uniform(80, 600, B).astype(np.float32)
    x = (0.05 * rng.standard_normal((B, n))).astype(np.float32) + w["dc"]
    for h in range(1, 4):
        x += (0.3 / h) * np.sin((2 * np.pi * h) * f0[:, None] * t[None, :] + h).astype(np.float32)
    return x


def reference_ms_per_clip(w, x, clips=2):
    kw = dict(sr=w["sr"], lf=w["low_fre"], r2=w["radix2_exp"], wt=None, slide=w["slide"])

    def prepare(lib):
        def clip(i):
            st, o = HO.c_new(lib, **kw)
            HO.c_ratio(lib, o, x[i])
            lib.harmonicRatioObj_free(o)
        return clip
    return K.reference_ms_per_clip(prepare, clips)      # construction included


def run(name, steps, warmup):
    w = WORKLOADS[name]
    r, B, length = w["radix2_exp"], w["clips"], w["length"]
    n = 2 << r
    obj = af.HarmonicRatio(samplate=w["sr"], low_fre=w["low_fre"], radix2_exp=r, slide_length=w["slide"])
    T = obj.cal_time_length(length)
    x = clips(w)
    xd = torch.from_numpy(x).cuda()

    def fn():
        return obj.harmonic_ratio_batch(xd)
    times, out = K.event_times(fn, steps, warmup)
    ms = float(np.median(times))
    p = HO.params(w["sr"], w["low_fre"], r, w["slide"])
    want, cands, own = HO.harmonic_ratio(x[0], p["W"], p["slide"], p["max_length"])
    scale = max(np.abs(want).max(), 1e-30)
    ok, alt = HO.agree(out[0].cpu().numpy(), want, cands, 1e-4 * scale)
    err = float(np.abs(out[0].cpu().numpy() - want).max() / scale)
    del out
    carry_frac = sum(o is None for o in own) / len(own)          # clip 0's share of frames without a crossing
    # per launch (one of each per call here): the average stays right when the trace drops a call's events
    per = K.kernel_times(fn, ("k_harmonic_ratio_carry", "k_harmonic_ratio"), per_launch=True)
    nbytes = B * length * 4 + B * T * 4
    flop = 2 * 2.5 * n * (r + 1) * T * B
    res = dict(workload=name, clips=B, samples=length, window=1 << r, fft_length=n, slide=w["slide"],
               max_length=p["max_length"], frames=T * B, carry_fraction_clip0=round(carry_frac, 4),
               **K.ms_stats(times, 4),
               kernels_ms={k: round(v, 4) for k, v in per.items()},
               compulsory_bytes=nbytes, hbm_share=round(nbytes / (ms * 1e-3) / K.HBM, 5),
               fft_tflops=round(flop / (ms * 1e-3) / 1e12, 3),
               parity_worst_frame_clip0=err, parity_undetermined_frames_clip0=len(alt), parity_ok=bool(ok),
               card=K.card())
    k = per.get("k_harmonic_ratio")
    if k:
        res["k_harmonic_ratio_tflops"] = round(flop / (k * 1e-3) / 1e12, 3)
    res["reference_ms_per_clip_1core"] = reference_ms_per_clip(w, x)
    return res


if __name__ == "__main__":
    K.main(run, "h12,h11,h13,h12dc", steps=20, warmup=3)
