"""PitchYIN throughput on the device (device-resident clips, CUDA-event timing, median of the timed calls after warm-up):

  y12  n = 2^12, 1024 clips x 160 000 samples (5 s at 32 kHz), the Python defaults (27 .. 2000 Hz, slide 1024,
       autoLength 2048): 156 672 frames
  y11  n = 2^11, 1024 clips x 110 250 samples (5 s at 22.05 kHz), slide 512, autoLength 1024
  y13  n = 2^13,   64 clips x 2 646 000 samples (60 s at 44.1 kHz), slide 2048: long clips, a large frame

Per workload: ms per call and frames per second, the kernel's own time (torch.profiler, a separate run), the FFT rate
counting 2.5 N log2 N flops per real N-point transform (three of n points per frame), compulsory bytes (clips in, fre,
value1 and value2 out) and their share of 3.35 TB/s, a parity gate on clip 0 against the float64 interval oracle, the
card's name, power limit and max SM clock, and where oracle/_ref exists the reference build's time per clip on one CPU
core.  Prints one JSON line per workload.

    python tools/bench_pitch_yin.py [--steps 20] [--warmup 3] [--workloads y12,y11,y13] [--out results.json]"""
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.realpath(__file__)))
import _bench_kit as K  # noqa: E402

import torch  # noqa: E402

import audioflux_b200 as af  # noqa: E402
import _pitch_yin_oracle as YO  # noqa: E402

WORKLOADS = {
    "y12": dict(radix2_exp=12, clips=1024, length=160000, sr=32000, slide=1024, auto=2048),
    "y11": dict(radix2_exp=11, clips=1024, length=110250, sr=22050, slide=512, auto=1024),
    "y13": dict(radix2_exp=13, clips=64, length=2646000, sr=44100, slide=2048, auto=4096),
}


def clips(w):
    """seeded noise with a harmonic tone per clip (f0 80 .. 600 Hz)"""
    rng = np.random.default_rng(0)
    B, n = w["clips"], w["length"]
    t = np.arange(n, dtype=np.float32) / np.float32(w["sr"])
    f0 = rng.uniform(80, 600, B).astype(np.float32)
    x = (0.05 * rng.standard_normal((B, n))).astype(np.float32)
    for h in range(1, 4):
        x += (0.3 / h) * np.sin((2 * np.pi * h) * f0[:, None] * t[None, :] + h).astype(np.float32)
    return x


def reference_ms_per_clip(w, x, clips=1):
    kw = dict(sr=w["sr"], lf=27.0, hf=2000.0, r2=w["radix2_exp"], slide=w["slide"], auto=w["auto"])

    def prepare(lib):
        def clip(i):
            st, o = YO.c_new(lib, **kw)
            YO.c_pitch(lib, o, x[i])
            lib.pitchYINObj_free(o)
        return clip
    return K.reference_ms_per_clip(prepare, clips)      # construction included


def run(name, steps, warmup):
    w = WORKLOADS[name]
    r, B, length = w["radix2_exp"], w["clips"], w["length"]
    n = 1 << r
    obj = af.PitchYIN(samplate=w["sr"], radix2_exp=r, slide_length=w["slide"], auto_length=w["auto"])
    p = YO.params(sr=w["sr"], lf=27.0, hf=2000.0, r2=r, slide=w["slide"], auto=w["auto"])
    T = obj.cal_time_length(length)
    x = clips(w)
    xd = torch.from_numpy(x).cuda()

    def fn():
        return obj.pitch_batch(xd)
    times, out = K.event_times(fn, steps, warmup)
    ms = float(np.median(times))
    ok, msg, alt = YO.check(*(o[0].cpu().numpy() for o in out), YO.pitch(x[0], p), p, 0.0)
    del out
    per = K.kernel_times(fn, ("k_pitch_yin",), per_launch=True)          # one launch per call
    nbytes = B * length * 4 + 3 * B * T * 4
    flop = 3 * 2.5 * n * r * T * B
    res = dict(workload=name, clips=B, samples=length, samplate=w["sr"], frame=n, slide=w["slide"], auto=w["auto"],
               lags=[p["min_index"], p["max_index"]], frames=T * B, **K.ms_stats(times, 4),
               frames_per_s=round(T * B / (ms * 1e-3)), kernels_ms={k: round(v, 4) for k, v in per.items()},
               compulsory_bytes=nbytes, hbm_share=round(nbytes / (ms * 1e-3) / K.HBM, 5),
               fft_tflops=round(flop / (ms * 1e-3) / 1e12, 3),
               parity_undetermined_frames_clip0=len(alt), parity_ok=bool(ok), parity_message=msg, card=K.card())
    k = per.get("k_pitch_yin")
    if k:
        res["k_pitch_yin_tflops"] = round(flop / (k * 1e-3) / 1e12, 3)
        res["k_pitch_yin_hbm_share"] = round(nbytes / (k * 1e-3) / K.HBM, 5)
    res["reference_ms_per_clip_1core"] = reference_ms_per_clip(w, x)
    return res


if __name__ == "__main__":
    K.main(run, "y12,y11,y13", steps=20, warmup=3)
