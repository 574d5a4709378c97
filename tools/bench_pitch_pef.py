"""PitchPEF throughput on the device (device-resident clips, CUDA-event timing, median of the timed calls after warm-up):

  p12  n = 2^12, 1024 clips x 160 000 samples (5 s at 32 kHz), the reference's defaults (slide 1024, 32 .. 2000 Hz,
       cut 4000 Hz, alpha 10, beta 0.5, gamma 1.8): a 4n-point correlation per frame, 156 672 frames
  p11  n = 2^11, 1024 clips x 110 250 samples (5 s at 22.05 kHz), slide 512
  p13  n = 2^13,   64 clips x 2 646 000 samples (60 s at 44.1 kHz), slide 2048: long clips, the largest frame

Per workload: ms per call and frames per second, the kernel's own time (torch.profiler, a separate run), the FFT rate
counting 2.5 N log2 N flops per real N-point transform (one of 2n points and two of L points per frame), compulsory
bytes (clips in, frequencies out) and their share of 3.35 TB/s, a parity gate on clip 0 against the float64 oracle, the
card's name, power limit and max SM clock, and where oracle/_ref exists the reference build's time per clip on one CPU
core.  Prints one JSON line per workload.

    python tools/bench_pitch_pef.py [--steps 20] [--warmup 3] [--workloads p12,p11,p13] [--out results.json]"""
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.realpath(__file__)))
import _bench_kit as K  # noqa: E402

import torch  # noqa: E402

import audioflux_b200 as af  # noqa: E402
import _pitch_pef_oracle as PO  # noqa: E402

WORKLOADS = {
    "p12": dict(radix2_exp=12, clips=1024, length=160000, sr=32000, slide=1024),
    "p11": dict(radix2_exp=11, clips=1024, length=110250, sr=22050, slide=512),
    "p13": dict(radix2_exp=13, clips=64, length=2646000, sr=44100, slide=2048),
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
    kw = dict(sr=w["sr"], r2=w["radix2_exp"], slide=w["slide"])

    def prepare(lib):
        def clip(i):
            st, o = PO.c_new(lib, **kw)
            PO.c_pitch(lib, o, x[i])
            lib.pitchPEFObj_free(o)
        return clip
    return K.reference_ms_per_clip(prepare, clips)      # construction included


def run(name, steps, warmup):
    w = WORKLOADS[name]
    r, B, length = w["radix2_exp"], w["clips"], w["length"]
    n = 1 << r
    obj = af.PitchPEF(samplate=w["sr"], radix2_exp=r, slide_length=w["slide"])
    p = PO.params(sr=w["sr"], r2=r, slide=w["slide"], lf=32.0, hf=2000.0, cf=4000.0)
    need = max(p["pad"] + 2 * n, n + p["max_index"] + 1)
    L = 1 << math.ceil(math.log2(need))                   # the kernel's correlation length (kernels/pitch_pef.cu)
    T = obj.cal_time_length(length)
    x = clips(w)
    xd = torch.from_numpy(x).cuda()

    def fn():
        return obj.pitch_batch(xd)
    times, out = K.event_times(fn, steps, warmup)
    ms = float(np.median(times))
    want, cands = PO.pitch(x[0], p)
    ok, alt = PO.agree(out[0].cpu().numpy(), want, cands, p)
    del out
    per = K.kernel_times(fn, ("k_pitch_pef",), per_launch=True)          # one launch per call
    nbytes = B * length * 4 + B * T * 4
    flop = (2.5 * 2 * n * (r + 1) + 2 * 2.5 * L * math.log2(L)) * T * B
    res = dict(workload=name, clips=B, samples=length, samplate=w["sr"], frame=n, slide=w["slide"],
               correlation_length=L, lags=[p["min_index"], p["max_index"]], frames=T * B, **K.ms_stats(times, 4),
               frames_per_s=round(T * B / (ms * 1e-3)), kernels_ms={k: round(v, 4) for k, v in per.items()},
               compulsory_bytes=nbytes, hbm_share=round(nbytes / (ms * 1e-3) / K.HBM, 5),
               fft_tflops=round(flop / (ms * 1e-3) / 1e12, 3),
               parity_undetermined_frames_clip0=len(alt), parity_ok=bool(ok), card=K.card())
    k = per.get("k_pitch_pef")
    if k:
        res["k_pitch_pef_tflops"] = round(flop / (k * 1e-3) / 1e12, 3)
        res["k_pitch_pef_hbm_share"] = round(nbytes / (k * 1e-3) / K.HBM, 5)
    res["reference_ms_per_clip_1core"] = reference_ms_per_clip(w, x)
    return res


if __name__ == "__main__":
    K.main(run, "p12,p11,p13", steps=20, warmup=3)
