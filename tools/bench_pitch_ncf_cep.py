"""PitchNCF and PitchCEP throughput on the device (device-resident clips, CUDA-event timing, median of the timed calls
after warm-up), each tracker on three workloads:

  12  n = 2^12, 1024 clips x 160 000 samples (5 s at 32 kHz), the Python defaults (32 .. 2000 Hz, slide 1024): 156 672
      frames
  11  n = 2^11, 1024 clips x 110 250 samples (5 s at 22.05 kHz), slide 512
  13  n = 2^13,   64 clips x 2 646 000 samples (60 s at 44.1 kHz), slide 2048: long clips, a large frame

(workload names ncf12, ncf11, ncf13, cep12, cep11, cep13).  Per workload: ms per call and frames per second, the
kernel's own time (torch.profiler, a separate run), the FFT rate counting 2.5 N log2 N flops per real N-point transform
(two of 2n points per frame), compulsory bytes (clips in, fre out) and their share of 3.35 TB/s, a parity gate on clip 0
against the float64 oracle, the card's name, power limit and max SM clock, and where oracle/_ref exists the reference
build's time per clip on one CPU core.  Prints one JSON line per workload.

    python tools/bench_pitch_ncf_cep.py [--steps 20] [--warmup 3] [--workloads ncf12,cep12] [--out results.json]"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.realpath(__file__)))
import _bench_kit as K  # noqa: E402

import torch  # noqa: E402

import audioflux_b200 as af  # noqa: E402
import _pitch_ncf_cep_oracle as PO  # noqa: E402

SIZES = {
    "12": dict(radix2_exp=12, clips=1024, length=160000, sr=32000, slide=1024),
    "11": dict(radix2_exp=11, clips=1024, length=110250, sr=22050, slide=512),
    "13": dict(radix2_exp=13, clips=64, length=2646000, sr=44100, slide=2048),
}
WORKLOADS = {kind + size: dict(w, kind=kind) for kind in PO.KINDS for size, w in SIZES.items()}
KERNEL = {"ncf": "k_pitch_ncf", "cep": "k_pitch_cep"}


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
    kw = dict(sr=w["sr"], lf=32.0, hf=2000.0, r2=w["radix2_exp"], slide=w["slide"])

    def prepare(lib):
        def clip(i):
            st, o = PO.c_new(lib, w["kind"], **kw)
            PO.c_pitch(lib, w["kind"], o, x[i])
            PO.c_free(lib, w["kind"], o)
        return clip
    return K.reference_ms_per_clip(prepare, clips)      # construction included


def run(name, steps, warmup):
    w = WORKLOADS[name]
    kind, r, B, length = w["kind"], w["radix2_exp"], w["clips"], w["length"]
    n = 1 << r
    cls = af.PitchNCF if kind == "ncf" else af.PitchCEP
    obj = cls(samplate=w["sr"], radix2_exp=r, slide_length=w["slide"])
    p = PO.params(kind, sr=w["sr"], lf=32.0, hf=2000.0, r2=r, slide=w["slide"])
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
    kname = KERNEL[kind]
    per = K.kernel_times(fn, (kname,), per_launch=True)                 # one launch per call
    nbytes = B * length * 4 + B * T * 4
    flop = 2 * 2.5 * (2 * n) * (r + 1) * T * B
    res = dict(workload=name, clips=B, samples=length, samplate=w["sr"], frame=n, slide=w["slide"],
               lags=[p["min_index"], p["max_index"]], frames=T * B, **K.ms_stats(times, 4),
               frames_per_s=round(T * B / (ms * 1e-3)), kernels_ms={k: round(v, 4) for k, v in per.items()},
               compulsory_bytes=nbytes, hbm_share=round(nbytes / (ms * 1e-3) / K.HBM, 5),
               fft_tflops=round(flop / (ms * 1e-3) / 1e12, 3),
               parity_undetermined_frames_clip0=len(alt), parity_ok=bool(ok), card=K.card())
    k = per.get(kname)
    if k:
        res[f"{kname}_tflops"] = round(flop / (k * 1e-3) / 1e12, 3)
        res[f"{kname}_hbm_share"] = round(nbytes / (k * 1e-3) / K.HBM, 5)
    res["reference_ms_per_clip_1core"] = reference_ms_per_clip(w, x)
    return res


if __name__ == "__main__":
    K.main(run, ",".join(WORKLOADS), steps=20, warmup=3)
