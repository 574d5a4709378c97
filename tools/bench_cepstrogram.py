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
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.realpath(__file__)))
import _bench_kit as K  # noqa: E402

import torch  # noqa: E402

import audioflux_b200 as af  # noqa: E402
import _cepstrogram_oracle as CO  # noqa: E402

WORKLOADS = {
    "c12": dict(radix2_exp=12, clips=1024, length=160000, slide=1024, cep_num=4),
    "c10": dict(radix2_exp=10, clips=1024, length=80000, slide=256, cep_num=20),
    "c14": dict(radix2_exp=14, clips=256, length=441000, slide=4096, cep_num=128),
}


def reference_ms_per_clip(w, x, clips=2):
    kw = dict(radix2_exp=w["radix2_exp"], window_type=CO.W_RECT, slide=w["slide"], cep_num=w["cep_num"])
    return K.reference_ms_per_clip(lambda lib: lambda i: CO.c_case(lib, kw, x[i]), clips)   # construction included


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
    times, out = K.event_times(fn, steps, warmup)
    ms = float(np.median(times))
    *want, logs = CO.cepstrogram(x[0], n, w["slide"], CO.W_RECT, c)
    err = max(float(CO.frame_errors(o[0].cpu().numpy(), wt, logs).max()) for o, wt in zip(out, want))
    del out
    per = K.kernel_times(fn, ("k_cepstrogram",))
    nbytes = B * length * 4 + 3 * B * T * (n // 2 + 1) * 4
    flop = 4 * 2.5 * n * r * T * B
    res = dict(workload=name, clips=B, samples=length, fft_length=n, slide=w["slide"], cep_num=c, frames=T * B,
               **K.ms_stats(times, 4),
               kernels_ms={k: round(v, 4) for k, v in per.items()},
               compulsory_bytes=nbytes, hbm_share=round(nbytes / (ms * 1e-3) / K.HBM, 4),
               fft_tflops=round(flop / (ms * 1e-3) / 1e12, 3),
               parity_worst_frame_clip0=err, parity_ok=bool(err <= 1e-4), card=K.card())
    k = per.get("k_cepstrogram")
    if k:
        res["k_cepstrogram_hbm_share"] = round(nbytes / (k * 1e-3) / K.HBM, 4)
        res["k_cepstrogram_tflops"] = round(flop / (k * 1e-3) / 1e12, 3)
    res["reference_ms_per_clip_1core"] = reference_ms_per_clip(w, x)
    return res


if __name__ == "__main__":
    K.main(run, "c12,c10,c14", steps=20, warmup=3)
