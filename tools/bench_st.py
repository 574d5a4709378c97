"""ST / FST throughput on the device (device-resident clips, CUDA-event timing, median of the timed calls after warm-up):

  st12   ST  at 2^12, rows 1 .. 2047, 128 clips   (8.6 GB of output planes per call)
  fst12  FST at 2^12, rows 1 .. 2047, 128 clips   (the same output: a pure store stream after two small kernels)
  st14   ST  at 2^14, rows 1000 .. 1063, 128 clips (the in-place shared-memory path)

Per workload: ms per call, the kernels' own times (torch.profiler, a separate run), compulsory bytes (clips in, planes
out) and their share of 3.35 TB/s, for ST the FP32 rate of the inverse FFTs (5 N log2 N per row), a parity gate on
clip 0 against the float64 oracle, the card's name, power limit and max SM clock, and where oracle/_ref exists the
reference build's time per clip on one CPU core.  Prints one JSON line per workload.

    python tools/bench_st.py [--steps 20] [--warmup 3] [--workloads st12,fst12,st14] [--out results.json]"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.realpath(__file__)))
import _bench_kit as K  # noqa: E402

import torch  # noqa: E402

import audioflux_b200 as af  # noqa: E402
import _st_oracle as SO  # noqa: E402

WORKLOADS = {
    "st12": dict(kind="st", radix2_exp=12, lo=1, hi=2047, batch=128),
    "fst12": dict(kind="fst", radix2_exp=12, lo=1, hi=2047, batch=128),
    "st14": dict(kind="st", radix2_exp=14, lo=1000, hi=1063, batch=128),
}


def reference_ms_per_clip(w, x, clips=2):
    kw = dict(radix2_exp=w["radix2_exp"], min_index=w["lo"], max_index=w["hi"])
    case = SO.c_st_case if w["kind"] == "st" else SO.c_fst_case
    return K.reference_ms_per_clip(lambda lib: lambda i: case(lib, kw, x[i]), clips)   # construction included


def run(name, steps, warmup):
    w = WORKLOADS[name]
    r, B = w["radix2_exp"], w["batch"]
    n, rows = 1 << r, w["hi"] - w["lo"] + 1
    if w["kind"] == "st":
        obj = af.ST(radix2_exp=r, min_index=w["lo"], max_index=w["hi"])
        fn = obj.st_batch
    else:
        obj = af.FST(radix2_exp=r, min_index=w["lo"], max_index=w["hi"])
        fn = obj.fst_batch
    rng = np.random.default_rng(0)
    x = (0.1 * rng.standard_normal((B, n))).astype(np.float32)
    x[0] = SO.case_signal(1, n)
    xd = torch.from_numpy(x).cuda()
    times, (re, im) = K.event_times(lambda: fn(xd), steps, warmup)
    ms = float(np.median(times))
    want = SO.st(x[0], list(range(w["lo"], w["hi"] + 1))) if w["kind"] == "st" else SO.fst(x[0], w["lo"], w["hi"])
    err, _ = SO.row_errors(re[0].cpu().numpy(), im[0].cpu().numpy(), want)
    del re, im
    per = K.kernel_times(lambda: fn(xd), ("k_st_rows", "k_fst_segments", "k_fst_expand", "k_stft_generic"))
    nbytes = B * n * 4 + B * rows * n * 8
    res = dict(workload=name, kind=w["kind"], clips=B, samples=n, rows=rows,
               **K.ms_stats(times, 4),
               kernels_ms={k: round(v, 4) for k, v in per.items()},
               compulsory_bytes=nbytes, hbm_share=round(nbytes / (ms * 1e-3) / K.HBM, 4),
               parity_worst_row_clip0=float(err.max()), parity_ok=bool(err.max() <= 1e-4), card=K.card())
    if w["kind"] == "st":
        flop = 5.0 * n * r * rows * B
        res["fft_tflops"] = round(flop / (ms * 1e-3) / 1e12, 3)
        k = per.get("k_st_rows")
        if k:
            res["k_st_rows_hbm_share"] = round(B * rows * n * 8 / (k * 1e-3) / K.HBM, 4)
            res["k_st_rows_tflops"] = round(flop / (k * 1e-3) / 1e12, 3)
    else:
        k = per.get("k_fst_expand")
        if k:
            res["k_fst_expand_hbm_share"] = round(B * rows * n * 8 / (k * 1e-3) / K.HBM, 4)
    res["reference_ms_per_clip_1core"] = reference_ms_per_clip(w, x)
    return res


if __name__ == "__main__":
    K.main(run, "st12,fst12,st14", steps=20, warmup=3)
