"""Discrete wavelet transform throughput on the device (device-resident clips, CUDA-event timing, median of the timed
calls after warm-up):

  dwt12   DWT sym4, 2^12 samples x 4096 clips, num 11 (every level), coef and mDataArr
  dwt16   DWT sym4, 2^16 samples x 256 clips, num 15
  wpt12   WPT db4, num 6, 2^12 samples x 4096 clips, coef and the 64 leaf rows
  swt14   SWT sym4, num 8, 2^14 samples x 1024 clips

The outputs dominate the traffic, so the bound is HBM write bandwidth: per workload, ms per call, the kernels' own times
(torch.profiler, a separate run), the compulsory bytes (clips in; coef and mDataArr, or both SWT planes, out) and their
share of 3.35 TB/s, a parity gate on clip 0 against the float64 oracle, the card's name, power limit and max SM clock,
and where oracle/_ref exists the reference build's time per clip on one CPU core.  Prints one JSON line per workload.

    python tools/bench_wavelet.py [--steps 20] [--warmup 3] [--workloads dwt12,dwt16,wpt12,swt14] [--out results.json]"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.realpath(__file__)))
import _bench_kit as K  # noqa: E402

import torch  # noqa: E402

import audioflux_b200 as af  # noqa: E402
import _wavelet_oracle as W  # noqa: E402
from test_wavelet_cpu import TABLE  # noqa: E402

WORKLOADS = {
    "dwt12": dict(kind="dwt", num=11, size=12, clips=4096, ty=2, t1=4),
    "dwt16": dict(kind="dwt", num=15, size=16, clips=256, ty=2, t1=4),
    "wpt12": dict(kind="wpt", num=6, size=12, clips=4096, ty=1, t1=4),
    "swt14": dict(kind="swt", num=8, size=1 << 14, clips=1024, ty=2, t1=4),
}


def run(name, steps, warmup):
    w = WORKLOADS[name]
    kind, num, size, B = w["kind"], w["num"], w["size"], w["clips"]
    n = size if kind == "swt" else 1 << size
    ty = af.WaveletDiscreteType(w["ty"])
    if kind == "swt":
        obj = af.SWT(num, n, wavelet_type=ty, t1=w["t1"])
    else:
        obj = (af.DWT if kind == "dwt" else af.WPT)(num=num, radix2_exp=size, wavelet_type=ty, t1=w["t1"])
    rows = 2 * num if kind == "swt" else 1 + (num if kind == "dwt" else 1 << num)
    x = np.stack([W.signal(n, i) for i in range(8)] * (B // 8))
    xd = torch.from_numpy(x).cuda()
    fn = lambda: getattr(obj, f"{kind}_batch")(xd)        # noqa: E731
    times, out = K.event_times(fn, steps, warmup)
    ms = float(np.median(times))
    got = np.concatenate([o[0].cpu().numpy().ravel() for o in out])
    del out
    lo, hi = (v.astype(np.float64) for v in TABLE[(w["ty"], w["t1"], 0)])
    want = np.concatenate([a.ravel() for a in getattr(W, kind)(x[0].astype(np.float64), num, lo, hi)])
    err = float(np.abs(got - want).max() / np.abs(want).max())
    per = K.kernel_times(fn, ("k_wavelet_level", "k_wavelet_expand", "k_swt_level"))
    nbytes = B * n * 4 * (1 + rows)
    written = B * n * 4 * rows
    res = dict(workload=name, transform=kind, clips=B, samples=n, num=num, **K.ms_stats(times, 4),
               kernels_ms={k: round(v, 4) for k, v in per.items()},
               compulsory_bytes=nbytes, written_bytes=written,
               achieved_tb_s=round(nbytes / (ms * 1e-3) / 1e12, 3), hbm_share=round(nbytes / (ms * 1e-3) / K.HBM, 4),
               parity_rel_err_clip0=err, parity_ok=bool(err <= 1e-4), card=K.card())

    def prepare(lib):
        def clip(i):
            W.run(lib, kind, num, size, w["ty"], w["t1"], 0, x[i])
        return clip
    res["reference_ms_per_clip_1core"] = K.reference_ms_per_clip(prepare, 2)     # construction included
    return res


if __name__ == "__main__":
    K.main(run, "dwt12,dwt16,wpt12,swt14", steps=20, warmup=3)
