"""Cross-correlation and CZT throughput on the device (device-resident rows, CUDA-event timing, median of the timed calls
after warm-up):

  xc_cross  4096 pairs x 4096 samples, cross-correlation with Coeff (M = 8192, k_xcorr)
  xc_auto   4096 autocorrelations x 8192 samples (M = 16384, k_xcorr at its largest size)
  xc_long   32 pairs x 2^19 samples, cross-correlation (M = 2^20: the four-step long path)
  czt10     CZT radix2Exp 10 x 16384 rows, complex input, band (0.15, 0.25)
  czt13     CZT radix2Exp 13 x 1024 rows, real input, band (0, 1) (M = 16384, k_czt at its largest size)

Per workload: ms per call, the kernels' own times (torch.profiler, a separate run), compulsory bytes (rows in, lags or
bins out, maxima) and their share of 3.35 TB/s, a parity gate on row 0 against the float64 oracle (1e-4 of its max),
the card's name, power limit and max SM clock, and where oracle/_ref exists the reference build's time per call on one
CPU core.  Prints one JSON line per workload.

    python tools/bench_dsp.py [--steps 20] [--warmup 3] [--workloads xc_cross,xc_auto,xc_long,czt10,czt13] [--out f.json]"""
import ctypes as C
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.realpath(__file__)))
import _bench_kit as K  # noqa: E402

import torch  # noqa: E402

import audioflux_b200 as af  # noqa: E402
import _dsp_oracle as D  # noqa: E402

WORKLOADS = {
    "xc_cross": dict(kind="xcorr", rows=4096, n=4096, cross=True, norm=1),
    "xc_auto": dict(kind="xcorr", rows=4096, n=8192, cross=False, norm=0),
    "xc_long": dict(kind="xcorr", rows=32, n=1 << 19, cross=True, norm=0),
    "czt10": dict(kind="czt", rows=16384, r=10, cplx=True, band=(0.15, 0.25)),
    "czt13": dict(kind="czt", rows=1024, r=13, cplx=False, band=(0.0, 1.0)),
}
KERNELS = ("k_xcorr_pad", "k_xcorr_cross", "k_xcorr_finish", "k_xcorr_argmax", "k_xcorr", "k_czt_filter", "k_czt",
           "k_cwt_cols", "k_cwt_rows")


def reference_ms(w, host):
    """the reference build's time per call on one CPU core (fresh Xcorr object per call; one CZT object)"""
    def prepare(lib):
        if w["kind"] == "xcorr":
            a, b = host
            return lambda i: D.c_xcorr(lib, a[i], None if b is None else b[i], w["norm"])
        st, o = D.c_czt_new(lib, w["r"])
        re, im = host
        return lambda i: D.c_czt(lib, o, re[i], None if im is None else im[i], *w["band"], 1 << w["r"])
    return K.reference_ms_per_clip(prepare, 2)


def run(name, steps, warmup):
    w = WORKLOADS[name]
    rng = np.random.default_rng(0)
    B = w["rows"]
    res = dict(workload=name, rows=B)
    if w["kind"] == "xcorr":
        n = w["n"]
        a = rng.standard_normal((B, n)).astype(np.float32)
        b = rng.standard_normal((B, n)).astype(np.float32) if w["cross"] else None
        ad = torch.from_numpy(a).cuda()
        bd = None if b is None else torch.from_numpy(b).cuda()
        obj = af.Xcorr()
        nt = af.XcorrNormalType(w["norm"])

        def fn():
            return obj.xcorr_batch(ad, bd, nt)
        times, out = K.event_times(fn, steps, warmup)
        want, _, _ = D.xcorr(a[0], None if b is None else b[0], w["norm"])
        err = float(np.abs(out[0][0].cpu().numpy() - want).max() / np.abs(want).max())
        nbytes = (B * n * (2 if w["cross"] else 1) + B * (2 * n - 1) + 2 * B) * 4
        res.update(samples=n, fft_length=1 << int(np.ceil(np.log2(2 * n))), cross=w["cross"], coeff=bool(w["norm"]))
        host = (a, b)
    else:
        N = 1 << w["r"]
        re = rng.standard_normal((B, N)).astype(np.float32)
        im = rng.standard_normal((B, N)).astype(np.float32) if w["cplx"] else None
        x = torch.complex(torch.from_numpy(re), torch.from_numpy(im)).cuda() if w["cplx"] else torch.from_numpy(re).cuda()
        obj = af.CZT(w["r"])

        def fn():
            return obj.czt_batch(x, *w["band"])
        times, out = K.event_times(fn, steps, warmup)
        x0 = re[0].astype(np.float64) + (0 if im is None else 1j * im[0].astype(np.float64))
        want = D.czt(x0, w["r"], *w["band"])
        err = float(np.abs(out[0].cpu().numpy() - want).max() / np.abs(want).max())
        nbytes = (B * N * (2 if w["cplx"] else 1) + B * 4 * N) * 4
        res.update(radix2_exp=w["r"], fft_length=2 * N, complex_input=w["cplx"], band=list(w["band"]))
        host = (re, im)
    del out
    ms = float(np.median(times))
    per = K.kernel_times(fn, KERNELS)
    res.update(**K.ms_stats(times, 4), kernels_ms={k: round(v, 4) for k, v in per.items()}, compulsory_bytes=nbytes,
               hbm_bytes_per_s=round(nbytes / (ms * 1e-3), 0), hbm_share=round(nbytes / (ms * 1e-3) / K.HBM, 5),
               parity_worst_row0=err, parity_ok=bool(err <= 1e-4), card=K.card())
    res["reference_ms_per_call_1core"] = reference_ms(w, host)
    return res


if __name__ == "__main__":
    K.main(run, "xc_cross,xc_auto,xc_long,czt10,czt13", steps=20, warmup=3)
