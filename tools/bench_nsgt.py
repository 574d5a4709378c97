"""NSGT throughput on the device, two workloads (device-resident clips, CUDA-event timing after warm-up):

  (a) 1024 clips x 2^15 samples at 32 kHz, Octave 84, 12 bins per octave, Slaney, BandWidth (the reference class's
      defaults at the length of its docs example)
  (b) 64 clips x 2^19 samples at 44.1 kHz, Octave 84 (widest band 5587 points: the direct path runs)

Per workload: ms per call, split into the forward FFT and the band kernels (torch.profiler, a separate run), compulsory
bytes (clips in, matrix out) and their share of 3.35 TB/s, a parity gate against the oracle on clip 0, and for (a) the
reference build's time per clip on one CPU core when oracle/_ref exists.  Prints one JSON line per workload.

    python tools/bench_nsgt.py [--steps 20] [--warmup 3] [--out results.json]"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.realpath(__file__)))
import _bench_kit as K  # noqa: E402

import torch  # noqa: E402

import audioflux_b200 as af  # noqa: E402
import _nsgt_oracle as NO  # noqa: E402
from oracle import af_oracle as O  # noqa: E402

WORKLOADS = {
    "a": dict(batch=1024, radix2_exp=15, samplate=32000),
    "b": dict(batch=64, radix2_exp=19, samplate=44100),
}


def reference_ms_per_clip(kw, x, clips=5):
    from oracle import ref_lib as R
    if not R.available():
        return None
    lib = R.get_ref_lib()
    st, obj = NO.c_new(lib, **kw)
    if st != 0:
        return None
    NO.c_nsgt(lib, obj, x[0], kw["num"])          # builds nothing new, but touches the matrices once
    try:
        return K.reference_ms_per_clip(lambda lib: lambda i: NO.c_nsgt(lib, obj, x[i % len(x)], kw["num"]), clips)
    finally:
        lib.nsgtObj_free(obj)


def run(name, steps, warmup):
    w = WORKLOADS[name]
    kw = dict(num=84, radix2_exp=w["radix2_exp"], samplate=w["samplate"], low_fre=32.703196, bin_per_octave=12,
              scale_type=O.SCALE_OCTAVE, style_type=O.STYLE_SLANEY, normal_type=O.NORM_BANDWIDTH)
    t = af.NSGT(num=84, radix2_exp=w["radix2_exp"], samplate=w["samplate"], bin_per_octave=12)
    n, B = 1 << w["radix2_exp"], w["batch"]
    rng = np.random.default_rng(0)
    x = (0.1 * rng.standard_normal((B, n))).astype(np.float32)
    x[0] = NO.case_signal(1, n, w["samplate"])
    xd = torch.from_numpy(x).cuda()
    times, (re, im) = K.event_times(lambda: t.nsgt_batch(xd), steps, warmup)
    ms = float(np.median(times))
    _, p = NO.params(**kw)
    _, m = NO.transform(x[0], p)
    r0, i0 = re[0].cpu().numpy(), im[0].cpu().numpy()
    err = max(np.abs(r0 - m.real).max() / np.abs(m.real).max(), np.abs(i0 - m.imag).max() / np.abs(m.imag).max())
    per = K.kernel_times(lambda: t.nsgt_batch(xd), ())
    band = sum(v for k, v in per.items() if "k_nsgt_" in k)
    fwd = sum(per.values()) - band
    T = t.get_max_time_length()
    nbytes = B * n * 4 + B * 84 * T * 8
    res = dict(workload=name, clips=B, samples=n, samplate=w["samplate"], max_len=T,
               total_len=t.get_total_time_length(), widest=int(t.get_time_length_arr().max()),
               **K.ms_stats(times, 4),
               ms_forward_fft=round(fwd, 4), ms_band_kernels=round(band, 4),
               kernels_ms={k: round(v, 4) for k, v in per.items()},
               compulsory_bytes=nbytes, hbm_share=round(nbytes / (ms * 1e-3) / K.HBM, 4),
               parity_rel_err_clip0=float(err), parity_ok=bool(err <= 1e-4), card=K.card())
    if name == "a":
        res["reference_ms_per_clip_1core"] = reference_ms_per_clip(kw, x)
    return res


if __name__ == "__main__":
    K.main(run, "ab", steps=20, warmup=3, split=list)
