"""Pitch tracker throughput on the device (device-resident clips, CUDA-event timing, median of the timed calls after
warm-up): PitchPEF (p), PitchYIN (y), PitchNCF (ncf) and PitchCEP (cep), each on three workloads:

  12  n = 2^12, 1024 clips x 160 000 samples (5 s at 32 kHz), the Python defaults (slide 1024; PEF 32 .. 2000 Hz, cut
      4000 Hz, alpha 10, beta 0.5, gamma 1.8; YIN 27 .. 2000 Hz, autoLength 2048; NCF / CEP 32 .. 2000 Hz): 156 672
      frames
  11  n = 2^11, 1024 clips x 110 250 samples (5 s at 22.05 kHz), slide 512 (YIN autoLength 1024)
  13  n = 2^13,   64 clips x 2 646 000 samples (60 s at 44.1 kHz), slide 2048 (YIN autoLength 4096): long clips, a
      large frame

(workload names p12 p11 p13 y12 y11 y13 ncf12 ncf11 ncf13 cep12 cep11 cep13).  Per workload: ms per call and frames
per second, the kernel's own time (torch.profiler, a separate run), the FFT rate counting 2.5 N log2 N flops per real
N-point transform (per frame: PEF one of 2n points and two of L points, YIN three of n points, NCF / CEP two of 2n
points), compulsory bytes (clips in; fre out, and YIN's value1 and value2) and their share of 3.35 TB/s, a parity gate
on clip 0 against the float64 oracle, the card's name, power limit and max SM clock, and where oracle/_ref exists the
reference build's time per clip on one CPU core.  Prints one JSON line per workload.  torch.profiler stops reporting
kernels after about five profiled workloads in one process, so run one tracker per call to get every kernel time.

    python tools/bench_pitch.py [--steps 20] [--warmup 3] [--workloads p12,y12,ncf12] [--out results.json]"""
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.realpath(__file__)))
import _bench_kit as K  # noqa: E402

import torch  # noqa: E402

import audioflux_b200 as af  # noqa: E402
import _pitch_c as PC  # noqa: E402
import _pitch_ncf_cep_oracle as NO  # noqa: E402
import _pitch_pef_oracle as PO  # noqa: E402
import _pitch_yin_oracle as YO  # noqa: E402

SIZES = {
    "12": dict(radix2_exp=12, clips=1024, length=160000, sr=32000, slide=1024, auto=2048),
    "11": dict(radix2_exp=11, clips=1024, length=110250, sr=22050, slide=512, auto=1024),
    "13": dict(radix2_exp=13, clips=64, length=2646000, sr=44100, slide=2048, auto=4096),
}


def _pef(w, n):
    p = PO.params(sr=w["sr"], r2=w["radix2_exp"], slide=w["slide"], lf=32.0, hf=2000.0, cf=4000.0)
    need = max(p["pad"] + 2 * n, n + p["max_index"] + 1)
    L = 1 << math.ceil(math.log2(need))                   # the kernel's correlation length (kernels/pitch_pef.cu)
    return p, dict(correlation_length=L), 2.5 * 2 * n * (w["radix2_exp"] + 1) + 2 * 2.5 * L * math.log2(L)


def _agree(O):
    def parity(out, x, p):
        want, cands = O.pitch(x, p)
        ok, alt = O.agree(out[0].cpu().numpy(), want, cands, p)
        return ok, alt, {}
    return parity


def _yin_parity(out, x, p):
    ok, msg, alt = YO.check(*(o[0].cpu().numpy() for o in out), YO.pitch(x, p), p, 0.0)
    return ok, alt, dict(parity_message=msg)


# per tracker: the class and its arguments; the C constructor's arguments for the reference timing; the oracle's
# parameters, extra result fields and FFT flops per frame; the parity check; the kernel; the output planes
TRACKERS = {
    "p": dict(kind="pef", cls=lambda w: af.PitchPEF(samplate=w["sr"], radix2_exp=w["radix2_exp"],
                                                    slide_length=w["slide"]),
              ctor=lambda w: dict(sr=w["sr"], r2=w["radix2_exp"], slide=w["slide"]),
              model=_pef, parity=_agree(PO), kernel="k_pitch_pef", planes=1),
    "y": dict(kind="yin", cls=lambda w: af.PitchYIN(samplate=w["sr"], radix2_exp=w["radix2_exp"],
                                                    slide_length=w["slide"], auto_length=w["auto"]),
              ctor=lambda w: dict(sr=w["sr"], lf=27.0, hf=2000.0, r2=w["radix2_exp"], slide=w["slide"], auto=w["auto"]),
              model=lambda w, n: (YO.params(**TRACKERS["y"]["ctor"](w)), dict(auto=w["auto"]),
                                  3 * 2.5 * n * w["radix2_exp"]),
              parity=_yin_parity, kernel="k_pitch_yin", planes=3),
}
for _t, _cls in (("ncf", af.PitchNCF), ("cep", af.PitchCEP)):
    TRACKERS[_t] = dict(kind=_t, cls=lambda w, c=_cls: c(samplate=w["sr"], radix2_exp=w["radix2_exp"],
                                                         slide_length=w["slide"]),
                        ctor=lambda w: dict(sr=w["sr"], lf=32.0, hf=2000.0, r2=w["radix2_exp"], slide=w["slide"]),
                        model=lambda w, n, t=_t: (NO.params(t, **TRACKERS[t]["ctor"](w)), {},
                                                  2 * 2.5 * (2 * n) * (w["radix2_exp"] + 1)),
                        parity=_agree(NO), kernel=f"k_pitch_{_t}", planes=1)
WORKLOADS = {t + size: (t, w) for t in TRACKERS for size, w in SIZES.items()}


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


def reference_ms_per_clip(kind, ctor, x, clips=1):
    def prepare(lib):
        def clip(i):
            st, o = PC.c_new(lib, kind, **ctor)
            PC.c_pitch(lib, kind, o, x[i])
            PC.c_free(lib, kind, o)
        return clip
    return K.reference_ms_per_clip(prepare, clips)      # construction included


def run(name, steps, warmup):
    t, w = WORKLOADS[name]
    tr = TRACKERS[t]
    r, B, length = w["radix2_exp"], w["clips"], w["length"]
    n = 1 << r
    obj = tr["cls"](w)
    p, extra, frame_flop = tr["model"](w, n)
    T = obj.cal_time_length(length)
    x = clips(w)
    xd = torch.from_numpy(x).cuda()

    def fn():
        return obj.pitch_batch(xd)
    times, out = K.event_times(fn, steps, warmup)
    ms = float(np.median(times))
    ok, alt, message = tr["parity"](out, x[0], p)
    del out
    kname = tr["kernel"]
    per = K.kernel_times(fn, (kname,), per_launch=True)                 # one launch per call
    nbytes = B * length * 4 + tr["planes"] * B * T * 4
    flop = frame_flop * T * B
    res = dict(workload=name, clips=B, samples=length, samplate=w["sr"], frame=n, slide=w["slide"], **extra,
               lags=[p["min_index"], p["max_index"]], frames=T * B, **K.ms_stats(times, 4),
               frames_per_s=round(T * B / (ms * 1e-3)), kernels_ms={k: round(v, 4) for k, v in per.items()},
               compulsory_bytes=nbytes, hbm_share=round(nbytes / (ms * 1e-3) / K.HBM, 5),
               fft_tflops=round(flop / (ms * 1e-3) / 1e12, 3),
               parity_undetermined_frames_clip0=len(alt), parity_ok=bool(ok), **message, card=K.card())
    k = per.get(kname)
    if k:
        res[f"{kname}_tflops"] = round(flop / (k * 1e-3) / 1e12, 3)
        res[f"{kname}_hbm_share"] = round(nbytes / (k * 1e-3) / K.HBM, 5)
    res["reference_ms_per_clip_1core"] = reference_ms_per_clip(tr["kind"], tr["ctor"](w), x)
    return res


if __name__ == "__main__":
    K.main(run, ",".join(WORKLOADS), steps=20, warmup=3)
