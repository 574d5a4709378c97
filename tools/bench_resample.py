"""Resampler throughput on the device (device-resident seeded clips of 5 s at the source rate, 1024 per call,
CUDA-event timing, median of the timed calls after warm-up):

  best_48k_16k   Best quality, 48 000 -> 16 000
  mid_48k_16k    Mid quality,  48 000 -> 16 000
  fast_48k_16k   Fast quality, 48 000 -> 16 000
  best_44k_16k   Best quality, 44 100 -> 16 000
  best_16k_48k   Best quality, 16 000 -> 48 000

Per workload: ms per call, the kernel's own time (torch.profiler, a separate run), output samples and taps per second
(taps counted with the reference's tap-count rule), the compulsory HBM bytes (clips in, outputs out) over kernel time and
their share of 3.35 TB/s, a parity gate on clip 0 against the float64 oracle, the card's name, power limit and max SM
clock, and where oracle/_ref exists the reference build's time per clip on one CPU core.  Prints one JSON line per
workload.

    python tools/bench_resample.py [--steps 20] [--warmup 3] [--workloads best_48k_16k,...] [--out results.json]"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.realpath(__file__)))
import _bench_kit as K  # noqa: E402

import torch  # noqa: E402

import audioflux_b200 as af  # noqa: E402
import _resample_oracle as RO  # noqa: E402

CLIPS = 1024
WORKLOADS = {
    "best_48k_16k": dict(qual=0, src=48000, dst=16000),
    "mid_48k_16k": dict(qual=1, src=48000, dst=16000),
    "fast_48k_16k": dict(qual=2, src=48000, dst=16000),
    "best_44k_16k": dict(qual=0, src=44100, dst=16000),
    "best_16k_48k": dict(qual=0, src=16000, dst=48000),
}


def reference_ms_per_clip(w, x, clips=2):
    def prepare(lib):
        def clip(i):                       # construction included, as a user pays it
            st, o = RO.c_new(lib, w["qual"])
            lib.resampleObj_setSamplate(o, w["src"], w["dst"])
            RO.c_resample(lib, o, x[i])
            lib.resampleObj_free(o)
        return clip
    return K.reference_ms_per_clip(prepare, clips)


def run(name, steps, warmup):
    w = WORKLOADS[name]
    length = 5 * w["src"]
    obj = af.Resample(af.ResampleQualityType(w["qual"]))
    obj.set_samplate(w["src"], w["dst"])
    m = obj.cal_data_length(length)
    rng = np.random.default_rng(0)
    x = (0.1 * rng.standard_normal((CLIPS, length))).astype(np.float32)
    x[0] = RO.case_signal(name, dict(length=length))
    xd = torch.from_numpy(x).cuda()

    def fn():
        return obj.resample_batch(xd)
    times, out = K.event_times(fn, steps, warmup)
    ms = float(np.median(times))
    o = RO.Resampler(w["qual"])
    o.set_samplate(w["src"], w["dst"])
    want = o.resample(x[0])
    got = out[0].cpu().numpy()
    err = float(np.abs(got - want).max() / np.abs(want).max())
    del out
    per = K.kernel_times(fn, ("k_resample",), per_launch=True)
    taps = int(o.taps(length).sum()) * CLIPS
    nbytes = CLIPS * (length + m) * 4
    res = dict(workload=name, clips=CLIPS, samples=length, outputs=m, quality=w["qual"], rates=[w["src"], w["dst"]],
               **K.ms_stats(times, 4),
               kernels_ms={k: round(v, 4) for k, v in per.items()},
               taps_per_output=round(taps / (CLIPS * m), 2),
               outputs_per_s=round(CLIPS * m / (ms * 1e-3), 1), taps_per_s=round(taps / (ms * 1e-3), 1),
               compulsory_bytes=nbytes, parity_clip0=err, parity_ok=bool(err <= 1e-4), card=K.card())
    k = per.get("k_resample")
    if k:
        res["k_resample_hbm_share"] = round(nbytes / (k * 1e-3) / K.HBM, 4)
        res["k_resample_taps_per_s"] = round(taps / (k * 1e-3), 1)
    res["reference_ms_per_clip_1core"] = reference_ms_per_clip(w, x)
    return res


if __name__ == "__main__":
    K.main(run, ",".join(WORKLOADS), steps=20, warmup=3)
