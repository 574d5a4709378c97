"""Harmonic-percussive separation throughput on the device (device-resident seeded clips, CUDA-event timing, median of
the timed calls after warm-up):

  n12_32k       1024 clips of 5 s at 32 kHz, fftLength 2^12, hOrder 21 / pOrder 31 (the defaults)
  n11_22k       1024 clips of 5 s at 22.05 kHz, fftLength 2^11, defaults
  n12_44k_60s   64 clips of 60 s at 44.1 kHz, fftLength 2^12, hOrder 31 / pOrder 31

Per workload: ms per call; per-kernel device time per call from torch.profiler (a separate run): the STFT, the mask
kernel and the two inverse STFTs; the compulsory HBM bytes of the call (clips in, h and p out) and of the mask kernel
(two half-spectrum planes in, four out) over their times; the window elements the two medians visit per bin (runs of 32
outputs: the first window's rank counts, at most order^2, then one pass of order elements per output) beside the
order_h^2 + order_p^2 of a rank count at every output; a parity gate on clip 0 against the float64 oracle; the card's
name, power limit and max SM clock; and where oracle/_ref exists the reference build's time per clip on one CPU core.
Prints one JSON line per workload.

    python tools/bench_hpss.py [--steps 10] [--warmup 2] [--workloads n12_32k,...] [--out results.json]"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.realpath(__file__)))
import _bench_kit as K  # noqa: E402

import torch  # noqa: E402

import audioflux_b200 as af  # noqa: E402
import _hpss_oracle as HO  # noqa: E402

RUN = 32                     # outputs per median run of k_hpss_mask (its frame tile and its bin run)
WORKLOADS = {
    "n12_32k": dict(clips=1024, seconds=5, sr=32000, r=12, h=21, p=31),
    "n11_22k": dict(clips=1024, seconds=5, sr=22050, r=11, h=21, p=31),
    "n12_44k_60s": dict(clips=64, seconds=60, sr=44100, r=12, h=31, p=31),
}
KERNELS = ("k_hpss_mask", "k_stft_generic", "k_istft_frames", "k_istft_ola")


def median_visits(order):
    """window elements visited per output along one axis: a run's first window by rank counts (at most order^2), then
    one pass of order elements for each of the other RUN - 1 outputs; an order of 1 visits nothing"""
    return 0.0 if order == 1 else (order * order + (RUN - 1) * order) / RUN


def reference_ms_per_clip(w, x, clips=1):
    def prepare(lib):
        def clip(i):                       # construction included, as a user pays it
            st, o = HO.c_new(lib, w["r"], None, None, w["h"], w["p"])
            HO.c_hpss(lib, o, x[i])
            lib.hpssObj_free(o)
        return clip
    return K.reference_ms_per_clip(prepare, clips)


def run(name, steps, warmup):
    w = WORKLOADS[name]
    length, clips, n = w["seconds"] * w["sr"], w["clips"], 1 << w["r"]
    obj = af.HPSS(radix2_exp=w["r"], h_order=w["h"], p_order=w["p"])
    m = obj.cal_data_length(length)
    T, W = HO.time_length(length, n), n // 2 + 1
    rng = np.random.default_rng(0)
    x = (0.1 * rng.standard_normal((clips, length))).astype(np.float32)
    x[0] = HO.case_signal(name, dict(length=length))
    xd = torch.from_numpy(x).cuda()

    def fn():
        return obj.hpss_batch(xd)
    times, out = K.event_times(fn, steps, warmup)
    ms = float(np.median(times))
    want = HO.hpss(x[0], w["r"], w["h"], w["p"])
    kw = dict(radix2_exp=w["r"], length=length)
    err = max(max(HO.errors(out[k][0].cpu().numpy(), want[k], kw)) for k in range(2))
    del out
    per = K.kernel_times(fn, KERNELS)
    bins = clips * T * W
    call_bytes = clips * (length + 2 * m) * 4
    mask_bytes = bins * 6 * 4
    res = dict(workload=name, clips=clips, samples=length, frames=T, bins_per_frame=W, fft_length=n,
               orders=[w["h"], w["p"]], **K.ms_stats(times, 3),
               kernels_ms_per_call={k: round(v, 3) for k, v in per.items()},
               call_compulsory_bytes=call_bytes, call_GBps=round(call_bytes / (ms * 1e-3) / 1e9, 1),
               median_visits_per_bin=round(median_visits(w["h"]) + median_visits(w["p"]), 1),
               rank_count_per_bin=w["h"] ** 2 + w["p"] ** 2, parity_clip0=err, parity_ok=bool(err <= 1e-4), card=K.card())
    k = per.get("k_hpss_mask")
    if k:
        res["mask_compulsory_bytes"] = mask_bytes
        res["mask_GBps"] = round(mask_bytes / (k * 1e-3) / 1e9, 1)
        res["mask_hbm_share"] = round(mask_bytes / (k * 1e-3) / K.HBM, 4)
        res["stft_istft_ms_per_call"] = round(sum(v for kk, v in per.items() if kk in KERNELS[1:]), 3)
    res["reference_ms_per_clip_1core"] = reference_ms_per_clip(w, x)
    return res


if __name__ == "__main__":
    K.main(run, ",".join(WORKLOADS), steps=10, warmup=2)
