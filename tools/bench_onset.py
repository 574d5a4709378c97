"""Onset detection throughput on the device (device-resident spectrograms of seeded clips, CUDA-event timing, median of
the timed calls after warm-up):

  mel_flux     1024 clips of 5 s at 32 kHz, hop 512: 128-band mel power spectrogram in dB (af.BFT, fftLength 2^12), FLUX
               with the reference Python's default NoveltyParam, filter order 1
  linear_pd    the same clips as a 2049-bin linear magnitude + phase (fftLength 2^12, hop 512), PD, filter order 3

Per workload: ms per onset_batch call; per-kernel device time per call from torch.profiler (a separate run): the max
filter, the novelty (k_spectral) and the peak picking; the compulsory HBM bytes of the call (spectrogram and phase in;
evn, points and counts out) over its time and as a share of the H100 SXM's 3.35 TB/s; a parity gate on clip 0 (evn
within 1e-4 of the numpy oracle, points exactly the oracle's peak picking of the GPU's own evn); the card's name, power
limit and max SM clock; and where oracle/_ref exists the reference build's time per clip on one CPU core.
Prints one JSON line per workload.

    python tools/bench_onset.py [--steps 10] [--warmup 2] [--workloads mel_flux,linear_pd] [--out results.json]"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.realpath(__file__)))
import _bench_kit as K  # noqa: E402

import torch  # noqa: E402

import audioflux_b200 as af  # noqa: E402
import _onset_oracle as OO  # noqa: E402

SR, SECONDS, HOP, R = 32000, 5, 512, 12
WORKLOADS = {
    "mel_flux": dict(clips=1024, kind=af.NoveltyType.FLUX, order=1),
    "linear_pd": dict(clips=1024, kind=af.NoveltyType.PD, order=3),
}
KERNELS = ("k_onset_maxfilter", "k_spectral", "k_onset_pick")


def clips(n):
    """n seeded clips: noise with a decaying tone burst every 0.3 s (clip 0 shifted per clip)"""
    rng = np.random.default_rng(0)
    length = SR * SECONDS
    x = (0.02 * rng.standard_normal((n, length))).astype(np.float32)
    t = np.arange(2000)
    burst = (np.sin(2 * np.pi * 440 * t / SR) * np.exp(-t / 400)).astype(np.float32)
    for k in range(0, length - 2000, 9600):
        x[:, k:k + 2000] += burst
    return x


def spectrograms(name, x):
    """device spectrograms [clips, T, bins] (and phase) of the workload"""
    xd = torch.from_numpy(x).cuda()
    if name == "mel_flux":
        b = af.BFT(num=128, radix2_exp=R, samplate=SR, slide_length=HOP,
                   scale_type=af.SpectralFilterBankScaleType.MEL, data_type=af.SpectralDataType.POWER)
        p = b.bft_batch(xd, result_type=1)                                   # [clips, T, 128]
        db = 10 * torch.log10(p / p.amax(dim=(1, 2), keepdim=True))
        return torch.clamp(db, min=-80.0).contiguous(), None
    mags, phs = [], []
    win = torch.hann_window(1 << R, device="cuda")
    for c0 in range(0, len(xd), 128):
        s = torch.stft(xd[c0:c0 + 128], 1 << R, HOP, window=win, center=False, return_complex=True).transpose(1, 2)
        mags.append(s.abs().contiguous())
        phs.append(s.angle().float().contiguous())
        del s
    return torch.cat(mags), torch.cat(phs)


def reference_ms_per_clip(w, spec, phase, clips=3):
    T, M = spec.shape[1], spec.shape[2]

    def prepare(lib):
        def clip(i):                       # construction included, as a user pays it
            st, o = OO.c_new(lib, T, M, HOP, SR, w["order"], w["kind"].value)
            OO.c_onset(lib, o, spec[i], None if phase is None else phase[i])
            lib.onsetObj_free(o)
        return clip
    return K.reference_ms_per_clip(prepare, clips)


def run(name, steps, warmup):
    w = WORKLOADS[name]
    x = clips(w["clips"])
    spec, phase = spectrograms(name, x)
    n, T, M = spec.shape
    obj = af.Onset(time_length=T, fre_length=M, slide_length=HOP, samplate=SR, filter_order=w["order"],
                   novelty_type=w["kind"])

    def fn():
        return obj.onset_batch(spec, phase)
    times, out = K.event_times(fn, steps, warmup)
    ms = float(np.median(times))
    evn, pts, counts = (t.cpu().numpy() for t in out)
    del out
    pp = OO.peak_params(SR, HOP)
    s0, p0 = spec[0].cpu().numpy(), None if phase is None else phase[0].cpu().numpy()
    want, _ = OO.onset(s0, p0, w["kind"].value, w["order"], OO.DEFAULT_PARAM, None, pp)
    err = float(np.abs(evn[0].astype(np.float64) - want).max())
    pick_ok = bool(np.array_equal(OO.pick(evn[0], pp), pts[0][:counts[0]]))
    per = K.kernel_times(fn, KERNELS)
    planes = 1 if phase is None else 2
    call_bytes = n * T * M * 4 * planes + n * T * 8 + n * 4
    res = dict(workload=name, clips=n, frames=T, bins=M, novelty=w["kind"].name, filter_order=w["order"],
               **K.ms_stats(times, 3), kernels_ms_per_call={k: round(v, 3) for k, v in per.items()},
               call_compulsory_bytes=call_bytes, call_GBps=round(call_bytes / (ms * 1e-3) / 1e9, 1),
               call_hbm_share=round(call_bytes / (ms * 1e-3) / K.HBM, 4),
               points_per_clip=round(float(counts.mean()), 1), parity_clip0=err, pick_exact_clip0=pick_ok,
               parity_ok=bool(err <= 1e-4 and pick_ok), card=K.card())
    sh, ph = spec[:3].cpu().numpy(), None if phase is None else phase[:3].cpu().numpy()
    res["reference_ms_per_clip_1core"] = reference_ms_per_clip(w, sh, ph)
    return res


if __name__ == "__main__":
    K.main(run, ",".join(WORKLOADS), steps=10, warmup=2)
