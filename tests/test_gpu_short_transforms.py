"""The shared-memory STFT / ISTFT frames (2^1 .. 2^14 points) and every CWT / PWT length outside the 2^19 fast path,
row by row against the float64 oracle.

The counterpart of test_gpu_long_transforms.py, with its per-row bar (`check_rows`): every output row -- one frame, or
one scale of one clip -- must be within 1e-4 of that row's own max |want|, and rows the oracle gives as exactly zero
must come out zero.  Covered here:

  - STFT frames, every size 2^1 .. 2^14: k_stft_n2 (n = 2), the 32-thread floor (n <= 128), the radix-2 tail of the
    Stockham passes (odd log2(n/2)), the shared-memory opt-in (n >= 8192) and two butterflies per thread (16384); FULL
    planes through the legacy entry, HALF planes through the batched one, the SQUARE / POWER / MAG store modes through
    BFT on the Linear scale (always the composed path: the bins reach the output through k_copy_cols or the 0/1 bank),
    and the three padding modes.
  - ISTFT frames, every size 2^1 .. 2^14 (k_istft_frames, k_istft_frames_inplace at 16384, k_istft_ola), both methods,
    HALF and FULL planes, non-Hermitian FULL planes, hops below, at and above the frame length.  The bar is per output
    sample (see `check_istft`).
  - CWT, every length 2^1 .. 2^24 except the 2^19 fast path: the single leg (N <= 2^12) and the four-step legs with every
    tile shape `fill_params` picks, padded at 2^2 .. 2^16, all eight wavelet families, six scales, the derivative
    transform; PWT's tabulated bank rows at the single-leg and rows-kernel crops.

Inputs make a mixed-up clip or frame index show: 3 clips per call (2 at CWT lengths 2^21 .. 2^24), the middle one 1000x
louder and reversed.  STFT / ISTFT clips join sections of loud noise, tones at 1e-3, noise at 1e-6 and exact zeros, each
at least 2n + hop samples long, so frames of every level and all-zero frames exist.  CWT / PWT clips are white noise
(quiet rows occur naturally) and tones.
"""
import numpy as np
import pytest

import audioflux_b200 as af
from audioflux_b200.base import Batch
from audioflux_b200.lib import AfB200Error
from conftest import noise, rel_max, tones
from oracle import af_oracle as O
from test_gpu_long_transforms import check_rows, cwt_bank, cwt_oracle, pwt_oracle
from test_gpu_long_transforms import report, torch_cuda  # noqa: F401 (fixtures)
from test_next_rows_cpu import istft_conditioned

pytestmark = pytest.mark.gpu

TOL = 1e-4
SR = 48000
W, S, D, WIN = af.WaveletContinueType, af.SpectralFilterBankScaleType, af.SpectralDataType, af.WindowType
PADPOS, PADMODE = af.PaddingPositionType, af.PaddingModeType
USER = "user"                                   # a window handed over with use_window_data_arr


def sectioned(seed, n, hop):
    """Loud noise, tones at 1e-3, noise at 1e-6, exact zeros, loud noise: every section at least 2n + hop samples, so
    frames lie in each level and at least one frame is all zero."""
    sec = max(2 * n + hop, 64)
    rng = np.random.default_rng(seed)
    t = np.arange(sec)
    parts = [0.5 * rng.standard_normal(sec),
             1e-3 * (np.sin(2 * np.pi * 0.0371 * t) + np.sin(2 * np.pi * 0.213 * t + 1.0)),
             1e-6 * rng.standard_normal(sec),
             np.zeros(sec),
             0.5 * rng.standard_normal(sec)]
    return np.concatenate(parts).astype(np.float32)


def three_clips(seed, n, hop):
    """3 clips, the middle one 1000x louder and reversed."""
    return np.stack([sectioned(seed, n, hop), 1000 * sectioned(seed + 1, n, hop)[::-1], sectioned(seed + 2, n, hop)])


def window_of(wt, n, seed=0):
    if wt == USER:
        return np.random.default_rng(1000 + seed).uniform(0.1, 1.0, n).astype(np.float32)
    return O.fft_window(af.enum_value(wt), n)


def stft_object(r, wt, hop):
    n = 1 << r
    if wt == USER:
        s = af.STFT(r, WIN.RECT, hop)
        s.use_window_data_arr(window_of(USER, n, r))
    else:
        s = af.STFT(r, wt, hop)
    return s


# ------------------------------------------------------------------ 1. STFT frames, n = 2^1 .. 2^14
# Two cases per size: one hop below n, one at n, above n (frames with gaps between them) or not dividing n.
STFT_CASES = [(1, WIN.RECT, 1), (1, WIN.HANN, 3),
              (2, WIN.HAMM, 1), (2, WIN.RECT, 4),
              (3, WIN.BLACKMAN, 3), (3, USER, 8),
              (4, WIN.HANN, 4), (4, WIN.BLACKMAN, 20),
              (5, USER, 8), (5, WIN.HAMM, 32),
              (6, WIN.RECT, 48), (6, WIN.HANN, 100),
              (7, WIN.HAMM, 32), (7, WIN.RECT, 128),
              (8, WIN.BLACKMAN, 100), (8, WIN.HANN, 300),
              (9, WIN.HANN, 128), (9, USER, 512),
              (10, WIN.RECT, 256), (10, WIN.HAMM, 1500),
              (11, WIN.HAMM, 512), (11, WIN.BLACKMAN, 2048),
              (12, USER, 1000), (12, WIN.HANN, 5000),
              (13, WIN.HANN, 2048), (13, WIN.RECT, 8192),
              (14, WIN.BLACKMAN, 4096), (14, WIN.HAMM, 20000)]


def _win_name(wt):
    return wt if wt == USER else wt.name


@pytest.mark.parametrize("r,wt,hop", STFT_CASES, ids=[f"2^{r}-{_win_name(w)}-hop{h}" for r, w, h in STFT_CASES])
def test_stft_frames_rows(torch_cuda, report, r, wt, hop):
    torch = torch_cuda
    n = 1 << r
    x = three_clips(300 + r, n, hop)
    s = stft_object(r, wt, hop)
    win = window_of(wt, n, r)
    half_re, half_im = s.stft_batch(torch.from_numpy(x).cuda())
    for b in range(3):
        wr, wi = O.stft(x[b], n, hop, win)
        re, im = s.stft_planes(x[b])
        zero = check_rows(report, f"full clip {b}", re, im, wr, wi)
        check_rows(report, f"half clip {b}", half_re[b], half_im[b], wr[:, :n // 2 + 1], wi[:, :n // 2 + 1])
        assert zero.any(), "no all-zero frame: the input does not test the zero rows"


@pytest.mark.parametrize("mode", [PADMODE.CONSTANT, PADMODE.REFLECT, PADMODE.WRAP], ids=lambda m: m.name)
def test_stft_padded_short_clip_2pow14(torch_cuda, report, mode):
    """Centre padding of n/2 = 8192 samples on each side of 2048 valid samples (3000 minus the tail past the last hop):
    the reflect and wrap extensions go round the data several times; constant padding with two non-zero values."""
    torch = torch_cuda
    r, hop, L = 14, 1024, 3000
    n = 1 << r
    x = np.stack([noise(330, L), 1000 * noise(331, L)[::-1], tones(332, L, SR)])
    v1, v2 = (0.25, -0.5) if mode == PADMODE.CONSTANT else (0.0, 0.0)
    s = af.STFT(r, WIN.HANN, hop)
    s.enable_padding(True)
    s.set_padding(PADPOS.CENTER, mode, v1, v2)
    assert s.cal_time_length(L) == L // hop + 1
    half_re, half_im = s.stft_batch(torch.from_numpy(np.ascontiguousarray(x)).cuda())
    for b in range(3):
        wr, wi = O.stft(x[b], n, hop, O.fft_window(O.W_HANN, n), is_pad=True, position=O.PAD_CENTER,
                        mode=af.enum_value(mode), value1=v1, value2=v2)
        re, im = s.stft_planes(x[b])
        check_rows(report, f"full clip {b}", re, im, wr, wi)
        check_rows(report, f"half clip {b}", half_re[b], half_im[b], wr[:, :n // 2 + 1], wi[:, :n // 2 + 1])


# ------------------------------------------------------------------ 1b. store modes through BFT on the Linear scale
# (result_type, data_type, normValue): real POWER with and without the powf, real MAG with and without the bank's
# post-power, complex POWER (the SQUARE store) and complex MAG (the HALF store)
BFT_MODES = [(1, D.POWER, 1.0), (1, D.POWER, 0.5), (1, D.MAG, 1.0), (1, D.MAG, 2.0), (0, D.POWER, 1.0), (0, D.MAG, 1.0)]
BFT_MODE_IDS = ["power", "power-norm0.5", "mag", "mag-norm2", "complex-square", "complex-half"]


@pytest.mark.parametrize("rt,dt,nv", BFT_MODES, ids=BFT_MODE_IDS)
@pytest.mark.parametrize("r", [1, 2, 4, 7, 11, 13, 14], ids=lambda r: f"2^{r}")
def test_bft_linear_store_modes_rows(torch_cuda, report, r, rt, dt, nv):
    """Every bin 0 .. n/2 of every frame (num = n/2 + 1 from 0 Hz), against O.bft; complex rows as complex values."""
    torch = torch_cuda
    n = 1 << r
    hop = max(1, n // 4)
    num = n // 2 + 1
    x = three_clips(340 + r, n, hop)
    b = af.BFT(num, r, SR, window_type=WIN.HANN, slide_length=hop, scale_type=S.LINEAR, data_type=dt)
    if nv != 1.0:
        b.set_data_norm_value(nv)
    got = b.bft_batch(torch.from_numpy(x).cuda(), result_type=rt)
    for i in range(3):
        want = O.bft(x[i], num, r, SR, hop, O.W_HANN, O.SCALE_LINEAR, O.STYLE_SLANEY, O.NORM_NONE, af.enum_value(dt),
                     result_type=rt, norm_value=nv)
        if rt == 0:
            zero = check_rows(report, f"clip {i}", got[0][i], got[1][i], *want)
        else:
            zero = check_rows(report, f"clip {i}", got[i], None, want, None)
        assert zero.any()


# ------------------------------------------------------------------ 2. ISTFT frames, n = 2^1 .. 2^14
def check_istft(report, case, got, re, im, n, hop, window, method):
    """Per output sample: |got - want| <= 1e-4 * (the largest |Re IFFT| of the frames covering the sample) / (the
    sample's window-sum normaliser), instead of the clip's maximum.  Samples that only all-zero frames cover (or no
    frame: gaps of hop > n) must be exactly 0.  Where the normaliser is ill-conditioned (istft_conditioned) the bound
    is 1e-2 of the clip's max |want|, as elsewhere in the suite."""
    got = np.asarray(got, dtype=np.float64)
    T = re.shape[0]
    y = np.fft.ifft(np.asarray(re, np.float64) + 1j * np.asarray(im, np.float64), axis=1).real
    peak = np.abs(y).max(axis=1)
    w = np.asarray(window, dtype=np.float64) ** (2 if method == 0 else 1)
    L = (T - 1) * hop + n
    norm, cover = np.zeros(L), np.zeros(L)
    for t in range(T):
        sl = slice(t * hop, t * hop + n)
        norm[sl] += w
        cover[sl] = np.maximum(cover[sl], peak[t])
    norm[norm < 1e-6] = 1.0
    want = O.istft(re, im, n, hop, window, method).astype(np.float64)
    assert got.shape == want.shape
    err = np.abs(got - want)
    ok = istft_conditioned(n, hop, T, window, method)
    scale = cover / norm
    live = scale > 0
    tight = ok & live
    rel = err[tight] / scale[tight]
    worst = float(rel.max()) if rel.size else 0.0
    report(case, worst, rel_max(got, want))
    assert worst < TOL, (case, "samples above the per-sample bar", np.nonzero(tight)[0][rel >= TOL][:20].tolist())
    assert not (~live).any() or np.abs(got[~live]).max() == 0, (case, "samples of all-zero frames are not 0")
    loose = ~ok & live
    assert not loose.any() or err[loose].max() <= 1e-2 * np.abs(want).max(), (case, "ill-conditioned samples")
    return ~live


# methods 0 ('weight') and 1 ('overlap-add') at every size; hops below, at and (2^14) above the frame length.  Overlap-add
# at hop = n divides each sample by the window value alone: with a window that reaches 0 (Hann at 2^12: 6e-7 next to
# the edge) float32 rounding of the frame divided by it is 2.6e-2 of the clip's peak, beyond the bound for
# ill-conditioned samples, so those cases use the Rect and Hamming windows.
ISTFT_CASES = [(1, WIN.HANN, 1, 0), (1, WIN.RECT, 2, 1),
               (2, WIN.HAMM, 1, 0), (2, WIN.HANN, 3, 1),
               (3, WIN.RECT, 8, 0), (3, WIN.HAMM, 2, 1),
               (4, WIN.HANN, 4, 0), (4, WIN.BLACKMAN, 16, 1),
               (5, WIN.BLACKMAN, 8, 0), (5, WIN.HANN, 12, 1),
               (6, WIN.HAMM, 16, 0), (6, WIN.RECT, 64, 1),
               (7, WIN.HANN, 32, 0), (7, WIN.HAMM, 100, 1),
               (8, WIN.RECT, 256, 0), (8, WIN.HANN, 64, 1),
               (9, WIN.HANN, 128, 0), (9, WIN.BLACKMAN, 200, 1),
               (10, WIN.BLACKMAN, 256, 0), (10, WIN.HANN, 512, 1),
               (11, WIN.HANN, 512, 0), (11, WIN.RECT, 1500, 1),
               (12, WIN.HANN, 1024, 0), (12, WIN.HAMM, 4096, 1),
               (13, WIN.HANN, 2048, 0), (13, WIN.HAMM, 8192, 1),
               (14, WIN.HANN, 4096, 0), (14, WIN.RECT, 19384, 1)]


@pytest.mark.parametrize("r,wt,hop,method", ISTFT_CASES,
                         ids=[f"2^{r}-{w.name}-hop{h}-m{m}" for r, w, h, m in ISTFT_CASES])
def test_istft_frames_samples(torch_cuda, report, r, wt, hop, method):
    """Planes of the sectioned clips: HALF planes of all 3 clips through one batched device call, FULL planes of each
    clip through the legacy entry."""
    torch = torch_cuda
    n = 1 << r
    win = O.fft_window(af.enum_value(wt), n)
    x = three_clips(360 + r, n, hop)
    planes = [O.stft(x[b], n, hop, win) for b in range(3)]
    s = af.STFT(r, wt, hop)
    hre = torch.from_numpy(np.stack([p[0][:, :n // 2 + 1] for p in planes])).cuda()
    him = torch.from_numpy(np.stack([p[1][:, :n // 2 + 1] for p in planes])).cuda()
    half = s.istft_batch(hre, him, method).cpu().numpy()
    for b, (re, im) in enumerate(planes):
        check_istft(report, f"half clip {b}", half[b], re, im, n, hop, win, method)
        zero = check_istft(report, f"full clip {b}", s.istft_planes(re, im, method), re, im, n, hop, win, method)
        assert zero.any(), "no sample of all-zero frames: the input does not test them"


@pytest.mark.parametrize("r,method", [(6, 0), (13, 1), (14, 0)], ids=["2^6", "2^13", "2^14"])
def test_istft_non_hermitian_full_planes(torch_cuda, report, r, method):
    """Random re / im over all n bins: the library, like the reference, takes Re IFFT of whatever it is given.  Through
    the legacy entry and the batched entry with width n; 2^13 runs k_istft_frames, 2^14 k_istft_frames_inplace."""
    torch = torch_cuda
    n, T = 1 << r, 6
    hop = n // 4
    win = O.fft_window(O.W_HANN, n)
    rng = np.random.default_rng(370 + r)
    planes = [(rng.standard_normal((T, n)) * a).astype(np.float32) for a in (1.0, 1.0, 1e3, 1e3, 1e-3, 1e-3)]
    clips = [(planes[0], planes[1]), (planes[2], planes[3]), (planes[4], planes[5])]
    s = af.STFT(r, WIN.HANN, hop)
    batched = s.istft_batch(torch.from_numpy(np.stack([c[0] for c in clips])).cuda(),
                            torch.from_numpy(np.stack([c[1] for c in clips])).cuda(), method).cpu().numpy()
    for b, (re, im) in enumerate(clips):
        check_istft(report, f"full clip {b}", s.istft_planes(re, im, method), re, im, n, hop, win, method)
        check_istft(report, f"batched clip {b}", batched[b], re, im, n, hop, win, method)


# ------------------------------------------------------------------ 3. CWT, every length 2^1 .. 2^24 except 2^19
# fill_params: N <= 2^12 one leg (padded: FFT 2^(r+1), so padded r <= 11 crops in the single leg, 12 .. 16 in
# k_cwt_rows<1>); 2^13 .. 2^17 8 columns / 16 rows per CTA, 2^18 8 / 8, 2^20 4 / 4, 2^21 2 / 4, 2^22 2 / 2, 2^23 1 / 2,
# 2^24 1 / 1.
WAVELETS = [W.MORSE, W.MORLET, W.BUMP, W.PAUL, W.DOG, W.MEXICAN, W.HERMIT, W.RICKER]
SCALES = [S.OCTAVE, S.LINEAR, S.MEL, S.BARK, S.ERB, S.LOG]
CWT_NUM = {r: (1 << (r - 1)) + 1 for r in range(1, 8)}            # every band a short transform has: N/2 + 1
CWT_NUM.update({r: 60 for r in range(8, 19)})
CWT_NUM.update({20: 24, 21: 24, 22: 16, 23: 12, 24: 8})
DET = {(3, False), (12, True), (13, False), (17, False), (22, False), (24, False)}
# The families and scales take turns, except where that pair leaves the transform empty or puts a row near float32's
# subnormal range.  Up to 2^6 the Octave scale (from 16 Hz) leaves the bands of a few bins empty, and some families have
# no support on those bins.  A row whose peak is below 2^-126 / 1e-4 (a bank row of a single bin at 7e-39, say) has
# values where float32 keeps fewer than 24 bits, so no float32 pipeline holds it to 1e-4 of its own scale: measured,
# such rows of 2^6 padded Morlet-Octave (peak 4.7e-42) and 2^9 padded Morse-Erb (8.3e-42) are 3.0e-4 and 1.7e-4 off.
# `cwt_want` refuses them, so the pairs below are chosen to have none.
CHOSEN = {(1, False): (W.PAUL, S.MEL), (2, False): (W.DOG, S.BARK), (2, True): (W.MEXICAN, S.MEL),
          (3, False): (W.MORSE, S.LINEAR), (3, True): (W.RICKER, S.ERB), (4, False): (W.RICKER, S.LOG),
          (4, True): (W.HERMIT, S.ERB), (5, False): (W.BUMP, S.LINEAR), (5, True): (W.PAUL, S.BARK),
          (6, False): (W.MEXICAN, S.ERB), (6, True): (W.PAUL, S.OCTAVE), (9, True): (W.MORLET, S.ERB)}
QUIET_FLOOR = np.finfo(np.float32).tiny / TOL


def _cwt_cases():
    keys = sorted([(r, False) for r in range(1, 25) if r != 19] + [(r, True) for r in range(2, 17)])
    return [(r, pad, *CHOSEN.get((r, pad), (WAVELETS[i % 8], SCALES[i % 6])), CWT_NUM[r], (r, pad) in DET)
            for i, (r, pad) in enumerate(keys)]


CWT_CASES = _cwt_cases()
CWT_IDS = [f"2^{r}{'-pad' if pad else ''}-{w.name}-{s.name}-{num}{'-det' if det else ''}"
           for r, pad, w, s, num, det in CWT_CASES]


def cwt_clips(seed, r):
    """White noise, the same 1000x louder and reversed, and tones; 2 clips (noise, loud reversed tones) from 2^21 on."""
    N = 1 << r
    if r >= 21:
        return np.stack([noise(seed, N), 1000 * tones(seed + 1, N, SR)[::-1]])
    return np.stack([noise(seed, N), 1000 * noise(seed + 1, N)[::-1], tones(seed + 2, N, SR)])


def cwt_want(w, x, det, bank):
    """The oracle's rows, none of them between zero and QUIET_FLOOR."""
    re, im = cwt_oracle(w, x, det=det, bank=bank)
    peak = np.sqrt(re.astype(np.float64) ** 2 + im.astype(np.float64) ** 2).max(axis=1)
    assert not ((peak > 0) & (peak < QUIET_FLOOR)).any(), ("rows near float32's subnormal range", peak.min())
    return re, im


@pytest.mark.parametrize("r,pad,wav,scale,num,det", CWT_CASES, ids=CWT_IDS)
def test_cwt_rows(torch_cuda, report, r, pad, wav, scale, num, det):
    torch = torch_cuda
    x = cwt_clips(400 + r, r)
    w = af.CWT(num, r, SR, wavelet_type=wav, scale_type=scale, is_padding=pad)
    bank = cwt_bank(w)
    xd = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    if det:
        w.enable_det(True)
    for d in ([False, True] if det else [False]):
        re, im = (w.cwt_det_batch if d else w.cwt_batch)(xd)
        name = "det" if d else "cwt"
        for b in range(x.shape[0]):
            if r < 22:
                zero = check_rows(report, f"{name} clip {b}", re[b], im[b], *cwt_want(w, x[b], d, bank))
                assert not zero.all()
                continue
            step = (1 << 26) >> r                 # float64 planes of every scale would be GBs: 2^26 points at a time
            for s in range(0, num, step):
                check_rows(report, f"{name} clip {b} rows {s}..{s + step - 1}", re[b, s:s + step], im[b, s:s + step],
                           *cwt_want(w, x[b], d, bank[s:s + step]))
        del re, im


# ------------------------------------------------------------------ 4. PWT: tabulated bank rows
PWT_CASES = [(2, False, dict(num=3, scale_type=S.LINEAR)),
             (11, True, dict(num=60, scale_type=S.MEL, high_fre=16000.)),        # single-leg crop (FFT 2^12)
             (13, False, dict(num=84, scale_type=S.OCTAVE)),
             (16, True, dict(num=48, scale_type=S.BARK)),                        # FFT 2^17: the rows-kernel crop
             (21, False, dict(num=12, scale_type=S.MEL))]                        # 2 columns per CTA


@pytest.mark.parametrize("r,pad,kw", PWT_CASES, ids=[f"2^{r}{'-pad' if p else ''}" for r, p, _ in PWT_CASES])
def test_pwt_rows(torch_cuda, report, r, pad, kw):
    torch = torch_cuda
    x = cwt_clips(450 + r, r)
    p = af.PWT(radix2_exp=r, samplate=SR, is_padding=pad, **kw)
    p.enable_det(True)
    xd = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    for d in (False, True):
        re, im = (p.pwt_det_batch if d else p.pwt_batch)(xd)
        for b in range(x.shape[0]):
            check_rows(report, f"{'det' if d else 'pwt'} clip {b}", re[b], im[b], *pwt_oracle(p, x[b], det=d))
        del re, im


# ------------------------------------------------------------------ 5. the CWT length range
def test_cwt_pwt_2pow25_refused_outputs_untouched(torch_cuda):
    """radix2Exp 25 constructs (as in the reference) but the transform stops at 2^24: each call fails with a message
    and writes nothing."""
    torch = torch_cuda
    r = 25
    x = torch.zeros((1, 1 << r), dtype=torch.float32, device="cuda")
    objs = [(af.CWT(2, r, SR, scale_type=S.LINEAR, is_padding=False), ["cwtObj_cwtBatch", "cwtObj_cwtDetBatch"]),
            (af.PWT(2, r, SR, scale_type=S.LINEAR, is_padding=False), ["pwtObj_pwtBatch", "pwtObj_pwtDetBatch"])]
    for obj, names in objs:
        obj.enable_det(True)
        for name in names:
            re = torch.full((1, 2, 1 << r), 7.0, device="cuda")
            im = torch.full((1, 2, 1 << r), -7.0, device="cuda")
            b = Batch(x)
            with pytest.raises(AfB200Error, match=r"2\^25 is outside \[2\^1, 2\^24\]"):
                obj._call(name, b, b.x, b.rows, re, im)
            torch.cuda.synchronize()
            assert bool((re == 7.0).all()) and bool((im == -7.0).all()), name
            del re, im
