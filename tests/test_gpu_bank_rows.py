"""The general filter-bank, cepstral and temporal kernels of bank_xxcc.cu element by element against float64 oracles.

Every composed BFT / Spectrogram / MFCC / LFCC / GTCC / XXCC / chroma / cqcc call ends in one of k_bank_banded,
k_bank_dense, k_copy_cols, k_phase, k_xxcc, k_xxcc_standard, k_chroma or k_temporal.  The per-tensor bar says little
about one quiet band or one high cepstral coefficient of a smooth spectrum, and a bare relative bar is ill-conditioned
there.  So each kernel is fed the exact float32 input it consumed, and every output element is held to 1e-4 of its own
scale: the sum of the absolute values of the terms that make it up, pushed through the same operator.
  - bank: the band's sum |w| |P| over the plane P the bank consumed (the band value itself in real mode; ^postPow after);
  - DCT: the coefficient's sum |l_m D[m, c]| over the rectified row l;
  - delta / delta-delta: sum_j |b_j| scale(c_{i-j}) along the coefficient axis;
  - chroma: the class value itself (non-negative terms), then / norm;
  - temporal: the energy itself; the zero-crossing rate is exact (numpy's float32 products round as the device's do).
Elements whose scale is zero must be exactly zero, and the per-tensor bar holds as well.

Where the input comes from:
  - a bank's plane: a Linear BFT with num = n/2 + 1 from 0 Hz at the same fftLength, window, hop, data type and norm
    value makes the same af_launch_stft store, and its k_copy_cols output is that plane bit for bit (complex mode: the
    SQUARE or HALF planes).  `test_linear_plane_is_the_stft_store` pins that premise;
  - XXCC after a composed MFCC: the same object's bft_batch output;
  - XXCC, xxccStandard and chroma called directly: what the test passes.
Every call carries 3 clips (row groups), the middle one 1000x louder and reversed, so a mixed-up clip index shows.
Every bank case asserts the kernel it claims (banded iff nnz * 4 <= num * width, af_bft.c) and every MFCC case the
composed route before it compares.  The run prints the worst element per case.
"""
import numpy as np
import pytest

import audioflux_b200 as af
from conftest import noise, rel_max, tones
from oracle import af_oracle as O
from test_gpu_long_transforms import report  # noqa: F401  (fixture)

gpu = pytest.mark.gpu

TOL = 1e-4
SR = 32000
S, ST, D, WIN = af.SpectralFilterBankScaleType, af.SpectralFilterBankStyleType, af.SpectralDataType, af.WindowType
CR, CE, CN = af.CepstralRectifyType, af.CepstralEnergyType, af.ChromaDataNormalType
MFCC_COMPOSED = -1
TINY = 2.0 ** -149                      # the smallest float32 denormal


def check_elems(report, case, got, want, scale):
    """every element within TOL of its own scale, zero-scale elements exactly 0, and the per-tensor bar"""
    got = np.asarray(got.cpu().numpy() if hasattr(got, "cpu") else got, np.float64)
    want, scale = np.asarray(want, np.float64), np.asarray(scale, np.float64)
    assert got.shape == want.shape == scale.shape, (case, got.shape, want.shape, scale.shape)
    err = np.abs(got - want)
    live = scale > 0
    rel = err[live] / scale[live]
    worst = float(rel.max()) if rel.size else 0.0
    tensor = rel_max(got, want)
    report(case, worst, tensor)
    assert np.isfinite(got).all(), (case, "non-finite output")
    assert tensor < TOL, (case, "per tensor", tensor)
    bad = np.argwhere(live & (err > TOL * scale))
    assert bad.size == 0, (case, "elements above their own scale", bad[:10].tolist(),
                           (err[live & (err > TOL * scale)] / scale[live & (err > TOL * scale)])[:10].tolist())
    assert (got[~live] == 0).all(), (case, "zero-scale elements not zero", np.argwhere(~live & (got != 0))[:10].tolist())


def three(x):
    """3 clips or row groups for one call: the middle one 1000x louder and reversed"""
    x = np.stack([x[0], x[1][::-1] * np.float32(1e3), x[2]]) if len(x) == 3 else x
    return np.ascontiguousarray(x, np.float32)


def clips(n, hop, T, seed=0):
    L = (T - 1) * hop + n
    return three([tones(seed, L, SR), noise(seed + 1, L), tones(seed + 2, L, SR) * np.float32(1e-2)])


# ------------------------------------------------------------------ filter banks: k_bank_banded, k_bank_dense
def bank_support(bank):
    """(kernel the launcher picks, smallest band's tap count): support lengths as af_bands_build counts them"""
    lens = []
    for row in bank:
        nz = np.nonzero(row)[0]
        lens.append(int(nz[-1] - nz[0] + 1) if nz.size else 0)
    return ("banded" if sum(lens) * 4 <= bank.size else "dense"), min(lens)


def linear_source(b, data_type, norm):
    """the Linear BFT from 0 Hz whose output is the plane b's bank consumes"""
    n = b.fft_length
    lin = af.BFT(n // 2 + 1, b.radix2_exp, SR, low_fre=0.0, high_fre=SR / 2, window_type=b.window_type,
                 slide_length=b.slide_length, scale_type=S.LINEAR, data_type=data_type)
    assert np.array_equal(lin.get_bin_band_arr(), np.arange(n // 2 + 1))
    if norm is not None and data_type == D.POWER:      # POWER takes the norm value in the STFT store; MAG after the bank
        lin.set_data_norm_value(norm)
    return lin


# name: (num, radix2_exp, scale, style, kernel, smallest band's taps or None, bands reach (bin 0, Nyquist))
BANKS = {
    "mel2_r2": (2, 2, S.MEL, ST.SLANEY, "banded", 0, None),
    "mel8_r5": (8, 5, S.MEL, ST.SLANEY, "banded", 0, None),
    "mel24_r8": (24, 8, S.MEL, ST.SLANEY, "banded", 1, None),
    "mel31_r12": (31, 12, S.MEL, ST.SLANEY, "banded", None, None),
    "mel32_r10": (32, 10, S.MEL, ST.SLANEY, "banded", None, None),
    "bark33_r12": (33, 12, S.BARK, ST.SLANEY, "banded", None, None),
    "log33_r12": (33, 12, S.LOG, ST.SLANEY, "banded", None, (False, True)),
    "linspace40_r12": (40, 12, S.LINSPACE, ST.SLANEY, "banded", None, (True, True)),
    "erb65_r12": (65, 12, S.ERB, ST.SLANEY, "banded", None, None),
    "mel128_r9": (128, 9, S.MEL, ST.SLANEY, "banded", 0, None),
    "mel128_r14": (128, 14, S.MEL, ST.SLANEY, "banded", None, None),
    "mel257_r13": (257, 13, S.MEL, ST.SLANEY, "banded", None, None),
    "mel2_r12": (2, 12, S.MEL, ST.SLANEY, "dense", None, None),
    "linspace16_r6_gt": (16, 6, S.LINSPACE, ST.GAMMATONE, "dense", None, (True, True)),
    "mel63_r12_gt": (63, 12, S.MEL, ST.GAMMATONE, "dense", None, None),
    "erb64_r10_gt": (64, 10, S.ERB, ST.GAMMATONE, "dense", None, None),
    "mel65_r9_gt": (65, 9, S.MEL, ST.GAMMATONE, "dense", None, None),
    "erb129_r13_gt": (129, 13, S.ERB, ST.GAMMATONE, "dense", None, None),
}
# (data type, norm value, result type); 1 = real mode, 0 = complex mode (both planes).  Real mode at fftLength 2048 with
# a banded bank runs the fused kernels, so no case here uses radix2_exp 11.
MODES = {
    "power": (D.POWER, None, 1),
    "power_norm0.5": (D.POWER, 0.5, 1),
    "mag": (D.MAG, None, 1),
    "mag_norm2": (D.MAG, 2.0, 1),
    "mag_norm0.7": (D.MAG, 0.7, 1),
    "complex_square": (D.POWER, None, 0),
    "complex_half": (D.MAG, None, 0),
}
BANK_MODES = [(name, mode) for name in BANKS for mode in
              (MODES if name in ("mel128_r9", "erb64_r10_gt", "mel63_r12_gt") else ("power", "mag_norm2", "complex_square"))]


def make_bank(name, **kw):
    num, r, scale, style, kernel, taps, edges = BANKS[name]
    b = af.BFT(num, r, SR, scale_type=scale, style_type=style, window_type=WIN.HANN, **kw)
    bank = b.get_filter_bank_arr()
    got_kernel, shortest = bank_support(bank)
    assert got_kernel == kernel, (name, got_kernel)
    if taps is not None:
        assert shortest == taps, (name, shortest)
    if edges is not None:
        assert (bool(bank[:, 0].any()), bool(bank[:, -1].any())) == edges, name
    return b, bank


@pytest.mark.parametrize("name", list(BANKS))
def test_bank_claims(name):
    """host only: every bank case is served by the kernel it claims, with the band shapes it claims"""
    b, bank = make_bank(name)
    assert bank.shape == (b.num, b.fft_length // 2 + 1)


@gpu
def test_linear_plane_is_the_stft_store(cuda_device):
    """the premise: a Linear BFT's output is bit-reproducible across objects, and is the STFT's |z|^2 within a few ulps"""
    r, hop, T = 10, 256, 21
    x = clips(1 << r, hop, T)
    a = linear_source(af.BFT(64, r, SR, slide_length=hop, scale_type=S.MEL), D.POWER, None)
    b = linear_source(af.BFT(64, r, SR, slide_length=hop, scale_type=S.MEL), D.POWER, None)
    pa, pb = a.bft_batch(x, 1), b.bft_batch(x, 1)
    assert np.array_equal(pa, pb)
    re, im = af.STFT(r, window_type=WIN.HANN, slide_length=hop).stft_batch(x)
    want = (re.astype(np.float64) ** 2 + im.astype(np.float64) ** 2).astype(np.float32)
    assert (np.abs(pa - want) <= 4 * np.spacing(want) + TINY).all()
    sq_re, sq_im = a.bft_batch(x, 0)                       # complex mode: the SQUARE planes z^2
    z2 = (re.astype(np.float64) + 1j * im.astype(np.float64)) ** 2
    bound = 4 * np.spacing(np.abs(z2).astype(np.float32)) + TINY
    assert (np.abs(sq_re - z2.real) <= bound).all() and (np.abs(sq_im - z2.imag) <= bound).all()


@gpu
@pytest.mark.parametrize("name,mode", BANK_MODES)
def test_bank_bands(report, cuda_device, name, mode):
    data_type, norm, result_type = MODES[mode]
    r = BANKS[name][1]
    n = 1 << r
    hop = max(n // 4, 1)
    T = 45 if r <= 12 else 7                                 # 135 or 21 rows: neither a multiple of 8 nor of 64
    b, bank = make_bank(name, slide_length=hop, data_type=data_type)
    if norm is not None:
        b.set_data_norm_value(norm)
    lin = linear_source(b, data_type, norm)
    x = clips(n, hop, T, seed=r)
    w = bank.astype(np.float64)
    if result_type == 1:
        got = b.bft_batch(x, 1)
        P = lin.bft_batch(x, 1).astype(np.float64)
        want, scale = P @ w.T, np.abs(P) @ np.abs(w).T
        post = norm if (norm is not None and data_type == D.MAG) else 1.0
        check_elems(report, f"{name} {mode}", got, want ** post, scale ** post)
    else:
        got_re, got_im = b.bft_batch(x, 0)
        for plane, got, P in zip(("re", "im"), (got_re, got_im), lin.bft_batch(x, 0)):
            P = P.astype(np.float64)
            check_elems(report, f"{name} {mode} {plane}", got, P @ w.T, np.abs(P) @ np.abs(w).T)


# ------------------------------------------------------------------ k_copy_cols / k_phase
@gpu
@pytest.mark.parametrize("r,low", [(9, 500.0), (12, 1234.0), (14, 15000.0)])
def test_linear_slice_and_phase(report, cuda_device, r, low):
    n = 1 << r
    hop, T = n // 4, 13
    s = af.Spectrogram(samplate=SR, low_fre=low, radix2_exp=r, filter_bank_type=S.LINEAR, data_type=D.POWER)
    lo = int(s.get_bin_band_arr()[0])
    assert lo > 0
    x = clips(n, hop, T, seed=r)
    x[2, : x.shape[1] // 2] = 0                              # frames of zeros: re = im = 0, phase atan2(0, 1e-16)
    spec, phase = s.spectrogram_batch(x, is_phase_arr=True)
    lin = linear_source(af.BFT(2, r, SR, slide_length=hop), D.POWER, None)
    assert np.array_equal(spec, lin.bft_batch(x, 1)[..., lo:lo + s.num])
    re, im = af.STFT(r, window_type=WIN.HANN, slide_length=hop).stft_batch(x)
    re, im = re[..., lo:lo + s.num].astype(np.float64), im[..., lo:lo + s.num].astype(np.float64)
    clamped = re < np.float32(1e-16)
    want = np.arctan2(im, np.where(clamped, np.float64(np.float32(1e-16)), re))
    err = np.abs(phase - want)
    worst = float((err / np.maximum(np.abs(want), 1e-30)).max())
    report(f"phase r={r} lo={lo}", worst, rel_max(phase, want))
    assert (err <= 4 * np.spacing(np.abs(want).astype(np.float32)) + TINY).all(), worst
    assert clamped.any() and (~clamped).any()


# ------------------------------------------------------------------ k_xxcc
def dct_block(num, c0, c1):
    """rows c0 .. c1-1 of the ortho DCT-II matrix, in float64"""
    k = np.arange(c0, c1)[:, None]
    scale = np.where(k == 0, np.sqrt(1.0 / num), np.sqrt(2.0 / num))
    return scale * np.cos(np.pi * (np.arange(num)[None, :] + 0.5) * k / num)


def rectified(m, rectify):
    m = m.astype(np.float64)
    return np.cbrt(m) if rectify == CR.CUBIC_ROOT else np.log10(np.maximum(m, np.float64(np.float32(1e-8))))


def xxcc_oracle(m, cc, rectify):
    """(want, scale) of the first cc ortho DCT-II coefficients of rectify(m), rows along the last axis"""
    num = m.shape[-1]
    l = rectified(m, rectify).reshape(-1, num)
    want, scale = np.empty((l.shape[0], cc)), np.empty((l.shape[0], cc))
    for c0 in range(0, cc, 1024):                            # 1024 rows of the DCT at a time: all of num = 8193 is 537 MB
        Dc = dct_block(num, c0, min(c0 + 1024, cc))
        want[:, c0:c0 + 1024], scale[:, c0:c0 + 1024] = l @ Dc.T, np.abs(l) @ np.abs(Dc).T
    return want.reshape(m.shape[:-1] + (cc,)), scale.reshape(m.shape[:-1] + (cc,))


def cepstral_input(num, T, seed):
    """3 row groups of a positive spectrum with entries below the 1e-8 floor, exact zeros and an all-zero row"""
    rng = np.random.default_rng(seed)
    m = (rng.random((3, T, num)) ** 4).astype(np.float32)
    m[rng.random((3, T, num)) < 0.05] = np.float32(3e-10)
    m[rng.random((3, T, num)) < 0.02] = 0
    m[:, 2] = 0
    return three(m)


XXCC_NUMS = (2, 3, 31, 32, 33, 128, 1025, 1536, 1537, 2049, 4097, 8193)


@gpu
@pytest.mark.parametrize("num", XXCC_NUMS)
def test_xxcc(report, cuda_device, num):
    T = 5 if num > 2049 else 7
    m = cepstral_input(num, T, num)
    x = af.XXCC(num)
    for rectify in (CR.LOG, CR.CUBIC_ROOT):
        for cc in sorted({c for c in (1, 31, 32, 33, num) if c <= num}):
            want, scale = xxcc_oracle(m, cc, rectify)
            check_elems(report, f"num={num} cc={cc} {rectify.name}", x.xxcc_batch(m, cc, rectify), want, scale)


@gpu
@pytest.mark.parametrize("name,num,r,scale_type,cc", [
    ("mel40_r12", 40, 12, S.MEL, 13),
    ("mel128_r10", 128, 10, S.MEL, 128),
    ("linear1537_r12", 1537, 12, S.LINEAR, 33),
    ("linear2049_r12", 2049, 12, S.LINEAR, 40),
])
def test_mfcc_composed(report, cuda_device, name, num, r, scale_type, cc):
    """BFT.mfcc_batch on the composed path: k_xxcc on the same object's bank output"""
    n = 1 << r
    hop = n // 4
    b = af.BFT(num, r, SR, low_fre=0.0 if scale_type == S.LINEAR else None,
               high_fre=(num - 1) * SR / n if scale_type == S.LINEAR else None, slide_length=hop,
               scale_type=scale_type, data_type=D.POWER)
    x = clips(n, hop, 9, seed=num)
    got = b.mfcc_batch(x, cc)
    assert b._lib.bftObj_mfccPlanMode(b._obj) == MFCC_COMPOSED
    mel = b.bft_batch(x, 1)
    want, scale = xxcc_oracle(mel, cc, CR.LOG)
    check_elems(report, name, got, want, scale)


@gpu
def test_legacy_lfcc_linear_4096(report, cuda_device):
    """spectrogramObj_lfcc of a Linear spectrogram at fftLength 4096 (2049 bands), one clip per legacy call"""
    n, hop = 4096, 1024
    s = af.Spectrogram(samplate=SR, radix2_exp=12, filter_bank_type=S.LINEAR, data_type=D.POWER)
    assert s.num == 2049
    x = clips(n, hop, 11, seed=7)
    for i in range(3):
        spec = s.spectrogram(x[i])                           # [num, T]
        got = s._cc("spectrogramObj_lfcc", spec, 20)
        want, scale = xxcc_oracle(np.ascontiguousarray(spec.T), 20, CR.LOG)
        check_elems(report, f"clip {i}", got.T, want, scale)


# ------------------------------------------------------------------ k_xxcc_standard
def fir(x, order, absolute=False):
    m = order // 2
    v1 = float(sum(i * i for i in range(1, m + 1)))
    b = np.array([(m - j) / v1 for j in range(order)])
    y = np.zeros_like(x)
    for j in range(min(order, x.shape[-1])):
        y[..., j:] += (abs(b[j]) if absolute else b[j]) * x[..., :x.shape[-1] - j]
    return y


def standard_oracle(m, energy, cc, window, energy_type, rectify):
    order = window if (window >= 3 and window % 2 == 1) else 9
    want, scale = xxcc_oracle(m, cc, rectify)
    if energy_type != CE.IGNORE:
        e = np.log(np.maximum(energy.astype(np.float64), np.float64(np.float32(1e-8))))[..., None]
        if energy_type == CE.REPLACE:
            want[..., :1], scale[..., :1] = e, np.abs(e)
        else:
            want, scale = np.concatenate([e, want], -1), np.concatenate([np.abs(e), scale], -1)
    d1, s1 = fir(want, order), fir(scale, order, True)
    return (want, scale), (d1, s1), (fir(d1, order), fir(s1, order, True))


# (num, ccNum, delta window, energy type, rectify): ccNum / ccNum + 1 across 32 / 33, windows 3 / 9 / 11 and the
# fall-back to 9 for 4 and 1, windows longer than W, zero energies
STANDARD = [
    (8, 8, 11, CE.REPLACE, CR.LOG), (8, 5, 11, CE.APPEND, CR.CUBIC_ROOT), (8, 2, 3, CE.IGNORE, CR.CUBIC_ROOT),
    (8, 8, 4, CE.APPEND, CR.LOG),
    (1023, 31, 9, CE.APPEND, CR.LOG), (1023, 32, 3, CE.APPEND, CR.LOG), (1023, 1023, 11, CE.APPEND, CR.CUBIC_ROOT),
    (1024, 32, 1, CE.REPLACE, CR.LOG), (1024, 33, 9, CE.IGNORE, CR.CUBIC_ROOT), (1024, 13, 11, CE.REPLACE, CR.CUBIC_ROOT),
    (1025, 32, 9, CE.APPEND, CR.LOG), (1025, 33, 3, CE.REPLACE, CR.LOG), (1025, 1025, 9, CE.IGNORE, CR.LOG),
    (2049, 31, 11, CE.APPEND, CR.CUBIC_ROOT), (2049, 33, 9, CE.REPLACE, CR.LOG), (2049, 2049, 9, CE.APPEND, CR.LOG),
]


@gpu
@pytest.mark.parametrize("num", sorted({c[0] for c in STANDARD}))
def test_xxcc_standard(report, cuda_device, num):
    T = 7
    m = cepstral_input(num, T, num + 1)
    energy = three((np.random.default_rng(num).random((3, T)) * 10).astype(np.float32))
    energy[:, 3] = 0
    x = af.XXCC(num)
    for _, cc, window, energy_type, rectify in (c for c in STANDARD if c[0] == num):
        got = x.xxcc_standard_batch(m, energy, cc, window, energy_type, rectify)
        want = standard_oracle(m, energy, cc, window, energy_type, rectify)
        for part, g, (w, s) in zip(("coe", "d1", "d2"), got, want):
            check_elems(report, f"cc={cc} win={window} {energy_type.name} {rectify.name} {part}", g, w, s)


# ------------------------------------------------------------------ k_chroma
@gpu
@pytest.mark.parametrize("bpo,chroma_num", [(12, 12), (24, 12), (24, 24), (36, 36), (48, 48), (48, 12)])
def test_chroma(report, cuda_device, bpo, chroma_num):
    q = af.CQT(num=bpo * 7, samplate=SR, bin_per_octave=bpo)
    T = 11
    rng = np.random.default_rng(bpo + chroma_num)
    re, im = (three(rng.standard_normal((3, T, q.num)).astype(np.float32)) for _ in range(2))
    bank = O.chroma_cqt_bank(chroma_num, q.num, bpo, q.low_fre).astype(np.float64)
    re[:, 4], im[:, 4] = 0, 0                                # all-zero rows: a zero norm leaves the row
    re[0, 5, bank[0] > 0], im[0, 5, bank[0] > 0] = 0, 0      # an empty class: the min norm is zero
    for data_type in (D.POWER, D.MAG):
        s = (re.astype(np.float64) ** 2 + im.astype(np.float64) ** 2)
        if data_type == D.MAG:
            s = np.sqrt(s)
        v = s @ bank.T
        for norm in (CN.NONE, CN.MAX, CN.MIN, CN.P1, CN.P2):
            a = np.abs(v)
            red = {CN.NONE: np.zeros(v.shape[:-1]), CN.MAX: a.max(-1), CN.MIN: a.min(-1), CN.P1: a.sum(-1),
                   CN.P2: np.sqrt((a * a).sum(-1))}[norm]
            red = np.where(red > 0, red, 1.0)[..., None]
            got = q.chroma_batch(re, im, chroma_num, data_type, norm)
            check_elems(report, f"{data_type.name} {norm.name}", got, v / red, a / red)


# ------------------------------------------------------------------ k_temporal
def temporal_clip(n, hop, T):
    """tones, then a quiet (1e-20) section, exact zeros, and the same tones 1000x louder and reversed"""
    L = (T - 1) * hop + n
    x = tones(n, L, SR)
    q = L // 4
    x[q:2 * q] *= np.float32(1e-20)
    x[2 * q:3 * q] = 0
    x[3 * q:] = x[3 * q:][::-1] * np.float32(1e3)
    return x


@gpu
@pytest.mark.parametrize("r", range(1, 15))
def test_temporal(report, cuda_device, r):
    n = 1 << r
    win = af.STFT(r, window_type=WIN.HANN).get_window_data_arr()
    for hop in sorted({max(n // 4, 1), n, n + n // 2 + 1}):
        T = 13
        x = temporal_clip(n, hop, T)
        b = af.BFT(2, r, SR, slide_length=hop, scale_type=S.LINEAR, is_temporal=True)
        b.bft(x, 1)
        e, rms, zcr = b.get_temporal_data(x.size)
        frames = np.stack([x[t * hop:t * hop + n] for t in range(T)]) * win       # float32, as the device rounds it
        want_e = (frames.astype(np.float64) ** 2).sum(-1)
        cross = ((frames[:, 1:] * frames[:, :-1]) < 0).sum(-1)
        assert np.array_equal(zcr, (cross / n).astype(np.float32)), (r, hop, zcr, cross / n)
        # each square below the denormal range rounds to a multiple of 2^-149: n of those bound the absolute error
        err_e = np.abs(e - want_e)
        normal = want_e >= np.finfo(np.float32).tiny                                 # reported: frames above the denormals
        report(f"n={n} hop={hop}", float((err_e[normal] / want_e[normal]).max()), rel_max(e, want_e))
        assert (err_e <= TOL * want_e + n * TINY).all(), (r, hop)
        assert (e[want_e == 0] == 0).all()
        assert np.array_equal(rms, np.sqrt(e / np.float32(n))), (r, hop)          # float32 division and sqrt, as on the device
