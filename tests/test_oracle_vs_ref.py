"""Pins the numpy restatement (oracle/af_oracle.py) to the reference compiled in oracle/_ref.

Where that library is absent the reference side comes from tests/golden/oracle_vs_ref*.npz: for every case, each small
reference output in full, and of each larger one a fixed sample (the flat positions are stored beside the values, half of
them drawn among the non-zero entries) with the output's max |value|, recorded from the reference build with
AFB200_RECORD_GOLDEN=1."""
import ctypes as C
import os
import zlib

import numpy as np
import pytest

import audioflux_b200 as af
from conftest import GOLDEN, noise
from oracle import af_oracle as O
from oracle import ref_lib as R

GOLD_PATH = os.path.join(GOLDEN, "oracle_vs_ref.npz")
GOLD_BANKS = os.path.join(GOLDEN, "oracle_vs_ref_banks.npz")      # test_filter_banks / test_gammatone_bank
SAMPLE = 256                     # largest output stored in full, and positions stored of a larger one
_record = {}


class Sampled:
    """A reference output known only at `idx` (flat positions) plus its max |value|."""

    def __init__(self, idx, values, amax, shape):
        self.idx, self.values, self.amax, self.shape = idx, values, amax, shape


def _choose_positions(key, a, sample):
    """recording only: every position of a small output, else `sample` sorted positions, half among the non-zero entries"""
    if a.size <= SAMPLE:
        return np.arange(a.size)
    rng = np.random.default_rng(zlib.crc32(key.encode()))
    nz = np.flatnonzero(a.reshape(-1))
    pick = set(rng.choice(nz, min(sample // 2, nz.size), replace=False).tolist()) if nz.size else set()
    rest = rng.permutation(a.size)
    for q in rest:
        if len(pick) >= sample:
            break
        pick.add(int(q))
    return np.array(sorted(pick), np.int64)


def reference(request, name, compute, path=GOLD_PATH, sample=SAMPLE):
    """`compute(lib)` -> reference output(s) from the reference build when it is built (recorded into the golden file
    `path` under AFB200_RECORD_GOLDEN=1), else the stored output or sample of each output as `Sampled`."""
    key = f"{request.node.name}/{name}"
    if R.available():
        out = compute(R.get_ref_lib())
        if os.environ.get("AFB200_RECORD_GOLDEN") == "1":
            rec = _record.setdefault(path, {})
            for i, a in enumerate(out if isinstance(out, tuple) else (out,)):
                a = np.asarray(a)
                pos = _choose_positions(f"{key}/{i}", a, sample)
                npos = pos.size if pos.size != a.size else 0
                # one float64 record: max |a|, ndim, shape, number of stored positions (0: all), positions, values
                rec[f"{key}/{i}"] = np.concatenate([[np.abs(a).max() if a.size else 0.0, a.ndim], a.shape, [npos],
                                                    pos if npos else [], a.reshape(-1)[pos]]).astype(np.float64)
        return out
    if not os.path.exists(path):
        pytest.skip(f"no reference build and no {os.path.relpath(path, GOLDEN)} under tests/golden")
    g = np.load(path)
    res = []
    i = 0
    while f"{key}/{i}" in g.files:
        r = g[f"{key}/{i}"]
        nd = int(r[1])
        shape = tuple(int(v) for v in r[2:2 + nd])
        npos = int(r[2 + nd])
        body = r[3 + nd:]
        if npos:
            res.append(Sampled(body[:npos].astype(np.int64), body[npos:], float(r[0]), shape))
        else:
            res.append(body.reshape(shape))
        i += 1
    assert res, f"{key} missing from {path}"
    return tuple(res) if len(res) > 1 else res[0]


def positions(ref):
    """flat positions at which `ref` is known"""
    return ref.idx if isinstance(ref, Sampled) else np.arange(np.asarray(ref).size)


def at(ours, ref):
    """(ours, ref, max |ref|) over the positions where the reference output is known"""
    ours = np.asarray(ours)
    if isinstance(ref, Sampled):
        assert ours.shape == ref.shape
        return ours.reshape(-1)[ref.idx], ref.values, ref.amax
    ref = np.asarray(ref)
    assert ours.shape == ref.shape
    return ours.reshape(-1), ref.reshape(-1), float(np.abs(ref).max()) if ref.size else 0.0


def rel_err(ours, ref):
    """rel_max of conftest over the known positions: max |ours - ref| / max |ref|"""
    a, b, m = at(ours, ref)
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max() / max(m, 1e-30))


def abs_err(ours, ref):
    a, b, _ = at(ours, ref)
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max())


def teardown_module(module):
    for path, rec in _record.items():
        np.savez_compressed(path, **rec)

S, ST, N, D, W = (af.SpectralFilterBankScaleType, af.SpectralFilterBankStyleType,
                  af.SpectralFilterBankNormalType, af.SpectralDataType, af.WindowType)


@pytest.mark.parametrize("wt", range(14))
def test_windows(request, wt):
    for n in (16, 512, 2048):
        def ref(lib):
            p = lib.window_calFFTWindow(wt, n)
            return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_float)), shape=(n,)).copy()
        w = reference(request, f"n{n}", ref)
        assert abs_err(O.fft_window(wt, n), w) < 2e-6


def _ref_bank(ref, num, n, sr, scale, style, norm, low, high, bpo):
    bank = np.zeros((num + 4, n // 2 + 1), np.float32)
    fb = np.zeros(num + 2, np.float32)
    bb = np.zeros(num + 2, np.int32)
    ref.auditory_filterBank(num, n, sr, 0, scale, style, norm, low, high, bpo, bank.ctypes.data, fb.ctypes.data, bb.ctypes.data)
    return bank[:num], fb[:num], bb[:num]


def bank_cases():
    for scale in range(1, 7):
        for style in (0, 1, 3, 4, 5, 6, 7, 8, 9, 10):
            for norm in (0, 1, 2):
                yield scale, style, norm


@pytest.mark.parametrize("scale,style,norm", list(bank_cases()))
def test_filter_banks(request, scale, style, norm):
    for num, n, sr in ((128, 2048, 48000), (40, 1024, 16000)):
        low = 32.703196 if scale in (5, 6) else None
        high = None
        if scale == 1:                       # the reference writes out of bounds when revised edges leave [0, sr/2]
            low, high = 1000.0, sr / 2 - 1000.0
        if scale == 6:
            low, high = 32.703196, sr / 2 * 0.8
        lo, hi, _, _ = O.bft_revise_range(num, n, sr, low, high, scale, 12)
        if scale == 5 and float(hi) > sr / 2:
            continue
        b1, f1, i1 = reference(request, f"{num}-{n}", lambda lib: _ref_bank(lib, num, n, sr, scale, style, norm, float(lo),
                                                                             float(hi), 12), GOLD_BANKS, 64)
        b2, f2, i2 = O.auditory_filterbank(num, n, sr, scale, style, norm, float(lo), float(hi), 12)
        assert np.array_equal(i1, i2)
        _, _, amax = at(b2, b1)
        assert abs_err(b2, b1) <= 5e-5 * max(1.0, amax)
        np.testing.assert_allclose(f1, f2, rtol=2e-6, atol=1e-3)


@pytest.mark.parametrize("r,hop,wt", [(11, 512, 1), (9, 100, 2), (10, 1024, 0), (12, 1000, 4)])
def test_stft(request, r, hop, wt):
    x = noise(1, 20000)
    re, im = reference(request, "planes", lambda lib: tuple(af.STFT(r, W(wt), hop, _lib=lib).stft_planes(x)))
    re2, im2 = O.stft(x, 1 << r, hop, O.fft_window(wt, 1 << r))
    assert rel_err(re2, re) < 2e-6 and rel_err(im2, im) < 2e-6


@pytest.mark.parametrize("scale,style,norm,dt,rt,nv", [
    (2, 0, 0, 0, 1, 1.0), (2, 0, 1, 1, 1, 1.0), (3, 1, 0, 0, 1, 0.5), (4, 0, 2, 1, 1, 2.0), (2, 0, 0, 0, 0, 1.0),
    (3, 0, 1, 1, 0, 1.0), (0, 0, 0, 0, 1, 1.0), (0, 0, 0, 1, 0, 1.0), (5, 0, 0, 0, 1, 1.0), (6, 1, 1, 1, 1, 1.0)])
def test_bft_modes(request, scale, style, norm, dt, rt, nv):
    x = noise(2, 20000)
    kw = dict(low_fre=32.703196, high_fre=16000.) if scale == 6 else {}

    def ref(lib):
        b = af.BFT(64, 10, 44100, slide_length=256, scale_type=S(scale), style_type=ST(style), normal_type=N(norm),
                   data_type=D(dt), _lib=lib, **kw)
        if nv != 1.0:
            b.set_data_norm_value(nv)
        re, im = b.bft_planes(x, rt)
        return re if rt == 1 else (re, im)
    got = reference(request, "planes", ref)
    o = O.bft(x, 64, 10, 44100, 256, 1, scale, style, norm, dt, low=32.703196 if scale in (5, 6) else None,
              high=kw.get("high_fre"), result_type=rt, norm_value=nv)
    if rt == 1:
        assert rel_err(o, got) < 2e-5
    else:
        assert rel_err(o[0], got[0]) < 2e-5 and rel_err(o[1], got[1]) < 2e-5


def test_xxcc(request):
    m = np.abs(noise(3, 50 * 128).reshape(50, 128)) + 1e-9
    m[3, :5] = 0.0

    def ref(lib):
        x = af.XXCC(128, _lib=lib)
        x2 = af.XXCC(60, _lib=lib)          # non power of two -> dense DCT in the reference
        return (x.xxcc_planes(m, 40), x2.xxcc_planes(m[:, :60], 13), x.xxcc_planes(m, 20, af.CepstralRectifyType.CUBIC_ROOT))
    c40, c13, c20 = reference(request, "cc", ref)
    assert abs_err(O.xxcc(m, 40), c40) < 2e-5
    assert abs_err(O.xxcc(m[:, :60], 13), c13) < 2e-5
    assert abs_err(O.xxcc(m, 20, O.RECT_CUBIC), c20) < 2e-5


def test_decimator(request):
    x = noise(4, 20001)

    def ref(ref_lib):
        ro = C.c_void_p()
        ref_lib.resampleObj_new.argtypes = [C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
        ref_lib.resampleObj_new(C.byref(ro), C.byref(C.c_int(2)), C.byref(C.c_int(1)), None)
        ref_lib.resampleObj_setSamplate.argtypes = [C.c_void_p, C.c_int, C.c_int]
        ref_lib.resampleObj_setSamplate(ro, 2, 1)
        ref_lib.resampleObj_resample.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        ref_lib.resampleObj_resample.restype = C.c_int
        out = np.zeros(len(x), np.float32)
        n = ref_lib.resampleObj_resample(ro, x.ctypes.data, len(x), out.ctypes.data)
        return out[:n]
    out = reference(request, "y", ref)
    y = O.resample_down2(x)
    assert len(y) == len(x) // 2
    assert rel_err(y, out) < 2e-6


@pytest.mark.parametrize("L,sr,norm,hop,scale", [(48037, 48000, 1, None, True), (30000, 32000, 0, None, True),
                                                  (22050, 22050, 2, 64, False)])
def test_cqt(request, L, sr, norm, hop, scale):
    x = noise(5, L)
    re, im = reference(request, "planes", lambda lib: tuple(
        af.CQT(84, sr, normal_type=N(norm), slide_length=hop, is_scale=scale, _lib=lib).cqt_planes(x)))
    re2, im2 = O.cqt(x, 84, sr, norm=norm, hop=hop, is_scale=scale)
    assert rel_err(re2, re) < 1e-5 and rel_err(im2, im) < 1e-5


@pytest.mark.parametrize("r,wav,scale,pad", [(12, 1, 5, False), (12, 0, 5, False), (12, 2, 5, False), (11, 3, 5, False),
                                             (11, 4, 5, False), (11, 5, 5, False), (11, 6, 5, False), (11, 7, 5, False),
                                             (12, 1, 2, False), (12, 0, 3, False), (12, 1, 5, True), (10, 1, 0, False)])
def test_cwt(request, r, wav, scale, pad):
    x = noise(6, 1 << r)
    kw = dict(low_fre=1000.) if scale == 0 else {}
    num = 40 if scale == 0 else 84
    re, im = reference(request, "planes", lambda lib: tuple(
        af.CWT(num, r, 48000, wavelet_type=af.WaveletContinueType(wav), scale_type=S(scale),
               is_padding=pad, _lib=lib, **kw).cwt_planes(x)))
    re2, im2 = O.cwt(x, num, r, 48000, wav, scale, low=kw.get("low_fre", 32.703196 if scale in (5, 6) else None), is_pad=pad)
    assert rel_err(re2, re) < 1e-5 and rel_err(im2, im) < 1e-5


@pytest.mark.parametrize("num,n,sr,scale,norm", [(64, 1024, 32000, 4, 0), (64, 1024, 32000, 4, 1), (40, 2048, 16000, 2, 2),
                                                  (128, 2048, 48000, 4, 0), (32, 512, 22050, 3, 1), (24, 1024, 44100, 1, 0)])
def test_gammatone_bank(request, num, n, sr, scale, norm):
    lo, hi = (100.0, sr / 2 - 100.0) if scale == 1 else (0.0, sr / 2)

    def ref(lib):
        b = np.zeros((num + 4, n // 2 + 1), np.float32)
        f = np.zeros(num + 2, np.float32)
        bi = np.zeros(num + 2, np.int32)
        lib.auditory_filterBank(num, n, sr, 0, scale, 2, norm, C.c_float(lo), C.c_float(hi), 12, b.ctypes.data, f.ctypes.data,
                                bi.ctypes.data)
        return b[:num], f[:num], bi[:num], b[:num].max(axis=1)
    b, f, bi, rowmax = reference(request, "bank", ref, GOLD_BANKS, 256)
    ob, of, obi = O.auditory_filterbank(num, n, sr, scale, O.STYLE_GAMMATONE, norm, lo, hi)
    assert np.array_equal(obi, bi)
    np.testing.assert_allclose(of, f, rtol=2e-6, atol=1e-3)
    pos = positions(b)
    tol = np.maximum(np.asarray(rowmax)[pos // ob.shape[1]], 1e-30)            # per position: its row's maximum
    assert (np.abs(at(ob, b)[0] - at(ob, b)[1]) <= 2e-5 * tol).all()
    # given the reference's own centre frequencies the restatement is bit-exact (area norm: up to its summation order)
    exact = O.gammatone_bank(num, n, sr, norm, np.asarray(f, np.float32))
    assert (np.abs(at(exact, b)[0] - at(exact, b)[1]) <= (1e-5 if norm == 1 else 0.0) * tol).all()
