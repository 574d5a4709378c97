"""Cross-correlation and the chirp z-transform without a GPU: the float64 oracle against the reference build (or its
stored outputs in tests/golden/dsp.npz) over every length, cross and auto, normType None / Coeff / NULL, impulse, silent
and unbalanced inputs; every CZT size 2^0 .. 2^13 with the bands and real-only, imaginary-only and complex inputs; one
CZT object through a valid, invalid, valid band sequence; the refusals (which need no device); the exported and bound
symbols of include/afb200_xcorr.h, afb200_czt.h and afb200_ext.h; and the Python classes' arguments."""
import ctypes as C

import numpy as np
import pytest

import _dsp_oracle as D
from _parity_kit import GoldenStore, check_symbols, ref_lib_or_none

TOL = 1e-5                 # of max |want| of the row
XC = dict(D.xcorr_cases())
CZ = dict(D.czt_cases())
SEQ_R = 10


def _gold_keys():
    """the cases the golden file keeps: outputs up to 8191 lags or 2^10-point CZTs, and the band sequence"""
    return ({k for k, kw in XC.items() if kw["n"] <= 4096} | {k for k, kw in CZ.items() if kw["r"] <= 10} |
            {"c_sequence"})


def _seq_input():
    return np.random.default_rng(5).standard_normal(1 << SEQ_R).astype(np.float32)


def _live(keys):
    lib = ref_lib_or_none()
    out = {}
    for k in keys:
        if k in XC:
            v, mv, i = D.c_xcorr_case(lib, k, XC[k])
            out[k] = np.concatenate([v, np.float32([mv, i])])
        elif k in CZ:
            out[k] = D.c_czt_case(lib, k, CZ[k]).astype(np.complex64)
        else:
            out[k] = np.stack(D.c_czt_sequence(lib, SEQ_R, _seq_input())).astype(np.complex64)
    return out


GOLD = GoldenStore("dsp.npz", _live, _gold_keys, equal=lambda a, b: np.array_equal(a, b, equal_nan=True))


def _scale(want):
    w = np.abs(want)
    return max(np.nanmax(w) if np.isfinite(w).any() else 0.0, 1e-30)


def check_xcorr(got, gv, gi, want, wv, wi, what, tol=TOL, exact_index=True):
    """values within tol of max |want|, NaN exactly where the oracle has NaN; the index equal (or, with
    exact_index=False, equal unless the values at both indices are within the bar); maxValue within the bar"""
    assert got.shape == want.shape, what
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), (what, "NaN pattern")
    bar = tol * _scale(want)
    if (~nan).any():
        err = np.abs(got[~nan] - want[~nan]).max()
        assert err <= bar, (what, err / _scale(want))
    if exact_index or nan.all():
        assert gi == wi, (what, gi, wi)
    else:
        assert gi == wi or abs(want[gi] - want[wi]) <= bar, (what, gi, wi, want[gi], want[wi])
    assert (np.isnan(gv) and np.isnan(wv)) or abs(gv - wv) <= bar, (what, gv, wv)


@pytest.mark.parametrize("name", list(XC))
def test_xcorr_oracle_matches_reference(name):
    got = GOLD.outputs({name}).get(name)
    if got is None:
        pytest.skip("not in tests/golden/dsp.npz and no reference build")
    want, wv, wi = D.xcorr_case(name, XC[name])
    check_xcorr(got[:-2], got[-2], int(got[-1]), want, wv, wi, name)


@pytest.mark.parametrize("name", list(CZ))
def test_czt_oracle_matches_reference(name):
    got = GOLD.outputs({name}).get(name)
    if got is None:
        pytest.skip("not in tests/golden/dsp.npz and no reference build")
    want = D.czt_case(name, CZ[name])
    assert got.shape == want.shape
    assert np.abs(got - want).max() <= TOL * _scale(want), (name, np.abs(got - want).max() / _scale(want))


def test_czt_band_sequence_matches_reference():
    """valid, invalid (kept tables), valid (rebuilt): the second call equals the first, the third is its own band"""
    got = GOLD.outputs({"c_sequence"})["c_sequence"]
    want = D.czt_sequence_oracle(SEQ_R, _seq_input())
    for g, w in zip(got, want):
        assert np.abs(g - w).max() <= TOL * _scale(w)
    assert np.array_equal(got[0], got[1]) and not np.allclose(got[1], got[2])


def test_golden_file_matches_reference_build():
    GOLD.check_file()


def test_refusals(product_lib):
    """xcorr: length < 1 -> -1, length > 2^19 -> -2; czt: radix2Exp < 0 -> -1, > 13 -> -2; both CZT inputs NULL refused.
    A message is recorded and the outputs stay untouched."""
    L = product_lib
    x = np.ones(8, np.float32)
    for n, st, what in ((0, -1, b"length=0"), (-3, -1, b"length=-3"), ((1 << 19) + 1, -2, b"largest supported is 524288")):
        o = C.c_void_p()
        assert L.xcorrObj_new(C.byref(o)) == 0
        out = np.full(8, 7.0, np.float32)
        mv = C.c_float(7.0)
        assert L.xcorrObj_xcorr(o, x.ctypes.data, None, n, None, out.ctypes.data, C.byref(mv)) == st
        assert what in L.afb200_lastError(), L.afb200_lastError()
        assert (out == 7).all() and mv.value == 7
        idx = np.full(2, 7, np.int32)
        assert L.xcorrObj_xcorrBatch(o, x.ctypes.data, None, n, 2, None, out.ctypes.data, None, idx.ctypes.data, 0,
                                     None) == st
        assert (out == 7).all() and (idx == 7).all()
        # vArr1 NULL: 0, nothing written
        assert L.xcorrObj_xcorr(o, None, None, 4, None, out.ctypes.data, C.byref(mv)) == 0 and (out == 7).all()
        L.xcorrObj_free(o)
    for r, st in ((-1, -1), (14, -2), (30, -2)):
        s, o = D.c_czt_new(L, r)
        assert s == st and not o, (r, s)
        assert f"radix2Exp={r}".encode() in L.afb200_lastError()
    s, o = D.c_czt_new(L, 4)
    assert s == 0 and o and L.afb200_lastError() == b""
    out = np.full(32, 7.0, np.float32)
    L.cztObj_czt(o, None, None, 0.1, 0.2, out.ctypes.data, out.ctypes.data)
    assert (out == 7).all() and b"both input planes NULL" in L.afb200_lastError()
    assert L.cztObj_cztBatch(o, x.ctypes.data, None, -1, 0.1, 0.2, out.ctypes.data, out.ctypes.data, 0, None) == -1
    L.cztObj_free(o)
    L.cztObj_free(None)
    L.xcorrObj_free(None)


def test_dsp_symbols_exported_and_bound(product_lib):
    from audioflux_b200 import capi
    check_symbols(product_lib, "afb200_xcorr.h", "xcorrObj_", {k: v for k, v in capi.DSP_API.items() if k.startswith("x")},
                  {"xcorrObj_new", "xcorrObj_xcorr", "xcorrObj_free"}, {"xcorrObj_xcorrBatch"})
    check_symbols(product_lib, "afb200_czt.h", "cztObj_", {k: v for k, v in capi.DSP_API.items() if k.startswith("c")},
                  {"cztObj_new", "cztObj_czt", "cztObj_free"}, {"cztObj_cztBatch"})
    assert any(t is capi.DSP_API for t in capi.bind.__defaults__[0])


def test_python_classes(product_lib):
    import audioflux_b200 as af
    assert [t.value for t in af.XcorrNormalType] == [0, 1]
    x = af.Xcorr()
    with pytest.raises(ValueError, match="1D"):
        x.xcorr(np.ones((2, 3), np.float32))
    with pytest.raises(ValueError, match="must be equal"):
        x.xcorr(np.ones(3, np.float32), np.ones(4, np.float32))
    with pytest.raises(ValueError, match="at least one sample"):
        x.xcorr_batch(np.ones((2, 0), np.float32))
    arr, mv, idx = x.xcorr_batch(np.ones((0, 5), np.float32))
    assert arr.shape == (0, 9) and mv.shape == (0,) and idx.shape == (0,) and idx.dtype == np.int32
    c = af.CZT(4)
    assert c.fft_length == 16 and c.radix2_exp == 4
    for r in (-1, 14):
        with pytest.raises(ValueError, match="cztObj_new failed with status"):
            af.CZT(r)
    with pytest.raises(ValueError, match="below 2\\*\\*radix2_exp"):
        c.czt(np.ones(15, np.float32), 0.1, 0.2)
    with pytest.raises(ValueError, match="16 samples"):
        c.czt_batch(np.ones((2, 17), np.float32), 0.1, 0.2)
    assert c.czt_batch(np.ones((0, 16), np.complex64), 0.1, 0.2).shape == (0, 32)
    from audioflux_b200.lib import AfB200Error
    if product_lib.afb200_deviceCount() <= 0:          # no CPU fallback: the compute call fails loudly
        with pytest.raises(AfB200Error, match="no CUDA device"):
            x.xcorr(np.ones(8, np.float32))
        with pytest.raises(AfB200Error, match="no CUDA device"):
            c.czt_batch(np.ones(16, np.float32), 0.1, 0.2)
