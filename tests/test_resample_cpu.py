"""Resampler without a GPU: the numpy oracle against the reference build (or its stored outputs in
tests/golden/resample.npz), the constructor statuses and calDataLength of both libraries over a grid of parameters and
rate settings, the refusals (which need no device), the exported and bound symbols of include/afb200_resample.h and
afb200_ext.h, and the Python classes' argument checks."""
import itertools
import os

import numpy as np
import pytest

import _resample_oracle as RO
from _parity_kit import GoldenStore, check_symbols, ref_lib_or_none

ORACLE_TOL = 1e-5          # of max|reference output|; worst seen: 1.3e-6 (the reference's float32 sums)
GOLDEN_MAX_LEN = 20000     # cases with inputs up to this many samples go to the golden file
CASES = dict(RO.cases())


def _keys(name):
    """one key per call of the case: one, or one per chunk in continue mode"""
    return [f"{name}__{k}" for k in range(len(CASES[name].get("chunks", [None])))]


def golden_names():
    return {name for name, kw in RO.cases() if RO.case_signal(name, kw).size <= GOLDEN_MAX_LEN}


def _live(keys):
    lib = ref_lib_or_none()
    out = {}
    for n in sorted({k.split("__")[0] for k in keys}):
        out.update((k, o) for k, o in zip(_keys(n), RO.c_case(lib, n, CASES[n])) if k in keys)
    return out


GOLD = GoldenStore("resample.npz", _live, lambda: {k for n in golden_names() for k in _keys(n)})


@pytest.mark.parametrize("name,kw", RO.cases(), ids=[c[0] for c in RO.cases()])
def test_oracle_matches_reference(name, kw):
    if ref_lib_or_none() is None and name not in golden_names():
        pytest.skip("case not in tests/golden/resample.npz and no reference build")
    out = GOLD.outputs(set(_keys(name)))
    got = [out[k] for k in _keys(name)]
    want = RO.oracle_case(name, kw)
    assert len(got) == len(want), name
    for k, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape, (name, k, g.shape, w.shape)
        if g.size:
            err = np.abs(g - w).max() / max(np.abs(g).max(), 1e-30)
            assert err <= ORACLE_TOL, (name, k, err)


def test_golden_file_matches_reference_build():
    GOLD.check_file()


def test_golden_file_covers_the_rules():
    names = golden_names()
    assert {"best_48000_16000", "mid_16000_48000", "fast_8000_44100", "fast_equal", "win13_v0.3", "win_rules",
            "ratio_0.37", "ratio_2.5", "chain", "scale_up_init", "len1_down", "len2_up",
            "continue_48000_16000", "continue_44100_48000"} <= names
    assert all(f"win{w}_null" in names for w in range(1, 14))
    assert os.path.getsize(GOLD.path) < 400 * 1024


WINDOWS = [dict(), dict(zero_num=16, nbit=7, win_type=4, value=None, roll_off=None),
           dict(zero_num=0, nbit=0, win_type=0, value=0.0, roll_off=0.0),
           dict(zero_num=-5, nbit=30, win_type=None, value=-1.0, roll_off=1.0001),
           dict(zero_num=7, nbit=3, win_type=8, value=0.0, roll_off=1.0),
           dict(zero_num=3, nbit=1, win_type=13, value=0.7, roll_off=0.5)]
SETTINGS = [[], [("rate", 48000, 16000)], [("rate", 44100, 48000)], [("rate", 16000, 48000)], [("rate", 7, 7)],
            [("rate", -1, 16000)], [("ratio", 0.37)], [("ratio", -2.0)], [("ratio", 2.5)],
            [("rate", 44100, 16000), ("rate", 16000, 22050), ("ratio", 1.0)]]
LENGTHS = [0, 1, 2, 3, 146, 147, 148, 1000, 44100, 12345677]


def test_statuses_and_lengths_match_reference(product_lib, ref_lib):
    for q, scale, cont in itertools.product((None, 0, 1, 2), (None, 1), (None, 0, 1)):
        for ops in SETTINGS:
            got = []
            for lib in (product_lib, ref_lib):
                st, o = RO.c_new(lib, q, None, scale, cont)
                RO.c_apply(lib, o, ops)
                got.append((st, [lib.resampleObj_calDataLength(o, n) for n in LENGTHS]))
                lib.resampleObj_enableContinue(o, 1)
                got[-1][1].extend(lib.resampleObj_calDataLength(o, n) for n in LENGTHS)
                lib.resampleObj_free(o)
            assert got[0] == got[1], (q, scale, cont, ops)
    for w in WINDOWS:
        got = []
        for lib in (product_lib, ref_lib):
            st, o = RO.c_new(lib, None, w)
            lib.resampleObj_setSamplate(o, 22050, 16000)
            got.append((st, [lib.resampleObj_calDataLength(o, n) for n in LENGTHS]))
            lib.resampleObj_free(o)
        assert got[0] == got[1], w


def test_lengths_match_the_oracle(product_lib):
    for ops in SETTINGS:
        for cont in (0, 1):
            st, o = RO.c_new(product_lib, 1, None, 0, cont)
            r = RO.Resampler(1, is_continue=bool(cont))
            RO.c_apply(product_lib, o, ops)
            for op in ops:
                r.set_samplate(*op[1:]) if op[0] == "rate" else r.set_ratio(op[1])
            for n in LENGTHS:
                assert product_lib.resampleObj_calDataLength(o, n) == r.lengths(n)[1], (ops, cont, n)
            product_lib.resampleObj_free(o)


def _untouched(lib, o, n=3000, fill=7.0):
    x = RO.case_signal("r", dict(length=n))
    buf = np.full(4 * n, fill, np.float32)
    ret = lib.resampleObj_resample(o, x.ctypes.data, n, buf.ctypes.data)
    return ret == 0 and (buf == fill).all()


def test_refusals(product_lib):
    """every refusal happens before any device work, so it holds without a GPU"""
    L = product_lib
    for w in (14, 100, -2):                # WindowType is unsigned: -2 is above Tukey too (the reference crashes on both)
        st, o = RO.c_new(L, None, dict(win_type=w))
        assert st == -1 and not o.value and f"winType={w}".encode() in L.afb200_lastError(), w
    for z, nb in ((64, 17), (1 << 20, 9), (3, 29), (1 << 30, 29)):
        st, o = RO.c_new(L, None, dict(zero_num=z, nbit=nb))
        assert st == -2 and not o.value and b"table entries" in L.afb200_lastError(), (z, nb)
    st, o = RO.c_new(L, None, dict(zero_num=1 << 13, nbit=9))                 # 2^22 + 1 entries: the largest
    assert st == 0
    L.resampleObj_free(o)
    st, o = RO.c_new(L, 0)
    # ratio * 2^nbit < 1: no tap stride
    L.resampleObj_setSamplateRatio(o, 0.0019)
    assert _untouched(L, o) and b"below 1" in L.afb200_lastError()
    L.resampleObj_setSamplateRatio(o, 0.0)
    assert _untouched(L, o)
    # continue mode with q <= 1
    for ops in ([("rate", 16000, 48000)], [("ratio", 0.5)], [("rate", 16000, 16000)]):
        st, c = RO.c_new(L, 0, None, 0, 1)
        RO.c_apply(L, c, ops)
        if ops[0][1] == 16000 and ops[0][2] == 16000:
            L.resampleObj_setSamplate(c, 16000, 32000)                     # q = 1
        assert _untouched(L, c) and b"continue mode" in L.afb200_lastError(), ops
        L.resampleObj_free(c)
    # continue mode where sourceLength * p overflows int, and a one-shot output length beyond int
    st, c = RO.c_new(L, 2, None, 0, 1)
    L.resampleObj_setSamplate(c, 2, 2147483647)
    assert _untouched(L, c) and b"does not fit" in L.afb200_lastError()
    L.resampleObj_enableContinue(c, 0)
    assert _untouched(L, c) and b"does not fit" in L.afb200_lastError()
    L.resampleObj_free(c)
    # the batch refuses continue mode and bad arguments
    x = RO.case_signal("r", dict(length=300))
    out = np.full(300, 7.0, np.float32)
    L.resampleObj_setSamplate(o, 48000, 16000)
    L.resampleObj_enableContinue(o, 1)
    assert L.resampleObj_resampleBatch(o, x.ctypes.data, 300, 1, out.ctypes.data, 0, None) != 0
    assert b"continue mode" in L.afb200_lastError()
    L.resampleObj_enableContinue(o, 0)
    for args in ((None, 300, 1, out.ctypes.data), (x.ctypes.data, 0, 1, out.ctypes.data),
                 (x.ctypes.data, 300, -1, out.ctypes.data), (x.ctypes.data, 300, 1, None)):
        assert L.resampleObj_resampleBatch(o, *args, 0, None) != 0
    assert (out == 7.0).all()
    L.resampleObj_debug(o)
    L.resampleObj_free(o)


def test_resample_symbols_exported_and_bound(product_lib):
    from audioflux_b200 import capi
    check_symbols(product_lib, "afb200_resample.h", "resampleObj_", capi.RESAMPLE_API, 9, {"resampleObj_resampleBatch"})


def test_python_class_checks(product_lib):
    import audioflux_b200 as af
    for alias, q in (("best", 0), ("af_mid", 1), ("audio_fast", 2), (af.ResampleQualityType.MID, 1)):
        assert af.Resample(alias).qual_type.value == q
    for bad in ("good", 3, None):
        with pytest.raises(ValueError, match="not supported"):
            af.Resample(bad)
    with pytest.raises(ValueError, match="status -2"):
        af.WindowResample(zero_num=64, nbit=20)
    with pytest.raises(ValueError, match="status -1"):
        af.WindowResample(win_type=14)
    r = af.Resample("fast")
    assert r.cal_data_length(48000) == 24000                                 # the initial 32000 -> 16000
    r.set_samplate(48000, 16000)
    assert (r.source_rate, r.target_rate) == (48000, 16000) and r.cal_data_length(48000) == 16000
    r.set_samplate(16000, 96000)
    assert r.cal_data_length(1000) == 6000                                   # beyond the reference's 5 * n buffer
    w = af.WindowResample()
    assert (w.zero_num, w.nbit, w.win_type, w.value, w.roll_off, w.is_scale) == (64, 9, af.WindowType.HANN, None, 0.945,
                                                                                 False)
    w.set_samplate(48000, 16000)
    with pytest.raises(ValueError, match="at least one dimension"):
        w.resample(np.float32(1.0))
    with pytest.raises(ValueError, match="empty"):
        w.resample(np.zeros((2, 0), np.float32))
    # fewer samples than one output: no device work, an empty result of the right shape
    assert w.resample(np.zeros((2, 3, 2), np.float32)).shape == (2, 3, 0)
    assert w.resample_batch(np.zeros((4, 1), np.float32)).shape == (4, 0)
