"""Harmonic-percussive separation without a GPU: the numpy oracle against the reference build (or its stored outputs in
tests/golden/hpss.npz), the constructor statuses and calDataLength of both libraries over a grid of parameters, the
refusals (which need no device), the exported and bound symbols of include/afb200_hpss.h and afb200_ext.h, and the
Python class's argument checks."""
import itertools
import os

import numpy as np
import pytest

import _hpss_oracle as HO
from _parity_kit import GoldenStore, check_symbols, ref_lib_or_none

ORACLE_TOL = 2e-5          # of max|reference output| where the normaliser is >= 1e-2 (elsewhere 1e-2); worst seen: 2e-6
GOLDEN_MAX_LEN = 5000      # cases with outputs up to this many samples go to the golden file
CASES = dict(HO.cases())


def _key(name, k):
    return f"{name}__{k}"


def golden_names():
    return {name for name, kw in HO.cases() if HO.data_length(kw["length"], 1 << kw["radix2_exp"]) <= GOLDEN_MAX_LEN}


def _golden_keys():
    """h is output 0 and p output 1; a skipped output has no key"""
    return {_key(n, k) for n in golden_names() for k, c in enumerate("hp") if c in CASES[n].get("outputs", "hp")}


def _live(keys):
    lib = ref_lib_or_none()
    out = {}
    for n in sorted({k.split("__")[0] for k in keys}):
        for k, o in enumerate(HO.c_case(lib, n, CASES[n])):
            if o is not None and _key(n, k) in keys:
                out[_key(n, k)] = o
    return out


GOLD = GoldenStore("hpss.npz", _live, _golden_keys)


@pytest.mark.parametrize("name,kw", HO.cases(), ids=[c[0] for c in HO.cases()])
def test_oracle_matches_reference(name, kw):
    if ref_lib_or_none() is None and name not in golden_names():
        pytest.skip("case not in tests/golden/hpss.npz and no reference build")
    out = GOLD.outputs({_key(name, k) for k in range(2)})
    got = [out.get(_key(name, k)) for k in range(2)]
    want = HO.oracle_case(name, kw)
    for k, (g, w) in enumerate(zip(got, want)):
        assert (g is None) == (w is None), (name, k)
        if w is None:
            continue
        assert g.shape == w.shape, (name, k, g.shape, w.shape)
        err, ill = HO.errors(w, g, kw)
        assert err <= ORACLE_TOL and ill <= 1e-2, (name, k, err, ill)


def test_golden_file_matches_reference_build():
    GOLD.check_file()


def test_golden_file_covers_the_rules():
    names = golden_names()
    assert {"hamm_n10_defaults", "hann_n9", "rect_n9", "hamm_n6", "hamm_n6_orders_121_45", "h_order_1", "p_order_1",
            "orders_1_1", "orders_even_zero", "orders_negative_even", "t1", "t1_tail", "h_only", "p_only",
            "init_buffers"} <= names
    assert os.path.getsize(GOLD.path) < 300 * 1024


ORDERS = [None, -3, 0, 1, 2, 3, 20, 21, 31, 255, 383, 385, 1001]
LENGTHS = [-5, 0, 1, 3, 4, 15, 16, 17, 100, 1023, 1024, 1025, 2047, 2048, 2049, 44100, 160000]


def test_statuses_and_lengths_match_reference(product_lib, ref_lib):
    for r, w, slide in itertools.product(range(2, 17), (None, 0, 1, 2), (None, -1, 7, 1024)):
        got = []
        for lib in (product_lib, ref_lib):
            st, o = HO.c_new(lib, r, w, slide, 21, 31)
            got.append((st, [lib.hpssObj_calDataLength(o, n) for n in LENGTHS]))
            lib.hpssObj_free(o)
        assert got[0] == got[1], (r, w, slide)
        assert got[0][1] == [HO.data_length(n, 1 << r) for n in LENGTHS], r
    for ho, po in itertools.product(ORDERS, ORDERS):
        for lib in (product_lib, ref_lib):
            st, o = HO.c_new(lib, 11, None, None, ho, po)
            assert st == 0 and lib.hpssObj_calDataLength(o, 5000) == HO.data_length(5000, 2048), (ho, po)
            lib.hpssObj_free(o)


def _untouched(lib, o, n, outputs="hp", fill=7.0):
    x = HO.case_signal("u", dict(length=max(n, 1)))
    h, p = HO.c_hpss(lib, o, x[:n] if n > 0 else x, outputs, fill=fill)
    return all(b is None or (b == fill).all() for b in (h, p))


def test_refusals(product_lib):
    """every refusal happens before any device work, so it holds without a GPU"""
    L = product_lib
    # shorter than one frame (the reference crashes)
    st, o = HO.c_new(L, 11)
    for n in (100, 2047):
        for outs in ("hp", "h", "p"):
            x = HO.case_signal("short", dict(length=n))
            h = np.full(2000, 7.0, np.float32)
            p = np.full(2000, 7.0, np.float32)
            L.hpssObj_hpss(o, x.ctypes.data, n, h.ctypes.data if "h" in outs else None,
                           p.ctypes.data if "p" in outs else None)
            assert (h == 7.0).all() and (p == 7.0).all(), (n, outs)
            assert b"shorter than one frame" in L.afb200_lastError(), n
    # the batch: bad arguments, no outputs, and the same rules
    x = HO.case_signal("b", dict(length=3000))
    out = np.full(3000, 7.0, np.float32)
    for args in ((None, 3000, 1, out.ctypes.data, out.ctypes.data), (x.ctypes.data, 0, 1, out.ctypes.data, None),
                 (x.ctypes.data, 3000, -1, out.ctypes.data, None), (x.ctypes.data, 3000, 1, None, None)):
        assert L.hpssObj_hpssBatch(o, *args, 0, None) != 0
    assert L.hpssObj_hpssBatch(o, x.ctypes.data, 2047, 1, out.ctypes.data, None, 0, None) != 0
    assert b"shorter than one frame" in L.afb200_lastError()
    assert (out == 7.0).all()
    L.hpssObj_debug(o)
    L.hpssObj_free(o)
    # radix2Exp the STFT path cannot serve, or with no hop
    for r in (0, 1, 21, 22):
        st, o = HO.c_new(L, r)
        assert st == 0
        assert _untouched(L, o, 1 << 12) and b"radix2Exp" in L.afb200_lastError(), r
        assert L.hpssObj_hpssBatch(o, x.ctypes.data, 3000, 1, out.ctypes.data, None, 0, None) != 0
        L.hpssObj_free(o)
    # orders above the cap
    for ho, po in ((385, 31), (21, 385), (1001, 1001)):
        st, o = HO.c_new(L, 10, None, None, ho, po)
        assert st == 0
        assert _untouched(L, o, 3000) and b"orders up to 383" in L.afb200_lastError(), (ho, po)
        L.hpssObj_free(o)
    # both outputs NULL: nothing happens, as in the reference
    st, o = HO.c_new(L, 10)
    L.hpssObj_hpss(o, x.ctypes.data, 3000, None, None)
    L.hpssObj_free(o)
    L.hpssObj_free(None)


def test_hpss_symbols_exported_and_bound(product_lib):
    from audioflux_b200 import capi
    check_symbols(product_lib, "afb200_hpss.h", "hpssObj_", capi.HPSS_API,
                  {"hpssObj_new", "hpssObj_calDataLength", "hpssObj_hpss", "hpssObj_free", "hpssObj_debug"},
                  {"hpssObj_hpssBatch"})


def test_python_class_checks(product_lib):
    import audioflux_b200 as af
    h = af.HPSS()
    assert (h.radix2_exp, h.window_type, h.slide_length, h.h_order, h.p_order) == (12, af.WindowType.HAMM, 1024, 21, 31)
    assert h.cal_data_length(160000) == HO.data_length(160000, 4096)
    assert h.cal_data_length(100) == 3072
    h2 = af.HPSS(radix2_exp=11, window_type=af.WindowType.HANN, slide_length=300, h_order=20, p_order=-1)
    assert h2.cal_data_length(5000) == HO.data_length(5000, 2048)          # slide_length is ignored, as in the reference
    with pytest.raises(ValueError, match="at least one dimension"):
        h.hpss(np.float32(1.0))
    with pytest.raises(ValueError, match="empty"):
        h.hpss(np.zeros((2, 0), np.float32))
    from audioflux_b200.lib import AfB200Error
    with pytest.raises(AfB200Error, match="shorter than one frame"):
        h.hpss(np.zeros((2, 4095), np.float32))
    with pytest.raises(AfB200Error, match="orders up to"):
        af.HPSS(radix2_exp=10, h_order=385).hpss(np.zeros(5000, np.float32))
    # no channels: no device work, empty results of the right shape
    a, b = h.hpss_batch(np.zeros((0, 5000), np.float32))
    assert a.shape == b.shape == (0, HO.data_length(5000, 4096))
