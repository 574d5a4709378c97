"""Cepstrogram without a GPU: the numpy oracle against the reference build (or its stored outputs in
tests/golden/cepstrogram.npz), cepstrogramObj_new statuses and calTimeLength of both libraries over a grid, the
refusals (which need no device), the exported and bound symbols of include/afb200_cepstrogram.h and afb200_ext.h, and
the Python class's argument checks."""
import os

import numpy as np
import pytest

import _cepstrogram_oracle as CO
from _parity_kit import GoldenStore, check_symbols, ref_lib_or_none

ORACLE_TOL = 5e-5          # per frame, of max|log S|; worst seen: 1.6e-5 (details at 2^14, the reference's float32 FFTs)
GOLDEN_MAX_CELLS = 1600    # cases with at most this many T x (N/2+1) cells go to the golden file (about 250 KB)


def golden_names():
    out = set()
    for name, kw in CO.cases():
        n = 1 << kw["radix2_exp"]
        if CO.time_length(kw["length"], n, kw["slide"]) * (n // 2 + 1) <= GOLDEN_MAX_CELLS:
            out.add(name)
    return out


def _live(names):
    """{name: [cep, env, det] stacked}"""
    lib = ref_lib_or_none()
    return {name: np.stack(CO.c_case(lib, kw, CO.case_signal(name, kw))) for name, kw in CO.cases() if name in names}


GOLD = GoldenStore("cepstrogram.npz", _live, golden_names)


@pytest.mark.parametrize("name,kw", CO.cases(), ids=[c[0] for c in CO.cases()])
def test_oracle_matches_reference(name, kw):
    if ref_lib_or_none() is None and name not in golden_names():
        pytest.skip("case not in tests/golden/cepstrogram.npz and no reference build")
    got = GOLD.outputs({name})[name]
    *want, logs = CO.oracle_case(name, kw)
    for k in range(3):
        assert got[k].shape == want[k].shape, (name, k)
        if got[k].size:
            err = CO.frame_errors(got[k], want[k], logs)
            assert err.max() <= ORACLE_TOL, (name, k, err.max())


def test_golden_file_matches_reference_build():
    GOLD.check_file()


def test_golden_file_covers_the_rules():
    names = golden_names()
    assert {"r1_c1", "r8_c128", "r8_c127", "r8_t0", "r8_t1", "r8_silent", "r9_slide512", "r9_slide700"} <= names
    assert os.path.getsize(GOLD.path) < 400 * 1024


def _grid():
    for r in range(1, 15):
        n = 1 << r
        for slide in (None, -3, 0, 1, 7, max(1, n // 2), n, n + 3, 3 * n):
            yield r, slide


def _lengths(n, hop):
    return sorted({0, 1, n - 1, n, n + 1, n + hop - 1, n + hop, 5 * n + 17})


def test_new_and_time_length_match_reference(product_lib, ref_lib):
    for r in (-1, 0, 31):
        assert CO.c_new(product_lib, r)[0] == CO.c_new(ref_lib, r)[0] == -100, r
    for r, slide in _grid():
        n = 1 << r
        hop = slide if slide is not None and slide > 0 else n // 4
        if hop == 0:                                  # N = 2 without a slide: the reference divides by zero
            continue
        sp, po = CO.c_new(product_lib, r, CO.W_HANN, slide)
        sr, ro = CO.c_new(ref_lib, r, CO.W_HANN, slide)
        assert sp == sr == 0, (r, slide)
        for length in _lengths(n, hop):
            tp = product_lib.cepstrogramObj_calTimeLength(po, length)
            assert tp == ref_lib.cepstrogramObj_calTimeLength(ro, length), (r, slide, length)
        product_lib.cepstrogramObj_free(po)
        ref_lib.cepstrogramObj_free(ro)


def test_new_statuses_and_time_length(product_lib):
    for r in (-5, 0, 31, 40):
        s, o = CO.c_new(product_lib, r)
        assert s == -100 and not o.value, r
    for r in (15, 16, 30):
        s, o = CO.c_new(product_lib, r, CO.W_HANN, 1024)
        assert s == -2 and not o.value, r
        assert b"largest supported is 14" in product_lib.afb200_lastError()
    for r, slide in _grid():
        n = 1 << r
        s, o = CO.c_new(product_lib, r, CO.W_HANN, slide)
        assert s == 0 and o.value
        hop = slide if slide is not None and slide > 0 else max(n // 4, 1)
        for length in _lengths(n, hop):
            assert product_lib.cepstrogramObj_calTimeLength(o, length) == CO.time_length(length, n, hop), (r, slide, length)
        product_lib.cepstrogramObj_enableDebug(o, 1)
        product_lib.cepstrogramObj_free(o)


def test_refusals_leave_outputs_untouched(product_lib):
    """cepNum outside 1 .. N/2 fails before any device work, so this holds without a GPU"""
    n = 256
    x = CO.signal(1, 2000)
    s, o = CO.c_new(product_lib, 8, CO.W_HANN, 128)
    T = product_lib.cepstrogramObj_calTimeLength(o, x.size)
    re = np.ones((T, n), np.float32)
    for c in (0, -1, n // 2 + 1, 1000):
        out = CO.c_cepstrogram(product_lib, o, n, c, x, fill=7.0)
        assert all((p == 7.0).all() for p in out), c
        assert f"cepNum={c}".encode() in product_lib.afb200_lastError()
        out = CO.c_cepstrogram2(product_lib, o, n, c, re, re, fill=7.0)
        assert all((p == 7.0).all() for p in out), c
        assert b"cepstrogram2" in product_lib.afb200_lastError()
        cep = np.full((T, n // 2 + 1), 7.0, np.float32)
        st = product_lib.cepstrogramObj_cepstrogramBatch(o, c, x.ctypes.data, x.size, 1, cep.ctypes.data, None, None, 0,
                                                         None)
        assert st != 0 and (cep == 7.0).all() and b"1 .. 128" in product_lib.afb200_lastError()
        st = product_lib.cepstrogramObj_cepstrogram2Batch(o, c, re.ctypes.data, re.ctypes.data, T, n, None, None,
                                                          cep.ctypes.data, 0, None)
        assert st != 0 and (cep == 7.0).all()
    # bad widths and no output at all
    assert product_lib.cepstrogramObj_cepstrogram2Batch(o, 4, re.ctypes.data, re.ctypes.data, T, n - 1, cep.ctypes.data,
                                                        None, None, 0, None) != 0
    assert b"specWidth" in product_lib.afb200_lastError()
    assert product_lib.cepstrogramObj_cepstrogramBatch(o, 4, x.ctypes.data, x.size, 1, None, None, None, 0, None) != 0
    product_lib.cepstrogramObj_free(o)


def test_cepstrogram_symbols_exported_and_bound(product_lib):
    from audioflux_b200 import capi
    check_symbols(product_lib, "afb200_cepstrogram.h", "cepstrogramObj_", capi.CEPSTROGRAM_API, 6,
                  {"cepstrogramObj_cepstrogramBatch", "cepstrogramObj_cepstrogram2Batch"})


def test_python_class_checks(product_lib):
    import audioflux_b200 as af
    with pytest.raises(ValueError, match="status -2"):
        af.Cepstrogram(radix2_exp=15)
    with pytest.raises(ValueError, match="status -100"):
        af.Cepstrogram(radix2_exp=0)
    t = af.Cepstrogram(radix2_exp=10, samplate=16000, window_type=af.WindowType.HANN, slide_length=256)
    assert t.cal_time_length(4000) == (4000 - 1024) // 256 + 1 and t.cal_time_length(1000) == 0
    assert np.array_equal(t.y_coords(), np.linspace(0, 8000, 514))
    assert np.array_equal(t.x_coords(4000), np.linspace(0, 4000 / 16000, t.cal_time_length(4000) + 1))
    with pytest.raises(ValueError):
        t.x_coords(1000)
    x = CO.signal(2, 4000)
    for c in (0, 513, -4):
        with pytest.raises(ValueError, match="cep_num"):
            t.cepstrogram(x, c)
        with pytest.raises(ValueError, match="cep_num"):
            t.cepstrogram2_batch(np.ones((3, 1024), np.float32), np.ones((3, 1024), np.float32), c)
    with pytest.raises(ValueError, match="request"):
        t.cepstrogram_batch(x, 4, cep=False, env=False, det=False)
    with pytest.raises(ValueError, match="width"):
        t.cepstrogram2_batch(np.ones((3, 600), np.float32), np.ones((3, 600), np.float32))
    # a clip shorter than one frame needs no device: empty outputs of the right shape
    cep, env, det = t.cepstrogram(np.zeros((2, 1000), np.float32))
    assert cep.shape == env.shape == det.shape == (2, 513, 0)
