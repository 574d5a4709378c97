"""ST / FST without a GPU: the numpy oracle against the reference build (or its stored outputs in tests/golden/st.npz),
the constructor statuses of both libraries, the exported and bound symbols of include/afb200_st.h, and the Python
classes' argument checks."""
import numpy as np
import pytest

import _st_oracle as SO
from _parity_kit import GoldenStore, check_symbols, ref_lib_or_none

ORACLE_TOL = 2e-5          # worst row seen: 5.4e-6 (the reference's float32 FFTs)
# cases whose output has at most this many complex values go to the golden file.  FST rows repeat each value N/len
# times and compress well; the limits keep the file near 200 KB while covering the bin-0, Nyquist, bin-list and
# fallback rules of both transforms.
GOLDEN_MAX_CELLS = {"st": 8320, "fst": 40000}


def _cases():
    return [("st", n, kw) for n, kw in SO.st_cases()] + [("fst", n, kw) for n, kw in SO.fst_cases()]


def _signal(kind, kw):
    return SO.case_signal(3 if kind == "st" else 4, 1 << kw["radix2_exp"])


def _live(names):
    """{name: [re, im] stacked}"""
    lib = ref_lib_or_none()
    res = {}
    for kind, name, kw in _cases():
        if name in names:
            x = _signal(kind, kw)
            res[name] = np.stack(SO.c_st_case(lib, kw, x) if kind == "st" else SO.c_fst_case(lib, kw, x))
    return res


def golden_names():
    out = set()
    for kind, name, kw in _cases():
        n = 1 << kw["radix2_exp"]
        rows = len(SO.st_rows(kw)) if kind == "st" else SO.fst(np.zeros(n), kw["min_index"], kw["max_index"]).shape[0]
        if rows * n <= GOLDEN_MAX_CELLS[kind]:
            out.add(name)
    return out


GOLD = GoldenStore("st.npz", _live, golden_names)


@pytest.mark.parametrize("kind,name,kw", _cases(), ids=[c[1] for c in _cases()])
def test_oracle_matches_reference(kind, name, kw):
    if ref_lib_or_none() is None and name not in golden_names():
        pytest.skip("case not in tests/golden/st.npz and no reference build")
    got = GOLD.outputs({name})[name]
    x = _signal(kind, kw)
    want = SO.oracle_st_case(kw, x) if kind == "st" else SO.fst(x, kw["min_index"], kw["max_index"])
    assert got.shape[1:] == want.shape
    err, _ = SO.row_errors(got[0], got[1], want)
    assert err.max() <= ORACLE_TOL, (name, err.max())


def test_golden_file_matches_reference_build():
    GOLD.check_file()


def _st_sweep():
    for r in range(1, 13):
        n = 1 << r
        for lo, hi in ((0, 0), (1, n // 2), (0, n // 2), (-1, 3), (2, n // 2 + 1), (3, 2), (n // 4, n // 4 + 1)):
            yield r, lo, hi


def test_st_constructor_matches_reference(product_lib, ref_lib):
    for r, lo, hi in _st_sweep():
        sp, po = SO.c_st_new(product_lib, r, lo, hi)
        sr, ro = SO.c_st_new(ref_lib, r, lo, hi)
        assert sp == sr == 0, (r, lo, hi)
        a, b = SO.st_range(r, lo, hi)
        assert product_lib.stObj_getBinLength(po) == b - a + 1
        product_lib.stObj_free(po)
        ref_lib.stObj_free(ro)


def test_fst_constructor_matches_reference(product_lib, ref_lib):
    for r in range(0, 13):
        sp, po = SO.c_fst_new(product_lib, r)
        sr, ro = SO.c_fst_new(ref_lib, r)
        assert sp == sr == (0 if r >= 3 else -1), r
        assert bool(po.value) == bool(ro.value) == (r >= 3), r
        if sp == 0:
            product_lib.fstObj_free(po)
            ref_lib.fstObj_free(ro)


def test_constructor_statuses_without_reference(product_lib):
    for r, lo, hi in list(_st_sweep()) + [(13, 0, 0), (14, 1, 8192), (14, 0, 0)]:
        s, o = SO.c_st_new(product_lib, r, lo, hi, 0.5, 2.0)
        assert s == 0
        a, b = SO.st_range(r, lo, hi)
        assert product_lib.stObj_getBinLength(o) == b - a + 1
        product_lib.stObj_free(o)
    for r in range(-1, 15):
        s, o = SO.c_fst_new(product_lib, r)
        assert s == (0 if r >= 3 else -1), r
        product_lib.fstObj_free(o)
    s, o = SO.c_st_new(product_lib, 0, 0, 0)
    assert s == -1 and not o.value


def test_use_bin_arr_rules(product_lib):
    s, o = SO.c_st_new(product_lib, 9, 10, 20)
    assert product_lib.stObj_getBinLength(o) == 11
    for bad in ([4, 300, 5], [4, -1], [257]):
        SO.c_use_bins(product_lib, o, bad)
        assert product_lib.stObj_getBinLength(o) == 11, bad
    longer = np.arange(700) % 257                                  # longer than N: taken (the reference overruns)
    SO.c_use_bins(product_lib, o, longer)
    assert product_lib.stObj_getBinLength(o) == 700
    SO.c_use_bins(product_lib, o, [256, 0, 256])
    assert product_lib.stObj_getBinLength(o) == 3
    product_lib.stObj_free(o)


def test_refusals_above_2e14(product_lib):
    for r in (15, 16, 30):
        s, o = SO.c_st_new(product_lib, r, 1, 100)
        assert s == -2 and not o.value, r
        assert b"radix2Exp" in product_lib.afb200_lastError()
        s, o = SO.c_fst_new(product_lib, r)
        assert s == -2 and not o.value, r
        assert b"largest supported is 14" in product_lib.afb200_lastError()


def test_st_symbols_exported_and_bound(product_lib):
    from audioflux_b200 import capi
    check_symbols(product_lib, "afb200_st.h", "stObj_|fstObj_", capi.ST_API, 8,
                  {"stObj_stBatch", "stObj_getBinLength", "fstObj_fstBatch"})


def test_python_class_checks(product_lib):
    import audioflux_b200 as af
    for cls in (af.ST, af.FST):
        with pytest.raises(ValueError):
            cls(radix2_exp=10, min_index=0)
        with pytest.raises(ValueError):
            cls(radix2_exp=10, max_index=512)
        with pytest.raises(ValueError):
            cls(radix2_exp=10, min_index=20, max_index=20)
        with pytest.raises(ValueError, match="status -2"):
            cls(radix2_exp=15)
        t = cls(radix2_exp=10, min_index=3, max_index=40, samplate=16000)
        assert t.num == 38
        assert t.get_fre_band_arr().dtype == np.float32 and t.get_fre_band_arr()[0] == 3 * 16000 / 1024
        assert t.y_coords().shape == (39,) and t.x_coords().shape == (1025,)
    with pytest.raises(ValueError, match="status -1"):
        af.FST(radix2_exp=2, min_index=1, max_index=1.5)
    t = af.ST(radix2_exp=10, min_index=3, max_index=40)
    t.use_bin_arr([5, 0, 512, 5])
    assert t.num == 4 and product_lib.stObj_getBinLength(t._obj) == 4
    assert np.array_equal(t.get_fre_band_arr(), np.array([5, 0, 512, 5], np.float32) * 32000 / 1024)
    t.use_bin_arr([5, 513])
    assert t.num == 4
    with pytest.raises(ValueError):
        t.use_bin_arr([[1, 2]])
    t.set_value(0.5, 2.0)
    assert (t.factor, t.norm) == (0.5, 2.0)
