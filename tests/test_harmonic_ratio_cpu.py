"""Harmonic ratio without a GPU: the float64 oracle against the reference build (or its stored outputs in
tests/golden/harmonic_ratio.npz) over every window size, the parameter fallbacks, slides, frame counts, window types and
signals; frames without a crossing and the carry of the last crossing; the statuses of new and calTimeLength against
the reference; the refusals (which need no device); the exported and bound symbols of include/afb200_harmonic_ratio.h
and afb200_ext.h; and the Python class's arguments."""
import numpy as np
import pytest

import _harmonic_ratio_oracle as HO
from _parity_kit import GoldenStore, check_symbols, ref_lib_or_none

TOL = 1e-5                 # of max |value| of the clip
CASES = dict(HO.cases())


def _live(keys):
    lib = ref_lib_or_none()
    return {k: HO.c_case(lib, k, CASES[k]) for k in keys}


GOLD = GoldenStore("harmonic_ratio.npz", _live, lambda: set(CASES))


def _scale(want):
    return max(np.abs(want).max(initial=0.0), 1e-30)


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference(name):
    got = GOLD.outputs({name})[name]
    want, cands, _ = HO.oracle_case(name, CASES[name])
    ok, alt = HO.agree(got, want, cands, TOL * _scale(want))
    assert ok, (name, alt, got[alt], want[alt])
    assert len(alt) <= max(2, len(want) // 10), (name, alt)


def test_carry_is_exercised():
    """frames without a crossing exist, from frame 0 and after frames with one, and reuse the last index found"""
    for name in ("sig_dc", "sig_low", "sig_dc_then_tones", "sig_tones_dc_tones", "h12_dc", "sr8000_lf3999.5"):
        _, _, own = HO.oracle_case(name, CASES[name])
        assert any(o is None for o in own), name
    _, _, own = HO.oracle_case("sig_dc_then_tones", CASES["sig_dc_then_tones"])
    assert own[0] is None and any(o is not None for o in own)
    _, _, own = HO.oracle_case("sig_tones_dc_tones", CASES["sig_tones_dc_tones"])
    first_none = own.index(None)
    assert first_none > 0 and own[first_none - 1] is not None
    # the carried index matters: the carry frames' values differ from what minIndex 0 would give
    kw = CASES["sig_tones_dc_tones"]
    p = HO.case_params(kw)
    r, E = HO._frame_parts(HO.case_signal("sig_tones_dc_tones", kw), p["W"], p["slide"], p["max_length"])
    m = own[first_none - 1]
    v_carry = HO._values(r[first_none], E[first_none], p["W"], p["max_length"], m)[0]
    v_zero = HO._values(r[first_none], E[first_none], p["W"], p["max_length"], 0)[0]
    assert m > 0 and abs(v_carry - v_zero) > 1e-3


def test_golden_file_matches_reference_build():
    GOLD.check_file()


def test_statuses_match_reference(product_lib, ref_lib):
    """new accepts what the reference accepts (outside the two refusals), and calTimeLength agrees"""
    grid = []
    for sr in (None, -1, 0, 1, 49, 50, 8000, 196000, 196001):
        for lf in (None, -2.0, 0.0, 24.0, 100.0, 4000.0, 1e9):
            for r2 in (None, -1, 1, 5, 13, 29, 30):
                for slide in (None, -1, 0, 1, 700):
                    grid.append((sr, lf, r2, slide))
    rng = np.random.default_rng(0)
    grid = [grid[i] for i in rng.choice(len(grid), 300, replace=False)]
    for sr, lf, r2, slide in grid:
        p = HO.params(sr, lf, r2, slide)
        if p["W"] > 1 << 13 or p["max_length"] < 1:
            continue
        # at W = 2 the default slide W/4 is 0: the reference divides by zero, this library uses 1
        zero_slide = p["W"] < 4 and not (slide is not None and slide > 0)
        st_p, o_p = HO.c_new(product_lib, sr, lf, r2, HO.W_HAMM, slide)
        assert st_p == 0, (sr, lf, r2, slide)
        if not zero_slide:
            st_r, o_r = HO.c_new(ref_lib, sr, lf, r2, HO.W_HAMM, slide)
            assert st_r == 0
        for n in (0, 1, p["W"] - 1, p["W"], p["W"] + 1, p["W"] + p["slide"], 5 * p["W"] + 3, 100000):
            got = product_lib.harmonicRatioObj_calTimeLength(o_p, n)
            assert got == HO.time_length(n, p["W"], max(1, p["slide"])), (sr, lf, r2, slide, n)
            if not zero_slide:
                assert got == ref_lib.harmonicRatioObj_calTimeLength(o_r, n), (sr, lf, r2, slide, n)
        product_lib.harmonicRatioObj_free(o_p)
        if not zero_slide:
            ref_lib.harmonicRatioObj_free(o_r)


def test_refusals(product_lib):
    """radix2Exp above 13 and an empty lag range are refused at construction with a status and a reason; the object
    pointer stays NULL.  A call with too few samples leaves the output untouched."""
    L = product_lib
    for args, st, what in (((32000, 100.0, 14, None, 512), -2, b"largest supported is 13"),
                           ((32000, 100.0, 29, None, 512), -2, b"largest supported is 13"),
                           ((32000, 100.0, 0, None, None), -3, b"maxLength=0"),
                           ((20, None, 10, None, None), -3, b"maxLength=0"),
                           ((20, 11.0, 10, None, None), -3, b"maxLength=0")):
        s, o = HO.c_new(L, *args)
        assert s == st and not o, (args, s)
        assert what in L.afb200_lastError(), L.afb200_lastError()
    s, o = HO.c_new(L, 30, None, 10)                       # samplate 25 .. 49 with lowFre 25: maxLength 1, accepted
    assert s == 0 and o and L.afb200_lastError() == b""
    out = HO.c_ratio(L, o, np.ones(1023, np.float32), fill=7.0, extra=4)
    assert (out == 7).all()
    L.harmonicRatioObj_free(o)
    s, o = HO.c_new(L, 32000, 100.0, 10)
    v = np.zeros(4, np.float32)
    assert L.harmonicRatioObj_harmonicRatioBatch(o, None, 2048, 1, v.ctypes.data, 0, None) != 0
    assert b"bad argument" in L.afb200_lastError()
    assert L.harmonicRatioObj_harmonicRatioBatch(o, v.ctypes.data, 4, -1, v.ctypes.data, 0, None) != 0
    L.harmonicRatioObj_free(o)
    L.harmonicRatioObj_free(None)
    L.harmonicRatioObj_harmonicRatio(None, None, 0, None)


def test_harmonic_ratio_symbols_exported_and_bound(product_lib):
    from audioflux_b200 import capi
    check_symbols(product_lib, "afb200_harmonic_ratio.h", "harmonicRatioObj_", capi.HARMONIC_RATIO_API,
                  {"harmonicRatioObj_new", "harmonicRatioObj_calTimeLength", "harmonicRatioObj_harmonicRatio",
                   "harmonicRatioObj_free"}, {"harmonicRatioObj_harmonicRatioBatch"})


def test_python_class(product_lib):
    import audioflux_b200 as af
    h = af.HarmonicRatio()
    assert (h.samplate, h.radix2_exp, h.slide_length, h.window_type, h.fft_length) == \
        (32000, 12, 1024, af.WindowType.HAMM, 4096)
    assert abs(h.low_fre - 32.703196) < 1e-6
    assert h.cal_time_length(160000) == (160000 - 4096) // 1024 + 1 and h.cal_time_length(4095) == 0
    assert af.HarmonicRatio(radix2_exp=40).fft_length == 2048
    assert af.HarmonicRatio(radix2_exp=-1, slide_length=0).cal_time_length(2048 + 512) == 2
    with pytest.raises(ValueError, match="status -2"):
        af.HarmonicRatio(radix2_exp=14)
    with pytest.raises(ValueError, match="status -3: .*maxLength=0"):
        af.HarmonicRatio(radix2_exp=0)
    with pytest.raises(ValueError, match="at least one dimension"):
        h.harmonic_ratio(np.float32(1))
    # no frames or no clips: no device work, empty results of the right shapes
    assert h.harmonic_ratio(np.zeros((2, 3, 100), np.float32)).shape == (2, 3, 0)
    assert h.harmonic_ratio_batch(np.zeros((0, 8000), np.float32)).shape == (0, 4)
    from audioflux_b200.lib import AfB200Error
    if product_lib.afb200_deviceCount() <= 0:          # no CPU fallback: the compute call fails loudly
        with pytest.raises(AfB200Error, match="no CUDA device"):
            h.harmonic_ratio(np.ones(8000, np.float32))
