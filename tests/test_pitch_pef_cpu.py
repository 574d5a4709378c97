"""PitchPEF without a GPU: the float64 oracle against the reference build (or its stored outputs in
tests/golden/pitch_pef.npz) over frame sizes, samplates, cut frequencies, filter parameters, slides, windows and
signals; the statuses of new and calTimeLength against the reference, streaming included; setFilterParams changing
nothing; the refusals (which need no device); the exported and bound symbols of include/afb200_pitch_pef.h and
afb200_ext.h; and the Python class's arguments.

Run as a script, it rewrites tests/golden/pitch_pef.npz from the reference build (oracle/_ref):

    python tests/test_pitch_pef_cpu.py"""
import numpy as np
import pytest

from _parity_kit import GoldenStore, check_symbols, ref_lib_or_none      # first: conftest puts the root on sys.path
import _pitch_c as PC
import _pitch_pef_oracle as PO

CASES = dict(PO.cases())


def _live(keys):
    lib = ref_lib_or_none()
    return {k: PO.c_case(lib, k, CASES[k]) for k in keys}


GOLD = GoldenStore("pitch_pef.npz", _live, lambda: set(CASES))


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference(name):
    kw = CASES[name]
    p = PO.case_params(kw)
    assert p["status"] == 0
    got = GOLD.outputs({name})[name]
    want, cands = PO.oracle_case(name, kw)
    ok, alt = PO.agree(got, want, cands, p)
    assert ok, (name, alt, got[alt], want[alt])
    assert len(alt) <= max(2, len(want) // 10), (name, alt)


def test_cases_cover_the_tables():
    """the padding-free filter (L = 4n), slides above n, odd integer samplate/2, a cut above samplate/2, n = 2^11 .. 2^13"""
    ps = {k: PO.case_params(kw) for k, kw in CASES.items()}
    assert ps["beta1"]["pad"] == 0 and ps["beta1"]["xcorr_length"] == 4 * ps["beta1"]["n"]
    assert ps["default"]["pad"] > 0 and ps["default"]["xcorr_length"] == 8 * ps["default"]["n"]
    assert ps["slide_gt_n"]["slide"] > ps["slide_gt_n"]["n"]
    assert ps["cut_at_nyquist_odd"]["sr"] % 2 == 1 and ps["cut_above_nyquist"]["cut"] > ps["cut_above_nyquist"]["sr"] // 2
    assert {ps[k]["n"] for k in ("r11", "default", "r13")} == {2048, 4096, 8192}


def test_golden_file_matches_reference_build():
    GOLD.check_file()


def _grid():
    grid = []
    for sr in (None, -1, 8000, 11025, 32000, 196001):
        for lf in (None, 20.0, 27.0, 100.0):
            for hf in (None, 90.0, 1000.0, 5000.0, 20000.0):
                for cf in (None, 500.0, 3000.0, 5512.0, 12000.0):
                    for r2 in (None, 0, 3, 11, 13, 14, 31):
                        grid.append(dict(sr=sr, lf=lf, hf=hf, cf=cf, r2=r2))
    rng = np.random.default_rng(0)
    return [grid[i] for i in rng.choice(len(grid), 250, replace=False)]


def test_statuses_match_reference(product_lib, ref_lib):
    """new accepts exactly what the oracle accepts, refuses the rest with the oracle's status, and calTimeLength agrees
    with the reference wherever both build the object"""
    seen = set()
    for kw in _grid():
        for slide in (None, 700):
            p = PO.params(**kw, slide=slide)
            st_p, o_p = PC.c_new(product_lib, "pef", **kw, slide=slide)
            assert st_p == p["status"], (kw, slide, st_p, p["status"])
            seen.add(st_p)
            if st_p:
                assert not o_p
                continue
            st_r, o_r = PC.c_new(ref_lib, "pef", **kw, slide=slide)
            assert st_r == 0
            for n in (0, 1, p["n"] - 1, p["n"], p["n"] + 1, p["n"] + p["slide"], 5 * p["n"] + 3, 100000):
                got = product_lib.pitchPEFObj_calTimeLength(o_p, n)
                assert got == PC.time_length(n, p["n"], p["slide"]) == ref_lib.pitchPEFObj_calTimeLength(o_r, n)
            product_lib.pitchPEFObj_free(o_p)
            ref_lib.pitchPEFObj_free(o_r)
    assert seen == {0, -2, -3}, seen


def test_streaming_in_the_reference():
    """isContinue: pieces of a clip (some shorter than a frame) give the frames of one call over the clip, with a slide
    below n and one above it (a negative carry); calTimeLength counts the carry"""
    lib = ref_lib_or_none()
    if lib is None:
        pytest.skip("needs the reference build")
    x = PC.signal("glide", 40000, 16000, 5)
    for r2, slide in ((11, 512), (10, 1500)):
        st, whole = PC.c_new(lib, "pef", sr=16000, r2=r2, slide=slide)
        want = PC.c_pitch(lib, "pef", whole, x)
        st, o = PC.c_new(lib, "pef", sr=16000, r2=r2, slide=slide, cont=1)
        got = PC.c_stream(lib, "pef", o, x, (700, 3000, 100, 9000, 1, 27199))
        assert np.array_equal(got, want), (r2, slide)
        lib.pitchPEFObj_free(o)
        lib.pitchPEFObj_free(whole)


def test_refusals(product_lib):
    """radix2Exp above 13, an empty lag range and the clipped peak search are refused at construction with a status and
    a reason; the object pointer stays NULL"""
    L = product_lib
    hf_top = float(PO.params(r2=11, beta=1.0)["log"][-1]) - 0.01          # nearest the top grid point of n = 2^11
    for kw, st, what in ((dict(r2=14), -2, b"largest supported is 13"),
                         (dict(r2=30), -2, b"largest supported is 13"),
                         (dict(hf=3999.0, cf=3999.0), -3, b"is empty"),
                         (dict(sr=8000, hf=3999.5), -3, b"is empty"),
                         (dict(r2=11, beta=1.0, hf=hf_top, cf=4000.0), -4, b"reads past")):
        p = PO.params(**kw)
        assert p["status"] == st, (kw, p["status"])
        s, o = PC.c_new(L, "pef", **kw)
        assert s == st and not o, (kw, s)
        assert what in L.afb200_lastError(), L.afb200_lastError()
    s, o = PC.c_new(L, "pef", r2=1)                         # n = 2: the default slide n/4 = 0 becomes 1
    assert s == 0 and L.pitchPEFObj_calTimeLength(o, 10) == 9
    L.pitchPEFObj_free(o)
    s, o = PC.c_new(L, "pef", r2=10)
    assert (PC.c_pitch(L, "pef", o, np.ones(1023, np.float32), fill=7.0, extra=4) == 7).all()
    v = np.zeros(4, np.float32)
    assert L.pitchPEFObj_pitchBatch(o, None, 2048, 1, v.ctypes.data, 0, None) != 0
    assert b"bad argument" in L.afb200_lastError()
    assert L.pitchPEFObj_pitchBatch(o, v.ctypes.data, 4, -1, v.ctypes.data, 0, None) != 0
    L.pitchPEFObj_free(o)
    L.pitchPEFObj_free(None)
    L.pitchPEFObj_pitch(None, None, 0, None)


def test_set_filter_params_changes_nothing():
    """the reference's setFilterParams recomputes the filter from the stored parameters: outputs stay the same"""
    lib = ref_lib_or_none()
    if lib is None:
        pytest.skip("needs the reference build")
    x = PC.signal("missing", 30000, 32000, 3)
    st, o = PC.c_new(lib, "pef", r2=12, slide=1024)
    before = PC.c_pitch(lib, "pef", o, x)
    lib.pitchPEFObj_setFilterParams(o, 3.0, 0.9, 1.2)
    after = PC.c_pitch(lib, "pef", o, x)
    lib.pitchPEFObj_free(o)
    st, o = PC.c_new(lib, "pef", r2=12, slide=1024, alpha=3.0, beta=0.9, gamma=1.2)
    other = PC.c_pitch(lib, "pef", o, x)
    lib.pitchPEFObj_free(o)
    assert np.array_equal(before, after) and not np.array_equal(before, other)


def test_pitch_pef_symbols_exported_and_bound(product_lib):
    from audioflux_b200 import capi
    check_symbols(product_lib, "afb200_pitch_pef.h", "pitchPEFObj_", capi.PITCH_PEF_API,
                  {"pitchPEFObj_new", "pitchPEFObj_calTimeLength", "pitchPEFObj_setFilterParams", "pitchPEFObj_pitch",
                   "pitchPEFObj_enableDebug", "pitchPEFObj_free"}, {"pitchPEFObj_pitchBatch"})


def test_python_class(product_lib):
    import audioflux_b200 as af
    h = af.PitchPEF()
    assert (h.samplate, h.low_fre, h.high_fre, h.cut_fre, h.radix2_exp, h.slide_length, h.window_type, h.alpha,
            h.beta, h.gamma, h.fft_length) == (32000, 32.0, 2000.0, 4000.0, 12, 1024, af.WindowType.HAMM, 10.0, 0.5,
                                               1.8, 4096)
    assert h.cal_time_length(160000) == (160000 - 4096) // 1024 + 1 and h.cal_time_length(4095) == 0
    for kw, msg in ((dict(low_fre=300.0, high_fre=200.0), "low_fre"), (dict(high_fre=5000.0), "high_fre"),
                    (dict(alpha=0.0), "alpha"), (dict(beta=1.5), "beta"), (dict(gamma=1.0), "gamma")):
        with pytest.raises(ValueError, match=msg):
            af.PitchPEF(**kw)
    with pytest.raises(ValueError, match="status -2"):
        af.PitchPEF(radix2_exp=14)
    with pytest.raises(ValueError, match="status -3: .*is empty"):
        af.PitchPEF(samplate=8000, high_fre=3999.5, cut_fre=4000.5)
    h.set_filter_params(2.0, 0.3, 1.5)
    assert (h.alpha, h.beta, h.gamma) == (2.0, 0.3, 1.5)
    with pytest.raises(ValueError, match="gamma"):
        h.set_filter_params(2.0, 0.3, 0.5)
    with pytest.raises(ValueError, match="at least one dimension"):
        h.pitch(np.float32(1))
    assert h.pitch(np.zeros((2, 3, 100), np.float32)).shape == (2, 3, 0)
    assert h.pitch_batch(np.zeros((0, 8000), np.float32)).shape == (0, 4)
    from audioflux_b200.lib import AfB200Error
    if product_lib.afb200_deviceCount() <= 0:          # no CPU fallback: the compute call fails loudly
        with pytest.raises(AfB200Error, match="no CUDA device"):
            h.pitch(np.ones(8000, np.float32))


if __name__ == "__main__":
    import sys
    if ref_lib_or_none() is None:
        sys.exit("oracle/_ref/libaudioflux_ref.so not built")
    print(f"{GOLD.name}: {GOLD.write()} arrays")
