"""PitchYIN without a GPU: the float64 interval oracle against the reference build (or its stored outputs in
tests/golden/pitch_yin.npz) over frame sizes, samplates, autocorrelation lengths, slides, thresholds, signals and the
shortest yin rows, for fre, value1, value2 and the trough rows; the statuses of new and calTimeLength against the
reference over a grid with NULL pointers and fallbacks; streaming in the reference; the refusals (which need no
device); the exported and bound symbols of include/afb200_pitch_yin.h and afb200_ext.h; and the Python
class's arguments.

Run as a script, it rewrites tests/golden/pitch_yin.npz from the reference build (oracle/_ref):

    python tests/test_pitch_yin_cpu.py"""
import numpy as np
import pytest

from _parity_kit import GoldenStore, check_symbols, ref_lib_or_none      # first: conftest puts the root on sys.path
import _pitch_c as PC
import _pitch_yin_oracle as YO

CASES = dict(YO.cases())
FILL = 7.0                       # the outputs start as this; frames without a trough keep it in fre and value1
PLANES = ("fre", "value1", "value2", "mfre", "mtrough", "lens")


def _live(keys):
    lib = ref_lib_or_none()
    out = {}
    for name in {k.split("/")[0] for k in keys}:
        res = dict(zip(PLANES, YO.c_case(lib, name, CASES[name], FILL)))
        # the reference leaves entries past each row's count from earlier calls: keep only the counted ones
        live = np.arange(res["mfre"].shape[1])[None, :] < res["lens"][:, None]
        res["mfre"], res["mtrough"] = np.where(live, res["mfre"], 0), np.where(live, res["mtrough"], 0)
        out.update({f"{name}/{k}": v for k, v in res.items()})
    return {k: out[k] for k in keys}


GOLD = GoldenStore("pitch_yin.npz", _live, lambda: {f"{c}/{k}" for c in CASES for k in PLANES})


def reference_outputs(name):
    g = GOLD.outputs({f"{name}/{k}" for k in PLANES})
    return [g[f"{name}/{k}"] for k in PLANES]


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference(name):
    kw = CASES[name]
    p = YO.case_params(kw)
    assert p["status"] == 0
    fre, v1, v2, mfre, mtrough, lens = reference_outputs(name)
    frames = YO.oracle_case(name, kw)
    ok, msg, alt = YO.check(fre, v1, v2, frames, p, FILL)
    assert ok, (name, msg)
    assert len(alt) <= max(2, len(frames) // 10), (name, alt)
    ok, msg = YO.check_troughs(mfre, mtrough, lens, frames, p)
    assert ok, (name, msg)
    has = lens > 0
    assert np.array_equal(mfre[has, 0], fre[has]) and np.array_equal(mtrough[has, 0], v1[has])
    assert (fre[~has] == FILL).all() and (v1[~has] == FILL).all()


def test_cases_cover_the_parameters():
    """radix2Exp 8 .. 14, the seven samplates, autoLength 0 / small / n/2 / clamped, slides below / at / above n,
    yinLength 1 and 2, thresholds at and above 1, and frames with and without a trough"""
    ps = {k: YO.case_params(kw) for k, kw in CASES.items()}
    assert {p["r2"] for p in ps.values()} >= set(range(8, 15)) | {1}
    assert {p["sr"] for p in ps.values()} >= {8000, 16000, 22050, 32000, 44100, 48000, 96000}
    assert ps["auto0"]["auto"] == 0 and ps["auto_near_n"]["max_index"] == ps["auto_near_n"]["n"] - 1901
    assert ps["slide_lt_n"]["slide"] < 2048 == ps["slide_eq_n"]["slide"] < ps["slide_gt_n"]["slide"]
    assert ps["yin1"]["yin_length"] == 1 and ps["yin2"]["yin_length"] == 2 == ps["yin2_exact"]["yin_length"]
    assert ps["default_null"]["high"] == 2094 and ps["hf_rejected"]["high"] == 2093
    assert {kw["thresh"] for kw in CASES.values()} >= {None, 0.05, 0.3, 0.9, 1.5}


def test_golden_file_matches_reference_build():
    GOLD.check_file()


def _grid():
    grid = []
    for sr in (None, -1, 2000, 8000, 11025, 32000, 196001):
        for lf in (None, 20.0, 27.0, 300.0):
            for hf in (None, 90.0, 1000.0, 5000.0, 20000.0):
                for r2 in (None, 0, 3, 11, 14, 15, 31):
                    for auto in (None, -1, 0, 100, 1020, 1 << 20):
                        grid.append(dict(sr=sr, lf=lf, hf=hf, r2=r2, auto=auto))
    rng = np.random.default_rng(0)
    return [grid[i] for i in rng.choice(len(grid), 400, replace=False)]


def test_statuses_match_reference(product_lib, ref_lib):
    """new accepts exactly what the oracle accepts, refuses the rest with the oracle's status, and calTimeLength agrees
    with the reference wherever both build the object"""
    seen = set()
    for kw in _grid():
        for slide in (None, 700):
            p = YO.params(**kw, slide=slide)
            st_p, o_p = PC.c_new(product_lib, "yin", **kw, slide=slide)
            assert st_p == p["status"], (kw, slide, st_p, p["status"])
            seen.add(st_p)
            if st_p:
                assert not o_p
                continue
            st_r, o_r = PC.c_new(ref_lib, "yin", **kw, slide=slide)
            assert st_r == 0
            for n in (0, 1, p["n"] - 1, p["n"], p["n"] + 1, p["n"] + p["slide"], 5 * p["n"] + 3, 100000):
                got = product_lib.pitchYINObj_calTimeLength(o_p, n)
                assert got == PC.time_length(n, p["n"], p["slide"]) == ref_lib.pitchYINObj_calTimeLength(o_r, n)
            assert product_lib.pitchYINObj_getTroughData(o_p, None, None, None) == p["m_len"]
            product_lib.pitchYINObj_free(o_p)
            ref_lib.pitchYINObj_free(o_r)
    assert seen == {0, -2, -3}, seen


def test_streaming_in_the_reference():
    """isContinue: pieces of a clip (some shorter than a frame) give the frames of one call over the clip, with a slide
    below n and one above it (a negative carry); calTimeLength counts the carry"""
    lib = ref_lib_or_none()
    if lib is None:
        pytest.skip("needs the reference build")
    x = PC.signal("glide", 40000, 16000, 5)
    for r2, slide in ((11, 512), (10, 1500)):
        st, whole = PC.c_new(lib, "yin", sr=16000, r2=r2, slide=slide)
        want = PC.c_pitch(lib, "yin", whole, x)
        st, o = PC.c_new(lib, "yin", sr=16000, r2=r2, slide=slide, cont=1)
        got = PC.c_stream(lib, "yin", o, x, (700, 3000, 100, 9000, 1, 27199))
        for g, w in zip(got, want):
            assert np.array_equal(g, w), (r2, slide)
        lib.pitchYINObj_free(o)
        lib.pitchYINObj_free(whole)


def test_refusals(product_lib):
    """radix2Exp above 14, minIndex 0 and an empty lag range are refused at construction with a status and a reason;
    the object pointer stays NULL"""
    L = product_lib
    for kw, st, what in ((dict(r2=15), -2, b"largest supported is 14"),
                         (dict(r2=30), -2, b"largest supported is 14"),
                         (dict(sr=2000), -3, b"minIndex=0"),
                         (dict(sr=1500, r2=10, slide=256), -3, b"minIndex=0"),
                         (dict(sr=8000, r2=10, auto=1021), -3, b"yinLength=0 is empty")):
        p = YO.params(**kw)
        assert p["status"] == st, (kw, p["status"])
        s, o = PC.c_new(L, "yin", **kw)
        assert s == st and not o, (kw, s)
        assert what in L.afb200_lastError(), L.afb200_lastError()
    s, o = PC.c_new(L, "yin", sr=4000, r2=1, auto=0)          # n = 2: the default slide n/4 = 0 becomes 1
    assert s == 0 and L.pitchYINObj_calTimeLength(o, 10) == 9
    L.pitchYINObj_free(o)
    s, o = PC.c_new(L, "yin", r2=10)
    assert all((v == 7).all() for v in PC.c_pitch(L, "yin", o, np.ones(1023, np.float32), fill=7.0, extra=4))
    assert L.pitchYINObj_getTroughData(o, None, None, None) == YO.params(r2=10)["m_len"]
    v = np.zeros(4, np.float32)
    assert L.pitchYINObj_pitchBatch(o, None, 2048, 1, v.ctypes.data, None, None, None, None, None, 0, None) != 0
    assert b"bad argument" in L.afb200_lastError()
    assert L.pitchYINObj_pitchBatch(o, v.ctypes.data, 4, -1, v.ctypes.data, None, None, None, None, None, 0, None) != 0
    assert L.pitchYINObj_pitchBatch(o, v.ctypes.data, 2048, 1, None, None, None, None, None, None, 0, None) != 0
    L.pitchYINObj_setThresh(o, -1.0)
    L.pitchYINObj_enableDebug(o, 1)
    L.pitchYINObj_free(o)
    L.pitchYINObj_free(None)
    L.pitchYINObj_pitch(None, None, 0, None, None, None)


def test_pitch_yin_symbols_exported_and_bound(product_lib):
    from audioflux_b200 import capi
    check_symbols(product_lib, "afb200_pitch_yin.h", "pitchYINObj_", capi.PITCH_YIN_API,
                  {"pitchYINObj_new", "pitchYINObj_setThresh", "pitchYINObj_calTimeLength", "pitchYINObj_pitch",
                   "pitchYINObj_getTroughData", "pitchYINObj_enableDebug", "pitchYINObj_free"},
                  {"pitchYINObj_pitchBatch"})


def test_python_class(product_lib):
    import audioflux_b200 as af
    h = af.PitchYIN()
    assert (h.samplate, h.low_fre, h.high_fre, h.radix2_exp, h.slide_length, h.auto_length, h.thresh,
            h.fft_length) == (32000, 27.0, 2000.0, 12, 1024, 2048, 0.1, 4096)
    assert h.cal_time_length(160000) == (160000 - 4096) // 1024 + 1 and h.cal_time_length(4095) == 0
    for th in (0.0, 1.0, -0.5, 1.5):
        with pytest.raises(ValueError, match="thresh"):
            h.set_thresh(th)
    h.set_thresh(0.3)
    assert h.thresh == 0.3
    with pytest.raises(ValueError, match="status -2"):
        af.PitchYIN(radix2_exp=15)
    with pytest.raises(ValueError, match="status -3: .*minIndex=0"):
        af.PitchYIN(samplate=1500, radix2_exp=10, slide_length=256, auto_length=512)
    with pytest.raises(ValueError, match="status -3: .*is empty"):
        af.PitchYIN(samplate=8000, radix2_exp=10, slide_length=256, auto_length=1021)
    with pytest.raises(ValueError, match="at least one dimension"):
        h.pitch(np.float32(1))
    assert all(o.shape == (2, 3, 0) for o in h.pitch(np.zeros((2, 3, 100), np.float32)))
    assert all(o.shape == (0, 4) for o in h.pitch_batch(np.zeros((0, 8000), np.float32)))
    from audioflux_b200.lib import AfB200Error
    if product_lib.afb200_deviceCount() <= 0:          # no CPU fallback: the compute call fails loudly
        with pytest.raises(AfB200Error, match="no CUDA device"):
            h.pitch(np.ones(8000, np.float32))


if __name__ == "__main__":
    import sys
    if ref_lib_or_none() is None:
        sys.exit("oracle/_ref/libaudioflux_ref.so not built")
    print(f"{GOLD.name}: {GOLD.write()} arrays")
