"""Onset detection without a GPU: the numpy oracle against the reference build (or its stored outputs in
tests/golden/onset.npz) over every novelty type, filter order, bin list, step, parameter variation and peak-parameter
set; the peak parameters of onsetObj_new; the refusals (which need no device); the exported and bound symbols of
include/afb200_onset.h and afb200_ext.h; and the Python class's argument checks."""
import ctypes as C

import numpy as np
import pytest

import _onset_oracle as OO
from _parity_kit import GoldenStore, check_symbols, ref_lib_or_none

TOL = 1e-4                 # absolute: evn is normalised to [0, 1]
CASES = dict(OO.cases())


def _live(keys):
    lib = ref_lib_or_none()
    out = {}
    for n in sorted({k.split("__")[0] for k in keys}):
        evn, pts = OO.c_case(lib, n, CASES[n])
        out[f"{n}__evn"], out[f"{n}__pts"] = evn, pts
    return {k: v for k, v in out.items() if k in keys}


def _golden_keys():
    return {f"{n}__{k}" for n in CASES for k in ("evn", "pts")}


GOLD = GoldenStore("onset.npz", _live, _golden_keys)


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference(name):
    kw = CASES[name]
    out = GOLD.outputs({f"{name}__evn", f"{name}__pts"})
    evn, pts = out[f"{name}__evn"], out[f"{name}__pts"]
    pp = OO.peak_params(kw["sr"], kw["hop"])
    # the peak picking restated exactly: on the reference's own curve it gives the reference's points
    assert np.array_equal(OO.pick(evn, pp), pts), name
    want_evn, want_pts = OO.oracle_case(name, kw)
    assert evn.shape == want_evn.shape
    assert np.abs(evn.astype(np.float64) - want_evn).max() <= TOL, name
    assert np.array_equal(want_pts, pts), (name, want_pts, pts)


def test_grid_has_points():
    """the cases are not vacuous: most clips have several onsets, the click trains one per click"""
    counts = [len(OO.oracle_case(n, kw)[1]) for n, kw in CASES.items()]
    assert np.median(counts) >= 5 and min(counts) >= 1


def test_golden_file_matches_reference_build():
    GOLD.check_file()


def _debug(lib, o, capfd):
    lib.onsetObj_debug(o)
    C.CDLL(None).fflush(None)
    return capfd.readouterr().out


@pytest.mark.parametrize("sr,hop", [(None, 512), (32000, 512), (8000, 512), (44100, 256), (22050, 0), (-5, -1),
                                    (48000, 100), (16000, 4096)])
def test_peak_parameters(product_lib, capfd, sr, hop):
    """onsetObj_debug's peak parameters are the oracle's (and the reference build's, where it is built)"""
    st, o = OO.c_new(product_lib, 200, 64, hop, sr, 3)
    assert st == 0
    got = _debug(product_lib, o, capfd)
    product_lib.onsetObj_free(o)
    pm, qm, pa, qa, w, d = OO.peak_params(sr, hop)
    assert f"preMax={pm},postMax={qm}, preAvg={pa},postAvg={qa}, wait={w},delta={d:f}" in got, got
    assert "timeLength=200,freNum=64, step=0,order=3" in got, got
    ref = ref_lib_or_none()
    if ref is not None:
        st, o = OO.c_new(ref, 200, 64, hop, sr, 3)
        assert _debug(ref, o, capfd) == got
        ref.onsetObj_free(o)


def _refused(lib, o, x, ph=None, prm=OO.DEFAULT_PARAM, idx=None, what=b""):
    """onsetObj_onset and onsetObj_onsetBatch both refuse, leave their outputs as they were and say why"""
    evn, pts, n, whole = OO.c_onset(lib, o, x, ph, prm, idx, fill=7)
    assert n == 0 and (evn == 7).all() and (whole == 7).all()
    assert what in lib.afb200_lastError(), lib.afb200_lastError()
    T = max(x.shape[0], 1)
    e, p, c = np.full(T, 7, np.float32), np.full(T, 7, np.int32), np.full(1, 7, np.int32)
    par = None if prm is None else OO.NoveltyParam(*prm)
    rc = lib.onsetObj_onsetBatch(o, x.ctypes.data, None if ph is None else ph.ctypes.data,
                                 1, None if par is None else C.addressof(par), None if idx is None else idx.ctypes.data,
                                 0 if idx is None else len(idx), e.ctypes.data, p.ctypes.data, c.ctypes.data, 0, None)
    assert rc != 0 and what in lib.afb200_lastError()
    assert (e == 7).all() and (p == 7).all() and (c == 7).all()


def test_refusals(product_lib):
    """every refusal happens before any device work, so it holds without a GPU"""
    L = product_lib
    x, ph = OO.case_signal("refusal", dict(T=50, M=32))
    for T, M in ((0, 32), (50, 0), (-3, 32)):
        st, o = OO.c_new(L, T, M, 512)
        assert st == 0
        _refused(L, o, x, what=b"must be at least 1")
        L.onsetObj_free(o)
    st, o = OO.c_new(L, 50, 32, 512, None, 3, 0)
    for idx in ([0, 5, 32], [-1], [31, 40]):
        _refused(L, o, x, idx=np.array(idx, np.int32), what=b"outside [0, 32)")
    _refused(L, o, x, idx=np.zeros(0, np.int32), what=b"indexLength=0")
    _refused(L, o, x, prm=(51,) + OO.DEFAULT_PARAM[1:], what=b"step=51 is above nLength=50")
    L.onsetObj_free(o)
    for kind in OO.PHASE:
        st, o = OO.c_new(L, 50, 32, 512, None, 1, kind)
        _refused(L, o, x, what=b"needs the phase")
        L.onsetObj_free(o)
    # bad arguments of the batch
    st, o = OO.c_new(L, 50, 32, 512)
    e = np.zeros(50, np.float32)
    p = np.zeros(50, np.int32)
    for args in ((None, None, 1, None, None, 0, e.ctypes.data, p.ctypes.data, p.ctypes.data),
                 (x.ctypes.data, None, -1, None, None, 0, e.ctypes.data, p.ctypes.data, p.ctypes.data),
                 (x.ctypes.data, None, 1, None, None, 0, None, p.ctypes.data, p.ctypes.data),
                 (x.ctypes.data, None, 1, None, None, 0, e.ctypes.data, p.ctypes.data, None)):
        assert L.onsetObj_onsetBatch(o, *args, 0, None) != 0
        assert b"bad argument" in L.afb200_lastError()
    assert L.onsetObj_onset(o, None, None, None, None, 0, e.ctypes.data, p.ctypes.data) == 0
    assert L.onsetObj_onset(None, x.ctypes.data, None, None, None, 0, e.ctypes.data, p.ctypes.data) == 0
    L.onsetObj_free(o)
    L.onsetObj_free(None)
    L.onsetObj_debug(None)


def test_constructor_status_matches_reference(product_lib, ref_lib):
    for T, M, hop, sr, order, kind in ((100, 64, 512, None, None, None), (1, 1, 0, 0, 0, 3), (100, 64, -4, -1, -7, 10),
                                       (300, 2049, 256, 44100, 5, 5)):
        for lib in (product_lib, ref_lib):
            st, o = OO.c_new(lib, T, M, hop, sr, order, kind)
            assert st == 0 and o
            lib.onsetObj_free(o)


def test_onset_symbols_exported_and_bound(product_lib):
    from audioflux_b200 import capi
    check_symbols(product_lib, "afb200_onset.h", "onsetObj_", capi.ONSET_API,
                  {"onsetObj_new", "onsetObj_onset", "onsetObj_free", "onsetObj_debug"}, {"onsetObj_onsetBatch"})


def test_python_class_checks(product_lib):
    import audioflux_b200 as af
    o = af.Onset(time_length=40, fre_length=16, slide_length=256)
    assert (o.time_length, o.fre_length, o.slide_length, o.samplate, o.filter_order, o.novelty_type) == \
        (40, 16, 256, 32000, 1, af.NoveltyType.FLUX)
    assert [t.value for t in af.NoveltyType] == list(range(11))
    assert [f for f, _ in af.NoveltyParam._fields_] == [f for f, _ in OO.NoveltyParam._fields_]
    assert C.sizeof(af.NoveltyParam) == C.sizeof(OO.NoveltyParam) == 32
    with pytest.raises(ValueError, match="two dimensions"):
        o.onset(np.zeros(16, np.float32))
    with pytest.raises(ValueError, match="same shape"):
        o.onset(np.zeros((16, 40), np.float32), np.zeros((16, 41), np.float32))
    with pytest.raises(ValueError, match="NoveltyParam"):
        o.onset(np.zeros((16, 40), np.float32), novelty_param=(1, 2, 0, 1, 0, 0, 0, 1))
    with pytest.raises(ValueError, match="time_length, fre_length"):
        o.onset(np.zeros((16, 41), np.float32))
    with pytest.raises(ValueError, match="needs the phase"):
        af.Onset(40, 16, 256, novelty_type=af.NoveltyType.CD).onset(np.zeros((16, 40), np.float32))
    # no clips: no device work, empty results of the right shapes
    evn, pts, counts = o.onset_batch(np.zeros((0, 40, 16), np.float32))
    assert evn.shape == pts.shape == (0, 40) and counts.shape == (0,) and pts.dtype == counts.dtype == np.int32
    from audioflux_b200.lib import AfB200Error
    with pytest.raises(AfB200Error, match="step=41"):
        o.onset(np.zeros((16, 40), np.float32), novelty_param=af.NoveltyParam(41, 1, 1, 0, 1, 0, 1, 1))
    if product_lib.afb200_deviceCount() <= 0:          # no CPU fallback: the compute call fails loudly
        with pytest.raises(AfB200Error, match="no CUDA device"):
            o.onset(np.ones((16, 40), np.float32))
