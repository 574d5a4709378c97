"""Spectral descriptors without a GPU: the numpy oracle against the reference build (or its stored outputs in
tests/golden/spectral.npz), the argument rules of SpectralObj, the exported C API and the loud failure without a GPU."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT
import _spectral_cases as SC
from _parity_kit import GoldenStore, check_symbols, ref_lib_or_none

import audioflux_b200 as af
from audioflux_b200 import capi


def _key(setname, mode, vi, part=0):
    return f"{setname}/{mode}/{vi}/{part}"


def _cases():
    for setname, x, ph, fre in SC.spectrogram_sets():
        for mode in ("full", "range", "list"):
            for vi, (name, kw) in enumerate(SC.VARIANTS):
                if name in SC.SO.PHASE and ph is None:
                    continue
                yield setname, x, ph, fre, mode, vi, name, kw


def _keys():
    return {_key(setname, mode, vi, part) for setname, _, _, _, mode, vi, name, _ in _cases()
            for part in range(2 if name in SC.TWO_OUTPUTS else 1)}


def _live(keys):
    lib = ref_lib_or_none()
    res = {}
    for setname, x, ph, fre, mode, vi, name, kw in _cases():
        out = SC.call_c(lib, name, x, fre, mode, ph, **kw)
        for part, o in enumerate(out if isinstance(out, tuple) else (out,)):
            if _key(setname, mode, vi, part) in keys:
                res[_key(setname, mode, vi, part)] = o
    return res


GOLD = GoldenStore("spectral.npz", _live, _keys, equal=lambda a, b: SC.agree(a, b, exact=True) is None)


@pytest.fixture(scope="module")
def ref_out():
    return GOLD.outputs(_keys())


def test_oracle_matches_reference(ref_out):
    bad = []
    for setname, x, ph, fre, mode, vi, name, kw in _cases():
        want = SC.oracle(name, x, fre, mode, ph, **kw)
        for part, w in enumerate(want if isinstance(want, tuple) else (want,)):
            r = ref_out[_key(setname, mode, vi, part)]
            msg = SC.agree(w, r, exact=SC.is_exact(name, kw) or (name == "max" and part == 1))
            if msg:
                bad.append(f"{setname}/{mode}/{name}{kw}[{part}]: {msg}")
    assert not bad, "\n".join(bad[:20])


def test_golden_file_matches_reference_build():
    GOLD.check_file()


def test_constructor_and_edge_rules(product_lib):
    lib = product_lib
    obj = C.c_void_p()
    assert lib.spectralObj_new(C.byref(obj), 1, None) == -1
    fre = np.arange(16, dtype=np.float32)
    assert lib.spectralObj_new(C.byref(obj), 16, fre.ctypes.data) == 0
    lib.spectralObj_setEdge(obj, 5, 16)          # end > num-1: ignored
    lib.spectralObj_setEdge(obj, 4, 4)           # empty: ignored
    lib.spectralObj_setEdge(obj, -1, 3)          # ignored
    lib.spectralObj_setEdge(obj, 2, 9)           # accepted
    # setEdgeArr takes ownership: an invalid list is freed and ignored, a valid one replaces (and frees) the old one
    for idx in ([3, 99], [5, 1, 5, 0], [15, -1], [2, 2]):
        p = SC._libc.calloc(len(idx), 4)
        (C.c_int * len(idx)).from_address(p)[:] = idx
        lib.spectralObj_setEdgeArr(obj, C.c_void_p(p), len(idx))
    lib.spectralObj_free(obj)
    with pytest.raises(ValueError):
        af.Spectral(1, np.zeros(1, np.float32))
    s = af.Spectral(16, fre)
    with pytest.raises(ValueError):
        s.set_edge(3, 16)
    with pytest.raises(ValueError):
        s.set_edge(5, 5)
    s.set_edge_arr([4, 2, 2, 9])
    with pytest.raises(ValueError):
        s.spectral_batch(np.zeros((3, 15), np.float32), ["centroid"])
    with pytest.raises(ValueError):
        s.spectral_batch(np.zeros((3, 16), np.float32), ["pd"])
    with pytest.raises(ValueError):
        s.spectral_batch(np.zeros((3, 16), np.float32), ["nope"])


def test_batch_rejects_bad_requests(product_lib):
    lib = product_lib
    obj = C.c_void_p()
    assert lib.spectralObj_new(C.byref(obj), 8, None) == 0
    x = np.ones((2, 8), np.float32)
    out = np.full(4, 7.0, np.float32)
    par = np.zeros(4, np.float32)
    for req in (99, 3):      # unknown id; centroid without freBandArr
        r = np.array([req], np.int32)
        assert lib.spectralObj_spectralBatch(obj, x.ctypes.data, None, 2, 1, 1, r.ctypes.data, par.ctypes.data,
                                             out.ctypes.data, 0, None) != 0
    r = np.array([18], np.int32)  # pd without phase planes
    assert lib.spectralObj_spectralBatch(obj, x.ctypes.data, None, 2, 1, 1, r.ctypes.data, par.ctypes.data,
                                         out.ctypes.data, 0, None) != 0
    assert (out == 7.0).all()
    lib.spectralObj_free(obj)


def test_spectral_api_declared_and_exported(product_lib):
    check_symbols(product_lib, "afb200_spectral.h", "spectralObj_", capi.SPECTRAL_API, 35,
                  {"spectralObj_spectralBatch"})


def test_feature_ids_match_header():
    src = open(os.path.join(ROOT, "include", "afb200_ext.h")).read()
    body = src[src.index("AFB200_SPECTRAL_FLATNESS = 0"):src.index("AFB200_SPECTRAL_COUNT")]
    ids = [n.lower() for n in re.findall(r"AFB200_SPECTRAL_([A-Z]+)", body)]
    from audioflux_b200 import spectral
    assert [n.replace("_", "") for n in spectral.FEATURES] == ids


def test_no_gpu_means_loud_failure_spectral(product_lib):
    if product_lib.afb200_deviceCount() > 0:
        return
    fre = np.arange(32, dtype=np.float32)
    s = af.Spectral(32, fre)
    x = np.ones((2, 5, 32), np.float32)
    with pytest.raises(af.lib.AfB200Error, match="no CUDA device"):
        s.spectral_batch(x, ["centroid", "flux"])
    out = np.full(5, 7.0, np.float32)
    obj = C.c_void_p()
    assert product_lib.spectralObj_new(C.byref(obj), 32, fre.ctypes.data) == 0
    product_lib.spectralObj_setTimeLength(obj, 5)
    product_lib.spectralObj_centroid(obj, x[0].ctypes.data, out.ctypes.data)
    assert (out == 7.0).all()
    assert b"no CUDA device" in product_lib.afb200_lastError()
    product_lib.spectralObj_free(obj)
