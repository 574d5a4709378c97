"""Spectral descriptors without a GPU: the numpy oracle against the reference build (or its stored outputs in
tests/golden/spectral.npz), frame by frame on the crafted rows and rolloff look-back runs of tests/_spectral_frames.py
(tests/golden/spectral_frames.npz), the argument rules of SpectralObj, the exported C API and the loud failure without a
GPU.

Run as a script, it rewrites tests/golden/spectral_frames.npz from the reference build (oracle/_ref):

    python tests/test_spectral_cpu.py"""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT
import _spectral_cases as SC
import _spectral_frames as SF
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


def test_frames_golden_file_matches_reference_build():
    GOLD_FRAMES.check_file()


def _frame_cases():
    """(case, x [B, T, num], phase or None, fre, mode, idx, variants): the crafted rows in each bin-list mode, a quiet
    and a loud clip over one bin and over two (where log(1 + u) rounds 1 + u to float32), and the two rolloff
    look-back clips"""
    for mode, idx in SF.extreme_modes().items():
        x, ph, fre = SF.extreme_clip(mode)
        yield f"crafted-{mode}", x[None], ph[None], fre, mode, idx, SC.VARIANTS
    for setname, mode in (("linear", "one"), ("cqt", "two")):    # a quiet clip (1e-2) and a loud one (1e2)
        x, ph, fre = SF.clips(setname, 40, 2, seed=6)
        yield f"quiet-{setname}-{mode}", x, ph, fre, mode, SF.bin_sets()[(setname, mode)], \
            [v for v in SC.VARIANTS if ph is not None or v[0] not in SC.SO.PHASE]
    for kind, variants in SF.LOOKBACK_VARIANTS.items():
        x, fre, _, _ = SF.lookback_clips(kind)
        yield f"lookback-{kind}", x, None, fre, "full", list(range(x.shape[-1])), \
            [v for v in variants or SC.VARIANTS if v[0] not in SC.SO.PHASE]


def _frame_key(case, b, variant, part):
    name, kw = variant
    return f"{case}/{b}/{name}{sorted(kw.items())}/{part}"


def _frame_keys():
    return {_frame_key(case, b, v, part) for case, x, _, _, _, _, variants in _frame_cases()
            for v in variants for b in range(x.shape[0]) for part in range(2 if v[0] in SC.TWO_OUTPUTS else 1)}


def _frame_live(keys):
    lib = ref_lib_or_none()
    res = {}
    for case, x, ph, fre, mode, idx, variants in _frame_cases():
        for v in variants:
            for b in range(x.shape[0]):
                out = SC.call_c(lib, v[0], x[b], fre, mode, None if ph is None else ph[b], idx=idx, **v[1])
                for part, o in enumerate(out if isinstance(out, tuple) else (out,)):
                    if _frame_key(case, b, v, part) in keys:
                        res[_frame_key(case, b, v, part)] = o
    return res


GOLD_FRAMES = GoldenStore("spectral_frames.npz", _frame_live, _frame_keys,
                          equal=lambda a, b: SC.agree(a, b, exact=True) is None)


def test_oracle_matches_reference_frame_by_frame():
    """NaN / +-inf / denormal / negative / zero / tied rows, one- and two-bin lists of a quiet clip, and rolloff runs
    without a crossing: inputs of tests/test_gpu_spectral_frames.py on which the GPU is judged by the oracle, each
    frame on its own scale"""
    ref = GOLD_FRAMES.outputs(_frame_keys())
    rep = SF.Report()
    for case, x, ph, fre, mode, idx, variants in _frame_cases():
        for v in variants:
            for b in range(x.shape[0]):
                nparts = 2 if v[0] in SC.TWO_OUTPUTS else 1
                got = [ref[_frame_key(case, b, v, part)] for part in range(nparts)]
                SF.check_clip(rep, f"{case} b={b}", v[0], v[1], got, x[b], idx, fre, None if ph is None else ph[b])
    assert rep.ok(), rep.text()


@pytest.mark.parametrize("kind", list(SF.LOOKBACK_VARIANTS))
def test_look_back_runs_are_what_they_claim(kind):
    """the frames lookback_clips marks as crossing are exactly those whose rolloff crosses in the oracle's float32, and
    every non-crossing run of 5 .. 70 frames is there"""
    x, fre, thr, cross = SF.lookback_clips(kind)
    for b in range(2):
        r = np.asarray(x[b], np.float32)
        s = np.add.accumulate(r, axis=1, dtype=np.float32)[:, -1]
        with np.errstate(invalid="ignore"):
            hit = (np.add.accumulate(np.abs(r), axis=1, dtype=np.float32) >= (s * np.float32(thr))[:, None]).any(1)
        assert np.array_equal(hit, cross[b]), kind
    runs = [len(r) for b in range(2) for r in "".join("x" if c else "." for c in cross[b]).split("x") if r]
    assert {5, 31, 32, 33, 64, 70} <= set(runs) and not cross[0, 0] and not cross[1, 0]


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


if __name__ == "__main__":
    import sys
    if ref_lib_or_none() is None:
        sys.exit("oracle/_ref/libaudioflux_ref.so not built")
    print(f"{GOLD_FRAMES.name}: {GOLD_FRAMES.write()} arrays")
