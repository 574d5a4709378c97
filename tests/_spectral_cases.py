"""Inputs, parameter variants and a ctypes driver of the reference's SpectralObj C functions, shared by
tests/test_spectral_cpu.py and tests/test_gpu_spectral.py.  The driver works on any library exporting those symbols
(the reference build or libaudioflux_b200.so) and gives every call a fresh object, so the reference's cached sums
(src/feature/spectral_algorithm.c:150-157) never leak from one call into the next."""
import ctypes as C

import numpy as np

import _spectral_oracle as SO

_libc = C.CDLL(None)
_libc.calloc.restype = C.c_void_p
_libc.calloc.argtypes = [C.c_size_t, C.c_size_t]

NOVELTY = [dict(method_type=m, data_type=d, threshold=th) for m in range(4) for d in range(2) for th in (0., 0.5)]
VARIANTS = [
    ("flatness", {}), ("flux", {}), ("flux", dict(step=2, p=1, is_positive=True, is_exp=True, tp=1)),
    ("flux", dict(p=3, is_exp=True)), ("rolloff", {}), ("rolloff", dict(threshold=0.5)), ("rolloff", dict(threshold=1.5)),
    ("centroid", {}), ("spread", {}), ("skewness", {}), ("kurtosis", {}), ("entropy", {}), ("entropy", dict(is_norm=True)),
    ("crest", {}), ("slope", {}), ("decrease", {}), ("band_width", {}), ("band_width", dict(p=4)),("band_width", dict(p=3)),
    ("rms", {}), ("energy", {}), ("energy", dict(is_log=True, gamma=5.)), ("energy", dict(is_log=True, gamma=-1.)),
    ("hfc", {}), ("sd", {}), ("sd", dict(step=3, is_positive=True)), ("sf", {}), ("sf", dict(step=2, is_positive=True)),
    ("mkl", {}), ("mkl", dict(tp=1)), ("pd", {}), ("wpd", {}), ("nwpd", {}), ("cd", {}), ("rcd", {}),
    ("broadband", {}), ("broadband", dict(threshold=3.)), ("eef", {}), ("eef", dict(is_norm=True)), ("eer", {}),
    ("eer", dict(is_norm=True, gamma=10.)), ("max", {}), ("mean", {}), ("var", {}),
] + [("novelty", kw) for kw in NOVELTY]
EXACT = ("rolloff", "max", "broadband")        # integer outcomes (and novelty with data_type NUMBER)


def is_exact(name, kw):
    return name in EXACT or (name == "novelty" and kw.get("data_type", 0) == 1)


def spectrogram_sets(seed=0, T=14):
    """(name, x [T, num] float32, phase or None, fre [num]): Linear magnitude with phase, Mel power, CQT magnitude;
    frame 5 of each is all zero."""
    rng = np.random.default_rng(seed)
    out = []
    for name, num, power, with_phase in (("linear", 1025, False, True), ("mel", 128, True, False), ("cqt", 84, False, False)):
        x = np.abs(rng.standard_normal((T, num))).astype(np.float32) * np.linspace(2, 0.1, num, dtype=np.float32)
        if power:
            x = (x * x).astype(np.float32)
        x[5] = 0
        ph = rng.uniform(-np.pi, np.pi, (T, num)).astype(np.float32) if with_phase else None
        fre = (np.arange(num) * 48000.0 / 2048).astype(np.float32) if name == "linear" else \
            np.geomspace(30, 16000, num).astype(np.float32)
        out.append((name, x, ph, fre))
    return out


def edges(num):
    """edge mode -> bin list: full, setEdge range, unsorted setEdgeArr with a duplicate"""
    return {"full": list(range(num)), "range": list(range(3, num // 2 + 1)),
            "list": [num // 3, 1, num - 1, 7, num // 3, 0, num // 2, 2]}


def apply_edge(lib, obj, mode, num, idx=None):
    """mode 'full', 'range...' (setEdge) or any other name (setEdgeArr) over edges(num)[mode], or over idx when given"""
    idx = edges(num)[mode] if idx is None else list(idx)
    if mode.startswith("range"):
        lib.spectralObj_setEdge(obj, idx[0], idx[-1])
    elif mode != "full":
        p = _libc.calloc(len(idx), 4)
        (C.c_int * len(idx)).from_address(p)[:] = idx
        lib.spectralObj_setEdgeArr(obj, C.c_void_p(p), len(idx))     # the object owns the array from here on
    return idx


TWO_OUTPUTS = ("max", "mean", "var")        # features whose call returns (value, fre)


def call_c(lib, name, x, fre, mode="full", phase=None, idx=None, **kw):
    """one reference-signature call on a fresh object; x [T, num] -> [T] (or (value, fre) for max / mean / var).
    idx: the bin list of the mode in place of edges(num)[mode]"""
    x = np.ascontiguousarray(x, np.float32)
    T, num = x.shape
    fre = np.ascontiguousarray(fre, np.float32)
    obj = C.c_void_p()
    assert lib.spectralObj_new(C.byref(obj), num, fre.ctypes.data) == 0
    apply_edge(lib, obj, mode, num, idx)
    lib.spectralObj_setTimeLength(obj, T)
    o1, o2 = np.zeros(T, np.float32), np.zeros(T, np.float32)
    X, O1, O2 = x.ctypes.data, o1.ctypes.data, o2.ctypes.data
    ph = None if phase is None else np.ascontiguousarray(phase, np.float32)
    ib = lambda v: C.byref(C.c_int(int(v)))
    fn = getattr(lib, "spectralObj_" + ("bandWidth" if name == "band_width" else name))
    if name == "flux":
        fn(obj, X, kw.get("step", 1), kw.get("p", 2), int(kw.get("is_positive", False)), ib(kw.get("is_exp", False)),
           ib(kw.get("tp", 0)), O1)
    elif name == "rolloff":
        fn(obj, X, kw.get("threshold", 0.95), O1)
    elif name in ("entropy", "eef"):
        fn(obj, X, int(kw.get("is_norm", False)), O1)
    elif name == "eer":
        fn(obj, X, int(kw.get("is_norm", False)), kw.get("gamma", 1.), O1)
    elif name == "band_width":
        fn(obj, X, kw.get("p", 2), O1)
    elif name == "energy":
        fn(obj, X, int(kw.get("is_log", False)), kw.get("gamma", 10.), O1)
    elif name in ("sd", "sf"):
        fn(obj, X, kw.get("step", 1), int(kw.get("is_positive", False)), O1)
    elif name == "mkl":
        fn(obj, X, kw.get("tp", 0), O1)
    elif name in SO.PHASE:
        fn(obj, X, ph.ctypes.data, O1)
    elif name == "broadband":
        fn(obj, X, kw.get("threshold", 0), O1)
    elif name == "novelty":
        fn(obj, X, kw.get("step", 1), kw.get("threshold", 0.), ib(kw.get("method_type", 0)), ib(kw.get("data_type", 0)), O1)
    elif name in TWO_OUTPUTS:
        fn(obj, X, O1, O2)
    else:
        fn(obj, X, O1)
    lib.spectralObj_free(obj)
    return (o1, o2) if name in TWO_OUTPUTS else o1


def oracle(name, x, fre, mode="full", phase=None, **kw):
    return SO.compute(name, x, edges(x.shape[1])[mode], fre, phase, **kw)


def agree(got, want, exact=False, tol=1e-4):
    """NaN / inf positions equal; exact: equal values; else max|a-b| <= tol * max|b| over the finite values"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    if got.shape != want.shape:
        return f"shape {got.shape} != {want.shape}"
    if not (np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(np.isposinf(got), np.isposinf(want))
            and np.array_equal(np.isneginf(got), np.isneginf(want))):
        return f"non-finite positions differ: {got} vs {want}"
    fin = np.isfinite(want)
    g, w = got[fin], want[fin]
    if exact:
        return None if np.array_equal(g, w) else f"not exact at {np.flatnonzero(g != w)[:8]}: {g[g != w][:4]} vs {w[g != w][:4]}"
    if not w.size:
        return None
    err = np.abs(g - w).max() / max(np.abs(w).max(), 1e-30)
    return None if err <= tol else f"rel err {err:.3e}"
