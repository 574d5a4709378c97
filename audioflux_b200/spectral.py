"""Spectral descriptors of a spectrogram: flatness, flux, rolloff, centroid, ..., max / mean / var
(reference binding: python/audioflux/feature/spectral.py:15-2651; C: src/feature/spectral_algorithm.c, src/flux_spectral.c).

Every method computes from its own input: unlike the reference, nothing is cached in the object between calls, so
repeated calls and multi-channel input return each input's own values.  All channels of a call go to the GPU in one
``spectralObj_spectralBatch`` call."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .base import Base, Batch, as_f32, np_ptr
from .types import SpectralNoveltyMethodType, SpectralNoveltyDataType, enum_value

# feature ids of include/afb200_ext.h (AFB200_SPECTRAL_*)
FEATURES = ("flatness", "flux", "rolloff", "centroid", "spread", "skewness", "kurtosis", "entropy", "crest", "slope",
            "decrease", "band_width", "rms", "energy", "hfc", "sd", "sf", "mkl", "pd", "wpd", "nwpd", "cd", "rcd",
            "broadband", "novelty", "eef", "eer", "max", "mean", "var")
FEATURE_ID = {n: i for i, n in enumerate(FEATURES)}
PHASE_FEATURES = ("pd", "wpd", "nwpd", "cd", "rcd")
TWO_PLANES = ("max", "mean", "var")
MAX_REQ = 64


def encode(name, kw=None):
    """(name, kwargs with the reference method's argument names) -> (feature id, [step, p, threshold, flags])."""
    kw = dict(kw or {})
    if name not in FEATURE_ID:
        raise ValueError(f"unknown spectral feature {name!r}; one of {', '.join(FEATURES)}")

    def take(key, default):
        return kw.pop(key, default)
    step, p, thr, flags = 0, 0.0, 0.0, 0
    if name == "flux":
        step, p = take("step", 1), take("p", 2)
        flags = (1 if take("is_positive", False) else 0) | (2 if take("is_exp", False) else 0) | (4 if take("tp", 0) else 0)
    elif name == "rolloff":
        thr = take("threshold", 0.95)
    elif name in ("entropy", "eef"):
        flags = 1 if take("is_norm", False) else 0
    elif name == "band_width":
        p = take("p", 2)
    elif name == "energy":
        flags, p = (1 if take("is_log", False) else 0), take("gamma", 10.)
    elif name in ("sd", "sf"):
        step, flags = take("step", 1), (1 if take("is_positive", False) else 0)
    elif name == "mkl":
        flags = 4 if take("tp", 0) else 0
    elif name == "broadband":
        thr = take("threshold", 0)
    elif name == "novelty":
        step, thr = take("step", 1), take("threshold", 0.)
        mt = enum_value(take("method_type", SpectralNoveltyMethodType.SUB))
        dt = enum_value(take("data_type", SpectralNoveltyDataType.VALUE))
        flags = (mt & 3) | (4 if dt else 0)
    elif name == "eer":
        flags, p = (1 if take("is_norm", False) else 0), take("gamma", 1.)
    if kw:
        raise TypeError(f"{name}: unexpected arguments {sorted(kw)}")
    return FEATURE_ID[name], [float(step), float(p), float(thr), float(flags)]


class Spectral(Base):
    """Spectral features of a [..., fre, time] spectrogram of `num` bins whose centre frequencies are `fre_band_arr`
    (copied at construction)."""

    def __init__(self, num, fre_band_arr, _lib=None):
        super().__init__(_lib)
        if num < 2:
            raise ValueError("num must be >= 2")
        self.num = num
        self.fre_band_arr = None if fre_band_arr is None else as_f32(fre_band_arr).reshape(-1)
        if self.fre_band_arr is not None and self.fre_band_arr.shape[0] < num:
            raise ValueError(f"fre_band_arr holds {self.fre_band_arr.shape[0]} values, num={num}")
        self.time_length = 0
        fre = None if self.fre_band_arr is None else np_ptr(self.fre_band_arr)
        self._new("spectralObj_new", "spectralObj_free", num, fre)

    def set_time_length(self, time_length):
        self._lib.spectralObj_setTimeLength(self._obj, int(time_length))
        self.time_length = int(time_length)

    def set_edge(self, start, end):
        if not 0 <= start < end:
            raise ValueError(f'start={start} must be in range [0, {end})')
        if not start < end <= self.num - 1:
            raise ValueError(f'end={end} must be in range ({start}, {self.num - 1}]')
        self._lib.spectralObj_setEdge(self._obj, int(start), int(end))

    def set_edge_arr(self, index_arr):
        """Any order, repeats allowed; the C object takes ownership of a calloc'd copy (as the reference's binding)."""
        index_arr = np.asarray(index_arr, dtype=np.int32).reshape(-1)
        n = len(index_arr)
        if n < 1:
            raise ValueError("index_arr must not be empty")
        calloc = self._lib["calloc"]
        calloc.argtypes, calloc.restype = [C.c_size_t, C.c_size_t], C.c_void_p
        addr = calloc(n, C.sizeof(C.c_int))
        if not addr:
            raise MemoryError("calloc failed")
        C.memmove(addr, np.ascontiguousarray(index_arr).ctypes.data, n * C.sizeof(C.c_int))
        self._lib.spectralObj_setEdgeArr(self._obj, C.c_void_p(addr), n)

    # ---- additive batched entry point
    def spectral_batch(self, m_tn, features, phase=None):
        """m_tn [..., T, num] time-major (numpy host | torch cuda), features [(name, kwargs), ...] ->
        {name: [..., T]} ((value, fre) for max / mean / var) from one spectralObj_spectralBatch call.
        `phase` (same shape and kind as m_tn) is needed by pd / wpd / nwpd / cd / rcd."""
        feats = [(f, {}) if isinstance(f, str) else (f[0], dict(f[1] or {})) for f in features]
        names = [f[0] for f in feats]
        if not feats or len(feats) > MAX_REQ:
            raise ValueError(f"between 1 and {MAX_REQ} features per call")
        if len(set(names)) != len(names):
            raise ValueError("each feature may appear once per call")
        enc = [encode(n, kw) for n, kw in feats]
        req = np.array([e[0] for e in enc], np.int32)
        par = np.array([e[1] for e in enc], np.float32).reshape(-1)
        planes = sum(2 if n in TWO_PLANES else 1 for n in names)
        if m_tn.shape[-1] != self.num:
            raise ValueError(f"last axis holds {m_tn.shape[-1]} bins, the object has num={self.num}")
        if any(n in PHASE_FEATURES for n in names) and phase is None:
            raise ValueError("pd / wpd / nwpd / cd / rcd need the phase planes")
        b = Batch(m_tn)
        lead, T = b.lead[:-1], b.lead[-1]
        batch = int(np.prod(lead))
        ph = None if phase is None else b.second(phase, "phase")
        out = b.alloc(planes, batch, T, zero=True)
        self._call("spectralObj_spectralBatch", b, b.x, ph, T, batch, len(enc), req, par, out)
        res, k = {}, 0
        for n in names:
            if n in TWO_PLANES:
                res[n] = (out[k].reshape(*lead, T), out[k + 1].reshape(*lead, T))
                k += 2
            else:
                res[n] = out[k].reshape(*lead, T)
                k += 1
        return res

    # ---- the reference's methods: [..., fre, time] -> [..., time]
    def _run(self, name, m_data_arr, m_phase_arr=None, **kw):
        m = np.asarray(m_data_arr)
        if m.ndim < 2:
            raise ValueError("m_data_arr must be [..., fre, time]")
        self.set_time_length(m.shape[-1])
        tn = np.ascontiguousarray(np.swapaxes(as_f32(m), -1, -2))
        ph = None if m_phase_arr is None else np.ascontiguousarray(np.swapaxes(as_f32(m_phase_arr), -1, -2))
        return self.spectral_batch(tn, [(name, kw)], phase=ph)[name]

    def flatness(self, m_data_arr):
        return self._run("flatness", m_data_arr)

    def flux(self, m_data_arr, step=1, p=2, is_positive=False, is_exp=False, tp=0):
        return self._run("flux", m_data_arr, step=step, p=p, is_positive=is_positive, is_exp=is_exp, tp=tp)

    def rolloff(self, m_data_arr, threshold=0.95):
        return self._run("rolloff", m_data_arr, threshold=threshold)

    def centroid(self, m_data_arr):
        return self._run("centroid", m_data_arr)

    def spread(self, m_data_arr):
        return self._run("spread", m_data_arr)

    def skewness(self, m_data_arr):
        return self._run("skewness", m_data_arr)

    def kurtosis(self, m_data_arr):
        return self._run("kurtosis", m_data_arr)

    def entropy(self, m_data_arr, is_norm=False):
        return self._run("entropy", m_data_arr, is_norm=is_norm)

    def crest(self, m_data_arr):
        return self._run("crest", m_data_arr)

    def slope(self, m_data_arr):
        return self._run("slope", m_data_arr)

    def decrease(self, m_data_arr):
        return self._run("decrease", m_data_arr)

    def band_width(self, m_data_arr, p=2):
        return self._run("band_width", m_data_arr, p=p)

    def rms(self, m_data_arr):
        return self._run("rms", m_data_arr)

    def energy(self, m_data_arr, is_log=False, gamma=10.):
        return self._run("energy", m_data_arr, is_log=is_log, gamma=gamma)

    def hfc(self, m_data_arr):
        return self._run("hfc", m_data_arr)

    def sd(self, m_data_arr, step=1, is_positive=False):
        return self._run("sd", m_data_arr, step=step, is_positive=is_positive)

    def sf(self, m_data_arr, step=1, is_positive=False):
        return self._run("sf", m_data_arr, step=step, is_positive=is_positive)

    def mkl(self, m_data_arr, tp=0):
        return self._run("mkl", m_data_arr, tp=tp)

    def pd(self, m_data_arr, m_phase_arr):
        return self._run("pd", m_data_arr, m_phase_arr)

    def wpd(self, m_data_arr, m_phase_arr):
        return self._run("wpd", m_data_arr, m_phase_arr)

    def nwpd(self, m_data_arr, m_phase_arr):
        return self._run("nwpd", m_data_arr, m_phase_arr)

    def cd(self, m_data_arr, m_phase_arr):
        return self._run("cd", m_data_arr, m_phase_arr)

    def rcd(self, m_data_arr, m_phase_arr):
        return self._run("rcd", m_data_arr, m_phase_arr)

    def broadband(self, m_data_arr, threshold=0):
        return self._run("broadband", m_data_arr, threshold=threshold)

    def novelty(self, m_data_arr, step=1, threshold=0., method_type=SpectralNoveltyMethodType.SUB,
                data_type=SpectralNoveltyDataType.VALUE):
        return self._run("novelty", m_data_arr, step=step, threshold=threshold, method_type=method_type,
                         data_type=data_type)

    def eef(self, m_data_arr, is_norm=False):
        return self._run("eef", m_data_arr, is_norm=is_norm)

    def eer(self, m_data_arr, is_norm=False, gamma=1.):
        return self._run("eer", m_data_arr, is_norm=is_norm, gamma=gamma)

    def max(self, m_data_arr):
        return self._run("max", m_data_arr)

    def mean(self, m_data_arr):
        return self._run("mean", m_data_arr)

    def var(self, m_data_arr):
        return self._run("var", m_data_arr)
