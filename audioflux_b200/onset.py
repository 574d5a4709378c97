"""Onset detection (reference binding: python/audioflux/mir/onset.py; C: src/mir/onset_algorithm.c).

Same constructor, argument names and defaults as the reference's ``Onset``, and the same ``onset`` with its
``[..., fre, time]`` layout and results.  ``onset`` sends all channels to the GPU in one batched call; ``onset_batch``
takes time-major spectrograms as numpy arrays or CUDA tensors and returns the same kind."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .base import MEM_HOST, Base, Batch, swap_last2
from .types import NoveltyType, enum_value

__all__ = ["Onset", "NoveltyParam"]

PHASE_TYPES = (NoveltyType.PD, NoveltyType.WPD, NoveltyType.NWPD, NoveltyType.CD, NoveltyType.RCD)


class NoveltyParam(C.Structure):
    """Parameters of the novelty function (include/mir/onset_algorithm.h:32-44).  Read: step, p, isPostive, isExp and
    type (FLUX / SD / SF / MKL) and threshold (BROADBAND); isNorm and gamma are unused, as in the reference."""
    _fields_ = [
        ("step", C.c_int),
        ("p", C.c_float),
        ("isPostive", C.c_int),
        ("isExp", C.c_int),
        ("type", C.c_int),
        ("threshold", C.c_float),
        ("isNorm", C.c_int),
        ("gamma", C.c_float),
    ]


def _default_param():
    """the reference Python's default (mir/onset.py:156-158)"""
    return NoveltyParam(1, 1, 1, 0, 1, 0, 1, 1)


class Onset(Base):
    """Onset detection on a spectrogram of time_length frames x fre_length bins: optional max filter over frequency
    (filter_order >= 2), a novelty function, normalisation to [0, 1] and peak picking with parameters derived from
    samplate / slide_length."""

    def __init__(self, time_length, fre_length, slide_length, samplate=32000, filter_order=1,
                 novelty_type=NoveltyType.FLUX, _lib=None):
        super().__init__(_lib)
        self.time_length = time_length
        self.fre_length = fre_length
        self.samplate = samplate
        self.slide_length = slide_length
        self.filter_order = filter_order
        self.novelty_type = novelty_type
        self._new("onsetObj_new", "onsetObj_free", int(time_length), int(fre_length), int(slide_length),
                  C.byref(C.c_int(int(samplate))), C.byref(C.c_int(int(filter_order))),
                  C.byref(C.c_int(enum_value(novelty_type))))

    def _needs_phase(self):
        return enum_value(self.novelty_type) in [t.value for t in PHASE_TYPES]

    def onset_batch(self, spec, phase=None, novelty_param=None, index_arr=None):
        """spec (and phase for PD / WPD / NWPD / CD / RCD) [..., time_length, fre_length], time-major (numpy host |
        torch cuda) -> (evn float32 [..., time_length], points int32 [..., time_length], counts int32 [...]) of the
        same kind: each clip's points first, 0 after them.  One onsetObj_onsetBatch call for all clips."""
        T, M = int(self.time_length), int(self.fre_length)
        if tuple(spec.shape[-2:]) != (T, M):
            raise ValueError(f"spec must end in (time_length, fre_length) = {(T, M)}, got {tuple(spec.shape)}")
        if novelty_param is None:
            novelty_param = _default_param()
        elif not isinstance(novelty_param, NoveltyParam):
            raise ValueError("novelty_param must be type of NoveltyParam")
        b = Batch(spec.reshape(*spec.shape[:-2], T * M))
        ph = None
        if self._needs_phase():
            if phase is None:
                raise ValueError(f"novelty type {NoveltyType(enum_value(self.novelty_type)).name} needs the phase")
            if tuple(phase.shape) != tuple(spec.shape):
                raise ValueError("spec and phase must be the same shape")
            ph = b.second(phase.reshape(*phase.shape[:-2], T * M), "phase")
        idx = None
        if index_arr is not None:
            idx = np.ascontiguousarray(np.asarray(index_arr).astype(np.int32).reshape(-1))
        evn = b.alloc(b.rows, T)
        points, counts = self._ints_out(b, b.rows, T), self._ints_out(b, b.rows)
        if b.rows:
            self._call("onsetObj_onsetBatch", b, b.x, ph, b.rows, C.addressof(novelty_param), idx,
                       0 if idx is None else len(idx), evn, points, counts)
        return b.shaped(evn), b.shaped(points), counts.reshape(b.lead)

    @staticmethod
    def _ints_out(b, *shape):
        if b.kind == MEM_HOST:
            return np.empty(shape, np.int32)
        import torch
        return torch.empty(shape, dtype=torch.int32, device=b.device)

    def onset(self, m_data_arr1, m_data_arr2=None, novelty_param=None, index_arr=None):
        """m_data_arr1 (and m_data_arr2, the phase) [..., fre, time] -> (point_arr, evn_arr, time_arr, value_arr) as
        the reference returns them: for one clip the points and their values; for several, [..., points] padded with
        0 to the largest count."""
        x = np.asarray(m_data_arr1, dtype=np.float32, order='C')
        if x.ndim < 2:
            raise ValueError("m_data_arr1 must have at least two dimensions (fre, time)")
        spec = swap_last2(x)
        phase = None
        if m_data_arr2 is not None:
            y = np.asarray(m_data_arr2, dtype=np.float32, order='C')
            if y.shape != x.shape:
                raise ValueError('m_data_arr1 and m_data_arr2 must be the same shape')
            phase = swap_last2(y)
        evn, points, counts = self.onset_batch(spec, phase, novelty_param, index_arr)
        if x.ndim == 2:
            point_arr = points[:int(counts)]
            value_arr = evn[point_arr]
        else:
            n = int(counts.max()) if counts.size else 0
            point_arr = points[..., :n]
            value_arr = np.take_along_axis(evn, point_arr, -1)
            value_arr[np.arange(n) >= counts[..., None]] = 0
        time_arr = 1.0 * point_arr * self.slide_length / self.samplate
        return point_arr, evn, time_arr, value_arr
