"""Pitch by YIN (reference binding: python/audioflux/mir/pitch_yin.py; C: src/mir/_pitch_yin.c).

Same constructor, argument names and defaults as the reference's ``PitchYIN``, and the same ``set_thresh`` (with its
``ValueError`` outside (0, 1)), ``cal_time_length`` and ``pitch``.  ``pitch`` returns zero-filled ``(fre, value1,
value2)`` arrays as the reference does: frames without a trough below the threshold keep 0 in ``fre`` and ``value1``.
It sends all channels to the GPU in one batched call; ``pitch_batch`` takes numpy arrays or CUDA tensors and returns the
same kind.

Differences from the reference, on purpose (``ValueError`` from the constructor): ``radix2_exp`` above 14; a
``samplate / high_fre`` below 1 (minIndex 0, where the reference reads before its buffer); and an empty lag range
(``samplate / low_fre`` clamped by ``2**radix2_exp - auto_length - 1`` below ``samplate / high_fre``)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .base import Base, Batch, FrameAxis

__all__ = ["PitchYIN"]


class PitchYIN(FrameAxis, Base):
    """Per frame of 2**radix2_exp samples: the cumulative mean normalised difference over the lags samplate/high_fre
    .. samplate/low_fre; the frequency of the first trough below the threshold, that trough's value and the row's
    minimum."""

    def __init__(self, samplate=32000, low_fre=27.0, high_fre=2000.0, radix2_exp=12, slide_length=1024,
                 auto_length=2048, _lib=None):
        super().__init__(_lib)
        self.samplate = samplate
        self.low_fre = low_fre
        self.high_fre = high_fre
        self.radix2_exp = radix2_exp
        self.slide_length = slide_length
        self.auto_length = auto_length
        self.thresh = 0.1
        self.is_continue = False
        f = lambda v: C.byref(C.c_float(float(v)))  # noqa: E731
        i = lambda v: C.byref(C.c_int(int(v)))      # noqa: E731
        self._new("pitchYINObj_new", "pitchYINObj_free", i(samplate), f(low_fre), f(high_fre), i(radix2_exp),
                  i(slide_length), i(auto_length), i(self.is_continue))
        # the frame: 2**radix2_exp, or the reference's fallback 2**12 outside 1 .. 30
        self.fft_length = 1 << (int(radix2_exp) if 1 <= radix2_exp <= 30 else 12)

    def set_thresh(self, thresh):
        if thresh <= 0.0 or thresh >= 1.0:
            raise ValueError('`thresh` must be between 0.0 and 1.0.')
        self._lib.pitchYINObj_setThresh(self._obj, float(thresh))
        self.thresh = thresh

    def cal_time_length(self, data_length):
        return self._lib.pitchYINObj_calTimeLength(self._obj, int(data_length))

    def pitch_batch(self, data):
        """data [..., n] (numpy host | torch cuda) -> (fre, value1, value2), each [..., cal_time_length(n)] float32 of
        the same kind, zero where a frame has no trough.  One pitchYINObj_pitchBatch call for all channels; each row is
        bit-identical to a legacy call."""
        b = Batch(data)
        t = self.cal_time_length(b.n)
        out = [b.alloc(b.rows, t, zero=True) for _ in range(3)]
        if b.rows and t:
            self._call("pitchYINObj_pitchBatch", b, b.x, b.n, b.rows, *out, None, None, None)
        return tuple(b.shaped(o) for o in out)

    def pitch(self, data_arr):
        """data_arr [..., n] -> (fre_arr, value1_arr, value2_arr), each [..., time] float32"""
        data_arr = np.asarray(data_arr, dtype=np.float32, order='C')
        if data_arr.ndim == 0:
            raise ValueError('Audio data must have at least one dimension')
        if data_arr.shape[-1] == 0:
            raise ValueError('Audio data must not be empty')
        return self.pitch_batch(data_arr)
