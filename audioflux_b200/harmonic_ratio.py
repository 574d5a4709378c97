"""Harmonic ratio (reference binding: python/audioflux/mir/harmonic_ratio.py; C: src/mir/harmonicRatio_algorithm.c).

Same constructor, argument names and defaults as the reference's ``HarmonicRatio``, and the same ``cal_time_length`` /
``harmonic_ratio``.  ``harmonic_ratio`` sends all channels to the GPU in one batched call; ``harmonic_ratio_batch`` takes
numpy arrays or CUDA tensors and returns the same kind.  As in the reference, ``window_type`` is kept but not used: the
window is always Hamming.

Differences from the reference, on purpose: ``radix2_exp`` above 13, or a configuration whose lag range is empty
(``radix2_exp=0``, or a samplate below 25 with the default low frequency), raises ``ValueError``."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .base import C1_HZ, Base, Batch, FrameAxis
from .types import WindowType, enum_value

__all__ = ["HarmonicRatio"]


class HarmonicRatio(FrameAxis, Base):
    """Per frame of 2**radix2_exp samples: the maximum of the normalised autocorrelation beyond its first zero
    crossing, over lags up to samplate / low_fre."""

    def __init__(self, samplate=32000, low_fre=C1_HZ, radix2_exp=12, window_type=WindowType.HAMM, slide_length=1024,
                 _lib=None):
        super().__init__(_lib)
        self.samplate = samplate
        self.low_fre = low_fre
        self.radix2_exp = radix2_exp
        self.window_type = window_type
        self.slide_length = slide_length
        self._new("harmonicRatioObj_new", "harmonicRatioObj_free", C.byref(C.c_int(int(samplate))),
                  C.byref(C.c_float(float(low_fre))), C.byref(C.c_int(int(radix2_exp))),
                  C.byref(C.c_int(enum_value(window_type))), C.byref(C.c_int(int(slide_length))))
        # the window: 2**radix2_exp, or the reference's fallback 2**11 outside 0 .. 29
        self.fft_length = 1 << (int(radix2_exp) if 0 <= radix2_exp <= 29 else 11)

    def cal_time_length(self, data_length):
        return self._lib.harmonicRatioObj_calTimeLength(self._obj, int(data_length))

    def harmonic_ratio_batch(self, data):
        """data [..., n] (numpy host | torch cuda) -> [..., cal_time_length(n)] float32 of the same kind.  One
        harmonicRatioObj_harmonicRatioBatch call for all channels; each row is bit-identical to a legacy call."""
        b = Batch(data)
        t = self.cal_time_length(b.n)
        out = b.alloc(b.rows, t)
        if b.rows and t:
            self._call("harmonicRatioObj_harmonicRatioBatch", b, b.x, b.n, b.rows, out)
        return b.shaped(out)

    def harmonic_ratio(self, data_arr):
        """data_arr [..., n] -> [..., time] float32"""
        data_arr = np.asarray(data_arr, dtype=np.float32, order='C')
        if data_arr.ndim == 0:
            raise ValueError('Audio data must have at least one dimension')
        if data_arr.shape[-1] == 0:
            raise ValueError('Audio data must not be empty')
        return self.harmonic_ratio_batch(data_arr)
