"""Pitch by the pitch estimation filter (reference binding: python/audioflux/mir/pitch_pef.py; C: src/mir/_pitch_pef.c).

Same constructor, argument names, defaults and ``ValueError`` checks as the reference's ``PitchPEF``, and the same
``cal_time_length`` / ``set_filter_params`` / ``pitch``.  ``pitch`` sends all channels to the GPU in one batched call;
``pitch_batch`` takes numpy arrays or CUDA tensors and returns the same kind.  As in the reference, ``set_filter_params``
checks and stores its arguments but the filter stays the one built by the constructor.

Differences from the reference, on purpose (``ValueError`` from the constructor): ``radix2_exp`` above 13; a lag range
that is empty (``high_fre`` at or above the top of the log grid, or ``low_fre`` and ``high_fre`` between the same two
grid points); and ``beta`` = 1 with ``high_fre`` nearest the top grid point, where the reference's peak search reads past
its buffer."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .base import Base, Batch, FrameAxis
from .types import WindowType, enum_value

__all__ = ["PitchPEF"]


def _check_filter(alpha, beta, gamma):
    if alpha <= 0:
        raise ValueError('`alpha` must be greater than 0.')
    if beta < 0 or beta > 1:
        raise ValueError('`beta` must be between 0 and 1.')
    if gamma <= 1:
        raise ValueError('`gamma` must be greater than 1.')


class PitchPEF(FrameAxis, Base):
    """Per frame of 2**radix2_exp samples: the log-frequency power spectrum, cross-correlated with the pitch estimation
    filter; the frequency of the largest correlation between low_fre and high_fre."""

    def __init__(self, samplate=32000, low_fre=32.0, high_fre=2000.0, cut_fre=4000.0, radix2_exp=12, slide_length=1024,
                 window_type=WindowType.HAMM, alpha=10.0, beta=0.5, gamma=1.8, _lib=None):
        if low_fre >= high_fre:
            raise ValueError('`low_fre` must be smaller than `high_fre`')
        if high_fre >= cut_fre:
            raise ValueError('`high_fre` must be smaller than `cut_fre`')
        _check_filter(alpha, beta, gamma)
        super().__init__(_lib)
        self.samplate = samplate
        self.low_fre = low_fre
        self.high_fre = high_fre
        self.cut_fre = cut_fre
        self.radix2_exp = radix2_exp
        self.slide_length = slide_length
        self.window_type = window_type
        self.alpha = alpha
        self.beta = beta
        self.gamma = gamma
        self.is_continue = False
        f = lambda v: C.byref(C.c_float(float(v)))  # noqa: E731
        i = lambda v: C.byref(C.c_int(int(v)))      # noqa: E731
        self._new("pitchPEFObj_new", "pitchPEFObj_free", i(samplate), f(low_fre), f(high_fre), f(cut_fre),
                  i(radix2_exp), i(slide_length), i(enum_value(window_type)), f(alpha), f(beta), f(gamma),
                  i(self.is_continue))
        # the frame: 2**radix2_exp, or the reference's fallback 2**12 outside 1 .. 30
        self.fft_length = 1 << (int(radix2_exp) if 1 <= radix2_exp <= 30 else 12)

    def cal_time_length(self, data_length):
        return self._lib.pitchPEFObj_calTimeLength(self._obj, int(data_length))

    def set_filter_params(self, alpha, beta, gamma):
        _check_filter(alpha, beta, gamma)
        self._lib.pitchPEFObj_setFilterParams(self._obj, float(alpha), float(beta), float(gamma))
        self.alpha = alpha
        self.beta = beta
        self.gamma = gamma

    def pitch_batch(self, data):
        """data [..., n] (numpy host | torch cuda) -> [..., cal_time_length(n)] float32 of the same kind.  One
        pitchPEFObj_pitchBatch call for all channels; each row is bit-identical to a legacy call."""
        b = Batch(data)
        t = self.cal_time_length(b.n)
        out = b.alloc(b.rows, t)
        if b.rows and t:
            self._call("pitchPEFObj_pitchBatch", b, b.x, b.n, b.rows, out)
        return b.shaped(out)

    def pitch(self, data_arr):
        """data_arr [..., n] -> fre_arr [..., time] float32"""
        data_arr = np.asarray(data_arr, dtype=np.float32, order='C')
        if data_arr.ndim == 0:
            raise ValueError('Audio data must have at least one dimension')
        if data_arr.shape[-1] == 0:
            raise ValueError('Audio data must not be empty')
        return self.pitch_batch(data_arr)
