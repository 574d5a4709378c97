"""Pitch by the normalised correlation function (reference binding: python/audioflux/mir/pitch_ncf.py; C:
src/mir/_pitch_ncf.c).

Same constructor, argument names and defaults as the reference's ``PitchNCF`` (window RECT), and the same
``cal_time_length`` and ``pitch``.  ``pitch`` sends all channels to the GPU in one batched call; ``pitch_batch`` takes
numpy arrays or CUDA tensors and returns the same kind.

Differences from the reference, on purpose (``ValueError`` from the constructor): ``radix2_exp`` above 14; a
``samplate / low_fre`` (rounded) of ``2**radix2_exp`` or more, where the reference writes past its buffer; a
``samplate / high_fre`` (rounded) below 1, where it clears a negative count of floats; and an empty lag range
(``samplate / low_fre`` below ``samplate / high_fre``, rounded)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .base import Base, Batch, FrameAxis
from .types import WindowType, enum_value

__all__ = ["PitchNCF"]


class _PitchLag(FrameAxis, Base):
    """The body PitchNCF and PitchCEP share: the constructor, cal_time_length and the batched pitch call of the C
    object named by _prefix."""
    _prefix = ""

    def __init__(self, samplate, low_fre, high_fre, radix2_exp, slide_length, window_type, _lib):
        super().__init__(_lib)
        self.samplate = samplate
        self.low_fre = low_fre
        self.high_fre = high_fre
        self.radix2_exp = radix2_exp
        self.slide_length = slide_length
        self.window_type = window_type
        self.is_continue = False
        f = lambda v: C.byref(C.c_float(float(v)))  # noqa: E731
        i = lambda v: C.byref(C.c_int(int(v)))      # noqa: E731
        self._new(f"{self._prefix}_new", f"{self._prefix}_free", i(samplate), f(low_fre), f(high_fre), i(radix2_exp),
                  i(slide_length), i(enum_value(window_type)), i(self.is_continue))
        # the frame: 2**radix2_exp, or the reference's fallback 2**12 outside 1 .. 30
        self.fft_length = 1 << (int(radix2_exp) if 1 <= radix2_exp <= 30 else 12)

    def cal_time_length(self, data_length):
        return getattr(self._lib, f"{self._prefix}_calTimeLength")(self._obj, int(data_length))

    def pitch_batch(self, data):
        """data [..., n] (numpy host | torch cuda) -> [..., cal_time_length(n)] float32 of the same kind.  One
        batched call for all channels; each row is bit-identical to a legacy call."""
        b = Batch(data)
        t = self.cal_time_length(b.n)
        out = b.alloc(b.rows, t)
        if b.rows and t:
            self._call(f"{self._prefix}_pitchBatch", b, b.x, b.n, b.rows, out)
        return b.shaped(out)

    def pitch(self, data_arr):
        """data_arr [..., n] -> fre_arr [..., time] float32"""
        data_arr = np.asarray(data_arr, dtype=np.float32, order='C')
        if data_arr.ndim == 0:
            raise ValueError('Audio data must have at least one dimension')
        if data_arr.shape[-1] == 0:
            raise ValueError('Audio data must not be empty')
        return self.pitch_batch(data_arr)


class PitchNCF(_PitchLag):
    """Per frame of 2**radix2_exp samples: the autocorrelation normalised by the frame's energy; the frequency of its
    largest value over the lags samplate/high_fre .. samplate/low_fre."""
    _prefix = "pitchNCFObj"

    def __init__(self, samplate=32000, low_fre=32.0, high_fre=2000.0, radix2_exp=12, slide_length=1024,
                 window_type=WindowType.RECT, _lib=None):
        super().__init__(samplate, low_fre, high_fre, radix2_exp, slide_length, window_type, _lib)
