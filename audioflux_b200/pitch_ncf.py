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

from .base import PitchBase, c_float, c_int
from .types import WindowType, enum_value

__all__ = ["PitchNCF"]


class _PitchLag(PitchBase):
    """The constructor PitchNCF and PitchCEP share"""

    def __init__(self, samplate, low_fre, high_fre, radix2_exp, slide_length, window_type, _lib):
        super().__init__(_lib)
        self.samplate = samplate
        self.low_fre = low_fre
        self.high_fre = high_fre
        self.radix2_exp = radix2_exp
        self.slide_length = slide_length
        self.window_type = window_type
        self.is_continue = False
        self._open(radix2_exp, c_int(samplate), c_float(low_fre), c_float(high_fre), c_int(radix2_exp),
                   c_int(slide_length), c_int(enum_value(window_type)), c_int(self.is_continue))


class PitchNCF(_PitchLag):
    """Per frame of 2**radix2_exp samples: the autocorrelation normalised by the frame's energy; the frequency of its
    largest value over the lags samplate/high_fre .. samplate/low_fre."""
    _prefix = "pitchNCFObj"

    def __init__(self, samplate=32000, low_fre=32.0, high_fre=2000.0, radix2_exp=12, slide_length=1024,
                 window_type=WindowType.RECT, _lib=None):
        super().__init__(samplate, low_fre, high_fre, radix2_exp, slide_length, window_type, _lib)
