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

from .base import PitchBase, c_float, c_int

__all__ = ["PitchYIN"]


class PitchYIN(PitchBase):
    """Per frame of 2**radix2_exp samples: the cumulative mean normalised difference over the lags samplate/high_fre
    .. samplate/low_fre; the frequency of the first trough below the threshold, that trough's value and the row's
    minimum.  pitch_batch returns (fre, value1, value2), zero where a frame has no trough; the trough rows are not
    requested."""
    _prefix = "pitchYINObj"
    _planes, _zero, _unset = 3, True, (None, None, None)

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
        self._open(radix2_exp, c_int(samplate), c_float(low_fre), c_float(high_fre), c_int(radix2_exp),
                   c_int(slide_length), c_int(auto_length), c_int(self.is_continue))

    def set_thresh(self, thresh):
        if thresh <= 0.0 or thresh >= 1.0:
            raise ValueError('`thresh` must be between 0.0 and 1.0.')
        self._lib.pitchYINObj_setThresh(self._obj, float(thresh))
        self.thresh = thresh
