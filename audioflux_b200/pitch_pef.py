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

from .base import PitchBase, c_float, c_int
from .types import WindowType, enum_value

__all__ = ["PitchPEF"]


def _check_filter(alpha, beta, gamma):
    if alpha <= 0:
        raise ValueError('`alpha` must be greater than 0.')
    if beta < 0 or beta > 1:
        raise ValueError('`beta` must be between 0 and 1.')
    if gamma <= 1:
        raise ValueError('`gamma` must be greater than 1.')


class PitchPEF(PitchBase):
    """Per frame of 2**radix2_exp samples: the log-frequency power spectrum, cross-correlated with the pitch estimation
    filter; the frequency of the largest correlation between low_fre and high_fre."""
    _prefix = "pitchPEFObj"

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
        self._open(radix2_exp, c_int(samplate), c_float(low_fre), c_float(high_fre), c_float(cut_fre),
                   c_int(radix2_exp), c_int(slide_length), c_int(enum_value(window_type)), c_float(alpha),
                   c_float(beta), c_float(gamma), c_int(self.is_continue))

    def set_filter_params(self, alpha, beta, gamma):
        _check_filter(alpha, beta, gamma)
        self._lib.pitchPEFObj_setFilterParams(self._obj, float(alpha), float(beta), float(gamma))
        self.alpha = alpha
        self.beta = beta
        self.gamma = gamma
