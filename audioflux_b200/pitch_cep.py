"""Pitch by the cepstrum (reference binding: python/audioflux/mir/pitch_cep.py; C: src/mir/_pitch_cep.c).

Same constructor, argument names, defaults (window HAMM) and ``ValueError`` as the reference's ``PitchCEP``, and the
same ``cal_time_length`` and ``pitch``.  ``pitch`` sends all channels to the GPU in one batched call; ``pitch_batch``
takes numpy arrays or CUDA tensors and returns the same kind.  As in the reference, a window after HAMM is replaced by
HAMM.

Differences from the reference, on purpose (``ValueError`` from the constructor): ``radix2_exp`` above 14; a
``samplate / low_fre`` (rounded) of ``2**(radix2_exp + 1)`` or more, where the reference's peak search reads past its
row; and an empty lag range (``samplate / low_fre`` below ``samplate / high_fre``, rounded, which the reference's
fallback for a rejected ``high_fre`` can produce)."""
from __future__ import annotations

from .pitch_ncf import _PitchLag
from .types import WindowType

__all__ = ["PitchCEP"]


class PitchCEP(_PitchLag):
    """Per frame of 2**radix2_exp samples: the real cepstrum (the inverse FFT of the log power spectrum); the frequency
    of its largest value over the quefrencies samplate/high_fre .. samplate/low_fre."""
    _prefix = "pitchCEPObj"

    def __init__(self, samplate=32000, low_fre=32.0, high_fre=2000.0, radix2_exp=12, slide_length=1024,
                 window_type=WindowType.HAMM, _lib=None):
        if low_fre >= high_fre:
            raise ValueError('`low_fre` must be smaller than `high_fre`')
        super().__init__(samplate, low_fre, high_fre, radix2_exp, slide_length, window_type, _lib)
