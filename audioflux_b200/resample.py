"""Resampler (reference binding: python/audioflux/dsp/resample.py; C: src/dsp/resample_algorithm.c).

Same constructors, argument names, defaults and quality aliases as the reference's ``Resample`` and ``WindowResample``,
and the same ``set_samplate`` / ``cal_data_length`` / ``resample``.  ``resample`` sends all channels to the GPU in one
batched call; ``resample_batch`` takes numpy arrays or CUDA tensors and returns the same kind.

Differences from the reference, on purpose: ``cal_data_length`` returns the length (the reference's returns None), and
outputs are sized by it rather than cut from a ``5 * n`` buffer, so upsampling by more than 5 works."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .base import Base, Batch
from .types import ResampleQualityType, WindowType, enum_value

__all__ = ["Resample", "WindowResample"]


def _get_quality_type(tp):
    if isinstance(tp, ResampleQualityType):
        return tp
    if not isinstance(tp, str):
        raise ValueError(f'ResampleQualityType[{tp}] not supported')
    if tp in ('af_best', 'audio_best', 'best'):
        return ResampleQualityType.BEST
    if tp in ('af_mid', 'audio_mid', 'mid'):
        return ResampleQualityType.MID
    if tp in ('af_fast', 'audio_fast', 'fast'):
        return ResampleQualityType.FAST
    raise ValueError(f'ResampleQualityType[{tp}] not supported')


class ResampleBase(Base):
    def __init__(self, _lib=None):
        super().__init__(_lib)
        self.source_rate = None
        self.target_rate = None

    def set_samplate(self, source_rate, target_rate):
        self._lib.resampleObj_setSamplate(self._obj, int(source_rate), int(target_rate))
        self.source_rate = source_rate
        self.target_rate = target_rate

    def cal_data_length(self, data_length):
        """samples resample() returns for data_length input samples"""
        return self._lib.resampleObj_calDataLength(self._obj, int(data_length))

    def resample_batch(self, data):
        """data [..., n] (numpy host | torch cuda) -> [..., cal_data_length(n)] of the same kind.  One
        resampleObj_resampleBatch call for all channels; each is bit-identical to a legacy call into a zeroed buffer."""
        b = Batch(data)
        m = self.cal_data_length(b.n)
        out = b.alloc(b.rows, m)
        if b.rows and m > 0:
            self._call("resampleObj_resampleBatch", b, b.x, b.n, b.rows, out)
        return b.shaped(out)

    def resample(self, data_arr):
        """data_arr [..., n] -> float32 [..., cal_data_length(n)]"""
        data_arr = np.asarray(data_arr, dtype=np.float32, order='C')
        if data_arr.ndim == 0:
            raise ValueError('Audio data must have at least one dimension')
        if data_arr.shape[-1] == 0:
            raise ValueError('Audio data must not be empty')
        return self.resample_batch(data_arr)


class Resample(ResampleBase):
    """Resampling with one of the three Kaiser-windowed presets (ResampleQualityType or 'best' / 'mid' / 'fast')."""

    def __init__(self, qual_type=ResampleQualityType.BEST, is_scale=False, _lib=None):
        super().__init__(_lib)
        self.qual_type = _get_quality_type(qual_type)
        self.is_scale = is_scale
        self.is_continue = False
        self._new("resampleObj_new", "resampleObj_free", C.byref(C.c_int(self.qual_type.value)),
                  C.byref(C.c_int(int(is_scale))), C.byref(C.c_int(0)))


class WindowResample(ResampleBase):
    """Resampling with a windowed-sinc table of zero_num zero crossings, 2**nbit entries per crossing."""

    def __init__(self, zero_num=64, nbit=9, win_type=WindowType.HANN, value=None, roll_off=0.945, is_scale=False,
                 _lib=None):
        super().__init__(_lib)
        self.zero_num, self.nbit, self.win_type = zero_num, nbit, win_type
        self.value, self.roll_off, self.is_scale = value, roll_off, is_scale
        self.is_continue = False
        self._new("resampleObj_newWithWindow", "resampleObj_free", C.byref(C.c_int(int(zero_num))),
                  C.byref(C.c_int(int(nbit))), C.byref(C.c_int(enum_value(win_type))),
                  None if value is None else C.byref(C.c_float(value)), C.byref(C.c_float(roll_off)),
                  C.byref(C.c_int(int(is_scale))), C.byref(C.c_int(0)))
