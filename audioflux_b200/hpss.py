"""Harmonic-percussive source separation (reference binding: python/audioflux/mir/hpss.py; C: src/mir/hpss_algorithm.c).

Same constructor, argument names and defaults as the reference's ``HPSS``, and the same ``cal_data_length`` /
``hpss``.  ``hpss`` sends all channels to the GPU in one batched call; ``hpss_batch`` takes numpy arrays or CUDA tensors
and returns the same kind.  As in the reference, ``slide_length`` is kept but not used: the hop is always
``2**radix2_exp // 4``."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .base import Base, Batch
from .types import WindowType, enum_value

__all__ = ["HPSS"]


class HPSS(Base):
    """Median-filtering HPSS: h_order frames for the harmonic part, p_order bins for the percussive part (odd orders;
    any other value takes the default)."""

    def __init__(self, radix2_exp=12, window_type=WindowType.HAMM, slide_length=1024, h_order=21, p_order=31, _lib=None):
        super().__init__(_lib)
        self.radix2_exp = radix2_exp
        self.window_type = window_type
        self.slide_length = slide_length
        self.h_order = h_order
        self.p_order = p_order
        self._new("hpssObj_new", "hpssObj_free", int(radix2_exp), C.byref(C.c_int(enum_value(window_type))),
                  C.byref(C.c_int(int(slide_length))), C.byref(C.c_int(int(h_order))), C.byref(C.c_int(int(p_order))))

    def cal_data_length(self, data_length):
        """samples of each output of hpss() for data_length input samples"""
        return self._lib.hpssObj_calDataLength(self._obj, int(data_length))

    def hpss_batch(self, data):
        """data [..., n] (numpy host | torch cuda) -> (h, p), each [..., cal_data_length(n)] of the same kind.  One
        hpssObj_hpssBatch call for all channels; each is bit-identical to a legacy call into zeroed buffers."""
        b = Batch(data)
        m = self.cal_data_length(b.n)
        h, p = b.alloc(b.rows, m), b.alloc(b.rows, m)
        if b.rows:
            self._call("hpssObj_hpssBatch", b, b.x, b.n, b.rows, h, p)
        return b.shaped(h), b.shaped(p)

    def hpss(self, data_arr):
        """data_arr [..., n] -> (h_arr, p_arr), float32 [..., cal_data_length(n)] each"""
        data_arr = np.asarray(data_arr, dtype=np.float32, order='C')
        if data_arr.ndim == 0:
            raise ValueError('Audio data must have at least one dimension')
        if data_arr.shape[-1] == 0:
            raise ValueError('Audio data must not be empty')
        return self.hpss_batch(data_arr)
