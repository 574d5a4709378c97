"""Stockwell transforms (reference bindings: python/audioflux/st.py:15-241 and fst.py:15-195; C: src/st_algorithm.c,
src/fst_algorithm.c).

Same constructors, argument checks, ``st`` / ``fst``, ``set_value`` and plot coordinates as the reference classes.
``st`` / ``fst`` send all channels to the GPU in one batched call; ``st_batch`` / ``fst_batch`` take numpy arrays or
CUDA tensors and return the (re, im) planes.

Two differences from the reference's ``ST``, both on purpose:
  - ``use_bin_arr`` passes the list as int32, as the C function expects, and updates ``num`` to the new row count.  The
    reference passes a float32 array to the C ``int *`` parameter, so the C side reads float bit patterns: any non-zero
    bin becomes an integer far above N/2 and the whole list is rejected (a list of zeros is taken as zeros), and ``num``
    never changes.
  - ``get_fre_band_arr`` (and ``y_coords``) give the frequencies of the current bin list; they equal the reference's
    ``min_index .. max_index`` grid until ``use_bin_arr`` is called."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .base import Base, SampleAxis, fit_length


def _range_checks(fft_length, min_index, max_index):
    if min_index < 1:
        raise ValueError(f'min_index={min_index} must be a positive integer.')
    if max_index >= (fft_length / 2):
        raise ValueError(f'max_index={max_index} must be less than or equal to fft_length/2={fft_length / 2}')
    if min_index >= max_index:
        raise ValueError(f'min_index={min_index} must be less than max_index={max_index}')


class _Stockwell(Base, SampleAxis):
    def y_coords(self):
        fre = self.get_fre_band_arr()
        return np.insert(fre, 0, fre[0])


class ST(_Stockwell):
    def __init__(self, radix2_exp=12, min_index=1, max_index=None, samplate=32000, factor=1., norm=1., _lib=None):
        super().__init__(_lib)
        self.fft_length = fft_length = 1 << radix2_exp
        if max_index is None:
            max_index = fft_length // 2 - 1
        _range_checks(fft_length, min_index, max_index)
        self.radix2_exp, self.samplate = radix2_exp, samplate
        self.min_index, self.max_index = min_index, max_index
        self.factor, self.norm = factor, norm
        self._new("stObj_new", "stObj_free", radix2_exp, min_index, max_index, C.byref(C.c_float(factor)),
                  C.byref(C.c_float(norm)))
        self._bins = np.arange(min_index, max_index + 1, dtype=np.int32)
        self.num = len(self._bins)

    def use_bin_arr(self, bin_arr):
        """rows of the transform: any bins in [0, fft_length/2], in any order, repeats allowed.  A list with a bin outside
        that range is ignored as a whole (the object keeps its rows)."""
        bin_arr = np.ascontiguousarray(np.asarray(bin_arr), dtype=np.int32)
        if bin_arr.ndim != 1:
            raise ValueError('bin_arr is only defined for 1D arrays')
        self._lib.stObj_useBinArr(self._obj, bin_arr.ctypes.data_as(C.c_void_p), len(bin_arr))
        if ((bin_arr >= 0) & (bin_arr <= self.fft_length // 2)).all():
            self._bins = bin_arr.copy()
        self.num = len(self._bins)

    def set_value(self, factor, norm):
        self._lib.stObj_setValue(self._obj, C.c_float(factor), C.c_float(norm))
        self.factor, self.norm = factor, norm

    def get_fre_band_arr(self):
        return self._bins.astype(np.float32) * self.samplate / self.fft_length

    def st_batch(self, data):
        """data [..., 2**radix2_exp] (numpy host | torch cuda) -> (re, im) each [..., num, 2**radix2_exp].
        One stObj_stBatch call."""
        return self._window_batch("stObj_stBatch", data)

    def st(self, data_arr):
        """data_arr [..., 2**radix2_exp] (padded / truncated with a warning, as the reference) -> complex
        [..., num, 2**radix2_exp]"""
        re, im = self.st_batch(fit_length(data_arr, self.fft_length, warn=True))
        return re + im * 1j


class FST(_Stockwell):
    def __init__(self, radix2_exp=12, min_index=1, max_index=None, samplate=32000, _lib=None):
        super().__init__(_lib)
        self.fft_length = fft_length = 1 << radix2_exp
        if max_index is None:
            max_index = fft_length // 2 - 1
        _range_checks(fft_length, min_index, max_index)
        self.radix2_exp, self.samplate = radix2_exp, samplate
        self.min_index, self.max_index = min_index, max_index
        self.num = max_index - min_index + 1
        self._new("fstObj_new", "fstObj_free", radix2_exp)

    def get_fre_band_arr(self):
        return np.arange(self.min_index, self.max_index + 1, dtype=np.float32) * self.samplate / self.fft_length

    def fst_batch(self, data):
        """data [..., 2**radix2_exp] (numpy host | torch cuda) -> (re, im) each [..., num, 2**radix2_exp], rows
        min_index .. max_index.  One fstObj_fstBatch call."""
        return self._window_batch("fstObj_fstBatch", data, self.min_index, self.max_index)

    def fst(self, data_arr):
        """data_arr [..., 2**radix2_exp] (padded / truncated with a warning, as the reference) -> complex
        [..., num, 2**radix2_exp]"""
        re, im = self.fst_batch(fit_length(data_arr, self.fft_length, warn=True))
        return re + im * 1j
