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
import warnings

import numpy as np

from .base import Base, SampleAxis, as_f32, split_batch
from .lib import check


def _range_checks(fft_length, min_index, max_index):
    if min_index < 1:
        raise ValueError(f'min_index={min_index} must be a positive integer.')
    if max_index >= (fft_length / 2):
        raise ValueError(f'max_index={max_index} must be less than or equal to fft_length/2={fft_length / 2}')
    if min_index >= max_index:
        raise ValueError(f'min_index={min_index} must be less than max_index={max_index}')


def _fit_length(data_arr, fft_length):
    """data [..., n] as float32, zero-padded or truncated to fft_length with the reference's warnings
    (python/audioflux/utils/util.py:98-110)"""
    data_arr = np.asarray(data_arr, dtype=np.float32, order='C')
    if data_arr.ndim == 0:
        raise ValueError('Audio data must have at least one dimension')
    n = data_arr.shape[-1]
    if n < fft_length:
        pad = fft_length - n
        warnings.warn(f'The audio length={n} is not enough for fft_length={fft_length}(2**radix2_exp), '
                      f'and {pad} zeros are automatically filled after the audio')
        data_arr = np.pad(data_arr, (*[(0, 0)] * (data_arr.ndim - 1), (0, pad)))
    elif n > fft_length:
        warnings.warn(f'fft_length={fft_length}(2**radix2_exp) is too small for data_arr length={n}, '
                      f'only the first fft_length={fft_length} data are valid')
        data_arr = data_arr[..., :fft_length].copy()
    return as_f32(data_arr)


class _Stockwell(Base, SampleAxis):
    def _new_failed(self, name, status):
        raise ValueError(f"{name} failed with status {status}"
                         + (f": {self._lib.afb200_lastError().decode()}" if self._is_product and status == -2 else ""))

    def y_coords(self):
        fre = self.get_fre_band_arr()
        return np.insert(fre, 0, fre[0])

    def _run(self, name, data, *args):
        fn = self._require_ext(name)
        x2, lead, kind, ptr, stream, alloc = split_batch(data)
        if x2.shape[-1] != self.fft_length:
            raise ValueError(f"data length must be 2**radix2_exp = {self.fft_length}")
        batch = x2.shape[0]
        re, im = alloc(batch, self.num, self.fft_length), alloc(batch, self.num, self.fft_length)
        check(fn(self._obj, ptr(x2), batch, *args, ptr(re), ptr(im), kind, stream), name)
        return re.reshape(*lead, self.num, self.fft_length), im.reshape(*lead, self.num, self.fft_length)


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
        status = self._lib.stObj_new(C.byref(self._obj), radix2_exp, min_index, max_index,
                                     C.byref(C.c_float(factor)), C.byref(C.c_float(norm)))
        if status != 0 or not self._obj:
            self._new_failed("stObj_new", status)
        self._is_created = True
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
        return self._run("stObj_stBatch", data)

    def st(self, data_arr):
        """data_arr [..., 2**radix2_exp] (padded / truncated with a warning, as the reference) -> complex
        [..., num, 2**radix2_exp]"""
        re, im = self.st_batch(_fit_length(data_arr, self.fft_length))
        return re + im * 1j

    def __del__(self):
        if getattr(self, "_is_created", False):
            self._lib.stObj_free(self._obj)
            self._is_created = False


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
        status = self._lib.fstObj_new(C.byref(self._obj), radix2_exp)
        if status != 0 or not self._obj:
            self._new_failed("fstObj_new", status)
        self._is_created = True

    def get_fre_band_arr(self):
        return np.arange(self.min_index, self.max_index + 1, dtype=np.float32) * self.samplate / self.fft_length

    def fst_batch(self, data):
        """data [..., 2**radix2_exp] (numpy host | torch cuda) -> (re, im) each [..., num, 2**radix2_exp], rows
        min_index .. max_index.  One fstObj_fstBatch call."""
        return self._run("fstObj_fstBatch", data, self.min_index, self.max_index)

    def fst(self, data_arr):
        """data_arr [..., 2**radix2_exp] (padded / truncated with a warning, as the reference) -> complex
        [..., num, 2**radix2_exp]"""
        re, im = self.fst_batch(_fit_length(data_arr, self.fft_length))
        return re + im * 1j

    def __del__(self):
        if getattr(self, "_is_created", False):
            self._lib.fstObj_free(self._obj)
            self._is_created = False
