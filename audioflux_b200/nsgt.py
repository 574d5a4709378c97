"""Non-stationary Gabor transform object (reference binding: python/audioflux/nsgt.py:16-367; C: src/nsgt_algorithm.c).

Same constructor, argument checks, getters, ``set_min_length``, ``nsgt`` and plot coordinates as the reference class.
``nsgt`` sends all channels to the GPU in one ``nsgtObj_nsgtBatch`` call; ``nsgt_batch`` takes numpy arrays or CUDA
tensors and returns the (re, im) planes."""
from __future__ import annotations

import ctypes as C
import warnings

import numpy as np

from .base import Base, as_f32, split_batch
from .capi import opt_int, opt_float
from .lib import check
from .types import (NSGTFilterBankType, SpectralFilterBankScaleType, SpectralFilterBankStyleType,
                    SpectralFilterBankNormalType, enum_value)

_C1 = 32.703195662574764        # note_to_hz('C1')


class NSGT(Base):
    def __init__(self, num=84, radix2_exp=12, samplate=32000, low_fre=None, high_fre=None, bin_per_octave=12,
                 min_len=3, nsgt_filter_bank_type=NSGTFilterBankType.EFFICIENT,
                 scale_type=SpectralFilterBankScaleType.OCTAVE, style_type=SpectralFilterBankStyleType.SLANEY,
                 normal_type=SpectralFilterBankNormalType.BAND_WIDTH, _lib=None):
        super().__init__(_lib)
        self.fft_length = fft_length = 1 << radix2_exp
        scale = enum_value(scale_type)
        log_like = scale in (SpectralFilterBankScaleType.OCTAVE.value, SpectralFilterBankScaleType.LOG.value)
        if num > fft_length // 2 + 1:
            raise ValueError(f'num={num} is too large')
        if scale == SpectralFilterBankScaleType.OCTAVE.value and bin_per_octave < 1:
            raise ValueError(f'bin_per_octave={bin_per_octave} must be a positive integer')
        if enum_value(style_type) == SpectralFilterBankStyleType.GAMMATONE.value:
            raise ValueError(f'style_type={SpectralFilterBankStyleType(enum_value(style_type)).name} is unsupported')
        if enum_value(normal_type) not in (SpectralFilterBankNormalType.NONE.value,
                                           SpectralFilterBankNormalType.BAND_WIDTH.value):
            raise ValueError(f'normal_type={SpectralFilterBankNormalType(enum_value(normal_type)).name} is unsupported')
        if low_fre is None:
            low_fre = _C1 if log_like else 0
        if high_fre is None:
            high_fre = samplate / 2
        if log_like and low_fre < round(_C1, 3):
            raise ValueError(f'{SpectralFilterBankScaleType(scale).name} low_fre={low_fre} must be greater than or '
                             f'equal to 32.703')
        if low_fre < 0:
            raise ValueError(f'{SpectralFilterBankScaleType(scale).name} low_fre={low_fre} must be a non-negative number')
        self.num, self.radix2_exp, self.samplate = num, radix2_exp, samplate
        self.low_fre, self.high_fre, self.bin_per_octave, self.min_len = low_fre, high_fre, bin_per_octave, min_len
        self.nsgt_filter_bank_type, self.scale_type = nsgt_filter_bank_type, scale_type
        self.style_type, self.normal_type = style_type, normal_type
        status = self._lib.nsgtObj_new(
            C.byref(self._obj), num, radix2_exp, opt_int(samplate), opt_float(low_fre), opt_float(high_fre),
            opt_int(bin_per_octave), opt_int(min_len), opt_int(enum_value(nsgt_filter_bank_type)), opt_int(scale),
            opt_int(enum_value(style_type)), opt_int(enum_value(normal_type)))
        if status != 0 or not self._obj:
            raise ValueError(f"nsgtObj_new failed with status {status}"
                             + (f": {self._lib.afb200_lastError().decode()}" if self._is_product and status == -2 else ""))
        self._is_created = True

    def get_max_time_length(self):
        return int(self._lib.nsgtObj_getMaxTimeLength(self._obj))

    def get_total_time_length(self):
        return int(self._lib.nsgtObj_getTotalTimeLength(self._obj))

    def _ints(self, p):
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_int)), shape=(self.num,)).copy()

    def get_time_length_arr(self):
        return self._ints(self._lib.nsgtObj_getTimeLengthArr(self._obj))

    def get_fre_band_arr(self):
        p = self._lib.nsgtObj_getFreBandArr(self._obj)
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_float)), shape=(self.num,)).copy()

    def get_bin_band_arr(self):
        return self._ints(self._lib.nsgtObj_getBinBandArr(self._obj))

    def set_min_length(self, min_length=3):
        if min_length < 1:
            raise ValueError(f'min_length={min_length} cannot be less than 1')
        self._lib.nsgtObj_setMinLength(self._obj, int(min_length))
        self.min_len = min_length

    def nsgt_batch(self, data, with_cells=False):
        """data [..., 2**radix2_exp] (numpy host | torch cuda) -> (re, im) each [..., num, max_time_length], plus the cells
        (cell_re, cell_im) each [..., total_time_length] when with_cells.  One nsgtObj_nsgtBatch call."""
        fn = self._require_ext("nsgtObj_nsgtBatch")
        x2, lead, kind, ptr, stream, alloc = split_batch(data)
        if x2.shape[-1] != self.fft_length:
            raise ValueError(f"data length must be 2**radix2_exp = {self.fft_length}")
        batch, T, tot = x2.shape[0], self.get_max_time_length(), self.get_total_time_length()
        re, im = alloc(batch, self.num, T), alloc(batch, self.num, T)
        cre = alloc(batch, tot) if with_cells else None
        cim = alloc(batch, tot) if with_cells else None
        check(fn(self._obj, ptr(x2), batch, ptr(re), ptr(im), None if cre is None else ptr(cre),
                 None if cim is None else ptr(cim), kind, stream), "nsgtObj_nsgtBatch")
        out = (re.reshape(*lead, self.num, T), im.reshape(*lead, self.num, T))
        if with_cells:
            out += (cre.reshape(*lead, tot), cim.reshape(*lead, tot))
        return out

    def nsgt(self, data_arr):
        """data_arr [..., 2**radix2_exp] (padded / truncated with a warning, as the reference) -> complex
        [..., num, max_time_length]"""
        data_arr = np.asarray(data_arr, dtype=np.float32, order='C')
        if data_arr.ndim == 0:
            raise ValueError('Audio data must have at least one dimension')
        n = data_arr.shape[-1]
        if n < self.fft_length:
            pad = self.fft_length - n
            warnings.warn(f'The audio length={n} is not enough for fft_length={self.fft_length}(2**radix2_exp), '
                          f'and {pad} zeros are automatically filled after the audio')
            data_arr = np.pad(data_arr, (*[(0, 0)] * (data_arr.ndim - 1), (0, pad)))
        elif n > self.fft_length:
            warnings.warn(f'fft_length={self.fft_length}(2**radix2_exp) is too small for data_arr length={n}, '
                          f'only the first fft_length={self.fft_length} data are valid')
            data_arr = data_arr[..., :self.fft_length].copy()
        re, im = self.nsgt_batch(as_f32(data_arr))
        return re + im * 1j

    def y_coords(self):
        return np.insert(self.get_fre_band_arr(), 0, self.low_fre)

    def x_coords(self, data_length):
        return np.linspace(0, data_length * 1. / self.samplate, self.get_max_time_length() + 1)

    def __del__(self):
        if getattr(self, "_is_created", False):
            self._lib.nsgtObj_free(self._obj)
            self._is_created = False
