"""Non-stationary Gabor transform object (reference binding: python/audioflux/nsgt.py:16-367; C: src/nsgt_algorithm.c).

Same constructor, argument checks, getters, ``set_min_length``, ``nsgt`` and plot coordinates as the reference class.
``nsgt`` sends all channels to the GPU in one ``nsgtObj_nsgtBatch`` call; ``nsgt_batch`` takes numpy arrays or CUDA
tensors and returns the (re, im) planes."""
from __future__ import annotations

import numpy as np

from .base import C1_HZ, Base, Batch, band_range, fit_length, is_log_scale
from .capi import opt_int, opt_float
from .types import (NSGTFilterBankType, SpectralFilterBankScaleType, SpectralFilterBankStyleType,
                    SpectralFilterBankNormalType, enum_value)


class NSGT(Base):
    def __init__(self, num=84, radix2_exp=12, samplate=32000, low_fre=None, high_fre=None, bin_per_octave=12,
                 min_len=3, nsgt_filter_bank_type=NSGTFilterBankType.EFFICIENT,
                 scale_type=SpectralFilterBankScaleType.OCTAVE, style_type=SpectralFilterBankStyleType.SLANEY,
                 normal_type=SpectralFilterBankNormalType.BAND_WIDTH, _lib=None):
        super().__init__(_lib)
        self.fft_length = fft_length = 1 << radix2_exp
        scale = enum_value(scale_type)
        if num > fft_length // 2 + 1:
            raise ValueError(f'num={num} is too large')
        if scale == SpectralFilterBankScaleType.OCTAVE.value and bin_per_octave < 1:
            raise ValueError(f'bin_per_octave={bin_per_octave} must be a positive integer')
        if enum_value(style_type) == SpectralFilterBankStyleType.GAMMATONE.value:
            raise ValueError(f'style_type={SpectralFilterBankStyleType(enum_value(style_type)).name} is unsupported')
        if enum_value(normal_type) not in (SpectralFilterBankNormalType.NONE.value,
                                           SpectralFilterBankNormalType.BAND_WIDTH.value):
            raise ValueError(f'normal_type={SpectralFilterBankNormalType(enum_value(normal_type)).name} is unsupported')
        low_fre, high_fre = band_range(low_fre, high_fre, scale, samplate)
        if is_log_scale(scale) and low_fre < round(C1_HZ, 3):
            raise ValueError(f'{SpectralFilterBankScaleType(scale).name} low_fre={low_fre} must be greater than or '
                             f'equal to 32.703')
        if low_fre < 0:
            raise ValueError(f'{SpectralFilterBankScaleType(scale).name} low_fre={low_fre} must be a non-negative number')
        self.num, self.radix2_exp, self.samplate = num, radix2_exp, samplate
        self.low_fre, self.high_fre, self.bin_per_octave, self.min_len = low_fre, high_fre, bin_per_octave, min_len
        self.nsgt_filter_bank_type, self.scale_type = nsgt_filter_bank_type, scale_type
        self.style_type, self.normal_type = style_type, normal_type
        self._new("nsgtObj_new", "nsgtObj_free", num, radix2_exp, opt_int(samplate), opt_float(low_fre),
                  opt_float(high_fre), opt_int(bin_per_octave), opt_int(min_len),
                  opt_int(enum_value(nsgt_filter_bank_type)), opt_int(scale), opt_int(enum_value(style_type)),
                  opt_int(enum_value(normal_type)))

    def get_max_time_length(self):
        return int(self._lib.nsgtObj_getMaxTimeLength(self._obj))

    def get_total_time_length(self):
        return int(self._lib.nsgtObj_getTotalTimeLength(self._obj))

    def get_time_length_arr(self):
        return self._ints("nsgtObj_getTimeLengthArr", self.num)

    def get_fre_band_arr(self):
        return self._floats("nsgtObj_getFreBandArr", self.num)

    def get_bin_band_arr(self):
        return self._ints("nsgtObj_getBinBandArr", self.num)

    def set_min_length(self, min_length=3):
        if min_length < 1:
            raise ValueError(f'min_length={min_length} cannot be less than 1')
        self._lib.nsgtObj_setMinLength(self._obj, int(min_length))
        self.min_len = min_length

    def nsgt_batch(self, data, with_cells=False):
        """data [..., 2**radix2_exp] (numpy host | torch cuda) -> (re, im) each [..., num, max_time_length], plus the cells
        (cell_re, cell_im) each [..., total_time_length] when with_cells.  One nsgtObj_nsgtBatch call."""
        b = Batch(data)
        if b.n != self.fft_length:
            raise ValueError(f"data length must be 2**radix2_exp = {self.fft_length}")
        T, tot = self.get_max_time_length(), self.get_total_time_length()
        re, im = b.alloc(b.rows, self.num, T), b.alloc(b.rows, self.num, T)
        cre, cim = (b.alloc(b.rows, tot), b.alloc(b.rows, tot)) if with_cells else (None, None)
        self._call("nsgtObj_nsgtBatch", b, b.x, b.rows, re, im, cre, cim)
        out = (b.shaped(re), b.shaped(im))
        return out + (b.shaped(cre), b.shaped(cim)) if with_cells else out

    def nsgt(self, data_arr):
        """data_arr [..., 2**radix2_exp] (padded / truncated with a warning, as the reference) -> complex
        [..., num, max_time_length]"""
        re, im = self.nsgt_batch(fit_length(data_arr, self.fft_length, warn=True))
        return re + im * 1j

    def y_coords(self):
        return np.insert(self.get_fre_band_arr(), 0, self.low_fre)

    def x_coords(self, data_length):
        return np.linspace(0, data_length * 1. / self.samplate, self.get_max_time_length() + 1)
