"""Pseudo wavelet transform: FFT -> auditory filter bank x spectrum -> IFFT per band
(reference binding: python/audioflux/pwt.py:20-257; C: src/pwt_algorithm.c)."""
from __future__ import annotations

import numpy as np

from .base import Base, BandAxis, SampleAxis, as_f32, band_range, fit_length, is_log_scale, np_ptr, per_clip
from .capi import opt_int, opt_float
from .lib import check
from .types import (SpectralFilterBankScaleType, SpectralFilterBankStyleType, SpectralFilterBankNormalType, enum_value)


class PWT(BandAxis, SampleAxis, Base):
    def __init__(self, num=84, radix2_exp=12, samplate=32000, low_fre=None, high_fre=None, bin_per_octave=12,
                 scale_type=SpectralFilterBankScaleType.OCTAVE, style_type=SpectralFilterBankStyleType.SLANEY,
                 normal_type=SpectralFilterBankNormalType.NONE, is_padding=True, _lib=None):
        super().__init__(_lib)
        self.fft_length = 1 << radix2_exp
        if num > self.fft_length // 2 + 1:
            raise ValueError(f"num={num} is too large")
        low_fre, high_fre = band_range(low_fre, high_fre, scale_type, samplate)
        if is_log_scale(scale_type) and low_fre < 32.703:
            raise ValueError(f"low_fre={low_fre} must be greater than or equal to 32.703")
        if low_fre < 0:
            raise ValueError(f"low_fre={low_fre} must be a non-negative number")
        self.num, self.radix2_exp, self.samplate = num, radix2_exp, samplate
        self.low_fre, self.high_fre, self.bin_per_octave = low_fre, high_fre, bin_per_octave
        self.scale_type, self.style_type, self.normal_type, self.is_padding = scale_type, style_type, normal_type, is_padding
        self._new("pwtObj_new", "pwtObj_free", num, radix2_exp, opt_int(samplate), opt_float(low_fre),
                  opt_float(high_fre), opt_int(bin_per_octave), opt_int(enum_value(scale_type)),
                  opt_int(enum_value(style_type)), opt_int(enum_value(normal_type)), opt_int(int(is_padding)))

    def get_fre_band_arr(self):
        return self._floats("pwtObj_getFreBandArr", self.num)

    def get_bin_band_arr(self):
        return self._ints("pwtObj_getBinBandArr", self.num)

    def enable_det(self, flag=True):
        self._lib.pwtObj_enableDet(self._obj, int(flag))

    def _planes(self, fn, data_arr):
        re = np.zeros((self.num, self.fft_length), np.float32)
        im = np.zeros((self.num, self.fft_length), np.float32)
        if data_arr is None:
            fn(self._obj, None, np_ptr(re), np_ptr(im))
        else:
            x = as_f32(data_arr)
            if x.shape[-1] != self.fft_length:
                raise ValueError(f"data length must be 2**radix2_exp = {self.fft_length}")
            fn(self._obj, np_ptr(x), np_ptr(re), np_ptr(im))
        return re, im

    def pwt_planes(self, data_arr):
        """Raw C layout: (re, im) each [num, N]."""
        return self._planes(self._lib.pwtObj_pwt, data_arr)

    def pwt_det_planes(self, data_arr=None):
        return self._planes(self._lib.pwtObj_pwtDet, data_arr)

    def pwt(self, data_arr):
        """-> complex [..., num, N] as pwt.py:190-257 (no row flip, unlike CWT)."""
        re, im = per_clip(self.pwt_planes, fit_length(data_arr, self.fft_length, warn=False))
        return re + 1j * im

    def pwt_batch(self, data):
        """Additive: data [B, N] (numpy host | torch cuda) -> (re, im) each [B, num, N]."""
        return self._window_batch("pwtObj_pwtBatch", data)

    def pwt_det_batch(self, data):
        return self._window_batch("pwtObj_pwtDetBatch", data)

    def get_filter_bank_arr(self):
        fn = self._require_ext("pwtObj_getFilterBankArr")
        # rows of the TRANSFORM length: 2 * fft_length when the object pads (is_padding, data lengths up to 1e5)
        width = 2 * self.fft_length if self.is_padding else self.fft_length
        out = np.zeros((self.num, width), np.float32)
        check(fn(self._obj, np_ptr(out)), "pwtObj_getFilterBankArr")
        return out
