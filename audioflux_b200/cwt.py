"""Continuous wavelet transform object (reference binding: python/audioflux/cwt.py:17-278;
C: src/cwt_algorithm.c)."""
from __future__ import annotations

import numpy as np

from .base import Base, BandAxis, SampleAxis, as_f32, band_range, fit_length, np_ptr, per_clip
from .capi import opt_int, opt_float
from .lib import check
from .types import WaveletContinueType, SpectralFilterBankScaleType, enum_value

_DEFAULT_GAMMA_BETA = {0: (3, 20), 1: (6, 2), 2: (5, 0.6), 3: (4, 0), 4: (2, 2), 5: (0, 2),
                       6: (5, 2), 7: (4, 0)}


class CWT(BandAxis, SampleAxis, Base):
    def __init__(self, num=84, radix2_exp=12, samplate=32000, low_fre=None, high_fre=None,
                 bin_per_octave=12, wavelet_type=WaveletContinueType.MORSE,
                 scale_type=SpectralFilterBankScaleType.OCTAVE, gamma=None, beta=None,
                 is_padding=True, _lib=None):
        super().__init__(_lib)
        self.fft_length = 1 << radix2_exp
        if num > self.fft_length // 2 + 1:
            raise ValueError(f"num={num} is too large")
        low_fre, high_fre = band_range(low_fre, high_fre, scale_type, samplate)
        g0, b0 = _DEFAULT_GAMMA_BETA[enum_value(wavelet_type)]
        gamma = g0 if gamma is None else gamma
        beta = b0 if beta is None else beta
        self.num, self.radix2_exp, self.samplate = num, radix2_exp, samplate
        self.low_fre, self.high_fre, self.bin_per_octave = low_fre, high_fre, bin_per_octave
        self.wavelet_type, self.scale_type = wavelet_type, scale_type
        self.gamma, self.beta, self.is_padding = gamma, beta, is_padding
        self._new("cwtObj_new", "cwtObj_free", num, radix2_exp, opt_int(samplate), opt_float(low_fre),
                  opt_float(high_fre), opt_int(bin_per_octave), opt_int(enum_value(wavelet_type)),
                  opt_int(enum_value(scale_type)), opt_float(gamma), opt_float(beta), opt_int(int(is_padding)))

    def get_fre_band_arr(self):
        return self._floats("cwtObj_getFreBandArr", self.num)

    def get_bin_band_arr(self):
        return self._ints("cwtObj_getBinBandArr", self.num)

    def cwt_planes(self, data_arr):
        """Raw C layout: (re, im) each [num, N], row 0 = highest band."""
        x = as_f32(data_arr)
        if x.shape[-1] != self.fft_length:
            raise ValueError(f"data length must be 2**radix2_exp = {self.fft_length}")
        re = np.zeros((self.num, self.fft_length), np.float32)
        im = np.zeros((self.num, self.fft_length), np.float32)
        self._lib.cwtObj_cwt(self._obj, np_ptr(x), np_ptr(re), np_ptr(im))
        return re, im

    def cwt(self, data_arr):
        """-> complex [..., num, N] low->high frequency rows, as cwt.py:236-278."""
        re, im = per_clip(self.cwt_planes, fit_length(data_arr, self.fft_length, warn=False))
        return np.ascontiguousarray((re + 1j * im)[..., ::-1, :])

    def ccwt(self, data_arr):
        """Continuous CWT of long audio (reference: cwt.py:280-320): windows of 2**radix2_exp samples every half window, the
        middle half of each kept (the first / last window also keep their outer quarter) -> [..., num, time].  With the
        product library all windows go through ONE cwtObj_cwtBatch call (every (window, scale) item is one CTA-resident
        transform for the default radix2_exp); any other library takes the reference's per-window loop."""
        x = as_f32(data_arr)
        N = self.fft_length
        quarter, step = N // 4, N // 2
        count = x.shape[-1] // step - 1
        if count < 1:
            raise ValueError(f"data length {x.shape[-1]} is shorter than one window of {N} samples")
        lead = x.shape[:-1]
        x2 = x.reshape(-1, x.shape[-1])
        win = np.lib.stride_tricks.sliding_window_view(x2, N, axis=-1)[:, ::step][:, :count]      # [B, count, N]
        if self._is_product and hasattr(self._lib, "cwtObj_cwtBatch"):
            re, im = self.cwt_batch(np.ascontiguousarray(win).reshape(-1, N))
            spec = (re + 1j * im).reshape(x2.shape[0], count, self.num, N)[:, :, ::-1]
        else:
            spec = self.cwt(np.ascontiguousarray(win))
        parts = [spec[:, i, :, (0 if i == 0 else quarter):(N if i == count - 1 else 3 * quarter)] for i in range(count)]
        out = np.concatenate(parts, axis=-1)
        return np.ascontiguousarray(out.reshape(*lead, self.num, out.shape[-1]))

    def enable_det(self, flag=True):
        self._lib.cwtObj_enableDet(self._obj, int(flag))

    def cwt_det_planes(self, data_arr=None):
        """Raw C layout of the derivative transform (cwtObj_cwtDet): (re, im) each [num, N].  data_arr=None reuses the
        spectrum of the preceding cwt / cwt_det call on this object."""
        re = np.zeros((self.num, self.fft_length), np.float32)
        im = np.zeros((self.num, self.fft_length), np.float32)
        if data_arr is None:
            self._lib.cwtObj_cwtDet(self._obj, None, np_ptr(re), np_ptr(im))
        else:
            x = as_f32(data_arr)
            if x.shape[-1] != self.fft_length:
                raise ValueError(f"data length must be 2**radix2_exp = {self.fft_length}")
            self._lib.cwtObj_cwtDet(self._obj, np_ptr(x), np_ptr(re), np_ptr(im))
        return re, im

    def cwt_det_batch(self, data):
        """Additive: data [B, N] (numpy host | torch cuda) -> (re, im) each [B, num, N] of the derivative transform."""
        return self._window_batch("cwtObj_cwtDetBatch", data)

    def cwt_batch(self, data):
        """Additive: data [B, N] (numpy host | torch cuda) -> (re, im) each [B, num, N] (C row order)."""
        return self._window_batch("cwtObj_cwtBatch", data)

    def get_filter_bank_arr(self):
        fn = self._require_ext("cwtObj_getFilterBankArr")
        # rows of the TRANSFORM length: 2 * fft_length when the object pads (is_padding, data lengths up to 1e5)
        width = 2 * self.fft_length if self.is_padding else self.fft_length
        out = np.zeros((self.num, width), np.float32)
        check(fn(self._obj, np_ptr(out)), "cwtObj_getFilterBankArr")
        return out
