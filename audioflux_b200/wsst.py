"""Synchrosqueezing objects (reference binding: python/audioflux/wsst.py:131-345, python/audioflux/synsq.py:60-200;
C: src/wsst_algorithm.c, src/synsq_algorithm.c)."""
from __future__ import annotations

import numpy as np

from .base import Base, BandAxis, SampleAxis, as_f32, band_range, fit_length, np_ptr, per_clip
from .capi import opt_int, opt_float
from .types import WaveletContinueType, SpectralFilterBankScaleType, enum_value
from .cwt import _DEFAULT_GAMMA_BETA


class WSST(BandAxis, SampleAxis, Base):
    def __init__(self, num=84, radix2_exp=12, samplate=32000, low_fre=None, high_fre=None, bin_per_octave=12,
                 wavelet_type=WaveletContinueType.MORLET, scale_type=SpectralFilterBankScaleType.OCTAVE,
                 gamma=None, beta=None, thresh=0.001, is_padding=True, _lib=None):
        super().__init__(_lib)
        low_fre, high_fre = band_range(low_fre, high_fre, scale_type, samplate)
        g0, b0 = _DEFAULT_GAMMA_BETA[enum_value(wavelet_type)]
        gamma = g0 if gamma is None else gamma
        beta = b0 if beta is None else beta
        self.num, self.radix2_exp, self.samplate, self.fft_length = num, radix2_exp, samplate, 1 << radix2_exp
        self.low_fre, self.high_fre, self.bin_per_octave = low_fre, high_fre, bin_per_octave
        self.wavelet_type, self.scale_type, self.gamma, self.beta = wavelet_type, scale_type, gamma, beta
        self.thresh, self.is_padding, self.order = thresh, is_padding, 1
        self._new("wsstObj_new", "wsstObj_free", num, radix2_exp, opt_int(samplate), opt_float(low_fre),
                  opt_float(high_fre), opt_int(bin_per_octave), opt_int(enum_value(wavelet_type)),
                  opt_int(enum_value(scale_type)), opt_float(gamma), opt_float(beta), opt_float(thresh),
                  opt_int(int(is_padding)))

    def get_fre_band_arr(self):
        return self._floats("wsstObj_getFreBandArr", self.num)

    def get_bin_band_arr(self):
        return self._ints("wsstObj_getBinBandArr", self.num)

    def set_order(self, order):
        self._lib.wsstObj_setOrder(self._obj, int(order))
        self.order = order

    def wsst_planes(self, data_arr):
        """Raw C layout: (re, im, cwt_re, cwt_im) each [num, N]."""
        x = as_f32(data_arr)
        if x.shape[-1] != self.fft_length:
            raise ValueError(f"data length must be 2**radix2_exp = {self.fft_length}")
        out = [np.zeros((self.num, self.fft_length), np.float32) for _ in range(4)]
        self._lib.wsstObj_wsst(self._obj, np_ptr(x), *[np_ptr(o) for o in out])
        return tuple(out)

    def wsst(self, data_arr):
        """-> (wsst, cwt) complex [..., num, N] as wsst.py:258-330."""
        re, im, cr, ci = per_clip(self.wsst_planes, fit_length(data_arr, self.fft_length, warn=False))
        return re + 1j * im, cr + 1j * ci


class Synsq(Base):
    def __init__(self, num, radix2_exp=12, samplate=32000, order=1, thresh=0.001, _lib=None):
        super().__init__(_lib)
        self.num, self.radix2_exp, self.samplate, self.order, self.thresh = num, radix2_exp, samplate, order, thresh
        self.fft_length = 1 << radix2_exp
        self._new("synsqObj_new", "synsqObj_free", num, radix2_exp, opt_int(samplate), opt_int(order), opt_float(thresh))

    def synsq_planes(self, fre_arr, scale_type, re, im):
        """Raw C layout: planes [num, N] -> squeezed (re, im) [num, N]."""
        re, im, fre = as_f32(re), as_f32(im), as_f32(fre_arr)
        o_re, o_im = np.zeros_like(re), np.zeros_like(im)
        self._lib.synsqObj_synsq(self._obj, np_ptr(fre), enum_value(scale_type), np_ptr(re), np_ptr(im), np_ptr(o_re), np_ptr(o_im))
        return o_re, o_im

    def synsq(self, m_data_arr, filter_bank_type, fre_arr):
        """complex [..., num, N] -> complex [..., num, N] as synsq.py:126-190."""
        z = np.asarray(m_data_arr)
        if not np.iscomplexobj(z):
            raise ValueError(f"m_data_arr with dtype={z.dtype} is not of complex type")
        if z.ndim < 2:
            raise ValueError(f"m_data_arr.ndim=[{z.ndim}] should be greater than 1")
        re, im = per_clip(lambda clip: self.synsq_planes(fre_arr, filter_bank_type, clip.real, clip.imag), z, clip_ndim=2)
        return re + 1j * im
