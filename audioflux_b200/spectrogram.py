"""Spectrogram front door: STFT -> power/magnitude -> Linear slice or mel/bark/erb/... bank, plus the
cepstral calls (reference binding: python/audioflux/spectrogram.py:31-503, 1771-2270;
C: src/spectrogram_algorithm.c).  Chroma / Deep bank types and the spectral descriptors are outside the path."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .base import Base, BandAxis, Batch, as_f32, band_range, is_log_scale, np_ptr, per_clip, swap_last2
from .capi import opt_int, opt_float
from .types import (WindowType, SpectralFilterBankScaleType, SpectralFilterBankStyleType,
                    SpectralFilterBankNormalType, SpectralDataType, CepstralRectifyType, enum_value)


class Spectrogram(BandAxis, Base):
    def __init__(self, num=0, samplate=32000, low_fre=None, high_fre=None, bin_per_octave=12, radix2_exp=12,
                 window_type=None, slide_length=None, data_type=SpectralDataType.POWER,
                 filter_bank_type=SpectralFilterBankScaleType.LINEAR,
                 style_type=SpectralFilterBankStyleType.SLANEY,
                 normal_type=SpectralFilterBankNormalType.NONE, is_continue=False, _lib=None):
        super().__init__(_lib)
        scale = enum_value(filter_bank_type)
        if scale == 5:
            if bin_per_octave not in (12, 24, 36):
                raise ValueError(f"bin_per_octave={bin_per_octave} must be 12, 24 or 36")
            if num % bin_per_octave != 0:
                raise ValueError(f"num={num} must be an integer multiple of bin_per_octave={bin_per_octave}")
        low_fre, high_fre = band_range(low_fre, high_fre, scale, samplate)
        if window_type is None:
            window_type = WindowType.HANN
        if is_log_scale(scale) and low_fre < 32.703:
            raise ValueError(f"low_fre={low_fre} must be greater than or equal to 32.703")
        if low_fre < 0:
            raise ValueError(f"low_fre={low_fre} must be a non-negative number")
        self.fft_length = 1 << radix2_exp
        if slide_length is None:
            slide_length = self.fft_length // 4
        self.samplate, self.low_fre, self.high_fre = samplate, low_fre, high_fre
        self.bin_per_octave, self.radix2_exp, self.window_type = bin_per_octave, radix2_exp, window_type
        self.slide_length, self.is_continue, self.data_type = slide_length, is_continue, data_type
        self.filter_bank_type, self.style_type, self.normal_type = filter_bank_type, style_type, normal_type
        self._new("spectrogramObj_new", "spectrogramObj_free", int(num), opt_int(samplate), opt_float(low_fre),
                  opt_float(high_fre), opt_int(bin_per_octave), opt_int(radix2_exp), opt_int(enum_value(window_type)),
                  opt_int(slide_length), opt_int(int(is_continue)), opt_int(enum_value(data_type)), opt_int(scale),
                  opt_int(enum_value(style_type)), opt_int(enum_value(normal_type)))
        self.num = self.get_band_num()

    def set_data_norm_value(self, norm_value):
        self._lib.spectrogramObj_setDataNormValue(self._obj, C.c_float(norm_value))

    def cal_time_length(self, data_length):
        return self._lib.spectrogramObj_calTimeLength(self._obj, data_length)

    def get_band_num(self):
        return self._lib.spectrogramObj_getBandNum(self._obj)

    def get_bin_band_length(self):
        return self._lib.spectrogramObj_getBinBandLength(self._obj)

    def get_fre_band_arr(self):
        return self._floats("spectrogramObj_getFreBandArr", self.get_bin_band_length())

    def get_bin_band_arr(self):
        return self._ints("spectrogramObj_getBinBandArr", self.get_bin_band_length())

    def spectrogram_planes(self, data_arr, is_phase_arr=False):
        """Raw C layout: one clip -> [T, num] (and phase [T, num], Linear bank only)."""
        x = as_f32(data_arr)
        T = self.cal_time_length(x.shape[-1])
        spec = np.zeros((T, self.num), np.float32)
        phase = np.zeros((T, self.num), np.float32) if is_phase_arr else None
        self._lib.spectrogramObj_spectrogram(self._obj, np_ptr(x), x.shape[-1], np_ptr(spec),
                                             np_ptr(phase) if is_phase_arr else None)
        return (spec, phase) if is_phase_arr else spec

    def spectrogram(self, data_arr, is_phase_arr=False):
        """data [..., L] -> [..., num, T] (and phase) as spectrogram.py:239-326."""
        if is_phase_arr and enum_value(self.filter_bank_type) != 0:
            raise ValueError("Only LINEAR bank type has phase arr")
        x = as_f32(data_arr)
        if is_phase_arr:
            return tuple(map(swap_last2, per_clip(lambda clip: self.spectrogram_planes(clip, True), x)))
        spec, = per_clip(lambda clip: (self.spectrogram_planes(clip),), x)
        return swap_last2(spec)

    def spectrogram_batch(self, data, is_phase_arr=False):
        """Additive: data [B, L] (numpy host | torch cuda) -> [B, T, num] (time-major; + phase for LINEAR)."""
        b = Batch(data)
        T = self.cal_time_length(b.n)
        spec = b.alloc(b.rows, T, self.num)
        phase = b.alloc(b.rows, T, self.num) if is_phase_arr else None
        self._call("spectrogramObj_spectrogramBatch", b, b.x, b.n, b.rows, spec, phase)
        return (b.shaped(spec), b.shaped(phase)) if is_phase_arr else b.shaped(spec)

    def mfcc_batch(self, data, cc_num=13, rectify_type=CepstralRectifyType.LOG):
        """Additive: the fused STFT -> bank -> log -> DCT kernel. data [B, L] -> [B, T, cc_num]."""
        b = Batch(data)
        out = b.alloc(b.rows, self.cal_time_length(b.n), cc_num)
        self._call("spectrogramObj_mfccBatch", b, b.x, b.n, b.rows, cc_num, enum_value(rectify_type), out)
        return b.shaped(out)

    def _cc(self, fn_name, m_data_arr, cc_num, rectify_type=None):
        """[num, T] of the LAST spectrogram call -> [cc_num, T]."""
        m = as_f32(m_data_arr)
        if m.ndim != 2:
            raise ValueError("cepstral calls work on the [num, T] result of the preceding spectrogram() call")
        if cc_num > self.num:
            raise ValueError("cc_num must be <= num")
        mt = np.ascontiguousarray(m.T)
        out = np.zeros((mt.shape[0], cc_num), np.float32)
        fn = getattr(self._lib, fn_name)
        if fn_name == "spectrogramObj_xxcc":
            fn(self._obj, np_ptr(mt), cc_num, opt_int(enum_value(rectify_type)), np_ptr(out))
        else:
            fn(self._obj, np_ptr(mt), cc_num, np_ptr(out))
        return np.ascontiguousarray(out.T)

    def xxcc(self, m_data_arr, cc_num=13, rectify_type=CepstralRectifyType.LOG):
        return self._cc("spectrogramObj_xxcc", m_data_arr, cc_num, rectify_type)

    def mfcc(self, m_data_arr, cc_num=13):
        if enum_value(self.filter_bank_type) != 2:
            raise ValueError("mfcc needs the MEL bank type")
        return self._cc("spectrogramObj_mfcc", m_data_arr, cc_num)

    def bfcc(self, m_data_arr, cc_num=13):
        if enum_value(self.filter_bank_type) != 3:
            raise ValueError("bfcc needs the BARK bank type")
        return self._cc("spectrogramObj_bfcc", m_data_arr, cc_num)

    def gtcc(self, m_data_arr, cc_num=13):
        if enum_value(self.style_type) != 2:
            raise ValueError("gtcc needs the GAMMATONE style")
        return self._cc("spectrogramObj_gtcc", m_data_arr, cc_num)

    def x_coords(self, data_length):
        """Frame start times in seconds: slide_length / samplate apart (plot axis of the reference's spectrogram classes)."""
        if data_length < self.fft_length:
            raise ValueError(f"radix2_exp={self.radix2_exp}(fft_length={self.fft_length}) is too large for data_length={data_length}")
        return np.arange(self.cal_time_length(data_length) + 1) * (self.slide_length / self.samplate)

    def deconv(self, m_data_arr):
        """[num, T] of the LAST spectrogram call -> (tone, pitch), each [num, T] (spectrogram.py:328-362 of the reference)."""
        m = as_f32(m_data_arr)
        if m.ndim != 2:
            raise ValueError("deconv works on the [num, T] result of the preceding spectrogram() call")
        mt = np.ascontiguousarray(m.T)
        tone, pitch = np.zeros_like(mt), np.zeros_like(mt)
        self._lib.spectrogramObj_deconv(self._obj, np_ptr(mt), np_ptr(tone), np_ptr(pitch))
        return np.ascontiguousarray(tone.T), np.ascontiguousarray(pitch.T)

    def deconv_batch(self, m_tn):
        """Additive: [..., T, num] (numpy host | torch cuda, time-major as spectrogram_batch returns it) -> (tone, pitch)."""
        b = Batch(m_tn)
        if b.n != self.num:
            raise ValueError(f"last dimension must be num={self.num}")
        tone, pitch = b.alloc(b.rows, b.n), b.alloc(b.rows, b.n)
        self._call("spectrogramObj_deconvBatch", b, b.x, b.rows, tone, pitch)
        return b.shaped(tone), b.shaped(pitch)


def _scaled(scale, default_num):
    class _S(Spectrogram):
        def __init__(self, num=0, samplate=32000, low_fre=None, high_fre=None, radix2_exp=12,
                     window_type=WindowType.HANN, slide_length=None,
                     style_type=SpectralFilterBankStyleType.SLANEY,
                     normal_type=SpectralFilterBankNormalType.NONE,
                     data_type=SpectralDataType.POWER, is_continue=False, _lib=None):
            super().__init__(num=num or default_num, samplate=samplate, low_fre=low_fre, high_fre=high_fre,
                             radix2_exp=radix2_exp, window_type=window_type, slide_length=slide_length,
                             data_type=data_type, filter_bank_type=scale, style_type=style_type,
                             normal_type=normal_type, is_continue=is_continue, _lib=_lib)
    return _S


MelSpectrogram = _scaled(SpectralFilterBankScaleType.MEL, 128)     # spectrogram.py:1948-2054
MelSpectrogram.__name__ = "MelSpectrogram"
BarkSpectrogram = _scaled(SpectralFilterBankScaleType.BARK, 128)   # spectrogram.py:2056-2162
BarkSpectrogram.__name__ = "BarkSpectrogram"
ErbSpectrogram = _scaled(SpectralFilterBankScaleType.ERB, 128)     # spectrogram.py:2164-2270
ErbSpectrogram.__name__ = "ErbSpectrogram"
