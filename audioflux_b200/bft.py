"""BFT object: STFT -> power/magnitude -> mel/bark/erb/... filter bank
(reference binding: python/audioflux/bft.py:16-390; C: src/bft_algorithm.c)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .base import MEM_DEVICE, Base, BandAxis, Batch, FrameAxis, as_f32, band_range, is_torch, np_ptr, per_clip, swap_last2
from .capi import opt_int, opt_float
from .lib import check
from .types import (WindowType, SpectralFilterBankScaleType, SpectralFilterBankStyleType,
                    SpectralFilterBankNormalType, SpectralDataType, CepstralRectifyType, enum_value)


class BFT(BandAxis, FrameAxis, Base):
    def __init__(self, num, radix2_exp=12, samplate=32000, low_fre=None, high_fre=None,
                 bin_per_octave=12, window_type=WindowType.HANN, slide_length=None,
                 scale_type=SpectralFilterBankScaleType.LINEAR,
                 style_type=SpectralFilterBankStyleType.SLANEY,
                 normal_type=SpectralFilterBankNormalType.NONE,
                 data_type=SpectralDataType.MAG, is_reassign=False, is_temporal=False, _lib=None):
        super().__init__(_lib)
        self.fft_length = fft_length = 1 << radix2_exp
        if num > fft_length // 2 + 1:
            raise ValueError(f"num={num} is too large")
        low_fre, high_fre = band_range(low_fre, high_fre, scale_type, samplate)
        if slide_length is None:
            slide_length = fft_length // 4
        self.num, self.radix2_exp, self.samplate = num, radix2_exp, samplate
        self.low_fre, self.high_fre, self.bin_per_octave = low_fre, high_fre, bin_per_octave
        self.window_type, self.slide_length = window_type, slide_length
        self.scale_type, self.style_type, self.normal_type = scale_type, style_type, normal_type
        self.data_type = data_type
        self.result_type = 0
        self.is_reassign, self.is_temporal = is_reassign, is_temporal
        self._new("bftObj_new", "bftObj_free", num, radix2_exp, opt_int(samplate), opt_float(low_fre),
                  opt_float(high_fre), opt_int(bin_per_octave), opt_int(enum_value(window_type)),
                  opt_int(slide_length), opt_int(enum_value(scale_type)), opt_int(enum_value(style_type)),
                  opt_int(enum_value(normal_type)), opt_int(enum_value(data_type)),
                  opt_int(int(is_reassign)), opt_int(int(is_temporal)))

    def cal_time_length(self, data_length):
        return self._lib.bftObj_calTimeLength(self._obj, data_length)

    def get_fre_band_arr(self):
        return self._floats("bftObj_getFreBandArr", self.num)

    def get_bin_band_arr(self):
        return self._ints("bftObj_getBinBandArr", self.num)

    def get_filter_bank_arr(self):
        """Additive: dense bank [num, fft_length//2+1] the device kernels consume."""
        fn = self._require_ext("bftObj_getFilterBankArr")
        out = np.zeros((self.num, self.fft_length // 2 + 1), np.float32)
        check(fn(self._obj, np_ptr(out)), "bftObj_getFilterBankArr")
        return out

    def set_result_type(self, result_type):
        self._lib.bftObj_setResultType(self._obj, int(result_type))
        self.result_type = int(result_type)

    def set_data_norm_value(self, norm_value):
        self._lib.bftObj_setDataNormValue(self._obj, C.c_float(norm_value))

    def bft_planes(self, data_arr, result_type=0):
        """Raw C layout: (re, im) each [T, num] for one clip."""
        x = as_f32(data_arr)
        if result_type != self.result_type:
            self.set_result_type(result_type)
        T = self.cal_time_length(x.shape[-1])
        re = np.zeros((T, self.num), np.float32)
        im = np.zeros((T, self.num), np.float32)
        self._lib.bftObj_bft(self._obj, np_ptr(x), x.shape[-1], np_ptr(re), np_ptr(im))
        return re, im

    def get_temporal_data(self, data_length):
        """(energy, rms, zero-crossing rate) of the frames of the LAST `bft` call, each [T] (bft.py:391-417,
        bftObj_getTemporalData); needs is_temporal=True."""
        if not self.is_temporal:
            raise ValueError("Please set the parameter is_temporal=True when creating the BFT object")
        T = self.cal_time_length(data_length)
        ptrs = [C.POINTER(C.c_float)() for _ in range(3)]
        self._lib.bftObj_getTemporalData(self._obj, *[C.byref(q) for q in ptrs])
        if not all(bool(q) for q in ptrs):
            raise ValueError("Please call the `BFT.bft()` method before calling this method")
        return tuple(np.ctypeslib.as_array(q, shape=(T,)).copy() for q in ptrs)

    def bft(self, data_arr, result_type=0):
        """-> [..., num, T] complex (result_type 0) or float32 (1), as bft.py:310-389."""
        x = as_f32(data_arr)
        if x.shape[-1] < self.fft_length:
            raise ValueError(f"radix2_exp={self.radix2_exp} is too large for data length {x.shape[-1]}")
        re, im = per_clip(lambda clip: self.bft_planes(clip, result_type), x)
        return swap_last2(re if result_type else re + 1j * im)

    # ---- additive batched / device-pointer entry points (include/afb200_ext.h) ----
    def bft_batch(self, data, result_type=1):
        """data [B, L] (numpy host | torch cuda) -> [B, T, num] real, or (re, im) for result_type 0."""
        if result_type != self.result_type:
            self.set_result_type(result_type)
        b = Batch(data)
        T = self.cal_time_length(b.n)
        re = b.alloc(b.rows, T, self.num)
        im = b.alloc(b.rows, T, self.num) if result_type == 0 else None
        self._call("bftObj_bftBatch", b, b.x, b.n, b.rows, re, im)
        return b.shaped(re) if result_type else (b.shaped(re), b.shaped(im))

    def mfcc_batch(self, data, cc_num=13, rectify_type=CepstralRectifyType.LOG, out=None):
        """Fused STFT -> |.|^2 (or |.|) -> bank -> log10/cbrt -> DCT-II(ortho) -> first cc_num.
        data [B, L] -> [B, T, cc_num].  Equals bft(result_type=1) followed by XXCC.xxcc.
        Host arrays go through the library's chunked copy-in / transform / copy-out pipeline; pass page-locked arrays
        (and a page-locked `out`) to run it at PCIe speed."""
        b = Batch(data)
        T = self.cal_time_length(b.n)
        if out is None:
            out = b.alloc(b.rows, T, cc_num)
        elif (is_torch(out) != (b.kind == MEM_DEVICE) or tuple(out.shape) != (b.rows, T, cc_num)
              or not (out.flags["C_CONTIGUOUS"] if hasattr(out, "flags") else out.is_contiguous())):
            raise ValueError(f"out must be a contiguous float32 array of shape {(b.rows, T, cc_num)} in the memory of data")
        self._call("bftObj_mfccBatch", b, b.x, b.n, b.rows, cc_num, enum_value(rectify_type), out)
        return b.shaped(out)
