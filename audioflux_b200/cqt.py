"""Constant-Q transform object (reference binding: python/audioflux/cqt.py:20-150, 515-655;
C: src/cqt_algorithm.c)."""
from __future__ import annotations

import numpy as np

from .base import C1_HZ, Base, BandAxis, Batch, FrameAxis, as_f32, np_ptr, per_clip, swap_last2
from .capi import opt_int, opt_float
from .lib import check
from .types import (WindowType, SpectralFilterBankNormalType, SpectralDataType, ChromaDataNormalType,
                    CepstralRectifyType, enum_value)


class CQT(BandAxis, FrameAxis, Base):
    _needs_full_frame = False            # padded frames: any data length gives data_length // slide + 1 columns
    def __init__(self, num=84, samplate=32000, low_fre=C1_HZ, bin_per_octave=12, factor=1., beta=0.,
                 thresh=0.01, window_type=WindowType.HANN, slide_length=None,
                 normal_type=SpectralFilterBankNormalType.AREA, is_scale=True, is_continue=False, _lib=None):
        super().__init__(_lib)
        if low_fre < 27.5:
            raise ValueError("low_fre must be >= 27.5")
        self.num, self.samplate, self.low_fre = num, samplate, low_fre
        self.bin_per_octave, self.factor, self.beta, self.thresh = bin_per_octave, factor, beta, thresh
        self.window_type, self.slide_length = window_type, slide_length
        self.normal_type, self.is_scale = normal_type, is_scale
        self.is_continue = is_continue
        self._new("cqtObj_newWith", "cqtObj_free", num, opt_int(samplate), opt_float(low_fre), opt_int(bin_per_octave),
                  opt_float(factor), opt_float(beta), opt_float(thresh), opt_int(enum_value(window_type)),
                  opt_int(slide_length), opt_int(int(is_continue)), opt_int(enum_value(normal_type)), opt_int(int(is_scale)))
        self.fft_length = self.get_fft_length()
        if self.slide_length is None:
            self.slide_length = self.fft_length // 4

    def cal_time_length(self, data_length):
        return self._lib.cqtObj_calTimeLength(self._obj, data_length)

    def get_fft_length(self):
        return self._lib.cqtObj_getFFTLength(self._obj)

    def get_fre_band_arr(self):
        return self._floats("cqtObj_getFreBandArr", self.num)

    def set_scale(self, flag=True):
        self._lib.cqtObj_setScale(self._obj, int(flag))

    def get_kernel_bank(self):
        """Additive: (kr, ki) spectral kernels [bin_per_octave (num when beta != 0: VQT), fft_length//2+1]."""
        fn = self._require_ext("cqtObj_getKernelBank")
        kr = np.zeros((self.num if self.beta else self.bin_per_octave, self.fft_length // 2 + 1), np.float32)
        ki = np.zeros_like(kr)
        check(fn(self._obj, np_ptr(kr), np_ptr(ki)), "cqtObj_getKernelBank")
        return kr, ki

    OCTAVE_KERNELS = ("wgmma", "mma.sync", "fp32 loop", "direct")

    def octave_plan(self):
        """Additive diagnostics: per octave, top octave first, a dict of the kernel that computes it (a name of
        OCTAVE_KERNELS), its hop, frames per CTA (0: direct kernel), threads per CTA, tap segments and dynamic shared memory
        bytes (cqtObj_octavePlan; host only, needs no device)."""
        fn = self._require_ext("cqtObj_octavePlan")
        octs = self.num // self.bin_per_octave
        cols = {k: np.zeros(octs, np.int32) for k in ("kernel", "hop", "frames", "threads", "segs", "smem")}
        n = fn(self._obj, *(np_ptr(cols[k]) for k in ("kernel", "hop", "frames", "threads", "segs", "smem")))
        if n != octs:
            raise RuntimeError(f"cqtObj_octavePlan returned {n} for {octs} octaves")
        return [dict(kernel=self.OCTAVE_KERNELS[cols["kernel"][k]], **{c: int(cols[c][k]) for c in cols if c != "kernel"})
                for k in range(octs)]

    def cqt_planes(self, data_arr):
        x = as_f32(data_arr)
        T = self.cal_time_length(x.shape[-1])
        re = np.zeros((T, self.num), np.float32)
        im = np.zeros((T, self.num), np.float32)
        self._lib.cqtObj_cqt(self._obj, np_ptr(x), x.shape[-1], np_ptr(re), np_ptr(im))
        return re, im

    def cqt(self, data_arr):
        """-> complex [..., num, T] as cqt.py:107-150."""
        re, im = per_clip(self.cqt_planes, as_f32(data_arr))
        return swap_last2(re + 1j * im)

    def cqt_batch(self, data):
        """Additive: data [B, L] (numpy host | torch cuda) -> (re, im) each [B, T, num]."""
        b = Batch(data)
        T = self.cal_time_length(b.n)
        re, im = b.alloc(b.rows, T, self.num), b.alloc(b.rows, T, self.num)
        self._call("cqtObj_cqtBatch", b, b.x, b.n, b.rows, re, im)
        return b.shaped(re), b.shaped(im)

    def chroma_planes(self, re, im, chroma_num=12, data_type=SpectralDataType.POWER,
                      norm_type=ChromaDataNormalType.MAX):
        """Raw C layout: planes [T, num] of the LAST cqt call -> [T, chroma_num] (cqtObj_chroma,
        src/cqt_algorithm.c:484-600)."""
        re, im = as_f32(re), as_f32(im)
        out = np.zeros((re.shape[0], chroma_num), np.float32)
        self._lib.cqtObj_chroma(self._obj, opt_int(chroma_num), opt_int(enum_value(data_type)),
                                opt_int(enum_value(norm_type)), np_ptr(re), np_ptr(im), np_ptr(out))
        return out

    def chroma(self, m_cqt_data, chroma_num=12, data_type=SpectralDataType.POWER,
               norm_type=ChromaDataNormalType.MAX):
        """complex [num, T] (result of the last ``cqt`` call) -> [chroma_num, T] as cqt.py:153-221."""
        z = np.asarray(m_cqt_data)
        if z.ndim != 2:
            raise ValueError("chroma works on the [num, T] result of the preceding cqt() call")
        zt = np.swapaxes(z, -1, -2)
        return swap_last2(self.chroma_planes(zt.real, zt.imag, chroma_num, data_type, norm_type))

    def chroma_batch(self, re, im, chroma_num=12, data_type=SpectralDataType.POWER,
                     norm_type=ChromaDataNormalType.MAX):
        """Additive: planes [..., T, num] (numpy host | torch cuda) -> [..., T, chroma_num]."""
        b = Batch(re)
        im = b.second(im, "im")
        out = b.alloc(b.rows, chroma_num)
        self._call("cqtObj_chromaBatch", b, b.x, im, b.rows, chroma_num, enum_value(data_type), enum_value(norm_type), out)
        return b.shaped(out)

    def cqcc_planes(self, m_tn, cc_num=13, rectify_type=CepstralRectifyType.LOG):
        """Raw C layout: [T, num] of the LAST cqt call -> [T, cc_num] (cqtObj_cqcc, src/cqt_algorithm.c:602-660)."""
        m = as_f32(m_tn)
        out = np.zeros((m.shape[0], cc_num), np.float32)
        self._lib.cqtObj_cqcc(self._obj, np_ptr(m), cc_num, opt_int(enum_value(rectify_type)), np_ptr(out))
        return out

    def cqcc(self, m_data_arr, cc_num=13, rectify_type=CepstralRectifyType.LOG):
        """[num, T] power / magnitude of the last cqt call -> [cc_num, T] as cqt.py:223-275."""
        m = np.asarray(m_data_arr)
        if np.iscomplexobj(m):
            m = np.abs(m)
        return swap_last2(self.cqcc_planes(np.swapaxes(as_f32(m), -1, -2), cc_num, rectify_type))

    def cqcc_batch(self, m_tn, cc_num=13, rectify_type=CepstralRectifyType.LOG):
        """Additive: [..., T, num] (numpy host | torch cuda) -> [..., T, cc_num]."""
        b = Batch(m_tn)
        out = b.alloc(b.rows, cc_num)
        self._call("cqtObj_cqccBatch", b, b.x, b.rows, cc_num, enum_value(rectify_type), out)
        return b.shaped(out)

    def cqhc_planes(self, m_tn, hc_num=20):
        """Raw C layout: [T, num] of the LAST cqt call -> [T, hc_num] (cqtObj_cqhc, src/cqt_algorithm.c:662-714)."""
        m = as_f32(m_tn)
        out = np.zeros((m.shape[0], hc_num), np.float32)
        self._lib.cqtObj_cqhc(self._obj, np_ptr(m), int(hc_num), np_ptr(out))
        return out

    def cqhc(self, m_data_arr, hc_num=20):
        """[num, T] power / magnitude (complex input: power) of the last cqt call -> [hc_num, T] as cqt.py:277-323."""
        m = np.asarray(m_data_arr)
        if np.iscomplexobj(m):
            m = np.abs(m) ** 2
        return swap_last2(self.cqhc_planes(np.swapaxes(as_f32(m), -1, -2), hc_num))

    def deconv_planes(self, m_tn):
        """Raw C layout: [T, num] of the LAST cqt call -> (timbre, pitch) each [T, num] (cqtObj_deconv, :716-781)."""
        m = as_f32(m_tn)
        tone, pitch = np.zeros_like(m), np.zeros_like(m)
        self._lib.cqtObj_deconv(self._obj, np_ptr(m), np_ptr(tone), np_ptr(pitch))
        return tone, pitch

    def deconv(self, m_data_arr):
        """[num, T] magnitude / power (complex input: magnitude) -> (tone, pitch) each [num, T] as cqt.py:325-375."""
        m = np.asarray(m_data_arr)
        if np.iscomplexobj(m):
            m = np.abs(m)
        tone, pitch = self.deconv_planes(np.swapaxes(as_f32(m), -1, -2))
        return swap_last2(tone), swap_last2(pitch)

    def cqhc_batch(self, m_tn, hc_num=20):
        """Additive: [..., T, num] (numpy host | torch cuda) -> [..., T, hc_num]."""
        b = Batch(m_tn)
        out = b.alloc(b.rows, hc_num)
        self._call("cqtObj_cqhcBatch", b, b.x, b.rows, int(hc_num), out)
        return b.shaped(out)

    def deconv_batch(self, m_tn):
        """Additive: [..., T, num] (numpy host | torch cuda) -> (timbre, pitch) each [..., T, num]."""
        b = Batch(m_tn)
        tone, pitch = b.alloc(b.rows, b.n), b.alloc(b.rows, b.n)
        self._call("cqtObj_deconvBatch", b, b.x, b.rows, tone, pitch)
        return b.shaped(tone), b.shaped(pitch)
