"""STFT object (reference binding: python/audioflux/stft.py:14-300; C: src/stft_algorithm.c)."""
from __future__ import annotations

import numpy as np

from .base import Base, Batch, as_f32, np_ptr, per_clip
from .capi import opt_int, opt_float
from .types import WindowType, PaddingPositionType, PaddingModeType, enum_value


class STFT(Base):
    def __init__(self, radix2_exp=12, window_type=WindowType.RECT, slide_length=1024, is_continue=False, _lib=None):
        super().__init__(_lib)
        self.radix2_exp = radix2_exp
        self.fft_length = 1 << radix2_exp
        self.window_type = window_type
        self.slide_length = slide_length
        self.is_continue = is_continue
        self._new("stftObj_new", "stftObj_free", radix2_exp, opt_int(enum_value(window_type)), opt_int(slide_length),
                  opt_int(int(is_continue)))

    def set_slide_length(self, slide_length):
        self._lib.stftObj_setSlideLength(self._obj, slide_length)
        self.slide_length = slide_length

    def enable_continue(self, flag=False):
        """streaming mode (src/stft_algorithm.c:180-183, 474-599): successive stft() calls continue one signal"""
        self._lib.stftObj_enableContinue(self._obj, int(flag))
        self.is_continue = bool(flag)

    def enable_padding(self, flag=False):
        self._lib.stftObj_enablePadding(self._obj, int(flag))

    def set_padding(self, position_type=PaddingPositionType.CENTER, mode_type=PaddingModeType.CONSTANT,
                    value1=0.0, value2=0.0):
        self._lib.stftObj_setPadding(self._obj, opt_int(enum_value(position_type)),
                                     opt_int(enum_value(mode_type)), opt_float(value1), opt_float(value2))

    def use_window_data_arr(self, data_arr):
        w = as_f32(data_arr)
        if w.shape != (self.fft_length,):
            raise ValueError("window must have fft_length samples")
        self._lib.stftObj_useWindowDataArr(self._obj, np_ptr(w))

    def get_window_data_arr(self):
        return self._floats("stftObj_getWindowDataArr", self.fft_length)

    def cal_time_length(self, data_length):
        return self._lib.stftObj_calTimeLength(self._obj, data_length)

    def stft_planes(self, data_arr):
        """Raw C layout: (re, im) each [T, fft_length] (full mirrored spectrum), one clip."""
        x = as_f32(data_arr)
        T = self.cal_time_length(x.shape[-1])
        re = np.zeros((T, self.fft_length), np.float32)
        im = np.zeros((T, self.fft_length), np.float32)
        self._lib.stftObj_stft(self._obj, np_ptr(x), x.shape[-1], np_ptr(re), np_ptr(im))
        return re, im

    def stft(self, data_arr):
        """-> complex [..., fft_length//2+1, T] like the reference wrapper (stft.py:259-300)."""
        re, im = per_clip(self.stft_planes, as_f32(data_arr))
        return np.ascontiguousarray(np.swapaxes(re + 1j * im, -1, -2)[..., : self.fft_length // 2 + 1, :])

    def stft_batch(self, data):
        """Additive batched entry point: data [B, L] (numpy host or torch cuda) ->
        (re, im) each [B, T, fft_length//2+1]."""
        b = Batch(data)
        T = self.cal_time_length(b.n)
        re, im = b.alloc(b.rows, T, self.fft_length // 2 + 1), b.alloc(b.rows, T, self.fft_length // 2 + 1)
        self._call("stftObj_stftBatch", b, b.x, b.n, b.rows, re, im)
        return b.shaped(re), b.shaped(im)

    def cal_data_length(self, time_length):
        return self._lib.stftObj_calDataLength(self._obj, int(time_length))

    def y_coords(self, samplate=32000):
        """Bin frequencies 0 .. samplate//2 with a leading 0 (plot axis, stft.py of the reference)."""
        return np.concatenate(([0.0], np.linspace(0, samplate // 2, self.fft_length // 2 + 1)))

    def x_coords(self, data_length, samplate=32000):
        if data_length < self.fft_length:
            raise ValueError(f"radix2_exp={self.radix2_exp}(fft_length={self.fft_length}) is too large for data_length={data_length}")
        return np.linspace(0, data_length / samplate, self.cal_time_length(data_length) + 1)

    def istft_planes(self, re, im, method_type=0):
        """Raw C layout: planes [T, fft_length] (full mirrored spectrum) -> data [(T-1)*slide + fft_length]."""
        re, im = as_f32(re), as_f32(im)
        out = np.zeros(self.cal_data_length(re.shape[0]), np.float32)
        self._lib.stftObj_istft(self._obj, np_ptr(re), np_ptr(im), re.shape[0], int(method_type), np_ptr(out))
        return out

    def istft(self, m_data_arr, method_type=0):
        """complex [..., fft_length//2+1, T] -> [..., data_length] like the reference wrapper (stft.py:302-361):
        method_type 0 'weight', 1 'overlap-add'."""
        z = np.asarray(m_data_arr)
        if not np.iscomplexobj(z):
            raise ValueError("m_data_arr must be of type np.complex")
        if z.ndim < 2:
            raise ValueError("m_data_arr's dimensions must be greater than 1")
        mirror = np.conj(z[..., ::-1, :][..., 1:-1, :])
        full = np.swapaxes(np.concatenate([z, mirror], axis=-2), -1, -2)          # [..., T, fft_length]
        out, = per_clip(lambda clip: (self.istft_planes(clip.real, clip.imag, method_type),), full, clip_ndim=2)
        return out

    def istft_batch(self, re, im, method_type=0):
        """Additive: planes [B, T, W] with W = fft_length//2+1 (as stft_batch returns them) or fft_length
        (numpy host | torch cuda) -> data [B, (T-1)*slide + fft_length]."""
        b = Batch(re)
        im = b.second(im, "im")
        if len(b.lead) < 1:
            raise ValueError("planes must be [..., T, W]")
        T = b.lead[-1]
        out = b.alloc(b.rows // T, self.cal_data_length(T), zero=True)
        self._call("stftObj_istftBatch", b, b.x, im, T, b.rows // T, b.n, int(method_type), out)
        return out.reshape(*b.lead[:-1], -1)
