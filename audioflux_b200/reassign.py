"""Time-frequency reassignment (reference binding: python/audioflux/reassign.py:94-282; C: src/reassign_algorithm.c)."""
from __future__ import annotations

import numpy as np

from .base import Base, Batch, as_f32, np_ptr, per_clip, swap_last2
from .capi import opt_int, opt_float
from .types import ReassignType, WindowType, enum_value


class Reassign(Base):
    def __init__(self, radix2_exp=12, samplate=32000, window_type=WindowType.HANN, slide_length=None,
                 re_type=ReassignType.ALL, thresh=0.001, is_padding=False, _lib=None):
        super().__init__(_lib)
        self.fft_length = 1 << radix2_exp
        self.radix2_exp, self.samplate, self.window_type = radix2_exp, samplate, window_type
        self.slide_length = self.fft_length // 4 if slide_length is None else slide_length
        self.re_type, self.thresh, self.is_padding = re_type, thresh, is_padding
        self.is_continue, self.order, self.result_type = False, 1, 0
        self._new("reassignObj_new", "reassignObj_free", radix2_exp, opt_int(samplate), opt_int(enum_value(window_type)),
                  opt_int(self.slide_length), opt_int(enum_value(re_type)), opt_float(thresh), opt_int(int(is_padding)),
                  opt_int(0))

    def cal_time_length(self, data_length):
        return self._lib.reassignObj_calTimeLength(self._obj, int(data_length))

    def set_result_type(self, result_type):
        self._lib.reassignObj_setResultType(self._obj, int(result_type))
        self.result_type = result_type

    def set_order(self, order):
        self._lib.reassignObj_setOrder(self._obj, int(order))
        self.order = order

    def reassign_planes(self, data_arr, result_type=0):
        """Raw C layout for one clip: (re, im, stft_re, stft_im), each [T, fft_length/2+1]."""
        x = as_f32(data_arr)
        if result_type != self.result_type:
            self.set_result_type(result_type)
        shape = (self.cal_time_length(x.shape[-1]), self.fft_length // 2 + 1)
        out = [np.zeros(shape, np.float32) for _ in range(4)]
        self._lib.reassignObj_reassign(self._obj, np_ptr(x), x.shape[-1], *[np_ptr(o) for o in out])
        return tuple(out)

    def reassign(self, data_arr, result_type=0):
        """-> (reassigned, stft): [..., fre, time]; complex (result_type 0) or amplitude (1) as reassign.py:177-246."""
        re, im, sr, si = per_clip(lambda clip: self.reassign_planes(clip, result_type), as_f32(data_arr))
        return swap_last2(re + 1j * im if result_type == 0 else re), swap_last2(sr + 1j * si)

    def reassign_batch(self, data, result_type=0):
        """Additive batched form (numpy host arrays or CUDA torch tensors): -> (re, im, stft_re, stft_im), each
        [..., T, fft_length/2+1], one call for the whole batch."""
        if result_type != self.result_type:
            self.set_result_type(result_type)
        b = Batch(data)
        T, W = self.cal_time_length(b.n), self.fft_length // 2 + 1
        outs = [b.alloc(b.rows, T, W, zero=k < 2) for k in range(4)]      # the reassigned planes are scattered into
        self._call("reassignObj_reassignBatch", b, b.x, b.n, b.rows, *outs)
        return tuple(map(b.shaped, outs))

    def y_coords(self):
        return np.linspace(0, self.samplate / 2, self.fft_length // 2 + 1 + 1)

    def x_coords(self, data_length):
        if data_length < self.fft_length:
            raise ValueError(f"radix2_exp={self.radix2_exp}(fft_length={self.fft_length}) is too large for data_length={data_length}")
        x_coords = np.linspace(0, data_length / self.samplate, self.cal_time_length(data_length) + 1)
        return x_coords
