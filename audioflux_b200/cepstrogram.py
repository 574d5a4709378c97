"""Cepstrogram (reference binding: python/audioflux/cepstrogram.py:14-227; C: src/cepstrogram_algorithm.c).

Same constructor, ``cal_time_length``, ``cepstrogram`` and plot coordinates as the reference class.  ``cepstrogram``
sends all channels to the GPU in one batched call.  ``cepstrogram_batch`` takes numpy arrays or CUDA tensors and
returns the C layout ``[..., time, fre]``; ``cepstrogram2_batch`` starts from STFT planes.  Both can skip outputs.

One difference from the reference, on purpose: ``cep_num`` outside 1 .. fft_length/2 raises ``ValueError`` (the
reference's C code reads and writes out of bounds there)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .base import Base, Batch, FrameAxis, swap_last2
from .types import WindowType, enum_value


class Cepstrogram(FrameAxis, Base):
    def __init__(self, radix2_exp=12, samplate=32000, window_type=WindowType.RECT, slide_length=1024, _lib=None):
        super().__init__(_lib)
        self.radix2_exp, self.samplate = radix2_exp, samplate
        self.window_type, self.slide_length = window_type, slide_length
        self.fft_length = 1 << radix2_exp
        self._new("cepstrogramObj_new", "cepstrogramObj_free", radix2_exp, C.byref(C.c_int(enum_value(window_type))),
                  C.byref(C.c_int(slide_length)))

    def cal_time_length(self, data_length):
        return self._lib.cepstrogramObj_calTimeLength(self._obj, int(data_length))

    def y_coords(self):
        return np.linspace(0, self.samplate / 2, self.fft_length // 2 + 2)

    def _check_cep_num(self, cep_num):
        if not 1 <= cep_num <= self.fft_length // 2:
            raise ValueError(f"cep_num={cep_num} must be in 1 .. fft_length/2 = {self.fft_length // 2}")

    def _outputs(self, b, shape, want):
        return [b.alloc(*shape, self.fft_length // 2 + 1) if w else None for w in want]

    def cepstrogram_batch(self, data, cep_num=4, cep=True, env=True, det=True):
        """data [..., n] (numpy host | torch cuda) -> (cepstrums, envelope, details), each [..., time, fft_length/2+1]
        or None when not requested.  One cepstrogramObj_cepstrogramBatch call."""
        self._check_cep_num(cep_num)
        if not (cep or env or det):
            raise ValueError("request at least one of cep, env, det")
        b = Batch(data)
        t = self.cal_time_length(b.n)
        out = self._outputs(b, (b.rows, t), (cep, env, det))
        if b.rows and t:
            self._call("cepstrogramObj_cepstrogramBatch", b, cep_num, b.x, b.n, b.rows, *out)
        return tuple(map(b.shaped, out))

    def cepstrogram2_batch(self, m_real, m_imag, cep_num=4, cep=True, env=True, det=True):
        """STFT planes [..., rows, width], width fft_length (the mirrored layout of the legacy STFT) or
        fft_length/2+1 (the layout of STFT.stft_batch) -> (cepstrums, envelope, details), each
        [..., rows, fft_length/2+1] or None.  The planes are read only.  One cepstrogramObj_cepstrogram2Batch call."""
        self._check_cep_num(cep_num)
        if not (cep or env or det):
            raise ValueError("request at least one of cep, env, det")
        b = Batch(m_real)
        im = b.second(m_imag, "m_imag")
        if b.n not in (self.fft_length, self.fft_length // 2 + 1):
            raise ValueError(f"plane width {b.n} must be fft_length={self.fft_length} or fft_length/2+1")
        out = self._outputs(b, (b.rows,), (cep, env, det))
        if b.rows:
            self._call("cepstrogramObj_cepstrogram2Batch", b, cep_num, b.x, im, b.rows, b.n, *out)
        return tuple(map(b.shaped, out))

    def cepstrogram(self, data_arr, cep_num=4):
        """data_arr [..., n] -> (cepstrums, envelope, details), each [..., fft_length/2+1, time] float32"""
        data_arr = np.asarray(data_arr, dtype=np.float32, order='C')
        if data_arr.ndim == 0:
            raise ValueError('Audio data must have at least one dimension')
        return tuple(swap_last2(o) for o in self.cepstrogram_batch(data_arr, cep_num))
