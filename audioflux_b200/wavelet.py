"""Discrete wavelet transforms (reference bindings: python/audioflux/{dwt,swt,wpt}.py; C: src/{dwt,swt,wpt}_algorithm.c).

Same constructors, argument names and defaults as the reference's ``DWT``, ``SWT`` and ``WPT``, and the same ``dwt`` /
``swt`` / ``wpt`` tuples.  Each sends all channels to the GPU in one batched call; ``*_batch`` takes numpy arrays or
CUDA tensors and returns the same kind.

Differences from the reference, on purpose:
- ``DWT`` passes ``wavelet_type``, ``t1`` and ``t2`` to the C constructor.  The reference's binding passes the samplate
  where the wavelet type belongs, so its ``DWT`` always computes sym4.
- A filter this library does not generate (db40, sym7, sym10, sym20, sym30, coif, fk, bior4.4 / 5.5 / 6.8, dmey), or a
  transform longer than 2**20 samples, raises ``ValueError`` (see include/afb200_dwt.h)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .base import Base, Batch, as_f32, fit_length
from .types import WaveletDiscreteType, enum_value

__all__ = ["DWT", "SWT", "WPT"]


def _type_args(wavelet_type, t1, t2):
    return (C.byref(C.c_int(enum_value(wavelet_type))), C.byref(C.c_int(int(t1))), C.byref(C.c_int(int(t2))))


class _Tree(Base):
    """DWT and WPT: 2**radix2_exp samples -> coef [..., n] and m_data [..., rows, n]"""
    _name = None

    def __init__(self, num, radix2_exp, samplate, wavelet_type, t1, t2, _lib):
        super().__init__(_lib)
        if num is None:
            num = radix2_exp - 1
        self.num, self.radix2_exp, self.samplate = num, radix2_exp, samplate
        self.wavelet_type, self.t1, self.t2 = wavelet_type, t1, t2
        self.fft_length = 1 << radix2_exp
        self._new(f"{self._name}Obj_new", f"{self._name}Obj_free", C.c_int(int(num)), C.c_int(int(radix2_exp)),
                  *_type_args(wavelet_type, t1, t2))

    def _batch(self, data, m_data=True):
        b = Batch(data)
        if b.n != self.fft_length:
            raise ValueError(f"data length must be 2**radix2_exp = {self.fft_length}")
        coef = b.alloc(b.rows, b.n)
        m = b.alloc(b.rows, self._rows, b.n) if m_data else None
        if b.rows:
            self._call(f"{self._name}Obj_{self._name}Batch", b, b.x, b.rows, coef, m)
        return b.shaped(coef), b.shaped(m)

    def _transform(self, data_arr):
        x = np.asarray(data_arr, dtype=np.float32, order='C')
        if x.ndim == 0:
            raise ValueError('Audio data must have at least one dimension')
        return self._batch(fit_length(x, self.fft_length, warn=True))

    def y_coords(self):
        fre_arr = self.get_fre_band_arr()
        return np.insert(fre_arr, 0, fre_arr[0])

    def x_coords(self):
        return np.linspace(0, self.fft_length / self.samplate, self.fft_length + 1)


class DWT(_Tree):
    """Discrete wavelet transform: num levels of a 2**radix2_exp-sample signal."""
    _name = "dwt"

    def __init__(self, num=None, radix2_exp=12, samplate=32000, wavelet_type=WaveletDiscreteType.SYM, t1=4, t2=0,
                 _lib=None):
        n = radix2_exp - 1 if num is None else num
        if n >= radix2_exp or n <= 0:
            raise ValueError(f'The num={n} range is [1, {radix2_exp - 1}]')
        super().__init__(num, radix2_exp, samplate, wavelet_type, t1, t2, _lib)
        self._rows = self.num

    def get_fre_band_arr(self):
        """the reference's bands: 16000 / 2^k, lowest first, the first num of radix2_exp-1"""
        base = 16000 / 2.0 ** np.arange(self.radix2_exp - 1)
        return np.array(base[::-1][:self.num], dtype=np.float32)

    def dwt_batch(self, data, m_data=True):
        """data [..., 2**radix2_exp] (numpy host | torch cuda) -> (coef [..., n], m_data [..., num, n] or None)"""
        return self._batch(data, m_data)

    def dwt(self, data_arr):
        """data_arr [..., n] (padded or cut to 2**radix2_exp) -> (coef_arr [..., n], m_data_arr [..., num, n])"""
        return self._transform(data_arr)


class WPT(_Tree):
    """Wavelet packet transform: the full tree of num levels; 2**num leaves."""
    _name = "wpt"

    def __init__(self, num=None, radix2_exp=12, samplate=32000, wavelet_type=WaveletDiscreteType.SYM, t1=4, t2=0,
                 _lib=None):
        super().__init__(num, radix2_exp, samplate, wavelet_type, t1, t2, _lib)
        self._rows = 1 << self.num

    def get_fre_band_arr(self):
        return np.linspace(0, 16000, (1 << self.num), dtype=np.float32)

    def wpt_batch(self, data, m_data=True):
        """data [..., 2**radix2_exp] (numpy host | torch cuda) -> (coef [..., n], m_data [..., 2**num, n] or None)"""
        return self._batch(data, m_data)

    def wpt(self, data_arr):
        """data_arr [..., n] (padded or cut to 2**radix2_exp) -> (coef_arr [..., n], m_data_arr [..., 2**num, n])"""
        return self._transform(data_arr)


class SWT(Base):
    """Stationary wavelet transform: num undecimated levels of an fft_length-sample signal."""

    def __init__(self, num, fft_length, wavelet_type=WaveletDiscreteType.SYM, t1=4, t2=0, _lib=None):
        super().__init__(_lib)
        self.num, self.fft_length = num, fft_length
        self.wavelet_type, self.t1, self.t2 = wavelet_type, t1, t2
        self._new("swtObj_new", "swtObj_free", C.c_int(int(num)), C.c_int(int(fft_length)),
                  *_type_args(wavelet_type, t1, t2))

    def swt_batch(self, data):
        """data [..., fft_length] (numpy host | torch cuda) -> (approximations, details), each [..., num, fft_length]"""
        b = Batch(data)
        if b.n != self.fft_length:
            raise ValueError(f"data length must be fft_length = {self.fft_length}")
        m1, m2 = b.alloc(b.rows, self.num, b.n), b.alloc(b.rows, self.num, b.n)
        if b.rows and self.num:
            self._call("swtObj_swtBatch", b, b.x, b.rows, m1, m2)
        return b.shaped(m1), b.shaped(m2)

    def swt(self, data_arr):
        """data_arr [..., fft_length] -> (m_data_arr1, m_data_arr2), each [..., num, fft_length]"""
        x = as_f32(data_arr)
        if x.ndim == 0:
            raise ValueError('Audio data must have at least one dimension')
        return self.swt_batch(x)
