"""Chirp z-transform (reference binding: python/audioflux/dsp/czt.py; C: src/dsp/czt_algorithm.c).

Same constructor, ``czt`` method and argument names as the reference's ``CZT``: ``czt`` casts its input to float32 as
the reference does (a complex input loses its imaginary part) and returns complex [..., 2n] for n input samples: the
N = 2**radix2_exp CZT bins, then the N tail values the C function writes behind them, then zeros.  ``czt_batch``
transforms many rows in one call, takes real or complex numpy arrays or CUDA tensors (a complex row keeps its imaginary
part) and returns the same kind.

Differences from the reference, on purpose: ``radix2_exp`` above 13 or below 0 raises ``ValueError`` (the 2N-point
transforms run in one CTA's shared memory); ``czt`` raises ``ValueError`` when n < 2**radix2_exp, where the reference
reads and writes past its arrays."""
from __future__ import annotations

import numpy as np

from .base import MEM_HOST, Base, Batch, is_torch

__all__ = ["CZT"]


class CZT(Base):
    """The N = 2**radix2_exp point chirp z-transform over the band [low_w, high_w) of the normalised frequency."""

    def __init__(self, radix2_exp, _lib=None):
        super().__init__(_lib)
        self.radix2_exp = radix2_exp
        self._new("cztObj_new", "cztObj_free", int(radix2_exp))
        self.fft_length = 1 << int(radix2_exp)

    def czt_batch(self, data, low_w, high_w):
        """data [..., N] real or complex (numpy host | torch cuda) -> complex64 [..., 2N] of the same kind: the CZT, then
        the tail.  One cztObj_cztBatch call; each row is bit-identical to a legacy call on it.  A band outside
        0 <= low_w < high_w <= 1 keeps the object's last valid band, as in the reference."""
        if is_torch(data):
            cplx = data.is_complex()
            re, im = (data.real, data.imag) if cplx else (data, None)
        else:
            data = np.asarray(data)
            cplx = np.iscomplexobj(data)
            re, im = (data.real, data.imag) if cplx else (data, None)
        b = Batch(re)
        if b.n != self.fft_length:
            raise ValueError(f"rows must hold 2**radix2_exp = {self.fft_length} samples, not {b.n}")
        y = b.second(im, "the imaginary part") if cplx else None
        re3, im3 = b.alloc(b.rows, 2 * b.n), b.alloc(b.rows, 2 * b.n)
        if b.rows:
            self._call("cztObj_cztBatch", b, b.x, y, b.rows, float(low_w), float(high_w), re3, im3)
        if b.kind == MEM_HOST:
            out = (re3 + 1j * im3).astype(np.complex64)
        else:
            import torch
            out = torch.complex(re3, im3)
        return b.shaped(out)

    def czt(self, data_arr, low_w, high_w):
        """data_arr [..., n] as float32, n >= 2**radix2_exp (the first 2**radix2_exp samples are used) -> complex64
        [..., 2n]"""
        data_arr = np.asarray(data_arr, dtype=np.float32, order='C')
        if data_arr.ndim == 0:
            raise ValueError('Audio data must have at least one dimension')
        n = data_arr.shape[-1]
        if n < self.fft_length:
            raise ValueError(f"data length {n} is below 2**radix2_exp = {self.fft_length}")
        head = self.czt_batch(data_arr[..., :self.fft_length], low_w, high_w)
        out = np.zeros((*data_arr.shape[:-1], 2 * n), np.complex64)
        out[..., :2 * self.fft_length] = head
        return out
