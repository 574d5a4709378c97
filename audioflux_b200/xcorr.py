"""Cross-correlation (reference binding: python/audioflux/dsp/xcorr.py; C: src/dsp/xcorr_algorithm.c).

Same constructor, ``xcorr`` method, argument names, checks and defaults as the reference's ``Xcorr``: the Python default
normalisation is ``XcorrNormalType.NONE``, while a NULL normType in C means ``Coeff``.  ``xcorr_batch`` correlates many
pairs (or autocorrelates many rows) in one call, takes numpy arrays or CUDA tensors and returns the same kind.

Differences from the reference, on purpose: every call is computed from its own inputs.  The reference keeps buffers of
the transform length between calls and copies only ``n`` samples into them, so a later, shorter call with the same
transform length correlates samples left over from the earlier one."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .base import MEM_HOST, Base, Batch
from .types import XcorrNormalType, enum_value

__all__ = ["Xcorr"]


class Xcorr(Base):
    """Cross-correlation of two 1-D sequences of n samples: 2n-1 lags, numpy.correlate(a, b, 'full')."""

    def __init__(self, _lib=None):
        super().__init__(_lib)
        self._new("xcorrObj_new", "xcorrObj_free")

    def xcorr_batch(self, a, b=None, xcorr_normal_type=XcorrNormalType.NONE):
        """a [..., n] (numpy host | torch cuda), b of the same shape and memory or None (autocorrelation) ->
        (arr [..., 2n-1] float32, max_val [...] float32, index [...] int32) of the same kind: each row's lags, its
        maximum and the first index of the maximum.  One xcorrObj_xcorrBatch call; each row is bit-identical to a
        legacy call on its pair."""
        shape = a.shape if hasattr(a, "shape") else np.shape(a)
        if len(shape) == 0 or shape[-1] < 1:
            raise ValueError("the sequences must hold at least one sample")
        ba = Batch(a)
        y = None if b is None else ba.second(b, "b")
        out, mv = ba.alloc(ba.rows, 2 * ba.n - 1), ba.alloc(ba.rows)
        if ba.kind == MEM_HOST:
            idx = np.zeros(ba.rows, np.int32)
        else:
            import torch
            idx = torch.zeros(ba.rows, dtype=torch.int32, device=ba.device)
        if ba.rows:
            self._call("xcorrObj_xcorrBatch", ba, ba.x, y, ba.n, ba.rows,
                       C.byref(C.c_int(enum_value(xcorr_normal_type))), out, mv, idx)
        return ba.shaped(out), mv.reshape(ba.lead), idx.reshape(ba.lead)

    def xcorr(self, data_arr1, data_arr2=None, xcorr_normal_type=XcorrNormalType.NONE):
        """data_arr1 [n], data_arr2 [n] or None (autocorrelation) -> (arr [2n-1] float32, max_val float)"""
        data_arr1 = np.asarray(data_arr1, dtype=np.float32, order='C')
        data_arr2 = None if data_arr2 is None else np.asarray(data_arr2, dtype=np.float32, order='C')
        if data_arr1.ndim != 1:
            raise ValueError(f"data_arr1[ndim={data_arr1.ndim}] must be a 1D array")
        if data_arr2 is not None and data_arr2.ndim != 1:
            raise ValueError(f"data_arr2[ndim={data_arr2.ndim}] must be a 1D array")
        if data_arr2 is not None and data_arr1.shape != data_arr2.shape:
            raise ValueError(f"data_arr1.shape={data_arr1.shape} must be equal to data_arr2.shape={data_arr2.shape}")
        arr, mv, _ = self.xcorr_batch(data_arr1, data_arr2, xcorr_normal_type)
        return arr, float(mv)
