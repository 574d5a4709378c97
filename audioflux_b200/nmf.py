"""Non-negative matrix factorisation (reference binding: python/audioflux/classic/nmf.py; C: src/classic/nmf.c).

``nmf`` has the reference's signature, defaults and ``arange`` initialisation and returns ``(h_arr, w_arr)``.
``nmf_batch`` factorises a stack of matrices in one call, takes numpy arrays or CUDA tensors and returns the same kind;
each matrix gives the same bits as ``nmf`` on it."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import lib as _libmod
from .base import MEM_DEVICE, MEM_HOST, _arg, as_f32, is_torch

__all__ = ["nmf", "nmf_batch"]


def _arange_init(lead, n, m, k):
    h = np.arange(1, k * m + 1, dtype=np.float32).reshape(k, m)
    w = np.arange(1, n * k + 1, dtype=np.float32).reshape(n, k)
    return np.broadcast_to(h, (*lead, k, m)).copy(), np.broadcast_to(w, (*lead, n, k)).copy()


def nmf_batch(X, k, max_iter=300, tp=0, thresh=1e-3, norm=0, w_init=None, h_init=None, return_iters=False):
    """X [..., n, m] (numpy host | torch cuda) -> (h [..., k, m], w [..., n, k]) float32 of the same kind, and with
    return_iters the iterations each matrix ran ([...] int32).  w_init / h_init (same lead axes and memory as X) replace
    the reference's arange initialisation; they are not modified.  tp 0 KL, 1 IS, other Euclidean; norm 1 | 2 column
    p-norm of W, other column max."""
    k = int(k)
    if k < 1:
        raise ValueError(f"k={k} must be at least 1")
    if X.ndim < 2:
        raise ValueError(f"X[ndim={X.ndim}] must have at least 2 dimensions")
    lead, (n, m) = tuple(X.shape[:-2]), tuple(X.shape[-2:])
    batch = int(np.prod(lead, dtype=np.int64))
    torch_in = is_torch(X)
    if torch_in:
        import torch
        if not X.is_cuda:
            raise ValueError("torch inputs must live on a CUDA device; pass numpy arrays for host data")
        dev = X.device
        x = X.contiguous().float()
        kind, stream = MEM_DEVICE, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        conv = (lambda a: torch.as_tensor(a).to(dev).float().contiguous().clone())
        iters = torch.zeros(lead, dtype=torch.int32, device=dev)
    else:
        x = as_f32(X)
        kind, stream = MEM_HOST, C.c_void_p(None)
        conv = (lambda a: np.array(a, dtype=np.float32, order='C', copy=True))
        iters = np.zeros(lead, np.int32)
    h0, w0 = _arange_init(lead, n, m, k)
    h = conv(h0 if h_init is None else h_init)
    w = conv(w0 if w_init is None else w_init)
    if tuple(h.shape) != (*lead, k, m) or tuple(w.shape) != (*lead, n, k):
        raise ValueError(f"h_init must be {(*lead, k, m)} and w_init {(*lead, n, k)}")
    if batch and n and m:
        fn = _libmod.get_lib().nmfBatch
        _libmod.check(fn(_arg(x), batch, n, m, k, _arg(w), _arg(h), C.byref(C.c_int(int(max_iter))),
                         C.byref(C.c_int(int(tp))), C.byref(C.c_float(float(thresh))), C.byref(C.c_int(int(norm))),
                         _arg(iters), kind, stream), "nmfBatch")
    return (h, w, iters) if return_iters else (h, w)


def nmf(X, k, max_iter=300, tp=0, thresh=1e-3, norm=0):
    """X [n, m] -> (h_arr [k, m], w_arr [n, k]) float32, as the reference's nmf"""
    X = np.asarray(X, dtype=np.float32, order='C')
    if X.ndim != 2:
        raise ValueError(f"X[ndim={X.ndim}] must be a 2D array")
    return nmf_batch(X, k, max_iter=max_iter, tp=tp, thresh=thresh, norm=norm)
