"""Discrete wavelet transforms on the GPU: every supported filter on DWT, WPT and SWT within 1e-4 of the float64 oracle
and of the reference build, at small and long transforms; the batched entry points against the legacy call bit for bit
(host pointers across staging chunks, device pointers back to back); a NULL mDataArr leaving only coefArr written; and
the reference's own Python classes on this library."""
import ctypes as C

import numpy as np
import pytest

import _wavelet_oracle as W
from _parity_kit import dptr, raf, ref_lib_or_none, stream  # noqa: F401  (raf: a fixture)
from test_wavelet_cpu import CASES, TABLE, oracle

import audioflux_b200 as af

TOL = 1e-4                 # of max |value| of the output
gpu = pytest.mark.gpu
LONG = {f"{k}_{a}_{b}_{c}_long": (k, 4, 16 if k != "swt" else 1 << 16, a, b, c, 5) for k in ("dwt", "wpt", "swt")
        for a, b, c in ((2, 4, 0), (1, 30, 0), (0, 0, 0))}


def _flat(a, b):
    return np.concatenate([a.ravel(), b.ravel()])


@gpu
@pytest.mark.parametrize("name", list(CASES) + list(LONG))
def test_against_oracle_and_reference(product_lib, cuda_device, name):
    case = CASES.get(name) or LONG[name]
    kind, num, size, ty, t1, t2, seed = case
    n = size if kind == "swt" else 1 << size
    got = _flat(*W.run(product_lib, kind, num, size, ty, t1, t2, W.signal(n, seed)))
    want = oracle(*case)
    scale = np.abs(want).max()
    assert np.abs(got - want).max() <= TOL * scale, name
    ref = ref_lib_or_none()
    if ref is not None:
        r = _flat(*W.run(ref, kind, num, size, ty, t1, t2, W.signal(n, seed)))
        assert np.abs(got - r).max() <= TOL * scale, name


def _legacy(kind, num, size, x):
    lib = af.lib.get_lib()
    return np.stack([_flat(*W.run(lib, kind, num, size, 2, 4, 0, c)) for c in x])


@gpu
@pytest.mark.parametrize("kind,num,size,batch", [("wpt", 6, 12, 80), ("dwt", 11, 12, 400), ("swt", 8, 1 << 14, 140)])
def test_batch_equals_legacy(cuda_device, kind, num, size, batch):
    """host pointers: more than one 64 MB staging chunk; device pointers: one call; both bit for bit per clip"""
    import torch
    n = size if kind == "swt" else 1 << size
    rng = np.random.default_rng(3)
    x = rng.standard_normal((batch, n)).astype(np.float32)
    obj = {"dwt": af.DWT, "wpt": af.WPT}[kind](num=num, radix2_exp=size) if kind != "swt" else af.SWT(num, n)
    call = getattr(obj, f"{kind}_batch")
    rows = (num if kind == "dwt" else 1 << num) if kind != "swt" else num
    assert batch * rows * n * 4 > 64 << 20
    host = np.concatenate([a.reshape(batch, -1) for a in call(x)], axis=1)
    dev = torch.cat([a.reshape(batch, -1) for a in call(torch.from_numpy(x).cuda())], dim=1)
    torch.cuda.synchronize()
    assert np.array_equal(host, dev.cpu().numpy())
    pick = [0, batch // 2, batch - 1]
    assert np.array_equal(host[pick], _legacy(kind, num, size, x[pick]))


def _planes(obj, kind, x, rows, n, offset):
    """coef and mData of one device call whose mData starts `offset` floats into a 7.0-filled buffer (None: NULL
    mData), each with a 64-float 7.0 tail behind it -> (coef buffer, mData buffer or None)"""
    import torch
    b = x.shape[0]
    coef = torch.full((b * n + 64,), 7.0, device="cuda")
    m = None if offset is None else torch.full((offset + b * rows * n + 64,), 7.0, device="cuda")
    fn = getattr(obj._lib, f"{kind}Obj_{kind}Batch")
    mp = None if m is None else C.c_void_p(m.data_ptr() + 4 * offset)
    assert fn(obj._obj, dptr(x), b, dptr(coef), mp, 1, stream()) == 0
    torch.cuda.synchronize()
    return coef, m


@gpu
@pytest.mark.parametrize("kind", ["dwt", "wpt"])
def test_null_m_data_writes_only_coef(cuda_device, kind):
    """mDataArr = NULL: coefArr as with mDataArr, nothing written past it; a following call with mDataArr still writes
    it as a fresh object does"""
    import torch
    n, num, b = 1 << 10, 5, 4
    rows = num if kind == "dwt" else 1 << num
    x = torch.from_numpy(W.signal(n * b, 2).reshape(b, n)).cuda()
    mk = lambda: af.DWT(num=num, radix2_exp=10) if kind == "dwt" else af.WPT(num=num, radix2_exp=10)  # noqa: E731
    full_coef, full_m = getattr(mk(), f"{kind}_batch")(x)
    obj = mk()
    coef, _ = _planes(obj, kind, x, rows, n, None)
    assert torch.equal(coef[:b * n].view(b, n), full_coef) and bool((coef[b * n:] == 7.0).all())
    coef2, m2 = _planes(obj, kind, x, rows, n, 0)
    assert torch.equal(coef2[:b * n].view(b, n), full_coef)
    assert torch.equal(m2[:b * rows * n].view(b, rows, n), full_m) and bool((m2[b * rows * n:] == 7.0).all())


@gpu
@pytest.mark.parametrize("kind", ["dwt", "wpt"])
@pytest.mark.parametrize("offset", [1, 2, 3])
def test_m_data_not_16_byte_aligned(cuda_device, kind, offset):
    """a device mDataArr that is float-aligned but not 16-byte aligned gets the same rows as an aligned one, and the
    floats before and after it stay untouched"""
    import torch
    n, num, b = 1 << 9, 4, 3
    rows = num if kind == "dwt" else 1 << num
    x = torch.from_numpy(W.signal(n * b, 6).reshape(b, n)).cuda()
    obj = af.DWT(num=num, radix2_exp=9) if kind == "dwt" else af.WPT(num=num, radix2_exp=9)
    _, aligned = _planes(obj, kind, x, rows, n, 0)
    _, shifted = _planes(obj, kind, x, rows, n, offset)
    assert torch.equal(shifted[offset:offset + b * rows * n], aligned[:b * rows * n])
    assert bool((shifted[:offset] == 7.0).all()) and bool((shifted[offset + b * rows * n:] == 7.0).all())


@gpu
def test_reference_python_classes_on_b200(raf, cuda_device):
    """the reference's own SWT, WPT and DWT (which always builds sym4) give on this library what they give on the
    reference build, within the tolerance; this package's classes give the same arrays as the legacy calls"""
    x = W.signal(4096 * 3, 4).reshape(3, 4096)
    res = {}
    for which in ("ref", "b200"):
        raf.fftlib.set_fft_lib(lib_ext="b200" if which == "b200" else None)
        s = raf.SWT(num=5, fft_length=4096, wavelet_type=raf.type.WaveletDiscreteType.DB, t1=4, t2=0)
        w = raf.WPT(num=5, radix2_exp=12, wavelet_type=raf.type.WaveletDiscreteType.SYM, t1=4, t2=0)
        d = raf.DWT(num=11, radix2_exp=12, wavelet_type=raf.type.WaveletDiscreteType.DB, t1=4, t2=0)
        res[which] = [np.concatenate([a.ravel() for a in o]) for o in (s.swt(x), w.wpt(x), d.dwt(x[0]))]
    raf.fftlib.set_fft_lib(None)
    for g, r in zip(res["b200"], res["ref"]):
        assert np.abs(g - r).max() <= TOL * np.abs(r).max()
    own = af.DWT(num=11, radix2_exp=12)       # sym4: what the reference's DWT computes
    c, m = own.dwt(x[0])
    assert np.array_equal(np.concatenate([c.ravel(), m.ravel()]), res["b200"][2])


@gpu
def test_ctor_refusal_and_python_shapes(cuda_device):
    with pytest.raises(ValueError, match="not supported"):
        af.WPT(num=3, radix2_exp=8, wavelet_type=af.WaveletDiscreteType.DMEY)
    d = af.DWT(num=4, radix2_exp=8)
    c, m = d.dwt(np.zeros((2, 3, 256), np.float32))
    assert c.shape == (2, 3, 256) and m.shape == (2, 3, 4, 256) and d.y_coords().shape == (5,)
    a1, a2 = af.SWT(3, 96).swt(np.ones(96, np.float32))
    assert a1.shape == a2.shape == (3, 96)

