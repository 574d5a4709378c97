"""The discrete wavelet kernels of wavelet.cu level by level and element by element against float64 oracles, and every
mDataArr row bit for bit.

k_wavelet_level (DWT and WPT) and k_swt_level run once per level, so a wrong level is wrong only on its own rows, which
can sit far below the tensor's maximum: on a smooth clip the finest DWT details cancel to ~1e-8 of the approximation.
So each level is fed the exact float32 input it consumed, and every output element is held to 1e-4 of its own scale,
sum_j |h_j| |x[idx_j]| over its taps (h = loD for approximations, hiD for details), plus dec subnormal ulps where that
scale underflows float32; elements whose scale is 0 must be exactly 0.  The float64 steps (_wavelet_oracle.level,
wpt_level, swt_level) read the unpadded input with the kernels' modulo indexing; tests/test_wavelet_cpu.py pins them
against the literal padding and convolution.

Where each level's input comes from:
  - DWT: level k reads coef[: n >> k] of a num = k run (the clip for k = 0) and writes coef[: n >> k] of a num = k + 1
    run.  The levels below k run the same kernels on the same data, so that input is exactly what the num = k + 1 run
    consumed; the details of every level below k must be bit-identical between the two runs, which pins that premise
    and the coef layout;
  - WPT: level k reads the coef of a num = k run (2^k nodes of n >> k samples) and writes the coef of a num = k + 1
    run, the children of the even non-zero nodes swapped;
  - SWT: row i reads approximation row i - 1 of the same call (the clip for i = 0) at dilation 2^i.
On the white-noise clips every row of at least MIN_ROW samples (a DWT detail level, the final approximation, a WPT
node, an SWT row) is also held end to end to 1e-4 of its own max |want| against the whole float64 transform.  Shorter
rows are left to the per-element bar: a 2-sample WPT leaf of white noise can peak at 2e-6 of the clip's rms (2^20,
num 19) while it inherits rounding from 19 levels of ancestors, so no float32 pipeline meets that bar there.

mDataArr, a copy of coefficients, must equal coef through _wavelet_oracle.m_data_index bit for bit, on the 16-byte
store path (dwt_batch / wpt_batch) and on the 4-byte one (the raw entry at 1, 2 and 3 floats past a 16-byte boundary),
with guard floats on both sides untouched.  Every call asserts its launches: num levels, plus one k_wavelet_expand
when mDataArr is requested.  Every call runs the four clips of _wavelet_oracle.level_clips.  The run prints the worst
element per case.
"""
import ctypes as C

import numpy as np
import pytest

import _wavelet_oracle as W
from _parity_kit import count_launches, dptr, stream
from test_wavelet_cpu import LEVEL_CASES, TABLE

import audioflux_b200 as af

gpu = pytest.mark.gpu

TOL = 1e-4
MIN_ROW = 16
TINY = 2.0 ** -149             # the smallest float32 subnormal
NORMAL = 1e-30                 # scales from here up report their worst element: far above float32's subnormals
GUARD = 16                     # guard floats before a raw mDataArr: 64 bytes, so its offset sets its alignment


@pytest.fixture
def report(request, capsys):
    """report(case, what, worst): prints a case's worst relative error past pytest's capture and records it"""
    def emit(case, what, worst):
        request.node.user_properties.append((f"{case} {what}", worst))     # (name, value), as junitxml reads them
        with capsys.disabled():
            print(f"\n    {case} {what}: {worst:.2e}", end="")
    return emit


def check_elems(case, got, want, scale, dec):
    """every element within TOL of its own scale plus dec float32 underflows (dec * TINY: an impulse through db30 leaves
    subnormal tails, where float32 keeps no relative precision), zero-scale elements exactly 0 -> worst |got - want| /
    scale over the elements of normal scale"""
    got, want, scale = (np.asarray(a, np.float64) for a in (got, want, scale))
    assert got.shape == want.shape == scale.shape, (case, got.shape, want.shape)
    assert np.isfinite(got).all(), (case, "non-finite output")
    err = np.abs(got - want)
    live = scale > 0
    over = live & (err > TOL * scale + dec * TINY)
    bad = np.argwhere(over)
    assert bad.size == 0, (case, "elements above their own scale", bad[:10].tolist(),
                           (err[over] / scale[over])[:10].tolist())
    assert (got[~live] == 0).all(), (case, "zero-scale elements not zero",
                                     np.argwhere(~live & (got != 0))[:10].tolist())
    normal = scale >= NORMAL
    return float((err[normal] / scale[normal]).max()) if normal.any() else 0.0


def check_rows(case, got, want):
    """got, want [..., width]: every row of at least MIN_ROW samples within TOL of its own max |want| -> worst"""
    if got.shape[-1] < MIN_ROW:
        return 0.0
    got, want = (np.asarray(a, np.float64).reshape(-1, got.shape[-1]) for a in (got, want))
    rel = np.abs(got - want).max(-1) / np.abs(want).max(-1)
    assert (rel <= TOL).all(), (case, "rows above their own max", np.argwhere(rel > TOL).ravel()[:10].tolist(),
                                rel.max())
    return float(rel.max())


def _tree(kind, num, e, key):
    ty, t1, t2 = key
    return (af.DWT if kind == "dwt" else af.WPT)(num=num, radix2_exp=e, wavelet_type=ty, t1=t1, t2=t2)


def run_tree(lib, kind, num, e, key, x, m_data):
    """(coef, mData or None) as numpy of dwt_batch / wpt_batch on the device clips x, a fresh object; asserts the call's
    launches"""
    obj, out = _tree(kind, num, e, key), []
    launches = count_launches(lib, lambda: out.append(getattr(obj, f"{kind}_batch")(x, m_data)), warm=True)
    assert launches == num + bool(m_data), (kind, num, e, launches)
    coef, m = out[-1]
    return coef.cpu().numpy(), None if m is None else m.cpu().numpy()


def _names(kind):
    return [k for k, c in LEVEL_CASES.items() if c[0] == kind]


@gpu
@pytest.mark.parametrize("name", _names("dwt"))
def test_dwt_levels(product_lib, cuda_device, report, name):
    import torch
    _, num, e, key, m_data = LEVEL_CASES[name]
    lo, hi = TABLE[key]
    n = 1 << e
    x = W.level_clips(n, e)
    xd = torch.from_numpy(x).cuda()
    prev, worst = x, 0.0
    for k in range(num):
        coef, m = run_tree(product_lib, "dwt", k + 1, e, key, xd, m_data and k == num - 1)
        L = n >> k
        assert np.array_equal(coef[:, L:], prev[:, L:]), (name, k, "details of the levels below differ")
        a, d, sa, sd = W.level(prev[:, :L], lo, hi)
        worst = max(worst, check_elems(f"{name} level {k}", coef[:, :L], np.concatenate([a, d], -1),
                                       np.concatenate([sa, sd], -1), len(lo)))
        prev = coef
    report(name, "k_wavelet_level worst element", worst)
    want = W.dwt_fast(x[W.NOISE], num, lo, hi)
    rows = [(0, n >> num)] + [(n >> (k + 1), n >> k) for k in range(num)]
    report(name, "end to end worst row",
           max(check_rows(f"{name} row {r}", coef[W.NOISE, a:b], want[:, a:b]) for r, (a, b) in enumerate(rows)))
    if m_data:
        assert np.array_equal(m, coef[:, W.m_data_index(n, num, "dwt")]), name


@gpu
@pytest.mark.parametrize("name", _names("wpt"))
def test_wpt_levels(product_lib, cuda_device, report, name):
    import torch
    _, num, e, key, m_data = LEVEL_CASES[name]
    lo, hi = TABLE[key]
    n = 1 << e
    x = W.level_clips(n, e)
    xd = torch.from_numpy(x).cuda()
    prev, worst = x, 0.0
    for k in range(num):
        coef, m = run_tree(product_lib, "wpt", k + 1, e, key, xd, m_data and k == num - 1)
        want, scale = W.wpt_level(prev, k, lo, hi)
        worst = max(worst, check_elems(f"{name} level {k}", coef, want, scale, len(lo)))
        prev = coef
    report(name, "k_wavelet_level worst element", worst)
    want = W.wpt_fast(x[W.NOISE], num, lo, hi)
    rows = (2, 1 << num, n >> num)
    report(name, "end to end worst row", check_rows(name, coef[W.NOISE].reshape(rows), want.reshape(rows)))
    if m_data:
        assert np.array_equal(m, coef[:, W.m_data_index(n, num, "wpt")]), name


@gpu
@pytest.mark.parametrize("name", _names("swt"))
def test_swt_levels(product_lib, cuda_device, report, name):
    import torch
    _, num, n, key, _ = LEVEL_CASES[name]
    ty, t1, t2 = key
    lo, hi = TABLE[key]
    x = W.level_clips(n, n)
    xd = torch.from_numpy(x).cuda()
    obj, out = af.SWT(num, n, wavelet_type=ty, t1=t1, t2=t2), []
    assert count_launches(product_lib, lambda: out.append(obj.swt_batch(xd)), warm=True) == num
    a, d = (t.cpu().numpy() for t in out[-1])
    worst = 0.0
    for i in range(num):
        wa, wd, sa, sd = W.swt_level(x if i == 0 else a[:, i - 1], 1 << i, lo, hi)
        worst = max(worst, check_elems(f"{name} row {i}", np.stack([a[:, i], d[:, i]]), np.stack([wa, wd]),
                                       np.stack([sa, sd]), len(lo)))
    report(name, "k_swt_level worst element", worst)
    wa, wd = W.swt_fast(x[W.NOISE], num, lo, hi)
    report(name, "end to end worst row",
           check_rows(name, np.stack([a[W.NOISE], d[W.NOISE]]), np.stack([wa, wd])))


@gpu
def test_swt_num_0_leaves_outputs_untouched(product_lib, cuda_device):
    """num = 0: no launch, and neither output plane is written, with device or host pointers"""
    import torch
    n = 96
    obj = af.SWT(0, n)
    x = torch.from_numpy(W.level_clips(n, 0)).cuda()
    m1, m2 = (torch.full((4 * n,), 7.0, device="cuda") for _ in range(2))
    rc = []
    fn = product_lib.swtObj_swtBatch
    call = lambda: rc.append(fn(obj._obj, dptr(x), 4, dptr(m1), dptr(m2), 1, stream()))  # noqa: E731
    assert count_launches(product_lib, call, warm=True) == 0 and rc == [0, 0]
    assert bool((m1 == 7.0).all()) and bool((m2 == 7.0).all())
    h1, h2 = np.full(n, 7.0, np.float32), np.full(n, 7.0, np.float32)
    xh = np.ascontiguousarray(W.level_clips(n, 0)[0])
    product_lib.swtObj_swt(obj._obj, *(a.ctypes.data_as(C.c_void_p) for a in (xh, h1, h2)))
    assert (h1 == 7.0).all() and (h2 == 7.0).all()
    a1, a2 = obj.swt_batch(x)
    assert a1.shape == a2.shape == (4, 0, n)


@gpu
@pytest.mark.parametrize("kind", ["dwt", "wpt"])
@pytest.mark.parametrize("e,num", [(2, 1), (3, 1), (3, 2), (20, 3)])
def test_m_data_both_store_paths(product_lib, cuda_device, kind, e, num):
    """log2n 2 (one float4 per row), 3 and 20: the aligned 16-byte stores of dwt_batch / wpt_batch and the 4-byte stores
    at offsets of 1, 2 and 3 floats (the raw *Batch entry) both give coef through the index map bit for bit, and leave
    the guard floats before and after mDataArr untouched"""
    import torch
    n = 1 << e
    rows = num if kind == "dwt" else 1 << num
    size = 4 * rows * n
    x = torch.from_numpy(W.level_clips(n, e)).cuda()
    obj = _tree(kind, num, e, W.SYM4)
    out = []
    assert count_launches(product_lib, lambda: out.append(getattr(obj, f"{kind}_batch")(x)), warm=True) == num + 1
    coef, m = out[-1]
    assert m.data_ptr() % 16 == 0
    coef = coef.cpu().numpy()
    want = coef[:, W.m_data_index(n, num, kind)]
    assert np.array_equal(m.cpu().numpy(), want), (kind, e, num)
    fn = getattr(product_lib, f"{kind}Obj_{kind}Batch")
    for offset in (1, 2, 3):
        c2 = torch.empty((4, n), device="cuda")
        buf = torch.full((GUARD + offset + size + 64,), 7.0, device="cuda")
        assert buf.data_ptr() % 64 == 0
        mp = C.c_void_p(buf.data_ptr() + 4 * (GUARD + offset))
        rc = []
        call = lambda: rc.append(fn(obj._obj, dptr(x), 4, dptr(c2), mp, 1, stream()))  # noqa: E731
        assert count_launches(product_lib, call, warm=True) == num + 1 and rc == [0, 0]
        got = buf.cpu().numpy()
        assert np.array_equal(c2.cpu().numpy(), coef), (kind, e, num, offset)
        assert np.array_equal(got[GUARD + offset:GUARD + offset + size], want.ravel()), (kind, e, num, offset)
        assert (got[:GUARD + offset] == 7.0).all() and (got[GUARD + offset + size:] == 7.0).all(), (kind, e, offset)
