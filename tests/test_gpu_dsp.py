"""Cross-correlation and the chirp z-transform on the GPU: every oracle case through xcorrObj_xcorr / cztObj_czt against
the float64 oracle and the reference build (its stored outputs where it is not built), within 1e-4 of the row's max
|want|, the Xcorr index equal to the reference's unless the values at both indices are within that bar; every transform
length 2^1 .. 2^20 row by row, both sides of the switch to the long path; the batch bit-identical to the legacy call
with host pointers across staging chunks and with device pointers back to back around a CZT table change; the CZT
tables and the long Xcorr workspace ordered across streams (busy caller streams, the host-pointer pipeline's own
stream, a second stream); every call as on a fresh object; one launch per chunk (plus one per CZT table change); and the
reference's own Xcorr and CZT classes on libaudioflux_b200.so."""
import ctypes as C
import warnings

import numpy as np
import pytest

import _dsp_oracle as D
from _parity_kit import Out, count_launches, dptr, raf, run_batch, stream  # noqa: F401  (raf: a fixture)
from test_dsp_cpu import CZ, GOLD, XC, _scale, check_xcorr

import audioflux_b200 as af

TOL = 1e-4                 # of max |want| of the row
gpu = pytest.mark.gpu


def _stored(name):
    """the reference's output of a case: live from the build, else from the golden file, else None"""
    v = GOLD.outputs({name}).get(name)
    return (v[:-2], v[-2], int(v[-1])) if v is not None and name in XC else v


@gpu
@pytest.mark.parametrize("name", list(XC))
def test_xcorr_case(product_lib, cuda_device, name):
    got, gv, gi = D.c_xcorr_case(product_lib, name, XC[name])
    assert product_lib.afb200_lastError() in (b"", None)
    want, wv, wi = D.xcorr_case(name, XC[name])
    check_xcorr(got, gv, gi, want, wv, wi, (name, "oracle"), TOL, exact_index=False)
    ref = _stored(name)
    if ref is not None:
        check_xcorr(got, gv, gi, ref[0].astype(np.float64), ref[1], ref[2], (name, "reference"), TOL, exact_index=False)


@gpu
@pytest.mark.parametrize("name", list(CZ))
def test_czt_case(product_lib, cuda_device, name):
    got = D.c_czt_case(product_lib, name, CZ[name])
    want = D.czt_case(name, CZ[name])
    for half, what in ((slice(0, want.size // 2), "head"), (slice(want.size // 2, None), "tail")):
        err = np.abs(got[half] - want[half]).max() / _scale(want[half])
        assert err <= TOL, (name, what, "oracle", err)
    ref = _stored(name)
    if ref is not None:
        assert np.abs(got - ref).max() <= TOL * _scale(ref), (name, "reference")


@gpu
def test_czt_band_sequence(product_lib, cuda_device):
    """valid, invalid (the tables stay), valid (rebuilt) on one object, against the oracle"""
    for r in (3, 10, 13):
        x = np.random.default_rng(r).standard_normal(1 << r).astype(np.float32)
        got = D.c_czt_sequence(product_lib, r, x)
        for g, w in zip(got, D.czt_sequence_oracle(r, x)):
            assert np.abs(g - w).max() <= TOL * _scale(w), r
        assert np.array_equal(got[0], got[1])


def _rows(n, seed):
    """3 rows: noise, the middle one 1000 times louder and reversed"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((3, n)).astype(np.float32)
    x[1] = 1000 * x[1, ::-1]
    return x


@gpu
def test_every_transform_length(product_lib, cuda_device):
    """M = 2^1 .. 2^20 (n = M/2, and n = M/2 - 1 from M = 4), cross with Coeff and auto without, row by row"""
    x = af.Xcorr()
    for k in range(1, 21):
        for n in sorted({(1 << k) // 2, max(1, (1 << k) // 2 - 1)}):
            if n < 1 or (n == (1 << k) // 2 - 1 and k < 2):
                continue
            a, b = _rows(n, k), _rows(n, 100 + k)
            for bb, norm in ((b, af.XcorrNormalType.COEFF), (None, af.XcorrNormalType.NONE)):
                arr, mv, idx = x.xcorr_batch(a, bb, norm)
                for r in range(3):
                    want, wv, wi = D.xcorr(a[r], None if bb is None else bb[r], norm.value)
                    check_xcorr(arr[r], mv[r], int(idx[r]), want, wv, wi, (k, n, r, bb is None), TOL, exact_index=False)


def _xcorr_batch_c(lib, o, a, b, norm, device):
    B, n = a.shape
    outs = Out(np.full((B, 2 * n - 1), 7.0, np.float32)), Out(np.full(B, 7.0, np.float32)), Out(np.full(B, 7, np.int32))
    return run_batch(lib, "xcorrObj_xcorrBatch", (o, a, b, n, B, C.byref(C.c_int(norm)), *outs), device)


def _same_as_legacy(lib, res, a, b, norm, rows):
    out, mv, ix = res
    for r in rows:
        v, m, i = D.c_xcorr(lib, a[r], None if b is None else b[r], norm)
        assert np.array_equal(out[r], v, equal_nan=True) and ix[r] == i, r
        assert np.array_equal(mv[r], np.float32(m), equal_nan=True), r


@gpu
def test_xcorr_batch_equals_legacy(product_lib, cuda_device):
    """host pointers across three staging chunks (4100 pairs of 4096 samples, 2032 per chunk) and device pointers; the
    long path across two workspace groups (14 pairs of 2^19 samples)"""
    o = C.c_void_p()
    assert product_lib.xcorrObj_new(C.byref(o)) == 0
    rng = np.random.default_rng(3)
    a = rng.standard_normal((4100, 4096)).astype(np.float32)
    b = rng.standard_normal((4100, 4096)).astype(np.float32)
    a[7] = 0.0                                             # a silent row: NaN lags with Coeff
    host = _xcorr_batch_c(product_lib, o, a, b, 1, False)
    _same_as_legacy(product_lib, host, a, b, 1, (0, 7, 2031, 2032, 4063, 4064, 4099))
    dev = _xcorr_batch_c(product_lib, o, a[:300], None, 0, True)
    _same_as_legacy(product_lib, dev, a[:300], None, 0, (0, 7, 299))
    a = rng.standard_normal((14, 1 << 19)).astype(np.float32)
    b = rng.standard_normal((14, 1 << 19)).astype(np.float32)
    for dv in (False, True):
        res = _xcorr_batch_c(product_lib, o, a, b, 1, dv)
        _same_as_legacy(product_lib, res, a, b, 1, (0, 11, 12, 13))
    product_lib.xcorrObj_free(o)


def _czt_batch_c(lib, o, re, im, band):
    """cztObj_cztBatch with host pointers -> (real, imaginary) numpy [B, 2N]"""
    B, N = (re if re is not None else im).shape
    return run_batch(lib, "cztObj_cztBatch", (o, re, im, B, *band, Out(np.full((B, 2 * N), 7.0, np.float32)),
                                              Out(np.full((B, 2 * N), 7.0, np.float32))), False)


@gpu
def test_czt_batch_equals_legacy(product_lib, cuda_device):
    """host pointers across three staging chunks (9000 rows of 2^10, 4096 per chunk); device pointers queued back to
    back on one stream around table changes and an invalid band, compared after one synchronise"""
    import torch
    rng = np.random.default_rng(4)
    r, N = 10, 1 << 10
    st, o = D.c_czt_new(product_lib, r)
    st2, leg = D.c_czt_new(product_lib, r)
    re = rng.standard_normal((9000, N)).astype(np.float32)
    im = rng.standard_normal((9000, N)).astype(np.float32)
    band = (0.15, 0.25)
    hr, hi = _czt_batch_c(product_lib, o, re, im, band)
    for k in (0, 4095, 4096, 8191, 8192, 8999):
        want = D.c_czt(product_lib, leg, re[k], im[k], *band, N)
        assert np.array_equal(hr[k], want.real.astype(np.float32)) and np.array_equal(hi[k], want.imag.astype(np.float32)), k
    calls = []
    for band, (x, y) in (((0.0, 1.0), (re[:50], None)), ((0.01, 0.02), (None, im[:70])), ((0.3, 0.2), (re[:5], im[:5])),
                         ((0.0, 0.5), (re[:40], im[:40])), ((0.0, 1.0), (re[:3], None))):
        B = (x if x is not None else y).shape[0]
        keep = [None if v is None else torch.from_numpy(v).cuda() for v in (x, y)]
        o3 = [torch.full((B, 2 * N), 7.0, device="cuda") for _ in range(2)]
        rc = product_lib.cztObj_cztBatch(o, *(None if t is None else dptr(t) for t in keep), B, *band, dptr(o3[0]),
                                         dptr(o3[1]), 1, stream())
        assert rc == 0, product_lib.afb200_lastError()
        calls.append((band, x, y, o3, keep))
    torch.cuda.synchronize()
    for band, x, y, o3, _ in calls:
        B = (x if x is not None else y).shape[0]
        for k in (0, B - 1):
            want = D.c_czt(product_lib, leg, None if x is None else x[k], None if y is None else y[k], *band, N)
            assert np.array_equal(o3[0][k].cpu().numpy(), want.real.astype(np.float32)), (band, k)
            assert np.array_equal(o3[1][k].cpu().numpy(), want.imag.astype(np.float32)), (band, k)
    product_lib.cztObj_free(o)
    product_lib.cztObj_free(leg)


def _on(stream_obj):
    return C.c_void_p(stream_obj.cuda_stream)


@gpu
def test_czt_tables_ordered_across_streams(product_lib, cuda_device):
    """the object's first use and a band change queued on a stream busy for about 100 ms, then calls with the same band
    on the host-pointer pipeline's own stream and on a second stream; then a band change from the host while launches
    on two other streams still read the old tables.  Every result equals a legacy object's bit for bit."""
    import torch
    lib, r, N, B = product_lib, 12, 1 << 12, 64
    rng = np.random.default_rng(21)
    x = rng.standard_normal((B, N)).astype(np.float32)
    st, o = D.c_czt_new(lib, r)
    st2, leg = D.c_czt_new(lib, r)
    xd = torch.from_numpy(x).cuda()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    outs = [[torch.full((B, 2 * N), 7.0, device="cuda") for _ in range(2)] for _ in range(4)]
    torch.cuda.synchronize()
    A, Bd = (0.1, 0.2), (0.3, 0.4)

    def dev(k, band, s):
        rc = lib.cztObj_cztBatch(o, dptr(xd), None, B, *band, dptr(outs[k][0]), dptr(outs[k][1]), 1, _on(s))
        assert rc == 0, lib.afb200_lastError()

    with torch.cuda.stream(s1):
        torch.cuda._sleep(200_000_000)
    dev(0, A, s1)                                          # first use + band A, behind the busy stream
    h1r, h1i = _czt_batch_c(lib, o, x, None, A)            # same band, the pipeline's stream
    dev(1, A, s2)                                          # same band, a second stream
    with torch.cuda.stream(s2):
        torch.cuda._sleep(200_000_000)
    dev(2, A, s2)                                          # still reading band A long after ...
    dev(3, A, s1)                                          # ... this one, the last launch on the object
    h2r, h2i = _czt_batch_c(lib, o, x, None, Bd)           # band B overwrites the tables
    torch.cuda.synchronize()
    for k in (0, B - 1):
        wa = D.c_czt(lib, leg, x[k], None, *A, N)
        for got in [(h1r[k], h1i[k])] + [(t[0][k].cpu().numpy(), t[1][k].cpu().numpy()) for t in outs]:
            assert np.array_equal(got[0], wa.real.astype(np.float32)) and np.array_equal(got[1], wa.imag.astype(np.float32)), k
        wb = D.c_czt(lib, leg, x[k], None, *Bd, N)
        assert np.array_equal(h2r[k], wb.real.astype(np.float32)) and np.array_equal(h2i[k], wb.imag.astype(np.float32)), k
    lib.cztObj_free(o)
    lib.cztObj_free(leg)


@gpu
def test_xcorr_long_workspace_across_streams(product_lib, cuda_device):
    """the long path's workspace, kept by the object, shared by a call queued on a busy stream, a host-pointer call, a
    call on a second stream and a larger call that grows the workspace; each equal to a legacy call bit for bit"""
    import torch
    lib, n = product_lib, (1 << 18) + 5
    rng = np.random.default_rng(22)
    a = rng.standard_normal((4, 3, n)).astype(np.float32)
    b = rng.standard_normal((4, 3, n)).astype(np.float32)
    o = C.c_void_p()
    assert lib.xcorrObj_new(C.byref(o)) == 0
    ad, bd = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    outs = [torch.full((3, 2 * n - 1), 7.0, device="cuda") for _ in range(3)]
    idx = [torch.full((3,), 7, dtype=torch.int32, device="cuda") for _ in range(3)]
    torch.cuda.synchronize()

    def dev(k, s):
        rc = lib.xcorrObj_xcorrBatch(o, dptr(ad[k]), dptr(bd[k]), n, 3, C.byref(C.c_int(1)), dptr(outs[k]), None,
                                     dptr(idx[k]), 1, _on(s))
        assert rc == 0, lib.afb200_lastError()

    with torch.cuda.stream(s1):
        torch.cuda._sleep(200_000_000)
    dev(0, s1)
    host = _xcorr_batch_c(lib, o, np.ascontiguousarray(a[1]), np.ascontiguousarray(b[1]), 1, False)
    dev(2, s2)
    big_a = rng.standard_normal((20, n)).astype(np.float32)    # more pairs: a larger workspace
    big = _xcorr_batch_c(lib, o, big_a, None, 0, False)
    torch.cuda.synchronize()
    for k, (res_out, res_idx) in ((0, (outs[0], idx[0])), (2, (outs[2], idx[2]))):
        got = res_out.cpu().numpy(), None, res_idx.cpu().numpy()
        for r in (0, 2):
            v, _, i = D.c_xcorr(lib, a[k, r], b[k, r], 1)
            assert np.array_equal(got[0][r], v) and got[2][r] == i, (k, r)
    _same_as_legacy(lib, host, a[1], b[1], 1, (0, 2))
    _same_as_legacy(lib, big, big_a, None, 0, (0, 19))
    lib.xcorrObj_free(o)


@gpu
def test_xcorr_calls_are_fresh(product_lib, cuda_device):
    """1000 samples, then 900 on the same object (the same transform length): the second call is np.correlate of its own
    inputs (the reference's object gives 0.51 relative error there)"""
    x = af.Xcorr()
    rng = np.random.default_rng(9)
    a1, b1 = rng.standard_normal((2, 1000)).astype(np.float32)
    a2, b2 = rng.standard_normal((2, 900)).astype(np.float32)
    x.xcorr(a1, b1)
    got, _ = x.xcorr(a2, b2)
    want = np.correlate(a2.astype(np.float64), b2.astype(np.float64), "full")
    assert np.abs(got - want).max() <= TOL * np.abs(want).max()
    o = C.c_void_p()
    assert product_lib.xcorrObj_new(C.byref(o)) == 0
    for a, b in ((a1, b1), (a2, b2)):
        out = np.empty(2 * a.size - 1, np.float32)
        product_lib.xcorrObj_xcorr(o, a.ctypes.data, b.ctypes.data, a.size, C.byref(C.c_int(0)), out.ctypes.data, None)
    want = np.correlate(a2.astype(np.float64), b2.astype(np.float64), "full")
    assert np.abs(out - want).max() <= TOL * np.abs(want).max()
    product_lib.xcorrObj_free(o)


@gpu
def test_launch_count(product_lib, cuda_device):
    """k_xcorr: one launch per staging chunk; k_czt: one per chunk, plus k_czt_filter once per table change"""
    import torch
    x = af.Xcorr()
    a = np.random.default_rng(1).standard_normal((8, 4096)).astype(np.float32)
    ad = torch.from_numpy(a).cuda()
    assert count_launches(product_lib, lambda: x.xcorr_batch(ad, ad), warm=True) == 1
    assert count_launches(product_lib, lambda: x.xcorr(a[0]), warm=True) == 1
    big = np.random.default_rng(2).standard_normal((4100, 4096)).astype(np.float32)
    assert count_launches(product_lib, lambda: x.xcorr_batch(big), warm=True) == 3
    c = af.CZT(10)
    z = np.random.default_rng(3).standard_normal((8, 1024)).astype(np.float32)
    zd = torch.from_numpy(z).cuda()
    assert count_launches(product_lib, lambda: c.czt_batch(zd, 0.0, 1.0), warm=False) == 2   # first call: H
    assert count_launches(product_lib, lambda: c.czt_batch(zd, 0.0, 1.0), warm=False) == 1
    assert count_launches(product_lib, lambda: c.czt_batch(zd, 0.1, 0.2), warm=False) == 2   # new band
    assert count_launches(product_lib, lambda: c.czt_batch(zd, 0.3, 0.2), warm=False) == 1   # invalid: kept
    zb = np.random.default_rng(4).standard_normal((9000, 1024)).astype(np.float32)
    assert count_launches(product_lib, lambda: c.czt_batch(zb, 0.1, 0.2), warm=False) == 3


@gpu
def test_reference_classes_on_b200(raf, cuda_device):
    """the reference's own Xcorr and CZT classes on the reference build and on libaudioflux_b200.so, and this package's
    classes giving the same arrays"""
    rng = np.random.default_rng(11)
    a, b = rng.standard_normal((2, 3000)).astype(np.float32)
    z = rng.standard_normal((2, 3, 4096)).astype(np.float32)
    res = {}
    for which in ("ref", "b200"):
        raf.fftlib.set_fft_lib(lib_ext="b200" if which == "b200" else None)
        x = raf.Xcorr()
        xt = raf.type.XcorrNormalType
        c = raf.CZT(10)
        res[which] = (x.xcorr(a, b), x.xcorr(a, None, xt.COEFF), c.czt(z[0, 0], 0.15, 0.25), c.czt(z, 0.0, 0.5))
    raf.fftlib.set_fft_lib(None)
    (g1, gv1), (g2, gv2), g3, g4 = res["b200"]
    (r1, rv1), (r2, rv2), r3, r4 = res["ref"]
    w1, wv1, _ = D.xcorr(a, b, 0)
    w2, wv2, _ = D.xcorr(a, None, 1)
    for g, gv, r, rv, w, wv in ((g1, gv1, r1, rv1, w1, wv1), (g2, gv2, r2, rv2, w2, wv2)):
        for v, mv in ((g, gv), (r, rv)):
            assert np.abs(v - w).max() <= TOL * _scale(w) and abs(mv - wv) <= TOL * _scale(w)
    for g, r, x, band in ((g3, r3, z[0, 0], (0.15, 0.25)), (g4[1, 2], r4[1, 2], z[1, 2], (0.0, 0.5))):
        assert g.shape == r.shape == (8192,)
        w = D.czt(x, 10, *band)
        for v in (g, r):
            assert np.abs(v[:2048] - w).max() <= TOL * _scale(w) and not v[2048:].any()
    own = af.Xcorr()
    assert np.array_equal(own.xcorr(a, b)[0], g1) and np.array_equal(own.xcorr(a, None, af.XcorrNormalType.COEFF)[0], g2)
    oc = af.CZT(10)
    assert np.array_equal(oc.czt(z, 0.0, 0.5), g4) and np.array_equal(oc.czt(z[0, 0], 0.15, 0.25), g3)
    with warnings.catch_warnings():                        # numpy's ComplexWarning: czt casts to float32, as the reference
        warnings.simplefilter("ignore")
        assert np.array_equal(oc.czt(z[0, 0] + 1j * z[0, 1], 0.15, 0.25), g3)

