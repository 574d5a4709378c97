"""Harmonic-percussive separation on the GPU: every oracle case through the legacy call (into zeroed and non-zero
buffers, H only, P only) against the float64 oracle and the reference build; the batch bit-identical to the legacy call
into zeroed buffers with host and device pointers, across staging chunks and workspace groups, with neighbouring clips
of very different levels; the launch count; device calls queued back to back on one object; and the reference's own
HPSS class running on libaudioflux_b200.so."""
import numpy as np
import pytest

import _hpss_oracle as HO
from _parity_kit import Out, count_launches, dptr, ref_lib_or_none, run_batch, stream
from _parity_kit import raf  # noqa: F401  (a fixture)

import audioflux_b200 as af

pytestmark = pytest.mark.gpu
TOL = 1e-4          # per output: max|got - want| <= TOL * max|want| where the normaliser is >= 1e-2, 1e-2 elsewhere
CASES = dict(HO.cases())


def _check(got, want, kw, what):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    err, ill = HO.errors(got, want, kw)
    assert err <= TOL and ill <= 1e-2, (what, err, ill)


def _batch(lib, o, x, device, outputs="hp"):
    """hpssObj_hpssBatch on x [batch, n] -> (h, p) numpy [batch, m] (None for a skipped output)"""
    x = np.ascontiguousarray(x, np.float32)
    b, n = x.shape
    m = lib.hpssObj_calDataLength(o, n)
    planes = [Out(np.full((b, m), 7.0, np.float32)) if c in outputs else None for c in "hp"]
    got = iter(run_batch(lib, "hpssObj_hpssBatch", (o, x, n, b, *planes), device))
    return [None if p is None else next(got) for p in planes]


def _legacy(lib, o, x, outputs="hp"):
    m = lib.hpssObj_calDataLength(o, x.size)
    h, p = HO.c_hpss(lib, o, x, outputs)
    assert lib.afb200_lastError() in (b"", None)
    return [None if b is None else b[:m].copy() for b in (h, p)]


def _new(lib, kw):
    st, o = HO.c_new(lib, kw["radix2_exp"], kw.get("window"), 1024, kw.get("h_order"), kw.get("p_order"))
    assert st == 0
    return o


@pytest.mark.parametrize("name", list(CASES))
def test_case_matches_oracle_and_reference(product_lib, cuda_device, name):
    kw = CASES[name]
    got = HO.c_case(product_lib, name, kw)
    assert product_lib.afb200_lastError() in (b"", None)
    want = HO.oracle_case(name, kw)
    ref = ref_lib_or_none()
    refs = HO.c_case(ref, name, kw) if ref is not None else None
    for k in range(2):
        assert (got[k] is None) == (want[k] is None), (name, k)
        if want[k] is None:
            continue
        _check(got[k], want[k], kw, (name, k, "oracle"))
        if refs is not None:
            _check(got[k], refs[k], kw, (name, k, "reference"))
    # the batch, host and device pointers, against the legacy call into zeroed buffers; the second clip is 1000 times
    # louder and reversed, so that a median window reaching into the neighbouring clip would show
    o = _new(product_lib, kw)
    outs = kw.get("outputs", "hp")
    x = HO.case_signal(name, kw)
    clips = np.stack([x, 1000 * x[::-1]])
    legacy = [_legacy(product_lib, o, c, outs) for c in clips]
    for device in (False, True):
        b = _batch(product_lib, o, clips, device, outs)
        for k in range(2):
            if b[k] is None:
                continue
            for c in range(2):
                assert np.array_equal(b[k][c], legacy[c][k]), (name, device, k, c)
    if kw.get("init") is None:
        for k in range(2):
            if want[k] is not None:
                _check(legacy[0][k], want[k], kw, (name, k, "batch oracle"))
    product_lib.hpssObj_free(o)


def test_launch_count(product_lib, cuda_device):
    """per workspace group, up to fftLength 2^14: one STFT, one mask, two per inverse STFT (frames, overlap-add)"""
    import torch
    h = af.HPSS(radix2_exp=11)
    x = (0.1 * np.random.default_rng(1).standard_normal((8, 40000))).astype(np.float32)
    xd = torch.from_numpy(x).cuda()
    assert count_launches(product_lib, lambda: h.hpss_batch(xd), warm=False) == 6
    assert count_launches(product_lib, lambda: h.hpss(x), warm=False) == 6
    o = h._obj
    m = h.cal_data_length(40000)
    out = torch.empty((8, m), device="cuda")
    for ptrs in ((dptr(out), None), (None, dptr(out))):
        call = lambda: product_lib.hpssObj_hpssBatch(o, dptr(xd), 40000, 8, *ptrs, 1, stream())  # noqa: E731
        assert count_launches(product_lib, call, warm=False) == 4


def test_batch_across_chunks_and_groups(product_lib, cuda_device):
    """240 clips of 5 s at 32 kHz: 5 host staging chunks of 48 clips, and on the device more than one workspace group
    (about 10 MB of workspace per clip, at most 2 GB per group); quiet and loud clips alternate"""
    import torch
    h = af.HPSS()
    rng = np.random.default_rng(2)
    n = 160000
    x = np.empty((240, n), np.float32)
    for k in range(240):
        x[k] = HO.case_signal(f"clip{k % 7}", dict(length=n)) * (1000.0 if k % 2 else 0.001)
        x[k] += (0.01 * rng.standard_normal(n)).astype(np.float32)
    host = {}
    launches = count_launches(product_lib, lambda: host.setdefault("o", h.hpss_batch(x)), warm=False)
    assert launches == 6 * 5, launches
    xd = torch.from_numpy(x).cuda()
    dev = {}
    launches = count_launches(product_lib, lambda: dev.setdefault("o", h.hpss_batch(xd)), warm=False)
    assert launches % 6 == 0 and launches >= 12, launches                 # several workspace groups
    for k in range(2):
        assert np.array_equal(dev["o"][k].cpu().numpy(), host["o"][k]), k
    del xd, dev
    for c in (0, 47, 48, 95, 191, 192, 212, 213, 214, 215, 239):
        legacy = _legacy(product_lib, h._obj, x[c])
        for k in range(2):
            assert np.array_equal(host["o"][k][c], legacy[k]), (c, k)
    want = HO.hpss(x[1], 12)
    for k in range(2):
        _check(host["o"][k][1], want[k], dict(radix2_exp=12, length=n), k)


def test_device_calls_back_to_back(product_lib, cuda_device):
    """calls of different lengths and clip counts queued on one object without a synchronise between them"""
    import torch
    h = af.HPSS(radix2_exp=10, h_order=11, p_order=17)
    xs = [np.stack([HO.case_signal(f"b2b{k}{c}", dict(length=n)) for c in range(b)])
          for k, (b, n) in enumerate(((3, 20000), (17, 5000), (2, 60000), (5, 1024)))]
    outs = [h.hpss_batch(torch.from_numpy(x).cuda()) for x in xs]
    torch.cuda.synchronize()
    for x, (hd, pd) in zip(xs, outs):
        for c in (0, len(x) - 1):
            legacy = _legacy(product_lib, h._obj, x[c])
            assert np.array_equal(hd[c].cpu().numpy(), legacy[0]) and np.array_equal(pd[c].cpu().numpy(), legacy[1])


def test_refusals_on_the_device(product_lib, cuda_device):
    import torch
    xd = torch.from_numpy(HO.case_signal("ref", dict(length=5000))).cuda()
    out = torch.full((8192,), 7.0, device="cuda")
    st, o = HO.c_new(product_lib, 13)
    assert product_lib.hpssObj_hpssBatch(o, dptr(xd), 5000, 1, dptr(out), None, 1, stream()) != 0
    assert b"shorter than one frame" in product_lib.afb200_lastError()
    product_lib.hpssObj_free(o)
    st, o = HO.c_new(product_lib, 10, None, None, 21, 401)
    assert product_lib.hpssObj_hpssBatch(o, dptr(xd), 5000, 1, None, dptr(out), 1, stream()) != 0
    assert b"orders up to" in product_lib.afb200_lastError()
    product_lib.hpssObj_free(o)
    torch.cuda.synchronize()
    assert (out == 7.0).all()


def test_reference_classes_on_b200(raf, cuda_device):
    mono = HO.case_signal("mono", dict(length=30000))
    multi = (0.1 * np.random.default_rng(5).standard_normal((2, 3, 9000))).astype(np.float32)
    res = {}
    for which in ("ref", "b200"):
        raf.fftlib.set_fft_lib(lib_ext="b200" if which == "b200" else None)
        a = raf.HPSS(radix2_exp=11, window_type=raf.type.WindowType.HANN, slide_length=512, h_order=13, p_order=19)
        b = raf.HPSS()
        res[which] = [*a.hpss(mono), *a.hpss(multi), *b.hpss(mono)]
    raf.fftlib.set_fft_lib(None)
    a = af.HPSS(radix2_exp=11, window_type=af.WindowType.HANN, slide_length=512, h_order=13, p_order=19)
    b = af.HPSS()
    own = [*a.hpss(mono), *a.hpss(multi), *b.hpss(mono)]
    for k in range(6):
        g, r = res["b200"][k], res["ref"][k]
        assert g.shape == r.shape == own[k].shape, k
        n = g.shape[-1]
        kw = dict(radix2_exp=12 if k >= 4 else 11, length=30000 if k in (0, 1, 4, 5) else 9000,
                  window=None if k >= 4 else HO.W_HANN)
        assert HO.data_length(kw["length"], 1 << kw["radix2_exp"]) == n
        for gr, rr in zip(g.reshape(-1, n), r.reshape(-1, n)):
            _check(gr, rr, kw, k)
        assert np.array_equal(own[k], g), k
