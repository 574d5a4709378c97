"""Harmonic ratio on the GPU: every oracle case through harmonicRatioObj_harmonicRatio against the float64 oracle and the
reference build (within 1e-4 of max |value| of the clip, a frame whose crossing or arg-max the oracle finds undetermined
equal to one of its candidates instead, and the count of such frames capped); the batch bit-identical to the legacy
call with host pointers across staging chunks, with device pointers back to back, and for clips whose carry starts at
frame 0; two launches per chunk; the refusals; and the reference's own HarmonicRatio class on libaudioflux_b200.so."""
import numpy as np
import pytest

import _harmonic_ratio_oracle as HO
from _parity_kit import Out, count_launches, dptr, raf, run_batch, stream  # noqa: F401  (raf: a fixture)
from test_harmonic_ratio_cpu import GOLD

import audioflux_b200 as af

TOL = 1e-4                 # of max |value| of the clip
CASES = dict(HO.cases())
gpu = pytest.mark.gpu
UNDETERMINED = []          # (case, frames) decided by a candidate, reported at the end


def _reference(name):
    return GOLD.outputs({name})[name]


def _check(got, want, cands, what):
    ok, alt = HO.agree(got, want, cands, TOL * max(np.abs(want).max(initial=0.0), 1e-30))
    assert ok, (what, "differs away from an undetermined decision at frame", alt, got[alt], want[alt])
    assert len(alt) <= max(2, len(want) // 10), (what, alt)
    return alt


@gpu
@pytest.mark.parametrize("name", list(CASES))
def test_case_matches_oracle_and_reference(product_lib, cuda_device, name):
    kw = CASES[name]
    got = HO.c_case(product_lib, name, kw)
    assert product_lib.afb200_lastError() in (b"", None)
    want, cands, _ = HO.oracle_case(name, kw)
    alt = _check(got, want, cands, (name, "oracle"))
    ref = _reference(name)
    assert got.shape == ref.shape
    scale = max(np.abs(ref).max(initial=0.0), 1e-30)
    far = np.flatnonzero(~(np.abs(got - ref) <= TOL * scale))
    # where the GPU and the reference differ by more, both must be outcomes the oracle allows
    for t in far:
        assert any(abs(got[t] - c) <= TOL * scale + s for c, s in cands[t]), (name, t, got[t], ref[t])
        assert any(abs(ref[t] - c) <= TOL * scale + s for c, s in cands[t]), (name, t, got[t], ref[t])
    assert len(far) <= max(2, len(want) // 10), (name, far)
    if alt:
        UNDETERMINED.append((name, alt))
    # the batch with host and device pointers: clip 1 is clip 0 reversed and 1000 times louder
    x = HO.case_signal(name, kw)
    xs = np.stack([x, 1000 * x[::-1]])
    st, o = HO.c_new(product_lib, kw["sr"], kw["lf"], kw["r2"], kw["wt"], kw["slide"])
    legacy = [HO.c_ratio(product_lib, o, c) for c in xs]
    assert np.array_equal(legacy[0], got)
    for device in (False, True):
        out = _batch(product_lib, o, xs, device)
        for k in range(2):
            assert np.array_equal(out[k], legacy[k]), (name, device, k)
    product_lib.harmonicRatioObj_free(o)


def _batch(lib, o, x, device, fill=7.0):
    b, n = x.shape
    T = lib.harmonicRatioObj_calTimeLength(o, n)
    return run_batch(lib, "harmonicRatioObj_harmonicRatioBatch",
                     (o, np.ascontiguousarray(x, np.float32), n, b, Out(np.full((b, T), fill, np.float32))), device)[0]


def _clips(n, length, seed, dc_every=3):
    """harmonic tones, noise and, every `dc_every` clips, a DC offset over the first half (carry from frame 0)"""
    rng = np.random.default_rng(seed)
    t = np.arange(length) / 32000
    f0 = rng.uniform(80, 600, (n, 1))
    x = sum(0.3 / h * np.sin(2 * np.pi * f0 * h * t + h) for h in range(1, 5)) + 0.05 * rng.standard_normal((n, length))
    x[::dc_every, :length // 2] = 1.0 + 0.05 * rng.standard_normal((len(x[::dc_every]), length // 2))
    return x.astype(np.float32)


@gpu
def test_batch_across_chunks(product_lib, cuda_device):
    """200 clips of 160 000 samples: three host staging chunks of at most 96 clips; host and device batches equal the
    legacy call, and the clips whose first frames have no crossing start their carry at 0"""
    x = _clips(200, 160000, 1)
    st, o = HO.c_new(product_lib, 32000, 32.703196, 12, None, 1024)
    assert st == 0
    host = _batch(product_lib, o, x, False)
    dev = _batch(product_lib, o, x, True)
    assert np.array_equal(host, dev)
    for c in (0, 1, 95, 96, 97, 191, 192, 199):
        assert np.array_equal(host[c], HO.c_ratio(product_lib, o, x[c])), c
    p = HO.params(32000, 32.703196, 12, 1024)
    for c in (0, 1):
        want, cands, own = HO.harmonic_ratio(x[c], p["W"], p["slide"], p["max_length"])
        assert (own[0] is None) == (c == 0)
        _check(host[c], want, cands, ("chunks", c))
    product_lib.harmonicRatioObj_free(o)


@gpu
def test_device_calls_back_to_back(product_lib, cuda_device):
    """calls with different clip counts and lengths queued on one object without a synchronise"""
    import torch
    st, o = HO.c_new(product_lib, 44100, 50.0, 11, None, 512)
    calls = []
    for k, (b, n) in enumerate(((3, 30000), (17, 9000), (1, 2048), (40, 22050), (2, 60000))):
        x = _clips(b, n, 10 + k, dc_every=2)
        xd = torch.from_numpy(x).cuda()
        T = product_lib.harmonicRatioObj_calTimeLength(o, n)
        v = torch.empty((b, T), device="cuda")
        rc = product_lib.harmonicRatioObj_harmonicRatioBatch(o, dptr(xd), n, b, dptr(v), 1, stream())
        assert rc == 0, product_lib.afb200_lastError()
        calls.append((x, xd, v))
    torch.cuda.synchronize()
    for x, _, v in calls:
        for k in (0, len(x) - 1):
            assert np.array_equal(v[k].cpu().numpy(), HO.c_ratio(product_lib, o, x[k]))
    product_lib.harmonicRatioObj_free(o)


@gpu
def test_launch_count(product_lib, cuda_device):
    """two launches per staging chunk: every frame, then the frames without a crossing"""
    import torch
    h = af.HarmonicRatio(radix2_exp=11, slide_length=512)
    x = _clips(8, 20000, 3)
    xd = torch.from_numpy(x).cuda()
    assert count_launches(product_lib, lambda: h.harmonic_ratio_batch(xd), warm=True) == 2
    assert count_launches(product_lib, lambda: h.harmonic_ratio(x[0]), warm=True) == 2
    big = _clips(200, 160000, 4)                         # 64 MB staging chunks: three of them
    assert count_launches(product_lib, lambda: h.harmonic_ratio(big), warm=True) == 6


@gpu
def test_refusals_on_device(product_lib, cuda_device):
    """a refused constructor leaves no object; a call with fewer samples than the window leaves the output untouched"""
    st, o = HO.c_new(product_lib, 32000, 100.0, 14)
    assert st == -2 and not o
    st, o = HO.c_new(product_lib, 32000, 100.0, 10)
    assert (HO.c_ratio(product_lib, o, np.ones(1000, np.float32), fill=7.0, extra=3) == 7).all()
    assert (_batch(product_lib, o, np.ones((2, 1000), np.float32), True).size == 0)
    product_lib.harmonicRatioObj_free(o)


@gpu
def test_reference_harmonic_ratio_on_b200(raf, cuda_device):
    """the reference's own HarmonicRatio class (its docstring example's settings), on the reference build and on
    libaudioflux_b200.so, per channel of a multi-channel array; and this package's class giving the same arrays"""
    x = _clips(6, 48000, 7).reshape(2, 3, 48000)
    res = {}
    for which in ("ref", "b200"):
        raf.fftlib.set_fft_lib(lib_ext="b200" if which == "b200" else None)
        h = raf.HarmonicRatio(radix2_exp=12, samplate=32000, slide_length=1024)
        res[which] = (h.harmonic_ratio(x[0, 0]), h.harmonic_ratio(x))
    raf.fftlib.set_fft_lib(None)
    p = HO.params(32000, 32.703196, 12, 1024)
    for g, r, c in ((res["b200"][0], res["ref"][0], x[0, 0]), (res["b200"][1][1, 2], res["ref"][1][1, 2], x[1, 2])):
        want, cands, _ = HO.harmonic_ratio(c, p["W"], p["slide"], p["max_length"])
        _check(g, want, cands, "b200")
        _check(r, want, cands, "ref")
    own = af.HarmonicRatio(radix2_exp=12, samplate=32000, slide_length=1024)
    assert np.array_equal(own.harmonic_ratio(x[0, 0]), res["b200"][0])
    got = own.harmonic_ratio(x)
    assert got.shape == res["b200"][1].shape and got.dtype == np.float32 and np.array_equal(got, res["b200"][1])


@gpu
def test_report_undetermined():
    """the frames an undetermined decision settled, over the cases run above"""
    total = sum(len(a) for _, a in UNDETERMINED)
    print(f"harmonic ratio: {total} frame(s) decided by an oracle candidate: {UNDETERMINED}")
    assert total <= 20

