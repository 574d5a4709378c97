"""PitchPEF on the GPU: every oracle case through pitchPEFObj_pitch against the float64 oracle and the reference build
(the exact frequency, except on frames whose arg-max the oracle finds undetermined, where the frequency of one of its
candidate lags; the count of such frames capped and reported); the batch bit-identical to the legacy call with host
pointers across staging chunks and with device pointers; streaming in uneven pieces equal to one call over the clip;
one launch per chunk; the refusals; and the reference's own PitchPEF class on libaudioflux_b200.so."""
import numpy as np
import pytest

import _pitch_c as PC
import _pitch_pef_oracle as PO
from _parity_kit import Out, count_launches, dptr, raf, run_batch, stream  # noqa: F401  (raf: a fixture)
from test_pitch_pef_cpu import GOLD

import audioflux_b200 as af

CASES = dict(PO.cases())
gpu = pytest.mark.gpu
UNDETERMINED = []          # (case, frames) decided by a candidate, reported at the end


def _check(got, want, cands, p, what):
    ok, alt = PO.agree(got, want, cands, p)
    assert ok, (what, "differs away from an undetermined arg-max at frame", alt, got[alt], want[alt])
    assert len(alt) <= max(2, len(want) // 10), (what, alt)
    return alt


def _batch(lib, o, x, device, fill=7.0):
    b, n = x.shape
    p = lib.pitchPEFObj_calTimeLength(o, n)
    return run_batch(lib, "pitchPEFObj_pitchBatch",
                     (o, np.ascontiguousarray(x, np.float32), n, b, Out(np.full((b, p), fill, np.float32))), device)[0]


@gpu
@pytest.mark.parametrize("name", list(CASES))
def test_case_matches_oracle_and_reference(product_lib, cuda_device, name):
    kw = CASES[name]
    p = PO.case_params(kw)
    got = PO.c_case(product_lib, name, kw)
    assert product_lib.afb200_lastError() in (b"", None)
    want, cands = PO.oracle_case(name, kw)
    alt = _check(got, want, cands, p, (name, "oracle"))
    ref = GOLD.outputs({name})[name]
    assert got.shape == ref.shape
    far = np.flatnonzero(got != ref)
    for t in far:                          # where the GPU and the reference differ, both are outcomes the oracle allows
        assert got[t] in {p["log"][k] for k in cands[t]} and ref[t] in {p["log"][k] for k in cands[t]}, (name, t)
    assert len(far) <= max(2, len(want) // 10), (name, far)
    if alt:
        UNDETERMINED.append((name, alt))
    # the batch with host and device pointers: clip 1 is clip 0 reversed and 1000 times louder
    x = PO.case_signal(name, kw)
    xs = np.stack([x, 1000 * x[::-1]])
    st, o = PC.c_new(product_lib, "pef", **kw["ctor"])
    legacy = [PC.c_pitch(product_lib, "pef", o, c) for c in xs]
    assert np.array_equal(legacy[0], got)
    for device in (False, True):
        out = _batch(product_lib, o, xs, device)
        for k in range(2):
            assert np.array_equal(out[k], legacy[k]), (name, device, k)
    product_lib.pitchPEFObj_free(o)


@gpu
def test_batch_across_chunks(product_lib, cuda_device):
    """200 clips of 160 000 samples: three host staging chunks; host and device batches equal the legacy call"""
    x = PC.clips(200, 160000, 32000, 1)
    st, o = PC.c_new(product_lib, "pef", r2=12, slide=1024)
    assert st == 0
    host = _batch(product_lib, o, x, False)
    dev = _batch(product_lib, o, x, True)
    assert np.array_equal(host, dev)
    for c in (0, 1, 95, 96, 97, 191, 192, 199):
        assert np.array_equal(host[c], PC.c_pitch(product_lib, "pef", o, x[c])), c
    p = PO.params(r2=12, slide=1024)
    for c in (0, 1):
        want, cands = PO.pitch(x[c], p)
        _check(host[c], want, cands, p, ("chunks", c))
    product_lib.pitchPEFObj_free(o)


@gpu
def test_device_calls_back_to_back(product_lib, cuda_device):
    """calls with different clip counts and lengths queued on one object without a synchronise"""
    import torch
    st, o = PC.c_new(product_lib, "pef", sr=44100, r2=11, slide=512, beta=1.0)
    calls = []
    for k, (b, n) in enumerate(((3, 30000), (17, 9000), (1, 2048), (40, 22050), (2, 60000))):
        x = PC.clips(b, n, 44100, 10 + k)
        xd = torch.from_numpy(x).cuda()
        T = product_lib.pitchPEFObj_calTimeLength(o, n)
        v = torch.empty((b, T), device="cuda")
        rc = product_lib.pitchPEFObj_pitchBatch(o, dptr(xd), n, b, dptr(v), 1, stream())
        assert rc == 0, product_lib.afb200_lastError()
        calls.append((x, xd, v))
    torch.cuda.synchronize()
    for x, _, v in calls:
        for k in (0, len(x) - 1):
            assert np.array_equal(v[k].cpu().numpy(), PC.c_pitch(product_lib, "pef", o, x[k]))
    product_lib.pitchPEFObj_free(o)


@gpu
def test_streaming_equals_one_call(product_lib, cuda_device):
    """isContinue: uneven pieces (some shorter than a frame) give the frames of one call over the clip, for a slide
    below n and one above it; a batch call in between neither reads nor moves the carry"""
    x = PC.signal("glide", 40000, 16000, 5)
    for r2, slide in ((11, 512), (10, 1500)):
        st, whole = PC.c_new(product_lib, "pef", sr=16000, r2=r2, slide=slide)
        want = PC.c_pitch(product_lib, "pef", whole, x)
        st, o = PC.c_new(product_lib, "pef", sr=16000, r2=r2, slide=slide, cont=1)
        pieces = (700, 3000, 100, 9000, 1, 27199)
        got, start = [], 0
        for k, size in enumerate(pieces):
            got.append(PC.c_pitch(product_lib, "pef", o, x[start:start + size]))
            start += size
            if k == 2:
                _batch(product_lib, o, np.stack([x, x]), True)
        assert np.array_equal(np.concatenate(got), want), (r2, slide)
        product_lib.pitchPEFObj_free(o)
        product_lib.pitchPEFObj_free(whole)


@gpu
def test_launch_count(product_lib, cuda_device):
    """one launch per staging chunk"""
    import torch
    h = af.PitchPEF(radix2_exp=11, slide_length=512)
    x = PC.clips(8, 20000, 32000, 3)
    xd = torch.from_numpy(x).cuda()
    assert count_launches(product_lib, lambda: h.pitch_batch(xd), warm=True) == 1
    assert count_launches(product_lib, lambda: h.pitch(x[0]), warm=True) == 1
    big = PC.clips(200, 160000, 32000, 4)                  # 64 MB staging chunks: three of them
    assert count_launches(product_lib, lambda: h.pitch(big), warm=True) == 3


@gpu
def test_refusals_on_device(product_lib, cuda_device):
    """a refused constructor leaves no object; a call with fewer samples than the frame leaves the output untouched"""
    st, o = PC.c_new(product_lib, "pef", r2=14)
    assert st == -2 and not o
    st, o = PC.c_new(product_lib, "pef", r2=10)
    assert (PC.c_pitch(product_lib, "pef", o, np.ones(1000, np.float32), fill=7.0, extra=3) == 7).all()
    assert _batch(product_lib, o, np.ones((2, 1000), np.float32), True).size == 0
    product_lib.pitchPEFObj_free(o)


@gpu
def test_reference_pitch_pef_on_b200(raf, cuda_device):
    """the reference's own PitchPEF class, on the reference build and on libaudioflux_b200.so, per channel of a
    multi-channel array; and this package's class giving the same arrays"""
    x = PC.clips(6, 48000, 32000, 7).reshape(2, 3, 48000)
    res = {}
    for which in ("ref", "b200"):
        raf.fftlib.set_fft_lib(lib_ext="b200" if which == "b200" else None)
        h = raf.PitchPEF(samplate=32000, radix2_exp=12, slide_length=1024)
        res[which] = (h.pitch(x[0, 0]), h.pitch(x))
    raf.fftlib.set_fft_lib(None)
    p = PO.params(sr=32000, r2=12, slide=1024, lf=32.0, hf=2000.0, cf=4000.0)
    for g, r, c in ((res["b200"][0], res["ref"][0], x[0, 0]), (res["b200"][1][1, 2], res["ref"][1][1, 2], x[1, 2])):
        want, cands = PO.pitch(c, p)
        _check(g, want, cands, p, "b200")
        _check(r, want, cands, p, "ref")
    own = af.PitchPEF(samplate=32000, radix2_exp=12, slide_length=1024)
    assert np.array_equal(own.pitch(x[0, 0]), res["b200"][0])
    got = own.pitch(x)
    assert got.shape == res["b200"][1].shape and got.dtype == np.float32 and np.array_equal(got, res["b200"][1])


@gpu
def test_report_undetermined():
    """the frames an undetermined arg-max settled, over the cases run above"""
    total = sum(len(a) for _, a in UNDETERMINED)
    print(f"pitch PEF: {total} frame(s) decided by an oracle candidate: {UNDETERMINED}")
    assert total <= 20
