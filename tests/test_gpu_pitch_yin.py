"""PitchYIN on the GPU: every oracle case through pitchYINObj_pitch against the float64 interval oracle and the reference
build (where the GPU and the reference differ, both outcomes the oracle allows; the frames whose first trough the oracle
finds undetermined capped and reported), with the trough rows of getTroughData; the batch bit-identical to the legacy
call with host pointers across staging chunks, with device pointers back to back, with NULL value outputs and with the
caller's values kept in frames without a trough; streaming in uneven pieces equal to one call over the clip; one
launch per chunk; the refusals; and the reference's own PitchYIN class on libaudioflux_b200.so."""
import numpy as np
import pytest

import _pitch_c as PC
import _pitch_yin_oracle as YO
from _parity_kit import Out, count_launches, dptr, raf, run_batch, stream  # noqa: F401  (raf: a fixture)
from test_pitch_yin_cpu import FILL, reference_outputs

import audioflux_b200 as af

CASES = dict(YO.cases())
gpu = pytest.mark.gpu
UNDETERMINED = []          # (case, frames) with more than one first-trough candidate, reported at the end
GAP = []                   # (largest relative frequency difference from the reference, case)


def _check(out, frames, p, what, fill=FILL):
    ok, msg, alt = YO.check(*out[:3], frames, p, fill)
    assert ok, (what, msg)
    assert len(alt) <= max(2, len(frames) // 10), (what, alt)
    return alt


def _batch(lib, o, x, device, fill=FILL, values=True, troughs=True):
    """pitchYINObj_pitchBatch -> (fre, value1, value2, mFre, mTrough, lens), the planes not requested as None"""
    b, n = x.shape
    T = lib.pitchYINObj_calTimeLength(o, n)
    m = lib.pitchYINObj_getTroughData(o, None, None, None)
    plane = lambda *shape: Out(np.full((b, *shape), fill, np.float32))    # noqa: E731
    args = [plane(T), plane(T) if values else None, plane(T) if values else None,
            plane(T, m) if troughs else None, plane(T, m) if troughs else None,
            Out(np.full((b, T), -1, np.int32)) if troughs else None]
    got = iter(run_batch(lib, "pitchYINObj_pitchBatch", (o, np.ascontiguousarray(x, np.float32), n, b, *args), device))
    return tuple(next(got) if a is not None else None for a in args)


@gpu
@pytest.mark.parametrize("name", list(CASES))
def test_case_matches_oracle_and_reference(product_lib, cuda_device, name):
    kw = CASES[name]
    p = YO.case_params(kw)
    got = YO.c_case(product_lib, name, kw, FILL)
    assert product_lib.afb200_lastError() in (b"", None)
    frames = YO.oracle_case(name, kw)
    alt = _check(got, frames, p, (name, "oracle"))
    fre, v1, v2, mfre, mtrough, lens = got
    ok, msg = YO.check_troughs(mfre, mtrough, lens, frames, p)
    assert ok, (name, msg)
    has = lens > 0
    assert np.array_equal(mfre[has, 0], fre[has]) and np.array_equal(mtrough[has, 0], v1[has])
    assert (fre[~has] == FILL).all() and (v1[~has] == FILL).all()
    live = np.arange(mfre.shape[1])[None, :] < lens[:, None]
    assert (mfre[~live] == 0).all() and (mtrough[~live] == 0).all()
    # the reference passes the same oracle (the CPU suite); the frequencies differ by the correlation's rounding, and
    # whether a frame has a trough at all may differ only where the oracle finds that undetermined
    ref = reference_outputs(name)
    both = (fre != FILL) & (ref[0] != FILL)
    assert set(np.flatnonzero((fre != FILL) != (ref[0] != FILL))) <= set(alt), name
    if both.any():
        GAP.append((float(np.max(np.abs(fre[both] / ref[0][both] - 1))), name))
    if alt:
        UNDETERMINED.append((name, alt))
    # the batch with host and device pointers: clip 1 is clip 0 reversed and 1000 times louder
    x = YO.case_signal(name, kw)
    xs = np.stack([x, 1000 * x[::-1]])
    st, o = PC.c_new(product_lib, "yin", **kw["ctor"])
    if kw["thresh"] is not None:
        product_lib.pitchYINObj_setThresh(o, kw["thresh"])
    legacy = []
    for c in xs:
        res = PC.c_pitch(product_lib, "yin", o, c, FILL)
        legacy.append(res + YO.c_troughs(product_lib, o, len(res[0])))
    for a, b in zip(legacy[0], got):
        assert np.array_equal(a, b)
    for device in (False, True):
        out = _batch(product_lib, o, xs, device)
        for k in range(2):
            for i in range(6):
                assert np.array_equal(out[i][k], legacy[k][i]), (name, device, k, i)
    product_lib.pitchYINObj_free(o)


@gpu
def test_batch_across_chunks(product_lib, cuda_device):
    """200 clips of 160 000 samples: three host staging chunks; host and device batches equal the legacy call, also
    without the value outputs and without the trough rows"""
    x = PC.clips(200, 160000, 32000, 1, silent_every=5)
    st, o = PC.c_new(product_lib, "yin", sr=32000, lf=27.0, hf=2000.0, r2=12, slide=1024, auto=2048)
    assert st == 0
    host = _batch(product_lib, o, x, False)
    dev = _batch(product_lib, o, x, True)
    for a, b in zip(host, dev):
        assert np.array_equal(a, b)
    bare = _batch(product_lib, o, x, False, values=False, troughs=False)
    assert np.array_equal(bare[0], host[0]) and bare[1:] == (None,) * 5
    bare = _batch(product_lib, o, x[:40], True, values=False)
    assert np.array_equal(bare[0], host[0][:40]) and all(np.array_equal(bare[i], host[i][:40]) for i in (3, 4, 5))
    assert (host[0] == FILL).any()                     # silent halves: frames without a trough keep the fill
    for c in (0, 1, 95, 96, 97, 191, 192, 199):
        res = PC.c_pitch(product_lib, "yin", o, x[c], FILL)
        for i in range(3):
            assert np.array_equal(host[i][c], res[i]), (c, i)
    p = YO.params(sr=32000, lf=27.0, hf=2000.0, r2=12, slide=1024, auto=2048)
    for c in (0, 5):
        _check([h[c] for h in host], YO.pitch(x[c], p), p, ("chunks", c))
    product_lib.pitchYINObj_free(o)


@gpu
def test_device_calls_back_to_back(product_lib, cuda_device):
    """calls with different clip counts and lengths queued on one object without a synchronise"""
    import torch
    st, o = PC.c_new(product_lib, "yin", sr=44100, r2=11, slide=512, auto=1024)
    m = product_lib.pitchYINObj_getTroughData(o, None, None, None)
    calls = []
    for k, (b, n) in enumerate(((3, 30000), (17, 9000), (1, 2048), (40, 22050), (2, 60000))):
        x = PC.clips(b, n, 44100, 10 + k, silent_every=5)
        xd = torch.from_numpy(x).cuda()
        T = product_lib.pitchYINObj_calTimeLength(o, n)
        outs = [torch.full((b, T), FILL, device="cuda") for _ in range(3)]
        rows = [torch.empty((b, T, m), device="cuda") for _ in range(2)]
        lens = torch.empty((b, T), dtype=torch.int32, device="cuda")
        rc = product_lib.pitchYINObj_pitchBatch(o, dptr(xd), n, b, *map(dptr, outs + rows + [lens]), 1, stream())
        assert rc == 0, product_lib.afb200_lastError()
        calls.append((x, xd, outs, rows, lens))
    torch.cuda.synchronize()
    for x, _, outs, rows, lens in calls:
        for k in (0, len(x) - 1):
            res = PC.c_pitch(product_lib, "yin", o, x[k], FILL)
            res = res + YO.c_troughs(product_lib, o, len(res[0]))
            for i, v in enumerate(outs + rows + [lens]):
                assert np.array_equal(v[k].cpu().numpy(), res[i]), (len(x), k, i)
    product_lib.pitchYINObj_free(o)


@gpu
def test_streaming_equals_one_call(product_lib, cuda_device):
    """isContinue: uneven pieces (some shorter than a frame) give the frames of one call over the clip, for a slide
    below n and one above it; a batch call in between neither reads nor moves the carry"""
    x = PC.signal("glide", 40000, 16000, 5)
    for r2, slide in ((11, 512), (10, 1500)):
        st, whole = PC.c_new(product_lib, "yin", sr=16000, r2=r2, slide=slide)
        want = PC.c_pitch(product_lib, "yin", whole, x)
        st, o = PC.c_new(product_lib, "yin", sr=16000, r2=r2, slide=slide, cont=1)
        pieces = (700, 3000, 100, 9000, 1, 27199)
        got, start = [], 0
        for k, size in enumerate(pieces):
            got.append(PC.c_pitch(product_lib, "yin", o, x[start:start + size]))
            start += size
            if k == 2:
                _batch(product_lib, o, np.stack([x, x]), True)
        for i in range(3):
            assert np.array_equal(np.concatenate([g[i] for g in got]), want[i]), (r2, slide, i)
        product_lib.pitchYINObj_free(o)
        product_lib.pitchYINObj_free(whole)


@gpu
def test_launch_count(product_lib, cuda_device):
    """one launch per staging chunk"""
    import torch
    h = af.PitchYIN(radix2_exp=11, slide_length=512, auto_length=1024)
    x = PC.clips(8, 20000, 32000, 3, silent_every=5)
    xd = torch.from_numpy(x).cuda()
    assert count_launches(product_lib, lambda: h.pitch_batch(xd), warm=True) == 1
    assert count_launches(product_lib, lambda: h.pitch(x[0]), warm=True) == 1
    big = PC.clips(200, 160000, 32000, 4, silent_every=5)                  # 64 MB staging chunks: three of them
    assert count_launches(product_lib, lambda: h.pitch(big), warm=True) == 3


@gpu
def test_refusals_on_device(product_lib, cuda_device):
    """a refused constructor leaves no object; a call with fewer samples than the frame leaves the outputs untouched"""
    for kw, want in ((dict(r2=15), -2), (dict(sr=2000), -3), (dict(sr=8000, r2=10, auto=1021), -3)):
        st, o = PC.c_new(product_lib, "yin", **kw)
        assert st == want and not o
    st, o = PC.c_new(product_lib, "yin", r2=10)
    assert all((v == 7).all() for v in PC.c_pitch(product_lib, "yin", o, np.ones(1000, np.float32), fill=7.0, extra=3))
    assert _batch(product_lib, o, np.ones((2, 1000), np.float32), True)[0].size == 0
    product_lib.pitchYINObj_free(o)


@gpu
def test_reference_pitch_yin_on_b200(raf, cuda_device):
    """the reference's own PitchYIN class (with set_thresh), on the reference build and on libaudioflux_b200.so, per
    channel of a multi-channel array; and this package's class giving the same arrays"""
    x = PC.clips(6, 48000, 32000, 7, silent_every=5).reshape(2, 3, 48000)
    res = {}
    for which in ("ref", "b200"):
        raf.fftlib.set_fft_lib(lib_ext="b200" if which == "b200" else None)
        h = raf.PitchYIN(samplate=32000)
        h.set_thresh(0.2)
        res[which] = (h.pitch(x[0, 0]), h.pitch(x))
    raf.fftlib.set_fft_lib(None)
    p = YO.params(sr=32000, lf=27.0, hf=2000.0, r2=12, slide=1024, auto=2048)
    for g, r, c in ((res["b200"][0], res["ref"][0], x[0, 0]),
                    ([a[1, 2] for a in res["b200"][1]], [a[1, 2] for a in res["ref"][1]], x[1, 2])):
        frames = YO.pitch(c, p, 0.2)
        _check(g, frames, p, "b200", 0.0)
        _check(r, frames, p, "ref", 0.0)
    own = af.PitchYIN(samplate=32000)
    own.set_thresh(0.2)
    for a, b in zip(own.pitch(x[0, 0]), res["b200"][0]):
        assert np.array_equal(a, b)
    for a, b in zip(own.pitch(x), res["b200"][1]):
        assert a.shape == b.shape and a.dtype == np.float32 and np.array_equal(a, b)
    import torch
    for a, b in zip(own.pitch_batch(torch.from_numpy(x).cuda()), res["b200"][1]):
        assert a.is_cuda and np.array_equal(a.cpu().numpy(), b)


@gpu
def test_report_undetermined():
    """the frames with an undetermined first trough, over the cases run above"""
    total = sum(len(a) for _, a in UNDETERMINED)
    print(f"pitch YIN: {total} frame(s) with more than one first-trough candidate: {UNDETERMINED}; largest relative "
          f"frequency difference from the reference: {max(GAP, default=None)}")
    assert total <= 30
