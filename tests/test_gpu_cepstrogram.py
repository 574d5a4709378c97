"""Cepstrogram on the GPU: the legacy call against the oracle and the reference build at every supported size (per frame,
within 1e-4 of the frame's max |log S|), every NULL-output combination, silent frames, both batched entry points (host
and device pointers, batches that span several staging chunks) bit-identical to the legacy calls, cepstrogram2 on full
and half STFT planes and on a non-Hermitian plane, the launch count, the refusals, and the reference's own Cepstrogram
class running on libaudioflux_b200.so."""
import ctypes as C
import itertools

import numpy as np
import pytest

import _cepstrogram_oracle as CO
from _parity_kit import count_launches, dptr, raf, ref_lib_or_none, stream  # noqa: F401  (raf: a fixture)

import audioflux_b200 as af

pytestmark = pytest.mark.gpu
TOL = 1e-4          # per frame, of the frame's max |log S|; and per tensor, of max |want|
LOG_CLAMP = float(np.log(np.float32(1e-16)))


def _check(got, want, logs, what):
    """the per-frame bar, the per-tensor bar, and frames that are exactly zero in `want` exactly 0 in `got`"""
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if not got.size:
        return
    err = CO.frame_errors(got, want, logs)
    assert err.max() <= TOL, (what, int(np.argmax(err)), float(err.max()))
    assert np.abs(got - want).max() <= TOL * max(np.abs(want).max(), 1e-30) or not np.abs(want).max(), what
    zero = ~want.any(axis=1)
    assert not got[zero].any(), (what, "zero rows")


@pytest.mark.parametrize("name,kw", CO.cases(), ids=[c[0] for c in CO.cases()])
def test_legacy_matches_oracle_and_reference(product_lib, cuda_device, name, kw):
    x = CO.case_signal(name, kw)
    got = CO.c_case(product_lib, kw, x)
    assert product_lib.afb200_lastError() in (b"", None)
    *want, logs = CO.oracle_case(name, kw)
    for k in range(3):
        _check(got[k], want[k], logs, (name, k, "oracle"))
    ref = ref_lib_or_none()
    if ref is not None:
        for k, r in enumerate(CO.c_case(ref, kw, x)):
            _check(got[k], r.astype(np.float64), logs, (name, k, "reference"))


@pytest.mark.parametrize("r,c", [(10, 20), (14, 128), (6, 32), (1, 1)])
def test_skipped_outputs_do_not_change_the_others(product_lib, cuda_device, r, c):
    n = 1 << r
    kw = dict(radix2_exp=r, window_type=CO.W_HAMM, slide=max(1, n // 3), cep_num=c)
    x = CO.signal(r, 3 * n + 5)
    full = CO.c_case(product_lib, kw, x)
    for want in itertools.product((0, 1), repeat=3):
        if not any(want):
            continue
        part = CO.c_case(product_lib, kw, x, want)
        for k in range(3):
            assert (part[k] is None) == (not want[k])
            if want[k]:
                assert np.array_equal(part[k], full[k]), (want, k)


def test_silent_frames_hit_the_clamp(product_lib, cuda_device):
    for name, kw in CO.cases():
        if not kw.get("silent"):
            continue
        n, hop = 1 << kw["radix2_exp"], kw["slide"]
        x = CO.case_signal(name, kw)
        cep, env, det = CO.c_case(product_lib, kw, x)
        silent = [t for t in range(cep.shape[0]) if not x[t * hop:t * hop + n].any()]
        assert silent, name
        for t in silent:
            assert abs(cep[t, 0] - LOG_CLAMP) <= 1e-6 * abs(LOG_CLAMP), (name, t, cep[t, 0])
            assert not cep[t, 1:].any() and not det[t].any(), (name, t)
            assert (env[t] == cep[t, 0]).all(), (name, t)


def test_batches_bit_identical_to_legacy(product_lib, cuda_device):
    """2^12 frames of 160 000-sample clips: 3.8 MB of output per clip, so a host batch of 40 runs in three staging
    chunks; device batches run at once"""
    import torch
    r, hop, c, length, B = 12, 1024, 4, 160000, 40
    n = 1 << r
    x = np.stack([CO.signal(s, length) * (1 + 3 * (s % 3)) for s in range(B)])
    t = af.Cepstrogram(radix2_exp=r, window_type=af.WindowType.HANN, slide_length=hop)
    legacy = [CO.c_cepstrogram(product_lib, t._obj, n, c, x[b]) for b in range(B)]
    host = t.cepstrogram_batch(x, c)
    dev = t.cepstrogram_batch(torch.from_numpy(x).cuda(), c)
    torch.cuda.synchronize()
    for b in range(B):
        for k in range(3):
            assert np.array_equal(host[k][b], legacy[b][k]), (b, k)
            assert np.array_equal(dev[k][b].cpu().numpy(), legacy[b][k]), (b, k, "device")
    # one output only, a [2, 3, L] lead shape
    small = x[:6, :9000].reshape(2, 3, 9000)
    cep, env, det = t.cepstrogram_batch(small, c, cep=False, env=False)
    assert cep is None and env is None and det.shape == (2, 3, t.cal_time_length(9000), n // 2 + 1)
    for b in range(6):
        want = CO.c_cepstrogram(product_lib, t._obj, n, c, x[b, :9000])[2]
        assert np.array_equal(det.reshape(6, -1, n // 2 + 1)[b], want), b
    # the reference layout of the Python front door
    cep2, env2, det2 = t.cepstrogram(x[:2], c)
    assert cep2.shape == (2, n // 2 + 1, legacy[0][0].shape[0])
    assert np.array_equal(cep2[1], legacy[1][0].T) and np.array_equal(det2[0], legacy[0][2].T)


def _stft_full(lib, r, window, hop, x):
    obj = C.c_void_p()
    assert lib.stftObj_new(C.byref(obj), r, C.byref(C.c_int(window)), C.byref(C.c_int(hop)), None) == 0
    n = 1 << r
    T = lib.stftObj_calTimeLength(obj, x.size)
    re, im = np.zeros((T, n), np.float32), np.zeros((T, n), np.float32)
    lib.stftObj_stft(obj, x.ctypes.data, x.size, re.ctypes.data, im.ctypes.data)
    lib.stftObj_free(obj)
    return re, im


def test_cepstrogram2_full_and_half_planes(product_lib, cuda_device):
    import torch
    for r, c, w, hop in ((8, 4, CO.W_HANN, 64), (11, 20, CO.W_HAMM, 512), (14, 128, CO.W_RECT, 4096)):
        n = 1 << r
        x = CO.signal(r + 100, 4 * n + 33)
        s, obj = CO.c_new(product_lib, r, w, hop)
        base = CO.c_cepstrogram(product_lib, obj, n, c, x)
        *_, logs = CO.cepstrogram(x, n, hop, w, c)
        re, im = _stft_full(product_lib, r, w, hop, x)
        re0, im0 = re.copy(), im.copy()
        full = CO.c_cepstrogram2(product_lib, obj, n, c, re, im)
        assert np.array_equal(re, re0) and np.array_equal(im, im0)
        assert product_lib.afb200_lastError() in (b"", None)
        want2 = CO.cepstrogram2(re, im, c)
        for k in range(3):
            _check(full[k], base[k].astype(np.float64), logs, (r, k, "full vs cepstrogram"))
            _check(full[k], want2[k], want2[3], (r, k, "full vs oracle"))
        # half planes from stftObj_stftBatch on the device, cepstrogram2Batch on the device
        sobj = C.c_void_p()
        assert product_lib.stftObj_new(C.byref(sobj), r, C.byref(C.c_int(w)), C.byref(C.c_int(hop)), None) == 0
        T = base[0].shape[0]
        xd = torch.from_numpy(x).cuda()
        hre = torch.empty((T, n // 2 + 1), device="cuda")
        him = torch.empty_like(hre)
        assert product_lib.stftObj_stftBatch(sobj, dptr(xd), x.size, 1, dptr(hre), dptr(him), 1, stream()) == 0
        outs = [torch.full((T, n // 2 + 1), 7.0, device="cuda") for _ in range(3)]
        h0 = (hre.clone(), him.clone())
        assert product_lib.cepstrogramObj_cepstrogram2Batch(obj, c, dptr(hre), dptr(him), T, n // 2 + 1,
                                                            *map(dptr, outs), 1, stream()) == 0
        torch.cuda.synchronize()
        assert torch.equal(hre, h0[0]) and torch.equal(him, h0[1])
        for k in range(3):
            _check(outs[k].cpu().numpy(), base[k].astype(np.float64), logs, (r, k, "half vs cepstrogram"))
        product_lib.stftObj_free(sobj)
        product_lib.cepstrogramObj_free(obj)


def test_cepstrogram2_non_hermitian_plane(product_lib, cuda_device):
    """width N: every bin is used, y = Re IFFT_N(log S) over all N bins"""
    rng = np.random.default_rng(8)
    for r, c in ((3, 2), (9, 20), (13, 4095)):
        n = 1 << r
        re = rng.standard_normal((5, n)).astype(np.float32)
        im = rng.standard_normal((5, n)).astype(np.float32)
        s, obj = CO.c_new(product_lib, r)
        got = CO.c_cepstrogram2(product_lib, obj, n, c, re, im)
        *want, logs = CO.cepstrogram2(re, im, c)
        for k in range(3):
            _check(got[k], want[k], logs, (r, k))
        t = af.Cepstrogram(radix2_exp=r)
        py = t.cepstrogram2_batch(re.reshape(5, 1, n), im.reshape(5, 1, n), c)
        for k in range(3):
            assert np.array_equal(py[k].reshape(5, -1), got[k]), (r, k)
        product_lib.cepstrogramObj_free(obj)


def test_cepstrogram2_batch_spans_chunks(product_lib, cuda_device):
    import torch
    r, c, rows = 12, 20, 5000
    n = 1 << r
    rng = np.random.default_rng(3)
    re = rng.standard_normal((rows, n)).astype(np.float32)
    im = rng.standard_normal((rows, n)).astype(np.float32)
    t = af.Cepstrogram(radix2_exp=r)
    host = t.cepstrogram2_batch(re, im, c)
    dev = t.cepstrogram2_batch(torch.from_numpy(re).cuda(), torch.from_numpy(im).cuda(), c)
    torch.cuda.synchronize()
    for b in (0, 2047, 2048, 4095, 4096, rows - 1):
        legacy = CO.c_cepstrogram2(product_lib, t._obj, n, c, re[b:b + 1], im[b:b + 1])
        for k in range(3):
            assert np.array_equal(host[k][b], legacy[k][0]), (b, k)
            assert np.array_equal(dev[k][b].cpu().numpy(), legacy[k][0]), (b, k, "device")


def test_one_launch_per_chunk(product_lib, cuda_device):
    import torch
    t = af.Cepstrogram(radix2_exp=12, window_type=af.WindowType.HANN, slide_length=1024)
    x = np.stack([CO.signal(s, 160000) for s in range(40)])
    xd = torch.from_numpy(x).cuda()
    assert count_launches(product_lib, lambda: t.cepstrogram_batch(xd, 4), warm=True) == 1
    assert count_launches(product_lib, lambda: t.cepstrogram_batch(xd, 4, env=False), warm=True) == 1
    assert count_launches(product_lib, lambda: t.cepstrogram_batch(x, 4), warm=True) == 3          # 16 + 16 + 8 clips
    assert count_launches(product_lib, lambda: t.cepstrogram_batch(x[:1], 4), warm=True) == 1
    for r in (1, 8, 14):
        u = af.Cepstrogram(radix2_exp=r)
        xr = torch.from_numpy(CO.signal(r, 5 * (1 << r))).cuda()
        assert count_launches(product_lib, lambda: u.cepstrogram_batch(xr, 1), warm=True) == 1, r


def test_refusals_on_the_device(product_lib, cuda_device):
    import torch
    n = 1024
    t = af.Cepstrogram(radix2_exp=10, slide_length=256)
    xd = torch.from_numpy(CO.signal(4, 5000)).cuda()
    T = t.cal_time_length(5000)
    outs = [torch.full((T, n // 2 + 1), 7.0, device="cuda") for _ in range(3)]
    for c in (0, n // 2 + 1):
        st = product_lib.cepstrogramObj_cepstrogramBatch(t._obj, c, dptr(xd), 5000, 1, *map(dptr, outs), 1, stream())
        assert st != 0 and f"cepNum={c}".encode() in product_lib.afb200_lastError()
        torch.cuda.synchronize()
        assert all((o == 7.0).all() for o in outs)
    # the largest legal cepNum runs, and its details are exactly 0
    st = product_lib.cepstrogramObj_cepstrogramBatch(t._obj, n // 2, dptr(xd), 5000, 1, *map(dptr, outs), 1, stream())
    torch.cuda.synchronize()
    assert st == 0 and not outs[2].any() and (outs[0] != 7.0).all()


def test_reference_class_on_b200(raf, cuda_device):
    rng = np.random.default_rng(5)
    mono = CO.signal(11, 20000)
    multi = (0.1 * rng.standard_normal((2, 3, 9000))).astype(np.float32)
    res = {}
    for which in ("ref", "b200"):
        raf.fftlib.set_fft_lib(lib_ext="b200" if which == "b200" else None)
        s = raf.Cepstrogram(radix2_exp=11, samplate=16000, window_type=raf.type.WindowType.HANN, slide_length=512)
        out = [*s.cepstrogram(mono, cep_num=20), *s.cepstrogram(multi)]
        out += [s.x_coords(20000), s.y_coords(), np.array(s.cal_time_length(20000))]
        res[which] = out
    raf.fftlib.set_fft_lib(None)
    mine = af.Cepstrogram(radix2_exp=11, samplate=16000, window_type=af.WindowType.HANN, slide_length=512)
    own = [*mine.cepstrogram(mono, cep_num=20), *mine.cepstrogram(multi)]
    own += [mine.x_coords(20000), mine.y_coords(), np.array(mine.cal_time_length(20000))]
    g, r = res["b200"], res["ref"]
    for k in range(6):
        cep_num = 20 if k < 3 else 4
        x = mono if k < 3 else multi
        assert g[k].shape == r[k].shape == own[k].shape, k
        # (..., fre, time) -> frames; the scale is the float64 log spectrum of each frame
        logs = np.concatenate([CO.cepstrogram(c, 2048, 512, CO.W_HANN, cep_num)[3] for c in x.reshape(-1, x.shape[-1])])
        flat = [np.swapaxes(a, -1, -2).reshape(-1, a.shape[-2]) for a in (g[k], r[k], own[k])]
        _check(flat[0], flat[1].astype(np.float64), logs, (k, "reference class on b200"))
        assert np.array_equal(flat[2], flat[0]), k
    for k in range(6, 9):
        assert np.array_equal(g[k], r[k]) and np.array_equal(own[k], r[k]), k
