"""Onset detection on the GPU: every oracle case through onsetObj_onset against the numpy oracle and the reference build
(novelty curve within 1e-4, the peak picking exact on the GPU's own curve, the points equal to the reference's up to
named near-ties); the batch bit-identical to the legacy call with host and device pointers and across staging chunks;
device calls queued back to back; the launch count; one clip of 100 000 frames; and the reference's own Onset class
running on libaudioflux_b200.so."""
import ctypes as C

import numpy as np
import pytest

import _onset_oracle as OO
from _parity_kit import Out, count_launches, dptr, raf, run_batch, stream  # noqa: F401  (raf: a fixture)
from test_onset_cpu import GOLD

import audioflux_b200 as af

TOL = 1e-4          # absolute: evn is normalised to [0, 1]
CASES = dict(OO.cases())
gpu = pytest.mark.gpu


def _check_points(evn, pts, evn_b, pts_b, pp, what):
    ok, diff = OO.points_agree(evn, pts, evn_b, pts_b, pp)
    assert ok, (what, "decisions differ away from a near-tie at frames", diff)


def _reference(name):
    """the reference build's (evn, points) of a case, from the golden file where the build is missing"""
    out = GOLD.outputs({f"{name}__evn", f"{name}__pts"})
    return out[f"{name}__evn"], out[f"{name}__pts"]


def _batch(lib, o, x, ph, prm, idx, device):
    """onsetObj_onsetBatch on x [batch, T, M] -> numpy (evn, points, counts)"""
    b, T, _ = x.shape
    par = None if prm is None else OO.NoveltyParam(*prm)
    ph = None if ph is None else np.ascontiguousarray(ph, np.float32)
    return run_batch(lib, "onsetObj_onsetBatch",
                     (o, np.ascontiguousarray(x, np.float32), ph, b, None if par is None else C.addressof(par),
                      None if idx is None else idx.ctypes.data, 0 if idx is None else len(idx),
                      Out(np.full((b, T), 7, np.float32)), Out(np.full((b, T), 7, np.int32)),
                      Out(np.full(b, 7, np.int32))), device)


def _legacy(lib, o, x, ph, prm, idx):
    evn, pts, _, _ = OO.c_onset(lib, o, x, ph, prm, idx)
    assert lib.afb200_lastError() in (b"", None)
    return evn, pts


@gpu
@pytest.mark.parametrize("name", list(CASES))
def test_case_matches_oracle_and_reference(product_lib, cuda_device, name):
    kw = CASES[name]
    pp = OO.peak_params(kw["sr"], kw["hop"])
    evn, pts = OO.c_case(product_lib, name, kw)
    assert product_lib.afb200_lastError() in (b"", None)
    # the pick stage exactly: the oracle's peak picking on the GPU's own curve
    assert np.array_equal(OO.pick(evn, pp), pts), name
    want_evn, want_pts = OO.oracle_case(name, kw)
    ref_evn, ref_pts = _reference(name)
    assert np.abs(evn.astype(np.float64) - want_evn).max() <= TOL, name
    assert np.abs(evn.astype(np.float64) - ref_evn).max() <= TOL, name
    _check_points(evn, pts, want_evn, want_pts, pp, (name, "oracle"))
    _check_points(evn, pts, ref_evn, ref_pts, pp, (name, "reference"))
    # the batch with host and device pointers, against the legacy call: a second clip 1000 times louder and reversed in
    # time, so that a novelty or a window reaching into the neighbouring clip would show
    x, ph = OO.case_signal(name, kw)
    phase = kw["kind"] in OO.PHASE
    xs = np.stack([x, 1000 * x[::-1]])
    phs = np.stack([ph, ph[::-1]]) if phase else None
    idx = OO.case_index(name, kw)
    st, o = OO.c_new(product_lib, x.shape[0], x.shape[1], kw["hop"], kw["sr"], kw["order"], kw["kind"])
    legacy = [_legacy(product_lib, o, xs[c], None if phs is None else phs[c], kw["prm"], idx) for c in range(2)]
    assert np.array_equal(legacy[0][0], evn) and np.array_equal(legacy[0][1], pts)
    for device in (False, True):
        e, p, c = _batch(product_lib, o, xs, phs, kw["prm"], idx, device)
        for k in range(2):
            n = len(legacy[k][1])
            assert c[k] == n and np.array_equal(e[k], legacy[k][0]), (name, device, k)
            assert np.array_equal(p[k][:n], legacy[k][1]) and not p[k][n:].any(), (name, device, k)
    product_lib.onsetObj_free(o)


def _clips(n, T, M, seed):
    rng = np.random.default_rng(seed)
    x = (rng.random((n, T, M)) + 0.01).astype(np.float32)
    x[:, ::17] *= 4                                       # an onset every 17 frames
    return x, rng.uniform(-np.pi, np.pi, (n, T, M)).astype(np.float32)


@gpu
def test_batch_across_chunks(product_lib, cuda_device):
    """40 clips of 313 frames x 1025 bins with phase: three host staging chunks of at most 16 clips"""
    x, ph = _clips(40, 313, 1025, 1)
    x[1::2] *= 1000.0
    idx = np.arange(3, 1000, 2, dtype=np.int32)
    st, o = OO.c_new(product_lib, 313, 1025, 512, 32000, 3, 6)           # WPD: the magnitudes weight the phase
    launches = count_launches(product_lib, lambda: _batch(product_lib, o, x, ph, OO.DEFAULT_PARAM, idx, False), warm=True)
    assert launches == 3 * 3, launches
    host = _batch(product_lib, o, x, ph, OO.DEFAULT_PARAM, idx, False)
    dev = _batch(product_lib, o, x, ph, OO.DEFAULT_PARAM, idx, True)
    for k in range(3):
        assert np.array_equal(host[k], dev[k]), k
    for c in (0, 15, 16, 31, 32, 39):
        e, p = _legacy(product_lib, o, x[c], ph[c], OO.DEFAULT_PARAM, idx)
        assert np.array_equal(host[0][c], e) and host[2][c] == len(p) and np.array_equal(host[1][c][:len(p)], p), c
    want_evn, want_pts = OO.onset(x[0], ph[0], 6, 3, OO.DEFAULT_PARAM, idx, OO.peak_params(32000, 512))
    assert np.abs(host[0][0] - want_evn).max() <= TOL
    assert host[2][0] >= 5
    product_lib.onsetObj_free(o)


@gpu
def test_device_calls_back_to_back(product_lib, cuda_device):
    """calls with different bin lists, parameters and clip counts queued on one object without a synchronise"""
    import torch
    T, M = 200, 96
    st, o = OO.c_new(product_lib, T, M, 256, 22050, 2, 0)
    calls = []
    for k, (b, idx, prm) in enumerate(((3, None, OO.DEFAULT_PARAM), (17, np.arange(10, 60, dtype=np.int32), None),
                                       (2, np.array([95, 0, 40], np.int32), (2, 2.0, 0, 1, 0, 0.0, 0, 1.0)),
                                       (5, np.arange(10, 60, dtype=np.int32), OO.DEFAULT_PARAM))):
        x, _ = _clips(b, T, M, 10 + k)
        xd = torch.from_numpy(x).cuda()
        e = torch.empty((b, T), device="cuda")
        p = torch.empty((b, T), dtype=torch.int32, device="cuda")
        c = torch.empty((b,), dtype=torch.int32, device="cuda")
        par = None if prm is None else OO.NoveltyParam(*prm)
        rc = product_lib.onsetObj_onsetBatch(o, dptr(xd), None, b, None if par is None else C.addressof(par),
                                             None if idx is None else idx.ctypes.data, 0 if idx is None else len(idx),
                                             dptr(e), dptr(p), dptr(c), 1, stream())
        assert rc == 0, product_lib.afb200_lastError()
        calls.append((x, idx, prm, xd, e, p, c))
    torch.cuda.synchronize()
    for x, idx, prm, _, e, p, c in calls:
        for k in (0, len(x) - 1):
            le, lp = _legacy(product_lib, o, x[k], None, prm, idx)
            assert np.array_equal(e[k].cpu().numpy(), le) and int(c[k]) == len(lp)
            assert np.array_equal(p[k].cpu().numpy()[:len(lp)], lp)
    product_lib.onsetObj_free(o)


@gpu
def test_launch_count(product_lib, cuda_device):
    """a warm call: the max filter (filter order >= 2), the novelty and the peak picking"""
    import torch
    x = torch.from_numpy(_clips(8, 157, 128, 3)[0]).cuda()
    for order, n in ((1, 2), (3, 3)):
        on = af.Onset(157, 128, 512, filter_order=order)
        assert count_launches(product_lib, lambda: on.onset_batch(x), warm=True) == n, order
        assert count_launches(product_lib, lambda: on.onset(x[0].cpu().numpy().T), warm=True) == n, order


@gpu
def test_long_clip(product_lib, cuda_device):
    """one clip of 100 000 frames: no limit on the clip length"""
    T, M = 100_000, 48
    x, _ = _clips(1, T, M, 4)
    prm = OO.DEFAULT_PARAM
    st, o = OO.c_new(product_lib, T, M, 512, 32000, 2, 0)
    evn, pts = _legacy(product_lib, o, x[0], None, prm, None)
    product_lib.onsetObj_free(o)
    pp = OO.peak_params(32000, 512)
    assert np.array_equal(OO.pick(evn, pp), pts)
    want_evn, want_pts = OO.onset(x[0], None, 0, 2, prm, None, pp)
    assert np.abs(evn.astype(np.float64) - want_evn).max() <= TOL
    assert len(pts) > 1000
    _check_points(evn, pts, want_evn, want_pts, pp, "long clip")


@gpu
def test_reference_onset_on_b200(raf, cuda_device):
    """the reference's Onset example (mel power BFT, dB, FLUX with NoveltyParam(1, 2, 0, 1, 0, 0, 0, 1)), HFC with the
    default parameters per channel of a multi-channel array, and PD with phase and a bin list, each through the
    reference's own Onset class on the reference build and on libaudioflux_b200.so; and this package's Onset giving the
    same arrays, including its multi-channel call"""
    T = raf.type
    sr = 32000
    x = (0.05 * np.random.default_rng(6).standard_normal(sr * 3)).astype(np.float32)
    for k in range(0, len(x) - 400, 3000):
        x[k:k + 400] += np.sin(np.arange(400) * 0.3).astype(np.float32) * np.linspace(1, 0, 400, dtype=np.float32)
    multi = (np.random.default_rng(7).random((2, 3, 64, 120)) + 0.01).astype(np.float32)
    mag, ph = _clips(1, 150, 80, 8)
    mag, ph = mag[0].T.copy(), ph[0].T.copy()
    dbs = {}
    for which in ("ref", "b200"):
        raf.fftlib.set_fft_lib(lib_ext="b200" if which == "b200" else None)
        b = raf.BFT(num=128, samplate=sr, radix2_exp=12, slide_length=2048, scale_type=T.SpectralFilterBankScaleType.MEL,
                    data_type=T.SpectralDataType.POWER)
        dbs[which] = _power_to_db(np.abs(b.bft(x)))
    db = dbs["b200"]
    assert np.abs(db - dbs["ref"]).max() < 1e-2                             # the BFT on the GPU, dB on the host
    res = {}
    for which in ("ref", "b200"):                      # both onsets on the same dB spectrogram: the GPU's
        raf.fftlib.set_fft_lib(lib_ext="b200" if which == "b200" else None)
        o = raf.Onset(time_length=db.shape[1], fre_length=db.shape[0], slide_length=2048, samplate=sr,
                      novelty_type=T.NoveltyType.FLUX)
        out = [o.onset(db, novelty_param=raf.NoveltyParam(1, 2, 0, 1, 0, 0, 0, 1))]
        o2 = raf.Onset(time_length=120, fre_length=64, slide_length=256, samplate=22050, filter_order=3,
                       novelty_type=T.NoveltyType.HFC)
        # the reference binding's multi-channel path stores each clip's points into a row of the frame count, which
        # fails unless every clip has a point at every frame; it fails the same way on both libraries
        with pytest.raises(ValueError, match="could not broadcast"):
            o2.onset(multi)
        out += [o2.onset(c) for c in multi.reshape(-1, 64, 120)]
        o3 = raf.Onset(time_length=150, fre_length=80, slide_length=512, novelty_type=T.NoveltyType.PD)
        out.append(o3.onset(mag, ph, index_arr=np.arange(5, 70)))
        res[which] = out
    raf.fftlib.set_fft_lib(None)
    pps = [OO.peak_params(sr, 2048)] + [OO.peak_params(22050, 256)] * 6 + [OO.peak_params(32000, 512)]
    for k, pp in enumerate(pps):
        (pg, eg, _, vg), (pr, er, _, vr) = res["b200"][k], res["ref"][k]
        assert eg.shape == er.shape and np.abs(eg - er).max() <= TOL, k
        assert np.array_equal(OO.pick(eg, pp), pg) and np.array_equal(OO.pick(er, pp), pr), k
        _check_points(eg, pg, er, pr, pp, k)
        assert np.array_equal(vg, eg[pg]) and np.array_equal(vr, er[pr]), k
    assert len(res["b200"][0][0]) >= 3
    # this package's class on the same inputs gives what the reference class gives on this library; its multi-channel
    # call pads each clip's points and values with 0 to the largest count
    own = [af.Onset(db.shape[1], 128, 2048, sr).onset(db, novelty_param=af.NoveltyParam(1, 2, 0, 1, 0, 0, 0, 1)),
           af.Onset(150, 80, 512, novelty_type=af.NoveltyType.PD).onset(mag, ph, index_arr=np.arange(5, 70))]
    for a, b in zip(own, (res["b200"][0], res["b200"][7])):
        for u, v in zip(a, b):
            assert u.shape == v.shape and u.dtype == v.dtype and np.array_equal(u, v)
    pm, em, tm, vm = af.Onset(120, 64, 256, 22050, 3, af.NoveltyType.HFC).onset(multi)
    n = max(len(r[0]) for r in res["b200"][1:7])
    assert pm.shape == vm.shape == tm.shape == (2, 3, n) and em.shape == (2, 3, 120) and pm.dtype == np.int32
    for c, (p1, e1, t1, v1) in enumerate(res["b200"][1:7]):
        i, j = divmod(c, 3)
        m = len(p1)
        assert np.array_equal(em[i, j], e1) and np.array_equal(pm[i, j, :m], p1) and np.array_equal(vm[i, j, :m], v1)
        assert np.array_equal(tm[i, j, :m], t1) and not pm[i, j, m:].any() and not vm[i, j, m:].any()


def _power_to_db(p, min_db=-80.0):
    """util_powerToDB of the reference (src/util/flux_util.c:549-571) in float32: 10 log10(p / max), floored"""
    p = np.asarray(p, np.float32)
    with np.errstate(all="ignore"):
        v = (np.float32(10) * np.log10((p / p.max()).astype(np.float32))).astype(np.float32)
    return np.maximum(v, np.float32(min_db)).astype(np.float32)

