"""Spectral descriptors on the GPU: the reference's entry points against the oracle and the reference build, the batched
entry point (host and device pointers, one launch, clip boundaries), the documented differences (stateless objects,
step >= timeLength) and the reference's own Spectral class running on libaudioflux_b200.so."""
import numpy as np
import pytest

import _spectral_cases as SC
from _parity_kit import count_launches, raf, ref_lib_or_none  # noqa: F401  (raf: a fixture)

import audioflux_b200 as af
from audioflux_b200 import spectral as SP

pytestmark = pytest.mark.gpu


def _parts(v):
    return v if isinstance(v, tuple) else (v,)


def test_legacy_entry_points_match_oracle_and_reference(product_lib, cuda_device):
    ref = ref_lib_or_none()
    bad = []
    for setname, x, ph, fre in SC.spectrogram_sets(seed=3):
        for mode in ("full", "range", "list"):
            for name, kw in SC.VARIANTS:
                if name in SC.SO.PHASE and ph is None:
                    continue
                got = SC.call_c(product_lib, name, x, fre, mode, ph, **kw)
                want = SC.oracle(name, x, fre, mode, ph, **kw)
                refs = SC.call_c(ref, name, x, fre, mode, ph, **kw) if ref is not None else None
                for part, (g, w) in enumerate(zip(_parts(got), _parts(want))):
                    exact = SC.is_exact(name, kw) or (name == "max")
                    msg = SC.agree(g, w, exact=exact)
                    if refs is not None:
                        msg = msg or SC.agree(g, _parts(refs)[part], exact=exact)
                    if msg:
                        bad.append(f"{setname}/{mode}/{name}{kw}[{part}]: {msg}")
    assert not bad, "\n".join(bad[:20])


def _all_features():
    seen, feats = set(), []
    for name, kw in SC.VARIANTS:
        if name not in seen:
            seen.add(name)
            feats.append((name, kw))
    return feats


def _clips(num=257, T=23, B=5, seed=11):
    rng = np.random.default_rng(seed)
    x = np.abs(rng.standard_normal((B, T, num))).astype(np.float32)
    x[:, 4] = 0
    x[B // 2] *= 50      # clips of very different level next to each other
    ph = rng.uniform(-np.pi, np.pi, (B, T, num)).astype(np.float32)
    fre = np.linspace(0, 8000, num).astype(np.float32)
    return x, ph, fre


def test_batch_host_device_and_per_clip_agree(product_lib, cuda_device):
    import torch
    x, ph, fre = _clips()
    feats = _all_features()
    for mode in ("full", "list"):
        s = af.Spectral(x.shape[-1], fre)
        idx = SC.edges(x.shape[-1])[mode]
        if mode == "list":
            s.set_edge_arr(idx)
        host = s.spectral_batch(x, feats, phase=ph)
        dev = s.spectral_batch(torch.from_numpy(x).cuda(), feats, phase=torch.from_numpy(ph).cuda())
        torch.cuda.synchronize()
        for name, kw in feats:
            for h, d in zip(_parts(host[name]), _parts(dev[name])):
                assert np.array_equal(h, d.cpu().numpy(), equal_nan=True), (mode, name)
            # one request per call is bit-identical to all requests in one call
            single = s.spectral_batch(x, [(name, kw)], phase=ph)[name]
            for h, g in zip(_parts(host[name]), _parts(single)):
                assert np.array_equal(h, g, equal_nan=True), (mode, name, "single")
            # each clip alone (legacy entry point, batch 1): frame 0 of clip b never sees clip b-1
            for b in range(x.shape[0]):
                legacy = SC.call_c(product_lib, name, x[b], fre, mode, ph[b], **kw)
                for h, g in zip(_parts(host[name]), _parts(legacy)):
                    assert np.array_equal(h[b], g, equal_nan=True), (mode, name, b)
                want = SC.oracle(name, x[b], fre, mode, ph[b], **kw)
                for h, w in zip(_parts(host[name]), _parts(want)):
                    assert SC.agree(h[b], w, exact=SC.is_exact(name, kw) or name == "max") is None, (mode, name, b)


def test_one_launch_per_device_call(product_lib, cuda_device):
    import torch
    x, ph, fre = _clips(B=3)
    s = af.Spectral(x.shape[-1], fre)
    xd, pd = torch.from_numpy(x).cuda(), torch.from_numpy(ph).cuda()
    s.spectral_batch(xd, ["centroid"])
    # the first call with phase planes, and the first with every feature, each launch one kernel
    for feats in (["centroid"], _all_features()):
        assert count_launches(product_lib, lambda: s.spectral_batch(xd, feats, phase=pd), warm=False) == 1


def test_step_at_least_time_length_is_clamped(product_lib, cuda_device):
    x, ph, fre = _clips(T=6, B=2)
    s = af.Spectral(x.shape[-1], fre)
    for name in ("flux", "sd", "sf", "novelty"):
        for step in (6, 9):
            out = s.spectral_batch(x, [(name, dict(step=step))])[name]
            assert out.shape == (2, 6) and (out == 0).all()
    out = s.spectral_batch(x, [("flux", dict(step=5))])["flux"]
    assert (out[:, :5] == 0).all() and (out[:, 5] > 0).all()


@pytest.mark.parametrize("num", [2, 84, 128, 1025, 2049, 32769])
def test_bin_counts(product_lib, cuda_device, num):
    rng = np.random.default_rng(num)
    T = 7 if num < 30000 else 4
    x = np.abs(rng.standard_normal((2, T, num))).astype(np.float32)
    fre = np.linspace(0, 24000, num).astype(np.float32)
    feats = [("centroid", {}), ("rolloff", {}), ("flux", {}), ("max", {}), ("entropy", {}), ("flatness", {}),
             ("hfc", {}), ("var", {})]
    got = af.Spectral(num, fre).spectral_batch(x, feats)
    for name, kw in feats:
        for b in range(2):
            want = SC.SO.compute(name, x[b], range(num), fre, **kw)
            for g, w in zip(_parts(got[name]), _parts(want)):
                assert SC.agree(g[b], w, exact=name in ("rolloff", "max")) is None, (num, name, b)


def test_stateless_repeated_and_multichannel(product_lib, cuda_device):
    """the reference returns A's centroid for B and the first channel's values for every channel (cached sums)"""
    x, ph, fre = _clips(B=3)
    s = af.Spectral(x.shape[-1], fre)
    m = np.ascontiguousarray(np.swapaxes(x, -1, -2))      # [..., fre, time]
    idx = range(x.shape[-1])
    for name in ("centroid", "spread", "flatness", "rolloff", "crest", "decrease", "entropy", "mean"):
        a = getattr(s, name)(m[0])
        b = getattr(s, name)(m[1])
        multi = getattr(s, name)(m)
        for k, got in ((0, a), (1, b)):
            for g, w in zip(_parts(got), _parts(SC.SO.compute(name, x[k], idx, fre))):
                assert SC.agree(g, w, exact=name == "rolloff") is None, (name, k)
        for k in range(3):
            for g, w in zip(_parts(multi), _parts(SC.SO.compute(name, x[k], idx, fre))):
                assert SC.agree(g[k], w, exact=name == "rolloff") is None, (name, k)


def test_reference_spectral_class_on_b200(raf, cuda_device):
    """every method of the reference's unmodified Spectral class, single channel, fresh object per call"""
    T = raf.type
    _, x, ph, fre = SC.spectrogram_sets(seed=5)[0]
    m, p = np.ascontiguousarray(x.T), np.ascontiguousarray(ph.T)     # [fre, time]
    # the class itself refuses rolloff / broadband thresholds outside [0, 1] (feature/spectral.py:366, 2105)
    calls = [(n, kw) for n, kw in SC.VARIANTS if n != "novelty" and kw.get("threshold", 0) <= 1] + [
        ("novelty", dict(method_type=T.SpectralNoveltyMethodType(kw["method_type"]),
                         data_type=T.SpectralNoveltyDataType(kw["data_type"]), threshold=kw["threshold"]))
        for kw in SC.NOVELTY]
    bad = []
    for name, kw in calls:
        res = {}
        for which in ("ref", "b200"):
            raf.fftlib.set_fft_lib(lib_ext="b200" if which == "b200" else None)
            s = raf.Spectral(num=x.shape[1], fre_band_arr=fre)
            s.set_time_length(x.shape[0])
            s.set_edge_arr([3, 1, 200, 3, 50])
            fn = getattr(s, name)
            res[which] = fn(m, p, **kw) if name in SC.SO.PHASE else fn(m, **kw)
        for part, (g, r) in enumerate(zip(_parts(res["b200"]), _parts(res["ref"]))):
            plain = {k: getattr(v, "value", v) for k, v in kw.items()}
            msg = SC.agree(g, r, exact=SC.is_exact(name, plain) or name == "max")
            if msg:
                bad.append(f"{name}{plain}[{part}]: {msg}")
    raf.fftlib.set_fft_lib(None)
    assert not bad, "\n".join(bad)
