"""Spectral descriptors on the GPU frame by frame against the float64 oracle (tests/_spectral_frames.py): clips of many
32-frame tiles (k_spectral gives each CTA one tile of one clip), temporal steps and rolloff look-backs that reach into
earlier tiles, every request alone and all of them in one call, crafted rows (NaN, +-inf, denormals, negative bins,
zero frames, max ties across and within lanes), the reference's per-feature entry points on long clips, outputs that
start pre-filled, and a host batch that spans three staging chunks.  Each feature's worst per-frame error ratio
(|got - want| / (1e-4 scale_t)) is printed at the end of the module."""
import numpy as np
import pytest

import _spectral_cases as SC
import _spectral_frames as SF
from _parity_kit import ref_lib_or_none

pytestmark = pytest.mark.gpu

REPORT = SF.Report()


@pytest.fixture(scope="module", autouse=True)
def worst_ratios():
    yield
    print("\nworst per-frame error ratio of each feature (1 = the bar):\n" + REPORT.table())


def _check(rep, label, x, ph, fre, idx, variants, got, prefill=None):
    """got {variant index: planes [B, T]} against the oracle, clip by clip"""
    for i, (name, kw) in enumerate(variants):
        for b in range(x.shape[0]):
            pre = None if prefill is None else prefill[i][:, b]
            SF.check_clip(rep, f"{label} b={b}", name, kw, [g[b] for g in got[i]], x[b], idx, fre,
                          None if ph is None else ph[b], pre)


def _finish(rep):
    for k, v in rep.worst.items():
        REPORT.worst[k] = max(REPORT.worst.get(k, 0.0), v)
    assert rep.ok(), rep.text()


def _variants(ph):
    return [(n, kw) for n, kw in SC.VARIANTS if ph is not None or n not in SC.SO.PHASE]


@pytest.mark.parametrize("setname,mode", list(SF.bin_sets()), ids=lambda v: str(v))
def test_every_variant_across_tiles(product_lib, cuda_device, setname, mode):
    """T in {1, 31, 32, 33, 64, 65, 97, 465} x batch {1, 3} (two lengths for the edge lists): every variant in one call
    (host pointers) and each alone (device pointers), every frame of every clip against the oracle"""
    idx = SF.bin_sets()[(setname, mode)]
    rep = SF.Report()
    shapes = [(T, B) for T in SF.CLIP_T for B in (1, 3)] if mode == "full" else [(33, 3), (97, 3)]
    for T, B in shapes:
        x, ph, fre = SF.clips(setname, T, B)
        s = SF.spectral(x.shape[-1], fre, idx, mode)
        variants = _variants(ph)
        assert len(variants) <= 64
        label = f"{setname}/{mode} T={T} B={B}"
        _check(rep, label + " one call", x, ph, fre, idx, variants, SF.batch_call(s, x, ph, variants))
        alone = {i: SF.batch_call(s, x, ph, [v], device=True)[0] for i, v in enumerate(variants)}
        _check(rep, label + " alone", x, ph, fre, idx, variants, alone)
    _finish(rep)


@pytest.mark.parametrize("setname", ["linear", "mel"])
def test_temporal_steps_across_tiles(product_lib, cuda_device, setname):
    """flux / sd / sf / novelty with step 1, 2, 31, 32, 33, T - 1, T, T + 5: frames t < step are 0, the others read
    row t - step of the same clip, in an earlier tile or (never) in the previous clip"""
    rep = SF.Report()
    for T in (33, 64, 65, 97, 465):
        x, ph, fre = SF.clips(setname, T, 3, seed=1)
        idx = list(range(x.shape[-1]))
        variants = SF.temporal_variants(T)
        got = SF.batch_call(SF.spectral(x.shape[-1], fre, idx, "full"), x, None, variants)
        _check(rep, f"{setname} T={T}", x, None, fre, idx, variants, got)
    _finish(rep)


@pytest.mark.parametrize("kind", ["nan", "neg"])
def test_rolloff_look_back_runs(product_lib, cuda_device, kind):
    """rolloff on runs of 5 .. 70 frames that never cross (rows holding a NaN; or positive rows under threshold 1.5,
    the crossing rows holding negative bins): each takes the bin of the last crossing frame of its clip, fre[0] before
    any, however many 32-frame rounds the look-back needs"""
    x, fre, thr, cross = SF.lookback_clips(kind)
    idx = list(range(x.shape[-1]))
    variants = SF.LOOKBACK_VARIANTS[kind] or _variants(None)
    rep = SF.Report()
    s = SF.spectral(x.shape[-1], fre, idx, "full")
    _check(rep, f"lookback/{kind}", x, None, fre, idx, variants, SF.batch_call(s, x, None, variants))
    r = SF.batch_call(s, x, None, [("rolloff", dict(threshold=thr))], device=True)[0][0]
    for b in range(2):          # the look-back really falls back: runs hold the bin of the frame before them
        t = np.flatnonzero(~cross[b])
        prev = np.array([max((u for u in range(tt) if cross[b, u]), default=-1) for tt in t])
        want = np.where(prev >= 0, r[b][np.maximum(prev, 0)], fre[0])
        assert np.array_equal(r[b][t], want), (kind, b)
    _finish(rep)


@pytest.mark.parametrize("mode", list(SF.extreme_modes()))
def test_crafted_rows(product_lib, cuda_device, mode):
    """NaN at list position 0 (max keeps it) and mid-list, +-inf, denormals, small negative bins, zero frames next to
    loud ones, and the largest value at several positions across lanes and within a lane (the first position wins)"""
    idx = SF.extreme_modes()[mode]
    x, ph, fre = SF.extreme_clip(mode)
    x, ph = x[None], ph[None]
    variants = _variants(ph)
    rep = SF.Report()
    s = SF.spectral(x.shape[-1], fre, idx, mode)
    _check(rep, f"crafted/{mode} one call", x, ph, fre, idx, variants, SF.batch_call(s, x, ph, variants))
    alone = {i: SF.batch_call(s, x, ph, [v])[0] for i, v in enumerate(variants)}
    _check(rep, f"crafted/{mode} alone", x, ph, fre, idx, variants, alone)
    _finish(rep)


def test_legacy_entry_points_long_clips(product_lib, cuda_device):
    """the reference's per-feature entry points at T = 465 against the oracle and, when built, the reference"""
    ref = ref_lib_or_none()
    rep = SF.Report()
    for setname in ("linear", "mel", "cqt"):
        x, ph, fre = SF.clips(setname, 465, 1, seed=2)
        x, ph = x[0], None if ph is None else ph[0]
        for mode in ("full", "list"):
            idx = SC.edges(x.shape[-1])[mode]
            for name, kw in _variants(ph):
                got = SC.call_c(product_lib, name, x, fre, mode, ph, **kw)
                got = got if isinstance(got, tuple) else (got,)
                SF.check_clip(rep, f"legacy {setname}/{mode}", name, kw, got, x, idx, fre, ph)
                if ref is not None:
                    r = SC.call_c(ref, name, x, fre, mode, ph, **kw)
                    r = r if isinstance(r, tuple) else (r,)
                    rep.check(f"legacy-vs-reference {setname}/{mode}", name, kw, got, r,
                              SF.mags_of(name, kw, x, idx, fre))
    _finish(rep)


def test_prefilled_outputs(product_lib, cuda_device):
    """broadband adds its counts into the output from frame 1 on; pd / wpd / nwpd leave frame 1 as it was; var over
    one bin leaves every frame"""
    rng = np.random.default_rng(3)
    rep = SF.Report()
    for setname, mode, variants in (("linear", "full", [("broadband", {}), ("broadband", dict(threshold=3.)),
                                                        ("pd", {}), ("wpd", {}), ("nwpd", {})]),
                                    ("linear", "one", [("var", {}), ("broadband", {})])):
        idx = SF.bin_sets()[(setname, mode)]
        for T, B in ((65, 3), (33, 1)):
            x, ph, fre = SF.clips(setname, T, B, seed=4)
            planes = [2 if n in SC.TWO_OUTPUTS else 1 for n, _ in variants]
            out0 = rng.uniform(-5, 5, (sum(planes), B, T)).astype(np.float32)
            s = SF.spectral(x.shape[-1], fre, idx, mode)
            for device in (False, True):
                got = SF.batch_call(s, x, ph, variants, out0=out0, device=device)
                pre, k = {}, 0
                for i, n in enumerate(planes):
                    pre[i] = out0[k:k + n]
                    k += n
                _check(rep, f"prefilled {setname}/{mode} T={T} B={B} device={device}", x, ph, fre, idx, variants,
                       got, prefill=pre)
    _finish(rep)


def test_host_batch_of_three_chunks_against_oracle(product_lib, cuda_device):
    """one host-pointer call on T = 465 clips that the staging pipeline splits into three chunks (about 64 MB of
    input each, a multiple of 16 clips): the clips on both sides of each chunk edge against the oracle"""
    T, num = 465, 84
    per = (64 << 20) // (T * num * 4)
    per -= per % 16
    B = 2 * per + per // 2 + 1
    x, _, fre = SF.clips("cqt", T, B, seed=5)
    idx = list(range(num))
    variants = [("rolloff", {}), ("centroid", {}), ("flux", dict(step=33)), ("max", {}), ("slope", {}), ("mkl", {})]
    got = SF.batch_call(SF.spectral(num, fre, idx, "full"), x, None, variants)
    rep = SF.Report()
    for b in sorted({0, per - 1, per, 2 * per - 1, 2 * per, B - 1}):
        for i, (name, kw) in enumerate(variants):
            SF.check_clip(rep, f"staged clip {b}", name, kw, [g[b] for g in got[i]], x[b], idx, fre)
    _finish(rep)
