"""Which kernel and tile computes each CQT octave (cqtObj_octavePlan), pinned per configuration; and the float64 oracle
pinned to the reference build at the non-power-of-two hops of the FP32 loop.

cqtObj_octavePlan and the compute path call the same planner (af_cqt_octave_plan, host/af_cqt.c), so the table below is
what cqtObj_cqtBatch launches.  A retune of any tile shows up here as a diff of the table.  The GPU side of the same
matrix is tests/test_gpu_cqt_octave_paths.py.  No test here needs a GPU.
"""
import numpy as np
import pytest

import audioflux_b200 as af
from conftest import noise, rel_max, tones
from oracle import af_oracle as O

KB = 1024

# case -> constructor arguments of af.CQT, one or two configurations per case
CASES = {
    "A": [dict(num=84, samplate=48000)],                                                    # bench.py C3, N 512
    "B": [dict(num=84, samplate=22050, slide_length=64)],                                   # N 256
    "C": [dict(num=12, samplate=8000, low_fre=65.4, factor=0.5, slide_length=64)],          # N 2048
    "D": [dict(num=12, samplate=8000, factor=0.5, slide_length=128)],                       # N 4096
    "E": [dict(num=12, samplate=8000, factor=4, slide_length=64)],                          # N 32768
    "F": [dict(num=36, samplate=48000, low_fre=261.6256)],                                  # N 1024
    "G": [dict(num=24, samplate=8000, low_fre=1000, factor=0.5, slide_length=128),          # N 64
          dict(num=36, samplate=16000, low_fre=1000, factor=0.5)],                          # N 64
    "H": [dict(num=84, samplate=8000, slide_length=64)],                                    # N 128
    "I": [dict(num=84, samplate=48000, slide_length=1000)],                                 # N 512
    "J": [dict(num=84, samplate=48000, slide_length=96)],                                   # N 512
    "K": [dict(num=24, samplate=8000, factor=4),                                            # N 16384
          dict(num=72, samplate=16000, bin_per_octave=24, factor=4, slide_length=1000)],    # N 32768
    "L": [dict(num=48, samplate=44100, bin_per_octave=24),                                  # N 32768
          dict(num=12, samplate=8000, slide_length=3000)],                                  # N 8192
    "M": [dict(num=36, bin_per_octave=36, samplate=8000, factor=0.25, slide_length=64),     # N 4096
          dict(num=48, bin_per_octave=24, samplate=8000, low_fre=1000, factor=0.5, slide_length=64)],   # N 128
}

WG, TC, LOOP, DIRECT = "wgmma", "mma.sync", "fp32 loop", "direct"
# per configuration: fftLength, then per octave (top octave first) (kernel, hop, frames per CTA, threads per CTA, segs)
PLANS = {
    "A": [(512, [(WG, 128, 256, 256, 1), (WG, 64, 128, 256, 1), (WG, 32, 256, 256, 1), (WG, 16, 256, 256, 1),
                 (WG, 8, 256, 256, 1), (WG, 4, 256, 256, 1), (WG, 2, 256, 256, 1)])],
    "B": [(256, [(WG, 64, 128, 256, 1), (WG, 32, 256, 256, 1), (WG, 16, 256, 256, 1), (WG, 8, 256, 256, 1),
                 (WG, 4, 256, 256, 1), (WG, 2, 256, 256, 1), (LOOP, 1, 512, 256, 1)])],
    "C": [(2048, [(WG, 64, 64, 128, 1)])],
    "D": [(4096, [(WG, 128, 128, 256, 1)])],
    "E": [(32768, [(WG, 64, 64, 128, 1)])],
    "F": [(1024, [(TC, 256, 32, 32, 1), (WG, 128, 256, 256, 1), (WG, 64, 128, 256, 1)])],
    "G": [(64, [(TC, 128, 64, 64, 1), (TC, 64, 256, 256, 1)]),
          (64, [(TC, 16, 256, 256, 1), (TC, 8, 256, 256, 1), (TC, 4, 256, 256, 1)])],
    "H": [(128, [(TC, 64, 256, 256, 1), (TC, 32, 256, 256, 1), (TC, 16, 256, 256, 1), (TC, 8, 256, 256, 1),
                 (TC, 4, 256, 256, 1), (TC, 2, 256, 256, 1), (LOOP, 1, 512, 256, 1)])],
    "I": [(512, [(LOOP, 1000, 32, 16, 1), (LOOP, 500, 64, 64, 2), (LOOP, 250, 128, 128, 2), (LOOP, 125, 256, 512, 4),
                 (LOOP, 62, 512, 512, 2), (LOOP, 31, 256, 512, 4), (LOOP, 15, 512, 512, 2)])],
    "J": [(512, [(LOOP, 96, 256, 512, 4), (LOOP, 48, 256, 512, 4), (LOOP, 24, 512, 512, 2), (LOOP, 12, 512, 512, 2),
                 (LOOP, 6, 512, 512, 2), (LOOP, 3, 512, 512, 2), (LOOP, 1, 512, 512, 2)])],
    "K": [(16384, [(DIRECT, 4096, 0, 256, 1), (LOOP, 2048, 8, 32, 8)]),
          (32768, [(DIRECT, 1000, 0, 256, 1), (LOOP, 500, 8, 256, 64), (LOOP, 250, 16, 512, 64)])],
    "L": [(32768, [(DIRECT, 8192, 0, 256, 1), (DIRECT, 4096, 0, 256, 1)]),
          (8192, [(DIRECT, 3000, 0, 256, 1)])],
    "M": [(4096, [(LOOP, 64, 512, 512, 2)]),
          (128, [(LOOP, 64, 256, 128, 1), (LOOP, 32, 512, 256, 1)])],
}


def make(cfg, **kw):
    return af.CQT(**cfg, **kw)


def variants(cfg, octave):
    """The tile variants one planned octave exercises (labels of the coverage table below)."""
    kernel, hop, tt, threads, segs, smem = (octave[k] for k in ("kernel", "hop", "frames", "threads", "segs", "smem"))
    layout = "polyphase" if hop >= 8 else "linear"
    if kernel == WG:
        wg = threads // 128
        return {f"wgmma {wg}x{tt // (64 * wg)} {'113' if smem <= 113 * KB else '227'} KB", f"wgmma {layout}"}
    if kernel == TC:
        return {f"mma.sync {threads // 32} warps", f"mma.sync {layout}"}
    pow2 = hop & (hop - 1) == 0
    if kernel == DIRECT:
        return {f"direct {'power-of-two' if pow2 else 'odd'} hop"}
    bpo = cfg.get("bin_per_octave", 12)
    return {f"loop TT {tt}", f"loop segs {segs}", f"loop {'shift' if pow2 else 'division'} polyphase split",
            f"loop pitch {'hop < 32' if hop < 32 else 'hop >= 32'}", f"loop {bpo // 12} bin passes"}


# Every tile variant the planner can choose, with the case that reaches it.  Left out, because no power-of-two fftLength
# reaches them: the 4-warp mma.sync tile (mma.sync runs only for fftLength 64 / 128 -- where 8 warps fit up to hop 64 and
# hop 128 needs 2 -- or for hops >= 256, where 1 warp is all that fits), and the linear wgmma tile with fewer than
# 2 x 2 m-tiles (a hop of 2 or 4 always fits the full tile under 113 KB).
REACHABLE = {
    "wgmma 2x2 113 KB": "A", "wgmma 2x2 227 KB": "A", "wgmma 2x1 113 KB": "A", "wgmma 2x1 227 KB": "D",
    "wgmma 1x1 113 KB": "C", "wgmma 1x1 227 KB": "E", "wgmma polyphase": "A", "wgmma linear": "A",
    "mma.sync 8 warps": "H", "mma.sync 2 warps": "G", "mma.sync 1 warps": "F",
    "mma.sync polyphase": "H", "mma.sync linear": "H",
    "loop TT 512": "B", "loop TT 256": "I", "loop TT 128": "I", "loop TT 64": "I", "loop TT 32": "I", "loop TT 16": "K",
    "loop TT 8": "K", "loop segs 1": "I", "loop segs 2": "I", "loop segs 4": "I", "loop segs 8": "K",
    "loop segs 64": "K", "loop shift polyphase split": "B", "loop division polyphase split": "I",
    "loop pitch hop < 32": "J", "loop pitch hop >= 32": "J",
    "loop 1 bin passes": "I", "loop 2 bin passes": "M", "loop 3 bin passes": "M",
    "direct power-of-two hop": "L", "direct odd hop": "L",
}


def plans(case):
    return [make(cfg).octave_plan() for cfg in CASES[case]]


@pytest.mark.parametrize("case", sorted(CASES))
def test_plan_table(case):
    for cfg, (n, want), plan in zip(CASES[case], PLANS[case], plans(case)):
        assert make(cfg).fft_length == n, (case, cfg)
        got = [(o["kernel"], o["hop"], o["frames"], o["threads"], o["segs"]) for o in plan]
        assert got == want, (case, cfg)
        for o in plan:
            assert 0 < o["threads"] <= 1024
            assert (o["smem"] == 0) == (o["kernel"] == DIRECT)
            assert o["smem"] <= 227 * KB


def test_every_reachable_variant_is_planned():
    seen = {}
    for case, cfgs in CASES.items():
        for cfg, plan in zip(cfgs, plans(case)):
            for o in plan:
                for v in variants(cfg, o):
                    seen.setdefault(v, case)
    assert set(seen) == set(REACHABLE), (sorted(set(REACHABLE) - set(seen)), sorted(set(seen) - set(REACHABLE)))
    for v, case in REACHABLE.items():
        assert any(v in variants(cfg, o) for cfg, plan in zip(CASES[case], plans(case)) for o in plan), (v, case)


def test_plan_hops_are_the_integer_halved_hop():
    c = make(CASES["I"][0])
    assert [o["hop"] for o in c.octave_plan()] == [1000, 500, 250, 125, 62, 31, 15]


def test_plan_query_arguments(product_lib):
    c = make(CASES["A"][0])
    kernel = np.zeros(7, np.int32)
    assert product_lib.cqtObj_octavePlan(c._obj, kernel.ctypes.data, None, None, None, None, None) == 7
    assert kernel.tolist() == [0] * 7
    assert product_lib.cqtObj_octavePlan(None, None, None, None, None, None, None) < 0


def test_plan_does_not_depend_on_scale_or_streaming():
    for case in ("A", "H", "I"):
        cfg = CASES[case][0]
        assert make(cfg, is_scale=False).octave_plan() == make(cfg).octave_plan()
        assert make(cfg, is_continue=True).octave_plan() == make(cfg).octave_plan()


# ---- the oracle against the reference build at non-power-of-two hops (cases I and J) ----
# integer hop halving (1000 -> 500 -> ... -> 15, 96 -> ... -> 3 -> 1), Tn = min(T, frames) and the tail dropped at every
# octave (valid = len - len % hop), centre-padded and streaming.
#
# The reference sizes its per-octave STFT buffers for the top octave's frames + 1 (cqt_algorithm.c:930-945).  When the
# integer halving makes a lower octave's hop less than half the one above (125 -> 62, 3 -> 1), that octave has more
# frames and the reference writes past its heap buffer once the clip is long enough.  The lengths below stay inside
# its buffers (`reference_buffer_fits`); the 84-bin case J (hop 1 at the bottom octave: 1.5x the top octave's frames)
# only does so for clips of a few frames (191 samples: its padding buffers also overflow at 319 once an object is
# reused), so J is also pinned with its first six octaves (72 bins, hops 96 ... 3).
J72 = dict(CASES["J"][0], num=72)


def reference_buffer_fits(cfg, L):
    hop, top = cfg["slide_length"], L // cfg["slide_length"] + 1
    for k in range(cfg["num"] // cfg.get("bin_per_octave", 12)):
        if (L >> k) // (hop >> k) + 1 > top + 1:
            return False
    return True


def _oracle_kw(cfg, is_scale=True):
    return dict(num=cfg["num"], sr=cfg["samplate"], hop=cfg["slide_length"], is_scale=is_scale, norm=O.NORM_AREA)


@pytest.mark.parametrize("cfg,L,signal", [(CASES["I"][0], 36001, "noise"), (CASES["I"][0], 47001, "tones"),
                                          (CASES["J"][0], 191, "noise"), (J72, 9601, "noise"), (J72, 20011, "tones")],
                         ids=["I-36001", "I-47001-tones", "J-191", "J72-9601", "J72-20011-tones"])
@pytest.mark.parametrize("is_scale", [True, False], ids=["scale", "noscale"])
def test_oracle_matches_reference_at_non_pow2_hops(ref_lib, cfg, L, signal, is_scale):
    assert reference_buffer_fits(cfg, L)
    x = noise(91, L) if signal == "noise" else tones(91, L, cfg["samplate"])
    rr, ri = make(cfg, is_scale=is_scale, _lib=ref_lib).cqt_planes(x)
    wr, wi = O.cqt(x, **_oracle_kw(cfg, is_scale))
    assert rr.shape == wr.shape == (L // cfg["slide_length"] + 1, cfg["num"])
    assert rel_max(wr, rr) < 1e-5 and rel_max(wi, ri) < 1e-5


@pytest.mark.parametrize("cfg,chunks", [(CASES["I"][0], (5000, 2600, 777, 9001)), (J72, (1000, 513, 4097, 700))],
                         ids=["I", "J72"])
def test_oracle_streaming_matches_reference_at_non_pow2_hops(ref_lib, cfg, chunks):
    """chunk by chunk through cqtObj_cqt(isContinue = 1); every chunk is at least one frame long (the reference
    corrupts its heap on shorter chunks)"""
    x = noise(92, sum(chunks))
    q = make(cfg, is_continue=True, _lib=ref_lib)
    model = O.CqtStream(cfg["num"], cfg["samplate"], hop=cfg["slide_length"], norm=O.NORM_AREA)
    pos, frames = 0, 0
    for n in chunks:
        piece = x[pos:pos + n]
        pos += n
        assert reference_buffer_fits(cfg, n + q.fft_length)
        rr, ri = q.cqt_planes(piece)
        wr, wi = model.push(piece)
        assert rr.shape == wr.shape
        frames += rr.shape[0]
        if rr.size:
            assert rel_max(wr, rr) < 1e-5 and rel_max(wi, ri) < 1e-5
    assert frames > 0
