"""Every CQT octave kernel and tile variant, by name, column by column against the float64 oracle.

Each octave runs on the kernel and tile cqtObj_octavePlan reports (wgmma, mma.sync, the FP32 loop or the direct kernel;
the configurations and the pinned plan table are in tests/test_cqt_octave_plan.py).  Every case first asserts that its
plan holds the variant it claims to test, then compares the output per (clip, bin) column over the column's T frames:
max |got - want| (complex) <= 1e-4 * the column's own max |want|.  An octave is one launch on one decimated signal, so a
wrong octave kernel is wrong on its bins only, and those bins may sit far below the plane's maximum (the low octaves,
bins away from a tone, is_scale off); the per-tensor bar is kept too, so a failure shows which bar broke.  Columns the
oracle gives as exactly zero must come out below 1e-20.  The run prints the worst column of every octave with its
planned kernel and tile.
"""
import numpy as np
import pytest

import audioflux_b200 as af
from conftest import noise, rel_max, tones
from oracle import af_oracle as O
from test_cqt_octave_plan import CASES, J72, make, reference_buffer_fits, variants
from test_gpu_long_transforms import report, row_rel, torch_cuda  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

TOL = 1e-4
ZERO_COL = 1e-20


def bpo_of(cfg):
    return cfg.get("bin_per_octave", 12)


def oracle(cfg, x, is_continue=False, **kw):
    """float64 oracle of one clip -> (re, im) [T, num]"""
    return O.cqt(x, cfg["num"], cfg["samplate"], cfg.get("low_fre", 32.703196), bpo_of(cfg), cfg.get("factor", 1.0),
                 kw.get("beta", 0.0), hop=cfg.get("slide_length"), norm=O.NORM_AREA, is_scale=kw.get("is_scale", True),
                 is_continue=is_continue)


def label(o):
    if o["kernel"] == "direct":
        return f"hop {o['hop']} direct"
    return f"hop {o['hop']} {o['kernel']} TT {o['frames']} x{o['threads']} segs {o['segs']} {o['smem'] // 1024} KB"


def check_columns(report, case, plan, bpo, got_re, got_im, want_re, want_im):
    """Per-column and per-tensor bar on planes [clips, T, num]; prints the worst column of every octave."""
    got_re, got_im = (np.asarray(a.cpu().numpy() if hasattr(a, "cpu") else a) for a in (got_re, got_im))
    want_re, want_im = np.asarray(want_re), np.asarray(want_im)
    assert got_re.shape == want_re.shape, (case, got_re.shape, want_re.shape)
    clips, T, num = want_re.shape
    col = lambda a: np.ascontiguousarray(np.swapaxes(a, 1, 2))          # [clips, num, T]: time along the last axis
    rel, zero = row_rel(col(got_re), col(got_im), col(want_re), col(want_im))
    rel, zero = rel.reshape(clips, num), zero.reshape(clips, num)
    tensor = max(rel_max(got_re, want_re), rel_max(got_im, want_im))
    octs = num // bpo
    for k, o in enumerate(plan):                                        # plan: top octave first
        bins = slice((octs - 1 - k) * bpo, (octs - k) * bpo)
        r, z = rel[:, bins], zero[:, bins]
        report(f"{case} T {T} octave {k} {label(o)}", float(r[~z].max()) if (~z).any() else 0.0, tensor)
    assert tensor < TOL, (case, "per tensor", tensor)
    bad = np.argwhere(~zero & (rel >= TOL))
    assert bad.size == 0, (case, "(clip, bin) columns above the per-column bar", bad[:20].tolist(),
                           rel[tuple(bad[:20].T)].tolist())
    assert not zero.any() or rel[zero].max() < ZERO_COL, (case, "all-zero columns", np.argwhere(zero)[:20].tolist())


def clips(cfg, L, n=3, seed=0):
    """n clips of L samples: white noise, the last one tones()"""
    return np.stack([noise(seed + 100 + i, L) for i in range(n - 1)] + [tones(seed + 100, L, cfg["samplate"])])


def run(torch, cfg, x, **kw):
    c = make(cfg, **kw)
    re, im = c.cqt_batch(torch.from_numpy(x).cuda())
    torch.cuda.synchronize()
    return c, re, im


def assert_claims(cfg, plan, claims):
    have = set().union(*(variants(cfg, o) for o in plan))
    assert set(claims) <= have, ("plan lacks the claimed variants", sorted(set(claims) - have), plan)


# ------------------------------------------------------------------ 1. the matrix, per column
# (id, configuration, clip length, variants the case claims).  T = L // hop + 1 frames in every octave; L is odd and
# chosen so that the octaves with the widest tile still span two or more CTAs plus a partial tile.
MATRIX = [
    ("A", CASES["A"][0], 70221, ["wgmma 2x2 227 KB", "wgmma 2x1 113 KB", "wgmma 2x2 113 KB", "wgmma polyphase", "wgmma linear"]),
    ("B", CASES["B"][0], 70367, ["wgmma linear", "loop TT 512", "loop shift polyphase split"]),
    ("C", CASES["C"][0], 9569, ["wgmma 1x1 113 KB"]),
    ("D", CASES["D"][0], 38277, ["wgmma 2x1 227 KB"]),
    ("E", CASES["E"][0], 9553, ["wgmma 1x1 227 KB"]),
    ("F", CASES["F"][0], 76555, ["mma.sync 1 warps", "wgmma 2x2 227 KB"]),
    ("G-2warps", CASES["G"][0], 76675, ["mma.sync 2 warps", "mma.sync 8 warps"]),
    ("G-linear", CASES["G"][1], 9589, ["mma.sync 8 warps", "mma.sync linear"]),
    ("H", CASES["H"][0], 70345, ["mma.sync 8 warps", "mma.sync polyphase", "mma.sync linear", "loop TT 512"]),
    ("I", CASES["I"][0], 599321, ["loop division polyphase split", "loop segs 1", "loop segs 2", "loop segs 4",
                                  "loop TT 32", "loop TT 64", "loop TT 128", "loop TT 256", "loop TT 512"]),
    ("J", CASES["J"][0], 105545, ["loop division polyphase split", "loop pitch hop < 32", "loop pitch hop >= 32"]),
    ("K-segs8", CASES["K"][0], 77923, ["loop TT 8", "loop segs 8", "loop shift polyphase split", "direct power-of-two hop"]),
    ("K-segs64", CASES["K"][1], 36123, ["loop TT 8", "loop TT 16", "loop segs 64", "loop 2 bin passes", "direct odd hop"]),
    ("L-pow2", CASES["L"][0], 90113, ["direct power-of-two hop"]),
    ("L-odd", CASES["L"][1], 27001, ["direct odd hop"]),
    ("M-3passes", CASES["M"][0], 70343, ["loop 3 bin passes", "loop TT 512", "loop segs 2"]),
    ("M-2passes", CASES["M"][1], 70343, ["loop 2 bin passes", "loop TT 256"]),
]


@pytest.mark.parametrize("case,cfg,L,claims", MATRIX, ids=[m[0] for m in MATRIX])
def test_octave_paths_per_column(torch_cuda, report, case, cfg, L, claims):
    torch = torch_cuda
    x = clips(cfg, L)
    c, re, im = run(torch, cfg, x)
    plan = c.octave_plan()
    assert_claims(cfg, plan, claims)
    want = [oracle(cfg, x[i]) for i in range(x.shape[0])]
    check_columns(report, case, plan, bpo_of(cfg), re, im, np.stack([w[0] for w in want]), np.stack([w[1] for w in want]))


@pytest.mark.parametrize("case", ["A", "I", "K-segs64"])
def test_octave_paths_per_column_unscaled(torch_cuda, report, case):
    """is_scale off: the low octaves come out sqrt(2^k) times the scaled ones, each bin without its 1 / sqrt(length)"""
    torch = torch_cuda
    _, cfg, L, _ = next(m for m in MATRIX if m[0] == case)
    x = clips(cfg, L)
    c, re, im = run(torch, cfg, x, is_scale=False)
    want = [oracle(cfg, x[i], is_scale=False) for i in range(x.shape[0])]
    check_columns(report, case + " unscaled", c.octave_plan(), bpo_of(cfg), re, im,
                  np.stack([w[0] for w in want]), np.stack([w[1] for w in want]))


# ------------------------------------------------------------------ 2. frame-tile edges of one octave
# (case, octave): T below one tile, a whole number of tiles, and one frame past it, in batches of 3 clips with odd L
EDGES = [("A", 0), ("A", 1), ("A", 5), ("C", 0), ("D", 0), ("E", 0), ("F", 0), ("G-2warps", 0), ("H", 0), ("H", 5),
         ("I", 0), ("I", 3), ("I", 5), ("J", 5), ("K-segs8", 1), ("K-segs64", 1), ("M-3passes", 0)]


@pytest.mark.parametrize("case,octave", EDGES, ids=[f"{c}-oct{k}" for c, k in EDGES])
def test_frame_tile_edges(torch_cuda, report, case, octave):
    torch = torch_cuda
    cfg = next(m[1] for m in MATRIX if m[0] == case)
    c = make(cfg)
    plan = c.octave_plan()
    tt, hop = plan[octave]["frames"], c.slide_length
    assert tt > 0
    for T in (max(1, tt - 3), 2 * tt, 2 * tt + 1):
        L = (T - 1) * hop + 1                      # T = L // hop + 1; odd, as every top hop here is even
        assert L % 2 == 1 and c.cal_time_length(L) == T
        x = clips(cfg, L, seed=T)
        _, re, im = run(torch, cfg, x)
        want = [oracle(cfg, x[i]) for i in range(3)]
        check_columns(report, f"{case} octave {octave} TT {tt}", plan, bpo_of(cfg), re, im,
                      np.stack([w[0] for w in want]), np.stack([w[1] for w in want]))


# ------------------------------------------------------------------ 3. bit-stability
@pytest.mark.parametrize("case", ["A", "F", "H", "I", "K-segs64", "L-odd", "M-3passes"])
def test_batch_is_bit_stable(torch_cuda, case):
    """a clip's output is the same bits alone, at any position of a batch, and through the legacy entry point"""
    torch = torch_cuda
    _, cfg, L, _ = next(m for m in MATRIX if m[0] == case)
    L = min(L, 40001)
    x = np.stack([noise(300 + i, L) for i in range(5)])
    c, re, im = run(torch, cfg, x)
    for i in range(5):
        r1, i1 = c.cqt_batch(torch.from_numpy(x[i:i + 1]).cuda())
        assert torch.equal(r1[0], re[i]) and torch.equal(i1[0], im[i]), (case, "single clip", i)
    r2, i2 = c.cqt_batch(torch.from_numpy(x[2:5]).cuda())
    assert torch.equal(r2, re[2:5]) and torch.equal(i2, im[2:5]), (case, "sub-batch at offset 2")
    lr, li = c.cqt_planes(x[3])
    assert np.array_equal(lr, re[3].cpu().numpy()) and np.array_equal(li, im[3].cpu().numpy()), (case, "cqt_planes")


# ------------------------------------------------------------------ 4. streaming and VQT on the same paths
@pytest.mark.parametrize("case,chunks", [("A", (20000, 9000, 31001, 700)), ("I", (30000, 12345, 50001, 999))])
def test_streaming_per_column(cuda_device, report, case, chunks):
    """is_continue (padLeft = 0, right padding) chunk by chunk against O.CqtStream"""
    cfg = CASES[case][0]
    c = make(cfg, is_continue=True)
    model = O.CqtStream(cfg["num"], cfg["samplate"], hop=cfg.get("slide_length"), norm=O.NORM_AREA)
    plan = c.octave_plan()
    x = noise(400, sum(chunks))
    pos, frames = 0, 0
    for n in chunks:
        piece = x[pos:pos + n]
        pos += n
        re, im = c.cqt_planes(piece)
        wr, wi = model.push(piece)
        assert re.shape == wr.shape, (case, n)
        if wr.size:
            frames += wr.shape[0]
            check_columns(report, f"{case} streaming +{n}", plan, 12, re[None], im[None], wr[None], wi[None])
    assert frames > 0


@pytest.mark.parametrize("case,kernel", [("A", "wgmma"), ("H", "mma.sync"), ("I", "fp32 loop")])
def test_vqt_per_column(torch_cuda, report, case, kernel):
    """beta 5: one kernel set per octave, at its offset into the wgmma images / mma.sync fragments / FP32 kernels"""
    torch = torch_cuda
    _, cfg, L, _ = next(m for m in MATRIX if m[0] == case)
    L = min(L, 150001)
    x = clips(cfg, L)
    c, re, im = run(torch, cfg, x, beta=5.0)
    plan = c.octave_plan()
    assert sum(o["kernel"] == kernel for o in plan) >= 6, plan
    want = [oracle(cfg, x[i], beta=5.0) for i in range(x.shape[0])]
    check_columns(report, case + " vqt", plan, 12, re, im, np.stack([w[0] for w in want]), np.stack([w[1] for w in want]))


# ------------------------------------------------------------------ 5. the reference build at non-power-of-two hops
# Per tensor only: per column the limit is the reference's own float32 radix-2 FFT (DESIGN section 2).  Lengths inside
# the reference's per-octave buffers (see test_cqt_octave_plan.py).
@pytest.mark.parametrize("cfg,L", [(CASES["I"][0], 47001), (CASES["J"][0], 191), (J72, 20011)], ids=["I", "J", "J72"])
def test_non_pow2_hops_against_reference_build(torch_cuda, ref_lib, cfg, L):
    torch = torch_cuda
    assert reference_buffer_fits(cfg, L)
    x = clips(cfg, L)
    _, re, im = run(torch, cfg, x)
    q = make(cfg, _lib=ref_lib)
    for i in range(x.shape[0]):
        rr, ri = q.cqt_planes(x[i])
        assert rel_max(re[i].cpu().numpy(), rr) < TOL and rel_max(im[i].cpu().numpy(), ri) < TOL, i
