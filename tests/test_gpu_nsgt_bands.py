"""The NSGT band kernels (k_nsgt_bluestein, k_nsgt_direct in kernels/nsgt.cu) band by band against the float64 oracle.

The per-tensor bar of test_gpu_nsgt.py is set by the loudest band.  On tonal clips a third or more of the bands of an
Octave 84 bank peak below 1e-2 of the matrix maximum, so a quiet band could be wrong by a few percent of its own scale
and pass.  Here every band of every clip is held to 1e-4 of its own max |want|, and a band the oracle gives as exactly
zero must be exactly zero (`_nsgt_oracle.check_bands`).

The oracle's band step runs on the GPU's own spectrum: `STFT.stft_batch` with a rect window and a hop of one frame makes
the same af_launch_stft call as nsgtObj_nsgtBatch.  The forward FFT's error scales with the whole spectrum, so it is
kept out of a quiet band's bar.  White-noise clips, where every band sits at a comparable level, are also checked end to
end against the float64 FFT of the clip.

Every case runs 3 clips in one call, the second scaled by 1e3 (a mixed-up clip index shows), checks every band of every
clip and asserts that the matrix is the gather of the cells, bit for bit.  What is covered:
  - a length sweep on one object through set_min_length: every Bluestein size M = 8 ... 8192 on both sides of each
    doubling, and direct lengths that need one, two and three passes of 6144 outputs.  All direct lengths exceed the
    2^12-point clip, so they also read the clamp at bin N - 1 and the conjugate mirror above N/2;
  - two 2^18 banks whose launches mix Bluestein groups of many sizes with direct bands of many lengths;
  - group packing: 2000 bands of 3 points (M = 8: groups of 1024 and 976 bands), two bands of M = 4096 per group with an
    odd band count, and banks with bands of 1 and 2 points, some with all-zero windows.
The CPU tests pin the lengths every configuration claims, through libaudioflux_b200.so's getters and the oracle's bank,
so that a change to a bank cannot silently drop coverage.  The run prints the worst band error per kernel path.
"""
import numpy as np
import pytest

import _nsgt_oracle as NO
import audioflux_b200 as af
from conftest import noise
from oracle import af_oracle as O
from test_gpu_nsgt import _cell_gather, _gpu_spectrum

gpu = pytest.mark.gpu

# Linear, 24 bands at 2^12: every natural length is 3, so set_min_length(L) makes every band exactly L points long
SWEEP = dict(num=24, radix2_exp=12, samplate=32000, min_len=1, scale_type=O.SCALE_LINEAR, style_type=O.STYLE_HANN,
             normal_type=O.NORM_NONE)
SWEEP_BLUESTEIN = (3, 4, 5, 8, 9, 16, 17, 32, 33, 64, 65, 128, 129, 256, 257, 512, 513, 1024, 1025, 2048, 2049, 4095, 4096)
SWEEP_DIRECT = (4097, 4160, 5120, 6143, 6144, 6145, 8192, 12287, 12288, 12289, 16383, 16384)
SWEEP_LENGTHS = SWEEP_BLUESTEIN + SWEEP_DIRECT
SWEEP_FRESH = (12289, 5, 4097, 4096)            # rebuilt upwards and downwards, then compared with a fresh object
SWEEP_END_TO_END = (513, 6145, 16384)

# 2^18 banks: (kw, (shortest, longest, direct bands, bands needing three direct passes))
MIXED = {
    "log120": (dict(num=120, radix2_exp=18, samplate=44100, low_fre=32.703196, scale_type=O.SCALE_LOG,
                    style_type=O.STYLE_HANN), (23, 14749, 24, 4)),
    "mel60": (dict(num=60, radix2_exp=18, samplate=22050, scale_type=O.SCALE_MEL, style_type=O.STYLE_SLANEY),
              (825, 12589, 25, 1)),
}

# uniform banks: (kw, the length of every band).  Bluestein groups are runs of consecutive bands with sum M <= 8192:
# 2000 bands of M = 8 make one group of 1024 bands and one of 976; 7 bands of M = 4096 make three pairs and a single
PACKING = {
    "lin2000_L3": (dict(num=2000, radix2_exp=12, samplate=32000, min_len=3, scale_type=O.SCALE_LINEAR,
                        style_type=O.STYLE_HANN, normal_type=O.NORM_NONE), 3),
    "lin7_L1025": (dict(SWEEP, num=7, min_len=1025), 1025),
    "lin7_L2048": (dict(SWEEP, num=7, min_len=2048), 2048),
}

# banks with bands of 1 and 2 points: cases of _nsgt_oracle.cases(), and Bark with ETSI windows at minLen 2, whose
# 2-point symmetric Bartlett windows are [0, 0]
TINY = {name: kw for name, kw in NO.cases() if name in ("b0s5t1", "b0s6t3", "b1s4t1", "b1s5t0", "b1s5t3")}
TINY["b0s5t1_etsi2"] = dict(TINY["b0s5t1"], min_len=2, style_type=O.STYLE_ETSI)


def make(kw):
    """af.NSGT from a keyword set of _nsgt_oracle.params (nsgtObj_new's defaults where kw leaves a value out)"""
    return af.NSGT(num=kw["num"], radix2_exp=kw["radix2_exp"], samplate=kw.get("samplate") or 32000,
                   low_fre=kw.get("low_fre"), high_fre=kw.get("high_fre"), bin_per_octave=kw.get("bin_per_octave") or 12,
                   min_len=kw.get("min_len") or 3, nsgt_filter_bank_type=kw.get("bank_type") or NO.EFFICIENT,
                   scale_type=kw.get("scale_type", O.SCALE_OCTAVE), style_type=kw.get("style_type", O.STYLE_HANN),
                   normal_type=kw.get("normal_type", O.NORM_BANDWIDTH))


def params_of(t):
    """the oracle's parameters of what the object passed to nsgtObj_new (and its current minimum length)"""
    ev = af.enum_value
    st, p = NO.params(num=t.num, radix2_exp=t.radix2_exp, samplate=t.samplate, low_fre=t.low_fre, high_fre=t.high_fre,
                      bin_per_octave=t.bin_per_octave, min_len=t.min_len, bank_type=ev(t.nsgt_filter_bank_type),
                      scale_type=ev(t.scale_type), style_type=ev(t.style_type), normal_type=ev(t.normal_type))
    assert st == 0
    return p


def lengths(t):
    """the band lengths from the library's getter, checked against the oracle's bank"""
    lens = t.get_time_length_arr()
    assert np.array_equal(lens, NO.bank(params_of(t))["lens"])
    assert t.get_max_time_length() == lens.max() and t.get_total_time_length() == lens.sum()
    return lens


def mixed_claims(lens):
    return (int(lens.min()), int(lens.max()), int((lens > NO.BLUESTEIN_MAX).sum()), int((lens > 2 * NO.DIRECT_PASS).sum()))


def clips(n, sr, white=False, seed=0):
    """3 clips for one device call, the second scaled by 1e3: tones over noise, or white noise"""
    x = np.stack([noise(seed + s, n) if white else NO.case_signal(seed + s, n, sr) for s in range(3)])
    x[1] *= 1e3
    return x


@pytest.fixture
def report(request, capsys):
    """report(case, {path: worst band error}): prints it past pytest's capture and records it"""
    def emit(case, worst):
        for path, e in worst.items():
            request.node.user_properties.append((f"{case} {path}", e))
        with capsys.disabled():
            order = sorted(worst, key=lambda path: (len(path), path))          # M = 2^3 before M = 2^10
            print(f"\n    {case}: " + ", ".join(f"{path} {worst[path]:.2e}" for path in order), end="")
    return emit


def check_case(report, case, t, x, X=None):
    """every band of every clip of one nsgt_batch call against the oracle's band step on X (default: the GPU's own
    spectrum of x), and the matrix against the gather of the cells"""
    p = params_of(t)
    b = NO.bank(p)
    lens = b["lens"]
    assert np.array_equal(lens, t.get_time_length_arr()), case
    re, im, cr, ci = t.nsgt_batch(x, with_cells=True)
    X = _gpu_spectrum(x) if X is None else X
    cmap = NO.column_map(lens, p["fft_length"], p["samplate"])
    worst = {}
    for c in range(len(x)):
        assert np.array_equal(re[c] + 1j * im[c], _cell_gather(cr[c], ci[c], lens, cmap)), (case, c)
        want, _ = NO.transform_spectrum(X[c], p, b)
        for path, e in NO.check_bands(NO.split_cells(cr[c], ci[c], lens), want, lens, what=f"{case} clip {c}").items():
            worst[path] = max(worst.get(path, 0.0), e)
    report(case, worst)
    return re, im


# ------------------------------------------------------------------ CPU: the coverage each configuration claims
def test_sweep_lengths_reach_their_paths(product_lib):
    t = make(SWEEP)
    assert (lengths(t) == 3).all()
    for L in SWEEP_LENGTHS:
        t.set_min_length(L)
        assert (lengths(t) == L).all(), L
    # every Bluestein size, from both sides of each doubling of M
    assert sorted({NO.log2_m(L) for L in SWEEP_BLUESTEIN}) == list(range(3, 14))
    for k in range(2, 12):
        assert {1 << k, (1 << k) + 1} <= set(SWEEP_BLUESTEIN) and NO.log2_m((1 << k) + 1) == NO.log2_m(1 << k) + 1
    assert {4095, 4096, 4097} <= set(SWEEP_LENGTHS) and max(SWEEP_BLUESTEIN) == NO.BLUESTEIN_MAX
    # one, two and three direct passes, each at its edges; the coarse / fine twiddle split, a whole number of tiles
    assert all(L > NO.BLUESTEIN_MAX for L in SWEEP_DIRECT)
    P = NO.DIRECT_PASS
    assert {P - 1, P, P + 1, 2 * P - 1, 2 * P, 2 * P + 1, NO.MAX_LEN - 1, NO.MAX_LEN} <= set(SWEEP_DIRECT)
    assert {NO.band_path(L) for L in SWEEP_DIRECT} == {"direct 1 pass", "direct 2 passes", "direct 3 passes"}
    assert 4160 == 65 * 64 and 5120 % 1024 == 0
    # longer than the clip: the bands read the clamp at N - 1 and the mirror above N/2
    assert min(SWEEP_DIRECT) > 1 << SWEEP["radix2_exp"]
    assert set(SWEEP_FRESH) <= set(SWEEP_LENGTHS) and set(SWEEP_END_TO_END) <= set(SWEEP_LENGTHS)


@pytest.mark.parametrize("name", MIXED)
def test_mixed_banks_reach_their_lengths(product_lib, name):
    kw, claims = MIXED[name]
    assert mixed_claims(lengths(make(kw))) == claims
    _, p = NO.params(**kw)
    assert mixed_claims(NO.bank(p)["lens"]) == claims


@pytest.mark.parametrize("name", PACKING)
def test_packing_banks_reach_their_lengths(product_lib, name):
    kw, L = PACKING[name]
    assert (lengths(make(kw)) == L).all()
    assert (NO.bank(NO.params(**kw)[1])["lens"] == L).all()
    M = 1 << NO.log2_m(L)
    assert kw["num"] * M > 8192 and kw["num"] % (8192 // M) != 0       # more than one group, the last one short


def test_tiny_banks_reach_their_lengths(product_lib):
    seen, zero = set(), 0
    for name, kw in TINY.items():
        lens = lengths(make(kw))
        assert lens.min() <= 2, name
        seen |= set(lens.tolist())
        zero += sum(not np.any(w) for w in NO.bank(NO.params(**kw)[1])["windows"])
    assert {1, 2} <= seen and zero > 0


# ------------------------------------------------------------------ GPU
@gpu
def test_size_one_bands_equal_the_stft_bins(cuda_device):
    """The premise of feeding the oracle the GPU's spectrum: a 1-point Bluestein transform is exact (c0 = 1, H = 1), so
    the 1-point rect bands of this bank are the bins of STFT.stft_batch themselves, bit for bit."""
    t = make(dict(num=84, radix2_exp=12, samplate=32000, min_len=1, scale_type=O.SCALE_OCTAVE,
                  style_type=O.STYLE_RECT, normal_type=O.NORM_NONE))
    lens = lengths(t)
    one = np.flatnonzero(lens == 1)
    bins = t.get_bin_band_arr()[one]
    assert bins.tolist() == [4, 5, 6, 7]
    x = clips(1 << 12, 32000)
    _, _, cr, ci = t.nsgt_batch(x, with_cells=True)
    sre, sim = af.STFT(12, af.WindowType.RECT, 1 << 12).stft_batch(x)
    off = np.concatenate([[0], np.cumsum(lens)[:-1]])[one]
    for c in range(len(x)):
        assert np.array_equal(cr[c][off], sre[c, 0, bins]) and np.array_equal(ci[c][off], sim[c, 0, bins]), c


@pytest.fixture(scope="module")
def sweep(cuda_device):
    """one object for the whole sweep, its clips and their GPU spectrum"""
    t = make(SWEEP)
    x = clips(1 << SWEEP["radix2_exp"], SWEEP["samplate"])
    return t, x, _gpu_spectrum(x)


@gpu
@pytest.mark.parametrize("L", SWEEP_LENGTHS)
def test_length_sweep(sweep, report, L):
    t, x, X = sweep
    t.set_min_length(L)
    assert (t.get_time_length_arr() == L).all()
    check_case(report, f"L={L}", t, x, X)


@gpu
def test_length_sweep_rebuild_equals_fresh_object(sweep):
    t, x, _ = sweep
    for L in SWEEP_FRESH:
        t.set_min_length(L)
        got = t.nsgt_batch(x, with_cells=True)
        want = make(dict(SWEEP, min_len=L)).nsgt_batch(x, with_cells=True)
        for g, w in zip(got, want):
            assert np.array_equal(g, w), L


@gpu
@pytest.mark.parametrize("name", MIXED)
def test_mixed_banks_2e18(cuda_device, report, name):
    kw, claims = MIXED[name]
    t = make(kw)
    assert mixed_claims(lengths(t)) == claims
    check_case(report, name, t, clips(1 << kw["radix2_exp"], kw["samplate"]))


@gpu
@pytest.mark.parametrize("name", PACKING)
def test_group_packing(cuda_device, report, name):
    kw, L = PACKING[name]
    t = make(kw)
    assert (lengths(t) == L).all()
    check_case(report, name, t, clips(1 << kw["radix2_exp"], kw["samplate"]))


@gpu
@pytest.mark.parametrize("name", TINY)
def test_tiny_bands(cuda_device, report, name):
    kw = TINY[name]
    t = make(kw)
    assert lengths(t).min() <= 2
    check_case(report, name, t, clips(1 << kw["radix2_exp"], kw.get("samplate") or 32000))


END_TO_END = [(name, kw) for name, (kw, _) in MIXED.items()] + [(f"L={L}", dict(SWEEP, min_len=L))
                                                                  for L in SWEEP_END_TO_END]


@gpu
@pytest.mark.parametrize("name,kw", END_TO_END, ids=[c[0] for c in END_TO_END])
def test_end_to_end_white_noise(cuda_device, report, name, kw):
    """the same per-band bar against the float64 FFT of white-noise clips: the forward FFT and the bands together"""
    t = make(kw)
    x = clips(1 << kw["radix2_exp"], kw["samplate"], white=True, seed=10)
    check_case(report, f"{name} end to end", t, x, np.fft.fft(x.astype(np.float64)))
