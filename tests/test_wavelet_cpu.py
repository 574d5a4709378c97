"""Discrete wavelet transforms without a GPU: the generated filters (audioflux_b200/csrc/kernels/wavelet_coef_gen.h)
against the reference's dwt_filterCoef for every supported combination; the refusals of every other listed one; the
float64 oracle against the reference build (or its stored outputs in tests/golden/wavelet.npz) over every family,
radix2Exp 2 .. 16 and num 1 .. radix2Exp-1; the modulo indexing the kernels use against the literal padding; the
vectorised level steps and mDataArr index map of the level-by-level GPU suite against the literal oracle; the
constructor statuses against the reference; and the symbols of the three headers."""
import os
import re

import numpy as np
import pytest

import _wavelet_oracle as W
from _parity_kit import GoldenStore, check_symbols, ref_lib_or_none
from conftest import ROOT

from audioflux_b200 import capi

TOL = 1e-5                 # of max |value| of the output
GEN = os.path.join(ROOT, "audioflux_b200", "csrc", "kernels", "wavelet_coef_gen.h")


def generated():
    """{(type, t1, t2): (loD, hiD)} and {(type, t1, t2): reason} of the generated header"""
    src = open(GEN).read()
    arrays = {m.group(1): np.array([float(v.rstrip("f")) for v in m.group(2).split(",")], np.float32)
              for m in re.finditer(r"static const float (\w+)\[\d+\] = \{([^}]*)\};", src)}
    table = {}
    for m in re.finditer(r"\{(\d+), (\d+), (\d+), (\d+), (\w+)_lo, (\w+)_hi\}", src):
        table[tuple(map(int, m.groups()[:3]))] = (arrays[m.group(5) + "_lo"], arrays[m.group(5) + "_hi"])
    refused = {tuple(map(int, m.groups()[:3])): m.group(4)
               for m in re.finditer(r'\{(\d+), (\d+), (\d+), "([^"]*)"\}', src)}
    return table, refused


TABLE, REFUSED = generated()
KINDS = ("dwt", "wpt", "swt")


def _ref_key(k):
    ty, t1, t2 = k
    return ty, (1 if ty in (0, 6) else t1), t2


def cases():
    """(name, (kind, num, size, type, t1, t2, seed)): every supported filter on each object, and the sizes"""
    out = []
    fams = sorted(TABLE)
    for i, (ty, t1, t2) in enumerate(fams):
        e = 6 + i % 5
        out.append((f"dwt_{ty}_{t1}_{t2}", ("dwt", e - 1 - i % 3, e, ty, t1, t2, i)))
        out.append((f"wpt_{ty}_{t1}_{t2}", ("wpt", 1 + i % 4, e, ty, t1, t2, i)))
        out.append((f"swt_{ty}_{t1}_{t2}", ("swt", 1 + i % 5, 96 * (1 + i % 3), ty, t1, t2, i)))
    for e in range(2, 17):
        for num in sorted({1, (e - 1 + 1) // 2, e - 1}):
            if num >= 1:
                out.append((f"dwt_e{e}_n{num}", ("dwt", num, e, 2, 4, 0, e)))
                if e <= 12:
                    out.append((f"wpt_e{e}_n{num}", ("wpt", min(num, 6), e, 1, 2, 0, e)))
    for n, num in ((2, 1), (64, 6), (1000, 3), (4096, 8), (1 << 14, 8)):
        out.append((f"swt_n{n}_l{num}", ("swt", num, n, 2, 4, 0, n)))
    return out


CASES = dict(cases())


def _live(keys):
    lib = ref_lib_or_none()
    out = {}
    for k in keys:
        if k.startswith("coef/"):
            ty, t1, t2 = map(int, k.split("/")[1].split("_"))
            lo, hi = W.filters(lib, ty, t1, t2)
            out[k] = np.stack([lo, hi])
        else:
            kind, num, size, ty, t1, t2, seed = CASES[k.split("/")[1]]
            n = size if kind == "swt" else 1 << size
            a, b = W.run(lib, kind, num, size, ty, t1, t2, W.signal(n, seed))
            out[k] = np.concatenate([a.ravel(), b.ravel()])
    return out


def _outputs(kind, num, size, *_):
    n = size if kind == "swt" else 1 << size
    return n * (2 * num if kind == "swt" else 1 + (num if kind == "dwt" else 1 << num))


def _golden_keys():
    """the filters, and the cases of up to 2^14 output floats (the larger ones need the reference build)"""
    return {f"coef/{a}_{b}_{c}" for a, b, c in map(_ref_key, TABLE)} | \
        {f"case/{n}" for n, c in CASES.items() if _outputs(*c) <= 1 << 14}


GOLD = GoldenStore("wavelet.npz", _live, _golden_keys)


def oracle(kind, num, size, ty, t1, t2, seed):
    lo, hi = (v.astype(np.float64) for v in TABLE[(ty, t1, t2)])
    n = size if kind == "swt" else 1 << size
    a, b = getattr(W, kind)(W.signal(n, seed).astype(np.float64), num, lo, hi)
    return np.concatenate([a.ravel(), b.ravel()])


def test_case_coverage():
    assert len(CASES) >= 40
    assert {c[0] for c in CASES.values()} == set(KINDS)
    assert {c[3] for c in CASES.values()} == {0, 1, 2, 5}
    assert {c[2] for c in CASES.values() if c[0] == "dwt"} >= set(range(2, 17))


@pytest.mark.parametrize("key", sorted(TABLE), ids=lambda k: "_".join(map(str, k)))
def test_generated_filters_match_reference(key):
    """every tap equals dwt_filterCoef's to the 6 printed decimals"""
    ref = GOLD.outputs({f"coef/{'_'.join(map(str, _ref_key(key)))}"})
    want = next(iter(ref.values()))
    lo, hi = TABLE[key]
    assert want.shape == (2, len(lo))
    assert np.array_equal(np.round(want.astype(np.float64), 6), np.round(np.stack([lo, hi]).astype(np.float64), 6))


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference(name):
    got = GOLD.outputs({f"case/{name}"}).get(f"case/{name}")
    if got is None:
        pytest.skip("not in tests/golden/wavelet.npz: needs the reference build")
    want = oracle(*CASES[name])
    assert got.shape == want.shape
    assert np.abs(got - want).max() <= TOL * np.abs(want).max(), name


def test_golden_file_is_current():
    GOLD.check_file()


LEVEL_CASES = W.level_cases(TABLE)


def _swt_level_pairs():
    """(n, dec * 2^i) of every SWT level the level-by-level GPU suite runs"""
    return {(n, len(TABLE[key][0]) << i) for kind, num, n, key, _ in LEVEL_CASES.values() if kind == "swt"
            for i in range(num)}


def test_modulo_indexing_equals_literal_padding():
    """padded[m] = x[(m - f/2) mod L] for every length and filter length the objects produce: DWT / WPT levels
    (L = 2^k >= 4 against every filter length), SWT levels (any L, f = dec * 2^i up to past 8 L), and every SWT level
    of the level-by-level GPU suite, where f reaches 30 L"""
    decs = sorted({len(v[0]) for v in TABLE.values()})
    pairs = [(1 << k, d) for k in range(2, 17) for d in decs]
    pairs += [(n, d << i) for n in range(1, 300) for d in decs for i in range(12) if (d << i) <= 8 * n + 80]
    levels = _swt_level_pairs()
    assert max(f / n for n, f in levels) == 30 and sum(f > 8 * n + 80 for n, f in levels) >= 20
    short = 0
    for n, f in pairs + sorted(levels):
        x = np.arange(n, dtype=np.float64) + 1
        lit = W.period_padding(x, f)
        assert lit.shape == (n + f,) and np.array_equal(lit, W.modulo_padding(x, f)), (n, f)
        short += n < f // 2
    assert short > 1000


def test_level_case_coverage():
    """what the level-by-level GPU suite claims to run"""
    by = lambda kind: [c for c in LEVEL_CASES.values() if c[0] == kind]  # noqa: E731
    for kind in KINDS:
        assert {c[3] for c in by(kind)} == set(TABLE), kind
    dwt, wpt, swt = by("dwt"), by("wpt"), by("swt")
    assert {(e, num) for _, num, e, *_ in dwt} >= {(e, e - 1) for e in range(2, 21)}
    assert all(len({c[3] for c in dwt if c[2] == e}) >= 2 for e in range(2, 21))
    assert any(len(TABLE[key][0]) == 60 for _, num, e, key, _ in dwt if num == e - 1 and e >= 10)    # 15 wraps at L = 4
    assert {(e, num) for _, num, e, *_ in wpt} >= {(e, num) for e in range(2, 15) for num in range(1, e)}
    assert {(e, num, m) for _, num, e, _, m in wpt if e >= 18} == {(e, num, False) for e in (18, 19, 20)
                                                                  for num in (3, e - 1)}
    assert max(len(TABLE[key][0]) * (1 << num - 1) // 2 / n for _, num, n, key, _ in swt) == 15  # dec s/2 / n
    assert {n // (1 << num) for _, num, n, *_ in swt} >= {1, 3, 5} and max(c[1] for c in swt) == 12
    assert ("swt", 10, 1 << 20) in {c[:3] for c in swt}
    for kind, num, size, key, m_data in dwt + wpt:
        rows = num if kind == "dwt" else 1 << num
        assert m_data == (4 * rows * (4 << size) <= W.M_DATA_BYTES and not (kind == "wpt" and size >= 18))


def _small_level_cases():
    """the level suite's DWT / WPT cases up to 2^10 and SWT cases up to 1280 samples, and every filter at num 1 .. 3"""
    out = [c[:4] for c in LEVEL_CASES.values() if c[2] <= (10 if c[0] != "swt" else 1280)]
    out += [(kind, num, 6 if kind != "swt" else 96, key) for kind in KINDS for num in (1, 2, 3) for key in TABLE]
    return out


@pytest.mark.parametrize("kind", KINDS)
def test_vectorised_oracle_matches_literal(kind):
    """level(), wpt_level() and swt_level(), gathers over the unpadded input as the kernels read it, chained level by
    level, equal the literal oracle (padding, convolution, decimation, WPT's _node order and swap) within float64
    rounding, for every small case of the level suite"""
    cases = [c for c in _small_level_cases() if c[0] == kind]
    assert len(cases) >= 100
    for _, num, size, key in cases:
        lo, hi = (v.astype(np.float64) for v in TABLE[key])
        n = size if kind == "swt" else 1 << size
        x = W.level_clips(n, size)
        for clip in x:
            if kind == "swt":
                want, got = np.stack(W.swt(clip, num, lo, hi)), np.stack(W.swt_fast(clip, num, lo, hi))
            else:
                want = getattr(W, kind)(clip, num, lo, hi, m_data=False)[0]
                got = getattr(W, f"{kind}_fast")(clip, num, lo, hi)
            assert got.shape == want.shape
            assert np.abs(got - want).max() <= 1e-12 * max(np.abs(want).max(), 1.0), (kind, num, size, key)
        batched = getattr(W, f"{kind}_fast")(x, num, lo, hi)            # leading axes: the four clips at once
        single = [getattr(W, f"{kind}_fast")(c, num, lo, hi) for c in x]
        if kind == "swt":
            batched, single = np.stack(batched, 1), np.stack([np.stack(s) for s in single])
        assert np.array_equal(batched, single)


def test_level_scales():
    """the scales level() and swt_level() return are the steps applied to |h| and |x|"""
    rng = np.random.default_rng(1)
    lo, hi = (v.astype(np.float64) for v in TABLE[W.DB30])
    x = rng.standard_normal((3, 64))
    a, d, sa, sd = W.level(x, lo, hi)
    assert np.array_equal(sa, W.level(np.abs(x), np.abs(lo), np.abs(hi))[0])
    assert np.array_equal(sd, W.level(np.abs(x), np.abs(lo), np.abs(hi))[1])
    a, d, sa, sd = W.swt_level(x, 8, lo, hi)
    assert np.array_equal(sa, W.swt_level(np.abs(x), 8, np.abs(lo), np.abs(hi))[0])
    assert (sa >= np.abs(a)).all() and (sd >= np.abs(d)).all()


@pytest.mark.parametrize("kind", ["dwt", "wpt"])
def test_m_data_index_matches_literal_loops(kind):
    """m_data_index(), the vectorised map the GPU suite checks mDataArr through, equals the literal loops of the
    reference's mData layout, for every radix2Exp 2 .. 10 and num 1 .. radix2Exp - 1"""
    lo, hi = (v.astype(np.float64) for v in TABLE[W.SYM4])
    for e in range(2, 11):
        x = np.random.default_rng(e).standard_normal(1 << e)
        for num in range(1, e):
            coef, m = getattr(W, kind)(x, num, lo, hi)
            idx = W.m_data_index(1 << e, num, kind)
            assert idx.shape == m.shape and np.array_equal(coef[idx], m), (e, num)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("key", sorted(REFUSED), ids=lambda k: "_".join(map(str, k)))
def test_refused_filters(product_lib, kind, key):
    """every listed filter this library does not generate is refused with -2 and a message"""
    ty, t1, t2 = key
    st, obj = W.new(product_lib, kind, 3, 256 if kind == "swt" else 8, ty, t1, t2)
    assert st == -2 and not obj.value
    msg = product_lib.afb200_lastError().decode()
    assert "not supported" in msg and REFUSED[key] in msg


def test_unknown_filters_fall_back_to_sym4(product_lib):
    """combinations the reference does not list build sym4 (the reference's python DWT only sends such ones)"""
    for ty, t1, t2 in ((2, 11, 0), (1, 41, 0), (5, 4, 5), (32000, 5, 3), (-1, 4, 4), (3, 6, 0), (4, 5, 0)):
        st, obj = W.new(product_lib, "dwt", 4, 8, ty, t1, t2)
        assert st == 0 and obj.value, (ty, t1, t2)
        product_lib.dwtObj_free(obj)
    ref = ref_lib_or_none()
    if ref is not None:
        for ty, t1, t2 in ((32000, 5, 3), (2, 11, 0)):
            assert np.array_equal(np.stack(W.filters(ref, ty, t1, t2)), np.stack(TABLE[(2, 4, 0)]))


STATUS_ARGS = [("dwt", num, e) for e in (-1, 0, 1, 2, 3, 12, 20, 30, 31) for num in (-1, 0, 1, 2, e - 1, e)] + \
              [("wpt", num, e) for e in (0, 1, 2, 5, 31) for num in (0, 1, e - 1, e)] + \
              [("swt", num, n) for n in (0, 1, 2, 3, 96, 100, 1 << 20) for num in (0, 1, 2, 5, 7)]


def test_constructor_statuses_match_reference(product_lib):
    ref = ref_lib_or_none()
    args = STATUS_ARGS + [("dwt", 1, 21), ("wpt", 3, 21), ("swt", 0, 1 << 21), ("swt", 1, (1 << 20) + 2)]
    for kind, num, size in args:
        st, obj = W.new(product_lib, kind, num, size, 2, 4, 4)
        if obj.value:
            getattr(product_lib, f"{kind}Obj_free")(obj)
        big = (size > 20 and kind != "swt") or (kind == "swt" and size > 1 << 20)
        if big and st != -1 and st != -100:
            assert st == -2, (kind, num, size, st)
            continue
        if ref is not None:
            rst, robj = W.new(ref, kind, num, size, 2, 4, 4)
            if robj.value:
                getattr(ref, f"{kind}Obj_free")(robj)
            assert st == rst, (kind, num, size, st, rst)
        else:
            assert st in (0, -1, -100), (kind, num, size, st)


def test_generator_reproduces_committed_header(tmp_path):
    """gen/gen_wavelets.py, run now, writes exactly the committed kernels/wavelet_coef_gen.h"""
    pytest.importorskip("mpmath")
    import importlib.util
    spec = importlib.util.spec_from_file_location(
        "gen_wavelets", os.path.join(ROOT, "audioflux_b200", "csrc", "gen", "gen_wavelets.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    out = tmp_path / "wavelet_coef_gen.h"
    gen.emit(str(out))
    assert out.read_text() == open(GEN).read()


@pytest.mark.parametrize("kind", KINDS)
def test_header_symbols(product_lib, kind):
    api = {k: v for k, v in capi.WAVELET_API.items() if k.startswith(f"{kind}Obj_")}
    check_symbols(product_lib, f"afb200_{kind}.h", f"{kind}Obj_", api, {f"{kind}Obj_new", f"{kind}Obj_{kind}",
                                                                         f"{kind}Obj_free"}, {f"{kind}Obj_{kind}Batch"})
