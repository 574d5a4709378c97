"""NMF without a GPU: the float32 / float64-accumulated oracle against the reference build (or its stored outputs in
tests/golden/nmf.npz) over the types (0, 1, 2, the Euclidean 3 and -1, and NULL), the W norms, k from 1 to
min(n, m), shapes from 1x1 and 8x8 to 513x431, maxIter 0 / 1 / 5 / 50 / 300 and thresholds that stop early, W and H
within 1e-4 of their max and the iteration counts equal (modulo an undetermined stop); the header's symbols; and the
Python function's argument checks."""
import numpy as np
import pytest

import _nmf_oracle as NO
from _parity_kit import GoldenStore, check_symbols, ref_lib_or_none

TOL = 1e-4                 # of max |ref| of W, and of H
CASES = dict(NO.cases())


def _live(keys):
    lib = ref_lib_or_none()
    out = {}
    for name in sorted({k.split("/")[0] for k in keys}):
        kw = CASES[name]
        W, H = NO.c_nmf(lib, kw)
        _, _, guess, _ = NO.oracle_case(kw)
        out[f"{name}/W"], out[f"{name}/H"] = W, H
        out[f"{name}/iters"] = np.array(NO.c_iters(lib, kw, W, H, guess))
    return {k: out[k] for k in keys}


GOLD = GoldenStore("nmf.npz", _live, lambda: {f"{n}/{a}" for n in CASES for a in ("W", "H", "iters")})


def check_against(kw, W, H, iters, what):
    """(W, H) after `iters` iterations agree with the oracle: the count within an undetermined stop, W and H within
    TOL of their max of the oracle at that count.  -> True when the counts differ"""
    r = NO.resolved(kw)
    Wo, Ho, it, _ = NO.oracle_case(kw)
    if iters != it:
        _, _, _, stat = NO.oracle_case(kw, stop=False)
        assert NO.counts_agree(iters, it, stat, r["thresh"]), (what, iters, it, stat[min(iters, it) - 1:max(iters, it)])
        Wo, Ho, _, _ = NO.oracle_case(kw, stop=False, max_iter=iters)
    for got, want, nm in ((W, Wo, "W"), (H, Ho, "H")):
        assert got.shape == want.shape, (what, nm)
        scale = max(float(np.abs(want).max()), 1e-30)
        err = float(np.abs(got.astype(np.float64) - want).max()) / scale
        assert err <= TOL, (what, nm, err)
    return iters != it


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference(name):
    kw = CASES[name]
    g = GOLD.outputs({f"{name}/{a}" for a in ("W", "H", "iters")})
    iters = int(g[f"{name}/iters"])
    assert iters >= 0, (name, "the reference's iteration count was not found")
    check_against(kw, g[f"{name}/W"], g[f"{name}/H"], iters, name)


def test_cases_cover_the_issue():
    """types 0/1/2, 3 and -1 (Euclidean) and NULL, norms 0/1/2, k 1 .. 16 and k = min(n, m), 1x1 .. 513x431, maxIter
    0/1/5/50/300, early stops (the oracle stops before maxIter)"""
    kws = list(CASES.values())
    assert {kw["tp"] for kw in kws} >= {0, 1, 2, 3, -1, None} and {kw["norm"] for kw in kws} >= {0, 1, 2}
    assert set(range(1, 4)) | {5, 8, 9, 16} <= {kw["k"] for kw in kws}
    assert any(kw["k"] == min(kw["n"], kw["m"]) and kw["k"] > 1 for kw in kws)
    assert {(8, 8), (513, 431), (1, 1)} <= {(kw["n"], kw["m"]) for kw in kws}
    assert {0, 1, 5, 50, 300, None} <= {kw["max_iter"] for kw in kws}
    early = [n for n, kw in CASES.items() if NO.oracle_case(kw)[2] < NO.resolved(kw)["max_iter"]]
    assert len(early) >= 3, early
    assert 35 <= len(kws) <= 60


def test_golden_file_matches_reference_build():
    GOLD.check_file()


def test_oracle_restates_reference_steps():
    """the oracle's W normalisation: column max (a zero entry stays 0), the sequential float p-norms"""
    W = np.array([[0, 2], [3, 4], [1, 0]], np.float32)
    assert np.array_equal(NO._normalise(W, 0), np.array([[0, .5], [1, 1], [1 / 3, 0]], np.float32))
    assert np.array_equal(NO._normalise(W, 1), (W / np.array([4, 6], np.float32)).astype(np.float32))
    assert np.allclose(NO._normalise(W, 2), W / np.sqrt((W * W).sum(0)))
    V = NO.matrix(0, 6, 5)
    W0, H0, it, stat = NO.run(V, 2, max_iter=0)
    assert it == 0 and len(stat) == 0 and np.array_equal(H0, np.arange(1, 11, dtype=np.float32).reshape(2, 5))
    assert NO.counts_agree(3, 3, [], 1e-3)
    assert NO.counts_agree(2, 3, np.array([5e-3, 1.005e-3, 9e-4]), 1e-3)
    assert not NO.counts_agree(2, 3, np.array([5e-3, 5e-4, 4e-4]), 1e-3)


def test_nmf_symbols_exported_and_bound(product_lib):
    from audioflux_b200 import capi
    check_symbols(product_lib, "afb200_nmf.h", "nmf", capi.NMF_API, {"nmf"}, {"nmfBatch"})


def test_batch_refusals(product_lib):
    """-1 for n, m, k or batch below 1 and for NULL arrays, before any device work"""
    L = product_lib
    a = np.ones(64, np.float32)
    p = a.ctypes.data
    for args in ((p, 1, 4, 4, 0), (p, 1, 0, 4, 2), (p, 1, 4, 0, 2), (p, 0, 4, 4, 2), (None, 1, 4, 4, 2)):
        assert L.nmfBatch(*args, p, p, None, None, None, None, None, 0, None) == -1, args
        assert b"bad argument" in L.afb200_lastError()
    assert L.nmfBatch(p, 1, 4, 4, 2, None, p, None, None, None, None, None, 0, None) == -1
    assert L.nmfBatch(p, 1, 4, 4, 2, p, None, None, None, None, None, None, 0, None) == -1
    L.nmf(None, 4, 4, 2, None, None, None, None, None, None)          # writes nothing, does not crash


def test_python_function_arguments(product_lib):
    import audioflux_b200 as af
    with pytest.raises(ValueError, match="2D array"):
        af.nmf(np.ones(5, np.float32), 2)
    with pytest.raises(ValueError, match="at least 1"):
        af.nmf_batch(np.ones((4, 4), np.float32), 0)
    with pytest.raises(ValueError, match="h_init must be"):
        af.nmf_batch(np.ones((2, 4, 4), np.float32), 2, h_init=np.ones((2, 4), np.float32))
    from audioflux_b200.lib import AfB200Error
    if product_lib.afb200_deviceCount() <= 0:          # no CPU fallback: the compute call fails loudly
        with pytest.raises(AfB200Error, match="no CUDA device"):
            af.nmf(np.ones((4, 4), np.float32), 2)
