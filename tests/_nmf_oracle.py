"""Non-negative matrix factorisation in numpy: src/classic/nmf.c restated in float32, each product rounded to float32
and summed in float64 (the reference's __mdot / __mdot2 accumulate in double), every other step rounded to float32 in
the reference's order, the stop norms summed sequentially in float32 as __vnorm does.  The run records each
iteration's stop statistic max(||dW||, ||dH||), so that a stop decision within STOP_RTOL of thresh (undetermined: the
two norms are differences of nearly equal iterates, far more sensitive to the last bits of W and H than W and H
themselves) accepts both outcomes.  Also: the test cases and the C calls shared by the CPU and GPU suites."""
import ctypes as C

import numpy as np

F = np.float32
EPS = F(1e-16)
STOP_RTOL = 1e-2
DEFAULTS = dict(max_iter=300, tp=1, thresh=1e-3, norm=0)        # the C function's NULL fallbacks


def _dot(a, b):
    """a @ b with each product rounded to float32 and the products summed in float64, as __mdot / __mdot2"""
    return (a[:, :, None] * b[None, :, :]).sum(axis=1, dtype=np.float64).astype(F)


def _normalise(W, norm):
    if norm in (1, 2):
        a = np.abs(W)
        v = np.cumsum(a if norm == 1 else a * a, axis=0, dtype=F)[-1]     # sequential float sums, as __mnorm
        if norm == 2:
            v = np.sqrt(v)
    else:
        v = W.max(axis=0)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(W != 0, W / v[None, :], F(0)).astype(F)


def _vnorm(d):
    return np.sqrt(np.cumsum((d * d).ravel(), dtype=F)[-1]) if d.size else F(0)


def run(V, k, max_iter=300, tp=1, thresh=1e-3, norm=0, W=None, H=None, stop=True):
    """-> (W, H, iters, stat): W n x k, H k x m after `iters` iterations; stat[i] = max of iteration i's two norms.
    stop=False runs all max_iter iterations."""
    V = np.asarray(V, F)
    n, m = V.shape
    H = (np.arange(1, k * m + 1, dtype=F).reshape(k, m) if H is None else np.array(H, F))
    W = (np.arange(1, n * k + 1, dtype=F).reshape(n, k) if W is None else np.array(W, F))
    W = _normalise(W, norm)
    thresh = F(thresh)
    stat = []
    it = 0
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for it in range(1, max(max_iter, 0) + 1):
            W1, H1 = W, H
            D = _dot(W, H)
            if tp == 0:
                D2, D3 = V / (D + EPS), None
            elif tp == 1:
                D2 = (1.0 / (D * D + EPS).astype(np.float64) * V.astype(np.float64)).astype(F)
                D3 = (1.0 / (D + EPS).astype(np.float64)).astype(F)
            else:
                D2, D3 = V, D
            A = _dot(W.T, D2)
            B = np.broadcast_to(W.astype(np.float64).sum(0).astype(F)[:, None], A.shape) if D3 is None else _dot(W.T, D3)
            H = H * A / (B + EPS) if tp in (0, 1) else H * (A / (B + EPS))
            A = _dot(D2, H.T)
            B = np.broadcast_to(H.astype(np.float64).sum(1).astype(F)[None, :], A.shape) if D3 is None else _dot(D3, H.T)
            W = W * A / (B + EPS) if tp in (0, 1) else W * (A / (B + EPS))
            W = _normalise(W, norm)
            w1, h1 = _vnorm(W - W1), _vnorm(H - H1)
            stat.append(max(float(w1), float(h1)) if not (np.isnan(w1) or np.isnan(h1)) else np.nan)
            if stop and w1 < thresh and h1 < thresh:
                break
    return W, H, (it if max_iter > 0 else 0), np.array(stat)


def undetermined(stat, thresh):
    """per iteration: True where the stop decision lies within STOP_RTOL of thresh"""
    return np.abs(np.asarray(stat) - thresh) <= STOP_RTOL * thresh


def counts_agree(got, want, stat, thresh):
    """iteration counts got and want agree, with stat the statistics of a run without stopping: equal, or the earlier
    stop's decision is undetermined and every later decision before the later stop is either undetermined or not a
    stop"""
    if got == want:
        return True
    lo, hi = min(got, want), max(got, want)
    if lo < 1 or len(stat) < hi:
        return False
    und, stops = undetermined(stat, thresh), np.asarray(stat) < thresh
    return bool(und[lo - 1]) and all(und[j - 1] or not stops[j - 1] for j in range(lo + 1, hi))


# ---- cases ----------------------------------------------------------------------------------------------------------

def matrix(seed, n, m, kind="noise"):
    rng = np.random.default_rng(seed)
    if kind == "noise":                                  # |noise|^2, a power spectrogram of white noise
        return (np.abs(rng.standard_normal((n, m))) ** 2).astype(F)
    if kind == "lowrank":                                # exactly rank 3 plus a little noise
        a, b = rng.random((n, 3)), rng.random((3, m))
        return (a @ b + 0.01 * rng.random((n, m))).astype(F)
    if kind == "sparse":                                 # zeros in V
        x = rng.random((n, m)).astype(F)
        x[rng.random((n, m)) < 0.3] = 0
        return x
    raise ValueError(kind)


def cases():
    """[(name, kw)]: kw holds n, m, k, kind, seed and the C arguments (None: NULL)"""
    out = []

    def add(name, n, m, k, mi=300, tp=0, th=1e-3, norm=0, kind="noise", seed=0):
        out.append((name, dict(n=n, m=m, k=k, max_iter=mi, tp=tp, thresh=th, norm=norm, kind=kind, seed=seed)))

    for tp in (0, 1, 2, None):
        for norm in (0, 1, 2):
            add(f"tp{tp}_norm{norm}", 40, 30, 4, mi=50, tp=tp, norm=norm, seed=1)
    for k in (1, 2, 3, 5, 8, 9, 16):
        add(f"k{k}", 48, 36, k, mi=50, tp=0, seed=2 + k)
    add("k_full_n", 12, 20, 12, mi=50, tp=2, seed=20)                  # k = min(n, m)
    add("k_full_m", 17, 9, 9, mi=50, tp=0, seed=21)
    add("s8x8", 8, 8, 2, mi=300, tp=0, seed=22)
    add("s8x8_euc", 8, 8, 3, mi=300, tp=2, norm=2, seed=23)
    add("s1x1", 1, 1, 1, mi=5, tp=0, seed=24)
    add("s1xm", 1, 40, 1, mi=5, tp=2, seed=25)
    add("s257x128_euc", 257, 128, 2, mi=50, tp=2, seed=26)
    add("s257x200_kl", 257, 200, 4, mi=50, tp=0, seed=27)
    add("s513x431_kl", 513, 431, 8, mi=5, tp=0, seed=28)
    add("s513x431_is", 513, 431, 8, mi=5, tp=1, norm=2, seed=29)
    add("s513x431_euc", 513, 431, 8, mi=5, tp=2, norm=1, seed=30)
    for mi in (0, 1, 5, 50, 300):
        add(f"iter{mi}", 64, 50, 4, mi=mi, tp=0, seed=31)
    add("iter300_is", 64, 50, 3, mi=300, tp=1, seed=32)
    add("iter300_euc", 64, 50, 3, mi=300, tp=2, seed=33)
    add("lowrank_stop_kl", 60, 40, 3, mi=300, tp=0, th=1e-2, kind="lowrank", seed=34)
    add("lowrank_stop_euc", 60, 40, 3, mi=300, tp=2, th=5e-2, kind="lowrank", seed=35)
    add("lowrank_default_th", 30, 20, 3, mi=300, tp=0, kind="lowrank", seed=36)
    add("sparse_kl", 50, 40, 4, mi=50, tp=0, kind="sparse", seed=37)
    add("sparse_euc", 50, 40, 4, mi=50, tp=2, norm=1, kind="sparse", seed=38)
    add("null_all", 32, 24, 3, mi=None, tp=None, th=None, norm=None, seed=39)
    add("tp3_is_euclidean", 40, 30, 4, mi=50, tp=3, norm=1, seed=40)     # every type but 0 and 1 is Euclidean
    add("tp_neg1_is_euclidean", 40, 30, 4, mi=50, tp=-1, seed=41)
    return out


def resolved(kw):
    """the case's arguments with NULL replaced by the C defaults"""
    d = {a: kw[a] if kw[a] is not None else DEFAULTS[a] for a in DEFAULTS}
    return d


def case_matrix(kw):
    return matrix(kw["seed"], kw["n"], kw["m"], kw["kind"])


def oracle_case(kw, stop=True, max_iter=None):
    r = resolved(kw)
    if max_iter is not None:
        r["max_iter"] = max_iter
    return run(case_matrix(kw), kw["k"], stop=stop, **r)


def _opt(ctype, v):
    return None if v is None else C.byref(ctype(v))


def c_nmf(lib, kw, max_iter="case"):
    """(W, H) from lib's nmf on the case, arange-initialised as the reference's Python binding; max_iter overrides"""
    V = case_matrix(kw)
    n, m, k = kw["n"], kw["m"], kw["k"]
    H = np.arange(1, k * m + 1, dtype=F).reshape(k, m)
    W = np.arange(1, n * k + 1, dtype=F).reshape(n, k)
    mi = kw["max_iter"] if max_iter == "case" else max_iter
    vp = C.c_void_p
    lib.nmf(V.ctypes.data_as(vp), n, m, k, W.ctypes.data_as(vp), H.ctypes.data_as(vp), _opt(C.c_int, mi),
            _opt(C.c_int, kw["tp"]), _opt(C.c_float, kw["thresh"]), _opt(C.c_int, kw["norm"]))
    return W, H


def c_iters(lib, kw, W, H, guess):
    """the iterations lib's nmf ran to give (W, H) on the case: `guess` when maxIter = guess gives the same bits (at a
    fixed point earlier counts do too), else the least j near it that does; -1 when none is found"""
    mi = resolved(kw)["max_iter"]
    same = lambda j: all(np.array_equal(a, b, equal_nan=True) for a, b in zip(c_nmf(lib, kw, j), (W, H)))  # noqa: E731
    if same(guess):
        return guess
    for j in range(max(0, guess - 3), min(mi, guess + 3) + 1):
        if same(j):
            return j
    return -1
