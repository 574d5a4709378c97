"""numpy restatement of onset detection (src/mir/onset_algorithm.c), the yardstick of tests/test_*onset*.py, and ctypes
drivers of onsetObj_* for either library.  The novelty functions come from tests/_spectral_oracle.py (float64); the max
filter, the normalisation and the peak picking are float32 in the reference's order, so that given the same novelty
curve the points are exactly the reference's."""
import ctypes as C
import zlib

import numpy as np

import _spectral_oracle as SO

f32 = np.float32
NAMES = ("flux", "hfc", "sd", "sf", "mkl", "pd", "wpd", "nwpd", "cd", "rcd", "broadband")
PHASE = tuple(range(5, 10))
DEFAULT_PARAM = (1, 1.0, 1, 0, 1, 0.0, 1, 1.0)     # the reference Python's NoveltyParam(1, 1, 1, 0, 1, 0, 1, 1)


class NoveltyParam(C.Structure):
    _fields_ = [("step", C.c_int), ("p", C.c_float), ("isPostive", C.c_int), ("isExp", C.c_int), ("type", C.c_int),
                ("threshold", C.c_float), ("isNorm", C.c_int), ("gamma", C.c_float)]


def peak_params(samplate=32000, slide_length=512):
    """(preMax, postMax, preAvg, postAvg, wait, delta) of onsetObj_new (:123-133): double, then floored as a float"""
    sr = samplate if samplate and samplate > 0 else 32000
    hop = slide_length if slide_length >= 1 else 512
    fl = lambda v: int(np.floor(f32(v)))  # noqa: E731
    return (fl(0.03 * sr / hop), fl(0.0 * sr / hop + 1), fl(0.1 * sr / hop), fl(0.1 * sr / hop + 1),
            fl(0.03 * sr / hop), f32(0.07))


def maxfilter(x, order):
    """__mmaxfilter along bins: window [k - order/2, k - 1 + order - order/2] clipped to the frame"""
    x = np.asarray(x, f32)
    if order < 2:
        return x
    M = x.shape[1]
    left, right = order // 2, order - order // 2
    out = np.empty_like(x)
    for k in range(M):
        out[:, k] = x[:, max(k - left, 0):min(k - 1 + right, M - 1) + 1].max(1)
    return out


def _param(prm):
    """the fields onsetObj_onset reads (:135-179); prm None: the C defaults"""
    step, p, pos, exp, tp, thr = 1, 1.0, 1, 0, 0, 0.0
    if prm is not None:
        step = prm[0] if prm[0] > 0 else 1
        p = float(f32(prm[1])) if prm[1] != 0 else 1.0
        pos, exp, tp, thr = prm[2], prm[3], prm[4], float(f32(prm[5]))
    return step, p, pos, exp, tp, thr


def novelty(kind, x, ph, idx, prm):
    """the raw novelty curve (before normalisation), float64"""
    step, p, pos, exp, tp, thr = _param(prm)
    name = NAMES[kind] if 0 <= kind < len(NAMES) else "flux"
    if name in ("pd", "wpd", "nwpd", "cd", "rcd"):
        return SO.compute(name, x, idx, None, phase=ph)
    kw = dict(flux=dict(step=step, p=p, is_positive=bool(pos), is_exp=bool(exp), tp=tp),
              sd=dict(step=step, is_positive=bool(pos)), sf=dict(step=step, is_positive=bool(pos)),
              mkl=dict(tp=tp), broadband=dict(threshold=thr)).get(name, {})
    return SO.compute(name, x, idx, None, **kw)


def normalise(v):
    """evn -= min, evn /= max when max > 0, float32, with the sequential scans' rule for NaN"""
    v = np.asarray(v, f32)
    with np.errstate(all="ignore"):
        mn = v[0] if np.isnan(v[0]) else f32(np.nanmin(v))
        v = (v - mn).astype(f32)
        mx = v[0] if np.isnan(v[0]) else f32(np.nanmax(v))
        if mx > 0:
            v = (v / mx).astype(f32)
    return v


def _windows(T, pre, post):
    i = np.arange(T)
    return np.maximum(i - pre, 0), np.where(i + post < T, i - 1 + post, T - 1)


def candidates(e, pp):
    """frames that pass the max and the mean tests of __peakPick (:438-448), float32 as the reference evaluates them"""
    e = np.asarray(e, f32)
    T = len(e)
    preMax, postMax, preAvg, postAvg, _, delta = pp
    s1, t1 = _windows(T, preMax, postMax)
    m = e[s1].copy()
    for k in range(1, preMax + postMax + 1):
        j = s1 + k
        w = e[np.minimum(j, T - 1)]
        m = np.where((j <= t1) & (m < w), w, m)
    s2, t2 = _windows(T, preAvg, postAvg)
    s = np.zeros(T, f32)
    for k in range(preAvg + postAvg + 1):          # summed from the window's left end, as __vmean does
        j = s2 + k
        s = np.where(j <= t2, (s + e[np.minimum(j, T - 1)]).astype(f32), s)
    with np.errstate(all="ignore"):
        mean = (s / (t2 - s2 + 1).astype(f32)).astype(f32)
        return (e == m) & (e >= (mean + f32(delta)).astype(f32))


def suppress(cand, wait):
    """the greedy wait rule in frame order (:449-454)"""
    out, pre = [], -wait - 1
    for i in np.flatnonzero(cand):
        if i - pre > wait:
            out.append(int(i))
            pre = int(i)
    return np.array(out, np.int32)


def pick(e, pp):
    return suppress(candidates(e, pp), pp[4])


def near_ties(e, pp, eps=1e-5):
    """frames whose max or mean decision a change of evn below eps could flip: |evn[i] - max of the rest of its max
    window| < eps, or |evn[i] - (mean + delta)| < eps"""
    e = np.asarray(e, np.float64)
    T = len(e)
    preMax, postMax, preAvg, postAvg, _, delta = pp
    s1, t1 = _windows(T, preMax, postMax)
    s2, t2 = _windows(T, preAvg, postAvg)
    out = np.zeros(T, bool)
    for i in range(T):
        rest = np.concatenate((e[s1[i]:i], e[i + 1:t1[i] + 1]))
        if rest.size and abs(e[i] - rest.max()) < eps:
            out[i] = True
        if abs(e[i] - (e[s2[i]:t2[i] + 1].mean() + float(delta))) < eps:
            out[i] = True
    return out


def points_agree(e_a, p_a, e_b, p_b, pp, eps=1e-5):
    """(ok, frames): the two point lists are equal, or every frame where the candidate decisions on the two curves
    differ is a near-tie of one of them (the suppression is then the only thing that can move later points)"""
    if np.array_equal(p_a, p_b):
        return True, []
    diff = np.flatnonzero(candidates(e_a, pp) != candidates(e_b, pp))
    ties = near_ties(e_a, pp, eps) | near_ties(e_b, pp, eps)
    return bool(diff.size) and bool(ties[diff].all()), diff.tolist()


def onset(x, ph, kind, order=1, prm=DEFAULT_PARAM, idx=None, pp=None):
    """one clip x [T, M] (time-major) -> (evn float32 [T], points int32)"""
    x = np.asarray(x, f32)
    idx = list(range(x.shape[1])) if idx is None else list(idx)
    raw = novelty(kind, maxfilter(x, order), ph, idx, prm)
    evn = normalise(np.asarray(raw, np.float64).astype(f32))
    return evn, pick(evn, pp if pp is not None else peak_params())


# ---- the test grid
SR_HOP = ((32000, 512), (8000, 512), (44100, 256))     # preMax / wait 1, 0 and 5


def _seed(name):
    return zlib.crc32(name.encode())


def case_signal(name, kw):
    """(spec [T, M] > 0, phase [T, M]) of a case: random, or a click train (sparse loud frames over a quiet floor)"""
    T, M = kw.get("T", 160), kw.get("M", 96)
    rng = np.random.default_rng(_seed(name))
    ph = rng.uniform(-np.pi, np.pi, (T, M)).astype(f32)
    if kw.get("sig", "rand") == "rand":
        return (rng.random((T, M)) + 0.01).astype(f32), ph
    x = 0.01 * (1 + rng.random((T, M)))
    t = 3
    while t < T:
        x[t] += rng.uniform(0.5, 2.0) * (1 + rng.random(M))
        t += int(rng.integers(9, 23))
    return x.astype(f32), ph


def case_index(name, kw):
    if kw.get("idx") is None:
        return None
    rng = np.random.default_rng(_seed(name) + 1)
    M = kw.get("M", 96)
    return rng.choice(M, M // 3, replace=False).astype(np.int32)


def _variants(kind):
    """NoveltyParam variations of a type (fields it does not read stay at the Python default)"""
    d = DEFAULT_PARAM
    if kind == 0:
        return {"default": d, "p2_abs_exp": (1, 2.0, 0, 1, 0, 0.0, 0, 1.0), "p05_abs": (1, 0.5, 0, 0, 0, 0.0, 0, 1.0)}
    if kind in (2, 3):
        return {"default": d, "abs": (1, 1.0, 0, 0, 1, 0.0, 1, 1.0)}
    if kind == 4:
        return {"default": d, "sum": (1, 1.0, 1, 0, 0, 0.0, 1, 1.0)}
    if kind == 10:
        return {"default": d, "thr3": (1, 1.0, 1, 0, 1, 3.0, 1, 1.0)}
    return {"default": d}


def cases():
    """[(name, kw)]: every type at filter orders 1 / 2 / 3 / 7, with and without a bin list, the samplate / hop pairs
    in turn; the parameter variations; step 3; the C defaults (param NULL); and a click train per type"""
    out = []
    n = 0
    for kind, name in enumerate(NAMES):
        for order in (1, 2, 3, 7):
            for idx in (None, "sub"):
                sr, hop = SR_HOP[n % len(SR_HOP)]
                n += 1
                out.append((f"{name}_o{order}{'_idx' if idx else ''}_sr{sr}",
                            dict(kind=kind, order=order, idx=idx, prm=DEFAULT_PARAM, sr=sr, hop=hop)))
        for vname, prm in _variants(kind).items():
            if vname != "default":
                out.append((f"{name}_{vname}", dict(kind=kind, order=2, prm=prm, sr=32000, hop=512)))
        out.append((f"{name}_step3", dict(kind=kind, order=1, prm=(3,) + DEFAULT_PARAM[1:], sr=8000, hop=512)))
        out.append((f"{name}_cdefaults", dict(kind=kind, order=1, prm=None, sr=44100, hop=256)))
        out.append((f"{name}_clicks", dict(kind=kind, order=1, prm=DEFAULT_PARAM, sr=32000, hop=512, sig="clicks")))
        out.append((f"{name}_clicks_o3", dict(kind=kind, order=3, prm=DEFAULT_PARAM, sr=8000, hop=512, sig="clicks",
                                              idx="sub")))
    # a filter order above the number of bins: every window is clipped to the frame
    out.append(("sf_order_above_bins", dict(kind=3, order=150, prm=DEFAULT_PARAM, sr=32000, hop=512, sig="clicks")))
    return out


def oracle_case(name, kw):
    x, ph = case_signal(name, kw)
    return onset(x, ph, kw["kind"], kw["order"], kw["prm"], case_index(name, kw), peak_params(kw["sr"], kw["hop"]))


# ---- ctypes drivers (either library; both are bound by audioflux_b200.capi)
def _opt(v):
    return None if v is None else C.byref(C.c_int(int(v)))


def c_new(lib, T, M, hop, sr=None, order=None, kind=None):
    o = C.c_void_p()
    st = lib.onsetObj_new(C.byref(o), int(T), int(M), int(hop), _opt(sr), _opt(order), _opt(kind))
    return st, o


def c_onset(lib, o, x, ph=None, prm=DEFAULT_PARAM, idx=None, fill=0):
    """onsetObj_onset on one clip x [T, M] into buffers holding `fill` -> (evn [T], points[:count], count, the whole
    point buffer)"""
    x = np.ascontiguousarray(x, f32)
    T = x.shape[0]
    evn = np.full(T, fill, f32)
    pts = np.full(T, fill, np.int32)
    par = None if prm is None else NoveltyParam(*prm)
    ph = None if ph is None else np.ascontiguousarray(ph, f32)
    n = lib.onsetObj_onset(o, x.ctypes.data, None if ph is None else ph.ctypes.data,
                           None if par is None else C.addressof(par), None if idx is None else idx.ctypes.data,
                           0 if idx is None else len(idx), evn.ctypes.data, pts.ctypes.data)
    return evn, pts[:n].copy(), n, pts


def c_case(lib, name, kw):
    """(evn, points) of a case through onsetObj_onset of lib"""
    x, ph = case_signal(name, kw)
    st, o = c_new(lib, x.shape[0], x.shape[1], kw["hop"], kw["sr"], kw["order"], kw["kind"])
    assert st == 0
    evn, pts, _, _ = c_onset(lib, o, x, ph if kw["kind"] in PHASE else None, kw["prm"], case_index(name, kw))
    lib.onsetObj_free(o)
    return evn, pts
