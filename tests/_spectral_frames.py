"""Frame-by-frame checks of the spectral descriptors (k_spectral, csrc/kernels/spectral.cu) against the float64 oracle
of tests/_spectral_oracle.py, shared by tests/test_gpu_spectral_frames.py and tests/test_spectral_cpu.py.

Every feature, output plane and frame is judged on its own scale, so a wrong value in a quiet frame is not hidden by a
loud one:
  - exact: rolloff, max (value and frequency), broadband, novelty counting hits, mean's frequency plane;
  - sums of non-negative terms and their ratios: |got - want| <= 1e-4 |want_t|;
  - features whose sums cancel (slope, skewness, decrease, band_width with odd p, novelty values): |got - want| <=
    1e-4 M_t, where M_t is the same expression with every summed term replaced by its absolute value;
  - NaN and +-inf sit in the same frames.
The inputs cross the 32-frame tiles of the kernel: clip lengths around multiples of 32, temporal steps around the tile,
runs of frames whose rolloff never crosses (the look-back of 1, 2 and 3 ballot rounds), and crafted rows (NaN, +-inf,
denormals, negative bins, zero frames, max ties across and within lanes)."""
import ctypes as C

import numpy as np

import _spectral_cases as SC
import _spectral_oracle as SO
from audioflux_b200.spectral import TWO_PLANES, encode

TOL = 1e-4
TILE = 32                       # frames per CTA of k_spectral
STEPS = (1, 2, 31, 32, 33)      # with T - 1, T and T + 5 per clip length
CLIP_T = (1, 31, 32, 33, 64, 65, 97, 465)
LEVELS = (1e-2, 1e2)            # adjacent clips differ in level by 1e4
CANCEL = ("slope", "skewness", "decrease")


# ---------------------------------------------------------------------------------------------------- the comparator
def _kind(name, kw, part):
    """'exact', 'nonneg' or 'cancel' for one output plane of a feature"""
    if name in ("rolloff", "max", "broadband") or (name == "mean" and part == 1):
        return "exact"
    if name == "novelty":
        return "exact" if kw.get("data_type", 0) else "cancel"
    if name in CANCEL or (name == "band_width" and kw.get("p", 2) % 2 == 1):
        return "cancel"
    return "nonneg"


def magnitude(name, x, idx, fre, kw):
    """M_t [T] of a feature whose sums cancel: its expression with every summed term replaced by |term|"""
    idx = list(idx)
    r = np.asarray(x, np.float64)[:, idx]
    f = np.asarray(fre, np.float64)[idx]
    with np.errstate(all="ignore"):
        if name == "slope":
            d = f - SO._mean_fre(idx, fre)
            m = (d * d).sum()
            n = np.abs(d[None, :] * (r - r.mean(1, keepdims=True))).sum(1)
            return n / m if m else np.zeros(r.shape[0])
        if name == "skewness":
            c = SO.centroid(x, idx, fre)
            n = (np.abs(f[None, :] - c[:, None]) ** 3 * np.abs(r)).sum(1)
            m = np.abs(SO.spread(x, idx, fre) ** 3 * r.sum(1))
            return np.where(m != 0, n / np.where(m != 0, m, 1), 0.0)
        if name == "decrease":
            n = (np.abs(r[:, 1:] - r[:, :1]) / np.asarray(idx[1:], np.float64)[None, :]).sum(1)
            m = np.abs(r.sum(1) - r[:, 0])
            return np.where(m != 0, n / np.where(m != 0, m, 1), 0.0)
        if name == "band_width":         # odd p: s = sum x d^p, then s^(1/p); the bound also covers d(s^(1/p))/ds
            p = kw.get("p", 2)
            d = f[None, :] - SO.centroid(x, idx, fre)[:, None]
            s, a = (r * d ** p).sum(1), (np.abs(r) * np.abs(d) ** p).sum(1)
            if p == 1:
                return a
            # s = 0 (a zero frame, one bin where d = 0): the slope term is inf * a, and a = 0 there; use a^(1/p)
            slope = np.where(s != 0, np.abs(s) ** (1.0 / p - 1) * a / p, 0.0)
            return np.maximum(a ** (1.0 / p), slope)
        if name == "novelty":
            return _novelty_mag(x, idx, kw)
    raise KeyError(name)


def _novelty_mag(x, idx, kw):
    """sum of |v| over the terms that pass the threshold, with v and the hit rule of SO.novelty"""
    mt = int(kw.get("method_type", 0))
    thr = np.float32(kw.get("threshold", 0.))
    step = max(int(kw.get("step", 1)), 1)
    r = np.asarray(x, np.float64)[:, list(idx)]
    out = np.zeros(r.shape[0])
    with np.errstate(all="ignore"):
        for t in range(step, r.shape[0]):
            c, q = r[t], r[t - step]
            c32, q32 = c.astype(np.float32), q.astype(np.float32)
            if mt == 0:
                v = (c32 - q32).astype(np.float64)
            else:
                qq = c / (q + 1e-16)
                lq = np.log(qq.astype(np.float32))
                v = lq if mt == 1 else c32 * lq if mt == 2 else (qq - lq.astype(np.float64) - 1).astype(np.float32)
                v = np.asarray(v, np.float64)
            out[t] = np.abs(v[v > thr]).sum()
    return out


# The reference takes logf(1.f + u) with 1 + u rounded to float32: for u below about 1e-3 (quiet frames, one or two
# bins) that rounding alone moves the result by more than 1e-4 of itself, and for u below 2^-24 it makes the log 0 (so
# eer's 0 / 0 entropy of one bin is NaN, not inf).  These restate log energy, mkl and eer with that sum rounded as the
# reference rounds it; the logarithm and the sums stay float64.
f32 = np.float32


def _log_one_plus(u32):
    with np.errstate(all="ignore"):
        return np.log((f32(1) + np.asarray(u32, f32)).astype(np.float64))


def _energy(x, idx, fre=None, is_log=False, gamma=10.):
    if not is_log:
        return SO.energy(x, idx, fre, is_log, gamma)
    r = np.asarray(x, f32)[:, idx]
    g = f32(10. if gamma <= 0 else gamma)
    return _log_one_plus(g * (r * r)).sum(1) / len(idx)


def _mkl(x, idx, fre=None, tp=0):
    r = np.asarray(x, np.float64)[:, idx]
    out = np.zeros(r.shape[0])
    with np.errstate(all="ignore"):
        for t in range(1, r.shape[0]):
            s = _log_one_plus((r[t] / (r[t - 1] + 1e-16)).astype(f32)).sum()
            out[t] = s / len(idx) if tp else s
    return out


def _eer(x, idx, fre=None, is_norm=False, gamma=1.):
    e = SO.energy(x, idx).astype(f32)
    with np.errstate(all="ignore"):
        return np.sqrt(1 + np.abs(_log_one_plus(e * f32(gamma)) / SO.entropy(x, idx, is_norm=is_norm)))


F32_ONE_PLUS = {"energy": _energy, "mkl": _mkl, "eer": _eer}


def want_of(name, kw, x, idx, fre, phase=None, prefill=None):
    """the oracle's planes (a tuple) for one clip, with the rules of frames the library leaves as they were (var with
    fewer than two bins, pd / wpd / nwpd frame 1) or adds into (broadband from frame 1) applied to `prefill`
    ([planes, T], zeros when None)"""
    T = x.shape[0]
    nparts = 2 if name in TWO_PLANES else 1
    pre = np.zeros((nparts, T)) if prefill is None else np.asarray(prefill, np.float64).reshape(nparts, T)
    if name == "var" and len(idx) < 2:
        return tuple(pre)
    if name in F32_ONE_PLUS:
        w = (F32_ONE_PLUS[name](x, list(idx), **kw),)
    else:
        w = SO.compute(name, x, list(idx), fre, phase, **kw)
    w = tuple(np.asarray(v, np.float64) for v in (w if isinstance(w, tuple) else (w,)))
    if name in ("pd", "wpd", "nwpd") and T > 1:
        w[0][1] = pre[0][1]
    if name == "broadband":                          # counts added into the float32 output
        w[0][1:] = (pre[0][1:].astype(f32) + w[0][1:].astype(f32)).astype(np.float64)
    return w


class Report:
    """failures and the worst per-frame error ratio |got - want| / (1e-4 scale_t) of each feature"""

    def __init__(self):
        self.bad, self.worst = [], {}

    def ok(self):
        return not self.bad

    def text(self, n=25):
        return "\n".join(self.bad[:n]) + (f"\n... {len(self.bad)} failures" if len(self.bad) > n else "")

    def table(self):
        return "\n".join(f"  {k:<34s} {v:.3g}" for k, v in sorted(self.worst.items()))

    def frames(self, ts, T):
        """failing frames, the ones the kernel treats specially (0, 1, 2 and each tile's first two) marked"""
        out = []
        for t in ts[:8]:
            tag = "start" if t < 3 else "tile" if t % TILE < 2 else ""
            out.append(f"t={t}(tile {t // TILE}+{t % TILE}{',' + tag if tag else ''})")
        return " ".join(out) + (f" ... {len(ts)} frames" if len(ts) > 8 else "")

    def check(self, label, name, kw, got, want, mags=None):
        """got / want: tuples of [T] planes of one clip; mags: M_t for the cancelling features (computed when None
        is passed with mags_of)"""
        key = name + (str({k: kw[k] for k in sorted(kw)}) if kw else "")
        for part, (g, w) in enumerate(zip(got, want)):
            g, w = np.asarray(g, np.float64), np.asarray(w, np.float64)
            T = w.shape[0]
            where = f"{label} {key}[{part}]"
            if g.shape != w.shape:
                self.bad.append(f"{where}: shape {g.shape} != {w.shape}")
                continue
            nf = [np.isnan, np.isposinf, np.isneginf]
            diff = np.zeros(T, bool)
            for fn in nf:
                diff |= fn(g) != fn(w)
            if diff.any():
                ts = np.flatnonzero(diff)
                self.bad.append(f"{where}: non-finite frames differ at {self.frames(ts, T)}: got {g[ts[:3]]} "
                                f"want {w[ts[:3]]}")
            fin = np.isfinite(w) & np.isfinite(g)
            kind = _kind(name, kw, part)
            err = np.abs(np.where(fin, g, 0) - np.where(fin, w, 0))
            if kind == "exact":
                ratio = np.where(err > 0, np.inf, 0.0)
            else:
                scale = np.abs(w) if kind == "nonneg" else np.asarray(mags, np.float64)
                if (fin & ~np.isfinite(scale)).any():     # a NaN or inf bar would accept any value
                    ts = np.flatnonzero(fin & ~np.isfinite(scale))
                    self.bad.append(f"{where} ({kind}): the bar is not finite at {self.frames(ts, T)}: "
                                    f"{scale[ts[:3]]}")
                scale = np.where(fin, TOL * scale, 1.0)
                with np.errstate(all="ignore"):
                    ratio = np.where(err > 0, err / scale, 0.0)
            ratio = np.where(fin, ratio, 0.0)
            ratio = np.where(np.isnan(ratio), np.inf, ratio)
            if T:
                wk = f"{name}[{part}]"
                self.worst[wk] = max(self.worst.get(wk, 0.0), float(ratio.max()))
            if (ratio > 1).any():
                ts = np.flatnonzero(ratio > 1)
                self.bad.append(f"{where} ({kind}): {self.frames(ts, T)}: got {g[ts[:3]]} want {w[ts[:3]]} "
                                f"ratio {ratio[ts[:3]]}")


def mags_of(name, kw, x, idx, fre):
    return magnitude(name, x, idx, fre, kw) if _kind(name, kw, 0) == "cancel" else None


def check_clip(rep, label, name, kw, got, x, idx, fre, phase=None, prefill=None):
    """one clip's planes against the oracle"""
    want = want_of(name, kw, x, idx, fre, phase, prefill)
    rep.check(label, name, kw, got, want, mags_of(name, kw, x, idx, fre))


# ---------------------------------------------------------------------------------------------------- the batched call
def batch_call(s, x, phase, variants, out0=None, device=False):
    """spectralObj_spectralBatch with the requests `variants` (repeats allowed, at most 64) on x [B, T, num]:
    -> {variant index: tuple of [B, T] planes}.  out0 [planes, B, T] pre-fills the output (zeros when None)."""
    from _parity_kit import Out, run_batch
    B, T, _ = x.shape
    enc = [encode(n, kw) for n, kw in variants]
    req = np.array([e[0] for e in enc], np.int32)
    par = np.array([e[1] for e in enc], np.float32).reshape(-1)
    planes = sum(2 if n in TWO_PLANES else 1 for n, _ in variants)
    out0 = np.zeros((planes, B, T), np.float32) if out0 is None else np.array(out0, np.float32)   # a copy: written
    ph = None if phase is None else np.ascontiguousarray(phase, np.float32)
    (out,) = run_batch(s._lib, "spectralObj_spectralBatch",
                       (s._obj, np.ascontiguousarray(x, np.float32), ph, T, B, len(variants),
                        C.c_void_p(req.ctypes.data), C.c_void_p(par.ctypes.data), Out(out0)), device)
    res, k = {}, 0
    for i, (n, _) in enumerate(variants):
        np_ = 2 if n in TWO_PLANES else 1
        res[i] = tuple(out[k + j] for j in range(np_))
        k += np_
    return res


def spectral(num, fre, idx, mode, lib=None):
    """an af.Spectral over the bin list idx (a setEdge range when mode starts with 'range', else setEdgeArr)"""
    import audioflux_b200 as af
    s = af.Spectral(num, fre, _lib=lib)
    if mode.startswith("range"):
        s.set_edge(idx[0], idx[-1])
    elif mode != "full":
        s.set_edge_arr(idx)
    return s


# ---------------------------------------------------------------------------------------------------- inputs
def bin_sets():
    """(set, mode) -> bin list: the spectrogram sets of SC.spectrogram_sets in full, setEdge ranges of the linear set
    whose length mod 128 (the pass-1 stride) is 0, 1, 31 and 127, the unsorted list with a duplicate, one bin, two"""
    out = {("linear", "full"): list(range(1025)), ("mel", "full"): list(range(128)), ("cqt", "full"): list(range(84))}
    for n in (512, 513, 415, 639):
        out[("linear", f"range{n}")] = list(range(3, 3 + n))
    out[("linear", "list")] = SC.edges(1025)["list"]
    out[("mel", "list")] = SC.edges(128)["list"]
    out[("linear", "one")] = [700]
    out[("cqt", "two")] = [83, 2]
    return out


def clips(setname, T, B, seed=0):
    """(x [B, T, num] float32, phase or None, fre [num]) shaped as SC.spectrogram_sets; clip b is scaled by
    LEVELS[b % 2] and frames t = 5 + 11 b (mod 29) are all zero"""
    num, power, with_phase = {"linear": (1025, False, True), "mel": (128, True, False), "cqt": (84, False, False)}[setname]
    rng = np.random.default_rng([seed, T, B, num])
    x = np.abs(rng.standard_normal((B, T, num))).astype(np.float32) * np.linspace(2, 0.1, num, dtype=np.float32)
    if power:
        x = (x * x).astype(np.float32)
    for b in range(B):
        x[b] *= np.float32(LEVELS[b % 2])
        x[b, np.arange(T) % 29 == (5 + 11 * b) % 29] = 0
    ph = rng.uniform(-np.pi, np.pi, (B, T, num)).astype(np.float32) if with_phase else None
    fre = (np.arange(num) * 48000.0 / 2048).astype(np.float32) if setname == "linear" else \
        np.geomspace(30, 16000, num).astype(np.float32)
    return x, ph, fre


def temporal_variants(T):
    """flux / sd / sf / novelty at every step of STEPS, T - 1, T and T + 5"""
    steps = sorted({s for s in STEPS + (T - 1, T, T + 5) if s >= 1})
    out = []
    for s in steps:
        out += [("flux", dict(step=s)), ("sd", dict(step=s, is_positive=True)), ("sf", dict(step=s)),
                ("novelty", dict(step=s)), ("novelty", dict(step=s, method_type=2, data_type=1, threshold=0.5))]
    return out


# crafted rows: one clip of EXTREME_T frames over a list of EXTREME_NB positions (duplicates allowed) of EXTREME_NUM bins
EXTREME_NUM, EXTREME_T = 300, 70


def extreme_modes():
    """mode -> bin list of the crafted-row case: all bins, a range of 257 (1 past two pass-1 strides), a list of 200
    positions in no order with duplicates"""
    rng = np.random.default_rng(17)
    lst = rng.integers(0, EXTREME_NUM, 200)
    lst[[3, 77]] = lst[11]
    return {"full": list(range(EXTREME_NUM)), "range": list(range(3, 260)), "list": [int(v) for v in lst]}


# frames of the crafted case and what each holds
EXTREME_ROWS = {0: "NaN at list position 0", 3: "NaN mid-list", 6: "+inf mid-list", 9: "-inf mid-list",
                12: "denormals among normal bins", 15: "small negative bins", 18: "all zero", 19: "loud (x1e3)",
                20: "all zero", 24: "max tie across lanes", 25: "max tie within a lane", 26: "max tie across and within",
                31: "all zero", 32: "loud (x1e3)", 33: "+inf at list position 0", 40: "NaN at list position 0 and +inf"}


def extreme_clip(mode):
    """(x [T, num] float32, phase, fre) with the rows of EXTREME_ROWS over the bin list of extreme_modes()[mode];
    everything else is positive noise"""
    idx = extreme_modes()[mode]
    nb = len(idx)
    rng = np.random.default_rng(23)
    x = (np.abs(rng.standard_normal((EXTREME_T, EXTREME_NUM))) + 0.05).astype(np.float32)
    ph = rng.uniform(-np.pi, np.pi, x.shape).astype(np.float32)
    fre = np.linspace(0, 16000, EXTREME_NUM).astype(np.float32)
    pos = lambda p: idx[p % nb]                                           # noqa: E731
    x[0, pos(0)] = np.nan
    x[3, pos(nb // 2)] = np.nan
    x[6, pos(nb // 3)] = np.inf
    x[9, pos(nb // 3 + 5)] = -np.inf
    x[12, [pos(p) for p in range(0, nb, 7)]] = np.float32(3e-41)
    x[15, [pos(p) for p in range(1, nb, 9)]] = np.float32(-1e-3)
    x[[18, 20, 31]] = 0
    x[[19, 32]] *= 1e3
    x[33, pos(0)] = np.inf
    x[40, pos(0)] = np.nan
    x[40, pos(nb // 2)] = np.inf
    # the largest value at several list positions: different lanes (17, 40 -> lanes 17, 8), one lane (9, 41, 137:
    # lane 9, unrolled slots 0 and 1, then the next 128-position round)
    for t, ps in ((24, (40, 17, 66)), (25, (137, 41, 9)), (26, (82, 146, 18, 50))):
        top = np.float32(x[t].max() * 4)
        ps = [p for p in ps if p < nb] or [0]
        x[t, [pos(p) for p in ps]] = top
    return x, ph, fre


def lookback_clips(kind):
    """(x [2, T, num], fre, threshold) whose rolloff fails to cross on runs of frames: kind 'nan' has rows holding a NaN
    (threshold 0.95), kind 'neg' has positive rows that cannot reach threshold 1.5 while the crossing rows hold
    negative bins.  Runs start at frame 0 and follow crossing frames; they last 5, 31, 32, 33, 64 and 70 frames, so
    the look-back takes one, two and three 32-frame rounds and straddles tiles.  Clip 1 starts with a run of its own:
    frame 0 of clip 1 must fall back to fre[0], not to clip 0's last crossing."""
    num, T = 97, 300
    rng = np.random.default_rng(29 if kind == "nan" else 31)
    fre = np.linspace(10, 9000, num).astype(np.float32)
    x = (np.abs(rng.standard_normal((2, T, num))) + 0.1).astype(np.float32)
    runs = ([5, 31, 32, 33, 64, 70, 20], [40, 3, 33, 64, 70, 32, 31])
    cross = np.ones((2, T), bool)
    for b in range(2):
        t = 0
        for k, n in enumerate(runs[b]):
            cross[b, t:t + n] = False
            t += n + 1 + (k % 2)             # one or two crossing frames between runs
    for b in range(2):
        for t in range(T):
            if kind == "nan" and not cross[b, t]:
                x[b, t, rng.integers(num)] = np.nan
            elif kind == "neg" and cross[b, t]:
                # every third bin negative: the net sum is about a third of the sum of |x|, so 1.5 times it is reached
                x[b, t, (np.arange(num) + t) % 3 == 0] *= -1
    return x, fre, 0.95 if kind == "nan" else 1.5, cross


LOOKBACK_VARIANTS = {"nan": None,               # None: every variant
                     "neg": [("rolloff", dict(threshold=1.5)), ("rolloff", {}), ("max", {}), ("broadband", {})]}
