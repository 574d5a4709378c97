"""Float64 numpy restatement of the reference's harmonic ratio, the case list, and ctypes drivers that work on either
library.

src/mir/harmonicRatio_algorithm.c, with W = 2^radix2Exp and N = 2W:
  - new (:52-155): samplate outside (0, 196000] -> 32000; lowFre outside (0, samplate/2) (the integer samplate/2) -> 25;
    radix2Exp outside 0 .. 29 -> W = 2^11; slideLength <= 0 -> W/4; maxLength = floorf(samplate / lowFre) in float,
    at most W-1.  The window is always the periodic Hamming window (windowType is not read);
  - calTimeLength (:157-170): 0 when dataLength < W, else (dataLength - W) / slide + 1;
  - per frame (:224-286): x = frame * window; r = Re IFFT_N(|FFT_N(x)|^2) (the 1/N of the inverse FFT kept);
    E[j] = sum of x[m]^2 for m <= W-2-j; minIndex = (first j in 2 .. maxLength where r[j], r[j-1] change sign, zeros
    included) - 1, else the last frame's (0 at the start of the call); g[k] = r[j] / sqrt(r[0] E[j] + 1e-16) for
    j = minIndex+1 .. maxLength-1; the first arg-max of g, refined by the parabola through its neighbours unless it is
    the first or the last of g; 0 when g is empty.

Everything is float64 except where a float32 value decides something: the sign tests of the crossing and the arg-max
(with its first-of-equal rule) run on the float32 roundings of r and g, so that exact zeros and exact ties (silence)
decide as in the reference.  Where the float64 values leave a decision undetermined -- |r[j]| or |r[j-1]| within
EPS_R r[0] of 0, or a g within EPS_G max|g| of the top -- every outcome is kept as a candidate, and a candidate crossing
carries its candidates into the frames without one."""
import ctypes as C

import numpy as np

from oracle import af_oracle as O

W_RECT, W_HANN, W_HAMM = O.W_RECT, O.W_HANN, O.W_HAMM
f32 = np.float32
EPS_R = 1e-5      # a sign test is undetermined when r[j] or r[j-1] lies within EPS_R r[0] of 0
EPS_G = 1e-5      # an arg-max is undetermined among the g within EPS_G max|g| of the top


def params(samplate=None, low_fre=None, radix2_exp=None, slide=None):
    """:52-155 -> dict(sr, W, slide, max_length, lf)"""
    sr = samplate if samplate is not None and 0 < samplate <= 196000 else 32000
    lf = f32(low_fre) if low_fre is not None else None
    if lf is None or not (lf > 0 and lf < f32(sr // 2)):
        lf = f32(25)
    log2w = radix2_exp if radix2_exp is not None and 1 <= radix2_exp + 1 <= 30 else 11
    W = 1 << log2w
    hop = slide if slide is not None and slide > 0 else W // 4
    q = np.floor(f32(sr) / lf)
    ml = W - 1 if q > W - 1 else int(q)
    return dict(sr=sr, W=W, slide=hop, max_length=ml, lf=lf)


def time_length(n, W, hop):
    return 0 if n < W else (n - W) // hop + 1


def _interp(v1, v2, v3):
    """util_qaudInterp (src/util/flux_util.c) in float64"""
    p = (v3 - v1) / (2 * (2 * v2 - v3 - v1) + 1e-16)
    return v2 - 0.25 * (v1 - v3) * p


def _frame_parts(x, W, hop, ml):
    """per frame: r[0 .. ml] and E[0 .. W-1] (prefix sums of x^2), float64"""
    x = np.asarray(x, np.float64)
    T = time_length(x.size, W, hop)
    idx = np.arange(T)[:, None] * hop + np.arange(W)[None, :]
    xw = x[idx] * O.fft_window(W_HAMM, W).astype(np.float64)[None, :]
    n = 2 * W
    r = np.fft.irfft(np.abs(np.fft.rfft(xw, n, axis=1)) ** 2, n, axis=1)[:, :ml + 1]
    return r, np.cumsum(xw * xw, axis=1)


def _own_crossings(r, ml):
    """(primary minIndex or None, set of candidate minIndex, 'none' possible) of one frame"""
    if ml < 2:
        return None, set(), True
    r32 = r.astype(f32)
    a, b = r32[2:ml + 1], r32[1:ml]
    cross = ((a >= 0) & (b <= 0)) | ((a <= 0) & (b >= 0))
    near = np.minimum(np.abs(r[2:ml + 1]), np.abs(r[1:ml])) < EPS_R * abs(r[0])
    hit = np.flatnonzero(cross)
    primary = int(hit[0]) + 1 if hit.size else None               # j - 1 with j = 2 + index
    stop = np.flatnonzero(cross & ~near)
    end = int(stop[0]) if stop.size else ml - 1
    cands = {int(i) + 1 for i in np.flatnonzero(near[:end])} | ({end + 1} if stop.size else set())
    return primary, cands, not stop.size


def _values(r, E, W, ml, m):
    """(primary value, set of candidate (value, slack)) of one frame with minIndex m.  The slack of a lag is what an
    error of EPS_R r[0] in r[j] moves g by, r[j] / sqrt(r[0] E[j]): large only where E[j] is tiny, at the window's end."""
    n = ml - m - 1
    if n <= 0:
        return 0.0, {(0.0, 0.0)}
    j = np.arange(m + 1, ml)
    d = np.sqrt(r[0] * E[W - 2 - j] + 1e-16)
    g = r[j] / d
    u = EPS_R * abs(r[0]) / d + EPS_G * np.nanmax(np.abs(g))
    g32 = g.astype(f32)

    def out(k):
        if k == 0 or k == n - 1:
            return float(g[k]), float(u[k])
        return float(_interp(g[k - 1], g[k], g[k + 1])), 2 * float(u[k - 1:k + 2].max())

    k0 = 0 if np.isnan(g32[0]) else int(np.argmax(g32))     # np.argmax: the first of equal values
    near = np.flatnonzero(g + u >= np.nanmax(g - u))
    return out(k0)[0], {out(k) for k in near} | {out(k0)}


def harmonic_ratio(x, W, hop, ml):
    """one clip -> (values [T] float64, candidates: list of sets of (value, slack), own crossing per frame or None)"""
    if time_length(len(x), W, hop) == 0:
        return np.zeros(0), [], []
    r, E = _frame_parts(x, W, hop, ml)
    vals, cands, own = [], [], []
    carry, carry_set = 0, {0}
    for t in range(r.shape[0]):
        primary, cm, none_possible = _own_crossings(r[t], ml)
        m = carry if primary is None else primary
        ms = cm | (carry_set if none_possible else set())
        v, vs = _values(r[t], E[t], W, ml, m)
        for mm in ms - {m}:
            vs |= _values(r[t], E[t], W, ml, mm)[1]
        vals.append(v)
        cands.append(vs)
        own.append(primary)
        if primary is not None:
            carry = primary
        carry_set = ms if none_possible else cm
    return np.array(vals), cands, own


def agree(got, want, cands, tol):
    """(ok, frames decided by a candidate): each frame within tol of the primary value, or within tol plus its slack of
    one of its candidates"""
    got = np.asarray(got, np.float64)
    if got.shape != want.shape:
        return False, []
    alt = []
    for t in np.flatnonzero(~(np.abs(got - want) <= tol)):
        if not any(abs(got[t] - c) <= tol + s for c, s in cands[t]):
            return False, [int(t)]
        alt.append(int(t))
    return True, alt


# ---- test signals ----

def signal(kind, length, sr, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(length) / sr
    if kind == "silence":
        x = np.zeros(length)
    elif kind == "noise":
        x = 0.1 * rng.standard_normal(length)
    elif kind == "tones":                       # a harmonic tone: 220 Hz and five overtones, a little noise
        x = sum(0.3 / h * np.sin(2 * np.pi * 220 * h * t + h) for h in range(1, 7)) + 0.01 * rng.standard_normal(length)
    elif kind == "sweep":
        x = 0.5 * np.sin(2 * np.pi * (100 * t + 0.5 * (sr / 8 - 100) * t * t / max(t[-1], 1e-9)))
    elif kind == "impulses":                    # a click every 160 samples
        x = np.zeros(length)
        x[::160] = 1.0
        x += 1e-3 * rng.standard_normal(length)
    elif kind == "dc":                          # a large offset: no autocorrelation crosses zero below maxLength
        x = 1.0 + 0.05 * rng.standard_normal(length)
    elif kind == "low":                         # a sine far below lowFre: the first crossing lies beyond maxLength
        x = np.sin(2 * np.pi * 3 * t) + 0.001 * rng.standard_normal(length)
    elif kind == "dc_then_tones":               # frames without a crossing from frame 0, then frames with one
        x = np.where(t < t[length // 2], 1.0 + 0.05 * rng.standard_normal(length),
                     np.sin(2 * np.pi * 440 * t) + 0.1 * rng.standard_normal(length))
    elif kind == "tones_dc_tones":              # crossings, a stretch without, crossings again: the carry in the middle
        x = sum(0.3 / h * np.sin(2 * np.pi * 310 * h * t) for h in range(1, 4)) + 0.02 * rng.standard_normal(length)
        x[length // 3:2 * length // 3] = 2.0 + 0.01 * rng.standard_normal(length // 3 + 1)[:2 * length // 3 - length // 3]
    else:
        raise ValueError(kind)
    return np.asarray(x, f32)


def cases():
    """[(name, dict(sr, lf, r2, wt, slide, length, kind))]: None arguments are passed as NULL"""
    out = []
    for r2 in range(1, 14):
        W = 1 << r2
        length = 2 * W + 7 if r2 >= 12 else W + 5 * max(1, W // 2) + 3
        out.append((f"r{r2}", dict(sr=32000, lf=200.0, r2=r2, wt=W_HAMM, slide=max(1, W // 2), length=length,
                                   kind="tones")))
    for sr, lf in ((None, None), (0, 100.0), (-5, 100.0), (196000, 100.0), (196001, 100.0), (8000, None), (8000, 0.0),
                   (8000, -1.0), (8000, 4000.0), (8000, 3999.5), (8001, 4000.0), (44100, 1.0), (16000, 30.0)):
        out.append((f"sr{sr}_lf{lf}", dict(sr=sr, lf=lf, r2=10, wt=W_HAMM, slide=256, length=6000, kind="tones")))
    for slide in (None, 0, -3, 1, 1024, 1500):
        out.append((f"slide{slide}", dict(sr=16000, lf=50.0, r2=10, wt=W_HAMM, slide=slide,
                                          length=1024 + 40 if slide == 1 else 8000, kind="noise")))
    out += [
        ("capped", dict(sr=44100, lf=5.0, r2=9, wt=W_HAMM, slide=200, length=5000, kind="tones")),
        ("r2default", dict(sr=32000, lf=100.0, r2=None, wt=W_HAMM, slide=1000, length=9000, kind="tones")),
        ("r2_minus1", dict(sr=32000, lf=100.0, r2=-1, wt=W_HAMM, slide=1000, length=9000, kind="noise")),
        ("t0", dict(sr=32000, lf=100.0, r2=10, wt=W_HAMM, slide=256, length=1023, kind="noise")),
        ("t1", dict(sr=32000, lf=100.0, r2=10, wt=W_HAMM, slide=256, length=1024, kind="noise")),
        ("hann", dict(sr=32000, lf=100.0, r2=10, wt=W_HANN, slide=256, length=6000, kind="tones")),
        ("rect", dict(sr=32000, lf=100.0, r2=10, wt=W_RECT, slide=256, length=6000, kind="tones")),
        ("wt_null", dict(sr=32000, lf=100.0, r2=10, wt=None, slide=256, length=6000, kind="tones")),
    ]
    for kind in ("silence", "noise", "tones", "sweep", "impulses", "dc", "low", "dc_then_tones", "tones_dc_tones"):
        out.append((f"sig_{kind}", dict(sr=32000, lf=32.703196, r2=11, wt=W_HAMM, slide=512, length=32000, kind=kind)))
    out.append(("h12_dc", dict(sr=32000, lf=32.703196, r2=12, wt=W_HAMM, slide=1024, length=20000, kind="dc")))
    return out


def case_signal(name, kw):
    return signal(kw["kind"], kw["length"], kw["sr"] if kw["sr"] and 0 < kw["sr"] <= 196000 else 32000,
                  sum(map(ord, name)))


def case_params(kw):
    return params(kw["sr"], kw["lf"], kw["r2"], kw["slide"])


def oracle_case(name, kw):
    p = case_params(kw)
    return harmonic_ratio(case_signal(name, kw), p["W"], p["slide"], p["max_length"])


# ---- ctypes drivers (either library) ----

def _ip(v):
    return None if v is None else C.byref(C.c_int(v))


def c_new(lib, sr=None, lf=None, r2=None, wt=None, slide=None):
    obj = C.c_void_p()
    st = lib.harmonicRatioObj_new(C.byref(obj), _ip(sr), None if lf is None else C.byref(C.c_float(lf)), _ip(r2),
                                  _ip(wt), _ip(slide))
    return st, obj


def c_ratio(lib, obj, x, fill=0.0, extra=0):
    """harmonicRatioObj_harmonicRatio -> the output buffer of T + extra floats, which started as `fill`"""
    x = np.ascontiguousarray(x, f32)
    T = lib.harmonicRatioObj_calTimeLength(obj, x.size)
    out = np.full(T + extra, fill, f32)
    lib.harmonicRatioObj_harmonicRatio(obj, x.ctypes.data, x.size, out.ctypes.data)
    return out


def c_case(lib, name, kw):
    st, obj = c_new(lib, kw["sr"], kw["lf"], kw["r2"], kw["wt"], kw["slide"])
    assert st == 0, (name, st)
    out = c_ratio(lib, obj, case_signal(name, kw))
    lib.harmonicRatioObj_free(obj)
    return out
