"""Float64 numpy restatement of the reference's pitch estimation filter (PitchPEF), the case list, and ctypes drivers
that work on either library.

src/mir/_pitch_pef.c, with n = 2^radix2Exp:
  - new (:106-231): samplate outside (0, 196000] -> 32000; lowFre < 27 -> 32; highFre not in (lowFre, samplate/2)
    (integer samplate/2) -> lowFre 32, highFre 2000; cutFre < highFre -> highFre (NULL: 4000); radix2Exp outside
    1 .. 30 -> 12; alpha <= 0 -> 10; beta <= 0 -> 0.5; gamma <= 1 -> 1.8; slideLength <= 0 -> n/4;
  - the tables (__pitchPEFObj_initData, :428-522): lin = linspace(0, samplate/2, n+1); fre1 = cutFre if samplate/2 >
    cutFre else samplate/2 - 1; log = 10^linspace(1, log10f(fre1), 2n); minIndex / maxIndex by the reference's loop;
    bandWidth[j] = (log[j+1] - log[j-1]) / 4n with both ends copied;
  - the filter (__pitchPEFObj_calEstimateFilter, :696-785): q = 10^linspace(log10 beta, log10(alpha+beta), n),
    h = 1/(gamma - cosf(2 pi q)), det = sum(d h) / sum(d) over the interval widths d, filter = h - det, P = #{q < 1},
    xcorrFFTLength = 8n if P else 4n;
  - per frame (:258-382): power of the 2n-point FFT of the windowed frame, bins 0 .. n; __vinterp_linear onto the log
    grid (src/vector/flux_vectorOp.c:580); times bandWidth, after P zeros; c = IFFT(FFT(s) conj(FFT(filter)));
  - the result (:384-426): util_peakPick's one peak (src/util/flux_util.c:783), __vmax's first maximum, over the lags
    minIndex .. maxIndex when len = maxIndex + 1 (len is clipped only when P = 0 and maxIndex = 2n - 1, a case this
    library refuses); freArr[t] = log[lag].
The tables are built in float32, each operation rounded as in the reference, with the C library's powf, log10f and cosf
(through ctypes), so that minIndex, maxIndex, P and every output frequency are exact.  The per-frame pipeline is float64.

The arg-max is undetermined when several lags lie within EPS ||s|| ||filter|| of the top correlation value (the
Cauchy-Schwarz bound of |c|, the scale of a float32 rounding error of c): each of those lags is then a candidate.  A
frame whose correlation is exactly 0 everywhere (silence) has the first lag as its only outcome."""
import ctypes as C
import ctypes.util
import math

import numpy as np

from _pitch_c import c_free, c_new, c_pitch, signal, time_length
from oracle import af_oracle as O

W_RECT, W_HANN, W_HAMM = O.W_RECT, O.W_HANN, O.W_HAMM
f32 = np.float32
EPS = 4e-6

_libm = C.CDLL(ctypes.util.find_library("m"))
for _name, _args in (("powf", [C.c_float, C.c_float]), ("log10f", [C.c_float]), ("cosf", [C.c_float])):
    getattr(_libm, _name).restype = C.c_float
    getattr(_libm, _name).argtypes = _args


def _linspace(start, stop, length):
    """__vlinspace (src/vector/flux_vector.c:2145) in float32"""
    start, stop = f32(start), f32(stop)
    step = f32(stop - start) / f32(length - 1 if length - 1 > 0 else 1)
    return np.array([f32(start + f32(f32(i) * step)) for i in range(length)], f32)


def _logspace(start, stop, length):
    """__vlogspace (:2164): powf(10, linspace)"""
    return np.array([_libm.powf(10.0, float(v)) for v in _linspace(start, stop, length)], f32)


def params(sr=None, lf=None, hf=None, cf=None, r2=None, slide=None, wt=None, alpha=None, beta=None, gamma=None):
    """:106-231 and the tables -> dict; status 0, or this library's refusals -2 (radix2Exp > 13), -3 (empty lag range),
    -4 (the clipped peak search)"""
    sr = sr if sr is not None and 0 < sr <= 196000 else 32000
    sr2 = sr // 2
    low = f32(lf) if lf is not None and f32(lf) >= 27 else f32(32)
    high, cut = f32(2000), f32(4000)
    if hf is not None:
        if f32(hf) > low and f32(hf) < f32(sr2):
            high = f32(hf)
        else:
            low, high = f32(32), f32(2000)
    if cf is not None:
        cut = f32(cf) if f32(cf) >= high else high
    r2 = r2 if r2 is not None and 1 <= r2 <= 30 else 12
    n = 1 << r2
    hop = slide if slide is not None and slide > 0 else max(1, n // 4)
    al = f32(alpha) if alpha is not None and f32(alpha) > 0 else f32(10)
    be = f32(beta) if beta is not None and f32(beta) > 0 else f32(0.5)
    ga = f32(gamma) if gamma is not None and f32(gamma) > 1 else f32(1.8)
    p = dict(sr=sr, n=n, r2=r2, slide=hop, low=low, high=high, cut=cut, wt=W_HAMM if wt is None else wt,
             alpha=al, beta=be, gamma=ga)
    if r2 > 13:
        return dict(p, status=-2)
    lin = _linspace(0, sr2, n + 1)
    fre1 = cut if f32(sr2) > cut else f32(sr2 - 1)
    lg = _logspace(1, _libm.log10f(float(fre1)), 2 * n)
    mi, ma = -1, 0
    for i in range(1, 2 * n):
        if high < lg[i]:
            ma = i if lg[i] - high < high - lg[i - 1] else i - 1
            break
        if mi != -1:
            continue
        if low < lg[i]:
            mi = i if lg[i] - low < low - lg[i - 1] else i - 1
    bw = np.zeros(2 * n, f32)
    bw[1:2 * n - 1] = (lg[2:] - lg[:-2]) / f32(4 * n)
    bw[0], bw[-1] = bw[1], bw[-2]
    q = _logspace(_libm.log10f(float(be)), _libm.log10f(float(f32(al + be))), n)
    P = int(np.count_nonzero(q < 1))
    h = np.array([f32(1) / f32(ga - f32(_libm.cosf(float(f32(2 * math.pi * float(v)))))) for v in q], f32)
    d = np.empty(n + 1, f32)
    d[0] = q[0]
    d[1:n] = (q[:-1] + q[1:]) / f32(2)
    d[n] = q[n - 1]
    d = d[1:] - d[:-1]
    v1 = f32(np.cumsum(d.astype(np.float64))[-1])
    v2 = f32(np.cumsum((d * h).astype(np.float64))[-1])
    filt = h - f32(v2 / v1)
    p.update(lin=lin, log=lg, bw=bw, min_index=mi, max_index=ma, pad=P, filter=filt,
             xcorr_length=8 * n if P else 4 * n)
    if mi < 0 or ma <= mi:
        return dict(p, status=-3)
    if P == 0 and ma >= 2 * n - 1:
        return dict(p, status=-4)
    return dict(p, status=0)


def correlations(x, p):
    """per frame, c over the lags min_index .. max_index and the Cauchy-Schwarz scale ||s|| ||filter||, float64"""
    n, hop = p["n"], p["slide"]
    x = np.asarray(x, np.float64)
    T = time_length(x.size, n, hop)
    idx = np.arange(T)[:, None] * hop + np.arange(n)[None, :]
    xw = x[idx] * O.fft_window(p["wt"], n).astype(np.float64)[None, :]
    power = np.abs(np.fft.rfft(xw, 2 * n, axis=1)) ** 2                       # T x (n + 1)
    lin, lg = p["lin"].astype(np.float64), p["log"].astype(np.float64)
    seg = np.minimum(np.searchsorted(p["lin"], p["log"], side="left") - 1, n)   # __vinterp_linear's index
    seg = np.maximum.accumulate(np.maximum(seg, 0))
    inner = seg < n
    j = np.minimum(seg, n - 1)
    x1, x2 = lin[j], lin[j + 1]
    y1, y2 = power[:, j], power[:, j + 1]
    v = np.where(inner[None, :], y1 + (lg - x1)[None, :] * (y2 - y1) / (x2 - x1)[None, :], power[:, n:n + 1])
    L, P = p["xcorr_length"], p["pad"]
    s = np.zeros((T, L))
    s[:, P:P + 2 * n] = v * p["bw"].astype(np.float64)[None, :]
    F = np.fft.rfft(p["filter"].astype(np.float64), L)
    c = np.fft.irfft(np.fft.rfft(s, axis=1) * np.conj(F)[None, :], L, axis=1)
    scale = np.linalg.norm(s, axis=1) * np.linalg.norm(p["filter"].astype(np.float64))
    return c[:, p["min_index"]:p["max_index"] + 1], scale


def pitch(x, p, block=64):
    """one clip -> (frequencies [T] float32, candidate lags per frame as sets); `block` frames at a time"""
    n, hop = p["n"], p["slide"]
    lo = p["min_index"]
    best, cands = [], []
    for t0 in range(0, time_length(len(x), n, hop), block):
        _decide(*correlations(x[t0 * hop:(t0 + block - 1) * hop + n], p), lo, best, cands)
    return p["log"][np.array(best, int)] if best else np.zeros(0, f32), cands


def _decide(c, scale, lo, best, cands):
    for t in range(c.shape[0]):
        if scale[t] == 0:
            best.append(lo)
            cands.append({lo})
            continue
        k = int(np.argmax(c[t]))
        best.append(lo + k)
        cands.append({lo + int(i) for i in np.flatnonzero(c[t] >= c[t, k] - EPS * scale[t])})


def agree(got, want, cands, p):
    """(ok, frames decided by a candidate): each frame's frequency is exactly the oracle's, or exactly the frequency of
    one of its candidate lags"""
    got = np.asarray(got)
    if got.shape != want.shape:
        return False, []
    alt = []
    for t in np.flatnonzero(got != want):
        if got[t] not in {p["log"][k] for k in cands[t]}:
            return False, [int(t)]
        alt.append(int(t))
    return True, alt


# ---- cases ----

def cases():
    """[(name, dict(ctor=dict(...), length, kind))]: ctor arguments left out are passed as NULL"""
    out = []

    def add(name, length, kind="tones", **ctor):
        out.append((name, dict(ctor=ctor, length=length, kind=kind)))

    add("default", 4096 + 30 * 1024)
    add("default_null", 4096 + 20 * 1024, slide=None)
    for r2 in (11, 13):
        n = 1 << r2
        add(f"r{r2}", n + 24 * (n // 4), sr=32000, r2=r2, slide=n // 4)
    for sr in (11025, 22050, 44100, 16000):
        add(f"sr{sr}", 2 * sr, sr=sr, r2=12, slide=1000)
    add("cut_above_nyquist", 16000, sr=8000, hf=1500.0, cf=6000.0, r2=11, slide=512)
    add("cut_at_nyquist_odd", 22050, sr=11025, hf=3000.0, cf=5512.0, r2=12, slide=700)
    add("cut_low", 32000, sr=32000, lf=60.0, hf=800.0, cf=1000.0, r2=12, slide=1024)
    add("beta1", 32000, beta=1.0, r2=12, slide=1024)
    add("beta1_r11", 16000, sr=16000, beta=1.0, r2=11, slide=400)
    add("slide_gt_n", 60000, r2=12, slide=5000)
    add("slide1", 2048 + 40, r2=11, slide=1, kind="noise")
    add("alpha5_gamma15", 32000, alpha=5.0, gamma=1.5, r2=12, slide=1024)
    add("beta02", 32000, beta=0.2, r2=12, slide=1024)
    add("hann", 32000, wt=W_HANN, r2=12, slide=1024)
    add("rect", 32000, wt=W_RECT, r2=12, slide=1024)
    add("lf_fallback", 32000, lf=20.0, hf=1000.0, r2=12, slide=1024)
    add("hf_fallback", 32000, sr=8000, lf=100.0, hf=4500.0, r2=12, slide=1024)
    add("sr_fallback", 32000, sr=0, r2=12, slide=1024)
    add("params_fallback", 32000, alpha=-1.0, beta=0.0, gamma=0.5, r2=12, slide=1024)
    add("r5", 600, r2=5, slide=16)
    for kind in ("silence", "dc", "noise", "tones", "missing", "glide"):
        add(f"sig_{kind}", 48000, kind=kind, sr=32000, r2=12, slide=1024)
    add("sig_missing_r11", 48000, kind="missing", sr=22050, r2=11, slide=512)
    add("sig_glide_r13", 8192 + 30 * 2048, kind="glide", sr=44100, r2=13, slide=2048)
    return out


def case_params(kw):
    return params(**kw["ctor"])


def case_signal(name, kw):
    return signal(kw["kind"], kw["length"], case_params(kw)["sr"], sum(map(ord, name)))


def oracle_case(name, kw):
    p = case_params(kw)
    return pitch(case_signal(name, kw), p)


def c_case(lib, name, kw):
    st, obj = c_new(lib, "pef", **kw["ctor"])
    assert st == 0, (name, st)
    out = c_pitch(lib, "pef", obj, case_signal(name, kw))
    c_free(lib, "pef", obj)
    return out
