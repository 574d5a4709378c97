"""Float64 numpy restatement of the reference's YIN pitch tracker (PitchYIN) with error intervals, the case list, and
ctypes drivers that work on either library.

src/mir/_pitch_yin.c, with n = 2^radix2Exp and A = autoLength:
  - new (:87-195): samplate outside (0, 196000] -> 32000; lowFre < 27 -> 27; highFre NULL -> 2094; highFre not in
    (lowFre, samplate/2) (integer samplate/2) -> lowFre 27, highFre 2093; radix2Exp outside 1 .. 30 -> 12;
    slideLength <= 0 -> n/4; autoLength outside [0, n) -> n/2; minIndex = floorf(samplate/highFre), maxIndex =
    ceilf(samplate/lowFre) clamped to n - A - 1 (float quotients); yinLength = maxIndex - minIndex + 1; thresh 0.1;
  - per frame (:350-453): r[k] = sum_{m<=A} x[m] x[m+k] (the float32 FFT correlation), E the float32 running sum of
    x^2, e2[j] = E[A+j] - E[j], both set to 0 below 1e-6; d = e2[0] + e2[j] - 2 r[j]; mean = float32 running sums of
    d[1 ..] over their counts; yin[k] = d[minIndex+k] / (mean[minIndex-1+k] + 1e-16) in double;
  - offsets (:462-503) and troughs (:541-625) as include/afb200_pitch_yin.h restates them.
E and e2 are computed literally in float32 (np.add.accumulate is sequential), so they are exact.  r is computed in
float64; the float32 FFT correlation of either library is within KAPPA ||frame|| ||x[0..A]|| of it.  KAPPA: a float32
radix-2 FFT of n <= 2^14 points has an l2 error of about 2^-24 log2 n <= 8.4e-7 of its output's norm; the correlation
runs two forward transforms, a product and one inverse, whose errors add to about 4 x 8.4e-7 of ||x|| ||y|| in l2, a
bound on every lag (the same form and value as the PEF oracle's 4e-6).  That bound, the
float32 rounding of d, of the running sums and of each division, are carried as intervals through d, the mean, yin,
the offsets and the frequencies.  A comparison whose intervals overlap is undetermined: a trough flag is then certain,
impossible or undetermined, and the first trough's candidates are every index from the first flag that is not
impossible up to the first certain one (and "no trough" when no flag is certain)."""
import ctypes as C

import numpy as np

from _pitch_c import c_free, c_new, c_pitch, signal, time_length

f32 = np.float32
KAPPA = 4e-6
U = 2.0 ** -24                    # float32 unit roundoff


def params(sr=None, lf=None, hf=None, r2=None, slide=None, auto=None):
    """:87-195 -> dict; status 0, or this library's refusals -2 (radix2Exp > 14) and -3 (minIndex < 1 or yinLength < 1)"""
    sr = sr if sr is not None and 0 < sr <= 196000 else 32000
    low = f32(lf) if lf is not None and f32(lf) >= 27 else f32(27)
    high = f32(2094)
    if hf is not None:
        if f32(hf) > low and f32(hf) < f32(sr // 2):
            high = f32(hf)
        else:
            low, high = f32(27), f32(2093)
    r2 = r2 if r2 is not None and 1 <= r2 <= 30 else 12
    n = 1 << r2
    hop = slide if slide is not None and slide > 0 else max(1, n // 4)
    A = auto if auto is not None and 0 <= auto < n else n // 2
    mi = int(np.floor(f32(sr) / high))
    ma = min(int(np.ceil(f32(sr) / low)), n - A - 1)
    p = dict(sr=sr, n=n, r2=r2, slide=hop, auto=A, low=low, high=high, min_index=mi, max_index=ma,
             yin_length=ma - mi + 1, m_len=(ma - mi + 1) // 2 + 1, thresh=f32(0.1))
    if r2 > 14:
        return dict(p, status=-2)
    if mi < 1 or ma < mi:
        return dict(p, status=-3)
    return dict(p, status=0)


def _frames(x, p):
    n, hop = p["n"], p["slide"]
    T = time_length(x.size, n, hop)
    return x[np.arange(T)[:, None] * hop + np.arange(n)[None, :]]


def _clamp(lo, hi):
    """the 1e-6 clamp of a value known to lie in [lo, hi]"""
    keep = np.minimum(np.abs(lo), np.abs(hi)) >= 1e-6
    keep &= np.sign(lo) == np.sign(hi)
    drop = np.maximum(np.abs(lo), np.abs(hi)) < 1e-6
    return (np.where(keep, lo, np.where(drop, 0.0, np.minimum(lo, 0.0))),
            np.where(keep, hi, np.where(drop, 0.0, np.maximum(hi, 0.0))))


def _div(alo, ahi, blo, bhi):
    """[alo, ahi] / [blo, bhi], unbounded where the divisor's interval holds 0"""
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.stack([alo / blo, alo / bhi, ahi / blo, ahi / bhi])
        lo, hi = q.min(0), q.max(0)
    zero = (blo <= 0) & (bhi >= 0)
    return np.where(zero, -np.inf, lo), np.where(zero, np.inf, hi)


def _widen(lo, hi, rel):
    return lo - rel * np.abs(lo), hi + rel * np.abs(hi)


def yin_rows(x, p):
    """one clip -> (lo, hi) of every frame's yin row [T, yinLength], float64 intervals"""
    n, A, M, mi = p["n"], p["auto"], p["max_index"], p["min_index"]
    xf = _frames(np.asarray(x, f32), p)                                 # T x n float32
    T = xf.shape[0]
    if T == 0:
        z = np.zeros((0, p["yin_length"]))
        return z, z
    x64 = xf.astype(np.float64)
    y = np.zeros_like(x64)
    y[:, :A + 1] = x64[:, A::-1]
    c = np.fft.irfft(np.fft.rfft(x64, axis=1) * np.fft.rfft(y, axis=1), n, axis=1)
    r = c[:, A:A + M + 1]
    delta = KAPPA * np.linalg.norm(x64, axis=1) * np.linalg.norm(x64[:, :A + 1], axis=1)
    rlo, rhi = _clamp(r - delta[:, None], r + delta[:, None])
    E = np.add.accumulate(xf * xf, axis=1, dtype=f32)                   # sequential float32, as :388-398
    e2 = (E[:, A:A + M + 1] - E[:, :M + 1]).astype(np.float64)
    e2 = np.where(np.abs(e2) >= 1e-6, e2, 0.0)
    s = e2[:, :1] + e2                                                  # exact in float32 and float64 alike
    dlo, dhi = s - 2 * rhi, s - 2 * rlo
    dlo, dhi = _widen(dlo, dhi, 2 * U)                                  # d rounded to float32
    # the float32 running sums of d[1 .. k+1]: each partial sum rounded, so the sum drifts by U |S_i| per step
    Slo, Shi = np.cumsum(dlo[:, 1:], axis=1), np.cumsum(dhi[:, 1:], axis=1)
    drift = 1.01 * U * np.cumsum(np.maximum(np.abs(Slo), np.abs(Shi)), axis=1)
    cnt = np.arange(1, M + 1, dtype=np.float64)
    mlo, mhi = _widen((Slo - drift) / cnt, (Shi + drift) / cnt, 2 * U)  # the float division
    k = np.arange(p["yin_length"])
    ylo, yhi = _div(dlo[:, mi + k], dhi[:, mi + k], mlo[:, mi - 1 + k] + 1e-16, mhi[:, mi - 1 + k] + 1e-16)
    return _widen(ylo, yhi, 2 * U)


def _lt(alo, ahi, blo, bhi):
    """a < b: 1 certain, 0 impossible, -1 undetermined"""
    return np.where(ahi < blo, 1, np.where(alo >= bhi, 0, -1))


def _le(alo, ahi, blo, bhi):
    return np.where(ahi <= blo, 1, np.where(alo > bhi, 0, -1))


def _and(*conds):
    out = np.ones_like(conds[0])
    for c in conds:
        out = np.where((out == 0) | (c == 0), 0, np.where((out == 1) & (c == 1), 1, -1))
    return out


def trough_flags(lo, hi, thresh):
    """[T, Y] of 1 (certain), 0 (impossible) or -1 (undetermined), :546-572"""
    T, Y = lo.shape
    flags = np.zeros((T, Y), int)
    th = float(thresh)
    below = np.where(hi < th, 1, np.where(lo >= th, 0, -1))
    if Y >= 2:
        flags[:, 0] = _and(_lt(lo[:, 0], hi[:, 0], lo[:, 1], hi[:, 1]), below[:, 0])
    if Y >= 3:
        j = np.arange(1, Y - 1)
        flags[:, j] = _and(_le(lo[:, j], hi[:, j], lo[:, j + 1], hi[:, j + 1]),
                           _lt(lo[:, j], hi[:, j], lo[:, j - 1], hi[:, j - 1]), below[:, j])
    return flags


def fre_interval(lo, hi, k, p):
    """interval of samplate / (minIndex + k + offset[k]) for one row's yin interval, :485-501 and :575-578"""
    Y = lo.size
    olo = ohi = 0.0
    if 1 <= k <= Y - 2 and not np.isfinite(np.r_[lo[k - 1:k + 2], hi[k - 1:k + 2]]).all():
        olo, ohi = -1.0, 1.0
    elif 1 <= k <= Y - 2:
        # num and den in float32: each sum rounded (U of its terms), then halved exactly
        a = np.abs(np.r_[lo[k - 1:k + 2], hi[k - 1:k + 2]]).max()
        nlo, nhi = (lo[k + 1] - hi[k - 1]) / 2 - U * a, (hi[k + 1] - lo[k - 1]) / 2 + U * a
        dlo = (lo[k - 1] + lo[k + 1] - 2 * hi[k]) / 2 - 4 * U * a
        dhi = (hi[k - 1] + hi[k + 1] - 2 * lo[k]) / 2 + 4 * U * a
        q = _div(np.array(-nhi), np.array(-nlo), np.array(2 * dlo + 1e-16), np.array(2 * dhi + 1e-16))
        qlo, qhi = float(q[0]), float(q[1])
        qlo, qhi = qlo - 8 * U * abs(qlo) - 1e-30, qhi + 8 * U * abs(qhi) + 1e-30
        if qlo >= -1 and qhi <= 1:
            olo, ohi = qlo, qhi
        elif qhi < -1 or qlo > 1:
            olo = ohi = 0.0
        else:
            olo, ohi = max(min(qlo, 0.0), -1.0), min(max(qhi, 0.0), 1.0)
    base = p["min_index"] + k
    flo, fhi = p["sr"] / (base + ohi), p["sr"] / (base + olo)
    return flo * (1 - 4 * U), fhi * (1 + 4 * U)


def pitch(x, p, thresh=None):
    """one clip -> per frame dict(cands=[first-trough candidates, None for 'no trough'], lo, hi, flags)"""
    th = p["thresh"] if thresh is None else f32(thresh)
    lo, hi = yin_rows(x, p)
    flags = trough_flags(lo, hi, th)
    out = []
    for t in range(lo.shape[0]):
        f = flags[t]
        cands = []
        for k in np.flatnonzero(f != 0):
            cands.append(int(k))
            if f[k] == 1:
                break
        else:
            cands.append(None)
        out.append(dict(cands=cands, lo=lo[t], hi=hi[t], flags=f))
    return out


def _within(v, lo, hi):
    return lo <= v <= hi or (np.isnan(lo) and np.isnan(hi))


def check(fre, v1, v2, frames, p, fill):
    """(ok, message, undetermined frames): fre / value1 against the first trough's candidates (the fill value where a
    frame may have none), value2 against the bound of the row minimum"""
    alt = []
    if not (len(fre) == len(v1) == len(v2) == len(frames)):
        return False, "lengths", alt
    for t, fr in enumerate(frames):
        lo, hi = fr["lo"], fr["hi"]
        if len(fr["cands"]) > 1:
            alt.append(t)
        ok = False
        for k in fr["cands"]:
            if k is None:
                ok = fre[t] == fill and v1[t] == fill
            else:
                flo, fhi = fre_interval(lo, hi, k, p)
                ok = flo <= fre[t] <= fhi and _within(v1[t], lo[k], hi[k])
            if ok:
                break
        if not ok:
            return False, f"frame {t}: fre {fre[t]} value1 {v1[t]}, candidates {fr['cands']}", alt
        if not lo.min() <= v2[t] <= hi.min():
            return False, f"frame {t}: value2 {v2[t]} outside [{lo.min()}, {hi.min()}]", alt
    return True, "", alt


def check_troughs(mfre, mtrough, lens, frames, p):
    """(ok, message): each row's count within the certain .. possible flags; in rows without an undetermined flag every
    entry at its trough's bounds; entries past the count zero (this library's rows; pass mfre None for the reference)"""
    for t, fr in enumerate(frames):
        f = fr["flags"]
        certain, possible = int((f == 1).sum()), int((f != 0).sum())
        if not certain <= lens[t] <= possible:
            return False, f"frame {t}: {lens[t]} troughs, {certain} .. {possible} possible"
        if possible == certain:
            for i, k in enumerate(np.flatnonzero(f == 1)):
                flo, fhi = fre_interval(fr["lo"], fr["hi"], int(k), p)
                if not (flo <= mfre[t, i] <= fhi and _within(mtrough[t, i], fr["lo"][k], fr["hi"][k])):
                    return False, f"frame {t} trough {i}: {mfre[t, i]}, {mtrough[t, i]}"
    return True, ""


# ---- cases ----

def cases():
    """[(name, dict(ctor=dict(...), length, kind, thresh))]: ctor arguments left out are passed as NULL"""
    out = []

    def add(name, length, kind="tones", thresh=None, **ctor):
        out.append((name, dict(ctor=ctor, length=length, kind=kind, thresh=thresh)))

    add("default", 4096 + 30 * 1024, sr=32000, lf=27.0, hf=2000.0, r2=12, slide=1024, auto=2048)
    add("default_null", 4096 + 20 * 1024)
    for r2 in (8, 9, 10, 11, 13, 14):
        n = 1 << r2
        add(f"r{r2}", n + 12 * (n // 4), sr=8000 if r2 < 10 else 32000, lf=60.0 if r2 < 10 else None, r2=r2)
    for sr in (8000, 16000, 22050, 44100, 48000, 96000):
        add(f"sr{sr}", sr, sr=sr, r2=12, slide=1000)
    add("auto0", 16000, r2=11, auto=0, slide=512)
    add("auto_small", 16000, r2=11, auto=64, slide=512)
    add("auto_near_n", 16000, r2=11, lf=100.0, auto=1900, slide=512)      # maxIndex clamped to n - A - 1
    add("slide_lt_n", 6000, r2=11, slide=7)
    add("slide_eq_n", 40000, r2=11, slide=2048)
    add("slide_gt_n", 60000, r2=11, slide=5000)
    for th in (0.05, 0.3, 0.9, 1.5):
        add(f"thresh{th}", 30000, kind="missing", thresh=th, r2=12, slide=1024)
    for kind in ("silence", "noise", "missing", "glide", "half", "quiet", "loud"):
        add(f"sig_{kind}", 40000, kind=kind, sr=32000, r2=12, slide=1024)
    add("sig_missing_r11", 30000, kind="missing", sr=22050, r2=11, slide=512)
    add("sig_glide_r13", 8192 + 30 * 2048, kind="glide", sr=44100, r2=13, slide=2048)
    add("yin1", 4000, sr=8000, hf=2000.0, r2=10, slide=256, auto=1019)     # minIndex 4 = maxIndex (clamped)
    add("yin2", 4000, sr=8000, hf=2000.0, r2=10, slide=256, auto=1018)     # lags 4 .. 5
    add("yin2_exact", 4000, sr=8000, lf=2700.0, hf=3000.0, r2=10, slide=256, kind="noise")   # lags 2 .. 3
    add("hf_null_fallback", 16000, sr=16000, lf=300.0, r2=11, slide=512)    # highFre 2094
    add("hf_rejected", 16000, sr=16000, lf=300.0, hf=9000.0, r2=11, slide=512)   # 27 .. 2093
    add("lf_low", 16000, sr=16000, lf=20.0, hf=1500.0, r2=11, slide=512)
    add("sr_fallback", 32000, sr=0, r2=12, slide=1024)
    add("radix_fallback", 32000, r2=0, slide=1024)
    add("r1", 5000, sr=4000, r2=1, slide=1, auto=0)                          # n = 2: lag 1 only
    return out


def case_params(kw):
    return params(**kw["ctor"])


def case_signal(name, kw):
    return signal(kw["kind"], kw["length"], case_params(kw)["sr"], sum(map(ord, name)))


def oracle_case(name, kw):
    return pitch(case_signal(name, kw), case_params(kw), kw["thresh"])


# ---- ctypes drivers (either library) ----

def c_troughs(lib, obj, T):
    """copies of getTroughData's arrays for T frames -> (mFre [T, mLen], mTrough [T, mLen], lens [T])"""
    fp, tp, lp = C.POINTER(C.c_float)(), C.POINTER(C.c_float)(), C.POINTER(C.c_int)()
    m = lib.pitchYINObj_getTroughData(obj, C.byref(fp), C.byref(tp), C.byref(lp))
    if T == 0:
        return np.zeros((0, m), f32), np.zeros((0, m), f32), np.zeros(0, np.int32)
    return (np.ctypeslib.as_array(fp, (T, m)).copy(), np.ctypeslib.as_array(tp, (T, m)).copy(),
            np.ctypeslib.as_array(lp, (T,)).copy())


def c_case(lib, name, kw, fill=0.0):
    """-> (fre, value1, value2, mFre, mTrough, lens)"""
    st, obj = c_new(lib, "yin", **kw["ctor"])
    assert st == 0, (name, st)
    if kw["thresh"] is not None:
        lib.pitchYINObj_setThresh(obj, C.c_float(kw["thresh"]))
    x = case_signal(name, kw)
    out = c_pitch(lib, "yin", obj, x, fill)
    tr = c_troughs(lib, obj, len(out[0]))
    c_free(lib, "yin", obj)
    return out + tr
