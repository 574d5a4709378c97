"""numpy restatement of the spectral descriptors (src/flux_spectral.c, src/feature/spectral_algorithm.c), the yardstick
of tests/test_spectral_*.py.  Computed fresh on every call: one clip x [T, num] time-major, a bin list `idx` (the
contiguous range of setEdge or the list of setEdgeArr) and the float32 band frequencies `fre`.  Sums are float64 except
where the outcome is an integer decided by float32 comparisons: rolloff's two sums run float32 in list order."""
import numpy as np

f32 = np.float32
PHASE = ("pd", "wpd", "nwpd", "cd", "rcd")


def _rows(x, idx):
    return np.asarray(x, np.float64)[:, idx]


def _sum(x, idx):
    return _rows(x, idx).sum(1)


def flatness(x, idx, fre=None):                                   # flux_spectral.c:21-55
    r = np.asarray(x, f32)[:, idx]
    lg = np.log((r.astype(np.float64) + 2e-16).astype(f32)).astype(np.float64).sum(1) / len(idx)
    g = np.exp(lg)
    m = _sum(x, idx) / len(idx)
    with np.errstate(all="ignore"):
        return np.where(m != 0, g / np.where(m != 0, m, 1), 0.0)


def _pos(v):
    """the reference's `v > 0 ? v : 0`: a NaN difference (NaN or inf - inf) counts as 0"""
    with np.errstate(invalid="ignore"):
        return np.where(v > 0, v, 0.0)


def _temporal(x, idx, step, fn):
    T = x.shape[0]
    out = np.zeros(T)
    step = max(int(step), 1)
    r = _rows(x, idx)
    for t in range(step, T):
        out[t] = fn(r[t], r[t - step])
    return out


def flux(x, idx, fre=None, step=1, p=2, is_positive=False, is_exp=False, tp=0):     # :58-105
    def f(c, q):
        v = c - q
        v = _pos(v) if is_positive else np.abs(v)
        with np.errstate(all="ignore"):
            s = (v * v if p == 2 else np.power(v, p)).sum()
        if tp:
            s /= len(idx)
        return s ** (1.0 / p) if is_exp else s
    return _temporal(x, idx, step, f)


def rolloff(x, idx, fre, threshold=0.95):                          # :107-146, float32 in list order
    x = np.asarray(x, f32)
    out = np.zeros(x.shape[0])
    index = 0
    for t in range(x.shape[0]):
        row = x[t, idx]
        s = np.add.accumulate(row, dtype=f32)[-1]                  # accumulate is sequential (np.sum is pairwise)
        m1 = f32(s * f32(threshold))
        with np.errstate(all="ignore"):
            hit = np.flatnonzero(np.add.accumulate(np.abs(row), dtype=f32) >= m1)
        if hit.size:
            index = idx[hit[0]]
        out[t] = fre[index]
    return out


def centroid(x, idx, fre):                                         # :148-173
    s = _sum(x, idx)
    n = (_rows(x, idx) * np.asarray(fre, np.float64)[idx]).sum(1)
    with np.errstate(all="ignore"):
        return np.where(s != 0, n / np.where(s != 0, s, 1), 0.0)


def _moment(x, idx, fre, k):
    c = centroid(x, idx, fre)
    d = np.asarray(fre, np.float64)[idx][None, :] - c[:, None]
    return (d ** k * _rows(x, idx)).sum(1), _sum(x, idx)


def spread(x, idx, fre):                                           # :175-202
    n, s = _moment(x, idx, fre, 2)
    with np.errstate(all="ignore"):
        return np.where(s != 0, np.sqrt(n / np.where(s != 0, s, 1)), 0.0)


def skewness(x, idx, fre, k=3):                                    # :204-260
    n, s = _moment(x, idx, fre, k)
    m = spread(x, idx, fre) ** k * s
    with np.errstate(all="ignore"):
        return np.where(m != 0, n / np.where(m != 0, m, 1), 0.0)


def kurtosis(x, idx, fre):
    return skewness(x, idx, fre, 4)


def entropy(x, idx, fre=None, is_norm=False):                      # :262-293; a zero-sum frame is NaN
    s = _sum(x, idx)
    with np.errstate(all="ignore"):
        v = _rows(x, idx) / s[:, None]
        n = (v * np.log2(v + 1e-16)).sum(1)
    if is_norm:
        m = np.log2(len(idx))
        return -n / m if m else np.zeros_like(n)
    return -n


def crest(x, idx, fre=None):                                       # :295-321
    m = _sum(x, idx) / len(idx)
    mx = max_(x, idx, np.zeros(x.shape[1]))[0]
    with np.errstate(all="ignore"):
        return np.where(m != 0, mx / np.where(m != 0, m, 1), 0.0)


def _mean_fre(idx, fre):                                           # spectral_algorithm.c:1124-1130, float32 in order
    s = f32(0)
    for k in idx:
        s = f32(s + f32(fre[k]))
    return float(f32(s / f32(len(idx))))


def slope(x, idx, fre):                                            # flux_spectral.c:323-350
    d = np.asarray(fre, np.float64)[idx] - _mean_fre(idx, fre)
    mv = _sum(x, idx) / len(idx)
    n = (d[None, :] * (_rows(x, idx) - mv[:, None])).sum(1)
    m = (d * d).sum()
    return n / m if m else np.zeros(x.shape[0])


def decrease(x, idx, fre=None):                                    # :352-376, divides by the absolute bin index
    r = _rows(x, idx)
    m = r.sum(1) - r[:, 0]
    with np.errstate(all="ignore"):
        n = ((r[:, 1:] - r[:, :1]) / np.asarray(idx[1:], np.float64)[None, :]).sum(1)
        return np.where(m != 0, n / np.where(m != 0, m, 1), 0.0)


def band_width(x, idx, fre, p=2):                                  # :378-407
    c = centroid(x, idx, fre)
    d = np.asarray(fre, np.float64)[idx][None, :] - c[:, None]
    with np.errstate(all="ignore"):
        d = d * d if p == 2 else np.power(d, p)
        v = (_rows(x, idx) * d).sum(1)
        return v if p == 1 else np.power(v, 1.0 / p)


def rms(x, idx, fre=None):                                         # :409-435, normalised by num
    num = x.shape[1]
    w = np.ones(len(idx))
    ia = np.asarray(idx)
    w[(ia == 0) | ((num % 2 == 0) & (ia == num - 1))] = 0.5
    nn = float(np.array(num * num, np.int64).astype(np.int32))    # the reference's int product, wrapped
    return np.sqrt(2 * (_rows(x, idx) ** 2 * w).sum(1) / nn)


def energy(x, idx, fre=None, is_log=False, gamma=10.):             # :794-823 with isPower = 0
    v = _rows(x, idx) ** 2
    if is_log:
        g = 10. if gamma <= 0 else gamma
        v = np.log(1 + g * v)
    return v.sum(1) / len(idx)


def hfc(x, idx, fre=None):                                         # :439-458, absolute bin index
    return (_rows(x, idx) * np.asarray(idx, np.float64)[None, :]).sum(1)


def sd(x, idx, fre=None, step=1, is_positive=False):               # :461-492
    return _temporal(x, idx, step, lambda c, q: (_pos(c - q) if is_positive else np.abs(c - q)).sum())


def sf(x, idx, fre=None, step=1, is_positive=False):               # :495-526
    return _temporal(x, idx, step, lambda c, q: ((_pos(c - q) if is_positive else np.abs(c - q)) ** 2).sum())


def mkl(x, idx, fre=None, tp=0):                                   # :529-555
    def f(c, q):
        s = np.log(1 + c / (q + 1e-16)).sum()
        return s / len(idx) if tp else s
    return _temporal(x, idx, 1, f)


def _pd(x, ph, idx, weight, norm):                                 # :557-599; frame 1 is left as it was (0 here)
    r, P = _rows(x, idx), _rows(ph, idx)
    out = np.zeros(x.shape[0])
    for t in range(2, x.shape[0]):
        v = np.abs(P[t] - 2 * P[t - 1] + P[t - 2])
        if weight or norm:
            v = v * r[t]
        s = v.sum() / len(idx)
        if norm:
            s = s / (r[t].sum() / len(idx) + 1e-16)
        out[t] = s
    return out


def pd(x, ph, idx):
    return _pd(x, ph, idx, 0, 0)


def wpd(x, ph, idx):
    return _pd(x, ph, idx, 1, 0)


def nwpd(x, ph, idx):
    return _pd(x, ph, idx, 0, 1)


def _cd(x, ph, idx, rectify):                                      # :631-680
    r, P = _rows(x, idx), _rows(ph, idx)
    out = np.zeros(x.shape[0])
    for t in range(1, x.shape[0]):
        re, im = r[t] * np.cos(P[t]), r[t] * np.sin(P[t])
        if t > 1:
            v2 = 2 * P[t - 1] - P[t - 2]
            re, im = re - r[t - 1] * np.cos(v2), im - r[t - 1] * np.sin(v2)
        v = np.sqrt(re * re + im * im)
        if rectify:
            v = np.where(r[t] <= r[t - 1], 0, v)
        out[t] = v.sum()
    return out


def cd(x, ph, idx):
    return _cd(x, ph, idx, 0)


def rcd(x, ph, idx):
    return _cd(x, ph, idx, 1)


def broadband(x, idx, fre=None, threshold=0):                      # :703-720, float32 log10 as log10f
    r = np.asarray(x, f32)[:, idx]
    out = np.zeros(x.shape[0])
    with np.errstate(all="ignore"):
        for t in range(1, x.shape[0]):
            d = (10.0 * np.log10((r[t] / r[t - 1]).astype(f32)).astype(np.float64)).astype(f32)
            out[t] = float((d > f32(threshold)).sum())
    return out


def novelty(x, idx, fre=None, step=1, threshold=0., method_type=0, data_type=0):   # :728-792
    mt, dt = int(getattr(method_type, "value", method_type)), int(getattr(data_type, "value", data_type))

    def f(c, q):      # float32 where the reference is float: logf of the double quotient, cur * logf, the IS difference
        with np.errstate(all="ignore"):
            c32, q32 = c.astype(f32), q.astype(f32)
            if mt == 0:
                v = (c32 - q32).astype(np.float64)
            else:
                qq = c / (q + 1e-16)
                lq = np.log(qq.astype(f32))
                v = lq if mt == 1 else c32 * lq if mt == 2 else (qq - lq.astype(np.float64) - 1).astype(f32)
                v = v.astype(np.float64)
            hit = v > f32(threshold)
            return float(hit.sum()) if dt else float(v[hit].sum())
    return _temporal(x, idx, step, f)


def eef(x, idx, fre=None, is_norm=False):                          # spectral_algorithm.c:781-815
    return np.sqrt(1 + np.abs(energy(x, idx) * entropy(x, idx, is_norm=is_norm)))


def eer(x, idx, fre=None, is_norm=False, gamma=1.):                # :818-852
    with np.errstate(all="ignore"):
        return np.sqrt(1 + np.abs(np.log(1 + energy(x, idx) * gamma) / entropy(x, idx, is_norm=is_norm)))


def max_(x, idx, fre):                                             # :855-891, ties -> first list position
    r = np.asarray(x, f32)[:, idx]
    val = np.zeros(x.shape[0])
    fr = np.zeros(x.shape[0])
    for t in range(x.shape[0]):
        row = r[t]
        j = 0
        if not np.isnan(row[0]):
            ok = ~np.isnan(row)
            m = row[ok].max()
            j = int(np.flatnonzero(ok & (row == m))[0])
        val[t], fr[t] = row[j], fre[idx[j]]
    return val, fr


def mean(x, idx, fre):                                             # :893-901, 1102-1147
    return _sum(x, idx) / len(idx), np.full(x.shape[0], _mean_fre(idx, fre))


def var(x, idx, fre):                                              # :903-956
    mv = _sum(x, idx) / len(idx)
    v1 = ((mv[:, None] - _rows(x, idx)) ** 2).sum(1) / (len(idx) - 1)
    d = _mean_fre(idx, fre) - np.asarray(fre, np.float64)[idx]
    return v1, np.full(x.shape[0], (d * d).sum() / (len(idx) - 1))


def compute(name, x, idx, fre, phase=None, **kw):
    """one feature by the Spectral method name"""
    idx = list(idx)
    if name in ("pd", "wpd", "nwpd", "cd", "rcd"):
        return globals()[name](x, phase, idx)
    if name == "max":
        return max_(x, idx, fre)
    return globals()[name](x, idx, fre, **kw)
