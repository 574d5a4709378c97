"""Float64 numpy restatements of the reference's cross-correlation and chirp z-transform, the case lists, and ctypes
drivers that work on either library.

Xcorr (src/dsp/xcorr_algorithm.c:49-115, 182-243), n = length, M = util_ceilPowerTwo(2n):
  - vArr3[n-1+m] = sum_k a[k+m] b[k] for m = -(n-1) .. n-1: numpy.correlate(a, b, 'full'); b = NULL is a with itself;
  - Coeff (normType NULL or XcorrNormal_Coeff, :55-109): every value divided by sqrtf(sum1 * sum2), each sum the float of
    a double sum of the float squares (__vsum, src/vector/flux_vector.c:1493-1501), the product in float;
  - the return value and *maxValue: __vmax (flux_vector.c:1536-1557), max = v[0] and then `max < v[i]`: the first index
    of the maximum, a NaN v[0] stays the maximum and later NaNs are passed over.
CZT (src/dsp/czt_algorithm.c:50-257), N = 2^radix2Exp, M = 2N:
  - the float32 tables of _cztObj_dealAW (:114-161) over nArr (:68-74: -(N-1) .. N-1 and a last entry left at 0),
    with the C library's cosf / sinf;
  - g = x * (A^-n W^(n^2/2)) for n < N, zero above; h = conj(W^(nArr^2/2)) with its last entry 0; y = IFFT_M(FFT_M(g)
    FFT_M(h)); the output is y[N-1+k] W^(k^2/2) for k < N, then y[N .. M-1] (:253-255), here in float64 from the
    float32 tables."""
import ctypes as C
import zlib

import numpy as np

f32 = np.float32
MAX_LENGTH = 1 << 19
MAX_EXP = 13
NORMS = {"none": 0, "coeff": 1, "null": None}
BANDS = {"full": (0.0, 1.0), "zoom": (0.15, 0.25), "narrow": (0.01, 0.02), "half": (0.0, 0.5)}

_libm = C.CDLL("libm.so.6")
for _f in (_libm.cosf, _libm.sinf):
    _f.restype, _f.argtypes = C.c_float, [C.c_float]


# ---------------- Xcorr ----------------

def coeff_scale(a, b):
    """sqrtf(sum1 * sum2) of :85-103, float32"""
    s1 = f32(np.sum((a * a).astype(f32), dtype=np.float64))
    s2 = s1 if b is None else f32(np.sum((b * b).astype(f32), dtype=np.float64))
    with np.errstate(invalid="ignore", over="ignore"):
        return np.sqrt(f32(s1 * s2))


def vmax(v):
    """__vmax: (index, value)"""
    if not v[0] == v[0]:
        return 0, v[0]
    w = np.where(np.isnan(v), -np.inf, v)
    i = int(np.argmax(w))
    return i, v[i]


def xcorr(a, b=None, norm=None):
    """-> (lags [2n-1] float64, maxValue, index); norm: 0 None, 1 Coeff, None the C default (Coeff)"""
    a = np.asarray(a, f32)
    bb = a if b is None else np.asarray(b, f32)
    n = a.size
    M = 1 << max(0, int(np.ceil(np.log2(2 * n))))
    A = np.fft.rfft(a.astype(np.float64), M)
    B = A if b is None else np.fft.rfft(bb.astype(np.float64), M)
    r = np.fft.irfft(A * np.conj(B), M)
    out = np.concatenate([r[M - (n - 1):], r[:n]]) if n > 1 else r[:1]
    if norm is None or norm == 1:
        with np.errstate(invalid="ignore", divide="ignore"):
            out = out / np.float64(coeff_scale(a, None if b is None else bb))
    i, v = vmax(out)
    return out, v, i


def c_xcorr(lib, a, b, norm, fill=7.0, extra=0):
    """one xcorrObj_xcorr call on a fresh object of lib -> (vArr3 [2n-1 + extra], maxValue, return value).  A fresh
    object per call: the reference's object carries samples from one call into the next."""
    a = np.ascontiguousarray(a, f32)
    n = a.size
    o = C.c_void_p()
    assert lib.xcorrObj_new(C.byref(o)) == 0
    out = np.full(max(2 * n - 1, 0) + extra, fill, f32)
    mv = C.c_float(fill)
    nt = None if norm is None else C.byref(C.c_int(norm))
    bp = None if b is None else np.ascontiguousarray(b, f32).ctypes.data
    idx = lib.xcorrObj_xcorr(o, a.ctypes.data, bp, n, nt, out.ctypes.data, C.byref(mv))
    lib.xcorrObj_free(o)
    return out, mv.value, idx


def _rng(name):
    return np.random.default_rng(zlib.crc32(name.encode()))


def xcorr_cases():
    """(name, dict(n, auto, norm, sig)) for every length, cross / auto, normType None / Coeff / NULL, and the
    special signals"""
    out = []
    for n in (1, 2, 3, 17, 1000, 4096, 4097, 8192, 8193, (1 << 15) + 3, 1 << 19):
        for auto in (False, True):
            for norm in NORMS:
                out.append((f"x_{'auto' if auto else 'cross'}_{n}_{norm}", dict(n=n, auto=auto, norm=norm, sig="noise")))
    for n in (1, 5, 1000, 8193):
        out.append((f"x_impulse_{n}", dict(n=n, auto=False, norm="coeff", sig="impulse")))
    for norm in NORMS:
        out.append((f"x_silent_{norm}", dict(n=1000, auto=False, norm=norm, sig="silent")))
        out.append((f"x_silent_auto_{norm}", dict(n=700, auto=True, norm=norm, sig="silent")))
    for ratio in ("1e-4", "1e4"):
        for n in (1000, 8192, 40000):
            out.append((f"x_ratio{ratio}_{n}", dict(n=n, auto=False, norm="none", sig="ratio" + ratio)))
    return out


def xcorr_signals(name, kw):
    """(a, b or None) of a case"""
    rng, n = _rng(name), kw["n"]
    a = rng.standard_normal(n).astype(f32)
    b = rng.standard_normal(n).astype(f32) + 0.5 * np.roll(a, n // 7)
    if kw["sig"] == "impulse":
        b = a
        a = np.zeros(n, f32)
        a[(3 * n) // 5] = 1.0
    elif kw["sig"] == "silent":
        b = rng.standard_normal(n).astype(f32)
        a = np.zeros(n, f32)
    elif kw["sig"].startswith("ratio"):
        b = (b * float(kw["sig"][5:])).astype(f32)
    return a, None if kw["auto"] else b.astype(f32)


def xcorr_case(name, kw):
    a, b = xcorr_signals(name, kw)
    return xcorr(a, b, NORMS[kw["norm"]])


def c_xcorr_case(lib, name, kw):
    a, b = xcorr_signals(name, kw)
    return c_xcorr(lib, a, b, NORMS[kw["norm"]])


# ---------------- CZT ----------------

_TABLES = {}


def czt_tables(r, low_w, high_w):
    """(pre [N], post [N], h [M]) complex128 holding the reference's float32 values"""
    key = (r, f32(low_w), f32(high_w))
    if key in _TABLES:
        return _TABLES[key]
    N = 1 << r
    M = 2 * N
    low_w, high_w = f32(low_w), f32(high_w)
    tA = f32(2 * np.pi * np.float64(low_w))
    tW = f32(-2 * np.pi * np.float64(f32(high_w - low_w)) / N)
    n = np.zeros(M, f32)
    n[:M - 1] = np.arange(M - 1) - (N - 1)
    n1, n2 = -n, (n * n) / f32(2)
    arg_a, arg_w = (n1 * tA).astype(f32), (n2 * tW).astype(f32)
    aR = np.array([_libm.cosf(float(v)) for v in arg_a], f32)
    aI = np.array([_libm.sinf(float(v)) for v in arg_a], f32)
    wR = np.array([_libm.cosf(float(v)) for v in arg_w], f32)
    wI = np.array([_libm.sinf(float(v)) for v in arg_w], f32)
    s = slice(N - 1, M - 1)
    pre = (aR[s] * wR[s] - aI[s] * wI[s]).astype(f32) + 1j * (aI[s] * wR[s] + aR[s] * wI[s]).astype(f32)
    post = wR[s].astype(np.float64) + 1j * wI[s]
    h = wR.astype(np.float64) - 1j * wI
    h[M - 1] = 0
    _TABLES[key] = (pre, post, h)
    return _TABLES[key]


def czt(x, r, low_w, high_w):
    """x [N] real or complex -> complex128 [2N]: the head, then the tail"""
    N = 1 << r
    pre, post, h = czt_tables(r, low_w, high_w)
    g = np.asarray(x, np.complex128)[:N] * pre
    y = np.fft.ifft(np.fft.fft(g, 2 * N) * np.fft.fft(h))
    return np.concatenate([y[N - 1:2 * N - 1] * post, y[N:]])


def czt_cases():
    """(name, dict(r, band, inp)): every radix2Exp 0 .. 13 with the bands and inputs in turn, and every band and input
    at 3 and 10"""
    out, inps, bands = [], ("re", "im", "cplx"), list(BANDS)
    for r in range(MAX_EXP + 1):
        for j in range(2):
            band, inp = bands[(r + 2 * j) % 4], inps[(r + j) % 3]
            out.append((f"c_{r}_{band}_{inp}", dict(r=r, band=band, inp=inp)))
    for r in (3, 10):
        for band in bands:
            for inp in inps:
                name = f"c_{r}_{band}_{inp}"
                if name not in dict(out):
                    out.append((name, dict(r=r, band=band, inp=inp)))
    return out


def czt_input(name, kw):
    """(re or None, im or None) of a case, N samples each"""
    rng, N = _rng(name), 1 << kw["r"]
    t = np.arange(N)
    x = np.cos(2 * np.pi * 0.2 * t + 0.3) + 0.5 * rng.standard_normal(N)
    y = np.sin(2 * np.pi * 0.17 * t) + 0.5 * rng.standard_normal(N)
    re, im = x.astype(f32), y.astype(f32)
    return (re, None) if kw["inp"] == "re" else (None, im) if kw["inp"] == "im" else (re, im)


def czt_case(name, kw):
    re, im = czt_input(name, kw)
    x = (0 if re is None else re.astype(np.float64)) + (0 if im is None else 1j * im.astype(np.float64))
    return czt(x, kw["r"], *BANDS[kw["band"]])


def c_czt(lib, o, re, im, low_w, high_w, N, fill=7.0):
    """cztObj_czt -> complex128 [2N].  The inputs are passed zero-padded to 2N: the reference reads 2N samples"""
    def pad(v):
        return None if v is None else np.concatenate([np.asarray(v, f32), np.zeros(N, f32)])
    rp, ip = pad(re), pad(im)
    o3 = [np.full(2 * N, fill, f32) for _ in range(2)]
    lib.cztObj_czt(o, None if rp is None else rp.ctypes.data, None if ip is None else ip.ctypes.data, low_w, high_w,
                   o3[0].ctypes.data, o3[1].ctypes.data)
    return o3[0].astype(np.float64) + 1j * o3[1]


def c_czt_new(lib, r):
    o = C.c_void_p()
    st = lib.cztObj_new(C.byref(o), r)
    return st, o


def c_czt_case(lib, name, kw):
    st, o = c_czt_new(lib, kw["r"])
    assert st == 0
    re, im = czt_input(name, kw)
    out = c_czt(lib, o, re, im, *BANDS[kw["band"]], 1 << kw["r"])
    lib.cztObj_free(o)
    return out


# one object through a valid, an invalid and a valid band: the invalid call keeps the first band's tables
SEQUENCE = ((0.15, 0.25), (0.3, 0.2), (0.01, 0.02))


def czt_sequence_oracle(r, x):
    bands = [SEQUENCE[0], SEQUENCE[0], SEQUENCE[2]]
    return [czt(x, r, *b) for b in bands]


def c_czt_sequence(lib, r, x):
    st, o = c_czt_new(lib, r)
    assert st == 0
    out = [c_czt(lib, o, x, None, *b, 1 << r) for b in SEQUENCE]
    lib.cztObj_free(o)
    return out
