"""Float64 numpy restatement of the reference's Stockwell transforms, and ctypes wrappers that drive either library.

ST  (src/st_algorithm.c): X = FFT_N(x), used periodically (:184-186).  Row of bin i != 0: IFFT_N(X[(m + i) mod N] G_i[m])
    (:189-198) with G_i[m] = exp(v m^2) + exp(v (m - N)^2) (:225-244).  v = -factor 2 pi^2 / powf(i, 2 norm) is
    evaluated in double and stored as a float, and m^2 is a float product (:227-230); both are rounded here the same
    way.  Bin 0: the clip's mean in the real row (:199-206).
FST (src/fst_algorithm.c): the FFT of ifftshift(x), fftshifted and times 1/sqrt(N) (:173-193), cut into the partition
    lengths 1, N/4 .. 2, 1, 1, 1, 2 .. N/4 (:293-317); every segment of two or more points becomes
    fftshift(ifft(ifftshift(seg))) sqrt(len) (:196-262).  Row k (frequency f = minIndex + k) is the segment that holds
    partition position N/2 - 1 + f, column l its element l len / N (the index table of :319-362, read at :265-275).
Range rules: stObj_new (:90-93), fstObj_fst (:160-171)."""
import ctypes as C

import numpy as np


def case_signal(seed, n):
    """tones at a few bins plus noise: rows of very different magnitude"""
    t = np.arange(n)
    rng = np.random.default_rng(seed)
    x = sum(a * np.cos(2 * np.pi * k * t / n + p) for a, k, p in ((0.5, max(1, n // 37), 0.3), (0.3, max(1, n // 5), 1.1),
                                                                     (0.2, max(1, n // 3 + 1), 2.0)))
    return (x + 0.05 * rng.standard_normal(n) + 0.02).astype(np.float32)


def st_range(radix2_exp, min_index, max_index):
    n = 1 << radix2_exp
    if min_index >= max_index or min_index < 0 or max_index > n // 2:
        return 0, n // 2
    return min_index, max_index


def fst_range(radix2_exp, min_index, max_index):
    n = 1 << radix2_exp
    min_index = max(min_index, 0)
    max_index = min(max_index, n // 2)
    if min_index > max_index:
        return 0, n // 2
    return min_index, max_index


def st_v(i, factor=1.0, norm=1.0):
    """the float the reference stores: double arithmetic on the float factor and powf(i, 2 norm)"""
    f32 = np.float32
    p = float(np.power(f32(i), f32(2) * f32(norm), dtype=f32))
    return f32(float(f32(-f32(factor) * f32(2))) * np.pi * np.pi / p)


def st(x, bins, factor=1.0, norm=1.0):
    """complex [len(bins), N]"""
    n = x.size
    X = np.fft.fft(x.astype(np.float64))
    m = np.arange(n)
    m1 = (m.astype(np.float32) * m.astype(np.float32)).astype(np.float64)
    m2 = ((m - n).astype(np.float32) * (m - n).astype(np.float32)).astype(np.float64)
    out = np.empty((len(bins), n), np.complex128)
    for r, i in enumerate(bins):
        if i == 0:
            out[r] = x.astype(np.float64).mean()
            continue
        v = float(st_v(i, factor, norm))
        g = np.exp(v * m1) + np.exp(v * m2)
        out[r] = np.fft.ifft(X[(m + i) % n] * g)
    return out


def fst_lengths(radix2_exp):
    length = 2 * radix2_exp
    lens = [0] * length
    lens[0] = lens[length // 2 - 1] = lens[length // 2] = 1
    for i in range(1, length // 2 - 1):
        lens[i] = 2 ** (length // 2 - 1 - i)
    for j, i in enumerate(range(length // 2 + 1, length)):
        lens[i] = 2 ** j
    return lens


def fst_partition(x):
    """complex [N]: the whole partition, every segment transformed"""
    n = x.size
    r = n.bit_length() - 1
    X = np.fft.fft(np.fft.ifftshift(x.astype(np.float64)))
    P = np.fft.fftshift(X) / np.sqrt(n)
    part = P.copy()
    start = 0
    for ln in fst_lengths(r):
        if ln > 1:
            seg = P[start:start + ln]
            part[start:start + ln] = np.fft.fftshift(np.fft.ifft(np.fft.ifftshift(seg))) * np.sqrt(ln)
        start += ln
    return part


def fst_segment_of(radix2_exp, f):
    """(first partition position, length) of the segment that row f reads"""
    q = (1 << radix2_exp) // 2 - 1 + f
    start = 0
    for ln in fst_lengths(radix2_exp):
        if start <= q < start + ln:
            return start, ln
        start += ln
    raise ValueError(f)


def fst(x, min_index, max_index):
    """complex [rows, N] after the range rules"""
    n = x.size
    r = n.bit_length() - 1
    lo, hi = fst_range(r, min_index, max_index)
    part = fst_partition(x)
    out = np.empty((hi - lo + 1, n), np.complex128)
    for k, f in enumerate(range(lo, hi + 1)):
        start, ln = fst_segment_of(r, f)
        out[k] = part[start + np.arange(n) * ln // n]
    return out


# ---- ctypes drivers (either library) ----

def c_st_new(lib, radix2_exp, min_index, max_index, factor=None, norm=None):
    obj = C.c_void_p()
    f = None if factor is None else C.byref(C.c_float(factor))
    nm = None if norm is None else C.byref(C.c_float(norm))
    st_ = lib.stObj_new(C.byref(obj), radix2_exp, min_index, max_index, f, nm)
    return st_, obj


def c_st(lib, obj, x, rows):
    """(re, im) [rows, N]; the planes start as zeros, as the reference's Python passes them"""
    n = x.size
    re = np.zeros((rows, n), np.float32)
    im = np.zeros((rows, n), np.float32)
    x = np.ascontiguousarray(x, np.float32)
    lib.stObj_st(obj, x.ctypes.data, re.ctypes.data, im.ctypes.data)
    return re, im


def c_use_bins(lib, obj, bins):
    b = np.ascontiguousarray(bins, np.int32)
    lib.stObj_useBinArr(obj, b.ctypes.data, len(b))


def c_fst_new(lib, radix2_exp):
    obj = C.c_void_p()
    return lib.fstObj_new(C.byref(obj), radix2_exp), obj


def c_fst(lib, obj, x, min_index, max_index):
    n = x.size
    lo, hi = fst_range(n.bit_length() - 1, min_index, max_index)
    re = np.zeros((hi - lo + 1, n), np.float32)
    im = np.zeros((hi - lo + 1, n), np.float32)
    x = np.ascontiguousarray(x, np.float32)
    lib.fstObj_fst(obj, x.ctypes.data, min_index, max_index, re.ctypes.data, im.ctypes.data)
    return re, im


# ---- the case sets shared by the CPU and GPU tests ----

def st_cases():
    """name -> dict(radix2_exp, min_index, max_index, factor, norm, bins (useBinArr list or None), set_value)"""
    out = []
    for r in range(3, 13):                                        # default full band (0 .. N/2 through the fallback)
        out.append((f"st{r}_full", dict(radix2_exp=r, min_index=0, max_index=0)))
    out += [
        ("st9_band", dict(radix2_exp=9, min_index=5, max_index=60, factor=0.5, norm=0.8)),
        ("st10_nyq", dict(radix2_exp=10, min_index=500, max_index=512, factor=2.0, norm=1.2)),
        ("st8_bin0", dict(radix2_exp=8, min_index=0, max_index=9)),
        ("st8_neg", dict(radix2_exp=8, min_index=-3, max_index=40)),           # min < 0: full band
        ("st8_over", dict(radix2_exp=8, min_index=3, max_index=129)),          # max > N/2: full band
        ("st8_nullfac", dict(radix2_exp=8, min_index=1, max_index=127, factor=-1.0, norm=0.0)),
        ("st9_nyq", dict(radix2_exp=9, min_index=250, max_index=256)),
        ("st11_bins", dict(radix2_exp=11, min_index=1, max_index=20, bins=[700, 3, 0, 1024, 3, 17, 512, 3])),
        ("st9_bins", dict(radix2_exp=9, min_index=1, max_index=20, bins=[200, 3, 0, 256, 3, 17, 128, 3])),
        ("st9_badbins", dict(radix2_exp=9, min_index=10, max_index=20, bins=[4, 300, 5])),   # ignored: 300 > N/2
        ("st8_negbins", dict(radix2_exp=8, min_index=10, max_index=20, bins=[4, -1])),      # ignored
        ("st10_setvalue", dict(radix2_exp=10, min_index=1, max_index=300, set_value=(1.7, 0.9))),
        ("st12_factor", dict(radix2_exp=12, min_index=1, max_index=2047, factor=0.3, norm=1.0)),
        ("st13_narrow", dict(radix2_exp=13, min_index=100, max_index=130)),
        ("st14_narrow", dict(radix2_exp=14, min_index=3000, max_index=3012, factor=1.5, norm=1.1)),
        ("st14_nyq", dict(radix2_exp=14, min_index=8189, max_index=8192)),
    ]
    return out


def fst_cases():
    """name -> dict(radix2_exp, min_index, max_index)"""
    out = [(f"fst{r}_full", dict(radix2_exp=r, min_index=0, max_index=1 << (r - 1))) for r in range(3, 13)]
    out += [
        ("fst6_band", dict(radix2_exp=6, min_index=1, max_index=31)),
        ("fst11_narrow", dict(radix2_exp=11, min_index=200, max_index=300)),
        ("fst9_clamp", dict(radix2_exp=9, min_index=-5, max_index=1000)),     # -> 0 .. 256
        ("fst9_swap", dict(radix2_exp=9, min_index=40, max_index=10)),        # min > max: full band
        ("fst10_one", dict(radix2_exp=10, min_index=7, max_index=7)),
        ("fst13_narrow", dict(radix2_exp=13, min_index=1000, max_index=1040)),
        ("fst14_narrow", dict(radix2_exp=14, min_index=8150, max_index=8192)),
    ]
    return out


def st_rows(kw):
    """the bin list a case ends with"""
    lo, hi = st_range(kw["radix2_exp"], kw["min_index"], kw["max_index"])
    bins = list(range(lo, hi + 1))
    b = kw.get("bins")
    n = 1 << kw["radix2_exp"]
    if b is not None and all(0 <= v <= n // 2 for v in b):
        bins = list(b)
    return bins


def st_params(kw):
    """(factor, norm) in effect when the transform runs"""
    if kw.get("set_value"):
        return kw["set_value"]
    f, nm = kw.get("factor"), kw.get("norm")
    return (f if f is not None and f > 0 else 1.0), (nm if nm is not None and nm > 0 else 1.0)


def c_st_case(lib, kw, x):
    """run a case through a library: (re, im)"""
    s, obj = c_st_new(lib, kw["radix2_exp"], kw["min_index"], kw["max_index"], kw.get("factor"), kw.get("norm"))
    assert s == 0
    if kw.get("bins") is not None:
        c_use_bins(lib, obj, kw["bins"])
    if kw.get("set_value"):
        lib.stObj_setValue(obj, *kw["set_value"])
    out = c_st(lib, obj, x, len(st_rows(kw)))
    lib.stObj_free(obj)
    return out


def c_fst_case(lib, kw, x):
    s, obj = c_fst_new(lib, kw["radix2_exp"])
    assert s == 0
    out = c_fst(lib, obj, x, kw["min_index"], kw["max_index"])
    lib.fstObj_free(obj)
    return out


def oracle_st_case(kw, x):
    f, nm = st_params(kw)
    return st(x, st_rows(kw), f, nm)


def row_errors(got_re, got_im, want):
    """per row: max |got - want| / max |want| of that row (rows whose want is exactly 0: the absolute max)"""
    g = got_re.astype(np.float64) + 1j * got_im.astype(np.float64)
    d = np.abs(g - want).max(axis=1)
    s = np.abs(want).max(axis=1)
    return np.where(s > 0, d / np.where(s > 0, s, 1), d), s
