"""Float64 restatement of DWTObj, WPTObj and SWTObj (src/dwt_algorithm.c, src/wpt_algorithm.c, src/swt_algorithm.c),
literal where the reference is: its periodic padding with both branches, valid / full convolution, odd-sample
decimation, the coefArr layout, the reassign indices for every num, WPT's node order and swap, SWT's dilation and
offset.  Filters are passed in (the float32 values of the C table), so the oracle judges the transform alone."""
import ctypes as C
import math

import numpy as np


def period_padding(x, filter_length):
    """__periodPadding (dwt_algorithm.c:308-351): x of length1 -> length1 + filter_length samples"""
    length1 = len(x)
    total = length1 + filter_length
    half = filter_length // 2
    if length1 >= half:
        return np.concatenate([x[length1 - half:], x, x[:half]])
    first = int(math.fmod(length1 - half + 1, length1))     # C's %: the sign of the dividend
    if first < 0:
        first = length1 + first
    first = length1 - 1 if first == 0 else first - 1
    n = int(math.floor((total - (length1 - first)) * 1.0 / length1))
    last = total - (length1 - first) - n * length1 - 1
    return np.concatenate([x[first:]] + [x] * n + [x[:last + 1]])


def modulo_padding(x, filter_length):
    """what the kernels read instead: padded[m] = x[(m - filter_length/2) mod length]"""
    m = np.arange(len(x) + filter_length)
    return x[(m - filter_length // 2) % len(x)]


def _split(x, lo, hi):
    """one DWT / WPT step: pad, valid convolution, odd samples"""
    p = period_padding(x, len(lo))
    a = np.convolve(p, lo, mode="valid")[1::2][:len(x) // 2]
    d = np.convolve(p, hi, mode="valid")[1::2][:len(x) // 2]
    return a, d


def dwt(x, num, lo, hi, m_data=True):
    n = len(x)
    coef = np.zeros(n)
    ca, c_len = np.asarray(x, np.float64), 0
    for _ in range(num):
        ca, cd = _split(ca, lo, hi)
        c_len += len(ca)
        coef[n - c_len:n - c_len + len(cd)] = cd
    coef[:len(ca)] = ca
    if not m_data:
        return coef, None
    m = np.zeros((num, n))
    for i in range(num, 0, -1):                       # :291-303
        start, end = 1 << i, (1 << (i + 1)) - 1
        k_len = n // (end - start + 1)
        for k in range(k_len):
            for l, j in enumerate(range(k, n, k_len)):
                m[i - 1, j] = coef[start + l]
    return coef, m


def _node(index, n):
    """__getNodeOffset (wpt_algorithm.c:357-382): (offset, length) in the (num+1) x n node array"""
    if index == 0:
        return 0, n
    base = int(math.floor(math.log2(index + 1)))
    j = index + 1 - (1 << base)
    length = n // (1 << base)
    return base * n + j * length, length


def wpt(x, num, lo, hi, m_data=True):
    n = len(x)
    nodes = np.zeros((num + 1) * n)
    nodes[:n] = x
    node_index = 1
    for i in range((1 << num) - 1):
        off, length = _node(i, n)
        a, d = _split(nodes[off:off + length], lo, hi)
        first, second = (d, a) if i and i % 2 == 0 else (a, d)
        o1, l1 = _node(node_index, n)
        nodes[o1:o1 + l1] = first
        o2, l2 = _node(node_index + 1, n)
        nodes[o2:o2 + l2] = second
        node_index += 2
    coef = nodes[num * n:(num + 1) * n].copy()
    if not m_data:
        return coef, None
    down = n >> num
    m = np.zeros((1 << num, n))
    for i in range(1 << num):
        k_len = n // down
        for k in range(k_len):
            for l, j in enumerate(range(k, n, k_len)):
                m[i, j] = coef[i * down + l]
    return coef, m


def m_data_index(n, num, kind):
    """the index map of mDataArr: row r of DWT is coef[2^(r+1) + (j >> (log2n - r - 1))], row i of WPT is
    coef[i (n >> num) + (j >> num)] -> int32 [rows, n], the literal loops of dwt / wpt above as one gather"""
    log2n = n.bit_length() - 1
    j = np.arange(n, dtype=np.int32)
    if kind == "dwt":
        r = np.arange(num, dtype=np.int32)[:, None]
        return (2 << r) + (j >> (log2n - r - 1))
    i = np.arange(1 << num, dtype=np.int32)[:, None]
    return i * (n >> num) + (j >> num)


# ---- the kernels' steps, vectorised: each output is a gather of dec shifted index arrays over the unpadded input ----

def level(x, lo, hi):
    """one DWT / WPT step on the last axis of x (length L, any leading axes), with the modulo indexing:
    a[i] = sum_j lo[j] x[(2i + dec - dec/2 - j) mod L], d[i] likewise with hi.  -> float64 [4, ..., L/2]: a, d and
    their scales sum_j |lo[j]| |x[...]|, sum_j |hi[j]| |x[...]|"""
    x = np.asarray(x, np.float64)
    L, dec = x.shape[-1], len(lo)
    base = 2 * np.arange(L // 2) + dec - dec // 2
    out = np.zeros((4,) + x.shape[:-1] + (L // 2,))
    for j in range(dec):
        v = x[..., (base - j) % L]
        out[0] += float(lo[j]) * v
        out[1] += float(hi[j]) * v
        v = np.abs(v)
        out[2] += abs(float(lo[j])) * v
        out[3] += abs(float(hi[j])) * v
    return out


def wpt_level(nodes, k, lo, hi):
    """level k of WPT on the last axis of nodes (2^k nodes of L samples, as coefArr of a num = k run) -> float64
    [2, ..., 2^k L]: the next level's nodes and their scales.  Node p is node g = 2^k - 1 + p of the tree; its children
    2g + 1, 2g + 2 sit at p L and p L + L/2, with the detail first where g is even and non-zero"""
    nodes = np.asarray(nodes, np.float64)
    x = nodes.reshape(nodes.shape[:-1] + (1 << k, nodes.shape[-1] >> k))
    a, d, sa, sd = level(x, lo, hi)
    g = (1 << k) - 1 + np.arange(1 << k)
    swap = ((g > 0) & (g % 2 == 0))[:, None]
    out = [np.concatenate([np.where(swap, q, p), np.where(swap, p, q)], axis=-1) for p, q in ((a, d), (sa, sd))]
    return np.stack(out).reshape((2,) + nodes.shape)


def swt_level(x, s, lo, hi):
    """one SWT level at dilation s on the last axis of x (length n), with the modulo indexing:
    lo_out[t] = sum_j lo[j] x[(t + dec s / 2 - j s) mod n].  -> float64 [4, ..., n] as level()"""
    x = np.asarray(x, np.float64)
    n, dec = x.shape[-1], len(lo)
    t = np.arange(n) + dec * s // 2
    out = np.zeros((4,) + x.shape)
    for j in range(dec):
        v = x[..., (t - j * s) % n]
        out[0] += float(lo[j]) * v
        out[1] += float(hi[j]) * v
        v = np.abs(v)
        out[2] += abs(float(lo[j])) * v
        out[3] += abs(float(hi[j])) * v
    return out


def dwt_fast(x, num, lo, hi):
    """coefArr of dwt() through level(), for any leading axes"""
    x = np.asarray(x, np.float64)
    n = x.shape[-1]
    coef = np.zeros(x.shape)
    for k in range(num):
        x, d = level(x, lo, hi)[:2]
        coef[..., n >> (k + 1):n >> k] = d
    coef[..., :n >> num] = x
    return coef


def wpt_fast(x, num, lo, hi):
    """coefArr of wpt() through wpt_level(), for any leading axes"""
    for k in range(num):
        x = wpt_level(x, k, lo, hi)[0]
    return np.asarray(x, np.float64)


def swt_fast(x, num, lo, hi):
    """(approximations, details) of swt() through swt_level(), each [..., num, n]"""
    rows, x = [], np.asarray(x, np.float64)
    for i in range(num):
        a, d = swt_level(x, 1 << i, lo, hi)[:2]
        rows.append((a, d))
        x = a
    shape = x.shape[:-1] + (num, x.shape[-1])
    return tuple(np.stack([r[p] for r in rows], axis=-2) if rows else np.zeros(shape) for p in (0, 1))


def swt(x, num, lo, hi):
    n = len(x)
    dec = len(lo)
    m1, m2 = np.zeros((num, n)), np.zeros((num, n))
    lo2, hi2 = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    up = dec
    for i in range(num):
        src = np.asarray(x, np.float64) if i == 0 else m1[i - 1]
        p = period_padding(src, up)
        m1[i] = np.convolve(p, lo2[:up])[up:up + n]
        m2[i] = np.convolve(p, hi2[:up])[up:up + n]
        lo2, hi2 = np.zeros(up * 2), np.zeros(up * 2)
        lo2[::1 << (i + 1)][:dec] = lo
        hi2[::1 << (i + 1)][:dec] = hi
        up *= 2
    return m1, m2


# ---- the C objects (reference build or this library) ----

def new(lib, kind, num, size, ty, t1, t2):
    """status, object of dwtObj_new / wptObj_new (size = radix2Exp) or swtObj_new (size = fftLength)"""
    obj = C.c_void_p()
    st = getattr(lib, f"{kind}Obj_new")(C.byref(obj), num, size, C.byref(C.c_int(ty)), C.byref(C.c_int(t1)),
                                        C.byref(C.c_int(t2)))
    return st, obj


def run(lib, kind, num, size, ty, t1, t2, x):
    """the legacy call of the object on one clip: (coef, m_data) or (m_data1, m_data2)"""
    st, obj = new(lib, kind, num, size, ty, t1, t2)
    assert st == 0 and obj, (kind, num, size, ty, t1, t2, st)
    x = np.ascontiguousarray(x, np.float32)
    n = len(x)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)
    try:
        if kind == "swt":
            a, b = np.zeros((num, n), np.float32), np.zeros((num, n), np.float32)
        else:
            a = np.zeros(n, np.float32)
            b = np.zeros((num if kind == "dwt" else 1 << num, n), np.float32)
        getattr(lib, f"{kind}Obj_{kind}")(obj, ptr(x), ptr(a), ptr(b))
    finally:
        getattr(lib, f"{kind}Obj_free")(obj)
    return a, b


def filters(lib, ty, t1, t2):
    """loD, hiD of the reference's dwt_filterCoef (float32 values)"""
    f = lib.dwt_filterCoef
    f.restype = C.c_int
    f.argtypes = [C.c_int] * 4 + [C.POINTER(C.POINTER(C.c_float))] * 2
    lo, hi = C.POINTER(C.c_float)(), C.POINTER(C.c_float)()
    n = f(ty, t1, t2, 0, C.byref(lo), C.byref(hi))
    return np.array(lo[:n], np.float32), np.array(hi[:n], np.float32)


def signal(n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    return (0.5 * np.sin(2 * np.pi * t * 0.013 * (1 + seed % 5)) + 0.3 * rng.standard_normal(n)).astype(np.float32)


# ---- the level-by-level GPU suite (tests/test_gpu_wavelet_levels.py): its clips and cases ----

NOISE = [0, 2]                 # the white-noise clips of level_clips()
SYM4, DB30, HAAR = (2, 4, 0), (1, 30, 0), (0, 0, 0)
M_DATA_BYTES = 256 << 20       # the largest mDataArr (all clips of a call) the suite requests


def level_clips(n, seed):
    """the four clips of every call: white noise; a smooth low sine (3 cycles), whose finest details cancel to ~1e-8 of
    the approximation; the noise 1000x louder and reversed; a unit impulse, so most elements have scale 0"""
    noise = np.random.default_rng(seed).standard_normal(n)
    impulse = np.zeros(n)
    impulse[n // 3] = 1.0
    sine = np.sin(2 * np.pi * 3 * np.arange(n) / n)
    return np.stack([noise, sine, 1e3 * noise[::-1], impulse]).astype(np.float32)


def level_cases(table):
    """{name: (kind, num, size, filter key, mData requested)}: size is radix2Exp for DWT / WPT, n for SWT.
    - every filter: DWT 2^10 with num 9 (the last levels have L = 4 < dec), WPT 2^8 with num 7 (nodes of 2), SWT
      n = 2^8 with num 8;
    - DWT: radix2Exp 2 .. 20 at num radix2Exp - 1 and a middle num, with sym4 and db30 (60 taps: 15 wraps at L = 4), and
      haar as well above 2^16;
    - WPT: sym4 at every num 1 .. radix2Exp - 1 for radix2Exp 2 .. 14; num 3 and radix2Exp - 1 at 2^18 .. 2^20 without
      mData;
    - SWT: db30 at n = 2^num, 3 2^num and 5 2^num for num 1 .. 12 (the last level's dec s / 2 is 15 n, 5 n and 3 n),
      sym4 at those n for num 4, 8, 12, and sym4 at n = 2^20 with num 10.
    mData is requested where all four clips' mDataArr fits M_DATA_BYTES."""
    out = {}

    def tree(kind, num, e, key, m_data=True):
        rows = num if kind == "dwt" else 1 << num
        fits = 4 * rows * (4 << e) <= M_DATA_BYTES
        out[f"{kind}_e{e}_n{num}_{'_'.join(map(str, key))}"] = (kind, num, e, key, m_data and fits)

    def swt_case(num, n, key):
        out[f"swt_{n}_n{num}_{'_'.join(map(str, key))}"] = ("swt", num, n, key, False)

    for key in sorted(table):
        tree("dwt", 9, 10, key)
        tree("wpt", 7, 8, key)
        swt_case(8, 256, key)
    for e in range(2, 21):
        for num in sorted({e - 1, max(1, e // 2)}):
            for key in (SYM4, DB30) + ((HAAR,) if e > 16 else ()):
                tree("dwt", num, e, key)
    for e in range(2, 15):
        for num in range(1, e):
            tree("wpt", num, e, SYM4)
    for e in (18, 19, 20):
        for num in (3, e - 1):
            tree("wpt", num, e, SYM4, m_data=False)
    for num in range(1, 13):
        for n in (1 << num, 3 << num, 5 << num):
            swt_case(num, n, DB30)
            if num % 4 == 0:
                swt_case(num, n, SYM4)
    swt_case(10, 1 << 20, SYM4)
    return out
