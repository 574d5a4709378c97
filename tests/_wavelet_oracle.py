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
