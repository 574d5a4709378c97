"""Float64 numpy restatement of the reference's harmonic-percussive separation, the case list, and ctypes drivers that
work on either library.

src/mir/hpss_algorithm.c:
  - hpssObj_new (:40-94): Hamm window by default; an order is taken when > 0 and odd, else 21 (h) / 31 (p); the hop is
    always fftLength / 4, whatever slideLength says; the STFT has no padding;
  - hpssObj_calDataLength (:96-111): (T - 1) * hop + fftLength, T = 0 below one frame;
  - hpssObj_hpss (:118-345): mag = |X| over the half spectrum, mH = the median over hOrder frames of each bin, mP = the
    median over pOrder bins of each frame (centred windows, zeros beyond the edges: scipy's median_filter with
    mode="constant", cval=0); an order of 1 leaves that median at 0 (the filter does not run); h1 = mH^2, p1 = mP^2,
    v = max(h1 + p1, 1e-16); H = h1 / v * mag and P = p1 / v * mag with the phase X / max(mag, 1e-16), mirrored to the
    full spectrum and taken through stftObj_istft (method 0), which adds into the caller's buffer and then divides."""
import ctypes as C

import numpy as np
from scipy.ndimage import median_filter

from oracle import af_oracle as O

f32 = np.float32
W_RECT, W_HANN, W_HAMM = O.W_RECT, O.W_HANN, O.W_HAMM


def rules(h_order=None, p_order=None, window=None):
    """:40-94 -> (hOrder, pOrder, windowType); None is a NULL pointer"""
    h = h_order if h_order is not None and h_order > 0 and h_order & 1 else 21
    p = p_order if p_order is not None and p_order > 0 and p_order & 1 else 31
    return h, p, W_HAMM if window is None else window


def time_length(L, n):
    return 0 if L < n else (L - n) // (n // 4) + 1


def data_length(L, n):
    return (time_length(L, n) - 1) * (n // 4) + n


def _median(mag, order, axis):
    if order == 1:
        return np.zeros_like(mag)
    size = (order, 1) if axis == 0 else (1, order)
    return median_filter(mag, size=size, mode="constant", cval=0.0)


def hpss(x, radix2_exp, h_order=None, p_order=None, window=None, init_h=None, init_p=None):
    """-> (h, p) float32, each data_length(len(x)) samples"""
    n = 1 << radix2_exp
    hop = n // 4
    ho, po, w = rules(h_order, p_order, window)
    win = O.fft_window(w, n)
    re, im = O.stft(x, n, hop, win)
    W = n // 2 + 1
    X = re[:, :W].astype(np.float64) + 1j * im[:, :W].astype(np.float64)
    mag = np.abs(X)
    phase = X / np.maximum(mag, 1e-16)
    h1, p1 = _median(mag, ho, 0) ** 2, _median(mag, po, 1) ** 2
    v = np.maximum(h1 + p1, 1e-16)
    out = []
    for part, init in ((h1 / v * mag, init_h), (p1 / v * mag, init_p)):
        Y = phase * part
        full = np.concatenate([Y, np.conj(Y[:, 1:n // 2][:, ::-1])], axis=1)
        out.append(O.istft(full.real, full.imag, n, hop, win, 0, init))
    return out[0], out[1]


def istft_norm(T, radix2_exp, window=None):
    """the inverse STFT's per-sample normaliser (sum of the squared window), for the DESIGN section 2 rule"""
    n = 1 << radix2_exp
    w = O.fft_window(rules(None, None, window)[2], n).astype(np.float64) ** 2
    norm = np.zeros((T - 1) * (n // 4) + n)
    for t in range(T):
        norm[t * (n // 4):t * (n // 4) + n] += w
    return norm


def errors(got, want, kw):
    """-> (max error where the inverse STFT's normaliser is >= 1e-2, max error elsewhere), both over max|want|; 0 for
    outputs that are both all zero, inf when only one is (the 1e-2 rule of DESIGN section 2)"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    scale = np.abs(want).max()
    d = np.abs(got - want)
    if scale == 0:
        return (0.0, 0.0) if not d.any() else (np.inf, np.inf)
    n = 1 << kw["radix2_exp"]
    good = istft_norm(time_length(kw["length"], n), kw["radix2_exp"], kw.get("window")) >= 1e-2
    return d[good].max(initial=0) / scale, d[~good].max(initial=0) / scale


def cases():
    """(name, kw): radix2_exp, length, window / h_order / p_order (None: a NULL pointer), outputs "hp" | "h" | "p",
    init: seed of the values the legacy call's buffers hold before the call (None: zeros)"""
    out = []

    def add(name, r, length, **kw):
        out.append((name, dict(radix2_exp=r, length=length, **kw)))
    add("hamm_n10_defaults", 10, 4800)                                  # hOrder 21 > T = 15
    add("hann_n9", 9, 2000, window=W_HANN, h_order=5, p_order=7)
    add("rect_n9", 9, 2000, window=W_RECT, h_order=3, p_order=3)
    add("hamm_n6", 6, 1500)                                             # pOrder 31 next to W = 33
    add("hamm_n6_orders_121_45", 6, 1500, h_order=121, p_order=45)     # larger than T = 90 and W = 33
    add("hamm_n6_orders_201_301", 6, 1500, h_order=201, p_order=301)   # more than twice T and W: both medians 0
    add("hann_n7", 7, 2000, window=W_HANN, h_order=9, p_order=15)
    add("hamm_n8", 8, 2000, window=W_HAMM)
    add("hamm_n9", 9, 2500, h_order=21, p_order=31)
    add("h_order_1", 9, 2000, h_order=1)
    add("p_order_1", 9, 2000, p_order=1)
    add("orders_1_1", 9, 2000, h_order=1, p_order=1)
    add("orders_even_zero", 9, 2000, h_order=20, p_order=0)
    add("orders_negative_even", 9, 2000, h_order=-3, p_order=4)
    add("t1", 10, 1024, h_order=1)
    add("t1_tail", 10, 1279, window=W_HANN, h_order=1, p_order=5)
    add("h_only", 9, 2000, h_order=7, outputs="h")
    add("p_only", 9, 2000, outputs="p")
    add("init_buffers", 9, 2000, h_order=7, init=7)
    add("orders_383", 10, 1024 + 250 * 256, h_order=383, p_order=383)  # the largest supported, T = 251, W = 513
    add("hamm_n11", 11, 10000, h_order=9)
    add("hamm_n12", 12, 14336, h_order=7)
    add("hann_n12_init", 12, 9000, window=W_HANN, h_order=3, init=11)
    add("hamm_n13", 13, 16384 + 3 * 2048, h_order=5)
    add("hamm_n14", 14, 16384 + 3 * 4096, h_order=3, p_order=301)
    add("hamm_n15", 15, 32768 + 2 * 8192, h_order=3)                  # the four-step STFT / inverse STFT
    return out


def case_signal(name, kw, length=None):
    """tones (harmonic) + clicks every 0.1 s (percussive) + noise, seeded by the name"""
    n = kw["length"] if length is None else length
    rng = np.random.default_rng(sum(map(ord, name)))
    t = np.arange(n) / 16000.0
    x = 0.3 * np.sin(2 * np.pi * 440 * t) + 0.2 * np.sin(2 * np.pi * 1320 * t + 0.5) + 0.01 * rng.standard_normal(n)
    x[::1600] += 1.0
    x[1::1600] -= 0.6
    return x.astype(np.float32)


def case_init(kw, m, which):
    if kw.get("init") is None:
        return None
    return np.random.default_rng(kw["init"] + which).standard_normal(m).astype(np.float32)


def oracle_case(name, kw):
    """-> [h, p] float32 of the requested outputs (None for a skipped one)"""
    x = case_signal(name, kw)
    m = data_length(x.size, 1 << kw["radix2_exp"])
    h, p = hpss(x, kw["radix2_exp"], kw.get("h_order"), kw.get("p_order"), kw.get("window"), case_init(kw, m, 0),
                case_init(kw, m, 1))
    outs = kw.get("outputs", "hp")
    return [h if "h" in outs else None, p if "p" in outs else None]


# ------------------------------------------------------------------------------------------------ ctypes drivers
def _oi(v):
    return None if v is None else C.byref(C.c_int(int(v)))


def c_new(lib, radix2_exp, window=None, slide_length=None, h_order=None, p_order=None):
    """-> (status, obj)"""
    o = C.c_void_p()
    st = lib.hpssObj_new(C.byref(o), int(radix2_exp), _oi(window), _oi(slide_length), _oi(h_order), _oi(p_order))
    return st, o


def c_hpss(lib, o, x, outputs="hp", init_h=None, init_p=None, extra=16, fill=0.0):
    """one legacy call into buffers of calDataLength + extra floats (init, else `fill`) -> (h, p) buffers (None when
    not requested)"""
    x = np.ascontiguousarray(x, np.float32)
    m = lib.hpssObj_calDataLength(o, x.size)
    bufs = []
    for k, init in ((0, init_h), (1, init_p)):
        if "hp"[k] not in outputs:
            bufs.append(None)
            continue
        b = np.full(max(m, 0) + extra, fill, np.float32)
        if init is not None:
            b[:m] = init[:m]
        bufs.append(b)
    lib.hpssObj_hpss(o, x.ctypes.data, x.size, None if bufs[0] is None else bufs[0].ctypes.data,
                     None if bufs[1] is None else bufs[1].ctypes.data)
    return bufs[0], bufs[1]


def c_case(lib, name, kw):
    """-> [h, p] float32 outputs of the library, like oracle_case"""
    st, o = c_new(lib, kw["radix2_exp"], kw.get("window"), 1024, kw.get("h_order"), kw.get("p_order"))
    assert st == 0, (name, st)
    try:
        x = case_signal(name, kw)
        m = lib.hpssObj_calDataLength(o, x.size)
        h, p = c_hpss(lib, o, x, kw.get("outputs", "hp"), case_init(kw, m, 0), case_init(kw, m, 1))
        return [None if b is None else b[:m].copy() for b in (h, p)]
    finally:
        lib.hpssObj_free(o)
