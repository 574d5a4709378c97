"""numpy restatement of audioFlux's non-stationary Gabor transform (NSGTObj), and ctypes drivers of its C API that run
against either libaudioflux_b200.so or the reference build.

    constructor  src/nsgt_algorithm.c:72-251      bank   src/filterbank/nsgt_filterBank.c:48-239 (edges :482-555,
    time grids   src/nsgt_algorithm.c:253-290              standard windows :247-305, efficient windows :307-365)
    transform    src/nsgt_algorithm.c:483-605     inverse DFT src/dsp/dft_algorithm.c:106-152

Integer outcomes (bins, lengths, the column map) are reproduced with the reference's float32 arithmetic; the transform
itself runs in float64 (numpy FFTs)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import af_oracle as O

f32 = np.float32
EFFICIENT, STANDARD = 0, 1
MAX_LEN = 16384             # longest band window libaudioflux_b200 accepts (nsgtObj_new returns -2 above)
STYLES = (O.STYLE_SLANEY, O.STYLE_ETSI, O.STYLE_HANN, O.STYLE_HAMM, O.STYLE_BLACKMAN, O.STYLE_BOHMAN, O.STYLE_KAISER,
          O.STYLE_GAUSS, O.STYLE_RECT)
_STYLE_WINDOW = {O.STYLE_SLANEY: O.W_TRIANG, O.STYLE_ETSI: O.W_BARTLETT, O.STYLE_HANN: O.W_HANN,
                 O.STYLE_HAMM: O.W_HAMM, O.STYLE_BLACKMAN: O.W_BLACKMAN, O.STYLE_BOHMAN: O.W_BOHMAN,
                 O.STYLE_KAISER: O.W_KAISER, O.STYLE_GAUSS: O.W_GAUSS}


def params(num, radix2_exp, samplate=None, low_fre=None, high_fre=None, bin_per_octave=None, min_len=None,
           bank_type=None, scale_type=None, style_type=None, normal_type=None):
    """nsgtObj_new's defaults, clamps and status codes (nsgt_algorithm.c:104-214) -> (status, p); None = NULL pointer"""
    p = dict(num=num, radix2_exp=radix2_exp, min_len=min_len if min_len is not None and min_len > 0 else 3)
    if radix2_exp and not 1 <= radix2_exp <= 30:
        return -100, None
    n = 1 << radix2_exp
    sr = samplate if samplate is not None and 0 < samplate <= 196000 else 32000
    scale = O.SCALE_OCTAVE if scale_type is None else scale_type
    if scale > O.SCALE_LOG:
        return 1, None
    style = O.STYLE_HANN if style_type is None else style_type
    style = O.STYLE_HANN if style == O.STYLE_GAMMATONE else style
    norm = O.NORM_BANDWIDTH if normal_type is None else normal_type
    norm = O.NORM_BANDWIDTH if norm == O.NORM_AREA else norm
    bpo = bin_per_octave if bin_per_octave is not None and 4 <= bin_per_octave <= 48 else 12
    lo, hi, _, _ = O.bft_revise_range(num, n, sr, None if low_fre is None else float(f32(low_fre)),
                                      None if high_fre is None else float(f32(high_fre)), scale, bpo)
    if scale in (O.SCALE_LINEAR, O.SCALE_OCTAVE) and float(hi) > sr / 2.0:
        return -1, None
    if num < 2 or num > n // 2 + 1:
        return -1, None
    p.update(fft_length=n, samplate=sr, low=lo, high=hi, bpo=bpo, scale=scale, style=style, norm=norm,
             bank=STANDARD if bank_type == STANDARD else EFFICIENT)
    return 0, p


def window(style, length, periodic):
    """window_createXxx(length, flag) (src/dsp/flux_window.c:64-78 and siblings): flag 1 = symmetric of length+1,
    truncated, for every type; length 1 = {1}; Point / Rect = ones"""
    kind = _STYLE_WINDOW.get(style)
    if kind is None or length == 1:
        return np.ones(length, f32)
    w = O._symmetric_window(kind, length + 1)[:length] if periodic else O._symmetric_window(kind, length)
    return w.astype(f32)


def bank(p, min_len=None):
    """nsgt_filterBank -> dict(lens, offs, bins, fre, windows [list], max_len, total_len)"""
    num, n, sr = p["num"], p["fft_length"], p["samplate"]
    min_len = p["min_len"] if min_len is None else min_len
    low, high, ref = O.revise_edges(num, p["low"], p["high"], p["scale"], n, sr, p["bpo"], is_edge=False)
    fre, bins = O.band_edges(num, n, sr, low, high, p["scale"], ref, False, False)
    lens, offs, wins = [], [], []
    for i in range(num):
        left, cur, right = int(bins[i]), int(bins[i + 1]), int(bins[i + 2])
        if p["bank"] == STANDARD:                                             # :145-152
            ln = right - left + 1
        else:                                                                 # :153-182
            ln = 2 * max(cur - left, right - cur) + 1 if right - left >= 1 else 0
        ln = max(ln, min_len)
        lens.append(ln)
        offs.append(max(cur - ln // 2, 0))                                    # :259-263
        w = window(p["style"], ln, p["bank"] == STANDARD)
        if p["norm"] == O.NORM_BANDWIDTH:
            w = (w / f32(np.sqrt(f32(ln)))).astype(f32)
        wins.append(w)
    lens = np.array(lens, np.int64)
    return dict(lens=lens, offs=np.array(offs, np.int64), bins=bins[1:num + 1].astype(np.int64),
                fre=fre[1:num + 1].astype(f32), windows=wins, max_len=int(lens.max()), total_len=int(lens.sum()))


def column_map(lens, fft_length, samplate):
    """step 3 of nsgtObj_nsgt (:585-604) on the grids of __nsgtObj_dealTime (:253-290): map[i][j] = k-1 for the first k
    with maxTime[j] < time_i[k], -1 where there is none"""
    max_len = int(max(lens))
    time = f32(f32(fft_length) / f32(samplate))
    max_time = O._linspace_f32(0, time, max_len + 1)[:max_len]
    out = np.full((len(lens), max_len), -1, np.int64)
    for i, ln in enumerate(lens):
        cur = f32(ln)
        det = f32(ln - 2) if ln - 2 >= 0 else f32(0)
        off = f32(time / f32(cur + det))
        grid = O._linspace_f32(f32(-off), f32(time + off), int(ln) + 1)
        k = np.searchsorted(grid, max_time, side="right")       # grid is non-decreasing, so this is the reference's scan
        out[i] = np.where(k <= ln, k - 1, -1)
    return out


def transform(x, p, b=None):
    """-> (cells [list of complex128 arrays], matrix complex128 [num, max_len])"""
    X = np.fft.fft(np.asarray(x, np.float64))                # the reference's full complex FFT of the real clip
    return transform_spectrum(X, p, b)


def transform_spectrum(X, p, b=None):
    """the band step of the transform from the clip's full complex spectrum X [fft_length]
    -> (cells [list of complex128 arrays], matrix complex128 [num, max_len])"""
    b = bank(p) if b is None else b
    n = p["fft_length"]
    X = np.asarray(X, np.complex128)
    cells = []
    for ln, off, w in zip(b["lens"], b["offs"], b["windows"]):
        j = np.arange(ln)
        a = np.zeros(ln, np.complex128)
        a[(j + ln - ln // 2) % ln] = X[np.clip(off + j, 0, n - 1)] * w.astype(np.float64)
        cells.append(np.fft.ifft(a))                          # (1/L) sum_k a_k e^{+2 pi i k n / L}
    cmap = column_map(b["lens"], n, p["samplate"])
    m = np.zeros(cmap.shape, np.complex128)
    for i, c in enumerate(cells):
        ok = cmap[i] >= 0
        m[i, ok] = c[cmap[i, ok]]
    return cells, m


# ---- per-band comparison of the band kernels (kernels/nsgt.cu) ----
BLUESTEIN_MAX = 4096        # longest band of k_nsgt_bluestein; longer bands run k_nsgt_direct
DIRECT_PASS = 1024 * 6      # outputs k_nsgt_direct computes per pass (1024 threads x 6)
BAND_TOL = 1e-4


def log2_m(ln):
    """log2 of k_nsgt_bluestein's convolution size M = 2^ceil(log2(2L - 1))"""
    return int(2 * ln - 2).bit_length()


def band_path(ln):
    """the kernel path of a band of length ln, e.g. "bluestein M=2^13" or "direct 3 passes" """
    if ln <= BLUESTEIN_MAX:
        return f"bluestein M=2^{log2_m(ln)}"
    passes = -(-int(ln) // DIRECT_PASS)
    return f"direct {passes} pass{'es' if passes > 1 else ''}"


def full_spectrum(re, im):
    """half-spectrum planes [..., N/2 + 1] -> the full complex128 spectrum [..., N] the band kernels read: bins above N/2
    are the conjugate mirror X[k] = conj(X[N - k])"""
    h = np.asarray(re, np.float64) + 1j * np.asarray(im, np.float64)
    return np.concatenate([h, np.conj(h[..., -2:0:-1])], axis=-1)


def split_cells(cr, ci, lens):
    """one clip's cell planes [total_len] -> [complex128 array per band]"""
    c = np.asarray(cr, np.float64) + 1j * np.asarray(ci, np.float64)
    return np.split(c, np.cumsum(lens)[:-1])


def check_bands(got, want, lens, tol=BAND_TOL, what=""):
    """Per band: max |got - want| <= tol * max |want| of that band; a band whose want is exactly zero must be exactly
    zero in got.  got, want: [complex array per band].  -> {band_path: worst relative error}.  AssertionError naming
    every failing band (index, L, log2 M, path)."""
    worst, bad = {}, []
    for i, (g, w, ln) in enumerate(zip(got, want, lens)):
        assert g.shape == w.shape == (ln,), (what, i, g.shape, w.shape, ln)
        path = band_path(ln)
        peak = np.abs(w).max()
        if peak == 0:
            err = 0.0 if not np.any(g) else np.inf
        else:
            err = float(np.abs(g - w).max() / peak)
        worst[path] = max(worst.get(path, 0.0), err)
        if not err <= tol:
            bad.append(f"band {i} L={ln} log2M={log2_m(ln) if ln <= BLUESTEIN_MAX else '-'} {path}: "
                       + ("want exactly 0, got max |.| %.3e" % np.abs(g).max() if peak == 0 else f"{err:.3e}"))
    assert not bad, f"{what}: {len(bad)} of {len(lens)} bands above {tol:g} of their own max\n" + "\n".join(bad[:30])
    return worst


# ---- the C API (libaudioflux_b200.so or the reference build) ----
def _ip(v):
    return None if v is None else C.byref(C.c_int(int(v)))


def _fp(v):
    return None if v is None else C.byref(C.c_float(float(v)))


def c_new(lib, num, radix2_exp, samplate=None, low_fre=None, high_fre=None, bin_per_octave=None, min_len=None,
          bank_type=None, scale_type=None, style_type=None, normal_type=None):
    obj = C.c_void_p()
    st = lib.nsgtObj_new(C.byref(obj), num, radix2_exp, _ip(samplate), _fp(low_fre), _fp(high_fre), _ip(bin_per_octave),
                         _ip(min_len), _ip(bank_type), _ip(scale_type), _ip(style_type), _ip(normal_type))
    return st, obj


def c_tables(lib, obj, num):
    max_len, total = lib.nsgtObj_getMaxTimeLength(obj), lib.nsgtObj_getTotalTimeLength(obj)
    lens = np.ctypeslib.as_array((C.c_int * num).from_address(lib.nsgtObj_getTimeLengthArr(obj))).astype(np.int64)
    bins = np.ctypeslib.as_array((C.c_int * num).from_address(lib.nsgtObj_getBinBandArr(obj))).astype(np.int64)
    fre = np.ctypeslib.as_array((C.c_float * num).from_address(lib.nsgtObj_getFreBandArr(obj))).copy()
    return dict(max_len=max_len, total_len=total, lens=lens, bins=bins, fre=fre)


def c_nsgt(lib, obj, x, num):
    """nsgtObj_nsgt + nsgtObj_getCellData -> (matrix re, im, cells re, im)"""
    max_len, total = lib.nsgtObj_getMaxTimeLength(obj), lib.nsgtObj_getTotalTimeLength(obj)
    x = np.ascontiguousarray(x, np.float32)
    re = np.zeros((num, max_len), np.float32)
    im = np.zeros_like(re)
    lib.nsgtObj_nsgt(obj, x.ctypes.data, re.ctypes.data, im.ctypes.data)
    pr, pi = C.c_void_p(), C.c_void_p()
    lib.nsgtObj_getCellData(obj, C.byref(pr), C.byref(pi))
    cr = np.ctypeslib.as_array((C.c_float * total).from_address(pr.value)).copy()
    ci = np.ctypeslib.as_array((C.c_float * total).from_address(pi.value)).copy()
    return re, im, cr, ci


def c_filterbank(lib, p, min_len=None):
    """the reference's exported nsgt_filterBank (nsgt_filterBank.c:48-239) with the revised range of nsgtObj_new"""
    num = p["num"]
    lens, fre = np.zeros(num, np.int32), np.zeros(num, np.float32)
    bins, offs = np.zeros(num, np.int32), np.zeros(num, np.int32)
    wp, mx, tot = C.c_void_p(), C.c_int(), C.c_int()
    lib.nsgt_filterBank(num, p["fft_length"], p["samplate"], p["min_len"] if min_len is None else min_len,
                        1 if p["bank"] == STANDARD else 0, p["scale"], p["style"], p["norm"], float(p["low"]),
                        float(p["high"]), p["bpo"], C.byref(wp), lens.ctypes.data, fre.ctypes.data, bins.ctypes.data,
                        offs.ctypes.data, C.byref(mx), C.byref(tot))
    w = np.ctypeslib.as_array((C.c_float * tot.value).from_address(wp.value)).copy()
    return dict(lens=lens.astype(np.int64), fre=fre, bins=bins.astype(np.int64), offs=offs.astype(np.int64),
                win=w, max_len=mx.value, total_len=tot.value)


def case_signal(seed, n, sr):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    x = 0.2 * np.sin(2 * np.pi * 440 * t) + 0.1 * np.sin(2 * np.pi * 97.3 * t) + 0.05 * rng.standard_normal(n)
    return x.astype(np.float32)


def cases():
    """the CPU case set: both banks x all seven scales, with the styles, norms, minimum lengths and sizes cycled through,
    plus three 2^15 cases -> [(name, kwargs of c_new / params)]"""
    out = []
    for i, (bank_t, scale) in enumerate([(b, s) for b in (EFFICIENT, STANDARD) for s in range(7)]):
        for t in range(4):
            idx = 4 * i + t
            radix = 8 if t < 2 else 12
            kw = dict(num=24 if radix == 8 else 48, radix2_exp=radix, samplate=32000 if t != 3 else 44100,
                      low_fre=None, high_fre=None, bin_per_octave=12 if t % 2 == 0 else 24,
                      min_len=(1, 3, 20)[idx % 3], bank_type=bank_t, scale_type=scale,
                      style_type=STYLES[idx % len(STYLES)], normal_type=(O.NORM_NONE, O.NORM_BANDWIDTH)[(idx // 2) % 2])
            if scale in (O.SCALE_OCTAVE, O.SCALE_LOG):
                kw["low_fre"] = 32.703196
            out.append((f"b{bank_t}s{scale}t{t}", kw))
    out.append(("docs84", dict(num=84, radix2_exp=15, samplate=32000, low_fre=32.703196, high_fre=None, bin_per_octave=12,
                               min_len=3, bank_type=EFFICIENT, scale_type=O.SCALE_OCTAVE, style_type=O.STYLE_SLANEY,
                               normal_type=O.NORM_BANDWIDTH)))
    out.append(("mel40std", dict(num=40, radix2_exp=15, samplate=22050, low_fre=None, high_fre=2000.0, bin_per_octave=12,
                                 min_len=3, bank_type=STANDARD, scale_type=O.SCALE_MEL, style_type=O.STYLE_HANN,
                                 normal_type=O.NORM_NONE)))
    out.append(("lin30", dict(num=30, radix2_exp=15, samplate=32000, low_fre=1000.0, high_fre=None, bin_per_octave=12,
                              min_len=20, bank_type=EFFICIENT, scale_type=O.SCALE_LINEAR, style_type=O.STYLE_KAISER,
                              normal_type=O.NORM_BANDWIDTH)))
    return out
