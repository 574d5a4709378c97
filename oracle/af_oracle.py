"""CPU restatement (numpy) of audioFlux's time-frequency hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``audioflux_b200/`` may import this
module; it is the checker used by ``tests/``, ``__graft_entry__.smoke()`` and
the ``cpu_baseline`` leg of ``bench.py``.

Every function cites the reference file:line (relative to the audioFlux source tree) it
restates.  Arithmetic is done in float64 unless the reference's float32
rounding decides an *integer* outcome (band-edge bin indices, kernel lengths),
in which case the float32 steps are reproduced explicitly.

Pinning: the reference ships no tests or golden vectors for this path
(SURVEY.md section 4), so this restatement is pinned by (i) the reference itself
compiled into ``oracle/_ref`` (tests/test_oracle_vs_ref.py, run wherever that
library exists) and (ii) fixtures generated from that library and committed
under ``tests/golden`` (tests/golden/make_golden.py).
"""
from __future__ import annotations

import math
import numpy as np

f32 = np.float32

# ---------------------------------------------------------------------------
# enums (src/flux_base.h:14-168) -- plain ints shared with the C ABI
# ---------------------------------------------------------------------------
W_RECT, W_HANN, W_HAMM, W_BLACKMAN, W_KAISER, W_BARTLETT, W_TRIANG, W_FLATTOP, \
    W_GAUSS, W_BLACKMAN_HARRIS, W_BLACKMAN_NUTTALL, W_BARTLETT_HANN, W_BOHMAN, W_TUKEY = range(14)
DATA_POWER, DATA_MAG = 0, 1
SCALE_LINEAR, SCALE_LINSPACE, SCALE_MEL, SCALE_BARK, SCALE_ERB, SCALE_OCTAVE, SCALE_LOG = range(7)
STYLE_SLANEY, STYLE_ETSI, STYLE_GAMMATONE, STYLE_POINT, STYLE_RECT, STYLE_HANN, STYLE_HAMM, \
    STYLE_BLACKMAN, STYLE_BOHMAN, STYLE_KAISER, STYLE_GAUSS = range(11)
NORM_NONE, NORM_AREA, NORM_BANDWIDTH = 0, 1, 2
RECT_LOG, RECT_CUBIC = 0, 1
WAVE_MORSE, WAVE_MORLET, WAVE_BUMP, WAVE_PAUL, WAVE_DOG, WAVE_MEXICAN, WAVE_HERMIT, WAVE_RICKER = range(8)


# ---------------------------------------------------------------------------
# windows  (src/dsp/flux_window.c)
# ---------------------------------------------------------------------------
def _bessel_i0_series(a):
    """15-term power series the reference uses (flux_window.c `__besselZeroOne`)."""
    a = np.asarray(a, dtype=np.float64)
    b = a / 2.0
    s = np.ones_like(b)
    num = np.ones_like(b)
    den = 1.0
    for k in range(1, 16):
        num = num * b
        den = den * k
        s = s + (num / den) ** 2
    return s


def _symmetric_window(kind, L, value=None):
    """Symmetric window of length L (flag=0 creators, flux_window.c:281-640, 737-850)."""
    if L == 1:
        return np.ones(1)
    i = np.arange(L, dtype=np.float64)
    M = L - 1
    if kind == W_HANN:
        w = 0.5 - 0.5 * np.cos(2 * np.pi * i / M)
    elif kind == W_HAMM:
        w = 0.54 - 0.46 * np.cos(2 * np.pi * i / M)
    elif kind == W_BLACKMAN:
        w = 0.42 - 0.5 * np.cos(2 * np.pi * i / M) + 0.08 * np.cos(4 * np.pi * i / M)
        w[0] = w[-1] = 0.0
    elif kind == W_KAISER:
        beta = 5.0 if value is None or value <= 0 else value
        v = 2.0 * i / M - 1.0
        w = _bessel_i0_series(beta * np.sqrt(np.maximum(0.0, 1 - v * v))) / _bessel_i0_series(beta)
    elif kind == W_BARTLETT:
        w = 1.0 - np.abs(2.0 * i / M - 1.0)
    elif kind == W_TRIANG:
        if L % 2 == 0:
            half = 2.0 * (np.arange(L // 2) + 0.5) / L
            w = np.concatenate([half, half[::-1]])
        else:
            half = 2.0 * (np.arange((L + 1) // 2) + 1.0) / (L + 1)
            w = np.concatenate([half, half[-2::-1]])
    elif kind == W_FLATTOP:
        a = (0.21557895, 0.41663158, 0.277263158, 0.083578947, 0.006947368)
        w = (a[0] - a[1] * np.cos(2 * np.pi * i / M) + a[2] * np.cos(4 * np.pi * i / M)
             - a[3] * np.cos(6 * np.pi * i / M) + a[4] * np.cos(8 * np.pi * i / M))
    elif kind == W_GAUSS:
        alpha = 2.5 if value is None or value <= 0 else value
        w = np.exp(-0.5 * (alpha * (i - M / 2.0) / (M / 2.0)) ** 2)
    elif kind == W_BLACKMAN_HARRIS:
        a = (0.35875, 0.48829, 0.14128, 0.01168)
        w = (a[0] - a[1] * np.cos(2 * np.pi * i / M) + a[2] * np.cos(4 * np.pi * i / M)
             - a[3] * np.cos(6 * np.pi * i / M))
    elif kind == W_BLACKMAN_NUTTALL:
        a = (0.3635819, 0.4891775, 0.1365995, 0.0106411)
        w = (a[0] - a[1] * np.cos(2 * np.pi * i / M) + a[2] * np.cos(4 * np.pi * i / M)
             - a[3] * np.cos(6 * np.pi * i / M))
    elif kind == W_BARTLETT_HANN:
        r = i / M - 0.5
        w = 0.62 - 0.48 * np.abs(r) + 0.38 * np.cos(2 * np.pi * r)
        w[0] = w[-1] = 0.0
    elif kind == W_BOHMAN:
        l = np.abs(-1.0 + 2.0 * i / M)
        w = (1 - l) * np.cos(np.pi * l) + np.sin(np.pi * l) / np.pi
        w[0] = w[-1] = 0.0
    elif kind == W_TUKEY:
        a = 0.5 if value is None or not (0 <= value <= 1) else value
        if a == 0:
            return np.ones(L)
        if a == 1:
            return _symmetric_window(W_HANN, L)
        x = i / M
        w = np.ones(L)
        lo = x < a / 2
        hi = x >= 1 - a / 2
        w[lo] = 0.5 * (1 + np.cos(2 * np.pi / a * (x[lo] - a / 2)))
        w[hi] = 0.5 * (1 + np.cos(2 * np.pi / a * (x[hi] - 1 + a / 2)))
    else:
        w = np.ones(L)
    return w


def fft_window(win_type: int, n: int) -> np.ndarray:
    """`window_calFFTWindow` (flux_window.c:890-940): periodic variants = symmetric
    window of length n+1 truncated to n, except Bartlett/Triang/Bartlett-Hann/Bohman
    which stay symmetric."""
    if win_type == W_RECT or win_type < 0 or win_type > W_TUKEY:
        return np.ones(n, dtype=f32)
    if win_type in (W_BARTLETT, W_TRIANG, W_BARTLETT_HANN, W_BOHMAN):
        return _symmetric_window(win_type, n).astype(f32)
    return _symmetric_window(win_type, n + 1)[:n].astype(f32)


# ---------------------------------------------------------------------------
# STFT  (src/stft_algorithm.c:225-287, 696-803; fft sign src/dsp/fft_algorithm.c:882-891)
# ---------------------------------------------------------------------------
def stft_time_length(L, n, hop, is_pad=False):
    """stft_algorithm.c:225-262."""
    if not is_pad:
        return 0 if L < n else (L - n) // hop + 1
    return 0 if L <= 0 else L // hop + 1


PAD_CENTER, PAD_RIGHT, PAD_LEFT = 0, 1, 2
PAD_CONSTANT, PAD_REFLECT, PAD_WRAP = 0, 1, 2


def stft_pad(x, n, hop, position=PAD_CENTER, mode=PAD_CONSTANT, value1=0.0, value2=0.0):
    """`__stftObj_dealPadData` (stft_algorithm.c:583-694): drop the `L % hop` tail when more than one frame exists,
    then add n samples: n/2 + n/2 (Center), n left (Left), n right (Right) -- a constant (Left/Right: the value is
    passed as `int`, src/vector/flux_vectorOp.c:641-652), the mirror image (== numpy 'reflect', :654-723) or the
    periodic extension (== numpy 'wrap', :736-770); reflect / wrap of fewer than two samples add zeros."""
    x = np.asarray(x, dtype=np.float64)
    L = x.shape[0]
    T = stft_time_length(L, n, hop, True)
    tail = (L % hop) if T > 1 else 0
    v = x[:L - tail]
    left, right = {PAD_CENTER: (n // 2, n - n // 2), PAD_LEFT: (n, 0), PAD_RIGHT: (0, n)}[position]
    if mode == PAD_CONSTANT:
        if position == PAD_CENTER:
            c1, c2 = float(f32(value1)), float(f32(value2))
        else:
            c1 = c2 = float(int(value1))
        return np.concatenate([np.full(left, c1), v, np.full(right, c2)])
    if len(v) < 2:
        return np.concatenate([np.zeros(left), v, np.zeros(right)])
    # numpy's reflect / wrap iterate when the pad is longer than the data, exactly like the reference's index walk
    return np.pad(v, (left, right), mode="reflect" if mode == PAD_REFLECT else "wrap")


def stft(x, n, hop, window, is_pad=False, position=PAD_CENTER, mode=PAD_CONSTANT, value1=0.0, value2=0.0):
    """Full mirrored n-point spectrum per frame -> (re[T,n], im[T,n]).

    is_pad=True: frames are cut from the padded signal of `stft_pad` (default = the centre / constant-zero padding
    CQT uses, stft_algorithm.c:601-694, 813-826)."""
    x = np.asarray(x, dtype=np.float64)
    L = x.shape[0]
    T = stft_time_length(L, n, hop, is_pad)
    if is_pad:
        x = stft_pad(x, n, hop, position, mode, value1, value2)
    if T == 0:
        return np.zeros((0, n), f32), np.zeros((0, n), f32)
    idx = np.arange(T)[:, None] * hop + np.arange(n)[None, :]
    fr = x[idx] * np.asarray(window, dtype=np.float64)[None, :]
    X = np.fft.fft(fr, axis=1)
    return X.real.astype(f32), X.imag.astype(f32)


def istft(re, im, n, hop, window, method_type=0, initial=None):
    """`stftObj_istft` (stft_algorithm.c:304-409): full-spectrum planes (T, n) -> data ((T-1)*hop + n).
    method_type 0 'weight': frames * w, normaliser sum w^2; else 'overlap-add': frames, normaliser sum w;
    normaliser < 1e-6 -> 1.  `initial` = what the caller's buffer held (the reference adds onto it)."""
    X = np.asarray(re, dtype=np.float64) + 1j * np.asarray(im, dtype=np.float64)
    T = X.shape[0]
    w = np.asarray(window, dtype=np.float64)
    y = np.fft.ifft(X, axis=1).real
    e = 1 if method_type == 0 else 0
    L = (T - 1) * hop + n
    out = np.zeros(L) if initial is None else np.asarray(initial, dtype=np.float64).copy()
    norm = np.zeros(L)
    for t in range(T):
        out[t * hop:t * hop + n] += y[t] * w ** e
        norm[t * hop:t * hop + n] += w ** (e + 1)
    norm[norm < 1e-6] = 1.0
    return (out / norm).astype(f32)


# ---------------------------------------------------------------------------
# auditory scales  (src/filterbank/auditory_filterBank.c:1023-1190) -- float32 semantics
# ---------------------------------------------------------------------------
def _fre_to_scale(fre, scale, ref=0.0):
    fre = f32(fre)
    if scale == SCALE_LINEAR:
        return f32(np.round(f32(fre / f32(ref))))          # roundf(fre/detFre)
    if scale == SCALE_LINSPACE:
        return fre
    if scale == SCALE_MEL:
        return f32(f32(2595) * f32(libm.log10f(f32(f32(1) + f32(fre / f32(700))))))        # log10f of the C library, as :1054
    if scale == SCALE_BARK:
        b = 26.81 * float(fre) / float(f32(f32(1960) + fre)) - 0.53    # double expression
        b = f32(b)
        if b < 2:
            b = f32(float(b) + 0.15 * float(f32(f32(2) - b)))
        elif float(b) > 20.1:
            b = f32(float(b) + 0.22 * (float(b) - 20.1))
        return b
    if scale == SCALE_ERB:
        a = f32(21.3654)
        return f32(a * f32(libm.log10f(f32(1.0 + float(fre) * 0.004368))))
    if scale == SCALE_OCTAVE:
        return f32(np.round(f32(float(f32(ref)) * math.log2(float(f32(fre / f32(440)))))))
    if scale == SCALE_LOG:
        return f32(math.log2(float(f32(fre / f32(440)))))
    raise ValueError(scale)


def _scale_to_fre(v, scale, ref=0.0):
    v = f32(v)
    if scale == SCALE_LINEAR:
        return f32(v * f32(ref))
    if scale == SCALE_LINSPACE:
        return v
    if scale == SCALE_MEL:
        return f32(f32(700) * f32(f32(libm.powf(10.0, f32(v / f32(2595)))) - f32(1)))          # powf of the C library, as :1062
    if scale == SCALE_BARK:
        b = v
        if b < 2:
            b = f32((float(b) - 0.3) / 0.85)
        elif float(b) > 20.1:
            b = f32((float(b) + 4.422) / 1.22)
        return f32(1960 * (float(b) + 0.53) / (26.28 - float(b)))
    if scale == SCALE_ERB:
        a = f32(21.3654)
        return f32(float(f32(f32(libm.powf(10.0, f32(v / a))) - f32(1))) / 0.004368)
    if scale == SCALE_OCTAVE:
        return f32(math.pow(2.0, float(f32(v / f32(ref)))) * 440)
    if scale == SCALE_LOG:
        return f32(math.pow(2.0, float(v)) * 440)
    raise ValueError(scale)


def _linspace_f32(start, stop, length):
    """`__vlinspace` type 0 (src/vector/flux_vector.c:2145-2162): start + i*step in float32."""
    start, stop = f32(start), f32(stop)
    step = f32(f32(stop - start) / f32(length - 1 if length - 1 > 0 else 1))
    i = np.arange(length).astype(f32)
    return (start + (i * step).astype(f32)).astype(f32)


def revise_edges(num, low, high, scale, n_fft_or_data, sr, bpo, is_edge):
    """`__revise*Fre` (auditory_filterBank.c:946-1021) applied inside the bank builder."""
    low, high = f32(low), f32(high)
    det, off = (0, 0) if is_edge else (2, 1)
    ref = 0.0
    if scale == SCALE_OCTAVE:
        ref = float(bpo) if 4 <= bpo <= 48 else 12.0
        lo = f32(_fre_to_scale(low, SCALE_OCTAVE, ref) - f32(off))
        hi = f32(lo + f32(num - 1 + det))
        low, high = _scale_to_fre(lo, SCALE_OCTAVE, ref), _scale_to_fre(hi, SCALE_OCTAVE, ref)
    elif scale == SCALE_LINEAR:
        ref = float(f32(sr * 1.0 / n_fft_or_data))
        lo = f32(np.round(f32(low / f32(ref))) - f32(off))
        hi = f32(lo + f32(num - 1 + det))
        low, high = f32(lo * f32(ref)), f32(hi * f32(ref))
    elif scale == SCALE_LINSPACE:
        if not is_edge:
            d = f32(f32(high - low) / f32(num - 1))
            low, high = f32(low - d), f32(high + d)
    elif scale == SCALE_LOG:
        if not is_edge:
            lo = _fre_to_scale(low, SCALE_LOG)
            hi = _fre_to_scale(high, SCALE_LOG)
            d = f32(f32(hi - lo) / f32(num - 1))
            low, high = _scale_to_fre(f32(lo - d), SCALE_LOG), _scale_to_fre(f32(hi + d), SCALE_LOG)
    return low, high, ref


def band_edges(num, n_fft, sr, low, high, scale, ref, is_edge, slaney_bins):
    """`__auditory_calBandEdge` (auditory_filterBank.c:594-677)."""
    det = 0 if is_edge else 2
    lo = _fre_to_scale(low, scale, ref)
    hi = _fre_to_scale(high, scale, ref)
    pts = _linspace_f32(lo, hi, num + det)
    fre = np.array([_scale_to_fre(p, scale, ref) for p in pts], dtype=f32)
    if not slaney_bins:
        bins = np.round((f32(n_fft) * fre).astype(f32) / f32(sr)).astype(np.int64)
    else:
        grid = _linspace_f32(0, f32(f32(sr) - f32(f32(sr) / f32(n_fft))), n_fft)
        bins = np.zeros(num + det, dtype=np.int64)
        for i in range(num + det):
            j = np.nonzero(grid > fre[i])[0]
            bins[i] = j[0] if j.size else 0
    return fre, bins



# ---------------------------------------------------------------------------
# gammatone bank (src/filterbank/auditory_filterBank.c:509-591, coefficients :691-924, response
# src/dsp/filterDesign_freqz.c:8-118): magnitude response of Slaney's four cascaded biquads at the FFT bins.
# The lowest bands are numerically degenerate (the gain and the biquad responses lose most float32 digits to
# cancellation) and the reference's values there are what a float32 evaluation in ITS order with ITS libm produces:
# numpy's own float32 cos/sin/exp differ from glibc's in the last bit and move six of 64 rows by up to 3e-4.  So this
# restatement is float32 operation by operation and takes cosf / sinf / expf / powf from the C library (ctypes); given the
# reference's centre frequencies it reproduces the reference bank bit for bit, and within 5e-6 of a row's maximum from
# its own centre frequencies (tests/test_golden.py, tests/test_oracle_vs_ref.py).
# ---------------------------------------------------------------------------
import ctypes as _C
import ctypes.util as _Cu

_libm = _C.CDLL(_Cu.find_library("m") or "libm.so.6")
for _n in ("cosf", "sinf", "expf", "powf", "log10f"):
    _fn = getattr(_libm, _n)
    _fn.restype = _C.c_float
    _fn.argtypes = [_C.c_float] * (2 if _n == "powf" else 1)


class libm:                                   # float32 in, float32 out, glibc rounding
    cosf = staticmethod(lambda x: _libm.cosf(float(x)))
    sinf = staticmethod(lambda x: _libm.sinf(float(x)))
    expf = staticmethod(lambda x: _libm.expf(float(x)))
    powf = staticmethod(lambda x, y: _libm.powf(float(x), float(y)))
    log10f = staticmethod(lambda x: _libm.log10f(float(x)))


cosf = lambda x: f32(libm.cosf(x))            # noqa: E731
sinf = lambda x: f32(libm.sinf(x))            # noqa: E731
expf = lambda x: f32(libm.expf(x))            # noqa: E731
sqrtf = lambda x: f32(np.sqrt(f32(x)))        # noqa: E731


def gammatone_bank(num, n_fft, sr, norm, fre):
    width=n_fft//2+1
    t=f32(1.0/sr)
    p15=f32(libm.powf(2.0,1.5))
    pv=sqrtf(f32(3)+p15); nv=sqrtf(f32(3)-p15)
    wEnd=f32(2*math.pi); wStep=f32(f32(f32(wEnd-f32(wEnd/f32(n_fft)))-f32(0))/f32(n_fft-1))
    w=(f32(0)+np.arange(width).astype(f32)*wStep).astype(f32)
    # per-bin trig with libm for exactness
    if True:
        c1=np.array([libm.cosf(float(-x)) for x in w],f32); s1=np.array([libm.sinf(float(-x)) for x in w],f32)
        w2=(-w*f32(2)).astype(f32)
        c2=np.array([libm.cosf(float(x)) for x in w2],f32); s2=np.array([libm.sinf(float(x)) for x in w2],f32)
    bank=np.zeros((num,width),f32)
    for i in range(num):
        cf=f32(fre[i])
        bw=f32((float(cf)/9.26449+24.7)*2*math.pi*1.019)
        arg=f32(float(f32(cf*f32(2)))*math.pi*float(t))
        v=f32(-t*expf(f32(-t*bw)))
        cs,sn=cosf(arg),sinf(arg)
        a4=f32(4*math.pi*float(t)*float(cf))
        c2r,c2i=cosf(a4),sinf(a4)
        e1=expf(f32(-bw*t))
        a2=2*math.pi*float(t)*float(cf)
        gr=f32(float(f32(f32(f32(2)*t)*e1))*math.cos(a2)); gi=f32(float(f32(f32(f32(2)*t)*e1))*math.sin(a2))
        den1=f32(f32(f32(-2)*cs)/expf(f32(bw*t))); den2=expf(f32(f32(f32(-2)*t)*bw))
        k=[f32(cs+f32(pv*sn)),f32(cs-f32(pv*sn)),f32(cs+f32(nv*sn)),f32(cs-f32(nv*sn))]
        num1=[f32(v*kk) for kk in k]
        mags=[]
        for s in range(4):
            re=f32(f32(f32(f32(-2)*t)*c2r)+f32(gr*k[s])); im=f32(f32(f32(f32(-2)*t)*c2i)+f32(gi*k[s]))
            mags.append(sqrtf(f32(f32(re*re)+f32(im*im))))
        e2=expf(f32(f32(f32(2)*t)*bw)); e3=expf(f32(t*bw))
        r5=f32(f32(f32(f32(-2)/e2)-f32(f32(2)*c2r))+f32(f32(f32(2)*f32(f32(1)+c2r))/e3))
        i5=f32(f32(f32(-2)*c2i)+f32(f32(f32(2)*c2i)/e3))
        q=f32(f32(r5*r5)+f32(i5*i5))
        gain=f32(f32(f32(f32(mags[0]*mags[1])*mags[2])*mags[3])/f32(q*q))
        sec=[]
        for s in range(4):
            b0=f32(t/gain) if s==0 else t
            b1=f32(num1[0]/gain) if s==0 else num1[s]
            b2=f32(f32(0)/gain) if s==0 else f32(0)
            sec.append((b0,b1,b2,f32(1),den1,den2))
        def poly(c0,c1_,c2_):
            re=np.zeros(width,f32); im=np.zeros(width,f32)
            re=(re+ (np.ones(width,f32)*c0).astype(f32)).astype(f32)   # cos(0)*c0 ; sin(-0)*c0=0 (-0*c0)
            im=(im+ (np.zeros(width,f32)*c0).astype(f32)).astype(f32)
            re=(re+(c1*c1_).astype(f32)).astype(f32); im=(im+(s1*c1_).astype(f32)).astype(f32)
            re=(re+(c2*c2_).astype(f32)).astype(f32); im=(im+(s2*c2_).astype(f32)).astype(f32)
            return re,im
        def cdiv(a,b):
            d=(b[0]*b[0]).astype(f32)+(b[1]*b[1]).astype(f32); d=d.astype(f32)
            return (((a[0]*b[0]).astype(f32)+(a[1]*b[1]).astype(f32)).astype(f32)/d).astype(f32), (((a[1]*b[0]).astype(f32)-(a[0]*b[1]).astype(f32)).astype(f32)/d).astype(f32)
        def cmul(a,b):
            return ((a[0]*b[0]).astype(f32)-(a[1]*b[1]).astype(f32)).astype(f32), ((a[0]*b[1]).astype(f32)+(a[1]*b[0]).astype(f32)).astype(f32)
        h=cdiv(poly(*sec[0][:3]),poly(*sec[0][3:]))
        for s in range(1,4): h=cmul(h,cdiv(poly(*sec[s][:3]),poly(*sec[s][3:])))
        row=np.sqrt(((h[0]*h[0]).astype(f32)+(h[1]*h[1]).astype(f32)).astype(f32)).astype(f32)
        if norm in (1,2):
            if norm==1:
                inner=f32(0)
                for j in range(1,width-1): inner=f32(inner+row[j])
                wt=f32(row[0]+row[width-1]); wt=f32(wt+f32(inner*f32(2)))
            else:
                wt=f32(1.019*24.7*(0.00437*float(fre[i])+1)); wt=f32(wt/f32(2))
            row=np.where(row!=0,(row/wt).astype(f32),row)
        row[1:width-1]=(row[1:width-1]*f32(2)).astype(f32)
        bank[i]=row
    return bank

def auditory_filterbank(num, n_fft, sr, scale=SCALE_MEL, style=STYLE_SLANEY, norm=NORM_NONE,
                        low=0.0, high=None, bpo=12):
    """`auditory_filterBank` (auditory_filterBank.c:56-207) for the Slaney / ETSI / window styles and gammatone.

    Returns (bank[num, n_fft/2+1] float32, fre_band[num], bin_band[num])."""
    if high is None:
        high = sr / 2.0
    if style == STYLE_GAMMATONE:                   # the num points are the centre frequencies themselves (isEdge = 1)
        lo_g, hi_g, ref_g = revise_edges(num, low, high, scale, n_fft, sr, bpo, is_edge=True)
        fre_g, bins_g = band_edges(num, n_fft, sr, lo_g, hi_g, scale, ref_g, True, False)
        return gammatone_bank(num, n_fft, sr, norm, fre_g), fre_g.astype(f32), bins_g
    m = n_fft // 2 + 1
    low, high, ref = revise_edges(num, low, high, scale, n_fft, sr, bpo, is_edge=False)
    fre, bins = band_edges(num, n_fft, sr, low, high, scale, ref, False, style == STYLE_SLANEY)
    bank = np.zeros((num, m), dtype=np.float64)
    fre64 = fre.astype(np.float64)
    if scale == SCALE_LINEAR:                      # :339-365
        bins = bins.copy()
        for i in range(1, num + 1):
            bins[i] -= 1
            bank[i - 1, bins[i]] = 1.0
    elif style == STYLE_SLANEY:                    # :435-500, triangles in Hz
        grid = _linspace_f32(0, f32(f32(sr) - f32(f32(sr) / f32(n_fft))), n_fft).astype(np.float64)
        w = (fre[1:] - fre[:-1]).astype(f32).astype(np.float64)
        for i in range(num):
            for j in range(bins[i], bins[i + 1]):
                bank[i, j] = f32(f32(f32(grid[j]) - fre[i]) / f32(w[i]))
            for j in range(bins[i + 1], bins[i + 2]):
                bank[i, j] = f32(f32(fre[i + 2] - f32(grid[j])) / f32(w[i + 1]))
    elif style == STYLE_ETSI:                      # :373-426, triangles in bins
        for i in range(1, num + 1):
            l, c, r = bins[i - 1], bins[i], bins[i + 1]
            if c > l:
                for j in range(l, c + 1):
                    bank[i - 1, j] = (j - l) / (c - l)
            for j in range(c + 1, r + 1):
                bank[i - 1, j] = (r - j) / (r - c)
    elif style == STYLE_POINT:                     # :229-237
        for i in range(1, num + 1):
            bank[i - 1, bins[i]] = 1.0
    elif style == STYLE_RECT:                      # :238-248
        for i in range(1, num + 1):
            bank[i - 1, bins[i - 1]:bins[i + 1] + 1] = 1.0
    else:                                          # window-design styles :249-316
        kind = {STYLE_HANN: W_HANN, STYLE_HAMM: W_HAMM, STYLE_BLACKMAN: W_BLACKMAN,
                STYLE_BOHMAN: W_BOHMAN, STYLE_KAISER: W_KAISER}.get(style, W_GAUSS)
        for i in range(1, num + 1):
            l, c, r = bins[i - 1], bins[i], bins[i + 1]
            if c > l:
                w = _symmetric_window(kind, 2 * (c - l) + 1)
                bank[i - 1, l:c + 1] = w[:c - l + 1]
            if r > c:
                w = _symmetric_window(kind, 2 * (r - c) + 1)
                k0 = (2 * (r - c) + 1) // 2 + 1
                bank[i - 1, c + 1:r + 1] = w[k0:k0 + (r - c)]
    bank = bank.astype(f32)
    if scale != SCALE_LINEAR and norm in (NORM_AREA, NORM_BANDWIDTH):   # :479-496
        if norm == NORM_AREA:
            wt = bank.astype(np.float64).sum(axis=1)
        else:
            wt = (fre64[2:] - fre64[:-2]) / 2.0
        with np.errstate(divide="ignore", invalid="ignore"):   # `__mdiv_vector` keeps exact zeros (flux_vector.c:289-308)
            bank = np.where(bank != 0, bank / wt[:, None].astype(f32), f32(0)).astype(f32)
    return bank, fre[1:num + 1].copy(), bins[1:num + 1].astype(np.int32)


# ---------------------------------------------------------------------------
# BFT  (src/bft_algorithm.c:87-276 defaults, 397-540 compute)
# ---------------------------------------------------------------------------
def bft_revise_range(num, n_fft, sr, low, high, scale, bpo):
    """Range defaults/revisions done in `bftObj_new` (bft_algorithm.c:158-230)."""
    lo = f32(0.0)
    hi = f32(sr / 2.0)
    if low is not None and 0 <= low < sr / 2.0:
        lo = f32(low)
    if lo == 0 and scale in (SCALE_OCTAVE, SCALE_LOG):
        lo = f32(f32(math.pow(2.0, float(f32(-45 / 12.0)))) * f32(440))
        hi = f32(f32(math.pow(2.0, float(f32(38 / 12.0)))) * f32(440))
    if high is not None and 0 < high <= sr / 2.0:
        hi = f32(high)
    if hi < lo:
        lo, hi = f32(0.0), f32(sr / 2.0)
        if scale in (SCALE_OCTAVE, SCALE_LOG):
            lo = f32(f32(math.pow(2.0, float(f32(-45 / 12.0)))) * f32(440))
            hi = f32(f32(math.pow(2.0, float(f32(38 / 12.0)))) * f32(440))
    low_idx = high_idx = 0
    if scale == SCALE_LINEAR:
        det = f32(f32(sr) / f32(n_fft))
        l2 = f32(np.round(f32(lo / det)))
        h2 = f32(l2 + f32(num - 1))
        lo, hi = f32(l2 * det), f32(h2 * det)
        low_idx, high_idx = int(np.round(f32(lo / det))), int(np.round(f32(hi / det)))
    elif scale == SCALE_OCTAVE:
        l2 = _fre_to_scale(lo, SCALE_OCTAVE, float(bpo))
        h2 = f32(l2 + f32(num - 1))
        lo, hi = _scale_to_fre(l2, SCALE_OCTAVE, float(bpo)), _scale_to_fre(h2, SCALE_OCTAVE, float(bpo))
    return lo, hi, low_idx, high_idx


def bft(x, num, radix2_exp, sr, hop=None, window_type=W_HANN, scale=SCALE_MEL, style=STYLE_SLANEY,
        norm=NORM_NONE, data_type=DATA_POWER, low=None, high=None, bpo=12, result_type=1,
        norm_value=1.0, bank=None):
    """`bftObj_bft` (bft_algorithm.c:397-540).  result_type 1 -> real (T,num);
    0 -> (re, im) each (T,num)."""
    n = 1 << radix2_exp
    hop = n // 4 if hop is None or hop <= 0 else hop
    lo, hi, low_idx, high_idx = bft_revise_range(num, n, sr, low, high, scale, bpo)
    if bank is None and scale != SCALE_LINEAR:
        bank, _, _ = auditory_filterbank(num, n, sr, scale, style, norm, lo, hi, bpo)
    re, im = stft(x, n, hop, fft_window(window_type, n))
    re = re[:, :n // 2 + 1].astype(np.float64)
    im = im[:, :n // 2 + 1].astype(np.float64)
    if result_type == 0:                                    # :457-486
        if data_type == DATA_POWER:
            re, im = re * re - im * im, 2 * re * im
        if scale == SCALE_LINEAR:
            return re[:, low_idx:high_idx + 1].astype(f32), im[:, low_idx:high_idx + 1].astype(f32)
        B = bank.astype(np.float64)
        return (re @ B.T).astype(f32), (im @ B.T).astype(f32)
    p = re * re + im * im                                   # :488-529
    if data_type == DATA_MAG:
        p = np.sqrt(p)
    elif norm_value != 1:
        p = np.power(p, norm_value)
    if scale == SCALE_LINEAR:
        out = p[:, low_idx:high_idx + 1]
    else:
        out = p.astype(f32).astype(np.float64) @ bank.astype(np.float64).T
    if data_type == DATA_MAG and norm_value != 1:
        out = np.power(out, norm_value)
    return out.astype(f32)


# ---------------------------------------------------------------------------
# xxcc  (src/feature/xxcc_algorithm.c:95-156; DCT src/dsp/fft_algorithm.c:625-674,
#        src/dsp/dct_algorithm.c:81-110)
# ---------------------------------------------------------------------------
def dct2_ortho_matrix(num):
    k = np.arange(num)[:, None]
    j = np.arange(num)[None, :]
    C = np.cos(np.pi * (j + 0.5) * k / num)
    s = np.full((num, 1), math.sqrt(2.0 / num))
    s[0, 0] = math.sqrt(1.0 / num)
    return C * s


def xxcc(m, cc_num, rectify=RECT_LOG):
    m = np.asarray(m, dtype=f32)
    T, num = m.shape
    if cc_num > num:
        return None
    if rectify == RECT_CUBIC:
        r = np.power(m.astype(np.float64), 1.0 / 3)
    else:
        r = np.log10(np.maximum(m, f32(1e-8)).astype(np.float64))
    return (r.astype(f32).astype(np.float64) @ dct2_ortho_matrix(num)[:cc_num].T).astype(f32)


# ---------------------------------------------------------------------------
# down-by-2 resampler used inside CQT (src/dsp/resample_algorithm.c:350-403, 430-521, 546-634)
# ---------------------------------------------------------------------------
def decimator_taps():
    """Quality 'Fast': 16 zero crossings, 512 samples per crossing, Kaiser beta 8.5555046,
    roll-off 0.85, scaled by ratio 0.5 -> taps interp[256*j].  32 left taps (j=0..31) and
    31 right taps (j=0..30, applied to x[n+1+j]) because of the integer division
    (interpLength-offset)/step with offset 0 (left) / 256 (right)."""
    zero_num, bit_len = 16, 512
    L = zero_num * bit_len + 1
    t = np.linspace(0, zero_num, L) * 0.85
    sinc = np.where(t == 0, 1.0, np.sin(np.pi * t) / np.where(t == 0, 1.0, np.pi * t)) * 0.85
    win = _symmetric_window(W_KAISER, 2 * (L - 1) + 1, 8.5555046)[L - 1:]
    interp = sinc * win * 0.5
    left = interp[0:L:256][:32]            # offset 0: (8193-0)//256 = 32 taps
    right = interp[256:L:256][:31]         # offset 256: (8193-256)//256 = 31 taps
    return left.astype(f32), right.astype(f32)


def resample_down2(x):
    x = np.asarray(x, dtype=np.float64)
    L = x.shape[0]
    out_len = L // 2
    left, right = decimator_taps()
    left = left.astype(np.float64)
    right = right.astype(np.float64)
    xp = np.concatenate([np.zeros(32), x, np.zeros(64)])
    n = 2 * np.arange(out_len) + 32
    y = np.zeros(out_len)
    for j in range(32):
        y += left[j] * xp[n - j]
    for j in range(31):
        y += right[j] * xp[n + 1 + j]
    return (y / math.sqrt(0.5)).astype(f32)


# ---------------------------------------------------------------------------
# CQT  (src/cqt_algorithm.c:123-247, 845-1061, 1181-1265; src/filterbank/cqt_filterBank.c)
# ---------------------------------------------------------------------------
def cqt_fre_arr(min_fre, num, bpo):
    """cqt_filterBank.c:159-184 (float32 running product)."""
    arr = np.zeros(num, dtype=f32)
    v = f32(math.pow(2.0, float(f32(1.0 / bpo))))      # powf, correctly rounded
    for i in range(num // bpo):
        f = f32(f32(min_fre) * f32(1 << i))
        arr[i * bpo] = f
        for j in range(1, bpo):
            f = f32(f * v)
            arr[i * bpo + j] = f
    return arr


def cqt_len_arr(fre, sr, bpo, factor=1.0, beta=0.0):
    """cqt_filterBank.c:187-213."""
    value = f32(f32(math.pow(2.0, float(f32(1.0 / bpo)))) - f32(1))
    q = f32(f32(factor) / value)
    return np.array([f32(f32(q * f32(sr)) / f32(f + f32(f32(beta) / value))) for f in fre], dtype=f32)


def _ceil_pow2(v):
    p = 1
    while p < v:
        p <<= 1
    return p


def cqt_kernel_bank(num, sr, min_fre=32.703196, bpo=12, factor=1.0, beta=0.0, thresh=0.01,
                    win_type=W_HANN, norm=NORM_NONE):
    """Spectral kernels (cqt_algorithm.c:1181-1265, cqt_filterBank.c:57-148, 253-336): the top octave's `bpo` rows,
    shared by all octaves -- or, beta != 0 (VQT, vFlag), `num` rows: every octave's rows from its own float
    frequencies and the integer-halved sample rate, all with the TOP octave's kernel lengths.

    Returns dict(fft_length, fre, slen(sqrt lengths), kr, ki, vqt) with kr/ki [rows, n/2+1]."""
    octs = num // bpo
    fre = cqt_fre_arr(min_fre, num, bpo)
    top = fre[(octs - 1) * bpo:]
    value = f32(f32(math.pow(2.0, float(f32(1.0 / bpo)))) - f32(1))
    q = f32(f32(factor) / value)
    n = _ceil_pow2(int(np.ceil(f32(f32(q * f32(sr)) / f32(top[0] + f32(f32(beta) / value))))))
    len_top = cqt_len_arr(top, sr, bpo, factor, beta)
    slen = np.sqrt(cqt_len_arr(fre, sr, bpo, factor, beta)).astype(f32)
    wt = win_type if win_type != W_RECT else W_HANN
    vqt = beta != 0
    rows = num if vqt else bpo
    kr = np.zeros((rows, n // 2 + 1), dtype=f32)
    ki = np.zeros((rows, n // 2 + 1), dtype=f32)
    full = np.concatenate([fre, [0.0, 0.0]])
    sr_oct = int(sr)
    for octv in range(octs - 1, (0 if vqt else octs - 1) - 1, -1):
        for i in range(bpo):
            f_bin = fre[octv * bpo + i]
            ln = int(np.ceil(len_top[i]))
            w = fft_window(wt, ln).astype(np.float64)
            j = np.arange(ln, dtype=np.float64)
            ph = 2 * np.pi * j * float(f_bin) / sr_oct
            weight = float(len_top[i]) if norm == NORM_NONE else 1.0
            tr = np.cos(ph) * w / weight
            ti = np.sin(ph) * w / weight
            if norm == NORM_AREA:
                s = np.sqrt(tr * tr + ti * ti).sum()
                tr, ti = tr / s, ti / s
            elif norm == NORM_BANDWIDTH:
                k = octv * bpo + i
                bw = (float(full[k + 1]) - float(full[k - 1] if k > 0 else 0.0)) / 2
                tr, ti = tr / bw, ti / bw
            tr = tr * (float(len_top[i]) / n)
            ti = ti * (float(len_top[i]) / n)
            buf = np.zeros(n, dtype=np.complex128)
            st = (n - ln) // 2
            buf[st:st + ln] = tr + 1j * ti
            K = np.fft.fft(buf)[:n // 2 + 1]
            keep = (K.real.astype(f32).astype(np.float64) ** 2 + K.imag.astype(f32).astype(np.float64) ** 2) > float(f32(thresh) * f32(thresh))
            row = octv * bpo + i if vqt else i
            kr[row] = np.where(keep, K.real, 0).astype(f32)
            ki[row] = np.where(keep, K.imag, 0).astype(f32)
        sr_oct //= 2
    return dict(fft_length=n, fre=fre, slen=slen, kr=kr, ki=ki, octs=octs, vqt=vqt)


def cqt(x, num=84, sr=32000, min_fre=32.703196, bpo=12, factor=1.0, beta=0.0, thresh=0.01,
        win_type=W_HANN, hop=None, norm=NORM_NONE, is_scale=True, bank=None, is_continue=False):
    """`cqtObj_cqt` (cqt_algorithm.c:463-478, 845-1061) -> (re, im) [T, num].  is_continue: the streaming variant run on
    the assembled samples -- frames start at t * hop (right zero padding, :1317-1319) and only the whole frames of the
    full-rate signal count, T = (L - n) / hop + 1 (:923-928)."""
    if bank is None:
        bank = cqt_kernel_bank(num, sr, min_fre, bpo, factor, beta, thresh, win_type, norm)
    n, octs, slen = bank["fft_length"], bank["octs"], bank["slen"].astype(np.float64)
    K = bank["kr"].astype(np.float64) + 1j * bank["ki"].astype(np.float64)
    hop = n // 4 if hop is None or hop <= 0 else hop
    x = np.asarray(x, dtype=f32)
    L = x.shape[0]
    T = L // hop + 1 if not is_continue else ((L - n) // hop + 1 if L >= n else 0)
    out = np.zeros((T, num), dtype=np.complex128)
    cur = x
    rect = np.ones(n)
    for o in range(octs - 1, -1, -1):
        k = octs - 1 - o
        if k > 0:
            cur = resample_down2(cur)
            hop //= 2
        re, im = stft(cur, n, hop, rect, is_pad=True, position=PAD_RIGHT if is_continue else PAD_CENTER)
        S = (re[:, :n // 2 + 1].astype(np.float64) + 1j * im[:, :n // 2 + 1].astype(np.float64))
        Tn = min(T, S.shape[0])
        Ko = K[o * bpo:(o + 1) * bpo] if bank.get("vqt") else K
        v = S[:Tn] @ Ko.T
        v = v * math.sqrt(float(1 << k)) if k > 0 else v
        if is_scale:
            v = v / slen[None, o * bpo:(o + 1) * bpo]
        out[:Tn, o * bpo:(o + 1) * bpo] = v
    return out.real.astype(f32), out.imag.astype(f32)


# ---------------------------------------------------------------------------
# CWT  (src/cwt_algorithm.c:73-334, 361-483; src/filterbank/cwt_filterBank.c:85-290, 361-640)
# ---------------------------------------------------------------------------
_WAVE_DEFAULTS = {WAVE_MORSE: (3.0, 20.0), WAVE_MORLET: (6.0, 2.0), WAVE_BUMP: (5.0, 0.6),
                  WAVE_PAUL: (4.0, 20.0), WAVE_DOG: (2.0, 2.0), WAVE_MEXICAN: (3.0, 2.0),
                  WAVE_HERMIT: (5.0, 2.0), WAVE_RICKER: (4.0, 20.0)}


def cwt_revise_range(num, n, sr, low, high, scale, bpo):
    """Range handling in `cwtObj_new` (cwt_algorithm.c:137-196): same rules as BFT."""
    lo, hi, _, _ = bft_revise_range(num, n, sr, low, high, scale, bpo)
    return lo, hi


def cwt_filterbank(num, n, sr, wavelet=WAVE_MORLET, scale=SCALE_OCTAVE, low=None, high=None, bpo=12,
                   gamma=None, beta=None, pad_length=0):
    """`cwt_filterBank` (cwt_filterBank.c:85-290).  Returns (bank[num, n+2*pad] f32, fre_band[num])."""
    g0, b0 = _WAVE_DEFAULTS[wavelet]
    gamma = g0 if gamma is None or gamma <= 0 else gamma
    beta = b0 if beta is None or beta <= 0 else beta
    if wavelet == WAVE_DOG:
        p = int(np.round(gamma))
        gamma = float(p) if p % 2 == 0 else 2.0
    lo, hi = cwt_revise_range(num, n, sr, low, high, scale, bpo)
    lo, hi, ref = revise_edges(num, lo, hi, scale, n, sr, bpo, is_edge=False)
    fre, _ = band_edges(num, n, sr, lo, hi, scale, ref, False, False)
    if wavelet == WAVE_MORSE:
        cf = float(f32(np.exp(f32(1.0 / gamma * float(f32(np.log(f32(beta)) - np.log(f32(gamma))))))))
    elif wavelet in (WAVE_MORLET, WAVE_BUMP, WAVE_RICKER):
        cf = gamma
    elif wavelet == WAVE_PAUL:
        cf = gamma + 0.5
    elif wavelet == WAVE_DOG:
        cf = math.sqrt(gamma + 0.5)
    elif wavelet == WAVE_MEXICAN:
        cf = math.sqrt(2.5)
    else:
        cf = gamma + 1
    wl = n + 2 * pad_length
    w = np.zeros(wl)
    half = wl // 2
    w[:half + 1] = np.arange(half + 1) * 2 * np.pi / wl
    for i, j in zip(range(half + 1, wl), range(half - 1, -1, -1)):
        w[i] = -w[j]
    w = w.astype(f32).astype(np.float64)
    fsel = np.maximum(fre[1:num + 1][::-1].astype(np.float64), 1e-6)
    s = (cf / (fsel / sr * 2 * np.pi)).astype(f32).astype(np.float64)
    sw = (s[:, None] * w[None, :]).astype(f32).astype(np.float64)
    pos = sw > 0
    swp = np.where(pos, sw, 1.0)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        if wavelet == WAVE_MORSE:
            fac = math.exp(-beta * math.log(cf) + cf ** gamma)
            bank = np.where(pos, 2 * fac * np.exp(beta * np.log(swp) - swp ** gamma), 0.0)
        elif wavelet == WAVE_MORLET:
            bank = np.where(pos, 2 * np.exp(-(swp - gamma) ** 2 / beta), 0.0)
        elif wavelet == WAVE_BUMP:
            v1 = (sw - gamma) / beta
            v2 = -1.0 / (1 - v1 * v1)
            bank = np.where(np.abs(v1) < 1 - 1e-6, 2 * math.e * np.exp(v2), 0.0)
            bank = np.nan_to_num(bank, nan=0.0)
        elif wavelet == WAVE_PAUL:
            p = int(np.round(gamma))
            prod = 1.0
            for i in range(2 * p - 1, 1, -1):
                prod *= i
            fac = 2.0 ** p / math.sqrt(p * prod)
            bank = np.where(pos, fac * swp ** gamma * np.exp(-swp), 0.0)
        elif wavelet in (WAVE_DOG, WAVE_MEXICAN):
            g = 2.0 if wavelet == WAVE_MEXICAN else gamma
            p = int(np.round(g))
            fac = -1.0 / math.sqrt(math.gamma(p + 0.5))
            if (p // 2) % 2 == 1:
                fac = -fac
            bank = np.where(pos, fac * swp ** g * np.exp(-swp * swp / beta), 0.0)
        elif wavelet == WAVE_HERMIT:
            fac = 2.0 / math.sqrt(gamma) * math.pi ** -0.25
            d = swp - gamma
            bank = np.where(pos, fac * d * (1 + d) * np.exp(-d * d / beta), 0.0)
        else:  # ricker
            fac = 2.0 / math.sqrt(math.pi)
            bank = np.where(pos, fac * swp * swp / gamma ** 3 * np.exp(-swp * swp / (gamma * gamma)), 0.0)
    return bank.astype(f32), fre[1:num + 1].copy()


def cwt(x, num=84, radix2_exp=12, sr=32000, wavelet=WAVE_MORLET, scale=SCALE_OCTAVE, low=None,
        high=None, bpo=12, gamma=None, beta=None, is_pad=False, bank=None, det=False):
    """`cwtObj_cwt` (cwt_algorithm.c:346-350, 361-483) -> (re, im) [num, N]; row 0 = highest band.
    det=True: `cwtObj_cwtDet` (:352-358, 485-528): the bank is multiplied by omega_k (float32: 2 pi k / L for k <= L/2,
    mirrored negative above) and by j before the inverse transform."""
    N = 1 << radix2_exp
    x = np.asarray(x, dtype=np.float64)[:N]
    pad = 0
    if is_pad:
        pad = N // 2 if N <= 1e5 else int(math.ceil(math.log2(N)))
    if bank is None:
        bank, _ = cwt_filterbank(num, N, sr, wavelet, scale, low, high, bpo, gamma, beta, pad)
    if pad:
        x = np.concatenate([x[:pad][::-1], x, x[N - pad:][::-1]])
    X = np.fft.fft(x)
    B = bank.astype(np.float64)
    if det:
        Lf = B.shape[1]
        w = np.zeros(Lf, f32)
        w[:Lf // 2 + 1] = (np.arange(Lf // 2 + 1) * 2 * math.pi / Lf).astype(f32)
        w[Lf // 2 + 1:] = -w[Lf // 2 - 1:0:-1][:Lf - Lf // 2 - 1]
        B = (bank * w[None, :]).astype(f32).astype(np.float64) * 1j
    y = np.fft.ifft(B * X[None, :], axis=1)
    if pad:
        y = y[:, pad:pad + N]
    return y.real.astype(f32), y.imag.astype(f32)


# ---------------------------------------------------------------------------
# convenience: the benchmark path (BFT mel power, result_type=1 -> xxcc)
# ---------------------------------------------------------------------------
def mfcc(x, sr=48000, radix2_exp=11, hop=512, n_mels=128, cc_num=40, norm=NORM_NONE, bank=None):
    m = bft(x, n_mels, radix2_exp, sr, hop, W_HANN, SCALE_MEL, STYLE_SLANEY, norm, DATA_POWER,
            result_type=1, bank=bank)
    return xxcc(m, cc_num, RECT_LOG)


# ---------------------------------------------------------------------------
# SURVEY section 8(f) rows: xxccStandard, CQT chroma / cqcc, SpectrogramObj front door
# ---------------------------------------------------------------------------
ENERGY_REPLACE, ENERGY_APPEND, ENERGY_IGNORE = 0, 1, 2
CHROMA_NORM_NONE, CHROMA_NORM_MAX, CHROMA_NORM_MIN, CHROMA_NORM_P2, CHROMA_NORM_P1 = range(5)


def delta_fir(x, order):
    """`util_delta` (src/util/flux_util.c:803-815): causal FIR with taps b[j] = (m - j) / sum_{i<=m} i^2,
    j = 0..order-1, m = order//2 (`filterDesign_smooth1`, src/dsp/filterDesign_fir.c:194-217, run through
    `filterDesign_filter`, :229-248, with the first `order` taps), along the LAST axis."""
    x = np.asarray(x, dtype=np.float64)
    m = order // 2
    v1 = float(sum(i * i for i in range(1, m + 1)))
    b = np.array([(m - j) / v1 for j in range(order)])
    y = np.zeros_like(x)
    n = x.shape[-1]
    for j in range(min(order, n)):
        y[..., j:] += b[j] * x[..., :n - j]
    return y


def xxcc_standard(m, energy, cc_num, delta_window_length=9, energy_type=ENERGY_REPLACE, rectify=RECT_LOG):
    """`xxccObj_xxccStandard` (src/feature/xxcc_algorithm.c:168-296) -> (coe, delta, delta2), each (T, W).
    The delta FIR runs along the coefficient axis of each frame, as the reference does."""
    order = delta_window_length if (delta_window_length >= 3 and delta_window_length % 2 == 1) else 9
    cc = xxcc(m, cc_num, rectify).astype(np.float64)
    if energy_type != ENERGY_IGNORE:
        e = np.log(np.maximum(np.asarray(energy, dtype=f32), f32(1e-8)).astype(np.float64))
    if energy_type == ENERGY_REPLACE:
        coe = cc.copy()
        coe[:, 0] = e
    elif energy_type == ENERGY_APPEND:
        coe = np.concatenate([e[:, None], cc], axis=1)
    else:
        coe = cc
    coe = coe.astype(f32)
    d1 = delta_fir(coe, order).astype(f32)
    d2 = delta_fir(d1, order).astype(f32)
    return coe, d1, d2


def chroma_cqt_bank(num, cqt_length, bpo=12, min_fre=32.703196):
    """`chroma_cqtFilterBank` (src/filterbank/chroma_filterBank.c:176-262): 0/1 matrix (num, cqt_length)."""
    if num > bpo or bpo % num != 0:
        return None
    n = bpo // num
    offset = int(math.ceil(n / 2.0))
    sub = n - offset
    arr = np.zeros((num, cqt_length), f32)
    j = np.arange(cqt_length) % bpo
    arr[0, (j < offset) | ((sub > 0) & (j >= bpo - sub))] = 1
    for i in range(1, num):
        start = offset + (i - 1) * n
        arr[i, (j >= start) & (j < start + n)] = 1
    midi = int(np.round(f32(12 * math.log2(float(f32(f32(min_fre) / f32(440)))) + 69))) % 12
    if midi > 6:
        midi = 12 - midi
    shift = midi * (num // bpo)
    return np.roll(arr, -shift, axis=0) if shift else arr


def cqt_chroma(re, im, chroma_num=12, data_type=DATA_POWER, norm=CHROMA_NORM_MAX, bpo=12, min_fre=32.703196):
    """`cqtObj_chroma` (src/cqt_algorithm.c:484-600); normalisation `__mnormalize` axis 1
    (src/vector/flux_vector.c:1058-1150)."""
    re = np.asarray(re, dtype=np.float64)
    im = np.asarray(im, dtype=np.float64)
    s = (re * re + im * im).astype(f32).astype(np.float64)
    if data_type == DATA_MAG:
        s = np.sqrt(s).astype(f32).astype(np.float64)
    bank = chroma_cqt_bank(chroma_num, re.shape[1], bpo, min_fre).astype(np.float64)
    out = (s @ bank.T).astype(f32).astype(np.float64)
    if norm != CHROMA_NORM_NONE:
        a = np.abs(out)
        if norm == CHROMA_NORM_MAX:
            v = a.max(axis=1)
        elif norm == CHROMA_NORM_MIN:
            v = a.min(axis=1)
        elif norm == CHROMA_NORM_P2:
            v = np.sqrt((a * a).sum(axis=1))
        else:
            v = a.sum(axis=1)
        v = v.astype(f32).astype(np.float64)
        nz = v != 0
        out[nz] = out[nz] / v[nz, None]
    return out.astype(f32)


def spectrogram_params(num, sr=32000, low=None, high=None, bpo=12, radix2_exp=12, scale=SCALE_LINEAR):
    """Parameter rules of `spectrogramObj_new` (src/spectrogram_algorithm.c:326-583) for the scale types on
    the path -> dict(num, low, high, low_idx, high_idx, bpo)."""
    n = 1 << radix2_exp
    if bpo is None or bpo <= 0 or bpo % 12 != 0:
        bpo = 12
    if scale == SCALE_LINEAR:
        lo, hi = f32(0.0), f32(sr / 2.0)
        if low is not None and 0 <= low < sr / 2.0:
            lo = f32(low)
        if high is not None and 0 < high <= sr / 2.0:
            hi = f32(high)
        if hi < lo:
            lo, hi = f32(0.0), f32(sr / 2.0)
        det = f32(f32(sr) / f32(n))
        li, hj = int(np.round(f32(lo / det))), int(np.round(f32(hi / det)))
        return dict(num=hj - li + 1, low=lo, high=hi, low_idx=li, high_idx=hj, bpo=bpo)
    lo, hi, _, _ = bft_revise_range(num, n, sr, low, high, scale, bpo)
    return dict(num=num, low=lo, high=hi, low_idx=0, high_idx=0, bpo=bpo)


def spectrogram(x, num=0, sr=32000, low=None, high=None, bpo=12, radix2_exp=12, window_type=W_HANN, hop=None,
                data_type=DATA_POWER, scale=SCALE_LINEAR, style=STYLE_SLANEY, norm=NORM_NONE, norm_value=1.0,
                want_phase=False, bank=None):
    """`spectrogramObj_spectrogram` (src/spectrogram_algorithm.c:864-1395) -> spec (T, bandNum)
    [, phase (T, bandNum), Linear scale only: atan2f(im, max(re, 1e-16)), :1040-1056]."""
    n = 1 << radix2_exp
    hop = n // 4 if hop is None or hop <= 0 else hop
    p = spectrogram_params(num, sr, low, high, bpo, radix2_exp, scale)
    re, im = stft(x, n, hop, fft_window(window_type, n))
    re = re[:, :n // 2 + 1].astype(np.float64)
    im = im[:, :n // 2 + 1].astype(np.float64)
    s = re * re + im * im
    if data_type == DATA_MAG:
        s = np.sqrt(s)
    elif norm_value != 1:
        s = np.power(s, norm_value)
    if scale == SCALE_LINEAR:
        out = s[:, p["low_idx"]:p["high_idx"] + 1]
    else:
        if bank is None:
            bank, _, _ = auditory_filterbank(p["num"], n, sr, scale, style, norm, p["low"], p["high"], p["bpo"])
        out = s.astype(f32).astype(np.float64) @ bank.astype(np.float64).T
    if data_type == DATA_MAG and norm_value != 1:
        out = np.power(out, norm_value)
    out = out.astype(f32)
    if not want_phase or scale != SCALE_LINEAR:
        return out
    r = re[:, p["low_idx"]:p["high_idx"] + 1].astype(f32)
    i = im[:, p["low_idx"]:p["high_idx"] + 1].astype(f32)
    phase = np.arctan2(i, np.where(r < f32(1e-16), f32(1e-16), r)).astype(f32)
    return out, phase


def spectrogram_linear_bands(sr, radix2_exp, low_idx, num):
    """`__spectrogramObj_calLinearBandArr` (src/spectrogram_algorithm.c:1909-1941)."""
    n = 1 << radix2_exp
    grid = _linspace_f32(f32(0), f32(sr / 2.0), n // 2 + 1)
    return grid[low_idx:low_idx + num].copy(), np.arange(low_idx, low_idx + num, dtype=np.int32)


def pwt(x, num=84, radix2_exp=12, sr=32000, low=None, high=None, bpo=12, scale=SCALE_OCTAVE, style=STYLE_SLANEY,
        norm=NORM_NONE, is_pad=False, det=False):
    """`pwtObj_pwt` / `pwtObj_pwtDet` (src/pwt_algorithm.c:63-348, 392-520): the CWT structure with the auditory bank of
    `auditory_filterBank(isPseudo=1)` (rows of fftLength entries, zero above fftLength/2) built for the PADDED length.
    Range rules = `bft_revise_range` with the unpadded length (:135-195)."""
    N = 1 << radix2_exp
    lo, hi, _, _ = bft_revise_range(num, N, sr, low, high, scale, bpo)
    pad = 0
    if is_pad:
        pad = N // 2 if N <= 1e5 else int(math.ceil(math.log2(N)))
    Lf = N + 2 * pad
    half, fre, bins = auditory_filterbank(num, Lf, sr, scale, style, norm, float(lo), float(hi), bpo)
    bank = np.zeros((num, Lf), f32)
    bank[:, :Lf // 2 + 1] = half
    re, im = cwt(x, num, radix2_exp, sr, is_pad=is_pad, bank=bank, det=det)
    return re, im, fre, bins


# ---------------------------------------------------------------------------
# Synchrosqueezing: WSST (src/wsst_algorithm.c:64-352) and Synsq (src/synsq_algorithm.c:38-300)
# ---------------------------------------------------------------------------
def _complex_div(ar, ai, br, bi):
    """__complexDiv (src/vector/flux_complex.c): (ar + i ai) / (br + i bi), float32 arithmetic"""
    ar, ai, br, bi = (np.asarray(v, dtype=f32) for v in (ar, ai, br, bi))
    with np.errstate(divide="ignore", invalid="ignore"):
        den = (br * br + bi * bi).astype(f32)
        re = ((ar * br + ai * bi).astype(f32) / den).astype(f32)
        im = ((ai * br - ar * bi).astype(f32) / den).astype(f32)
    return re, im


def squeeze_index(inst_fre, fre_arr, sr, scale, num):
    """row index of an instantaneous frequency (cycles / sample): wsst_algorithm.c:268-296, synsq_algorithm.c:167-193.
    Octave / Log: round((log2|f| - log2 fmin) num / (log2 fmax - log2 fmin)); Linear / Linspace: round(|f - fmin| num /
    (fmax - fmin)); Mel / Bark / Erb: nearest band (`__arr_roundIndex`, -1 outside).  int conversion of NaN / inf as C
    does it on x86 (INT_MIN)."""
    f = np.asarray(inst_fre, dtype=f32)
    fre = np.asarray(fre_arr, dtype=f32)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        if scale in (SCALE_OCTAVE, SCALE_LOG):
            fmin, fmax = f32(fre[0] / f32(sr)), f32(fre[num - 1] / f32(sr))
            v = np.round(((np.log2(np.abs(f)).astype(f32) - np.log2(fmin)) * f32(num) / (np.log2(fmax) - np.log2(fmin))).astype(f32))
        elif scale in (SCALE_LINEAR, SCALE_LINSPACE):
            fmin, fmax = f32(fre[0] / f32(sr)), f32(fre[num - 1] / f32(sr))
            v = np.round((np.abs(f - fmin) * f32(num) / (fmax - fmin)).astype(f32))
        else:
            arr = (fre / f32(sr)).astype(f32)
            a = np.abs(f)
            idx = np.full(f.shape, -1, dtype=np.int64)
            j = np.searchsorted(arr, a, side="right") - 1          # arr[j] <= a < arr[j + 1]
            ok = (j >= 0) & (j < num - 1)
            jj = np.clip(j, 0, num - 2)
            left, right = a - arr[jj], arr[jj + 1] - a
            idx[ok] = np.where(left < right, jj, jj + 1)[ok]
            return idx
    out = np.full(f.shape, np.iinfo(np.int32).min, dtype=np.int64)
    fin = np.isfinite(v) & (np.abs(v) < 2 ** 31)
    out[fin] = v[fin].astype(np.int64)
    return out


def squeeze_scatter(re, im, idx, thresh):
    """out[idx[i, j], j] += W[i, j] for rows i in ascending order where 0 <= idx < num and |W|^2 > thresh^2
    (wsst_algorithm.c:318-341): float32 accumulation in the reference's order"""
    num, n = re.shape
    o_re = np.zeros((num, n), dtype=f32)
    o_im = np.zeros((num, n), dtype=f32)
    cols = np.arange(n)
    t2 = f32(thresh) * f32(thresh)
    for i in range(num):
        v1, v2 = re[i].astype(f32), im[i].astype(f32)
        ok = (idx[i] >= 0) & (idx[i] < num) & ((v1 * v1 + v2 * v2).astype(f32) > t2)
        r = idx[i][ok]
        o_re[r, cols[ok]] += v1[ok]
        o_im[r, cols[ok]] += v2[ok]
    return o_re, o_im


def wsst(x, num=84, radix2_exp=12, sr=32000, wavelet=WAVE_MORLET, scale=SCALE_OCTAVE, low=None, high=None, bpo=12,
         gamma=None, beta=None, thresh=0.001, is_pad=False, cwt_planes=None):
    """`wsstObj_wsst` (order 1) -> (re, im, cwt_re, cwt_im), each [num, N] in the reference's row order.
    cwt_planes = (W_re, W_im, dW_re, dW_im) overrides the transforms (used to test the squeezing alone)."""
    if cwt_planes is None:
        w_re, w_im = cwt(x, num, radix2_exp, sr, wavelet, scale, low, high, bpo, gamma, beta, is_pad)
        d_re, d_im = cwt(x, num, radix2_exp, sr, wavelet, scale, low, high, bpo, gamma, beta, is_pad, det=True)
    else:
        w_re, w_im, d_re, d_im = cwt_planes
    _, fre = cwt_filterbank(num, 1 << radix2_exp, sr, wavelet, scale, low, high, bpo, gamma, beta, 0)
    _, ph = _complex_div(d_re, d_im, w_re, w_im)
    ph = (ph / f32(2 * math.pi)).astype(f32)
    idx = squeeze_index(ph, fre, sr, scale, num)
    o_re, o_im = squeeze_scatter(w_re, w_im, idx, thresh)
    return o_re, o_im, w_re, w_im


def unwrap_rows(p):
    """`__vunwrap` in place along the last axis (src/vector/flux_vector.c:1792-1830): float32 storage, the correction
    t * 2 pi evaluated in double as the C expression does"""
    p = np.array(p, dtype=f32)
    two_pi = 2 * math.pi
    for r in range(p.shape[0]):
        a = p[r]
        for i in range(1, a.shape[0]):
            sub = float(f32(abs(f32(a[i] - a[i - 1]))))
            if sub >= math.pi:
                t = int(math.floor(float(f32(sub / two_pi))))        # floorf(double) -> the argument is rounded to float
                mod = float(f32(sub - t * two_pi))
                if mod > math.pi:
                    t += 1
                a[i] = f32(float(a[i]) - t * two_pi) if a[i] > a[i - 1] else f32(float(a[i]) + t * two_pi)
    return p


def synsq(fre_arr, re, im, sr=32000, scale=SCALE_OCTAVE, thresh=0.001):
    """`synsqObj_synsq` (order 1): phase = atan2f(re, im) (the reference's argument order), unwrap along time, first
    difference (last column repeated), / 2 pi, index, scatter -> (re, im) [num, N]"""
    re, im = np.asarray(re, dtype=f32), np.asarray(im, dtype=f32)
    num, n = re.shape
    ph = unwrap_rows(np.arctan2(re, im).astype(f32))
    d = np.zeros_like(ph)
    d[:, 1:] = (ph[:, 1:] - ph[:, :-1]).astype(f32)
    d[:, n - 1] = d[:, n - 2]
    d = (d / f32(2 * math.pi)).astype(f32)
    idx = squeeze_index(d, fre_arr, sr, scale, num)
    return squeeze_scatter(re, im, idx, thresh)


# ---------------------------------------------------------------------------
# streaming STFT (isContinue = 1, non-padding): `__stftObj_dealData` (src/stft_algorithm.c:474-599)
# ---------------------------------------------------------------------------
class StftStream:
    """successive `push(chunk)` calls give the frames `stftObj_stft` returns in continue mode: the samples that did not
    complete a hop are carried over (tail length (total - n) % hop + (n - hop); negative = samples to skip when hop > n)"""

    def __init__(self, n, hop, window):
        self.n, self.hop, self.window = n, hop, np.asarray(window, dtype=np.float64)
        self.tail = np.zeros(0, np.float64)
        self.skip = 0

    def push(self, chunk):
        x = np.asarray(chunk, dtype=np.float64)
        if self.skip:
            k = min(self.skip, x.shape[0])
            x, self.skip = x[k:], self.skip - k
        cur = np.concatenate([self.tail, x])
        n, hop = self.n, self.hop
        if cur.shape[0] < n:
            self.tail = cur
            return np.zeros((0, n), f32), np.zeros((0, n), f32)
        tail_len = (cur.shape[0] - n) % hop + (n - hop)
        re, im = stft(cur, n, hop, self.window)
        if tail_len >= 0:
            self.tail = cur[cur.shape[0] - tail_len:]
        else:
            self.tail, self.skip = np.zeros(0, np.float64), -tail_len
        return re, im


class CqtStream:
    """`cqtObj_cqt` with isContinue = 1 (`_cqtObj_dealData`, cqt_algorithm.c:346-456): full-rate samples that do not
    complete a hop are carried to the next call; every call transforms the assembled samples on their own"""

    def __init__(self, num=84, sr=32000, **kw):
        self.num, self.sr, self.kw = num, sr, kw
        self.bank = cqt_kernel_bank(num, sr, kw.get("min_fre", 32.703196), kw.get("bpo", 12), kw.get("factor", 1.0),
                                    kw.get("beta", 0.0), kw.get("thresh", 0.01), kw.get("win_type", W_HANN), kw.get("norm", NORM_NONE))
        self.n = self.bank["fft_length"]
        self.hop = kw.get("hop") or self.n // 4
        self.tail = np.zeros(0, f32)
        self.skip = 0

    def push(self, chunk):
        x = np.asarray(chunk, dtype=f32)
        if self.skip:
            k = min(self.skip, x.shape[0])
            x, self.skip = x[k:], self.skip - k
        cur = np.concatenate([self.tail, x])
        n, hop = self.n, self.hop
        if cur.shape[0] < n:
            self.tail = cur
            return np.zeros((0, self.num), f32), np.zeros((0, self.num), f32)
        tail_len = (cur.shape[0] - n) % hop + (n - hop)
        out = cqt(cur, self.num, self.sr, bank=self.bank, hop=hop, is_scale=self.kw.get("is_scale", True),
                  bpo=self.kw.get("bpo", 12), is_continue=True)
        if tail_len >= 0:
            self.tail = cur[cur.shape[0] - tail_len:]
        else:
            self.tail, self.skip = np.zeros(0, f32), -tail_len
        return out


# ---------------------------------------------------------------------------
# Reassignment (src/reassign_algorithm.c:83-186 constructor, :200-414 transform, :417-451 windows, :587-822 steps)
# ---------------------------------------------------------------------------
REASSIGN_ALL, REASSIGN_FRE, REASSIGN_TIME, REASSIGN_NONE = range(4)


def reassign_windows(window):
    """`_reassignObj_initWindowData` (reassign_algorithm.c:417-451): h, dh = central difference of the periodically
    wrapped window (`__vgradient` of [w[n-1], w[0..n-1], w[0]], entries 1..n), th = n * w(n), n = -N/2 .. N/2-1."""
    w = np.asarray(window, dtype=f32)
    n = w.shape[0]
    der = np.concatenate([w[-1:], w, w[:1]]).astype(f32)
    dh = ((der[2:] - der[:-2]).astype(f32) / f32(2)).astype(f32)
    th = (np.arange(-(n // 2), n // 2).astype(f32) * w).astype(f32)
    return w, dh, th


def _c_int_cast(v):
    """(int) of a float as C does it on x86: NaN / inf / out of range -> INT_MIN"""
    out = np.full(v.shape, np.iinfo(np.int32).min, dtype=np.int64)
    fin = np.isfinite(v) & (np.abs(v) < 2 ** 31)
    out[fin] = v[fin].astype(np.int64)
    return out


def _roundf(v):
    """roundf: halves away from zero (numpy rounds halves to even)"""
    v = np.asarray(v, dtype=f32)
    return (np.sign(v) * np.floor(np.abs(v) + f32(0.5))).astype(f32)


def reassign_coords(s1, s2, s3, n, sr, hop, re_type=REASSIGN_ALL, thresh=0.001):
    """steps 3 + 4 (`_reassignObj_reassignTimeFre` :612-703, `_reassignObj_filterTimeFre` :709-822): reassigned
    frequency / time of every cell [T, n/2+1] in float32, thresholded on |S_h|^2 >= thresh^2 and clipped."""
    (r1, i1), W = s1, n // 2 + 1
    T = r1.shape[0]
    fre = _linspace_f32(0, sr / 2.0, W)
    tarr = ((np.arange(T).astype(f32) * f32(hop)).astype(f32) / f32(sr)).astype(f32)
    power = ((r1 * r1).astype(f32) + (i1 * i1).astype(f32)).astype(f32)
    keep = power >= f32(thresh) * f32(thresh)
    re_f = np.broadcast_to(fre[None, :], (T, W)).astype(f32).copy()
    re_t = np.broadcast_to(tarr[:, None], (T, W)).astype(f32).copy()
    fmax, tmax = fre[W - 1], tarr[T - 1]
    with np.errstate(all="ignore"):
        if re_type in (REASSIGN_FRE, REASSIGN_ALL):
            _, qi = _complex_div(s2[0], s2[1], r1, i1)
            v = ((qi * f32(-0.5 * sr / math.pi)).astype(f32) + fre[None, :]).astype(f32)     # __mmul_value takes a float
            v = np.where(keep, v, re_f)
            v = np.where(v < 0, f32(0), v)             # NaN compares false in both clips and survives, as in C
            re_f = np.where(v > fmax, fmax, v).astype(f32)
        if re_type in (REASSIGN_TIME, REASSIGN_ALL):
            qr, _ = _complex_div(s3[0], s3[1], r1, i1)
            v = ((qr * f32(1.0 / sr)).astype(f32) + tarr[:, None]).astype(f32)
            v = np.where(keep, v, re_t)
            v = np.where(v < 0, f32(0), v)
            re_t = np.where(v > tmax, tmax, v).astype(f32)
    return re_f, re_t, fre, tarr


def reassign_indices(re_f, re_t, fre, tarr, n, order=1):
    """`_reassignObj_rearrage` index part (:268-323): roundf of the affine maps, then order-1 further look-ups of the
    frequency index along the row (the scratch keeps its previous content where the index leaves the row)."""
    T, W = re_f.shape
    fmin, fmax, tmin, tmax = fre[0], fre[W - 1], tarr[0], tarr[T - 1]
    with np.errstate(all="ignore"):
        ti = np.zeros((T, W), dtype=np.int64)
        if T > 1:
            ti = _c_int_cast(_roundf(((re_t - tmin).astype(f32) * f32(T - 1)).astype(f32) / f32(tmax - tmin)))
        fi = _c_int_cast(_roundf(((re_f - fmin).astype(f32) * f32(n // 2)).astype(f32) / f32(fmax - fmin)))
    if order > 1:
        tmp = np.zeros((T, W), dtype=np.int64)
        rows = np.arange(T)[:, None]
        for _ in range(order - 1):
            ok = (fi >= 0) & (fi < W)
            look = fi[rows, np.clip(fi, 0, W - 1)]
            tmp = np.where(ok, look, tmp)
            fi = tmp.copy()
    return ti, fi


def reassign(x, radix2_exp=12, sr=32000, window_type=W_HANN, hop=None, re_type=REASSIGN_ALL, thresh=0.001,
             is_pad=False, order=1, result_type=0, indices=False):
    """`reassignObj_reassign` (reassign_algorithm.c:200-414) -> (re4, im4, re5, im5), planes [T, n/2+1]; the reference
    ADDS into re4 / im4 (zero planes here), re5 / im5 = the plain half spectrum S_h.  float32 accumulation in the
    reference's (frame, bin) order.  indices=True also returns (time index, frequency index)."""
    n = 1 << radix2_exp
    hop = hop if hop else n // 4
    W = n // 2 + 1
    h, dh, th = reassign_windows(fft_window(window_type, n))
    s = []
    for w in (h, dh, th):
        r, i = stft(x, n, hop, w, is_pad=is_pad)
        s.append((np.ascontiguousarray(r[:, :W]), np.ascontiguousarray(i[:, :W])))
    T = s[0][0].shape[0]
    if re_type == REASSIGN_NONE:
        out = (s[0][0].copy(), s[0][1].copy(), None, None)
        return out + (None, None) if indices else out
    re_f, re_t, fre, tarr = reassign_coords(s[0], s[1], s[2], n, sr, hop, re_type, thresh)
    ti, fi = reassign_indices(re_f, re_t, fre, tarr, n, order)
    o_re = np.zeros((T, W), dtype=f32)
    o_im = np.zeros((T, W), dtype=f32)
    sign = np.where(np.arange(W) % 2 == 1, f32(-1), f32(1)).astype(f32)
    v1 = (s[0][0] * sign[None, :]).astype(f32)
    v2 = (s[0][1] * sign[None, :]).astype(f32)
    ok = (ti >= 0) & (ti < T) & (fi >= 0) & (fi < W)
    amp = np.sqrt((v1 * v1 + v2 * v2).astype(f32)).astype(f32)
    for i in range(T):                                  # float32 += in source order (rows, then bins)
        m = ok[i]
        if result_type == 0:
            np.add.at(o_re, (ti[i][m], fi[i][m]), v1[i][m])
            np.add.at(o_im, (ti[i][m], fi[i][m]), v2[i][m])
        else:
            np.add.at(o_re, (ti[i][m], fi[i][m]), amp[i][m])
    out = (o_re, o_im, s[0][0], s[0][1])
    return out + (ti, fi) if indices else out


# ---------------------------------------------------------------------------
# cepstral deconvolution of constant-Q spectra: cqtObj_cqhc / cqtObj_deconv (src/cqt_algorithm.c:662-781)
# ---------------------------------------------------------------------------
def cq_deconv(m, bpo=12):
    """m [T, num] magnitudes / powers -> (timbre, pitch), each [T, num]: rows zero-padded to L = ceilPow2(2 num);
    timbre = Re IFFT(|FFT(row)|), pitch = Re IFFT(FFT(row) / max(|FFT(row)|, 1e-16))"""
    m = np.asarray(m, dtype=np.float64)
    T, num = m.shape
    L = _ceil_pow2(2 * num)
    X = np.fft.fft(np.concatenate([m, np.zeros((T, L - num))], axis=1), axis=1)
    mag = np.abs(X).astype(f32).astype(np.float64)
    timbre = np.fft.ifft(mag, axis=1).real
    pitch = np.fft.ifft(X / np.maximum(mag, 1e-16), axis=1).real
    return timbre[:, :num].astype(f32), pitch[:, :num].astype(f32)


def cqhc(m, hc_num=20, bpo=12):
    """`cqtObj_cqhc`: timbre[round(bpo log2(j + 1))], j < hc_num (index from float32 log2f / roundf)"""
    m = np.asarray(m, dtype=np.float64)
    T, num = m.shape
    L = _ceil_pow2(2 * num)
    X = np.fft.fft(np.concatenate([m, np.zeros((T, L - num))], axis=1), axis=1)
    timbre = np.fft.ifft(np.abs(X).astype(f32).astype(np.float64), axis=1).real
    idx = _roundf(f32(bpo) * np.log2(np.arange(1, hc_num + 1).astype(f32)).astype(f32)).astype(int)
    return timbre[:, idx].astype(f32)
