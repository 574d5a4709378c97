"""Float64 numpy restatement of the reference's cepstrogram, the case list, and ctypes drivers that work on either library.

src/cepstrogram_algorithm.c, per frame t of the STFT without padding (cepstrogramObj_calTimeLength, :104-109):
  1. X = the full N-point FFT of the windowed frame (:210-212);
  2. S = re^2 + im^2, values below 1e-16 replaced by the float 1e-16, then log (:219-229);
  3. y = Re IFFT_N(log S), the inverse FFT scaled by 1/N (:232-234);
  4. cepstrums = y[0 .. N/2] (:236-239);
  5. envelope: e = y[0 .. c], then e[N-1-j] = e[j+1] for j < c, zero elsewhere; Re FFT_N(e)[0 .. N/2] (:257-265);
  6. details: d = y on c+1 .. c+1 + (N-2c) - 1 = N-c, zero elsewhere; Re FFT_N(d)[0 .. N/2] (:283-287).
The index sets are taken literally: no closed form, no even-part shortcut.  cepstrogram2 (:119-125) is restated as
its documented intent (include/afb200_cepstrogram.h): the same steps from the caller's planes, every bin of a width-N
plane used as it is."""
import ctypes as C

import numpy as np

from oracle import af_oracle as O

W_RECT, W_HANN, W_HAMM, W_BLACKMAN = O.W_RECT, O.W_HANN, O.W_HAMM, O.W_BLACKMAN
CLAMP = float(np.float32(1e-16))


def time_length(length, n, hop):
    """:104-109 (stftObj_calTimeLength without padding, src/stft_algorithm.c:225-262)"""
    return 0 if length < n else (length - n) // hop + 1


def log_power(re, im):
    """:219-229 in float64: the clamp stores the float 1e-16"""
    s = np.asarray(re, np.float64) ** 2 + np.asarray(im, np.float64) ** 2
    return np.log(np.where(s < 1e-16, CLAMP, s))


def from_log_spectrum(L, cep_num):
    """L [T, N] (every bin) -> (cepstrums, envelope, details) [T, N/2+1], steps 3-6"""
    T, n = L.shape
    c, h = cep_num, n // 2 + 1
    y = np.fft.ifft(L, axis=1).real                                # :233
    e = np.zeros((T, n))
    e[:, :c + 1] = y[:, :c + 1]                                    # :259
    e[:, n - 1 - np.arange(c)] = e[:, 1 + np.arange(c)]            # :260-262
    d = np.zeros((T, n))
    d[:, c + 1:c + 1 + n - 2 * c] = y[:, c + 1:c + 1 + n - 2 * c]  # :284
    return y[:, :h], np.fft.fft(e, axis=1).real[:, :h], np.fft.fft(d, axis=1).real[:, :h]


def frames_spectrum(x, n, hop, window_type):
    """complex [T, N]: the full FFT of every windowed frame"""
    x = np.asarray(x, np.float64)
    T = time_length(x.size, n, hop)
    if T == 0:
        return np.zeros((0, n), np.complex128)
    idx = np.arange(T)[:, None] * hop + np.arange(n)[None, :]
    return np.fft.fft(x[idx] * O.fft_window(window_type, n).astype(np.float64)[None, :], axis=1)


def cepstrogram(x, n, hop, window_type, cep_num):
    """(cepstrums, envelope, details, log S) for one clip; log S [T, N/2+1] is the scale of the per-frame bar"""
    X = frames_spectrum(x, n, hop, window_type)
    L = log_power(X.real, X.imag)
    return (*from_log_spectrum(L, cep_num), L[:, :n // 2 + 1])


def cepstrogram2(re, im, cep_num):
    """from STFT planes [rows, width]: width N used as given (the literal Re IFFT of all N bins), width N/2+1 mirrored
    as a Hermitian spectrum"""
    re, im = np.asarray(re, np.float64), np.asarray(im, np.float64)
    L = log_power(re, im)
    width = L.shape[1]
    if width % 2:                                                 # N/2+1 -> N
        n = 2 * (width - 1)
        L = np.concatenate([L, L[:, n // 2 - 1:0:-1]], axis=1)
    return (*from_log_spectrum(L, cep_num), L[:, :L.shape[1] // 2 + 1])


def frame_errors(got, want, logs):
    """per frame: max_k |got - want| / max_k |log S[k]|"""
    g = np.asarray(got, np.float64)
    return np.abs(g - want).max(axis=1, initial=0) / np.abs(logs).max(axis=1, initial=0)


# ---- test signals ----

def signal(seed, length, silent=0.0):
    """white noise with two tones riding on it: every bin stays within about 80 dB of its frame's peak (the log of a
    bin far below the peak is ill-conditioned in float32).  silent: the fraction of the clip, from its start, that is
    zeros (1: a silent clip); frames inside it hit the clamp exactly."""
    rng = np.random.default_rng(seed)
    t = np.arange(length)
    x = 0.1 * rng.standard_normal(length) + 0.05 * np.cos(0.0931 * t + 0.4) + 0.03 * np.cos(1.2345 * t)
    x[:int(round(silent * length))] = 0
    return x.astype(np.float32)


def cases():
    """[(name, dict(radix2_exp, window_type, slide, cep_num, length, silent))]"""
    out = []
    for r in range(1, 13):
        n = 1 << r
        for c in sorted({c for c in (1, 4, 20, 128, n // 2 - 1, n // 2) if 1 <= c <= n // 2}):
            out.append((f"r{r}_c{c}", dict(radix2_exp=r, window_type=W_HANN, slide=max(1, n // 2), cep_num=c,
                                           length=n + 5 * max(1, n // 2) + 3)))
    for r in (13, 14):
        n = 1 << r
        for c in (4, 128, n // 2 - 1, n // 2):
            out.append((f"r{r}_c{c}", dict(radix2_exp=r, window_type=W_HANN, slide=n // 2, cep_num=c, length=2 * n + 7)))
    for w, wn in ((W_RECT, "rect"), (W_HAMM, "hamm"), (W_BLACKMAN, "blackman")):
        out.append((f"r10_{wn}", dict(radix2_exp=10, window_type=w, slide=256, cep_num=20, length=4000)))
    out += [
        ("r9_slide100", dict(radix2_exp=9, window_type=W_HANN, slide=100, cep_num=20, length=1500)),
        ("r9_slide512", dict(radix2_exp=9, window_type=W_RECT, slide=512, cep_num=4, length=3000)),
        ("r9_slide700", dict(radix2_exp=9, window_type=W_HAMM, slide=700, cep_num=128, length=3000)),
        ("r8_t0", dict(radix2_exp=8, window_type=W_HANN, slide=64, cep_num=4, length=200)),
        ("r8_t1", dict(radix2_exp=8, window_type=W_HANN, slide=512, cep_num=4, length=300)),
        ("r8_silent", dict(radix2_exp=8, window_type=W_HANN, slide=128, cep_num=4, length=1000, silent=1.0)),
        ("r10_halfsilent", dict(radix2_exp=10, window_type=W_HANN, slide=256, cep_num=20, length=4000, silent=0.5)),
        ("r12_halfsilent", dict(radix2_exp=12, window_type=W_RECT, slide=1024, cep_num=128, length=12000, silent=0.5)),
        ("r12_default", dict(radix2_exp=12, window_type=W_RECT, slide=1024, cep_num=4, length=16000)),
    ]
    return out


def case_signal(name, kw):
    return signal(sum(map(ord, name)), kw["length"], kw.get("silent", 0.0))


def oracle_case(name, kw):
    return cepstrogram(case_signal(name, kw), 1 << kw["radix2_exp"], kw["slide"], kw["window_type"], kw["cep_num"])


# ---- ctypes drivers (either library) ----

def c_new(lib, radix2_exp, window_type=None, slide=None):
    obj = C.c_void_p()
    w = None if window_type is None else C.byref(C.c_int(window_type))
    s = None if slide is None else C.byref(C.c_int(slide))
    return lib.cepstrogramObj_new(C.byref(obj), radix2_exp, w, s), obj


def _planes(rows, n, want, fill):
    return [np.full((rows, n // 2 + 1), fill, np.float32) if w else None for w in want]


def _p(a):
    return None if a is None else a.ctypes.data


def c_cepstrogram(lib, obj, n, cep_num, x, want=(1, 1, 1), fill=0.0, rows=None):
    """[cep, env, det] [T, N/2+1] (None where not requested); the planes start as `fill`"""
    x = np.ascontiguousarray(x, np.float32)
    if rows is None:
        rows = lib.cepstrogramObj_calTimeLength(obj, x.size)
    out = _planes(rows, n, want, fill)
    lib.cepstrogramObj_cepstrogram(obj, cep_num, x.ctypes.data, x.size, *map(_p, out))
    return out


def c_cepstrogram2(lib, obj, n, cep_num, re, im, want=(1, 1, 1), fill=0.0):
    re, im = np.ascontiguousarray(re, np.float32), np.ascontiguousarray(im, np.float32)
    out = _planes(re.shape[0], n, want, fill)
    lib.cepstrogramObj_cepstrogram2(obj, cep_num, re.ctypes.data, im.ctypes.data, re.shape[0], *map(_p, out))
    return out


def c_case(lib, kw, x, want=(1, 1, 1)):
    s, obj = c_new(lib, kw["radix2_exp"], kw["window_type"], kw["slide"])
    assert s == 0
    out = c_cepstrogram(lib, obj, 1 << kw["radix2_exp"], kw["cep_num"], x, want)
    lib.cepstrogramObj_free(obj)
    return out
