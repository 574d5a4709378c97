"""What the frame-wise pitch trackers' tests share, whatever the algorithm: ctypes drivers of the C objects that work on
either library, keyed by tracker (pef, yin, ncf, cep), the test signals and the batch clips.

The drivers pass a constructor argument left out as NULL.  c_pitch returns the legacy call's output plane (PEF, NCF,
CEP) or its three planes fre, value1, value2 as a tuple (YIN)."""
import ctypes as C

import numpy as np

f32 = np.float32


def ip(v):
    return None if v is None else C.byref(C.c_int(int(v)))


def fp(v):
    return None if v is None else C.byref(C.c_float(float(v)))


# the C prefix, the constructor's arguments in order (name, pointer) and the legacy call's output planes
_LAG = (("sr", ip), ("lf", fp), ("hf", fp), ("r2", ip), ("slide", ip), ("wt", ip), ("cont", ip))
TRACKERS = {
    "pef": ("pitchPEFObj", (("sr", ip), ("lf", fp), ("hf", fp), ("cf", fp), ("r2", ip), ("slide", ip), ("wt", ip),
                            ("alpha", fp), ("beta", fp), ("gamma", fp), ("cont", ip)), 1),
    "yin": ("pitchYINObj", (("sr", ip), ("lf", fp), ("hf", fp), ("r2", ip), ("slide", ip), ("auto", ip),
                            ("cont", ip)), 3),
    "ncf": ("pitchNCFObj", _LAG, 1),
    "cep": ("pitchCEPObj", _LAG, 1),
}


def prefix(kind):
    return TRACKERS[kind][0]


def c_new(lib, kind, **ctor):
    """new -> (status, object)"""
    name, args, _ = TRACKERS[kind]
    unknown = set(ctor) - {a for a, _ in args}
    if unknown:
        raise TypeError(f"{name}_new takes no {sorted(unknown)}")
    obj = C.c_void_p()
    return getattr(lib, name + "_new")(C.byref(obj), *(ptr(ctor.get(a)) for a, ptr in args)), obj


def c_time_length(lib, kind, obj, n):
    return getattr(lib, prefix(kind) + "_calTimeLength")(obj, n)


def c_free(lib, kind, obj):
    getattr(lib, prefix(kind) + "_free")(obj)


def c_pitch(lib, kind, obj, x, fill=0.0, extra=0):
    """pitch -> the output planes of T + extra floats (T from calTimeLength before the call), which started as
    `fill`"""
    x = np.ascontiguousarray(x, f32)
    T = c_time_length(lib, kind, obj, x.size)
    out = [np.full(T + extra, fill, f32) for _ in range(TRACKERS[kind][2])]
    getattr(lib, prefix(kind) + "_pitch")(obj, x.ctypes.data, x.size, *(o.ctypes.data for o in out))
    return tuple(out) if len(out) > 1 else out[0]


def c_stream(lib, kind, obj, x, pieces):
    """pitch over consecutive pieces of x (isContinue objects) -> the output planes of all calls, concatenated"""
    outs, start = [], 0
    for size in pieces:
        outs.append(c_pitch(lib, kind, obj, x[start:start + size]))
        start += size
    if TRACKERS[kind][2] == 1:
        return np.concatenate(outs)
    return tuple(np.concatenate([o[i] for o in outs]) for i in range(TRACKERS[kind][2]))


def time_length(length, n, hop):
    return 0 if length < n else (length - n) // hop + 1


def signal(kind, length, sr, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(length) / sr
    if kind == "silence":
        x = np.zeros(length)
    elif kind == "dc":
        x = np.full(length, 0.5)
    elif kind == "alt":                         # +1, -1, ...
        x = np.where(np.arange(length) % 2, -1.0, 1.0)
    elif kind == "noise":
        x = 0.1 * rng.standard_normal(length)
    elif kind == "tones":                       # 220 Hz and five overtones, a little noise
        x = sum(0.3 / h * np.sin(2 * np.pi * 220 * h * t + h) for h in range(1, 7)) + 0.01 * rng.standard_normal(length)
    elif kind == "low":                         # 95 Hz and its overtones, a little noise
        x = sum(0.4 / h * np.sin(2 * np.pi * 95 * h * t + h) for h in range(1, 9)) + 0.01 * rng.standard_normal(length)
    elif kind == "missing":                     # overtones 2 .. 6 of 180 Hz without the fundamental
        x = sum(0.3 / h * np.sin(2 * np.pi * 180 * h * t + h) for h in range(2, 7)) + 0.01 * rng.standard_normal(length)
    elif kind == "glide":                       # a harmonic tone gliding from 120 to 700 Hz, in noise
        f = 120 + (700 - 120) * t / max(t[-1], 1e-9)
        ph = 2 * np.pi * np.cumsum(f) / sr
        x = sum(0.4 / h * np.sin(h * ph) for h in range(1, 5)) + 0.05 * rng.standard_normal(length)
    elif kind == "gaps":                        # tones with runs of silence longer than a frame
        x = signal("tones", length, sr, seed).astype(np.float64)
        for a in range(length // 5, length, 2 * length // 5):
            x[a:a + length // 6] = 0.0
    elif kind == "half":                        # the tone in the second half only
        x = np.where(t >= t[-1] / 2, signal("tones", length, sr, seed), 0.0)
    elif kind == "quiet":                       # near YIN's 1e-6 clamps of r and e2
        x = 3e-4 * signal("tones", length, sr, seed)
    elif kind == "loud":
        x = 3e3 * signal("tones", length, sr, seed)
    elif kind == "nan":                         # noise with one NaN sample
        x = 0.1 * rng.standard_normal(length)
        x[length // 2] = np.nan
    elif kind == "tone4638":                    # 32000 / 69 Hz: every correlation between lags 33 and 36 is negative
        x = np.sin(2 * np.pi * (32000 / 69) * t)
    else:
        raise ValueError(kind)
    return np.asarray(x, f32)


def clips(n, length, sr, seed, silent_every=0):
    """harmonic tones of random f0 (80 .. 600 Hz), some without their fundamental, in noise; with silent_every = k,
    every k-th clip silent in its second half"""
    rng = np.random.default_rng(seed)
    t = np.arange(length) / sr
    f0 = rng.uniform(80, 600, (n, 1))
    first = rng.integers(1, 3, (n, 1))
    x = sum(np.where(first <= h, 0.3 / h, 0.0) * np.sin(2 * np.pi * f0 * h * t + h) for h in range(1, 6))
    x = x + 0.05 * rng.standard_normal((n, length))
    if silent_every:
        x[::silent_every, length // 2:] = 0
    return x.astype(f32)
