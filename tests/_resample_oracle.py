"""Float64 numpy restatement of the reference's resampler, the case list, and ctypes drivers that work on either library.

src/dsp/resample_algorithm.c, with the float32 index arithmetic taken literally:
  - the table (:546-634) in float32: x = i * (zeroNum / (L-1)) * rollOff, rollOff * sinf(pi x) / (pi x), times the right
    half of the symmetric window of length 2(L-1)+1; scaled in place by the ratio while the ratio is below 1, and divided
    by the old ratio before a rescale (:281-293, :536-540), every step rounded to float32;
  - the difference table (:542-543): float32 a[k+1] - a[k], 0 for the last entry;
  - per output i (:468-520): t = float32(i / ratio) (double division), n = floorf(t), scale = min(1, ratio),
    step = floorf(scale * 2^nbit), phases and offsets in float32, tap counts by integer division;
  - the weights a[o] + delta * d[o] and the sums in float64.
Continue mode (:219-251, :350-403): each call resamples the first L - L % q samples into (L - L % q) * p / q outputs and
drops the rest; the reference's tail carry starts only from a non-empty tail, which it never creates."""
import ctypes as C

import numpy as np

from oracle import af_oracle as O

f32 = np.float32
QUALITIES = {0: (64, 9, f32(14.7696565), f32(0.9475937)),      # :59-97: zeroNum, nbit, Kaiser beta, rollOff
             1: (32, 9, f32(11.6625806), f32(0.8987969)),
             2: (16, 9, f32(8.5555046), f32(0.85))}
W_HANN, W_KAISER, W_GAUSS, W_TUKEY = O.W_HANN, O.W_KAISER, O.W_GAUSS, O.W_TUKEY


def window_rules(zero_num=None, nbit=None, win_type=None, value=None, roll_off=None):
    """:115-175 -> (zeroNum, nbit, winType, value, rollOff); None is a NULL pointer"""
    z = zero_num if zero_num is not None and zero_num > 0 else 64
    nb = nbit if nbit is not None and 0 < nbit < 30 else 9
    w = win_type if win_type is not None and win_type > O.W_RECT else W_HANN
    v = f32(0)
    if value is not None:
        if value >= 0:
            v = f32(value)
        if v == 0:
            v = f32(5) if w == W_KAISER else f32(2.5) if w == W_GAUSS else v
    r = f32(roll_off) if roll_off is not None and 0 < f32(roll_off) <= 1 else f32(0.945)
    return z, nb, w, v, r


def table(z, nb, w, v, r):
    """the unscaled float32 table (:546-634)"""
    L = z * (1 << nb) + 1
    step = f32(z) / f32(L - 1)
    x = (np.arange(L).astype(f32) * step) * r
    val = (x.astype(np.float64) * np.pi).astype(f32)
    with np.errstate(invalid="ignore", divide="ignore"):
        s = np.where(np.abs(val) < 1e-9, f32(1), np.sin(val) / val).astype(f32)
    win = O._symmetric_window(w, 2 * (L - 1) + 1, float(v)).astype(f32)
    return (s * r) * win[L - 1:]


class Resampler:
    """one reference object: its rates, its float32 table with the scaling history, its continue flag"""

    def __init__(self, qual=None, window=None, is_scale=False, is_continue=False):
        if window is None:
            z, nb, v, r = QUALITIES[0 if qual is None else qual]
            params = (z, nb, W_KAISER, v, r)
        else:
            params = window_rules(**window)
        self.zero_num, self.nbit = params[0], params[1]
        self.bit_length = 1 << self.nbit
        self.a = table(*params)
        self.ratio, self.p, self.q = f32(1), 1, 2
        self._set_ratio(f32(0.5))
        self.is_scale, self.is_continue = is_scale, is_continue

    def _set_ratio(self, ratio):
        ratio = f32(ratio)
        if ratio != self.ratio and (self.ratio < 1 or ratio < 1):
            if self.ratio < 1:
                self.a = (self.a / self.ratio).astype(f32)
            if ratio < 1:
                self.a = (self.a * ratio).astype(f32)
        self.ratio = ratio

    def set_samplate(self, src, dst):
        """:253-301"""
        if src == dst or src <= 0 or dst <= 0:
            return
        g = int(np.gcd(src, dst))
        self._set_ratio(f32(dst) / f32(src))
        self.p, self.q = dst // g, src // g

    def set_ratio(self, r):
        """:303-332"""
        if r < 0:
            return
        self._set_ratio(r)
        self.p = self.q = 0

    def lengths(self, n):
        """:219-251 -> (source length, target length)"""
        if not self.is_continue:
            return n, int(np.floor(f32(n) * self.ratio))
        if self.q > 1:
            src = n - n % self.q
            return src, src * self.p // self.q
        return 0, 0

    def step(self):
        scale = self.ratio if 1.0 > self.ratio else f32(1)
        return scale, int(np.floor(scale * f32(self.bit_length)))

    def taps(self, n):
        """taps summed per output of a call on n samples (:493-495, :509-511)"""
        src, tgt = self.lengths(n)
        scale, step = self.step()
        t = (np.arange(tgt) / np.float64(self.ratio)).astype(f32)
        m = np.floor(t).astype(np.int64)
        factor = (scale * (t - m.astype(f32))).astype(f32)
        count = 0
        for f, lim in ((factor, m + 1), ((scale - factor).astype(f32), src - m - 1)):
            off = np.floor((f * f32(self.bit_length)).astype(f32)).astype(np.int64)
            count = count + np.maximum(np.minimum(lim, (self.a.size - off) // step), 0)
        return count

    def resample(self, x, init=None):
        """one call: x float32 [n] -> float64 [target length]; init = the caller's buffer (added into)"""
        x = np.asarray(x, np.float64)
        src, tgt = self.lengths(x.size)
        scale, step = self.step()
        out = np.zeros(tgt) if init is None else np.asarray(init[:tgt], np.float64).copy()
        if tgt <= 0:
            return out
        a = self.a.astype(np.float64)
        d = np.zeros_like(a)
        d[:-1] = (self.a[1:] - self.a[:-1]).astype(np.float64)        # float32 differences (__vdiff)
        L, bits = a.size, f32(self.bit_length)
        i = np.arange(tgt)
        t = (i / np.float64(self.ratio)).astype(f32)
        n = np.floor(t).astype(np.int64)
        xz = np.concatenate([x, [0.0]])                                  # a left tap at or beyond the clip end reads 0

        def side(factor, count, index):
            fv = (factor * bits).astype(f32)
            off = np.floor(fv).astype(np.int64)
            delta = (fv - off.astype(f32)).astype(np.float64)
            cnt = np.minimum(count, (L - off) // step)
            acc = np.zeros(tgt)
            for j in range(int(cnt.max(initial=0))):
                m = j < cnt
                o = np.where(m, off + j * step, 0)
                g = np.clip(index(j), 0, x.size)
                acc += np.where(m, (a[o] + delta * d[o]) * xz[g], 0.0)
            return acc

        factor = (scale * (t - n.astype(f32))).astype(f32)
        left = side(factor, n + 1, lambda j: np.minimum(n - j, x.size))
        right = side((scale - factor).astype(f32), src - n - 1, lambda j: n + j + 1)
        out = out + left + right
        if self.is_scale:
            out = out / np.float64(np.sqrt(self.ratio, dtype=f32))
        return out


# ---------------------------------------------------------------------------------------------------------- the cases
RATES = [(48000, 16000), (44100, 16000), (16000, 48000), (22050, 44100), (44100, 48000), (48000, 44100), (8000, 44100)]
BIG = (1 << 24) + 10007


def _len_for(ratio):
    return int(min(1500, 2000 / ratio))


def cases():
    """[(name, kw)]: kw = ctor ('qual' or 'window'), ops (('rate', s, d) | ('ratio', r)), length, is_scale, init seed,
    chunks (continue mode)"""
    out = []
    names = {0: "best", 1: "mid", 2: "fast"}
    for q in (0, 1, 2):
        for s, d in RATES:
            out.append((f"{names[q]}_{s}_{d}", dict(qual=q, ops=[("rate", s, d)], length=_len_for(d / s))))
        out.append((f"{names[q]}_equal", dict(qual=q, ops=[("rate", 44100, 44100)], length=1500)))
    for w in range(O.W_HANN, O.W_TUKEY + 1):
        out.append((f"win{w}_null", dict(window=dict(zero_num=16, nbit=7, win_type=w), ops=[("rate", 44100, 16000)],
                                         length=1500)))
    for w, vals in ((W_KAISER, (0.0, 9.0)), (W_GAUSS, (0.0, 3.5)), (W_TUKEY, (0.0, 0.3, 1.0, 2.0))):
        for v in vals:
            out.append((f"win{w}_v{v}", dict(window=dict(zero_num=24, nbit=6, win_type=w, value=v, roll_off=0.9),
                                              ops=[("rate", 48000, 44100)], length=1500)))
    out.append(("win_defaults", dict(window=dict(), ops=[("rate", 22050, 16000)], length=1500)))
    out.append(("win_rules", dict(window=dict(zero_num=-3, nbit=30, win_type=0, value=-1.0, roll_off=1.5),
                                  ops=[("rate", 16000, 22050)], length=1200)))
    for r in (0.37, 1.0, 2.5):
        out.append((f"ratio_{r}", dict(qual=1, ops=[("ratio", r)], length=_len_for(r))))
    out.append(("chain", dict(qual=0, ops=[("rate", 44100, 16000), ("rate", 16000, 48000), ("ratio", 0.37),
                                           ("rate", 48000, 22050), ("rate", 22050, 44100), ("rate", 44100, 32000)],
                              length=1500)))
    out.append(("scale_down", dict(qual=1, ops=[("rate", 48000, 16000)], length=1500, is_scale=1)))
    out.append(("scale_up_init", dict(qual=2, ops=[("rate", 16000, 48000)], length=600, is_scale=1, init=3)))
    out.append(("init_44100_48000", dict(qual=0, ops=[("rate", 44100, 48000)], length=1500, init=4)))
    for n in (1, 2, 17):
        out.append((f"len{n}_down", dict(qual=0, ops=[("rate", 48000, 16000)], length=n)))
        out.append((f"len{n}_up", dict(qual=0, ops=[("rate", 16000, 48000)], length=n)))
    out.append(("continue_48000_16000", dict(qual=2, ops=[("rate", 48000, 16000)], chunks=[1000, 777, 1, 2, 4096, 333])))
    out.append(("continue_44100_48000", dict(qual=1, ops=[("rate", 44100, 48000)], chunks=[2000, 146, 147, 1500, 900])))
    out.append(("big_fast", dict(qual=2, ops=[("rate", 48000, 16000)], length=BIG)))
    return out


def case_signal(name, kw):
    """the input of a case: one clip, or the concatenated chunks of a continue case"""
    n = sum(kw["chunks"]) if "chunks" in kw else kw["length"]
    seed = sum(map(ord, name))
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 8000.0
    x = 0.3 * np.sin(2 * np.pi * 440 * t + 0.2 * np.sin(2 * np.pi * 3 * t)) + 0.05 * rng.standard_normal(n)
    return x.astype(np.float32)


def case_init(kw, m):
    if kw.get("init") is None:
        return None
    return np.random.default_rng(kw["init"]).standard_normal(m).astype(np.float32)


def _apply(obj_set_rate, obj_set_ratio, ops):
    for op in ops:
        if op[0] == "rate":
            obj_set_rate(op[1], op[2])
        else:
            obj_set_ratio(op[1])


def oracle_case(name, kw):
    """-> list of float64 outputs (one per chunk of a continue case, else one)"""
    r = Resampler(kw.get("qual"), kw.get("window"), bool(kw.get("is_scale")), "chunks" in kw)
    _apply(r.set_samplate, r.set_ratio, kw["ops"])
    x = case_signal(name, kw)
    if "chunks" in kw:
        pos, out = 0, []
        for c in kw["chunks"]:
            out.append(r.resample(x[pos:pos + c]))
            pos += c
        return out
    m = r.lengths(x.size)[1]
    return [r.resample(x, case_init(kw, m))]


# ------------------------------------------------------------------------------------------------ ctypes drivers
def _oi(v):
    return None if v is None else C.byref(C.c_int(int(v)))


def _of(v):
    return None if v is None else C.byref(C.c_float(float(v)))


def c_new(lib, qual=None, window=None, is_scale=0, is_continue=0):
    """-> (status, obj)"""
    o = C.c_void_p()
    if window is None:
        st = lib.resampleObj_new(C.byref(o), _oi(qual), _oi(is_scale), _oi(is_continue))
    else:
        w = window
        st = lib.resampleObj_newWithWindow(C.byref(o), _oi(w.get("zero_num")), _oi(w.get("nbit")), _oi(w.get("win_type")),
                                           _of(w.get("value")), _of(w.get("roll_off")), _oi(is_scale), _oi(is_continue))
    return st, o


def c_apply(lib, o, ops):
    _apply(lambda s, d: lib.resampleObj_setSamplate(o, s, d), lambda r: lib.resampleObj_setSamplateRatio(o, r), ops)


def c_resample(lib, o, x, init=None, extra=16):
    """one legacy call into a buffer of calDataLength + extra floats (init, else zeros) -> (returned length, buffer)"""
    x = np.ascontiguousarray(x, np.float32)
    m = lib.resampleObj_calDataLength(o, x.size)
    buf = np.zeros(max(m, 0) + extra, np.float32)
    if init is not None:
        buf[:m] = init[:m]
    n = lib.resampleObj_resample(o, x.ctypes.data, x.size, buf.ctypes.data)
    return n, buf


def c_case(lib, name, kw):
    """-> list of float32 outputs of the library, like oracle_case"""
    st, o = c_new(lib, kw.get("qual"), kw.get("window"), kw.get("is_scale", 0), 1 if "chunks" in kw else 0)
    assert st == 0, (name, st)
    c_apply(lib, o, kw["ops"])
    x = case_signal(name, kw)
    out = []
    try:
        if "chunks" in kw:
            pos = 0
            for c in kw["chunks"]:
                n, buf = c_resample(lib, o, x[pos:pos + c])
                out.append(buf[:n].copy())
                pos += c
        else:
            m = lib.resampleObj_calDataLength(o, x.size)
            n, buf = c_resample(lib, o, x, case_init(kw, m))
            assert n == m, (name, n, m)
            out.append(buf[:n].copy())
    finally:
        lib.resampleObj_free(o)
    return out
