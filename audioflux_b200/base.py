"""Common plumbing of the host-side mirror classes (reference: python/audioflux/base.py:4-8): the object lifecycle, the
array getters, the batched-call path, the per-clip loop of the reference-style methods and the argument defaults
several classes share."""
from __future__ import annotations

import ctypes as C
import warnings

import numpy as np

from . import lib as _libmod
from .types import enum_value

MEM_HOST, MEM_DEVICE = 0, 1
C1_HZ = 32.703196                # note_to_hz('C1'), the default lower edge of the Octave / Log scales


class Base(object):
    _free = None                     # the C free function, set once the constructor has succeeded

    def __init__(self, _lib=None):
        self._lib = _libmod.get_lib() if _lib is None else _lib
        self._obj = C.c_void_p()
        self._is_product = _lib is None or hasattr(self._lib, "afb200_version")

    def _new(self, new_name, free_name, *args):
        """self._obj = new_name(&obj, *args); ValueError on a non-zero status or a NULL object, with the library's
        recorded reason when it has one (product library)"""
        status = getattr(self._lib, new_name)(C.byref(self._obj), *args)
        if status != 0 or not self._obj:
            reason = (self._lib.afb200_lastError() or b"").decode() if self._is_product else ""
            raise ValueError(f"{new_name} failed with status {status}" + (f": {reason}" if reason else ""))
        self._free = getattr(self._lib, free_name)

    def __del__(self):
        free, self._free = self._free, None
        if free is not None:
            free(self._obj)

    def _require_ext(self, name):
        if not hasattr(self._lib, name):
            raise AttributeError(f"library does not export the additive entry point {name} "
                                 f"(include/afb200_ext.h); it is not libaudioflux_b200")
        return getattr(self._lib, name)

    def _array(self, fn_name, ctype, n):
        p = getattr(self._lib, fn_name)(self._obj)
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(ctype)), shape=(n,)).copy()

    def _floats(self, fn_name, n):
        """copy of the n floats the getter fn_name(obj) points at"""
        return self._array(fn_name, C.c_float, n)

    def _ints(self, fn_name, n):
        return self._array(fn_name, C.c_int, n)

    def _call(self, name, batch, *args):
        """name(obj, *args, kind, stream) for a Batch; arrays and tensors among args are passed by address"""
        fn = self._require_ext(name)
        _libmod.check(fn(self._obj, *map(_arg, args), batch.kind, batch.stream), name)


def _arg(a):
    if isinstance(a, np.ndarray):
        return np_ptr(a)
    if is_torch(a):
        return C.c_void_p(a.data_ptr())
    return a


class Batch:
    """The first operand of a batched call, flattened to x [rows, n], with what the call's other planes need: the lead
    shape, the memory kind and stream (numpy: host, torch: its CUDA device and current stream), alloc and second."""

    def __init__(self, x):
        if is_torch(x):
            import torch
            if not x.is_cuda:
                raise ValueError("torch inputs must live on a CUDA device; pass numpy arrays for host data")
            x = x.contiguous().float()
            self.kind, self.device = MEM_DEVICE, x.device
            self.stream = C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)
        else:
            x = as_f32(x)
            self.kind, self.device, self.stream = MEM_HOST, None, C.c_void_p(None)
        self.lead = tuple(x.shape[:-1])
        self.x = x.reshape(-1, x.shape[-1])
        self.rows, self.n = self.x.shape

    def alloc(self, *shape, zero=False):
        """float32 output in the operand's memory; zero=True where the library adds into it"""
        if self.kind == MEM_HOST:
            return (np.zeros if zero else np.empty)(shape, np.float32)
        import torch
        return (torch.zeros if zero else torch.empty)(shape, dtype=torch.float32, device=self.device)

    def second(self, operand, what, shape=None):
        """Another input plane of the call, flattened the same way (to one axis when `shape` has one).  ValueError
        unless it lives where the first operand does and its flattened shape is `shape` (default: the first's)."""
        other = Batch(operand)
        if (other.kind, other.device) != (self.kind, self.device):
            raise ValueError(f"{what} must live in the same memory as the first operand")
        want = self.x.shape if shape is None else shape
        flat = other.x.reshape(-1) if len(want) == 1 else other.x
        if tuple(flat.shape) != tuple(want):
            raise ValueError(f"{what} flattens to {tuple(flat.shape)}, {tuple(want)} is needed")
        return flat

    def shaped(self, out):
        """an output [rows, ...] as [*lead, ...]"""
        return None if out is None else out.reshape(*self.lead, *out.shape[1:])


def per_clip(fn, x, clip_ndim=1, y=None):
    """fn(clip) -> tuple of planes, for every clip of x [..., *clip] (clip_ndim trailing axes) -> tuple of the
    stacked planes [..., *plane].  With y [..., k] (the same lead axes), fn(clip, y_clip)."""
    lead = x.shape[:x.ndim - clip_ndim]
    clips = x.reshape(-1, *x.shape[len(lead):])
    res = [fn(*c) for c in (zip(clips) if y is None else zip(clips, y.reshape(len(clips), -1)))]
    return tuple(np.stack(p).reshape(*lead, *p[0].shape) for p in zip(*res))


def fit_length(data_arr, n, warn):
    """data [..., m] as contiguous float32, zero-padded or truncated to n samples; warn=True gives the reference's
    warnings (python/audioflux/utils/util.py:98-110)"""
    x = np.asarray(data_arr, dtype=np.float32, order='C')
    if x.ndim == 0:
        raise ValueError('Audio data must have at least one dimension')
    m = x.shape[-1]
    if m < n:
        if warn:
            warnings.warn(f'The audio length={m} is not enough for fft_length={n}(2**radix2_exp), '
                          f'and {n - m} zeros are automatically filled after the audio')
        x = np.pad(x, (*[(0, 0)] * (x.ndim - 1), (0, n - m)))
    elif m > n:
        if warn:
            warnings.warn(f'fft_length={n}(2**radix2_exp) is too small for data_arr length={m}, '
                          f'only the first fft_length={n} data are valid')
        x = x[..., :n]
    return as_f32(x)


def is_log_scale(scale_type):
    """Octave and Log filter-bank scales"""
    return enum_value(scale_type) in (5, 6)


def band_range(low_fre, high_fre, scale_type, samplate):
    """the reference's band edges: low_fre defaults to C1 on the Octave / Log scales, else 0; high_fre to samplate/2"""
    if low_fre is None:
        low_fre = C1_HZ if is_log_scale(scale_type) else 0.0
    return low_fre, samplate / 2 if high_fre is None else high_fre


class BandAxis:
    """Plot-axis helper of the banded transforms (reference: the y_coords of bft.py / cqt.py / cwt.py / pwt.py / wsst.py):
    the band frequencies with the lower edge in front."""

    def y_coords(self):
        return np.concatenate(([self.low_fre], self.get_fre_band_arr()))


class FrameAxis:
    """Time axis of a framed transform: data_length / samplate seconds cut into cal_time_length frames."""
    _needs_full_frame = True

    def x_coords(self, data_length):
        if self._needs_full_frame and data_length < self.fft_length:
            raise ValueError(f"radix2_exp={self.radix2_exp}(fft_length={self.fft_length}) is too large for data_length={data_length}")
        return np.linspace(0, data_length / self.samplate, self.cal_time_length(data_length) + 1)


class PitchBase(FrameAxis, Base):
    """The body of the frame-wise pitch trackers (PitchPEF, PitchYIN, PitchNCF, PitchCEP): the constructor call,
    cal_time_length and the batched pitch call of the C object named by _prefix.  {_prefix}_pitchBatch fills _planes
    output planes [rows, T]; _zero: they start at 0 (in-out planes whose frames without a result keep their value);
    _unset: trailing optional outputs passed as NULL."""
    _prefix = ""
    _planes, _zero, _unset = 1, False, ()

    def _open(self, radix2_exp, *args):
        """{_prefix}_new(&obj, *args) and fft_length"""
        self._new(f"{self._prefix}_new", f"{self._prefix}_free", *args)
        # the frame: 2**radix2_exp, or the reference's fallback 2**12 outside 1 .. 30
        self.fft_length = 1 << (int(radix2_exp) if 1 <= radix2_exp <= 30 else 12)

    def cal_time_length(self, data_length):
        return getattr(self._lib, f"{self._prefix}_calTimeLength")(self._obj, int(data_length))

    def pitch_batch(self, data):
        """data [..., n] (numpy host | torch cuda) -> the output planes, each [..., cal_time_length(n)] float32 of the
        same kind (a tuple when there are several).  One batched call for all channels; each row is bit-identical to a
        legacy call."""
        b = Batch(data)
        t = self.cal_time_length(b.n)
        out = [b.alloc(b.rows, t, zero=self._zero) for _ in range(self._planes)]
        if b.rows and t:
            self._call(f"{self._prefix}_pitchBatch", b, b.x, b.n, b.rows, *out, *self._unset)
        out = tuple(b.shaped(o) for o in out)
        return out if self._planes > 1 else out[0]

    def pitch(self, data_arr):
        """data_arr [..., n] -> pitch_batch's planes, each [..., time] float32"""
        data_arr = np.asarray(data_arr, dtype=np.float32, order='C')
        if data_arr.ndim == 0:
            raise ValueError('Audio data must have at least one dimension')
        if data_arr.shape[-1] == 0:
            raise ValueError('Audio data must not be empty')
        return self.pitch_batch(data_arr)


def c_int(v):
    """a pointer to the int v (the constructors' NULL-able arguments, always given here)"""
    return C.byref(C.c_int(int(v)))


def c_float(v):
    return C.byref(C.c_float(float(v)))


class SampleAxis:
    """Time axis of a per-sample transform (CWT family): one column per sample of the 2**radix2_exp window; and the
    family's batched call."""

    def x_coords(self):
        return np.linspace(0, self.fft_length / self.samplate, self.fft_length + 1)

    def _window_batch(self, name, data, *args):
        """data [..., fft_length] -> (re, im) each [..., num, fft_length] from name(obj, x, rows, *args, re, im, ...)"""
        b = Batch(data)
        if b.n != self.fft_length:
            raise ValueError(f"data length must be 2**radix2_exp = {self.fft_length}")
        re, im = b.alloc(b.rows, self.num, b.n), b.alloc(b.rows, self.num, b.n)
        self._call(name, b, b.x, b.rows, *args, re, im)
        return b.shaped(re), b.shaped(im)


def as_f32(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32))


def np_ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def is_torch(x) -> bool:
    return type(x).__module__.startswith("torch")


def swap_last2(a):
    if is_torch(a):
        return a.transpose(-1, -2).contiguous()
    return np.ascontiguousarray(np.swapaxes(a, -1, -2))
