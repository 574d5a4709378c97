"""The shared plumbing of the Python mirror classes (audioflux_b200/base.py): constructor failures and their messages,
teardown, the second-operand check of the batched calls and the reference's pad / truncate warnings.  No GPU needed."""
import warnings

import numpy as np
import pytest

import audioflux_b200 as af
from audioflux_b200.base import Base, fit_length
from audioflux_b200.types import SpectralFilterBankStyleType


@pytest.mark.parametrize("make, name", [
    # classes that used to report the status only
    (lambda: af.STFT(radix2_exp=31), "stftObj_new"),
    (lambda: af.Synsq(0, 9), "synsqObj_new"),
    # classes that used to add the recorded reason for status -2 only
    (lambda: af.Cepstrogram(radix2_exp=20), "cepstrogramObj_new"),
    (lambda: af.Cepstrogram(radix2_exp=31), "cepstrogramObj_new"),
    (lambda: af.NSGT(num=8, radix2_exp=31), "nsgtObj_new"),
    # classes that used to add it for any non-zero status
    (lambda: af.WindowResample(win_type=99), "resampleObj_newWithWindow"),
])
def test_failed_constructor_raises_with_status(product_lib, make, name):
    with pytest.raises(ValueError) as e:
        make()
    assert str(e.value).startswith(f"{name} failed with status ")


def test_recorded_reason_is_appended(product_lib):
    with pytest.raises(ValueError, match=r"^cepstrogramObj_new failed with status -100: cepstrogramObj_new: radix2Exp=31"):
        af.Cepstrogram(radix2_exp=31)
    with pytest.raises(ValueError, match=r"^resampleObj_newWithWindow failed with status -1: .*winType=99"):
        af.WindowResample(win_type=99)


def test_failure_does_not_carry_an_earlier_reason(product_lib):
    with pytest.raises(ValueError, match="Gammatone") as first:
        af.PWT(32, 9, style_type=SpectralFilterBankStyleType.GAMMATONE)
    reason = str(first.value).split(": ", 1)[1]
    # fstObj_new refuses radix2Exp < 3 without recording a reason; FST's own range checks stop that case earlier
    with pytest.raises(ValueError) as second:
        Base()._new("fstObj_new", "fstObj_free", 2)
    assert str(second.value) == "fstObj_new failed with status -1"
    assert reason not in str(second.value)
    with pytest.raises(ValueError) as third:
        af.STFT(radix2_exp=31)
    assert str(third.value) == "stftObj_new failed with status -100"


class _FakeLib:
    """a C library whose fooObj_new fails or succeeds on request and counts fooObj_free calls"""

    def __init__(self, status, obj):
        self.status, self.obj, self.freed = status, obj, []

    def fooObj_new(self, ref):
        self.obj._obj.value = 0x1000 if self.status == 0 else None
        return self.status

    def fooObj_free(self, handle):
        self.freed.append(handle.value)


def _half_built(status):
    obj = Base.__new__(Base)
    lib = _FakeLib(status, obj)
    Base.__init__(obj, _lib=lib)
    return obj, lib


def test_del_frees_once_and_never_after_a_failed_constructor():
    obj, lib = _half_built(-3)
    with pytest.raises(ValueError, match=r"^fooObj_new failed with status -3$"):
        obj._new("fooObj_new", "fooObj_free")
    obj.__del__()
    assert lib.freed == []

    obj, lib = _half_built(0)
    obj._new("fooObj_new", "fooObj_free")
    obj.__del__()
    obj.__del__()
    assert lib.freed == [0x1000]


def test_del_of_an_object_stopped_before_its_constructor():
    b = af.BFT.__new__(af.BFT)
    with pytest.raises(ValueError, match="too large"):
        b.__init__(10 ** 6, 10)
    b.__del__()                                   # no C object and no free function: nothing to do
    assert b._free is None


def _no_library_call(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("the library was called")
    monkeypatch.setattr(Base, "_call", refuse)


def _second_operand_cases():
    rng = np.random.default_rng(0)
    re = rng.standard_normal((2, 5, 513)).astype(np.float32)
    m = np.abs(rng.standard_normal((2, 5, 40))).astype(np.float32) + 0.1
    cq = rng.standard_normal((2, 5, 84)).astype(np.float32)
    # (method, object, call(obj, first, second), first, a matching second, a second of another flattened shape)
    return [
        ("istft_batch", lambda: af.STFT(10), lambda o, a, b: o.istft_batch(a, b), re, re, re[:, :4]),
        ("chroma_batch", lambda: af.CQT(84), lambda o, a, b: o.chroma_batch(a, b), cq, cq, cq[:, :, :80]),
        ("cepstrogram2_batch", lambda: af.Cepstrogram(10), lambda o, a, b: o.cepstrogram2_batch(a, b), re, re, re[:1]),
        ("xxcc_standard_batch", lambda: af.XXCC(40), lambda o, a, b: o.xxcc_standard_batch(a, b), m, m[..., 0],
         m[:, :4, 0]),
        ("spectral_batch", lambda: af.Spectral(40, np.arange(40.)),
         lambda o, a, b: o.spectral_batch(a, ["pd"], phase=b), m, m, m[:, :, :39]),
    ]


_CASE_IDS = dict(ids=lambda v: v if isinstance(v, str) else None)


@pytest.mark.parametrize("name, make, call, first, good, bad", _second_operand_cases(), **_CASE_IDS)
def test_second_operand_shape_is_checked_before_the_library(product_lib, monkeypatch, name, make, call, first, good, bad):
    obj = make()
    _no_library_call(monkeypatch)
    with pytest.raises(ValueError, match="flattens to"):
        call(obj, first, bad)
    with pytest.raises(AssertionError, match="the library was called"):
        call(obj, first, good)                    # a matching operand gets as far as the library call


@pytest.mark.gpu
@pytest.mark.parametrize("name, make, call, first, good, bad", _second_operand_cases(), **_CASE_IDS)
def test_host_second_operand_next_to_a_device_first_is_refused(cuda_device, monkeypatch, name, make, call, first, good,
                                                               bad):
    import torch
    obj = make()
    _no_library_call(monkeypatch)
    first_d = torch.from_numpy(first).cuda()
    with pytest.raises(ValueError, match="must live in the same memory"):
        call(obj, first_d, good)
    with pytest.raises(AssertionError, match="the library was called"):
        call(obj, first_d, torch.from_numpy(np.ascontiguousarray(good)).cuda())


def test_fit_length_warnings():
    x = np.ones((2, 3, 100), np.float32)
    with pytest.warns(UserWarning) as w:
        y = fit_length(x, 128, warn=True)
    assert [str(r.message) for r in w] == ["The audio length=100 is not enough for fft_length=128(2**radix2_exp), "
                                           "and 28 zeros are automatically filled after the audio"]
    assert y.shape == (2, 3, 128) and y.dtype == np.float32 and not y[..., 100:].any()
    with pytest.warns(UserWarning) as w:
        y = fit_length(x, 64, warn=True)
    assert [str(r.message) for r in w] == ["fft_length=64(2**radix2_exp) is too small for data_arr length=100, "
                                           "only the first fft_length=64 data are valid"]
    assert y.shape == (2, 3, 64) and y.flags["C_CONTIGUOUS"]
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        assert fit_length(x, 100, warn=True).shape == x.shape
        assert fit_length(x, 128, warn=False).shape == (2, 3, 128)
        assert fit_length(x, 64, warn=False).shape == (2, 3, 64)
    with pytest.raises(ValueError, match="at least one dimension"):
        fit_length(np.float32(1), 64, warn=True)


@pytest.mark.parametrize("make, method, warns", [
    (lambda: af.NSGT(num=48, radix2_exp=10), "nsgt", True),
    (lambda: af.ST(10), "st", True),
    (lambda: af.FST(10), "fst", True),
    (lambda: af.CWT(num=32, radix2_exp=10), "cwt", False),
    (lambda: af.PWT(num=32, radix2_exp=10), "pwt", False),
    (lambda: af.WSST(num=32, radix2_exp=10), "wsst", False),
])
def test_which_methods_warn(product_lib, monkeypatch, make, method, warns):
    """NSGT, ST and FST warn as the reference does when they pad or truncate; CWT, PWT and WSST do it silently"""
    obj = make()
    n = obj.fft_length
    if warns:
        monkeypatch.setattr(type(obj), f"{method}_batch", lambda self, x: (x, x))
    else:
        planes = 4 if method == "wsst" else 2
        monkeypatch.setattr(type(obj), f"{method}_planes",
                            lambda self, x: tuple(np.zeros((self.num, n), np.float32) for _ in range(planes)))
    for length in (n - 100, n + 100):
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            getattr(obj, method)(np.ones((2, length), np.float32))
        assert len(w) == (1 if warns else 0), [str(r.message) for r in w]
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        getattr(obj, method)(np.ones((2, n), np.float32))
    assert not w
