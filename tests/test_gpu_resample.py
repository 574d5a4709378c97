"""Resampler on the GPU: every oracle case through the legacy call (into zeroed and non-zero buffers, continue mode fed
chunk by chunk) and the batch against the float64 oracle and the reference build; the batch bit-identical to the legacy
call into zeroed buffers with host and device pointers, across staging chunks, for ratios down to 2^-nbit and for
upsampling by 6; a clip longer than 2^24 samples; device calls at different ratios queued back to back; the launch
count; the refusals; and the reference's own Resample / WindowResample classes running on libaudioflux_b200.so."""
import numpy as np
import pytest

import _resample_oracle as RO
from _parity_kit import Out, count_launches, dptr, ref_lib_or_none, run_batch, stream
from _parity_kit import raf  # noqa: F401  (a fixture)

import audioflux_b200 as af

pytestmark = pytest.mark.gpu
TOL = 1e-4          # per tensor: max|got - want| <= TOL * max|want|
CASES = dict(RO.cases())


def _check(got, want, what):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if got.size:
        err = np.abs(np.asarray(got, np.float64) - want).max() / max(np.abs(want).max(), 1e-30)
        assert err <= TOL, (what, err)


def _batch(lib, o, x, device):
    """resampleObj_resampleBatch on x [batch, n] -> [batch, m] numpy"""
    x = np.ascontiguousarray(x, np.float32)
    b, n = x.shape
    m = lib.resampleObj_calDataLength(o, n)
    return run_batch(lib, "resampleObj_resampleBatch", (o, x, n, b, Out(np.full((b, m), 7.0, np.float32))), device)[0]


def _legacy_rows(lib, o, x):
    rows = []
    for row in np.atleast_2d(x):
        n, buf = RO.c_resample(lib, o, row)
        rows.append(buf[:n])
    return np.stack(rows)


@pytest.mark.parametrize("name", [n for n in CASES if n != "big_fast"])
def test_case_matches_oracle_and_reference(product_lib, cuda_device, name):
    kw = CASES[name]
    got = RO.c_case(product_lib, name, kw)
    assert product_lib.afb200_lastError() in (b"", None)
    want = RO.oracle_case(name, kw)
    ref = ref_lib_or_none()
    refs = RO.c_case(ref, name, kw) if ref is not None else None
    for k, (g, w) in enumerate(zip(got, want)):
        _check(g, w, (name, k, "oracle"))
        if refs is not None:
            _check(g, refs[k].astype(np.float64), (name, k, "reference"))
    if "chunks" in kw:
        return
    # the batch, host and device pointers, against the legacy call into a zeroed buffer and the oracle
    st, o = RO.c_new(product_lib, kw.get("qual"), kw.get("window"), kw.get("is_scale", 0))
    RO.c_apply(product_lib, o, kw["ops"])
    x = RO.case_signal(name, kw)
    legacy = _legacy_rows(product_lib, o, x)
    for device in (False, True):
        b = _batch(product_lib, o, np.stack([x, x[::-1]]), device)
        assert np.array_equal(b[0], legacy[0]), (name, device)
        assert np.array_equal(b[1], _legacy_rows(product_lib, o, x[::-1])[0]), (name, device)
    if kw.get("init") is None:
        _check(legacy[0], want[0], (name, "batch oracle"))
    product_lib.resampleObj_free(o)


def test_clip_beyond_2_24_samples(product_lib, cuda_device):
    """positions above 2^24 fall on the float grid of the reference's t: the same outputs as the reference build"""
    name, kw = "big_fast", CASES["big_fast"]
    got = RO.c_case(product_lib, name, kw)[0]
    assert got.size == int(np.floor(np.float32(RO.BIG) * np.float32(1 / 3)))
    _check(got, RO.oracle_case(name, kw)[0], "oracle")
    ref = ref_lib_or_none()
    if ref is not None:
        _check(got, RO.c_case(ref, name, kw)[0].astype(np.float64), "reference")
    st, o = RO.c_new(product_lib, 2)
    RO.c_apply(product_lib, o, kw["ops"])
    assert np.array_equal(_batch(product_lib, o, RO.case_signal(name, kw)[None], True)[0], got)
    product_lib.resampleObj_free(o)


def test_batch_across_staging_chunks_and_launch_count(product_lib, cuda_device):
    import torch
    r = af.Resample("best")
    r.set_samplate(48000, 16000)
    rng = np.random.default_rng(3)
    x = (0.1 * rng.standard_normal((20, 1_200_000))).astype(np.float32)      # 4.8 MB clips: 13 per 64 MB chunk
    host = {}
    assert count_launches(product_lib, lambda: host.setdefault("o", r.resample_batch(x)), warm=False) == 2
    xd = torch.from_numpy(x).cuda()
    dev = {}
    assert count_launches(product_lib, lambda: dev.setdefault("o", r.resample_batch(xd)), warm=False) == 1
    assert np.array_equal(dev["o"].cpu().numpy(), host["o"])
    for k in (0, 12, 13, 19):
        n, buf = RO.c_resample(product_lib, r._obj, x[k])
        assert np.array_equal(host["o"][k], buf[:n]), k
    assert count_launches(product_lib, lambda: r.resample(x[:1, :5000]), warm=False) == 1


@pytest.mark.parametrize("qual", [0, 2])
def test_ratios_down_to_2_pow_minus_nbit(product_lib, cuda_device, qual):
    x = RO.case_signal("low", dict(length=30000))[None]
    for ratio in (2.0 ** -9, 0.0021, 0.004, 0.013, 0.11):
        st, o = RO.c_new(product_lib, qual)
        product_lib.resampleObj_setSamplateRatio(o, ratio)
        legacy = _legacy_rows(product_lib, o, x)
        for device in (False, True):
            assert np.array_equal(_batch(product_lib, o, x, device), legacy), (qual, ratio, device)
        r = RO.Resampler(qual)
        r.set_ratio(ratio)
        _check(legacy[0], r.resample(x[0]), (qual, ratio, "oracle"))
        product_lib.resampleObj_free(o)


def test_upsampling_by_6(product_lib, cuda_device):
    x = np.stack([RO.case_signal("up6", dict(length=7001)), RO.case_signal("up6b", dict(length=7001))])
    r = af.Resample("mid")
    r.set_samplate(8000, 48000)
    assert r.cal_data_length(7001) == 6 * 7001
    got = r.resample(x)
    assert got.shape == (2, 6 * 7001)
    assert np.array_equal(got, _legacy_rows(product_lib, r._obj, x))
    o = RO.Resampler(1)
    o.set_samplate(8000, 48000)
    for k in range(2):
        _check(got[k], o.resample(x[k]), k)


def test_device_calls_at_different_ratios_back_to_back(product_lib, cuda_device):
    """each table rebuild waits for the kernels queued before it that read the old table"""
    import torch
    x = np.stack([RO.case_signal(f"b2b{k}", dict(length=400_000)) for k in range(8)])
    xd = torch.from_numpy(x).cuda()
    r = af.Resample("best")
    outs, rates = [], [(48000, 16000), (16000, 44100), (44100, 16000), (22050, 8000)]
    for s, d in rates:
        r.set_samplate(s, d)
        outs.append(r.resample_batch(xd))                 # no synchronise between the calls
    torch.cuda.synchronize()
    for (s, d), got in zip(rates, outs):
        fresh = af.Resample("best")
        fresh.set_samplate(s, d)
        want = fresh.resample(x[:2])
        o = RO.Resampler(0)
        o.set_samplate(48000, 16000)
        for s2, d2 in rates[1:rates.index((s, d)) + 1]:
            o.set_samplate(s2, d2)
        _check(got[0].cpu().numpy(), o.resample(x[0]), (s, d, "oracle"))
        # the table's history differs between the two objects only in the last bits
        _check(got[:2].cpu().numpy(), want.astype(np.float64), (s, d, "fresh object"))


def test_refusals_on_the_device(product_lib, cuda_device):
    import torch
    xd = torch.from_numpy(RO.case_signal("ref", dict(length=5000))).cuda()
    st, o = RO.c_new(product_lib, 0)
    product_lib.resampleObj_setSamplateRatio(o, 0.0019)                      # 0.0019 * 512 < 1
    out = torch.full((64,), 7.0, device="cuda")
    assert product_lib.resampleObj_resampleBatch(o, dptr(xd), 5000, 1, dptr(out), 1, stream()) != 0
    assert b"below 1" in product_lib.afb200_lastError()
    product_lib.resampleObj_setSamplate(o, 16000, 48000)
    product_lib.resampleObj_enableContinue(o, 1)                             # q = 1
    assert product_lib.resampleObj_resampleBatch(o, dptr(xd), 5000, 1, dptr(out), 1, stream()) != 0
    torch.cuda.synchronize()
    assert (out == 7.0).all()
    product_lib.resampleObj_free(o)


def test_reference_classes_on_b200(raf, cuda_device):
    mono = RO.case_signal("mono", dict(length=9000))
    multi = (0.1 * np.random.default_rng(5).standard_normal((2, 3, 4000))).astype(np.float32)
    res = {}
    for which in ("ref", "b200"):
        raf.fftlib.set_fft_lib(lib_ext="b200" if which == "b200" else None)
        a = raf.Resample(qual_type="mid", is_scale=True)
        a.set_samplate(44100, 16000)
        w = raf.WindowResample(zero_num=32, nbit=8, win_type=raf.type.WindowType.BLACKMAN, roll_off=0.9)
        w.set_samplate(16000, 48000)
        res[which] = [a.resample(mono), a.resample(multi), w.resample(mono), w.resample(multi)]
    raf.fftlib.set_fft_lib(None)
    a = af.Resample(qual_type="mid", is_scale=True)
    a.set_samplate(44100, 16000)
    w = af.WindowResample(zero_num=32, nbit=8, win_type=af.WindowType.BLACKMAN, roll_off=0.9)
    w.set_samplate(16000, 48000)
    own = [a.resample(mono), a.resample(multi), w.resample(mono), w.resample(multi)]
    for k in range(4):
        g, r = res["b200"][k], res["ref"][k]
        assert g.shape == r.shape == own[k].shape, k
        _check(g, r.astype(np.float64), k)
        assert np.array_equal(own[k], g), k
