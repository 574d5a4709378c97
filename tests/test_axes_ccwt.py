"""Plot-axis helpers (x_coords / y_coords) and CWT.ccwt of the host-side mirror classes against the reference's own
Python package (python/audioflux/{bft,cqt,cwt,stft,pwt,wsst}.py, cwt.py:280-320), both bound to the reference build on
the CPU; the product library's ccwt (one cwtObj_cwtBatch call over all windows) against that on the GPU."""
import numpy as np
import pytest

from conftest import noise, rel_max

from oracle import ref_lib as R
from oracle import ref_python as RP


@pytest.fixture(scope="module")
def raf(ref_lib):
    if not RP.available():
        pytest.skip("oracle/_ref/pyref not built (make -C oracle REF=<audioFlux tree>)")
    import os
    from conftest import ROOT
    mod = RP.load(R.REF_PATH, os.path.join(ROOT, "audioflux_b200", "lib", "libaudioflux_b200.so"))
    mod.fftlib.set_fft_lib(None)
    return mod


def test_axis_helpers_match_the_reference_package(raf, ref_lib):
    import audioflux_b200 as af
    T = raf.type
    pairs = [
        (af.BFT(64, 10, 16000, _lib=ref_lib), raf.BFT(num=64, radix2_exp=10, samplate=16000), (5000,)),
        (af.CQT(84, 32000, _lib=ref_lib), raf.CQT(num=84, samplate=32000), (5000,)),
        (af.CWT(40, 11, 16000, _lib=ref_lib), raf.CWT(num=40, radix2_exp=11, samplate=16000), ()),
        (af.PWT(40, 11, 16000, _lib=ref_lib), raf.PWT(num=40, radix2_exp=11, samplate=16000), ()),
        (af.WSST(40, 11, 16000, _lib=ref_lib), raf.WSST(num=40, radix2_exp=11, samplate=16000), ()),
    ]
    for mine, ref, xargs in pairs:
        np.testing.assert_allclose(mine.y_coords(), ref.y_coords(), rtol=1e-6)
        np.testing.assert_allclose(mine.x_coords(*xargs), ref.x_coords(*xargs), rtol=1e-12)
    ms, rs = af.MelSpectrogram(64, 16000, radix2_exp=10, _lib=ref_lib), raf.MelSpectrogram(num=64, samplate=16000, radix2_exp=10)
    np.testing.assert_allclose(ms.y_coords(), rs.y_coords(), rtol=1e-6)
    np.testing.assert_allclose(ms.x_coords(5000), rs.x_coords(5000), rtol=1e-12)
    s, q = af.STFT(10, _lib=ref_lib), raf.STFT(radix2_exp=10)
    np.testing.assert_allclose(s.y_coords(16000), q.y_coords(16000))
    np.testing.assert_allclose(s.x_coords(5000, 16000), q.x_coords(5000, 16000))
    with pytest.raises(ValueError):
        s.x_coords(100)
    with pytest.raises(ValueError):
        pairs[0][0].x_coords(100)
    assert len(pairs[1][0].x_coords(100)) == pairs[1][0].cal_time_length(100) + 1      # CQT pads: any length is legal


@pytest.mark.parametrize("shape,r", [((12388,), 12), ((2, 3, 6000), 10), ((4096,), 11)])
def test_ccwt_splicing_matches_the_reference_package(raf, ref_lib, shape, r):
    import audioflux_b200 as af
    x = noise(31, int(np.prod(shape))).reshape(shape)
    kw = dict(num=24, radix2_exp=r, samplate=16000)
    want = raf.CWT(wavelet_type=raf.type.WaveletContinueType.MORLET, **kw).ccwt(x)
    got = af.CWT(wavelet_type=af.WaveletContinueType.MORLET, _lib=ref_lib, **kw).ccwt(x)
    assert got.shape == want.shape and np.iscomplexobj(got)
    assert np.array_equal(got, want)                                   # same library, same windows: identical
    with pytest.raises(ValueError):
        af.CWT(_lib=ref_lib, **kw).ccwt(x[..., :(1 << r) - 1])


@pytest.mark.gpu
@pytest.mark.parametrize("shape,r,wavelet", [((12388,), 12, "MORLET"), ((3, 9000), 10, "MORSE"), ((2, 40000), 13, "MORLET")])
def test_ccwt_on_the_gpu(cuda_device, ref_lib, shape, r, wavelet):
    """all windows of all clips through one cwtObj_cwtBatch call == the reference build window by window"""
    import audioflux_b200 as af
    x = noise(32, int(np.prod(shape))).reshape(shape)
    kw = dict(num=36, radix2_exp=r, samplate=16000, wavelet_type=getattr(af.WaveletContinueType, wavelet))
    got = af.CWT(**kw).ccwt(x)
    want = af.CWT(_lib=ref_lib, **kw).ccwt(x)
    assert got.shape == want.shape
    assert float(np.abs(got - want).max() / np.abs(want).max()) < 1e-4
