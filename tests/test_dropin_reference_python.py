"""The drop-in claim of INTEGRATION.md section 1, proven with the reference's OWN Python package (unmodified
python/audioflux, byte-compiled into oracle/_ref/pyref by `make -C oracle`): after
`audioflux.fftlib.set_fft_lib(lib_ext='b200')` (python/audioflux/fftlib.py:96-124) its BFT / XXCC / CQT / CWT /
MelSpectrogram classes run on libaudioflux_b200.so and return what the reference build returns."""
import os

import numpy as np
import pytest

from conftest import ROOT, noise, tones, rel_max

from oracle import af_oracle as O
from oracle import ref_lib as R
from oracle import ref_python as RP

TOL = 1e-4
B200 = os.path.join(ROOT, "audioflux_b200", "lib", "libaudioflux_b200.so")


@pytest.fixture(scope="module")
def raf(product_lib):
    """the reference package, default library = the reference build, lib_ext 'b200' = the product"""
    if not (RP.available() and R.available()):
        pytest.skip("oracle/_ref/pyref or oracle/_ref/libaudioflux_ref.so not built (make -C oracle REF=<audioFlux tree>)")
    mod = RP.load(R.REF_PATH, B200)
    yield mod
    mod.fftlib.set_fft_lib(None)


def _use(raf, which):
    raf.fftlib.set_fft_lib(lib_ext="b200" if which == "b200" else None)
    assert raf.fftlib.get_fft_lib_fp().endswith("libaudioflux_b200.so" if which == "b200" else "libaudioflux.so")


def test_reference_package_binds_the_product_library(raf):
    """CPU-only: objects are created through the reference classes on libaudioflux_b200.so and the setup-time getters
    agree with the reference build (no compute call, so no GPU needed)."""
    T = raf.type
    out = {}
    for which in ("ref", "b200"):
        _use(raf, which)
        b = raf.BFT(num=128, radix2_exp=11, samplate=48000, slide_length=512, scale_type=T.SpectralFilterBankScaleType.MEL,
                    data_type=T.SpectralDataType.POWER)
        c = raf.CQT(num=84, samplate=48000)
        w = raf.CWT(num=84, radix2_exp=12, samplate=48000, wavelet_type=T.WaveletContinueType.MORLET)
        s = raf.MelSpectrogram(num=128, samplate=48000, radix2_exp=11, slide_length=512)
        out[which] = (b.get_fre_band_arr(), b.get_bin_band_arr(), b.cal_time_length(48000), c.get_fre_band_arr(),
                      c.cal_time_length(240000), w.get_fre_band_arr(), s.get_fre_band_arr(), s.cal_time_length(48000))
    for a, b in zip(out["ref"], out["b200"]):
        np.testing.assert_allclose(np.asarray(a, np.float64), np.asarray(b, np.float64), rtol=1e-6)


@pytest.mark.gpu
def test_reference_bft_xxcc_on_b200(raf, cuda_device, golden):
    T = raf.type
    g = golden("c1_mel_mfcc.npz")
    x = g["x"] if "x" in g.files else noise(11, 48000)
    res = {}
    for which in ("ref", "b200"):
        _use(raf, which)
        b = raf.BFT(num=128, radix2_exp=11, samplate=48000, slide_length=512, scale_type=T.SpectralFilterBankScaleType.MEL,
                    data_type=T.SpectralDataType.POWER)
        mel = b.bft(x, result_type=1)                      # [num, T]
        xx = raf.XXCC(num=128)
        xx.set_time_length(mel.shape[-1])
        cc = xx.xxcc(mel, cc_num=40)
        res[which] = (mel, cc)
    assert res["b200"][0].shape == res["ref"][0].shape == (128, O.stft_time_length(len(x), 2048, 512))
    assert rel_max(res["b200"][0], res["ref"][0]) < TOL
    assert rel_max(res["b200"][1], res["ref"][1]) < TOL
    assert rel_max(res["b200"][1].T, O.mfcc(x, 48000, 11, 512, 128, 40)) < TOL


@pytest.mark.gpu
def test_reference_cqt_cwt_on_b200(raf, cuda_device):
    T = raf.type
    x = tones(5, 48000, 48000)
    xw = noise(6, 4096)
    res = {}
    for which in ("ref", "b200"):
        _use(raf, which)
        c = raf.CQT(num=84, samplate=48000)
        w = raf.CWT(num=84, radix2_exp=12, samplate=48000, wavelet_type=T.WaveletContinueType.MORLET)
        res[which] = (c.cqt(x), w.cwt(xw))
    for a, b in zip(res["b200"], res["ref"]):
        assert a.shape == b.shape and np.iscomplexobj(a)
        assert rel_max(np.abs(a - b), np.abs(b)) < 1.0 and float(np.abs(a - b).max() / np.abs(b).max()) < TOL


@pytest.mark.gpu
def test_reference_mel_spectrogram_mfcc_on_b200(raf, cuda_device):
    x = noise(9, 48000)
    res = {}
    for which in ("ref", "b200"):
        _use(raf, which)
        s = raf.MelSpectrogram(num=128, samplate=48000, radix2_exp=11, slide_length=512)
        spec = s.spectrogram(x)
        res[which] = (spec, s.mfcc(spec, cc_num=40))
    assert rel_max(res["b200"][0], res["ref"][0]) < TOL
    assert rel_max(res["b200"][1], res["ref"][1]) < TOL
