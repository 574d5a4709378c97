"""The numpy oracle against fixtures generated from the reference itself
(tests/golden/make_golden.py).  Runs everywhere (no GPU, no reference build)."""
import numpy as np

from conftest import rel_max
from oracle import af_oracle as O

TOL = 2e-5   # oracle (float64 math) vs reference (float32 radix-2 FFT, double-accumulated dots)


def test_c1_mel_and_mfcc(golden):
    g = golden("c1_mel_mfcc.npz")
    mel = O.bft(g["x"], 128, 11, 48000, 512, O.W_HANN, O.SCALE_MEL, O.STYLE_SLANEY, O.NORM_NONE, O.DATA_POWER, result_type=1)
    assert mel.shape == (90, 128)
    assert rel_max(mel, g["mel"]) < TOL
    # values recorded in SURVEY.md section 8(c)
    assert abs(float(g["mel"].sum()) - 698303.625) < 1.0
    np.testing.assert_allclose(g["mel"][0, :4], [7.165208, 15.285028, 15.125343, 7.3538113], rtol=1e-5)
    mf = O.xxcc(mel, 40)
    assert rel_max(mf, g["mfcc"]) < TOL
    np.testing.assert_allclose(g["mfcc"][0, :4], [17.20224, -5.007658, 0.2310224, -0.40099555], rtol=1e-4)


def test_c1_complex_mode(golden):
    g = golden("c1_mel_mfcc.npz")
    re, im = O.bft(g["x"], 128, 11, 48000, 512, O.W_HANN, O.SCALE_MEL, O.STYLE_SLANEY, O.NORM_NONE, O.DATA_POWER, result_type=0)
    assert rel_max(re, g["cre"]) < TOL and rel_max(im, g["cim"]) < TOL


def test_band_tables(golden):
    g = golden("c1_mel_mfcc.npz")
    _, fre, bins = O.auditory_filterbank(128, 2048, 48000, O.SCALE_MEL, O.STYLE_SLANEY, O.NORM_NONE, 0.0, 24000.0)
    assert np.array_equal(bins, g["bin_band"])
    np.testing.assert_allclose(fre, g["fre_band"], rtol=2e-6)


def test_bark_etsi_mag(golden):
    g = golden("bark_etsi_mag.npz")
    m = O.bft(g["x"], 64, 10, 48000, 256, O.W_HANN, O.SCALE_BARK, O.STYLE_ETSI, O.NORM_AREA, O.DATA_MAG, result_type=1)
    assert rel_max(m, g["mel"]) < TOL
    assert rel_max(O.xxcc(g["mel"], 20), g["cc"]) < TOL
    assert rel_max(O.xxcc(g["mel"], 13, O.RECT_CUBIC), g["cc_cubic"]) < TOL


def test_stft(golden):
    g = golden("stft_512.npz")
    re, im = O.stft(g["x"], 512, 128, O.fft_window(O.W_HANN, 512))
    assert re.shape[0] == int(g["T"])
    assert rel_max(re[:8], g["re"]) < TOL and rel_max(im[:8], g["im"]) < TOL


def test_cqt(golden):
    g = golden("cqt_84.npz")
    re, im = O.cqt(g["x"], 84, 48000, norm=O.NORM_AREA)
    assert re.shape == g["re"].shape
    assert rel_max(re, g["re"]) < TOL and rel_max(im, g["im"]) < TOL


def test_cwt(golden):
    g = golden("cwt_morlet.npz")
    re, im = O.cwt(g["x"], 36, 11, 48000, O.WAVE_MORLET, O.SCALE_OCTAVE, low=32.703196, is_pad=False)
    assert rel_max(re, g["re"]) < TOL and rel_max(im, g["im"]) < TOL


def test_gammatone_bank_and_path(golden):
    """The oracle's gammatone bank is a float32, libm-faithful restatement (the reference's values in the lowest bands are
    float32 rounding artefacts): bit-identical to the reference given its centre frequencies, within 2e-5 of a row's
    maximum from the oracle's own; then the BFT / cepstrum path with it."""
    g = golden("erb_gammatone.npz")
    assert np.array_equal(O.gammatone_bank(64, 1024, 32000, O.NORM_NONE, g["fre_band"]), g["bank"])
    bank, fre, bins = O.auditory_filterbank(64, 1024, 32000, O.SCALE_ERB, O.STYLE_GAMMATONE, O.NORM_NONE, 0.0, 16000.0)
    assert np.array_equal(bins, g["bin_band"])
    np.testing.assert_allclose(fre, g["fre_band"], rtol=2e-6)
    assert (np.abs(bank - g["bank"]).max(axis=1) <= 2e-5 * g["bank"].max(axis=1)).all()
    m = O.bft(g["x"], 64, 10, 32000, 256, O.W_HANN, O.SCALE_ERB, O.STYLE_GAMMATONE, O.NORM_NONE, O.DATA_POWER, result_type=1)
    assert rel_max(m, g["mel"]) < TOL
    assert rel_max(O.xxcc(g["mel"], 13), g["cc"]) < TOL
