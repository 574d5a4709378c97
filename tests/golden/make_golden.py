#!/usr/bin/env python3
"""Generate tests/golden/*.npz from the UNMODIFIED reference build (oracle/_ref).

Run where the reference has been compiled by `make -C oracle REF=<audioFlux tree>`:
    python tests/golden/make_golden.py
The fixtures pin both the numpy oracle (tests/test_golden.py) and the CUDA path
(tests/test_gpu_parity.py) to outputs of the reference itself.  Inputs are seeded
(`np.random.default_rng(seed)`), amplitude 0.1, float32 -- SURVEY.md section 8(d).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.realpath(__file__))))
sys.path.insert(0, ROOT)

import audioflux_b200 as af  # noqa: E402  (host-side mirror classes, driven with the reference library)
from oracle.ref_lib import get_ref_lib  # noqa: E402

HERE = os.path.dirname(os.path.realpath(__file__))


def noise(seed, n):
    return (0.1 * np.random.default_rng(seed).standard_normal(n)).astype(np.float32)


def tones(seed, n, sr):
    t = np.arange(n) / sr
    x = 0.3 * (np.sin(2 * np.pi * 220 * t) + np.sin(2 * np.pi * 880 * t) + np.sin(2 * np.pi * 3520 * t))
    return (x + 0.01 * np.random.default_rng(seed).standard_normal(n)).astype(np.float32)


def main():
    ref = get_ref_lib()
    S, ST, N, D = (af.SpectralFilterBankScaleType, af.SpectralFilterBankStyleType,
                   af.SpectralFilterBankNormalType, af.SpectralDataType)
    # ---- C1: 1 s 48 kHz clip, BFT mel-128, n_fft 2048, hop 512 (+ MFCC-40) ----
    x = noise(0, 48000)
    b = af.BFT(128, 11, 48000, slide_length=512, scale_type=S.MEL, data_type=D.POWER, _lib=ref)
    mel, _ = b.bft_planes(x, 1)
    xx = af.XXCC(128, _lib=ref)
    mfcc = xx.xxcc_planes(mel, 40)
    zre, zim = b.bft_planes(x, 0)
    np.savez_compressed(os.path.join(HERE, "c1_mel_mfcc.npz"), x=x, mel=mel, mfcc=mfcc, cre=zre, cim=zim,
                        bin_band=b.get_bin_band_arr(), fre_band=b.get_fre_band_arr())
    # tones + area norm + magnitude, bark ETSI
    xt = tones(1, 24000, 48000)
    b2 = af.BFT(64, 10, 48000, slide_length=256, scale_type=S.BARK, style_type=ST.ETSI, normal_type=N.AREA,
                data_type=D.MAG, _lib=ref)
    m2, _ = b2.bft_planes(xt, 1)
    xx2 = af.XXCC(64, _lib=ref)
    np.savez_compressed(os.path.join(HERE, "bark_etsi_mag.npz"), x=xt, mel=m2, cc=xx2.xxcc_planes(m2, 20),
                        cc_cubic=xx2.xxcc_planes(m2, 13, af.CepstralRectifyType.CUBIC_ROOT))
    # ---- gammatone (dense bank) on the ERB scale, as af.gtcc uses it: bank + real-mode BFT + cepstrum ----
    xg = tones(5, 16000, 32000)
    b3 = af.BFT(64, 10, 32000, slide_length=256, scale_type=S.ERB, style_type=ST.GAMMATONE, normal_type=N.NONE,
                data_type=D.POWER, _lib=ref)
    import ctypes as C
    gbank = np.zeros((64, 513), np.float32)
    gf = np.zeros(66, np.float32)
    gb = np.zeros(66, np.int32)
    ref.auditory_filterBank(64, 1024, 32000, 0, 4, 2, 0, C.c_float(0.0), C.c_float(16000.0), 12, gbank.ctypes.data, gf.ctypes.data, gb.ctypes.data)
    m3, _ = b3.bft_planes(xg, 1)
    xx3 = af.XXCC(64, _lib=ref)
    np.savez_compressed(os.path.join(HERE, "erb_gammatone.npz"), x=xg, bank=gbank, mel=m3, cc=xx3.xxcc_planes(m3, 13),
                        fre_band=b3.get_fre_band_arr(), bin_band=b3.get_bin_band_arr())
    # ---- STFT (full mirrored planes), hann 512 / hop 128, first 8 frames ----
    s = af.STFT(9, af.WindowType.HANN, 128, _lib=ref)
    xs = noise(2, 4000)
    re, im = s.stft_planes(xs)
    np.savez_compressed(os.path.join(HERE, "stft_512.npz"), x=xs, re=re[:8], im=im[:8], T=np.int32(re.shape[0]))
    # ---- CQT 84 bins @ 48 kHz, 0.25 s ----
    xc = noise(3, 12037)
    c = af.CQT(84, 48000, _lib=ref)
    cre, cim = c.cqt_planes(xc)
    np.savez_compressed(os.path.join(HERE, "cqt_84.npz"), x=xc, re=cre, im=cim, fft_length=np.int32(c.fft_length))
    # ---- CWT morlet, 36 scales, N = 2048 ----
    xw = noise(4, 2048)
    w = af.CWT(36, 11, 48000, wavelet_type=af.WaveletContinueType.MORLET, is_padding=False, _lib=ref)
    wre, wim = w.cwt_planes(xw)
    np.savez_compressed(os.path.join(HERE, "cwt_morlet.npz"), x=xw, re=wre, im=wim, fre=w.get_fre_band_arr())
    # ---- SURVEY 8(f) rows: xxccStandard, CQT chroma / cqcc, SpectrogramObj front door ----
    E, CN = af.CepstralEnergyType, af.ChromaDataNormalType
    energy = (mel.sum(axis=1) / 128).astype(np.float32)
    std = {}
    for name, et, order in (("rep", E.REPLACE, 9), ("app", E.APPEND, 5), ("ign", E.IGNORE, 3)):
        coe, d1, d2 = xx.xxcc_standard_planes(mel[:24], energy[:24], 13, order, et)
        std[f"std_{name}_coe"], std[f"std_{name}_d1"], std[f"std_{name}_d2"] = coe, d1, d2
    c2 = af.CQT(84, 48000, _lib=ref)
    cre2, cim2 = c2.cqt_planes(xc)
    chroma_max = c2.chroma_planes(cre2, cim2, 12, D.POWER, CN.MAX)
    chroma_p2 = c2.chroma_planes(cre2, cim2, 12, D.MAG, CN.P2)
    cqcc = c2.cqcc_planes(cre2 * cre2 + cim2 * cim2, 20)
    xsp = tones(6, 6000, 48000)
    sl = af.Spectrogram(samplate=48000, low_fre=100., high_fre=8000., radix2_exp=10, slide_length=256, _lib=ref)
    lin, lin_phase = sl.spectrogram_planes(xsp, True)
    sm = af.MelSpectrogram(num=64, samplate=48000, radix2_exp=10, slide_length=256, data_type=D.MAG, _lib=ref)
    sm.set_data_norm_value(0.5)
    msp = sm.spectrogram_planes(xsp)
    mcc = sm.mfcc(np.ascontiguousarray(msp.T), 13).T
    wd = af.CWT(12, 10, 48000, wavelet_type=af.WaveletContinueType.MORLET, is_padding=False, _lib=ref)
    wd.enable_det(True)
    xdet = noise(7, 1024)
    det_re, det_im = wd.cwt_det_planes(xdet)
    np.savez_compressed(os.path.join(HERE, "next_rows.npz"), xdet=xdet, det_re=det_re, det_im=det_im, energy=energy[:24], chroma_max=chroma_max,
                        chroma_p2=chroma_p2, cqcc=cqcc, xsp=xsp, lin=lin, lin_phase=lin_phase,
                        lin_fre=sl.get_fre_band_arr(), lin_bin=sl.get_bin_band_arr(), mel_mag=msp, mel_cc=mcc,
                        mel_fre=sm.get_fre_band_arr(), **std)
    for f in sorted(os.listdir(HERE)):
        if f.endswith(".npz"):
            print(f, os.path.getsize(os.path.join(HERE, f)))


if __name__ == "__main__":
    main()
