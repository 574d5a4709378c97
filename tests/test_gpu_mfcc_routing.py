"""Which path serves a BFT object's fused-MFCC and real-mode filter-bank calls at fftLength 2048: the v2 kernel
(kernels/mfcc_fused2.cu), the v1 kernel (kernels/mfcc_fused.cu) or the composed STFT -> bank (-> DCT) kernels.

For every case the table pins bftObj_mfccPlanMode after mfcc_batch (1 = v2, 0 = v1, -1 = composed), the kernel launches
of that mfcc_batch call and the kernel launches of a real-mode bft_batch call on the same clips."""
import numpy as np
import pytest

import audioflux_b200 as af
from conftest import noise

pytestmark = pytest.mark.gpu

S, ST, N, D = af.SpectralFilterBankScaleType, af.SpectralFilterBankStyleType, af.SpectralFilterBankNormalType, af.SpectralDataType
MEL128 = dict(num=128, samplate=48000, scale_type=S.MEL)

# id, BFT arguments, clip length, clip offset in floats, ccNum, hook environment, (plan mode, mfcc launches, bft launches)
CASES = [
    # the nine banks of test_gpu_parity.py::test_mfcc_fused_bank_loop_modes
    ("mel-slaney-none", dict(num=128, samplate=48000, scale_type=S.MEL, style_type=ST.SLANEY, normal_type=N.NONE, data_type=D.POWER), 20480, 0, 20, {}, (1, 1, 1)),
    ("mel-slaney-area", dict(num=128, samplate=48000, scale_type=S.MEL, style_type=ST.SLANEY, normal_type=N.AREA, data_type=D.POWER), 20480, 0, 20, {}, (1, 1, 1)),
    ("mel-slaney-bw-mag", dict(num=128, samplate=48000, scale_type=S.MEL, style_type=ST.SLANEY, normal_type=N.BAND_WIDTH, data_type=D.MAG), 20480, 0, 20, {}, (1, 1, 1)),
    ("bark-etsi-area-64", dict(num=64, samplate=48000, scale_type=S.BARK, style_type=ST.ETSI, normal_type=N.AREA, data_type=D.POWER), 20480, 0, 20, {}, (-1, 3, 2)),
    ("erb-slaney-none", dict(num=128, samplate=48000, scale_type=S.ERB, style_type=ST.SLANEY, normal_type=N.NONE, data_type=D.POWER), 20480, 0, 20, {}, (1, 1, 1)),
    ("mel-etsi-none", dict(num=128, samplate=48000, scale_type=S.MEL, style_type=ST.ETSI, normal_type=N.NONE, data_type=D.POWER), 20480, 0, 20, {}, (1, 1, 1)),
    ("mel-hann-none", dict(num=128, samplate=48000, scale_type=S.MEL, style_type=ST.HANN, normal_type=N.NONE, data_type=D.POWER), 20480, 0, 20, {}, (1, 1, 1)),
    ("mel-40-16k", dict(num=40, samplate=16000, scale_type=S.MEL, style_type=ST.SLANEY, normal_type=N.NONE, data_type=D.POWER), 20480, 0, 20, {}, (-1, 3, 2)),
    ("erb-etsi-bw-77-mag", dict(num=77, samplate=22050, scale_type=S.ERB, style_type=ST.ETSI, normal_type=N.BAND_WIDTH, data_type=D.MAG), 20480, 0, 20, {}, (1, 1, 1)),
    # a bank only v1 serves (three filters on a bin), one outside v1's weight table, and a Linear bank
    ("mel-rect", dict(MEL128, style_type=ST.RECT), 20480, 0, 13, {}, (0, 1, 1)),
    ("bark-slaney-bw-128", dict(num=128, samplate=48000, scale_type=S.BARK, style_type=ST.SLANEY, normal_type=N.BAND_WIDTH), 20480, 0, 20, {}, (-1, 3, 2)),
    ("linear", dict(num=128, samplate=48000, scale_type=S.LINEAR), 20480, 0, 20, {}, (-1, 3, 2)),
    # call shapes outside the fused kernels
    ("norm-0.5", dict(MEL128, norm_value=0.5), 20480, 0, 20, {}, (-1, 3, 2)),
    ("hop-510", dict(MEL128, slide_length=510), 20480, 0, 20, {}, (-1, 3, 2)),
    ("length-not-4", dict(MEL128), 20481, 0, 20, {}, (-1, 3, 2)),
    ("offset-1-float", dict(MEL128), 20480, 1, 20, {}, (-1, 3, 2)),
    ("cc-65", dict(MEL128), 20480, 0, 65, {}, (-1, 2, 1)),
    ("mel-129", dict(MEL128, num=129), 20480, 0, 20, {}, (-1, 3, 2)),
    # the two hooks
    ("hook-v1-mel", dict(MEL128), 20480, 0, 20, {"AFB200_MFCC_KERNEL": "v1"}, (0, 1, 1)),
    ("hook-v1-rect", dict(MEL128, style_type=ST.RECT), 20480, 0, 13, {"AFB200_MFCC_KERNEL": "v1"}, (0, 1, 1)),
    ("hook-general-mel", dict(MEL128), 20480, 0, 20, {"AFB200_BFT_GENERAL": "1"}, (1, 1, 2)),
    ("hook-general-cc-65", dict(MEL128), 20480, 0, 65, {"AFB200_BFT_GENERAL": "1"}, (-1, 3, 2)),
]


def run_case(lib, torch, kw, length, offset, cc):
    """(plan mode after mfcc_batch, launches of mfcc_batch, launches of a real-mode bft_batch) on two device clips"""
    kw = dict(kw)
    norm_value = kw.pop("norm_value", None)
    b = af.BFT(kw.pop("num"), 11, kw.pop("samplate"), slide_length=kw.pop("slide_length", 512), **kw)
    if norm_value is not None:
        b.set_data_norm_value(norm_value)
    x = np.concatenate([np.zeros(offset, np.float32), noise(51, length), noise(52, length)])
    xd = torch.from_numpy(x).cuda()[offset:].view(2, length)
    n0 = lib.afb200_kernelLaunchCount()
    b.mfcc_batch(xd, cc)
    n1 = lib.afb200_kernelLaunchCount()
    mode = lib.bftObj_mfccPlanMode(b._obj)
    b.bft_batch(xd, result_type=1)
    n2 = lib.afb200_kernelLaunchCount()
    torch.cuda.synchronize()
    return mode, n1 - n0, n2 - n1


@pytest.mark.parametrize("case_id,kw,length,offset,cc,env,want", CASES, ids=[c[0] for c in CASES])
def test_fused_mfcc_routing(cuda_device, product_lib, monkeypatch, case_id, kw, length, offset, cc, env, want):
    import torch
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    assert run_case(product_lib, torch, kw, length, offset, cc) == want
