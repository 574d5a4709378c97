"""Full-batch parity for BASELINE configs 3 and 4 and for the chunkers (VERDICT r1, item 8): scattered clips of a
full-size batch -- first, chunk boundary +-1, last -- must equal the single-clip result BIT FOR BIT, and one of them
the oracle.  Catches clip-offset bugs in the device-side chunk loops (af_cwt.c:cwt_compute, bft_compute) and in the
host-pointer pipeline (af_ctx.c:af_run_batch) that one-clip tests cannot see."""
import os

import numpy as np
import pytest

from conftest import rel_max
from oracle import af_oracle as O

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
TOL = 1e-4


def _af():
    import audioflux_b200 as af
    return af


def test_cqt_config3_full_batch_device(cuda_device):
    af = _af()
    B, L = 1024, 240000
    g = torch.Generator(device="cuda").manual_seed(31)
    x = 0.1 * torch.randn((B, L), generator=g, device="cuda")
    c = af.CQT(84, 48000)
    re, im = c.cqt_batch(x)
    torch.cuda.synchronize()
    assert re.shape == (B, c.cal_time_length(L), 84)
    for i in (0, 1, 511, 512, 1022, 1023):
        r1, i1 = c.cqt_batch(x[i:i + 1].contiguous())
        torch.cuda.synchronize()
        assert torch.equal(re[i], r1[0]) and torch.equal(im[i], i1[0]), f"clip {i} of the full batch differs from the single-clip result"
    wr, wi = O.cqt(x[1023].cpu().numpy(), 84, 48000, norm=O.NORM_AREA)
    got = re[1023].cpu().numpy() + 1j * im[1023].cpu().numpy()
    assert float(np.abs(got - (wr + 1j * wi)).max() / np.abs(wr + 1j * wi).max()) < TOL


def test_cqt_host_pipeline_chunk_boundaries(cuda_device):
    """host pointers: af_run_batch cuts the batch into ~64 MB chunks (66 clips of 5 s); compare around every boundary"""
    af = _af()
    B, L = 200, 240000
    x = (0.1 * np.random.default_rng(5).standard_normal((B, L))).astype(np.float32)
    c = af.CQT(84, 48000)
    re, im = c.cqt_batch(x)
    per = max(1, (64 << 20) // (L * 4))
    per -= per % 16 if per >= 16 else 0
    idx = sorted({0, B - 1} | {k for b in range(per, B, per) for k in (b - 1, b)})
    for i in idx:
        r1, i1 = c.cqt_planes(x[i])
        assert np.array_equal(re[i], r1) and np.array_equal(im[i], i1), f"clip {i} (chunk size {per}) differs from the single-clip call"
    wr, wi = O.cqt(x[idx[2]], 84, 48000, norm=O.NORM_AREA)
    assert rel_max(re[idx[2]], wr) < TOL and rel_max(im[idx[2]], wi) < TOL


def test_cwt_config4_shape_chunked(cuda_device):
    """64 clips of 2^19 samples (config 4's clip shape), forced into workspace chunks of 24 clips"""
    af = _af()
    B, N = 64, 1 << 19
    g = torch.Generator(device="cuda").manual_seed(41)
    x = torch.zeros((B, N), device="cuda")
    x[:, :480000] = 0.1 * torch.randn((B, 480000), generator=g, device="cuda")
    os.environ["AFB200_CWT_CHUNK"] = "24"
    try:
        w = af.CWT(84, 19, 48000, wavelet_type=af.WaveletContinueType.MORLET, is_padding=False)
        re, im = w.cwt_batch(x)
        torch.cuda.synchronize()
    finally:
        del os.environ["AFB200_CWT_CHUNK"]
    for i in (0, 23, 24, 47, 48, 63):
        r1, i1 = w.cwt_batch(x[i:i + 1].contiguous())
        torch.cuda.synchronize()
        assert torch.equal(re[i], r1[0]) and torch.equal(im[i], i1[0]), f"clip {i} of the chunked batch differs from the single-clip result"
    wr, wi = O.cwt(x[48].cpu().numpy(), 84, 19, 48000, wavelet=O.WAVE_MORLET, is_pad=False)
    want = wr + 1j * wi
    got = re[48].cpu().numpy() + 1j * im[48].cpu().numpy()
    assert float(np.abs(got - want).max() / np.abs(want).max()) < TOL


def test_mfcc_config2_full_batch_and_host_pipeline(cuda_device):
    af = _af()
    S, D = af.SpectralFilterBankScaleType, af.SpectralDataType
    b = af.BFT(128, 11, 48000, slide_length=512, scale_type=S.MEL, data_type=D.POWER)
    B, L = 1024, 240000
    g = torch.Generator(device="cuda").manual_seed(51)
    x = 0.1 * torch.randn((B, L), generator=g, device="cuda")
    out = b.mfcc_batch(x, 40)
    torch.cuda.synchronize()
    for i in (0, 1, 147, 148, 1023):
        o1 = b.mfcc_batch(x[i:i + 1].contiguous(), 40)
        torch.cuda.synchronize()
        assert torch.equal(out[i], o1[0]), f"clip {i}: result depends on the batch it was computed in"
    assert rel_max(out[1023].cpu().numpy(), O.mfcc(x[1023].cpu().numpy(), 48000, 11, 512, 128, 40)) < TOL
    xh = x[:200].cpu().numpy()
    oh = b.mfcc_batch(xh, 40)                            # host pointers: chunked 3-stream pipeline
    assert np.array_equal(oh, out[:200].cpu().numpy())
