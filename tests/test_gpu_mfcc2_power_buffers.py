"""The fused MFCC v2 kernel (kernels/mfcc_fused2.cu) alternates two power tiles: a CTA's tile number `it` lands on
buffer it & 1.  A clip's fused MFCC and raw-mel output must not depend on which buffer its tiles used: the clip is moved
through a batch until every one of its tiles has run on both buffers, and every result must equal, bit for bit, the
clip transformed on its own.  The shapes include a tail tile with fewer frames than the tile holds and a hop at which
fewer than 13 frames fit the shared memory."""
import numpy as np
import pytest

import audioflux_b200 as af
from conftest import noise

pytestmark = pytest.mark.gpu

S, D = af.SpectralFilterBankScaleType, af.SpectralDataType
FRAMES = 13


def _frames_per_tile(lib, b, time_length, hop, cc, raw):
    bank = np.ascontiguousarray(b.get_filter_bank_arr(), np.float32)
    num = bank.shape[0]
    z = lambda n, t: np.zeros(n, t)                                        # noqa: E731
    owner, desc, table = z(1025, np.int32), z(num + 2, np.uint32), z(4 * 1408, np.float32)
    piece, prefix, assign, info = z(256, np.uint32), z(num + 2, np.uint16), z(256, np.uint16), z(16, np.int32)
    tab = lib.afb200_mfccBankPlan2(bank.ctypes.data, num, owner.ctypes.data, desc.ctypes.data, table.ctypes.data,
                                   piece.ctypes.data, prefix.ctypes.data, assign.ctypes.data, info.ctypes.data)
    assert tab > 0
    carve = np.zeros(16, np.int32)
    assert lib.afb200_mfccCarve2(time_length, hop, num, cc, tab, raw, carve.ctypes.data) > 0
    return int(carve[0])


def _positions(n_clips, tiles_per_clip, sms):
    """batch positions of the clip such that each of its tiles runs on both power buffers"""
    grid = min(n_clips * tiles_per_clip, sms)
    seen = [set() for _ in range(tiles_per_clip)]
    chosen = []
    for c in range(n_clips):
        bufs = [((c * tiles_per_clip + k) // grid) & 1 for k in range(tiles_per_clip)]
        if any(bf not in seen[k] for k, bf in enumerate(bufs)):
            chosen.append(c)
            for k, bf in enumerate(bufs):
                seen[k].add(bf)
    assert all(s == {0, 1} for s in seen), "the batch is too small to put every tile on both buffers"
    return chosen


@pytest.mark.parametrize("hop,length,mode", [
    (512, 48000, "mfcc"), (512, 48000, "mel"),            # 90 frames: 6 full tiles + a tail of 12
    (2048, 2048 * 75, "mfcc"), (2048, 2048 * 75, "mel"),  # fewer than 13 frames per tile fit
])
def test_output_does_not_depend_on_the_power_buffer(cuda_device, product_lib, hop, length, mode):
    import torch
    b = af.BFT(128, 11, 48000, slide_length=hop, scale_type=S.MEL, data_type=D.POWER)
    T = b.cal_time_length(length)
    F = _frames_per_tile(product_lib, b, T, hop, 20, mode == "mel")
    if hop == 2048:
        assert F < FRAMES
    assert T % F != 0                                                      # the clip ends in a partial tile
    tiles = -(-T // F)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n_clips = 4 * sms // tiles + 4
    run = (lambda x: b.mfcc_batch(x, 20)) if mode == "mfcc" else (lambda x: b.bft_batch(x, result_type=1))

    clip = torch.from_numpy(noise(7, length)).cuda().view(1, length)
    b.mfcc_batch(clip, 20)
    assert product_lib.bftObj_mfccPlanMode(b._obj) == 1                    # the bank is served by the v2 kernel
    n0 = product_lib.afb200_kernelLaunchCount()
    alone = run(clip)[0].cpu().numpy()
    assert product_lib.afb200_kernelLaunchCount() - n0 == 1                # in one fused launch
    clip = clip[0]
    batch = torch.from_numpy(np.stack([noise(100 + i, length) for i in range(n_clips)])).cuda()
    for c in _positions(n_clips, tiles, sms):
        x = batch.clone()
        x[c] = clip
        got = run(x)[c].cpu().numpy()
        assert np.array_equal(got, alone), (mode, hop, c, float(np.abs(got - alone).max()))
