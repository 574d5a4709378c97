"""The power-tile layout of the fused MFCC v2 kernel (kernels/mfcc_fused2.cu), checked in numpy without a GPU.

Stage C of a frame warp transposes its 32 x 32 complex columns (a real plane, then an imaginary plane) through its own
column of the power tile: float2 slot 13 s + w of frame w, s < 513 bin pairs.  Element pair j = n2 / 2 of plane row
r = k1 - 1 sits at slot s = r + 31 j.  The writers (lane n2, one 32-bit store per row) and the readers (lane k1, one
float2 per pair j; lane 0 reads row 0 with lane 1) must each take one shared-memory wavefront.  The launcher's
carve-up (two power tiles, no transpose scratch) must fit the 227 KB an H100 CTA may use at every hop."""
import numpy as np
import pytest

PAIRS, PITCH, FRAMES, ROWS = 513, 13, 13, 31
BUDGET = 227 * 1024
MAX_TAB = 1408
TILE_BYTES = PAIRS * PITCH * 8


def slot(r, j):
    return r + ROWS * j


def test_slot_map_stays_in_the_frame_column():
    r, j = np.meshgrid(np.arange(ROWS), np.arange(16), indexing="ij")
    s = slot(r, j)
    assert s.min() == 0 and s.max() < PAIRS
    for w in range(FRAMES):
        f2 = PITCH * s + w                                     # float2 index in the tile
        assert np.all(f2 % PITCH == w)                         # frame w's column, nobody else's
        assert f2.max() < PAIRS * PITCH


def test_slot_map_is_a_bijection_on_the_plane():
    words = {(slot(r, n2 // 2), n2 & 1) for r in range(ROWS) for n2 in range(32)}
    assert len(words) == ROWS * 32


@pytest.mark.parametrize("w", range(FRAMES))
def test_writers_hit_32_banks(w):
    lanes = np.arange(32)
    for r in range(ROWS):
        word = 2 * (PITCH * slot(r, lanes // 2) + w) + (lanes & 1)
        assert len(set(word % 32)) == 32, (w, r)


@pytest.mark.parametrize("w", range(FRAMES))
def test_readers_hit_16_bank_pairs_per_half_warp(w):
    lanes = np.arange(32)
    rows = np.where(lanes == 0, 0, lanes - 1)                  # lane 0 reads row 0 with lane 1
    for j in range(16):
        f2 = PITCH * slot(rows, j) + w
        for half in (f2[:16], f2[16:]):
            distinct = np.unique(half)                         # equal addresses are one broadcast access
            assert len(set(distinct % 16)) == len(distinct), (w, j)


def _carve(lib, time_length, hop, cc, tab, raw):
    info = np.zeros(16, np.int32)
    total = lib.afb200_mfccCarve2(time_length, hop, 128, cc, tab, raw, info.ctypes.data)
    return total, info


@pytest.mark.parametrize("raw", (0, 1))
@pytest.mark.parametrize("cc", (40, 64))
def test_carve_up_fits_at_every_hop(product_lib, raw, cc):
    for hop in range(4, 2049, 4):
        for tab in (0, MAX_TAB):
            total, info = _carve(product_lib, 465, hop, cc, tab, raw)
            frames, stages = int(info[0]), int(info[1])
            assert 0 < total <= BUDGET, (hop, tab, total)
            assert 1 <= frames <= FRAMES and stages in (1, 2), (hop, frames, stages)
            off = [int(v) for v in info[2:14]]
            assert off == sorted(off) and off[-1] < total, (hop, off)
            assert all(o % 16 == 0 for o in off), (hop, off)
            assert off[1] - off[0] >= stages * int(info[15]) * 4        # the TMA span(s)
            assert off[2] - off[1] >= 2 * TILE_BYTES                    # two power tiles


def test_carve_up_of_the_benchmark_shape(product_lib):
    total, info = _carve(product_lib, 465, 512, 40, MAX_TAB, 0)
    assert info[0] == FRAMES and total <= BUDGET
    total, info = _carve(product_lib, 465, 2048, 40, MAX_TAB, 0)
    assert info[0] < FRAMES                                             # the largest hop runs shorter tiles
    assert _carve(product_lib, 5, 512, 40, 0, 0)[1][0] == 5              # a clip shorter than a tile
