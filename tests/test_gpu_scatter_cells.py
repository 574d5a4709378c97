"""Reassignment and synchrosqueezing on the GPU, cell by cell on the GPU's own float32 planes.

The index and scatter steps are repeated by tests/_scatter_model.py on the very planes the GPU transformed, so the
outputs must agree bit for bit wherever the kernels' arithmetic is plain float32:
  * reassignment (kernels/reassign.cu): every cell of every plane, including the 64-bit fixed-point sum;
  * WSST on the Linear, Linspace, Mel, Bark and Erb scales: every column;
  * WSST on Octave / Log (log2f) and synsq (atan2f): the CUDA Math API's rounding is only bounded, so those columns go
    through the model's column verifier, with a cap on the share of undetermined columns.
The planes themselves are checked against the float64 oracle beside it (tests/test_gpu_reassign.py and
tests/test_gpu_squeeze.py compare the final planes with the reference's different float32 pipeline)."""
import numpy as np
import pytest

import _scatter_model as M
from conftest import rel_max
from oracle import af_oracle as O
from test_gpu_squeeze import _signal as _sq_signal
from test_reassign_cpu import _signal

pytestmark = pytest.mark.gpu
f32 = np.float32
WSST_LOG_CAP, SYNSQ_CAP = 0.01, 0.15


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a, f32).view(np.uint32), np.asarray(b, f32).view(np.uint32))


# ------------------------------------------------------------------------------------------------ reassignment
def _reassign_inputs(r, radix, window, hop, pad, xs):
    """S_dh and S_th of the batch through product STFT objects with the reassignment windows of r's window"""
    import audioflux_b200 as af
    h = af.STFT(radix, af.WindowType(window), hop).get_window_data_arr()
    out = []
    for win in O.reassign_windows(h):
        s = af.STFT(radix, af.WindowType(window), hop)
        s.enable_padding(bool(pad))
        s.use_window_data_arr(win)
        out.append(s.stft_batch(xs))
    return out


def _check_reassign(r, xs, radix, sr, window, hop, re_type, thresh, pad, order, result_type, start=None):
    got = r.reassign_batch(xs, result_type) if start is None else None
    if start is not None:                                         # accumulate into the caller's planes
        from audioflux_b200.base import np_ptr
        r.set_result_type(result_type)
        a, b = start[0].copy(), start[1].copy()
        sh = [np.zeros_like(a) for _ in range(2)]
        r._lib.reassignObj_reassign(r._obj, np_ptr(xs[0]), xs.shape[-1], np_ptr(a), np_ptr(b), np_ptr(sh[0]), np_ptr(sh[1]))
        got = tuple(p[None] for p in (a, b, sh[0], sh[1]))
    s_h, s_dh, s_th = _reassign_inputs(r, radix, window, hop, pad, xs)
    assert _bits_equal(s_h[0], got[2]) and _bits_equal(s_h[1], got[3]), "STFT(h) differs from the S_h reassignment returns"
    n = 1 << radix
    for c in range(xs.shape[0]):
        want_h = O.stft(xs[c], n, hop, O.fft_window(window, n), is_pad=bool(pad))
        if np.abs(xs[c]).max() > 0:
            assert rel_max(got[2][c], want_h[0][:, :n // 2 + 1]) < 1e-4 and rel_max(got[3][c], want_h[1][:, :n // 2 + 1]) < 1e-4
        ti, fi = M.reassign_index((s_h[0][c], s_h[1][c]), (s_dh[0][c], s_dh[1][c]), (s_th[0][c], s_th[1][c]), n, sr, hop,
                                  re_type, thresh, order)
        st = None if start is None else start
        want = M.reassign_fixed_point((s_h[0][c], s_h[1][c]), ti, fi, result_type, st)
        for k in ((0,) if result_type else (0, 1)):
            diff = int((got[k][c].view(np.uint32) != want[k].view(np.uint32)).sum())
            assert diff == 0, (c, k, diff)
        if result_type:
            want_im = np.zeros_like(got[1][c]) if start is None else start[1]
            assert _bits_equal(got[1][c], want_im)
    print(f"reassign 2^{radix} hop {hop} type {re_type} order {order} result {result_type}: "
          f"{got[0].shape[0]} clips x {got[0][0].size} cells bitwise, 0 undetermined")


LEVELS = [1e-4, 1e-2, 1.0, 10.0, 0.0]
REASSIGN = [  # radix, sr, window, hop, re_type, thresh, pad, order, result_type, length
    (8, 8000, 0, 64, 0, 0.0, 0, 1, 0, 4000), (9, 16000, 1, 128, 0, 0.001, 0, 1, 0, 9000),
    (9, 16000, 2, 100, 1, 0.001, 1, 2, 0, 9000), (9, 16000, 1, 128, 2, 0.001, 0, 3, 1, 9000),
    (10, 32000, 1, 300, 0, 0.01, 1, 1, 1, 12000), (11, 32000, 2, 512, 0, 0.0, 0, 2, 0, 12000),
    (12, 32000, 0, 1000, 1, 0.001, 1, 3, 1, 20000), (12, 32000, 1, 1024, 2, 0.01, 0, 1, 0, 4096),       # T = 1
    (12, 32000, 2, 1000, 0, 0.001, 0, 1, 0, 5096), (14, 32000, 1, 3000, 0, 0.001, 0, 2, 0, 40000)]     # T = 2


@pytest.mark.parametrize("radix,sr,window,hop,re_type,thresh,pad,order,result_type,length", REASSIGN)
def test_reassign_bitwise_on_its_own_planes(cuda_device, radix, sr, window, hop, re_type, thresh, pad, order, result_type, length):
    import audioflux_b200 as af
    xs = np.stack([_signal(length, sr, radix + k) * f32(v) for k, v in enumerate(LEVELS)]).astype(f32)
    r = af.Reassign(radix, sr, af.WindowType(window), hop, af.ReassignType(re_type), thresh, bool(pad))
    r.set_order(order)
    _check_reassign(r, xs, radix, sr, window, hop, re_type, thresh, pad, order, result_type)


@pytest.mark.parametrize("result_type", [0, 1])
def test_reassign_bitwise_accumulating_into_nonzero_planes(cuda_device, result_type):
    import audioflux_b200 as af
    x = _signal(9000, 16000, 3)[None]
    r = af.Reassign(9, 16000, slide_length=100)
    T = r.cal_time_length(9000)
    rng = np.random.default_rng(4)
    start = [rng.standard_normal((T, 257)).astype(f32) for _ in range(2)]
    _check_reassign(r, x, 9, 16000, 1, 100, 0, 0.001, 0, 1, result_type, start)


def test_reassign_bitwise_host_batch_across_staging_chunks(cuda_device):
    """2^8 points, hop 16: every clip's planes are ~13 MB, so six clips cross the 64 MB staging chunk"""
    import audioflux_b200 as af
    xs = np.stack([_signal(100000, 8000, k) * f32(10.0 ** (k - 3)) for k in range(6)]).astype(f32)
    r = af.Reassign(8, 8000, slide_length=16)
    _check_reassign(r, xs, 8, 8000, 1, 16, 0, 0.001, 0, 1, 0)


# ------------------------------------------------------------------------------------------------ WSST
def _wsst_case(radix, is_pad, scale, wavelet, thresh, start=None):
    import audioflux_b200 as af
    sr, num = 32000, 84
    x = _sq_signal(1 << radix, sr, radix)
    kw = dict(wavelet_type=af.WaveletContinueType(wavelet), scale_type=af.SpectralFilterBankScaleType(scale), is_padding=is_pad)
    w = af.WSST(num, radix, sr, thresh=thresh, **kw)
    if start is None:
        got = w.wsst_planes(x)
    else:
        from audioflux_b200.base import np_ptr
        got = [start[0].copy(), start[1].copy()] + [np.zeros_like(start[0]) for _ in range(2)]
        w._lib.wsstObj_wsst(w._obj, np_ptr(x), *[np_ptr(p) for p in got])
    c = af.CWT(num, radix, sr, **kw)
    c.enable_det(True)
    wp = c.cwt_planes(x)
    dw = c.cwt_det_planes(None)
    assert _bits_equal(wp[0], got[2]) and _bits_equal(wp[1], got[3]), "CWT planes differ from the W wsst returns"
    if radix <= 14:
        o = O.cwt(x, num, radix, sr, wavelet, scale, w.low_fre, w.high_fre, is_pad=is_pad)
        assert rel_max(wp[0], o[0]) < 1e-4 and rel_max(wp[1], o[1]) < 1e-4
    fre = w.get_fre_band_arr()
    index = M.wsst_index(wp, dw, fre, sr, scale)
    v = M.verify_columns(got[:2], wp, index, thresh, start)
    print(f"wsst 2^{radix} pad {is_pad} scale {scale} wavelet {wavelet} thresh {thresh}: {v['undetermined_cells']} "
          f"undetermined cells, {v['undetermined_columns']:.4%} of columns")
    assert not v["failures"], v["failures"][:20]
    if scale in (O.SCALE_OCTAVE, O.SCALE_LOG):
        assert v["undetermined_columns"] <= WSST_LOG_CAP
    else:
        assert v["undetermined_cells"] == 0
        want = M.scatter(wp, index.idx, thresh, start)
        assert _bits_equal(got[0], want[0]) and _bits_equal(got[1], want[1])
    return wp, fre


WSST = [  # radix, is_pad, scale, wavelet, thresh
    (10, False, O.SCALE_LINEAR, O.WAVE_MORLET, 0.001), (10, True, O.SCALE_OCTAVE, O.WAVE_PAUL, 0.0),
    (12, False, O.SCALE_LINSPACE, O.WAVE_MORSE, 0.001), (12, True, O.SCALE_MEL, O.WAVE_BUMP, 0.001),
    (12, False, O.SCALE_BARK, O.WAVE_MORLET, 0.1), (12, False, O.SCALE_ERB, O.WAVE_PAUL, 0.001),
    (12, False, O.SCALE_OCTAVE, O.WAVE_MORLET, 0.001), (12, True, O.SCALE_LOG, O.WAVE_MORSE, 0.001),
    (13, False, O.SCALE_LINEAR, O.WAVE_BUMP, 0.0), (13, True, O.SCALE_OCTAVE, O.WAVE_MORLET, 0.001),
    (14, False, O.SCALE_MEL, O.WAVE_MORLET, 0.001), (14, True, O.SCALE_LOG, O.WAVE_BUMP, 0.1),
    (16, False, O.SCALE_LINEAR, O.WAVE_MORLET, 0.001), (16, False, O.SCALE_OCTAVE, O.WAVE_MORSE, 0.001)]


@pytest.mark.parametrize("radix,is_pad,scale,wavelet,thresh", WSST)
def test_wsst_cells_on_its_own_planes(cuda_device, radix, is_pad, scale, wavelet, thresh):
    _wsst_case(radix, is_pad, scale, wavelet, thresh)


@pytest.mark.parametrize("scale", [O.SCALE_LINEAR, O.SCALE_OCTAVE])
def test_wsst_cells_accumulating_into_nonzero_planes(cuda_device, scale):
    rng = np.random.default_rng(9)
    start = [rng.standard_normal((84, 1 << 12)).astype(f32) for _ in range(2)]
    _wsst_case(12, False, scale, O.WAVE_MORLET, 0.001, start)


# ------------------------------------------------------------------------------------------------ synsq
@pytest.mark.parametrize("radix", [10, 12, 13, 14])
@pytest.mark.parametrize("scale", [O.SCALE_LINEAR, O.SCALE_OCTAVE, O.SCALE_BARK])
def test_synsq_cells_on_gpu_planes(cuda_device, radix, scale):
    """the GPU CWT planes of the WSST cases; the Linear scale reaches Nyquist, whose rows jump by 2 pi almost every
    sample.  k_synsq_index gives each thread N / 1024 samples: 1 to 16 per thread run."""
    import audioflux_b200 as af
    wp, fre = _wsst_case(radix, False, scale, O.WAVE_MORLET, 0.001)
    got = af.Synsq(84, radix, 32000).synsq_planes(fre, af.SpectralFilterBankScaleType(scale), *wp)
    index = M.synsq_index(*wp, fre, 32000, scale)
    v = M.verify_columns(got, wp, index, 0.001)
    print(f"synsq 2^{radix} scale {scale}: {v['undetermined_cells']} undetermined cells, "
          f"{v['undetermined_columns']:.4%} of columns ({v['enumerated_columns']} enumerated, {v['bounded_columns']} bounded)")
    assert not v["failures"], v["failures"][:20]
    assert v["undetermined_columns"] <= SYNSQ_CAP
    assert np.abs(got[0]).max() > 0


def test_synsq_threshold_is_evaluated_without_fma(cuda_device):
    """rows of crafted (v1, v2) whose |W|^2 falls on the other side of thresh^2 when contracted into an FMA; constant
    along time, so every cell's phase difference is 0 and its row on the Linear scale from 0 Hz is row 0.  Two rows of
    clearly kept cells keep row 0 non-zero."""
    import audioflux_b200 as af
    v1, v2, kept = M.crafted_threshold_pairs()
    num, radix = 16, 10
    n = 1 << radix
    re = np.zeros((num, n), f32)
    im = np.zeros((num, n), f32)
    re[:len(v1)], im[:len(v1)] = v1[:, None], v2[:, None]
    re[len(v1)], im[len(v1)] = f32(0.02), f32(-0.01)
    re[len(v1) + 1], im[len(v1) + 1] = f32(-0.003), f32(0.005)
    fre = np.linspace(0, 16000, num).astype(f32)
    got = af.Synsq(num, radix, 32000).synsq_planes(fre, af.SpectralFilterBankScaleType.LINEAR, re, im)
    index = M.synsq_index(re, im, fre, 32000, O.SCALE_LINEAR)
    assert not index.cands and (index.idx[:len(v1) + 2] == 0).all()
    want = M.scatter((re, im), index.idx, 0.001)
    clear = f32(f32(0.02) + f32(-0.003))
    assert want[0][0, 0] == (clear if not kept.any() else want[0][0, 0])
    assert _bits_equal(got[0], want[0]) and _bits_equal(got[1], want[1]), (got[0][0, :4], want[0][0, :4])
