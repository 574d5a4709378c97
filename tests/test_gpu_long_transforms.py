"""The long-transform FFT paths (2^15 .. 2^20 points) row by row against the float64 oracle.

Every transform longer than 16384 points runs through the four-step kernels of cwt.cu: CWT / PWT (and at N = 2^19 their
fast path -- warp-level legs, the persistent k_cwt_fused_w with its ring of item groups, per-row bank-support pruning),
long-frame STFT / BFT (`launch_stft_long`) and long-frame ISTFT (Hartley identity, `launch_istft_frames_long`).

The bar is applied per output ROW (one scale of one clip, one frame): max |got - want| over the row's complex values
<= 1e-4 * that row's own max |want|.  Quiet rows of a CWT plane peak at a few percent of the plane's maximum, so the
per-tensor bar of the rest of the suite lets a whole quiet row be wrong by 1e-3 of its own scale; the per-tensor bar is
kept as well, so a failure shows which one broke.  Rows the oracle gives as exactly zero must come out below 1e-20.
Inputs are white noise, so every band has content.  The run prints the worst row of every case.
"""
import numpy as np
import pytest

import audioflux_b200 as af
from conftest import noise, rel_max
from oracle import af_oracle as O
from test_next_rows_cpu import istft_conditioned

pytestmark = pytest.mark.gpu

TOL = 1e-4
ZERO_ROW = 1e-20
SR = 48000
N19 = 1 << 19
W, S, D, WIN = af.WaveletContinueType, af.SpectralFilterBankScaleType, af.SpectralDataType, af.WindowType


@pytest.fixture(scope="module")
def torch_cuda(cuda_device):
    import torch
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)
    return torch


@pytest.fixture
def report(request, capsys):
    """report(case, worst_row, tensor): prints the case's worst per-row error past pytest's capture and records it."""
    def emit(case, worst_row, tensor):
        request.node.user_properties.append((case, worst_row))
        with capsys.disabled():
            print(f"\n    {request.node.name} {case}: worst row {worst_row:.2e}, per tensor {tensor:.2e}", end="")
    return emit


def _host(a):
    return a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a)


def row_rel(got_re, got_im, want_re, want_im):
    """Per output row (the last axis runs along the row): max |got - want| over the row's complex values divided by the
    row's own max |want|.  A row the oracle gives as exactly zero reports max |got| instead, an absolute value.
    -> (values [rows], zero [rows] bool).  got_im / want_im may be None for real outputs."""
    planes = [None if a is None else np.asarray(a) for a in (got_re, got_im, want_re, want_im)]
    width = planes[0].shape[-1]
    gr, gi, wr, wi = (None if a is None else a.reshape(-1, width) for a in planes)
    rows = gr.shape[0]
    out, zero = np.empty(rows), np.zeros(rows, bool)
    for r in range(rows):                       # one row at a time: a 2^19-point plane of 84 rows is 352 MB in float64
        a_r, b_r = gr[r].astype(np.float64), wr[r].astype(np.float64)
        a_i = gi[r].astype(np.float64) if gi is not None else 0.0
        b_i = wi[r].astype(np.float64) if wi is not None else 0.0
        peak = np.sqrt(b_r * b_r + b_i * b_i).max()
        if peak == 0:
            zero[r] = True
            out[r] = np.sqrt(a_r * a_r + a_i * a_i).max()
        else:
            out[r] = np.sqrt((a_r - b_r) ** 2 + (a_i - b_i) ** 2).max() / peak
    return out, zero


def check_rows(report, case, got_re, got_im, want_re, want_im):
    """Per-row and per-tensor bar on one clip's planes; returns the zero-row mask."""
    got_re, got_im = _host(got_re), None if got_im is None else _host(got_im)
    rel, zero = row_rel(got_re, got_im, want_re, want_im)
    tensor = rel_max(got_re, want_re)
    if want_im is not None:
        tensor = max(tensor, rel_max(got_im, want_im))
    worst = float(rel[~zero].max()) if (~zero).any() else 0.0
    report(case, worst, tensor)
    assert tensor < TOL, (case, "per tensor", tensor)
    bad = np.nonzero(~zero & (rel >= TOL))[0]
    assert bad.size == 0, (case, "rows above the per-row bar", bad[:20].tolist(), rel[bad[:20]].tolist())
    assert not zero.any() or rel[zero].max() < ZERO_ROW, (case, "all-zero rows", np.nonzero(zero)[0].tolist(), rel[zero].max())
    return zero


# ------------------------------------------------------------------ CWT / PWT oracles
def cwt_oracle(w, x, det=False, bank=None):
    return O.cwt(x, w.num, w.radix2_exp, w.samplate, af.enum_value(w.wavelet_type), af.enum_value(w.scale_type),
                 low=w.low_fre, high=w.high_fre, bpo=w.bin_per_octave, gamma=w.gamma, beta=w.beta, is_pad=w.is_padding,
                 bank=bank, det=det)


def cwt_bank(w):
    """The oracle bank at the transform length: N + 2 * pad columns (pad = N / 2 when the object pads), band frequencies
    of the unpadded length."""
    pad = w.fft_length // 2 if w.is_padding else 0
    return O.cwt_filterbank(w.num, w.fft_length, w.samplate, af.enum_value(w.wavelet_type), af.enum_value(w.scale_type),
                            low=w.low_fre, high=w.high_fre, bpo=w.bin_per_octave, gamma=w.gamma, beta=w.beta,
                            pad_length=pad)[0]


def pwt_oracle(p, x, det=False):
    re, im, _, _ = O.pwt(x, p.num, p.radix2_exp, p.samplate, low=p.low_fre, high=p.high_fre, bpo=p.bin_per_octave,
                         scale=af.enum_value(p.scale_type), style=af.enum_value(p.style_type),
                         norm=af.enum_value(p.normal_type), is_pad=p.is_padding, det=det)
    return re, im


# ------------------------------------------------------------------ 1. CWT, N = 2^19 fast path
# Support classes (2^-28 rule) noted where they matter: 'single' rows span at most 32 rows of the 1024-point column and
# take the one-hot branch of cwt_cols_w_unit; 'Nyquist' rows have support up to bin N/2.
CWT19 = [
    (W.MORSE, S.OCTAVE, 84, {}),                        # the default wavelet
    (W.PAUL, S.MEL, 60, {}),                            # 30 Nyquist rows, rows covering the whole half spectrum
    (W.MORLET, S.MEL, 60, {}),                          # 11 Nyquist rows
    (W.DOG, S.OCTAVE, 84, dict(gamma=4)),
    (W.MEXICAN, S.LOG, 84, {}),                         # 19 Nyquist rows
    (W.BUMP, S.OCTAVE, 84, dict(gamma=6, beta=1.0)),    # every row 'single'
    (W.HERMIT, S.BARK, 60, {}),
    (W.RICKER, S.ERB, 60, {}),
    (W.MORLET, S.LINEAR, 83, {}),                       # 83 items: a one-item last group; the 0 Hz band is all zero
]
CWT19_IDS = [f"{w.name}-{s.name}-{n}" for w, s, n, _ in CWT19]


@pytest.mark.parametrize("wav,scale,num,kw", CWT19, ids=CWT19_IDS)
def test_cwt_2pow19_rows(torch_cuda, report, wav, scale, num, kw):
    torch = torch_cuda
    x = noise(100 + num, N19)
    w = af.CWT(num, 19, SR, wavelet_type=wav, scale_type=scale, is_padding=False, **kw)
    re, im = w.cwt_batch(torch.from_numpy(x[None]).cuda())
    want = cwt_oracle(w, x)
    zero = check_rows(report, "cwt", re[0], im[0], *want)
    assert zero.sum() == (1 if scale == S.LINEAR else 0)


def test_cwt_2pow19_three_clips_short_last_group(torch_cuda, report):
    """3 clips x 61 scales = 183 (clip, scale) items: items of clips 1 and 2 inside the fused kernel, and its groups of
    two end in a one-item group."""
    torch = torch_cuda
    x = np.stack([noise(110 + i, N19) for i in range(3)])
    w = af.CWT(61, 19, SR, wavelet_type=W.PAUL, scale_type=S.OCTAVE, is_padding=False)
    re, im = w.cwt_batch(torch.from_numpy(x).cuda())
    bank = cwt_bank(w)
    for b in range(3):
        check_rows(report, f"clip {b}", re[b], im[b], *cwt_oracle(w, x[b], bank=bank))


@pytest.mark.parametrize("wav,scale,num,kw", [CWT19[1], CWT19[5]], ids=[CWT19_IDS[1], CWT19_IDS[5]])
def test_cwt_det_2pow19_rows(torch_cuda, report, wav, scale, num, kw):
    torch = torch_cuda
    x = noise(120 + num, N19)
    w = af.CWT(num, 19, SR, wavelet_type=wav, scale_type=scale, is_padding=False, **kw)
    w.enable_det(True)
    re, im = w.cwt_det_batch(torch.from_numpy(x[None]).cuda())
    check_rows(report, "det", re[0], im[0], *cwt_oracle(w, x, det=True))


def test_cwt_det_2pow19_reuses_workspace_spectrum(cuda_device):
    """cwtObj_cwtDet(NULL) after cwtObj_cwt: the inverse legs run on the spectrum the forward legs left in the workspace,
    and must give what a full derivative call gives."""
    x = noise(130, N19)
    w = af.CWT(60, 19, SR, wavelet_type=W.PAUL, scale_type=S.MEL, is_padding=False)
    w.enable_det(True)
    w.cwt_planes(x)
    re, im = w.cwt_det_planes(None)
    re2, im2 = w.cwt_det_planes(x)
    assert re.any() and im.any()
    assert np.array_equal(re, re2) and np.array_equal(im, im2)


def test_cwt_2pow19_support_table_cached_per_object(torch_cuda):
    """The bank-support table is computed on an object's first fast-path call and reused: cwt, then det, then another
    batch size on ONE object equal the same calls on fresh objects bit for bit."""
    torch = torch_cuda
    x = torch.from_numpy(np.stack([noise(140, N19), noise(141, N19)])).cuda()

    def fresh(det=False):
        w = af.CWT(60, 19, SR, wavelet_type=W.PAUL, scale_type=S.MEL, is_padding=False)
        if det:
            w.enable_det(True)
        return w
    w = fresh(det=True)
    calls = [("cwt_batch", x[:1]), ("cwt_det_batch", x[:1]), ("cwt_batch", x)]
    for name, data in calls:
        got = getattr(w, name)(data)
        want = getattr(fresh(det=True), name)(data)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), name
        del got, want


# ------------------------------------------------------------------ 2. PWT, N = 2^19 fast path (tabulated bank)
PWT19 = [dict(num=84, scale_type=S.MEL, high_fre=16000.),     # Slaney Mel, top band below Nyquist
         dict(num=100, scale_type=S.LINEAR)]                   # Linear from bin 0 (DESIGN section 1)


@pytest.mark.parametrize("kw", PWT19, ids=["mel84-16k", "linear100"])
def test_pwt_2pow19_rows(torch_cuda, report, kw):
    torch = torch_cuda
    x = noise(150 + kw["num"], N19)
    p = af.PWT(radix2_exp=19, samplate=SR, is_padding=False, **kw)
    re, im = p.pwt_batch(torch.from_numpy(x[None]).cuda())
    check_rows(report, "pwt", re[0], im[0], *pwt_oracle(p, x))


def test_pwt_det_2pow19_rows(torch_cuda, report):
    torch = torch_cuda
    x = noise(160, N19)
    p = af.PWT(radix2_exp=19, samplate=SR, is_padding=False, **PWT19[0])
    p.enable_det(True)
    re, im = p.pwt_det_batch(torch.from_numpy(x[None]).cuda())
    check_rows(report, "pwt det", re[0], im[0], *pwt_oracle(p, x, det=True))


# ------------------------------------------------------------------ 3. general four-step inverse path
# 2^15 (N1 = 256, N2 = 128), 2^17 (512 x 256), 2^18 (512 x 512), 2^20 (1024 x 1024: 4 columns / 4 rows per CTA)
GENERAL = [(15, W.MORLET, S.OCTAVE, 84), (15, W.PAUL, S.MEL, 60),
           (17, W.MORSE, S.MEL, 60), (17, W.DOG, S.OCTAVE, 84),
           (18, W.MEXICAN, S.BARK, 48), (18, W.RICKER, S.OCTAVE, 84),
           (20, W.MORSE, S.OCTAVE, 24), (20, W.PAUL, S.MEL, 24)]


@pytest.mark.parametrize("r,wav,scale,num", GENERAL, ids=[f"2^{r}-{w.name}-{s.name}-{n}" for r, w, s, n in GENERAL])
def test_cwt_general_path_rows(torch_cuda, report, r, wav, scale, num):
    torch = torch_cuda
    x = np.stack([noise(170 + r, 1 << r), noise(171 + r, 1 << r)])
    w = af.CWT(num, r, SR, wavelet_type=wav, scale_type=scale, is_padding=False)
    re, im = w.cwt_batch(torch.from_numpy(x).cuda())
    bank = cwt_bank(w)
    for b in range(2):
        check_rows(report, f"clip {b}", re[b], im[b], *cwt_oracle(w, x[b], bank=bank))


# ------------------------------------------------------------------ 4. long-frame STFT / BFT
def long_chunk_frames(n):
    """Frames per workspace chunk of the long-frame STFT and ISTFT (`launch_stft_long` in stft_generic.cu,
    `launch_istft_frames_long` in istft.cu): 512 MiB at 20 bytes per sample (frame, spectrum, inter-leg buffer)."""
    return (512 << 20) // (20 * n)


STFT_LONG = [(15, 5000, WIN.HANN), (16, 30000, WIN.HAMM), (17, 40000, WIN.BLACKMAN), (18, 100000, WIN.HANN),
             (19, 200000, WIN.RECT), (20, 300000, WIN.HANN)]


@pytest.mark.parametrize("r,hop,wt", STFT_LONG, ids=[f"2^{r}" for r, _, _ in STFT_LONG])
def test_stft_long_frames_half_planes(torch_cuda, report, r, hop, wt):
    torch = torch_cuda
    n = 1 << r
    L = n + 2 * hop + 777
    x = np.stack([noise(180 + r, L), noise(181 + r, L)])
    s = af.STFT(r, wt, hop)
    re, im = s.stft_batch(torch.from_numpy(x).cuda())
    assert tuple(re.shape) == (2, 3, n // 2 + 1)
    for b in range(2):
        wr, wi = O.stft(x[b], n, hop, O.fft_window(af.enum_value(wt), n))
        check_rows(report, f"clip {b}", re[b], im[b], wr[:, :n // 2 + 1], wi[:, :n // 2 + 1])


def test_stft_long_frames_full_planes_2pow18(cuda_device, report):
    n, hop = 1 << 18, 90000
    x = noise(190, n + 3 * hop + 5)
    s = af.STFT(18, WIN.HAMM, hop)
    re, im = s.stft_planes(x)                                     # legacy entry: FULL mirrored planes
    assert re.shape == (4, n)
    check_rows(report, "full", re, im, *O.stft(x, n, hop, O.fft_window(O.W_HAMM, n)))


# SQUARE, HALF and MAG store modes.  Complex mode without squaring sums the signed spectrum over each band, and a Hann
# window makes neighbouring bins so alike that a wide triangular band nearly cancels: any float32 pipeline (numpy's
# included) is 7e-4 (2^16) .. 2e-2 (2^20) away from float64 there, so that mode is checked with a rectangular window.
BFT_MODES = [(0, D.POWER, 1.0, WIN.HANN), (0, D.MAG, 1.0, WIN.RECT), (1, D.MAG, 0.5, WIN.HANN)]


@pytest.mark.parametrize("rt,dt,nv,wt", BFT_MODES, ids=["complex-power", "complex-mag", "mag-norm0.5"])
@pytest.mark.parametrize("r", [16, 20])
def test_bft_long_frames_modes(torch_cuda, report, r, rt, dt, nv, wt):
    torch = torch_cuda
    n = 1 << r
    hop = n // 2
    L = n + 3 * hop + 11
    x = np.stack([noise(200 + r, L), noise(201 + r, L)])
    b = af.BFT(64, r, SR, window_type=wt, slide_length=hop, scale_type=S.MEL, data_type=dt)
    if nv != 1.0:
        b.set_data_norm_value(nv)
    got = b.bft_batch(torch.from_numpy(x).cuda(), result_type=rt)
    for i in range(2):
        want = O.bft(x[i], 64, r, SR, hop, af.enum_value(wt), O.SCALE_MEL, O.STYLE_SLANEY, O.NORM_NONE, af.enum_value(dt),
                     result_type=rt, norm_value=nv)
        if rt == 0:
            check_rows(report, f"clip {i}", got[0][i], got[1][i], *want)
        else:
            check_rows(report, f"clip {i}", got[i], None, want, None)


@pytest.mark.parametrize("r,T,hop", [(15, 500, 1024), (20, 16, 65536)], ids=["2^15", "2^20"])
def test_stft_long_frames_across_workspace_chunks(torch_cuda, report, r, T, hop):
    """2 clips whose frames do not fit one workspace chunk: the first boundary falls inside clip 1 (frame 319 at 2^15,
    frame 9 at 2^20).  The frame transform does not depend on the batch, so each clip equals its single-clip call bit for
    bit -- the frames on both sides of the boundary included -- and every frame matches the oracle."""
    torch = torch_cuda
    n = 1 << r
    chunk = long_chunk_frames(n)
    assert T < chunk < 2 * T
    L = n + (T - 1) * hop
    x = np.stack([noise(210 + r, L), noise(211 + r, L)])
    s = af.STFT(r, WIN.HANN, hop)
    assert s.cal_time_length(L) == T
    xd = torch.from_numpy(x).cuda()
    re, im = s.stft_batch(xd)
    for b in range(2):
        one_re, one_im = s.stft_batch(xd[b:b + 1])
        assert torch.equal(re[b], one_re[0]) and torch.equal(im[b], one_im[0]), b
        wr, wi = O.stft(x[b], n, hop, O.fft_window(O.W_HANN, n))
        check_rows(report, f"clip {b}", re[b], im[b], wr[:, :n // 2 + 1], wi[:, :n // 2 + 1])
        del wr, wi


# ------------------------------------------------------------------ 5. long-frame ISTFT
@pytest.mark.parametrize("r,hop,wt,method", [(18, 1 << 16, 1, 0), (19, 200000, 2, 1), (20, 1 << 18, 1, 0)],
                         ids=["2^18", "2^19", "2^20"])
def test_istft_long_frames_2pow18_to_2pow20(torch_cuda, report, r, hop, wt, method):
    """Full planes through the legacy host entry and half planes through the batched device entry, against the oracle
    (2^19: the fast path's forward legs inside the Hartley identity)."""
    torch = torch_cuda
    n = 1 << r
    w = O.fft_window(wt, n)
    x = noise(220 + r, n + 5 * hop)
    re, im = O.stft(x, n, hop, w)
    want = O.istft(re, im, n, hop, w, method)
    ok = istft_conditioned(n, hop, re.shape[0], w, method)
    s = af.STFT(r, WIN(wt), hop)
    full = s.istft_planes(re, im, method)
    hre = torch.from_numpy(np.ascontiguousarray(re[None, :, :n // 2 + 1])).cuda()
    him = torch.from_numpy(np.ascontiguousarray(im[None, :, :n // 2 + 1])).cuda()
    half = s.istft_batch(hre, him, method)[0].cpu().numpy()
    for name, y in (("full", full), ("half", half)):
        assert y.shape == want.shape
        err = rel_max(y[ok], want[ok])
        report(name, err, err)
        assert err < TOL, name
        assert np.abs(y - want).max() <= 1e-2 * np.abs(want).max(), name
    if method == 0 and n // hop >= 4:
        assert rel_max(full[n:-n], x[n:-n]) < TOL                    # round trip where the windows overlap fully


def test_istft_long_frames_across_workspace_chunks(torch_cuda, report):
    """More frames than one workspace chunk holds at 2^15 (see long_chunk_frames): the frame loop of the long ISTFT runs
    twice, and the frames of the second chunk must land at their own positions."""
    torch = torch_cuda
    r, hop = 15, 4096
    n = 1 << r
    T = long_chunk_frames(n) + 81
    w = O.fft_window(O.W_HANN, n)
    x = noise(230, n + (T - 1) * hop)
    re, im = O.stft(x, n, hop, w)
    assert re.shape[0] == T
    s = af.STFT(r, WIN.HANN, hop)
    hre = torch.from_numpy(np.ascontiguousarray(re[None, :, :n // 2 + 1])).cuda()
    him = torch.from_numpy(np.ascontiguousarray(im[None, :, :n // 2 + 1])).cuda()
    y = s.istft_batch(hre, him, 0)[0].cpu().numpy()
    del hre, him
    want = O.istft(re, im, n, hop, w, 0)
    ok = istft_conditioned(n, hop, T, w, 0)
    err = rel_max(y[ok], want[ok])
    report("half", err, err)
    assert y.shape == want.shape and err < TOL
    assert rel_max(y[n:-n], x[n:-n]) < TOL
