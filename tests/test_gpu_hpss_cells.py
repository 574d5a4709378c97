"""The masks of harmonic-percussive separation (k_hpss_mask, kernels/hpss.cu) cell by cell and bit for bit, on crafted
planes and on the GPU's own spectra.

k_hpss_mask's result can be predicted exactly: the medians are selections, hpss.cu is built with -fmad=false and without
fast-math (sqrtf and / are IEEE-rounded, subnormals are kept), and every mask step is one float32 operation in the order
its header gives.  So _hpss_oracle.mask_model, numpy float32 in that order, must match every H and P cell bit for bit,
sign of zero included; tests/test_hpss_cpu.py pins the model to scipy's median_filter and to the float64 formula.

  - Cells: af_launch_hpss_mask called through ctypes (_hpss_oracle.AfHpssArgs, pinned to csrc/af_internal.h on the CPU)
    on device planes [3 * T, W], on the current stream, at the shapes and orders of _hpss_oracle.MASK_SHAPES and every
    value pattern of _hpss_oracle.PATTERNS.  Each call carries three clips, the middle one 1000x louder and reversed in
    time, so a window that crossed into a neighbouring clip would show.  Each call asserts one launch, guard floats
    untouched before and after every output plane, and a skipped output (hRe or pRe NULL, its im pointer still set)
    left at its sentinel.  The host refuses even orders, order 0, orders above 383 and two NULL outputs with its own
    message and no launch.
  - The composed route: for every case of _hpss_oracle.cases(), HPSS.hpss_batch must equal, bit for bit, the same
    computation through public calls: STFT.stft_batch (hop N/4, no padding), mask_model, STFT.istft_batch (method 0).
    Both routes make the same af_launch_stft (half spectrum) and af_launch_istft calls.  Each output sample is also
    held to 1e-4 of its own share (_hpss_oracle.istft64) against the float64 formula and inverse STFT applied to the
    GPU's own spectra; samples whose share is 0 must be exactly 0.  The STFT's own error is left to its suites and to
    tests/test_gpu_hpss.py, which compares with the float64 oracle from the clip.

Inputs are finite.  NaN and inf magnitudes are left out: median_first gives 0 for a window it cannot rank.
"""
import ctypes as C

import numpy as np
import pytest

import _hpss_oracle as HO
from _parity_kit import count_launches, stream

import audioflux_b200 as af

pytestmark = pytest.mark.gpu

GUARD = 64                   # sentinel floats before and after each output plane
SENTINEL = 0x7FA5A5A5        # a NaN bit pattern, which no finite input produces
PLANES = ("hRe", "hIm", "pRe", "pIm")
TOL = 1e-4


@pytest.fixture
def report(request, capsys):
    """report(case, what, worst): prints a case's worst relative error past pytest's capture and records it"""
    def emit(case, what, worst):
        request.node.user_properties.append((f"{case} {what}", worst))     # (name, value), as junitxml reads them
        with capsys.disabled():
            print(f"\n    {case} {what}: {worst:.2e}", end="")
    return emit


def _ptr(t, offset=0):
    return C.cast(C.c_void_p(t.data_ptr() + 4 * offset), HO.FLOAT_P)


def launch(lib, re, im, T, W, h, p, outputs="hp"):
    """one af_launch_hpss_mask call over the device planes re / im [3 * T, W] into sentinel-filled buffers with GUARD
    floats on both sides; a skipped output passes NULL for its re plane and a live pointer for its im plane
    -> (status, launches, {plane: the whole buffer as int32 numpy})"""
    import torch
    n = re.numel()
    bufs = {k: torch.full((n + 2 * GUARD,), SENTINEL, dtype=torch.int32, device="cuda") for k in PLANES}
    a = HO.AfHpssArgs(re=_ptr(re), im=_ptr(im), clips=3, timeLength=T, width=W, hOrder=h, pOrder=p)
    for k, b in bufs.items():
        setattr(a, k, _ptr(b, GUARD))
    if "h" not in outputs:
        a.hRe = None
    if "p" not in outputs:
        a.pRe = None
    rc = []
    launches = count_launches(lib, lambda: rc.append(lib.af_launch_hpss_mask(C.byref(a), stream())), warm=False)
    return rc[0], launches, {k: b.cpu().numpy() for k, b in bufs.items()}


def check_cells(case, got, model, outputs):
    """guards untouched; requested planes equal the model bit for bit; skipped planes at their sentinel"""
    for k, name in enumerate(PLANES):
        b = got[name]
        assert (b[:GUARD] == SENTINEL).all() and (b[-GUARD:] == SENTINEL).all(), (case, name, "guard floats written")
        body = b[GUARD:-GUARD]
        if "hp"[k // 2] not in outputs:
            assert (body == SENTINEL).all(), (case, name, "skipped output written")
            continue
        want = model[k].view(np.int32).ravel()
        bad = np.flatnonzero(body != want)
        W = model[k].shape[1]
        assert bad.size == 0, (case, name, f"{bad.size} cells differ", [(int(i // W), int(i % W)) for i in bad[:8]],
                               body[bad[:8]].view(np.float32).tolist(), want[bad[:8]].view(np.float32).tolist())


def _shape_id(s):
    return "T{}_W{}_h{}_p{}".format(*s)


@pytest.mark.parametrize("shape", HO.MASK_SHAPES, ids=[_shape_id(s) for s in HO.MASK_SHAPES])
def test_mask_cells_bit_for_bit(product_lib, cuda_device, shape):
    """every value pattern with both outputs, then the Gaussian planes with H only and with P only"""
    import torch
    T, W, h, p = shape
    runs = [(pattern, "hp") for pattern in HO.PATTERNS] + [("gauss", "h"), ("gauss", "p")]
    for pattern, outputs in runs:
        case = (_shape_id(shape), pattern, outputs)
        re, im = HO.mask_planes(pattern, T, W)
        rc, launches, got = launch(product_lib, torch.from_numpy(re).cuda(), torch.from_numpy(im).cuda(), T, W, h, p,
                                   outputs)
        assert rc == 0 and launches == 1, (case, rc, launches, product_lib.afb200_lastError())
        check_cells(case, got, HO.mask_model(re, im, 3, h, p), outputs)


@pytest.mark.parametrize("h,p,outputs", [(2, 31, "hp"), (21, 30, "hp"), (0, 31, "hp"), (21, 0, "h"),
                                         (HO.MAX_ORDER + 2, 31, "hp"), (21, HO.MAX_ORDER + 2, "p"), (21, 31, "")])
def test_mask_refusals(product_lib, cuda_device, h, p, outputs):
    """checked on the host before any launch: a non-zero status, this call's own message (the error is cleared first,
    since the launcher does not clear it), and every buffer left at its sentinel"""
    import torch
    re, im = (torch.from_numpy(a).cuda() for a in HO.mask_planes("gauss", 33, 129))
    product_lib.af_clear_error()
    rc, launches, got = launch(product_lib, re, im, 33, 129, h, p, outputs)
    assert rc != 0 and launches == 0, (h, p, outputs, rc, launches)
    want = f"hpss mask: orders {h} / {p};" if outputs else "hpss mask: no output"
    assert product_lib.afb200_lastError().startswith(want.encode()), (want, product_lib.afb200_lastError())
    for k in PLANES:
        assert (got[k] == SENTINEL).all(), (h, p, outputs, k)


CASES = dict(HO.cases())


@pytest.mark.parametrize("name", list(CASES))
def test_composed_route_on_own_spectra(product_lib, cuda_device, report, name):
    import torch
    kw = CASES[name]
    r = kw["radix2_exp"]
    n = 1 << r
    ho, po, window = HO.rules(kw.get("h_order"), kw.get("p_order"), kw.get("window"))
    x = HO.case_signal(name, kw)
    clips = np.stack([x, 1000 * x[::-1], HO.case_signal(name + "_third", kw)])
    xd = torch.from_numpy(clips).cuda()
    got = af.HPSS(radix2_exp=r, window_type=window, h_order=ho, p_order=po).hpss_batch(xd)
    stft = af.STFT(r, window_type=window, slide_length=n // 4)
    re, im = (t.cpu().numpy() for t in stft.stft_batch(xd))
    T, W = re.shape[1:]
    re, im = re.reshape(3 * T, W), im.reshape(3 * T, W)
    planes = [torch.from_numpy(m.reshape(3, T, W)).cuda() for m in HO.mask_model(re, im, 3, ho, po)]
    mine = [stft.istft_batch(planes[2 * k], planes[2 * k + 1], 0) for k in range(2)]
    want = HO.mask_ref64(re, im, 3, ho, po)
    win = stft.get_window_data_arr()
    worst = 0.0
    for k in range(2):
        g = got[k].cpu().numpy()
        assert np.array_equal(g.view(np.int32), mine[k].cpu().numpy().view(np.int32)), (name, "hp"[k])
        for c in range(3):
            rows = slice(c * T, (c + 1) * T)
            y, share = HO.istft64(want[2 * k][rows], want[2 * k + 1][rows], n, win)
            err = np.abs(g[c].astype(np.float64) - y)
            live = share > 0
            bad = np.flatnonzero(live & (err > TOL * share))
            assert bad.size == 0, (name, "hp"[k], c, bad[:8].tolist(), (err[bad] / share[bad])[:8].tolist())
            assert (g[c][~live] == 0).all(), (name, "hp"[k], c, "zero-share samples not zero")
            if live.any():
                worst = max(worst, float((err[live] / share[live]).max()))
    report(name, "worst sample over its share", worst)
