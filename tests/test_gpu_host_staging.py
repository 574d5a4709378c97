"""Host-pointer staging of the batched entry points (af_run_batch, csrc/host/af_ctx.c): a host batch that spans at
least three chunks must give bit for bit what the device-pointer call gives, in-out planes that start non-zero must
accumulate to the same bits, and a batch of one must equal the legacy single-call entry point."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

MB64 = 64 << 20


def _af():
    import audioflux_b200 as af
    return af


def chunk_items(in_bytes, out_bytes, budget=MB64):
    """items per chunk: about `budget` bytes of the larger side, a multiple of 16 from 16 items on, at least 1"""
    per = max(1, budget // max(in_bytes, out_bytes))
    return per - per % 16 if per >= 16 else per


def three_chunks(in_bytes, out_bytes, budget=MB64):
    per = chunk_items(in_bytes, out_bytes, budget)
    return per, 2 * per + per // 2 + 1


def rand(rng, *shape, lo=0.0):
    return (lo + rng.random(shape)).astype(np.float32)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def same(host, device):
    d = device.cpu().numpy() if isinstance(device, torch.Tensor) else device
    assert host.shape == d.shape and np.array_equal(host, d)


def ptr(a):
    return C.c_void_p(a.data_ptr()) if isinstance(a, torch.Tensor) else a.ctypes.data_as(C.c_void_p)


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def run(fn, *args, device):
    from audioflux_b200.lib import check
    check(fn(*args, 1 if device else 0, stream() if device else C.c_void_p(None)), fn.__name__)
    if device:
        torch.cuda.synchronize()


def test_xxcc_rows_host_equals_device(cuda_device):
    af = _af()
    rng = np.random.default_rng(1)
    num, cc = 40, 13
    _, rows = three_chunks(4 * num, 4 * cc)
    m = rand(rng, rows, num, lo=0.01)
    x = af.XXCC(num)
    same(x.xxcc_batch(m, cc), x.xxcc_batch(dev(m), cc))
    x.set_time_length(50)
    same(x.xxcc_batch(m[:50], cc), x.xxcc_planes(m[:50], cc))
    e = rand(rng, rows, lo=0.5)
    W = cc + 1
    _, rows2 = three_chunks(4 * (num + 1), 3 * 4 * W)
    rows2 = min(rows2, rows)
    h = x.xxcc_standard_batch(m[:rows2], e[:rows2], cc, energy_type=af.CepstralEnergyType.APPEND)
    d = x.xxcc_standard_batch(dev(m[:rows2]), dev(e[:rows2]), cc, energy_type=af.CepstralEnergyType.APPEND)
    for a, b in zip(h, d):
        same(a, b)


def test_cqt_rows_host_equals_device(cuda_device):
    af = _af()
    rng = np.random.default_rng(2)
    c = af.CQT(84, 48000)
    _, rows = three_chunks(2 * 4 * 84, 4 * 12)
    re, im = rand(rng, rows, 84, lo=-0.5), rand(rng, rows, 84, lo=-0.5)
    mag = np.abs(re) + 0.01
    same(c.chroma_batch(re, im), c.chroma_batch(dev(re), dev(im)))
    same(c.cqcc_batch(mag, 20), c.cqcc_batch(dev(mag), 20))
    same(c.cqhc_batch(mag, 20), c.cqhc_batch(dev(mag), 20))
    _, rows = three_chunks(4 * 84, 2 * 4 * 84)
    for a, b in zip(c.deconv_batch(mag[:rows]), c.deconv_batch(dev(mag[:rows]))):
        same(a, b)
    T = c.cqt_planes(np.zeros(48000, np.float32))[0].shape[0]      # the legacy calls take the rows of the last cqt call
    same(c.chroma_batch(re[:T], im[:T]), c.chroma_planes(re[:T], im[:T]))
    same(c.cqcc_batch(mag[:T], 20), c.cqcc_planes(mag[:T], 20))
    same(c.cqhc_batch(mag[:T], 20), c.cqhc_planes(mag[:T], 20))
    for a, b in zip(c.deconv_batch(mag[:T]), c.deconv_planes(mag[:T])):
        same(a, b)


def test_spectrogram_deconv_and_phase_host_equals_device(cuda_device):
    af = _af()
    rng = np.random.default_rng(3)
    s = af.Spectrogram(samplate=48000, radix2_exp=11, slide_length=512)
    num = s.get_band_num()
    _, rows = three_chunks(4 * num, 2 * 4 * num)
    mag = rand(rng, rows, num, lo=0.01)
    for a, b in zip(s.deconv_batch(mag), s.deconv_batch(dev(mag))):
        same(a, b)
    L = 30720
    T = s.cal_time_length(L)
    _, B = three_chunks(4 * L, 2 * 4 * T * num)
    x = (0.1 * rng.standard_normal((B, L))).astype(np.float32)
    hs, hph = s.spectrogram_batch(x, is_phase_arr=True)
    ds, dph = s.spectrogram_batch(dev(x), is_phase_arr=True)
    same(hs, ds)
    same(hph, dph)
    ls, lph = s.spectrogram_planes(x[7], is_phase_arr=True)
    same(hs[7], ls)
    same(hph[7], lph)


def test_spectral_host_equals_device_with_preloaded_out(cuda_device):
    af = _af()
    from audioflux_b200.spectral import encode
    rng = np.random.default_rng(4)
    num, T = 128, 100
    s = af.Spectral(num, np.linspace(0, 16000, num).astype(np.float32))
    _, B = three_chunks(2 * 4 * T * num, 4 * 4 * T)
    spec, phase = rand(rng, B, T, num, lo=0.01), rand(rng, B, T, num, lo=-3.0)
    feats = ["pd", "var", "centroid"]                   # pd / var leave frames as they were: out is an in-out plane
    enc = [encode(f) for f in feats]
    req = np.array([e[0] for e in enc], np.int32)
    par = np.array([e[1] for e in enc], np.float32).reshape(-1)
    out0 = rand(rng, 4, B, T, lo=-1.0)
    fn = s._lib.spectralObj_spectralBatch
    oh = out0.copy()
    run(fn, s._obj, ptr(spec), ptr(phase), T, B, len(feats), ptr(req), ptr(par), ptr(oh), device=False)
    sd, pd_, od = dev(spec), dev(phase), dev(out0)
    run(fn, s._obj, ptr(sd), ptr(pd_), T, B, len(feats), ptr(req), ptr(par), ptr(od), device=True)
    same(oh, od)
    assert not np.array_equal(oh, out0)
    o1 = out0[:, :1].copy()
    run(fn, s._obj, ptr(spec[:1]), ptr(phase[:1]), T, 1, len(feats), ptr(req), ptr(par), ptr(o1), device=False)
    same(o1, oh[:, :1])


def test_istft_host_equals_device_accumulating(cuda_device):
    af = _af()
    rng = np.random.default_rng(5)
    st = af.STFT(9, af.WindowType.HANN, 128)
    n, T = 512, 20
    W = n // 2 + 1
    L = st.cal_data_length(T)
    _, B = three_chunks(2 * 4 * T * W, 4 * L)
    re, im = rand(rng, B, T, W, lo=-0.5), rand(rng, B, T, W, lo=-0.5)
    data0 = rand(rng, B, L, lo=-1.0)
    fn = st._lib.stftObj_istftBatch
    dh = data0.copy()
    run(fn, st._obj, ptr(re), ptr(im), T, B, W, 0, ptr(dh), device=False)
    rd, id_, dd = dev(re), dev(im), dev(data0)
    run(fn, st._obj, ptr(rd), ptr(id_), T, B, W, 0, ptr(dd), device=True)
    same(dh, dd)
    full = np.concatenate([re[0], re[0, :, -2:0:-1]], axis=-1), np.concatenate([im[0], -im[0, :, -2:0:-1]], axis=-1)
    full = [np.ascontiguousarray(a[None]) for a in full]
    z = np.zeros((1, L), np.float32)
    run(fn, st._obj, ptr(full[0]), ptr(full[1]), T, 1, n, 0, ptr(z), device=False)
    same(z[0], st.istft_planes(full[0][0], full[1][0]))


@pytest.mark.parametrize("re_type,result_type", [("ALL", 0), ("ALL", 1), ("NONE", 0)])
def test_reassign_host_equals_device_accumulating(cuda_device, re_type, result_type):
    af = _af()
    rng = np.random.default_rng(6)
    r = af.Reassign(9, 32000, re_type=getattr(af.ReassignType, re_type))
    r.set_result_type(result_type)
    L = 4096
    T, W = r.cal_time_length(L), 512 // 2 + 1
    _, B = three_chunks(4 * (L + 2 * T * W), 4 * 4 * T * W)
    x = (0.1 * rng.standard_normal((B, L))).astype(np.float32)
    init = [rand(rng, B, T, W, lo=-1.0) for _ in range(2)] + [np.zeros((B, T, W), np.float32) for _ in range(2)]
    fn = r._lib.reassignObj_reassignBatch
    h = [a.copy() for a in init]
    run(fn, r._obj, ptr(x), L, B, *[ptr(a) for a in h], device=False)
    xd, d = dev(x), [dev(a) for a in init]
    run(fn, r._obj, ptr(xd), L, B, *[ptr(a) for a in d], device=True)
    for k, (a, b) in enumerate(zip(h, d)):
        if k != 1 or result_type == 0 or re_type == "NONE":      # im4 comes back only when the result asks for it
            same(a, b)
    one = [np.zeros((1, T, W), np.float32) for _ in range(4)]
    run(fn, r._obj, ptr(x[:1]), L, 1, *[ptr(a) for a in one], device=False)
    re, im, sr, si = r.reassign_planes(x[0], result_type)
    same(one[0][0], re)
    if result_type == 0 or re_type == "NONE":
        same(one[1][0], im)
    if re_type != "NONE":
        same(one[2][0], sr)
        same(one[3][0], si)


def test_cwt_and_nsgt_cells_host_equals_device(cuda_device):
    af = _af()
    rng = np.random.default_rng(7)
    w = af.CWT(8, 10, 32000, wavelet_type=af.WaveletContinueType.MORLET, is_padding=False)
    N = 1 << 10
    _, B = three_chunks(4 * N, 2 * 4 * 8 * N, budget=1024 << 20)
    x = (0.1 * rng.standard_normal((B, N))).astype(np.float32)
    hr, hi = w.cwt_batch(x)
    dr, di = w.cwt_batch(dev(x))
    same(hr, dr)
    same(hi, di)
    del hr, hi, dr, di
    g = af.NSGT(84, 12, 32000)
    N = 1 << 12
    ho = g.nsgt_batch(np.zeros((1, N), np.float32), with_cells=True)
    per_out = sum(a[0].size for a in ho)
    _, B = three_chunks(4 * N, 4 * per_out)
    x = (0.1 * rng.standard_normal((B, N))).astype(np.float32)
    for a, b in zip(g.nsgt_batch(x, with_cells=True), g.nsgt_batch(dev(x), with_cells=True)):
        same(a, b)
