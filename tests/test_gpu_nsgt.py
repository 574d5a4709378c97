"""NSGT on the GPU: the reference's entry points against the oracle and the reference build, the batched entry point
(host and device pointers, any batch size), the matrix as a gather of the cells, the launch count, the direct path of
the widest bands (end to end, and band by band on the GPU's own spectrum), setMinLength, and the reference's own NSGT
class running on libaudioflux_b200.so.  test_gpu_nsgt_bands.py checks every band kernel path band by band."""
import numpy as np
import pytest

from conftest import rel_max
import _nsgt_oracle as NO
from _parity_kit import count_launches, raf, ref_lib_or_none  # noqa: F401  (raf: a fixture)

import audioflux_b200 as af
from oracle import af_oracle as O

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _cell_gather(cr, ci, lens, cmap):
    off = np.concatenate([[0], np.cumsum(lens)[:-1]])
    c = cr.astype(np.complex64) + 1j * ci.astype(np.complex64)
    return np.where(cmap >= 0, c[off[:, None] + np.maximum(cmap, 0)], 0)


@pytest.mark.parametrize("name,kw", NO.cases(), ids=[c[0] for c in NO.cases()])
def test_legacy_matches_oracle_and_reference(product_lib, cuda_device, name, kw):
    ref = ref_lib_or_none()
    _, p = NO.params(**kw)
    x = NO.case_signal(7, p["fft_length"], p["samplate"])
    st, obj = NO.c_new(product_lib, **kw)
    assert st == 0
    re, im, cr, ci = NO.c_nsgt(product_lib, obj, x, kw["num"])
    assert product_lib.afb200_lastError() in (b"", None)
    cells, m = NO.transform(x, p)
    c = np.concatenate(cells)
    assert rel_max(re, m.real) <= TOL and rel_max(im, m.imag) <= TOL, name
    assert rel_max(cr, c.real) <= TOL and rel_max(ci, c.imag) <= TOL, name
    b = NO.bank(p)
    cmap = NO.column_map(b["lens"], p["fft_length"], p["samplate"])
    assert np.array_equal(re + 1j * im, _cell_gather(cr, ci, b["lens"], cmap)), name      # matrix = its own cells, exactly
    if ref is not None:
        sr_, ro = NO.c_new(ref, **kw)
        rre, rim, rcr, rci = NO.c_nsgt(ref, ro, x, kw["num"])
        ref.nsgtObj_free(ro)
        assert rel_max(re, rre) <= TOL and rel_max(im, rim) <= TOL, name
        assert rel_max(cr, rcr) <= TOL and rel_max(ci, rci) <= TOL, name
    product_lib.nsgtObj_free(obj)


def test_batch_host_device_bit_identical_to_legacy(product_lib, cuda_device):
    import torch
    for kw in (NO.cases()[-3][1], dict(num=40, radix2_exp=12, scale_type=O.SCALE_MEL, style_type=O.STYLE_HANN,
                                         bank_type=NO.STANDARD)):
        n = 1 << kw["radix2_exp"]
        x = np.stack([NO.case_signal(s, n, kw.get("samplate") or 32000) * (1 + 10 * (s == 2)) for s in range(5)])
        st, obj = NO.c_new(product_lib, **kw)
        assert st == 0
        legacy = [NO.c_nsgt(product_lib, obj, x[b], kw["num"]) for b in range(len(x))]
        product_lib.nsgtObj_free(obj)
        t = af.NSGT(num=kw["num"], radix2_exp=kw["radix2_exp"], samplate=kw.get("samplate") or 32000,
                    low_fre=kw.get("low_fre"), min_len=kw.get("min_len") or 3,
                    nsgt_filter_bank_type=kw.get("bank_type") or 0, scale_type=kw["scale_type"],
                    style_type=kw["style_type"], normal_type=kw.get("normal_type", 2))
        for nb in (1, 2, 5):
            host = t.nsgt_batch(x[:nb], with_cells=True)
            dev = t.nsgt_batch(torch.from_numpy(x[:nb]).cuda(), with_cells=True)
            torch.cuda.synchronize()
            for b in range(nb):
                for k in range(4):
                    assert np.array_equal(host[k][b], legacy[b][k]), (nb, b, k)
                    assert np.array_equal(dev[k][b].cpu().numpy(), legacy[b][k]), (nb, b, k, "device")
        re, im = t.nsgt_batch(x)          # without cells: the pipelined host path
        for b in range(len(x)):
            assert np.array_equal(re[b], legacy[b][0]) and np.array_equal(im[b], legacy[b][1])


def test_launch_count(product_lib, cuda_device):
    """af_launch_stft's launches (one up to 2^14 points), one Bluestein launch, one direct launch when a band is wider
    than 4096"""
    import torch
    x12 = torch.zeros((3, 1 << 12), device="cuda")
    t = af.NSGT(num=84, radix2_exp=12)
    assert count_launches(product_lib, lambda: t.nsgt_batch(x12), warm=True) == 2
    x19 = torch.zeros((2, 1 << 19), device="cuda")
    wide = af.NSGT(num=84, radix2_exp=19, samplate=44100)             # widest band 5587: direct path
    narrow = af.NSGT(num=84, radix2_exp=19, samplate=196000)          # same FFT, every band <= 4096
    assert wide.get_time_length_arr().max() > 4096 >= narrow.get_time_length_arr().max()
    assert (count_launches(product_lib, lambda: wide.nsgt_batch(x19), warm=True) ==
            count_launches(product_lib, lambda: narrow.nsgt_batch(x19), warm=True) + 1)


def _gpu_spectrum(x):
    """the clips' forward FFT exactly as nsgtObj_nsgtBatch computes it (af_launch_stft: rect window, one frame, half
    planes), mirrored to the full complex128 spectrum [clips, N]"""
    r = x.shape[-1].bit_length() - 1
    re, im = af.STFT(r, af.WindowType.RECT, 1 << r).stft_batch(x)
    return NO.full_spectrum(re[:, 0], im[:, 0])


def _oracle_check(t, x, kw):
    """end to end against the float64 FFT of each clip per tensor, and every band against the oracle's band step on the
    GPU's own spectrum per band"""
    _, p = NO.params(**kw)
    b = NO.bank(p)
    re, im, cr, ci = t.nsgt_batch(x, with_cells=True)
    X = _gpu_spectrum(x)
    for c in range(len(x)):
        _, m = NO.transform(x[c], p, b)
        assert rel_max(re[c], m.real) <= TOL and rel_max(im[c], m.imag) <= TOL, (kw, c)
        want, _ = NO.transform_spectrum(X[c], p, b)
        NO.check_bands(NO.split_cells(cr[c], ci[c], b["lens"]), want, b["lens"], what=(kw, c))


def test_direct_path_octave84_2e19(product_lib, cuda_device):
    kw = dict(num=84, radix2_exp=19, samplate=44100, low_fre=32.703196, scale_type=O.SCALE_OCTAVE,
              style_type=O.STYLE_SLANEY)
    t = af.NSGT(num=84, radix2_exp=19, samplate=44100, scale_type=af.SpectralFilterBankScaleType.OCTAVE)
    lens = t.get_time_length_arr()
    assert lens.max() == 5587 and (lens > 4096).sum() >= 1
    x = np.stack([NO.case_signal(s, 1 << 19, 44100) for s in range(2)])
    _oracle_check(t, x, kw)


def test_direct_path_linear_2e15(product_lib, cuda_device):
    kw = dict(num=4, radix2_exp=15, samplate=32000, low_fre=1000.0, min_len=6000, scale_type=O.SCALE_LINEAR,
              style_type=O.STYLE_HANN, normal_type=O.NORM_NONE)
    t = af.NSGT(num=4, radix2_exp=15, low_fre=1000.0, min_len=6000, scale_type=af.SpectralFilterBankScaleType.LINEAR,
                style_type=af.SpectralFilterBankStyleType.HANN, normal_type=af.SpectralFilterBankNormalType.NONE)
    assert (t.get_time_length_arr() == 6000).all()
    x = np.stack([NO.case_signal(s, 1 << 15, 32000) for s in range(3)])
    _oracle_check(t, x, kw)


def test_set_min_length_equals_fresh_object(product_lib, cuda_device):
    x = NO.case_signal(3, 1 << 12, 32000)
    for start, to in ((20, 3), (3, 20), (3, 200), (200, 1)):
        a = af.NSGT(num=84, radix2_exp=12, min_len=start)
        a.nsgt(x)
        a.set_min_length(to)
        b = af.NSGT(num=84, radix2_exp=12, min_len=to)
        assert a.get_max_time_length() == b.get_max_time_length()
        assert np.array_equal(a.get_time_length_arr(), b.get_time_length_arr())
        assert np.array_equal(a.nsgt(x), b.nsgt(x)), (start, to)


def test_refusals(product_lib):
    for kw in (dict(num=84, radix2_exp=21), dict(num=4, radix2_exp=16, scale_type=O.SCALE_LINEAR, min_len=20000)):
        st, obj = NO.c_new(product_lib, **kw)
        assert st == -2 and not obj.value, kw
        assert product_lib.afb200_lastError()


def test_reference_nsgt_class_on_b200(raf, cuda_device):
    T = raf.type
    rng = np.random.default_rng(5)
    mono = NO.case_signal(11, 1 << 13, 32000)
    multi = (0.1 * rng.standard_normal((2, 3, 1 << 13))).astype(np.float32)
    configs = [dict(num=84, radix2_exp=13),
               dict(num=40, radix2_exp=13, scale_type=T.SpectralFilterBankScaleType.MEL,
                    style_type=T.SpectralFilterBankStyleType.HANN,
                    nsgt_filter_bank_type=T.NSGTFilterBankType.STANDARD,
                    normal_type=T.SpectralFilterBankNormalType.NONE)]
    for kw in configs:
        res = {}
        for which in ("ref", "b200"):
            raf.fftlib.set_fft_lib(lib_ext="b200" if which == "b200" else None)
            o = raf.NSGT(**kw)
            res[which] = (o.nsgt(mono), o.nsgt(multi), o.get_time_length_arr(), o.get_fre_band_arr(),
                          o.get_bin_band_arr(), o.get_max_time_length(), o.get_total_time_length(),
                          o.x_coords(1 << 13), o.y_coords())
            # downwards only: the reference's grids stay those of the larger lengths, so it stays in bounds; compare
            # this library after set_min_length with fresh reference objects
            shrunk = []
            for m in (9, 2):
                if which == "b200":
                    o2 = raf.NSGT(**dict(kw, min_len=20))
                    o2.set_min_length(m)
                else:
                    o2 = raf.NSGT(**dict(kw, min_len=m))
                shrunk.append(o2.nsgt(mono))
            res[which] += tuple(shrunk)
        raf.fftlib.set_fft_lib(None)
        g, r = res["b200"], res["ref"]
        for k in (0, 1, 9, 10):
            assert g[k].shape == r[k].shape, (kw, k)
            assert rel_max(g[k].real, r[k].real) <= TOL and rel_max(g[k].imag, r[k].imag) <= TOL, (kw, k)
        for k in (2, 3, 4, 5, 6, 7, 8):
            assert np.array_equal(np.asarray(g[k]), np.asarray(r[k])), (kw, k)
