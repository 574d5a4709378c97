"""ST / FST on the GPU: the reference's entry points against the oracle and the reference build at every supported size
(both shared-memory paths of k_st_rows), FST rows as the exact expansion of their partition segment, the batched entry
points (host and device pointers, batches that span several staging chunks) bit-identical to the legacy calls, the
launch count, and the reference's own ST / FST classes running on libaudioflux_b200.so."""
import numpy as np
import pytest

import _st_oracle as SO
from _parity_kit import count_launches, raf, ref_lib_or_none  # noqa: F401  (raf: a fixture)

import audioflux_b200 as af

pytestmark = pytest.mark.gpu
TOL = 1e-4          # per row, of the row's own max |want| (DESIGN section 2)
ZERO_TOL = 1e-20    # rows that are exactly zero in the want


def _check_rows(re, im, want, what):
    err, scale = SO.row_errors(re, im, want)
    bad = np.where(scale > 0, err > TOL, err > ZERO_TOL)
    assert not bad.any(), (what, int(np.argmax(err)), float(err.max()))


def _st_cases():
    return [("st1_full", dict(radix2_exp=1, min_index=0, max_index=0)),
            ("st2_full", dict(radix2_exp=2, min_index=0, max_index=0))] + SO.st_cases()


@pytest.mark.parametrize("name,kw", _st_cases(), ids=[c[0] for c in _st_cases()])
def test_st_legacy_matches_oracle_and_reference(product_lib, cuda_device, name, kw):
    x = SO.case_signal(3, 1 << kw["radix2_exp"])
    re, im = SO.c_st_case(product_lib, kw, x)
    assert product_lib.afb200_lastError() in (b"", None)
    _check_rows(re, im, SO.oracle_st_case(kw, x), (name, "oracle"))
    bins = SO.st_rows(kw)
    assert all(not im[r].any() for r, b in enumerate(bins) if b == 0)          # bin 0: an imaginary row of 0
    ref = ref_lib_or_none()
    if ref is not None and kw["radix2_exp"] >= 3:
        rre, rim = SO.c_st_case(ref, kw, x)
        _check_rows(re, im, rre.astype(np.float64) + 1j * rim, (name, "reference"))


@pytest.mark.parametrize("name,kw", SO.fst_cases(), ids=[c[0] for c in SO.fst_cases()])
def test_fst_legacy_matches_oracle_and_reference(product_lib, cuda_device, name, kw):
    x = SO.case_signal(4, 1 << kw["radix2_exp"])
    re, im = SO.c_fst_case(product_lib, kw, x)
    assert product_lib.afb200_lastError() in (b"", None)
    _check_rows(re, im, SO.fst(x, kw["min_index"], kw["max_index"]), (name, "oracle"))
    ref = ref_lib_or_none()
    if ref is not None:
        rre, rim = SO.c_fst_case(ref, kw, x)
        _check_rows(re, im, rre.astype(np.float64) + 1j * rim, (name, "reference"))


@pytest.mark.parametrize("r", [3, 6, 10, 12, 14])
def test_fst_rows_expand_their_segment_exactly(product_lib, cuda_device, r):
    """every row is one partition segment, each value repeated N/len times; rows of one segment are identical"""
    n = 1 << r
    x = SO.case_signal(9, n)
    s, obj = SO.c_fst_new(product_lib, r)
    re, im = SO.c_fst(product_lib, obj, x, 0, n // 2)
    product_lib.fstObj_free(obj)
    z = re + 1j * im.astype(np.complex64)
    first = {}
    for f in range(n // 2 + 1):
        start, ln = SO.fst_segment_of(r, f)
        blocks = z[f].reshape(ln, n // ln)
        assert np.array_equal(blocks, np.repeat(blocks[:, :1], n // ln, axis=1)), f
        if start in first:
            assert np.array_equal(z[f], z[first[start]]), f
        else:
            first[start] = f
    assert len(first) == r + 1                                    # 3 single points + segments of 2 .. N/4


def test_batches_bit_identical_to_legacy(product_lib, cuda_device):
    """host batches of 2^12 full-band clips run one clip per staging chunk (67 MB each); device batches run at once"""
    import torch
    n = 1 << 12
    x = np.stack([SO.case_signal(s, n) * (1 + 5 * (s == 1)) for s in range(3)])
    st = af.ST(radix2_exp=12, min_index=1, max_index=2047)
    st.use_bin_arr(np.arange(0, 2049))
    fs = af.FST(radix2_exp=12, min_index=1, max_index=2047)
    legacy_st = [SO.c_st(product_lib, st._obj, x[b], st.num) for b in range(3)]
    legacy_fst = [SO.c_fst(product_lib, fs._obj, x[b], 1, 2047) for b in range(3)]
    for fn, legacy in ((st.st_batch, legacy_st), (fs.fst_batch, legacy_fst)):
        for nb in (1, 3):
            host = fn(x[:nb])
            dev = fn(torch.from_numpy(x[:nb]).cuda())
            torch.cuda.synchronize()
            for b in range(nb):
                for k in range(2):
                    assert np.array_equal(host[k][b], legacy[b][k]), (fn, nb, b, k)
                    assert np.array_equal(dev[k][b].cpu().numpy(), legacy[b][k]), (fn, nb, b, k, "device")
    # many small clips in one chunk, and a [2, 3, N] lead shape
    small = np.stack([SO.case_signal(s, 256) for s in range(6)]).reshape(2, 3, 256)
    t = af.ST(radix2_exp=8, min_index=1, max_index=100, factor=0.7)
    re, im = t.st_batch(small)
    assert re.shape == (2, 3, 100, 256)
    for b in range(6):
        lr, li = SO.c_st(product_lib, t._obj, small.reshape(6, 256)[b], 100)
        assert np.array_equal(re.reshape(6, 100, 256)[b], lr) and np.array_equal(im.reshape(6, 100, 256)[b], li)


def test_launch_count_independent_of_rows(product_lib, cuda_device):
    """ST: the forward FFT and k_st_rows; FST: the forward FFT, k_fst_segments and k_fst_expand"""
    import torch
    for r in (8, 12, 14):
        xd = torch.zeros((3, 1 << r), device="cuda")
        hi = (1 << (r - 1)) - 1
        for rows in ((1, 2), (1, hi), (hi - 3, hi)):
            st = af.ST(radix2_exp=r, min_index=rows[0], max_index=rows[1])
            fst = af.FST(radix2_exp=r, min_index=rows[0], max_index=rows[1])
            assert count_launches(product_lib, lambda: st.st_batch(xd), warm=True) == 2
            assert count_launches(product_lib, lambda: fst.fst_batch(xd), warm=True) == 3


def test_set_value_and_bin_list_follow_the_object(product_lib, cuda_device):
    x = SO.case_signal(5, 1024)
    t = af.ST(radix2_exp=10, min_index=1, max_index=200)
    t.st(x)
    t.set_value(2.5, 0.7)
    t.use_bin_arr([300, 0, 7, 7, 512])
    got = t.st(x)
    want = SO.st(x, [300, 0, 7, 7, 512], 2.5, 0.7)
    _check_rows(got.real.astype(np.float32), got.imag.astype(np.float32), want, "set_value + use_bin_arr")


def test_reference_classes_on_b200(raf, cuda_device):
    rng = np.random.default_rng(5)
    mono = SO.case_signal(11, 1 << 11)
    multi = (0.1 * rng.standard_normal((2, 3, 1 << 11))).astype(np.float32)
    res = {}
    for which in ("ref", "b200"):
        raf.fftlib.set_fft_lib(lib_ext="b200" if which == "b200" else None)
        s = raf.ST(radix2_exp=11, min_index=1, max_index=600, factor=1.3, norm=0.9)
        out = [s.st(mono), s.st(multi)]
        s.set_value(0.8, 1.1)
        out.append(s.st(mono))
        s.use_bin_arr(np.array([3, 9, 27], np.float32))    # float bits through an int *: ignored by both libraries
        out.append(s.st(mono))
        f = raf.FST(radix2_exp=11, min_index=5, max_index=900)
        out += [f.fst(mono), f.fst(multi)]
        out += [s.get_fre_band_arr(), s.x_coords(), s.y_coords(), f.get_fre_band_arr(), f.y_coords()]
        res[which] = out
    raf.fftlib.set_fft_lib(None)
    g, r = res["b200"], res["ref"]
    for k in range(6):
        assert g[k].shape == r[k].shape, k
        want = r[k].reshape(-1, r[k].shape[-1])
        got = g[k].reshape(-1, g[k].shape[-1])
        _check_rows(got.real.astype(np.float32), got.imag.astype(np.float32), want.astype(np.complex128), k)
    for k in range(6, 11):
        assert np.array_equal(g[k], r[k]), k
