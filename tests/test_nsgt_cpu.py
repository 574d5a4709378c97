"""NSGT without a GPU: the numpy oracle against the reference build (or its stored outputs in tests/golden/nsgt.npz),
the column map on the reference's own outputs, and nsgtObj_new of libaudioflux_b200.so (status codes, getters, lengths,
its -2 refusals) against the reference over the same sweep."""
import numpy as np
import pytest

import _nsgt_oracle as NO
from _parity_kit import GoldenStore, ref_lib_or_none

from oracle import af_oracle as O

KINDS = ("lens", "bins", "fre", "offs", "win", "cells", "matrix")
# the golden file keeps every case's tables, but windows, cells and matrices only of the 2^8 cases (all styles, both
# banks) and the cells of the docs example; where the reference build exists everything is compared
GOLDEN_BULKY = ("win", "cells", "matrix")


def _signal(kw):
    return NO.case_signal(7, 1 << kw["radix2_exp"], kw["samplate"])


def _live(keys):
    """{"<case>/<kind>": array}: tables, windows, cells and matrices"""
    lib = ref_lib_or_none()
    res = {}
    for name, kw in NO.cases():
        if not any(f"{name}/{kind}" in keys for kind in KINDS):
            continue
        st, obj = NO.c_new(lib, **kw)
        assert st == 0, name
        _, p = NO.params(**kw)
        t = NO.c_tables(lib, obj, kw["num"])
        fb = NO.c_filterbank(lib, p)
        re, im, cr, ci = NO.c_nsgt(lib, obj, _signal(kw), kw["num"])
        lib.nsgtObj_free(obj)
        case = dict(lens=t["lens"].astype(np.int32), bins=t["bins"].astype(np.int32), fre=t["fre"],
                    offs=fb["offs"].astype(np.int32), win=fb["win"][:fb["total_len"]], cells=np.stack([cr, ci]),
                    matrix=np.stack([re, im]))
        res.update((f"{name}/{kind}", case[kind]) for kind in KINDS if f"{name}/{kind}" in keys)
    return res


def _golden_keys():
    """what tests/golden/nsgt.npz keeps"""
    return {f"{name}/{kind}" for name, kw in NO.cases() for kind in KINDS
            if kind not in GOLDEN_BULKY or kw["radix2_exp"] == 8 or (name, kind) == ("docs84", "cells")}


GOLD = GoldenStore("nsgt.npz", _live, _golden_keys)


@pytest.fixture(scope="module")
def ref_out():
    return GOLD.outputs({f"{name}/{kind}" for name, _ in NO.cases() for kind in KINDS})


@pytest.mark.parametrize("name,kw", NO.cases(), ids=[c[0] for c in NO.cases()])
def test_oracle_matches_reference(ref_out, name, kw):
    st, p = NO.params(**kw)
    assert st == 0
    b = NO.bank(p)
    assert np.array_equal(b["lens"], ref_out[f"{name}/lens"])
    assert np.array_equal(b["bins"], ref_out[f"{name}/bins"])
    assert np.array_equal(b["offs"], ref_out[f"{name}/offs"])
    assert np.abs(b["fre"] - ref_out[f"{name}/fre"]).max() <= 1e-6 * np.abs(ref_out[f"{name}/fre"]).max()
    if f"{name}/win" in ref_out:
        assert np.abs(np.concatenate(b["windows"]) - ref_out[f"{name}/win"]).max() <= 1e-6
    cells, m = NO.transform(_signal(kw), p, b)
    c = np.concatenate(cells)
    if f"{name}/cells" in ref_out:
        want = ref_out[f"{name}/cells"]
        scale = np.abs(want).max()
        assert np.abs(c.real - want[0]).max() <= 1e-5 * scale and np.abs(c.imag - want[1]).max() <= 1e-5 * scale
    if f"{name}/matrix" in ref_out:
        scale = np.abs(ref_out[f"{name}/matrix"]).max()
        w = ref_out[f"{name}/matrix"]
        assert np.abs(m.real - w[0]).max() <= 1e-5 * scale and np.abs(m.imag - w[1]).max() <= 1e-5 * scale


def test_transform_spectrum_is_the_band_step_of_transform():
    """the band step alone, from the float64 FFT of the clip, is the whole transform bit for bit; the mirrored half
    spectrum is the full one"""
    for name, kw in NO.cases():
        _, p = NO.params(**kw)
        x = _signal(kw)
        X = np.fft.fft(x.astype(np.float64))
        cells, m = NO.transform(x, p)
        cells2, m2 = NO.transform_spectrum(X, p)
        assert all(np.array_equal(a, b) for a, b in zip(cells, cells2)) and np.array_equal(m, m2), name
        h = np.fft.rfft(x.astype(np.float64))
        assert np.abs(NO.full_spectrum(h.real, h.imag) - X).max() <= 1e-12 * np.abs(X).max(), name


def test_check_bands_holds_each_band_to_its_own_scale():
    rng = np.random.default_rng(0)
    lens = [1, 3, 4097, 2]
    want = [rng.standard_normal(n) + 1j * rng.standard_normal(n) for n in lens]
    want[1] *= 1e-6                                           # a quiet band
    want[3][:] = 0                                            # an all-zero band
    worst = NO.check_bands([w.copy() for w in want], want, lens)
    assert set(worst) == {"bluestein M=2^0", "bluestein M=2^3", "direct 1 pass", "bluestein M=2^2"}
    got = [w.copy() for w in want]
    got[1][0] += 2e-4 * np.abs(want[1]).max()                 # far below the tensor's scale, 2e-4 of the band's own
    with pytest.raises(AssertionError, match="band 1 L=3 log2M=3"):
        NO.check_bands(got, want, lens)
    got = [w.copy() for w in want]
    got[3][1] = 1e-30
    with pytest.raises(AssertionError, match="band 3 L=2 log2M=2 bluestein M=2\\^2: want exactly 0"):
        NO.check_bands(got, want, lens)


@pytest.mark.parametrize("name,kw", NO.cases(), ids=[c[0] for c in NO.cases()])
def test_column_map_on_reference_outputs(ref_lib, name, kw):
    """the reference's matrix is its cells gathered with the oracle's column map, bit for bit"""
    _, p = NO.params(**kw)
    st, obj = NO.c_new(ref_lib, **kw)
    re, im, cr, ci = NO.c_nsgt(ref_lib, obj, _signal(kw), kw["num"])
    ref_lib.nsgtObj_free(obj)
    lens = NO.bank(p)["lens"]
    cmap = NO.column_map(lens, p["fft_length"], p["samplate"])
    off = np.concatenate([[0], np.cumsum(lens)[:-1]])
    idx = off[:, None] + np.maximum(cmap, 0)
    assert (cmap >= 0).all()
    assert np.array_equal(re, cr[idx]) and np.array_equal(im, ci[idx])


def test_golden_file_matches_reference_build():
    GOLD.check_file()


def _sweep():
    """the case set, the out-of-range parameters of nsgtObj_new, and NULL arguments"""
    for _, kw in NO.cases():
        yield kw
    base = dict(num=84, radix2_exp=12)
    for extra in (dict(radix2_exp=0), dict(radix2_exp=-1), dict(radix2_exp=31), dict(radix2_exp=1, num=2),
                  dict(num=1), dict(num=2049), dict(num=2050, radix2_exp=12, scale_type=O.SCALE_MEL),
                  dict(scale_type=7), dict(scale_type=10), dict(samplate=0), dict(samplate=200000),
                  dict(samplate=8000), dict(low_fre=-5.0), dict(low_fre=20000.0), dict(high_fre=100.0),
                  dict(high_fre=20.0, low_fre=40.0), dict(num=120, scale_type=O.SCALE_OCTAVE),
                  dict(num=400, scale_type=O.SCALE_LINEAR, low_fre=15000.0), dict(bin_per_octave=3),
                  dict(bin_per_octave=49), dict(bin_per_octave=24, num=168), dict(min_len=0), dict(min_len=-3),
                  dict(style_type=O.STYLE_GAMMATONE), dict(style_type=O.STYLE_POINT), dict(normal_type=O.NORM_AREA),
                  dict(bank_type=5), dict(scale_type=O.SCALE_LOG, samplate=4000), dict(scale_type=O.SCALE_LINSPACE),
                  dict(scale_type=O.SCALE_BARK, num=24), dict(scale_type=O.SCALE_ERB, num=40)):
        yield dict(base, **extra)
    yield dict(num=84, radix2_exp=12, samplate=None, low_fre=None, high_fre=None, bin_per_octave=None, min_len=None,
               bank_type=None, scale_type=None, style_type=None, normal_type=None)


def test_constructor_matches_reference(product_lib, ref_lib):
    bad = []
    for kw in _sweep():
        sp, po = NO.c_new(product_lib, **kw)
        sr, ro = NO.c_new(ref_lib, **kw)
        so, _ = NO.params(**kw)
        if not (sp == sr == so):
            bad.append(f"{kw}: status product {sp} reference {sr} oracle {so}")
            continue
        if sp != 0:
            continue
        tp, tr = NO.c_tables(product_lib, po, kw["num"]), NO.c_tables(ref_lib, ro, kw["num"])
        for k in ("max_len", "total_len", "lens", "bins", "fre"):
            if not np.array_equal(tp[k], tr[k]):
                bad.append(f"{kw}: {k}")
        product_lib.nsgtObj_free(po)
        ref_lib.nsgtObj_free(ro)
    assert not bad, "\n".join(bad[:20])


def test_constructor_without_reference(product_lib):
    """status codes and tables of the product against the oracle (runs where no reference build exists)"""
    bad = []
    for kw in _sweep():
        sp, po = NO.c_new(product_lib, **kw)
        so, p = NO.params(**kw)
        if sp != so:
            bad.append(f"{kw}: status {sp} oracle {so}")
            continue
        if sp:
            continue
        b = NO.bank(p)
        t = NO.c_tables(product_lib, po, kw["num"])
        if not (np.array_equal(t["lens"], b["lens"]) and np.array_equal(t["bins"], b["bins"]) and
                t["max_len"] == b["max_len"] and t["total_len"] == b["total_len"]):
            bad.append(f"{kw}: tables")
        product_lib.nsgtObj_free(po)
    assert not bad, "\n".join(bad[:20])


def test_refusals(product_lib):
    for kw in (dict(num=84, radix2_exp=21), dict(num=84, radix2_exp=30),
               dict(num=4, radix2_exp=16, scale_type=O.SCALE_LINEAR, min_len=16385)):
        st, obj = NO.c_new(product_lib, **kw)
        assert st == -2 and not obj.value, kw
        assert product_lib.afb200_lastError()
    st, obj = NO.c_new(product_lib, num=4, radix2_exp=16, scale_type=O.SCALE_LINEAR, min_len=16384)
    assert st == 0 and product_lib.nsgtObj_getMaxTimeLength(obj) == 16384
    # a minimum length beyond the limit leaves the object as it was
    product_lib.nsgtObj_setMinLength(obj, 20000)
    assert product_lib.nsgtObj_getMaxTimeLength(obj) == 16384
    product_lib.nsgtObj_free(obj)


def test_set_min_length_rebuilds_tables(product_lib):
    for start, to in ((20, 3), (3, 20), (1, 300)):
        st, a = NO.c_new(product_lib, num=84, radix2_exp=12, min_len=start)
        st2, b = NO.c_new(product_lib, num=84, radix2_exp=12, min_len=to)
        product_lib.nsgtObj_setMinLength(a, to)
        ta, tb = NO.c_tables(product_lib, a, 84), NO.c_tables(product_lib, b, 84)
        for k in ("max_len", "total_len", "lens", "bins", "fre"):
            assert np.array_equal(ta[k], tb[k]), (start, to, k)
        product_lib.nsgtObj_free(a)
        product_lib.nsgtObj_free(b)


def test_python_class_checks(product_lib):
    import audioflux_b200 as af
    with pytest.raises(ValueError):
        af.NSGT(num=3000, radix2_exp=12)
    with pytest.raises(ValueError):
        af.NSGT(style_type=af.SpectralFilterBankStyleType.GAMMATONE)
    with pytest.raises(ValueError):
        af.NSGT(normal_type=af.SpectralFilterBankNormalType.AREA)
    with pytest.raises(ValueError):
        af.NSGT(low_fre=20.0)
    with pytest.raises(ValueError, match="status -2"):
        af.NSGT(radix2_exp=21)
    t = af.NSGT(num=84, radix2_exp=12)
    assert t.get_max_time_length() == max(t.get_time_length_arr())
    assert t.y_coords().shape == (85,) and t.x_coords(4096).shape == (t.get_max_time_length() + 1,)
    with pytest.raises(ValueError):
        t.set_min_length(0)
    assert af.NSGTFilterBankType.STANDARD.value == 1
