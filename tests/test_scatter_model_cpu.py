"""The cell-by-cell model of reassignment and synchrosqueezing (tests/_scatter_model.py) on the CPU.

* On the reference build's own float32 planes, with glibc's log2f, the model reproduces the reference's reassigned and
  WSST planes bit for bit: the model's index and scatter are the reference's.
* On the oracle's float32 planes, the model's candidate sets contain the index a glibc evaluation gives, and the column
  verifier accepts the matching scatter but rejects one with a cell moved by one row or a value off by one ulp.
* The crafted threshold pairs that tests/test_gpu_scatter_cells.py feeds to the GPU really split the op-by-op and the
  FMA-contracted |W|^2 test (exact rational arithmetic).
* kernels/squeeze.cu's scatter, compiled as the Makefile compiles it, contains no FFMA, and its synsq index no DFMA."""
import os
import re
import shutil
import subprocess
import tempfile
from fractions import Fraction

import numpy as np
import pytest

import _scatter_model as M
from oracle import af_oracle as O
from test_gpu_squeeze import _signal as _sq_signal
from test_reassign_cpu import CASES, _signal

f32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.realpath(__file__)))


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a, f32).view(np.uint32), np.asarray(b, f32).view(np.uint32))


# ------------------------------------------------------------------------------------------ reference build, bitwise
@pytest.mark.parametrize("radix,sr,window,hop,re_type,thresh,pad,order,result_type", CASES)
def test_model_reproduces_reference_reassign(ref_lib, radix, sr, window, hop, re_type, thresh, pad, order, result_type):
    import audioflux_b200 as af
    x = _signal(20000, sr, radix)
    r = af.Reassign(radix, sr, af.WindowType(window), hop, af.ReassignType(re_type), thresh, bool(pad), _lib=ref_lib)
    r.set_order(order)
    want = r.reassign_planes(x, result_type)
    n, W = 1 << radix, (1 << radix) // 2 + 1
    # the reference's own window (its float32 values differ from the float64 oracle's in the last bit)
    h = af.STFT(radix, af.WindowType(window), hop, _lib=ref_lib).get_window_data_arr()
    planes = []
    for win in O.reassign_windows(h):
        s = af.STFT(radix, af.WindowType(window), hop, _lib=ref_lib)
        s.enable_padding(bool(pad))
        s.use_window_data_arr(win)
        a, b = s.stft_planes(x)
        planes.append((np.ascontiguousarray(a[:, :W]), np.ascontiguousarray(b[:, :W])))
    assert _bits_equal(planes[0][0], want[2]) and _bits_equal(planes[0][1], want[3])
    ti, fi = M.reassign_index(*planes, n, sr, hop, re_type, thresh, order)
    got = M.reassign_float_sum(planes[0], ti, fi, result_type)
    for k in ((0,) if result_type else (0, 1)):
        assert _bits_equal(got[k], want[k]), (k, int((got[k] != want[k]).sum()))


WSST_CASES = [(12, False, O.SCALE_OCTAVE, O.WAVE_MORLET), (12, True, O.SCALE_LOG, O.WAVE_MORSE),
              (12, False, O.SCALE_LINEAR, O.WAVE_MORLET), (12, False, O.SCALE_MEL, O.WAVE_BUMP),
              (11, False, O.SCALE_LINSPACE, O.WAVE_PAUL), (11, True, O.SCALE_BARK, O.WAVE_MORLET),
              (11, False, O.SCALE_ERB, O.WAVE_MORSE)]


@pytest.mark.parametrize("radix,is_pad,scale,wavelet", WSST_CASES)
def test_model_reproduces_reference_wsst(ref_lib, radix, is_pad, scale, wavelet):
    import audioflux_b200 as af
    sr, num = 32000, 84
    x = _sq_signal(1 << radix, sr, radix)
    kw = dict(wavelet_type=af.WaveletContinueType(wavelet), scale_type=af.SpectralFilterBankScaleType(scale),
              is_padding=is_pad, _lib=ref_lib)
    want = af.WSST(num, radix, sr, **kw).wsst_planes(x)
    c = af.CWT(num, radix, sr, **kw)
    c.enable_det(True)
    w = c.cwt_planes(x)
    dw = c.cwt_det_planes(None)
    assert _bits_equal(w[0], want[2]) and _bits_equal(w[1], want[3])
    index = M.wsst_index(w, dw, c.get_fre_band_arr(), sr, scale, libm=True)
    assert not index.cands
    got = M.scatter(w, index.idx, 0.001)
    assert _bits_equal(got[0], want[0]) and _bits_equal(got[1], want[1])
    assert np.abs(got[0]).max() > 0


# ------------------------------------------------------------------------------------------ oracle planes, candidates
def _oracle_cwt(radix, scale, wavelet=O.WAVE_MORLET, seed=7):
    sr, num = 32000, 84
    x = _sq_signal(1 << radix, sr, seed)
    w = O.cwt(x, num, radix, sr, wavelet, scale, is_pad=False)
    dw = O.cwt(x, num, radix, sr, wavelet, scale, is_pad=False, det=True)
    _, fre = O.cwt_filterbank(num, 1 << radix, sr, wavelet, scale, None, None, 12, None, None, 0)
    return [np.asarray(v, f32) for v in w], [np.asarray(v, f32) for v in dw], np.asarray(fre, f32)


def _determined(index):
    det = np.ones(index.idx.shape, bool)
    for k in index.cands:
        det[k] = False
    return det


# undetermined-column caps: measured on these planes with margin (DESIGN.md section 7)
WSST_LOG_CAP, SYNSQ_CAP = 0.01, 0.15


@pytest.mark.parametrize("scale", [O.SCALE_OCTAVE, O.SCALE_LOG, O.SCALE_LINEAR, O.SCALE_MEL])
def test_wsst_candidates_contain_the_glibc_index(scale):
    w, dw, fre = _oracle_cwt(12, scale)
    gpu = M.wsst_index(w, dw, fre, 32000, scale)
    ref = M.wsst_index(w, dw, fre, 32000, scale, libm=True)
    det = _determined(gpu)
    assert np.array_equal(gpu.idx[det], ref.idx[det])
    assert all(int(ref.idx[k]) in c for k, c in gpu.cands.items())
    out = M.scatter(w, ref.idx, 0.001)
    v = M.verify_columns(out, w, gpu, 0.001)
    assert not v["failures"], v
    assert v["undetermined_columns"] <= (WSST_LOG_CAP if scale in (O.SCALE_OCTAVE, O.SCALE_LOG) else 0.0), v
    print(f"wsst scale {scale}: {v['undetermined_cells']} undetermined cells, {v['undetermined_columns']:.4%} of columns")


@pytest.mark.parametrize("radix", [10, 12, 13])
@pytest.mark.parametrize("scale", [O.SCALE_OCTAVE, O.SCALE_LINEAR, O.SCALE_BARK])
def test_synsq_candidates_contain_the_glibc_index(radix, scale):
    w, _, fre = _oracle_cwt(radix, scale)
    gpu = M.synsq_index(*w, fre, 32000, scale)
    ref = M.synsq_index(*w, fre, 32000, scale, libm=True)
    det = _determined(gpu)
    assert np.array_equal(gpu.idx[det], ref.idx[det])
    assert all(c is None or int(ref.idx[k]) in c for k, c in gpu.cands.items())
    out = M.scatter(w, ref.idx, 0.001)
    v = M.verify_columns(out, w, gpu, 0.001)
    assert not v["failures"], v
    assert v["undetermined_columns"] <= SYNSQ_CAP, v
    print(f"synsq 2^{radix} scale {scale}: {v['undetermined_cells']} undetermined cells, "
          f"{v['undetermined_columns']:.4%} of columns")


def test_synsq_libm_index_matches_the_oracle_on_plain_rows():
    """the kernel's unwrap (a running count of +-2 pi jumps) and the reference's sequential unwrap agree on the
    oracle's planes wherever the oracle's own float32 steps are used"""
    w, _, fre = _oracle_cwt(12, O.SCALE_BARK)
    ref = M.synsq_index(*w, fre, 32000, O.SCALE_BARK, libm=True)
    want = O.synsq(fre, *w, 32000, O.SCALE_BARK)
    got = M.scatter(w, ref.idx, 0.001)
    same = (got[0] == want[0]).all(axis=0).mean()
    assert same >= 0.99, same


def test_verifier_rejects_a_moved_cell_and_a_one_ulp_error():
    w, dw, fre = _oracle_cwt(12, O.SCALE_OCTAVE)
    index = M.wsst_index(w, dw, fre, 32000, O.SCALE_OCTAVE)
    ref = M.wsst_index(w, dw, fre, 32000, O.SCALE_OCTAVE, libm=True)
    out = M.scatter(w, ref.idx, 0.001)
    assert not M.verify_columns(out, w, index, 0.001)["failures"]
    free = [j for j in range(out[0].shape[1]) if j not in set(index.columns())]
    j = next(j for j in free if np.count_nonzero(out[0][1:-1, j]))
    r = int(np.nonzero(out[0][1:-1, j])[0][0]) + 1
    moved = [p.copy() for p in out]
    for p in moved:
        p[r + 1, j], p[r, j] = p[r + 1, j] + p[r, j], 0
    assert M.verify_columns(moved, w, index, 0.001)["failures"] == [j]
    ulp = [p.copy() for p in out]
    ulp[1][r, j] = np.nextafter(ulp[1][r, j], f32(np.inf))
    assert M.verify_columns(ulp, w, index, 0.001)["failures"] == [j]


def test_reassign_fixed_point_model_is_exact_for_a_single_term():
    """one term per cell: the fixed-point round trip gives the float back exactly (36 bits below the clip maximum)"""
    rng = np.random.default_rng(1)
    re, im = (rng.standard_normal((6, 9)).astype(f32) for _ in range(2))
    ti, fi = np.repeat(np.arange(6)[:, None], 9, 1), np.repeat(np.arange(9)[None, :], 6, 0)
    out = M.reassign_fixed_point((re, im), ti, fi)
    sign = np.where(np.arange(9) % 2 == 1, f32(-1), f32(1))
    assert _bits_equal(out[0], re * sign) and _bits_equal(out[1], im * sign)


# ------------------------------------------------------------------------------------------ crafted threshold pairs
def _round_f32(q):
    """round a rational to the nearest float32 (ties to even), exactly"""
    c = f32(float(q))
    best = None
    for v in (np.nextafter(c, f32(-np.inf)), c, np.nextafter(c, f32(np.inf))):
        d = abs(Fraction(float(v)) - q)
        key = (d, int(np.asarray(v, f32).view(np.uint32)) & 1)
        if best is None or key < best[0]:
            best = (key, v)
    return Fraction(float(best[1]))


def test_crafted_threshold_pairs_split_op_by_op_and_fma():
    v1, v2, kept = M.crafted_threshold_pairs()
    t2 = _round_f32(Fraction(float(f32(0.001))) ** 2)
    for a, b, k in zip(v1, v2, kept):
        a2, b2 = Fraction(float(a)) ** 2, Fraction(float(b)) ** 2
        op = _round_f32(_round_f32(a2) + _round_f32(b2)) > t2
        fma_a = _round_f32(b2 + _round_f32(a2)) > t2
        fma_b = _round_f32(a2 + _round_f32(b2)) > t2
        assert op == k and fma_a != k and fma_b != k, (a, b)


# ------------------------------------------------------------------------------------------ SASS of the scatter
def _nvcc():
    for p in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if p and os.path.exists(p):
            return p
    return None


def _sass_by_kernel(src):
    nvcc = _nvcc()
    with tempfile.TemporaryDirectory() as tmp:
        cubin = os.path.join(tmp, "squeeze.cubin")
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-cubin", src, "-o", cubin],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        dump = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), "-sass", cubin], capture_output=True, text=True)
    assert dump.returncode == 0, dump.stderr
    out, name = {}, None
    for line in dump.stdout.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            out[name] = []
        elif name:
            out[name].append(line)
    return out


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not found")
def test_squeeze_scatter_and_synsq_unwrap_are_not_contracted():
    sass = _sass_by_kernel(os.path.join(ROOT, "audioflux_b200", "csrc", "kernels", "squeeze.cu"))
    scatter = [v for k, v in sass.items() if "k_squeeze_scatter" in k]
    synsq = [v for k, v in sass.items() if "k_synsq_index" in k]
    assert len(scatter) == 1 and len(synsq) == 1, list(sass)
    assert not [l for l in scatter[0] if re.search(r"\bFFMA\b", l)]
    assert any(re.search(r"\bFMUL\b", l) for l in scatter[0])
    assert not [l for l in synsq[0] if re.search(r"\bDFMA\b", l)]
