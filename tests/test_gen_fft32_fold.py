"""The fused MFCC frame path with the window and the column twiddles folded into the transforms (af_fft32_fma_win /
af_fft32_fma_tw in kernels/fft32_gen.cuh): op lists checked with numpy in float64 and in float32 with one rounding per
op, alone and composed into the whole 2048-point real DFT the frame warps and the producer warp compute."""
import importlib.util
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.realpath(__file__)))
GEN = os.path.join(ROOT, "audioflux_b200", "csrc", "gen", "gen_fft32.py")
HEADER = os.path.join(ROOT, "audioflux_b200", "csrc", "kernels", "fft32_gen.cuh")
EPS = 2.0 ** -24
WIN_BUDGET = 404        # af_fft32_fma (372) + one FMUL per first butterfly and component, instead of 64 window products
TW_BUDGET = 464         # af_fft32_fma + 2 FMAs per twiddled input + 30 FMULs, instead of 31 complex products (124)


def _mod():
    spec = importlib.util.spec_from_file_location("gen_fft32", GEN)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _f32(a):
    return np.asarray(a).astype(np.float32).astype(np.float64)


def _hann(n):
    return 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(n) / n)


def test_windowed_stage_b_is_the_real_dft_of_the_windowed_column():
    """packed z[m] = (s[2m], s[2m+1]), window pairs 0.5 (w[2m], w[2m+1]) -> R[0..32] of rfft(w s)"""
    m = _mod()
    rng = np.random.default_rng(11)
    for trial in range(40):
        s = _f32(rng.standard_normal(64))
        w = _f32(_hann(64) if trial % 2 else rng.uniform(0.0, 1.0, 64))
        R = np.fft.rfft(w * s)
        for dtype, tol in ((np.float64, 1e-12 * np.abs(R).max()), (np.float32, 4 * EPS * np.abs(R).max())):
            Z = m.run_numpy_fma_win(s[0::2] + 1j * s[1::2], 0.5 * (w[0::2] + 1j * w[1::2]), dtype)
            ops, outs = m.build_fma_post64()
            Rk = m.run_ops(ops, outs, Z, dtype)
            got = np.concatenate([[Rk[0].real], Rk[1:32], [Rk[0].imag]])
            assert np.abs(got - R).max() < tol, (trial, dtype)


def _tw_table(m):
    """(g, t)[n2][k1] as the kernel's plan rounds them to float32"""
    g, t = np.ones((32, 32)), np.zeros((32, 32))
    for n2 in range(1, 32):
        for k1 in range(32):
            g[n2, k1], t[n2, k1] = m.twiddle_gt(n2 * k1)
    return _f32(g), _f32(t)


def test_twiddled_stage_d_is_a_dft_of_the_twiddled_column():
    m = _mod()
    rng = np.random.default_rng(12)
    g, t = _tw_table(m)
    for k1 in (1, 9, 17, 19, 27, 30, 31):              # 17 * 30 and 19 * 27 sit next to cos = 0 (|t| up to 326)
        x = _f32(rng.standard_normal(32)) + 1j * _f32(rng.standard_normal(32))
        W = np.exp(-2j * np.pi * np.arange(32) * k1 / 2048)
        X = np.fft.fft(x * W)
        assert np.abs(m.run_numpy_fma_tw(x, g[:, k1], t[:, k1]) - X).max() < 1e-6 * np.abs(X).max()   # table in float32
        exact_g = np.array([1.0] + [m.twiddle_gt(n2 * k1)[0] for n2 in range(1, 32)])
        exact_t = np.array([0.0] + [m.twiddle_gt(n2 * k1)[1] for n2 in range(1, 32)])
        assert np.abs(m.run_numpy_fma_tw(x, exact_g, exact_t) - X).max() < 1e-12 * np.abs(X).max()
        assert np.abs(m.run_numpy_fma_tw(x, g[:, k1], t[:, k1], np.float32) - X).max() < 8 * EPS * np.abs(X).max()


def _frame_dft(m, s, w, dtype):
    """The frame path of k_mfcc_fused2 on numpy: bins 0..1024 of the 2048-point DFT of w s."""
    g, t = _tw_table(m)
    post_ops, post_outs = m.build_fma_post64()
    R = np.zeros((32, 33), complex)                    # [n2][k1]: stage B of lane n2
    for n2 in range(32):
        col, wc = s[n2::32], 0.5 * w[n2::32]
        Z = m.run_numpy_fma_win(col[0::2] + 1j * col[1::2], wc[0::2] + 1j * wc[1::2], dtype)
        Rk = m.run_ops(post_ops, post_outs, Z, dtype)
        R[n2, 0], R[n2, 32], R[n2, 1:32] = Rk[0].real, Rk[0].imag, Rk[1:32]
    X = np.zeros(2048, complex)
    for k1 in range(1, 32):                            # frame warps, lane k1: stage D over n2
        X[k1::64] = m.run_numpy_fma_tw(R[:, k1], g[:, k1], t[:, k1], dtype)
    X[0::64] = m.run_numpy_fma(R[:, 0], dtype)         # producer warp, kind 0
    b = np.array([R[n2, 32] * np.exp(-2j * np.pi * n2 / 64) for n2 in range(32)])
    b = (np.array([complex(np.float32(v.real), np.float32(v.imag)) for v in b]) if dtype == np.float32 else b)
    X[32::64] = m.run_numpy_fma(b, dtype)              # producer warp, kind 1
    k = np.arange(1025)
    upper = k % 64 > 32                                # bins 64 (k2 + 1) - k1: mirrored from 2048 - k
    X[k[upper]] = np.conj(X[2048 - k[upper]])
    return X[:1025]


def test_folded_frame_path_is_the_2048_point_real_dft():
    m = _mod()
    rng = np.random.default_rng(13)
    w = _f32(_hann(2048))
    for _ in range(2):
        s = _f32(rng.standard_normal(2048))
        X = np.fft.rfft(w * s)
        assert np.abs(_frame_dft(m, s, w, np.float64) - X).max() < 1e-6 * np.abs(X).max()     # tables in float32
        err32 = np.abs(_frame_dft(m, s, w, np.float32) - X).max() / (EPS * np.abs(X).max())
        assert err32 < 8, err32


def test_fold_op_counts_within_budget():
    m = _mod()
    n_win, n_tw = m.fp32_op_count(m.build_fma_fft32_win()[0]), m.fp32_op_count(m.build_fma_fft32_tw()[0])
    assert n_win <= WIN_BUDGET and n_tw <= TW_BUDGET
    text = open(HEADER).read()
    assert f"af_fft32_fma_win FP32 instruction count: {n_win}" in text
    assert f"af_fft32_fma_tw FP32 instruction count: {n_tw}" in text
