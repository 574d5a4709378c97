"""The FMA-oriented split-radix 32-point DFT and real 64-point post-pass of the fused MFCC frame path
(af_fft32_fma / af_rfft64_post_fma in kernels/fft32_gen.cuh): op lists checked with numpy in float64 and in float32
with one rounding per op, and their FP32 instruction counts held to a written budget."""
import importlib.util
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.realpath(__file__)))
GEN = os.path.join(ROOT, "audioflux_b200", "csrc", "gen", "gen_fft32.py")
HEADER = os.path.join(ROOT, "audioflux_b200", "csrc", "kernels", "fft32_gen.cuh")
FFT32_FMA_BUDGET = 372        # FP32 instructions per 32-point transform (radix-2 af_fft32: 456)
POST64_FMA_BUDGET = 156       # FP32 instructions of the real 64-point post-pass


def _mod():
    spec = importlib.util.spec_from_file_location("gen_fft32", GEN)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_fma_op_list_is_a_dft():
    m = _mod()
    rng = np.random.default_rng(6)
    for _ in range(4):
        x = rng.standard_normal(32) + 1j * rng.standard_normal(32)
        assert np.abs(m.run_numpy_fma(x) - np.fft.fft(x)).max() < 1e-12
        s = rng.standard_normal(64)
        assert np.abs(m.run_numpy_rfft64(s / 2) - np.fft.rfft(s)).max() < 1e-12


def test_fma_float32_within_a_few_ulps():
    """one rounding per op in float32: every twiddle ratio is <= 1 in magnitude, so no tangent blows up"""
    m = _mod()
    rng = np.random.default_rng(7)
    eps = 2.0 ** -24
    for _ in range(50):
        x = (rng.standard_normal(32) + 1j * rng.standard_normal(32)).astype(np.complex64).astype(np.complex128)
        X = np.fft.fft(x)
        assert np.abs(m.run_numpy_fma(x, np.float32) - X).max() < 4 * eps * np.abs(X).max()
        s = rng.standard_normal(64).astype(np.float32).astype(np.float64)
        R = np.fft.rfft(s)
        assert np.abs(m.run_numpy_rfft64(s / 2, np.float32) - R).max() < 4 * eps * np.abs(R).max()


def test_fma_op_counts_within_budget():
    m = _mod()
    n_fft, n_post = m.fp32_op_count(m.build_fma_fft32()[0]), m.fp32_op_count(m.build_fma_post64()[0])
    assert n_fft <= FFT32_FMA_BUDGET and n_post <= POST64_FMA_BUDGET
    text = open(HEADER).read()
    assert f"af_fft32_fma FP32 instruction count: {n_fft}" in text
    assert f"af_rfft64_post_fma FP32 instruction count: {n_post}" in text

