"""NMF throughput on the device (device-resident matrices, CUDA-event timing, median of the timed calls after warm-up):

  kl8    1024 x (513 x 431) |noise|^2 spectrograms, k = 8, KL, 300 iterations (thresh 1e-3: a noise spectrogram does
         not converge that far, so every matrix runs them all)
  euc2   4096 x (257 x 128), k = 2, Euclidean, maxIter 300, thresh 1e-3 (matrices stop on their own)

Per workload: ms per call and decompositions per second; the iterations run (mean over matrices); per iteration and
matrix the FLOPs (5 n m k products, each a multiply and an FP64 add) and the compulsory bytes of the four stages (V and
the D2 / D3 planes, W and H aside); the kernels' own times (torch.profiler, a separate run); the share of the FP64 bound
(the FP64 adds at 33.5 TFLOPS / 2 adds per second, the H100 SXM data-sheet FP64 rate) and of 3.35 TB/s; a parity gate on
matrix 0 against the oracle; the card's name, power limit and max SM clock; and where oracle/_ref exists the reference
build's time per decomposition on one CPU core, measured over 3 iterations and scaled to the mean iteration count.
Prints one JSON line per workload.

    python tools/bench_nmf.py [--steps 3] [--warmup 1] [--workloads kl8,euc2] [--out results.json]"""
import ctypes as C
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.realpath(__file__)))
import _bench_kit as K  # noqa: E402

import torch  # noqa: E402

import audioflux_b200 as af  # noqa: E402
import _nmf_oracle as NO  # noqa: E402

FP64_ADDS = 33.5e12 / 2
WORKLOADS = {
    "kl8": dict(batch=1024, n=513, m=431, k=8, tp=0, max_iter=300),
    "euc2": dict(batch=4096, n=257, m=128, k=2, tp=2, max_iter=300),
}
PLANES = {0: 4, 1: 7, 2: 6}     # n x m planes read or written per iteration: KL V, D2 x3; IS V, (D2, D3) x3; Euc V x3, D3 x3


def matrices(w):
    rng = np.random.default_rng(0)
    return (np.abs(rng.standard_normal((w["batch"], w["n"], w["m"]), dtype=np.float32)) ** 2).astype(np.float32)


def reference_ms(w, V, iters):
    from oracle import ref_lib as R
    if not R.available():
        return None
    lib = R.get_ref_lib()
    n, m, k = w["n"], w["m"], w["k"]
    W = np.arange(1, n * k + 1, dtype=np.float32).reshape(n, k)
    H = np.arange(1, k * m + 1, dtype=np.float32).reshape(k, m)
    vp = C.c_void_p
    t0 = time.perf_counter()
    lib.nmf(V.ctypes.data_as(vp), n, m, k, W.ctypes.data_as(vp), H.ctypes.data_as(vp), C.byref(C.c_int(3)),
            C.byref(C.c_int(w["tp"])), C.byref(C.c_float(-1.0)), C.byref(C.c_int(0)))
    return (time.perf_counter() - t0) * 1e3 / 3 * iters


def run(name, steps, warmup):
    w = WORKLOADS[name]
    B, n, m, k = w["batch"], w["n"], w["m"], w["k"]
    V = matrices(w)
    Vd = torch.from_numpy(V).cuda()

    def fn():
        return af.nmf_batch(Vd, k, max_iter=w["max_iter"], tp=w["tp"], return_iters=True)
    times, out = K.event_times(fn, steps, warmup)
    ms = float(np.median(times))
    h, wm, it = (x.cpu().numpy() for x in out)
    del out
    iters = it.astype(np.int64)
    Wo, Ho, io, _ = NO.run(V[0], k, max_iter=w["max_iter"], tp=w["tp"], thresh=1e-3, norm=0)
    err = max(float(np.abs(wm[0] - Wo).max() / np.abs(Wo).max()), float(np.abs(h[0] - Ho).max() / np.abs(Ho).max()))
    ok = err <= 1e-4 and int(iters[0]) == io
    per = K.kernel_times(fn, ("k_nmf_d", "k_nmf_h", "k_nmf_w", "k_nmf_norm"), calls=2)
    total_it = int(iters.sum())
    adds = 5 * n * m * k
    flop_it, bytes_it = 2 * adds, 4 * PLANES[w["tp"]] * n * m
    s = ms * 1e-3
    res = dict(workload=name, batch=B, n=n, m=m, k=k, type=w["tp"], max_iter=w["max_iter"],
               iters_mean=round(float(iters.mean()), 2), iters_min=int(iters.min()), iters_max=int(iters.max()),
               **K.ms_stats(times, 2), decompositions_per_s=round(B / s, 1),
               kernels_ms={kk: round(v, 2) for kk, v in per.items()},
               flop_per_iter=flop_it, bytes_per_iter=bytes_it,
               fp64_bound_share=round(adds * total_it / FP64_ADDS / s, 4),
               hbm_share=round(bytes_it * total_it / K.HBM / s, 4),
               parity_worst_matrix0=err, parity_iters_matrix0=(int(iters[0]), io), parity_ok=bool(ok),
               card=K.card())
    ref = reference_ms(w, V[0], float(iters.mean()))
    res["reference_ms_per_decomposition_1core"] = None if ref is None else round(ref, 1)
    return res


if __name__ == "__main__":
    K.main(run, "kl8,euc2", steps=3, warmup=1)
