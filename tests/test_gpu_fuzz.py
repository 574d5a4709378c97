"""Differential compute fuzz on the GPU: random configurations of BFT (+ complex mode, + xxcc), Spectrogram, STFT (all
padding modes), CQT / VQT, CWT (+ derivative transform), PWT, the fused MFCC / mel kernels' configuration space (fftLength
2048: bank families, odd hops and clip lengths, small batches through the batched entry points), ISTFT, xxccStandard, the
CQT post-processing calls (chroma, cqcc, cqhc, deconv) and streaming (STFT / Spectrogram / CQT chunk sequences) through the C ABI against the reference build run on the
CPU by tests/_fuzz_ref_worker.py (a separate process that never touches CUDA, each case fork-isolated).  Bar: 1e-4 of the
reference's maximum per output plane (BASELINE.md), as everywhere else.  Deterministic seeds."""
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from conftest import rel_max
from oracle import ref_lib as R

from _fuzz_cases import compute

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.realpath(__file__))
# the two planes of a complex result are judged on their common scale: the imaginary plane of a symmetric frame is pure
# rounding noise in both libraries
PAIRS = {"re": "im", "im": "re", "zre": "zim", "zim": "zre", "dre": "dim", "dim": "dre"}


def plane_scale(want, k):
    s = float(np.abs(want[k]).max()) if want[k].size else 0.0
    q = PAIRS.get(k)
    if q in want and want[q].size:
        s = max(s, float(np.abs(want[q]).max()))
    return s
TOL = 1e-4


def reference_results(kind, seed, cases):
    if not R.available():
        pytest.skip("oracle/_ref/libaudioflux_ref.so not built (make -C oracle REF=<audioFlux tree>)")
    with tempfile.TemporaryDirectory() as d:
        out = os.path.join(d, "ref.pkl")
        env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
        try:                                                   # the sanitizer build tells defined reference results from heap overruns
            asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True, timeout=30).stdout.strip()
        except Exception:
            asan = ""
        if os.path.isabs(asan) and os.path.exists(asan) and os.path.exists(R.REF_ASAN_PATH):
            env.update(LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=1", AFB200_FUZZ_ASAN="1")
        subprocess.run([sys.executable, os.path.join(HERE, "_fuzz_ref_worker.py"), kind, str(seed), str(cases), out], check=True,
                       env=env, timeout=900)
        with open(out, "rb") as f:
            return pickle.load(f)


def known_deviation(kind, a, got, want):
    """configurations where the two libraries legitimately differ (each documented where it is decided)"""
    if kind in ("cqt", "cqtpost", "stream") and "error" in got and "error" not in want:
        # hop 0 at the lowest octave: refused at _new.  (The reference ignores the non-positive hop -- stft_algorithm.c:171-178 --
        # so those octaves run at the previous hop over a signal half as long and the frames beyond its end are whatever the
        # previous octave left in the STFT buffer, cqt_algorithm.c:992-1010.)
        return "cannot be halved" in __import__("audioflux_b200").lib.last_error()
    if kind in ("cwt", "pwt") and "error" in got and "error" not in want:
        # documented refusals (status -2; tests/test_ctor_fuzz.py): Gammatone pseudo banks, band edges outside [0, Nyquist],
        # bump wavelets with beta > gamma, padded lengths that are not a power of two
        msg = __import__("audioflux_b200").lib.last_error()
        return any(t in msg for t in ("Gammatone", "above the Nyquist bin", "negative frequencies", "power-of-two"))
    return False


@pytest.mark.parametrize("kind,seed,cases", [("bft", 101, 70), ("spec", 102, 50), ("stft", 103, 70), ("cqt", 104, 50), ("cwt", 105, 70),
                                             ("pwt", 106, 60), ("mfcc", 107, 60), ("istft", 108, 50), ("xxccstd", 109, 50),
                                             ("cqtpost", 110, 30), ("stream", 111, 40)])
def test_random_configurations_match_the_reference_build(cuda_device, kind, seed, cases):
    ref = reference_results(kind, seed, cases)
    compared = skipped = 0
    worst = (0.0, None, None)
    fails = []                                              # every failing case is reported, not just the first
    for a, want in ref:
        if want == "crash":
            skipped += 1
            continue
        try:
            got = compute(kind, a)
        except Exception as e:                              # a product-side exception other than a constructor's ValueError
            fails.append(("exception", repr(e)[:200], a))
            continue
        if known_deviation(kind, a, got, want):
            skipped += 1
            continue
        if ("error" in got) != ("error" in want):
            fails.append(("status", got.get("error"), want.get("error"), a))
            continue
        if "error" in want:
            continue
        compared += 1
        if got.keys() != want.keys():
            fails.append(("keys", sorted(got), sorted(want), a))
            continue
        for k in want:
            if got[k].shape != want[k].shape:
                fails.append(("shape", k, got[k].shape, want[k].shape, a))
                continue
            if want[k].size == 0:
                continue
            scale = plane_scale(want, k)
            if scale < 1e-30:
                if not float(np.abs(got[k]).max()) < 1e-20:
                    fails.append(("nonzero", k, a))
                continue
            if not np.isfinite(got[k]).all():
                fails.append(("nonfinite", k, a))
                continue
            err = float(np.abs(got[k].astype(np.float64) - want[k]).max() / scale)
            if err > worst[0]:
                worst = (err, k, a)
            if not err < TOL:
                fails.append(("parity", k, err, a))
    print(f"{kind}: {compared} compared, {skipped} skipped, worst {worst[0]:.2e} ({worst[1]}), {len(fails)} failing")
    dump = os.environ.get("AFB200_FUZZ_DUMP")               # debugging aid: the failing cases with both results, for offline analysis
    if dump and fails:
        want_of = {id(f[-1]): w for a, w in ref for f in fails if f[-1] is a}
        with open(os.path.join(dump, f"fuzz_fail_{kind}.pkl"), "wb") as f:
            pickle.dump([(fl[:-1], fl[-1], want_of.get(id(fl[-1])), (compute(kind, fl[-1]) if fl[0] != "exception" else None)) for fl in fails[:8]], f)
    assert not fails, (kind, len(fails), fails[:12])
    assert compared >= cases // 3, (kind, compared, skipped)
