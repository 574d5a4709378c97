"""The numpy oracle against the reference build on RANDOM configurations (CPU): the same generators as the GPU fuzz
(tests/_fuzz_cases.py), the reference side produced by tests/_fuzz_ref_worker.py (fork-isolated, under AddressSanitizer
where gcc provides it, so results computed over a corrupted heap never count).  Pins af_oracle.{bft, xxcc, spectrogram,
stft, cqt, cwt, pwt, istft, xxcc_standard, cqt_chroma, cqhc, cq_deconv} well beyond the fixed cases of tests/test_oracle_vs_ref.py."""
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from conftest import rel_max
from oracle import af_oracle as O
from oracle import ref_lib as R

from _fuzz_cases import _sig

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


def reference_results(kind, seed, cases):
    if not R.available():
        pytest.skip("oracle/_ref/libaudioflux_ref.so not built (make -C oracle REF=<audioFlux tree>)")
    with tempfile.TemporaryDirectory() as d:
        out = os.path.join(d, "ref.pkl")
        env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
        try:
            asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True, timeout=30).stdout.strip()
        except Exception:
            asan = ""
        if os.path.isabs(asan) and os.path.exists(asan) and os.path.exists(R.REF_ASAN_PATH):
            env.update(LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=1", AFB200_FUZZ_ASAN="1")
        subprocess.run([sys.executable, os.path.join(HERE, "_fuzz_ref_worker.py"), kind, str(seed), str(cases), out], check=True,
                       env=env, timeout=900)
        with open(out, "rb") as f:
            return pickle.load(f)


def oracle(kind, a):
    """the oracle's answer in the layout tests/_fuzz_cases.compute returns, or None where it declines (see `declines`)"""
    x = _sig(a["seed"], a["L"], a["sr"]) if a["L"] else None
    if kind == "bft":
        kw = dict(hop=a["hop"], window_type=a["win"], scale=a["scale"], style=a["style"], norm=a["norm"], data_type=a["dt"],
                  low=a["lo"], high=a["hi"], bpo=a["bpo"])
        mel = O.bft(x, a["num"], a["r"], a["sr"], result_type=1, **kw)
        zr, zi = O.bft(x, a["num"], a["r"], a["sr"], result_type=0, **kw)
        return {"mel": mel.T, "zre": zr.T, "zim": zi.T, "cc": O.xxcc(mel, min(a["cc"], a["num"]), a["rect"]).T}
    if kind == "spec":
        spec = O.spectrogram(x, a["num"], a["sr"], a["lo"], a["hi"], a["bpo"], a["r"], a["win"], a["hop"], a["dt"], a["scale"], a["style"],
                             a["norm"])
        return {"spec": spec.T, "cc": O.xxcc(spec, min(a["cc"], spec.shape[1]), a["rect"]).T}
    if kind == "stft":
        n = 1 << a["r"]
        re, im = O.stft(x, n, a["hop"], O.fft_window(a["win"], n), bool(a["pad"]), a["pos"], a["mode"], a["v1"], a["v2"])
        return {"re": re, "im": im}
    if kind == "cqt":
        re, im = O.cqt(x, a["num"], a["sr"], a["lo"], a["bpo"], a["factor"], a["beta"], a["thresh"], a["win"], a["hop"] or None, a["norm"],
                       bool(a["is_scale"]))
        return {"re": re.T, "im": im.T}
    if kind == "cwt":
        re, im = O.cwt(x, a["num"], a["r"], a["sr"], a["wave"], a["scale"], a["lo"], a["hi"], a["bpo"], a["gamma"], a["beta"], bool(a["pad"]))
        out = {"re": re[::-1], "im": im[::-1]}
        if a["det"]:
            dr, di = O.cwt(x, a["num"], a["r"], a["sr"], a["wave"], a["scale"], a["lo"], a["hi"], a["bpo"], a["gamma"], a["beta"],
                           bool(a["pad"]), det=True)
            out["dre"], out["dim"] = dr, di
        return out
    if kind == "pwt":
        re, im, _, _ = O.pwt(x, a["num"], a["r"], a["sr"], a["lo"], a["hi"], a["bpo"], a["scale"], a["style"], a["norm"], bool(a["pad"]))
        return {"re": re, "im": im}
    if kind == "xxccstd":
        rng = np.random.default_rng(a["seed"])
        m = (rng.random((a["T"], a["num"])) ** 2 + 1e-3).astype(np.float32)
        e = (rng.random(a["T"]) + 0.1).astype(np.float32)
        c0, c1, c2 = O.xxcc_standard(m, e, a["cc"], a["win"], a["etype"], a["rect"])
        return {"coe": c0, "d1": c1, "d2": c2}
    if kind == "istft":
        n = 1 << a["r"]
        rng = np.random.default_rng(a["seed"])
        w = O.fft_window(a["win"], n)
        xx = (0.1 * rng.standard_normal((a["T"] - 1) * a["hop"] + n)).astype(np.float32)
        fr = np.stack([xx[t * a["hop"]:t * a["hop"] + n] * w for t in range(a["T"])])
        Z = np.fft.fft(fr, axis=1)
        re, im = np.ascontiguousarray(Z.real, dtype=np.float32), np.ascontiguousarray(Z.imag, dtype=np.float32)
        y = O.istft(re, im, n, a["hop"], w, a["method"])
        norm = np.zeros(len(y))
        for t in range(a["T"]):
            norm[t * a["hop"]:t * a["hop"] + n] += np.asarray(w, np.float64) ** (2 if a["method"] == 0 else 1)
        return {"y": np.where(norm > 1e-2, y, 0.0).astype(np.float32)}
    if kind == "cqtpost":
        hop = O.cqt_kernel_bank(a["num"], a["sr"], bpo=a["bpo"], norm=1)["fft_length"] // 4
        T = a["L"] // hop + 1
        rng = np.random.default_rng(a["seed"])
        z = ((rng.standard_normal((a["num"], T)) + 1j * rng.standard_normal((a["num"], T))) *
             np.exp(-np.arange(a["num"])[:, None] / 30.0)).astype(np.complex64)
        zt = z.T
        mag = np.abs(zt).astype(np.float32)
        tone, pitch = O.cq_deconv(mag, a["bpo"])
        out = {"cqcc": O.xxcc(mag, a["cc"], a["rect"]).T, "cqhc": O.cqhc((np.abs(zt) ** 2).astype(np.float32), a["hc"], a["bpo"]).T,
               "tone": tone.T, "pitch": pitch.T}
        if a["chroma"] <= a["bpo"] and a["bpo"] % a["chroma"] == 0:
            out["chroma"] = O.cqt_chroma(zt.real, zt.imag, a["chroma"], a["dt"], a["cnorm"], a["bpo"]).T
        return out
    raise KeyError(kind)


def declines(kind, a):
    """parameter regions the oracle (like the product) does not restate: the reference's own quirks there are documented in
    DESIGN.md section 1 and asserted in tests/test_ctor_fuzz.py"""
    if kind == "pwt":
        return a["style"] == 2 or (a["scale"] in (1, 6) and a["hi"] >= a["sr"] / 2)     # Gammatone pseudo banks; band edges beyond Nyquist
    if kind == "cwt":
        g, b = a["gamma"], a["beta"]
        return a["wave"] == 2 and g is not None and b is not None and b > g
    if kind in ("bft", "spec"):
        return a["scale"] in (1, 6) and a["hi"] >= a["sr"] / 2   # one-sided bank rows the reference overruns (Log / Linspace at Nyquist)
    return False


@pytest.mark.parametrize("kind,seed,cases,tol", [("bft", 201, 40, 2e-5), ("spec", 202, 30, 2e-5), ("stft", 203, 40, 2e-5), ("cqt", 204, 24, 2e-5),
                                                 ("cwt", 205, 40, 5e-5), ("pwt", 206, 40, 2e-5), ("xxccstd", 209, 30, 2e-5),
                                                 ("istft", 208, 30, 2e-5), ("cqtpost", 210, 24, 1e-4)])
def test_oracle_matches_the_reference_build_on_random_configurations(ref_lib, kind, seed, cases, tol):
    compared, fails = 0, []
    for a, want in reference_results(kind, seed, cases):
        if want == "crash" or "error" in want or declines(kind, a):
            continue
        try:
            got = oracle(kind, a)
        except (ZeroDivisionError, IndexError) as e:           # (hop 0 at the lowest CQT octave / bins beyond the one-sided bank)
            if kind == "cqt" and isinstance(e, ZeroDivisionError):
                continue
            fails.append(("exception", repr(e), a))
            continue
        compared += 1
        for k in want:
            if k not in got:                                    # (chroma where chromaNum does not divide binPerOctave: refused by both)
                continue
            if got[k].shape != want[k].shape:
                fails.append(("shape", k, got[k].shape, want[k].shape, a))
            elif want[k].size and plane_scale(want, k) > 1e-30:
                err = float(np.abs(got[k].astype(np.float64) - want[k]).max() / plane_scale(want, k))
                if not err < tol:
                    fails.append(("parity", k, err, a))
    assert not fails, (kind, len(fails), fails[:6])
    assert compared >= cases // 3, (kind, compared)
