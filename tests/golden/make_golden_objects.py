"""Writes the golden files of the per-object suites from the reference build: spectral.npz, nsgt.npz, st.npz,
cepstrogram.npz, resample.npz, hpss.npz, onset.npz, harmonic_ratio.npz, wavelet.npz, nmf.npz and dsp.npz, each from the
store (GOLD) of tests/test_<object>_cpu.py, so that their oracle tests run where no reference build exists.  Needs
oracle/_ref (make -C oracle REF=<audioFlux tree>).

    python tests/golden/make_golden_objects.py [--out DIR] [object ...]"""
import argparse
import importlib
import os
import sys

HERE = os.path.dirname(os.path.realpath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import ref_lib as R  # noqa: E402

OBJECTS = ("spectral", "nsgt", "st", "cepstrogram", "resample", "hpss", "onset", "harmonic_ratio", "wavelet", "nmf", "dsp")

if __name__ == "__main__":
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("objects", nargs="*", default=list(OBJECTS), help=f"any of {', '.join(OBJECTS)} (default: all)")
    ap.add_argument("--out", default=HERE, help="directory to write into (default: tests/golden)")
    a = ap.parse_args()
    for obj in set(a.objects) - set(OBJECTS):
        ap.error(f"unknown object {obj!r}")
    if not R.available():
        sys.exit("oracle/_ref/libaudioflux_ref.so not built")
    for obj in a.objects:
        store = importlib.import_module(f"test_{obj}_cpu").GOLD
        print(f"{store.name}: {store.write(a.out)} arrays")
