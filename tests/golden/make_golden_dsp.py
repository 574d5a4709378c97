"""Writes tests/golden/dsp.npz from the reference build, from the store (GOLD) of tests/test_dsp_cpu.py, so that the
cross-correlation and CZT oracle tests run where no reference build exists.  Needs oracle/_ref
(make -C oracle REF=<audioFlux tree>).

    python tests/golden/make_golden_dsp.py [--out DIR]"""
import argparse
import os
import sys

HERE = os.path.dirname(os.path.realpath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import ref_lib as R  # noqa: E402

if __name__ == "__main__":
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", default=HERE, help="directory to write into (default: tests/golden)")
    a = ap.parse_args()
    if not R.available():
        sys.exit("oracle/_ref/libaudioflux_ref.so not built")
    from test_dsp_cpu import GOLD  # noqa: E402
    print(f"{GOLD.name}: {GOLD.write(a.out)} arrays")
