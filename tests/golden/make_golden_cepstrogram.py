"""Writes tests/golden/cepstrogram.npz: the reference build's cepstrogram outputs (cepstrums, envelope, details stacked)
for the cases of tests/_cepstrogram_oracle.py with at most test_cepstrogram_cpu.GOLDEN_MAX_CELLS cells per output, so
that the oracle tests run where no reference build exists.  Needs oracle/_ref (make -C oracle REF=<audioFlux tree>).

    python tests/golden/make_golden_cepstrogram.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.realpath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import test_cepstrogram_cpu as T  # noqa: E402
from oracle import ref_lib as R  # noqa: E402

if __name__ == "__main__":
    if not R.available():
        sys.exit("oracle/_ref/libaudioflux_ref.so not built")
    res = T.reference_outputs(T.golden_names())
    np.savez_compressed(os.path.join(HERE, "cepstrogram.npz"), **res)
    print(f"{len(res)} arrays")
