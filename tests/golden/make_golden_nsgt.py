"""Writes tests/golden/nsgt.npz: the reference build's NSGT tables (lengths, bins, centre frequencies, offsets) for the
case set of tests/_nsgt_oracle.py, and the windows, cells and matrices of its 2^8 cases and the cells of the docs example
(test_nsgt_cpu.golden_subset), so that the oracle tests run where no reference build exists.  Needs oracle/_ref
(make -C oracle REF=<audioFlux tree>).

    python tests/golden/make_golden_nsgt.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.realpath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import test_nsgt_cpu as T  # noqa: E402
from oracle import ref_lib as R  # noqa: E402

if __name__ == "__main__":
    if not R.available():
        sys.exit("oracle/_ref/libaudioflux_ref.so not built")
    res = T.golden_subset(T.reference_outputs())
    np.savez_compressed(os.path.join(HERE, "nsgt.npz"), **res)
    print(f"{len(res)} arrays")
