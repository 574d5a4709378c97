"""Writes tests/golden/st.npz: the reference build's ST / FST outputs (re, im stacked) for the cases of
tests/_st_oracle.py whose output holds at most test_st_cpu.GOLDEN_MAX_CELLS complex values, so that the oracle tests run
where no reference build exists.  Needs oracle/_ref (make -C oracle REF=<audioFlux tree>).

    python tests/golden/make_golden_st.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.realpath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import test_st_cpu as T  # noqa: E402
from oracle import ref_lib as R  # noqa: E402

if __name__ == "__main__":
    if not R.available():
        sys.exit("oracle/_ref/libaudioflux_ref.so not built")
    res = T.reference_outputs(T.golden_names())
    np.savez_compressed(os.path.join(HERE, "st.npz"), **res)
    print(f"{len(res)} arrays")
