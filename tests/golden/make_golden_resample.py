"""Writes tests/golden/resample.npz: the reference build's resampler outputs (one array per call, key "<case>__<call>")
for the cases of tests/_resample_oracle.py with inputs of at most test_resample_cpu.GOLDEN_MAX_LEN samples, so that the
oracle tests run where no reference build exists.  Needs oracle/_ref (make -C oracle REF=<audioFlux tree>).

    python tests/golden/make_golden_resample.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.realpath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import test_resample_cpu as T  # noqa: E402
from oracle import ref_lib as R  # noqa: E402

if __name__ == "__main__":
    if not R.available():
        sys.exit("oracle/_ref/libaudioflux_ref.so not built")
    res = T.reference_outputs(sorted(T.golden_names()))
    arrays = {T._key(n, k): o for n, outs in res.items() for k, o in enumerate(outs)}
    np.savez_compressed(os.path.join(HERE, "resample.npz"), **arrays)
    print(f"{len(arrays)} arrays")
