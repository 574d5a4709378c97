"""Writes tests/golden/hpss.npz: the reference build's HPSS outputs (key "<case>__0" for h, "<case>__1" for p; a skipped
output has no key) for the cases of tests/_hpss_oracle.py with outputs of at most test_hpss_cpu.GOLDEN_MAX_LEN samples,
so that the oracle tests run where no reference build exists.  Needs oracle/_ref (make -C oracle REF=<audioFlux tree>).

    python tests/golden/make_golden_hpss.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.realpath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import test_hpss_cpu as T  # noqa: E402
from oracle import ref_lib as R  # noqa: E402

if __name__ == "__main__":
    if not R.available():
        sys.exit("oracle/_ref/libaudioflux_ref.so not built")
    res = T.reference_outputs(sorted(T.golden_names()))
    arrays = {T._key(n, k): o for n, outs in res.items() for k, o in enumerate(outs) if o is not None}
    np.savez_compressed(os.path.join(HERE, "hpss.npz"), **arrays)
    print(f"{len(arrays)} arrays")
