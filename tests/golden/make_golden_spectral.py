"""Writes tests/golden/spectral.npz: the reference build's SpectralObj outputs for the inputs and parameter variants of
tests/_spectral_cases.py (3 seeded spectrogram sets x 3 edge modes x every variant), so that the oracle tests run where
no reference build exists.  Needs oracle/_ref (make -C oracle REF=<audioFlux tree>).

    python tests/golden/make_golden_spectral.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.realpath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import test_spectral_cpu as T  # noqa: E402
from oracle import ref_lib as R  # noqa: E402

if __name__ == "__main__":
    if not R.available():
        sys.exit("oracle/_ref/libaudioflux_ref.so not built")
    res = T._reference_outputs()
    np.savez_compressed(os.path.join(HERE, "spectral.npz"), **{k: np.asarray(v, np.float32) for k, v in res.items()})
    print(f"{len(res)} arrays")
