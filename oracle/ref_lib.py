"""ctypes handle on the UNMODIFIED reference build in oracle/_ref (test infrastructure only).

The library is produced by `make -C oracle REF=<audioFlux tree>` (or by build() when
the audioFlux tree is present).  It is never loaded by the product package."""
from __future__ import annotations

import ctypes
import os

from audioflux_b200 import capi

_HERE = os.path.dirname(os.path.realpath(__file__))
REF_PATH = os.path.join(_HERE, "_ref", "libaudioflux_ref.so")
REF_OMP_PATH = os.path.join(_HERE, "_ref", "libaudioflux_ref_omp.so")
REF_ASAN_PATH = os.path.join(_HERE, "_ref", "libaudioflux_ref_asan.so")     # needs LD_PRELOAD=libasan in the loading process

_cache = {}


def available(omp: bool = False) -> bool:
    return os.path.exists(REF_OMP_PATH if omp else REF_PATH)


def get_ref_lib(omp: bool = False, asan: bool = False):
    path = REF_ASAN_PATH if asan else REF_OMP_PATH if omp else REF_PATH
    if path not in _cache:
        if not os.path.exists(path):
            raise FileNotFoundError(f"{path} missing: run `make -C oracle REF=<audioFlux tree>`")
        lib = ctypes.CDLL(path)
        capi.bind(lib)
        _cache[path] = lib
    return _cache[path]
