"""Loader for the product library ``libaudioflux_b200.so`` (C-ABI boundary).

Plays the role of python/audioflux/fftlib.py:96-124 in the reference.  There is
no CPU fallback: if the CUDA library is missing this raises, and compute entry
points fail loudly (non-zero status + message) when no GPU is usable.
"""
from __future__ import annotations

import ctypes
import os

from . import capi

_HERE = os.path.dirname(os.path.realpath(__file__))
LIB_NAME = "libaudioflux_b200.so"
# AFB200_LIB_PATH: another build of the SAME library (sanitizer build of the host code, tools/asan_host_check.sh) --
# never a different implementation: there is no CPU fallback to select
LIB_PATH = os.environ.get("AFB200_LIB_PATH") or os.path.join(_HERE, "lib", LIB_NAME)

__LIBRARY = {"lib": None, "present": None}


class LibraryNotBuilt(RuntimeError):
    pass


def load_library(path: str):
    lib = ctypes.CDLL(path)          # RTLD_LOCAL: the reference build exports the same symbol names
    present = capi.bind(lib)
    return lib, present


def get_lib():
    if __LIBRARY["lib"] is None:
        if not os.path.exists(LIB_PATH):
            raise LibraryNotBuilt(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                f"or `make -C audioflux_b200/csrc` (no CPU fallback exists)")
        __LIBRARY["lib"], __LIBRARY["present"] = load_library(LIB_PATH)
    return __LIBRARY["lib"]


def last_error() -> str:
    lib = get_lib()
    msg = lib.afb200_lastError()
    return msg.decode() if msg else ""


class AfB200Error(RuntimeError):
    pass


def check(status: int, what: str):
    if status != 0:
        raise AfB200Error(f"{what} failed with status {status}: {last_error()}")
