"""The reference's own Python package (byte-compiled by `make -C oracle` into oracle/_ref/pyref), importable next to a
chosen pair of shared libraries.  Test infrastructure only.

`load(default_lib, b200_lib)` copies the sourceless package into a temp dir whose `lib/` holds
    libaudioflux.so       -> default_lib   (what `import audioflux` loads, python/audioflux/fftlib.py:127)
    libaudioflux_b200.so  -> b200_lib      (what `fftlib.set_fft_lib(lib_ext='b200')` switches to, fftlib.py:96-124)
stubs the optional third-party imports (soundfile, matplotlib) and returns the imported `audioflux` module."""
from __future__ import annotations

import importlib
import os
import shutil
import sys
import tempfile
import types

_HERE = os.path.dirname(os.path.realpath(__file__))
PYREF = os.path.join(_HERE, "_ref", "pyref", "audioflux")
_state = {}


def available() -> bool:
    return os.path.exists(os.path.join(PYREF, "__init__.pyc"))


class _Stub(types.ModuleType):
    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return type(name, (), {})


def load(default_lib: str, b200_lib: str):
    if "mod" in _state:
        return _state["mod"]
    if not available():
        raise FileNotFoundError(f"{PYREF} missing: run `make -C oracle REF=<audioFlux tree>`")
    tmp = tempfile.mkdtemp(prefix="af_pyref_")
    pkg = os.path.join(tmp, "audioflux")
    shutil.copytree(PYREF, pkg)
    os.makedirs(os.path.join(pkg, "lib"), exist_ok=True)
    os.symlink(default_lib, os.path.join(pkg, "lib", "libaudioflux.so"))
    os.symlink(b200_lib, os.path.join(pkg, "lib", "libaudioflux_b200.so"))
    for m in ("soundfile", "matplotlib", "matplotlib.pyplot", "matplotlib.axes", "matplotlib.colors", "matplotlib.ticker",
              "matplotlib.cm", "matplotlib.axis", "matplotlib.transforms", "matplotlib.collections", "matplotlib.patches"):
        sys.modules.setdefault(m, _Stub(m))
    sys.path.insert(0, tmp)
    try:
        mod = importlib.import_module("audioflux")
    finally:
        sys.path.remove(tmp)
    _state["mod"], _state["tmp"] = mod, tmp
    return mod
