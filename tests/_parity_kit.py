"""What the per-object parity suites share: the reference build, the golden files that stand in for it where it is not
built, the check of an object's C API across the headers and libraries, the batched call with host or device pointers,
the helpers of direct calls on the device, and the reference's own Python package bound to this library."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

B200 = os.path.join(ROOT, "audioflux_b200", "lib", "libaudioflux_b200.so")


def ref_lib_or_none():
    """the reference build (oracle/_ref), or None where it is not built"""
    from oracle import ref_lib as R
    return R.get_ref_lib() if R.available() else None


class GoldenStore:
    """Outputs of the reference build under flat string keys, and tests/golden/<name> that keeps a subset of them so
    that the oracle tests also run where the reference build is missing.

    live(keys) -> {key: array} computes those outputs with the reference build; keys() is the exact key set the file
    holds; equal(live, stored) decides whether a stored array is still what the build computes."""

    def __init__(self, name, live, keys, equal=np.array_equal):
        self.name, self.live, self.keys, self.equal = name, live, keys, equal
        self.path = os.path.join(GOLDEN, name)

    def outputs(self, keys):
        """{key: array}: every key from the reference build when it is built, else the keys the golden file holds"""
        if ref_lib_or_none() is not None:
            return self.live(keys)
        if not os.path.exists(self.path):
            pytest.skip(f"no reference build and no tests/golden/{self.name}")
        g = np.load(self.path)
        return {k: g[k] for k in keys if k in g.files}

    def check_file(self):
        """the golden file holds exactly keys(), each array as the reference build computes it today"""
        if not (ref_lib_or_none() is not None and os.path.exists(self.path)):
            pytest.skip(f"needs both the reference build and tests/golden/{self.name}")
        g = np.load(self.path)
        keys = self.keys()
        assert set(g.files) == keys, sorted(set(g.files) ^ keys)[:20]
        live = self.live(keys)
        for k in g.files:
            assert self.equal(live[k], g[k]), k

    def write(self, directory=GOLDEN):
        """write the golden file from the reference build into directory; -> number of arrays"""
        arrays = self.live(self.keys())
        np.savez_compressed(os.path.join(directory, self.name), **arrays)
        return len(arrays)


def header_symbols(header, prefix):
    """functions include/<header> declares whose names match the regex prefix (comments ignored)"""
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", header)).read(), flags=re.S)
    return {m.group(1) for m in re.finditer(rf"\b((?:{prefix})[A-Za-z0-9_]*)\s*\(", src)}


def check_symbols(product_lib, header, prefix, api, names, ext):
    """The object's header declares `names` (the set, or how many) and afb200_ext.h declares the set `ext`; no other
    header under include/ declares the prefix; `api`, the object's table in capi, is exactly those; the product library
    exports all of them and the reference build, when present, those of the object's header."""
    own, own_ext = header_symbols(header, prefix), header_symbols("afb200_ext.h", prefix)
    assert (len(own) if isinstance(names, int) else own) == names, own
    assert own_ext == ext, own_ext
    declared = set().union(*(header_symbols(h, prefix) for h in os.listdir(os.path.join(ROOT, "include"))))
    assert declared == own | own_ext, declared ^ (own | own_ext)
    assert set(api) == own | own_ext
    for n in own | own_ext:
        assert hasattr(product_lib, n), n
    ref = ref_lib_or_none()
    if ref is not None:
        for n in own:
            assert hasattr(ref, n), n


def dptr(t):
    return C.c_void_p(t.data_ptr())


def stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class Out:
    """an argument of run_batch: a plane the call writes or updates in place, starting as the numpy array a"""

    def __init__(self, a):
        self.a = a


def run_batch(lib, name, args, device):
    """lib.<name>(*args, memKind, stream), a *Batch entry point, with host pointers (memKind 0, no stream) or with
    device pointers (memKind 1, the current stream).  Out(a) marks a plane the call writes; other numpy arrays are
    inputs, passed by address or first copied to a CUDA tensor; None, scalars and ctypes objects pass through unchanged.
    Asserts status 0, and synchronises after a call with device pointers.  -> the Out planes as numpy, in argument
    order"""
    planes = {k: np.ascontiguousarray(a.a if isinstance(a, Out) else a)
              for k, a in enumerate(args) if isinstance(a, (Out, np.ndarray))}
    if device:
        import torch
        planes = {k: torch.from_numpy(a).cuda() for k, a in planes.items()}
        ptrs, tail = {k: dptr(t) for k, t in planes.items()}, (1, stream())
    else:
        ptrs, tail = {k: a.ctypes.data for k, a in planes.items()}, (0, None)
    rc = getattr(lib, name)(*(ptrs.get(k, a) for k, a in enumerate(args)), *tail)
    assert rc == 0, lib.afb200_lastError()
    if device:
        torch.cuda.synchronize()
    return [planes[k].cpu().numpy() if device else planes[k] for k, a in enumerate(args) if isinstance(a, Out)]


def count_launches(lib, fn, warm):
    """kernels fn() launches.  warm=True counts a second call, after one that has done the lazy device set-up (plans,
    tables, workspaces); warm=False counts the first call, set-up included."""
    import torch
    if warm:
        fn()
    torch.cuda.synchronize()
    n0 = lib.afb200_kernelLaunchCount()
    fn()
    torch.cuda.synchronize()
    return lib.afb200_kernelLaunchCount() - n0


@pytest.fixture(scope="module")
def raf(product_lib):
    """the reference's own Python package: its default library is the reference build, lib_ext 'b200' this library"""
    from oracle import ref_lib as R
    from oracle import ref_python as RP
    if not (RP.available() and R.available()):
        pytest.skip("oracle/_ref/pyref or oracle/_ref/libaudioflux_ref.so not built (make -C oracle REF=<audioFlux tree>)")
    mod = RP.load(R.REF_PATH, B200)
    yield mod
    mod.fftlib.set_fft_lib(None)
