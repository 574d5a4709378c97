"""Multi-destination store path of the fused MFCC kernel (the all-gather fused into the epilogue).
One GPU: extra destinations are plain local buffers, which exercises the kernel and the C ABI; with >= 2 GPUs
a torchrun job maps real peer buffers (cudaIpc) and checks every rank's gathered array bit for bit."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import audioflux_b200 as af
from conftest import noise

pytestmark = pytest.mark.gpu

S, D = af.SpectralFilterBankScaleType, af.SpectralDataType
ROOT = os.path.dirname(os.path.dirname(os.path.realpath(__file__)))


@pytest.fixture(scope="module")
def torch_cuda(cuda_device):
    import torch
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)
    return torch


def test_scatter_to_local_destinations(torch_cuda, product_lib):
    torch = torch_cuda
    B, L, CC = 5, 30720, 40
    bft = af.BFT(128, 11, 48000, slide_length=512, scale_type=S.MEL, data_type=D.POWER)
    T = bft.cal_time_length(L)
    x = torch.from_numpy(np.stack([noise(40 + i, L) for i in range(B)])).cuda()
    want = bft.mfcc_batch(x, CC)
    for n_peer in (0, 1, 3, 15):
        outs = [torch.zeros((2, B, T, CC), device="cuda") for _ in range(n_peer + 1)]       # slot 1 of a 2-slot array
        off = B * T * CC * 4
        peers = (C.c_void_p * max(1, n_peer))(*[C.c_void_p(o.data_ptr() + off) for o in outs[1:]])
        n0 = product_lib.afb200_kernelLaunchCount()
        rc = product_lib.bftObj_mfccBatchScatter(bft._obj, C.c_void_p(x.data_ptr()), L, B, CC, 0,
                                                 C.c_void_p(outs[0].data_ptr() + off), n_peer, peers,
                                                 C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == 0, product_lib.afb200_lastError()
        torch.cuda.synchronize()
        assert product_lib.afb200_kernelLaunchCount() - n0 == 1               # still ONE launch
        for o in outs:
            assert torch.equal(o[1], want) and not o[0].any()                  # right slot, nothing else touched


def test_scatter_argument_checks(torch_cuda, product_lib):
    torch = torch_cuda
    bft = af.BFT(128, 11, 48000, slide_length=512, scale_type=S.MEL, data_type=D.POWER)
    x = torch.zeros((1, 4096), device="cuda")
    o = torch.zeros((1, 5, 40), device="cuda")
    peers = (C.c_void_p * 16)(*[C.c_void_p(o.data_ptr())] * 16)
    assert product_lib.bftObj_mfccBatchScatter(bft._obj, C.c_void_p(x.data_ptr()), 4096, 1, 40, 0, C.c_void_p(o.data_ptr()),
                                               16, peers, None) != 0          # more than 15 peers
    b2 = af.BFT(64, 10, 48000, slide_length=256, scale_type=S.MEL, data_type=D.POWER)    # not the fused configuration
    assert product_lib.bftObj_mfccBatchScatter(b2._obj, C.c_void_p(x.data_ptr()), 4096, 1, 20, 0, C.c_void_p(o.data_ptr()),
                                               1, peers, None) != 0
    assert b"fused" in product_lib.afb200_lastError()


def test_peer_buffer_export(torch_cuda, product_lib):
    torch = torch_cuda
    p = C.c_void_p()
    assert product_lib.afb200_peerAlloc(C.byref(p), 1 << 20) == 0 and p.value
    h = (C.c_ubyte * 64)()
    assert product_lib.afb200_ipcGetHandle(p, h) == 0 and any(h)
    from audioflux_b200.dist import _DevArray
    t = torch.as_tensor(_DevArray(p.value, (256, 1024)), device="cuda")
    t.fill_(3.0)
    assert float(t.sum()) == 3.0 * 256 * 1024 and t.data_ptr() == p.value       # zero-copy view
    del t
    assert product_lib.afb200_peerFree(p) == 0


def test_peer_scatter_single_rank_group(torch_cuda, tmp_path):
    """world = 1: no peers to map, the same object still produces the (1, B, T, cc) gathered array."""
    torch = torch_cuda
    import torch.distributed as dist
    from audioflux_b200.dist import PeerScatter
    dist.init_process_group("gloo", init_method=f"file://{tmp_path}/store", rank=0, world_size=1)
    try:
        bft = af.BFT(128, 11, 48000, slide_length=512, scale_type=S.MEL, data_type=D.POWER)
        x = torch.from_numpy(np.stack([noise(50 + i, 20480) for i in range(3)])).cuda()
        sc = PeerScatter(bft, 3, 20480, 13)
        out = sc(x)
        sc.fence()
        torch.cuda.synchronize()
        assert torch.equal(out[0], bft.mfcc_batch(x, 13))
        sc.close()
    finally:
        dist.destroy_process_group()


def test_peer_scatter_two_gpus(torch_cuda):
    torch = torch_cuda
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    n = 2 if n < 4 else 4 if n < 8 else 8
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}",
           "--master-addr", "127.0.0.1", "--master-port", "29533", os.path.join(ROOT, "tests", "_peer_scatter_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=420)
    assert r.returncode == 0 and f"PEER_SCATTER_OK {n}" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
