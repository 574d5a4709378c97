#!/usr/bin/env python3
"""Per-octave comparison of the CQT octave kernels (wgmma / mma.sync / fp32) against each other and the oracle."""
import os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.realpath(__file__)))
sys.path.insert(0, ROOT)
import torch
import audioflux_b200 as af
from oracle import af_oracle as O

def run(kernel, x):
    if kernel: os.environ["AFB200_CQT_KERNEL"] = kernel
    else: os.environ.pop("AFB200_CQT_KERNEL", None)
    c = af.CQT(84, 48000)
    re, im = c.cqt_batch(x)
    torch.cuda.synchronize()
    return (re.cpu().numpy() + 1j * im.cpu().numpy())

def main():
    rng = np.random.default_rng(3)
    L = int(os.environ.get("DBG_L", "48000"))
    xh = (0.1 * rng.standard_normal((2, L))).astype(np.float32)
    x = torch.from_numpy(xh).cuda()
    ref = run("fp32", x)
    wr, wi = O.cqt(xh[1], 84, 48000, norm=O.NORM_AREA)
    want = wr + 1j * wi
    print("fp32 vs oracle", float(np.abs(ref[1] - want).max() / np.abs(want).max()))
    for name, k in (("mma.sync", "mma"), ("wgmma", None)):
        got = run(k, x)
        for o in range(7):
            sl = slice(12 * o, 12 * o + 12)
            e = float(np.abs(got[1][:, sl] - want[:, sl]).max() / np.abs(want[:, sl]).max())
            e2 = float(np.abs(got[0][:, sl] - ref[0][:, sl]).max() / np.abs(ref[0][:, sl]).max())
            print(f"{name}: octave {o} (hop {2 << o}) rel err vs oracle {e:.3e} vs fp32 {e2:.3e} nan {int(np.isnan(got[:, :, sl]).sum())}")
    print("DEBUG_CQT_DONE")

if __name__ == "__main__":
    main()
