"""Tensor-core (wgmma) Fisher-vector kernel (update_umma.cu) against the FP32 tiled-GEMM kernel and the float64 oracle on Hopper-shaped
data, then timing at the cfg4 batch size.  Usage: python scripts/umma_fvp_check.py"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import policy as P          # noqa: E402
from rllab_b200 import _lib as L, ops   # noqa: E402


def make(O, A, H, N, T, dev, seed=0):
    rng = np.random.RandomState(seed)
    dims = P.Dims(O, (H, H), A)
    theta = P.init_params(dims, rng) + 0.05 * rng.randn(dims.P)
    theta[-A:] = -0.3 + 0.1 * np.arange(A)
    th32 = torch.tensor(theta, dtype=torch.float32, device=dev)
    theta = th32.double().cpu().numpy()
    b = ops.LaneBatch(O, A, N, T, dev)
    b.obs.copy_(torch.tensor(rng.randn(O, T, N), dtype=torch.float32))
    mean, ls = P.forward(theta, b.obs.cpu().numpy().reshape(O, -1).T.astype(np.float64), dims)
    b.mean.copy_(torch.tensor(mean.T.reshape(A, T, N), dtype=torch.float32))
    b.act.copy_(b.mean + torch.randn_like(b.mean) * 0.7)
    b.adv.copy_(torch.tensor(rng.randn(T, N), dtype=torch.float32))
    b.log_std.copy_(torch.tensor(ls, dtype=torch.float32))
    b.flags.zero_()
    return dims, theta, th32, b


def main():
    dev = torch.device("cuda:0")
    L.load()
    ok = True
    for (O, A, N, T) in ((20, 3, 509, 31), (4, 1, 300, 7), (13, 2, 128, 3)):
        dims, theta, th32, b = make(O, A, 64, N, T, dev)
        dd = (O, 64, 64, A)
        g = torch.zeros(dims.P, dtype=torch.float64, device=dev)
        hc = b.hcache(64, 64)
        ops.grad(L.LOSS_TRPO, th32, dd, 1e-6, b, g, None, hc)
        x = np.random.RandomState(1).randn(dims.P)
        xd = torch.tensor(x, dtype=torch.float64, device=dev)
        H_umma, H_gemm = torch.zeros_like(g), torch.zeros_like(g)
        ops.fvp(th32, dd, 1e-6, b, xd, 1e-5, 1.0, H_umma, hc)
        ops.fvp(th32, dd, 1e-6, b, xd, 1e-5, 1.0, H_gemm, None)
        torch.cuda.synchronize()
        batch = dict(obs=b.obs.cpu().numpy().reshape(O, -1).T.astype(np.float64))
        ref = P.fvp(theta, batch, xd.float().double().cpu().numpy(), dims, 0.0) + 1e-5 * x
        eu = np.abs(H_umma.cpu().numpy() - ref).max() / np.abs(ref).max()
        eg = np.abs(H_gemm.cpu().numpy() - ref).max() / np.abs(ref).max()
        print("O=%d A=%d B=%d: max err / max|ref|  wgmma %.3e   FP32 GEMM %.3e   nan=%s" %
              (O, A, N * T, eu, eg, bool(np.isnan(H_umma.cpu().numpy()).any())), flush=True)
        if not (eu < 2e-4):
            ok = False
            d = np.abs(H_umma.cpu().numpy() - ref) / np.abs(ref).max()
            names = ["W0", "b0", "W1", "b1", "Wo", "bo", "ls"]
            k = 0
            for nm, sh in zip(names, dims.shapes):
                n = int(np.prod(sh))
                print("    block %s: max err %.3e" % (nm, d[k:k + n].max()))
                k += n
    # timing at the cfg4 per-GPU batch (4096 lanes x 500 steps)
    dims, theta, th32, b = make(20, 3, 64, 4096, 500, dev)
    dd = (20, 64, 64, 3)
    g = torch.zeros(dims.P, dtype=torch.float64, device=dev)
    hc = b.hcache(64, 64)
    ops.grad(L.LOSS_TRPO, th32, dd, 1e-6, b, g, None, hc)
    xd = torch.randn(dims.P, dtype=torch.float64, device=dev)
    out = torch.zeros_like(g)
    for name, cache in (("wgmma (cached activations)", hc), ("FP32 tiled GEMM (no cache)", None)):
        for _ in range(2):
            ops.fvp(th32, dd, 1e-6, b, xd, 1e-5, 1.0, out, cache)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            ops.fvp(th32, dd, 1e-6, b, xd, 1e-5, 1.0, out, cache)
        e1.record()
        torch.cuda.synchronize()
        print("FVP %s: %.3f ms / %d samples" % (name, e0.elapsed_time(e1) / 10, b.B))
    print("OK" if ok else "MISMATCH")
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
