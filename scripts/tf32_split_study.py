"""Accuracy of TF32 tensor-core formulations of the policy GEMMs, emulated in NumPy (no GPU needed).

Question for the tensor-core update kernels (DESIGN.md section 8): which operand split keeps the float32-grade accuracy
the parity tests need?  wgmma .tf32 reads 32-bit operands and keeps sign + 8 exponent + 10 mantissa bits
(truncation), products are exact, accumulation is float32.  Variants:
  1xTF32        a_hi*b_hi
  3xTF32        a_hi*b_hi + a_lo*b_hi + a_hi*b_lo          (lo = x - hi, itself truncated to tf32)
against plain float32 FMA chains and the float64 truth, on the shapes of the Hopper net (K = 64 layers, Gram over 128
samples) with activations in (-1, 1) and weights ~ N(0, 1/sqrt(64))."""
import numpy as np


def tf32(x):
    b = np.asarray(x, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)
    return b.view(np.float32)


def split(x):
    hi = tf32(x)
    lo = tf32((np.asarray(x, np.float32) - hi).astype(np.float32))
    return hi, lo


def mm32(a, b):
    """float32 accumulation of exact products (the products of two tf32 numbers fit float32's 24 bits exactly when
    both have 11 significant bits; np.float32 matmul of float64-exact products is emulated by a float64 product
    rounded per k-step into a float32 accumulator)."""
    acc = np.zeros((a.shape[0], b.shape[1]), np.float32)
    for k in range(a.shape[1]):
        acc = (acc.astype(np.float64) + a[:, k:k + 1].astype(np.float64) * b[k:k + 1, :].astype(np.float64)).astype(np.float32)
    return acc


def study(M, K, N, rng, label):
    a = np.tanh(rng.randn(M, K)).astype(np.float32)
    b = (rng.randn(K, N) / np.sqrt(K)).astype(np.float32)
    truth = a.astype(np.float64) @ b.astype(np.float64)
    scale = np.abs(truth).max()
    ah, al = split(a)
    bh, bl = split(b)
    res = {
        "float32 FMA": mm32(a, b),
        "1xTF32": mm32(ah, bh),
        "3xTF32": (mm32(ah, bh).astype(np.float64) + mm32(al, bh) + mm32(ah, bl)).astype(np.float32),
    }
    print("%-34s" % label, "  ".join("%s max|err|/max|out| = %.2e" % (k, np.abs(v - truth).max() / scale) for k, v in res.items()))


if __name__ == "__main__":
    rng = np.random.RandomState(0)
    study(128, 64, 64, rng, "layer   [128 x 64] . [64 x 64]")
    study(64, 128, 64, rng, "Gram    [64 x 128] . [128 x 64]")
    study(128, 20, 64, rng, "input   [128 x 20] . [20 x 64]")
