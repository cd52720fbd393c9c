"""Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11) on the host, in the word layout of
pulse_b200/csrc/philox.cuh (TEST INFRASTRUCTURE): key = seed (lo, hi), counter = (index lo, index hi, offset lo, offset hi).  With the
kernels' `u01` and `box_muller`, tests regenerate a kernel's Philox draws, inject them, and compare with the kernel's own draws."""
import numpy as np

_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(seed: int, index, offset):
    """The four 32-bit words of the blocks (seed, index[i], offset[i]); index / offset are python ints or sequences of them (< 2^64).
    Returns four uint64 arrays holding 32-bit values."""
    idx = np.asarray(index, dtype=np.uint64)
    off = np.broadcast_to(np.asarray(offset, dtype=np.uint64), idx.shape)
    c0, c1, c2, c3 = idx & _M32, idx >> np.uint64(32), off & _M32, off >> np.uint64(32)
    k0, k1 = seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = c0 * np.uint64(0xD2511F53), c2 * np.uint64(0xCD9E8D57)
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ np.uint64(k0), p1 & _M32, (p0 >> np.uint64(32)) ^ c3 ^ np.uint64(k1), p0 & _M32
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return c0, c1, c2, c3


def u01(w) -> np.ndarray:
    """philox.cuh's u01: the top 24 bits on the 2^-24 grid, fp32 (exact)."""
    return ((np.asarray(w, dtype=np.uint64) >> np.uint64(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)).astype(np.float32)


def box_muller(a, b):
    """philox.cuh's box_muller in float64 (the kernel's __logf / __sincosf are approximations: compare within a tolerance)."""
    u1 = ((np.asarray(a, dtype=np.uint64) >> np.uint64(8)).astype(np.float64) + 1.0) / 16777216.0
    u2 = (np.asarray(b, dtype=np.uint64) >> np.uint64(8)).astype(np.float64) / 16777216.0
    r = np.sqrt(-2.0 * np.log(u1))
    return r * np.cos(2 * np.pi * u2), r * np.sin(2 * np.pi * u2)
