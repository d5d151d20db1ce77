"""numpy transcription of the per-sample noise generator (pfd_randn_f16, include/pfd_b200.h), used by
tests/test_rng_cpu.py and tests/test_rng_gpu.py.  Philox4x32-10 is bit-exact; the Box-Muller transform forms u1, u2
exactly as the kernel does in fp32 and evaluates log / sqrt / cos / sin in float64, so the kernel's fp16 output is
this value rounded once (within one fp16 ulp: the kernel's fp32 functions are accurate to a few fp32 ulps)."""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: 4 uint32 arrays (or scalars), key: 2 uint32 arrays -> 4 uint32 arrays."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint32) for c in ctr)
    k0, k1 = (np.asarray(k, dtype=np.uint32) for k in key)
    with np.errstate(over="ignore"):
        for r in range(10):
            if r:
                k0 = (k0 + W0).astype(np.uint32)
                k1 = (k1 + W1).astype(np.uint32)
            p0 = M0 * c0.astype(np.uint64)
            p1 = M1 * c2.astype(np.uint64)
            hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), (p0 & MASK).astype(np.uint32)
            hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), (p1 & MASK).astype(np.uint32)
            c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
    return c0, c1, c2, c3


def _box_muller(wa, wb):
    two32 = np.float32(2.0 ** -32)
    u1 = (wa.astype(np.float32) + np.float32(1.0)) * two32          # fp32, as the kernel forms it
    u2 = wb.astype(np.float32) * two32
    x = (np.float32(2.0) * u2).astype(np.float64)                   # sincospif(2 u2): 2 u2 is exact in fp32
    r = np.sqrt(-2.0 * np.log(u1.astype(np.float64)))
    return r * np.cos(np.pi * x), r * np.sin(np.pi * x)


def randn64(seed: int, n: int, stream: int, draw: int, first: int = 0) -> np.ndarray:
    """float64 values z(seed, stream, draw, e) for e in [first, first + n) (first a multiple of 4)."""
    assert first % 4 == 0
    g = np.arange(first // 4, (first + n + 3) // 4, dtype=np.uint64)
    ctr = ((g & MASK).astype(np.uint32), (g >> np.uint64(32)).astype(np.uint32),
           np.full(g.shape, draw & 0xFFFFFFFF, dtype=np.uint32), np.full(g.shape, stream & 0xFFFFFFFF, dtype=np.uint32))
    key = (np.uint32(seed & 0xFFFFFFFF), np.uint32(seed >> 32))
    w0, w1, w2, w3 = philox4x32_10(ctr, key)
    z0, z1 = _box_muller(w0, w1)
    z2, z3 = _box_muller(w2, w3)
    return np.stack([z0, z1, z2, z3], 1).reshape(-1)[:n]


def randn_batch64(seeds, n: int, stream: int, draw: int, scale: float = 1.0) -> np.ndarray:
    """[B, n] float64 = scale * z for each seed: pfd_randn_f16 before its fp16 rounding."""
    return np.stack([scale * randn64(int(s), n, stream, draw) for s in seeds])
