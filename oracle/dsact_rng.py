"""Host restatement of the device generator (csrc/kernels.cuh): Philox4x32-10, the (0,1] uniform map, Box-Muller, the
replay-index draw of `replay_index` and the noise layout of `noise_body`.  numpy only, CPU.

The integer parts (Philox words, replay indices) are bit-exact restatements.  `u01` repeats the kernel's float32
arithmetic exactly; Box-Muller runs in float64 on those float32 uniforms, so the device's `logf` / `sincospif` results
differ from it by a few float32 ulps."""
from __future__ import annotations

import numpy as np

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_LO32 = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)

NOISE_DOMAIN = 0x4E4F4953   # "NOIS": third counter word of every noise block
INDEX_DOMAIN = 0x49445853   # "IDXS": third counter word of every replay-index block


def _u32(x) -> np.ndarray:
    return np.asarray(x, dtype=np.uint64) & _LO32


def philox4x32_10(ctr, key):
    """Philox4x32-10 on counters ctr = (c0, c1, c2, c3) and key = (k0, k1); each word a uint32 scalar or array (broadcast).
    Returns the four output words as uint32 arrays."""
    x, y, z, w = (_u32(c) for c in ctr)
    x, y, z, w = np.broadcast_arrays(x, y, z, w)
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = _M0 * x, _M1 * z            # 32 x 32 -> 64 bits: exact in uint64
        x, y, z, w = ((p1 >> _S32) ^ y ^ np.uint64(k0), p1 & _LO32, (p0 >> _S32) ^ w ^ np.uint64(k1), p0 & _LO32)
        k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
    return tuple(v.astype(np.uint32) for v in (x, y, z, w))


def u01(x) -> np.ndarray:
    """`((float)x + 0.5f) * 2.3283064365386963e-10f` in float32: uint32 -> float32 rounds to nearest; the result is in (0, 1]."""
    f = np.asarray(x, dtype=np.uint32).astype(np.float32)
    return (f + np.float32(0.5)) * np.float32(2.3283064365386963e-10)


def box_muller(a, b):
    """The kernel's Box-Muller pair from two uint32 words, in float64 on the float32 uniforms."""
    r = np.sqrt(-2.0 * np.log(u01(a).astype(np.float64)))
    t = 2.0 * u01(b).astype(np.float64)      # sincospif(2 u): exact doubling in float32 as well
    return r * np.cos(np.pi * t), r * np.sin(np.pi * t)


def _key(seed: int):
    seed = int(seed) & (2 ** 64 - 1)
    return seed & 0xFFFFFFFF, seed >> 32


def _mulhi64(a: np.ndarray, b: int) -> np.ndarray:
    """High 64 bits of the 128-bit product of uint64 a and b (`__umul64hi`), on 32-bit limbs."""
    a = np.asarray(a, dtype=np.uint64)
    b = np.uint64(int(b) & (2 ** 64 - 1))
    a0, a1, b0, b1 = a & _LO32, a >> _S32, b & _LO32, b >> _S32
    p00, p01, p10, p11 = a0 * b0, a0 * b1, a1 * b0, a1 * b1
    mid = (p00 >> _S32) + (p01 & _LO32) + (p10 & _LO32)
    return p11 + (p01 >> _S32) + (p10 >> _S32) + (mid >> _S32)


def replay_indices(seed: int, counter: int, B: int, size: int) -> np.ndarray:
    """Rows 0..B-1 of `replay_index`: row r reads Philox block (r >> 1, counter, INDEX_DOMAIN, 0); even rows take words
    (x, y), odd rows (z, w), as the 64-bit value hi << 32 | lo; the index is its 64 x 64 -> high-64 product with `size`."""
    rows = np.arange(int(B), dtype=np.int64)
    x, y, z, w = philox4x32_10((rows >> 1, int(counter), INDEX_DOMAIN, 0), _key(seed))
    odd = (rows & 1).astype(bool)
    hi = np.where(odd, z, x).astype(np.uint64)
    lo = np.where(odd, w, y).astype(np.uint64)
    return _mulhi64((hi << _S32) | lo, size).astype(np.int64)


def device_noise(seed: int, counter: int, B: int, A: int):
    """eps1, eps2 [B, A] and z3, z4 [B] (float64) as `noise_body` lays them out: a stream of normal pairs, pair p drawn from
    Philox block (p >> 1, counter, NOISE_DOMAIN, 0) by Box-Muller on words (x, y) (even p) or (z, w) (odd p).  eps1 takes
    the first ceil(B*A/2) pairs, eps2 the next as many, then z3 and z4 ceil(B/2) each; a tensor of odd length drops the
    second value of its last pair."""
    B, A = int(B), int(A)
    n_ea, n_z = (B * A + 1) // 2, (B + 1) // 2
    total = 2 * n_ea + 2 * n_z
    blocks = np.arange((total + 1) // 2, dtype=np.int64)
    x, y, z, w = philox4x32_10((blocks, int(counter), NOISE_DOMAIN, 0), _key(seed))
    n0, n1 = box_muller(x, y)
    n2, n3 = box_muller(z, w)
    flat = np.stack([n0, n1, n2, n3], axis=1).reshape(-1)    # values 2p, 2p + 1 belong to pair p
    starts = (0, 2 * n_ea, 4 * n_ea, 4 * n_ea + 2 * n_z)
    eps1 = flat[starts[0]:starts[0] + B * A].reshape(B, A)
    eps2 = flat[starts[1]:starts[1] + B * A].reshape(B, A)
    return eps1, eps2, flat[starts[2]:starts[2] + B].copy(), flat[starts[3]:starts[3] + B].copy()
