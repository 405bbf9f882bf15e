"""Oracle for MatMulNBits with 4-bit weights and block-wise scales (the project's extension; the reference has no quantised MatMul).

Layout (include/it_b200.h, it_b200_matmul_nbits): B is uint8 [N, K / bs, bs / 2]; element k of column n is in byte
(n, k / bs, (k % bs) / 2), even k in the low nibble.  scales [N * K / bs], the scale of (n, block) at n * (K / bs) + block.  Zero
points are absent (z = 8) or nibble-packed, (K / bs) / 2 bytes per column, block b at byte b / 2, low nibble for even b.
W[k, n] = (q[n, k] - z[n, k / bs]) * s[n, k / bs].

* `unpack_codes`, `unpack_zero_points`, `dequantize` restate the layout in numpy (float64, exact);
* `reference` is the float64 product over the dequantised weights with the decode GEMMs' bound of tests/ref64.py,
  ulp_T(|ref|) + 2^-16 |A| . |W|;
* `emulate32` follows the decode kernel's arithmetic in float32: per block a float32 partial sum of x . (q - z), folded into the
  float32 accumulator as fma(partial, s, acc), one rounding to T.  `bugs` injects slips the bound must catch.
The graph oracle's MatMulNBits (tests/llama_oracle.py) runs on `dequantize`."""
import numpy as np

import oracle as O
from tests import ref64

F32, F16, BF16 = 1, 10, 16


def pack_codes(q):
    """q uint8 [N, K] of nibble values -> B uint8 [N, K / bs, bs / 2] flattened to [N, K / 2] (the same bytes)"""
    q = np.asarray(q, np.uint8)
    return (q[:, 0::2] | (q[:, 1::2] << 4)).astype(np.uint8)


def unpack_codes(b, K, swapped=False):
    """B (any shape with N * K / 2 bytes, column-major by n) -> q uint8 [N, K]"""
    b = np.asarray(b, np.uint8).reshape(-1, K // 2)
    lo, hi = b & 15, b >> 4
    if swapped:
        lo, hi = hi, lo
    q = np.empty((b.shape[0], K), np.uint8)
    q[:, 0::2], q[:, 1::2] = lo, hi
    return q


def pack_zero_points(z):
    """z uint8 [N, K / bs] -> packed uint8 [N * (K / bs) / 2]"""
    z = np.asarray(z, np.uint8)
    return (z[:, 0::2] | (z[:, 1::2] << 4)).astype(np.uint8).reshape(-1)


def unpack_zero_points(zp, N, nblk):
    """packed zero points -> z int [N, nblk]; None -> 8 everywhere"""
    if zp is None:
        return np.full((N, nblk), 8, np.int64)
    b = np.asarray(zp, np.uint8).reshape(N, nblk // 2)
    z = np.empty((N, nblk), np.int64)
    z[:, 0::2], z[:, 1::2] = b & 15, b >> 4
    return z


def dequantize(b, scales, zp, K, N, bs):
    """W [K, N] float64 = (q - z) * s, exact"""
    nblk = K // bs
    q = unpack_codes(b, K).astype(np.int64)
    z = np.repeat(unpack_zero_points(zp, N, nblk), bs, axis=1)
    s = np.repeat(np.asarray(scales, np.float64).reshape(N, nblk), bs, axis=1)
    return ((q - z) * s).T


def reference(x, b, scales, zp, K, N, bs, dt, rounded_weights=False):
    """(ref, bound) for Y = X . W in float64.  rounded_weights: the dequantise-then-GEMM path (more than 64 rows), whose weights are
    T((q - z) * s): the bound is widened by |A| . |W - T(W)|, the error that rounding adds."""
    w = dequantize(b, scales, zp, K, N, bs)
    ref, mag = ref64.product(np.asarray(x, np.float64), w)
    extra = None
    if rounded_weights:
        wt = O.round_to(w.astype(np.float32), dt).astype(np.float64)
        extra = np.abs(np.asarray(x, np.float64)) @ np.abs(w - wt)
        mag = mag + np.abs(np.asarray(x, np.float64)) @ np.abs(wt)
    return ref, ref64.bound(ref, mag, dt, extra)


def violations(got, ref, bound):
    return ~(np.abs(np.asarray(got, np.float64) - ref) <= bound)


def emulate32(x, b, scales, zp, K, N, bs, dt, bugs=()):
    """The decode kernel's arithmetic in float32, rounded to dt.  bugs: 'swapped_nibbles', 'z7', 'neighbour_scale',
    'boundary_16' (the fold 16 k late), 'scale_twice', 'weight_rounded' (W rounded to bf16 before the product)."""
    f = np.float32
    nblk = K // bs
    x = np.asarray(x, np.float32)
    q = unpack_codes(b, K, swapped="swapped_nibbles" in bugs).astype(np.float32)
    z = unpack_zero_points(zp, N, nblk).astype(np.float32)
    if "z7" in bugs:
        z = np.full_like(z, 7.0)
    s = np.asarray(scales, np.float32).reshape(N, nblk)
    if "neighbour_scale" in bugs:
        s = np.roll(s, -1, axis=1)
    wq = (q - np.repeat(z, bs, axis=1)).T  # [K, N], exact small integers
    acc = np.zeros((x.shape[0], N), np.float32)
    if "weight_rounded" in bugs:
        w = O.round_to((wq * np.repeat(s, bs, axis=1).T).astype(np.float32), BF16)
        return O.round_to((x @ w).astype(np.float32), dt)
    shift = 16 if "boundary_16" in bugs else 0
    for blk in range(nblk):
        k0, k1 = max(blk * bs + shift, 0), min((blk + 1) * bs + shift, K)
        part = (x[:, k0:k1] @ wq[k0:k1]).astype(np.float32)
        sc = s[:, blk].astype(np.float64)
        if "scale_twice" in bugs:
            sc = (s[:, blk] * s[:, blk]).astype(np.float32).astype(np.float64)
        acc = (part.astype(np.float64) * sc[None, :] + acc.astype(np.float64)).astype(f)  # one fma: exact in float64, one rounding
    return O.round_to(acc, dt)

