"""RoPE with an inv_freq table against float64, and a float32 emulation of the kernels' rule.

The kernels (rope_freq_kernel, and the RoPE folded into decode attention) rotate column pair c of every head by the angle
a = fp32(p * inv_freq[c]) -- one float32 product, exactly what numpy's float32 multiply gives -- take cosf(a) / sinf(a),
round them to the activation type T, and then round each product and the sum to T.  The reference here takes cos / sin of
the same angle in float64.  cosf / sinf are within 2 ulp of the true value (CUDA Programming Guide, single-precision
mathematical functions), so a cos / sin whose float64 value lies that close to a rounding point of T may come out as either
neighbour: every output element must lie between the results of the two candidates (equal to the nominal result where
there is only one)."""
import numpy as np

import oracle as O

F32, F16, BF16 = 1, 10, 16
TRIG_ULPS = 2  # cosf / sinf maximum error, ulp of the float32 result


def angles(pos, inv_freq, half):
    """fp32(p * inv_freq[c]) for every position (flattened) and column pair: [rows, half]"""
    p = np.asarray(pos).astype(np.int64).ravel().astype(np.int32).astype(np.float32)
    return p[:, None] * np.asarray(inv_freq, np.float32)[None, :half]


def _rotate(x, cs, sn, dim_head, dt):
    """the kernels' arithmetic in T on float32 x [rows, dim_model] with cos / sin [rows, half] already in T"""
    rows, dm = x.shape
    half = dim_head // 2
    xh = x.reshape(rows, dm // dim_head, dim_head)
    lo, hi = xh[..., :half], xh[..., half:]
    cs, sn = cs[:, None, :], sn[:, None, :]
    r = lambda a: O.round_to(np.ascontiguousarray(a, np.float32), dt)
    return np.concatenate([r(r(lo * cs) - r(hi * sn)), r(r(hi * cs) + r(lo * sn))], axis=-1).reshape(rows, dm)


class Bound:
    """The float64 reference of RoPE with a table on x [rows, dim_model] (values exact in T): `nominal` (cos / sin of the
    fp32 angle in float64, rounded to T) and per element the interval [lo, hi] that cosf / sinf's error allows"""

    def __init__(self, pos, x, inv_freq, dim_head, dt):
        x = np.asarray(x, np.float32)
        self.x = x.reshape(-1, x.shape[-1])
        a = angles(pos, inv_freq, dim_head // 2).astype(np.float64)
        c64, s64 = np.cos(a), np.sin(a)
        rnd = lambda v: O.round_to(v.astype(np.float32), dt)
        self.nominal = _rotate(self.x, rnd(c64), rnd(s64), dim_head, dt)

        def window(v):
            u = np.spacing(np.abs(v).astype(np.float32)).astype(np.float64) * (TRIG_ULPS + 1)
            return rnd(v - u), rnd(v + u)
        (clo, chi), (slo, shi) = window(c64), window(s64)
        corners = [_rotate(self.x, c, s, dim_head, dt) for c in (clo, chi) for s in (slo, shi)]
        self.lo, self.hi = np.minimum.reduce(corners), np.maximum.reduce(corners)
        self.share = float(np.mean(self.lo != self.hi))  # elements with two candidates

    def outside(self, got):
        got = np.asarray(got, np.float32).reshape(self.x.shape)
        return ~((got >= self.lo) & (got <= self.hi))


def base_table(dim_head):
    """the kernels' base-10000 rule, 10000^(-2c / dim_head) in float32"""
    c = np.arange(dim_head // 2, dtype=np.float32)
    return np.power(np.float32(10000.0), -(c * np.float32(2)) / np.float32(dim_head)).astype(np.float32)


def emulate(pos, x, inv_freq, dim_head, dt, slip=None):
    """the kernels' rule in float32 numpy (cos / sin of the fp32 angle via float64, rounded to float32 as a correctly
    rounded cosf would); `slip` injects one mistake: "base10000" (the table ignored), "column+1" (inv_freq read one column
    late), "angle64" (the angle formed in float64)"""
    x = np.asarray(x, np.float32).reshape(-1, np.shape(x)[-1])
    half = dim_head // 2
    table = np.asarray(inv_freq, np.float32)
    if slip == "base10000":
        table = base_table(dim_head)
    elif slip == "column+1":
        table = np.concatenate([table[1:half], table[half - 1:half]])
    if slip == "angle64":
        p = np.asarray(pos).astype(np.int64).ravel().astype(np.float64)
        a = p[:, None] * table[None, :half].astype(np.float64)
    else:
        a = angles(pos, table, half).astype(np.float64)
    rnd = lambda v: O.round_to(v.astype(np.float32), dt)
    return _rotate(x, rnd(np.cos(a)), rnd(np.sin(a)), dim_head, dt)


POSITIONS = np.array([0, 1, 2, 3, 7, 100, 2047, 2048, 4095, 8191, 8192, 8193, 16383, 32767, 65535, 100000, 130000, 131000,
                      131070, 131071], np.int64)


def case(D, dt, heads=4, seed=0):
    """(positions [rows], x [rows, heads * D] exact in T): POSITIONS plus a spread up to 131071"""
    rng = np.random.default_rng([seed, D, dt])
    pos = np.concatenate([POSITIONS, rng.integers(0, 131072, 44)])
    x = O.round_to((rng.standard_normal((pos.size, heads * D)) * 2.0).astype(np.float32), dt)
    return pos, x
