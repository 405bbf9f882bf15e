"""Float64 intervals of the RMSNorm and Silu.Mul operands: the values rmsnorm_kernel, silu_mul_kernel and the all-reduce +
residual + RMSNorm kernel may store, given that rinv and silu come from fp32 arithmetic.
rnd (gpt2_64.rnd: prefill64.rnd for f16 / bf16) rounds float64 straight to T; u = 2^-24.

* RMSNorm: xn = rnd(rnd(x rinv) w), rinv = 1 / sqrt(mean(x^2) + fp32(1e-5)).
* Silu.Mul: m = rnd(rnd(silu(g)) u).

Ambiguous roundings.  An element whose exact value lies within the fp32 error window of a T rounding midpoint may round
either way.  As prefill64 does, each path gets a relative window and the element is ambiguous where rnd at the two ends of
the window differ; c_lo / c_hi are the transformed operand at those ends.

* rinv: the sum of squares is a chain of L roundings of a positive sum (relative error <= L u), then the division by K and
  the eps add (1 u each), rsqrtf (<= 2 ulp, 4 u) and the product x * rinv (1 u): |error| <= (L / 2 + 7) u; the window is
  (L + 8) u.  For a kernel that reduces with block_sum (rmsnorm_kernel, allreduce_ll_kernel), L is the items of one thread,
  then two 5-level warp trees: items + 10 (`chain_length("block", ...)`).
* silu(g) = g / (1 + expf(-g)): expf <= 2 ulp (4 u relative to exp(-g)), the add <= 4 u + 1 u relative to 1 + exp(-g), the
  division 1 u: <= 6 u; the window is 8 u.
* The second rounding adds no ambiguity: rnd(x rinv) w and rnd(silu) up are products of two T values, 8 x 8 (bf16) or
  11 x 11 (f16) significant bits, exact in fp32's 24, so rnd of them is rnd of an exact value.
"""
import numpy as np

from tests import ref64
from tests.gpt2_64 import rnd

U = 2.0 ** -24
EPS32 = float(np.float32(1e-5))   # the kernels' 0.00001f
SILU_WINDOW = 8 * U


# ====================================================================== inputs
def norm_weight(k, dt, seed):
    """1 + U(-1/4, 1/4), exact in T"""
    return rnd(1.0 + 0.25 * np.random.default_rng(seed).uniform(-1, 1, k), dt)


def rows(m, k, dt, seed, scale=1.0):
    """[m, k]: standard normal x scale, row i x 2^((i mod 7) - 3) (ref64's row scaling), exact in T"""
    x = np.random.default_rng(seed).standard_normal((m, k)) * scale * ref64.row_scale(m)[:, None]
    return rnd(x, dt)


# ====================================================================== operand transforms and their ambiguity
def chain_length(path, K, nt=0, items=0):
    """longest chain of fp32 additions in the sum of squares: "x_raw" (a phase with no producer), "ss" (the hand-over from the
    previous residual phase's nt tiles) or "block" (rmsnorm_kernel, `items` per thread)"""
    if path == "x_raw":
        return K // 32 + 5
    if path == "ss":
        return 12 + -(-nt // 8)
    return items + 10


def rms_window(L):
    return (L + 8) * U


class Operand:
    """a GEMM operand: nominal value a; for a transformed one, the values c_lo / c_hi at the two ends of the fp32 window, and
    amb = |c_hi - c_lo| (0 where the rounding is not ambiguous)"""

    def __init__(self, a, lo=None, hi=None):
        self.a = np.asarray(a, np.float64)
        self.lo = self.a if lo is None else lo
        self.hi = self.a if hi is None else hi
        self.amb = np.abs(self.hi - self.lo)
        self.n_amb = int((self.amb > 0).sum())

    @property
    def share(self):
        return self.n_amb / max(self.a.size, 1)

    def outside(self, got):
        """elements of a kernel's transformed operand outside [min(c_lo, c_hi), max(c_lo, c_hi)]"""
        got = np.asarray(got, np.float64)
        return ~((got >= np.minimum(self.lo, self.hi)) & (got <= np.maximum(self.lo, self.hi)))


def _two_sided(y, window, tail, dt):
    """Operand tail(rnd(y)) when y carries a relative error up to `window`"""
    return Operand(tail(rnd(y, dt)), tail(rnd(y * (1 - window), dt)), tail(rnd(y * (1 + window), dt)))


def rinv64(x):
    x = np.asarray(x, np.float64)
    return 1.0 / np.sqrt((x * x).mean(1, keepdims=True) + EPS32)


def rmsnorm_operand(x, w, dt, L):
    """xn = rnd(rnd(x rinv) w) with rinv's window for a chain of L roundings"""
    x, w = np.asarray(x, np.float64), np.asarray(w, np.float64)
    return _two_sided(x * rinv64(x), rms_window(L), lambda r: rnd(r * w[None, :], dt), dt)


def silu64(g):
    g = np.asarray(g, np.float64)
    return g / (1.0 + np.exp(-g))


def silu_mul_operand(g, u, dt):
    """m = rnd(rnd(silu(g)) u)"""
    u = np.asarray(u, np.float64)
    return _two_sided(silu64(g), SILU_WINDOW, lambda r: rnd(r * u, dt), dt)


# ====================================================================== fp32 reductions
def _f(x):
    return np.asarray(x, np.float64).astype(np.float32)


def _xor_tree(v, levels):
    """lane 0 of a __shfl_xor_sync butterfly over the last axis (2^levels lanes)"""
    v = np.asarray(v, np.float32)
    n = v.shape[-1]
    o = n // 2
    while o:
        v = _f(v + v[..., np.arange(n) ^ o])
        o //= 2
    return v[..., 0]
