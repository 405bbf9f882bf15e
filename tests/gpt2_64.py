"""Float64 references, per-element bounds and float32 emulations of the GPT-2 forward's other two kernel families: the Linear
layers' GEMM epilogues (`gemm_tc_kernel` through `it_b200_matmul` / `it_b200_matmul_fused`) and LayerNorm (norm.cu).

Linear epilogues.  X [M, K] and W [K, N] are exact in f16 and bf16 (`attn64.exact`), so acc = X.W and S = |X|.|W| are exact
float64 values (computed once per shape at the largest M and sliced).  The kernel forms acc in fp32 (split-K partials summed
in rank order by the cluster's reduce-scatter when the launch splits) and then, in fp32, the epilogue:

    f = acc [rounded to T first with ITB_ACT_ROUND_BEFORE_BIAS] + b     x = rnd_T(f) (Gelu only)
    y = f | relu(f) | gelu(x)          out = rnd_T(y)   or, with a residual r,   out = rnd_T(rnd_T(y) + r)

The reference is that chain without the intermediate roundings: ref = act(acc + b) [+ r].  The bound adds each step's error:

* E0 = 2^-16 S: the fp32 accumulation (tests/ref64.py), split or not (at most 8 partials added in rank order);
* E1 = E0 + 2^-23 (|acc| + |b|) [+ ulp_T(acc)]: the fp32 bias add (2^-24, doubled) [and the rounding before the bias];
* Gelu: x = rnd_T(f) adds ulp_T(f); |Gelu'| <= 1.13 carries E1 + ulp_T(f) through the activation; the fp32 evaluation
  0.5 x (1 + erff(x / sqrt 2)) adds at most 2^-22 (|x| + |y|) + 2^-22 (erff <= 2 ulp of a value below 1, the argument's and the
  sum's roundings, the product's); Relu carries E1 unchanged (|relu'| <= 1);
* out: ulp_T(|ref|) for the final rounding, plus ulp_T(y) for the rounding before the residual add.

Bias values are scaled per column by 2^((n mod 3) - 1) and residuals by 2^((m mod 3) - 1) 2^((n mod 4) - 2), so a bias read
by row, or a residual read from another element, changes values by 2x or more.

LayerNorm.  y = scale (x - mu) / sqrt(var + eps) + bias with mu and var = mean((x - mu)^2) in float64 from the exact x.  The
kernels sum in fp32 along a chain of L additions (`chain_length`: per-thread items, then the shuffle / block trees), so:

* |mu^ - mu| <= dmu = (L + 2) 2^-24 mean|x| (the chain and the division by dim);
* the two-pass variance sums t = x - mu^ (t^2 = (x - mu)^2 - 2 (x - mu) dmu + dmu^2, and sum(x - mu) = 0): var^ lies within
  rho (var + eps) of var + eps with rho = (dmu^2 + (L + 6) 2^-24 (var + dmu^2)) / (var + eps) (the chain, the two roundings
  of t and t^2, the division, the eps add, two to spare);
* rsqrtf is within 2 ulp: rs^ / rs - 1 <= r = 1 / sqrt(1 - rho) - 1 + 5 2^-24;
* y^ = fp32(scale t rs^ + bias): |y^ - y| <= |scale| rs (dmu + |x - mu| (r + 3 2^-24)) (1 + r) + 2^-23 (|bias| + |y|),
  and the output rounding adds ulp_T(|y|) (fp32: 2^(e - 23)).

A one-pass variance E[x^2] - mu^2 loses about L 2^-24 mu^2 / var of var, which rows with |mean| / std = 1e3 (fp32) turn into a
relative error of several percent; the bound allows (L + 2) 2^-24 |mean| / std.
"""
import math

import numpy as np
from scipy.special import erf

from tests import attn64, ref64
from tests.ref64 import BF16, F16, F32

U = 2.0 ** -24
NUM_SMS = 132
GELU_SLOPE = 1.13


def rnd(x, dt):
    """float64 -> T (round to nearest even), as float64"""
    if dt == F32:
        return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)
    from tests.prefill64 import rnd as r
    return r(x, dt)


def gelu(x):
    return 0.5 * x * (1.0 + erf(x / math.sqrt(2.0)))


# ====================================================================== Linear layers
def tc_split(M, K, N):
    """cluster split of a fused gemm_tc launch (batch 1, bias / activation epilogue), as launch_tc_t chooses it:
    (split, rows per reduce-scatter rank, row chunk mpad, row chunks)"""
    mpad = 16
    while mpad < M and mpad < 128:
        mpad *= 2
    chunks = -(-M // mpad)
    tiles_n = -(-N // 128)
    kt = -(-K // 64)
    split = 1
    if kt >= 24 and tiles_n * chunks * 4 <= NUM_SMS:
        split = max(1, min(8, kt // 6, NUM_SMS // (tiles_n * chunks)))
    kps = -(-kt // split)
    split = -(-kt // kps)
    return split, -(-mpad // split), mpad, chunks


class Linear:
    """X [Mmax, K], W [K, N], bias [N], residual [Mmax, N] (float32, exact in f16 and bf16) and the float64 products"""

    def __init__(self, Mmax, K, N, seed):
        rng = np.random.default_rng(seed)
        self.K, self.N = K, N
        self.x = attn64.exact(rng.standard_normal((Mmax, K)) * 0.5 * ref64.row_scale(Mmax)[:, None])
        self.w = attn64.exact(rng.standard_normal((K, N)) * 0.05 * ref64.col_scale(N)[None, :])
        self.bias = attn64.exact(rng.standard_normal(N) * 0.5 * np.exp2((np.arange(N) % 3) - 1.0))
        self.res = attn64.exact(rng.standard_normal((Mmax, N)) * np.exp2((np.arange(Mmax) % 3) - 1.0)[:, None]
                                * np.exp2((np.arange(N) % 4) - 2.0)[None, :])
        self.acc, self.mag = ref64.product(self.x, self.w)


def linear_reference(L, M, act, residual, rb, dt):
    """(ref, bound) [M, N] of act(X W + b) [+ r]; act 0 none, 1 relu, 4 gelu"""
    acc, S, b = L.acc[:M], L.mag[:M], L.bias.astype(np.float64)[None, :]
    f = acc + b
    e = ref64.ACC_SLACK * S + 2 * U * (np.abs(acc) + np.abs(b)) + (ref64.ulp(acc, dt) if rb else 0)
    if act == 4:
        ex = e + ref64.ulp(f, dt)
        y = gelu(f)
        e = GELU_SLOPE * ex + 4 * U * (np.abs(f) + np.abs(y)) + 4 * U
    elif act == 1:
        y = np.maximum(f, 0.0)
    else:
        y = f
    if residual:
        ref = y + L.res[:M].astype(np.float64)
        return ref, e + ref64.ulp(y, dt) + ref64.ulp(ref, dt)
    return y, e + ref64.ulp(y, dt)


def _f(x):
    return np.asarray(x, np.float64).astype(np.float32)


LINEAR_MUTATIONS = ["rs_rows_off_by_one", "bias_by_row"]


def emulate_linear(L, M, act, residual, rb, dt, mutation=None):
    """the split-K reduce-scatter launch in float32: fp32 partials per k-tile of each split, summed in rank order, the
    epilogue of each rank's rows; rows no rank writes stay NaN"""
    K, N = L.K, L.N
    split, rows_per, mpad, chunks = tc_split(M, K, N)
    kt = -(-K // 64)
    kps = -(-kt // split)
    x, w = L.x[:M].astype(np.float64), L.w.astype(np.float64)
    parts = []
    for s in range(split):
        p = np.zeros((M, N), np.float32)
        for t in range(s * kps, min(kt, (s + 1) * kps)):
            p = _f(p + x[:, 64 * t:64 * t + 64] @ w[64 * t:64 * t + 64])
        parts.append(p)
    f = np.zeros((M, N), np.float32)
    for p in parts:
        f = _f(f + p)
    bias = L.bias.astype(np.float32)
    out = np.full((M, N), np.nan, np.float32)
    for c in range(chunks):
        for r in range(split):
            lo = r * rows_per + (1 if mutation == "rs_rows_off_by_one" else 0)
            hi = min(mpad, lo + rows_per)
            rows = np.arange(c * mpad + lo, min(M, c * mpad + hi))
            if not len(rows):
                continue
            v = f[rows]
            if rb:
                v = rnd(v, dt).astype(np.float32)
            if mutation == "bias_by_row":
                bv = np.where(rows < N, bias[np.minimum(rows, N - 1)], 0)[:, None]
            else:
                bv = bias[None, :]
            v = _f(v + bv)
            if act == 4:
                xx = rnd(v, dt)
                v = _f(0.5 * xx * (1.0 + _f(erf(_f(xx * 0.70710678118654752440)))))
            elif act == 1:
                v = np.maximum(v, 0).astype(np.float32)
            if residual:
                v = _f(rnd(v, dt) + L.res[rows])
            out[rows] = rnd(v, dt)
    return out


# ====================================================================== LayerNorm
def rowop_path(dt, dim, inner=1, aligned=True):
    """the launch_rowop branch a LayerNorm takes: "strided", "warp<I>", "vec<CHUNKS>", "block_cached", "block_uncached" """
    if inner != 1:
        return "strided"
    if dim <= 1024:
        if dt != F32 and dim % 8 == 0 and dim >= 64 and aligned:
            return f"vec{1 if dim <= 256 else 2 if dim <= 512 else 3 if dim <= 768 else 4}"
        items = 1 if dim <= 32 else 2 if dim <= 64 else 4 if dim <= 128 else 8 if dim <= 256 else 16 if dim <= 512 else 32
        return f"warp{items}"
    return "block_cached" if dim <= 12288 else "block_uncached"


def block_threads(dim):
    return 1024 if dim >= 8192 else 512


def chain_length(path, dim):
    """the longest chain of fp32 additions in the row sum of one path"""
    if path == "strided":
        return dim
    if path.startswith("vec"):
        return 8 * int(path[3:]) + 5
    if path.startswith("warp"):
        return int(path[4:]) + 5
    return -(-dim // block_threads(dim)) + 10


def ln_rows(rows, dim, dt, seed):
    """x [rows, dim] exact in dt: row r has std 2^((r mod 5) - 2) and |mean| / std cycling over 0, 1, 10, 100 and 1e3 (fp32) /
    100 (f16 / bf16); every 7th row is constant (variance 0)"""
    rng = np.random.default_rng(seed)
    ratios = [0.0, 1.0, 10.0, 100.0, 1e3 if dt == F32 else 100.0]
    sd = np.exp2((np.arange(rows) % 5) - 2.0)
    mu = np.array([ratios[r % 5] * (-1) ** r for r in range(rows)]) * sd
    x = mu[:, None] + sd[:, None] * rng.standard_normal((rows, dim))
    x[::7] = mu[::7, None] + sd[::7, None]
    return rnd(x, dt).astype(np.float32)


def ln_params(dim, size, dt, seed):
    rng = np.random.default_rng(seed)
    n = dim if size == "dim" else 1
    sc = rnd((0.5 + rng.random(n)) * np.exp2((np.arange(n) % 3) - 1.0), dt).astype(np.float32)
    bi = rnd(rng.standard_normal(n) * 0.5 * np.exp2((np.arange(n) % 4) - 2.0), dt).astype(np.float32)
    return sc, bi


def ln_reference(x, sc, bi, eps, dt, L):
    """(ref, bound) [rows, dim] for rows along the last axis"""
    x = x.astype(np.float64)
    sc = np.broadcast_to(sc.astype(np.float64), x.shape[-1:])[None, :]
    bi = np.broadcast_to(bi.astype(np.float64), x.shape[-1:])[None, :]
    mu = x.mean(1, keepdims=True)
    t = x - mu
    var = (t * t).mean(1, keepdims=True)
    rs = 1.0 / np.sqrt(var + eps)
    y = sc * t * rs + bi
    dmu = (L + 2) * U * np.abs(x).mean(1, keepdims=True)
    rho = (dmu * dmu + (L + 6) * U * (var + dmu * dmu)) / (var + eps)
    r = 1.0 / np.sqrt(np.maximum(1.0 - rho, 1e-6)) - 1.0 + 5 * U
    b = np.abs(sc) * rs * (dmu + np.abs(t) * (r + 3 * U)) * (1 + r) + 2 * U * (np.abs(bi) + np.abs(y)) + ref64.ulp(y, dt)
    return y, b


LN_MUTATIONS = ["one_pass_variance", "drop_last_chunk"]


def emulate_ln(x, sc, bi, eps, dt, path, mutation=None):
    """float32 emulation: per-thread sequential sums over the thread's elements, then a pairwise (xor) tree over the threads"""
    rows, dim = x.shape
    xs = x.astype(np.float32).copy()
    n_read = dim - 8 if mutation == "drop_last_chunk" else dim
    xs[:, n_read:] = 0
    thr = 1 if path == "strided" else 32 if not path.startswith("block") else block_threads(dim)
    pad = -(-dim // thr) * thr
    xp = np.zeros((rows, pad), np.float32)
    xp[:, :dim] = xs
    lanes = xp.reshape(rows, -1, thr)  # element d = thread + i * threads

    def tree(v):  # [rows, -1, thr] -> [rows]
        s = np.zeros((rows, thr), np.float32)
        for i in range(v.shape[1]):
            s = _f(s + v[:, i])
        while s.shape[1] > 1:
            h = s.shape[1] // 2
            s = _f(s[:, :h] + s[:, h:])
        return s[:, 0]

    mu = _f(tree(lanes) / np.float32(dim))
    if mutation == "one_pass_variance":
        var = _f(_f(tree(_f(lanes * lanes)) / np.float32(dim)) - _f(mu * mu))
    else:
        t = np.where(np.arange(pad)[None, :] < n_read, _f(xp - mu[:, None]), 0).astype(np.float32)
        var = _f(tree(_f(t * t).reshape(rows, -1, thr)) / np.float32(dim))
    rs = _f(1.0 / np.sqrt(_f(np.maximum(var, 0) + np.float32(eps)).astype(np.float64)))
    scf = np.broadcast_to(sc.astype(np.float32), (dim,))
    bif = np.broadcast_to(bi.astype(np.float32), (dim,))
    y = _f(_f(_f(scf[None, :] * _f(xs - mu[:, None])) * rs[:, None]) + bif[None, :])
    out = rnd(y, dt)
    out[:, n_read:] = np.nan
    return out
