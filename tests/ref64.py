"""Float64 reference for the decode GEMMs, with a per-element error bound.

Inputs are T-rounded float32 arrays, so they are exact in float64.  For C = A . W the reference is `ref = A64 @ W64` and the
magnitude term is `S = |A64| @ |W64|`; a kernel that accumulates in fp32 and rounds once to T must satisfy, element by element,

    |got - ref| <= ulp_T(|ref|) + 2^-16 * S

* ulp_T(x) = 2^(max(e, -126) - 7) for bf16, 2^(max(e, -14) - 10) for fp16 (and 2^(max(e, -126) - 23) for fp32, which
  tests/attn64.py uses), e = floor(log2 |x|).  The one rounding to T is
  at most half an ulp; a sum that crosses a binade while it is rounded can double that, so one whole ulp of |ref| is allowed.
* fp32 accumulation: the kernels add 16-product tensor-core partials into fp32 running sums of at most 11008 / 16 terms per
  split and then add at most 8 split partials.  Even if every one of those additions truncates, the running sums of products with
  random signs stay far below S, and the error stays below about 2^-19 * S.  2^-16 * S leaves at least 8x margin.
* The kernels are deterministic (fixed split order, fixed seeds), so a case that passes once passes every time.

The bound is about 15x tighter than the generic 2^-8 * sqrt(K) * max|a| * max|b| GEMM tolerance at the 4096-wide shapes: it
catches split partials rounded to T before their reduction (a few ulp) and a single lost k16 slice of one fragment.

Rows of X are scaled by 2^((i mod 7) - 3) and columns of W by 2^((j mod 5) - 2) before rounding, so a row or column mix-up in a
fragment or epilogue mapping changes a value by a factor of 2 or more.
"""
import numpy as np

import oracle

F32, F16, BF16 = 1, 10, 16
REF_ROWS = 64  # every shape's reference is computed once at 64 rows; a smaller M uses the first M rows
ACC_SLACK = 2.0 ** -16


def row_scale(m):
    return np.exp2((np.arange(m) % 7) - 3.0).astype(np.float32)


def col_scale(n):
    return np.exp2((np.arange(n) % 5) - 2.0).astype(np.float32)


def activations(m, k, dt, seed, scale=0.5):
    """X [m, k]: standard normal x scale, row i x 2^((i mod 7) - 3), rounded to dt (exact in float64)"""
    x = np.random.default_rng(seed).standard_normal((m, k), dtype=np.float32) * np.float32(scale)
    return oracle.round_to(x * row_scale(m)[:, None], dt)


def weights(k, n, dt, seed, scale=0.05):
    """W [k, n]: standard normal x scale, column j x 2^((j mod 5) - 2), rounded to dt"""
    w = np.random.default_rng(seed).standard_normal((k, n), dtype=np.float32) * np.float32(scale)
    return oracle.round_to(w * col_scale(n)[None, :], dt)


def product(a, w, block=4096):
    """(A64 @ W64, |A64| @ |W64|) in float64, W converted block by block of columns (W may be ~100M elements)"""
    a64 = np.asarray(a, np.float64)
    aa = np.abs(a64)
    m, n = a.shape[0], w.shape[1]
    ref, mag = np.empty((m, n)), np.empty((m, n))
    for j in range(0, n, block):
        wb = np.asarray(w[:, j:j + block], np.float64)
        ref[:, j:j + block] = a64 @ wb
        mag[:, j:j + block] = aa @ np.abs(wb)
    return ref, mag


def ulp(x, dt):
    """ulp of the storage type at |x| (the ulp of its smallest normal below that, as for subnormals)"""
    emin, mant = {BF16: (-126, 7), F16: (-14, 10), F32: (-126, 23)}[dt]
    ax = np.abs(np.asarray(x, np.float64))
    _, ex = np.frexp(ax)                  # ax = f * 2^ex with f in [0.5, 1): floor(log2 ax) = ex - 1
    e = np.where(ax > 0, ex - 1, emin)
    return np.exp2(np.maximum(e, emin) - mant)


def bound(ref, mag, dt, extra=None):
    b = ulp(ref, dt) + ACC_SLACK * mag
    return b if extra is None else b + extra


def violations(got, ref, mag, dt, extra=None):
    """boolean mask of the elements outside the bound"""
    got = np.asarray(got, np.float64)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    return ~(np.abs(got - ref) <= bound(ref, mag, dt, extra))


def assert_within(got, ref, mag, dt, what="", extra=None):
    bad = violations(got, ref, mag, dt, extra)
    if bad.any():
        got64 = np.asarray(got, np.float64)
        idx = np.argwhere(bad)
        i, j = idx[0]
        excess = (np.abs(got64 - ref) / bound(ref, mag, dt, extra))[bad].max()
        raise AssertionError(f"{what}: {bad.sum()} of {bad.size} elements outside |got - ref| <= ulp + 2^-16 S "
                             f"(worst {excess:.3g}x the bound); first at row {i}, col {j}: got {got64[i, j]!r}, "
                             f"ref {ref[i, j]!r}, S {mag[i, j]!r}; rows with errors {sorted(set(idx[:, 0].tolist()))[:16]}")
