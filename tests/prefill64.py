"""Float64 reference, per-element bound, input construction and float32 emulation of `attention_prefill_kernel`
(attention_prefill.cu), the fused prefill attention of the GPT-2 forward.

Reference.  The kernel promises the graph's rounding points, so the reference is that operator chain evaluated in float64
from the exact inputs (q, k, v and the mask are exact in T, hence in float64), with rnd_T rounding float64 straight to T
(`rnd`; `oracle.round_to` goes through float32 and can round twice):

    s1 = rnd_T(q.k)   s2 = rnd_T(s1 / c) | rnd_T(s1 * c) | s1   s3 = rnd_T(s2 + mask) | s2
    P_j = rnd_T(exp(s3_j - max s3) / sum exp(s3 - max s3))     ref = sum_j P_j v_j     (out = rnd_T of the fp32 sum)

A row whose every s3 is -inf (every key masked, or f16 sums that all overflow) is written as 0 by the kernel; the unfused
Softmax writes NaN there.  The reference is 0 for such rows and the tests require exact zeros.

Ambiguous roundings.  The kernel's intermediate values come from fp32 arithmetic, so a value within the fp32 error window
of a T rounding midpoint may round either way:

* q.k comes from D / 16 chained wgmma k16 steps into an fp32 accumulator.  Counting each step as 2 units of roundoff
  (truncation allowed, as tests/ref64.py does) gives |acc - q.k| <= e_j with e_j = C_QK 2^-24 sum_i |q_i k_ji|,
  C_QK = D / 8 (8 for D = 64, 16 for D = 128).
* s1 / c (a scale that is not a power of two) and s2 + mask are each one correctly rounded fp32 operation before the
  rounding to T: a window of 2^-24 of the result (none where the exact sum is a float32 value: the fp32 sum is then exact,
  and a tie rounds to even on both sides).  s1 * c is exact in fp32 (two 11-bit significands), and so is a division by
  a power of two, which the kernel performs as that multiplication.
* Every step is monotone, so the chain evaluated at both ends of the windows gives the lowest and highest s3 the kernel can
  produce; where they differ, the score is ambiguous, Delta_j = s3_hi - s3_lo.
* P_j = rnd_T(expf(s3_j - m) * (1 / l)) in fp32.  Its relative error before the rounding is at most
      2^-24 (|s3_j - m| + 6) + c_l + eps_row,
  |s3_j - m| 2^-24 for the fp32 subtraction, 4 (expf, <= 2 ulp), 1 (1 / l) and 1 (the product).  c_l bounds l's relative
  error: l is a sum of positive terms, so its relative error is at most the largest of the terms' (weighted), plus the
  roundings of the running sum: every term carries its own subtraction error and those of the rescales it passes through,
  whose maxima telescope to at most |s_i - m| twice more (3 2^-24 sum_i p_i |s_i - m| in all), 4 2^-24 for each expf on
  its path (its own, one rescale per 16-column chunk of its part, the part merge: 4 (2 + nch), where nch = 2 x the number
  of key tiles is the number of 16-column chunks one part sees), and one rounding per addition on the longest path (16 in
  a chunk, 2 per chunk for the rescale, 4 in the merge, and 4 to spare: 2 nch + 24).  eps_row = sum over the row's ambiguous scores of |exp(s3_hi - m) - exp(s3_lo - m)| / L, the shift of l that
  an ambiguous score can cause.  Where rnd_T at the two ends of that window differ (or the score itself is ambiguous), P_j
  is ambiguous.

Bound, element by element (L = sum exp(s3 - m), d_j = (exp(s3_hi,j - m) - exp(s3_lo,j - m)) / L):

    |got - ref| <= ulp_T(|ref|) + 2^-16 sum_j P_j |v_j| + sum_{ambiguous s_j} d_j |v_j - ref| / (1 - eps_row)
                   + sum_{ambiguous P_j} ulp_T(P_j) |v_j|

* ulp_T(|ref|): the output is rounded to T once (half an ulp, doubled for a rounding that crosses a binade).
* 2^-16 sum P|v|: O = P.V accumulates fp32 over at most 2048 / 16 = 128 wgmma k16 steps, 2 units of roundoff each (as
  tests/ref64.py counts them): 256 2^-24 = 2^-16 of sum P|v| even if every one errs the same way.
* d_j |v_j - ref| / (1 - eps_row): an ambiguous score moves its weight by d_j and, through l, every other weight by the
  same relative amount the other way; to first order that moves the output by d_j (v_j - ref), and 1 / (1 - eps_row) covers
  the second order (p = d_j P_j (e^Delta - 1) for Delta = s3_hi - s3_lo).
* ulp_T(P_j) |v_j|: an ambiguous P_j is one ulp of P away from the reference's.
* The two ambiguity terms are what a flipped rounding costs, no more: a kernel that takes the other side of every
  ambiguous rounding meets them exactly.  They are counted twice (AMB_MARGIN), so that an emulation that flips some of
  them can still be held to half of the bound, as the other terms are; ambiguous values are rare (the tests assert <= 1 %
  of the scores), so this costs the bound nothing elsewhere.

The float32 emulation below follows the kernel's order of operations (the four 32-column parts of every key tile, the
16-column chunks with an online (m, l) per part, the merge of the parts, P = rnd_T(expf(s - m) * (1 / l)), O += P V in
fp32 per k16 step) and stays within half of the bound on cases that carry every score regime (0.49 - 0.5: the output's
own rounding, half an ulp, is what comes closest, so the margin of 2 holds for everything but that rounding).
"""
import math

import numpy as np

from tests import attn64, ref64
from tests.ref64 import BF16, F16, ulp

NAMES = {F16: "f16", BF16: "bf16"}
U = 2.0 ** -24
BQ = BK = 128
PARTS, PCOLS = 4, 32
AMB_MARGIN = 2.0  # the ambiguity terms count twice (see the module docstring)
_FMT = {F16: (-14, 10, 15), BF16: (-126, 7, 127)}  # (emin, mantissa bits, emax)


def c_qk(D):
    return D / 8.0


# ====================================================================== float64 -> T rounding
def rnd(x, dt):
    """float64 -> the nearest value of T (round to nearest even), as float64; overflow to +-inf, NaN and +-inf kept.  Rounds
    once, straight from float64 (oracle.round_to rounds through float32)."""
    emin, mant, emax = _FMT[dt]
    x = np.asarray(x, np.float64)
    ax = np.abs(x)
    fin = np.isfinite(x) & (ax > 0)
    safe = np.where(fin, ax, 1.0)
    _, ex = np.frexp(safe)
    q = np.exp2(np.maximum(ex - 1, emin) - mant)
    r = np.round(np.where(fin, x, 0.0) / q) * q
    r = np.where(np.abs(r) >= 2.0 ** (emax + 1), np.copysign(np.inf, x), r)
    return np.where(fin, r, x)


BIG_NEG = {F16: -65504.0, BF16: float(rnd(-3.0e38, BF16))}  # the frontend's mask values as stored in T


# ====================================================================== inputs
REGIMES = ["flat", "late", "early", "sink", "diag", "past_diag", "neg150", "pos200", "part3"]


def _column_targets(regime, Skv, rng):
    """target score (after scaling) per key, or None where the key keeps the flat random score"""
    t = np.full(Skv, np.nan)
    if Skv == 0:
        return t
    peaks = sorted({min(Skv - 1, int(round(f * (Skv - 1)))) for f in (0.1, 0.35, 0.6, 0.85)})
    if regime == "late":
        t[peaks] = 6.0 + 3.0 * np.arange(len(peaks))
    elif regime == "early":
        t[peaks] = 15.0 - 3.0 * np.arange(len(peaks))
    elif regime == "sink":
        t[0] = 20.0
    elif regime == "neg150":
        t[:] = -150.0 + 3.0 * rng.standard_normal(Skv)
    elif regime == "pos200":  # a tent peaking at +200 two thirds of the way in
        top = (2 * (Skv - 1)) // 3
        t[:] = 200.0 - np.abs(np.arange(Skv) - top)
    elif regime == "part3":
        # the maximum in the last key tile's column part 3 (or on the last key when that tile has no part 3), far smaller
        # scores everywhere else.  Under a causal mask only the query rows that see that key -- the last one when Skv = Sq --
        # carry the part-3 maximum; the other rows' maxima fall in earlier parts
        last0 = ((Skv - 1) // BK) * BK
        cols = [j for j in range(last0, Skv) if (j % BK) // PCOLS == PARTS - 1]
        t[:] = -30.0
        t[cols[-1] if cols else Skv - 1] = 40.0
    return t


class Case:
    """One prefill attention problem: q [B, H, Sq, D], k, v [B, H, Skv, D] (float32, exact in f16 and bf16).  Score regimes
    cycle over the heads from `offset`; v row j is scaled by 2^((j mod 5) - 2) and head h by 2^((h mod 3) - 1).

    mask: None | "causal" (offset Skv - Sq, [1, 1, Sq, Skv]) | "causal_inf" (the same with -inf) | "pad" ([B, 1, 1, Skv]: the
    last 3 b + 1 keys of batch row b masked) | "batch" ([B, 1, Sq, Skv]: causal + a per-batch bias) | "head" ([B, H, Sq, Skv]:
    causal + a per-head bias) | "head_misaligned" (the same, heads stored Sq Skv + 4 elements apart) | "transposed" (causal,
    stored [Skv, Sq] and read with mi = 1, mj = Sq) | "full" (causal + rows masked with -inf everywhere, and for f16
    every key of some neg150 rows at -65504, whose sums all overflow).
    scale: None | ("div", c) | ("mul", c), c rounded to T."""

    def __init__(self, B, H, Sq, Skv, D, mask=None, scale=("div", None), seed=0, offset=0):
        self.B, self.H, self.Sq, self.Skv, self.D = B, H, Sq, Skv, D
        self.mask_kind, self.offset = mask, offset
        if scale is not None and scale[1] is None:
            scale = (scale[0], math.sqrt(D) if scale[0] == "div" else 1.0 / math.sqrt(D))
        self.scale = scale
        rng = np.random.default_rng(seed)
        self.q = np.empty((B, H, Sq, D), np.float32)
        self.k = np.empty((B, H, Skv, D), np.float32)
        self.v = np.empty((B, H, Skv, D), np.float32)
        self.regime = np.empty((B, H), object)
        ceff = 1.0 if scale is None else (scale[1] if scale[0] == "div" else 1.0 / scale[1])  # raw score = target * ceff
        vrow = np.exp2((np.arange(Skv) % 5) - 2.0)
        for b in range(B):
            for h in range(H):
                reg = REGIMES[(b * H + h + offset) % len(REGIMES)]
                self.regime[b, h] = reg
                q = np.zeros((Sq, D))
                k = np.zeros((Skv, D))
                # dims [0, D - 1): the flat part, s_i g_j sum_d u_id w_jd with u, w uniform in [0.5, 1.5], s_i = +-1 and
                # g_j ~ N(0, 1): every product of one score has the same sign, so sum |q k| = |q.k| and the fp32 window of
                # a score stays a few units of its own roundoff (random signs would make it ~ sqrt(D) times that)
                # (scaled score std about 1); dim D - 1 carries the targets
                nz = D - 1
                sig = math.sqrt(ceff / nz)
                q[:, :nz] = rng.uniform(0.5, 1.5, (Sq, nz)) * sig * rng.choice([-1.0, 1.0], (Sq, 1))
                k[:, :nz] = rng.uniform(0.5, 1.5, (Skv, nz)) * sig * rng.standard_normal((Skv, 1))
                alpha = 4.0
                q[:, D - 1] = alpha
                t = _column_targets(reg, Skv, rng)
                k[:, D - 1] = np.where(np.isnan(t), 0.0, t) * ceff / alpha
                if reg in ("diag", "past_diag"):
                    # a ramp over the keys: under the causal mask a query's largest visible score is on its diagonal, and
                    # with the steeper ramp the keys just past it, which the mask removes, are larger still
                    slope = 1.0 if reg == "diag" else 2.0
                    k[:, D - 1] = (slope * (np.arange(Skv) - (Skv - 1)) + 20.0) * ceff / alpha
                self.q[b, h] = attn64.exact(q)
                self.k[b, h] = attn64.exact(k)
                v = rng.standard_normal((Skv, D)) * 0.5 * vrow[:, None] * 2.0 ** ((h % 3) - 1)
                self.v[b, h] = attn64.exact(v)
        self._rng = rng
        self._mask_cache = {}
        self._prod = None

    # ------------------------------------------------------------------ the mask as stored and as read
    def mask(self, dt):
        """(storage float32 array or None, (mb, mh, mi, mj), element offset of the mask base, logical [B|1, H|1, Sq, Skv])"""
        if dt in self._mask_cache:
            return self._mask_cache[dt]
        B, H, Sq, Skv, kind = self.B, self.H, self.Sq, self.Skv, self.mask_kind
        r = None
        if kind is None:
            r = (None, (0, 0, 0, 0), 0, None)
        else:
            neg = -np.inf if kind == "causal_inf" else BIG_NEG[dt]
            causal = np.triu(np.full((Sq, Skv), neg, np.float32), 1 + Skv - Sq) if Sq and Skv else np.zeros((Sq, Skv), np.float32)
            rng = np.random.default_rng(7 + Sq + Skv)
            if kind in ("causal", "causal_inf"):
                r = (causal, (0, 0, Skv, 1), 0, causal[None, None])
            elif kind == "pad":
                m = np.zeros((B, 1, 1, Skv), np.float32)
                for b in range(B):
                    m[b, 0, 0, Skv - min(Skv, 3 * b + 1):] = neg
                r = (m, (Skv, 0, 0, 1), 0, m)
            elif kind == "batch":
                m = causal[None, None] + attn64.exact(rng.standard_normal((B, 1, Sq, Skv)))
                m = np.where(np.isfinite(causal)[None, None] & (causal[None, None] == 0), m, causal[None, None]).astype(np.float32)
                r = (m, (Sq * Skv, 0, Skv, 1), 0, m)
            elif kind in ("head", "head_misaligned", "full"):
                m = causal[None, None] + attn64.exact(rng.standard_normal((B, H, Sq, Skv)))
                m = np.where(causal[None, None] == 0, m, causal[None, None]).astype(np.float32)
                if kind == "full":
                    m[:, :, ::7] = -np.inf                         # every key of every 7th query row
                    if dt == F16:
                        for b in range(B):
                            for h in range(H):
                                if self.regime[b, h] == "neg150":
                                    m[b, h, 3::7] = BIG_NEG[F16]   # -65504 + (about -150): all overflow to -inf
                if kind == "head_misaligned":
                    pitch = Sq * Skv + 4  # odd heads start 8 bytes past a 16-byte boundary: their rows take the scalar path
                    store = np.zeros(B * H * pitch, np.float32)
                    for b in range(B):
                        for h in range(H):
                            o = (b * H + h) * pitch
                            store[o:o + Sq * Skv] = m[b, h].ravel()
                    r = (store, (H * pitch, pitch, Skv, 1), 0, m)
                else:
                    r = (m, (H * Sq * Skv, Sq * Skv, Skv, 1), 0, m)
            elif kind == "transposed":
                st = np.ascontiguousarray(causal.T)
                r = (st, (0, 0, 1, Sq), 0, causal[None, None])
            else:
                raise ValueError(kind)
        store = r[0]
        if store is not None:
            assert np.array_equal(rnd(store.astype(np.float64), dt), store.astype(np.float64), equal_nan=True), \
                "mask values must be exact in T"
        self._mask_cache[dt] = r
        return r

    def scale_value(self, dt):
        return None if self.scale is None else float(rnd(self.scale[1], dt))

    # ------------------------------------------------------------------ float64 products, shared by both types
    def products(self):
        if self._prod is None:
            x = np.empty((self.B, self.H, self.Sq, self.Skv))
            a = np.empty_like(x)
            for b in range(self.B):
                for h in range(self.H):
                    q, k = self.q[b, h].astype(np.float64), self.k[b, h].astype(np.float64)
                    x[b, h] = q @ k.T
                    a[b, h] = np.abs(q) @ np.abs(k).T
            self._prod = (x, a)
        return self._prod

    def head_mask(self, dt, b, h):
        lg = self.mask(dt)[3]
        if lg is None:
            return None
        return lg[b if lg.shape[0] > 1 else 0, h if lg.shape[1] > 1 else 0].astype(np.float64)


# ====================================================================== the chain, its windows and the bound
def score_chain(x, a, mask, scale, dt, D, wide):
    """s3 from the float64 product x (wide = 0), or the lowest / highest value the kernel can produce (wide = -1 / +1)"""
    with np.errstate(invalid="ignore", over="ignore"):
        s = rnd(x + wide * c_qk(D) * U * a, dt)
        if scale is not None:
            mode, c = scale
            c = float(rnd(c, dt))
            cm = c if mode == "mul" else 1.0 / c
            pow2 = mode == "div" and math.frexp(c)[0] == 0.5
            if mode == "mul" or pow2:
                s = rnd(s * cm, dt)  # exact in fp32
            else:
                y = s / c
                s = rnd(y + wide * U * np.where(np.isfinite(y), np.abs(y), 0.0), dt)
        if mask is not None:
            y = s + mask  # exact in float64; the fp32 sum is exact too wherever y is a float32 value
            inexact = np.isfinite(y) & (y.astype(np.float32).astype(np.float64) != y)
            s = rnd(y + wide * U * np.where(inexact, np.abs(y), 0.0), dt)
    return s


class HeadRef:
    """reference, bound and ambiguity shares of one head: every array [Sq, D] or [Sq]"""

    def __init__(self, x, a, mask, v, scale, dt, D, Skv):
        Sq = x.shape[0]
        v = v.astype(np.float64)
        av = np.abs(v)
        self.dead = np.ones(Sq, bool)
        self.ref = np.zeros((Sq, D))
        self.bound = np.zeros((Sq, D))
        self.n_scores = self.n_amb_s = self.n_p = self.n_amb_p = 0
        if Skv == 0 or Sq == 0:
            return
        s3 = score_chain(x, a, mask, scale, dt, D, 0)
        lo = score_chain(x, a, mask, scale, dt, D, -1)
        hi = score_chain(x, a, mask, scale, dt, D, +1)
        m = s3.max(1)
        live = m > -np.inf
        self.dead = ~live
        if not live.any():
            return
        s3, lo, hi, m = s3[live], lo[live], hi[live], m[live][:, None]
        with np.errstate(invalid="ignore", over="ignore"):
            E = np.exp(s3 - m)
            L = E.sum(1, keepdims=True)
            p = E / L
            P = rnd(p, dt)
            amb_s = lo != hi
            d = np.where(amb_s, (np.exp(hi - m) - np.exp(lo - m)) / L, 0.0)
            eps_row = d.sum(1, keepdims=True)
            nch = 2 * (-(-Skv // BK))
            dist = np.where(np.isfinite(s3), np.abs(s3 - m), 0.0)
            c_l = U * (3.0 * (p * dist).sum(1, keepdims=True) + 4.0 * (2 + nch) + 2.0 * nch + 24.0)
            w = U * (dist + 6.0) + c_l + eps_row
            amb_p = (rnd(p * (1 - w), dt) != rnd(p * (1 + w), dt)) | amb_s
        ref = P @ v
        b = ulp(ref, dt) + ref64.ACC_SLACK * (P @ av)
        pe = np.where(amb_p, ulp(np.maximum(P, rnd(p * (1 + w), dt)), dt), 0.0)
        amb = pe @ av
        ii, jj = np.nonzero(amb_s)
        if len(ii):
            st = np.zeros_like(ref)
            np.add.at(st, ii, d[ii, jj, None] * np.abs(v[jj] - ref[ii]))
            amb += st / np.maximum(1.0 - eps_row, 0.5)
        b += AMB_MARGIN * amb
        self.ref[live], self.bound[live] = ref, b
        finite = np.isfinite(s3)
        self.n_scores, self.n_amb_s = int(finite.sum()), int((amb_s & finite).sum())
        self.n_p, self.n_amb_p = int((P > 0).sum()), int((amb_p & (P > 0)).sum())


class Reference:
    """float64 reference of a case in one type: ref, bound [B, H, Sq, D], dead rows [B, H, Sq], ambiguity counts"""

    def __init__(self, case, dt):
        B, H, Sq, Skv, D = case.B, case.H, case.Sq, case.Skv, case.D
        self.ref = np.zeros((B, H, Sq, D))
        self.bound = np.zeros((B, H, Sq, D))
        self.dead = np.ones((B, H, Sq), bool)
        cnt = np.zeros(4, np.int64)
        if Sq and Skv:
            x, a = case.products()
        for b in range(B):
            for h in range(H):
                if not (Sq and Skv):
                    continue
                r = HeadRef(x[b, h], a[b, h], case.head_mask(dt, b, h), case.v[b, h], case.scale, dt, D, Skv)
                self.ref[b, h], self.bound[b, h], self.dead[b, h] = r.ref, r.bound, r.dead
                cnt += [r.n_scores, r.n_amb_s, r.n_p, r.n_amb_p]
        self.n_scores, self.n_amb_s, self.n_p, self.n_amb_p = (int(c) for c in cnt)

    def share_s(self):
        return self.n_amb_s / max(self.n_scores, 1)

    def share_p(self):
        return self.n_amb_p / max(self.n_p, 1)

    def violations(self, got, scale=1.0):
        """[B, H, Sq, D] mask of elements outside scale x the bound; dead rows must be exactly 0; NaN is outside"""
        got = np.asarray(got, np.float64)
        bad = ~(np.abs(got - self.ref) <= scale * self.bound)
        return bad | (self.dead[..., None] & (got != 0))

    def ratio(self, got):
        got = np.asarray(got, np.float64)
        with np.errstate(invalid="ignore", divide="ignore"):
            r = np.abs(got - self.ref) / self.bound
        r = np.where(self.dead[..., None], np.where(got == 0, 0.0, np.inf), r)
        return float(np.nanmax(np.where(np.isnan(got), np.inf, r))) if r.size else 0.0


def report(bad, got, R, what, limit=4):
    if not bad.any():
        return None
    lines = [f"{what}: {int(bad.sum())} of {bad.size} elements outside the bound"]
    rows = sorted({(int(b), int(h), int(i)) for b, h, i, _ in np.argwhere(bad)})
    for b, h, i in rows[:limit]:
        with np.errstate(invalid="ignore", divide="ignore"):
            e = np.where(bad[b, h, i], np.abs(got[b, h, i] - R.ref[b, h, i]) / np.maximum(R.bound[b, h, i], 1e-300), -1)
        d = int(np.nanargmax(np.where(np.isnan(e), np.inf, e)))
        mx = "dead row (all keys masked)" if R.dead[b, h, i] else ""
        lines.append(f"  (b {b}, h {h}, query row {i}): query tile {i // BQ}, head column {d} {mx}: got {float(got[b, h, i, d])!r}, "
                     f"float64 {R.ref[b, h, i, d]!r}, bound {R.bound[b, h, i, d]:.3g}")
    if len(rows) > limit:
        lines.append(f"  ... {len(rows)} rows in all: {rows[:16]}")
    return "\n".join(lines)


def where_max(case, dt, b, h, i):
    """(key tile, column part) of the largest s3 of query row i of head (b, h), for failure messages"""
    x, a = case.products()
    s3 = score_chain(x[b, h, i], a[b, h, i], None if case.head_mask(dt, b, h) is None else case.head_mask(dt, b, h)[i],
                     case.scale, dt, case.D, 0)
    j = int(np.argmax(s3))
    return j // BK, (j % BK) // PCOLS


# ====================================================================== float32 emulation of the kernel
def _f(x):
    return np.asarray(x, np.float64).astype(np.float32)


def _exp(x):
    with np.errstate(invalid="ignore", over="ignore"):
        return np.exp(np.asarray(x, np.float64)).astype(np.float32)


def _r32(x, dt):
    return rnd(np.asarray(x, np.float64), dt).astype(np.float32)


MUTATIONS = ["mask_shift_plus1", "mask_shift_minus1", "skip_last_tile_b", "part_l", "merge_no_rescale", "no_online_rescale",
             "p_unrounded", "p_rounded_twice", "s_unrounded", "mask_transposed", "stale_k"]


def emulate_head(q, k, v, mask, scale, dt, mutation=None, trace=None):
    """the kernel's output [Sq, D] (float32) for one head; mask [Sq, Skv] float64 (logical) or None.  trace: a dict that
    receives the emulated s3 and P, [Sq, Skv] each"""
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        return _emulate_head(q, k, v, mask, scale, dt, mutation, trace)


def _emulate_head(q, k, v, mask, scale, dt, mutation, trace):
    Sq, D = q.shape
    Skv = k.shape[0]
    out = np.zeros((Sq, D), np.float32)
    if Skv == 0:
        return out
    ntiles = -(-Skv // BK)
    if mask is not None and mutation in ("mask_shift_plus1", "mask_shift_minus1", "mask_transposed"):
        mm = np.zeros_like(mask)
        if mutation == "mask_transposed":
            n, c = min(Sq, Skv), mask
            mm[:n, :n] = c[:n, :n].T
        else:
            sft = 1 if mutation == "mask_shift_plus1" else -1
            src = np.arange(Skv) + sft
            ok = (src >= 0) & (src < Skv)
            mm[:, ok] = mask[:, src[ok]]
        mask = mm
    q32, k32 = q.astype(np.float64), k.astype(np.float64)

    def scores(kt):  # s3 of key tile kt's columns, [Sq, <= 128]
        j0, j1 = kt * BK, min(Skv, kt * BK + BK)
        acc = np.zeros((Sq, j1 - j0), np.float32)
        for kk in range(D // 16):
            sl = slice(16 * kk, 16 * kk + 16)
            acc = _f(acc + q32[:, sl] @ k32[j0:j1, sl].T)
        s = acc if mutation == "s_unrounded" else _r32(acc, dt)
        if scale is not None:
            mode, c = scale
            c = np.float32(rnd(c, dt))
            pow2 = mode == "div" and math.frexp(float(c))[0] == 0.5
            if mode == "mul":
                s = _r32(_f(s * c), dt)
            elif pow2:
                s = _r32(_f(s * np.float32(1.0 / c)), dt)
            else:
                s = _r32(_f(s.astype(np.float32) / c), dt)
        if mask is not None:
            s = _r32(_f(s + mask[:, j0:j1].astype(np.float32)), dt)
        return s.astype(np.float32)

    S = [scores(t) for t in range(ntiles)]
    # pass A: online (m, l) per column part over 16-column chunks
    m = np.full((PARTS, Sq), -np.inf, np.float32)
    l = np.zeros((PARTS, Sq), np.float32)
    for t in range(ntiles):
        for p in range(PARTS):
            for c0 in (p * PCOLS, p * PCOLS + 16):
                sv = np.full((Sq, 16), -np.inf, np.float32)
                n = max(0, min(16, S[t].shape[1] - c0))
                if n:
                    sv[:, :n] = S[t][:, c0:c0 + n]
                mx = np.maximum(m[p], sv.max(1))
                upd = mx > -np.inf
                add = np.zeros(Sq, np.float32)
                for j in range(16):
                    add = _f(add + _exp(_f(sv[:, j] - mx)))
                corr = np.ones(Sq, np.float32) if mutation == "no_online_rescale" else _exp(_f(m[p] - mx))
                corr = np.where(m[p] > -np.inf, corr, 0).astype(np.float32)
                lnew = _f(l[p].astype(np.float64) * corr + add)  # fmaf
                l[p] = np.where(upd, lnew, l[p])
                m[p] = np.where(upd, mx, m[p])
    # the parts meet
    mg = m.max(0)
    lg = np.zeros(Sq, np.float32)
    for p in range(PARTS):
        cw = np.ones(Sq, np.float32) if mutation == "merge_no_rescale" else _exp(_f(m[p] - mg))
        lg = np.where(m[p] > -np.inf, _f(l[p].astype(np.float64) * cw + lg), lg).astype(np.float32)
    inv = np.where(lg > 0, _f(1.0 / lg.astype(np.float64)), 0).astype(np.float32)
    # pass B
    o = np.zeros((Sq, D), np.float32)
    for t in range(ntiles):
        if mutation == "skip_last_tile_b" and t == ntiles - 1:
            continue
        s = S[t]
        if mutation == "stale_k" and t > 0:  # the previous tile's K: its scores for this tile's columns
            s = np.full_like(s, -np.inf)
            n = min(s.shape[1], S[t - 1].shape[1])
            s[:, :n] = S[t - 1][:, :n]
        n = s.shape[1]
        pr = np.zeros((Sq, n), np.float32)
        for p in range(PARTS):
            cols = slice(p * PCOLS, min(n, p * PCOLS + PCOLS))
            iv = inv
            if mutation == "part_l":
                iv = np.where(l[p] > 0, _f(1.0 / l[p].astype(np.float64)), 0).astype(np.float32)
            e = _exp(_f(s[:, cols] - mg[:, None]))
            if mutation == "p_rounded_twice":
                e = _r32(e, dt)
            pr[:, cols] = np.where(mg[:, None] > -np.inf, _f(e * iv[:, None]), 0)
        P = pr if mutation == "p_unrounded" else _r32(pr, dt)
        if trace is not None:
            trace.setdefault("s3", []).append(s)
            trace.setdefault("P", []).append(P)
        vt = v[t * BK:t * BK + n].astype(np.float64)
        for kk in range(-(-n // 16)):
            sl = slice(16 * kk, min(n, 16 * kk + 16))
            o = _f(o + P[:, sl].astype(np.float64) @ vt[sl])
    return _r32(o, dt)


def emulate(case, dt, mutation=None):
    out = np.zeros((case.B, case.H, case.Sq, case.D), np.float32)
    for b in range(case.B):
        for h in range(case.H):
            out[b, h] = emulate_head(case.q[b, h], case.k[b, h], case.v[b, h], case.head_mask(dt, b, h), case.scale, dt, mutation)
    return out


# ====================================================================== which load_mask path a case takes
def mask_paths(case, dt):
    """set of load_mask paths the case reaches: "vector", "scalar", "misaligned", "mi0", "mj" """
    store, (mb, mh, mi, mj), off, _ = case.mask(dt)
    r = set()
    if store is None:
        return r
    if mi == 0:
        r.add("mi0")
    if mj != 1:
        r.add("mj")
    for b in range(case.B):
        for h in range(case.H):
            base = off + b * mb + h * mh
            aligned = (base * 2) % 16 == 0
            if not aligned:
                r.add("misaligned")
            mvec = mj == 1 and mi % 8 == 0 and aligned
            for t in range(-(-case.Skv // BK)):
                for jc in range(0, BK, 8):
                    j = t * BK + jc
                    if j >= case.Skv:
                        continue
                    if mvec and j + 8 <= case.Skv:
                        r.add("vector")
                    else:
                        r.add("scalar")
    return r
