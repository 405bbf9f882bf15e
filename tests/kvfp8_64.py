"""Float64 reference, per-element bound and float32 emulation of decode attention over an FP8 E4M3 KV cache
(attn_stream_kv8_kernel, G = 1, and attn_gqa_kv8_kernel, G > 1, in attention.cu), on attn64's score regimes and dealing model.

Values.  A cache element is e4m3(code) * scale[KV head] (tests/kvfp8_oracle.py).  `Case` builds the problem in a unit domain
(attn64's regimes, with the scores computed from the decoded codes) and then carries it to KV head h by exact powers of two:
K values x f_k(h) = 2^((h mod 5) - 2), V values x f_v(h) = 2^((h mod 3) - 1), q / f_k(h), on scale bases 0.7 / 448 and 1.7 / 448
(times a power of two that fits the case's data), so the codes are those of the unit problem while the scales of
neighbouring heads, of K and V, and of a query head read as a KV head differ by 2x or more.

Reference.  Float64 over the dequantised caches after the append (row p_b = quantise(k / v), RoPE already applied).  With
s_j = q.k_j / sqrt(D), w = softmax(s) over rows 0 .. p and ref = sum_j w_j v_j:

    |got - ref| <= ulp_T(|ref|) + 2^-23 |ref| + 2^-16 sum_j w_j |v_j| + c_s 2^-24 sum_j w_j a_j |v_j - ref|
                   + 2^-126 (sum_j |v_j| + p + 1) / L  [+ 2^-25 sum_j |v_j| / L]
    a_j = sum_i |q_i k_ji| / sqrt(D),   L = sum_j exp(s_j - max s),   the last term for f16 in attn_gqa_kv8_kernel only

* ulp_T(|ref|), 2^-16 sum w|v| and the f16 hi + lo term: as attn64 (one rounding to T; fp32 softmax, P.V and merge chains
  over at most 264 partials; subnormal f16 weights).  The weights and P.V see the decoded codes, which are exact in T, times
  fp32 weights, so nothing there depends on the cache type.
* 2^-126 (sum |v_j| + p + 1) / L: a weight exp(s_j - max) or a product P_j v_j below fp32's smallest normal may be flushed
  to 0 (bf16 operands of the tensor core are), up to 2^-126 (|v_j| + 1) of absolute error per row, divided by the final l.
  It matters only where ref is itself near 2^-126: outputs made of weights near exp(-87), as on appended rows of zeros.
* 2^-23 |ref|: the output is fp32(fp32(A / L) * v_scale), two fp32 roundings before the rounding to T.
* c_s = 24: the error of one fp32 score, in units of 2^-24 a_j (an error d_j in s_j moves the output by sum_j w_j d_j (v_j - ref)
  to first order).  Codes decode exactly to fp32 and to T.
  - attn_stream_kv8_kernel: qs = fp32(k_scale * fp32(1 / sqrt(D))) (at D = 128 the constant is rounded: 1 unit; the product:
    1) and q_i * qs (1) scale every term alike: 3 units; each lane then runs an fma chain of 16 terms (16 roundings of a partial
    sum no larger than a_j) and the row's lanes meet in a shuffle tree of 3 (D 128, 8 lanes) or 2 (D 64, 4 lanes) additions:
    3 + 16 + 3 = 22 units.
  - attn_gqa_kv8_kernel: q (T) times a code widened to T is exact in fp32 (11 + 4 significant bits); D / 16 chained
    m16n8k16 steps add 16 products each into the fp32 accumulator, 2 units per step (truncation allowed, as attn64):
    16 (D 128) or 8 (D 64); then the product with ksc = fp32(k_scale * fp32(1 / sqrt(D))): 3 units.  19 at most.
  22 <= 24, which replaces kvfp8_oracle's 64.

`emulate` follows both kernels' order of operations in float32 through `Deal`'s split and merge (attn64's per-CTA partials
with the FP8 row layout, chunk rows and k order), the appended row through its codes, and stays within half of the bound.
"""
import math

import numpy as np

import oracle
from tests import attn64, ref64
from tests import kvfp8_oracle as KV
from tests.attn64 import BF16, F16, Deal

C_SCORE = 24.0
OUT_REL = 2.0 ** -23
TINY = 2.0 ** -126
K_BASE, V_BASE = np.float32(0.7) / np.float32(448), np.float32(1.7) / np.float32(448)
REGIMES = attn64.REGIMES + ["sat"]
NAN_CODES = (0x7F, 0xFF)
# the +200 tent stops at 152 (still 48 below the peak, exp(-48) of its weight): a k row of score s carries about s / 3 along
# its head's q, and E4M3's 2^-4 relative rounding of rows at s = -10^4 would leak scores of tens of units into the other
# query heads of the group
TENT_FLOOR = 152.0


def f_k(h):
    return 2.0 ** ((np.asarray(h) % 5) - 2)


def f_v(h):
    return 2.0 ** ((np.asarray(h) % 3) - 1)


def kscale(d):
    return np.float32(attn64.SCALE32 if d == 128 else 0.125)


def _pow2_over(amax, base):
    """the power of two M with amax / (base M) in (224, 448]: the unit problem's largest element just inside the E4M3 range"""
    return 2.0 ** math.ceil(math.log2(max(amax, 1e-6) / (448.0 * float(base))))


class Case:
    """one FP8 AttentionKVCache problem.  q [B, Hq, D] (exact in f16 and bf16); code caches kc, vc [B, Hkv, S, D] uint8 with
    NaN codes (0x7F / 0xFF mixed) from row p_b on; the appended rows kn, vn [B, Hkv, 1, D]; scales ksc, vsc [Hkv] float32.
    Regimes cycle over (batch row, query head) starting at `offset`; "sat" puts the peak on an appended k row whose large
    elements lie beyond +-448 * scale, with a v row saturated alike, so the saturated codes carry the output."""

    def __init__(self, B, Hq, Hkv, S, D, pos, seed, offset=0):
        self.B, self.Hq, self.Hkv, self.S, self.D, self.grp = B, Hq, Hkv, S, D, Hq // Hkv
        self.pos = np.clip(np.broadcast_to(np.asarray(pos, np.int64), (B,)), 0, S - 1)
        self.per_row = np.ndim(pos) > 0
        rng = np.random.default_rng(seed)
        g = self.grp
        qu = np.zeros((B, Hq, D))
        ku = [[None] * Hkv for _ in range(B)]
        vu = [[None] * Hkv for _ in range(B)]
        self.regime = np.empty((B, Hq), object)
        vrow = np.exp2((np.arange(S) % 5) - 2.0)
        sat_cols = {}
        for b in range(B):
            n = int(self.pos[b]) + 1
            for kv in range(Hkv):
                # orthogonal query heads, in blocks of at most D when the group is wider than the head (G 80 at D 64)
                qo = np.concatenate([np.linalg.qr(rng.standard_normal((D, min(D, g - r0))))[0].T for r0 in range(0, g, D)])
                qg = attn64.exact(qo * math.sqrt(D / 4.0)).astype(np.float64)
                regs = [REGIMES[(b * Hq + kv * g + r + offset) % len(REGIMES)] for r in range(g)]
                self.regime[b, kv * g:(kv + 1) * g] = regs
                taken = set()
                for r in [r for r in range(g) if regs[r] == "sat"]:
                    # four columns of the "sat" head that every other query head of the group ignores (q = 0 there): the
                    # saturated elements of the appended k row move this head's scores only
                    cols = [c for c in np.argsort(-np.abs(qg[r])) if c not in taken][:4]
                    taken.update(cols)
                    keep = qg[r, cols].copy()
                    qg[:, cols] = 0
                    qg[r, cols] = keep
                    sat_cols.setdefault((b, kv), []).append((r, cols))
                z = rng.standard_normal((n, D)) * 0.5
                k = z.copy()
                for r in range(g):
                    reg = regs[r]
                    reg = "append" if reg == "sat" else reg
                    for j, t in attn64.targets(reg, n - 1, rng).items():
                        t = max(t, TENT_FLOOR) if reg == "pos200" else t
                        k[j] += (t * math.sqrt(D) - qg[r] @ z[j]) / (qg[r] @ qg[r]) * qg[r]
                qu[b, kv * g:(kv + 1) * g] = qg
                ku[b][kv] = k
                vu[b][kv] = rng.standard_normal((n, D)) * 0.5 * vrow[:n, None]
        # one scale per KV head for the whole batch: the unit problem's cache rows (not the appended rows) just fit
        heads = np.arange(Hkv)
        self.ksc = np.empty(Hkv, np.float32)
        self.vsc = np.empty(Hkv, np.float32)
        for kv in heads:
            ka = max(np.abs(ku[b][kv][:-1]).max(initial=0) for b in range(B))
            va = max(np.abs(vu[b][kv][:-1]).max(initial=0) for b in range(B))
            ka = ka or max(np.abs(ku[b][kv]).max() for b in range(B))
            va = va or max(np.abs(vu[b][kv]).max() for b in range(B))
            self.ksc[kv] = np.float32(K_BASE * _pow2_over(ka, K_BASE) * f_k(kv))
            self.vsc[kv] = np.float32(V_BASE * _pow2_over(va, V_BASE) * f_v(kv))
        self.q = np.empty((B, Hq, D), np.float32)
        self.kc = np.empty((B, Hkv, S, D), np.uint8)
        self.vc = np.empty((B, Hkv, S, D), np.uint8)
        self.kn = np.empty((B, Hkv, 1, D), np.float32)
        self.vn = np.empty((B, Hkv, 1, D), np.float32)
        for b in range(B):
            p = int(self.pos[b])
            for kv in heads:
                hs = slice(kv * g, (kv + 1) * g)
                self.q[b, hs] = attn64.exact(qu[b, hs] / f_k(kv))
                k = ku[b][kv] * f_k(kv)
                v = vu[b][kv] * f_v(kv)
                for r, cols in sat_cols.get((b, kv), []):
                    # the appended k row 3x past +-448 scale on the head's own columns, signed with its q: a peak on top of
                    # the "append" target that only the saturated codes carry; v saturates on every third column
                    k[p, cols] = 3.0 * 448.0 * float(self.ksc[kv]) * np.sign(self.q[b, kv * g + r, cols])
                    v[p] = rng.standard_normal(D) * 448.0 * float(self.vsc[kv]) * np.where(np.arange(D) % 3 == 0, 2.0, 0.3)
                kx, vx = attn64.exact(k), attn64.exact(v)
                self.kn[b, kv, 0], self.vn[b, kv, 0] = kx[p], vx[p]
                self.kc[b, kv, :p] = KV.quantise(kx[:p], self.ksc[kv])
                self.vc[b, kv, :p] = KV.quantise(vx[:p], self.vsc[kv])
                poison = rng.choice(np.array(NAN_CODES, np.uint8), size=(2, S - p, D))
                self.kc[b, kv, p:], self.vc[b, kv, p:] = poison
        self.sat_cols = sat_cols

    def appended(self):
        """(k codes, v codes) of the appended rows [B, Hkv, D]"""
        return (KV.quantise(self.kn[:, :, 0], self.ksc[None, :, None]),
                KV.quantise(self.vn[:, :, 0], self.vsc[None, :, None]))

    def after_append(self):
        """the code caches as the step must leave them: row p_b <- the appended codes, every other row as before"""
        kc, vc = self.kc.copy(), self.vc.copy()
        ka, va = self.appended()
        for b in range(self.B):
            p = int(self.pos[b])
            kc[b, :, p], vc[b, :, p] = ka[b], va[b]
        return kc, vc

    def values(self, b, kv):
        """float64 K, V [p + 1, D] of KV head kv in batch row b after the append"""
        kc, vc = self.after_append() if not hasattr(self, "_after") else self._after
        self._after = (kc, vc)
        p = int(self.pos[b])
        return (KV.decode(kc[b, kv, :p + 1]) * float(self.ksc[kv]), KV.decode(vc[b, kv, :p + 1]) * float(self.vsc[kv]))

    def scores(self, b, h):
        K, _ = self.values(b, h // self.grp)
        return self.q[b, h].astype(np.float64) @ K.T / math.sqrt(self.D)

    def reference(self):
        """float64 (ref, sum w|v|, sum w a |v - ref|, sum |v| / L, (p + 1) / L), each [B, Hq, D]"""
        D = self.D
        out = [np.empty((self.B, self.Hq, D)) for _ in range(5)]
        for b in range(self.B):
            for kv in range(self.Hkv):
                hs = slice(kv * self.grp, (kv + 1) * self.grp)
                K, V = self.values(b, kv)
                q = self.q[b, hs].astype(np.float64)
                s = q @ K.T / math.sqrt(D)
                a = np.abs(q) @ np.abs(K).T / math.sqrt(D)
                e = np.exp(s - s.max(1, keepdims=True))
                L = e.sum(1, keepdims=True)
                w = e / L
                ref = w @ V
                out[0][b, hs], out[1][b, hs] = ref, w @ np.abs(V)
                out[2][b, hs] = [(w[r] * a[r]) @ np.abs(V - ref[r]) for r in range(self.grp)]
                out[3][b, hs] = np.abs(V).sum(0)[None, :] / L
                out[4][b, hs] = len(V) / L
        return out

    def deal(self, dt):
        return Deal(dt, self.B, self.Hq, self.Hkv, self.S, self.pos, self.D, kv8=True)


def bound(refs, dt, gqa):
    ref, wv, wav, vl, nl = refs
    b = (ref64.ulp(ref, dt) + OUT_REL * np.abs(ref) + ref64.ACC_SLACK * wv + C_SCORE * 2.0 ** -24 * wav
         + TINY * (vl + nl))
    return b + attn64.F16_P_ABS * vl if (gqa and dt == F16) else b


def violations(got, refs, dt, gqa, scale=1.0):
    """boolean [B, Hq, D] mask of the elements outside scale x the bound; NaN is outside"""
    return ~(np.abs(np.asarray(got, np.float64) - refs[0]) <= scale * bound(refs, dt, gqa))


def report(bad, got, refs, dt, gqa, case, deal, what, limit=4):
    """attn64.report with this bound, naming each head's regime"""
    if not bad.any():
        return None
    bd = bound(refs, dt, gqa)
    lines = [f"{what}: {int(bad.sum())} of {bad.size} elements outside the bound"]
    heads = sorted({(int(b), int(h)) for b, h, _ in np.argwhere(bad)})
    for b, h in heads[:limit]:
        d = int(np.argmax(np.where(bad[b, h], np.abs(got[b, h] - refs[0][b, h]) / bd[b, h], -1)))
        lines.append(f"  {deal.where(b, h)}, regime {case.regime[b, h]}; column {d}: got {float(got[b, h, d])!r}, "
                     f"float64 {refs[0][b, h, d]!r}, bound {bd[b, h, d]:.3g}")
    if len(heads) > limit:
        lines.append(f"  ... {len(heads)} heads in all: {heads[:24]}")
    return "\n".join(lines)


# ====================================================================== float32 emulation of both FP8 kernels
MUTATIONS = {
    "neighbour_k_scale": "the K scale of KV head h + 1",
    "kv_scales_swapped": "K's scale read for V and V's for K",
    "v_scale_partials": "V's scale applied to each CTA partial and again after the merge",
    "scale_by_query_head": "the scales indexed by query head instead of KV head",
    "unquantised_append": "the appended row contributes its unquantised values",
    "drop_last_row": "the last cache row of the last chunk dropped",
    "merge_ignore_max": "the merge adds partials without their maxima",
    "no_rescale": "no rescale when a later chunk raises the running maximum",
    "round_p_once": "P rounded once to T before P.V (grouped)",
}


def emulate(case, dt, mutation=None):
    """the kernel's output [B, Hq, D] as float32, segment by segment with the CTA split of `Deal`"""
    with np.errstate(invalid="ignore", over="ignore"):
        return _emulate(case, dt, mutation)


def _emulate(case, dt, mutation):
    deal = case.deal(dt)
    D, g = case.D, case.grp
    out = np.empty((case.B, case.Hq, D), np.float32)
    kca, vca = case.appended()
    base = mutation if mutation in ("drop_last_row", "merge_ignore_max", "no_rescale", "round_p_once") else None

    def scales(kv, i):
        """(k scale, v scale) a slip reads for KV head kv (i: the scale index it uses)"""
        ks, vs = case.ksc, case.vsc
        if mutation == "kv_scales_swapped":
            ks, vs = vs, ks
        if mutation == "neighbour_k_scale":
            return ks[(kv + 1) % case.Hkv], vs[kv]
        return ks[i], vs[i]

    for b in range(case.B):
        p = int(case.pos[b])
        for s in range(deal.segs):
            _, ctas, chunks = deal.segment(b, s)
            if g == 1:
                heads, kv = np.array([s]), s
            else:
                kv, qg = divmod(s, deal.NQG)
                heads = np.arange(kv * g + qg * deal.GP, min((kv + 1) * g, kv * g + (qg + 1) * deal.GP))
            # the scale index of each query head: its KV head, or (the slip) the query head itself, mod Hkv to stay in range
            src = heads % case.Hkv if mutation == "scale_by_query_head" else np.full(len(heads), kv)
            for i in np.unique(src):
                hs = heads[src == i]
                out[b, hs] = _segment(case, dt, deal, b, p, kv, hs, chunks, *scales(kv, i), mutation, base, kca, vca)
    return out


def _segment(case, dt, deal, b, p, kv, heads, chunks, ks, vs, mutation, base, kca, vca):
    """the output rows of query heads `heads` (one segment's, all of one KV head) with scales ks / vs"""
    D, g = case.D, case.grp
    K = KV.decode(case.kc[b, kv, :p]).astype(np.float32)
    V = KV.decode(case.vc[b, kv, :p]).astype(np.float32)
    if mutation == "unquantised_append":
        kn, vn = _f(case.kn[b, kv, 0] / np.float32(ks)), _f(case.vn[b, kv, 0] / np.float32(vs))
    else:
        kn, vn = KV.decode(kca[b, kv]).astype(np.float32), KV.decode(vca[b, kv]).astype(np.float32)
    sc = _f(np.float32(ks) * kscale(D))
    last = [ch[-1] == deal.nch[b] - 1 for ch in chunks]
    if g == 1:
        parts = [attn64.emulate_stream_partial(case.q[b, heads[0]], K, V, kn, vn, p, ch, la, dt, base, qs=sc, kv8=True)
                 for ch, la in zip(chunks, last)]
        parts = [(np.array([m]), np.array([l]), a[None]) for m, l, a in parts]
    else:
        Q = np.zeros((deal.GP, D), np.float32)
        Q[:len(heads)] = case.q[b, heads]
        parts = [attn64.emulate_gqa_partial(Q, K, V, kn, vn, p, ch, la, dt, base, sscale=sc, kv8=True)
                 for ch, la in zip(chunks, last)]
    if mutation == "v_scale_partials" and len(parts) > 1:
        parts = [(m, l, _f(a * np.float32(vs))) for m, l, a in parts]
    return attn64._merge(parts, dt, base, vscale=vs)[:len(heads)]


def _f(x):
    return np.asarray(x, np.float64).astype(np.float32)


# ====================================================================== the quantiser's edges
def pow2_edges(s):
    """(classes, midpoints): fp32 inputs for a power-of-two scale s, exact in f16 and bf16.  classes: +-0, +-448 s, +-464 s
    (rounds to 448), +-480 s and 2^14 s (saturate), +-inf, the smallest subnormal +-2^-9 s and half of it (ties to 0);
    midpoints: exact midpoints between adjacent E4M3 values times s, which tie to the even code, upward or downward"""
    e = [0.0, -0.0, 448.0, -448.0, 464.0, -464.0, 480.0, -480.0, 2.0 ** 14, np.inf, -np.inf, 2.0 ** -9, -(2.0 ** -9),
         2.0 ** -10, -(2.0 ** -10)]
    mids = (KV.DECODE[1:127] + KV.DECODE[0:126]) / 2
    mids = mids[(mids >= 2.0 ** -9) & (mids <= 416)]
    mids = np.stack([mids, -mids], 1).ravel()
    return (np.array(e) * s).astype(np.float32), (mids * s).astype(np.float32)


def disagreeing_inputs(dt, s, n=64):
    """values exact in T on which quantise(x, s) and quantise_reciprocal(x, s) give different codes (s not a power of two):
    every finite positive T value is tried, both signs returned"""
    bits = np.arange(0x0001, 0x7C00 if dt == F16 else 0x7F80, dtype=np.uint32)
    if dt == F16:
        x = bits.astype(np.uint16).view(np.float16).astype(np.float32)
    else:
        x = (bits << 16).view(np.float32)
    x = x[np.abs(x) <= 500 * float(s)]
    x = x[KV.quantise(x, s) != KV.quantise_reciprocal(x, s)]
    x = x[np.linspace(0, x.size - 1, min(n, x.size)).astype(int)] if x.size else x
    return np.concatenate([x, -x]).astype(np.float32)
