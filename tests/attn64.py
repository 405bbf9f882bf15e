"""Float64 reference, per-element bound, work-dealing model and float32 emulation of the decode attention kernels in
attention.cu: attn_stream_kernel (query heads = KV heads) and attn_gqa_kernel (G = Hq / Hkv query heads per KV head).

Reference.  The inputs are exact in f16, bf16 and fp32 (`exact`), so they are exact in float64.  Row `pos` of a batch row's
sequence is the appended k / v.  With s_j = q.k_j / sqrt(128), w = softmax(s) over rows 0 .. pos and ref = sum_j w_j v_j:

    |got - ref| <= ulp_T(|ref|) + 2^-16 sum_j w_j |v_j| + c_s 2^-24 sum_j w_j a_j |v_j - ref|  [+ 2^-25 sum_j |v_j| / L]
    a_j = sum_i |q_i k_ji| / sqrt(128),   L = sum_j exp(s_j - max s),   the last term for f16 in attn_gqa_kernel only

* ulp_T(|ref|) (tests/ref64.py; fp32: 2^(e - 23)): the output is rounded to T once, half an ulp, doubled for a rounding that
  crosses a binade.
* 2^-16 sum w|v|: fp32 softmax and P.V.  Each weight is expf (<= 2 ulp, 2^-22 relative) times at most a few expf
  rescales; l and acc are fp32 running sums with positive weights.  The longest chain a weight passes through is the merge of
  264 CTA partials (B = H = 1 at p 16383, fp32): <= 264 roundings of the running sum, 264 x 2^-24 < 2^-15.9 of
  sum w|v| even if every one errs the same way, and about 2^-20 for rounding errors of random sign.  The hi + lo split of P
  in attn_gqa_kernel keeps 16 (bf16) / 22 (f16) significant bits of each weight: <= 2^-17 relative.  A weight rounded once
  to bf16 (2^-9) is outside this term wherever |ref| is small against sum w|v|, which is what the term is for.
* c_s = 32: the error of one fp32 score.  An error d_j in s_j moves the output by sum_j w_j d_j (v_j - ref) to first order,
  so |d_j| <= c_s 2^-24 a_j gives the term.  attn_stream_kernel: q is scaled by fp32(1/sqrt(128)) (2 roundings), each product
  enters an fma chain of 8 terms per lane (f16 / bf16; 4 for fp32) and a 4-level (fp32: 5) shuffle tree: at most
  2 + 8 + 4 = 14 roundings of a partial sum no larger than a_j, so |d_j| <= 14 x 2^-24 a_j.  attn_gqa_kernel, f16 / bf16:
  the products are exact in fp32, 8 chained mma.m16n8k16 steps each add 16 of them into the fp32 accumulator; counting each
  step as 2 units of roundoff (truncation allowed, as tests/ref64.py does) and 2 more for the fp32 scale gives
  18 x 2^-24 a_j.  attn_gqa_kernel, fp32: one chain of 128 fmaf; its worst case (every rounding the same way on a partial
  sum of magnitude a_j) is 130 x 2^-24 a_j, but its rounding errors are independent and of either sign: Higham's
  probabilistic bound gives lambda sqrt(130) 2^-24 a_j, and c_s = 32 is lambda = 2.8 for one score; the output term sums
  those bounds over every row without cancellation, so an output that leaves it needs many scores at that tail at once.
* 2^-25 sum |v| / L (f16, attn_gqa_kernel): hi and lo of P are f16, whose subnormals below 2^-14 are spaced 2^-24 apart, so
  a weight below 2^-14 of the running maximum carries up to 2^-25 of absolute error; the running maximum is at most max s,
  so divided by the final l that is <= 2^-25 |v_j| / L per row.

The float32 emulation below, which follows both kernels' order of operations, stays within half of the bound on cases
carrying every score regime (test_attention_float64.py checks it); the rounding of the output to T, half an ulp, is what
comes closest.

The kernels deal (head or (KV head, query group), 64-row chunk) units (32 rows for fp32) of the whole batch in equal
contiguous ranges over min(units, 264) CTAs; `Deal` restates that dealing so failures can be located and so the tests can
show which dealing states their cases reach.  A chunk is 16 KiB of cache: `Deal` and the emulation below also take the head
width and FP8 caches (one byte per element, tests/kvfp8_64.py), whose chunks hold 16384 / D rows.
"""
import math

import numpy as np

import oracle
from tests import ref64

F32, F16, BF16 = 1, 10, 16
D = 128
GRID_MAX = 264                     # AS_CTAS_PER_SM x kNumSMs
C_SCORE = 32.0
F16_P_ABS = 2.0 ** -25
SCALE32 = np.float32(0.08838834764831845)  # the kernels' fp32 1/sqrt(128)
NAMES = {F32: "fp32", F16: "f16", BF16: "bf16"}


def chunk_rows(dt, d=D, kv8=False):
    """cache rows per 16 KiB chunk: 64 (f16 / bf16) or 32 (fp32) at D = 128, twice that at D = 64; FP8 codes: 16384 / D"""
    return 16384 // (d * (1 if kv8 else 4 if dt == F32 else 2))


# ====================================================================== dealing model
class Deal:
    """How attn_stream_kernel (grp = 1) and attn_gqa_kernel (grp > 1) deal their units.  A segment is a head (grp = 1) or a
    (KV head, query group) pair; unit u of the batch is (segment, chunk) in row-major order over batch rows."""

    def __init__(self, dt, B, Hq, Hkv, S, pos, d=D, kv8=False):
        self.dt, self.B, self.Hq, self.Hkv, self.S = dt, B, Hq, Hkv, S
        self.CH = chunk_rows(dt, d, kv8)
        self.grp = Hq // Hkv
        if self.grp == 1:
            self.QT, self.GP, self.NQG, self.segs = 1, 1, 1, Hq
        else:
            self.QT = 1 if self.grp <= 16 else 2
            self.GP = 16 * self.QT
            self.NQG = -(-self.grp // self.GP)
            self.segs = Hkv * self.NQG
        pos = np.broadcast_to(np.asarray(pos, np.int64), (B,))
        self.pos = np.clip(pos, 0, S - 1)
        self.nch = self.pos // self.CH + 1
        self.pre = np.concatenate([[0], np.cumsum(self.segs * self.nch)]).astype(np.int64)
        self.total = int(self.pre[-1])
        self.grid = int(min(B * self.segs * (S // self.CH + 1), GRID_MAX))
        self.ncta = min(self.grid, self.total)
        self.u0 = [c * self.total // self.ncta for c in range(self.ncta + 1)]  # CTA c owns units [u0[c], u0[c + 1])

    def owner(self, u):
        """the CTA owning unit u, as the merge computes it"""
        return ((u + 1) * self.ncta - 1) // self.total

    def cta_of(self, u):
        """the CTA owning unit u by the forward dealing"""
        return int(np.searchsorted(self.u0, u, side="right")) - 1

    def unit(self, u):
        """(batch row, segment, chunk) of unit u"""
        b = int(np.searchsorted(self.pre, u, side="right")) - 1
        s, c = divmod(u - int(self.pre[b]), int(self.nch[b]))
        return b, s, c

    def segment(self, b, s):
        """(first unit, CTAs of the segment in order, chunks per CTA) of segment s of batch row b"""
        hu0, n = int(self.pre[b]) + s * int(self.nch[b]), int(self.nch[b])
        ctas, chunks = [], []
        for c in range(n):
            o = self.owner(hu0 + c)
            if not ctas or ctas[-1] != o:
                ctas.append(o)
                chunks.append([])
            chunks[-1].append(c)
        return hu0, ctas, chunks

    def seg_of_head(self, h):
        """(segment, KV head, query group, row in the group) of query head h"""
        if self.grp == 1:
            return h, h, 0, 0
        kv, r = divmod(h, self.grp)
        qg, rr = divmod(r, self.GP)
        return kv * self.NQG + qg, kv, qg, rr

    def where(self, b, h):
        s, kv, qg, _ = self.seg_of_head(h)
        _, ctas, chunks = self.segment(b, s)
        grp = f", KV head {kv}, query group {qg} of {self.NQG} (QT {self.QT})" if self.grp > 1 else ""
        return (f"batch row {b} (pos {int(self.pos[b])}, {int(self.nch[b])} chunks of {self.CH}), query head {h}{grp}: "
                f"CTAs {ctas[0]}..{ctas[-1]} of {self.ncta} share it (nseg {len(ctas)}), chunks per CTA "
                f"{[len(c) for c in chunks][:8]}{'...' if len(chunks) > 8 else ''}")

    def ctas_units(self):
        return [[self.unit(u) for u in range(self.u0[c], self.u0[c + 1])] for c in range(self.ncta)]


# ====================================================================== inputs
REGIMES = ["flat", "late", "early", "sink", "prev", "append", "neg150", "pos200"]


def exact(x):
    """float32 -> rounded to bf16 with |x| < 2^-14 flushed to 0: exact in bf16, f16 and fp32 alike (asserted)"""
    y = oracle.round_to(np.asarray(x, np.float32), BF16)
    y[np.abs(y) < 2.0 ** -14] = 0
    assert np.all(np.abs(y) < 60000) and np.array_equal(oracle.round_to(y, F16), y)
    return y


def targets(regime, pos, rng):
    """{row: target score} for rows 0 .. pos of one query head (rows not listed keep the flat, random scores)"""
    n = pos + 1
    peaks = sorted({int(round(f * pos)) for f in (0.1, 0.35, 0.6, 0.85)} - {pos})
    if regime == "late" and peaks:
        return {j: 6.0 + 3.0 * i for i, j in enumerate(peaks)}
    if regime == "early" and peaks:
        return {j: 15.0 - 3.0 * i for i, j in enumerate(peaks)}
    if regime == "sink":
        return {0: 20.0}
    if regime == "prev" and pos >= 1:
        return {pos - 1: 20.0}
    if regime == "append":
        return {pos: 20.0}
    if regime == "neg150":
        return dict(enumerate(-150.0 + 3.0 * rng.standard_normal(n)))
    if regime == "pos200":  # a tent peaking at 200 two thirds of the way in: a later CTA's maximum far above an earlier one's
        top = (2 * pos) // 3
        return {j: 200.0 - abs(j - top) for j in range(n)}
    return {}


class Case:
    """one AttentionKVCache problem.  q [B, Hq, 128]; kseq, vseq [B, Hkv, S, 128] hold the whole sequence, row pos_b being
    the appended k / v of batch row b; the caches are kseq / vseq with rows >= pos_b set to NaN.  Regimes cycle over
    (batch row, query head) starting at `offset`."""

    def __init__(self, B, Hq, Hkv, S, pos, seed, offset=0):
        self.B, self.Hq, self.Hkv, self.S, self.grp = B, Hq, Hkv, S, Hq // Hkv
        self.pos = np.clip(np.broadcast_to(np.asarray(pos, np.int64), (B,)), 0, S - 1)
        self.per_row = np.ndim(pos) > 0
        rng = np.random.default_rng(seed)
        g = self.grp
        self.q = np.empty((B, Hq, D), np.float32)
        self.kseq = np.full((B, Hkv, S, D), np.nan, np.float32)
        self.vseq = np.full((B, Hkv, S, D), np.nan, np.float32)
        self.regime = np.empty((B, Hq), object)
        vrow = np.exp2((np.arange(S) % 5) - 2.0)
        for b in range(B):
            n = int(self.pos[b]) + 1
            for kv in range(Hkv):
                # the group's query heads are orthogonal before rounding (|q|^2 = 32, as N(0, 0.5^2) draws): each head's
                # targets move only its own scores
                qo, _ = np.linalg.qr(rng.standard_normal((D, g)))
                qg = exact(qo.T * math.sqrt(32.0)).astype(np.float64)
                z = rng.standard_normal((n, D)) * 0.5
                k = z.copy()
                for r in range(g):
                    h = kv * g + r
                    reg = REGIMES[(b * Hq + h + offset) % len(REGIMES)]
                    self.regime[b, h] = reg
                    for j, t in targets(reg, n - 1, rng).items():
                        k[j] += (t * math.sqrt(D) - qg[r] @ z[j]) / (qg[r] @ qg[r]) * qg[r]
                self.q[b, kv * g:(kv + 1) * g] = qg
                self.kseq[b, kv, :n] = exact(k)
                v = rng.standard_normal((n, D)) * 0.5 * vrow[:n, None] * 2.0 ** ((kv % 3) - 1)
                self.vseq[b, kv, :n] = exact(v)

    def caches(self):
        """(k cache, v cache, appended k, appended v): the caches poisoned with NaN from row pos_b on"""
        kc, vc = self.kseq.copy(), self.vseq.copy()
        kn = np.empty((self.B, self.Hkv, 1, D), np.float32)
        vn = np.empty_like(kn)
        for b in range(self.B):
            p = int(self.pos[b])
            kn[b, :, 0], vn[b, :, 0] = self.kseq[b, :, p], self.vseq[b, :, p]
            kc[b, :, p:] = np.nan
            vc[b, :, p:] = np.nan
        return kc, vc, kn, vn

    def reference(self):
        """float64 (ref, sum w|v|, sum w a |v - ref|, sum |v| / L), each [B, Hq, 128]"""
        out = [np.empty((self.B, self.Hq, D)) for _ in range(4)]
        for b in range(self.B):
            n = int(self.pos[b]) + 1
            for kv in range(self.Hkv):
                hs = slice(kv * self.grp, (kv + 1) * self.grp)
                q = self.q[b, hs].astype(np.float64)
                k = self.kseq[b, kv, :n].astype(np.float64)
                v = self.vseq[b, kv, :n].astype(np.float64)
                s = q @ k.T / math.sqrt(D)
                a = np.abs(q) @ np.abs(k).T / math.sqrt(D)
                e = np.exp(s - s.max(1, keepdims=True))
                L = e.sum(1, keepdims=True)
                w = e / L
                ref = w @ v
                out[0][b, hs], out[1][b, hs] = ref, w @ np.abs(v)
                out[2][b, hs] = [(w[r] * a[r]) @ np.abs(v - ref[r]) for r in range(self.grp)]
                out[3][b, hs] = np.abs(v).sum(0)[None, :] / L
        return out


def bound(refs, dt, gqa):
    ref, wv, wav, vl = refs
    b = ref64.ulp(ref, dt) + ref64.ACC_SLACK * wv + C_SCORE * 2.0 ** -24 * wav
    return b + F16_P_ABS * vl if (gqa and dt == F16) else b


def violations(got, refs, dt, gqa, scale=1.0):
    """boolean [B, Hq, 128] mask of the elements outside scale x the bound; NaN is outside"""
    return ~(np.abs(np.asarray(got, np.float64) - refs[0]) <= scale * bound(refs, dt, gqa))


def report(bad, got, refs, dt, gqa, deal, what, limit=4):
    if not bad.any():
        return None
    lines = [f"{what}: {int(bad.sum())} of {bad.size} elements outside the bound"]
    bd = bound(refs, dt, gqa)
    heads = sorted({(int(b), int(h)) for b, h, _ in np.argwhere(bad)})
    for b, h in heads[:limit]:
        d = int(np.argmax(np.where(bad[b, h], np.abs(got[b, h] - refs[0][b, h]) / bd[b, h], -1)))
        lines.append(f"  {deal.where(b, h)}; column {d}: got {float(got[b, h, d])!r}, float64 {refs[0][b, h, d]!r}, "
                     f"bound {bd[b, h, d]:.3g}")
    if len(heads) > limit:
        lines.append(f"  ... {len(heads)} heads in all: {heads[:24]}")
    return "\n".join(lines)


# ====================================================================== float32 emulation of the kernels' arithmetic
def _f(x):
    return np.asarray(x, np.float64).astype(np.float32)


def _fma(a, b, c):
    return (np.asarray(a, np.float64) * b + c).astype(np.float32)


def _exp(x):
    with np.errstate(invalid="ignore", over="ignore"):
        return np.exp(np.asarray(x, np.float64)).astype(np.float32)


def _out(A, L, dt, vscale):
    """the output write: A / L rounded to T, or for an FP8 cache fp32(A / L) * v_scale rounded to T"""
    o = _f(A / L[..., None])
    return oracle.round_to(o if vscale is None else _f(o * np.float32(vscale)), dt)


def _merge(parts, dt, mutation, vscale=None):
    """the last CTA's merge of (m, l, acc) partials in CTA order; also the whole-segment output when there is one partial"""
    if len(parts) == 1:
        m, l, a = parts[0]
        return _out(a, l, dt, vscale)
    if mutation == "merge_skip_last":
        parts = parts[:-1]
    mw = parts[0][0] if mutation == "merge_slot0_max" else np.max([p[0] for p in parts], axis=0)
    L, A = np.float32(0), np.float32(0)
    for m, l, a in parts:
        cw = np.ones_like(m) if mutation == "merge_ignore_max" else _exp(m - mw)
        L, A = _fma(l, cw, L), _fma(a, cw[..., None], A)
    with np.errstate(invalid="ignore", divide="ignore"):
        return _out(A, L, dt, vscale)


def _stream_dot(qf, k, lpr, epl):
    """per-lane fma chains over EPL columns, then the xor shuffle tree over the row's LPR lanes; k [..., 128]"""
    kr = k.reshape(k.shape[:-1] + (lpr, epl))
    qr = qf.reshape(lpr, epl)
    d = np.zeros(k.shape[:-1] + (lpr,), np.float32)
    for j in range(epl):
        d = _fma(qr[:, j], kr[..., j], d)
    o = lpr // 2
    while o:
        d = _f(d + d[..., np.arange(lpr) ^ o])
        o //= 2
    return d[..., 0]


def emulate_stream_partial(q, K, V, kn, vn, pos, chunks, last, dt, mutation=None, qs=SCALE32, kv8=False):
    """one CTA's (m, l, acc) of one head in attn_stream_kernel: the consumer warps' per-thread online softmax over `chunks`,
    the appended row (warp 0, sub-row 0) if `last`, then the sub-row and warp merges.  K, V: the head's rows < pos.
    FP8 caches (kv8): K, V, kn, vn are the decoded E4M3 values, a lane holds 16 codes of a row, and qs = fp32(k_scale / sqrt(D))."""
    dw = K.shape[-1]
    CH = chunk_rows(dt, dw, kv8)
    lpr = dw // 16 if kv8 else 32 if dt == F32 else dw // 8
    rpw, epl, U = 32 // lpr, dw // lpr, 4
    qf = _f(q.astype(np.float32) * np.float32(qs))
    m = np.full((8, rpw), -np.inf, np.float32)
    l = np.zeros((8, rpw), np.float32)
    acc = np.zeros((8, rpw, dw), np.float32)
    idx = np.arange(CH).reshape(8, U, rpw)  # chunk row = warp U RPW + uu RPW + sub
    for c in chunks:
        nvalid = pos - c * CH - (1 if mutation == "drop_last_row" and c == chunks[-1] and last else 0)
        ok = idx < nvalid
        rows = np.clip(c * CH + idx, 0, max(pos - 1, 0))
        kc = np.where(ok[..., None], K[rows] if pos else 0, 0).astype(np.float32)
        vc = np.where(ok[..., None], V[rows] if pos else 0, 0).astype(np.float32)
        sc = np.where(ok, _stream_dot(qf, kc, lpr, epl), -np.inf).astype(np.float32)
        mx = np.maximum(m, sc.max(1))
        upd = mx > -np.inf
        corr = np.where(upd, _exp(m - mx), 1).astype(np.float32)
        if mutation == "no_rescale":
            corr = np.ones_like(corr)
        l2, a2 = _f(l * corr), _f(acc * corr[..., None])
        for uu in range(U):
            p = np.where(ok[:, uu], _exp(sc[:, uu] - mx), 0).astype(np.float32)
            l2, a2 = _f(l2 + p), _fma(p[..., None], vc[:, uu], a2)
        l, acc, m = np.where(upd, l2, l), np.where(upd[..., None], a2, acc), np.where(upd, mx, m)
        if last and c == chunks[-1]:
            d = _stream_dot(qf, kn.astype(np.float32), lpr, epl)
            for _ in range(2 if mutation == "append_twice" else 1):
                mx2 = max(m[0, 0], d)
                corr, pn = _exp(m[0, 0] - mx2), _exp(d - mx2)
                l[0, 0] = _fma(l[0, 0], corr, pn)
                acc[0, 0] = _fma(pn, vn, _f(acc[0, 0] * corr))
                m[0, 0] = mx2
    o = 1
    while o < rpw:  # sub-row folds (shuffles xor LPR, 2 LPR, ...): sub-row i takes in sub-row i ^ o
        x = np.arange(rpw) ^ o
        m2, l2, a2 = m[:, x], l[:, x], acc[:, x]
        mm = np.maximum(m, m2)
        live = mm > -np.inf
        c1 = np.where(live, _exp(m - mm), 0).astype(np.float32)
        c2 = np.where(live, _exp(m2 - mm), 0).astype(np.float32)
        l = _f(_f(l * c1) + _f(l2 * c2))
        acc = _f(_f(acc * c1[..., None]) + _f(a2 * c2[..., None]))
        m = mm
        o *= 2
    m, l, acc = m[:, 0], l[:, 0], acc[:, 0]
    mw = m.max()
    cw = np.where(m > -np.inf, _exp(m - mw), 0).astype(np.float32)
    L, A = np.float32(0), np.zeros(dw, np.float32)
    for w in range(8):
        L, A = _fma(l[w], cw[w], L), _fma(acc[w], cw[w], A)
    return np.float32(mw), L, A


def gqa_k_steps(d, kv8=False):
    """the head-dim columns of each chained k16 MMA step of S = Q K^T: 16 consecutive columns, or for FP8 caches the permuted
    order (step 4 jj + st: columns 64 jj + 16 qc + 4 st + {0 .. 3} for qc = 0 .. 3)"""
    if not kv8:
        return [np.arange(16 * kk, 16 * kk + 16) for kk in range(d // 16)]
    return [np.array([64 * jj + 16 * qc + 4 * st + e for qc in range(4) for e in range(4)])
            for jj in range(d // 64) for st in range(4)]


def emulate_gqa_partial(Q, K, V, kn, vn, pos, chunks, last, dt, mutation=None, sscale=SCALE32, kv8=False):
    """one CTA's (m [GP], l [GP], acc [GP, D]) of one (KV head, query group) segment in attn_gqa_kernel.  Q [GP, D] with
    zero padding rows; S = Q K^T per chunk (D / 16 chained k16 MMA steps, or D fmaf for fp32) times sscale, the eight warps'
    row maxima and sums, P as hi + lo in T (f16 / bf16), O += P V.  FP8 caches (kv8): K, V, kn, vn are the decoded E4M3
    values and sscale = fp32(k_scale / sqrt(D))."""
    D = Q.shape[1]
    CH = chunk_rows(dt, D, kv8)
    nc = CH // 32
    gp = Q.shape[0]
    Q = Q.astype(np.float32)
    m = np.full(gp, -np.inf, np.float32)
    l = np.zeros(gp, np.float32)
    o = np.zeros((gp, D), np.float32)
    for c in chunks:
        nvalid = pos - c * CH
        if mutation == "drop_last_row" and last and c == chunks[-1]:
            nvalid -= 1
        nv = max(min(nvalid, CH), 0)
        kc, vc = np.zeros((CH, D), np.float32), np.zeros((CH, D), np.float32)
        kc[:nv], vc[:nv] = K[c * CH:c * CH + nv], V[c * CH:c * CH + nv]
        nrows = nv
        if last and c == chunks[-1]:
            for _ in range(2 if mutation == "append_twice" else 1):
                kc[nrows], vc[nrows] = kn, vn
                nrows += 1
        if dt == F32:
            d = np.zeros((gp, CH), np.float32)
            for dd in range(D):
                d = _fma(Q[:, dd, None], kc[None, :, dd], d)
        else:
            d = np.zeros((gp, CH), np.float32)
            for cols in gqa_k_steps(D, kv8):
                d = _f(d + Q[:, cols].astype(np.float64) @ kc[:, cols].T.astype(np.float64))
        s = _f(d * np.float32(sscale))
        s[:, nrows:] = -np.inf
        mnew = np.maximum(m, s.max(1))
        p = _exp(s - mnew[:, None])
        hi = oracle.round_to(p, dt)
        lo = np.zeros_like(p) if mutation == "round_p_once" else oracle.round_to(_f(p - hi), dt)
        t = p.reshape(gp, 8, 4, nc)
        ts = t[..., 0]
        for e in range(1, nc):
            ts = _f(ts + t[..., e])
        ts = _f(ts + ts[..., [1, 0, 3, 2]])
        ts = _f(ts + ts[..., [2, 3, 0, 1]])
        ls = np.zeros(gp, np.float32)
        for w in range(8):
            ls = _f(ls + ts[:, w, 0])
        corr = np.ones(gp, np.float32) if mutation == "no_rescale" else _exp(m - mnew)
        l = _fma(l, corr, ls)
        o = _f(o * corr[:, None])
        if dt == F32:
            for k in range(nrows):
                o = _fma(hi[:, k, None], vc[k], o)
        else:
            for kk in range(CH // 16):
                sl = slice(16 * kk, 16 * kk + 16)
                o = _f(o + lo[:, sl].astype(np.float64) @ vc[sl].astype(np.float64))
                o = _f(o + hi[:, sl].astype(np.float64) @ vc[sl].astype(np.float64))
        m = mnew
    return m, l, o


def emulate(case, dt, mutation=None):
    """the kernel's output [B, Hq, 128] as float32, emulated segment by segment with the CTA split of `Deal`"""
    with np.errstate(invalid="ignore", over="ignore"):  # -inf - -inf where a thread has seen no row yet (masked below)
        return _emulate(case, dt, mutation)


def _emulate(case, dt, mutation):
    deal = Deal(dt, case.B, case.Hq, case.Hkv, case.S, case.pos)
    out = np.empty((case.B, case.Hq, D), np.float32)
    for b in range(case.B):
        p = int(case.pos[b])
        for s in range(deal.segs):
            _, ctas, chunks = deal.segment(b, s)
            if deal.grp == 1:
                K, V = case.kseq[b, s, :p], case.vseq[b, s, :p]
                kn, vn = case.kseq[b, s, p], case.vseq[b, s, p]
                parts = [emulate_stream_partial(case.q[b, s], K, V, kn, vn, p, ch, ch[-1] == deal.nch[b] - 1, dt, mutation)
                         for ch in chunks]
                m, l, a = zip(*parts)
                out[b, s] = _merge([(np.array([mm]), np.array([ll]), aa[None]) for mm, ll, aa in zip(m, l, a)], dt,
                                   mutation)[0]
                continue
            kv, qg = divmod(s, deal.NQG)
            heads = np.arange(kv * deal.grp + qg * deal.GP, min((kv + 1) * deal.grp, kv * deal.grp + (qg + 1) * deal.GP))
            # which KV head each query head reads; "kv_mod" is the i mod Hkv mix-up (rows of a tile are independent)
            src = heads % case.Hkv if mutation == "kv_mod" else heads // deal.grp
            for kvs in np.unique(src):
                hs = heads[src == kvs]
                Q = np.zeros((deal.GP, D), np.float32)
                Q[:len(hs)] = case.q[b, hs]
                K, V = case.kseq[b, kvs, :p], case.vseq[b, kvs, :p]
                kn, vn = case.kseq[b, kvs, p], case.vseq[b, kvs, p]
                parts = [emulate_gqa_partial(Q, K, V, kn, vn, p, ch, ch[-1] == deal.nch[b] - 1, dt, mutation) for ch in chunks]
                out[b, hs] = _merge(parts, dt, mutation)[:len(hs)]
    return out
