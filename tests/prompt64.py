"""Float64 reference, per-element bound and float32 emulation of AttentionKVCache over a prompt chunk
(it_b200_attention_kvcache_prompt: kvcache_append_kernel + attention_kvcache_prompt_kernel in attention_prefill.cu).

Reference.  Batch row b holds a sequence of p_b + S rows per KV head; rows p_b .. p_b + S - 1 are the chunk's k / v.  Query i
of head h is a single-token AttentionKVCache at position p_b + i: with s_j = q_i.k_j / sqrt(D) over rows j = 0 .. p_b + i of
KV head h / G, w = softmax(s) and ref = sum_j w_j v_j, every output element must satisfy tests/attn64.py's bound

    |got - ref| <= ulp_T(|ref|) + 2^-16 sum_j w_j |v_j| + c_s 2^-24 sum_j w_j a_j |v_j - ref|  [+ 2^-25 sum_j |v_j| / L, f16]

with its terms re-derived for this kernel:
* c_s = 32 (attn64.C_SCORE).  S = Q K^T is a chain of D / 16 wgmma k16 steps into fp32 accumulators (8 at D = 128, 4 at
  D = 64), each counted as 2 units of roundoff (truncation allowed), and the fp32 scale by 1/sqrt(D) adds 2: at most
  18 x 2^-24 a_j.
* 2^-16 sum w|v|: the online softmax over 64-key tiles.  Per tile O is rescaled once and takes 2 x 4 k16 steps (hi and lo
  P operands); at p_b + S = 1777 rows that is 28 tiles, about 476 roundings of partial sums no larger than sum p|v| -- 2^-15.1
  if every one erred the same way, about 2^-19.6 for rounding errors of random sign (the argument attn64 makes for its
  longest merge chain).  P enters the product as hi + lo in T: 16 (bf16) / 22 (f16) significant bits, <= 2^-17 relative.
* 2^-25 sum |v| / L for f16: hi and lo of P are f16, whose subnormals carry up to 2^-25 absolute error per weight, as in
  attn_gqa_kernel.

The float32 emulation below follows the kernel's order of operations per 64-query tile; test_prompt_kvcache_host.py checks
that it stays within half of the bound on every score regime and that each of a set of injected bugs leaves the bound.
"""
import math

import numpy as np

import oracle
from tests import attn64

F16, BF16 = 10, 16
BQ = BK = 64
REGIMES = ["flat", "late", "early", "sink", "diag", "neg150", "pos200"]


def scale32(D):
    return np.float32(0.08838834764831845 if D == 128 else 0.125)


class Case:
    """One prompt chunk: B batch rows, Hq query heads over Hkv KV heads of width D, S new tokens at starts p [B] (already
    clamped) in caches of S_max rows.  kseq / vseq [B, Hkv, S_max, D] hold every row a query may read (rows >= p_b + S are
    NaN); q [B, Hq, S, D].  Query head h of batch row b carries regime REGIMES[(b Hq + h + offset) % 7]: its G query heads
    get orthogonal directions u_r, every key carries a component along each u_r that sets head r's scores, and the rest of
    q and k lies in the orthogonal complement (random, the flat part of every score)."""

    def __init__(self, B, Hq, Hkv, S, S_max, p, D, seed, offset=0, regimes=REGIMES):
        self.B, self.Hq, self.Hkv, self.S, self.S_max, self.D, self.G = B, Hq, Hkv, S, S_max, D, Hq // Hkv
        self.p = np.broadcast_to(np.asarray(p, np.int64), (B,)).copy()
        assert np.all(self.p + S <= S_max) and Hq // Hkv <= D
        rng = np.random.default_rng(seed)
        G = self.G
        self.q = np.empty((B, Hq, S, D), np.float32)
        self.kseq = np.full((B, Hkv, S_max, D), np.nan, np.float32)
        self.vseq = np.full((B, Hkv, S_max, D), np.nan, np.float32)
        self.regime = np.empty((B, Hq), object)
        a = math.sqrt(32.0)
        for b in range(B):
            n = int(self.p[b]) + S
            vrow = np.exp2((np.arange(n) % 5) - 2.0)
            for kv in range(Hkv):
                basis, _ = np.linalg.qr(rng.standard_normal((D, D)))
                U, W = basis[:, :G], basis[:, G:]  # head directions, complement
                z = rng.standard_normal((n, D - G)) * 0.5 @ W.T
                c = np.zeros((n, G))
                for r in range(G):
                    h = kv * G + r
                    reg = regimes[(b * Hq + h + offset) % len(regimes)]
                    self.regime[b, h] = reg
                    c[:, r] = self._targets(reg, n, int(self.p[b]), rng) * math.sqrt(D) / a
                    w = rng.standard_normal((S, D - G)) * 0.5 @ W.T
                    self.q[b, h] = attn64.exact(a * U[:, r][None, :] + w)
                self.kseq[b, kv, :n] = attn64.exact(z + c @ U.T)
                v = rng.standard_normal((n, D)) * 0.5 * vrow[:, None] * 2.0 ** ((kv % 3) - 1)
                self.vseq[b, kv, :n] = attn64.exact(v)

    @staticmethod
    def _targets(reg, n, p, rng):
        """head r's score target for each of the n rows (0: the flat, random part only)"""
        t = np.zeros(n)
        peaks = sorted({int(round(f * (n - 1))) for f in (0.1, 0.35, 0.6, 0.85)})
        if reg == "late":
            t[peaks] = 6.0 + 3.0 * np.arange(len(peaks))
        elif reg == "early":
            t[peaks] = 15.0 - 3.0 * np.arange(len(peaks))
        elif reg == "sink":
            t[0] = 20.0
        elif reg == "diag":  # the chunk's own rows: query i's largest scores are its own row and the chunk rows before it
            t[p:] = 12.0
        elif reg == "neg150":
            t[:] = -150.0 + 3.0 * rng.standard_normal(n)
        elif reg == "pos200":
            top = (2 * (n - 1)) // 3
            t[:] = 200.0 - np.abs(np.arange(n) - top)
        return t

    def inputs(self):
        """(k cache, v cache, k, v): the caches hold rows < p_b, NaN from p_b on; k / v [B, Hkv, S, D] are the chunk's rows"""
        kc, vc = self.kseq.copy(), self.vseq.copy()
        k = np.empty((self.B, self.Hkv, self.S, self.D), np.float32)
        v = np.empty_like(k)
        for b in range(self.B):
            p = int(self.p[b])
            k[b], v[b] = self.kseq[b, :, p:p + self.S], self.vseq[b, :, p:p + self.S]
            kc[b, :, p:] = np.nan
            vc[b, :, p:] = np.nan
        return kc, vc, k, v

    def reference(self):
        """float64 (ref, sum w|v|, sum w a |v - ref|, sum |v| / L), each [B, Hq, S, D]"""
        B, Hq, S, D, G = self.B, self.Hq, self.S, self.D, self.G
        out = [np.empty((B, Hq, S, D)) for _ in range(4)]
        for b in range(B):
            p = int(self.p[b])
            n = p + S
            lim = p + np.arange(S)
            mask = np.arange(n)[None, :] > lim[:, None]  # [S, n]
            for kv in range(self.Hkv):
                K = self.kseq[b, kv, :n].astype(np.float64)
                V = self.vseq[b, kv, :n].astype(np.float64)
                for h in range(kv * G, (kv + 1) * G):
                    Q = self.q[b, h].astype(np.float64)
                    s = np.where(mask, -np.inf, Q @ K.T / math.sqrt(D))
                    a = np.abs(Q) @ np.abs(K).T / math.sqrt(D)
                    e = np.exp(s - s.max(1, keepdims=True))
                    L = e.sum(1, keepdims=True)
                    w = e / L
                    ref = w @ V
                    out[0][b, h], out[1][b, h] = ref, w @ np.abs(V)
                    wa = (w * a).astype(np.float32)
                    Vf, rf = V.astype(np.float32), ref.astype(np.float32)
                    for i0 in range(0, S, 64):  # sum_j w_j a_j |v_j - ref_i|, 64 queries at a time
                        sl = slice(i0, min(i0 + 64, S))
                        out[2][b, h, sl] = np.einsum("ij,ijd->id", wa[sl], np.abs(Vf[None] - rf[sl, None]))
                    out[3][b, h] = (np.where(mask, 0.0, 1.0) @ np.abs(V)) / L
        return out


def bound(refs, dt):
    return attn64.bound(refs, dt, True)


def violations(got, refs, dt, scale=1.0):
    return ~(np.abs(np.asarray(got, np.float64) - refs[0]) <= scale * bound(refs, dt))


def report(bad, got, refs, dt, case, what, limit=4):
    if not bad.any():
        return None
    bd = bound(refs, dt)
    lines = [f"{what}: {int(bad.sum())} of {bad.size} elements outside the bound"]
    rows = sorted({(int(b), int(h), int(i)) for b, h, i, _ in np.argwhere(bad)})
    for b, h, i in rows[:limit]:
        d = int(np.argmax(np.where(bad[b, h, i], np.abs(got[b, h, i] - refs[0][b, h, i]) / bd[b, h, i], -1)))
        lines.append(f"  batch row {b} (p {int(case.p[b])}), head {h} ({case.regime[b, h]}), token {i} (query tile {i // BQ}), "
                     f"column {d}: got {float(got[b, h, i, d])!r}, float64 {refs[0][b, h, i, d]!r}, bound {bd[b, h, i, d]:.3g}")
    if len(rows) > limit:
        lines.append(f"  ... {len(rows)} query rows in all")
    return "\n".join(lines)


# ====================================================================== float32 emulation of the kernel
_f, _fma, _exp = attn64._f, attn64._fma, attn64._exp
MUTATIONS = ["round_p_once", "causal_off_by_one", "append_shifted", "kv_mod", "skip_diag_tile"]


def emulate(case, dt, mutation=None):
    """the kernel's output [B, Hq, S, D] as float32"""
    with np.errstate(invalid="ignore", over="ignore"):
        return _emulate(case, dt, mutation)


def _cache_rows(case, b, kv, mutation):
    """the cache of (b, kv) after the append launch: rows < p_b as given, the chunk at p_b .. (shifted by one: the row at p_b
    keeps its NaN poison)"""
    kc, vc, k, v = case.inputs()
    K, V = kc[b, kv].copy(), vc[b, kv].copy()
    p, S = int(case.p[b]), case.S
    d = 1 if mutation == "append_shifted" else 0
    n = min(S, case.S_max - p - d)
    K[p + d:p + d + n], V[p + d:p + d + n] = k[b, kv, :n], v[b, kv, :n]
    return K, V


def _emulate(case, dt, mutation):
    B, Hq, S, D, G = case.B, case.Hq, case.S, case.D, case.G
    out = np.empty((B, Hq, S, D), np.float32)
    sc = scale32(D)
    for b in range(B):
        p = int(case.p[b])
        for h in range(Hq):
            kv = h % case.Hkv if mutation == "kv_mod" else h // G
            K, V = _cache_rows(case, b, kv, mutation)
            K = np.pad(K, ((0, BK), (0, 0)))  # the tensor map's zero fill past S_max
            V = np.pad(V, ((0, BK), (0, 0)))
            for i0 in range(0, S, BQ):
                Q = np.zeros((BQ, D), np.float32)
                nq = min(BQ, S - i0)
                Q[:nq] = case.q[b, h, i0:i0 + nq]
                lim = p + np.minimum(i0 + np.arange(BQ), S - 1) + (1 if mutation == "causal_off_by_one" else 0)
                last = p + min(i0 + BQ - 1, S - 1)
                m = np.full(BQ, -np.inf, np.float32)
                l = np.zeros(BQ, np.float32)
                o = np.zeros((BQ, D), np.float32)
                for t in range(last // BK + 1):
                    j0 = t * BK
                    diag = j0 + BK - 1 > p + i0
                    if diag and mutation == "skip_diag_tile":
                        continue
                    Kt, Vt = K[j0:j0 + BK].copy(), V[j0:j0 + BK].copy()
                    if j0 + BK > p + S:
                        Vt[p + S - j0:] = 0
                    d = np.zeros((BQ, BK), np.float32)
                    for kk in range(D // 16):
                        sl = slice(16 * kk, 16 * kk + 16)
                        d = _f(d + Q[:, sl].astype(np.float64) @ Kt[:, sl].T.astype(np.float64))
                    keys = j0 + np.arange(BK)
                    s = np.where(diag & (keys[None, :] > lim[:, None]), -np.inf, _f(d * sc)).astype(np.float32)
                    mx = np.maximum(m, s.max(1))
                    pr = _exp(s - mx[:, None])
                    hi = oracle.round_to(pr, dt)
                    lo = np.zeros_like(pr) if mutation == "round_p_once" else oracle.round_to(_f(pr - hi), dt)
                    # per lane: columns 8 j + 2 lane + e in order (j, e), then the xor-1 and xor-2 shuffles
                    lane = pr.reshape(BQ, 8, 4, 2).transpose(0, 2, 1, 3).reshape(BQ, 4, 16)
                    ts = np.zeros((BQ, 4), np.float32)
                    for e in range(16):
                        ts = _f(ts + lane[:, :, e])
                    ts = _f(ts + ts[:, [1, 0, 3, 2]])
                    ts = _f(ts + ts[:, [2, 3, 0, 1]])
                    corr = _exp(m - mx)
                    l = _fma(l, corr, ts[:, 0])
                    o = _f(o * corr[:, None])
                    for P in (hi, lo):
                        for kk in range(BK // 16):
                            sl = slice(16 * kk, 16 * kk + 16)
                            o = _f(o + P[:, sl].astype(np.float64) @ Vt[sl].astype(np.float64))
                    m = mx
                with np.errstate(divide="ignore"):
                    inv = _f(np.float32(1) / l)
                out[b, h, i0:i0 + nq] = oracle.round_to(_f(o * inv[:, None]), dt)[:nq]
    return out
