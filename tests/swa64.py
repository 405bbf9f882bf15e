"""Float64 reference, per-element bound and float32 emulation of sliding-window AttentionKVCache (window W >= 1: the query
at position P reads cache rows (P - W, P] only).

Decode (attn_stream_win_kernel / attn_gqa_win_kernel).  A windowed head at position P runs exactly as an unwindowed head at
span = min(P, W - 1) over the cache rows from lo = P - span up: the same units, dealing and order of operations.  `deal`
is therefore tests/attn64.py's `Deal` at the span positions, and the float64 reference and bound are attn64's over rows
[lo, P] (`decode_refs`).

Prompt (attention_kvcache_prompt_win_kernel).  `Case` is tests/prompt64.py's chunk with a window: the reference masks key j
of query i (position p_b + i) unless p_b + i - W < j <= p_b + i, and the cache rows below the first query's window,
max(0, p_b - W + 1), are NaN, so a row that leaks into an output shows.  The bound is prompt64's.  `emulate` follows the
kernel per 64-query tile: key tiles from the one holding the tile's first query's window start, V rows below that start
zeroed, the leading edge masked per element, and a row's exponentials taken against 0 while it has met only masked keys.
`SLIPS` are the injected bugs the host tests show leave the bound.
"""
import math

import numpy as np

import oracle
from tests import attn64, prompt64

BQ = BK = prompt64.BQ
SLIPS = ["window_plus_one", "window_minus_one", "window_from_last_query", "no_lead_mask", "v_not_zeroed",
         "element0_lo_per_row", "no_max_guard"]


# ====================================================================== decode
def span(pos, window, S_max):
    """rows read below each (clamped) position: min(P, W - 1)"""
    p = np.clip(np.asarray(pos, np.int64), 0, S_max - 1)
    return np.minimum(p, window - 1)


def deal(dt, B, Hq, Hkv, S_max, pos, window, d=128, kv8=False):
    """attn64.Deal of the windowed kernels: the unwindowed dealing at the span positions"""
    return attn64.Deal(dt, B, Hq, Hkv, S_max, np.broadcast_to(span(pos, window, S_max), (B,)), d, kv8)


def split_states(dl):
    """the numbers of CTAs sharing each segment of a Deal"""
    return sorted({len(dl.segment(b, s)[1]) for b in range(dl.B) for s in range(dl.segs)})


def decode_refs(kc, vc, q, pos, window):
    """attn64's (ref, sum w|v|, sum w a |v - ref|, sum |v| / L), each [B, Hq, D], of one windowed decode step over caches
    kc / vc [B, Hkv, S_max, D] (float values, the appended row already in place); pos one per batch row (clamped)"""
    B, Hkv, S_max, D = kc.shape
    Hq = q.shape[1]
    G = Hq // Hkv
    out = [np.zeros((B, Hq, D)) for _ in range(4)]
    for b in range(B):
        P = int(np.clip(pos[b], 0, S_max - 1))
        lo = max(0, P - window + 1)
        for h in range(Hq):
            K = np.asarray(kc[b, h // G, lo:P + 1], np.float64)
            V = np.asarray(vc[b, h // G, lo:P + 1], np.float64)
            Q = np.asarray(q[b, h, 0], np.float64)
            s = K @ Q / math.sqrt(D)
            a = np.abs(K) @ np.abs(Q) / math.sqrt(D)
            e = np.exp(s - s.max())
            L = e.sum()
            w = e / L
            ref = w @ V
            out[0][b, h], out[1][b, h] = ref, w @ np.abs(V)
            out[2][b, h] = (w * a) @ np.abs(V - ref)
            out[3][b, h] = np.abs(V).sum(0) / L
    return out


# ====================================================================== prompt
class Case(prompt64.Case):
    """prompt64.Case with a window: rows below max(0, p_b - window + 1) of every KV head are NaN"""

    def __init__(self, B, Hq, Hkv, S, S_max, p, D, seed, window, offset=0):
        super().__init__(B, Hq, Hkv, S, S_max, p, D, seed, offset)
        self.window = window
        for b in range(B):
            lo = self.lo(b)
            self.kseq[b, :, :lo] = np.nan
            self.vseq[b, :, :lo] = np.nan

    def lo(self, b):
        """the first row any query of batch row b reads"""
        return max(0, int(self.p[b]) - self.window + 1)

    def reference(self):
        """float64 (ref, sum w|v|, sum w a |v - ref|, sum |v| / L), each [B, Hq, S, D], over each query's window"""
        B, Hq, S, D, G, W = self.B, self.Hq, self.S, self.D, self.G, self.window
        out = [np.empty((B, Hq, S, D)) for _ in range(4)]
        for b in range(B):
            p, lo = int(self.p[b]), self.lo(b)
            n = p + S
            j = np.arange(lo, n)[None, :]
            lim = p + np.arange(S)[:, None]
            mask = (j > lim) | (j <= lim - W)  # [S, n - lo]
            for kv in range(self.Hkv):
                K = self.kseq[b, kv, lo:n].astype(np.float64)
                V = self.vseq[b, kv, lo:n].astype(np.float64)
                for h in range(kv * G, (kv + 1) * G):
                    Q = self.q[b, h].astype(np.float64)
                    s = np.where(mask, -np.inf, Q @ K.T / math.sqrt(D))
                    a = np.where(mask, 0.0, np.abs(Q) @ np.abs(K).T / math.sqrt(D))
                    e = np.exp(s - s.max(1, keepdims=True))
                    L = e.sum(1, keepdims=True)
                    w = e / L
                    ref = w @ V
                    out[0][b, h], out[1][b, h] = ref, w @ np.abs(V)
                    wa = w * a
                    out[2][b, h] = np.einsum("ij,ijd->id", wa, np.abs(V[None] - ref[:, None]))
                    out[3][b, h] = (np.where(mask, 0.0, 1.0) @ np.abs(V)) / L
        return out


def emulate(case, dt, slip=None):
    """the windowed prompt kernel's output [B, Hq, S, D] as float32"""
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        return _emulate(case, dt, slip)


def _emulate(case, dt, slip):
    _f, _fma, _exp = attn64._f, attn64._fma, attn64._exp
    B, Hq, S, D, G = case.B, case.Hq, case.S, case.D, case.G
    W = case.window + {"window_plus_one": 1, "window_minus_one": -1}.get(slip, 0)
    out = np.empty((B, Hq, S, D), np.float32)
    sc = prompt64.scale32(D)
    for b in range(B):
        p = int(case.p[b])
        pw = int(case.p[0]) if slip == "element0_lo_per_row" else p  # the position the window is measured from
        for h in range(Hq):
            K, V = prompt64._cache_rows(case, b, h // G, None)
            K = np.pad(K, ((0, BK), (0, 0)))
            V = np.pad(V, ((0, BK), (0, 0)))
            for i0 in range(0, S, BQ):
                Q = np.zeros((BQ, D), np.float32)
                nq = min(BQ, S - i0)
                Q[:nq] = case.q[b, h, i0:i0 + nq]
                lim = p + np.minimum(i0 + np.arange(BQ), S - 1)
                last = p + min(i0 + BQ - 1, S - 1)
                wlim = pw + np.minimum(i0 + np.arange(BQ), S - 1)
                if slip == "window_from_last_query":
                    wlim = np.full(BQ, last)
                lo0 = max(int(wlim[0]) - W + 1, 0)
                m = np.full(BQ, -np.inf, np.float32)
                l = np.zeros(BQ, np.float32)
                o = np.zeros((BQ, D), np.float32)
                for t in range(lo0 // BK, last // BK + 1):
                    j0 = t * BK
                    Kt, Vt = K[j0:j0 + BK].copy(), V[j0:j0 + BK].copy()
                    if j0 + BK > p + S:
                        Vt[p + S - j0:] = 0
                    if j0 < lo0 and slip != "v_not_zeroed":
                        Vt[:lo0 - j0] = 0
                    d = np.zeros((BQ, BK), np.float32)
                    for kk in range(D // 16):
                        sl = slice(16 * kk, 16 * kk + 16)
                        d = _f(d + Q[:, sl].astype(np.float64) @ Kt[:, sl].T.astype(np.float64))
                    keys = (j0 + np.arange(BK))[None, :]
                    masked = keys > lim[:, None]
                    if slip != "no_lead_mask":
                        masked |= keys <= wlim[:, None] - W
                    s = np.where(masked, -np.inf, _f(d * sc)).astype(np.float32)
                    mx = np.maximum(m, s.max(1))
                    mxe = mx if slip == "no_max_guard" else np.where(mx == -np.inf, np.float32(0), mx)
                    pr = _exp(s - mxe[:, None])
                    hi = oracle.round_to(pr, dt)
                    lo = oracle.round_to(_f(pr - hi), dt)
                    lane = pr.reshape(BQ, 8, 4, 2).transpose(0, 2, 1, 3).reshape(BQ, 4, 16)
                    ts = np.zeros((BQ, 4), np.float32)
                    for e in range(16):
                        ts = _f(ts + lane[:, :, e])
                    ts = _f(ts + ts[:, [1, 0, 3, 2]])
                    ts = _f(ts + ts[:, [2, 3, 0, 1]])
                    corr = _exp(m - mxe)
                    l = _fma(l, corr, ts[:, 0])
                    o = _f(o * corr[:, None])
                    for P in (hi, lo):
                        for kk in range(BK // 16):
                            sl = slice(16 * kk, 16 * kk + 16)
                            o = _f(o + P[:, sl].astype(np.float64) @ Vt[sl].astype(np.float64))
                    m = mx
                inv = _f(np.float32(1) / l)
                out[b, h, i0:i0 + nq] = oracle.round_to(_f(o * inv[:, None]), dt)[:nq]
    return out
