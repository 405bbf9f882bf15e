"""Oracle pieces for 64-wide heads (GPT-2, TinyLlama): AttentionKVCache with the 1/sqrt(D) scale and RoPE with a head width.

The oracle's own AttentionKVCache restates the reference, whose scale is 1/sqrt(128) whatever D is (attention_kvcache.cu:72),
and the oracle graph handler's RoPE rotates 128-wide heads (rope.cc:25).  The kernels extend both to D = 64 with the rule
models with such heads use: scale 1/sqrt(D), rotate-half within each D-wide head.  At D = 128 everything here is the
oracle's own code, so a 128-wide graph is checked exactly as before."""
import math

import numpy as np

import oracle as O
from tests.gqa_oracle import GqaOracleHandler, attention_kvcache_gqa


def attention_kvcache_d(kc, vc, q, k, v, pos, dt):
    """AttentionKVCache at head width D = kc.shape[3] on float32 arrays; in place on kc / vc.  pos: one int (every batch row)
    or one per batch row.  Query head i reads KV head i // (Hq / Hkv).  D = 128 is the oracle's AttentionKVCache; other
    widths are a float64 softmax of q.k / sqrt(D) over rows 0 .. pos, the output rounded to dt once."""
    B, Hkv, S, D = kc.shape
    if D == 128:
        return attention_kvcache_gqa(kc, vc, q, k, v, pos, dt)
    Hq = q.shape[1]
    G = Hq // Hkv
    posv = np.broadcast_to(np.asarray(pos, np.int64).ravel(), (B,)) if np.ndim(pos) else np.full(B, int(pos), np.int64)
    out = np.empty((B, Hq, 1, D), np.float32)
    for b in range(B):
        p = int(min(max(int(posv[b]), 0), S - 1))
        kc[b, :, p] = k[b, :, 0]
        vc[b, :, p] = v[b, :, 0]
        K = kc[b, :, :p + 1].astype(np.float64)
        V = vc[b, :, :p + 1].astype(np.float64)
        Q = np.asarray(q[b, :, 0], np.float64).reshape(Hkv, G, D)
        s = np.einsum("hgd,hsd->hgs", Q, K) / math.sqrt(D)
        w = np.exp(s - s.max(-1, keepdims=True))
        w /= w.sum(-1, keepdims=True)
        out[b, :, 0] = np.einsum("hgs,hsd->hgd", w, V).reshape(Hq, D)
    return O.round_to(out, dt)


class HeadWidthOracleHandler(GqaOracleHandler):
    """The grouped-query graph oracle with RoPE(dim_head) and AttentionKVCache at the caches' head width."""

    head_widths = (64, 128)

    def RoPE(self, pos, x, y, dim_head=128):
        out = self._out(y, x.dims, x.dt)
        return self._rec(lambda: O.rope(pos.value, x.value, dim_head, x.dt), [pos, x], [out])

    def attentionKVCache(self, kc, vc, q, k, v, pos, y, per_row_positions=False):
        if q.dims[3] == 128:
            return super().attentionKVCache(kc, vc, q, k, v, pos, y, per_row_positions)
        out = self._out(y, q.dims, q.dt)

        def run():
            pv = np.asarray(pos.value).ravel()
            p = pv[:q.dims[0]] if per_row_positions else int(pv[0])
            return attention_kvcache_d(kc.value, vc.value, q.value, k.value, v.value, p, q.dt)
        return self._rec(run, [kc, vc, q, k, v, pos], [out])
