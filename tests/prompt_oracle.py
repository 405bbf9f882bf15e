"""AttentionKVCache over a prompt chunk of S > 1 tokens for the tests: S single-token AttentionKVCache steps in order.

Token i of batch row b is step i at position p_b + i: its k / v are appended at cache row p_b + i and query i attends over rows
0 .. p_b + i.  p_b is element 0 of the positions, or (per-row positions) row b's first element, flat index b * (numel / B), so
a [B, S] position tensor and a [B, 1] one both work; p_b is clamped to [0, S_max - S].  The single-token step is the oracle's
own (through HeadWidthOracleHandler: grouped-query heads and 64-wide heads), so S = 1 graphs run exactly as before."""
import numpy as np

from tests.head64_oracle import HeadWidthOracleHandler, attention_kvcache_d


def prompt_starts(pos, B, S, S_max, per_row):
    """p_b for every batch row"""
    pv = np.asarray(pos).ravel().astype(np.int64)
    start = pv[np.arange(B) * (pv.size // B)] if per_row else np.full(B, pv[0])
    return np.clip(start, 0, S_max - S)


def attention_kvcache_prompt(kc, vc, q, k, v, pos, dt, per_row=False):
    """in place on kc / vc (float32, C-contiguous [B, Hkv, S_max, D]); q [B, Hq, S, D], k / v [B, Hkv, S, D]; returns
    [B, Hq, S, D] float32 rounded to dt"""
    B, S = q.shape[0], q.shape[2]
    start = prompt_starts(pos, B, S, kc.shape[2], per_row)
    tok = [np.asarray(t, np.float32) for t in (q, k, v)]
    return np.concatenate([attention_kvcache_d(kc, vc, *(np.ascontiguousarray(t[:, :, i:i + 1]) for t in tok), start + i, dt)
                           for i in range(S)], axis=2)


class PromptOracleHandler(HeadWidthOracleHandler):
    """The graph oracle with AttentionKVCache over S >= 1 new tokens (S = 1: HeadWidthOracleHandler's own step)."""

    def attentionKVCache(self, kc, vc, q, k, v, pos, y, per_row_positions=False):
        if q.dims[2] == 1:
            return super().attentionKVCache(kc, vc, q, k, v, pos, y, per_row_positions)
        out = self._out(y, q.dims, q.dt)
        return self._rec(lambda: attention_kvcache_prompt(kc.value, vc.value, q.value, k.value, v.value, pos.value, q.dt,
                                                          per_row_positions), [kc, vc, q, k, v, pos], [out])
