"""The Llama graph oracle with a rolling KV cache (a config's rolling_cache, AttentionKVCache's `rolling`), and the
device-vs-oracle pair built on it.

`RingOracleHandler` is tests/swa_oracle.py's `SwaOracleHandler` whose AttentionKVCache also takes `rolling`: the caches
[B, Hkv, S_max, D] are a ring, position P in row P mod S_max.  A single-token step at position P gathers the rows of
positions lo .. P - 1 (lo = max(0, P - window + 1)) from the ring into a linear cache, runs swa_oracle's windowed step there
at position P - lo, and stores the appended row back at row P mod S_max.  Positions are clamped to [0, ring_pos_max], the
kernels' bound, with no S_max - 1 or S_max - S limit.  A prompt chunk is S such steps in order."""
from types import SimpleNamespace

import numpy as np

from tests import llama_oracle as LO
from tests import swa_oracle as SO

INT32_MAX = 2**31 - 1


def ring_pos_max(S_max):
    """the largest position a ring of S_max rows takes (common.cuh's ring_pos_max)"""
    return INT32_MAX - int(S_max)


def ring_rows(lo, hi, S_max):
    """the ring rows of positions lo .. hi - 1"""
    return np.arange(lo, hi, dtype=np.int64) % S_max


def ring_step(kc, vc, q, k, v, pos, dt, window, scales=None):
    """One rolling-cache AttentionKVCache step on float32 arrays (FP8: uint8 codes with scales = (k_scale, v_scale)), in place
    on the rings kc / vc.  pos: one position per batch row.  Returns [B, Hq, 1, D] float32 rounded to dt."""
    B, S_max = kc.shape[0], kc.shape[2]
    pos = np.clip(np.asarray(pos, np.int64).reshape(B), 0, ring_pos_max(S_max))
    outs = []
    for b in range(B):
        p = int(pos[b])
        lo = SO.window_start(p, window)
        rows = ring_rows(lo, p + 1, S_max)  # (the last one, P's row, is overwritten by the append)
        lk, lv = np.ascontiguousarray(kc[b:b + 1, :, rows]), np.ascontiguousarray(vc[b:b + 1, :, rows])
        sl = lambda t: np.ascontiguousarray(np.asarray(t)[b:b + 1])
        outs.append(SO.window_step(lk, lv, sl(q), sl(k), sl(v), [p - lo], dt, window, scales))
        kc[b, :, p % S_max], vc[b, :, p % S_max] = lk[0, :, p - lo], lv[0, :, p - lo]
    return np.concatenate(outs)


def ring_starts(pos, B, S_max, per_row):
    """p_b as llama_oracle.prompt_starts, clamped to [0, ring_pos_max] instead of [0, S_max - S]"""
    pv = np.asarray(pos).ravel().astype(np.int64)
    start = pv[np.arange(B) * (pv.size // B)] if per_row else np.full(B, pv[0])
    return np.clip(start, 0, ring_pos_max(S_max))


def ring_prompt(kc, vc, q, k, v, pos, dt, window, per_row=False):
    """S rolling-cache steps: token i of batch row b at position p_b + i.  Returns [B, Hq, S, D] float32 rounded to dt."""
    B, S = q.shape[0], q.shape[2]
    start = ring_starts(pos, B, kc.shape[2], per_row)
    tok = [np.asarray(t, np.float32) for t in (q, k, v)]
    return np.concatenate([ring_step(kc, vc, *(np.ascontiguousarray(t[:, :, i:i + 1]) for t in tok), start + i, dt, window)
                           for i in range(S)], axis=2)


def check_ring(window, S_max, S):
    """the shape rule of a rolling cache, with the operator's messages"""
    if window < 1:
        raise ValueError("AttentionKVCache: a rolling cache needs a window >= 1")
    if S_max < window:
        raise ValueError(f"AttentionKVCache: a rolling cache of {S_max} rows is shorter than the window of {window}")
    if S_max % 64:
        raise ValueError(f"AttentionKVCache: a rolling cache's length {S_max} is not a multiple of 64")
    if S_max < window + S - 1:
        raise ValueError(f"AttentionKVCache: a chunk of {S} tokens needs a rolling cache of window + {S - 1} = "
                         f"{window + S - 1} rows or more, not {S_max} (split the prompt)")


class RingOracleHandler(SO.SwaOracleHandler):
    """SwaOracleHandler whose windowed AttentionKVCache may run over a rolling cache"""

    rolling_cache = True

    def attentionKVCache(self, kc, vc, q, k, v, pos, y, per_row_positions=False, k_scale=None, v_scale=None, window=0,
                         rolling=False):
        if not rolling:
            return super().attentionKVCache(kc, vc, q, k, v, pos, y, per_row_positions, k_scale, v_scale, window)
        B, S, S_max = q.dims[0], q.dims[2], kc.dims[2]
        if S > 1 and k_scale is not None:
            raise ValueError("AttentionKVCache: an FP8 KV cache takes one new token per step (S = 1)")
        check_ring(window, S_max, S)
        out = self._out(y, q.dims, q.dt)

        def run():
            if S > 1:
                return ring_prompt(kc.value, vc.value, q.value, k.value, v.value, pos.value, q.dt, window, per_row_positions)
            pv = np.asarray(pos.value).ravel().astype(np.int64)
            p = pv[:B] if per_row_positions else np.full(B, pv[0])
            scales = None if k_scale is None else (k_scale.value, v_scale.value)
            return ring_step(kc.value, vc.value, q.value, k.value, v.value, p, q.dt, window, scales)
        ins = [kc, vc, q, k, v, pos] + ([] if k_scale is None else [k_scale, v_scale])
        return self._rec(run, ins, [out])


def oracle_graph(cfg, seq=1, caches=None):
    """(RingOracleHandler, graph) for (cfg, seq) with fill_llama_weights_host's weights and `caches` (default llama_caches)"""
    from infinitensor_b200 import graphs as G
    oh = RingOracleHandler()
    og = G.build_llama_decode(oh, cfg, seq=seq)
    G.fill_llama_weights_host(og)
    LO.load_caches(og, LO.llama_caches(cfg) if caches is None else caches)
    return oh, og


def llama_pair(cfg, seq=1, env=None, caches=None, oracle_caches=None, rt=None):
    """llama_oracle.llama_pair with the oracle side on RingOracleHandler"""
    from infinitensor_b200 import backend as B
    from infinitensor_b200 import graphs as G
    rt = rt or B.CudaRuntime(0)
    h = B.GraphHandler(rt)
    with LO._environ(env or {}):
        g = G.build_llama_decode(h, cfg, seq=seq)
        h.data_malloc()
        sched = h.schedule()
    G.fill_llama_weights_host(g)
    caches = LO.llama_caches(cfg) if caches is None else caches
    LO.load_caches(g, caches)
    oh, og = oracle_graph(cfg, seq, caches if oracle_caches is None else oracle_caches)
    return SimpleNamespace(cfg=cfg, rt=rt, h=h, g=g, oh=oh, og=og, schedule=sched)
