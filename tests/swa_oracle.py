"""The Llama graph oracle with sliding-window attention (a config's sliding_window, AttentionKVCache's `window`), and the
device-vs-oracle pair built on it.

`SwaOracleHandler` is tests/rope_oracle.py's `RopeOracleHandler` whose AttentionKVCache also takes `window`.  A windowed
single-token step at position P is the oracle's own rule run on the shifted view of the cache: rows [lo, P] with
lo = max(0, P - window + 1), as a cache whose row 0 is row lo, at position P - lo (the appended row goes to row P of the
real cache).  That is `attention_kvcache_d` for 16-bit and fp32 caches and `kvfp8_oracle.attention` for FP8 ones.  A prompt
chunk is S windowed single-token steps in order.  `oracle_graph` and `llama_pair` are rope_oracle's, building the oracle side
on this handler."""
from types import SimpleNamespace

import numpy as np

from tests import kvfp8_oracle as KV
from tests import llama_oracle as LO
from tests import rope_oracle as RO


def window_start(p, window):
    """the first cache row the query at (clamped) position p reads"""
    return max(0, int(p) - int(window) + 1)


def window_step(kc, vc, q, k, v, pos, dt, window, scales=None):
    """One windowed single-token AttentionKVCache step on float32 arrays (FP8: uint8 codes with scales = (k_scale, v_scale)),
    in place on kc / vc.  pos: one position per batch row (clamped here to [0, S_max - 1]).  Returns [B, Hq, 1, D] float32
    rounded to dt."""
    B, S_max = kc.shape[0], kc.shape[2]
    pos = np.clip(np.asarray(pos, np.int64).reshape(B), 0, S_max - 1)
    outs = []
    for b in range(B):
        p = int(pos[b])
        lo = window_start(p, window)
        qb, kb, vb = (np.ascontiguousarray(np.asarray(t, np.float32)[b:b + 1]) for t in (q, k, v))
        if scales is not None:
            KV.append(kc[b:b + 1], vc[b:b + 1], kb, vb, scales[0], scales[1], np.array([p]))
            kview, vview = np.ascontiguousarray(kc[b:b + 1, :, lo:p + 1]), np.ascontiguousarray(vc[b:b + 1, :, lo:p + 1])
            ref, _ = KV.attention(kview, vview, scales[0], scales[1], qb, np.array([p - lo]), dt)
            outs.append(LO.O.round_to(ref.astype(np.float32), dt))
        else:
            kview, vview = np.ascontiguousarray(kc[b:b + 1, :, lo:p + 1]), np.ascontiguousarray(vc[b:b + 1, :, lo:p + 1])
            outs.append(LO.attention_kvcache_d(kview, vview, qb, kb, vb, p - lo, dt))
            kc[b, :, p], vc[b, :, p] = kview[0, :, p - lo], vview[0, :, p - lo]
    return np.concatenate(outs)


def window_prompt(kc, vc, q, k, v, pos, dt, window, per_row=False):
    """S windowed single-token steps: token i of batch row b is appended at row p_b + i and its query reads rows
    (p_b + i - window, p_b + i]; p_b as llama_oracle.prompt_starts.  Returns [B, Hq, S, D] float32 rounded to dt."""
    B, S = q.shape[0], q.shape[2]
    start = LO.prompt_starts(pos, B, S, kc.shape[2], per_row)
    tok = [np.asarray(t, np.float32) for t in (q, k, v)]
    return np.concatenate([window_step(kc, vc, *(np.ascontiguousarray(t[:, :, i:i + 1]) for t in tok), start + i, dt, window)
                           for i in range(S)], axis=2)


class SwaOracleHandler(RO.RopeOracleHandler):
    """RopeOracleHandler whose AttentionKVCache takes a sliding window"""

    sliding_window = True

    def attentionKVCache(self, kc, vc, q, k, v, pos, y, per_row_positions=False, k_scale=None, v_scale=None, window=0):
        if not window:
            return super().attentionKVCache(kc, vc, q, k, v, pos, y, per_row_positions, k_scale, v_scale)
        if window < 0:
            raise ValueError(f"AttentionKVCache: window {window} is negative")
        B, S = q.dims[0], q.dims[2]
        if S > 1 and k_scale is not None:
            raise ValueError("AttentionKVCache: an FP8 KV cache takes one new token per step (S = 1)")
        out = self._out(y, q.dims, q.dt)

        def run():
            if S > 1:
                return window_prompt(kc.value, vc.value, q.value, k.value, v.value, pos.value, q.dt, window, per_row_positions)
            pv = np.asarray(pos.value).ravel().astype(np.int64)
            p = pv[:B] if per_row_positions else np.full(B, pv[0])
            scales = None if k_scale is None else (k_scale.value, v_scale.value)
            return window_step(kc.value, vc.value, q.value, k.value, v.value, p, q.dt, window, scales)
        ins = [kc, vc, q, k, v, pos] + ([] if k_scale is None else [k_scale, v_scale])
        return self._rec(run, ins, [out])


def oracle_graph(cfg, seq=1, caches=None):
    """(SwaOracleHandler, graph) for (cfg, seq) with fill_llama_weights_host's weights and `caches` (default llama_caches)"""
    from infinitensor_b200 import graphs as G
    oh = SwaOracleHandler()
    og = G.build_llama_decode(oh, cfg, seq=seq)
    G.fill_llama_weights_host(og)
    LO.load_caches(og, LO.llama_caches(cfg) if caches is None else caches)
    return oh, og


def llama_pair(cfg, seq=1, env=None, caches=None, oracle_caches=None, rt=None):
    """llama_oracle.llama_pair with the oracle side on SwaOracleHandler"""
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
