"""The Llama graph oracle with RoPE from an inv_freq table (a config's rope_theta / rope_scaling), and the device-vs-oracle
pair built on it.

`RopeOracleHandler` is tests/llama_oracle.py's `LlamaOracleHandler` whose RoPE also takes the optional inv_freq input:
`rope_freq`, the kernels' angle rule with cos / sin in float64.  `oracle_graph` and `llama_pair` are llama_oracle's, building
the oracle side on this handler; `llama_step`, `rel_err`, `check_appended_k` and the rest are used from llama_oracle as they
are."""
from types import SimpleNamespace

import numpy as np

import oracle as O
from tests import llama_oracle as LO


def rope_freq(pos, x, inv_freq, dim_head, dt):
    """RoPE with a table on float32 [B, S, dim_model]: column pair c of every dim_head-wide head rotates by the angle
    fp32(p * inv_freq[c]) (one float32 product, HF's inv_freq @ position_ids); cos / sin in float64, rounded to float32 and
    then to dt; each product and the sum rounded to dt, as the kernels do"""
    x = np.asarray(x, np.float32)
    B, S, dm = x.shape
    half = dim_head // 2
    p = np.asarray(pos).reshape(B, S).astype(np.int64).astype(np.int32).astype(np.float32)
    ang = p[:, :, None] * np.asarray(inv_freq, np.float32)[None, None, :half]
    cs = O.round_to(np.cos(ang.astype(np.float64)).astype(np.float32), dt)[:, :, None, :]
    sn = O.round_to(np.sin(ang.astype(np.float64)).astype(np.float32), dt)[:, :, None, :]
    xh = x.reshape(B, S, dm // dim_head, dim_head)
    lo, hi = xh[..., :half], xh[..., half:]
    r = lambda a: O.round_to(a, dt)
    out = np.concatenate([r(r(lo * cs) - r(hi * sn)), r(r(hi * cs) + r(lo * sn))], axis=-1)
    return out.reshape(B, S, dm)


class RopeOracleHandler(LO.LlamaOracleHandler):
    """LlamaOracleHandler whose RoPE takes an inv_freq table"""

    rope_inv_freq = True

    def RoPE(self, pos, x, y, dim_head=128, inv_freq=None):
        if inv_freq is None:
            return super().RoPE(pos, x, y, dim_head)
        out = self._out(y, x.dims, x.dt)
        return self._rec(lambda: rope_freq(pos.value, x.value, inv_freq.value, dim_head, x.dt), [pos, x, inv_freq], [out])


def oracle_graph(cfg, seq=1, caches=None):
    """(RopeOracleHandler, graph) for (cfg, seq) with fill_llama_weights_host's weights and `caches` (default llama_caches)"""
    from infinitensor_b200 import graphs as G
    oh = RopeOracleHandler()
    og = G.build_llama_decode(oh, cfg, seq=seq)
    G.fill_llama_weights_host(og)
    LO.load_caches(og, LO.llama_caches(cfg) if caches is None else caches)
    return oh, og


def llama_pair(cfg, seq=1, env=None, caches=None, oracle_caches=None, rt=None):
    """llama_oracle.llama_pair with the oracle side on RopeOracleHandler"""
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
