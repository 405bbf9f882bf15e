"""Grouped-query AttentionKVCache for the tests: the oracle's AttentionKVCache restatement run once per group member.

With Hq = G * Hkv query heads, query head i attends over KV head i // G (HF repeat_kv order).  For each g in [0, G) the
query heads g, G + g, 2G + g, ... (q.reshape(B, Hkv, G, 1, D)[:, :, g]) form an equal-heads AttentionKVCache over the
caches; every pass appends the same k / v row.  GqaOracleHandler is the graph oracle with that rule, so that whole GQA
graphs can be checked like the equal-heads ones (tests/smoke_impl.run_llama_parity's criterion)."""
import numpy as np

import oracle as O
from oracle.graph_oracle import OracleHandler


def attention_kvcache_gqa(kc, vc, q, k, v, pos, dt):
    """In place on kc / vc (float32, C-contiguous); pos: one int (element-0 rule) or one per batch row."""
    B, Hkv, _, D = kc.shape
    Hq = q.shape[1]
    assert Hq % Hkv == 0
    G = Hq // Hkv
    q = np.ascontiguousarray(q, np.float32).reshape(B, Hkv, G, 1, D)
    out = np.empty_like(q)
    for g in range(G):
        qg = np.ascontiguousarray(q[:, :, g])
        if np.ndim(pos) == 0:
            out[:, :, g] = O.attention_kvcache(kc, vc, qg, k, v, int(pos), dt)
        else:
            for b in range(B):
                out[b:b + 1, :, g] = O.attention_kvcache(kc[b:b + 1], vc[b:b + 1], qg[b:b + 1], k[b:b + 1], v[b:b + 1],
                                                         int(pos[b]), dt)
    return out.reshape(B, Hq, 1, D)


class GqaOracleHandler(OracleHandler):
    def attentionKVCache(self, kc, vc, q, k, v, pos, y, per_row_positions=False):
        out = self._out(y, q.dims, q.dt)

        def run():
            pv = np.asarray(pos.value).ravel()
            p = pv[:q.dims[0]] if per_row_positions else int(pv[0])
            return attention_kvcache_gqa(kc.value, vc.value, q.value, k.value, v.value, p, q.dt)
        return self._rec(run, [kc, vc, q, k, v, pos], [out])


def run_gqa_llama_parity(cfg, pos=5, steps=2, cudagraph=True, tol=None):
    """run_llama_parity for a grouped-query config: device graph vs GqaOracleHandler, logits rel-to-max error and the
    appended k rows of layer 0.  Returns the worst logits error."""
    from infinitensor_b200 import backend as B
    from infinitensor_b200 import graphs as G

    rt = B.CudaRuntime(0)
    h = B.GraphHandler(rt)
    g = G.build_llama_decode(h, cfg)
    h.data_malloc()
    G.fill_llama_weights_host(g)
    oh = GqaOracleHandler()
    og = G.build_llama_decode(oh, cfg)
    G.fill_llama_weights_host(og)
    for li in range(cfg.layers):
        for which, (ct, oct_) in (("k", (g.k_caches[li], og.k_caches[li])), ("v", (g.v_caches[li], og.v_caches[li]))):
            vals = G.to_storage(G.llama_cache_values(cfg, li, which), cfg.dtype)
            ct.copyin_numpy(vals)
            oct_.copyin_numpy(vals)
    rng = np.random.default_rng(1)
    worst = 0.0
    t = tol or {1: 1e-3, 10: 4e-3, 16: 3e-2}[cfg.dtype]
    for step in range(steps):
        ids = rng.integers(0, cfg.vocab, size=(cfg.batch, 1)).astype(np.int64)
        p = np.full((cfg.batch, 1), pos + step, np.int64)
        for gg in (g, og):
            gg.input_ids.copyin_numpy(ids)
            gg.position_ids.copyin_numpy(p)
        if cudagraph:
            h.run_with_cudagraph()
        else:
            h.run()
        oh.run()
        got = G.from_storage(g.logits.copyout_numpy(), cfg.dtype).astype(np.float64)
        ref = og.logits.f32().astype(np.float64)
        err = np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-6)
        worst = max(worst, err)
        assert err < t, f"step {step}: logits rel-to-max error {err:.3e} >= {t}"
        k_got = G.from_storage(g.k_caches[0].copyout_numpy(), cfg.dtype)
        assert np.allclose(k_got[:, :, pos + step], og.k_caches[0].f32()[:, :, pos + step], rtol=t, atol=t)
    if cudagraph:
        assert rt.cuda_graph_capture_count() == 1, "graph must be captured once and replayed"
    return worst, h.schedule()
