"""The graph oracle for every Llama decode variant, and the loop that checks a device graph against it.

`LlamaOracleHandler` is `oracle.graph_oracle.OracleHandler` (the reference, restated) with the project's extensions, each
picked from the operands of the call:
* grouped-query heads: query head i attends over KV head i // (Hq / Hkv) (HF repeat_kv order), the oracle's AttentionKVCache
  run once per group member (`attention_kvcache_gqa`);
* 64-wide heads: RoPE(dim_head) rotates within each D-wide head, and AttentionKVCache at D != 128 is a float64 softmax at
  1 / sqrt(D) (`attention_kvcache_d`).  The reference's scale is 1/sqrt(128) whatever D is (attention_kvcache.cu:72) and its
  RoPE rotates 128-wide heads (rope.cc:25); at D = 128 everything is the oracle's own code;
* prompt chunks, S > 1 new tokens: S single-token steps in order (`attention_kvcache_prompt`);
* FP8 E4M3 caches (k_scale / v_scale given): tests/kvfp8_oracle.py's append and attention;
* MatMulNBits: tests/w4_oracle.py's layout, the decode rule for at most 64 rows and the dequantise-then-GEMM rule above.

`llama_pair` builds a Llama graph on the device and on the oracle with the same weights and caches, `llama_step` runs one
step on both, and `run_llama_parity` is the decode loop on top of the two (smoke() and the graph tests)."""
import contextlib
import math
import os
from types import SimpleNamespace

import numpy as np

import oracle as O
from oracle.graph_oracle import OracleHandler
from tests import kvfp8_oracle as KV
from tests import w4_oracle as W

F32, F16, BF16 = 1, 10, 16
# end-to-end criterion of the reference: rtol = atol = 1e-3 else argmax-equal (examples/python/llama_kvcache_inference.py:133-141);
# 16-bit storage gets its rounding step
TOL = {F32: 1e-3, F16: 4e-3, BF16: 3e-2}


# ---------------------------------------------------------------- AttentionKVCache rules on float32 arrays
def attention_kvcache_gqa(kc, vc, q, k, v, pos, dt):
    """In place on kc / vc (float32, C-contiguous); pos: one int (element-0 rule) or one per batch row.  With Hq = G * Hkv, for
    each g in [0, G) the query heads g, G + g, 2G + g, ... (q.reshape(B, Hkv, G, 1, D)[:, :, g]) form an equal-heads
    AttentionKVCache over the caches; every pass appends the same k / v row."""
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


def prompt_starts(pos, B, S, S_max, per_row):
    """p_b for every batch row: element 0 of the positions, or (per-row positions) row b's first element, flat index
    b * (numel / B), so that a [B, S] position tensor and a [B, 1] one both work; clamped to [0, S_max - S]"""
    pv = np.asarray(pos).ravel().astype(np.int64)
    start = pv[np.arange(B) * (pv.size // B)] if per_row else np.full(B, pv[0])
    return np.clip(start, 0, S_max - S)


def attention_kvcache_prompt(kc, vc, q, k, v, pos, dt, per_row=False):
    """S single-token steps: token i of batch row b is appended at cache row p_b + i and query i attends over rows
    0 .. p_b + i.  In place on kc / vc (float32, C-contiguous [B, Hkv, S_max, D]); q [B, Hq, S, D], k / v [B, Hkv, S, D];
    returns [B, Hq, S, D] float32 rounded to dt"""
    B, S = q.shape[0], q.shape[2]
    start = prompt_starts(pos, B, S, kc.shape[2], per_row)
    tok = [np.asarray(t, np.float32) for t in (q, k, v)]
    return np.concatenate([attention_kvcache_d(kc, vc, *(np.ascontiguousarray(t[:, :, i:i + 1]) for t in tok), start + i, dt)
                           for i in range(S)], axis=2)


class LlamaOracleHandler(OracleHandler):
    """The graph oracle with grouped-query and 64-wide heads, prompt chunks, FP8 KV caches and MatMulNBits."""

    head_widths = (64, 128)

    def RoPE(self, pos, x, y, dim_head=128):
        out = self._out(y, x.dims, x.dt)
        return self._rec(lambda: O.rope(pos.value, x.value, dim_head, x.dt), [pos, x], [out])

    def attentionKVCache(self, kc, vc, q, k, v, pos, y, per_row_positions=False, k_scale=None, v_scale=None):
        B, S = q.dims[0], q.dims[2]
        if S > 1 and k_scale is not None:
            raise ValueError("AttentionKVCache: an FP8 KV cache takes one new token per step (S = 1)")
        out = self._out(y, q.dims, q.dt)

        def run():
            if S > 1:
                return attention_kvcache_prompt(kc.value, vc.value, q.value, k.value, v.value, pos.value, q.dt,
                                                per_row_positions)
            pv = np.asarray(pos.value).ravel()
            if k_scale is not None:
                p = np.clip(pv[:B] if per_row_positions else np.full(B, int(pv[0])), 0, kc.dims[2] - 1)
                KV.append(kc.value, vc.value, np.asarray(k.value, np.float32), np.asarray(v.value, np.float32), k_scale.value,
                          v_scale.value, p)
                ref, _ = KV.attention(kc.value, vc.value, k_scale.value, v_scale.value, q.value, p, q.dt)
                return O.round_to(ref.astype(np.float32), q.dt)
            p = pv[:B] if per_row_positions else int(pv[0])
            return attention_kvcache_d(kc.value, vc.value, q.value, k.value, v.value, p, q.dt)
        ins = [kc, vc, q, k, v, pos] + ([] if k_scale is None else [k_scale, v_scale])
        return self._rec(run, ins, [out])

    def matMulNBits(self, a, b, scales, zero_points, y, K, N, block_size, bits=4, g_idx=None, bias=None):
        assert bits == 4 and g_idx is None and bias is None
        out = self._out(y, list(a.dims[:-1]) + [N], a.dt)

        def run():
            x = np.asarray(a.value, np.float32).reshape(-1, K)
            zp = None if zero_points is None else zero_points.value
            w = W.dequantize(b.value, scales.value, zp, K, N, block_size)
            if x.shape[0] > 64:  # dequantise to T, then the 16-bit MatMul
                return O.matmul(x, O.round_to(w.astype(np.float32), a.dt), None, False, False, a.dt).reshape(out.dims)
            return O.round_to((x.astype(np.float64) @ w).astype(np.float32), a.dt).reshape(out.dims)
        ins = [a, b, scales] + ([] if zero_points is None else [zero_points])
        return self._rec(run, ins, [out])


# ---------------------------------------------------------------- device graph vs oracle graph
def llama_caches(cfg):
    """the caches every parity test starts from, k of every layer then v, in storage: llama_cache_values, or for an FP8 cache
    the codes of llama_kv_fp8_values (whose scales fill_llama_weights_host writes)"""
    from infinitensor_b200 import graphs as G
    if cfg.kv_fp8:
        return [G.llama_kv_fp8_values(cfg, li, w)[0] for w in "kv" for li in range(cfg.layers)]
    return [G.to_storage(G.llama_cache_values(cfg, li, w), cfg.dtype) for w in "kv" for li in range(cfg.layers)]


def load_caches(g, caches):
    for t, c in zip(g.k_caches + g.v_caches, caches):
        t.copyin_numpy(c)


def cache_values(g):
    """a graph's caches in storage, k of every layer then v"""
    return [t.copyout_numpy() for t in g.k_caches + g.v_caches]


def oracle_graph(cfg, seq=1, caches=None):
    """(LlamaOracleHandler, graph) for (cfg, seq) with fill_llama_weights_host's weights and `caches` (default llama_caches)"""
    from infinitensor_b200 import graphs as G
    oh = LlamaOracleHandler()
    og = G.build_llama_decode(oh, cfg, seq=seq)
    G.fill_llama_weights_host(og)
    load_caches(og, llama_caches(cfg) if caches is None else caches)
    return oh, og


@contextlib.contextmanager
def _environ(env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def llama_pair(cfg, seq=1, env=None, caches=None, oracle_caches=None, rt=None):
    """The device graph and the oracle graph of (cfg, seq) with the same weights.  Caches: `caches` on both sides (default
    llama_caches), or `oracle_caches` on the oracle's where the two differ (caches carried from a prompt step).  `env` is set
    while the device graph is planned and restored afterwards (ITB_NO_FUSION / ITB_FUSION_MASK select the schedule)."""
    from infinitensor_b200 import backend as B
    from infinitensor_b200 import graphs as G
    rt = rt or B.CudaRuntime(0)
    h = B.GraphHandler(rt)
    with _environ(env or {}):
        g = G.build_llama_decode(h, cfg, seq=seq)
        h.data_malloc()
        sched = h.schedule()
    G.fill_llama_weights_host(g)
    caches = llama_caches(cfg) if caches is None else caches
    load_caches(g, caches)
    oh, og = oracle_graph(cfg, seq, caches if oracle_caches is None else oracle_caches)
    return SimpleNamespace(cfg=cfg, rt=rt, h=h, g=g, oh=oh, og=og, schedule=sched)


def llama_step(p, ids, pos, cudagraph=True):
    """feed ids / positions to both graphs, run the device graph (replayed or eager) and the oracle; the logits of both as
    float64 (device, oracle)"""
    from infinitensor_b200 import graphs as G
    for g in (p.g, p.og):
        g.input_ids.copyin_numpy(ids)
        g.position_ids.copyin_numpy(pos)
    if cudagraph:
        p.h.run_with_cudagraph()
    else:
        p.h.run()
    p.oh.run()
    return G.from_storage(p.g.logits.copyout_numpy(), p.cfg.dtype).astype(np.float64), p.og.logits.f32().astype(np.float64)


def rel_err(got, ref):
    """logits rel-to-max error"""
    return np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-6)


def check_appended_k(p, rows, tol):
    """layer 0's k cache rows `rows` (this step's appends) on the device against the oracle's.  The RoPE arithmetic runs on the
    GPU's cosf / sinf, so 16-bit caches get the storage type's rounding step (tolerance, not bit-equality; rows that are not
    appended are checked bit-exact in tests/test_gpu_kernels.py::test_attention_parity).  FP8 codes come from activations that
    already differ in their last bits: a code step is allowed on a few."""
    from infinitensor_b200 import graphs as G
    kd = p.g.k_caches[0].copyout_numpy()[:, :, rows]
    ko = p.og.k_caches[0].copyout_numpy()[:, :, rows]
    if p.cfg.kv_fp8:
        assert np.mean(kd != ko) < 0.05, "appended k codes of layer 0 differ from the oracle's beyond rounding"
    else:
        assert np.allclose(G.from_storage(kd, p.cfg.dtype), G.from_storage(ko, p.cfg.dtype), rtol=tol, atol=tol), \
            "appended k rows of layer 0 differ from the oracle's"


def run_llama_parity(cfg, pos=5, steps=2, cudagraph=True, env=None, tol=None):
    """Decode steps at positions pos .. pos + steps - 1 on the device and on the oracle.  Every step: finite logits, rel-to-max
    error below tol (default TOL), layer 0's appended k row.  Replayed: the graph is captured once.  Returns (worst logits
    error, kernel launches, schedule)."""
    p = llama_pair(cfg, env=env)
    t = tol or TOL[cfg.dtype]
    rng = np.random.default_rng(1)
    worst = 0.0
    for step in range(steps):
        ids = rng.integers(0, cfg.vocab, size=(cfg.batch, 1)).astype(np.int64)
        got, ref = llama_step(p, ids, np.full((cfg.batch, 1), pos + step, np.int64), cudagraph)
        assert np.isfinite(got).all(), f"step {step}: non-finite logits"
        err = rel_err(got, ref)
        worst = max(worst, err)
        assert err < t, f"step {step}: logits rel-to-max error {err:.3e} >= {t}"
        check_appended_k(p, pos + step, t)
    if cudagraph:
        assert p.rt.cuda_graph_capture_count() == 1, "graph must be captured once and replayed"
    return worst, p.rt.kernel_launches(), p.schedule
