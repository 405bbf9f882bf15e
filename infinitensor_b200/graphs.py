"""Synthetic graph builders for the BASELINE.json configs, written against the GraphHandler API only
(the same calls OnnxStub makes, reference pyinfinitensor/src/pyinfinitensor/onnx.py:136-1117), so they
need no `onnx` package.  Every builder takes a duck-typed handler: `backend.GraphHandler` (the product)
or `oracle.graph_oracle.OracleHandler` (the CPU checker) -- one graph description, two executors.  Decode graphs with
attention heads narrower than 128 (GPT-2, TinyLlama) use an extension of the reference, whose AttentionKVCache scale and
RoPE are fixed at 128: they build only on a handler that lists the width in its `head_widths` (`GraphHandler` does;
`OracleHandler`, which restates the reference, does not), so no executor quietly applies the 128-wide rule to them.  Likewise
a Llama config with other RoPE frequencies than base 10000 (`rope_theta`, `rope_scaling`) builds only on a handler whose
RoPE takes an inv_freq table (`rope_inv_freq`).

  build_llama_decode   -- config C3/C5: Llama-7B-shape KV-cache decode step (op mix of
                          examples/python/llama_kvcache_inference.py:45-80 with fused RMSNorm / RoPE /
                          AttentionKVCache nodes), optionally tensor-parallel-sharded exactly where
                          examples/distributed/parallel_opt.py:9-247 cuts the graph.
  build_gpt2           -- config C2: GPT-2-small forward, B=1 S=128 (op mix of run_pytorch.py:89-108 export)
  build_gpt2_decode    -- one GPT-2 KV-cache decode step over the same weights (64-wide heads)
  build_resnet50       -- config C4: ResNet-50 forward (conv + BN + relu + pooling + fc)
  build_matmul         -- config C1: single MatMul
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

F32, F16, BF16, I64, I32 = 1, 10, 16, 7, 6
FP8 = 17  # FP8 E4M3 codes: weights (SURVEY 8(f-4)) and, with LlamaConfig.kv_fp8, the KV caches
U8 = 2  # packed 4-bit weight codes (LlamaConfig.int4_block)
LINEAR = 0


# ---------------------------------------------------------------- storage helpers (host side)
def f32_to_bf16_bits(a: np.ndarray) -> np.ndarray:
    """float32 -> bf16 bit pattern (uint16), round-to-nearest-even."""
    u = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)
    r = ((u >> 16) & 1) + 0x7FFF
    return ((u + r) >> 16).astype(np.uint16)


def bf16_bits_to_f32(b: np.ndarray) -> np.ndarray:
    return (b.astype(np.uint32) << 16).view(np.float32)


def to_storage(a: np.ndarray, dtype: int) -> np.ndarray:
    """float32 values -> array in the tensor's storage dtype (what copyin_numpy expects)."""
    if dtype == F32:
        return np.ascontiguousarray(a, dtype=np.float32)
    if dtype == F16:
        return np.ascontiguousarray(a, dtype=np.float32).astype(np.float16)
    if dtype == BF16:
        return f32_to_bf16_bits(a)
    return np.ascontiguousarray(a)


def from_storage(a: np.ndarray, dtype: int) -> np.ndarray:
    if dtype == BF16:
        return bf16_bits_to_f32(a)
    if dtype == F16:
        return a.astype(np.float32)
    return a


def _require_head_width(h, dh: int):
    if dh != 128 and dh not in getattr(h, "head_widths", (128,)):
        raise NotImplementedError(f"{type(h).__name__} does not execute {dh}-wide attention heads (the reference's are 128-wide)")


def _require_window(h):
    if not getattr(h, "sliding_window", False):
        raise NotImplementedError(f"{type(h).__name__} has no sliding-window AttentionKVCache: it cannot run a config with "
                                  "sliding_window (it would attend over every cache row)")


def _require_ring(h):
    if not getattr(h, "rolling_cache", False):
        raise NotImplementedError(f"{type(h).__name__} has no rolling KV cache: it cannot run a config with rolling_cache "
                                  "(it would index the cache by absolute position)")


def _require_rope_table(h, cfg):
    if not getattr(h, "rope_inv_freq", False):
        raise NotImplementedError(f"{type(h).__name__} has no RoPE inv_freq table: it cannot run rope_theta = {cfg.rope_theta}, "
                                  f"rope_scaling = {cfg.rope_scaling} (its RoPE is base 10000)")


def rope_inv_freq(dim_head: int, theta: float = 10000.0, scaling: dict | None = None) -> np.ndarray:
    """RoPE's inv_freq table, f32 [dim_head / 2], as Hugging Face transformers computes it in float32: the default rule
    1 / theta^(2c / dim_head), and with scaling {"type": "llama3", factor, low_freq_factor, high_freq_factor,
    original_max_position_embeddings} Llama-3.1's rule: columns whose wavelength 2 pi / inv_freq is below
    original / high_freq_factor keep their frequency, those above original / low_freq_factor are divided by factor, and the
    band between is interpolated.  Rope types that also scale attention (YaRN, LongRoPE) and dynamic NTK are not covered."""
    f32 = np.float32
    expo = np.arange(0, dim_head, 2, dtype=np.int64).astype(f32) / f32(dim_head)
    inv = f32(1.0) / np.power(np.float64(f32(theta)), expo.astype(np.float64)).astype(f32)  # (a correctly rounded f32 power)
    if scaling is None:
        return inv.astype(f32)
    kind = scaling.get("type", scaling.get("rope_type"))
    if kind != "llama3":
        raise ValueError(f"rope_scaling type {kind!r}: only 'llama3' is provided")
    factor, lo_f, hi_f = f32(scaling["factor"]), f32(scaling["low_freq_factor"]), f32(scaling["high_freq_factor"])
    old = f32(scaling["original_max_position_embeddings"])
    lo_wave, hi_wave = old / lo_f, old / hi_f
    wave = f32(2 * np.pi) / inv
    scaled = np.where(wave > lo_wave, inv / factor, inv)
    smooth = (old / wave - lo_f) / (hi_f - lo_f)
    smoothed = (f32(1) - smooth) * scaled / factor + smooth * scaled
    medium = ~(wave < hi_wave) & ~(wave > lo_wave)
    return np.where(medium, smoothed, scaled).astype(f32)


# ---------------------------------------------------------------- Llama decode (C3 / C5)
LLAMA31_ROPE_SCALING = {"type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                        "original_max_position_embeddings": 8192}


@dataclass
class LlamaConfig:
    layers: int = 32
    d_model: int = 4096
    heads: int = 32
    head_dim: int = 128
    ffn: int = 11008
    vocab: int = 32000
    s_max: int = 1024
    batch: int = 16
    dtype: int = BF16
    fp8_weights: bool = False  # the seven projection matrices of every layer + the logits head as FP8 E4M3 codes + f32 column scales
    kv_heads: int | None = None  # grouped-query attention: KV heads shared by heads // kv_heads query heads each; None = heads
    kv_fp8: bool = False  # KV caches as FP8 E4M3 codes + per-layer f32 [KV heads] k / v scales (one token per step)
    int4_block: int = 0  # 32 / 64 / 128: the seven projections of every layer + the logits head as MatMulNBits (4-bit, symmetric)
    rope_theta: float = 10000.0  # RoPE base
    rope_scaling: dict | None = None  # None, or {"type": "llama3", factor, low_freq_factor, high_freq_factor,
                                      # original_max_position_embeddings} (see rope_inv_freq)
    sliding_window: int | None = None  # every layer's query at position P attends over cache rows (P - W, P] only; None: all rows
    rolling_cache: bool = False  # (with a window) the caches are a ring of s_max rows, position P in row P mod s_max

    @property
    def n_kv(self) -> int:
        return self.heads if self.kv_heads is None else self.kv_heads

    @property
    def rope_default(self) -> bool:
        """base 10000 without scaling: the RoPE nodes take no inv_freq table"""
        return self.rope_theta == 10000.0 and self.rope_scaling is None

    @staticmethod
    def llama3_8b(batch=16, s_max=1024, dtype=BF16, layers=32, kv_fp8=False, int4_block=0):
        """Llama-3-8B shape: 32 query heads over 8 KV heads (G = 4).  A shape only: its RoPE is base 10000, not Llama-3's
        500 000; `llama31_8b` has Llama-3.1's frequencies."""
        return LlamaConfig(layers=layers, d_model=4096, heads=32, kv_heads=8, head_dim=128, ffn=14336, vocab=128256,
                           s_max=s_max, batch=batch, dtype=dtype, kv_fp8=kv_fp8, int4_block=int4_block)

    @staticmethod
    def llama31_8b(batch=16, s_max=1024, dtype=BF16, layers=32, kv_fp8=False, int4_block=0):
        """Llama-3.1-8B: the Llama-3-8B shape with its RoPE, base 500 000 and llama3 scaling (factor 8, low / high frequency
        factors 1 / 4, original context 8192)."""
        return LlamaConfig(layers=layers, d_model=4096, heads=32, kv_heads=8, head_dim=128, ffn=14336, vocab=128256,
                           s_max=s_max, batch=batch, dtype=dtype, kv_fp8=kv_fp8, int4_block=int4_block,
                           rope_theta=500000.0, rope_scaling=dict(LLAMA31_ROPE_SCALING))

    @staticmethod
    def mistral_7b_v01(batch=16, s_max=1024, dtype=BF16, layers=32, kv_fp8=False, int4_block=0, rolling_cache=False):
        """Mistral-7B-v0.1: 32 query heads over 8 KV heads of 128 (G = 4), ffn 14336, vocab 32000, RoPE base 10000 and a
        sliding window of 4096 rows (HF's sliding_window).  By default the cache is indexed by absolute position: s_max
        covers the longest position, not just the window.  rolling_cache=True makes it a ring of s_max rows (Mistral's
        rolling buffer cache): s_max >= 4096 and a multiple of 64, and prompt chunks of up to s_max - 4095 tokens, so
        s_max=4608 for 512-token chunks; decode then goes on past s_max."""
        return LlamaConfig(layers=layers, d_model=4096, heads=32, kv_heads=8, head_dim=128, ffn=14336, vocab=32000,
                           s_max=s_max, batch=batch, dtype=dtype, kv_fp8=kv_fp8, int4_block=int4_block, sliding_window=4096,
                           rolling_cache=rolling_cache)

    @staticmethod
    def tiny(dtype=BF16, layers=2, batch=4, kv_fp8=False):
        return LlamaConfig(layers=layers, d_model=256, heads=2, head_dim=128, ffn=512, vocab=1000, s_max=64,
                           batch=batch, dtype=dtype, kv_fp8=kv_fp8)

    @staticmethod
    def tinyllama_1b(batch=16, s_max=1024, dtype=BF16, layers=22, kv_fp8=False, int4_block=0):
        """TinyLlama-1.1B shape: 32 query heads of 64 over 4 KV heads (G = 8)."""
        return LlamaConfig(layers=layers, d_model=2048, heads=32, kv_heads=4, head_dim=64, ffn=5632, vocab=32000,
                           s_max=s_max, batch=batch, dtype=dtype, kv_fp8=kv_fp8, int4_block=int4_block)

    def weight_elems(self, world: int = 1) -> int:
        d, f, dkv = self.d_model, self.ffn, self.n_kv * self.head_dim
        per_layer = (2 * d * d + 2 * d * dkv + 3 * d * f) // world + 2 * d
        return self.layers * per_layer + d + self.vocab * d + self.vocab * d  # + embedding table

    def algorithmic_bytes(self, pos: int, world: int = 1) -> int:
        """SURVEY.md 8(d): weights read once + KV read/append + ~12 activation tensors per layer.  With a sliding window W a
        step reads min(pos + 1, W) cache rows per head instead of pos + 1."""
        e = 2 if self.dtype in (F16, BF16) else 4
        d, f, dkv = self.d_model, self.ffn, self.n_kv * self.head_dim
        proj = self.layers * ((2 * d * d + 2 * d * dkv + 3 * d * f) // world) + d * self.vocab
        norms = self.layers * 2 * d + d
        rows = pos + 2 if not self.sliding_window else min(pos + 1, self.sliding_window) + 1  # rows read + the appended one
        kv = self.layers * 2 * self.batch * (self.n_kv // world) * self.head_dim * rows
        act = self.layers * 12 * self.batch * d
        kv_bytes = kv * e
        if self.kv_fp8:  # one byte per cache element + the 4-byte k / v scale of every KV head
            kv_bytes = kv + self.layers * 2 * (self.n_kv // world) * 4
        if self.int4_block:  # half a byte per projection weight + one 16-bit scale per block of int4_block weights
            return proj // 2 + 2 * (proj // self.int4_block) + (norms + act) * e + kv_bytes
        if self.fp8_weights:  # one byte per projection weight + 4 bytes per output column
            cols = self.layers * ((d + 2 * dkv + 2 * f) // world + 2 * d) + self.vocab
            return proj + 4 * cols + (norms + act) * e + kv_bytes
        return (proj + norms + act) * e + kv_bytes


@dataclass
class LlamaGraph:
    cfg: LlamaConfig
    input_ids: object = None
    position_ids: object = None
    logits: object = None
    k_caches: list = field(default_factory=list)
    v_caches: list = field(default_factory=list)
    weights: dict = field(default_factory=dict)  # name -> (tensor, shape, kind, shard)


def build_llama_decode(h, cfg: LlamaConfig, world: int = 1, rank: int = 0, seq: int = 1) -> LlamaGraph:
    """One decode step, or with seq > 1 one prompt step: seq new tokens per batch row at positions p_b .. p_b + seq - 1
    (input_ids and position_ids [B, seq], logits [B, seq, vocab]; AttentionKVCache appends all of them and attends
    causally).  world > 1 applies the reference's tensor-parallel cut (parallel_opt.py):
    q/k/v + gate/up column-split, o/down row-split followed by AllReduceSum, KV cache split by head,
    embedding / norms / logits replicated.  cfg.kv_heads < cfg.heads builds grouped-query attention: k / v projections
    and caches carry the KV heads, query head i reads KV head i // (heads // kv_heads)."""
    assert cfg.heads % world == 0 and cfg.ffn % world == 0
    assert cfg.n_kv % world == 0 and cfg.heads % cfg.n_kv == 0
    # the FP8 weight GEMM takes at most 64 rows, and a tensor-parallel prompt step is not provided
    assert seq == 1 or (world == 1 and not cfg.fp8_weights), "prompt steps (seq > 1): one GPU, 16-bit weights"
    assert seq == 1 or not cfg.kv_fp8, "an FP8 KV cache takes one token per step (seq == 1)"
    if cfg.int4_block:
        if cfg.int4_block not in (32, 64, 128):
            raise ValueError(f"int4_block = {cfg.int4_block}: 32, 64 or 128")
        if world > 1:
            raise ValueError("int4 weights (int4_block): tensor-parallel sharding is not provided; world must be 1")
        if cfg.fp8_weights:
            raise ValueError("int4_block and fp8_weights exclude each other")
    B, d, H, dh, f, V, dt = cfg.batch, cfg.d_model, cfg.heads // world, cfg.head_dim, cfg.ffn // world, cfg.vocab, cfg.dtype
    Hkv = cfg.n_kv // world
    dl, dkv = H * dh, Hkv * dh  # local attention widths of q and of k / v
    _require_head_width(h, dh)
    rope_kw = {} if dh == 128 else {"dim_head": dh}  # 128-wide graphs make the reference's RoPE call
    if not cfg.rope_default:
        _require_rope_table(h, cfg)
    if cfg.sliding_window is not None and cfg.sliding_window < 0:
        raise ValueError(f"sliding_window = {cfg.sliding_window}: a window is at least 1 row (None: no window)")
    if cfg.sliding_window:
        _require_window(h)
    win_kw = {"window": cfg.sliding_window} if cfg.sliding_window else {}  # (unwindowed: the call as before)
    if cfg.rolling_cache:
        W = cfg.sliding_window
        if not W:
            raise ValueError("rolling_cache needs a sliding_window: a ring holds the window's rows")
        need = W + seq - 1
        if cfg.s_max < need or cfg.s_max % 64:
            raise ValueError(f"rolling_cache: s_max = {cfg.s_max}, but a ring for window {W} and {seq}-token steps needs "
                             f"s_max >= window + seq - 1 = {need} and a multiple of 64 (e.g. {-(-need // 64) * 64})")
        _require_ring(h)
        win_kw["rolling"] = True
    g = LlamaGraph(cfg)

    def weight(name, shape, kind, shard=None):
        t = h.tensor(list(shape), dt)
        t.set_weight()
        g.weights[name] = (t, tuple(shape), kind, shard)
        return t

    def linear(x_, name, shape, shard=None):
        """x . W: 16-bit weight, or (cfg.fp8_weights) FP8 E4M3 codes + per-column f32 scale dequantised inside the GEMM, or
        (cfg.int4_block) MatMulNBits: 4-bit codes [N, K / bs, bs / 2] + one scale of the activation type per block of bs"""
        if cfg.int4_block:
            K_, N_ = shape
            bs = cfg.int4_block
            wq = h.tensor([N_, K_ // bs, bs // 2], U8)
            wq.set_weight()
            sc = h.tensor([N_ * (K_ // bs)], dt)
            sc.set_weight()
            g.weights[name] = (wq, tuple(shape), "proj_int4", shard)
            g.weights[name + ".scale"] = (sc, (N_ * (K_ // bs),), "scale", None)
            return h.matMulNBits(x_, wq, sc, None, None, K_, N_, bs)
        if not cfg.fp8_weights:
            return h.matmul(x_, weight(name, shape, "proj", shard), None, False, False, None, LINEAR)
        assert world == 1, "fp8 weights: single GPU"
        wq = h.tensor(list(shape), FP8)
        wq.set_weight()
        sc = h.tensor([shape[1]], F32)
        sc.set_weight()
        g.weights[name] = (wq, tuple(shape), "proj_fp8", shard)
        g.weights[name + ".scale"] = (sc, (shape[1],), "scale", None)
        return h.matmul(x_, wq, None, False, False, None, LINEAR, w_scale=sc)

    g.input_ids = h.tensor([B, seq], I64)
    g.position_ids = h.tensor([B, seq], I64)
    g.input_ids.set_input()
    g.position_ids.set_input()
    emb = weight("embed", (V, d), "embed")
    if not cfg.rope_default:  # one table, shared by every RoPE (replicated on every rank)
        inv = h.tensor([dh // 2], F32)
        inv.set_weight()
        g.weights["rope.inv_freq"] = (inv, (dh // 2,), "inv_freq", None)
        rope_kw["inv_freq"] = inv
    x = h.gather(emb, g.input_ids, None, 0)  # [B,seq,d]
    for li in range(cfg.layers):
        p = f"l{li}."
        kc = h.tensor([B, Hkv, cfg.s_max, dh], FP8 if cfg.kv_fp8 else dt)
        vc = h.tensor([B, Hkv, cfg.s_max, dh], FP8 if cfg.kv_fp8 else dt)
        kc.set_input()
        vc.set_input()
        g.k_caches.append(kc)
        g.v_caches.append(vc)
        kv_scales = {}
        if cfg.kv_fp8:  # per-KV-head f32 scales of this layer's caches, sharded by head with them
            for which in ("k", "v"):
                t = h.tensor([Hkv], F32)
                t.set_weight()
                g.weights[f"{p}{which}_scale"] = (t, (Hkv,), "kv_scale", ("head", cfg.n_kv))
                kv_scales[which + "_scale"] = t
        hn = h.RMSNorm(x, weight(p + "ln1", (d,), "norm"), None)
        q = linear(hn, p + "wq", (d, dl), ("col", d))
        k = linear(hn, p + "wk", (d, dkv), ("col", d))
        v = linear(hn, p + "wv", (d, dkv), ("col", d))
        q = h.RoPE(g.position_ids, q, None, **rope_kw)
        k = h.RoPE(g.position_ids, k, None, **rope_kw)

        def heads(t, n=H):
            t = h.reshape(t, None, [B, seq, n, dh])
            return h.transpose(t, None, [0, 2, 1, 3])  # [B,n,seq,dh]

        attn = h.attentionKVCache(kc, vc, heads(q), heads(k, Hkv), heads(v, Hkv), g.position_ids, None, **kv_scales,
                                  **win_kw)
        a = h.reshape(h.transpose(attn, None, [0, 2, 1, 3]), None, [B, seq, dl])
        o = linear(a, p + "wo", (dl, d), ("row", d))
        if world > 1:
            o = h.allReduceSum(o, None)
        x = h.add(x, o, None)
        hn = h.RMSNorm(x, weight(p + "ln2", (d,), "norm"), None)
        gate = linear(hn, p + "wg", (d, f), ("col", cfg.ffn))
        up = linear(hn, p + "wu", (d, f), ("col", cfg.ffn))
        m = h.mul(h.silu(gate, None), up, None)
        dn = linear(m, p + "wd", (f, d), ("row", cfg.ffn))
        if world > 1:
            dn = h.allReduceSum(dn, None)
        x = h.add(x, dn, None)
    xf = h.RMSNorm(x, weight("ln_f", (d,), "norm"), None)
    g.logits = linear(xf, "lm_head", (d, V))
    g.logits.set_output()
    return g


def llama_weight_values(name: str, shape, kind: str, seed: int = 0) -> np.ndarray:
    """SURVEY.md 8(d) synthetic inputs: weights ~ N(0, 0.02^2), norm weights 1 + N(0, 0.02^2); a
    per-tensor stream so every rank / executor draws identical full tensors."""
    rng = np.random.default_rng([seed, abs(hash_name(name))])
    w = rng.standard_normal(shape, dtype=np.float32) * np.float32(0.02)
    if kind == "norm":
        w = w + np.float32(1.0)
    return w


def hash_name(name: str) -> int:
    hv = 2166136261
    for ch in name.encode():
        hv = ((hv ^ ch) * 16777619) & 0xFFFFFFFF
    return hv


def shard_weight(full: np.ndarray, shard, world: int, rank: int) -> np.ndarray:
    """parallel_opt.py:21-59 slicing: column split -> W[:, r*N/w:(r+1)*N/w]; row split -> W[r*K/w:(r+1)*K/w, :]."""
    if shard is None or world == 1:
        return full
    mode = shard[0]
    if mode == "col":
        n = full.shape[1] // world
        return np.ascontiguousarray(full[:, rank * n:(rank + 1) * n])
    n = full.shape[0] // world
    return np.ascontiguousarray(full[rank * n:(rank + 1) * n, :])


def quantize_fp8_host(w: np.ndarray):
    """per-output-column symmetric FP8 E4M3 quantisation (same rule as oracle.quantize_weight_fp8, restated so that the product
    never imports the oracle): codes uint8 [K, N], scale f32 [N] = max|column| / 448; round to nearest, ties to even."""
    w = np.asarray(w, np.float32)
    scale = np.maximum(np.abs(w).max(axis=0), 1e-12).astype(np.float32) / np.float32(448.0)
    return e4m3_codes_host((w / scale[None, :]).astype(np.float32)), scale


def e4m3_codes_host(x: np.ndarray) -> np.ndarray:
    """float32 -> FP8 E4M3 codes (uint8): round to nearest, ties to even, saturated to +-448 (finite inputs)."""
    x = np.asarray(x, np.float32)
    table = np.zeros(127, np.float64)
    for c in range(127):
        e, m = (c >> 3) & 15, c & 7
        table[c] = (m / 8.0) * 2.0 ** -6 if e == 0 else (1.0 + m / 8.0) * 2.0 ** (e - 7)
    mag = np.minimum(np.abs(x).astype(np.float64), 448.0)
    hi = np.clip(np.searchsorted(table, mag, side="left"), 0, 126)
    lo = np.clip(hi - 1, 0, 126)
    dlo, dhi = mag - table[lo], table[hi] - mag
    code = np.where((dhi < dlo) | ((dhi == dlo) & (hi % 2 == 0)), hi, lo).astype(np.uint8)
    return np.where(np.signbit(x), code | 0x80, code).astype(np.uint8)


def quantize_w4(w: np.ndarray, block: int, dtype: int = BF16):
    """Symmetric 4-bit block quantisation of W [K, N] in MatMulNBits' layout (no zero points, so z = 8): per column n and block b
    of `block` consecutive k, scale = amax / 7 rounded to the activation dtype, q = clamp(rint(w / scale) + 8, 0, 15), rint
    rounding half to even.  Returns (codes uint8 [N, K / block, block / 2] with even k in the low nibble, scale float32 [N * K / block]
    holding values exact in `dtype`)."""
    w = np.asarray(w, np.float32)
    K, N = w.shape
    assert K % block == 0
    wb = w.T.reshape(N, K // block, block)
    amax = np.abs(wb).max(axis=2)
    scale = from_storage(to_storage(amax / np.float32(7.0), dtype), dtype).astype(np.float32)
    safe = np.where(scale > 0, scale, np.float32(1.0))
    q = np.clip(np.rint(wb / safe[:, :, None]) + 8, 0, 15).astype(np.uint8)
    codes = (q[:, :, 0::2] | (q[:, :, 1::2] << 4)).astype(np.uint8)
    return codes, scale.reshape(-1)


def fill_llama_weights_host(g: LlamaGraph, world: int = 1, rank: int = 0, seed: int = 0):
    """Small configs only (host RNG): full tensors are drawn, then sharded like parallel_opt.py does."""
    for name, (t, shape, kind, shard) in g.weights.items():
        if kind == "scale":
            continue  # written together with its codes
        if kind == "inv_freq":
            t.copyin_numpy(rope_inv_freq(g.cfg.head_dim, g.cfg.rope_theta, g.cfg.rope_scaling))
            continue
        if kind == "kv_scale":  # the scale the cache helpers quantise with (llama_kv_fp8_values)
            li, which = int(name[1:name.index(".")]), name[name.index(".") + 1]
            t.copyin_numpy(llama_kv_fp8_values(g.cfg, li, which, world, rank)[1])
            continue
        if kind == "proj_int4":
            codes, scale = quantize_w4(llama_weight_values(name, list(shape), "proj", seed), g.cfg.int4_block, g.cfg.dtype)
            t.copyin_numpy(codes)
            g.weights[name + ".scale"][0].copyin_numpy(to_storage(scale, g.cfg.dtype))
            continue
        if kind == "proj_fp8":
            codes, scale = quantize_fp8_host(llama_weight_values(name, list(shape), "proj", seed))
            t.copyin_numpy(codes)
            g.weights[name + ".scale"][0].copyin_numpy(scale)
            continue
        full_shape = list(shape)
        if shard is not None and world > 1:
            full_shape[1 if shard[0] == "col" else 0] *= world
        w = shard_weight(llama_weight_values(name, full_shape, kind, seed), shard, world, rank)
        t.copyin_numpy(to_storage(w, g.cfg.dtype))


def llama_cache_values(cfg: LlamaConfig, layer: int, which: str, world: int = 1, rank: int = 0, seed: int = 2):
    """KV cache pre-filled with N(0,1)*0.5 (SURVEY 8(d)); full-head tensor then the rank's head slice."""
    rng = np.random.default_rng([seed, layer, 0 if which == "k" else 1])
    full = rng.standard_normal((cfg.batch, cfg.n_kv, cfg.s_max, cfg.head_dim), dtype=np.float32) * np.float32(0.5)
    hl = cfg.n_kv // world
    return np.ascontiguousarray(full[:, rank * hl:(rank + 1) * hl])


def llama_kv_fp8_values(cfg: LlamaConfig, layer: int, which: str, world: int = 1, rank: int = 0, seed: int = 2):
    """llama_cache_values quantised for an FP8 cache (cfg.kv_fp8): scale[h] = max |cache of KV head h| / 448 over the batch,
    codes = e4m3(value / scale[h]) -- the rule the append applies to new rows.  Returns (codes uint8 [B, Hkv_l, s_max, D],
    scale f32 [Hkv_l]) for the rank's heads."""
    x = llama_cache_values(cfg, layer, which, world, rank, seed)
    scale = (np.maximum(np.abs(x).max(axis=(0, 2, 3)), 1e-12).astype(np.float32) / np.float32(448.0)).astype(np.float32)
    return e4m3_codes_host(x / scale[None, :, None, None]), scale


# ---------------------------------------------------------------- single MatMul (C1)
def build_matmul(h, m=512, n=512, k=512, dtype=F32):
    a = h.tensor([m, k], dtype)
    b = h.tensor([k, n], dtype)
    a.set_input()
    b.set_input()
    c = h.matmul(a, b, None, False, False, None, LINEAR)
    c.set_output()
    return a, b, c


# ---------------------------------------------------------------- GPT-2 small (C2)
@dataclass
class GPT2Config:
    layers: int = 12
    d_model: int = 768
    heads: int = 12
    ffn: int = 3072
    vocab: int = 50257
    n_pos: int = 1024
    seq: int = 128
    batch: int = 1
    dtype: int = F16
    lm_head: bool = False  # the reference export is GPT2Model without LM head (run_pytorch.py:47,78-81)

    @staticmethod
    def tiny(dtype=F16):
        return GPT2Config(layers=2, d_model=64, heads=2, ffn=128, vocab=500, n_pos=64, seq=16, batch=1, dtype=dtype)

    def algorithmic_bytes(self, pos: int) -> int:
        """One decode step (build_gpt2_decode) at position `pos`, as LlamaConfig.algorithmic_bytes counts it: every layer's
        weights and biases read once, the KV cache read and appended, ~12 activation tensors per layer, the two embedding
        rows per batch row, and the tied logits head (the whole embedding table) when there is one."""
        e = 2 if self.dtype in (F16, BF16) else 4
        B, d, f = self.batch, self.d_model, self.ffn
        per_layer = 3 * d * d + 3 * d + d * d + d + 2 * d * f + f + d + 4 * d
        weights = self.layers * per_layer + 2 * d + 2 * B * d + (self.vocab * d if self.lm_head else 0)
        kv = self.layers * 2 * B * d * (pos + 2)
        act = self.layers * 12 * B * d
        return (weights + kv + act) * e


@dataclass
class GPT2Graph:
    cfg: GPT2Config
    input_ids: object = None
    position_ids: object = None
    out: object = None
    weights: dict = field(default_factory=dict)
    consts: dict = field(default_factory=dict)  # name -> (tensor, float32 ndarray)
    k_caches: list = field(default_factory=list)  # build_gpt2_decode: per layer [B, H, s_max, dh]
    v_caches: list = field(default_factory=list)


def build_gpt2(h, cfg: GPT2Config) -> GPT2Graph:
    B, S, d, H, f, dt = cfg.batch, cfg.seq, cfg.d_model, cfg.heads, cfg.ffn, cfg.dtype
    dh = d // H
    g = GPT2Graph(cfg)

    def weight(name, shape, kind):
        t = h.tensor(list(shape), dt)
        t.set_weight()
        g.weights[name] = (t, tuple(shape), kind, None)
        return t

    def const(name, arr):
        t = h.tensor(list(arr.shape), dt)
        t.set_weight()
        g.consts[name] = (t, np.asarray(arr, np.float32))
        return t

    g.input_ids = h.tensor([B, S], I64)
    g.position_ids = h.tensor([B, S], I64)
    g.input_ids.set_input()
    g.position_ids.set_input()
    x = h.add(h.gather(weight("wte", (cfg.vocab, d), "embed"), g.input_ids, None, 0),
              h.gather(weight("wpe", (cfg.n_pos, d), "embed"), g.position_ids, None, 0), None)  # [B,S,d]
    # causal mask as an additive 0/-inf constant: the frontend's rewrite of Where(mask, x, -inf) (onnx.py:1055-1081)
    big_neg = -65504.0 if dt == F16 else -3.0e38
    mask = const("mask", np.triu(np.full((S, S), big_neg, np.float32), 1).reshape(1, 1, S, S))
    scale = const("scale", np.array([np.sqrt(dh)], np.float32))
    for li in range(cfg.layers):
        p = f"h{li}."
        hn = h.layerNormalization(x, weight(p + "ln1.w", (d,), "norm"), None, weight(p + "ln1.b", (d,), "bias"), 1e-5, -1, 1)
        qkv = h.matmul(hn, weight(p + "attn.w", (d, 3 * d), "proj"), None, False, False,
                       weight(p + "attn.b", (3 * d,), "bias"), LINEAR)
        q, k, v = h.split(qkv, None, 2, 3)

        def heads(t):
            return h.transpose(h.reshape(t, None, [B, S, H, dh]), None, [0, 2, 1, 3])  # [B,H,S,dh]

        q, k, v = heads(q), heads(k), heads(v)
        kt = h.transpose(k, None, [0, 1, 3, 2])
        s = h.div(h.matmul(q, kt, None, False, False, None, LINEAR), scale, None)
        pr = h.softmax(h.add(s, mask, None), None, -1)
        a = h.matmul(pr, v, None, False, False, None, LINEAR)  # [B,H,S,dh]
        a = h.reshape(h.transpose(a, None, [0, 2, 1, 3]), None, [B, S, d])
        o = h.matmul(a, weight(p + "proj.w", (d, d), "proj"), None, False, False, weight(p + "proj.b", (d,), "bias"), LINEAR)
        x = h.add(x, o, None)
        hn = h.layerNormalization(x, weight(p + "ln2.w", (d,), "norm"), None, weight(p + "ln2.b", (d,), "bias"), 1e-5, -1, 1)
        m = h.matmul(hn, weight(p + "fc.w", (d, f), "proj"), None, False, False, weight(p + "fc.b", (f,), "bias"), LINEAR)
        m = h.gelu(m, None)
        m = h.matmul(m, weight(p + "fc2.w", (f, d), "proj"), None, False, False, weight(p + "fc2.b", (d,), "bias"), LINEAR)
        x = h.add(x, m, None)
    x = h.layerNormalization(x, weight("ln_f.w", (d,), "norm"), None, weight("ln_f.b", (d,), "bias"), 1e-5, -1, 1)
    if cfg.lm_head:
        x = h.matmul(x, g.weights["wte"][0], None, False, True, None, LINEAR)  # tied embedding
    g.out = x
    g.out.set_output()
    return g


def build_gpt2_decode(h, cfg: GPT2Config, s_max: int) -> GPT2Graph:
    """One KV-cache decode step of build_gpt2's model: input_ids / position_ids [B, 1] (position_ids[0] is every row's
    position, the AttentionKVCache rule), per layer LayerNorm, c_attn + bias split into q / k / v heads [B, H, 1, dh],
    AttentionKVCache over caches [B, H, s_max, dh] (graph inputs, appended in place), merge, proj + bias, residual, LayerNorm,
    fc + bias, Gelu, fc2 + bias, residual; the final LayerNorm and (cfg.lm_head) the tied-embedding logits.  Same weight
    names and shapes as build_gpt2, so fill_gpt2_weights_host fills either; the caches are in `k_caches` / `v_caches`."""
    B, d, H, f, dt = cfg.batch, cfg.d_model, cfg.heads, cfg.ffn, cfg.dtype
    dh = d // H
    _require_head_width(h, dh)
    g = GPT2Graph(cfg)

    def weight(name, shape, kind):
        t = h.tensor(list(shape), dt)
        t.set_weight()
        g.weights[name] = (t, tuple(shape), kind, None)
        return t

    def linear(x_, name, k, n):
        return h.matmul(x_, weight(name + ".w", (k, n), "proj"), None, False, False, weight(name + ".b", (n,), "bias"), LINEAR)

    def layer_norm(x_, name):
        return h.layerNormalization(x_, weight(name + ".w", (d,), "norm"), None, weight(name + ".b", (d,), "bias"), 1e-5, -1, 1)

    g.input_ids = h.tensor([B, 1], I64)
    g.position_ids = h.tensor([B, 1], I64)
    g.input_ids.set_input()
    g.position_ids.set_input()
    x = h.add(h.gather(weight("wte", (cfg.vocab, d), "embed"), g.input_ids, None, 0),
              h.gather(weight("wpe", (cfg.n_pos, d), "embed"), g.position_ids, None, 0), None)  # [B,1,d]
    for li in range(cfg.layers):
        p = f"h{li}."
        kc = h.tensor([B, H, s_max, dh], dt)
        vc = h.tensor([B, H, s_max, dh], dt)
        kc.set_input()
        vc.set_input()
        g.k_caches.append(kc)
        g.v_caches.append(vc)
        qkv = linear(layer_norm(x, p + "ln1"), p + "attn", d, 3 * d)
        q, k, v = h.split(qkv, None, 2, 3)

        def heads(t):
            return h.transpose(h.reshape(t, None, [B, 1, H, dh]), None, [0, 2, 1, 3])  # [B,H,1,dh]

        a = h.attentionKVCache(kc, vc, heads(q), heads(k), heads(v), g.position_ids, None)
        a = h.reshape(h.transpose(a, None, [0, 2, 1, 3]), None, [B, 1, d])
        x = h.add(x, linear(a, p + "proj", d, d), None)
        m = h.gelu(linear(layer_norm(x, p + "ln2"), p + "fc", d, f), None)
        x = h.add(x, linear(m, p + "fc2", f, d), None)
    x = layer_norm(x, "ln_f")
    if cfg.lm_head:
        x = h.matmul(x, g.weights["wte"][0], None, False, True, None, LINEAR)  # tied embedding
    g.out = x
    g.out.set_output()
    return g


def fill_gpt2_weights_host(g: GPT2Graph, seed: int = 0):
    for name, (t, shape, kind, _) in g.weights.items():
        w = llama_weight_values(name, shape, "norm" if kind == "norm" else "proj", seed)
        if kind == "bias":
            w = w * np.float32(0.5)
        t.copyin_numpy(to_storage(w, g.cfg.dtype))
    for name, (t, arr) in g.consts.items():
        t.copyin_numpy(to_storage(arr, g.cfg.dtype))


# ---------------------------------------------------------------- ResNet-50 (C4)
@dataclass
class ResNetConfig:
    batch: int = 64
    image: int = 224
    dtype: int = F16
    blocks: tuple = (3, 4, 6, 3)
    width: int = 64
    classes: int = 1000

    @staticmethod
    def tiny(dtype=F16):
        return ResNetConfig(batch=2, image=32, dtype=dtype, blocks=(1, 1, 1, 1), width=8, classes=10)


@dataclass
class ResNetGraph:
    cfg: ResNetConfig
    input: object = None
    out: object = None
    weights: dict = field(default_factory=dict)  # name -> (tensor, shape, kind, dtype)


def build_resnet50(h, cfg: ResNetConfig) -> ResNetGraph:
    """conv -> BatchNormalization -> Relu bottlenecks exactly as torchvision's export lowers through the
    frontend (Conv bias-free, BN as its own node, GlobalAveragePool -> AveragePool k=(H,W), onnx.py:489-503,
    Gemm -> MatMul(transB) + bias)."""
    dt = cfg.dtype
    g = ResNetGraph(cfg)

    def weight(name, shape, kind, dtype=None):
        t = h.tensor(list(shape), dtype or dt)
        t.set_weight()
        g.weights[name] = (t, tuple(shape), kind, dtype or dt)
        return t

    def conv_bn(x, name, cin, cout, k, stride, pad, relu=True):
        w = weight(name + ".w", (cout, cin, k, k), "conv")
        y = h.conv(x, w, None, pad, pad, stride, stride, 1, 1)
        y = h.batchNormalization(y, None, weight(name + ".bn.mean", (cout,), "bn_mean", F32),
                                 weight(name + ".bn.var", (cout,), "bn_var", F32),
                                 weight(name + ".bn.g", (cout,), "bn_g", F32), weight(name + ".bn.b", (cout,), "bn_b", F32),
                                 0.9, 1e-5, False)
        return h.relu(y, None) if relu else y

    g.input = h.tensor([cfg.batch, 3, cfg.image, cfg.image], dt)
    g.input.set_input()
    w0 = cfg.width
    x = conv_bn(g.input, "stem", 3, w0, 7, 2, 3)
    x = h.maxPool(x, None, 3, 3, 1, 1, 1, 1, 2, 2, 0)
    cin = w0
    for si, nb in enumerate(cfg.blocks):
        mid = w0 * (2 ** si)
        cout = mid * 4
        for bi in range(nb):
            stride = 2 if (bi == 0 and si > 0) else 1
            p = f"s{si}b{bi}"
            idn = x
            y = conv_bn(x, p + ".c1", cin, mid, 1, 1, 0)
            y = conv_bn(y, p + ".c2", mid, mid, 3, stride, 1)
            y = conv_bn(y, p + ".c3", mid, cout, 1, 1, 0, relu=False)
            if bi == 0:
                idn = conv_bn(x, p + ".down", cin, cout, 1, stride, 0, relu=False)
            x = h.relu(h.add(y, idn, None), None)
            cin = cout
    hw = x.shape()[2]
    x = h.avgPool(x, None, hw, hw, 1, 1, 0, 0, 1, 1, 0)
    x = h.flatten(x, None, 1)
    x = h.matmul(x, weight("fc.w", (cfg.classes, cin), "fc"), None, False, True, weight("fc.b", (cfg.classes,), "bias"),
                 LINEAR)
    g.out = x
    g.out.set_output()
    return g


def resnet_weight_values(name, shape, kind, seed=0):
    rng = np.random.default_rng([seed, abs(hash_name(name))])
    if kind == "conv":  # Kaiming-normal (SURVEY 8(d))
        fan_in = int(np.prod(shape[1:]))
        return rng.standard_normal(shape, dtype=np.float32) * np.float32(np.sqrt(2.0 / fan_in))
    if kind == "fc":
        return rng.standard_normal(shape, dtype=np.float32) * np.float32(0.02)
    if kind == "bn_var":
        return np.float32(1.0) + np.abs(rng.standard_normal(shape, dtype=np.float32)) * np.float32(0.1)
    if kind == "bn_g":
        return np.float32(1.0) + rng.standard_normal(shape, dtype=np.float32) * np.float32(0.1)
    return rng.standard_normal(shape, dtype=np.float32) * np.float32(0.1)  # bn_mean, bn_b, bias


def fill_resnet_weights_host(g: ResNetGraph, seed: int = 0):
    for name, (t, shape, kind, dtype) in g.weights.items():
        t.copyin_numpy(to_storage(resnet_weight_values(name, shape, kind, seed), dtype))
