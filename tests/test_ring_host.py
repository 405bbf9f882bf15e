"""CPU tier for the rolling KV cache (AttentionKVCache's `rolling`, LlamaConfig.rolling_cache): the shape rule and the
launchers' refusals, the attribute vector, unchanged default and windowed exports and schedules, ONNX round trips and
tensor-parallel sharding with a ring, the config checks, the refusals of handlers without rings, and the ring oracle against
the windowed oracle over a linear cache, bit for bit across several wraps."""
import ctypes
import dataclasses
import hashlib
import re

import numpy as np
import pytest

F32, F16, BF16, I64, FP8 = 1, 10, 16, 7, 17
RING = 0x400

# sha256 of the exports (and of the host schedules' repr) of windowed graphs, as written before rolling caches existed
WINDOWED_EXPORTS = {
    "win_decode": ("8481293ac8fb4ecfca9dd1dc5ab0846e1d827fed50844e53080e740e92b294e2",
                   "ab354e3b29ea79d0a18f592ee3b6699597d3581c61942db2949b9457e0dc5ab6"),
    "win_prompt": ("cad0bd5ba0fad60e6cf1e84db6870a4e8229affea0c2fd33ff05e64b548f2643",
                   "34b6f2a012cbf0b2c6ba1e5eda58a7a6d2fef87fe813c01a16b2d89cd8cd28e1"),
    "win_fp8": ("21cbc1c0e4536437105931cdb50f6d089a089a1fa857efc98a084698e1b9cb62",
                "ab354e3b29ea79d0a18f592ee3b6699597d3581c61942db2949b9457e0dc5ab6"),
    "mistral_2l": ("dd5dd83c4a0d2c09facdb801309351eacbd62c95a220715c43f6e139fc110c5f",
                   "ab354e3b29ea79d0a18f592ee3b6699597d3581c61942db2949b9457e0dc5ab6"),
}


@pytest.fixture(scope="module")
def B():
    from infinitensor_b200 import backend
    return backend


@pytest.fixture(scope="module")
def G():
    from infinitensor_b200 import graphs
    return graphs


def _attn(B, window, S=1, S_max=128, fp8=False, rolling=True):
    h = B.GraphHandler(B.HostPlanRuntime())
    Bn, Hq, Hkv, D = 2, 8, 2, 128
    cache = FP8 if fp8 else BF16
    kc, vc = h.tensor([Bn, Hkv, S_max, D], cache), h.tensor([Bn, Hkv, S_max, D], cache)
    q, k, v = h.tensor([Bn, Hq, S, D], BF16), h.tensor([Bn, Hkv, S, D], BF16), h.tensor([Bn, Hkv, S, D], BF16)
    sc = {"k_scale": h.tensor([Hkv], F32), "v_scale": h.tensor([Hkv], F32)} if fp8 else {}
    return h, h.attentionKVCache(kc, vc, q, k, v, h.tensor([Bn, S], I64), None, False, **sc, window=window, rolling=rolling)


# ---------------------------------------------------------------------------------------------------- shape rule, refusals
@pytest.mark.parametrize("window,S,S_max", [(1, 1, 64), (64, 1, 64), (100, 1, 128), (64, 65, 128), (4096, 513, 4608),
                                            (16, 8, 64)])
def test_shape_rule_accepts_rings(B, window, S, S_max):
    assert _attn(B, window, S, S_max)[1].shape() == [2, 8, S, 128]


def test_shape_rule_accepts_an_fp8_ring(B):
    assert _attn(B, 64, 1, 128, fp8=True)[1].shape() == [2, 8, 1, 128]


@pytest.mark.parametrize("window,S,S_max,fp8,msg", [
    (0, 1, 128, False, "AttentionKVCache: a rolling cache needs a window >= 1"),
    (129, 1, 128, False, "AttentionKVCache: a rolling cache of 128 rows is shorter than the window of 129"),
    (64, 1, 96, False, "AttentionKVCache: a rolling cache's length 96 is not a multiple of 64"),
    (100, 30, 128, False, "AttentionKVCache: a chunk of 30 tokens needs a rolling cache of window + 29 = 129 rows or more, "
                          "not 128 (split the prompt)"),
    (64, 8, 128, True, "AttentionKVCache: an FP8 KV cache takes one token per step"),
], ids=["no_window", "shorter_than_window", "not_64", "chunk_too_long", "fp8_prompt"])
def test_shape_rule_refusals(B, window, S, S_max, fp8, msg):
    with pytest.raises(RuntimeError, match=re.escape(msg)):
        _attn(B, window, S, S_max, fp8)


def test_rolling_false_is_the_windowed_operator(B):
    """rolling=False plans the schedule of the call without the keyword"""
    def sched(**kw):
        h = B.GraphHandler(B.HostPlanRuntime())
        kc, vc = h.tensor([2, 2, 128, 128], BF16), h.tensor([2, 2, 128, 128], BF16)
        q, k, v = h.tensor([2, 8, 1, 128], BF16), h.tensor([2, 2, 1, 128], BF16), h.tensor([2, 2, 1, 128], BF16)
        h.attentionKVCache(kc, vc, q, k, v, h.tensor([2, 1], I64), None, window=16, **kw).set_output()
        h.data_malloc()
        return h.schedule()
    assert sched() == sched(rolling=False)


def _fake(n=1):
    """host addresses that are never dereferenced: every refusal below happens before a launch"""
    return ctypes.c_void_p(0x1000 * n)


def _call(fn, flags, window=0, S=1, S_max=128):
    from infinitensor_b200 import _lib as L
    p = [_fake(i) for i in range(1, 16)]
    lib, ws = L.lib, 1 << 24
    if fn == "kvcache":
        return lib.it_b200_attention_kvcache(BF16, p[0], p[1], p[2], p[3], p[4], p[5], flags, p[6], 1, 4, S_max, 128, p[7], ws, None)
    if fn == "rope":
        return lib.it_b200_attention_kvcache_rope(BF16, p[0], p[1], p[2], p[3], p[4], p[5], flags, p[8], I64, p[6], 1, 4, S_max,
                                                  128, p[7], ws, None)
    if fn == "gqa":
        return lib.it_b200_attention_kvcache_gqa(BF16, p[0], p[1], p[2], p[3], p[4], p[5], flags, None, 0, p[6], 1, 4, 1, S_max,
                                                 128, p[7], ws, None)
    if fn == "fp8":
        return lib.it_b200_attention_kvcache_fp8(BF16, p[0], p[1], p[9], p[10], p[2], p[3], p[4], p[5], flags, None, 0, p[6], 1, 4,
                                                 1, S_max, 128, p[7], ws, None)
    if fn == "gqa_freq":
        return lib.it_b200_attention_kvcache_gqa_freq(BF16, p[0], p[1], p[2], p[3], p[4], p[5], flags, p[8], I64, p[11], F32, 64,
                                                      p[6], 1, 4, 1, S_max, 128, p[7], ws, None)
    if fn == "fp8_freq":
        return lib.it_b200_attention_kvcache_fp8_freq(BF16, p[0], p[1], p[9], p[10], p[2], p[3], p[4], p[5], flags, p[8], I64,
                                                      p[11], F32, 64, p[6], 1, 4, 1, S_max, 128, p[7], ws, None)
    if fn == "prompt":
        return lib.it_b200_attention_kvcache_prompt(BF16, p[0], p[1], p[2], p[3], p[4], p[5], flags, p[6], 1, 4, 1, 8, S_max, 128,
                                                    None)
    if fn == "window":
        return lib.it_b200_attention_kvcache_window(BF16, p[0], p[1], None, None, p[2], p[3], p[4], None, I64, None, F32, 0,
                                                    window, p[5], flags, p[6], 1, 4, 1, S_max, 128, p[7], ws, None)
    assert fn == "prompt_window"
    return lib.it_b200_attention_kvcache_prompt_window(BF16, p[0], p[1], p[2], p[3], p[4], p[5], flags, p[6], 1, 4, 1, S, S_max,
                                                       128, window, None)


@pytest.mark.parametrize("fn", ["kvcache", "rope", "gqa", "fp8", "gqa_freq", "fp8_freq", "prompt"])
def test_unwindowed_launchers_refuse_the_ring(B, fn):
    from infinitensor_b200 import _lib as L
    before = L.lib.it_b200_launch_count()
    assert _call(fn, I64 | RING) != 0
    err = L.last_error()
    assert "a rolling cache (ITB_POS_RING) needs a window" in err, err
    assert L.lib.it_b200_launch_count() == before


@pytest.mark.parametrize("fn", ["window", "prompt_window"])
@pytest.mark.parametrize("window,S,S_max,msg", [
    (0, 1, 128, "needs a window >= 1"),
    (129, 1, 128, "a rolling cache of 128 rows is shorter than the window of 129"),
    (64, 1, 96, "a rolling cache's length 96 is not a multiple of 64"),
    (100, 30, 128, "a chunk of 30 tokens needs a rolling cache of window + 29 = 129 rows or more, not 128"),
], ids=["no_window", "shorter_than_window", "not_64", "chunk_too_long"])
def test_windowed_launchers_refuse_each_ring_rule(B, fn, window, S, S_max, msg):
    from infinitensor_b200 import _lib as L
    if fn == "window" and S > 1:
        pytest.skip("the decode launcher takes one token per step")
    before = L.lib.it_b200_launch_count()
    assert _call(fn, I64 | RING, window, S, S_max) != 0
    err = L.last_error()
    assert err.startswith("AttentionKVCache prompt" if fn == "prompt_window" else "AttentionKVCache") and msg in err, err
    assert L.lib.it_b200_launch_count() == before


def test_native_attribute_vector(tmp_path):
    """AttentionKVCacheObj::getOpAttrVector: unchanged for a linear cache, {type, per-row flag, window, 1} for a ring (C++
    against core.cc / operators.cc / schedule.cc, no CUDA)"""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    host = os.path.join(root, "infinitensor_b200", "csrc", "host")
    exe = str(tmp_path / "test_ring_attrs")
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    cmd = [gxx, "-O1", "-std=c++17", "-Wall", "-I" + os.path.join(root, "include"), "-I" + host, "-o", exe,
           os.path.join(root, "tests", "native", "test_ring_attrs.cc")] + [os.path.join(host, f) for f in ("core.cc", "operators.cc", "schedule.cc")]
    subprocess.run(cmd, check=True, timeout=300)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and "passed" in r.stdout, r.stdout + r.stderr


# ---------------------------------------------------------------------------------------------------- graphs, ONNX
def _small(G, **kw):
    base = dict(layers=2, d_model=512, heads=4, kv_heads=2, head_dim=128, ffn=1024, vocab=128, s_max=64, batch=2,
                sliding_window=16)
    base.update(kw)
    return G.LlamaConfig(**base)


def _windowed_configs(G):
    return {"win_decode": (_small(G), 1), "win_prompt": (_small(G), 8), "win_fp8": (_small(G, kv_fp8=True), 1),
            "mistral_2l": (G.LlamaConfig.mistral_7b_v01(layers=2, batch=2, s_max=256), 1)}


def test_default_and_windowed_exports_unchanged(B, G):
    """rolling_cache False writes the export bytes and plans the schedules of graphs built before rings existed"""
    from infinitensor_b200 import onnx_lite as X
    from tests.test_kvfp8_host import EXPORT_SHA256
    from tests.test_swa_host import TINY_SHA256
    rt = B.HostPlanRuntime()
    exp = X.OnnxExporter(B.GraphHandler(rt))
    G.build_llama_decode(exp, dataclasses.replace(G.LlamaConfig.tiny(), rolling_cache=False))
    assert hashlib.sha256(exp.save()).hexdigest() == TINY_SHA256
    exp = X.OnnxExporter(B.GraphHandler(rt))
    G.build_llama_decode(exp, _small(G, kv_heads=None, s_max=32, batch=4, sliding_window=None))
    assert hashlib.sha256(exp.save()).hexdigest() == EXPORT_SHA256["llama"]
    for name, (cfg, seq) in _windowed_configs(G).items():
        exp = X.OnnxExporter(B.GraphHandler(rt))
        G.build_llama_decode(exp, cfg, seq=seq)
        h = B.GraphHandler(rt)
        G.build_llama_decode(h, cfg, seq=seq)
        h.data_malloc()
        got = (hashlib.sha256(exp.save()).hexdigest(), hashlib.sha256(repr(h.schedule()).encode()).hexdigest())
        assert got == WINDOWED_EXPORTS[name], name


def test_mistral_preset_with_a_ring(G):
    c = G.LlamaConfig.mistral_7b_v01(batch=32, s_max=4608, rolling_cache=True)
    assert (c.rolling_cache, c.sliding_window, c.s_max) == (True, 4096, 4608)
    assert not G.LlamaConfig.mistral_7b_v01().rolling_cache


@pytest.mark.parametrize("kw,seq", [({}, 1), ({}, 49), (dict(kv_fp8=True), 1), (dict(head_dim=64, d_model=256), 1),
                                    (dict(rope_theta=500000.0), 1), (dict(kv_heads=None), 8)],
                         ids=["gqa", "gqa_prompt_max", "kv_fp8", "d64", "table", "mha_prompt"])
def test_llama_graph_with_a_ring(B, G, kw, seq):
    """every layer's AttentionKVCache carries the ring; decode graphs still fold RoPE into it"""
    cfg = _small(G, rolling_cache=True, **kw)
    h = B.GraphHandler(B.HostPlanRuntime())
    G.build_llama_decode(h, cfg, seq=seq)
    h.data_malloc()
    sc = h.schedule()
    if seq == 1:
        assert sum(s.startswith("AttentionRope") for s in sc) == cfg.layers, sc


@pytest.mark.parametrize("kw,seq,msg", [
    (dict(sliding_window=None), 1, "rolling_cache needs a sliding_window"),
    (dict(s_max=96), 1, "s_max = 96"),
    (dict(), 50, "needs s_max >= window + seq - 1 = 65 and a multiple of 64 (e.g. 128)"),
    (dict(sliding_window=80), 1, "s_max = 64"),
], ids=["no_window", "not_64", "chunk_too_long", "shorter_than_window"])
def test_builder_checks_the_ring(B, G, kw, seq, msg):
    with pytest.raises(ValueError, match=re.escape(msg)):
        G.build_llama_decode(B.GraphHandler(B.HostPlanRuntime()), _small(G, rolling_cache=True, **kw), seq=seq)


@pytest.mark.parametrize("kw", [{}, dict(kv_fp8=True), dict(head_dim=64, d_model=256)], ids=["16bit", "kv_fp8", "d64"])
def test_onnx_round_trip_with_a_ring(B, G, kw):
    from infinitensor_b200 import onnx_lite as X
    rt = B.HostPlanRuntime()
    cfg = _small(G, rolling_cache=True, **kw)
    direct = B.GraphHandler(rt)
    G.build_llama_decode(direct, cfg)
    direct.data_malloc()
    exp = X.OnnxExporter(B.GraphHandler(rt))
    G.build_llama_decode(exp, cfg)
    blob = exp.save()
    m = X.load_model(blob)
    att = [n for n in m.graph.nodes if n.op_type == "AttentionKVCache"]
    assert len(att) == cfg.layers and all(int(n.attrs["window"]) == 16 and int(n.attrs["rolling"]) == 1 for n in att)
    h = B.GraphHandler(rt)
    X.OnnxStub(blob, handler=h, upload=False)
    h.data_malloc()
    assert h.schedule() == direct.schedule()
    exp2 = X.OnnxExporter(B.GraphHandler(rt))
    X.OnnxStub(blob, handler=exp2, upload=False)
    again = X.load_model(exp2.save())
    assert [(n.op_type, n.attrs) for n in again.graph.nodes] == [(n.op_type, n.attrs) for n in m.graph.nodes]


@pytest.mark.parametrize("world", [2, 4])
def test_parallel_model_keeps_the_ring(B, G, world):
    from infinitensor_b200 import onnx_lite as X
    rt = B.HostPlanRuntime()
    cfg = _small(G, heads=8, kv_heads=4, rolling_cache=True)
    exp = X.OnnxExporter(B.GraphHandler(rt))
    G.build_llama_decode(exp, cfg)
    for rank in range(world):
        direct = B.GraphHandler(rt)
        G.build_llama_decode(direct, cfg, world, rank)
        direct.data_malloc()
        sharded = X.parallel_model(exp.save(), world, rank)
        m = X.load_model(sharded) if isinstance(sharded, (bytes, bytearray)) else sharded
        att = [n for n in m.graph.nodes if n.op_type == "AttentionKVCache"]
        assert len(att) == cfg.layers and all(int(n.attrs["rolling"]) == 1 for n in att), "every rank keeps the ring"
        h = B.GraphHandler(rt)
        X.OnnxStub(sharded, handler=h, upload=False)
        h.data_malloc()
        assert h.schedule() == direct.schedule()


# ---------------------------------------------------------------------------------------------------- the CPU oracles
def test_handlers_without_rings_refuse_a_ring(B, G):
    """SwaOracleHandler has windows but no rings: it refuses a ring config from graphs and from an ONNX file"""
    from infinitensor_b200 import onnx_lite as X
    from tests import ring_oracle as RG
    from tests import swa_oracle as SO
    cfg = _small(G, kv_heads=None, rolling_cache=True)
    with pytest.raises(NotImplementedError, match="no rolling KV cache"):
        G.build_llama_decode(SO.SwaOracleHandler(), cfg)
    exp = X.OnnxExporter(B.GraphHandler(B.HostPlanRuntime()))
    G.build_llama_decode(exp, cfg)
    with pytest.raises(NotImplementedError, match="no rolling KV cache"):
        X.OnnxStub(exp.save(), handler=SO.SwaOracleHandler(), upload=False)
    G.build_llama_decode(SO.SwaOracleHandler(), dataclasses.replace(cfg, rolling_cache=False))
    G.build_llama_decode(RG.RingOracleHandler(), cfg)


def _linear_of(ring, lo, hi, total):
    """a linear cache of `total` rows holding positions lo .. hi - 1 of the ring (the rest NaN)"""
    S_max = ring.shape[2]
    lin = np.full(ring.shape[:2] + (total,) + ring.shape[3:], np.nan, ring.dtype)
    lin[:, :, lo:hi] = ring[:, :, np.arange(lo, hi) % S_max]
    return lin


@pytest.mark.parametrize("fp8", [False, True], ids=["16bit", "fp8"])
def test_ring_oracle_decode_equals_linear_window(fp8):
    """decode steps over a 64-row ring, wrapping it five times, equal the windowed oracle over a linear cache, bit for bit:
    the outputs, and the ring rows of the window after every step"""
    from tests import ring_oracle as RG
    from tests import swa_oracle as SO
    rng = np.random.default_rng(17)
    Bn, Hq, Hkv, S_max, D, W, steps = 2, 4, 2, 64, 64, 48, 330
    total = steps + 16
    starts = np.array([0, 9])  # rows at different wrap phases
    # the positions below the first step's hold the same values in both; the linear rows past the ring's are NaN
    lin, lin_v = (np.full((Bn, Hkv, total, D), np.nan, np.float32) for _ in range(2))
    scales = None
    if fp8:
        lin, lin_v = (np.full((Bn, Hkv, total, D), 0x7F, np.uint8) for _ in range(2))
        lin[:, :, :S_max], lin_v[:, :, :S_max] = (rng.integers(0, 0x70, (Bn, Hkv, S_max, D), dtype=np.uint8) for _ in range(2))
        scales = (np.full(Hkv, 0.02, np.float32), np.full(Hkv, 0.03, np.float32))
    else:
        lin[:, :, :S_max], lin_v[:, :, :S_max] = (rng.standard_normal((Bn, Hkv, S_max, D)).astype(np.float32) for _ in range(2))
    ring, ring_v = lin[:, :, :S_max].copy(), lin_v[:, :, :S_max].copy()
    for step in range(steps):
        q, k, v = (rng.standard_normal((Bn, n, 1, D)).astype(np.float32) for n in (Hq, Hkv, Hkv))
        pos = starts + step
        a = RG.ring_step(ring, ring_v, q, k, v, pos, BF16, W, scales)
        b = SO.window_step(lin, lin_v, q, k, v, pos, BF16, W, scales)
        assert np.array_equal(a, b), step
        for r in range(Bn):
            lo = max(0, pos[r] - W + 1)
            rows = np.arange(lo, pos[r] + 1)
            assert np.array_equal(ring[r][:, rows % S_max], lin[r][:, rows])


def test_ring_oracle_prompt_chunks_equal_linear_window():
    """prompt chunks of the largest size S_max - W + 1 over a ring, wrapping it several times, equal the windowed oracle
    over a linear cache bit for bit, and a chunk followed by decode steps equals decode steps alone"""
    from tests import ring_oracle as RG
    from tests import swa_oracle as SO
    rng = np.random.default_rng(23)
    Bn, Hq, Hkv, S_max, D, W = 2, 4, 2, 64, 64, 40
    S = S_max - W + 1
    total = 8 * S + 70
    lin, lin_v = (np.full((Bn, Hkv, total, D), np.nan, np.float32) for _ in range(2))
    lin[:, :, :S_max], lin_v[:, :, :S_max] = (rng.standard_normal((Bn, Hkv, S_max, D)).astype(np.float32) for _ in range(2))
    ring, ring_v = lin[:, :, :S_max].copy(), lin_v[:, :, :S_max].copy()
    starts = np.array([3, 30])
    p = starts.copy()
    for chunk in range(8):
        q, k, v = (rng.standard_normal((Bn, n, S, D)).astype(np.float32) for n in (Hq, Hkv, Hkv))
        pos = np.stack([p + i for i in range(S)], 1)
        a = RG.ring_prompt(ring, ring_v, q, k, v, pos, BF16, W, per_row=True)
        b = SO.window_prompt(lin, lin_v, q, k, v, pos, BF16, W, per_row=True)
        assert np.array_equal(a, b), chunk
        p = p + S
    for r in range(Bn):
        rows = np.arange(p[r] - W, p[r])
        assert np.array_equal(ring[r][:, rows % S_max], lin[r][:, rows])


def test_ring_oracle_far_positions_and_the_clamp():
    """a step at P near 10**6 equals the step at a small position over the same window contents, and positions are clamped
    to [0, INT32_MAX - S_max]"""
    from tests import ring_oracle as RG
    rng = np.random.default_rng(29)
    Bn, Hkv, S_max, D, W = 1, 1, 64, 64, 30
    base = rng.standard_normal((Bn, Hkv, S_max, D)).astype(np.float32)
    q, k, v = (rng.standard_normal((Bn, 1, 1, D)).astype(np.float32) for _ in range(3))
    outs = []
    for P in (100, 100 + 64 * 15625, RG.ring_pos_max(S_max), 2**40):
        kc, vc = base.copy(), base.copy() * 0.5
        shift = (min(P, RG.ring_pos_max(S_max)) - 100) % S_max  # rotate: the window's positions hold the same values
        kc, vc = np.roll(kc, shift, axis=2), np.roll(vc, shift, axis=2)
        outs.append(RG.ring_step(kc, vc, q, k, v, [P], BF16, W))
    assert np.array_equal(outs[0], outs[1]) and np.array_equal(outs[0], outs[2]) and np.array_equal(outs[2], outs[3])
    assert np.array_equal(RG.ring_starts([2**40], 1, S_max, False), [RG.ring_pos_max(S_max)])
    assert np.array_equal(RG.ring_starts([-5], 1, S_max, False), [0])


def test_ring_oracle_runs_a_ring_graph(G):
    """decode steps of a ring graph past s_max on the ring oracle equal the windowed oracle with a linear cache, bit for bit"""
    from tests import llama_oracle as LO
    from tests import ring_oracle as RG
    from tests import swa_oracle as SO
    ring_cfg = _small(G, layers=1, sliding_window=20, s_max=64, rolling_cache=True)
    lin_cfg = dataclasses.replace(ring_cfg, s_max=192, rolling_cache=False)
    ring_c = LO.llama_caches(ring_cfg)
    lin_c = LO.llama_caches(lin_cfg)
    for r, l in zip(ring_c, lin_c):  # the same 60-row prefix in both
        l[:, :, :60] = r[:, :, :60]
    rh, rg = RG.oracle_graph(ring_cfg, caches=ring_c)
    lh, lg = SO.oracle_graph(lin_cfg, caches=lin_c)
    for step in range(130):
        for g in (rg, lg):
            g.input_ids.copyin_numpy(np.array([[3 + step % 7], [5]], np.int64))
            g.position_ids.copyin_numpy(np.array([[59 + step], [59 + step]], np.int64))
        rh.run()
        lh.run()
        assert np.array_equal(rg.logits.f32(), lg.logits.f32()), step
