"""CPU tier for sliding-window attention (AttentionKVCache's `window`, LlamaConfig.sliding_window): the shape rule and the
launchers' refusals, default graphs unchanged, ONNX round trips and tensor-parallel sharding with a window, the AttentionRope
fold, the CPU oracle's refusal, the windowed test oracle against float64 and against itself, and a float32 emulation of the
windowed prompt kernel against the float64 bound the GPU tests apply (and the slips it must catch)."""
import ctypes
import dataclasses
import hashlib
import re

import numpy as np
import pytest

from tests import swa64

F32, F16, BF16, I64 = 1, 10, 16, 7
TINY_SHA256 = "634afe4b33636fcfc1a7ce0c2a4a96ae5a516cdacf294dc3bec882f14ccff0c1"


@pytest.fixture(scope="module")
def B():
    from infinitensor_b200 import backend
    return backend


@pytest.fixture(scope="module")
def G():
    from infinitensor_b200 import graphs
    return graphs


def _attn(B, window, S=1, S_max=64, fp8=False, per_row=False):
    """one AttentionKVCache on a host-planned graph: (handler, output)"""
    h = B.GraphHandler(B.HostPlanRuntime())
    Bn, Hq, Hkv, D = 2, 8, 2, 128
    cache = 17 if fp8 else BF16
    kc, vc = h.tensor([Bn, Hkv, S_max, D], cache), h.tensor([Bn, Hkv, S_max, D], cache)
    q, k, v = h.tensor([Bn, Hq, S, D], BF16), h.tensor([Bn, Hkv, S, D], BF16), h.tensor([Bn, Hkv, S, D], BF16)
    pos = h.tensor([Bn, S], I64)
    sc = {"k_scale": h.tensor([Hkv], F32), "v_scale": h.tensor([Hkv], F32)} if fp8 else {}
    return h, h.attentionKVCache(kc, vc, q, k, v, pos, None, per_row, **sc, window=window)


# ---------------------------------------------------------------------------------------------------- shape rule, refusals
@pytest.mark.parametrize("window", [0, 1, 16, 64, 100000])
@pytest.mark.parametrize("S", [1, 8])
def test_shape_rule_accepts_windows(B, window, S):
    assert _attn(B, window, S)[1].shape() == [2, 8, S, 128]


@pytest.mark.parametrize("S", [1, 8])
def test_shape_rule_refuses_a_negative_window(B, S):
    with pytest.raises(RuntimeError, match=re.escape("AttentionKVCache: window -1 is negative")):
        _attn(B, -1, S)


def _schedule(B, window, per_row=False, fp8=False):
    h, out = _attn(B, window, per_row=per_row, fp8=fp8)
    out.set_output()
    h.data_malloc()
    return h.schedule()


def test_window_zero_is_the_unwindowed_operator(B):
    """a window-0 AttentionKVCache plans the same schedule as the call without the keyword"""
    Bn, Hq, Hkv, D, S_max = 2, 8, 2, 128, 64
    a = _schedule(B, 0)
    h = B.GraphHandler(B.HostPlanRuntime())
    kc, vc = h.tensor([Bn, Hkv, S_max, D], BF16), h.tensor([Bn, Hkv, S_max, D], BF16)
    q, k, v = h.tensor([Bn, Hq, 1, D], BF16), h.tensor([Bn, Hkv, 1, D], BF16), h.tensor([Bn, Hkv, 1, D], BF16)
    h.attentionKVCache(kc, vc, q, k, v, h.tensor([Bn, 1], I64), None).set_output()
    h.data_malloc()
    assert a == h.schedule()


def _fake(n=1):
    """host addresses that are never dereferenced: every refusal below happens before a launch"""
    return ctypes.c_void_p(0x1000 * n)


@pytest.mark.parametrize("fn", ["decode", "decode_fp8", "decode_rope_table", "prompt"])
def test_launchers_refuse_a_negative_window_before_launching(B, fn):
    from infinitensor_b200 import _lib as L
    before = L.lib.it_b200_launch_count()
    p = [_fake(i) for i in range(1, 16)]
    if fn == "prompt":
        rc = L.lib.it_b200_attention_kvcache_prompt_window(BF16, p[0], p[1], p[2], p[3], p[4], p[5], I64, p[6], 1, 4, 1, 8, 64,
                                                           128, -3, None)
        what = "AttentionKVCache prompt"
    else:
        fp8 = fn == "decode_fp8"
        table = fn == "decode_rope_table"
        rc = L.lib.it_b200_attention_kvcache_window(BF16, p[0], p[1], p[7] if fp8 else None, p[8] if fp8 else None, p[2], p[3],
                                                    p[4], p[9] if table else None, I64, p[10] if table else None, F32, 64, -3,
                                                    p[5], I64, p[6], 1, 4, 1, 64, 128, p[11], 1 << 20, None)
        what = "AttentionKVCache"
    assert rc != 0
    err = L.last_error()
    assert err.startswith(what) and "window -3 is negative" in err, err
    assert L.lib.it_b200_launch_count() == before


def test_decode_launcher_refuses_half_a_scale_pair(B):
    from infinitensor_b200 import _lib as L
    p = [_fake(i) for i in range(1, 16)]
    rc = L.lib.it_b200_attention_kvcache_window(BF16, p[0], p[1], p[7], None, p[2], p[3], p[4], None, I64, None, F32, 0, 4,
                                                p[5], I64, p[6], 1, 4, 1, 64, 128, p[11], 1 << 20, None)
    assert rc != 0 and "k_scale and v_scale go together" in L.last_error()


# ---------------------------------------------------------------------------------------------------- graphs, ONNX
def _small(G, **kw):
    base = dict(layers=2, d_model=512, heads=4, kv_heads=2, head_dim=128, ffn=1024, vocab=128, s_max=64, batch=2,
                sliding_window=16)
    base.update(kw)
    return G.LlamaConfig(**base)


def test_mistral_preset(G):
    c = G.LlamaConfig.mistral_7b_v01(batch=8, s_max=16384)
    assert (c.layers, c.d_model, c.heads, c.n_kv, c.head_dim, c.ffn, c.vocab, c.rope_theta, c.sliding_window) == \
        (32, 4096, 32, 8, 128, 14336, 32000, 10000.0, 4096)
    assert c.rope_default and (c.batch, c.s_max) == (8, 16384)
    k = G.LlamaConfig.mistral_7b_v01(kv_fp8=True, int4_block=64, dtype=F16)
    assert (k.kv_fp8, k.int4_block, k.dtype) == (True, 64, F16)


def test_algorithmic_bytes(G):
    """a window counts min(pos + 1, W) cache rows read; every unwindowed config's count is unchanged"""
    m = G.LlamaConfig.mistral_7b_v01(batch=8, s_max=16384)
    nw = dataclasses.replace(m, sliding_window=None)
    per_row = m.layers * 2 * m.batch * m.n_kv * m.head_dim * 2  # bytes of one cache row of every layer, k and v
    assert nw.algorithmic_bytes(16383) - m.algorithmic_bytes(16383) == (16384 - 4096) * per_row
    assert m.algorithmic_bytes(100) == nw.algorithmic_bytes(100)
    assert m.algorithmic_bytes(4095) == nw.algorithmic_bytes(4095)
    # the formula of every unwindowed config, restated
    c = G.LlamaConfig.llama3_8b()
    e, d, f, dkv = 2, c.d_model, c.ffn, c.n_kv * c.head_dim
    want = (c.layers * (2 * d * d + 2 * d * dkv + 3 * d * f) + d * c.vocab + c.layers * 2 * d + d + c.layers * 12 * c.batch * d) * e \
        + c.layers * 2 * c.batch * c.n_kv * c.head_dim * (700 + 2) * e
    assert c.algorithmic_bytes(700) == want


@pytest.mark.parametrize("kw,seq", [({}, 1), ({}, 8), (dict(kv_fp8=True), 1), (dict(head_dim=64, d_model=256), 1),
                                    (dict(int4_block=64), 1), (dict(rope_theta=500000.0), 1), (dict(kv_heads=None), 8)],
                         ids=["gqa", "gqa_prompt", "kv_fp8", "d64", "int4", "table", "mha_prompt"])
def test_llama_graph_with_a_window(B, G, kw, seq):
    """every layer's AttentionKVCache carries the window; decode graphs fold RoPE into it"""
    cfg = _small(G, **kw)
    h = B.GraphHandler(B.HostPlanRuntime())
    G.build_llama_decode(h, cfg, seq=seq)
    h.data_malloc()
    sc = h.schedule()
    if seq == 1:
        assert sum(s.startswith("AttentionRope") for s in sc) == cfg.layers, sc


def test_default_graphs_unchanged(B, G):
    """sliding_window None (and 0) writes the pinned export bytes and plans the same schedule as before windows existed"""
    from infinitensor_b200 import onnx_lite as X
    from tests.test_kvfp8_host import EXPORT_SHA256
    rt = B.HostPlanRuntime()
    for sw in (None, 0):
        exp = X.OnnxExporter(B.GraphHandler(rt))
        G.build_llama_decode(exp, dataclasses.replace(G.LlamaConfig.tiny(), sliding_window=sw), seq=1)
        assert hashlib.sha256(exp.save()).hexdigest() == TINY_SHA256
    exp = X.OnnxExporter(B.GraphHandler(rt))
    G.build_llama_decode(exp, _small(G, kv_heads=None, s_max=32, batch=4, sliding_window=None))
    assert hashlib.sha256(exp.save()).hexdigest() == EXPORT_SHA256["llama"]
    scheds = []
    for sw in (None, 0):
        h = B.GraphHandler(rt)
        G.build_llama_decode(h, dataclasses.replace(G.LlamaConfig.tiny(), sliding_window=sw))
        h.data_malloc()
        scheds.append(h.schedule())
    assert scheds[0] == scheds[1]


def test_builder_refuses_a_negative_window(B, G):
    with pytest.raises(ValueError, match="sliding_window"):
        G.build_llama_decode(B.GraphHandler(B.HostPlanRuntime()), _small(G, sliding_window=-4))


@pytest.mark.parametrize("kw", [{}, dict(kv_fp8=True), dict(head_dim=64, d_model=256)], ids=["16bit", "kv_fp8", "d64"])
def test_onnx_round_trip_with_a_window(B, G, kw):
    from infinitensor_b200 import onnx_lite as X
    rt = B.HostPlanRuntime()
    cfg = _small(G, **kw)
    direct = B.GraphHandler(rt)
    G.build_llama_decode(direct, cfg)
    direct.data_malloc()
    exp = X.OnnxExporter(B.GraphHandler(rt))
    G.build_llama_decode(exp, cfg)
    blob = exp.save()
    m = X.load_model(blob)
    att = [n for n in m.graph.nodes if n.op_type == "AttentionKVCache"]
    assert len(att) == cfg.layers and all(int(n.attrs["window"]) == 16 for n in att)
    h = B.GraphHandler(rt)
    X.OnnxStub(blob, handler=h, upload=False)
    h.data_malloc()
    assert h.schedule() == direct.schedule()
    exp2 = X.OnnxExporter(B.GraphHandler(rt))
    X.OnnxStub(blob, handler=exp2, upload=False)
    again = X.load_model(exp2.save())
    assert [(n.op_type, n.attrs) for n in again.graph.nodes] == [(n.op_type, n.attrs) for n in m.graph.nodes]


def test_onnx_window_refused_by_a_handler_without_one(B, G):
    from infinitensor_b200 import onnx_lite as X
    from oracle.graph_oracle import OracleHandler
    exp = X.OnnxExporter(B.GraphHandler(B.HostPlanRuntime()))
    G.build_llama_decode(exp, _small(G, kv_heads=None))
    with pytest.raises(NotImplementedError, match="sliding window"):
        X.OnnxStub(exp.save(), handler=OracleHandler(), upload=False)


@pytest.mark.parametrize("world", [2, 4])
def test_parallel_model_keeps_the_window(B, G, world):
    from infinitensor_b200 import onnx_lite as X
    rt = B.HostPlanRuntime()
    cfg = _small(G, heads=8, kv_heads=4)
    exp = X.OnnxExporter(B.GraphHandler(rt))
    G.build_llama_decode(exp, cfg)
    for rank in range(world):
        direct = B.GraphHandler(rt)
        G.build_llama_decode(direct, cfg, world, rank)
        direct.data_malloc()
        sharded = X.parallel_model(exp.save(), world, rank)
        m = X.load_model(sharded) if isinstance(sharded, (bytes, bytearray)) else sharded
        att = [n for n in m.graph.nodes if n.op_type == "AttentionKVCache"]
        assert len(att) == cfg.layers and all(int(n.attrs["window"]) == 16 for n in att), "every rank keeps the window"
        h = B.GraphHandler(rt)
        X.OnnxStub(sharded, handler=h, upload=False)
        h.data_malloc()
        assert h.schedule() == direct.schedule()


@pytest.mark.parametrize("fp8", [False, True], ids=["16bit", "fp8"])
def test_rope_fold_carries_the_window(B, fp8):
    """RoPE(q), RoPE(k) fold into a windowed AttentionKVCache as into an unwindowed one; the window stays on the operator the
    fused step launches (its attribute vector)"""
    h = B.GraphHandler(B.HostPlanRuntime())
    Bn, Hq, Hkv, D, S = 2, 8, 2, 128, 64
    cache = 17 if fp8 else BF16
    pos = h.tensor([Bn, 1], I64)
    pos.set_input()
    q, k, v = h.tensor([Bn, 1, Hq * D], BF16), h.tensor([Bn, 1, Hkv * D], BF16), h.tensor([Bn, 1, Hkv * D], BF16)
    q, k = h.RoPE(pos, q, None), h.RoPE(pos, k, None)
    heads = lambda t, n: h.transpose(h.reshape(t, None, [Bn, 1, n, D]), None, [0, 2, 1, 3])
    kc, vc = h.tensor([Bn, Hkv, S, D], cache), h.tensor([Bn, Hkv, S, D], cache)
    sc = {"k_scale": h.tensor([Hkv], F32), "v_scale": h.tensor([Hkv], F32)} if fp8 else {}
    h.attentionKVCache(kc, vc, heads(q, Hq), heads(k, Hkv), heads(v, Hkv), pos, None, **sc, window=5).set_output()
    h.data_malloc()
    sc_ = h.schedule()
    assert sum(s.startswith("AttentionRope") for s in sc_) == 1 and not any(s.startswith("Single") and "RoPE" in s for s in sc_)


# ---------------------------------------------------------------------------------------------------- the CPU oracles
def test_oracle_handler_refuses_a_window(G):
    from oracle.graph_oracle import OracleHandler
    from tests import llama_oracle as LO
    from tests import rope_oracle as RO
    for h in (OracleHandler(), LO.LlamaOracleHandler(), RO.RopeOracleHandler()):
        with pytest.raises(NotImplementedError, match="sliding-window"):
            G.build_llama_decode(h, _small(G, kv_heads=None))
    G.build_llama_decode(OracleHandler(), _small(G, kv_heads=None, sliding_window=None))


@pytest.mark.parametrize("fp8", [False, True], ids=["16bit", "fp8"])
@pytest.mark.parametrize("D", [64, 128])
def test_oracle_window_step_against_float64(D, fp8):
    """the oracle's windowed step (its own rule on the shifted view) against the float64 windowed reference, within the bound"""
    from tests import attn64
    from tests import kvfp8_oracle as KV
    from tests import swa_oracle as SO
    rng = np.random.default_rng(3)
    Bn, Hq, Hkv, S_max, W = 3, 4, 2, 96, 20
    pos = np.array([5, 40, 95])
    kc = attn64.exact(rng.standard_normal((Bn, Hkv, S_max, D)).astype(np.float32))
    vc = attn64.exact(rng.standard_normal((Bn, Hkv, S_max, D)).astype(np.float32))
    q = attn64.exact(rng.standard_normal((Bn, Hq, 1, D)).astype(np.float32) * 2)
    k = attn64.exact(rng.standard_normal((Bn, Hkv, 1, D)).astype(np.float32))
    v = attn64.exact(rng.standard_normal((Bn, Hkv, 1, D)).astype(np.float32))
    for b in range(Bn):  # rows below the window and above the position are poison
        kc[b, :, :max(0, pos[b] - W + 1)] = np.nan
        vc[b, :, :max(0, pos[b] - W + 1)] = np.nan
        kc[b, :, pos[b]:] = np.nan
        vc[b, :, pos[b]:] = np.nan
    if fp8:
        ksc, vsc = np.full(Hkv, 0.02, np.float32), np.full(Hkv, 0.03, np.float32)
        kq, vq = KV.quantise(np.nan_to_num(kc), ksc[None, :, None, None]), KV.quantise(np.nan_to_num(vc), vsc[None, :, None, None])
        kq[np.isnan(kc)], vq[np.isnan(vc)] = 0x7F, 0x7F  # E4M3 NaN codes
        got = SO.window_step(kq, vq, q, k, v, pos, BF16, W, (ksc, vsc))
        for b in range(Bn):
            lo = max(0, pos[b] - W + 1)
            ref, bd = KV.attention(kq[b:b + 1, :, lo:], vq[b:b + 1, :, lo:], ksc, vsc, q[b:b + 1], [pos[b] - lo], BF16)
            assert np.isfinite(got[b]).all() and np.all(np.abs(got[b:b + 1].astype(np.float64) - ref) <= bd)
        return
    got = SO.window_step(kc, vc, q, k, v, pos, BF16, W)
    assert np.array_equal(kc[np.arange(Bn), :, pos], k[:, :, 0]) and np.array_equal(vc[np.arange(Bn), :, pos], v[:, :, 0])
    refs = swa64.decode_refs(kc, vc, q, pos, W)
    bad = attn64.violations(got[:, :, 0], refs, BF16, True)
    assert not bad.any()


@pytest.mark.parametrize("per_row", [False, True], ids=["element0", "per_row"])
def test_oracle_prompt_equals_decode_steps(G, per_row):
    """on the windowed oracle, a prompt step of S tokens followed by a decode step equals S + 1 decode steps, bit for bit"""
    from tests import swa_oracle as SO
    rng = np.random.default_rng(5)
    Bn, Hq, Hkv, S_max, D, S, W = 2, 4, 2, 64, 128, 12, 7
    kc0 = rng.standard_normal((Bn, Hkv, S_max, D)).astype(np.float32)
    vc0 = rng.standard_normal((Bn, Hkv, S_max, D)).astype(np.float32)
    q = rng.standard_normal((Bn, Hq, S + 1, D)).astype(np.float32)
    k = rng.standard_normal((Bn, Hkv, S + 1, D)).astype(np.float32)
    v = rng.standard_normal((Bn, Hkv, S + 1, D)).astype(np.float32)
    starts = np.array([20, 33]) if per_row else np.array([20, 20])
    pos = np.stack([starts + i for i in range(S)], 1)
    kc1, vc1 = kc0.copy(), vc0.copy()
    a = SO.window_prompt(kc1, vc1, q[:, :, :S], k[:, :, :S], v[:, :, :S], pos, BF16, W, per_row)
    a = np.concatenate([a, SO.window_step(kc1, vc1, q[:, :, S:], k[:, :, S:], v[:, :, S:], starts + S, BF16, W)], 2)
    kc2, vc2 = kc0.copy(), vc0.copy()
    b = np.concatenate([SO.window_step(kc2, vc2, q[:, :, i:i + 1], k[:, :, i:i + 1], v[:, :, i:i + 1], starts + i, BF16, W)
                        for i in range(S + 1)], 2)
    assert np.array_equal(a, b) and np.array_equal(kc1, kc2) and np.array_equal(vc1, vc2)


def test_oracle_window_beyond_the_position_is_no_window(G):
    """a window that covers every row gives the unwindowed oracle's output bit for bit"""
    from tests import llama_oracle as LO
    from tests import swa_oracle as SO
    rng = np.random.default_rng(7)
    kc = rng.standard_normal((2, 2, 48, 128)).astype(np.float32)
    vc = rng.standard_normal((2, 2, 48, 128)).astype(np.float32)
    q, k, v = (rng.standard_normal((2, n, 1, 128)).astype(np.float32) for n in (8, 2, 2))
    pos = np.array([30, 47])
    a = SO.window_step(kc.copy(), vc.copy(), q, k, v, pos, BF16, 48)
    b = LO.attention_kvcache_d(kc.copy(), vc.copy(), q, k, v, pos, BF16)
    assert np.array_equal(a, b)


def test_swa_oracle_runs_a_window_graph(G):
    """one decode step of a windowed graph on the windowed oracle: finite logits that differ from the unwindowed graph's"""
    from tests import swa_oracle as SO
    cfg = _small(G, layers=1, sliding_window=4)
    logits = []
    for c in (cfg, dataclasses.replace(cfg, sliding_window=None)):
        oh, og = SO.oracle_graph(c)
        og.input_ids.copyin_numpy(np.array([[3], [5]], np.int64))
        og.position_ids.copyin_numpy(np.array([[40], [63]], np.int64))
        oh.run()
        logits.append(og.logits.f32())
    assert np.isfinite(logits[0]).all() and not np.array_equal(logits[0], logits[1])


# ---------------------------------------------------------------------------------------------------- emulation vs bound
PROMPT_CASES = {
    # (B, Hq, Hkv, S, S_max, p, D, window): S below and above W, windows starting inside a key tile and on a tile boundary,
    # the first query's window starting at 0 and past it, per-row starts
    "inside_tile": (2, 2, 1, 80, 256, [100, 37], 128, 50),
    "on_tile": (1, 2, 2, 70, 256, 128, 64, 65),
    "s_above_w": (1, 4, 1, 150, 320, 90, 128, 33),
    "from_zero": (1, 2, 1, 64, 128, 10, 64, 40),
}


@pytest.mark.parametrize("dt", [F16, BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", sorted(PROMPT_CASES))
def test_prompt_emulation_within_half_the_bound(case, dt):
    c = swa64.Case(*PROMPT_CASES[case][:7], seed=11, window=PROMPT_CASES[case][7])
    refs = c.reference()
    got = swa64.emulate(c, dt)
    bad = swa64.prompt64.violations(got, refs, dt, 0.5)
    assert not bad.any(), swa64.prompt64.report(bad, got, refs, dt, c, case)


@pytest.mark.parametrize("slip", swa64.SLIPS)
def test_bound_catches_slips(slip):
    c = swa64.Case(2, 2, 1, 80, 256, [100, 37], 128, seed=11, window=50)
    refs = c.reference()
    got = swa64.emulate(c, BF16, slip)
    assert swa64.prompt64.violations(got, refs, BF16).any(), f"{slip} stays within the bound"


def test_decode_deal_reaches_every_split_state():
    """the windowed dealing (the unwindowed one at the span positions) reaches whole heads, 2-way, >= 3-way and 256-way merges
    on the GPU tests' decode cases"""
    from tests.test_gpu_swa import DECODE_CASES
    seen = set()
    for name, c in DECODE_CASES.items():
        dl = swa64.deal(c["dt"], c["B"], c["Hq"], c["Hkv"], c["S_max"], c["pos"], c["W"], c["D"], c.get("fp8", False))
        seen |= set(swa64.split_states(dl))
    assert 1 in seen and 2 in seen and any(3 <= n < 256 for n in seen) and max(seen) >= 256, sorted(seen)


def test_native_attribute_vector(tmp_path):
    """AttentionKVCacheObj::getOpAttrVector: {type, per-row flag} at window 0, as before windows existed, and the window
    appended otherwise (C++ against core.cc / operators.cc / schedule.cc, no CUDA)"""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    host = os.path.join(root, "infinitensor_b200", "csrc", "host")
    exe = str(tmp_path / "test_swa_attrs")
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    cmd = [gxx, "-O1", "-std=c++17", "-Wall", "-I" + os.path.join(root, "include"), "-I" + host, "-o", exe,
           os.path.join(root, "tests", "native", "test_swa_attrs.cc")] + [os.path.join(host, f) for f in ("core.cc", "operators.cc", "schedule.cc")]
    subprocess.run(cmd, check=True, timeout=300)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and "passed" in r.stdout, r.stdout + r.stderr
