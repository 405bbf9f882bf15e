"""CPU tier for grouped-query AttentionKVCache: the operator's shape rule, the schedule of a GQA Llama graph, the test
oracle's head mapping, the kernel's unit partition over KV heads, and ONNX / tensor-parallel handling of GQA graphs."""
import collections

import numpy as np
import pytest

F32, BF16, I64 = 1, 16, 7


@pytest.fixture(scope="module")
def B():
    from infinitensor_b200 import backend
    return backend


def _att(B, cache, q, k=None, v=None):
    h = B.GraphHandler(B.HostPlanRuntime())
    kc, vc = h.tensor(cache, F32), h.tensor(cache, F32)
    kt = k or [cache[0], cache[1], q[2], cache[3]]
    qt, kk, vv = h.tensor(q, F32), h.tensor(kt, F32), h.tensor(v or kt, F32)
    pos = h.tensor([1], I64)
    return h.attentionKVCache(kc, vc, qt, kk, vv, pos, None)


@pytest.mark.parametrize("G", [1, 2, 7, 32, 48])
def test_shape_rule_accepts_grouped_query_heads(B, G):
    out = _att(B, [2, 3, 16, 128], [2, 3 * G, 1, 128])
    assert out.shape() == [2, 3 * G, 1, 128]


@pytest.mark.parametrize("cache,q,k", [
    ([2, 3, 16, 128], [2, 8, 1, 128], None),                        # 8 query heads over 3 KV heads
    ([2, 4, 16, 128], [2, 8, 1, 128], [2, 8, 1, 128]),              # k / v head count differs from the caches'
    ([2, 4, 16, 128], [2, 8, 1, 64], [2, 4, 1, 64]),                # head dim differs from the caches'
    ([2, 4, 16, 128], [3, 8, 1, 128], [3, 4, 1, 128]),              # batch differs from the caches'
])
def test_shape_rule_rejects_malformed_graphs(B, cache, q, k):
    with pytest.raises(RuntimeError):
        _att(B, cache, q, k)


def _cfg(kv_heads, **kw):
    from infinitensor_b200 import graphs as G
    base = dict(layers=2, d_model=512, heads=4, head_dim=128, ffn=1024, vocab=128, s_max=32, batch=16)
    base.update(kw)
    return G.LlamaConfig(kv_heads=kv_heads, **base)


def test_gqa_llama_schedule(B):
    """both RoPEs fold into one AttentionRope step per layer"""
    from infinitensor_b200 import graphs as G
    rt = B.HostPlanRuntime()
    for kv in (2, 1):
        h = B.GraphHandler(rt)
        g = G.build_llama_decode(h, _cfg(kv))
        assert g.k_caches[0].shape() == [16, kv, 32, 128]
        assert g.weights["l0.wk"][0].shape() == [512, kv * 128] and g.weights["l0.wq"][0].shape() == [512, 512]
        sc = h.schedule()
        assert sc.count("AttentionRope:RoPE+RoPE+AttentionKVCache") == 2
        assert not any(s.startswith("Single:RoPE") for s in sc)
        kinds = collections.Counter(s.split(":")[0] for s in sc)
        assert kinds["AttentionRope"] == 2 and kinds["MatMulGroup"] == 4
        h.data_malloc()
    h = B.GraphHandler(rt)
    G.build_llama_decode(h, _cfg(2))
    assert sum(s.startswith("AttentionRope") for s in h.schedule()) == 2


def test_equal_heads_schedule_unchanged(B):
    """kv_heads=None and kv_heads=heads build the very graph the equal-heads builder always built"""
    from infinitensor_b200 import graphs as G
    rt = B.HostPlanRuntime()
    scheds = []
    for kv in (None, 4):
        h = B.GraphHandler(rt)
        G.build_llama_decode(h, _cfg(kv))
        scheds.append(h.schedule())
    assert scheds[0] == scheds[1]
    assert G.LlamaConfig().algorithmic_bytes(511) == G.LlamaConfig(kv_heads=32).algorithmic_bytes(511)
    assert G.LlamaConfig().weight_elems() == G.LlamaConfig(kv_heads=32).weight_elems()


def test_llama3_8b_bytes():
    """the Llama-3-8B shape: ~15.0 GB of weights, ~1.08 GB of KV at p = 511, ~16.1 GB per step"""
    from infinitensor_b200 import graphs as G
    c = G.LlamaConfig.llama3_8b()
    assert (c.heads, c.kv_heads, c.d_model, c.ffn, c.vocab, c.layers, c.batch, c.s_max) == (32, 8, 4096, 14336, 128256, 32, 16, 1024)
    kv = c.layers * 2 * c.batch * c.kv_heads * 128 * (511 + 2) * 2
    assert abs(kv / 1e9 - 1.08) < 0.01
    assert abs(c.algorithmic_bytes(511) / 1e9 - 16.1) < 0.1
    assert abs((c.weight_elems() - c.vocab * c.d_model) * 2 / 1e9 - 15.0) < 0.1  # the embedding table is gathered, not streamed


def _repeat_kv_reference(kc, vc, q, k, v, pos):
    """float64: append, expand the caches to Hq heads in repeat_kv order, stable softmax"""
    kc, vc = kc.astype(np.float64).copy(), vc.astype(np.float64).copy()
    kc[:, :, pos], vc[:, :, pos] = k[:, :, 0], v[:, :, 0]
    G = q.shape[1] // kc.shape[1]
    ke, ve = np.repeat(kc[:, :, :pos + 1], G, axis=1), np.repeat(vc[:, :, :pos + 1], G, axis=1)
    s = np.einsum("bhd,bhsd->bhs", q[:, :, 0].astype(np.float64), ke) / np.sqrt(128.0)
    p = np.exp(s - s.max(-1, keepdims=True))
    return (np.einsum("bhs,bhsd->bhd", p, ve) / p.sum(-1, keepdims=True))[:, :, None]


@pytest.mark.parametrize("G", [2, 4, 7, 32, 48])
def test_oracle_head_mapping(G):
    from tests.llama_oracle import attention_kvcache_gqa
    rng = np.random.default_rng(G)
    Bn, Hkv, S, pos = 2, 2, 40, 33
    kc = (rng.standard_normal((Bn, Hkv, S, 128)) * 0.5).astype(np.float32)
    vc = (rng.standard_normal((Bn, Hkv, S, 128)) * 0.5).astype(np.float32)
    q = (rng.standard_normal((Bn, Hkv * G, 1, 128)) * 0.5).astype(np.float32)
    k = (rng.standard_normal((Bn, Hkv, 1, 128)) * 0.5).astype(np.float32)
    v = (rng.standard_normal((Bn, Hkv, 1, 128)) * 0.5).astype(np.float32)
    ref = _repeat_kv_reference(kc, vc, q, k, v, pos)
    kc2, vc2 = kc.copy(), vc.copy()
    got = attention_kvcache_gqa(kc2, vc2, q, k, v, pos, F32)
    np.testing.assert_allclose(got, ref, rtol=1e-5, atol=1e-6)
    assert np.array_equal(kc2[:, :, pos], k[:, :, 0]) and np.array_equal(vc2[:, :, pos], v[:, :, 0])


def _check_partition(pre, Hkv, nch, grid):
    """attn_gqa_kernel: units (batch row, KV head, query group, chunk), Hkv here counting (KV head, query group) segments;
    pre[b] = units before row b = sum of Hkv * nch[b']"""
    total = pre[-1]
    ncta = min(grid, total)
    owner = {}
    for i in range(ncta):
        u0, u1 = i * total // ncta, (i + 1) * total // ncta
        assert u1 > u0
        b = 0
        while b + 1 < len(nch) and pre[b + 1] <= u0:
            b += 1
        assert pre[b] <= u0 < pre[b + 1]
        for u in range(u0, u1):
            assert u not in owner
            owner[u] = i
    assert len(owner) == total
    for b in range(len(nch)):
        for kvh in range(Hkv):
            hu0 = pre[b] + kvh * nch[b]
            first, last = ((hu0 + 1) * ncta - 1) // total, ((hu0 + nch[b]) * ncta - 1) // total
            assert sorted({owner[hu0 + c] for c in range(nch[b])}) == list(range(first, last + 1))
            assert last - first + 1 <= nch[b]  # the partial-slot index stays below slots per query head


def test_gqa_unit_partition_properties():
    rng = np.random.default_rng(0)
    # segments per batch row = KV heads x query groups (ceil(G / 32) groups when G > 32, e.g. 2 for G = 48)
    for Bn, Hkv in ((1, 1), (2, 2), (16, 8), (3, 4), (7, 3), (5, 1), (3, 1 * 2), (2, 2 * 3)):
        for uniform in (True, False):
            for _ in range(4):
                nch = [int(rng.integers(1, 17))] * Bn if uniform else rng.integers(1, 17, size=Bn).tolist()
                pre = [0]
                for b in range(Bn):
                    pre.append(pre[-1] + Hkv * nch[b])
                for grid in (1, 3, 8, 31, 264):
                    _check_partition(pre, Hkv, nch, grid)


def _gqa_onnx_cfg(kv, dtype=F32):
    from infinitensor_b200 import graphs as G
    return G.LlamaConfig(layers=2, d_model=512, heads=4, kv_heads=kv, head_dim=128, ffn=1024, vocab=128, s_max=32, batch=16,
                         dtype=dtype)


def test_gqa_onnx_roundtrip_schedule_and_oracle():
    """OnnxExporter -> OnnxStub of a GQA graph: same schedule on the C++ host, identical oracle bits"""
    from infinitensor_b200 import backend as B, graphs as G, onnx_lite as X
    from tests.llama_oracle import LlamaOracleHandler
    rt = B.HostPlanRuntime()
    cfg = _gqa_onnx_cfg(2)
    h = B.GraphHandler(rt)
    G.build_llama_decode(h, cfg)
    exp = X.OnnxExporter(B.GraphHandler(rt))
    G.build_llama_decode(exp, cfg)
    stub_h = B.GraphHandler(rt)
    X.OnnxStub(exp.save(), handler=stub_h, upload=False)
    assert stub_h.schedule() == h.schedule()

    small = G.LlamaConfig(layers=2, d_model=512, heads=4, kv_heads=1, head_dim=128, ffn=384, vocab=96, s_max=16, batch=3,
                          dtype=F32)
    exp = X.OnnxExporter(LlamaOracleHandler())
    ge = G.build_llama_decode(exp, small)
    exp.data_malloc()
    G.fill_llama_weights_host(ge)
    blob = exp.save()
    stub = X.OnnxStub(blob, handler=LlamaOracleHandler())
    oh = LlamaOracleHandler()
    gd = G.build_llama_decode(oh, small)
    oh.data_malloc()
    G.fill_llama_weights_host(gd)
    rng = np.random.default_rng(5)
    names_in = [t.name for t in exp._inputs]
    gi = [t for t in oh.tensors if t.is_input]
    assert len(gi) == len(names_in) == len(stub.inputs)
    for name, t in zip(names_in, gi):
        shp, dt = t.shape(), t.dtype()
        val = rng.integers(0, 7, size=shp).astype(np.int64) if dt == I64 else (rng.standard_normal(shp) * 0.5).astype(np.float32)
        t.copyin_numpy(val)
        stub.inputs[name].copyin_numpy(val)
    oh.run()
    stub.run()
    outs = [t for t in oh.tensors if t.is_output]
    assert len(outs) == len(stub.outputs) == 1
    for t, (_, s) in zip(outs, stub.outputs.items()):
        np.testing.assert_array_equal(t.copyout_numpy(), s.copyout_numpy())


def test_gqa_parallel_model_matches_direct_tp_build():
    from infinitensor_b200 import backend as B, graphs as G, onnx_lite as X
    rt = B.HostPlanRuntime()
    cfg = _gqa_onnx_cfg(2)
    direct = B.GraphHandler(rt)
    G.build_llama_decode(direct, cfg, 2, 1)
    exp = X.OnnxExporter(B.GraphHandler(rt))
    G.build_llama_decode(exp, cfg)
    sharded = X.parallel_model(exp.save(), 2, 1)
    h = B.GraphHandler(rt)
    X.OnnxStub(sharded, handler=h, upload=False)
    assert h.schedule() == direct.schedule()
    h.data_malloc()
    direct.data_malloc()
    assert h.arena_bytes() == direct.arena_bytes()
    # one KV head does not split over two ranks
    exp1 = X.OnnxExporter(B.GraphHandler(rt))
    G.build_llama_decode(exp1, _gqa_onnx_cfg(1))
    with pytest.raises(NotImplementedError, match="KV heads"):
        X.parallel_model(exp1.save(), 2, 0)
    with pytest.raises(AssertionError):
        G.build_llama_decode(B.GraphHandler(rt), _gqa_onnx_cfg(1), 2, 0)
