"""CPU tier for 64-wide decode heads: RoPE's dim_head attribute through every interface, the schedule of TinyLlama-shape
graphs, and GPT-2 decode on the oracle against the oracle's GPT-2 forward."""
import collections
import hashlib

import numpy as np
import pytest

F32, F16, BF16, I64 = 1, 10, 16, 7


@pytest.fixture(scope="module")
def B():
    from infinitensor_b200 import backend
    return backend


def _tinyllama(layers=2, **kw):
    from infinitensor_b200 import graphs as G
    base = dict(batch=16, s_max=64, layers=layers)
    base.update(kw)
    cfg = G.LlamaConfig.tinyllama_1b(**base)
    cfg.vocab = 256  # the logits head is not what these tests are about
    return cfg


def test_tinyllama_config():
    from infinitensor_b200 import graphs as G
    c = G.LlamaConfig.tinyllama_1b()
    assert (c.layers, c.d_model, c.heads, c.n_kv, c.head_dim, c.ffn, c.vocab) == (22, 2048, 32, 4, 64, 5632, 32000)


def _rope_graph(B, dim_head, width=256, heads_w=64):
    """RoPE(dim_head) on q -> heads of `heads_w` -> AttentionKVCache, and the same for k; returns the handler"""
    h = B.GraphHandler(B.HostPlanRuntime())
    n = width // heads_w
    pos = h.tensor([2, 1], I64)
    kc, vc = h.tensor([2, n, 16, heads_w], BF16), h.tensor([2, n, 16, heads_w], BF16)
    q, k, v = (h.tensor([2, 1, width], BF16) for _ in range(3))
    kw = {} if dim_head is None else {"dim_head": dim_head}
    qr, kr = h.RoPE(pos, q, None, **kw), h.RoPE(pos, k, None, **kw)

    def heads(t):
        return h.transpose(h.reshape(t, None, [2, 1, n, heads_w]), None, [0, 2, 1, 3])
    h.attentionKVCache(kc, vc, heads(qr), heads(kr), heads(v), pos, None)
    return h


@pytest.mark.parametrize("dim_head,heads_w,folds", [(64, 64, True), (None, 128, True), (128, 128, True), (128, 64, False),
                                                    (64, 128, False), (32, 64, False)])
def test_rope_width_decides_the_fold(B, dim_head, heads_w, folds):
    """the C-ABI carries dim_head to the operator: RoPE folds into the attention kernel exactly when its width is the
    caches' head width (64 or 128); otherwise both RoPEs run on their own before the attention"""
    sc = _rope_graph(B, dim_head, heads_w=heads_w).schedule()
    assert (sc.count("AttentionRope:RoPE+RoPE+AttentionKVCache") == 1) == folds
    assert sum(s == "Single:RoPE" for s in sc) == (0 if folds else 2)


@pytest.mark.parametrize("dim_head", [0, 3, -2])
def test_rope_rejects_bad_width(B, dim_head):
    h = B.GraphHandler(B.HostPlanRuntime())
    with pytest.raises(RuntimeError, match="dim_head"):
        h.RoPE(h.tensor([1, 1], I64), h.tensor([1, 1, 128], F32), None, dim_head=dim_head)


def test_rope_dim_head_onnx_roundtrip(B):
    """OnnxExporter writes dim_head only when it is not 128; OnnxStub reads it back; parallel_model keeps it"""
    from infinitensor_b200 import graphs as G, onnx_lite as X
    rt = B.HostPlanRuntime()
    cfg = _tinyllama()
    direct = B.GraphHandler(rt)
    G.build_llama_decode(direct, cfg)
    exp = X.OnnxExporter(B.GraphHandler(rt))
    G.build_llama_decode(exp, cfg)
    blob = exp.save()
    ropes = [n for n in X.load_model(blob).graph.nodes if n.op_type == "RoPE"]
    assert len(ropes) == 2 * cfg.layers and all(n.attrs == {"dim_head": 64} for n in ropes)
    stub_h = B.GraphHandler(rt)
    X.OnnxStub(blob, handler=stub_h, upload=False)
    assert stub_h.schedule() == direct.schedule()
    # stub -> exporter again: the same bytes
    again = X.OnnxExporter(B.GraphHandler(rt))
    X.OnnxStub(blob, handler=again, upload=False)
    assert [n.attrs for n in again.model().graph.nodes if n.op_type == "RoPE"] == [{"dim_head": 64}] * (2 * cfg.layers)
    sharded = X.parallel_model(blob, 2, 1)
    ropes = [n for n in sharded.graph.nodes if n.op_type == "RoPE"]
    assert len(ropes) == 2 * cfg.layers and all(n.attrs == {"dim_head": 64} for n in ropes)
    tp = B.GraphHandler(rt)
    X.OnnxStub(sharded, handler=tp, upload=False)
    ref = B.GraphHandler(rt)
    G.build_llama_decode(ref, cfg, 2, 1)
    assert tp.schedule() == ref.schedule()


def test_llama_export_bytes_unchanged(B):
    """ONNX files of 128-wide Llama graphs carry no dim_head attribute: byte for byte what the exporter wrote before the
    attribute existed (SHA-256 of the equal-heads tiny config and of a grouped-query config)"""
    from infinitensor_b200 import graphs as G, onnx_lite as X
    rt = B.HostPlanRuntime()
    want = ["634afe4b33636fcfc1a7ce0c2a4a96ae5a516cdacf294dc3bec882f14ccff0c1",
            "85582cf211a038e53ea35841376babfae71c3c093001cc1c1b9dcb96a3352abd"]
    cfgs = [G.LlamaConfig.tiny(), G.LlamaConfig(layers=2, d_model=512, heads=4, kv_heads=2, head_dim=128, ffn=1024, vocab=128,
                                                s_max=32, batch=16)]
    for cfg, w in zip(cfgs, want):
        exp = X.OnnxExporter(B.GraphHandler(rt))
        G.build_llama_decode(exp, cfg)
        assert hashlib.sha256(exp.save()).hexdigest() == w


def test_tinyllama_schedule(B):
    """TinyLlama-shape layers: both RoPEs fold into one AttentionRope step per layer, and a second build gets the same steps"""
    from infinitensor_b200 import graphs as G
    rt = B.HostPlanRuntime()
    cfg = _tinyllama()
    h = B.GraphHandler(rt)
    g = G.build_llama_decode(h, cfg)
    assert g.k_caches[0].shape() == [16, 4, 64, 64]
    sc = h.schedule()
    assert sc.count("AttentionRope:RoPE+RoPE+AttentionKVCache") == cfg.layers
    assert not any(s.startswith("Single:RoPE") for s in sc)
    kinds = collections.Counter(s.split(":")[0] for s in sc)
    assert kinds["AttentionRope"] == cfg.layers and kinds["MatMulGroup"] == 2 * cfg.layers
    h.data_malloc()
    h2 = B.GraphHandler(rt)
    G.build_llama_decode(h2, cfg)
    assert h2.schedule() == sc


def test_gpt2_decode_graph_shapes(B):
    from infinitensor_b200 import graphs as G
    cfg = G.GPT2Config(batch=16, lm_head=True)
    h = B.GraphHandler(B.HostPlanRuntime())
    g = G.build_gpt2_decode(h, cfg, 1024)
    assert len(g.k_caches) == 12 and g.k_caches[0].shape() == [16, 12, 1024, 64]
    assert g.out.shape() == [16, 1, cfg.vocab]
    fwd = G.build_gpt2(B.GraphHandler(B.HostPlanRuntime()), cfg)
    assert {k: v[1] for k, v in g.weights.items()} == {k: v[1] for k, v in fwd.weights.items()}
    sc = h.schedule()
    assert sum(s.startswith("Single:AttentionKVCache") for s in sc) == 12
    e = 2
    assert cfg.algorithmic_bytes(511) > 12 * 2 * 16 * 768 * 511 * e  # at least the KV cache read


def _gpt2_small_cfg(dtype=F16, T=20, batch=2):
    from infinitensor_b200 import graphs as G
    return G.GPT2Config(layers=2, d_model=128, heads=2, ffn=256, vocab=300, n_pos=64, seq=T, batch=batch, dtype=dtype,
                        lm_head=True)


@pytest.mark.parametrize("dtype", [F32, F16])
def test_gpt2_decode_on_oracle_matches_forward(dtype):
    """token by token from an empty cache, the decode step reproduces the rows of build_gpt2's forward over the same
    tokens (the oracle executing both graphs)"""
    from infinitensor_b200 import graphs as G
    from tests.llama_oracle import LlamaOracleHandler
    T = 20
    cfg = _gpt2_small_cfg(dtype, T)
    rng = np.random.default_rng(3)
    ids = rng.integers(0, cfg.vocab, size=(cfg.batch, T)).astype(np.int64)
    fh = LlamaOracleHandler()
    fg = G.build_gpt2(fh, cfg)
    G.fill_gpt2_weights_host(fg)
    fg.input_ids.copyin_numpy(ids)
    fg.position_ids.copyin_numpy(np.broadcast_to(np.arange(T, dtype=np.int64), (cfg.batch, T)).copy())
    fh.run()
    ref = fg.out.f32().astype(np.float64)  # [B, T, vocab]
    dh = LlamaOracleHandler()
    dg = G.build_gpt2_decode(dh, cfg, 32)
    G.fill_gpt2_weights_host(dg)
    for c in dg.k_caches + dg.v_caches:
        c.copyin_numpy(G.to_storage(np.zeros(c.shape(), np.float32), dtype))
    tol = {F32: 1e-4, F16: 2e-2}[dtype]
    for t in range(T):
        dg.input_ids.copyin_numpy(ids[:, t:t + 1])
        dg.position_ids.copyin_numpy(np.full((cfg.batch, 1), t, np.int64))
        dh.run()
        got = dg.out.f32().astype(np.float64)[:, 0]
        err = np.abs(got - ref[:, t]).max() / np.abs(ref[:, t]).max()
        assert err < tol, f"token {t}: rel-to-max error {err:.3e}"


def test_handlers_without_narrow_heads_refuse_them(B):
    """the oracle's graph handler restates the 128-only reference: a 64-wide decode graph, or an ONNX file with a RoPE
    dim_head, is refused on it instead of being run with the 128-wide scale and RoPE"""
    from infinitensor_b200 import graphs as G, onnx_lite as X
    from oracle.graph_oracle import OracleHandler
    with pytest.raises(NotImplementedError, match="64-wide"):
        G.build_llama_decode(OracleHandler(), _tinyllama())
    with pytest.raises(NotImplementedError, match="64-wide"):
        G.build_gpt2_decode(OracleHandler(), _gpt2_small_cfg(), 32)
    exp = X.OnnxExporter(B.GraphHandler(B.HostPlanRuntime()))
    G.build_llama_decode(exp, _tinyllama())
    with pytest.raises(NotImplementedError, match="dim_head 64"):
        X.OnnxStub(exp.save(), handler=OracleHandler(), upload=False)
    # 128-wide graphs still build on it, through the exporter too
    G.build_llama_decode(X.OnnxExporter(OracleHandler()), G.LlamaConfig.tiny())
