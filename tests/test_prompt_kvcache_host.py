"""CPU tier for AttentionKVCache over a prompt chunk (S > 1 new tokens): the operator's shape rule, the launcher's argument
checks, the test oracle's S-step loop against a float64 causal formula, the Llama prompt-step graph (schedule, ONNX round
trip, seq = 1 unchanged) and a prompt step followed by a decode step against single-token steps on the oracle."""
import collections
import hashlib

import numpy as np
import pytest

from tests import prompt64

F32, F16, BF16, I64 = 1, 10, 16, 7


@pytest.fixture(scope="module")
def B():
    from infinitensor_b200 import backend
    return backend


def _att(B, cache, q, npos, dt=BF16, per_row=False):
    h = B.GraphHandler(B.HostPlanRuntime())
    kc, vc = h.tensor(cache, dt), h.tensor(cache, dt)
    kv = [cache[0], cache[1], q[2], cache[3]]
    qt, kt, vt = h.tensor(q, dt), h.tensor(kv, dt), h.tensor(kv, dt)
    pos = h.tensor(npos, I64)
    return h.attentionKVCache(kc, vc, qt, kt, vt, pos, None, per_row)


@pytest.mark.parametrize("q,npos", [([2, 8, 16, 128], [2, 16]), ([2, 8, 16, 128], [2, 1]), ([2, 2, 64, 64], [2, 64]),
                                    ([1, 48, 5, 128], [1, 5]), ([1, 4, 64, 64], [1])])
def test_shape_rule_accepts_prompt_chunks(B, q, npos):
    out = _att(B, [q[0], 1 if q[1] == 48 else q[1] // 4 or 1, 64, q[3]], q, npos)
    assert out.shape() == q


@pytest.mark.parametrize("cache,q,npos,dt,what", [
    ([2, 2, 16, 128], [2, 8, 17, 128], [2, 17], BF16, "do not fit"),  # S > S_max
    ([2, 2, 16, 128], [2, 8, 4, 128], [2, 4], F32, "fp32"),          # fp32 prompt chunk
    ([2, 2, 16, 128], [2, 8, 4, 128], [2, 3], BF16, "position"),     # neither one position per row nor one per token
    ([2, 2, 16, 128], [2, 8, 4, 128], [1], BF16, "position"),        # one position for two rows
])
def test_shape_rule_rejects_bad_prompt_chunks(B, cache, q, npos, dt, what):
    with pytest.raises(RuntimeError, match=what):
        _att(B, cache, q, npos, dt)


def test_shape_rule_single_token_unchanged(B):
    """S = 1 keeps the decode rule: fp32, one position for every row, a one-row cache"""
    assert _att(B, [2, 2, 1, 128], [2, 8, 1, 128], [1], F32).shape() == [2, 8, 1, 128]


def test_launcher_refuses_before_any_launch():
    """fp32, S > S_max and a bad head width are refused by the C-ABI with a message naming the operator"""
    from infinitensor_b200 import _lib as L
    f = L.lib.it_b200_attention_kvcache_prompt
    for args, what in [((F32, 64, 128), "fp32"), ((BF16, 65, 128), "do not fit"), ((BF16, 8, 96), "head dim")]:
        dt, S, D = args
        assert f(dt, None, None, None, None, None, None, I64, None, 1, 1, 1, S, 64, D, None) != 0
        msg = L.last_error()
        assert "AttentionKVCache prompt" in msg and what in msg, msg


# ---------------------------------------------------------------- the test oracle's loop
@pytest.mark.parametrize("D,G,p,S,per_row", [(64, 4, [0, 5], 9, True), (128, 1, [3], 7, False), (128, 2, [0, 60], 4, True),
                                             (64, 1, [30], 34, False)])
def test_oracle_loop_matches_float64_causal_attention(D, G, p, S, per_row):
    from tests.llama_oracle import attention_kvcache_prompt
    Bn = len(p)
    # (scores up to 20: the oracle's 128-wide step exponentiates scores without subtracting their maximum, as the reference)
    c = prompt64.Case(Bn, 2 * G, 2, S, 64, p if per_row else p[0], D, seed=5, regimes=["flat", "late", "sink", "diag"])
    kc, vc, k, v = c.inputs()
    pos = (c.p[:, None] + np.arange(S)[None, :]) if per_row else np.array([p[0]])
    got = attention_kvcache_prompt(kc, vc, c.q, k, v, pos, BF16, per_row)
    refs = c.reference()
    # the oracle's own step (fp32, one rounding to bf16): within an ulp plus 2^-12 sum w|v|
    err = np.abs(got - refs[0])
    assert np.all(err <= oracle_ulp(refs[0]) + 2.0 ** -12 * refs[1]), float((err / (oracle_ulp(refs[0]) + 2.0 ** -12 * refs[1])).max())
    for b in range(Bn):
        q0 = int(c.p[b])
        np.testing.assert_array_equal(kc[b, :, q0:q0 + S], k[b])
        np.testing.assert_array_equal(vc[b, :, q0:q0 + S], v[b])
        assert np.array_equal(kc[b, :, :q0], c.kseq[b, :, :q0]) and np.isnan(kc[b, :, q0 + S:]).all()


def oracle_ulp(x):
    from tests import ref64
    return ref64.ulp(x, BF16)


def test_prompt_starts_rules():
    from tests.llama_oracle import prompt_starts
    pos = np.array([[5, 6, 7], [40, 41, 42]])
    assert list(prompt_starts(pos, 2, 3, 64, True)) == [5, 40]
    assert list(prompt_starts(pos, 2, 3, 64, False)) == [5, 5]
    assert list(prompt_starts(np.array([[3], [70]]), 2, 3, 64, True)) == [3, 61]  # clamped to S_max - S
    assert list(prompt_starts(np.array([-4]), 2, 3, 64, False)) == [0, 0]


def test_single_token_oracle_unchanged():
    """at S = 1 the oracle handler's AttentionKVCache is the single-token rule (64-wide grouped-query heads here): output and
    cache writes bit for bit attention_kvcache_d's on the same arrays"""
    import oracle
    from tests.llama_oracle import LlamaOracleHandler, attention_kvcache_d
    Bn, Hq, Hkv, Smax, D = 2, 8, 2, 16, 64
    rng = np.random.default_rng(4)
    vals = [oracle.round_to(rng.standard_normal(shape).astype(np.float32), BF16)
            for shape in ((Bn, Hkv, Smax, D), (Bn, Hkv, Smax, D), (Bn, Hq, 1, D), (Bn, Hkv, 1, D), (Bn, Hkv, 1, D))]
    h = LlamaOracleHandler()
    ts = [h.tensor(list(a.shape), BF16) for a in vals]
    for t, a in zip(ts, vals):
        t.set_f32(a)
    pos = h.tensor([Bn, 1], I64)
    pos.copyin_numpy(np.array([[4], [4]], np.int64))
    out = h.attentionKVCache(*ts, pos, None)
    kc, vc = vals[0].copy(), vals[1].copy()
    ref = attention_kvcache_d(kc, vc, *vals[2:], 4, BF16)
    h.run()
    assert np.array_equal(out.f32(), ref) and np.array_equal(ts[0].f32(), kc) and np.array_equal(ts[1].f32(), vc)


# ---------------------------------------------------------------- the Llama prompt-step graph
def _cfg(**kw):
    from infinitensor_b200 import graphs as G
    base = dict(layers=2, d_model=512, heads=4, kv_heads=2, head_dim=128, ffn=1024, vocab=128, s_max=32, batch=16)
    base.update(kw)
    return G.LlamaConfig(**base)


def test_seq1_graph_schedule_and_export_unchanged(B):
    from infinitensor_b200 import graphs as G, onnx_lite as X
    rt = B.HostPlanRuntime()
    for cfg in (G.LlamaConfig.tiny(), _cfg(), G.LlamaConfig.tinyllama_1b(layers=2, s_max=64)):
        a, b = B.GraphHandler(rt), B.GraphHandler(rt)
        G.build_llama_decode(a, cfg)
        G.build_llama_decode(b, cfg, seq=1)
        assert a.schedule() == b.schedule()
        blobs = []
        for kw in ({}, {"seq": 1}):
            exp = X.OnnxExporter(B.GraphHandler(rt))
            G.build_llama_decode(exp, cfg, **kw)
            blobs.append(exp.save())
        assert blobs[0] == blobs[1]
    # the 128-wide tiny config's export, byte for byte what test_head64_host pins
    exp = X.OnnxExporter(B.GraphHandler(rt))
    G.build_llama_decode(exp, G.LlamaConfig.tiny(), seq=1)
    assert hashlib.sha256(exp.save()).hexdigest() == "634afe4b33636fcfc1a7ce0c2a4a96ae5a516cdacf294dc3bec882f14ccff0c1"


@pytest.mark.parametrize("kv", [None, 2])
def test_prompt_graph_plans_without_decode_fusions(B, kv):
    """seq = 8 over 16 rows: 128 GEMM rows, so no MatMulGroup; the RoPE fold needs S = 1, so no AttentionRope"""
    from infinitensor_b200 import graphs as G
    h = B.GraphHandler(B.HostPlanRuntime())
    g = G.build_llama_decode(h, _cfg(kv_heads=kv), seq=8)
    assert g.input_ids.shape() == [16, 8] and g.position_ids.shape() == [16, 8] and g.logits.shape() == [16, 8, 128]
    sc = h.schedule()
    kinds = collections.Counter(s.split(":")[0] for s in sc)
    assert kinds["AttentionRope"] == 0 and kinds["MatMulGroup"] == 0
    assert sc.count("Single:AttentionKVCache") == 2 and sum(s == "Single:RoPE" for s in sc) == 4
    h.data_malloc()


def test_prompt_graph_builder_refusals(B):
    from infinitensor_b200 import graphs as G
    h = B.GraphHandler(B.HostPlanRuntime())
    with pytest.raises(AssertionError):
        G.build_llama_decode(h, _cfg(), world=2, seq=4)
    with pytest.raises(AssertionError):
        G.build_llama_decode(B.GraphHandler(B.HostPlanRuntime()), _cfg(fp8_weights=True), seq=4)


def test_prompt_graph_onnx_roundtrip(B):
    from infinitensor_b200 import graphs as G, onnx_lite as X
    rt = B.HostPlanRuntime()
    cfg = _cfg()
    direct = B.GraphHandler(rt)
    G.build_llama_decode(direct, cfg, seq=8)
    exp = X.OnnxExporter(B.GraphHandler(rt))
    G.build_llama_decode(exp, cfg, seq=8)
    blob = exp.save()
    stub = B.GraphHandler(rt)
    X.OnnxStub(blob, handler=stub, upload=False)
    assert stub.schedule() == direct.schedule()
    again = X.OnnxExporter(B.GraphHandler(rt))
    X.OnnxStub(blob, handler=again, upload=False)
    nodes = [(n.op_type, n.attrs) for n in X.load_model(blob).graph.nodes]
    assert [(n.op_type, n.attrs) for n in again.model().graph.nodes] == nodes
    assert sum(op == "AttentionKVCache" for op, _ in nodes) == cfg.layers


def _fill(g, cfg, seed=0):
    from infinitensor_b200 import graphs as G
    G.fill_llama_weights_host(g, seed=seed)


@pytest.mark.parametrize("head_dim,kv", [(128, None), (64, 2)])
def test_prompt_then_decode_equals_single_token_steps(head_dim, kv):
    """On the oracle, a prompt step of S tokens and one decode step give bit for bit the logits and caches of S + 1
    single-token steps: the oracle's GEMMs, norms and RoPE compute every row on its own, and its AttentionKVCache over S
    tokens is S single-token steps by definition, so nothing depends on how the tokens are batched."""
    from infinitensor_b200 import graphs as G
    from tests.llama_oracle import LlamaOracleHandler
    cfg = _cfg(head_dim=head_dim, kv_heads=kv, heads=4 if head_dim == 128 else 8, batch=2, dtype=BF16)
    S, p0 = 5, 3
    rng = np.random.default_rng(7)
    ids = rng.integers(0, cfg.vocab, size=(cfg.batch, S + 1)).astype(np.int64)
    cache0 = [G.to_storage(rng.standard_normal((cfg.batch, cfg.n_kv, cfg.s_max, head_dim)).astype(np.float32) * 0.5, BF16)
              for _ in range(2 * cfg.layers)]

    def graph(seq):
        h = LlamaOracleHandler()
        g = G.build_llama_decode(h, cfg, seq=seq)
        _fill(g, cfg)
        return h, g

    def load(g, caches):
        for t, c in zip(g.k_caches + g.v_caches, caches):
            t.copyin_numpy(c)

    def caches(g):
        return [G.to_storage(t.f32(), BF16) for t in g.k_caches + g.v_caches]

    # prompt step + decode step
    hp, gp = graph(S)
    load(gp, cache0)
    gp.input_ids.copyin_numpy(ids[:, :S])
    gp.position_ids.copyin_numpy(np.broadcast_to(p0 + np.arange(S), (cfg.batch, S)).copy())
    hp.run()
    prompt_logits = gp.logits.f32().copy()
    hd, gd = graph(1)
    load(gd, caches(gp))
    gd.input_ids.copyin_numpy(ids[:, S:])
    gd.position_ids.copyin_numpy(np.full((cfg.batch, 1), p0 + S, np.int64))
    hd.run()
    last = gd.logits.f32().copy()
    after = caches(gd)
    # S + 1 single-token steps
    hs, gs = graph(1)
    load(gs, cache0)
    step_logits = []
    for i in range(S + 1):
        gs.input_ids.copyin_numpy(ids[:, i:i + 1])
        gs.position_ids.copyin_numpy(np.full((cfg.batch, 1), p0 + i, np.int64))
        hs.run()
        step_logits.append(gs.logits.f32().copy())
    assert np.array_equal(prompt_logits, np.concatenate(step_logits[:S], axis=1))
    assert np.array_equal(last, step_logits[S])
    assert all(np.array_equal(a, b) for a, b in zip(after, caches(gs)))


# ---------------------------------------------------------------- the float64 bound and the kernel's emulation
EMU_CASES = [(2, 8, 2, 70, 200, [0, 77], 128, BF16), (1, 8, 1, 65, 130, 64, 64, F16), (1, 2, 1, 129, 300, 1, 128, F16),
             (2, 4, 4, 64, 128, [64, 0], 64, BF16), (1, 6, 3, 130, 130, 0, 128, BF16)]


@pytest.mark.parametrize("case", EMU_CASES)
def test_emulation_within_half_the_bound(case):
    Bn, Hq, Hkv, S, Smax, p, D, dt = case
    c = prompt64.Case(Bn, Hq, Hkv, S, Smax, p, D, seed=11)
    refs = c.reference()
    got = prompt64.emulate(c, dt)
    assert set(c.regime.ravel()) <= set(prompt64.REGIMES)
    msg = prompt64.report(prompt64.violations(got, refs, dt, 0.5), got, refs, dt, c, "emulation at half the bound")
    assert msg is None, msg


def test_every_regime_is_exercised():
    seen = set()
    for Bn, Hq, Hkv, S, Smax, p, D, dt in EMU_CASES:
        seen |= set(prompt64.Case(Bn, Hq, Hkv, 2, Smax, p, D, seed=11).regime.ravel())
    assert seen == set(prompt64.REGIMES)


@pytest.mark.parametrize("mutation", prompt64.MUTATIONS)
def test_injected_bugs_leave_the_bound(mutation):
    """P rounded once to bf16, the causal limit one row late, the append one row late, KV head h mod Hkv instead of h / G,
    and the diagonal key tiles skipped each put outputs outside the bound"""
    c = prompt64.Case(2, 8, 2, 70, 200, [0, 77], 128, seed=11)
    refs = c.reference()
    got = prompt64.emulate(c, BF16, mutation)
    assert prompt64.violations(got, refs, BF16).any()
