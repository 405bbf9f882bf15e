"""CPU tier for RoPE with a model's own frequencies (an inv_freq table): the table against Hugging Face's formulas in torch
float32, RoPE's shape rule and the launchers' refusals, the AttentionRope fold, ONNX round trips and tensor-parallel
replication of the table, default graphs unchanged, the CPU oracle's refusal, and a float32 emulation of the kernels' rule
against the float64 bound the GPU tests apply (and the slips it must catch)."""
import ctypes
import dataclasses
import hashlib
import math
import re

import numpy as np
import pytest

from tests import rope64

F32, F16, BF16, I64 = 1, 10, 16, 7
LLAMA31 = {"type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
           "original_max_position_embeddings": 8192}
TABLES = {"base1e4": (10000.0, None), "base5e5": (500000.0, None), "base1e6": (1000000.0, None), "llama31": (500000.0, LLAMA31)}


@pytest.fixture(scope="module")
def B():
    from infinitensor_b200 import backend
    return backend


@pytest.fixture(scope="module")
def G():
    from infinitensor_b200 import graphs
    return graphs


# ---------------------------------------------------------------------------------------------------- the table
def hf_inv_freq(dim, base, scaling):
    """transformers' _compute_default_rope_parameters / _compute_llama3_parameters, in torch float32 on the CPU"""
    import torch
    inv_freq = 1.0 / (base ** (torch.arange(0, dim, 2, dtype=torch.int64).to(dtype=torch.float) / dim))
    if scaling is None:
        return inv_freq.numpy()
    factor, low, high = scaling["factor"], scaling["low_freq_factor"], scaling["high_freq_factor"]
    old = scaling["original_max_position_embeddings"]
    low_wavelen, high_wavelen = old / low, old / high
    wavelen = 2 * math.pi / inv_freq
    inv_freq_llama = torch.where(wavelen > low_wavelen, inv_freq / factor, inv_freq)
    smooth = (old / wavelen - low) / (high - low)
    smoothed = (1 - smooth) * inv_freq_llama / factor + smooth * inv_freq_llama
    is_medium = ~(wavelen < high_wavelen) * ~(wavelen > low_wavelen)
    return torch.where(is_medium, smoothed, inv_freq_llama).numpy()


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("table", sorted(TABLES))
def test_table_matches_hf_formulas(G, D, table):
    got = G.rope_inv_freq(D, *TABLES[table])
    ref = hf_inv_freq(D, *TABLES[table])
    assert got.dtype == np.float32 and got.shape == (D // 2,)
    ulps = np.abs(got.view(np.int32).astype(np.int64) - ref.view(np.int32).astype(np.int64))
    assert ulps.max() <= 1, f"{table} D={D}: {ulps.max()} float32 ulps from HF's table"


def test_llama31_bands_by_hand(G):
    """Llama-3.1 at D = 128: wavelengths below 8192 / 4 = 2048 keep their frequency, above 8192 are divided by 8, and the band
    between is interpolated -- one column of each, worked out in float64 from the formula"""
    t = G.rope_inv_freq(128, 500000.0, LLAMA31)
    base = 500000.0 ** (-np.arange(0, 128, 2) / 128.0)
    wave = 2 * np.pi / base
    hi_col = 10   # wavelength ~ 92: high frequency, unchanged
    lo_col = 50   # wavelength ~ 2.4e5: divided by 8
    mid = [c for c in range(64) if 2048 <= wave[c] <= 8192]
    assert wave[hi_col] < 2048 and wave[lo_col] > 8192 and mid
    c = mid[len(mid) // 2]
    s = (8192 / wave[c] - 1) / (4 - 1)
    expect = {hi_col: base[hi_col], lo_col: base[lo_col] / 8, c: (1 - s) * base[c] / 8 + s * base[c]}
    for col, v in expect.items():
        assert abs(float(t[col]) - v) <= 4 * np.spacing(np.float32(v)), (col, float(t[col]), v)
    assert 1 / 8 < t[c] / base[c] < 1


def test_table_refuses_unknown_scaling(G):
    with pytest.raises(ValueError, match="llama3"):
        G.rope_inv_freq(128, 1e6, {"type": "yarn", "factor": 4.0})


def test_llama31_preset(G):
    c = G.LlamaConfig.llama31_8b(batch=2, s_max=64, kv_fp8=True, int4_block=64)
    three = G.LlamaConfig.llama3_8b(batch=2, s_max=64, kv_fp8=True, int4_block=64)
    assert (c.heads, c.n_kv, c.ffn, c.vocab, c.rope_theta) == (32, 8, 14336, 128256, 500000.0)
    assert c.rope_scaling == LLAMA31 and not c.rope_default
    assert dataclasses.replace(c, rope_theta=10000.0, rope_scaling=None) == three and three.rope_default


# ---------------------------------------------------------------------------------------------------- shape rule, launchers
def _rope(B, freq_shape=(64,), freq_dt=F32, dim_head=128):
    h = B.GraphHandler(B.HostPlanRuntime())
    pos, x = h.tensor([2, 1], I64), h.tensor([2, 1, 256], BF16)
    return h.RoPE(pos, x, None, dim_head, inv_freq=h.tensor(list(freq_shape), freq_dt))


def test_shape_rule_accepts_a_table(B):
    assert _rope(B).shape() == [2, 1, 256]
    assert _rope(B, (32,), dim_head=64).shape() == [2, 1, 256]


@pytest.mark.parametrize("kw", [dict(freq_dt=F16), dict(freq_dt=BF16), dict(freq_shape=(1, 64)), dict(freq_shape=(63,)),
                                dict(freq_shape=(65,)), dict(freq_shape=(64,), dim_head=64)],
                         ids=["f16", "bf16", "rank2", "short", "long", "width"])
def test_shape_rule_refuses(B, kw):
    with pytest.raises(RuntimeError, match=re.escape("RoPE: inv_freq must be f32 [dim_head / 2]")):
        _rope(B, **kw)


def _fake(n=1):
    """host addresses that are never dereferenced: every refusal below happens before a launch"""
    return ctypes.c_void_p(0x1000 * n)


REFUSALS = {"f16": (dict(freq_dtype=F16), "inv_freq must be f32"), "short": (dict(freq_len=63), "inv_freq has 63 entries"),
            "missing": (dict(inv_freq=None), "inv_freq table missing"), "ragged": (dict(ragged=True), "multiple of dim_head"),
            "no_rope_pos": (dict(rope_pos=None), "needs RoPE positions")}


@pytest.mark.parametrize("fn,why", [(f, w) for f in ("rope", "gqa", "fp8") for w in REFUSALS
                                    if w != ("no_rope_pos" if f == "rope" else "ragged")])
def test_launchers_refuse_before_launching(B, fn, why):
    """a bad table (and RoPE's ragged path, attention without RoPE positions) is refused with the operator's name, and no
    kernel is launched"""
    from infinitensor_b200 import _lib as L
    bad, msg = REFUSALS[why]
    a = dict(freq_dtype=F32, freq_len=64, inv_freq=_fake(7), rope_pos=_fake(6), ragged=False)
    a.update(bad)
    before = L.lib.it_b200_launch_count()
    if fn == "rope":
        rc = L.lib.it_b200_rope_freq(BF16, _fake(1), I64, _fake(2), _fake(3), 1, 1, 200 if a["ragged"] else 256, 128,
                                     a["inv_freq"], a["freq_dtype"], a["freq_len"], None)
        what = "rope"
    else:
        p = [_fake(i) for i in range(1, 6)]
        common = (p[0], I64, a["rope_pos"], I64, a["inv_freq"], a["freq_dtype"], a["freq_len"], _fake(8), 1, 4, 1, 64, 128,
                  _fake(9), 1 << 20, None)
        if fn == "gqa":
            rc = L.lib.it_b200_attention_kvcache_gqa_freq(BF16, _fake(10), _fake(11), p[1], p[2], p[3], *common)
            what = "AttentionKVCache+RoPE"
        else:
            rc = L.lib.it_b200_attention_kvcache_fp8_freq(BF16, _fake(10), _fake(11), _fake(12), _fake(13), p[1], p[2], p[3],
                                                          *common)
            what = "AttentionKVCache(FP8 cache)+RoPE"
    assert rc != 0
    err = L.last_error()
    assert err.startswith(what) and msg in err, err
    assert L.lib.it_b200_launch_count() == before


# ---------------------------------------------------------------------------------------------------- schedule
def _attn_graph(B, q_table, k_table, fp8=False):
    """RoPE(q), RoPE(k) -> reshape / transpose -> AttentionKVCache, with the named tables ("a", "b" or None)"""
    h = B.GraphHandler(B.HostPlanRuntime())
    Bn, Hq, Hkv, D, S = 2, 8, 2, 128, 64
    act, cache = BF16, (17 if fp8 else BF16)
    tables = {n: h.tensor([D // 2], F32) for n in ("a", "b")}
    for t in tables.values():
        t.set_weight()
    pos = h.tensor([Bn, 1], I64)
    pos.set_input()
    q, k, v = h.tensor([Bn, 1, Hq * D], act), h.tensor([Bn, 1, Hkv * D], act), h.tensor([Bn, 1, Hkv * D], act)
    kw = lambda n: {} if n is None else {"inv_freq": tables[n]}
    q = h.RoPE(pos, q, None, **kw(q_table))
    k = h.RoPE(pos, k, None, **kw(k_table))
    heads = lambda t, n: h.transpose(h.reshape(t, None, [Bn, 1, n, D]), None, [0, 2, 1, 3])
    kc, vc = h.tensor([Bn, Hkv, S, D], cache), h.tensor([Bn, Hkv, S, D], cache)
    sc = {"k_scale": h.tensor([Hkv], F32), "v_scale": h.tensor([Hkv], F32)} if fp8 else {}
    h.attentionKVCache(kc, vc, heads(q, Hq), heads(k, Hkv), heads(v, Hkv), pos, None, **sc).set_output()
    h.data_malloc()
    return h.schedule()


@pytest.mark.parametrize("fp8", [False, True], ids=["16bit", "fp8"])
@pytest.mark.parametrize("tables,fold", [(("a", "a"), True), ((None, None), True), (("a", "b"), False), (("a", None), False),
                                         ((None, "b"), False)], ids=["shared", "none", "differ", "q_only", "k_only"])
def test_fold_needs_one_table(B, tables, fold, fp8):
    sc = _attn_graph(B, *tables, fp8=fp8)
    folded = sum(s.startswith("AttentionRope") for s in sc)
    ropes = sum(s.startswith("Single") and "RoPE" in s for s in sc)
    assert (folded, ropes) == ((1, 0) if fold else (0, 2)), sc


def _small31(G, **kw):
    base = dict(layers=2, d_model=512, heads=4, kv_heads=2, head_dim=128, ffn=1024, vocab=128, s_max=32, batch=4,
                rope_theta=500000.0, rope_scaling=dict(LLAMA31))
    base.update(kw)
    return G.LlamaConfig(**base)


@pytest.mark.parametrize("kw", [{}, dict(kv_fp8=True), dict(head_dim=64, d_model=256), dict(int4_block=64)],
                         ids=["16bit", "kv_fp8", "d64", "int4"])
def test_llama_graph_with_table(B, G, kw):
    cfg = _small31(G, **kw)
    h = B.GraphHandler(B.HostPlanRuntime())
    g = G.build_llama_decode(h, cfg)
    t, shape, kind, shard = g.weights["rope.inv_freq"]
    assert (t.dtype(), t.shape(), shape, kind, shard) == (F32, [cfg.head_dim // 2], (cfg.head_dim // 2,), "inv_freq", None)
    h.data_malloc()
    sc = h.schedule()
    assert sum(s.startswith("AttentionRope") for s in sc) == cfg.layers, sc


def test_default_graphs_take_no_table(B, G):
    cfg = _small31(G, rope_theta=10000.0, rope_scaling=None)
    g = G.build_llama_decode(B.GraphHandler(B.HostPlanRuntime()), cfg)
    assert "rope.inv_freq" not in g.weights


# ---------------------------------------------------------------------------------------------------- ONNX
def _node_list(m):
    return [(n.op_type, len(n.inputs), len(n.outputs), sorted(n.attrs)) for n in m.graph.nodes]


@pytest.mark.parametrize("kw", [{}, dict(kv_fp8=True), dict(head_dim=64, d_model=256)], ids=["16bit", "kv_fp8", "d64"])
def test_onnx_round_trip_with_table(B, G, kw):
    from infinitensor_b200 import onnx_lite as X
    rt = B.HostPlanRuntime()
    cfg = _small31(G, **kw)
    direct = B.GraphHandler(rt)
    G.build_llama_decode(direct, cfg)
    exp = X.OnnxExporter(B.GraphHandler(rt))
    G.build_llama_decode(exp, cfg)
    blob = exp.save()
    m = X.load_model(blob)
    ropes = [n for n in m.graph.nodes if n.op_type == "RoPE"]
    assert len(ropes) == 2 * cfg.layers and len({n.inputs[2] for n in ropes if len(n.inputs) == 3}) == 1
    assert all(len(n.inputs) == 3 for n in ropes)
    h = B.GraphHandler(rt)
    X.OnnxStub(blob, handler=h, upload=False)
    assert h.schedule() == direct.schedule()
    exp2 = X.OnnxExporter(B.GraphHandler(rt))
    X.OnnxStub(blob, handler=exp2, upload=False)
    assert _node_list(X.load_model(exp2.save())) == _node_list(m)


def test_onnx_table_refused_by_a_handler_without_one(B, G):
    from infinitensor_b200 import onnx_lite as X
    from oracle.graph_oracle import OracleHandler
    exp = X.OnnxExporter(B.GraphHandler(B.HostPlanRuntime()))
    G.build_llama_decode(exp, _small31(G))
    with pytest.raises(NotImplementedError, match="inv_freq"):
        X.OnnxStub(exp.save(), handler=OracleHandler(), upload=False)


def test_default_exports_and_schedules_unchanged(B, G):
    """a config that spells out the defaults (rope_theta 10000, no scaling) writes the bytes pinned before tables existed"""
    from infinitensor_b200 import onnx_lite as X
    from tests.test_kvfp8_host import EXPORT_SHA256
    cfgs = {"llama": _small31(G, kv_heads=None, rope_theta=10000.0, rope_scaling=None),
            "gqa": _small31(G, rope_theta=10000.0, rope_scaling=None),
            "d64": dataclasses.replace(G.LlamaConfig.tinyllama_1b(batch=2, s_max=16, layers=2), rope_theta=10000.0)}
    for which, cfg in cfgs.items():
        exp = X.OnnxExporter(B.GraphHandler(B.HostPlanRuntime()))
        G.build_llama_decode(exp, cfg)
        assert hashlib.sha256(exp.save()).hexdigest() == EXPORT_SHA256[which], which
        h = B.GraphHandler(B.HostPlanRuntime())
        G.build_llama_decode(h, cfg)
        h.data_malloc()
        assert not any("inv_freq" in s for s in h.schedule())


def test_parallel_model_replicates_the_table(B, G):
    from infinitensor_b200 import onnx_lite as X
    rt = B.HostPlanRuntime()
    cfg = _small31(G, kv_heads=4)
    exp = X.OnnxExporter(B.GraphHandler(rt))
    G.build_llama_decode(exp, cfg)
    for rank in (0, 1):
        direct = B.GraphHandler(rt)
        G.build_llama_decode(direct, cfg, 2, rank)
        sharded = X.parallel_model(exp.save(), 2, rank)
        m = X.load_model(sharded) if isinstance(sharded, (bytes, bytearray)) else sharded
        dims = {v.name: list(v.dims) for v in m.graph.inputs}
        dims.update({t.name: list(np.shape(t.array)) if t.array is not None else list(t.dims) for t in m.graph.initializers})
        ropes = [n for n in m.graph.nodes if n.op_type == "RoPE"]
        assert len(ropes) == 4 and all(dims[n.inputs[2]] == [64] for n in ropes), "every rank holds the whole table"
        h = B.GraphHandler(rt)
        X.OnnxStub(sharded, handler=h, upload=False)
        assert h.schedule() == direct.schedule()


# ---------------------------------------------------------------------------------------------------- the CPU oracle
def test_oracle_handler_refuses_a_table(G):
    from oracle.graph_oracle import OracleHandler
    for cfg in (_small31(G), _small31(G, rope_scaling=None), _small31(G, rope_theta=1e6, rope_scaling=None)):
        with pytest.raises(NotImplementedError, match="rope_theta"):
            G.build_llama_decode(OracleHandler(), cfg)
    G.build_llama_decode(OracleHandler(), _small31(G, rope_theta=10000.0, rope_scaling=None))


def test_test_oracle_matches_the_emulation(G):
    """tests/rope_oracle.py's RoPE with a table is the rule the bound checks"""
    from tests import rope_oracle as RO
    pos, x = rope64.case(128, BF16)
    t = G.rope_inv_freq(128, 500000.0, LLAMA31)
    got = RO.rope_freq(pos.reshape(-1, 1), x.reshape(-1, 1, x.shape[-1]), t, 128, BF16).reshape(x.shape)
    assert np.array_equal(got, rope64.Bound(pos, x, t, 128, BF16).nominal)


def test_rope_oracle_runs_a_table_graph(G):
    """the graph oracle with a table takes a non-default config; one decode step gives finite logits that differ from the
    same graph's at base 10000"""
    from tests import rope_oracle as RO
    cfg = _small31(G, layers=1, batch=2, s_max=64)
    logits = []
    for c in (cfg, dataclasses.replace(cfg, rope_theta=10000.0, rope_scaling=None)):
        oh, og = RO.oracle_graph(c)
        og.input_ids.copyin_numpy(np.array([[3], [5]], np.int64))
        og.position_ids.copyin_numpy(np.array([[40], [63]], np.int64))
        oh.run()
        logits.append(og.logits.f32())
    assert np.isfinite(logits[0]).all() and not np.array_equal(logits[0], logits[1])


# ---------------------------------------------------------------------------------------------------- emulation vs bound
@pytest.mark.parametrize("dt", [F32, F16, BF16], ids=["fp32", "f16", "bf16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("table", sorted(TABLES))
def test_emulation_within_bound(G, table, D, dt):
    pos, x = rope64.case(D, dt)
    t = G.rope_inv_freq(D, *TABLES[table])
    b = rope64.Bound(pos, x, t, D, dt)
    assert not b.outside(rope64.emulate(pos, x, t, D, dt)).any()
    assert b.share <= (1.0 if dt == F32 else 0.05), f"{b.share:.2%} of the elements have two candidates"


@pytest.mark.parametrize("slip", ["base10000", "column+1", "angle64", "no_llama3_scaling"])
def test_bound_catches_slips(G, slip):
    fails = []
    for dt in (F32, F16, BF16):
        for D in (64, 128):
            pos, x = rope64.case(D, dt)
            t = G.rope_inv_freq(D, 500000.0, LLAMA31)
            if slip == "no_llama3_scaling":
                got = rope64.emulate(pos, x, G.rope_inv_freq(D, 500000.0), D, dt)
            else:
                got = rope64.emulate(pos, x, t, D, dt, slip=slip)
            fails.append(int(rope64.Bound(pos, x, t, D, dt).outside(got).sum()))
    assert all(f > 0 for f in fails[:2]) and sum(f > 0 for f in fails) >= 4, f"{slip}: elements outside per case {fails}"
