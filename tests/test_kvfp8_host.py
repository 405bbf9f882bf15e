"""CPU tier for the FP8 E4M3 KV cache: AttentionKVCache's shape rule with k_scale / v_scale, the test oracle's quantiser on
known answers, a float32 emulation of the kernel's arithmetic against the float64 bound (and slips it must catch), the
schedule of an FP8 Llama graph, ONNX round trips and tensor-parallel sharding of the scales."""
import re

import numpy as np
import pytest

from tests import kvfp8_oracle as KV

F32, F16, BF16, I64, FP8 = 1, 10, 16, 7, 17


@pytest.fixture(scope="module")
def B():
    from infinitensor_b200 import backend
    return backend


def _att(B, cache_dt=FP8, v_cache_dt=None, act=BF16, S=1, scales=True, kshape=None, vshape=None, sdt=F32, Hkv=4, Hq=8):
    h = B.GraphHandler(B.HostPlanRuntime())
    kc = h.tensor([2, Hkv, 64, 128], cache_dt)
    vc = h.tensor([2, Hkv, 64, 128], v_cache_dt or cache_dt)
    q, k, v = h.tensor([2, Hq, S, 128], act), h.tensor([2, Hkv, S, 128], act), h.tensor([2, Hkv, S, 128], act)
    pos = h.tensor([2], I64)
    kw = {}
    if scales:
        kw = {"k_scale": h.tensor(kshape or [Hkv], sdt), "v_scale": h.tensor(vshape or [Hkv], sdt)}
    return h.attentionKVCache(kc, vc, q, k, v, pos, None, **kw)


@pytest.mark.parametrize("act", [F16, BF16])
@pytest.mark.parametrize("Hq", [4, 8, 32])
def test_shape_rule_accepts_fp8_caches(B, act, Hq):
    assert _att(B, act=act, Hq=Hq).shape() == [2, Hq, 1, 128]


@pytest.mark.parametrize("kw,msg", [
    (dict(S=4), "one token per step"),                                  # a prompt chunk over an FP8 cache
    (dict(act=F32), "f16 / bf16"),                                      # fp32 activations
    (dict(scales=False), "needs k_scale and v_scale"),                  # scales missing
    (dict(kshape=[8]), "f32 [Hkv]"),                                    # one scale per query head, not per KV head
    (dict(vshape=[4, 1]), "f32 [Hkv]"),                                 # mis-shaped
    (dict(sdt=F16), "f32 [Hkv]"),                                       # scales not f32
    (dict(v_cache_dt=BF16), "both be FP8"),                             # mixed cache dtypes
    (dict(cache_dt=BF16), "FP8 caches only"),                           # scales without FP8 caches
])
def test_shape_rule_refuses(B, kw, msg):
    with pytest.raises(RuntimeError, match=re.escape(msg)):
        _att(B, **kw)


def test_scales_go_together(B):
    h = B.GraphHandler(B.HostPlanRuntime())
    t = h.tensor([4], F32)
    with pytest.raises(ValueError):
        h.attentionKVCache(t, t, t, t, t, t, None, k_scale=t)


# ---------------------------------------------------------------------------------------------------- quantiser
@pytest.mark.parametrize("x,code", [
    (0.0, 0x00), (-0.0, 0x80), (1.0, 0x38), (-1.0, 0xB8), (448.0, 0x7E), (-448.0, 0xFE),
    (464.0, 0x7E), (1e9, 0x7E), (-np.inf, 0xFE), (np.inf, 0x7E),       # saturation (satfinite): +-448, infinities too
    (2.0 ** -9, 0x01), (2.0 ** -10, 0x00), (1.5 * 2.0 ** -10, 0x01),   # smallest subnormal; half of it ties to even (0)
    (3 * 2.0 ** -10, 0x02),                                             # 1.5 x 2^-9: tie between codes 1 and 2 -> 2 (even)
    (1.0625, 0x38), (1.1875, 0x3A), (2.0 ** -6, 0x08), (7 * 2.0 ** -9, 0x07),
    (240.0, 0x77), (256.0, 0x78), (432.0, 0x7E),                       # 432 ties 416 / 448 -> 448 (even mantissa)
])
def test_quantiser_known_answers(x, code):
    assert int(KV.e4m3(np.float32(x))) == code
    if np.isfinite(x) and abs(x) <= 448:
        assert KV.decode(np.uint8(code)) == pytest.approx(KV.DECODE[code])


def test_quantiser_nan_and_table():
    assert int(KV.e4m3(np.float32(np.nan))) & 0x7F == 0x7F
    finite = [c for c in range(256) if (c & 0x7F) != 0x7F]
    vals = KV.decode(np.array(finite, np.uint8)).astype(np.float32)
    assert np.array_equal(KV.e4m3(vals), np.array(finite, np.uint8)), "every finite code round-trips"
    assert KV.DECODE[0x7E] == 448.0 and KV.DECODE[0x01] == 2.0 ** -9


def _tie_inputs(scales):
    """fp32 inputs within a few ulps of x = (midpoint between two E4M3 values) x scale: where the rounding of x / scale decides
    the code, so a quantiser that multiplies by a rounded reciprocal gives other codes on some of them"""
    mids = (KV.DECODE[1:127] + KV.DECODE[0:126]) / 2
    xs = []
    for sc in scales:
        base = (mids * np.float64(sc)).astype(np.float32)
        for d in range(-3, 4):
            xs.append(base + d * np.spacing(base))
    return np.concatenate(xs).astype(np.float32)


def test_quantiser_divides_rather_than_multiplying_by_a_reciprocal():
    scales = (np.float32(0.7) / np.float32(448), np.float32(0.3), np.float32(1.7) / np.float32(448))
    diff = sum(int(np.sum(KV.quantise(x, sc) != KV.quantise_reciprocal(x, sc))) for sc in scales
               for x in [_tie_inputs([sc])])
    assert diff > 0, "the two rules must be distinguishable"


def test_product_quantiser_agrees():
    from infinitensor_b200 import graphs as G
    x = np.random.default_rng(4).standard_normal(50000).astype(np.float32) * np.float32(300)
    assert np.array_equal(G.e4m3_codes_host(x), KV.e4m3(x))


# ---------------------------------------------------------------------------------------------------- emulation vs bound
def _case(H=4, S=1024, p=700, qscale=0.5, seed=0):
    rng = np.random.default_rng(seed)
    kc, ksc = KV.fill(rng.standard_normal((1, H, S, 128)).astype(np.float32) * np.float32(0.5))
    vc, vsc = KV.fill(rng.standard_normal((1, H, S, 128)).astype(np.float32) * np.float32(0.5))
    q = (rng.standard_normal((1, H, 1, 128)) * qscale).astype(np.float32)
    k, v = (rng.standard_normal((1, H, 1, 128)) * 0.5).astype(np.float32), (rng.standard_normal((1, H, 1, 128)) * 0.5).astype(np.float32)
    return kc, vc, ksc, vsc, q, k, v, np.array([p])


def _emulate(case, bugs=()):
    import oracle
    kc, vc, ksc, vsc, q, k, v, pos = case
    kc1, vc1 = kc.copy(), vc.copy()
    got = oracle.round_to(KV.emulate32(kc1, vc1, ksc, vsc, q, k, v, pos, bugs=bugs), BF16)
    kc2, vc2 = kc.copy(), vc.copy()
    KV.append(kc2, vc2, k, v, ksc, vsc, pos)
    ref, bound = KV.attention(kc2, vc2, ksc, vsc, q, pos, BF16)
    return got, ref, bound


@pytest.mark.parametrize("p,qscale", [(0, 0.5), (127, 0.5), (128, 0.5), (700, 0.5), (1023, 8.0), (300, 8.0)])
def test_emulation_within_bound(p, qscale):
    got, ref, bound = _emulate(_case(p=p, qscale=qscale))
    assert len(KV.violations(got, ref, bound)) == 0


@pytest.mark.parametrize("bug", ["scale_twice", "neighbour_scale", "unquantised_append", "chunk_off_by_one"])
def test_bound_catches_slips(bug):
    # two score regimes: a slip must leave the bound in at least one
    hits = 0
    for p, qscale, seed in ((700, 0.5, 1), (300, 8.0, 2), (5, 4.0, 5)):
        case = _case(p=p, qscale=qscale, seed=seed)
        if bug == "neighbour_scale":  # heads with distinct scales
            case[2][:] = case[2] * np.array([1, 2, 3, 4], np.float32)
            case[3][:] = case[3] * np.array([1, 2, 3, 4], np.float32)
        got, ref, bound = _emulate(case, bugs=(bug,))
        hits += len(KV.violations(got, ref, bound)) > 0
    assert hits > 0, f"{bug}: the emulation with the slip stays inside the bound"


def test_reciprocal_quantiser_caught_by_the_appended_codes():
    # one code off in the appended row moves the output far less than the bound: the GPU tests compare the appended codes bit
    # for bit, and this is the slip that comparison catches
    case = _case(H=4, p=10)
    kc, vc, ksc, vsc, q, k, v, pos = case
    k, ksc = k.copy(), np.array([0.7 / 448, 0.3, 1.7 / 448, 0.011], np.float32)
    found = 0
    for h in range(4):  # inputs on which the two rules disagree for this head's scale
        x = _tie_inputs([ksc[h]])
        x = x[KV.quantise(x, ksc[h]) != KV.quantise_reciprocal(x, ksc[h])][:128]
        k[0, h, 0, :x.size] = x
        found += x.size
    assert found > 0
    kc1, vc1, kc2, vc2 = kc.copy(), vc.copy(), kc.copy(), vc.copy()
    KV.emulate32(kc1, vc1, ksc, vsc, q, k, v, pos, bugs=("reciprocal",))
    KV.emulate32(kc2, vc2, ksc, vsc, q, k, v, pos)
    ref_k, ref_v = kc.copy(), vc.copy()
    KV.append(ref_k, ref_v, k, v, ksc, vsc, pos)
    assert np.array_equal(kc2, ref_k) and np.array_equal(vc2, ref_v)
    assert not np.array_equal(kc1, ref_k), "the reciprocal-multiply quantiser must give other codes on tie inputs"


# ---------------------------------------------------------------------------------------------------- graphs
def test_llama_fp8_graph_schedule_and_bytes(B):
    from infinitensor_b200 import graphs as G
    cfg = G.LlamaConfig(layers=2, d_model=512, heads=4, kv_heads=2, head_dim=128, ffn=1024, vocab=128, s_max=32, batch=4,
                        kv_fp8=True)
    h = B.GraphHandler(B.HostPlanRuntime())
    g = G.build_llama_decode(h, cfg)
    assert g.k_caches[0].dtype() == FP8 and g.k_caches[0].shape() == [4, 2, 32, 128]
    assert g.weights["l0.k_scale"][2] == "kv_scale" and g.weights["l1.v_scale"][1] == (2,)
    h.data_malloc()
    sc = h.schedule()
    assert sum(s.startswith("AttentionRope") for s in sc) == 2, sc   # RoPE(q), RoPE(k) still fold
    c16 = G.LlamaConfig(**{**cfg.__dict__, "kv_fp8": False})
    kv16 = c16.algorithmic_bytes(500) - cfg.algorithmic_bytes(500)
    elems = 2 * 2 * 4 * 2 * 128 * 502
    assert kv16 == elems - 2 * 2 * 2 * 4, "FP8 cache: one byte per element plus the scales"
    with pytest.raises(AssertionError):
        G.build_llama_decode(B.GraphHandler(B.HostPlanRuntime()), cfg, seq=4)


def test_llama_presets_take_kv_fp8():
    from infinitensor_b200 import graphs as G
    assert G.LlamaConfig.llama3_8b(kv_fp8=True).kv_fp8 and G.LlamaConfig.tinyllama_1b(kv_fp8=True).kv_fp8
    assert not G.LlamaConfig.llama3_8b().kv_fp8


def test_kv_fp8_cache_helpers_shard_by_head():
    from infinitensor_b200 import graphs as G
    cfg = G.LlamaConfig(layers=1, d_model=256, heads=4, kv_heads=4, head_dim=128, ffn=256, vocab=64, s_max=16, batch=2,
                        kv_fp8=True)
    full_c, full_s = G.llama_kv_fp8_values(cfg, 0, "k")
    c1, s1 = G.llama_kv_fp8_values(cfg, 0, "k", world=2, rank=1)
    assert np.array_equal(c1, full_c[:, 2:]) and np.array_equal(s1, full_s[2:])
    vals = G.llama_cache_values(cfg, 0, "k")
    dq = KV.decode(full_c) * full_s[None, :, None, None]
    assert np.abs(dq - vals).max() <= np.abs(vals).max() * 2.0 ** -4


# ---------------------------------------------------------------------------------------------------- ONNX
def _cfg(**kw):
    from infinitensor_b200 import graphs as G
    base = dict(layers=2, d_model=512, heads=4, kv_heads=2, head_dim=128, ffn=1024, vocab=128, s_max=32, batch=4, kv_fp8=True)
    base.update(kw)
    return G.LlamaConfig(**base)


def test_onnx_round_trip_with_scales(B):
    from infinitensor_b200 import graphs as G
    from infinitensor_b200 import onnx_lite as X
    rt = B.HostPlanRuntime()
    cfg = _cfg()
    direct = B.GraphHandler(rt)
    G.build_llama_decode(direct, cfg)
    exp = X.OnnxExporter(B.GraphHandler(rt))
    G.build_llama_decode(exp, cfg)
    blob = exp.save()
    m = X.load_model(blob)
    att = [n for n in m.graph.nodes if n.op_type == "AttentionKVCache"]
    assert len(att) == 2 and all(len(n.inputs) == 8 for n in att)
    elem = {v.name: (v.elem_type, list(v.dims)) for v in m.graph.inputs}
    assert elem[att[0].inputs[0]] == (FP8, [4, 2, 32, 128])
    h = B.GraphHandler(rt)
    X.OnnxStub(blob, handler=h, upload=False)
    assert h.schedule() == direct.schedule()


# sha256 of OnnxExporter.save() for 16-bit decode graphs, as the exporter wrote them before FP8 caches existed: the optional
# scale inputs are written only when given, so these files do not change
EXPORT_SHA256 = {
    "llama": "47cfdb3857dc63ff99e9f85a6b8d150623d7c9ef7c177a21f0b8a629fe82d814",
    "gqa": "74b1e5856209e1a7265f0bc9618994f737bd6ad05aecbdddd89b19175d5fac96",
    "d64": "a2b5cb9cf0215ccbdca3e19c3a17cdad3494b8fca8ba286a021dc85a9c6d7d47",
}


@pytest.mark.parametrize("which", sorted(EXPORT_SHA256))
def test_16bit_exports_unchanged(B, which):
    import hashlib
    from infinitensor_b200 import graphs as G
    from infinitensor_b200 import onnx_lite as X
    cfg = {"llama": _cfg(kv_heads=None, kv_fp8=False), "gqa": _cfg(kv_fp8=False),
           "d64": G.LlamaConfig.tinyllama_1b(batch=2, s_max=16, layers=2)}[which]
    exp = X.OnnxExporter(B.GraphHandler(B.HostPlanRuntime()))
    G.build_llama_decode(exp, cfg)
    assert hashlib.sha256(exp.save()).hexdigest() == EXPORT_SHA256[which]


def test_parallel_model_shards_scales_by_head(B):
    from infinitensor_b200 import graphs as G
    from infinitensor_b200 import onnx_lite as X
    rt = B.HostPlanRuntime()
    cfg = _cfg(kv_heads=4)
    direct = B.GraphHandler(rt)
    G.build_llama_decode(direct, cfg, 2, 1)
    exp = X.OnnxExporter(B.GraphHandler(rt))
    G.build_llama_decode(exp, cfg)
    sharded = X.parallel_model(exp.save(), 2, 1)
    m = X.load_model(sharded) if isinstance(sharded, (bytes, bytearray)) else sharded
    dims = {v.name: list(v.dims) for v in m.graph.inputs}
    dims.update({t.name: list(np.shape(t.array)) if t.array is not None else list(t.dims) for t in m.graph.initializers})
    att = [n for n in m.graph.nodes if n.op_type == "AttentionKVCache"]
    assert len(att) == 2
    for n in att:  # the rank's two of four KV heads, scales with them
        assert dims[n.inputs[0]] == [4, 2, 32, 128] and dims[n.inputs[6]] == [2] and dims[n.inputs[7]] == [2]
    h = B.GraphHandler(rt)
    X.OnnxStub(sharded, handler=h, upload=False)
    assert h.schedule() == direct.schedule()
