"""CPU tier for 4-bit MatMulNBits: the operator's shape rule and the launcher's refusals, the layout on hand-built known answers,
a float32 emulation of the decode kernel against the float64 bound (and the slips it must catch), the schedule of an int4 Llama
graph, ONNX round trips and the tensor-parallel refusal."""
import ctypes
import re

import numpy as np
import pytest

from tests import ref64
from tests import w4_oracle as W
from tests.llama_oracle import LlamaOracleHandler

F32, U8, F16, BF16, I64 = 1, 2, 10, 16, 7


@pytest.fixture(scope="module")
def B():
    from infinitensor_b200 import backend
    return backend


def _nbits(B, K=256, N=64, bs=64, act=BF16, bits=4, bshape=None, bdt=U8, sdt=None, ssize=None, zp=False, zsize=None, zdt=U8,
           g_idx=False, bias=False, adims=None):
    h = B.GraphHandler(B.HostPlanRuntime())
    a = h.tensor(adims or [4, K], act)
    b = h.tensor(bshape or [N, K // bs, bs // 2], bdt)
    s = h.tensor([ssize or N * (K // bs)], sdt or act)
    z = h.tensor([zsize or N * (K // bs) // 2], zdt) if zp else None
    gi = h.tensor([K], 6) if g_idx else None
    bi = h.tensor([N], act) if bias else None
    return h.matMulNBits(a, b, s, z, None, K, N, bs, bits=bits, g_idx=gi, bias=bi)


@pytest.mark.parametrize("act", [F16, BF16])
@pytest.mark.parametrize("zp", [False, True])
def test_shape_rule_accepts(B, act, zp):
    y = _nbits(B, act=act, zp=zp, adims=[2, 3, 256])
    assert y.shape() == [2, 3, 64] and y.dtype() == act


@pytest.mark.parametrize("kw,msg", [
    (dict(bits=8), "only 4-bit weights"),
    (dict(bs=16, bshape=[64, 16, 8]), "block_size = 16 is not 32, 64 or 128"),
    (dict(K=320, bs=128, bshape=[64, 2, 64], ssize=128), "K = 320 is not a positive multiple of block_size 128"),
    (dict(N=40, bshape=[40, 4, 32], ssize=160), "N = 40 is not a positive multiple of 16"),
    (dict(bshape=[64, 4, 16]), "B must be uint8 [N, K / block_size, block_size / 2]"),
    (dict(bdt=F16), "B must be uint8"),
    (dict(ssize=64), "scales must hold N * K / block_size = 256"),
    (dict(sdt=F16), "scales must hold"),                                # scales not of A's dtype
    (dict(K=192, bs=64, bshape=[64, 3, 32], ssize=192, zp=True, zsize=96), "zero points need an even number of blocks"),
    (dict(zp=True, zsize=64), "zero_points must be uint8 with N * (K / block_size) / 2 = 128"),
    (dict(zp=True, zdt=F16), "zero_points must be uint8"),
    (dict(act=F32, sdt=F32), "fp32 activations are not supported"),
    (dict(g_idx=True), "g_idx input (act-order) is not supported"),
    (dict(bias=True), "bias input is not supported"),
    (dict(adims=[4, 128]), "last dimension of A must be K = 256"),
])
def test_shape_rule_refuses(B, kw, msg):
    with pytest.raises(RuntimeError, match=re.escape(msg)):
        _nbits(B, **kw)


def _launch(dtype=BF16, ng=1, m=16, k=256, N=64, bs=64, zp=False, residual=False, align=0):
    """it_b200_matmul_nbits with dummy (never dereferenced) pointers: every refusal below returns before touching the device"""
    from infinitensor_b200 import _lib as L
    VP = ctypes.c_void_p
    p = 1 << 20
    arr = lambda n, base: (VP * max(n, 1))(*[base + 4096 * i for i in range(max(n, 1))])
    Ns = L.i32arr([N] * max(ng, 1))
    r = L.lib.it_b200_matmul_nbits(dtype, VP(p + align), ng, arr(ng, p), arr(ng, 2 * p), arr(ng, 3 * p) if zp else None,
                                   arr(ng, 4 * p), Ns, m, k, bs, VP(5 * p) if residual else None, None, 0, None)
    return r, L.last_error()


@pytest.mark.parametrize("kw,msg", [
    (dict(dtype=F32), "activations / scales must be f16 or bf16"),
    (dict(ng=0), "1..4 weight matrices"),
    (dict(ng=5), "1..4 weight matrices"),
    (dict(ng=2, residual=True), "a residual goes with a single weight matrix"),
    (dict(bs=48), "block_size 48 is not 32, 64 or 128"),
    (dict(k=320, bs=128), "K = 320 is not a positive multiple of block_size 128"),
    (dict(N=40), "N = 40 is not a positive multiple of 16"),
    (dict(k=192, zp=True), "zero points need an even number of blocks"),
    (dict(align=8), "X and the residual must be 16-byte aligned"),
    (dict(m=100), "workspace 0 <"),
])
def test_launcher_refuses(B, kw, msg):
    r, err = _launch(**kw)
    assert r != 0 and msg in err, err


def test_workspace_only_for_many_rows():
    from infinitensor_b200 import _lib as L
    Ns = L.i32arr([1024, 4096])
    assert L.lib.it_b200_matmul_nbits_workspace(BF16, 64, 4096, 2, Ns) == 0
    assert L.lib.it_b200_matmul_nbits_workspace(BF16, 65, 4096, 2, Ns) == 4096 * 4096 * 2


# ---------------------------------------------------------------------------------------------------- layout known answers
def test_nibble_order_and_default_zero_point():
    K, N, bs = 64, 16, 32
    b = np.zeros((N, K // bs, bs // 2), np.uint8)
    b[0, 0, 0] = 0x21   # column 0: k 0 -> 1, k 1 -> 2 (even k in the low nibble)
    b[3, 1, 5] = 0xF0   # column 3: k = 32 + 10 -> 0, k = 43 -> 15
    s = np.ones(N * K // bs, np.float32)
    w = W.dequantize(b, s, None, K, N, bs)
    assert w[0, 0] == 1 - 8 and w[1, 0] == 2 - 8 and w[2, 0] == -8
    assert w[42, 3] == -8 and w[43, 3] == 15 - 8


def test_block_order_of_scales():
    K, N, bs = 128, 16, 32
    b = np.full((N, K // bs, bs // 2), 0x99, np.uint8)  # q = 9 everywhere: (q - 8) = 1
    s = np.arange(N * K // bs, dtype=np.float32)          # the scale of (n, block) is element n * (K / bs) + block
    w = W.dequantize(b, s, None, K, N, bs)
    for n, k in [(0, 0), (0, 33), (2, 127), (15, 64)]:
        assert w[k, n] == n * (K // bs) + k // bs


def test_packed_zero_points():
    K, N, bs = 128, 16, 64
    b = np.zeros((N, K // bs, bs // 2), np.uint8)        # q = 0
    z = np.zeros(N * (K // bs) // 2, np.uint8)
    z[0] = 0x53   # column 0: block 0 -> z 3, block 1 -> z 5 (low nibble for the even block)
    z[7] = 0xA0   # column 7: block 0 -> 0, block 1 -> 10
    s = np.ones(N * K // bs, np.float32)
    w = W.dequantize(b, s, z, K, N, bs)
    assert w[0, 0] == -3 and w[63, 0] == -3 and w[64, 0] == -5 and w[127, 0] == -5
    assert w[0, 7] == 0 and w[100, 7] == -10 and w[5, 1] == 0


def test_quantize_w4_known_answers():
    """graphs.quantize_w4: scale = amax / 7 per block, rint half to even, + 8, clamped to [0, 15], the oracle's layout"""
    from infinitensor_b200 import graphs as G
    K, N, bs = 64, 16, 32
    w = np.zeros((K, N), np.float32)
    w[:bs, 0] = 0.25
    w[0, 0] = 1.75              # amax 1.75 -> scale 0.25: 1.75 -> 7, 0.25 -> 1
    w[1, 0] = -1.75 / 7 * 2.5   # -2.5 -> rint -2 (half to even)
    w[bs, 1] = -0.5             # block 1 of column 1: scale 0.5 / 7, -7 -> q 1
    codes, scale = G.quantize_w4(w, bs, F32)
    assert codes.shape == (N, K // bs, bs // 2) and scale.shape == (N * K // bs,)
    q = W.unpack_codes(codes, K)
    assert q[0, 0] == 15 and q[0, 1] == 6 and q[0, 2] == 9 and q[1, 32] == 1 and q[2, 0] == 8
    assert scale[0] == np.float32(0.25) and scale[1 * (K // bs) + 1] == np.float32(0.5) / np.float32(7)
    deq = W.dequantize(codes, scale, None, K, N, bs)
    assert abs(deq[0, 0] - 1.75) < 1e-7 and deq[1, 0] == -0.5


# ---------------------------------------------------------------------------------------------------- emulation vs bound
def _case(dt, bs, zp, K=1024, N=256, m=16, seed=0):
    rng = np.random.default_rng(seed + bs)
    x = ref64.activations(m, K, dt, seed)
    q = rng.integers(0, 16, size=(N, K), dtype=np.uint8)
    import oracle
    s = oracle.round_to((rng.uniform(0.5, 1.5, size=(N, K // bs)) * 0.01).astype(np.float32), dt).reshape(-1)
    z = W.pack_zero_points(rng.integers(0, 16, size=(N, K // bs), dtype=np.uint8)) if zp else None
    return x, W.pack_codes(q), s, z, K, N, bs, dt


@pytest.mark.parametrize("dt", [F16, BF16])
@pytest.mark.parametrize("bs", [32, 64, 128])
@pytest.mark.parametrize("zp", [False, True])
def test_emulation_within_bound(dt, bs, zp):
    x, b, s, z, K, N, bs, dt = _case(dt, bs, zp)
    ref, bound = W.reference(x, b, s, z, K, N, bs, dt)
    got = W.emulate32(x, b, s, z, K, N, bs, dt)
    assert not W.violations(got, ref, bound).any()
    assert (np.abs(got - ref) / bound).max() < 0.75  # with room to spare


@pytest.mark.parametrize("bug", ["swapped_nibbles", "z7", "neighbour_scale", "boundary_16", "scale_twice", "weight_rounded"])
@pytest.mark.parametrize("dt", [F16, BF16])
def test_bound_catches_slips(dt, bug):
    x, b, s, z, K, N, bs, dt = _case(dt, 64, False)
    ref, bound = W.reference(x, b, s, z, K, N, bs, dt)
    bad = W.violations(W.emulate32(x, b, s, z, K, N, bs, dt, bugs=(bug,)), ref, bound)
    assert bad.mean() > 0.05, f"{bug}: only {bad.sum()} elements outside the bound"


# ---------------------------------------------------------------------------------------------------- graphs
def _cfg(**kw):
    from infinitensor_b200 import graphs as G
    base = dict(layers=2, d_model=512, heads=4, kv_heads=2, head_dim=128, ffn=1024, vocab=128, s_max=32, batch=4)
    base.update(kw)
    return G.LlamaConfig(**base)


@pytest.mark.parametrize("seq", [1, 4])
def test_int4_llama_schedule_matches_16bit(B, seq):
    from infinitensor_b200 import graphs as G
    kinds = {}
    for bs in (0, 32, 128):
        h = B.GraphHandler(B.HostPlanRuntime())
        g = G.build_llama_decode(h, _cfg(int4_block=bs), seq=seq)
        h.data_malloc()
        kinds[bs] = [st.split(":")[0] for st in h.schedule()]
        if bs:
            assert g.weights["l0.wq"][2] == "proj_int4" and g.weights["lm_head.scale"][1] == (128 * 512 // bs,)
    assert kinds[32] == kinds[0] and kinds[128] == kinds[0]
    if seq == 1:
        assert kinds[0].count("MatMulGroup") == 4 and kinds[0].count("MatMulAdd") == 4


def test_int4_config_refusals_and_bytes(B):
    from infinitensor_b200 import graphs as G
    h = lambda: B.GraphHandler(B.HostPlanRuntime())
    with pytest.raises(ValueError, match="world must be 1"):
        G.build_llama_decode(h(), _cfg(int4_block=64, kv_heads=4), world=2)
    with pytest.raises(ValueError, match="exclude each other"):
        G.build_llama_decode(h(), _cfg(int4_block=64, fp8_weights=True))
    with pytest.raises(ValueError, match="32, 64 or 128"):
        G.build_llama_decode(h(), _cfg(int4_block=48))
    assert G.LlamaConfig.llama3_8b(int4_block=128).int4_block == 128 and G.LlamaConfig.tinyllama_1b(int4_block=32).int4_block == 32
    c16, c4 = G.LlamaConfig(), G.LlamaConfig(int4_block=128)
    d, f, V, L = 4096, 11008, 32000, 32
    proj = L * (4 * d * d + 3 * d * f) + d * V
    assert c16.algorithmic_bytes(511) - c4.algorithmic_bytes(511) == 2 * proj - (proj // 2 + 2 * proj // 128)


def _export(B, cfg, inner):
    """(exporter, graph) with the weights filled through the exporter"""
    from infinitensor_b200 import graphs as G
    from infinitensor_b200 import onnx_lite as X
    exp = X.OnnxExporter(inner)
    g = G.build_llama_decode(exp, cfg)
    G.fill_llama_weights_host(g)
    return exp, g


def test_onnx_round_trip_schedule(B):
    from infinitensor_b200 import graphs as G
    from infinitensor_b200 import onnx_lite as X
    rt = B.HostPlanRuntime()
    cfg = _cfg(int4_block=64)
    direct = B.GraphHandler(rt)
    G.build_llama_decode(direct, cfg)
    exp, _ = _export(B, cfg, B.GraphHandler(rt))
    blob = exp.save()
    m = X.load_model(blob)
    nb = [n for n in m.graph.nodes if n.op_type == "MatMulNBits"]
    assert len(nb) == 2 * 7 + 1 and all(n.domain == "com.microsoft" for n in nb)
    assert nb[0].attrs == {"K": 512, "N": 512, "bits": 4, "block_size": 64} and len(nb[0].inputs) == 3
    assert m.opset == 17
    h = B.GraphHandler(rt)
    X.OnnxStub(blob, handler=h, upload=False)
    assert h.schedule() == direct.schedule()


def test_onnx_round_trip_oracle_bit_identical():
    """the exported file, imported on the graph oracle, computes what the directly built graph computes, bit for bit"""
    from infinitensor_b200 import graphs as G
    from infinitensor_b200 import onnx_lite as X
    cfg = _cfg(int4_block=32, batch=2)
    exp, ge = _export(None, cfg, LlamaOracleHandler())
    blob = exp.save()
    oh = LlamaOracleHandler()
    og = G.build_llama_decode(oh, cfg)
    G.fill_llama_weights_host(og)
    ih = LlamaOracleHandler()
    stub = X.OnnxStub(blob, handler=ih)
    rng = np.random.default_rng(3)
    feeds = {ge.input_ids.name: rng.integers(0, cfg.vocab, size=(cfg.batch, 1)).astype(np.int64),
             ge.position_ids.name: np.full((cfg.batch, 1), 7, np.int64)}
    og.input_ids.copyin_numpy(feeds[ge.input_ids.name])
    og.position_ids.copyin_numpy(feeds[ge.position_ids.name])
    for li in range(cfg.layers):
        for which, ce, co in (("k", ge.k_caches[li], og.k_caches[li]), ("v", ge.v_caches[li], og.v_caches[li])):
            feeds[ce.name] = G.to_storage(G.llama_cache_values(cfg, li, which), cfg.dtype)
            co.copyin_numpy(feeds[ce.name])
    for name, arr in feeds.items():
        stub.inputs[name].copyin_numpy(arr)
    oh.run()
    ih.run()
    out = stub.outputs[ge.logits.name].copyout_numpy()
    assert np.array_equal(out, og.logits.copyout_numpy())


def test_domain_and_opset_only_when_used(B):
    from infinitensor_b200 import graphs as G
    from infinitensor_b200 import onnx_lite as X
    rt = B.HostPlanRuntime()
    exp16 = X.OnnxExporter(B.GraphHandler(rt))
    G.build_llama_decode(exp16, _cfg())
    b16 = exp16.save()
    assert b"com.microsoft" not in b16
    exp4 = X.OnnxExporter(B.GraphHandler(rt))
    G.build_llama_decode(exp4, _cfg(int4_block=128))
    b4 = exp4.save()
    assert b4.count(b"com.microsoft") == 2 * 7 + 1 + 1  # every MatMulNBits node + one opset import
    m = X.load_model(b4)
    assert all(n.domain == ("com.microsoft" if n.op_type == "MatMulNBits" else "") for n in m.graph.nodes)
    assert X.save_model(m) == b4  # the domain and the opset import survive a load / save


def test_onnx_import_refuses_g_idx_and_bias(B):
    """a hand-built MatMulNBits node with g_idx or bias inputs is refused by the backend with the operator's message"""
    from infinitensor_b200 import onnx_lite as X
    K, N, bs = 128, 32, 64
    for extra, msg in ((["", "", "bias"], "bias input"), (["", "g"], "g_idx input")):
        inits = [X.TensorProto("b", [N, K // bs, bs // 2], U8, np.zeros((N, K // bs, bs // 2), np.uint8)),
                 X.TensorProto("s", [N * K // bs], F16, np.ones(N * K // bs, np.float16)),
                 X.TensorProto("g", [K], 6, np.zeros(K, np.int32)), X.TensorProto("bias", [N], F16, np.zeros(N, np.float16))]
        node = X.Node("MatMulNBits", ["a", "b", "s"] + extra, ["y"], "n0", {"K": K, "N": N, "bits": 4, "block_size": bs,
                                                                           "accuracy_level": 4}, "com.microsoft")
        m = X.Model(X.Graph([node], inits, [X.ValueInfo("a", F16, [2, K])], [X.ValueInfo("y", F16, [2, N])]))
        with pytest.raises(RuntimeError, match=msg):
            X.OnnxStub(X.save_model(m), handler=B.GraphHandler(B.HostPlanRuntime()), upload=False)


def test_parallel_model_refuses(B):
    from infinitensor_b200 import onnx_lite as X
    exp, _ = _export(B, _cfg(int4_block=64, kv_heads=4), B.GraphHandler(B.HostPlanRuntime()))
    with pytest.raises(NotImplementedError, match="MatMulNBits"):
        X.parallel_model(exp.save(), 2, 0)
