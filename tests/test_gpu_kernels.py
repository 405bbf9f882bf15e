"""GPU parity tests: every C-ABI launcher vs (a) the reference's golden vectors and (b) the CPU oracle
on seeded inputs.  Tolerances are the ones SURVEY.md 8(c) states per op, written next to each check.
Run with `pytest -m gpu` on an H100."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import oracle
from tests.golden import reference_vectors as G

F32, F16, BF16 = 1, 10, 16
# relative tolerance of one rounding step in the storage dtype
EPS = {F32: 2.0 ** -23, F16: 2.0 ** -10, BF16: 2.0 ** -7}


@pytest.fixture(scope="module")
def K():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from tests import kernel_harness
    return kernel_harness


def close(got, exp, rel, abs_):
    got = np.asarray(got, np.float64).ravel()
    exp = np.asarray(exp, np.float64).ravel()
    assert got.shape == exp.shape, (got.shape, exp.shape)
    np.testing.assert_allclose(got, exp, rtol=rel, atol=abs_)


def rnd(shape, seed, dt=F32, scale=1.0):
    x = (np.random.default_rng(seed).standard_normal(shape) * scale).astype(np.float32)
    return oracle.round_to(x, dt)


# ------------------------------------------------------------------ golden vectors of the reference
@pytest.mark.parametrize("c", G.MATMUL)
def test_matmul_golden(K, c):
    close(K.matmul(c["a"], c["b"], transA=c["tA"], transB=c["tB"]), c["out"], 1e-6, 1e-6)


@pytest.mark.parametrize("c", G.CONV)
def test_conv_golden(K, c):
    close(K.conv2d(c["x"], c["w"], *c["args"]), c["out"], 1e-6, 1e-6)
    close(K.conv2d(c["x"], c["w"], *c["args"], dt=F16), oracle.conv2d(c["x"], c["w"], *c["args"], dt=F16), 1e-3, 1e-3)


@pytest.mark.parametrize("c", G.SOFTMAX)
def test_softmax_golden(K, c):
    close(K.softmax(c["x"], c["axis"], dt=c["dt"]), c["out"], 2e-6 if c["dt"] == 1 else 1e-6, 1e-9)


@pytest.mark.parametrize("c", G.LAYERNORM)
def test_layernorm_golden(K, c):
    bias = None if c["bias"] is None else np.array(c["bias"], np.float32)
    got = K.layer_norm(c["x"], np.array(c["scale"], np.float32), bias, 1e-5, c["axis"], dt=c["dt"])
    close(got, c["out"], 2e-6, 3e-7)


def test_attention_golden(K):
    c = G.ATTENTION
    z = np.zeros((1, 1, 1, 128), np.float32)
    one = np.ones((1, 1, 1, 128), np.float32)
    out, kc, vc = K.attention_kvcache(z, z, one, one, one, c["pos"], pos_np_dtype=np.uint32)
    close(out, c["out"], 1e-6, 0)
    assert np.array_equal(kc, one) and np.array_equal(vc, one)  # in-place append


def test_rope_golden(K):
    x = np.zeros((1, 1, 128), np.float32)
    x[..., :64] = 1.0
    out = K.rope(np.array([[1]]), x, pos_np_dtype=np.uint32)
    close(out[0, 0, :32], G.ROPE_COS, 2e-6, 1e-6)


@pytest.mark.parametrize("c", G.ELEMENTWISE)
def test_elementwise_golden(K, c):
    close(K.binary(c["op"], c["a"], c["b"]), c["out"], 1e-6, 0)


@pytest.mark.parametrize("c", G.POOL)
def test_pool_golden(K, c):
    close(K.pool2d(c["kind"], c["x"], *c["kdps"]), c["out"], 2e-6, 0)


def test_batchnorm_golden(K):
    c = G.BATCHNORM
    close(K.batch_norm(c["x"], c["mean"], c["var"], c["scale"], c["bias"], c["eps"]), c["out"], 2e-6, 1e-7)


@pytest.mark.parametrize("c", G.REDUCE)
def test_reduce_golden(K, c):
    close(K.reduce(c["kind"], c["x"], c["axes"], c["keep"]), c["out"], 1e-6, 0)


def test_movement_golden(K):
    c = G.TRANSPOSE
    assert K.transpose(c["x"], c["perm"]).ravel().tolist() == c["out"]
    for c in G.CONCAT:
        assert K.concat(c["xs"], c["dim"]).ravel().tolist() == c["out"]
    c = G.SPLIT
    assert [o.ravel().tolist() for o in K.split(c["x"], c["axis"], [3, 3, 4])] == c["outs"]
    for c in G.GATHER:
        assert K.gather(c["x"], c["idx"], c["axis"]).ravel().tolist() == c["out"]
    for c in G.WHERE:
        assert K.where(c["c"], c["x"], c["y"]).ravel().tolist() == c["out"]
    assert K.expand(G.EXPAND["x"], G.EXPAND["dims"]).ravel().tolist() == G.EXPAND["out"]
    c = G.PAD   # pads {1,0,1,1} axes {0,3} -> start = -begin
    assert K.pad_slice(c["x"], (3, 2, 3, 3), [-1, 0, 0, 0], [1, 1, 1, 1]).ravel().tolist() == c["out"]
    c = G.SLICE
    assert K.pad_slice(c["x"], (1, 2, 1, 4), [1, 0, 0, 1], [1, 1, 1, 1]).ravel().tolist() == c["out"]


# ------------------------------------------------------------------ seeded parity vs the oracle
@pytest.mark.parametrize("dt", [F32, F16, BF16])
@pytest.mark.parametrize("name", ["relu", "sigmoid", "tanh", "gelu", "silu", "erf", "neg", "abs", "sqrt",
                                  "hardsigmoid", "hardswish"])
def test_unary_parity(K, name, dt):
    x = rnd((3, 7, 129), 1, dt, 2.0)
    if name == "sqrt":
        x = np.abs(x)
    # fp32: <= 2 ulp vs oracle (reference test uses rel 1e-6); half types: 1 rounding step
    close(K.unary(name, x, dt), oracle.unary(name, x, dt), 4 * EPS[dt] if dt == F32 else 2 * EPS[dt], 5e-7)


@pytest.mark.parametrize("dt", [F32, F16, BF16])
@pytest.mark.parametrize("name", ["add", "sub", "mul", "div", "min", "max", "pow", "less"])
def test_binary_parity(K, name, dt):
    a, b = rnd((2, 1, 5, 64), 2, dt), rnd((3, 1, 64), 3, dt)
    if name in ("div",):
        b = np.where(np.abs(b) < 0.1, 0.5, b).astype(np.float32)
    if name == "pow":
        a = np.abs(a) + 0.1
    close(K.binary(name, a, b, dt), oracle.binary(name, a, b, dt), 8 * EPS[dt] if name == "pow" else 2 * EPS[dt], 1e-7)
    # same-shape + scalar fast paths
    c = rnd((4, 1000), 4, dt)
    c1 = oracle.round_to(np.abs(c) + 0.1, dt)
    c2 = oracle.round_to(np.abs(c[::-1].copy()) + 0.2, dt)
    close(K.binary(name, c1, c2, dt), oracle.binary(name, c1, c2, dt), 8 * EPS[dt], 1e-7)
    s = oracle.round_to(np.array([1.5], np.float32), dt)
    close(K.binary(name, c1, s, dt), oracle.binary(name, c1, s, dt), 8 * EPS[dt], 1e-7)


@pytest.mark.parametrize("dt", [F32, F16, BF16])
@pytest.mark.parametrize("shape,axis", [((2, 12, 128, 128), -1), ((4, 3000), 1), ((3, 5, 7), 1), ((2, 20000), -1)])
def test_softmax_parity(K, shape, axis, dt):
    x = rnd(shape, 5, dt, 3.0)
    tol = {F32: 1e-5, F16: 1e-3, BF16: 1e-2}[dt]  # SURVEY 8(c): norms/softmax 1e-5 / 1e-3 / 1e-2 rel
    close(K.softmax(x, axis, dt), oracle.softmax(x, axis, dt), tol, tol * 1e-3)


@pytest.mark.parametrize("dt", [F32, F16, BF16])
@pytest.mark.parametrize("shape,axis", [((1, 128, 768), -1), ((4, 2500), 1), ((3, 5, 6), 1)])
def test_layernorm_parity(K, shape, axis, dt):
    x = rnd(shape, 6, dt)
    dim = shape[axis]
    sc, bi = rnd((dim,), 7, dt), rnd((dim,), 8, dt)
    tol = {F32: 1e-5, F16: 1e-3, BF16: 1e-2}[dt]
    close(K.layer_norm(x, sc, bi, 1e-5, axis, dt), oracle.layer_norm(x, sc, bi, 1e-5, axis, dt), tol, tol)
    close(K.layer_norm(x, sc[:1], None, 1e-5, axis, dt), oracle.layer_norm(x, sc[:1], None, 1e-5, axis, dt), tol, tol)


@pytest.mark.parametrize("dt", [F32, F16, BF16])
@pytest.mark.parametrize("shape", [(16, 1, 4096), (3, 100), (5, 1000)])
def test_rmsnorm_parity(K, shape, dt):
    x, w = rnd(shape, 9, dt), 1 + rnd(shape[-1:], 10, dt, 0.02)
    w = oracle.round_to(w, dt)
    tol = {F32: 1e-5, F16: 1e-3, BF16: 1e-2}[dt]
    got, ref = K.rms_norm(x, w, dt), oracle.rms_norm(x, w, dt)
    close(got, ref, tol, tol * 1e-2)
    assert np.array_equal(got, K.rms_norm(x, w, dt, const_w=True))  # weight fetched ahead of the PDL wait: same bits
    if dt != F32:  # rounding order of rms_norm.cu:52 reproduced: overwhelmingly bit-identical
        assert np.mean(got == ref) > 0.98


@pytest.mark.parametrize("dt", [F32, F16, BF16])
def test_rope_parity(K, dt):
    x = rnd((16, 1, 4096), 11, dt)
    pos = np.full((16, 1), 511)
    pos[3, 0] = 0
    pos[5, 0] = 1023
    tol = {F32: 2e-4, F16: 2e-3, BF16: 1.6e-2}[dt]  # cos/sin of angles up to 1023 rad in float
    close(K.rope(pos, x, dt), oracle.rope(pos, x, dt=dt), tol, tol)
    x2 = rnd((2, 3, 256), 12, dt)
    pos2 = np.arange(6).reshape(2, 3) * 7
    close(K.rope(pos2, x2, dt, pos_np_dtype=np.int32), oracle.rope(pos2, x2, dt=dt), tol, tol)


@pytest.mark.parametrize("es", [np.uint8, np.float16, np.float32, np.int64])
def test_movement_parity(K, es):
    rng = np.random.default_rng(13)
    def mk(shape):
        return rng.integers(0, 100, size=shape).astype(es)
    x = mk((2, 128, 12, 64))
    assert np.array_equal(K.transpose(x, (0, 2, 1, 3)), oracle.transpose(x, (0, 2, 1, 3)))
    assert np.array_equal(K.transpose(x, (0, 2, 3, 1)), oracle.transpose(x, (0, 2, 3, 1)))
    assert np.array_equal(K.transpose(x, (3, 1, 0, 2)), oracle.transpose(x, (3, 1, 0, 2)))
    y = mk((5, 33, 65))
    assert np.array_equal(K.transpose(y, (2, 1, 0)), oracle.transpose(y, (2, 1, 0)))
    assert np.array_equal(K.transpose(y, (0, 2, 1)), oracle.transpose(y, (0, 2, 1)))
    assert np.array_equal(K.transpose(y, (0, 1, 2)), y)
    parts = [mk((3, 5, 8)), mk((3, 1, 8)), mk((3, 10, 8))]
    assert np.array_equal(K.concat(parts, 1), oracle.concat(parts, 1))
    many = [mk((2, 3)) for _ in range(40)]  # > 32 parts -> two launches
    assert np.array_equal(K.concat(many, 1), oracle.concat(many, 1))
    big = mk((1, 128, 2304))
    for got, ref in zip(K.split(big, 2, [768, 768, 768]), oracle.split(big, 2, 3)):
        assert np.array_equal(got, ref)
    emb = mk((1000, 96))
    idx = rng.integers(0, 1000, size=(16, 1)).astype(np.int64)
    assert np.array_equal(K.gather(emb, idx, 0), oracle.gather(emb, idx, 0))
    assert np.array_equal(K.gather(emb, idx.astype(np.int32), 1 - 1), oracle.gather(emb, idx, 0))
    g3 = mk((4, 9, 5))
    i3 = np.array([[8, 0], [3, -1]], np.int64)  # negative index wraps (ONNX)
    assert np.array_equal(K.gather(g3, i3, 1), oracle.gather(g3, i3, 1))
    c = rng.integers(0, 2, size=(2, 1, 5)).astype(np.uint8)
    a, b = mk((3, 1)), mk((2, 3, 5))
    assert np.array_equal(K.where(c, a, b), oracle.where(c, a, b))
    e = mk((2, 1, 4, 1))
    assert np.array_equal(K.expand(e, (2, 3, 4, 5)), oracle.expand(e, (2, 3, 4, 5)))
    s = mk((4, 6, 10))
    assert np.array_equal(K.pad_slice(s, (2, 3, 4), [1, 0, 9], [1, 2, -2]), oracle.slice_(s, [1, 0, 9], [3, 6, 1], None, [1, 2, -2]))
    assert np.array_equal(K.pad_slice(s, (5, 6, 13), [-1, 0, -2], [1, 1, 1]), oracle.pad(s, [1, 0, 2, 0, 0, 1]))


@pytest.mark.parametrize("dt", [F32, F16, BF16])
def test_reduce_pool_bn_parity(K, dt):
    x = rnd((2, 128, 768), 14, dt)
    tol = {F32: 1e-5, F16: 2e-3, BF16: 1.6e-2}[dt]
    close(K.reduce("mean", x, [-1], True, dt), oracle.reduce("mean", x, [-1], True, dt), tol, tol * 0.1)
    close(K.reduce("sum", x, [0, 2], False, dt), oracle.reduce("sum", x, [0, 2], False, dt), tol, tol)
    img = rnd((2, 8, 17, 19), 15, dt)
    close(K.pool2d("max", img, 3, 3, 1, 1, 1, 1, 2, 2, dt), oracle.pool2d("max", img, 3, 3, 1, 1, 1, 1, 2, 2, dt=dt), 0, 0)
    close(K.pool2d("avg", img, 3, 2, 1, 1, 1, 0, 2, 1, dt), oracle.pool2d("avg", img, 3, 2, 1, 1, 1, 0, 2, 1, dt=dt), tol, tol)
    m, v = rnd((8,), 16), np.abs(rnd((8,), 17)) + 0.5
    s, b = rnd((8,), 18), rnd((8,), 19)
    close(K.batch_norm(img, m, v, s, b, 1e-5, dt), oracle.batch_norm(img, m, v, s, b, 1e-5, dt), tol, tol)


@pytest.mark.parametrize("dt", [F32, F16, BF16])
def test_silu_mul_matches_two_kernels(K, dt):
    g, u = rnd((16, 11008), 50, dt, 2.0), rnd((16, 11008), 51, dt)
    fused = K.silu_mul(g, u, dt)
    two = K.binary("mul", K.unary("silu", g, dt), u, dt)
    assert np.array_equal(fused, two)  # same rounding points as Silu followed by Mul
    close(fused, oracle.binary("mul", oracle.unary("silu", g, dt), u, dt), 4 * EPS[dt], 1e-6)


def gemm_tol(dt, k, amax, bmax):
    """SURVEY 8(c): fp32 rel 1e-5*sqrt(K); 16-bit with fp32 accumulate: abs <= 2^-8 (bf16) / 2^-11 (fp16)
    * sqrt(K) * max|a| * max|b| against an fp32 oracle fed the same rounded inputs."""
    if dt == F32:
        return 1e-5 * np.sqrt(k) * amax * bmax
    return (2.0 ** -8 if dt == BF16 else 2.0 ** -11) * np.sqrt(k) * amax * bmax


@pytest.mark.parametrize("dt", [F32, F16, BF16])
@pytest.mark.parametrize("shape", [
    # (A shape, B shape, transA, transB, bias shape)
    ((512, 512), (512, 512), False, False, None),           # BASELINE config #1
    ((2, 3, 37, 53), (2, 3, 53, 29), False, False, None),   # batched, odd sizes -> SIMT path
    ((12, 128, 64), (12, 64, 128), False, False, None),     # GPT-2 q.k^T shape
    ((4, 70, 33), (33, 50), False, False, (50,)),           # batch-broadcast B + bias
    ((2, 40, 30), (2, 40, 20), True, False, None),          # transA
    ((5, 30, 40), (5, 20, 40), False, True, (5, 30, 20)),   # transB + full bias
])
def test_matmul_parity(K, shape, dt):
    sa, sb, tA, tB, sbias = shape
    a, b = rnd(sa, 20, dt), rnd(sb, 21, dt)
    bias = rnd(sbias, 22, dt) if sbias else None
    k = sa[-2] if tA else sa[-1]
    tol = gemm_tol(dt, k, np.abs(a).max(), np.abs(b).max())
    close(K.matmul(a, b, bias, tA, tB, dt), oracle.matmul(a, b, bias, tA, tB, dt), 2 * EPS[dt], tol)


SKINNY_SHAPES = [(16, 4096, 4096), (16, 4096, 11008), (16, 11008, 4096), (1, 256, 64), (7, 320, 200), (16, 4096, 32000),
                 (33, 1024, 1024), (64, 512, 4160), (16, 72, 64)]
TC_SHAPES = SKINNY_SHAPES + [(128, 768, 2304), (128, 3072, 768), (200, 512, 640), (256, 1024, 1024), (96, 64, 128)]


GEMM_IMPL = {"": 0, "skinny": 1, "tc": 2, "simt": 3}  # it_b200_matmul_select: "" = the production dispatch


@pytest.fixture
def gemm_impl(request):
    from infinitensor_b200 import _lib
    _lib.lib.it_b200_matmul_select(GEMM_IMPL[request.param], 0)
    yield request.param
    _lib.lib.it_b200_matmul_select(0, 0)


def _gemm_case(K, m, k, n, dt):
    a, b = rnd((m, k), 23, dt, 0.5), rnd((k, n), 24, dt, 0.05)
    tol = gemm_tol(dt, k, np.abs(a).max(), np.abs(b).max())
    got = K.matmul(a, b, None, False, False, dt)
    ref = oracle.matmul(a, b, None, False, False, dt)
    close(got, ref, 2 * EPS[dt], tol)
    bias = rnd((n,), 25, dt)
    close(K.matmul(a, b, bias, False, False, dt, act=1), np.maximum(oracle.matmul(a, b, bias, False, False, dt), 0),
          2 * EPS[dt], tol)


@pytest.mark.parametrize("gemm_impl", ["skinny"], indirect=True)
@pytest.mark.parametrize("dt", [BF16, F16])
@pytest.mark.parametrize("m,k,n", SKINNY_SHAPES)
def test_matmul_skinny_parity(K, gemm_impl, m, k, n, dt):
    """Decode-regime GEMM (TMA + mma.sync + cluster split-K) at the Llama-7B shapes of SURVEY 8a row a1."""
    _gemm_case(K, m, k, n, dt)


@pytest.mark.parametrize("gemm_impl", ["skinny"], indirect=True)
@pytest.mark.parametrize("dt", [BF16, F16])
def test_matmul_grouped_parity(K, gemm_impl, dt):
    """q/k/v- and gate/up-style grouped launches: several weight matrices sharing X in one kernel."""
    for m, k, ns in [(16, 4096, [4096, 4096, 4096]), (16, 1024, [2816, 2816]), (5, 512, [64, 128, 192, 256])]:
        x = rnd((m, k), 40, dt, 0.5)
        ws = [rnd((k, n), 41 + i, dt, 0.05) for i, n in enumerate(ns)]
        outs = K.matmul_grouped(x, ws, dt)
        for w, o in zip(ws, outs):
            close(o, oracle.matmul(x, w, None, False, False, dt), 2 * EPS[dt], gemm_tol(dt, k, np.abs(x).max(), np.abs(w).max()))


@pytest.mark.parametrize("dt", [BF16, F16])
def test_matmul_fused_epilogue_parity(K, dt):
    """MatMul + bias -> [Gelu] -> [+ residual] in the tcgen05 epilogue = the separate kernels (MatMul with bias, unary Gelu, binary
    Add), bit for bit -- the same fp32 sums and the same rounding points -- and the oracle chain within the GEMM tolerance."""
    from infinitensor_b200 import _lib
    for ci, (m, k, n) in enumerate([(128, 768, 768), (128, 768, 3072), (128, 3072, 768), (200, 3072, 776), (65, 64, 64)]):  # (third: split-K cluster)
        a, b = rnd((m, k), 420 + ci, dt, 0.5), rnd((k, n), 430 + ci, dt, 0.05)
        bias, res = rnd((n,), 440 + ci, dt, 0.5), rnd((m, n), 450 + ci, dt)
        tol = gemm_tol(dt, k, np.abs(a).max(), np.abs(b).max())
        _lib.lib.it_b200_matmul_select(GEMM_IMPL["tc"], 0)
        try:
            plain = K.matmul(a, b, bias, False, False, dt)
        finally:
            _lib.lib.it_b200_matmul_select(0, 0)
        for act, use_res in [(0, True), (4, False), (4, True), (1, True)]:
            got = K.matmul_fused(a, b, bias, res if use_res else None, act, dt)
            assert got is not None
            ref, ora = plain, oracle.matmul(a, b, bias, False, False, dt)
            if act == 4:
                ref, ora = K.unary("gelu", ref, dt), oracle.unary("gelu", ora, dt)
            if act == 1:
                ref, ora = np.maximum(ref, 0), np.maximum(ora, 0)
            if use_res:
                ref, ora = K.binary("add", ref, res, dt=dt), oracle.binary("add", ora, res, dt)
            assert np.array_equal(got, ref), f"case {ci} act={act} res={use_res}: max diff {np.abs(got - ref).max()}"
            close(got, ora, 4 * EPS[dt], 2 * tol)
    # decode rows (<= 64) and fp32 are not this kernel's: rc 2, the runtime runs the operators one by one
    a, b = rnd((16, 256), 460, dt), rnd((256, 256), 461, dt, 0.05)
    assert K.matmul_fused(a, b, None, rnd((16, 256), 462, dt), 0, dt) is not None  # (taken: the tcgen05 kernel has no row minimum)


@pytest.mark.parametrize("gemm_impl", ["", "tc"], indirect=True)
@pytest.mark.parametrize("dt", [BF16, F16])
def test_matmul_grouped_tcgen05_parity(K, gemm_impl, dt):
    """Grouped decode GEMMs whose 128-wide column tiles fill the machine (gate/up at the Llama-7B width: 2 x 86 tiles; ragged
    widths; 3 groups) run as ONE tcgen05 launch (tile index -> group); production dispatch and the pinned kernel agree with the oracle."""
    for m, k, ns in [(16, 4096, [11008, 11008]), (9, 320, [9600, 9608]), (33, 512, [6400, 6400, 6464])]:
        x = rnd((m, k), 340, dt, 0.5)
        ws = [rnd((k, n), 341 + i, dt, 0.05) for i, n in enumerate(ns)]
        outs = K.matmul_grouped(x, ws, dt)
        for w, o in zip(ws, outs):
            close(o, oracle.matmul(x, w, None, False, False, dt), 2 * EPS[dt], gemm_tol(dt, k, np.abs(x).max(), np.abs(w).max()))
    # logits-sized plain MatMul takes the same kernel by the dispatch rule (250 tiles)
    _gemm_case(K, 16, 1024, 32000, dt)


@pytest.mark.parametrize("gemm_impl", ["tc"], indirect=True)
@pytest.mark.parametrize("dt", [BF16, F16])
@pytest.mark.parametrize("m,k,n", TC_SHAPES)
def test_matmul_tcgen05_parity(K, gemm_impl, m, k, n, dt):
    """tcgen05 / TMEM / TMA swap-AB GEMM: decode shapes (M = 16) plus GPT-2 (M = 128) and M up to 256."""
    _gemm_case(K, m, k, n, dt)


@pytest.mark.parametrize("gemm_impl", ["tc"], indirect=True)
@pytest.mark.parametrize("dt", [BF16, F16])
@pytest.mark.parametrize("sa,sb", [((600, 256), (256, 384)),            # M > 256: row chunks of 256 on grid.z
                                   ((257, 72), (72, 200)),              # ragged last chunk, K and N not tile multiples
                                   ((12, 128, 64), (12, 64, 128)),      # GPT-2 q.k^T, batched on both sides
                                   ((12, 128, 128), (12, 128, 64)),     # GPT-2 p.v
                                   ((512, 576), (5, 576, 200)),         # conv form: broadcast filters x batched im2col
                                   ((3, 300, 64), (64, 96))])           # batched X, broadcast W
def test_matmul_tcgen05_batched_parity(K, gemm_impl, sa, sb, dt):
    """tcgen05 GEMM over grid.z = batch x 256-row chunks with 3-D tensor maps (conv im2col GEMMs, GPT-2 attention)."""
    a, b = rnd(sa, 28, dt, 0.5), rnd(sb, 29, dt, 0.1)
    tol = gemm_tol(dt, sa[-1], np.abs(a).max(), np.abs(b).max())
    close(K.matmul(a, b, None, False, False, dt), oracle.matmul(a, b, None, False, False, dt), 2 * EPS[dt], tol)
    bias = rnd((sb[-1],), 30, dt)
    close(K.matmul(a, b, bias, False, False, dt, act=1),
          np.maximum(oracle.matmul(a, b, bias, False, False, dt), 0), 2 * EPS[dt], tol)


@pytest.mark.parametrize("gemm_impl", ["tc"], indirect=True)
@pytest.mark.parametrize("dt", [BF16, F16])
@pytest.mark.parametrize("sa,sb", [((64, 2048), (1000, 2048)),      # ResNet-50 classifier (ONNX Gemm, transB = 1)
                                   ((128, 768), (2304, 768)), ((300, 72), (200, 72)), ((16, 4096), (4096, 4096))])
def test_matmul_tcgen05_transb_parity(K, gemm_impl, sa, sb, dt):
    """[N, K] weights (transB) feed the wgmma A operand K-major: one [128 x 64] box per stage, no transpose pass."""
    a, b = rnd(sa, 31, dt, 0.5), rnd(sb, 32, dt, 0.05)
    tol = gemm_tol(dt, sa[-1], np.abs(a).max(), np.abs(b).max())
    close(K.matmul(a, b, None, False, True, dt), oracle.matmul(a, b, None, False, True, dt), 2 * EPS[dt], tol)
    bias = rnd((sb[0],), 33, dt)
    close(K.matmul(a, b, bias, False, True, dt), oracle.matmul(a, b, bias, False, True, dt), 2 * EPS[dt], tol)


@pytest.mark.parametrize("dt", [F16, BF16])
def test_conv_resnet_shapes_parity(K, dt):
    """ResNet-50 bottleneck shapes (reduced batch): 1x1, 3x3 s1/s2, 7x7-stage P = 49, F up to 2048."""
    tol = {F16: 8e-3, BF16: 6e-2}[dt]
    for (xs, ws, args) in [((2, 64, 56, 56), (256, 64, 1, 1), (0, 0, 1, 1, 1, 1)),
                           ((2, 128, 28, 28), (128, 128, 3, 3), (1, 1, 1, 1, 1, 1)),
                           ((2, 256, 28, 28), (256, 256, 3, 3), (1, 1, 2, 2, 1, 1)),
                           ((2, 1024, 14, 14), (2048, 1024, 1, 1), (0, 0, 2, 2, 1, 1)),
                           ((2, 512, 7, 7), (512, 512, 3, 3), (1, 1, 1, 1, 1, 1)),
                           ((2, 2048, 7, 7), (512, 2048, 1, 1), (0, 0, 1, 1, 1, 1)),
                           ((2, 3, 64, 64), (64, 3, 7, 7), (3, 3, 2, 2, 1, 1))]:
        x, w = rnd(xs, 26, dt), rnd(ws, 27, dt, 0.05)
        close(K.conv2d(x, w, *args, dt=dt), oracle.conv2d(x, w, *args, dt=dt), tol, tol)


@pytest.mark.parametrize("dt", [F16, BF16])
def test_conv_fused_tail_bit_identical(K, dt):
    """Conv -> BatchNorm -> [+ residual] -> [ReLU] in the tcgen05 epilogue equals the separate kernels bit for bit, and the
    oracle chain within the conv tolerance; shapes off the tensor-core path answer rc 2 (nothing launched)."""
    tol = {F16: 2e-2, BF16: 1.5e-1}[dt]
    cases = [((2, 64, 56, 56), (256, 64, 1, 1), (0, 0, 1, 1, 1, 1)),      # batched 1x1, no repack
             ((2, 128, 28, 28), (128, 128, 3, 3), (1, 1, 1, 1, 1, 1)),   # folded im2col
             ((8, 256, 14, 14), (300, 256, 3, 3), (1, 1, 2, 2, 1, 1)),   # P = 49, F > 256 (two row chunks, ragged)
             ((8, 512, 7, 7), (128, 512, 1, 1), (0, 0, 1, 1, 1, 1)),     # 1x1 with P % 8 != 0 -> folded
             ((4, 3, 64, 64), (64, 3, 7, 7), (3, 3, 2, 2, 1, 1))]        # stem: K = 147 zero-padded to 152
    for ci, (xs, ws, args) in enumerate(cases):
        x, w = rnd(xs, 50 + ci, dt), rnd(ws, 60 + ci, dt, 0.05)
        F = ws[0]
        rng = np.random.default_rng(70 + ci)
        bn = (rng.standard_normal(F).astype(np.float32) * 0.1, rng.uniform(0.5, 1.5, F).astype(np.float32),
              rng.uniform(0.5, 1.5, F).astype(np.float32), rng.standard_normal(F).astype(np.float32) * 0.1)
        conv = K.conv2d(x, w, *args, dt=dt)
        res = rnd(conv.shape, 80 + ci, dt)
        for use_res, relu in [(False, False), (False, True), (True, True)]:
            got = K.conv2d_fused(x, w, *args, bn, 1e-5, res if use_res else None, relu, dt=dt)
            assert got is not None
            ref = K.batch_norm(conv, *bn, 1e-5, dt=dt)
            ora = oracle.batch_norm(oracle.conv2d(x, w, *args, dt=dt), *bn, 1e-5, dt)
            if use_res:
                ref = K.binary("add", ref, res, dt=dt)
                ora = oracle.binary("add", ora, res, dt)
            if relu:
                ref = np.maximum(ref, 0)
                ora = None if ora is None else np.maximum(ora, 0)
            assert np.array_equal(got, ref), f"case {ci} res={use_res} relu={relu}: max diff {np.abs(got - ref).max()}"
            if ci in (1, 2, 4) and K.L.lib.it_b200_conv2d_nchw_to_nhwc_supported(dt, *xs, ws[0], ws[2], ws[3], *args, 1):
                # the same GEMM scattering its result as NHWC (entry into the NHWC domain): identical values
                nh = K.conv2d_fused(x, w, *args, bn, 1e-5, res if use_res else None, relu, dt=dt, y_nhwc=True)
                assert nh is not None and np.array_equal(nh, ref)
            if ora is not None:
                close(got, ora, tol, tol)
    # fp32 / grouped / tiny-K convs are not taken: rc 2, the runtime runs the operators one by one
    x, w = rnd((1, 8, 9, 9), 90, dt), rnd((8, 2, 3, 3), 91, dt, 0.2)  # groups = 4
    z = np.zeros(8, np.float32)
    assert K.conv2d_fused(x, w, 1, 1, 2, 2, 1, 1, (z, z + 1, z + 1, z), 1e-5, None, True, dt=dt) is None
    x = rnd((2, 16, 8, 8), 92, dt)
    close(K.batch_norm_relu(x, *[np.full(16, v, np.float32) for v in (0.1, 1.3, 0.9, -0.2)], 1e-5, dt=dt),
          np.maximum(K.batch_norm(x, *[np.full(16, v, np.float32) for v in (0.1, 1.3, 0.9, -0.2)], 1e-5, dt=dt), 0), 0, 0)


@pytest.mark.parametrize("dt", [F16, BF16])
def test_pool_nhwc_parity(K, dt):
    """NHWC pooling = the NCHW kernel on the permuted tensor, bit for bit (same fp32 arithmetic)."""
    img = rnd((3, 24, 13, 11), 301, dt)
    for kind, args in [("max", (3, 3, 1, 1, 1, 1, 2, 2)), ("avg", (3, 3, 1, 1, 1, 1, 2, 1)), ("avg", (3, 2, 1, 1, 1, 0, 2, 1)),
                       ("max", (2, 2, 2, 1, 0, 1, 1, 2))]:
        assert np.array_equal(K.pool2d_nhwc(kind, img, *args, dt=dt), K.pool2d(kind, img, *args, dt))
    # global average pool: its own kernel (pixel groups reduced through shared memory -> another fp32 summation order)
    big = rnd((5, 264, 7, 7), 302, dt)
    close(K.pool2d_nhwc("avg", big, 7, 7, 1, 1, 0, 0, 1, 1, dt=dt), K.pool2d("avg", big, 7, 7, 1, 1, 0, 0, 1, 1, dt), 2 * EPS[dt], 1e-6)
    close(K.pool2d_nhwc("avg", img, 13, 11, 1, 1, 0, 0, 1, 1, dt=dt), K.pool2d("avg", img, 13, 11, 1, 1, 0, 0, 1, 1, dt), 2 * EPS[dt], 1e-6)


NHWC_CASES = [((2, 64, 56, 56), (256, 64, 1, 1), (0, 0, 1, 1, 1, 1)),      # 1x1, one k-tile, filters used as stored
              ((2, 128, 28, 28), (128, 128, 3, 3), (1, 1, 1, 1, 1, 1)),   # 3x3 s1 p1
              ((3, 256, 28, 28), (256, 256, 3, 3), (1, 1, 2, 2, 1, 1)),   # 3x3 s2 p1
              ((2, 1024, 14, 14), (2048, 1024, 1, 1), (0, 0, 2, 2, 1, 1)),  # 1x1 s2 downsample, 8 filter tiles
              ((5, 512, 7, 7), (512, 512, 3, 3), (1, 1, 1, 1, 1, 1)),     # P = 49: pixel tiles straddle images, ragged last tile
              ((2, 2048, 7, 7), (512, 2048, 1, 1), (0, 0, 1, 1, 1, 1)),
              ((3, 24, 19, 13), (40, 24, 3, 5), (1, 2, 2, 1, 1, 1)),      # ragged everything: C < 64, F < 64, asymmetric taps / pads / strides
              ((2, 72, 11, 9), (304, 72, 3, 3), (2, 1, 1, 2, 2, 1)),      # C = 64 + 8, F = 256 + 48, dilation 2 along h
              ((1, 8, 6, 6), (8, 8, 1, 1), (0, 0, 1, 1, 1, 1))]


@pytest.mark.parametrize("dt", [F16, BF16])
def test_conv_nhwc_parity(K, dt):
    """Implicit-GEMM conv over NHWC activations (TMA im2col mode -> tcgen05) against the oracle's direct convolution."""
    tol = {F16: 8e-3, BF16: 6e-2}[dt]
    for ci, (xs, ws, args) in enumerate(NHWC_CASES):
        x, w = rnd(xs, 126 + ci, dt), rnd(ws, 127 + ci, dt, 0.05)
        want = oracle.conv2d(x, w, *args, dt=dt)
        for y_nhwc in (True, False):
            got = K.conv2d_nhwc(x, w, *args, dt=dt, y_nhwc=y_nhwc)
            assert got.shape == want.shape
            close(got, want, tol, tol)


@pytest.mark.parametrize("dt", [F16, BF16])
def test_conv_stem_parity(K, dt):
    """The stem kernel (NCHW input with <= 4 channels -> NHWC, mma.sync fragments built from a shared-memory patch) against the
    oracle: the ResNet stem, ragged image sizes (blocks cut by the border), 1..4 channels, small filters, stride 1, F < 64."""
    tol = {F16: 8e-3, BF16: 6e-2}[dt]
    for ci, (xs, ws, args) in enumerate([((2, 3, 64, 64), (64, 3, 7, 7), (3, 3, 2, 2)),
                                         ((3, 3, 45, 37), (64, 3, 7, 7), (3, 3, 2, 2)),
                                         ((2, 4, 19, 23), (24, 4, 3, 3), (1, 1, 1, 1)),
                                         ((2, 1, 30, 17), (8, 1, 5, 8), (2, 0, 1, 2)),
                                         ((1, 2, 33, 33), (40, 2, 1, 1), (0, 0, 2, 1))]):
        x, w = rnd(xs, 226 + ci, dt), rnd(ws, 227 + ci, dt, 0.1)
        ph, pw, sh, sw = args
        want = oracle.conv2d(x, w, ph, pw, sh, sw, 1, 1, dt=dt)
        close(K.conv2d_stem(x, w, *args, dt=dt), want, tol, tol)
        F = ws[0]
        rng = np.random.default_rng(240 + ci)
        bn = (rng.standard_normal(F).astype(np.float32) * 0.1, rng.uniform(0.5, 1.5, F).astype(np.float32),
              rng.uniform(0.5, 1.5, F).astype(np.float32), rng.standard_normal(F).astype(np.float32) * 0.1)
        ora = np.maximum(oracle.batch_norm(want, *bn, 1e-5, dt), 0)
        close(K.conv2d_stem(x, w, *args, bn=bn, relu=True, dt=dt), ora, 2.5 * tol, 2.5 * tol)


@pytest.mark.parametrize("dt", [F16, BF16])
def test_conv_nhwc_fused_tail(K, dt):
    """Conv -> BatchNorm -> [+ residual] -> [ReLU] in the implicit-GEMM epilogue (fp32, one rounding) against the oracle chain
    (which rounds after every operator, like the reference's separate kernels)."""
    tol = {F16: 2e-2, BF16: 1.5e-1}[dt]
    for ci, (xs, ws, args) in enumerate(NHWC_CASES[:5] + NHWC_CASES[6:8]):
        x, w = rnd(xs, 150 + ci, dt), rnd(ws, 160 + ci, dt, 0.05)
        F = ws[0]
        rng = np.random.default_rng(170 + ci)
        bn = (rng.standard_normal(F).astype(np.float32) * 0.1, rng.uniform(0.5, 1.5, F).astype(np.float32),
              rng.uniform(0.5, 1.5, F).astype(np.float32), rng.standard_normal(F).astype(np.float32) * 0.1)
        conv = oracle.conv2d(x, w, *args, dt=dt)
        res = rnd(conv.shape, 180 + ci, dt)
        for use_res, relu, y_nhwc in [(False, False, True), (False, True, True), (True, True, True), (True, True, False)]:
            ora = oracle.batch_norm(conv, *bn, 1e-5, dt)
            if use_res:
                ora = oracle.binary("add", ora, res, dt)
            if relu:
                ora = np.maximum(ora, 0)
            got = K.conv2d_nhwc(x, w, *args, bn=bn, eps=1e-5, residual=res if use_res else None, relu=relu, dt=dt, y_nhwc=y_nhwc)
            close(got, ora, tol, tol)


@pytest.mark.parametrize("dt", [F32, F16, BF16])
def test_conv_parity(K, dt):
    tol = {F32: 1e-4, F16: 4e-3, BF16: 3e-2}[dt]
    for (xs, ws, args) in [((2, 16, 14, 14), (32, 16, 3, 3), (1, 1, 1, 1, 1, 1)),
                           ((2, 3, 32, 32), (8, 3, 7, 7), (3, 3, 2, 2, 1, 1)),
                           ((2, 64, 8, 8), (128, 64, 1, 1), (0, 0, 1, 1, 1, 1)),
                           ((1, 8, 9, 9), (8, 2, 3, 3), (1, 1, 2, 2, 1, 1))]:  # groups = 4
        x, w = rnd(xs, 26, dt), rnd(ws, 27, dt, 0.2)
        close(K.conv2d(x, w, *args, dt=dt), oracle.conv2d(x, w, *args, dt=dt), tol, tol)


@pytest.mark.parametrize("dt", [F32, F16, BF16])
@pytest.mark.parametrize("B,H,S,pos", [(2, 4, 64, 0), (2, 4, 64, 37), (16, 32, 1024, 511), (1, 2, 1024, 1023),
                                       (1, 32, 256, 100), (7, 9, 512, 257), (1, 1, 2048, 2047), (3, 40, 128, 64)])
def test_attention_parity(K, B, H, S, pos, dt):
    kc, vc = rnd((B, H, S, 128), 28, dt, 0.5), rnd((B, H, S, 128), 29, dt, 0.5)
    q, k, v = rnd((B, H, 1, 128), 30, dt, 0.5), rnd((B, H, 1, 128), 31, dt, 0.5), rnd((B, H, 1, 128), 32, dt, 0.5)
    kc_ref, vc_ref = kc.copy(), vc.copy()
    ref = oracle.attention_kvcache(kc_ref, vc_ref, q, k, v, pos, dt)
    out, kc_got, vc_got = K.attention_kvcache(kc, vc, q, k, v, pos, dt)
    tol = {F32: 1e-5, F16: 1e-3, BF16: 1e-2}[dt]  # SURVEY 8(c)
    close(out, ref, tol, tol * 0.05)
    assert np.array_equal(kc_got, kc_ref) and np.array_equal(vc_got, vc_ref)  # append is bit-exact, rest untouched


@pytest.mark.parametrize("dt", [F32, BF16])
@pytest.mark.parametrize("B,H,S,poss", [(4, 4, 256, [0, 37, 255, 64]), (16, 32, 1024, None), (3, 5, 128, [127, 0, 63]),
                                        (5, 2, 512, [200, 200, 1, 511, 300])])
def test_attention_per_row_positions(K, B, H, S, poss, dt):
    """SURVEY 8(f-3): ragged batches.  ITB_POS_PER_ROW: row b attends to position_id[b] + 1 rows and appends at
    position_id[b]; the oracle is the reference kernel's arithmetic (attention_kvcache.cu:8-145) applied row by row with that
    row's position.  ITB_POS_IN_STEP (no read ahead of griddepcontrol.wait) must not change a bit."""
    if poss is None:
        poss = np.random.default_rng(5).integers(0, S, size=B).tolist()
    kc, vc = rnd((B, H, S, 128), 28, dt, 0.5), rnd((B, H, S, 128), 29, dt, 0.5)
    q, k, v = rnd((B, H, 1, 128), 30, dt, 0.5), rnd((B, H, 1, 128), 31, dt, 0.5), rnd((B, H, 1, 128), 32, dt, 0.5)
    kc_ref, vc_ref = kc.copy(), vc.copy()
    ref = np.concatenate([oracle.attention_kvcache(kc_ref[b:b + 1], vc_ref[b:b + 1], q[b:b + 1], k[b:b + 1], v[b:b + 1],
                                                   int(poss[b]), dt) for b in range(B)])
    out, kc_got, vc_got = K.attention_kvcache(kc, vc, q, k, v, poss, dt)
    tol = {F32: 1e-5, F16: 1e-3, BF16: 1e-2}[dt]
    close(out, ref, tol, tol * 0.05)
    assert np.array_equal(kc_got, kc_ref) and np.array_equal(vc_got, vc_ref)
    out2, kc2, vc2 = K.attention_kvcache(kc, vc, q, k, v, poss, dt, flags=0x200)
    assert np.array_equal(out2, out) and np.array_equal(kc2, kc_got) and np.array_equal(vc2, vc_got)


@pytest.mark.parametrize("mode", ["DCR", "CRD"])
@pytest.mark.parametrize("dt", [F32, F16])
def test_depth_to_space_graph(mode, dt):
    """DepthToSpace through the graph API (registered kernel = the rank-6 permute of reference transpose.cc:48-90), bit-exact
    against the ONNX definition evaluated by the oracle handler."""
    from infinitensor_b200 import backend as B, graphs as GR
    from oracle.graph_oracle import OracleHandler
    x = np.random.default_rng(3).standard_normal((2, 16, 5, 7)).astype(np.float32)
    outs = []
    for h in (B.GraphHandler(B.CudaRuntime(0)), OracleHandler()):
        t = h.tensor([2, 16, 5, 7], dt)
        t.set_input()
        y = h.depthToSpace(t, None, 2, mode)
        y.set_output()
        h.data_malloc()
        t.copyin_numpy(GR.to_storage(x, dt))
        h.run()
        outs.append(np.asarray(y.f32()) if hasattr(y, "f32") else GR.from_storage(y.copyout_numpy(), dt))
    assert outs[0].shape == (2, 4, 10, 14)
    assert np.array_equal(outs[0].astype(np.float32), outs[1].reshape(outs[0].shape).astype(np.float32))


@pytest.mark.parametrize("dt", [F16, BF16])
@pytest.mark.parametrize("B,H,Sq,Skv,D,masked,div", [(1, 12, 128, 128, 64, True, True), (2, 3, 16, 16, 64, True, True),
                                                      (1, 2, 200, 200, 128, True, False), (2, 2, 96, 300, 64, False, True),
                                                      (1, 4, 257, 129, 128, True, True), (1, 1, 128, 128, 64, False, False)])
def test_attention_prefill_parity(K, B, H, Sq, Skv, D, masked, div, dt):
    """SURVEY 8(f-3): the fused tcgen05 prefill attention against the oracle executing the operator chain it replaces --
    MatMul(q, k^T) -> Div|Mul(scale) -> Add(mask) -> Softmax(-1) -> MatMul(., v), every intermediate rounded to the storage
    type (config C2's attention block: [1,12,128,64] heads, causal additive mask, scale sqrt(64))."""
    import torch
    from infinitensor_b200 import _lib as L
    q, k, v = rnd((B, H, Sq, D), 50, dt, 0.7), rnd((B, H, Skv, D), 51, dt, 0.7), rnd((B, H, Skv, D), 52, dt, 0.7)
    scale = oracle.round_to(np.array([np.sqrt(D) if div else 1.0 / np.sqrt(D)], np.float32), dt)
    big_neg = -65504.0 if dt == F16 else -3.0e38
    mask = None
    if masked:
        mask = oracle.round_to(np.triu(np.full((Sq, Skv), big_neg, np.float32), 1 + max(0, Skv - Sq)).reshape(1, 1, Sq, Skv), dt)
    s = oracle.matmul(q, np.ascontiguousarray(k.transpose(0, 1, 3, 2)), None, False, False, dt)
    s = oracle.binary("div" if div else "mul", s, scale, dt)
    if masked:
        s = oracle.binary("add", s, mask, dt)
    p = oracle.softmax(s, -1, dt)
    ref = oracle.matmul(p, v, None, False, False, dt)
    qd, kd, vd, sd = K.dev(q, dt), K.dev(k, dt), K.dev(v, dt), K.dev(scale, dt)
    md = K.dev(mask, dt) if masked else None
    out = torch.zeros((B, H, Sq, D), dtype=K.TORCH_DT[dt], device="cuda")
    L.check(L.lib.it_b200_attention_prefill(dt, K.ptr(qd), K.ptr(kd), K.ptr(vd), K.ptr(out), B, H, Sq, Skv, D, K.ptr(sd), int(div),
                                            K.ptr(md), 0, 0, Skv if masked else 0, 1 if masked else 0, K.stream()))
    K.sync()
    got = K.host(out)
    tol = {F16: 2e-3, BF16: 1.6e-2}[dt]  # attention tolerance of SURVEY 8(c): 1e-3 (fp16) / 1e-2 (bf16) relative, P rounded once more
    assert np.abs(got - ref).max() <= tol * max(np.abs(ref).max(), 1e-3), np.abs(got - ref).max() / np.abs(ref).max()


@pytest.mark.parametrize("dt", [F16, BF16])
@pytest.mark.parametrize("B,H,S,D", [(1, 12, 128, 64), (2, 3, 200, 64), (2, 2, 72, 128)])
def test_attention_prefill_strided_views(K, B, H, S, D, dt):
    """q / k / v as strided views of a fused projection output [B, S, 3 H D] and the result written as [B, S, H D] (what the
    schedule's extended PrefillAttention step passes) = the dense kernel on the materialised [B, H, S, D] copies, bit for bit."""
    import torch
    from infinitensor_b200 import _lib as L
    d = H * D
    qkv = rnd((B, S, 3 * d), 520, dt, 0.7)
    parts = [np.ascontiguousarray(qkv[:, :, i * d:(i + 1) * d].reshape(B, S, H, D).transpose(0, 2, 1, 3)) for i in range(3)]
    scale = oracle.round_to(np.array([np.sqrt(D)], np.float32), dt)
    big_neg = -65504.0 if dt == F16 else -3.0e38
    mask = oracle.round_to(np.triu(np.full((S, S), big_neg, np.float32), 1).reshape(1, 1, S, S), dt)
    sd, md = K.dev(scale, dt), K.dev(mask, dt)
    qd, kd, vd = [K.dev(t, dt) for t in parts]
    dense = torch.zeros((B, H, S, D), dtype=K.TORCH_DT[dt], device="cuda")
    L.check(L.lib.it_b200_attention_prefill(dt, K.ptr(qd), K.ptr(kd), K.ptr(vd), K.ptr(dense), B, H, S, S, D, K.ptr(sd), 1, K.ptr(md), 0, 0, S,
                                            1, K.stream()))
    xd = K.dev(qkv, dt)
    out = torch.zeros((B, S, d), dtype=K.TORCH_DT[dt], device="cuda")
    es = xd.element_size()
    view = L.i64arr([S * 3 * d, D, 3 * d])
    ost = L.i64arr([S * d, D, d])
    import ctypes
    base = xd.data_ptr()
    L.check(L.lib.it_b200_attention_prefill_strided(dt, ctypes.c_void_p(base), ctypes.c_void_p(base + d * es), ctypes.c_void_p(base + 2 * d * es),
                                                    K.ptr(out), B, H, S, S, D, view, view, view, ost, K.ptr(sd), 1, K.ptr(md), 0, 0, S, 1,
                                                    K.stream()))
    K.sync()
    want = K.host(dense).transpose(0, 2, 1, 3).reshape(B, S, d)
    assert np.array_equal(K.host(out), want)


@pytest.mark.parametrize("dt", [F32, F16, BF16])
def test_leaky_relu_elu_parity(K, dt):
    """LeakyRelu / Elu (reference unary.cu:97-106, 157-165; golden cases of test_cuda_unary.cc: alpha 0.1 / 1.0)."""
    import torch
    from infinitensor_b200 import _lib as L
    x = rnd((3, 1000), 70, dt, 2.0)
    xd = K.dev(x, dt)
    for op, name, alpha in ((12, "leakyrelu", 0.1), (13, "elu", 1.0), (13, "elu", 0.5)):
        y = torch.empty_like(xd)
        L.check(L.lib.it_b200_unary_alpha(op, dt, K.ptr(xd), K.ptr(y), xd.numel(), alpha, K.stream()))
        K.sync()
        ref = oracle.unary_alpha(name, x, alpha, dt)
        close(K.host(y), ref, 4 * EPS[dt] if dt != F32 else 2e-6, 1e-6)


def test_rope_partial_head_golden(K):
    """the reference's RoPE known-answer test as written: dim_model = 32 under 128-wide heads (test_cuda_rope.cc:17-35)."""
    x = np.ones((1, 1, 32), np.float32)
    out = K.rope(np.array([[1]]), x, pos_np_dtype=np.uint32)
    close(out[0, 0], G.ROPE_COS, 2e-6, 1e-6)


@pytest.mark.parametrize("dt", [BF16, F16])
@pytest.mark.parametrize("m,k,ns,res", [(16, 4096, [4096], False), (16, 4096, [4096, 4096, 4096], False), (16, 4096, [11008, 11008], False),
                                        (16, 11008, [4096], True), (16, 4096, [32000], False), (5, 512, [64, 128], False),
                                        (33, 1024, [256], True)])
def test_matmul_fp8_weights_parity(K, m, k, ns, res, dt):
    """SURVEY 8(f-4): weight-only FP8 E4M3 with the dequantisation inside the GEMM (codes -> activation type in the main loop,
    per-column scale on the fp32 sum in the epilogue), 1..3 matrices sharing X; against the fp32 oracle fed the DEQUANTISED
    weights.  Tolerance: the GEMM bound of SURVEY 8(c) on the dequantised operands."""
    import ctypes, torch
    from infinitensor_b200 import _lib as L
    x = rnd((m, k), 80, dt, 0.5)
    qs = [oracle.quantize_weight_fp8(np.random.default_rng(81 + i).standard_normal((k, n)).astype(np.float32) * 0.05) for i, n in enumerate(ns)]
    resid = rnd((m, ns[0]), 90, dt, 1.0) if res else None
    xd = K.dev(x, dt)
    cd = [K.raw(c) for c, _ in qs]
    sd = [K.raw(s) for _, s in qs]
    od = [torch.zeros((m, n), dtype=K.TORCH_DT[dt], device="cuda") for n in ns]
    rd = K.dev(resid, dt) if res else None
    VP = ctypes.c_void_p
    arr = lambda ts: (VP * len(ts))(*[t.data_ptr() for t in ts])
    L.check(L.lib.it_b200_matmul_fp8w(dt, K.ptr(xd), len(ns), arr(cd), arr(sd), arr(od), L.i32arr(ns), m, k, K.ptr(rd), K.stream()))
    K.sync()
    for (codes, scale), o in zip(qs, od):
        ref = oracle.matmul_fp8w(x, codes, scale, dt)
        if res:
            ref = oracle.binary("add", resid, ref, dt)
        wmax = np.abs(oracle.e4m3_decode(codes)).max() * scale.max()
        close(K.host(o), ref, 2 * EPS[dt], gemm_tol(dt, k, np.abs(x).max(), wmax))
    # the stand-alone DequantizeLinear kernel: bit-exact against the oracle
    y = torch.zeros((k, ns[0]), dtype=K.TORCH_DT[dt], device="cuda")
    L.check(L.lib.it_b200_dequantize_fp8(dt, K.ptr(cd[0]), K.ptr(sd[0]), K.ptr(y), k, ns[0], K.stream()))
    K.sync()
    assert np.array_equal(K.host(y), oracle.dequantize_fp8(qs[0][0], qs[0][1], dt))


def test_error_reporting(K):
    import torch
    from infinitensor_b200 import _lib as L
    x = torch.zeros(8, device="cuda")
    assert L.lib.it_b200_unary(99, 1, K.ptr(x), K.ptr(x), 8, K.stream()) != 0
    assert "bad op" in L.last_error()
    with pytest.raises(L.B200BackendError):
        L.check(L.lib.it_b200_attention_kvcache(1, K.ptr(x), K.ptr(x), K.ptr(x), K.ptr(x), K.ptr(x), K.ptr(x), 7,
                                                K.ptr(x), 1, 1, 1, 64, None, 0, K.stream()))
