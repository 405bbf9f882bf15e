"""4-bit MatMulNBits on the GPU: it_b200_matmul_nbits against the float64 oracle of tests/w4_oracle.py (per element, with its
bound), in NaN-poisoned guarded outputs and run twice bit for bit; the kernel's name in a profile; and int4 Llama graphs against
the graph oracle (tests/llama_oracle.py)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import oracle
from tests import llama_oracle as L
from tests import ref64
from tests import w4_oracle as W

F16, BF16 = 10, 16
GUARD = 64  # elements of NaN on each side of every output


@pytest.fixture(scope="module")
def K():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from tests import kernel_harness
    return kernel_harness


def make_matrix(K_, N, bs, dt, zp, seed):
    """random codes / scales / zero points of one [K, N] weight; column scales vary by 2^((n mod 5) - 2) so a column mix-up shows"""
    rng = np.random.default_rng(seed)
    nblk = K_ // bs
    q = rng.integers(0, 16, size=(N, K_), dtype=np.uint8)
    s = (rng.uniform(0.5, 1.5, size=(N, nblk)) * 0.01 * ref64.col_scale(N)[:, None]).astype(np.float32)
    s = oracle.round_to(s, dt).reshape(-1)
    z = W.pack_zero_points(rng.integers(0, 16, size=(N, nblk), dtype=np.uint8)) if zp else None
    return W.pack_codes(q).reshape(N, nblk, bs // 2), s, z


def nan_bits(dt):
    return np.uint16(0x7FFF) if dt == BF16 else np.uint16(0x7E00)


def launch(K, x, mats, k, bs, dt, residual=None):
    """one it_b200_matmul_nbits call; returns the outputs (float32) after checking the guards.  mats: [(B, scales, zp, N)]"""
    import ctypes
    import torch
    L = K.L
    m = x.shape[0]
    xd = K.dev(x, dt)
    keep, Wp, Sp, Zp, Cp, outs = [], [], [], [], [], []
    Ns = [N for *_, N in mats]
    for b, s, z, N in mats:
        bd, sd = K.raw(b), K.dev(s, dt)
        zd = K.raw(z) if z is not None else None
        buf = torch.from_numpy(np.full(m * N + 2 * GUARD, nan_bits(dt), np.uint16)).cuda()
        keep += [bd, sd, zd, buf]
        Wp.append(bd.data_ptr())
        Sp.append(sd.data_ptr())
        Zp.append(zd.data_ptr() if zd is not None else 0)
        Cp.append(buf.data_ptr() + 2 * GUARD)
        outs.append(buf)
    VP = ctypes.c_void_p
    arr = lambda v: (VP * len(v))(*v)
    rd = K.dev(residual, dt) if residual is not None else None
    n_arr = L.i32arr(Ns)
    wsb = int(L.lib.it_b200_matmul_nbits_workspace(dt, m, k, len(mats), n_arr))
    ws = torch.empty(max(wsb, 16), dtype=torch.uint8, device="cuda")
    zarr = arr(Zp) if mats[0][2] is not None else None
    L.check(L.lib.it_b200_matmul_nbits(dt, K.ptr(xd), len(mats), arr(Wp), arr(Sp), zarr, arr(Cp), n_arr, m, k, bs, K.ptr(rd),
                                       K.ptr(ws), wsb, K.stream()))
    K.sync()
    res = []
    for buf, N in zip(outs, Ns):
        h = buf.cpu().numpy()
        assert (h[:GUARD] == nan_bits(dt)).all() and (h[GUARD + m * N:] == nan_bits(dt)).all(), "write outside the output"
        t = torch.from_numpy(h[GUARD:GUARD + m * N].copy()).view(torch.bfloat16 if dt == BF16 else torch.float16)
        res.append(t.float().numpy().reshape(m, N))
    return res


def check(K, m, k, Ns, bs, zp, dt, res=False, seed=0):
    x = ref64.activations(m, k, dt, seed)
    mats = [make_matrix(k, N, bs, dt, zp, seed + 1 + i) + (N,) for i, N in enumerate(Ns)]
    r = ref64.activations(m, Ns[0], dt, seed + 9, scale=1.0) if res else None
    got = launch(K, x, mats, k, bs, dt, r)
    again = launch(K, x, mats, k, bs, dt, r)
    for i, (b, s, z, N) in enumerate(mats):
        assert np.array_equal(got[i].view(np.uint32), again[i].view(np.uint32)), "two runs differ"
        ref, bound = W.reference(x, b, s, z, k, N, bs, dt, rounded_weights=m > 64)
        if r is not None:  # the product rounded to T, then the residual added and rounded again
            ref = oracle.round_to(ref.astype(np.float32), dt).astype(np.float64) + r
            bound = bound + ref64.ulp(ref, dt)
        bad = W.violations(got[i], ref, bound)
        assert not bad.any(), (f"matrix {i}: {bad.sum()} of {bad.size} outside the bound; first {np.argwhere(bad)[0]}, "
                               f"worst {(np.abs(got[i] - ref) / bound).max():.3g}x")


# row-tile widths: every M the three 16-row tilings take, rotating dtype, block size and zero points
ROWS = [(m, (F16, BF16)[i % 2], (32, 64, 128)[i % 3], i % 2 == 1) for i, m in enumerate([1, 2, 8, 15, 16, 17, 32, 48, 64])]


@pytest.mark.parametrize("m,dt,bs,zp", ROWS)
def test_w4_rows(K, m, dt, bs, zp):
    check(K, m, 4096, [1024], bs, zp, dt)


@pytest.mark.parametrize("dt", [F16, BF16])
@pytest.mark.parametrize("bs", [32, 64, 128])
@pytest.mark.parametrize("zp", [False, True])
def test_w4_block_sizes(K, dt, bs, zp):
    check(K, 16, 4096, [4096], bs, zp, dt)  # 64 column tiles: the launcher splits K over a cluster


@pytest.mark.parametrize("k", [4096, 11008, 14336])
@pytest.mark.parametrize("dt", [F16, BF16])
def test_w4_k_splits(K, k, dt):
    check(K, 16, k, [4096], 128, False, dt, res=True)  # o / down: split-K, the residual epilogue


@pytest.mark.parametrize("Ns", [[4096, 1024, 1024], [11008, 11008], [1040, 512, 2048, 4096]])
@pytest.mark.parametrize("zp", [False, True])
def test_w4_groups(K, Ns, zp):
    check(K, 16, 4096, Ns, 128, zp, BF16)


@pytest.mark.parametrize("m", [1, 16])
def test_w4_logits_and_ragged_columns(K, m):
    check(K, m, 4096, [32000], 128, False, BF16)
    check(K, m, 2048, [1040], 64, True, F16)  # N not a multiple of 64


@pytest.mark.parametrize("m", [65, 200])
@pytest.mark.parametrize("dt", [F16, BF16])
def test_w4_many_rows_dequantised(K, m, dt):
    check(K, m, 2048, [1024, 512], 64, dt == F16, dt)
    check(K, m, 2048, [1024], 128, False, dt, res=True)


def test_w4_dequantize(K):
    """the stand-alone dequantiser: T((q - z) * s), the product in fp32 and rounded once"""
    import torch
    k, n, bs = 1024, 512, 64
    for dt in (F16, BF16):
        for zp in (False, True):
            b, s, z, = make_matrix(k, n, bs, dt, zp, 3)
            bd, sd = K.raw(b), K.dev(s, dt)
            zd = K.raw(z) if z is not None else None
            out = torch.empty((k, n), dtype=K.TORCH_DT[dt], device="cuda")
            K.L.check(K.L.lib.it_b200_dequantize_w4(dt, K.ptr(bd), K.ptr(sd), K.ptr(zd), K.ptr(out), k, n, bs, K.stream()))
            K.sync()
            want = oracle.round_to(W.dequantize(b, s, z, k, n, bs).astype(np.float32), dt)
            assert np.array_equal(K.host(out), want)


def profiled_kernel_names():
    import torch
    from tests import kernel_harness as K
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        check(K, 16, 4096, [1024], 128, False, BF16)
        torch.cuda.synchronize()
    return sorted({e.name for e in prof.events() if "CUDA" in str(e.device_type)})


def test_w4_kernel_names_in_profile(K):
    """in a child process, as the other profiler checks"""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = "import json; from tests.test_gpu_w4 import profiled_kernel_names as f; print(json.dumps(f()))"
    r = subprocess.run([sys.executable, "-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    names = json.loads(r.stdout.strip().splitlines()[-1])
    if not names:
        pytest.skip("the profiler recorded no CUDA kernel events (CUPTI activity tracing unavailable)")
    assert any("gemm_skinny_w4_kernel" in n for n in names), names


# ---------------------------------------------------------------------------------------------------- whole graphs
def run_graph(cfg, pos=5, steps=3, cudagraph=True, fused=True):
    """The device graph with int4 weights against the graph oracle (tests/llama_oracle.py); fused=False plans the unfused
    schedule (ITB_FUSION_MASK=0).  Returns the schedule."""
    return L.run_llama_parity(cfg, pos, steps, cudagraph, env=None if fused else {"ITB_FUSION_MASK": "0"}, tol=3e-2)[2]


@pytest.mark.parametrize("cudagraph", [False, True])
@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("bs", [32, 128])
def test_w4_llama_tiny(K, cudagraph, fused, bs):
    from infinitensor_b200 import graphs as G
    cfg = G.LlamaConfig.tiny()
    cfg.int4_block, cfg.vocab = bs, 1024  # (MatMulNBits takes N % 16 == 0)
    sched = run_graph(cfg, cudagraph=cudagraph, fused=fused)
    assert ("MatMulGroup" in str(sched)) == fused


@pytest.mark.parametrize("cudagraph", [False, True])
def test_w4_llama_tinyllama_width(K, cudagraph):
    from infinitensor_b200 import graphs as G
    run_graph(G.LlamaConfig.tinyllama_1b(batch=4, s_max=512, layers=2, int4_block=64), pos=300, cudagraph=cudagraph)


def test_w4_llama7b_width_two_layers(K):
    from infinitensor_b200 import graphs as G
    cfg = G.LlamaConfig(layers=2, batch=16, s_max=512, int4_block=128)
    cfg.vocab = 4096  # keeps the oracle's logits GEMM small
    run_graph(cfg, pos=200, steps=2)


@pytest.mark.parametrize("cudagraph", [False, True])
@pytest.mark.parametrize("shape", ["tiny", "tinyllama_width"])
def test_w4_llama_kv_fp8(K, shape, cudagraph):
    """int4 weights with an FP8 KV cache"""
    from infinitensor_b200 import graphs as G
    if shape == "tiny":
        cfg = G.LlamaConfig.tiny(kv_fp8=True)
        cfg.int4_block, cfg.vocab = 32, 1024
        run_graph(cfg, cudagraph=cudagraph)
    else:
        run_graph(G.LlamaConfig.tinyllama_1b(batch=4, s_max=512, layers=2, kv_fp8=True, int4_block=64), pos=300,
                  cudagraph=cudagraph)


@pytest.mark.parametrize("dt", [F16, BF16])
def test_w4_prompt_then_decode(K, dt):
    """a 40-token prompt step (dequantise path: 4 x 40 rows) fills the caches, then decode steps continue from them"""
    from infinitensor_b200 import backend as B
    from infinitensor_b200 import graphs as G
    cfg = G.LlamaConfig.tiny(dtype=dt, batch=4)
    cfg.int4_block, cfg.vocab = 64, 1024
    S, tol = 40, 3e-2
    rt = B.CudaRuntime(0)
    zeros = G.to_storage(np.zeros((cfg.batch, cfg.n_kv, cfg.s_max, cfg.head_dim), np.float32), dt)
    p = L.llama_pair(cfg, seq=S, caches=[zeros] * (2 * cfg.layers), rt=rt)
    rng = np.random.default_rng(4)
    ids = rng.integers(0, cfg.vocab, size=(cfg.batch, S)).astype(np.int64)
    got, ref = L.llama_step(p, ids, np.tile(np.arange(S, dtype=np.int64), (cfg.batch, 1)), cudagraph=False)
    assert np.isfinite(got).all() and L.rel_err(got, ref) < tol
    L.check_appended_k(p, slice(0, S), tol)
    # decode steps from the prompt's caches: each side continues from its own
    d = L.llama_pair(cfg, caches=L.cache_values(p.g), oracle_caches=L.cache_values(p.og), rt=rt)
    for step in range(3):
        ids1 = rng.integers(0, cfg.vocab, size=(cfg.batch, 1)).astype(np.int64)
        got, ref = L.llama_step(d, ids1, np.full((cfg.batch, 1), S + step, np.int64))
        assert np.isfinite(got).all() and L.rel_err(got, ref) < tol, f"decode step {step}"
        L.check_appended_k(d, S + step, tol)


def test_w4_onnx_import(K):
    """a tiny int4 Llama exported to ONNX and imported on the device computes what the graph oracle computes"""
    from infinitensor_b200 import backend as B
    from infinitensor_b200 import graphs as G
    from infinitensor_b200 import onnx_lite as X
    cfg = G.LlamaConfig.tiny(batch=2)
    cfg.int4_block, cfg.vocab = 32, 1024
    exp = X.OnnxExporter(B.GraphHandler(B.HostPlanRuntime()))
    ge = G.build_llama_decode(exp, cfg)
    G.fill_llama_weights_host(ge)
    stub = X.OnnxStub(exp.save(), handler=B.GraphHandler(B.CudaRuntime(0)))
    oh, og = L.oracle_graph(cfg)
    rng = np.random.default_rng(3)
    feeds = {ge.input_ids.name: rng.integers(0, cfg.vocab, size=(cfg.batch, 1)).astype(np.int64),
             ge.position_ids.name: np.full((cfg.batch, 1), 7, np.int64)}
    og.input_ids.copyin_numpy(feeds[ge.input_ids.name])
    og.position_ids.copyin_numpy(feeds[ge.position_ids.name])
    feeds.update((t.name, c) for t, c in zip(ge.k_caches + ge.v_caches, L.llama_caches(cfg)))
    for name, arr in feeds.items():
        stub.inputs[name].copyin_numpy(arr)
    stub.run()
    oh.run()
    got = G.from_storage(stub.outputs[ge.logits.name].copyout_numpy(), cfg.dtype).astype(np.float64)
    assert np.isfinite(got).all() and L.rel_err(got, og.logits.f32().astype(np.float64)) < 3e-2
