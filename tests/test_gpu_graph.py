"""GPU graph-level parity: the same graph description (infinitensor_b200/graphs.py) executed by the CUDA backend
backend through the C-ABI graph API and by the CPU oracle.  Covers the run loop, the memory planner, CUDA-graph
capture / replay / invalidation and the three BASELINE model families at reduced size."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F32, F16, BF16 = 1, 10, 16


@pytest.mark.parametrize("dtype", [F32, F16, BF16])
@pytest.mark.parametrize("cudagraph", [False, True])
def test_llama_decode_parity(dtype, cudagraph):
    from infinitensor_b200 import graphs as G
    from tests.llama_oracle import run_llama_parity
    _, launches, _ = run_llama_parity(G.LlamaConfig.tiny(dtype=dtype, layers=2, batch=4), pos=5, steps=3, cudagraph=cudagraph)
    assert launches > 0


def test_llama_decode_batch16_wide():
    """d=1024 / ffn=2816 / B=16: the skinny TMA GEMM path (M=16) inside the graph."""
    from infinitensor_b200 import graphs as G
    from tests.llama_oracle import run_llama_parity
    cfg = G.LlamaConfig(layers=2, d_model=1024, heads=8, head_dim=128, ffn=2816, vocab=2048, s_max=128, batch=16, dtype=BF16)
    run_llama_parity(cfg, pos=77, steps=2)


def test_llama_decode_baseline_width():
    """The BASELINE config's own per-layer shapes -- d = 4096, 32 heads, ffn = 11008, vocab = 32000, S_max = 1024, B = 16,
    position 511, bf16 -- two layers deep (the oracle stays within seconds): every GEMM shape of the bench (grouped q/k/v
    and gate/up, o, down, the 32000-wide logits), the 512-head streaming attention with folded RoPE, the fused schedule and
    CUDA-graph replay, end to end against the oracle."""
    from infinitensor_b200 import graphs as G
    from tests.llama_oracle import run_llama_parity
    cfg = G.LlamaConfig(layers=2, d_model=4096, heads=32, head_dim=128, ffn=11008, vocab=32000, s_max=1024, batch=16, dtype=BF16)
    run_llama_parity(cfg, pos=511, steps=1)


@pytest.mark.parametrize("dtype", [BF16, F16])
def test_llama_decode_fp8_weights(dtype):
    """SURVEY 8(f-4) through the graph: every projection (q/k/v grouped, o + residual, gate/up grouped, down + residual, logits)
    with FP8 E4M3 weight codes + per-column scales dequantised inside the GEMM; the oracle executes the same graph with the
    dequantised weights in fp32.  CUDA-graph replay, two steps."""
    from infinitensor_b200 import backend as B, graphs as G
    from tests.llama_oracle import run_llama_parity
    cfg = G.LlamaConfig(layers=2, d_model=1024, heads=8, head_dim=128, ffn=2816, vocab=2048, s_max=128, batch=16, dtype=dtype,
                        fp8_weights=True)
    h = B.GraphHandler(B.CudaRuntime(0))
    G.build_llama_decode(h, cfg)
    sc = h.schedule()
    assert sc.count("MatMulGroup:MatMul+MatMul+MatMul") == 2 and sc.count("MatMulAdd:MatMul+Add") == 4
    run_llama_parity(cfg, pos=77, steps=2)


def test_matmul_512_config1():
    """BASELINE config #1: MatmulObj fp32 512^3 through the graph API."""
    from infinitensor_b200 import backend as B, graphs as G
    import oracle
    rt = B.CudaRuntime(0)
    h = B.GraphHandler(rt)
    a, b, c = G.build_matmul(h)
    h.data_malloc()
    A = np.random.default_rng(0).standard_normal((512, 512)).astype(np.float32)
    Bm = np.random.default_rng(1).standard_normal((512, 512)).astype(np.float32)
    a.copyin_numpy(A)
    b.copyin_numpy(Bm)
    h.run()
    np.testing.assert_allclose(c.copyout_numpy(), oracle.matmul(A, Bm), rtol=1e-4, atol=1e-5 * np.sqrt(512) * 16)


@pytest.mark.parametrize("dtype", [F32, F16])
def test_gpt2_parity(dtype):
    from infinitensor_b200 import backend as B, graphs as G
    from oracle.graph_oracle import OracleHandler
    cfg = G.GPT2Config.tiny(dtype)
    rt = B.CudaRuntime(0)
    h, oh = B.GraphHandler(rt), OracleHandler()
    g, og = G.build_gpt2(h, cfg), G.build_gpt2(oh, cfg)
    h.data_malloc()
    G.fill_gpt2_weights_host(g)
    G.fill_gpt2_weights_host(og)
    ids = np.random.default_rng(1).integers(0, cfg.vocab, size=(cfg.batch, cfg.seq)).astype(np.int64)
    pos = np.arange(cfg.seq, dtype=np.int64).reshape(1, -1).repeat(cfg.batch, 0)
    for gg in (g, og):
        gg.input_ids.copyin_numpy(ids)
        gg.position_ids.copyin_numpy(pos)
    h.run_with_cudagraph()
    oh.run()
    got = G.from_storage(g.out.copyout_numpy(), dtype).astype(np.float64)
    ref = og.out.f32().astype(np.float64)
    tol = 1e-3 if dtype == F32 else 1e-2
    assert np.abs(got - ref).max() / np.abs(ref).max() < tol


def _gpt2_run(cfg, monkeypatch=None, env=None):
    from infinitensor_b200 import backend as B, graphs as G
    from oracle.graph_oracle import OracleHandler
    if env:
        for k, v in env.items():
            monkeypatch.setenv(k, v)
    rt = B.CudaRuntime(0)
    h, oh = B.GraphHandler(rt), OracleHandler()
    g, og = G.build_gpt2(h, cfg), G.build_gpt2(oh, cfg)
    sched = h.schedule()
    h.data_malloc()
    G.fill_gpt2_weights_host(g)
    G.fill_gpt2_weights_host(og)
    ids = np.random.default_rng(1).integers(0, cfg.vocab, size=(cfg.batch, cfg.seq)).astype(np.int64)
    pos = np.arange(cfg.seq, dtype=np.int64).reshape(1, -1).repeat(cfg.batch, 0)
    for gg in (g, og):
        gg.input_ids.copyin_numpy(ids)
        gg.position_ids.copyin_numpy(pos)
    h.run_with_cudagraph()
    oh.run()
    return G.from_storage(g.out.copyout_numpy(), cfg.dtype).astype(np.float64), og.out.f32().astype(np.float64), sched


def test_gpt2_small_full_size_config2(monkeypatch):
    """BASELINE config C2 at FULL size -- GPT-2-small, 12 layers, d = 768, 12 heads of 64, ffn 3072, vocab 50257, B = 1, S = 128,
    fp16 -- one forward through the fused schedule (PrefillAttention per layer) and CUDA-graph replay against the CPU oracle
    executing the operator graph; and the same graph with the attention chain unfused (ITB_FUSION_MASK without bit 8)."""
    from infinitensor_b200 import graphs as G
    cfg = G.GPT2Config()
    got, ref, sched = _gpt2_run(cfg)
    assert sum(s.startswith("PrefillAttention") for s in sched) == cfg.layers
    err = np.abs(got - ref).max() / np.abs(ref).max()
    assert err < 1e-2, err  # end-to-end fp16, 12 layers (SURVEY 8(c): 1e-3 per op, accumulated)
    got2, _, sched2 = _gpt2_run(cfg, monkeypatch, {"ITB_FUSION_MASK": "127"})
    assert not any(s.startswith("PrefillAttention") for s in sched2)
    assert np.abs(got2 - ref).max() / np.abs(ref).max() < 1e-2
    assert np.abs(got - got2).max() / np.abs(ref).max() < 5e-3  # fused vs unfused chain: same rounding points, other sum order


@pytest.mark.parametrize("dtype", [F32, F16])
def test_resnet_parity(dtype):
    from infinitensor_b200 import backend as B, graphs as G
    from oracle.graph_oracle import OracleHandler
    cfg = G.ResNetConfig.tiny(dtype)
    rt = B.CudaRuntime(0)
    h, oh = B.GraphHandler(rt), OracleHandler()
    g, og = G.build_resnet50(h, cfg), G.build_resnet50(oh, cfg)
    h.data_malloc()
    G.fill_resnet_weights_host(g)
    G.fill_resnet_weights_host(og)
    x = np.random.default_rng(3).standard_normal((cfg.batch, 3, cfg.image, cfg.image)).astype(np.float32)
    g.input.copyin_numpy(G.to_storage(x, dtype))
    og.input.copyin_numpy(G.to_storage(x, dtype))
    h.run()
    oh.run()
    got = G.from_storage(g.out.copyout_numpy(), dtype).astype(np.float64)
    ref = og.out.f32().astype(np.float64)
    tol = 1e-3 if dtype == F32 else 2e-2
    assert np.abs(got - ref).max() / np.abs(ref).max() < tol


def test_resnet50_full_width_config4():
    """BASELINE config C4 at FULL width and depth -- ResNet-50 (3-4-6-3 bottlenecks, 64..2048 channels, 224 x 224, 1000 classes),
    fp16, batch 8 (the oracle's CPU convolutions stay within a minute; every conv / GEMM shape is the B = 64 one except the batch
    fold) -- through the fused schedule (Conv+BN(+Add)(+ReLU) in the tcgen05 epilogue) against the CPU oracle executing the
    operator graph, plus top-1 agreement."""
    from infinitensor_b200 import backend as B, graphs as G
    from oracle.graph_oracle import OracleHandler
    cfg = G.ResNetConfig(batch=8)
    rt = B.CudaRuntime(0)
    h, oh = B.GraphHandler(rt), OracleHandler()
    g, og = G.build_resnet50(h, cfg), G.build_resnet50(oh, cfg)
    assert sum(s.startswith("ConvBnAct") for s in h.schedule()) == 53
    h.data_malloc()
    G.fill_resnet_weights_host(g)
    G.fill_resnet_weights_host(og)
    x = np.random.default_rng(3).standard_normal((cfg.batch, 3, cfg.image, cfg.image)).astype(np.float32)
    g.input.copyin_numpy(G.to_storage(x, F16))
    og.input.copyin_numpy(G.to_storage(x, F16))
    h.run_with_cudagraph()
    oh.run()
    got = G.from_storage(g.out.copyout_numpy(), F16).astype(np.float64)
    ref = og.out.f32().astype(np.float64)
    err = np.abs(got - ref).max() / np.abs(ref).max()
    assert err < 2e-2, err  # 53 fp16 convolutions deep: the per-op 1e-3 of SURVEY 8(c), accumulated
    assert (got.argmax(-1) == ref.argmax(-1)).mean() >= 0.75


def test_cudagraph_cache_semantics():
    """capture once / replay / invalidate on storage change / LRU (reference test/cuda/test_cudagraph.cc:80-320)."""
    from infinitensor_b200 import backend as B
    rt = B.CudaRuntime(0, 2)
    hs = []
    for i in range(3):
        h = B.GraphHandler(rt)
        a = h.tensor([4, 8], F32)
        b = h.tensor([4, 8], F32)
        a.set_input(); b.set_input()
        c = h.add(a, b, None)
        d = h.relu(c, None)
        d.set_output()
        h.data_malloc()
        a.copyin_numpy(np.full((4, 8), i + 1.0, np.float32))
        b.copyin_numpy(np.full((4, 8), -0.5, np.float32))
        hs.append((h, a, b, d))
    h, a, b, d = hs[0]
    h.run_with_cudagraph()
    assert rt.cuda_graph_capture_count() == 1 and rt.cuda_graph_cache_size() == 1
    h.run_with_cudagraph()
    assert rt.cuda_graph_capture_count() == 1  # replayed
    assert np.all(d.copyout_numpy() == 0.5)
    a.copyin_numpy(np.full((4, 8), 3.0, np.float32))  # new contents, same storage -> replay sees them
    h.run_with_cudagraph()
    assert rt.cuda_graph_capture_count() == 1 and np.all(d.copyout_numpy() == 2.5)
    h.data_malloc()  # re-plan -> new storage -> recapture
    a.copyin_numpy(np.full((4, 8), 3.0, np.float32)); b.copyin_numpy(np.full((4, 8), -0.5, np.float32))
    h.run_with_cudagraph()
    assert rt.cuda_graph_capture_count() == 2
    hs[1][0].run_with_cudagraph()
    hs[2][0].run_with_cudagraph()
    assert rt.cuda_graph_cache_size() == 2  # LRU capacity
    rt.clear_cuda_graph_cache()
    assert rt.cuda_graph_cache_size() == 0


def test_error_paths():
    from infinitensor_b200 import backend as B
    rt = B.CudaRuntime(0)
    h = B.GraphHandler(rt)
    a = h.tensor([2, 3], F32)
    b = h.tensor([4, 5], F32)
    with pytest.raises(RuntimeError):
        h.matmul(a, b, None, False, False, None, 0)  # K mismatch
    c = h.relu(a, None)
    with pytest.raises(RuntimeError):
        h.run()  # no storage yet
    h.data_malloc()
    with pytest.raises(RuntimeError):
        a.copyin_numpy(np.zeros((3, 2), np.float32))  # wrong shape


def test_smoke_entry():
    import __graft_entry__ as ge
    ge.smoke()


def _decode_once(dtype, env, monkeypatch):
    from infinitensor_b200 import backend as B, graphs as G
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    cfg = G.LlamaConfig(layers=2, d_model=1024, heads=8, head_dim=128, ffn=2816, vocab=2048, s_max=64, batch=16, dtype=dtype)
    rt = B.CudaRuntime(0)
    h = B.GraphHandler(rt)
    g = G.build_llama_decode(h, cfg)
    sched = h.schedule()
    h.data_malloc()
    G.fill_llama_weights_host(g)
    for li in range(cfg.layers):
        g.k_caches[li].copyin_numpy(G.to_storage(G.llama_cache_values(cfg, li, "k"), dtype))
        g.v_caches[li].copyin_numpy(G.to_storage(G.llama_cache_values(cfg, li, "v"), dtype))
    g.input_ids.copyin_numpy(np.arange(16, dtype=np.int64).reshape(16, 1) * 7 % cfg.vocab)
    g.position_ids.copyin_numpy(np.full((16, 1), 33, np.int64))
    h.run_with_cudagraph()
    h.run_with_cudagraph()
    return sched, g.logits.copyout_numpy().copy(), g.k_caches[1].copyout_numpy().copy(), cfg


@pytest.mark.parametrize("dtype", [F32, BF16])
def test_fused_schedule_matches_unfused(dtype, monkeypatch):
    """Alias elimination, MatMul+Add epilogue fusion, Silu*Mul fusion and RoPE-in-attention give EXACTLY the bits of the
    one-kernel-per-operator order (ITB_NO_FUSION=1).  Grouping q/k/v and gate/up into one launch may pick a different
    split-K partition (fp32 summation order), so that step is held to the GEMM tolerance instead."""
    from infinitensor_b200 import graphs as G
    _, base, base_k, cfg = _decode_once(dtype, {"ITB_NO_FUSION": "1"}, monkeypatch)
    sched, got, got_k, _ = _decode_once(dtype, {"ITB_NO_FUSION": "0", "ITB_FUSION_MASK": "61"}, monkeypatch)
    assert any(s.startswith("MatMulAdd") for s in sched) and any(s.startswith("Alias") for s in sched)
    assert any(s.startswith("AttentionRope") for s in sched) and any(s.startswith("SiluMul") for s in sched)
    assert np.array_equal(got, base) and np.array_equal(got_k, base_k)
    sched, got, got_k, _ = _decode_once(dtype, {"ITB_NO_FUSION": "0", "ITB_FUSION_MASK": "63"}, monkeypatch)
    if dtype == BF16:
        assert any(s.startswith("MatMulGroup") for s in sched)
    a, b = G.from_storage(got, dtype).astype(np.float64), G.from_storage(base, dtype).astype(np.float64)
    assert np.abs(a - b).max() <= (0 if dtype == F32 else 2.0 ** -6 * np.abs(b).max())


def _resnet_once(cfg, env, monkeypatch):
    from infinitensor_b200 import backend as B, graphs as G
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    rt = B.CudaRuntime(0)
    h = B.GraphHandler(rt)
    g = G.build_resnet50(h, cfg)
    sched = h.schedule()
    h.data_malloc()
    G.fill_resnet_weights_host(g)
    x = np.random.default_rng(3).standard_normal((cfg.batch, 3, cfg.image, cfg.image)).astype(np.float32)
    g.input.copyin_numpy(G.to_storage(x, cfg.dtype))
    h.run_with_cudagraph()
    h.run_with_cudagraph()
    return sched, g.out.copyout_numpy().copy()


def test_resnet_conv_tail_fusion_is_bit_identical(monkeypatch):
    """Full-width ResNet-50 (reduced image / batch): Conv+BatchNorm(+Add)(+Relu) steps on the tcgen05 epilogue produce the
    very bits of the one-kernel-per-operator schedule."""
    from infinitensor_b200 import graphs as G
    cfg = G.ResNetConfig(batch=4, image=64, dtype=F16)
    s1, fused = _resnet_once(cfg, {"ITB_FUSION_MASK": "127"}, monkeypatch)
    s0, plain = _resnet_once(cfg, {"ITB_FUSION_MASK": "63"}, monkeypatch)
    assert sum(s.startswith("ConvBnAct") for s in s1) == 53 and not any(s.startswith("ConvBnAct") for s in s0)
    assert np.isfinite(G.from_storage(fused, F16)).all()
    assert np.array_equal(fused, plain)


def test_matmul_tune_records_a_kernel_choice_per_shape(tmp_path):
    """run(tune=True): MatMul's tune() times the production dispatch and each GEMM kernel on the operator's own shape, stores the
    winner (kernel + tile width) in PerfEngine; the next run re-applies it and gives the same result within the GEMM tolerance."""
    import json
    from infinitensor_b200 import backend as B, graphs as G
    B.PerfEngine.clear()
    rt = B.CudaRuntime(0)
    h = B.GraphHandler(rt)
    x = h.tensor([16, 1024], BF16)
    x.set_input()
    w1 = h.tensor([1024, 4096], BF16)
    w1.set_weight()
    w2 = h.tensor([4096, 512], BF16)
    w2.set_weight()
    y = h.matmul(h.matmul(x, w1, None, False, False, None, 0), w2, None, False, False, None, 0)
    y.set_output()
    h.data_malloc()
    rng = np.random.default_rng(11)
    x.copyin_numpy(G.to_storage(rng.standard_normal((16, 1024)).astype(np.float32) * 0.5, BF16))
    w1.copyin_numpy(G.to_storage(rng.standard_normal((1024, 4096)).astype(np.float32) * 0.03, BF16))
    w2.copyin_numpy(G.to_storage(rng.standard_normal((4096, 512)).astype(np.float32) * 0.03, BF16))
    h.run()
    before = G.from_storage(y.copyout_numpy(), BF16).astype(np.float64)
    h.tune()
    assert B.PerfEngine.size() == 2 and h.get_perf_time() > 0
    out = tmp_path / "perf.json"
    B.PerfEngine.save(str(out))
    recs = [e[1] for e in json.loads(out.read_text())["data"]]
    assert all(r["type"] == 1 and r["impl"] in (0, 1, 2) and r["nb"] in (0, 1, 2) and r["data"] > 0 for r in recs)
    h.run()
    after = G.from_storage(y.copyout_numpy(), BF16).astype(np.float64)
    assert np.abs(after - before).max() <= 2.0 ** -6 * np.abs(before).max()
    B.PerfEngine.clear()


@pytest.mark.parametrize("tail", ["none", "relu_out", "flatten"])
def test_small_conv_net_enters_and_leaves_the_nhwc_domain(tail):
    """Conv (no BatchNorm) -> Relu -> MaxPool 2x2 -> Conv 1x1 [-> Relu] [-> Flatten] in f16: the first conv reads the NCHW graph
    input and writes NHWC through the im2col GEMM, Relu / MaxPool run on NHWC bytes, the implicit-GEMM conv writes the NCHW result
    (`@nhwc>`); against the oracle executing the operator graph."""
    from infinitensor_b200 import backend as B, graphs as G
    from oracle.graph_oracle import OracleHandler
    outs = []
    rng = np.random.default_rng(17)
    xv = rng.standard_normal((2, 16, 12, 12)).astype(np.float32)
    w1v = (rng.standard_normal((24, 16, 3, 3)) * 0.1).astype(np.float32)
    w2v = (rng.standard_normal((32, 24, 1, 1)) * 0.2).astype(np.float32)
    for h in (B.GraphHandler(B.CudaRuntime(0)), OracleHandler()):
        x = h.tensor([2, 16, 12, 12], F16)
        x.set_input()
        w1 = h.tensor([24, 16, 3, 3], F16)
        w1.set_weight()
        w2 = h.tensor([32, 24, 1, 1], F16)
        w2.set_weight()
        t = h.relu(h.conv(x, w1, None, 1, 1, 1, 1, 1, 1), None)
        t = h.maxPool(t, None, 2, 2, 1, 1, 0, 0, 2, 2, 0)
        t = h.conv(t, w2, None, 0, 0, 1, 1, 1, 1)
        if tail == "relu_out":
            t = h.relu(t, None)
        elif tail == "flatten":
            t = h.flatten(h.relu(t, None), None, 1)
        t.set_output()
        if isinstance(h, B.GraphHandler):
            sc = h.schedule()
            assert sc[0] == "Single:Conv@>nhwc" and sc[2] == "Single:MaxPool@nhwc" and sc[3] == "Single:Conv@nhwc>", sc
        h.data_malloc()
        for tt, v in ((x, xv), (w1, w1v), (w2, w2v)):
            tt.copyin_numpy(G.to_storage(v, F16))
        h.run()
        outs.append(np.asarray(t.f32(), np.float64) if hasattr(t, "f32") else G.from_storage(t.copyout_numpy(), F16).astype(np.float64))
    got, ref = outs[0].reshape(-1), outs[1].reshape(-1)
    assert np.abs(got - ref).max() <= 4e-3 * max(np.abs(ref).max(), 1.0)


def test_resnet_nhwc_domain_matches_nchw(monkeypatch):
    """The NHWC domain (implicit-GEMM convs, NHWC pools; fusion mask bit 9) against the NCHW schedule of the same graph: the
    logits agree within fp16 accumulation noise (the NHWC epilogue rounds once per chain, the NCHW one after every operator) and
    pick the same classes."""
    from infinitensor_b200 import graphs as G
    cfg = G.ResNetConfig(batch=4, image=64, dtype=F16)
    s1, nhwc = _resnet_once(cfg, {}, monkeypatch)
    s0, nchw = _resnet_once(cfg, {"ITB_FUSION_MASK": "383"}, monkeypatch)
    assert sum("@nhwc" in s for s in s1) == 54 and s1[0].endswith("@>nhwc") and not any("@" in s for s in s0)
    a, b = G.from_storage(nhwc, F16).astype(np.float64), G.from_storage(nchw, F16).astype(np.float64)
    assert np.isfinite(a).all()
    assert np.abs(a - b).max() / np.abs(b).max() < 2e-2
    assert (a.argmax(-1) == b.argmax(-1)).all()


@pytest.mark.parametrize("dtype", [F32, BF16])
def test_onnx_stub_drives_the_backend(dtype):
    """SURVEY 8(f-1): an ONNX file (written by OnnxExporter, read by the package-free protobuf reader) lowered by
    OnnxStub onto the CUDA runtime gives the oracle's logits for the same file."""
    from infinitensor_b200 import backend as B, graphs as G, onnx_lite as X
    from oracle.graph_oracle import OracleHandler
    cfg = G.LlamaConfig(layers=2, d_model=256, heads=2, head_dim=128, ffn=384, vocab=96, s_max=16, batch=3, dtype=dtype)
    exp = X.OnnxExporter(OracleHandler())
    ge = G.build_llama_decode(exp, cfg)
    exp.data_malloc()
    G.fill_llama_weights_host(ge)
    blob = exp.save()
    gpu = X.OnnxStub(blob, B.CudaRuntime(0))
    cpu = X.OnnxStub(blob, handler=OracleHandler())
    rng = np.random.default_rng(5)
    for name, t in gpu.inputs.items():
        shp, dt = t.shape(), t.dtype()
        v = rng.integers(0, 7, size=shp).astype(np.int64) if dt == 7 else G.to_storage((rng.standard_normal(shp) * 0.5).astype(np.float32), dt)
        t.copyin_numpy(v)
        cpu.inputs[name].copyin_numpy(v)
    gpu.run_with_cudagraph()
    cpu.run()
    (name, out), = [(k, v) for k, v in gpu.outputs.items()][:1]
    got = G.from_storage(out.copyout_numpy(), dtype).astype(np.float64)
    ref = cpu.outputs[name].f32().astype(np.float64)
    assert np.abs(got - ref).max() / np.abs(ref).max() < (1e-3 if dtype == F32 else 3e-2)
