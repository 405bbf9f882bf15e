"""CPU tier: the C-ABI library loads and exports every symbol include/it_b200.h declares, and the host
logic (operator shape rules, memory planner, error behaviour, tensor-parallel sharding rule) behaves like
the reference's -- exercised through the planning-only runtime (device -1).  No kernel runs here."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest


def _free_port():
    """an unused TCP port for the torchrun rendezvous of the gloo world-2 tests"""
    import socket
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        return sk.getsockname()[1]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def B():
    from infinitensor_b200 import backend
    return backend


def test_header_symbols_are_exported():
    import ctypes
    from infinitensor_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "it_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    names = set(re.findall(r"\b(it_b200_\w+|itb_\w+)\s*\(", hdr))
    names -= {"itb_runtime", "itb_graph", "itb_tensor"}
    assert len(names) > 60
    missing = [n for n in sorted(names) if not hasattr(_lib.lib, n)]
    assert not missing, f"declared in include/it_b200.h but not exported: {missing}"
    # the loader's signature tables must not drift from the header
    from infinitensor_b200 import backend
    for n in list(_lib.exported_symbols()) + backend.GRAPH_API_SYMBOLS:
        assert n in names or n == "it_b200_launch_count", n


def test_no_cpu_fallback(B):
    with pytest.raises(RuntimeError):
        B.cpu_runtime()
    rt = B.HostPlanRuntime()
    h = B.GraphHandler(rt)
    a = h.tensor([2, 2], 1)
    h.relu(a, None)
    h.data_malloc()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        h.run()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        h.run_with_cudagraph()


def test_cuda_runtime_fails_loudly_without_gpu(B):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError, match="CUDA"):
        B.CudaRuntime(0)


def test_product_never_imports_oracle():
    """the oracle is test infrastructure: nothing under infinitensor_b200/ may import or load it"""
    for dp, _, fs in os.walk(os.path.join(ROOT, "infinitensor_b200")):
        for f in fs:
            if f.endswith((".py", ".cc", ".cu", ".h", ".cuh")):
                txt = open(os.path.join(dp, f), errors="ignore").read()
                assert not re.search(r"^\s*(import oracle|from oracle)", txt, flags=re.M), f
                assert "it_oracle" not in txt, f


# ---- shape rules (reference test/operators/*.cc assert getOutput()->getDims())
def test_shape_inference(B):
    rt = B.HostPlanRuntime()
    h = B.GraphHandler(rt)
    T = lambda *d, dt=1: h.tensor(list(d), dt)
    assert h.matmul(T(1, 3, 5), T(1, 5, 2), None, False, False, None, 0).shape() == [1, 3, 2]
    assert h.matmul(T(2, 3, 4), T(2, 3, 2), None, True, False, None, 0).shape() == [2, 4, 2]   # test_matmul.cc
    assert h.matmul(T(2, 3, 5), T(5, 2), None, False, False, None, 0).shape() == [2, 3, 2]
    assert h.matmul(T(3, 1, 4, 5), T(2, 5, 6), None, False, False, None, 0).shape() == [3, 2, 4, 6]
    assert h.conv(T(1, 3, 4, 4), T(2, 3, 3, 3), None, 1, 1, 2, 1, 1, 2).shape() == [1, 2, 2, 2]  # test_cuda_conv.cc
    assert h.conv(T(2, 8, 9, 9), T(8, 2, 3, 3), None, 1, 1, 2, 2, 1, 1).shape() == [2, 8, 5, 5]  # groups = 4
    assert h.maxPool(T(1, 2, 5, 5), None, 3, 3, 1, 1, 1, 1, 2, 2, 0).shape() == [1, 2, 3, 3]
    assert h.maxPool(T(1, 2, 6, 6), None, 3, 3, 1, 1, 0, 0, 2, 2, 1).shape() == [1, 2, 3, 3]     # ceil mode
    assert h.transpose(T(1, 2, 3, 4), None, [0, 2, 1, 3]).shape() == [1, 3, 2, 4]
    assert h.concat([T(2, 2, 3, 1), T(2, 2, 1, 1), T(2, 2, 2, 1)], None, 2).shape() == [2, 2, 6, 1]
    assert [t.shape() for t in h.split(T(2, 10, 2, 1), None, 1, 3)] == [[2, 3, 2, 1], [2, 3, 2, 1], [2, 4, 2, 1]]
    assert [t.shape() for t in h.split(T(1, 6), None, 1, [1, 2])] == [[1, 2], [1, 4]]
    assert h.gather(T(2, 4, 2), T(3, 1, dt=6), None, 1).shape() == [2, 3, 1, 2]
    assert h.reshape(T(2, 3, 4), None, [4, -1]).shape() == [4, 6]
    assert h.flatten(T(2, 3, 4), None, 1).shape() == [2, 12]
    assert h.squeeze(T(1, 3, 1, 4), None, [0]).shape() == [3, 1, 4]
    assert h.unsqueeze(T(3, 4), None, [0, 3]).shape() == [1, 3, 4, 1]
    assert h.reduceMean(T(2, 3, 2, 2), None, [1, 2], False).shape() == [2, 2]
    assert h.reduceSum(T(3, 2, 2), None, None, True).shape() == [1, 1, 1]
    assert h.slice(T(3, 2, 1, 5), None, [1, 1], [2, 5], [0, 3], None).shape() == [1, 2, 1, 4]   # test_cuda_slice.cc
    assert h.slice(T(10,), None, [8], [-11], [0], [-3]).shape() == [3]
    assert h.pad(T(1, 2, 3, 2), None, [1, 0, 1, 1], [0, 3]).shape() == [3, 2, 3, 3]              # test_cuda_pad.cc
    assert h.expand(T(2, 1, 2, 1), None, [2, 2, 2, 3]).shape() == [2, 2, 2, 3]
    assert h.where(T(3,), T(2, 3, 1), T(2, 1, 3, 1, dt=2), None).shape() == [2, 2, 3, 3]
    assert h.less(T(2, 3), T(3,), None).dtype() == 9
    assert h.cast(T(4,), None, 10).dtype() == 10
    q = T(2, 4, 1, 128)
    assert h.attentionKVCache(T(2, 4, 64, 128), T(2, 4, 64, 128), q, T(2, 4, 1, 128), T(2, 4, 1, 128), T(2, 1, dt=7), None).shape() == [2, 4, 1, 128]
    for bad in (lambda: h.matmul(T(2, 3), T(4, 5), None, False, False, None, 0),
                lambda: h.add(T(2, 3), T(4,), None),
                lambda: h.transpose(T(2, 3), None, [0, 0]),
                lambda: h.reshape(T(2, 3), None, [4, 2]),
                lambda: h.concat([T(2, 3), T(3, 3, 1)], None, 0),
                lambda: h.relu(T(2, 3), T(3, 2))):
        with pytest.raises(RuntimeError):
            bad()


# ---- planner (reference test/core/test_graph.cc, test_lazy_allocator.cc)
def test_memory_plan_reuses_dead_activations(B):
    rt = B.HostPlanRuntime()
    h = B.GraphHandler(rt)
    n = 1 << 20
    x = h.tensor([n], 1)
    x.set_input()
    t = x
    for _ in range(10):
        t = h.relu(t, None)
    t.set_output()
    h.data_malloc()
    w, a = h.arena_bytes()
    assert w == 0
    # input + output pinned, chain needs two live activations at a time -> 4 buffers, not 11
    assert a <= 4 * n * 4 + 4 * 256, a
    ptrs = set()
    h2 = B.GraphHandler(rt)
    y = h2.tensor([n], 1); y.set_input()
    u = y
    outs = []
    for _ in range(4):
        u = h2.relu(u, None)
        outs.append(u)
    h2.data_malloc(True)  # naive allocator: every tensor its own slot
    assert h2.arena_bytes()[1] >= 5 * n * 4
    assert len({o.device_ptr() for o in outs}) == 4
    assert all(o.device_ptr() % 256 == 0 for o in outs)  # 256 B alignment (lazy_allocator.cc:13)


def test_weights_and_inputs_survive_replan(B):
    rt = B.HostPlanRuntime()
    h = B.GraphHandler(rt)
    a = h.tensor([4, 8], 1); a.set_input()
    w = h.tensor([8, 2], 1); w.set_weight()
    y = h.matmul(a, w, None, False, False, None, 0)
    h.data_malloc()
    A = np.arange(32, dtype=np.float32).reshape(4, 8); W = np.ones((8, 2), np.float32) * 3
    a.copyin_numpy(A); w.copyin_numpy(W)
    p0 = w.device_ptr()
    h.relu(y, None)
    h.data_malloc()  # re-plan after a topology change
    assert w.device_ptr() == p0, "weight arena is allocated once"
    assert np.array_equal(w.copyout_numpy(), W) and np.array_equal(a.copyout_numpy(), A)
    with pytest.raises(RuntimeError):
        a.copyin_numpy(np.zeros((8, 4), np.float32))
    with pytest.raises(RuntimeError):
        a.copyin_numpy(np.zeros((4, 8), np.float16))


def test_llama_graph_op_mix_and_tp_shapes(B):
    from infinitensor_b200 import graphs as G
    rt = B.HostPlanRuntime()
    cfg = G.LlamaConfig(layers=2, d_model=512, heads=4, head_dim=128, ffn=1024, vocab=100, s_max=32, batch=16)
    h = B.GraphHandler(rt)
    g = G.build_llama_decode(h, cfg)
    ops = h.operators()
    assert ops.count("MatMul") == 2 * 7 + 1 and ops.count("AttentionKVCache") == 2 and ops.count("RMSNorm") == 5
    assert "AllReduceSum" not in ops
    h2 = B.GraphHandler(rt)
    g2 = G.build_llama_decode(h2, cfg, world=2, rank=1)
    assert h2.operators().count("AllReduceSum") == 4          # 2 per layer (parallel_opt.py:195-210)
    assert g2.weights["l0.wq"][0].shape() == [512, 256]        # column split
    assert g2.weights["l0.wo"][0].shape() == [256, 512]        # row split
    assert g2.weights["l0.wd"][0].shape() == [512, 512]
    assert g2.weights["lm_head"][0].shape() == [512, 100]      # logits MatMul not sharded (:178-187)
    assert g2.k_caches[0].shape() == [16, 2, 32, 128]          # KV cache split by head (:61-69)
    assert cfg.algorithmic_bytes(511) > 0
    full = G.LlamaConfig()
    assert abs(full.algorithmic_bytes(511) / 1e9 - 17.56) < 0.1  # SURVEY 8(d)


def _tp_worker():
    """one rank of a world-size-2 gloo run: sharded oracle graph with a real all-reduce"""
    import torch.distributed as dist
    from infinitensor_b200 import graphs as G
    from oracle.graph_oracle import OracleHandler
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    cfg = G.LlamaConfig.tiny(dtype=1, layers=2, batch=3)
    oh = OracleHandler()
    g = G.build_llama_decode(oh, cfg, world, rank)
    G.fill_llama_weights_host(g, world, rank)
    for li in range(cfg.layers):
        g.k_caches[li].copyin_numpy(G.llama_cache_values(cfg, li, "k", world, rank))
        g.v_caches[li].copyin_numpy(G.llama_cache_values(cfg, li, "v", world, rank))
    g.input_ids.copyin_numpy(np.array([[1], [5], [7]], np.int64))
    g.position_ids.copyin_numpy(np.full((3, 1), 9, np.int64))
    oh.run()
    np.save(os.environ["TP_OUT"] + f".{rank}.npy", g.logits.f32())
    dist.barrier()


def test_tensor_parallel_rule_gloo_world2(tmp_path):
    """The TP cut (column/row split + all-reduce, parallel_opt.py) reproduces the unsharded graph: two gloo
    ranks on CPU vs the single-rank oracle."""
    from infinitensor_b200 import graphs as G
    from oracle.graph_oracle import OracleHandler
    out = str(tmp_path / "tp")
    env = dict(os.environ, TP_OUT=out, MASTER_ADDR="127.0.0.1", OMP_NUM_THREADS="2")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(_free_port()), os.path.abspath(__file__), "--tp-worker"]
    subprocess.run(cmd, check=True, env=env, cwd=ROOT, timeout=240)
    cfg = G.LlamaConfig.tiny(dtype=1, layers=2, batch=3)
    oh = OracleHandler()
    g = G.build_llama_decode(oh, cfg)
    G.fill_llama_weights_host(g)
    for li in range(cfg.layers):
        g.k_caches[li].copyin_numpy(G.llama_cache_values(cfg, li, "k"))
        g.v_caches[li].copyin_numpy(G.llama_cache_values(cfg, li, "v"))
    g.input_ids.copyin_numpy(np.array([[1], [5], [7]], np.int64))
    g.position_ids.copyin_numpy(np.full((3, 1), 9, np.int64))
    oh.run()
    ref = g.logits.f32()
    for r in range(2):
        got = np.load(out + f".{r}.npy")
        np.testing.assert_allclose(got, ref, rtol=1e-4, atol=1e-5)


if __name__ == "__main__" and "--tp-worker" in sys.argv:
    sys.path.insert(0, ROOT)
    _tp_worker()


def test_conv_bn_act_schedule(B, monkeypatch):
    """ResNet-50: every Conv takes its BatchNorm (+ residual Add) (+ Relu) into one ConvBnAct step; mask bit 6 off -> 1:1."""
    import collections
    from infinitensor_b200 import graphs as G
    rt = B.HostPlanRuntime()
    h = B.GraphHandler(rt)
    G.build_resnet50(h, G.ResNetConfig(batch=2, image=64))
    sc = h.schedule()
    kinds = collections.Counter(s.split(":")[0] for s in sc)
    assert kinds["ConvBnAct"] == 53
    # NHWC domain: the 3-channel stem reads the NCHW graph input and WRITES NHWC ("@>nhwc"); the max pool, every bottleneck conv
    # (implicit GEMM) and the global average pool (whose [N, C, 1, 1] result is layout-free) stay inside it ("@nhwc")
    assert sc.count("ConvBnAct:Conv+BatchNormalization+Relu@>nhwc") == 1             # stem
    assert sc.count("ConvBnAct:Conv+BatchNormalization+Relu@nhwc") == 16 * 2         # conv1 / conv2 of 16 blocks
    assert sc.count("ConvBnAct:Conv+BatchNormalization+Add+Relu@nhwc") == 16         # conv3 of every block
    assert sc.count("ConvBnAct:Conv+BatchNormalization@nhwc") == 4                   # the four downsample branches
    assert sc.count("Single:MaxPool@nhwc") == 1 and sc.count("Single:AveragePool@nhwc") == 1
    assert not any(s.startswith("Single:BatchNormalization") or s == "Single:Relu" or s == "Single:Add" for s in sc)
    h.data_malloc()
    # bit 9 off: the same fusion, every tensor NCHW
    monkeypatch.setenv("ITB_FUSION_MASK", str(127 | 256))
    h3 = B.GraphHandler(rt)
    G.build_resnet50(h3, G.ResNetConfig(batch=2, image=64))
    sc3 = h3.schedule()
    assert not any("@" in s for s in sc3) and sc3.count("ConvBnAct:Conv+BatchNormalization+Relu") == 1 + 16 * 2
    monkeypatch.setenv("ITB_FUSION_MASK", "63")
    h2 = B.GraphHandler(rt)
    G.build_resnet50(h2, G.ResNetConfig(batch=2, image=64))
    assert not any(s.startswith("ConvBnAct") for s in h2.schedule())


def test_nhwc_layout_pass_corner_cases(B):
    """The NHWC domain's fixpoint (schedule.cc LayoutPass): a tensor is channel-innermost only when EVERY step touching it can work
    that way -- a Conv chain ending in a layout-sensitive operator (Flatten of a [N, C, H, W] map), an fp32 graph, channels that are
    not a multiple of 8, or a graph output in the middle all keep the reference layout where they must."""
    rt = B.HostPlanRuntime()

    def build(dt, c_mid, tail):
        h = B.GraphHandler(rt)
        x = h.tensor([2, 16, 12, 12], dt)
        x.set_input()
        w1 = h.tensor([c_mid, 16, 3, 3], dt)
        w1.set_weight()
        w2 = h.tensor([32, c_mid, 1, 1], dt)
        w2.set_weight()
        t = h.relu(h.conv(x, w1, None, 1, 1, 1, 1, 1, 1), None)
        t = h.maxPool(t, None, 2, 2, 1, 1, 0, 0, 2, 2, 0)
        t = h.conv(t, w2, None, 0, 0, 1, 1, 1, 1)
        if tail == "relu_out":
            t = h.relu(t, None)
        elif tail == "flatten":
            t = h.flatten(h.relu(t, None), None, 1)
        t.set_output()
        return h.schedule()

    # f16, 8-multiple channels: the first conv reads the NCHW graph input and WRITES NHWC (the im2col GEMM scatters channel-innermost),
    # Relu / MaxPool stay inside, the last conv reads NHWC and writes the NCHW graph output
    assert build(10, 24, "none") == ["Single:Conv@>nhwc", "Single:Relu@nhwc", "Single:MaxPool@nhwc", "Single:Conv@nhwc>"]
    # ... and with a Relu producing the output, that Relu (flat elementwise: operands and result agree) pulls the last conv's result to NCHW
    assert build(10, 24, "relu_out") == ["Single:Conv@>nhwc", "Single:Relu@nhwc", "Single:MaxPool@nhwc", "Single:Conv@nhwc>", "Single:Relu"]
    # fp32: nothing is NHWC
    assert not any("@" in s for s in build(1, 24, "relu_out"))
    # 20 mid channels (not a multiple of 8): no NHWC pool kernel, no implicit-GEMM conv -> the whole chain stays NCHW
    assert not any("@" in s for s in build(10, 20, "relu_out"))
    # Flatten reads [N, C, H, W] as [N, C*H*W]: its input stays NCHW
    sc = build(10, 24, "flatten")
    assert sc[:4] == ["Single:Conv@>nhwc", "Single:Relu@nhwc", "Single:MaxPool@nhwc", "Single:Conv@nhwc>"] and "@" not in sc[4] and "@" not in sc[5]


def test_prefill_extension_and_linear_epilogue_negative_cases(B):
    """The extended PrefillAttention step and the biased-Linear epilogue only swallow what is provably private to them."""
    rt = B.HostPlanRuntime()
    Bt, S, H, D = 1, 128, 2, 64
    d = H * D

    def attention_block(extra_reader=False, swap_kv=False, rows=128):
        h = B.GraphHandler(rt)
        x = h.tensor([Bt, rows, d], 10)
        x.set_input()
        w = h.tensor([d, 3 * d], 10)
        w.set_weight()
        b = h.tensor([3 * d], 10)
        b.set_weight()
        wo = h.tensor([d, d], 10)
        wo.set_weight()
        bo = h.tensor([d], 10)
        bo.set_weight()
        sc = h.tensor([1], 10)
        sc.set_weight()
        qkv = h.matmul(x, w, None, False, False, b, 0)
        parts = h.split(qkv, None, 2, 3)
        q, k, v = parts
        if swap_kv:
            k, v = v, k
        heads = lambda t: h.transpose(h.reshape(t, None, [Bt, rows, H, D]), None, [0, 2, 1, 3])
        if extra_reader:
            side = h.relu(parts[0], None)  # a second consumer of the q third: it must stay a real tensor
            side.set_output()
        q, k, v = heads(q), heads(k), heads(v)
        s_ = h.div(h.matmul(q, h.transpose(k, None, [0, 1, 3, 2]), None, False, False, None, 0), sc, None)
        a = h.matmul(h.softmax(s_, None, -1), v, None, False, False, None, 0)
        a = h.reshape(h.transpose(a, None, [0, 2, 1, 3]), None, [Bt, rows, d])
        o = h.add(x, h.matmul(a, wo, None, False, False, bo, 0), None)
        o.set_output()
        return h.schedule()

    ext = [s for s in attention_block() if s.startswith("PrefillAttention:Split")]
    assert len(ext) == 1
    sc = attention_block(extra_reader=True)  # the Split has an outside reader -> the bare chain, Split / Transposes on their own
    assert any(s == "PrefillAttention:Transpose+MatMul+Div+Softmax+MatMul" for s in sc) and "Single:Split" in sc and sc.count("Single:Transpose") == 4
    sc = attention_block(swap_kv=True)      # k / v are not thirds 1 / 2 in order -> not the strided-view pattern
    assert not any(s.startswith("PrefillAttention:Split") for s in sc) and "Single:Split" in sc
    # 16 rows (decode regime): the biased projections keep their Add outside (the tcgen05 epilogue is for > 64 rows), 32-row attention is
    # still a prefill chain (q-len > 1) but never the biased-Linear fusion
    sc = attention_block(rows=16)
    assert "MatMulAdd:MatMul+Add" not in sc and "Single:Add" in sc


def test_gpt2_linear_epilogue_schedule(B, monkeypatch):
    """GPT-2: the biased Linear layers take the residual Add (c_proj, mlp c_proj) or the Gelu (c_fc) into their step (mask bit 10);
    off -> the Round-1 schedule with those operators on their own."""
    import collections
    from infinitensor_b200 import graphs as G
    rt = B.HostPlanRuntime()
    h = B.GraphHandler(rt)
    G.build_gpt2(h, G.GPT2Config())
    c = collections.Counter(h.schedule())
    assert c["MatMulAdd:MatMul+Add"] == 24 and c["MatMulAdd:MatMul+Gelu"] == 12 and c["Single:MatMul"] == 12
    assert c["Single:Gelu"] == 0 and c["Single:Add"] == 1 and len(h.schedule()) == 88
    # (bit 11) the head split / merge around each attention chain belongs to the attention step: no Split / Transpose launches left
    ext = "PrefillAttention:Split+Reshape+Transpose+Reshape+Transpose+Reshape+Transpose+Transpose+MatMul+Div+Add+Softmax+MatMul+Transpose+Reshape"
    assert c[ext] == 12 and not any(s.startswith(("Single:Transpose", "Single:Split", "Alias:")) for s in h.schedule())
    monkeypatch.setenv("ITB_FUSION_MASK", str(127 | 256 | 512 | 1024))
    h1 = B.GraphHandler(rt)
    G.build_gpt2(h1, G.GPT2Config())
    c1 = collections.Counter(h1.schedule())
    assert c1["PrefillAttention:Transpose+MatMul+Div+Add+Softmax+MatMul"] == 12 and c1["Single:Transpose"] == 48 and len(h1.schedule()) == 196
    monkeypatch.setenv("ITB_FUSION_MASK", str(127 | 256 | 512))
    h2 = B.GraphHandler(rt)
    G.build_gpt2(h2, G.GPT2Config())
    c2 = collections.Counter(h2.schedule())
    assert c2["Single:Gelu"] == 12 and c2["Single:Add"] == 25 and c2["Single:MatMul"] == 48 and len(h2.schedule()) == 232


def test_fused_schedule_and_alias_plan(B, monkeypatch):
    """The execution schedule groups q/k/v and gate/up MatMuls, folds the residual Adds and Silu*Mul, and turns
    the decode graph's Reshape / size-1 Transpose ops into storage aliases; ITB_NO_FUSION=1 gives the 1:1 order."""
    import collections
    from infinitensor_b200 import graphs as G
    rt = B.HostPlanRuntime()
    cfg = G.LlamaConfig(layers=2, d_model=512, heads=4, head_dim=128, ffn=1024, vocab=128, s_max=32, batch=16)
    h = B.GraphHandler(rt)
    G.build_llama_decode(h, cfg)
    sc = h.schedule()
    kinds = collections.Counter(s.split(":")[0] for s in sc)
    assert kinds == {"Alias": 16, "Single": 7, "MatMulGroup": 4, "MatMulAdd": 4, "SiluMul": 2, "AttentionRope": 2}
    assert "AttentionRope:RoPE+RoPE+AttentionKVCache" in sc
    assert "MatMulGroup:MatMul+MatMul+MatMul" in sc and "MatMulGroup:MatMul+MatMul" in sc
    launches = sum(1 for s in sc if not s.startswith("Alias"))
    assert launches == 2 * 8 + 3  # 8 kernels per layer + gather, final norm, logits
    # tensor-parallel graph: the all-reduce takes the residual Add and the following RMSNorm with it
    h_tp = B.GraphHandler(rt)
    G.build_llama_decode(h_tp, cfg, 2, 1)
    sc_tp = [s for s in h_tp.schedule() if not s.startswith("Alias")]
    assert sc_tp.count("AllReduceAddNorm:AllReduceSum+Add+RMSNorm") == 4 and sc_tp.count("Single:RMSNorm") == 1
    h.data_malloc()
    fused_bytes = h.arena_bytes()[1]
    monkeypatch.setenv("ITB_NO_FUSION", "1")
    h2 = B.GraphHandler(rt)
    G.build_llama_decode(h2, cfg)
    assert len(h2.schedule()) == len(h2.operators()) and all(s.startswith("Single:") for s in h2.schedule())
    h2.data_malloc()
    assert fused_bytes <= 1.1 * h2.arena_bytes()[1]  # grouped steps allocate their outputs together
    monkeypatch.delenv("ITB_NO_FUSION")
    # alias: a Reshape's output shares its input's storage unless it is a graph output / KV-cache operand
    h3 = B.GraphHandler(rt)
    x = h3.tensor([4, 6], 1); x.set_input()
    r = h3.reshape(h3.relu(x, None), None, [2, 12])
    t = h3.transpose(h3.reshape(r, None, [2, 1, 12]), None, [1, 0, 2])   # only moves a size-1 dim
    y = h3.relu(t, None)
    z = h3.reshape(y, None, [24])                                         # graph output: must stay a copy
    h3.data_malloc()
    sc3 = h3.schedule()
    assert sc3 == ["Single:Relu", "Alias:Reshape", "Alias:Reshape", "Alias:Transpose", "Single:Relu", "Single:Reshape"]
    assert r.device_ptr() == t.device_ptr() and z.device_ptr() != y.device_ptr()
    h4 = B.GraphHandler(rt)
    a = h4.tensor([2, 3, 4], 1); a.set_input()
    assert h4.schedule() == [] and h4.transpose(a, None, [0, 2, 1]) is not None
    assert h4.schedule() == ["Single:Transpose"]                          # a real permutation is never an alias


def test_conv_bn_act_matcher_edge_cases(B):
    """The ConvBnAct step only swallows single-consumer links, same-shape residuals and fp32 BatchNorm statistics."""
    F16, F32 = 10, 1
    rt = B.HostPlanRuntime()

    def net(build):
        h = B.GraphHandler(rt)
        x = h.tensor([2, 16, 8, 8], F16); x.set_input()
        w = h.tensor([16, 16, 3, 3], F16); w.set_weight()
        stats = [h.tensor([16], F32) for _ in range(4)]
        for s in stats: s.set_weight()
        build(h, x, w, stats)
        return h.schedule()

    def bn(h, t, stats, dtype_stats=None):
        return h.batchNormalization(t, None, stats[0], stats[1], stats[2], stats[3], 0.9, 1e-5, False)

    # plain chain, BN output is the graph output
    sc = net(lambda h, x, w, s: bn(h, h.conv(x, w, None, 1, 1, 1, 1, 1, 1), s).set_output())
    assert sc == ["ConvBnAct:Conv+BatchNormalization"]
    # conv output read twice: nothing may be folded (the second reader needs the tensor)
    def two_readers(h, x, w, s):
        c = h.conv(x, w, None, 1, 1, 1, 1, 1, 1)
        h.relu(c, None).set_output()
        bn(h, c, s).set_output()
    sc = net(two_readers)
    assert sorted(sc) == ["Single:BatchNormalization", "Single:Conv", "Single:Relu"]
    # residual of another shape (broadcast add): chain stops at the BatchNorm
    def bcast(h, x, w, s):
        r = h.tensor([1, 16, 1, 1], F16); r.set_input()
        h.relu(h.add(bn(h, h.conv(x, w, None, 1, 1, 1, 1, 1, 1), s), r, None), None).set_output()
    sc = net(bcast)
    assert sc == ["ConvBnAct:Conv+BatchNormalization", "Single:Add", "Single:Relu"]
    # same-shape residual + relu: everything in one step, the residual producer scheduled before it
    def residual(h, x, w, s):
        r = h.relu(x, None)
        h.relu(h.add(r, bn(h, h.conv(x, w, None, 1, 1, 1, 1, 1, 1), s), None), None).set_output()
    sc = net(residual)
    assert sc == ["Single:Relu", "ConvBnAct:Conv+BatchNormalization+Add+Relu"]


def test_perf_engine_json_roundtrip_in_the_reference_layout(B, tmp_path):
    """savePerfEngineData / loadPerfEngineData (reference src/core/perf_engine.cc:7-62): a file in nlohmann's layout of the
    reference's map (keys in any order, 64-bit hashes) loads, saves back with the same content, and load replaces the table."""
    import json
    ref_style = {"data": [
        [[[2, 7], {"opType": 7, "hashType": 18446744073709551557, "attrs": [16, 4096, 4096, 0, 0]}], {"type": 0, "data": 0.0125}],
        [[[2, 3], {"attrs": [], "hashType": 42, "opType": 3}], {"data": 3, "type": 0}],
    ]}
    p = tmp_path / "perf.json"
    p.write_text(json.dumps(ref_style, indent=1))
    B.PerfEngine.clear()
    B.PerfEngine.load(str(p))
    assert B.PerfEngine.size() == 2
    out = tmp_path / "perf_out.json"
    B.PerfEngine.save(str(out))
    back = json.loads(out.read_text())
    canon = lambda d: sorted((tuple(e[0][0]), e[0][1]["hashType"], e[0][1]["opType"], tuple(e[0][1]["attrs"]), float(e[1]["data"]), e[1]["type"])
                             for e in d["data"])
    assert canon(back) == canon(ref_style)
    p.write_text(json.dumps({"data": []}))
    B.PerfEngine.load(str(p))
    assert B.PerfEngine.size() == 0
    with pytest.raises(RuntimeError):
        B.PerfEngine.load(str(tmp_path / "missing.json"))
    # MatMul's tuned record (type 1: which GEMM kernel + tile width won on that shape) survives the round trip
    tuned = {"data": [[[[2, 7], {"opType": 7, "hashType": 99, "attrs": [16, 4096, 11008, 0, 0]}], {"type": 1, "data": 0.018, "impl": 2, "nb": 0}],
                      [[[2, 7], {"opType": 7, "hashType": 98, "attrs": [16, 4096, 4096, 0, 0]}], {"type": 1, "data": 0.010, "impl": 1, "nb": 1}]]}
    p.write_text(json.dumps(tuned))
    B.PerfEngine.load(str(p))
    B.PerfEngine.save(str(out))
    got = sorted((e[0][1]["hashType"], e[1]["type"], e[1]["impl"], e[1]["nb"], float(e[1]["data"])) for e in json.loads(out.read_text())["data"])
    assert got == [(98, 1, 1, 1, 0.010), (99, 1, 2, 0, 0.018)]
    B.PerfEngine.clear()


def test_native_host_core(tmp_path):
    """C++ unit tests of the host contract compiled against core.cc / operators.cc / schedule.cc alone (no CUDA): the
    LazyAllocator scenarios of the reference's test_lazy_allocator.cc, KernelRegistry / PerfEngine duplicate-key rules,
    topological sort + planner through GraphObj."""
    host = os.path.join(ROOT, "infinitensor_b200", "csrc", "host")
    exe = str(tmp_path / "test_host_core")
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    cmd = [gxx, "-O1", "-std=c++17", "-Wall", "-I" + os.path.join(ROOT, "include"), "-I" + host, "-o", exe,
           os.path.join(ROOT, "tests", "native", "test_host_core.cc")] + [os.path.join(host, f) for f in ("core.cc", "operators.cc", "schedule.cc")]
    subprocess.run(cmd, check=True, timeout=300)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and "passed" in r.stdout, r.stdout + r.stderr


def test_attention_unit_partition_properties():
    """The streaming attention kernel deals the flattened (head, chunk) units to CTAs with
         G = min(grid, total);  CTA i owns [i*total//G, (i+1)*total//G);  cta(u) = ((u+1)*G - 1)//total
       (attention.cu, attn_stream_kernel).  Re-stated here and checked exhaustively over small shapes: every unit is owned
       once, owners of a head are CONSECUTIVE CTAs (the partial-slot index blockIdx - first_cta stays below the slot
       count), and the closed form agrees with the ranges.  The first version of the kernel broke exactly this for
       total < grid."""
    for BH in (1, 2, 3, 7, 16, 33):
        for nch in (1, 2, 3, 5, 8, 16, 33):
            total = BH * nch
            for grid in (1, 2, 3, 5, 8, 31, 64, 296):
                G = min(grid, total)
                owner = {}
                for i in range(G):
                    u0, u1 = i * total // G, (i + 1) * total // G
                    assert u1 > u0, "every participating CTA owns at least one unit"
                    for u in range(u0, u1):
                        assert u not in owner
                        owner[u] = i
                        assert ((u + 1) * G - 1) // total == i
                assert len(owner) == total
                for bh in range(BH):
                    first = ((bh * nch + 1) * G - 1) // total
                    last = ((bh * nch + nch) * G - 1) // total
                    touching = sorted({owner[bh * nch + c] for c in range(nch)})
                    assert touching == list(range(first, last + 1))
                    assert last - first + 1 <= nch  # slots_per_head >= chunks per head covers the slot index


def test_skinny_gemm_split_k_partition_properties():
    """gemm_skinny.cu / gemm_tc.cu split-K: splitk = clamp(target // tiles, 1, 8), at least 4 k-tiles per split, then
    `per = ceil(ktiles / splitk)` and `splitk = ceil(ktiles / per)` so that NO split is empty and the splits cover K once."""
    for tiles in (1, 6, 32, 64, 172, 192, 250, 344, 500):
        for ktiles in (1, 2, 3, 4, 8, 16, 43, 64, 172):
            splitk = max(1, min(296 // tiles, 8))
            splitk = min(splitk, max(1, ktiles // 4))
            per = -(-ktiles // splitk)
            splitk = -(-ktiles // per)
            covered = []
            for s in range(splitk):
                b, e = s * per, min(ktiles, (s + 1) * per)
                assert e > b, (tiles, ktiles, splitk, per)
                covered += list(range(b, e))
            assert covered == list(range(ktiles)) and 1 <= splitk <= 8


def test_attention_unit_partition_with_per_row_positions():
    """Per-row positions (ITB_POS_PER_ROW): row b has its own chunk count, the units are the concatenation of every row's
    H x nch_b (head, chunk) grid and `pre[b]` = units before row b (attention.cu: s_pre).  Same properties as the uniform case:
    every unit owned once, a head's owners are consecutive CTAs, the closed forms for first / last CTA of a head hold."""
    rng = np.random.default_rng(0)
    for B, H in ((1, 1), (3, 2), (16, 4), (5, 9)):
        for _ in range(6):
            nch = rng.integers(1, 17, size=B).tolist()
            pre = [0]
            for b in range(B):
                pre.append(pre[-1] + H * nch[b])
            total = pre[-1]
            for grid in (1, 3, 8, 31, 296):
                G = min(grid, total)
                owner = {}
                for i in range(G):
                    u0, u1 = i * total // G, (i + 1) * total // G
                    assert u1 > u0
                    b = 0
                    while b + 1 < B and pre[b + 1] <= u0:
                        b += 1
                    assert pre[b] <= u0 < pre[b + 1]  # the kernel's starting-row search
                    for u in range(u0, u1):
                        owner[u] = i
                assert len(owner) == total
                for b in range(B):
                    for hh in range(H):
                        hu0 = pre[b] + hh * nch[b]
                        first, last = ((hu0 + 1) * G - 1) // total, ((hu0 + nch[b]) * G - 1) // total
                        assert sorted({owner[hu0 + c] for c in range(nch[b])}) == list(range(first, last + 1))
                        assert last - first + 1 <= nch[b]


def test_every_kernel_waits_for_its_predecessor():
    """Programmatic dependent launch invariant the peer-memory all-reduce's epoch hand-over relies on (allreduce.cu header):
    every __global__ kernel of the library that triggers its dependents also executes griddepcontrol.wait, so completion is
    transitive along the stream.  Checked on the sources: each kernel body mentions pdl_wait() or calls a helper that does."""
    kdir = os.path.join(ROOT, "infinitensor_b200", "csrc", "kernels")
    bad = []
    for f in sorted(os.listdir(kdir)):
        if not f.endswith(".cu"):
            continue
        src = open(os.path.join(kdir, f)).read()
        parts = re.split(r"__global__", src)
        for body in parts[1:]:
            name = re.search(r"(\w+)\s*\(", body.split("{", 1)[0].replace("__launch_bounds__", ""))
            # the kernel's text runs to the next top-level `}` at column 0
            end = body.find("\n}\n")
            text = body[: end if end > 0 else len(body)]
            if "pdl_trigger" in text and "pdl_wait" not in text:
                bad.append(f"{f}:{name.group(1) if name else '?'}")
            if "pdl_trigger" not in text and "pdl_wait" not in text:
                bad.append(f"{f}:{name.group(1) if name else '?'} (no PDL calls at all)")
    assert not bad, bad


def test_depth_to_space_shapes_and_oracle(B):
    """DepthToSpace (reference src/operators/transpose.cc:53-107): shape rule on the host core; the oracle handler follows the
    ONNX definition -- checked against the worked example of the ONNX operator documentation (DCR mode)."""
    from oracle.graph_oracle import OracleHandler
    h = B.GraphHandler(B.HostPlanRuntime())
    assert h.depthToSpace(h.tensor([1, 8, 2, 3], 1), None, 2, "DCR").shape() == [1, 2, 4, 6]
    assert h.depthToSpace(h.tensor([2, 16, 5, 7], 10), None, 2, "CRD").shape() == [2, 4, 10, 14]
    with pytest.raises(RuntimeError):
        h.depthToSpace(h.tensor([1, 6, 2, 2], 1), None, 2, "DCR")
    x = np.arange(48, dtype=np.float32).reshape(1, 8, 2, 3)
    want = np.array([[[[0., 18., 1., 19., 2., 20.], [36., 54., 37., 55., 38., 56.], [3., 21., 4., 22., 5., 23.], [39., 57., 40., 58., 41., 59.]],
                      [[9., 27., 10., 28., 11., 29.], [45., 63., 46., 64., 47., 65.], [12., 30., 13., 31., 14., 32.], [48., 66., 49., 67., 50., 68.]]]])
    x2 = np.array([[[[0., 1., 2.], [3., 4., 5.]], [[9., 10., 11.], [12., 13., 14.]], [[18., 19., 20.], [21., 22., 23.]], [[27., 28., 29.], [30., 31., 32.]],
                    [[36., 37., 38.], [39., 40., 41.]], [[45., 46., 47.], [48., 49., 50.]], [[54., 55., 56.], [57., 58., 59.]], [[63., 64., 65.], [66., 67., 68.]]]],
                  np.float32)
    oh = OracleHandler()
    t = oh.tensor([1, 8, 2, 3], 1)
    y = oh.depthToSpace(t, None, 2, "DCR")
    t.copyin_numpy(x2)
    oh.run()
    assert np.array_equal(np.asarray(y.f32()).reshape(want.shape), want)
    del x


def test_prefill_attention_schedule(B, monkeypatch):
    """GPT-2's attention block -- Transpose(k) -> MatMul -> Div -> Add(mask) -> Softmax -> MatMul -- becomes ONE PrefillAttention
    step per layer for f16 / bf16 (SURVEY 8(f-3)); fp32 graphs, 32-wide heads and ITB_FUSION_MASK without bit 8 keep the operators."""
    from infinitensor_b200 import graphs as G
    rt = B.HostPlanRuntime()
    cfg = G.GPT2Config(layers=2, d_model=128, heads=2, ffn=256, vocab=500, n_pos=64, seq=16, batch=1, dtype=10)
    h = B.GraphHandler(rt)
    G.build_gpt2(h, cfg)
    sc = h.schedule()
    assert sum(s.startswith("PrefillAttention:") and s.endswith("Transpose+MatMul+Div+Add+Softmax+MatMul+Transpose+Reshape") for s in sc) == 2, sc
    assert not any(s in ("Single:Softmax", "Single:Div") for s in sc)
    h.data_malloc()
    monkeypatch.setenv("ITB_FUSION_MASK", str(127 | 256))  # without bit 11: the bare chain
    hb = B.GraphHandler(rt)
    G.build_gpt2(hb, cfg)
    assert hb.schedule().count("PrefillAttention:Transpose+MatMul+Div+Add+Softmax+MatMul") == 2
    monkeypatch.delenv("ITB_FUSION_MASK")
    h32 = B.GraphHandler(rt)
    G.build_gpt2(h32, G.GPT2Config(layers=1, d_model=128, heads=2, ffn=256, vocab=500, n_pos=64, seq=16, batch=1, dtype=1))
    assert not any(s.startswith("PrefillAttention") for s in h32.schedule())
    hs = B.GraphHandler(rt)
    G.build_gpt2(hs, G.GPT2Config.tiny(10))  # 32-wide heads: not taken by the tensor-core kernel
    assert not any(s.startswith("PrefillAttention") for s in hs.schedule())
    monkeypatch.setenv("ITB_FUSION_MASK", "127")
    hm = B.GraphHandler(rt)
    G.build_gpt2(hm, cfg)
    assert not any(s.startswith("PrefillAttention") for s in hm.schedule())
