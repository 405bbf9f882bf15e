"""Grouped-query decode attention on the GPU: it_b200_attention_kvcache_gqa against the oracle's AttentionKVCache run
per group member (tests/llama_oracle.py), and whole GQA Llama graphs against the graph oracle with that rule."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import oracle
from tests.llama_oracle import attention_kvcache_gqa, oracle_graph, run_llama_parity

F32, F16, BF16 = 1, 10, 16
TOL = {F32: 1e-5, F16: 1e-3, BF16: 1e-2}  # as test_attention_parity (SURVEY 8(c))
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def K():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from tests import kernel_harness
    return kernel_harness


def rnd(shape, seed, dt, scale=0.5):
    return oracle.round_to(np.random.default_rng(seed).standard_normal(shape).astype(np.float32) * np.float32(scale), dt)


def close(got, exp, rel, abs_):
    np.testing.assert_allclose(np.asarray(got, np.float64).ravel(), np.asarray(exp, np.float64).ravel(), rtol=rel, atol=abs_)


def gqa(K, kc, vc, q, k, v, pos, dt, flags=0, rope_pos=None, entry="gqa"):
    """one launch; returns (out, k cache, v cache) as float32.  entry="equal" calls it_b200_attention_kvcache instead."""
    import torch
    L = K.L
    kcd, vcd = K.dev(kc, dt), K.dev(vc, dt)
    qd, kd, vd = K.dev(q, dt), K.dev(k, dt), K.dev(v, dt)
    B, Hkv, Smax, D = kc.shape
    Hq = q.shape[1]
    if np.ndim(pos) > 0:
        flags |= 0x100
    pd = K.raw(np.atleast_1d(np.asarray(pos)).astype(np.int64))
    rp = None if rope_pos is None else K.raw(np.asarray(rope_pos, np.int64))
    out = torch.empty_like(qd)
    wsb = L.lib.it_b200_attention_kvcache_workspace(B, Hq, Smax, D)
    ws = torch.empty(max(int(wsb), 16), dtype=torch.uint8, device="cuda")
    if entry == "gqa":
        L.check(L.lib.it_b200_attention_kvcache_gqa(dt, K.ptr(kcd), K.ptr(vcd), K.ptr(qd), K.ptr(kd), K.ptr(vd), K.ptr(pd),
                                                    7 | flags, K.ptr(rp), 7, K.ptr(out), B, Hq, Hkv, Smax, D, K.ptr(ws),
                                                    int(wsb), K.stream()))
    else:
        assert Hq == Hkv and rope_pos is None
        L.check(L.lib.it_b200_attention_kvcache(dt, K.ptr(kcd), K.ptr(vcd), K.ptr(qd), K.ptr(kd), K.ptr(vd), K.ptr(pd), 7 | flags,
                                                K.ptr(out), B, Hq, Smax, D, K.ptr(ws), int(wsb), K.stream()))
    K.sync()
    return K.host(out), K.host(kcd), K.host(vcd)


def inputs(B, Hq, Hkv, S, dt):
    kc, vc = rnd((B, Hkv, S, 128), 28, dt), rnd((B, Hkv, S, 128), 29, dt)
    q, k, v = rnd((B, Hq, 1, 128), 30, dt), rnd((B, Hkv, 1, 128), 31, dt), rnd((B, Hkv, 1, 128), 32, dt)
    return kc, vc, q, k, v


# G = 48, 64 and 40 (two query groups of up to 32 heads per KV head): multi-query layers with more than 32 heads
SHAPES = [(2, 8, 2, 64, 0), (2, 8, 2, 64, 37), (16, 32, 8, 1024, 511), (1, 64, 8, 2048, 2047), (3, 28, 4, 512, 257),
          (2, 16, 1, 256, 100), (1, 32, 1, 128, 64), (7, 6, 3, 512, 300), (2, 48, 1, 256, 100), (1, 64, 1, 512, 300),
          (2, 80, 2, 128, 64)]


@pytest.mark.parametrize("dt", [F32, F16, BF16])
@pytest.mark.parametrize("B,Hq,Hkv,S,pos", SHAPES)
def test_gqa_attention_parity(K, B, Hq, Hkv, S, pos, dt):
    kc, vc, q, k, v = inputs(B, Hq, Hkv, S, dt)
    kc_ref, vc_ref = kc.copy(), vc.copy()
    ref = attention_kvcache_gqa(kc_ref, vc_ref, q, k, v, pos, dt)
    out, kc_got, vc_got = gqa(K, kc, vc, q, k, v, pos, dt)
    close(out, ref, TOL[dt], TOL[dt] * 0.05)
    assert np.array_equal(kc_got, kc_ref) and np.array_equal(vc_got, vc_ref)  # append is bit-exact, rest untouched


@pytest.mark.parametrize("dt", [F32, BF16])
@pytest.mark.parametrize("B,Hq,Hkv,S,poss", [(4, 8, 2, 256, [0, 37, 255, 64]), (16, 32, 8, 1024, None),
                                             (3, 28, 4, 128, [127, 0, 63]), (5, 32, 1, 512, [200, 200, 1, 511, 300]),
                                             (3, 48, 1, 256, [10, 255, 0])])
def test_gqa_attention_per_row_positions(K, B, Hq, Hkv, S, poss, dt):
    """ITB_POS_PER_ROW with units counted over the KV heads; ITB_POS_IN_STEP must not change a bit."""
    if poss is None:
        poss = np.random.default_rng(5).integers(0, S, size=B).tolist()
    kc, vc, q, k, v = inputs(B, Hq, Hkv, S, dt)
    kc_ref, vc_ref = kc.copy(), vc.copy()
    ref = attention_kvcache_gqa(kc_ref, vc_ref, q, k, v, poss, dt)
    out, kc_got, vc_got = gqa(K, kc, vc, q, k, v, poss, dt)
    close(out, ref, TOL[dt], TOL[dt] * 0.05)
    assert np.array_equal(kc_got, kc_ref) and np.array_equal(vc_got, vc_ref)
    out2, kc2, vc2 = gqa(K, kc, vc, q, k, v, poss, dt, flags=0x200)
    assert np.array_equal(out2, out) and np.array_equal(kc2, kc_got) and np.array_equal(vc2, vc_got)


@pytest.mark.parametrize("dt", [F32, F16, BF16])
@pytest.mark.parametrize("B,Hq,Hkv,S,pos", [(2, 8, 2, 64, 37), (16, 32, 8, 1024, 511), (3, 28, 4, 512, 257),
                                           (2, 48, 1, 256, 100)])
def test_gqa_attention_rope_folded(K, B, Hq, Hkv, S, pos, dt):
    """RoPE folded in: q rotated per query head, k per KV head (the rotated k is appended), vs the oracle's RoPE followed
    by the grouped attention.  The kernel's cosf / sinf differ from the oracle's in the last bit, so the appended row is
    compared with the storage type's tolerance."""
    kc, vc, q, k, v = inputs(B, Hq, Hkv, S, dt)
    rpos = (np.arange(B, dtype=np.int64) * 3 + pos) % 4096
    qr = oracle.rope(rpos.reshape(B, 1), q.reshape(B, 1, Hq * 128), 128, dt).reshape(q.shape)
    kr = oracle.rope(rpos.reshape(B, 1), k.reshape(B, 1, Hkv * 128), 128, dt).reshape(k.shape)
    kc_ref, vc_ref = kc.copy(), vc.copy()
    ref = attention_kvcache_gqa(kc_ref, vc_ref, qr, kr, v, pos, dt)
    out, kc_got, vc_got = gqa(K, kc, vc, q, k, v, pos, dt, rope_pos=rpos)
    tol = max(TOL[dt], 4e-3 if dt == F16 else TOL[dt])
    close(out, ref, tol, tol * 0.05)
    rows = np.arange(S) != pos
    assert np.array_equal(kc_got[:, :, rows], kc_ref[:, :, rows]) and np.array_equal(vc_got, vc_ref)
    # fp32: cosf / sinf of angles up to ~500 rad differ from the oracle's by a few 1e-5
    close(kc_got[:, :, pos], kc_ref[:, :, pos], tol if dt != F32 else 1e-3, tol if dt != F32 else 1e-4)


@pytest.mark.parametrize("dt", [F32, BF16])
def test_gqa_entry_with_equal_heads_is_the_existing_launch(K, dt):
    """it_b200_attention_kvcache_gqa with Hq == Hkv routes to the existing decode kernel: identical bits."""
    kc, vc, q, k, v = inputs(7, 9, 9, 512, dt)
    a = gqa(K, kc, vc, q, k, v, 257, dt)
    b = gqa(K, kc, vc, q, k, v, 257, dt, entry="equal")
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def test_gqa_entry_rejects_bad_groups(K):
    import torch
    L = K.L
    x = torch.zeros(1 << 16, dtype=torch.float32, device="cuda")
    ws = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    with pytest.raises(RuntimeError):  # 12 query heads over 5 KV heads
        L.check(L.lib.it_b200_attention_kvcache_gqa(1, K.ptr(x), K.ptr(x), K.ptr(x), K.ptr(x), K.ptr(x), K.ptr(x), 7, None,
                                                    7, K.ptr(x), 1, 12, 5, 4, 128, K.ptr(ws), 1 << 20, K.stream()))
    # no heads: a no-op, as it always was for it_b200_attention_kvcache
    assert L.lib.it_b200_attention_kvcache(1, K.ptr(x), K.ptr(x), K.ptr(x), K.ptr(x), K.ptr(x), K.ptr(x), 7, K.ptr(x), 1, 0,
                                           4, 128, K.ptr(ws), 1 << 20, K.stream()) == 0


def _gqa_cfg(dtype, kv_heads, layers=2, d=512, heads=4, batch=16, s_max=64, ffn=1408, vocab=512):
    from infinitensor_b200 import graphs as G
    return G.LlamaConfig(layers=layers, d_model=d, heads=heads, kv_heads=kv_heads, head_dim=128, ffn=ffn, vocab=vocab,
                         s_max=s_max, batch=batch, dtype=dtype)


@pytest.mark.parametrize("dtype", [BF16, F32])
@pytest.mark.parametrize("kv_heads", [2, 1])
@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("cudagraph", [True, False])
def test_gqa_llama_graph_parity(dtype, kv_heads, fused, cudagraph):
    env = None if fused else {"ITB_NO_FUSION": "1"}
    _, _, sched = run_llama_parity(_gqa_cfg(dtype, kv_heads), pos=5, steps=2, cudagraph=cudagraph, env=env)
    if fused:
        assert sum(s.startswith("AttentionRope") for s in sched) == 2


def test_gqa_llama3_width_graph_parity():
    """two Llama-3-8B-width layers (32 query heads over 8 KV heads) at B 16, p 511"""
    from infinitensor_b200 import graphs as G
    full = G.LlamaConfig.llama3_8b()
    cfg = G.LlamaConfig(layers=2, d_model=full.d_model, heads=full.heads, kv_heads=full.kv_heads, head_dim=128, ffn=full.ffn,
                        vocab=2048, s_max=1024, batch=16, dtype=BF16)
    run_llama_parity(cfg, pos=511, steps=1)


def _ngpu():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


def test_gqa_tensor_parallel_two_gpus(tmp_path):
    """tools/tp_worker.py with 8 query heads over 2 KV heads: each rank holds 4 query heads over 1 KV head"""
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    from infinitensor_b200 import graphs as G
    out = str(tmp_path / "tp")
    env = dict(os.environ, TP_OUT=out, TP_DTYPE="16", TP_KV_HEADS="2", MASTER_ADDR="127.0.0.1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29619", os.path.join(ROOT, "tools", "tp_worker.py")]
    subprocess.run(cmd, check=True, env=env, cwd=ROOT, timeout=600)
    cfg = G.LlamaConfig(layers=2, d_model=1024, heads=8, kv_heads=2, head_dim=128, ffn=2816, vocab=2048, s_max=64, batch=16,
                        dtype=BF16)
    oh, g = oracle_graph(cfg)
    refs = []
    for step in range(3):
        g.input_ids.copyin_numpy((np.arange(cfg.batch, dtype=np.int64).reshape(-1, 1) * 7 + step) % cfg.vocab)
        g.position_ids.copyin_numpy(np.full((cfg.batch, 1), 9 + step, np.int64))
        oh.run()
        refs.append(g.logits.f32().copy())
    ref = np.stack(refs).astype(np.float64)
    for mode in ("p2p", "nccl"):
        got = [np.load(f"{out}.{mode}.{r}.npy").astype(np.float64) for r in range(2)]
        assert np.array_equal(got[0], got[1]), f"{mode}: ranks disagree"
        err = np.abs(got[0] - ref).max() / np.abs(ref).max()
        assert err < 3e-2, f"{mode}: rel-to-max error {err:.3e}"
