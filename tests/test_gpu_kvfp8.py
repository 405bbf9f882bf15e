"""Decode attention over an FP8 E4M3 KV cache on the GPU: it_b200_attention_kvcache_fp8 against the float64 oracle of
tests/kvfp8_oracle.py (per element, with its bound), the appended codes bit for bit, RoPE folded against RoPE + the unfused
launcher, and whole Llama graphs with LlamaConfig(kv_fp8=True) against the graph oracle with the same rule
(tests/llama_oracle.py)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import oracle
from tests import kvfp8_oracle as KV
from tests.llama_oracle import run_llama_parity

F16, BF16 = 10, 16
NAN = np.uint8(0x7F)
POS_PER_ROW, POS_IN_STEP = 0x100, 0x200


@pytest.fixture(scope="module")
def K():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from tests import kernel_harness
    return kernel_harness


def rnd(shape, seed, dt, scale=0.5):
    return oracle.round_to(np.random.default_rng(seed).standard_normal(shape).astype(np.float32) * np.float32(scale), dt)


def launch(K, kc, vc, ksc, vsc, q, k, v, pos, dt, flags=0, rope_pos=None):
    """One it_b200_attention_kvcache_fp8 launch on code caches (uint8); returns (out float32, k codes, v codes)."""
    import torch
    L = K.L
    kcd, vcd = K.raw(kc), K.raw(vc)
    ksd, vsd = K.raw(np.asarray(ksc, np.float32)), K.raw(np.asarray(vsc, np.float32))
    qd, kd, vd = K.dev(q, dt), K.dev(k, dt), K.dev(v, dt)
    B, Hkv, Smax, D = kc.shape
    Hq = q.shape[1]
    if np.ndim(pos) > 0:
        flags |= POS_PER_ROW
    pd = K.raw(np.atleast_1d(np.asarray(pos)).astype(np.int64))
    rp = None if rope_pos is None else K.raw(np.asarray(rope_pos, np.int64))
    out = torch.full_like(qd, float("nan"))
    wsb = L.lib.it_b200_attention_kvcache_workspace(B, Hq, Smax, D)
    ws = torch.full((max(int(wsb), 16),), 0xFF, dtype=torch.uint8, device="cuda")  # NaN in every fp32 slot
    L.check(L.lib.it_b200_attention_kvcache_fp8(dt, K.ptr(kcd), K.ptr(vcd), K.ptr(ksd), K.ptr(vsd), K.ptr(qd), K.ptr(kd), K.ptr(vd),
                                                K.ptr(pd), 7 | flags, K.ptr(rp), 7, K.ptr(out), B, Hq, Hkv, Smax, D, K.ptr(ws),
                                                int(wsb), K.stream()))
    K.sync()
    return K.host(out), K.host(kcd), K.host(vcd)


def make(B, Hq, Hkv, S, D, dt, seed=0, qscale=0.5):
    kc, ksc = KV.fill(rnd((B, Hkv, S, D), seed + 1, dt))
    vc, vsc = KV.fill(rnd((B, Hkv, S, D), seed + 2, dt))
    q = rnd((B, Hq, 1, D), seed + 3, dt, qscale)
    k, v = rnd((B, Hkv, 1, D), seed + 4, dt), rnd((B, Hkv, 1, D), seed + 5, dt)
    return kc, vc, ksc, vsc, q, k, v


def check(K, B, Hq, Hkv, S, D, pos, dt, flags=0, qscale=0.5, seed=0):
    kc, vc, ksc, vsc, q, k, v = make(B, Hq, Hkv, S, D, dt, seed, qscale)
    posv = np.broadcast_to(np.asarray(pos, np.int64), (B,)) if np.ndim(pos) else np.full(B, int(pos), np.int64)
    # rows past each position are NaN codes: the kernel must never read them, and must not write them
    for b in range(B):
        kc[b, :, posv[b] + 1:] = NAN
        vc[b, :, posv[b] + 1:] = NAN
    kc_ref, vc_ref = kc.copy(), vc.copy()
    KV.append(kc_ref, vc_ref, k, v, ksc, vsc, posv)
    ref, bound = KV.attention(kc_ref, vc_ref, ksc, vsc, q, posv, dt)
    for rep in range(2):  # twice: the append and the tickets must leave nothing behind
        got, kg, vg = launch(K, kc, vc, ksc, vsc, q, k, v, pos, dt, flags)
        assert np.array_equal(kg, kc_ref) and np.array_equal(vg, vc_ref), f"run {rep}: appended codes or other rows differ"
        bad = KV.violations(got, ref, bound)
        assert len(bad) == 0, (f"run {rep}: {len(bad)} elements outside the bound, first {tuple(bad[0])}: "
                               f"got {got[tuple(bad[0])]} ref {ref[tuple(bad[0])]} bound {bound[tuple(bad[0])]}")


# (B, Hq, Hkv, S_max, D, pos): G 1 / 2 / 4 / 8 / 32 / 48 (one and two query tiles), p at 0, at chunk edges (128 rows per chunk
# at D = 128, 256 at D = 64, streaming and grouped-query alike), 511 and 4095; small and large B x heads (every CTA split)
CASES = [
    (2, 4, 4, 256, 128, 0), (2, 4, 4, 512, 128, 127), (2, 4, 4, 512, 128, 128), (1, 2, 2, 1024, 128, 255),
    (16, 32, 32, 1024, 128, 511), (1, 1, 1, 4096, 128, 4095), (4, 32, 32, 4096, 128, 4095),
    (2, 4, 4, 512, 64, 255), (2, 4, 4, 512, 64, 256), (8, 32, 32, 1024, 64, 511), (1, 2, 2, 4096, 64, 4095),
    (2, 8, 4, 512, 128, 0), (2, 8, 4, 512, 128, 128), (16, 32, 8, 1024, 128, 511), (1, 32, 8, 4096, 128, 4095),
    (3, 16, 4, 512, 128, 257), (2, 64, 8, 1024, 128, 300), (2, 32, 1, 512, 128, 200), (2, 48, 1, 512, 128, 100),
    (2, 32, 4, 512, 64, 255), (2, 32, 4, 512, 64, 256), (16, 32, 4, 1024, 64, 511), (1, 32, 4, 4096, 64, 4095),
    (2, 96, 2, 512, 64, 300), (1, 8, 1, 128, 64, 64),
]


@pytest.mark.parametrize("dt", [F16, BF16])
@pytest.mark.parametrize("B,Hq,Hkv,S,D,pos", CASES)
def test_fp8_attention_vs_float64(K, B, Hq, Hkv, S, D, pos, dt):
    check(K, B, Hq, Hkv, S, D, pos, dt)


@pytest.mark.parametrize("dt", [F16, BF16])
@pytest.mark.parametrize("Hq,Hkv,D", [(8, 8, 128), (32, 8, 128), (8, 8, 64), (32, 4, 64), (48, 1, 128)])
def test_fp8_per_row_positions_and_in_step(K, Hq, Hkv, D, dt):
    pos = np.array([0, 127, 128, 511, 300, 1, 256, 1023], np.int64)
    check(K, 8, Hq, Hkv, 1024, D, pos, dt)
    check(K, 8, Hq, Hkv, 1024, D, pos, dt, flags=POS_IN_STEP)
    check(K, 3, Hq, Hkv, 512, D, 200, dt, flags=POS_IN_STEP)


@pytest.mark.parametrize("dt", [F16, BF16])
@pytest.mark.parametrize("Hq,Hkv,D,pos", [(4, 4, 128, 511), (32, 8, 128, 4095), (4, 4, 64, 1000), (32, 4, 64, 511)])
def test_fp8_large_score_range(K, Hq, Hkv, D, pos, dt):
    # q 16x larger: scores spread over tens of units, the softmax concentrates on a few rows of each head
    check(K, 2, Hq, Hkv, max(1024, pos + 1), D, pos, dt, qscale=8.0, seed=7)


def test_fp8_position_clamped(K):
    # positions past S_max - 1 append into (and attend up to) the last row, as for 16-bit caches
    kc, vc, ksc, vsc, q, k, v = make(2, 8, 2, 256, 128, BF16)
    got, kg, _ = launch(K, kc, vc, ksc, vsc, q, k, v, 1000, BF16)
    kc_ref, vc_ref = kc.copy(), vc.copy()
    KV.append(kc_ref, vc_ref, k, v, ksc, vsc, [255, 255])
    ref, bound = KV.attention(kc_ref, vc_ref, ksc, vsc, q, [255, 255], BF16)
    assert np.array_equal(kg, kc_ref) and len(KV.violations(got, ref, bound)) == 0


def rope_dev(K, pos, x, D, dt):
    """it_b200_rope over [B, 1, H*D] with head width D"""
    import torch
    xd = K.dev(x, dt)
    pd = K.raw(np.asarray(pos, np.int64))
    y = torch.empty_like(xd)
    B, S, dm = x.shape
    K.L.check(K.L.lib.it_b200_rope(dt, K.ptr(pd), 7, K.ptr(xd), K.ptr(y), B, S, dm, D, K.stream()))
    K.sync()
    return K.host(y)


@pytest.mark.parametrize("dt", [F16, BF16])
@pytest.mark.parametrize("Hq,Hkv,D", [(8, 8, 128), (32, 8, 128), (8, 8, 64), (32, 4, 64), (48, 1, 128)])
def test_fp8_rope_folded_matches_unfused(K, Hq, Hkv, D, dt):
    B, S = 3, 1024
    kc, vc, ksc, vsc, q, k, v = make(B, Hq, Hkv, S, D, dt, seed=11)
    pos = np.array([5, 700, 1023], np.int64)
    qr = rope_dev(K, pos.reshape(B, 1), q.reshape(B, 1, Hq * D), D, dt).reshape(B, Hq, 1, D)
    kr = rope_dev(K, pos.reshape(B, 1), k.reshape(B, 1, Hkv * D), D, dt).reshape(B, Hkv, 1, D)
    got_u, kg_u, vg_u = launch(K, kc, vc, ksc, vsc, qr, kr, v, pos, dt)
    got_f, kg_f, vg_f = launch(K, kc, vc, ksc, vsc, q, k, v, pos, dt, rope_pos=pos)
    assert np.array_equal(kg_f, kg_u) and np.array_equal(vg_f, vg_u), "appended codes differ"
    assert np.array_equal(got_f, got_u), "folded RoPE output differs from RoPE + the unfused launcher"


def test_fp8_refusals(K):
    import torch
    L = K.L
    kc, vc, ksc, vsc, q, k, v = make(1, 4, 4, 128, 128, BF16)
    args = lambda dt, ks: (dt, K.ptr(K.raw(kc)), K.ptr(K.raw(vc)), ks, K.ptr(K.raw(vsc)), K.ptr(K.dev(q, BF16)),
                           K.ptr(K.dev(k, BF16)), K.ptr(K.dev(v, BF16)), K.ptr(K.raw(np.array([3], np.int64))), 7, None, 7,
                           K.ptr(torch.empty(4 * 128, dtype=torch.bfloat16, device="cuda")), 1, 4, 4, 128, 128,
                           K.ptr(torch.empty(1 << 20, dtype=torch.uint8, device="cuda")), 1 << 20, K.stream())
    assert L.lib.it_b200_attention_kvcache_fp8(*args(1, K.ptr(K.raw(ksc)))) != 0, "fp32 activations must be refused"
    assert L.lib.it_b200_attention_kvcache_fp8(*args(BF16, None)) != 0, "a missing k_scale must be refused"


# ---------------------------------------------------------------------------------------------------- whole graphs
def run_graph(cfg, pos=5, steps=3, cudagraph=True, fused=True):
    """The device graph with FP8 caches against the graph oracle (tests/llama_oracle.py); fused=False disables the
    RoPE -> attention fold (ITB_FUSION_MASK without bit 5).  Returns the schedule."""
    env = None if fused else {"ITB_FUSION_MASK": str((127 | 256 | 512 | 1024 | 2048) & ~32)}
    return run_llama_parity(cfg, pos, steps, cudagraph, env=env, tol=3e-2)[2]


@pytest.mark.parametrize("cudagraph", [False, True])
@pytest.mark.parametrize("fused", [True, False])
def test_fp8_llama_tiny(K, cudagraph, fused):
    from infinitensor_b200 import graphs as G
    sched = run_graph(G.LlamaConfig.tiny(kv_fp8=True), cudagraph=cudagraph, fused=fused)
    assert ("AttentionRope" in str(sched)) == fused


@pytest.mark.parametrize("cudagraph", [False, True])
def test_fp8_llama_tinyllama_width(K, cudagraph):
    from infinitensor_b200 import graphs as G
    run_graph(G.LlamaConfig.tinyllama_1b(batch=4, s_max=512, layers=2, kv_fp8=True), pos=300, cudagraph=cudagraph)


@pytest.mark.parametrize("fused", [True, False])
def test_fp8_llama3_8b_width_two_layers(K, fused):
    from infinitensor_b200 import graphs as G
    cfg = G.LlamaConfig.llama3_8b(batch=2, s_max=512, layers=2, kv_fp8=True)
    cfg.vocab = 4096  # the head's width does not bear on the attention; keeps the oracle's logits GEMM small
    run_graph(cfg, pos=200, steps=2, fused=fused)


def profiled_kernel_names():
    """kernel names recorded by torch.profiler (CUDA activity only) for one streaming and one grouped-query FP8 launch"""
    import torch
    from tests import kernel_harness as K
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        check(K, 2, 4, 4, 512, 128, 300, BF16)
        check(K, 2, 32, 8, 512, 128, 300, BF16)
        torch.cuda.synchronize()
    return sorted({e.name for e in prof.events() if "CUDA" in str(e.device_type)})


def test_fp8_kernel_names_in_profile(K):
    """In a child process, as the other profiler checks: a profiler session in the test process loses kernel records of a
    later one in a full-suite run."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = "import json; from tests.test_gpu_kvfp8 import profiled_kernel_names as f; print(json.dumps(f()))"
    r = subprocess.run([sys.executable, "-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    names = json.loads(r.stdout.strip().splitlines()[-1])
    if not names:
        pytest.skip("the profiler recorded no CUDA kernel events (CUPTI activity tracing unavailable)")
    assert any("attn_stream_kv8_kernel" in n for n in names) and any("attn_gqa_kv8_kernel" in n for n in names), names
