"""RoPE with a model's own frequencies on the H100: it_b200_rope_freq against float64 up to position 131071, the RoPE folded
into decode attention with an inv_freq table bit for bit against RoPE-with-table then the unfused kernel (16-bit and FP8
caches, every query-group shape), and a reduced-width Llama-3.1-style graph at long context against the test oracle."""
import dataclasses

import numpy as np
import pytest

import oracle
from tests import llama_oracle as LO
from tests import rope64
from tests import rope_oracle as RO

F32, F16, BF16, I32, I64, U32 = 1, 10, 16, 6, 7, 12
LLAMA31 = {"type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
           "original_max_position_embeddings": 8192}
TABLES = {"base1e4": (10000.0, None), "base5e5": (500000.0, None), "base1e6": (1000000.0, None), "llama31": (500000.0, LLAMA31)}
POS_NP = {I64: np.int64, I32: np.int32, U32: np.uint32}


@pytest.fixture(scope="module")
def K():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from tests import kernel_harness
    return kernel_harness


def table(D, name):
    from infinitensor_b200 import graphs as G
    return G.rope_inv_freq(D, *TABLES[name])


def rope_freq_dev(K, dt, x, pos, pos_code, inv, S=1):
    """it_b200_rope_freq on a device tensor x [B * S, dim_model] taken as [B, S, dim_model], heads of 2 * len(inv)"""
    import torch
    y = torch.empty_like(x)
    (rows, dm), D = x.shape, inv.numel() * 2
    K.L.check(K.L.lib.it_b200_rope_freq(dt, K.ptr(pos), pos_code, K.ptr(x), K.ptr(y), rows // S, S, dm, D, K.ptr(inv), F32,
                                        inv.numel(), K.stream()))
    K.sync()
    return y


# ---------------------------------------------------------------------------------------------------- RoPE vs float64
@pytest.mark.gpu
@pytest.mark.parametrize("pos_code", [I64, I32, U32], ids=["i64", "i32", "u32"])
@pytest.mark.parametrize("name", sorted(TABLES))
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dt", [F32, F16, BF16], ids=["fp32", "f16", "bf16"])
def test_rope_freq_float64(K, dt, D, name, pos_code):
    """every element equals the float64 result rounded as the kernel rounds it, or where cosf / sinf's error reaches a rounding
    point of T, lies between the two candidates; positions 0 .. 131071"""
    pos, x = rope64.case(D, dt)
    inv = table(D, name)
    b = rope64.Bound(pos, x, inv, D, dt)
    y = rope_freq_dev(K, dt, K.dev(x, dt), K.raw(pos.astype(POS_NP[pos_code])), pos_code, K.raw(inv))
    got = K.host(y)
    bad = b.outside(got)
    if bad.any():
        i, j = np.argwhere(bad)[0]
        pytest.fail(f"{int(bad.sum())} elements outside; first (p {pos[i]}, col {j}): got {got[i, j]!r}, nominal "
                    f"{b.nominal[i, j]!r}, candidates {b.lo[i, j]!r} .. {b.hi[i, j]!r}")
    assert b.share <= (1.0 if dt == F32 else 0.05)
    # the same kernel over [B, S, dim_model] with S > 1 (a prompt chunk's layout) gives the same bits
    y2 = rope_freq_dev(K, dt, K.dev(x, dt), K.raw(pos.astype(POS_NP[pos_code])), pos_code, K.raw(inv), S=8)
    assert np.array_equal(K.host(y2), got)


# ---------------------------------------------------------------------------------------------------- folded = unfused
def bits(t):
    import torch
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()]).cpu().numpy()


FOLD_CASES = {  # B, Hq, Hkv, S_max, cache positions
    "g1": (3, 8, 8, 320, (5, 300, 64)),
    "g4": (2, 32, 8, 600, (511, 3, 200)),
    "g8": (2, 32, 4, 300, (130, 299, 0)),
    "g32": (1, 64, 2, 260, (257,)),
    "g48": (2, 96, 2, 400, (399, 17)),
}


def fold_inputs(K, case, dt, D, fp8, seed=0):
    from infinitensor_b200 import graphs as G
    B, Hq, Hkv, S, cpos = FOLD_CASES[case]
    rng = np.random.default_rng([seed, D, dt, Hq])
    rnd = lambda shape: oracle.round_to((rng.standard_normal(shape) * 0.7).astype(np.float32), dt)
    if fp8:
        kc = K.raw(G.e4m3_codes_host(rng.standard_normal((B, Hkv, S, D)).astype(np.float32) * 100))
        vc = K.raw(G.e4m3_codes_host(rng.standard_normal((B, Hkv, S, D)).astype(np.float32) * 100))
        scales = (K.raw((rng.random(Hkv) * 0.02 + 0.001).astype(np.float32)), K.raw((rng.random(Hkv) * 0.02 + 0.001).astype(np.float32)))
    else:
        kc, vc, scales = K.dev(rnd((B, Hkv, S, D)), dt), K.dev(rnd((B, Hkv, S, D)), dt), None
    q, k, v = K.dev(rnd((B, Hq, 1, D)), dt), K.dev(rnd((B, Hkv, 1, D)), dt), K.dev(rnd((B, Hkv, 1, D)), dt)
    rows = np.resize(np.array(cpos, np.int64), B)
    # RoPE positions: other than the cache positions, past 8192 and near 131071
    rope_pos = np.resize(np.array([131071, 8192, 130999, 8191, 100000], np.int64), B)
    return (kc, vc, q, k, v), scales, rows, rope_pos


def attend(K, dt, inputs, scales, Hq, Hkv, pos, flags, rope=None, inv=None):
    """one AttentionKVCache launch on copies of the caches, RoPE folded with the table when `rope` is given; raw bits of
    (out, k cache, v cache)"""
    import torch
    kc, vc, q, k, v = inputs
    kc, vc = kc.clone(), vc.clone()
    B, Hkv_, S, D = kc.shape
    out = torch.full_like(q, float("nan"))
    wsb = K.L.lib.it_b200_attention_kvcache_workspace(B, Hq, S, D)
    ws = torch.full((int(wsb) // 4,), float("nan"), dtype=torch.float32, device="cuda")
    lib, p = K.L.lib, K.ptr
    args = (p(q), p(k), p(v), p(pos), I64 | flags)
    tail = (p(out), B, Hq, Hkv, S, D, p(ws), int(wsb), K.stream())
    if scales is None and rope is None:
        rc = lib.it_b200_attention_kvcache_gqa(dt, p(kc), p(vc), *args, None, 0, *tail)
    elif scales is None:
        rc = lib.it_b200_attention_kvcache_gqa_freq(dt, p(kc), p(vc), *args, p(rope), I64, p(inv), F32, inv.numel(), *tail)
    elif rope is None:
        rc = lib.it_b200_attention_kvcache_fp8(dt, p(kc), p(vc), p(scales[0]), p(scales[1]), *args, None, 0, *tail)
    else:
        rc = lib.it_b200_attention_kvcache_fp8_freq(dt, p(kc), p(vc), p(scales[0]), p(scales[1]), *args, p(rope), I64, p(inv),
                                                    F32, inv.numel(), *tail)
    K.L.check(rc)
    K.sync()
    return bits(out), bits(kc), bits(vc)


@pytest.mark.gpu
@pytest.mark.parametrize("per_row", [False, True], ids=["pos0", "per_row"])
@pytest.mark.parametrize("cache", ["f32", "f16", "bf16", "fp8_f16", "fp8_bf16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("case", sorted(FOLD_CASES))
def test_folded_table_is_rope_then_attention(K, case, D, cache, per_row):
    """attention with RoPE folded from a Llama-3.1 table gives exactly the bits of it_b200_rope_freq on q and k followed by
    the unfused kernel: output, k cache (the rotated k is appended; FP8: its codes) and v cache.  RoPE positions are other
    than the cache positions and lie past 8192 and near 131071; ITB_POS_IN_STEP changes nothing."""
    fp8 = cache.startswith("fp8")
    dt = {"f32": F32, "f16": F16, "bf16": BF16, "fp8_f16": F16, "fp8_bf16": BF16}[cache]
    B, Hq, Hkv, S, _ = FOLD_CASES[case]
    inputs, scales, rows, rope_pos = fold_inputs(K, case, dt, D, fp8)
    inv = K.raw(table(D, "llama31"))
    flags = 0x100 if per_row else 0
    pos, rope = K.raw(rows), K.raw(rope_pos)
    kc, vc, q, k, v = inputs
    qr = rope_freq_dev(K, dt, q.view(B, Hq * D), rope, I64, inv).view(B, Hq, 1, D)
    kr = rope_freq_dev(K, dt, k.view(B, Hkv * D), rope, I64, inv).view(B, Hkv, 1, D)
    ref = attend(K, dt, [kc, vc, qr, kr, v], scales, Hq, Hkv, pos, flags)
    for extra in (0, 0x200):
        got = attend(K, dt, inputs, scales, Hq, Hkv, pos, flags | extra, rope=rope, inv=inv)
        for what, g, r in zip(("out", "k cache", "v cache"), got, ref):
            assert np.array_equal(g, r), f"{what} (flags {flags | extra:#x}): {np.sum(g != r)} elements differ"
    # the table is really read: base 10000 gives other bits
    base = attend(K, dt, inputs, scales, Hq, Hkv, pos, flags, rope=rope, inv=K.raw(rope64.base_table(D)))
    assert not np.array_equal(base[0], ref[0])


# ---------------------------------------------------------------------------------------------------- long-context graphs
def long_cfg(B=2, kv_fp8=False, **kw):
    """a reduced-width Llama-3.1-8B: the preset's heads ratio (G = 4), head width and RoPE, 2 layers, a 128K cache"""
    from infinitensor_b200 import graphs as G
    c = G.LlamaConfig.llama31_8b(batch=B, s_max=131072, layers=2, kv_fp8=kv_fp8)
    return dataclasses.replace(c, d_model=512, heads=4, kv_heads=1, ffn=1024, vocab=512, **kw)


def base_logits(p, ids, pos, cudagraph):
    """the device logits of the same graph and inputs with base-10000 RoPE, on a runtime of its own"""
    from infinitensor_b200 import backend as Bk
    from infinitensor_b200 import graphs as G
    cfg = dataclasses.replace(p.cfg, rope_theta=10000.0, rope_scaling=None)
    h = Bk.GraphHandler(Bk.CudaRuntime(0))
    g = G.build_llama_decode(h, cfg, seq=ids.shape[1])
    h.data_malloc()
    G.fill_llama_weights_host(g)
    LO.load_caches(g, LO.cache_values(p.g))
    g.input_ids.copyin_numpy(ids)
    g.position_ids.copyin_numpy(pos)
    h.run_with_cudagraph() if cudagraph else h.run()
    return G.from_storage(g.logits.copyout_numpy(), cfg.dtype).astype(np.float64)


def base_oracle_logits(cfg, ids, pos):
    """the oracle's logits of the same graph built with base-10000 RoPE, from the caches every parity test starts from"""
    oh, og = RO.oracle_graph(dataclasses.replace(cfg, rope_theta=10000.0, rope_scaling=None), seq=ids.shape[1],
                             caches=LO.llama_caches(cfg))
    og.input_ids.copyin_numpy(ids)
    og.position_ids.copyin_numpy(pos)
    oh.run()
    return og.logits.f32().astype(np.float64)


@pytest.mark.gpu
@pytest.mark.parametrize("kv_fp8,fused,cudagraph", [(False, True, False), (False, True, True), (False, False, False),
                                                    (False, False, True), (True, True, True), (True, False, False)],
                         ids=["bf16_cache-fused-eager", "bf16_cache-fused-replay", "bf16_cache-unfused-eager",
                              "bf16_cache-unfused-replay", "fp8_cache-fused-replay", "fp8_cache-unfused-eager"])
def test_long_context_decode(K, kv_fp8, fused, cudagraph):
    """decode steps at p 8191, 8192 and 131000 against the test oracle.  At the first step the logits of the same graph built
    with base-10000 RoPE lie several times farther from the device's than the oracle's do (over a random cache the attention
    is close to uniform, so RoPE moves these logits by only 2-7 %)"""
    cfg = long_cfg(B=1 if kv_fp8 else 2, kv_fp8=kv_fp8)
    p = RO.llama_pair(cfg, env=None if fused else {"ITB_NO_FUSION": "1"})
    assert sum(s.startswith("AttentionRope") for s in p.schedule) == (cfg.layers if fused else 0), p.schedule
    tol = LO.TOL[cfg.dtype]
    rng = np.random.default_rng(3)
    for at in (8191, 8192, 131000):
        ids = rng.integers(0, cfg.vocab, (cfg.batch, 1)).astype(np.int64)
        pos = np.full((cfg.batch, 1), at, np.int64)
        got, ref = LO.llama_step(p, ids, pos, cudagraph)
        assert np.isfinite(got).all()
        err = LO.rel_err(got, ref)
        assert err < tol, f"p {at}: logits rel-to-max error {err:.3e} >= {tol}"
        LO.check_appended_k(p, at, tol)
        if at == 8191:
            other = LO.rel_err(base_oracle_logits(cfg, ids, pos), got)
            assert other > 4 * err, f"base-10000 logits {other:.3e} from the table's, the oracle {err:.3e}"
    if cudagraph:
        assert p.rt.cuda_graph_capture_count() == 1


@pytest.mark.gpu
def test_long_context_prompt_then_decode(K):
    """a 64-token prompt chunk at p 130000 (RoPE with the table unfused over [B, 64, d]), then decode steps on the caches it
    filled, against the test oracle"""
    cfg = long_cfg(B=1)
    tol = LO.TOL[cfg.dtype]
    rng = np.random.default_rng(4)
    pp = RO.llama_pair(cfg, seq=64)
    ids = rng.integers(0, cfg.vocab, (1, 64)).astype(np.int64)
    pos = (130000 + np.arange(64, dtype=np.int64))[None]
    got, ref = LO.llama_step(pp, ids, pos, cudagraph=False)
    assert np.isfinite(got).all() and LO.rel_err(got, ref) < tol, LO.rel_err(got, ref)
    other = LO.rel_err(base_logits(pp, ids, pos, False), ref)
    assert other > 2 * LO.rel_err(got, ref), f"base-10000 logits {other:.3e} from the oracle"
    dec = RO.llama_pair(cfg, caches=LO.cache_values(pp.g), oracle_caches=LO.cache_values(pp.og), rt=pp.rt)
    for at in (130064, 130065):
        ids = rng.integers(0, cfg.vocab, (1, 1)).astype(np.int64)
        got, ref = LO.llama_step(dec, ids, np.full((1, 1), at, np.int64), cudagraph=True)
        assert np.isfinite(got).all() and LO.rel_err(got, ref) < tol, (at, LO.rel_err(got, ref))
        LO.check_appended_k(dec, at, tol)
