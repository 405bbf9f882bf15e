"""Sliding-window attention on the H100: the windowed decode kernels (stream / grouped-query x 16-bit / fp32 / FP8 caches x
D 64 / 128 x RoPE none / base / table) against float64, against the unwindowed kernel over a shifted cache bit for bit, and
with a window past the position against the window-0 call bit for bit; the windowed prompt kernel against float64; and
Mistral-7B-v0.1-width graphs against the windowed test oracle."""
import dataclasses

import numpy as np
import pytest

import oracle
from tests import attn64
from tests import kvfp8_oracle as KV
from tests import llama_oracle as LO
from tests import swa64
from tests import swa_oracle as SO

F32, F16, BF16, I64 = 1, 10, 16, 7
PER_ROW = 0x100
GUARD = 4096  # elements of NaN before and after every cache: nothing may be written there

# decode cases: W = 1, W below a chunk, W a multiple of the chunk and not; whole heads, 2-way, >= 3-way and 256-way merges
# (test_swa_host checks the dealing reaches each); per-row positions whose window starts differ by row
DECODE_CASES = {
    "w1_stream": dict(dt=BF16, B=2, Hq=4, Hkv=4, S_max=300, pos=[0, 250], W=1, D=128),
    "below_chunk_d64": dict(dt=F16, B=3, Hq=2, Hkv=2, S_max=400, pos=[399, 37, 120], W=20, D=64),
    "chunk_multiple_f32": dict(dt=F32, B=1, Hq=8, Hkv=8, S_max=512, pos=[500], W=128, D=128),
    "whole_heads": dict(dt=BF16, B=8, Hq=32, Hkv=32, S_max=256, pos=[200, 201, 90, 255, 64, 63, 5, 180], W=64, D=128),
    "two_way": dict(dt=BF16, B=1, Hq=132, Hkv=132, S_max=256, pos=[255], W=100, D=128),
    "way256": dict(dt=BF16, B=1, Hq=1, Hkv=1, S_max=20000, pos=[19999], W=16400, D=128),
    "fp8_stream": dict(dt=BF16, B=2, Hq=4, Hkv=4, S_max=1024, pos=[1000, 700], W=256, D=128, fp8=True),
    "fp8_stream_d64": dict(dt=F16, B=2, Hq=4, Hkv=4, S_max=1024, pos=[1023, 300], W=333, D=64, fp8=True),
    "gqa_g4": dict(dt=BF16, B=2, Hq=32, Hkv=8, S_max=2048, pos=[2047, 900], W=300, D=128),
    "gqa_g8_d64": dict(dt=F16, B=1, Hq=32, Hkv=4, S_max=600, pos=[599], W=70, D=64),
    "gqa_g32_fp8_d64": dict(dt=F16, B=2, Hq=64, Hkv=2, S_max=800, pos=[799, 10], W=500, D=64, fp8=True),
    "gqa_g4_fp8": dict(dt=BF16, B=2, Hq=16, Hkv=4, S_max=1500, pos=[1499, 600], W=512, D=128, fp8=True),
    "gqa_g48_f32": dict(dt=F32, B=1, Hq=96, Hkv=2, S_max=400, pos=[350], W=64, D=128),
}


@pytest.fixture(scope="module")
def K():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from tests import kernel_harness
    return kernel_harness


def bits(t):
    import torch
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()]).cpu().numpy()


def _lo(p, W):
    return max(0, int(p) - W + 1)


def decode_inputs(c, rope, seed=0):
    """host arrays: caches (float values, or FP8 codes), q / k / v, scales, positions, RoPE positions and table.  Cache rows
    below each row's window and from its position on are NaN (FP8: NaN codes)."""
    from infinitensor_b200 import graphs as G
    rng = np.random.default_rng([seed, c["Hq"], c["S_max"], c["D"]])
    B, Hq, Hkv, S, D, W, dt = c["B"], c["Hq"], c["Hkv"], c["S_max"], c["D"], c["W"], c["dt"]
    pos = np.array(c["pos"], np.int64)
    rnd = lambda shape, s=0.7: attn64.exact((rng.standard_normal(shape) * s).astype(np.float32))
    kc, vc = rnd((B, Hkv, S, D)), rnd((B, Hkv, S, D))
    poison = np.zeros((B, Hkv, S, D), bool)
    for b in range(B):
        poison[b, :, :_lo(pos[b], W)] = True
        poison[b, :, pos[b]:] = True
    scales = None
    if c.get("fp8"):
        kc, vc = G.e4m3_codes_host(kc * 100), G.e4m3_codes_host(vc * 100)
        kc[poison], vc[poison] = 0x7F, 0x7F
        scales = ((rng.random(Hkv) * 0.02 + 0.001).astype(np.float32), (rng.random(Hkv) * 0.02 + 0.001).astype(np.float32))
    else:
        kc[poison], vc[poison] = np.nan, np.nan
    q, k, v = rnd((B, Hq, 1, D), 2.0 if rope == "none" else 0.7), rnd((B, Hkv, 1, D)), rnd((B, Hkv, 1, D))
    rope_pos = (pos + 7000).astype(np.int64)
    inv = G.rope_inv_freq(D, 500000.0) if rope == "table" else None
    return dict(kc=kc, vc=vc, q=q, k=k, v=v, scales=scales, pos=pos, rope_pos=rope_pos, inv=inv)


def attend(K, c, x, window, pos=None, kc=None, vc=None, rope="none"):
    """one it_b200_attention_kvcache_window call on guarded device copies of the caches; raw bits of (out, k cache, v cache)"""
    import torch
    dt, B, Hq, Hkv, S, D = c["dt"], c["B"], c["Hq"], c["Hkv"], c["S_max"], c["D"]
    kc = x["kc"] if kc is None else kc
    vc = x["vc"] if vc is None else vc
    pos = x["pos"] if pos is None else pos
    fp8 = x["scales"] is not None

    def guarded(a):
        if fp8:
            buf = torch.full((a.size + 2 * GUARD,), 0x7F, dtype=torch.uint8, device="cuda")
            buf[GUARD:GUARD + a.size] = K.raw(a.ravel())
        else:
            buf = torch.full((a.size + 2 * GUARD,), float("nan"), dtype=K.TORCH_DT[dt], device="cuda")
            buf[GUARD:GUARD + a.size] = K.dev(a.ravel(), dt)
        return buf
    kb, vb = guarded(kc), guarded(vc)
    q, k, v = (K.dev(t, dt) for t in (x["q"], x["k"], x["v"]))
    out = torch.full_like(q, float("nan"))
    wsb = K.L.lib.it_b200_attention_kvcache_workspace(B, Hq, S, D)
    ws = torch.full((int(wsb) // 4,), float("nan"), dtype=torch.float32, device="cuda")
    pd = K.raw(np.asarray(pos, np.int64))
    sc = [K.raw(s) for s in x["scales"]] if fp8 else [None, None]
    rp = K.raw(x["rope_pos"]) if rope != "none" else None
    inv = K.raw(x["inv"]) if rope == "table" else None
    p = K.ptr
    kp, vp = (p(kb[GUARD:]), p(vb[GUARD:]))
    K.L.check(K.L.lib.it_b200_attention_kvcache_window(dt, kp, vp, p(sc[0]), p(sc[1]), p(q), p(k), p(v), p(rp), I64, p(inv), F32,
                                                       D // 2, window, p(pd), I64 | PER_ROW, p(out), B, Hq, Hkv, S, D, p(ws),
                                                       int(wsb), K.stream()))
    K.sync()
    n = kc.size
    for buf in (kb, vb):  # the guards are untouched
        g = torch.cat([buf[:GUARD], buf[GUARD + n:]])
        assert (g == 0x7F).all() if fp8 else torch.isnan(g).all(), "a cache guard region was written"
    shape = kc.shape
    return bits(out), bits(kb[GUARD:GUARD + n]).reshape(shape), bits(vb[GUARD:GUARD + n]).reshape(shape)


def values(K, dt, a):
    """raw bits of 16-bit or fp32 elements -> float32 values"""
    import torch
    return torch.from_numpy(a).view(K.TORCH_DT[dt]).float().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("rope", ["none", "base", "table"])
@pytest.mark.parametrize("case", sorted(DECODE_CASES))
def test_decode_window(K, case, rope):
    """float64 within the bound (RoPE none), the shifted-cache identity bit for bit, a window past the position equal to the
    window-0 call bit for bit, the appended rows bit for bit, and two runs alike"""
    c = DECODE_CASES[case]
    x = decode_inputs(c, rope)
    B, Hq, Hkv, S, D, W, dt = c["B"], c["Hq"], c["Hkv"], c["S_max"], c["D"], c["W"], c["dt"]
    out, kc, vc = attend(K, c, x, W, rope=rope)
    again = attend(K, c, x, W, rope=rope)
    assert all(np.array_equal(a, b) for a, b in zip((out, kc, vc), again)), "two runs differ"
    got = values(K, dt, out.reshape(B, Hq, 1, D))
    # the shifted-cache identity: rows [lo, pos) moved to [0, pos - lo), the unwindowed kernel at pos - lo
    lo = np.array([_lo(p, W) for p in x["pos"]])
    ks, vs = np.full_like(x["kc"], np.nan if not c.get("fp8") else 0x7F), np.full_like(x["vc"], np.nan if not c.get("fp8") else 0x7F)
    for b in range(B):
        n = int(x["pos"][b] - lo[b])
        ks[b, :, :n], vs[b, :, :n] = x["kc"][b, :, lo[b]:lo[b] + n], x["vc"][b, :, lo[b]:lo[b] + n]
    out2, kc2, vc2 = attend(K, c, x, 0, pos=x["pos"] - lo, kc=ks, vc=vs, rope=rope)
    assert np.array_equal(out, out2), f"shifted-cache identity: {np.sum(out != out2)} output elements differ"
    for b in range(B):
        p = int(x["pos"][b])
        assert np.array_equal(kc[b, :, p], kc2[b, :, p - lo[b]]) and np.array_equal(vc[b, :, p], vc2[b, :, p - lo[b]])
    # only row pos of each batch row changed
    for a, orig in ((kc, x["kc"]), (vc, x["vc"])):
        o = orig if c.get("fp8") else bits(K.dev(orig, dt))
        for b in range(B):
            keep = np.ones(S, bool)
            keep[int(x["pos"][b])] = False
            assert np.array_equal(a[b][:, keep], o[b][:, keep]), "a cache row other than the appended one changed"
    # a window that covers every row is the unwindowed call
    full = attend(K, c, x, S, rope=rope)
    zero = attend(K, c, x, 0, rope=rope)
    assert all(np.array_equal(a, b) for a, b in zip(full, zero)), "window >= pos + 1 differs from window 0"
    if rope != "none":
        return
    # float64: over rows [lo, pos] of the caches after the append
    if c.get("fp8"):
        ksc, vsc = x["scales"]
        for b in range(B):
            p = int(x["pos"][b])
            ref, bd = KV.attention(kc[b:b + 1, :, lo[b]:], vc[b:b + 1, :, lo[b]:], ksc, vsc, x["q"][b:b + 1], [p - lo[b]], dt)
            bad = ~(np.abs(got[b:b + 1].astype(np.float64) - ref) <= bd)
            assert not bad.any(), f"batch row {b}: {int(bad.sum())} elements outside the FP8 bound"
        return
    refs = swa64.decode_refs(values(K, dt, kc), values(K, dt, vc), x["q"], x["pos"], W)
    bad = attn64.violations(got[:, :, 0], refs, dt, Hq != Hkv)
    dl = swa64.deal(dt, B, Hq, Hkv, S, x["pos"], W, D)
    assert not bad.any(), attn64.report(bad, got[:, :, 0], refs, dt, Hq != Hkv, dl, case)


# ---------------------------------------------------------------------------------------------------- prompt
PROMPT_CASES = {  # (B, Hq, Hkv, S, S_max, p, D, W)
    "s_below_w_inside_tile": (2, 4, 1, 100, 512, [300, 77], 128, 150),
    "s_above_w_on_tile": (1, 8, 2, 300, 1024, 500, 64, 128),
    "from_zero": (1, 2, 2, 64, 256, 20, 128, 100),
    "g48": (1, 48, 1, 130, 512, 200, 64, 61),
    "w1": (1, 2, 1, 70, 256, 50, 128, 1),
    "s_above_w_inside_tile": (2, 2, 2, 200, 700, [450, 131], 128, 77),
}


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F16, BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", sorted(PROMPT_CASES))
def test_prompt_window_float64(K, case, dt):
    """every output element within the float64 bound; cache rows below every query's window are NaN; two runs alike; the
    append is it_b200_attention_kvcache_prompt's"""
    import torch
    B, Hq, Hkv, S, S_max, p, D, W = PROMPT_CASES[case]
    c = swa64.Case(B, Hq, Hkv, S, S_max, p, D, seed=5, window=W)
    refs = c.reference()
    kc, vc, k, v = c.inputs()
    flags = I64 | (PER_ROW | (S << 16) if B > 1 else 0)
    pos = (c.p[:, None] + np.arange(S)[None]).astype(np.int64)
    runs = []
    for _ in range(2):
        kd, vd = K.dev(kc, dt), K.dev(vc, dt)
        q, kk, vv = K.dev(c.q, dt), K.dev(k, dt), K.dev(v, dt)
        out = torch.full_like(q, float("nan"))
        K.L.check(K.L.lib.it_b200_attention_kvcache_prompt_window(dt, K.ptr(kd), K.ptr(vd), K.ptr(q), K.ptr(kk), K.ptr(vv),
                                                                  K.ptr(K.raw(pos)), flags, K.ptr(out), B, Hq, Hkv, S, S_max, D,
                                                                  W, K.stream()))
        K.sync()
        runs.append((bits(out), bits(kd), bits(vd)))
        got = K.host(out)
    assert all(np.array_equal(a, b) for a, b in zip(*runs)), "two runs differ"
    bad = swa64.prompt64.violations(got, refs, dt)
    assert not bad.any(), swa64.prompt64.report(bad, got, refs, dt, c, case)


# ---------------------------------------------------------------------------------------------------- graphs
def mistral_cfg(kv_fp8=False):
    """a 2-layer Mistral-7B-v0.1 at full width (vocab 1000), B 1, an 8K cache"""
    from infinitensor_b200 import graphs as G
    return dataclasses.replace(G.LlamaConfig.mistral_7b_v01(batch=1, s_max=8192, layers=2, kv_fp8=kv_fp8), vocab=1000)


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [True, False], ids=["fused", "unfused"])
@pytest.mark.parametrize("kv_fp8", [False, True], ids=["bf16_cache", "fp8_cache"])
def test_mistral_decode(K, kv_fp8, fused):
    """decode steps at p 4094, 4095, 4096 (the window's first row leaves 0) and 8000 against the windowed oracle, each run
    eagerly and then replayed (the replay appends the same row again)"""
    cfg = mistral_cfg(kv_fp8)
    p = SO.llama_pair(cfg, env=None if fused else {"ITB_NO_FUSION": "1"})
    assert sum(s.startswith("AttentionRope") for s in p.schedule) == (cfg.layers if fused else 0), p.schedule
    tol = LO.TOL[cfg.dtype]
    rng = np.random.default_rng(3)
    for at in (4094, 4095, 4096, 8000):
        ids = rng.integers(0, cfg.vocab, (cfg.batch, 1)).astype(np.int64)
        for cudagraph in (False, True):
            got, ref = LO.llama_step(p, ids, np.full((cfg.batch, 1), at, np.int64), cudagraph)
            assert np.isfinite(got).all()
            err = LO.rel_err(got, ref)
            assert err < tol, f"p {at} ({'replayed' if cudagraph else 'eager'}): logits rel-to-max error {err:.3e} >= {tol}"
            LO.check_appended_k(p, at, tol)
    assert p.rt.cuda_graph_capture_count() == 1


@pytest.mark.gpu
def test_mistral_prompt_then_decode(K):
    """a 600-token prompt chunk at p 3800 (its windows start past 0 from token 297 on), then decode steps on the caches it
    filled, against the windowed oracle"""
    cfg = mistral_cfg()
    tol = LO.TOL[cfg.dtype]
    rng = np.random.default_rng(4)
    pp = SO.llama_pair(cfg, seq=600)
    ids = rng.integers(0, cfg.vocab, (1, 600)).astype(np.int64)
    pos = (3800 + np.arange(600, dtype=np.int64))[None]
    got, ref = LO.llama_step(pp, ids, pos, cudagraph=False)
    assert np.isfinite(got).all() and LO.rel_err(got, ref) < tol, LO.rel_err(got, ref)
    dec = SO.llama_pair(cfg, caches=LO.cache_values(pp.g), oracle_caches=LO.cache_values(pp.og), rt=pp.rt)
    for at in (4400, 4401):
        ids = rng.integers(0, cfg.vocab, (1, 1)).astype(np.int64)
        got, ref = LO.llama_step(dec, ids, np.full((1, 1), at, np.int64), cudagraph=True)
        assert np.isfinite(got).all() and LO.rel_err(got, ref) < tol, (at, LO.rel_err(got, ref))
        LO.check_appended_k(dec, at, tol)


@pytest.mark.gpu
@pytest.mark.parametrize("seq", [1, 24])
def test_tiny_graph_per_row_positions(K, seq):
    """one AttentionKVCache with window 16 and per-row positions (decode and a prompt chunk) on the device against the
    windowed oracle, cache rows below every window NaN"""
    from infinitensor_b200 import backend as Bk
    from infinitensor_b200 import graphs as G
    Bn, Hq, Hkv, S_max, D, W, dt = 3, 8, 2, 128, 128, 16, BF16
    rng = np.random.default_rng(9)
    starts = np.array([3, 40, 100])
    pos = (starts[:, None] + np.arange(seq)[None]).astype(np.int64)
    kc = oracle.round_to(rng.standard_normal((Bn, Hkv, S_max, D)).astype(np.float32), dt)
    vc = oracle.round_to(rng.standard_normal((Bn, Hkv, S_max, D)).astype(np.float32), dt)
    for b in range(Bn):
        kc[b, :, :_lo(starts[b], W)] = np.nan
        vc[b, :, :_lo(starts[b], W)] = np.nan
    q, k, v = (oracle.round_to(rng.standard_normal((Bn, n, seq, D)).astype(np.float32), dt) for n in (Hq, Hkv, Hkv))
    res = []
    for h in (Bk.GraphHandler(Bk.CudaRuntime(0)), SO.SwaOracleHandler()):
        t = [h.tensor(list(a.shape), dt) for a in (kc, vc, q, k, v)]
        pt = h.tensor([Bn, seq], I64)
        for x in t + [pt]:
            x.set_input()
        y = h.attentionKVCache(*t, pt, None, True, window=W)
        y.set_output()
        h.data_malloc()
        for x, a in zip(t, (kc, vc, q, k, v)):
            x.copyin_numpy(G.to_storage(a, dt))
        pt.copyin_numpy(pos)
        h.run()
        res.append(G.from_storage(y.copyout_numpy(), dt).astype(np.float64))
    assert np.isfinite(res[0]).all()
    assert np.abs(res[0] - res[1]).max() <= 2 ** -7 * np.abs(res[1]).max(), np.abs(res[0] - res[1]).max()
