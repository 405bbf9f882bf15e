"""The rolling KV cache on the H100: every ring call against the same windowed launcher over a linear cache that holds the same
positions, bit for bit -- decode (stream / grouped-query x 16-bit / fp32 / FP8 caches x D 64 / 128 x RoPE none / base / table,
positions before the first wrap, just after it, around 10**6 and at the clamp, a chunk straddling the ring's end first, in the
middle and last in a head) and prompt chunks (f16 / bf16, D 64 / 128, G 1 .. 48, chunks that wrap, the largest chunk
S_max - W + 1); and 2-layer Mistral-width graphs with a 384-row ring against the same graphs over a 2048-row linear cache,
bit for bit at every step, and against the ring oracle."""
import dataclasses

import numpy as np
import pytest

from tests import attn64
from tests import llama_oracle as LO
from tests import ring_oracle as RG

F32, F16, BF16, I64 = 1, 10, 16, 7
PER_ROW, IN_STEP, RING = 0x100, 0x200, 0x400


@pytest.fixture(scope="module")
def K():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from tests import kernel_harness
    return kernel_harness


def bits(t):
    import torch
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()]).cpu().numpy()


def chunk_rows(dt, D, fp8):
    """cache rows per 16 KiB chunk, both decode bodies"""
    return 16384 // (D * (1 if fp8 else (4 if dt == F32 else 2)))


def straddle(S_max, W, CH, c, wraps=3):
    """a position P >= W - 1 whose window's chunk c crosses the ring's end in its middle"""
    lo = wraps * S_max - c * CH - CH // 2
    return lo + W - 1


# decode cases: (family by Hq / Hkv, cache dtype, D, W, S_max, per-row positions by kind).  Position kinds: "pre" before the
# first wrap, "just" just past it, "first" / "mid" / "last" a straddling chunk there, "far" ~10**6, "clamp" at the bound
# INT32_MAX - S_max, "over" an int64 position beyond it
DECODE_CASES = {
    "stream_bf16": dict(dt=BF16, Hq=4, Hkv=4, D=128, W=300, S_max=448, pos=["pre", "just", "first", "mid", "last", "far"]),
    "stream_f16_d64": dict(dt=F16, Hq=2, Hkv=2, D=64, W=500, S_max=512, pos=["first", "mid", "last", "clamp", "over"]),
    "stream_f32": dict(dt=F32, Hq=3, Hkv=3, D=128, W=200, S_max=256, pos=["just", "mid", "last", "far"]),
    "stream_fp8": dict(dt=BF16, Hq=4, Hkv=4, D=128, W=700, S_max=768, pos=["pre", "first", "mid", "last"], fp8=True),
    "stream_fp8_d64": dict(dt=F16, Hq=2, Hkv=2, D=64, W=1000, S_max=1024, pos=["mid", "last", "far", "clamp"], fp8=True),
    "gqa4_bf16": dict(dt=BF16, Hq=32, Hkv=8, D=128, W=600, S_max=640, pos=["pre", "first", "mid", "last", "far"]),
    "gqa8_f16_d64": dict(dt=F16, Hq=32, Hkv=4, D=64, W=256, S_max=256, pos=["just", "first", "last", "clamp"]),
    "gqa48_f32": dict(dt=F32, Hq=96, Hkv=2, D=128, W=100, S_max=128, pos=["first", "mid", "last"]),
    "gqa4_fp8": dict(dt=BF16, Hq=16, Hkv=4, D=128, W=900, S_max=1024, pos=["pre", "first", "mid", "last", "over"], fp8=True),
    "gqa32_fp8_d64": dict(dt=F16, Hq=64, Hkv=2, D=64, W=1, S_max=64, pos=["pre", "just", "far"], fp8=True),
    "stream_w1": dict(dt=BF16, Hq=4, Hkv=4, D=128, W=1, S_max=64, pos=["pre", "just", "far", "clamp"]),
    "one_head_many_way": dict(dt=BF16, Hq=1, Hkv=1, D=128, W=4096, S_max=4096, pos=["mid"]),
    "gqa_w_eq_smax": dict(dt=BF16, Hq=8, Hkv=2, D=128, W=1024, S_max=1024, pos=["first", "last", "far"]),
}


def positions(c):
    S_max, W = c["S_max"], c["W"]
    CH = chunk_rows(c["dt"], c["D"], c.get("fp8", False))
    nch = (W - 1) // CH + 1  # chunks of a full window
    kinds = {"pre": min(S_max - 1, W // 2 + 3), "just": S_max + 5, "first": straddle(S_max, W, CH, 0),
             "mid": straddle(S_max, W, CH, nch // 2), "last": straddle(S_max, W, CH, max(nch - 1, 0)),
             "far": 10**6 + 37, "clamp": RG.ring_pos_max(S_max), "over": 2**40}
    return np.array([kinds[k] for k in c["pos"]], np.int64)


def linear_position(P, W, S_max):
    """a position of a linear S_max-row cache with the same span (min(P, W - 1)) as P"""
    return P if P < S_max else W - 1 + P % (S_max - W + 1)


def decode_case(c, seed):
    """ring caches (rows outside every window NaN / NaN codes), the linear caches with the same window contents, and the rest
    of one step's inputs"""
    from infinitensor_b200 import graphs as G
    rng = np.random.default_rng([seed, c["Hq"], c["S_max"], c["D"]])
    dt, Hq, Hkv, S_max, D, W = c["dt"], c["Hq"], c["Hkv"], c["S_max"], c["D"], c["W"]
    fp8 = c.get("fp8", False)
    P = np.minimum(positions(c), RG.ring_pos_max(S_max))
    B = len(P)
    Pl = np.array([linear_position(p, W, S_max) for p in P], np.int64)
    if fp8:
        nan = 0x7F
        ring = [np.full((B, Hkv, S_max, D), nan, np.uint8) for _ in range(2)]
    else:
        nan = np.nan
        ring = [np.full((B, Hkv, S_max, D), nan, np.float32) for _ in range(2)]
    lin = [r.copy() for r in ring]
    for b in range(B):
        span = min(int(P[b]), W - 1)
        for r, l in zip(ring, lin):
            rows = attn64.exact((rng.standard_normal((Hkv, span, D)) * 0.7).astype(np.float32))
            if fp8:
                rows = G.e4m3_codes_host(rows * 100)
            r[b][:, np.arange(P[b] - span, P[b]) % S_max] = rows
            l[b][:, Pl[b] - span:Pl[b]] = rows
    rnd = lambda shape: attn64.exact((rng.standard_normal(shape) * 0.7).astype(np.float32))
    scales = None
    if fp8:
        scales = ((rng.random(Hkv) * 0.02 + 0.001).astype(np.float32), (rng.random(Hkv) * 0.02 + 0.001).astype(np.float32))
    return dict(P=P, raw_P=positions(c), Pl=Pl, ring=ring, lin=lin, q=rnd((B, Hq, 1, D)) * 2, k=rnd((B, Hkv, 1, D)),
                v=rnd((B, Hkv, 1, D)), scales=scales)


def decode_call(K, c, x, caches, pos, flags, rope):
    """one it_b200_attention_kvcache_window call; raw bits of (out, k cache, v cache)"""
    import torch
    dt, Hq, Hkv, S_max, D, W = c["dt"], c["Hq"], c["Hkv"], c["S_max"], c["D"], c["W"]
    B = len(pos)
    fp8 = x["scales"] is not None
    kc, vc = ((K.raw(a) if fp8 else K.dev(a, dt)) for a in caches)
    q, k, v = (K.dev(t, dt) for t in (x["q"], x["k"], x["v"]))
    out = torch.full_like(q, float("nan"))
    wsb = K.L.lib.it_b200_attention_kvcache_workspace(B, Hq, S_max, D)
    ws = torch.full((int(wsb) // 4,), float("nan"), dtype=torch.float32, device="cuda")
    pd = K.raw(np.asarray(pos, np.int64))
    sc = [K.raw(s) for s in x["scales"]] if fp8 else [None, None]
    rp = K.raw((x["P"] + 3).astype(np.int64)) if rope != "none" else None  # the real positions, for both calls
    from infinitensor_b200 import graphs as G
    inv = K.raw(G.rope_inv_freq(D, 500000.0)) if rope == "table" else None
    p = K.ptr
    K.L.check(K.L.lib.it_b200_attention_kvcache_window(dt, p(kc), p(vc), p(sc[0]), p(sc[1]), p(q), p(k), p(v), p(rp), I64, p(inv),
                                                       F32, D // 2, W, p(pd), I64 | flags, p(out), B, Hq, Hkv, S_max, D, p(ws),
                                                       int(wsb), K.stream()))
    K.sync()
    return bits(out), bits(kc), bits(vc)


@pytest.mark.gpu
@pytest.mark.parametrize("rope", ["none", "base", "table"])
@pytest.mark.parametrize("case", sorted(DECODE_CASES))
def test_decode_ring_equals_linear(K, case, rope):
    """the ring call at the real positions against the linear windowed call at positions with the same window contents: the
    output, the appended row (at P mod S_max against P'), and every other ring row unchanged, bit for bit"""
    c = DECODE_CASES[case]
    x = decode_case(c, seed=len(case))
    S_max = c["S_max"]
    o_r, k_r, v_r = decode_call(K, c, x, x["ring"], x["raw_P"], PER_ROW | RING, rope)
    o_l, k_l, v_l = decode_call(K, c, x, x["lin"], x["Pl"], PER_ROW, rope)
    assert np.array_equal(o_r, o_l), "output differs from the linear windowed call"
    fp8 = x["scales"] is not None
    for got, lin, before in ((k_r, k_l, x["ring"][0]), (v_r, v_l, x["ring"][1])):
        for b, (P, Pl) in enumerate(zip(x["P"], x["Pl"])):
            assert np.array_equal(got[b][:, P % S_max], lin[b][:, Pl]), "appended row"
            keep = np.arange(S_max) != P % S_max
            want = before[b][:, keep] if fp8 else bits(K.dev(before[b][:, keep], c["dt"]))
            assert np.array_equal(got[b][:, keep], want), "a ring row other than the appended one changed"


@pytest.mark.gpu
def test_decode_ring_element0_in_step(K):
    """element-0 positions with ITB_POS_IN_STEP: every batch row at the same ring position"""
    c = dict(dt=BF16, Hq=16, Hkv=4, D=128, W=600, S_max=640, pos=["mid"] * 3)
    x = decode_case(c, seed=5)
    o_r, k_r, _ = decode_call(K, c, x, x["ring"], x["raw_P"], RING | IN_STEP, "base")
    o_l, k_l, _ = decode_call(K, c, x, x["lin"], x["Pl"], IN_STEP, "base")
    assert np.array_equal(o_r, o_l) and np.array_equal(k_r[:, :, x["P"][0] % 640], k_l[:, :, x["Pl"][0]])


# ---------------------------------------------------------------------------------------------------- prompt
PROMPT_CASES = {
    # (dt, Hq, Hkv, D, W, S_max, S, starts): chunks that wrap, the largest chunk S_max - W + 1, starts whose first key tile
    # holds rows the chunk itself overwrites, far positions
    "bf16_max_chunk": (BF16, 4, 1, 128, 200, 320, 121, [1000, 5000]),
    "f16_d64_wrap": (F16, 8, 8, 64, 64, 192, 100, [150, 700]),
    "bf16_g48": (BF16, 96, 2, 128, 300, 512, 213, [10**6 + 17, 333]),
    "f16_first_tile_overwritten": (F16, 2, 2, 128, 130, 256, 127, [517, 2000]),
    "bf16_d64_g8_from_zero": (BF16, 32, 4, 64, 100, 256, 157, [0, 45]),
}


def prompt_call(K, dt, Hq, Hkv, D, S, S_max, W, caches, starts, q, k, v, flags):
    import torch
    B = len(starts)
    kc, vc = (K.dev(a, dt) for a in caches)
    qd, kd, vd = (K.dev(t, dt) for t in (q, k, v))
    out = torch.full_like(qd, float("nan"))
    pos = K.raw((np.asarray(starts, np.int64)[:, None] + np.arange(S)[None]).astype(np.int64))
    p = K.ptr
    K.L.check(K.L.lib.it_b200_attention_kvcache_prompt_window(dt, p(kc), p(vc), p(qd), p(kd), p(vd), p(pos),
                                                              I64 | PER_ROW | flags | (S << 16), p(out), B, Hq, Hkv, S, S_max, D,
                                                              W, K.stream()))
    K.sync()
    return bits(out), bits(kc), bits(vc)


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(PROMPT_CASES))
def test_prompt_ring_equals_linear(K, case):
    """a ring chunk against the linear windowed chunk at starts shifted by a multiple of 64 (the key tiles keep their place),
    ring rows outside every window NaN: the output and the appended rows, bit for bit"""
    dt, Hq, Hkv, D, W, S_max, S, starts = PROMPT_CASES[case]
    rng = np.random.default_rng(len(case))
    B = len(starts)
    starts = np.array(starts, np.int64)
    base = 64 * ((W + 63) // 64)
    lstarts = np.where(starts < base, starts, base + starts % 64)
    S_lin = 64 * ((int(lstarts.max()) + S + 63) // 64)
    ring = [np.full((B, Hkv, S_max, D), np.nan, np.float32) for _ in range(2)]
    lin = [np.full((B, Hkv, S_lin, D), np.nan, np.float32) for _ in range(2)]
    for b in range(B):
        lo = max(0, int(starts[b]) - W + 1)
        n = int(starts[b]) - lo
        for r, l in zip(ring, lin):
            rows = attn64.exact(rng.standard_normal((Hkv, n, D)).astype(np.float32))
            r[b][:, np.arange(lo, starts[b]) % S_max] = rows
            l[b][:, lstarts[b] - n:lstarts[b]] = rows
    q, k, v = (attn64.exact(rng.standard_normal((B, h, S, D)).astype(np.float32)) for h in (Hq, Hkv, Hkv))
    o_r, k_r, v_r = prompt_call(K, dt, Hq, Hkv, D, S, S_max, W, ring, starts, q, k, v, RING)
    o_l, k_l, v_l = prompt_call(K, dt, Hq, Hkv, D, S, S_lin, W, lin, lstarts, q, k, v, 0)
    assert np.array_equal(o_r, o_l), "output differs from the linear windowed chunk"
    for got, want in ((k_r, k_l), (v_r, v_l)):
        for b in range(B):
            assert np.array_equal(got[b][:, np.arange(starts[b], starts[b] + S) % S_max],
                                  want[b][:, lstarts[b]:lstarts[b] + S]), "appended rows"


# ---------------------------------------------------------------------------------------------------- graphs
def mistral_ring_cfg(rolling, kv_fp8=False, table=False):
    """a 2-layer Mistral-7B-v0.1 at full width (vocab 1000), B 1, window 256: a 384-row ring, or a 2048-row linear cache"""
    from infinitensor_b200 import graphs as G
    cfg = dataclasses.replace(G.LlamaConfig.mistral_7b_v01(batch=1, layers=2, kv_fp8=kv_fp8), vocab=1000, sliding_window=256,
                              s_max=384 if rolling else 2048, rolling_cache=rolling)
    if table:
        cfg = dataclasses.replace(cfg, rope_theta=500000.0, rope_scaling=dict(G.LLAMA31_ROPE_SCALING))
    return cfg


def _device_graph(cfg, seq, rt, env):
    from infinitensor_b200 import backend as Bk
    from infinitensor_b200 import graphs as G
    h = Bk.GraphHandler(rt)
    with LO._environ(env):
        g = G.build_llama_decode(h, cfg, seq=seq)
        h.data_malloc()
        h.schedule()
    G.fill_llama_weights_host(g)
    return h, g


def _run(h, g, ids, pos, cudagraph):
    from infinitensor_b200 import graphs as G
    g.input_ids.copyin_numpy(ids)
    g.position_ids.copyin_numpy(pos)
    h.run_with_cudagraph() if cudagraph else h.run()
    return G.from_storage(g.logits.copyout_numpy(), g.cfg.dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["fused_replay", "unfused_eager", "fp8_cache", "rope_table"])
def test_mistral_ring_graph(K, variant):
    """a 128-token prompt (not with the FP8 cache), then decode steps to position 1200 (about three wraps of the ring): the
    ring graph's logits equal the linear graph's bit for bit at every step, and the ring oracle's within the tolerance every
    100 steps (the oracle takes the device's caches there)"""
    fp8, table = variant == "fp8_cache", variant == "rope_table"
    env = {"ITB_NO_FUSION": "1"} if variant == "unfused_eager" else {}
    # (the fusion switch stays set while the graphs run: building one graph invalidates the other's schedule, which is
    # then planned again)
    with LO._environ(env):
        _mistral_ring_graph(variant, fp8, table, env, cudagraph=variant != "unfused_eager")


def _mistral_ring_graph(variant, fp8, table, env, cudagraph):
    from infinitensor_b200 import backend as Bk
    rt = Bk.CudaRuntime(0)
    rc, lc = mistral_ring_cfg(True, fp8, table), mistral_ring_cfg(False, fp8, table)
    rng = np.random.default_rng(11)
    start = 0
    caches = LO.llama_caches(rc)
    lcaches = [np.zeros(c.shape[:2] + (2048,) + c.shape[3:], c.dtype) for c in caches]
    for r, l in zip(caches, lcaches):
        l[:, :, :384] = r
    if not fp8:  # the prompt
        S = 128
        outs = []
        for cfg, cs in ((rc, caches), (lc, lcaches)):
            h, g = _device_graph(cfg, S, rt, env)
            LO.load_caches(g, cs)
            ids = rng.integers(0, cfg.vocab, (1, S)).astype(np.int64) if not outs else ids
            outs.append(_run(h, g, ids, np.arange(S, dtype=np.int64)[None], False))
            cs[:] = LO.cache_values(g)
        assert np.array_equal(outs[0], outs[1]), "prompt logits"
        start = S
    hr, gr = _device_graph(rc, 1, rt, env)
    hl, gl = _device_graph(lc, 1, rt, env)
    for name, (t, _, kind, _) in gr.weights.items():  # FP8 caches: the ring's k / v scales in both graphs
        if kind == "kv_scale":
            gl.weights[name][0].copyin_numpy(t.copyout_numpy())
    LO.load_caches(gr, caches)
    LO.load_caches(gl, lcaches)
    oh, og = RG.oracle_graph(rc, caches=caches)
    tol = LO.TOL[rc.dtype]
    for P in range(start, 1201):
        ids = rng.integers(0, rc.vocab, (1, 1)).astype(np.int64)
        pos = np.full((1, 1), P, np.int64)
        if P % 100 == 0:  # the oracle from the ring graph's caches before the step
            LO.load_caches(og, LO.cache_values(gr))
        a = _run(hr, gr, ids, pos, cudagraph)
        b = _run(hl, gl, ids, np.full((1, 1), min(P, 2047), np.int64), cudagraph)
        assert np.array_equal(a, b), f"p {P}: ring logits differ from the linear cache's"
        if P % 100 == 0:
            og.input_ids.copyin_numpy(ids)
            og.position_ids.copyin_numpy(pos)
            oh.run()
            err = LO.rel_err(a.astype(np.float64), og.logits.f32().astype(np.float64))
            assert err < tol, f"p {P}: logits rel-to-max error {err:.3e} against the ring oracle"
    if cudagraph:
        assert rt.cuda_graph_capture_count() >= 1
