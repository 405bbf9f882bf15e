"""AttentionKVCache over a prompt chunk (S > 1 new tokens) on the GPU: it_b200_attention_kvcache_prompt against float64
(tests/prompt64.py's per-element bound) over every score regime, head width, group size, chunk length and start; the append
bit for bit with NaN-poisoned caches, outputs and guard regions; the graph operator's dispatch; and Llama prompt steps followed
by decode steps against the graph oracle."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from tests import prompt64

F16, BF16, I32, I64 = 10, 16, 6, 7
POS_PER_ROW, STRIDE_SHIFT = 0x100, 16
GUARD = 4096  # elements of NaN on either side of every cache and output buffer


@pytest.fixture(scope="module")
def K():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from tests import kernel_harness
    return kernel_harness


def _bits(t):
    import torch
    return t.view(torch.int16)


def positions(case, mode, pos_dt, raw_p=None):
    """(position array, pos_flags): "elem0" -- [B, S] read at element 0 only; "rows_bs" -- [B, S] per row (stride S);
    "rows_b1" -- [B, 1] per row"""
    p = case.p if raw_p is None else np.asarray(raw_p, np.int64)
    B, S = case.B, case.S
    npdt = np.int64 if pos_dt == I64 else np.int32
    if mode == "rows_b1":
        return p.reshape(B, 1).astype(npdt), pos_dt | POS_PER_ROW | (1 << STRIDE_SHIFT)
    arr = (p[:, None] + np.arange(S)[None, :]).astype(npdt)
    if mode == "rows_bs":
        return arr, pos_dt | POS_PER_ROW | (S << STRIDE_SHIFT)
    return arr, pos_dt


def launch(K, case, dt, pos, flags):
    """one call on NaN-guarded buffers; returns (k cache buffer, v cache buffer, output buffer) before and after, as tensors"""
    import torch
    L = K.L
    kc, vc, k, v = case.inputs()

    def guarded(a):
        buf = K.dev(np.full(a.size + 2 * GUARD, np.nan, np.float32), dt)
        buf[GUARD:GUARD + a.size] = K.dev(a.ravel(), dt)
        return buf, buf[GUARD:GUARD + a.size].view(a.shape)

    (kb, kcd), (vb, vcd) = guarded(kc), guarded(vc)
    ob, od = guarded(np.full(case.q.shape, np.nan, np.float32))
    before = [kb.clone(), vb.clone(), ob.clone()]
    qd, kd, vd, pd = K.dev(case.q, dt), K.dev(k, dt), K.dev(v, dt), K.raw(pos)
    L.check(L.lib.it_b200_attention_kvcache_prompt(dt, K.ptr(kcd), K.ptr(vcd), K.ptr(qd), K.ptr(kd), K.ptr(vd), K.ptr(pd), flags,
                                                   K.ptr(od), case.B, case.Hq, case.Hkv, case.S, case.S_max, case.D, K.stream()))
    K.sync()
    return before, [kb, vb, ob], (kd, vd)


# (dt, D, B, Hq, Hkv, S, S_max, p, positions, position dtype): G = Hq / Hkv in {1, 4, 8, 32, 48}; S in {2, 63, 64, 65, 128, 129,
# 1000}; p in {0, 1, 64, 777}, p + S = S_max in three cases; per-row starts that differ by row
CASES = [
    (BF16, 128, 2, 8, 2, 65, 1024, [0, 777], "rows_bs", I64),
    (F16, 64, 1, 8, 1, 129, 256, 64, "elem0", I32),
    (BF16, 64, 1, 32, 1, 63, 64, 1, "rows_b1", I64),
    (F16, 128, 1, 48, 1, 2, 779, 777, "elem0", I64),
    (BF16, 128, 1, 2, 2, 1000, 1024, 0, "elem0", I32),
    (F16, 128, 3, 4, 4, 64, 1024, [0, 64, 777], "rows_b1", I32),
    (BF16, 64, 2, 8, 2, 128, 1024, [777, 1], "rows_bs", I32),
    (F16, 64, 1, 1, 1, 1000, 1001, 1, "elem0", I64),
    (BF16, 128, 1, 16, 2, 129, 512, 64, "rows_bs", I64),
    (F16, 64, 1, 4, 1, 1000, 2048, 777, "rows_b1", I64),
    (BF16, 64, 2, 32, 1, 2, 16, [3, 14], "rows_bs", I32),
]


@pytest.mark.parametrize("dt,D,B,Hq,Hkv,S,S_max,p,mode,pos_dt", CASES)
def test_prompt_attention_float64(K, dt, D, B, Hq, Hkv, S, S_max, p, mode, pos_dt):
    import torch
    case = prompt64.Case(B, Hq, Hkv, S, S_max, p, D, seed=S + 7 * Hq + D, offset=S)
    pos, flags = positions(case, mode, pos_dt)
    runs = [launch(K, case, dt, pos, flags) for _ in range(2)]
    for x, y in zip(runs[0][1], runs[1][1]):
        assert torch.equal(_bits(x), _bits(y)), "two runs of the same case differ"
    before, after, (kd, vd) = runs[0]
    # caches: rows [p_b, p_b + S) are k / v bit for bit, every other row and both guards untouched
    for b0, a0, src in ((before[0], after[0], kd), (before[1], after[1], vd)):
        want = b0.clone()
        view = want[GUARD:GUARD + B * Hkv * S_max * D].view(B, Hkv, S_max, D)
        for b in range(B):
            view[b, :, int(case.p[b]):int(case.p[b]) + S] = src[b]
        assert torch.equal(_bits(a0), _bits(want)), "cache rows outside the appended chunk (or its bits) changed"
    # output: guards untouched, every element finite and inside the float64 bound
    n = B * Hq * S * D
    ob = after[2]
    assert torch.equal(_bits(ob[:GUARD]), _bits(before[2][:GUARD])) and torch.equal(_bits(ob[GUARD + n:]), _bits(before[2][GUARD + n:]))
    got = K.host(ob[GUARD:GUARD + n]).reshape(B, Hq, S, D)
    refs = case.reference()
    msg = prompt64.report(prompt64.violations(got, refs, dt), got, refs, dt, case, f"{NAMES[dt]} D {D} G {Hq // Hkv} S {S}")
    assert msg is None, msg


NAMES = {F16: "f16", BF16: "bf16"}


def test_start_is_clamped(K):
    """p_b beyond S_max - S is clamped there, negative to 0: the same bits as the clamped start"""
    import torch
    case = prompt64.Case(2, 8, 2, 20, 64, [44, 0], 128, seed=3)
    outs = []
    for raw in ([5000, -7], [44, 0]):
        pos, flags = positions(case, "rows_b1", I64, raw_p=raw)
        outs.append(launch(K, case, BF16, pos, flags)[1])
    for x, y in zip(*outs):
        assert torch.equal(_bits(x), _bits(y))


# ---------------------------------------------------------------- the graph operator
def _op_graph(B_, rt, dt, Bn, Hq, Hkv, S, Smax, D, pos_shape, per_row):
    h = B_.GraphHandler(rt)
    kc, vc = h.tensor([Bn, Hkv, Smax, D], dt), h.tensor([Bn, Hkv, Smax, D], dt)
    q, k, v = h.tensor([Bn, Hq, S, D], dt), h.tensor([Bn, Hkv, S, D], dt), h.tensor([Bn, Hkv, S, D], dt)
    pos = h.tensor(pos_shape, I64)
    for t in (kc, vc, q, k, v, pos):
        t.set_input()
    out = h.attentionKVCache(kc, vc, q, k, v, pos, None, per_row)
    out.set_output()
    h.data_malloc()
    return h, (kc, vc, q, k, v, pos), out


@pytest.mark.parametrize("S,per_row,pos_shape", [(1, False, [2, 1]), (1, True, [2, 1]), (37, True, [2, 37]), (37, True, [2, 1]),
                                                 (37, False, [2, 37])])
def test_graph_operator_dispatch(K, S, per_row, pos_shape):
    """S = 1: the operator's output is bit for bit it_b200_attention_kvcache_gqa's; S > 1: it_b200_attention_kvcache_prompt's,
    with per-row positions read at the stride of a [B, S] or [B, 1] tensor"""
    import torch
    from infinitensor_b200 import backend as B_, graphs as G
    L = K.L
    Bn, Hq, Hkv, Smax, D = 2, 8, 2, 128, 128
    case = prompt64.Case(Bn, Hq, Hkv, S, Smax, [40, 3] if per_row else 40, D, seed=9, regimes=["flat", "late", "sink", "diag"])
    kc, vc, k, v = case.inputs()
    kc, vc = np.nan_to_num(kc), np.nan_to_num(vc)  # (the graph's caches hold zeros past p_b, like a fresh cache)
    posv = (case.p[:, None] + np.arange(pos_shape[1])[None, :]).astype(np.int64)
    h, ins, out = _op_graph(B_, B_.CudaRuntime(0), BF16, Bn, Hq, Hkv, S, Smax, D, pos_shape, per_row)
    for t, a in zip(ins, (kc, vc, case.q, k, v)):
        t.copyin_numpy(G.to_storage(a, BF16))
    ins[5].copyin_numpy(posv)
    h.run()
    got = torch.from_numpy(out.copyout_numpy().view(np.int16).copy())
    kcd, vcd = K.dev(kc, BF16), K.dev(vc, BF16)
    qd, kd, vd, pd = K.dev(case.q, BF16), K.dev(k, BF16), K.dev(v, BF16), K.raw(posv)
    od = torch.empty_like(qd)
    flags = I64 | (POS_PER_ROW if per_row else 0)
    if S == 1:
        wsb = L.lib.it_b200_attention_kvcache_workspace(Bn, Hq, Smax, D)
        ws = torch.empty(max(int(wsb), 16), dtype=torch.uint8, device="cuda")
        L.check(L.lib.it_b200_attention_kvcache_gqa(BF16, K.ptr(kcd), K.ptr(vcd), K.ptr(qd), K.ptr(kd), K.ptr(vd), K.ptr(pd), flags,
                                                    None, 0, K.ptr(od), Bn, Hq, Hkv, Smax, D, K.ptr(ws), int(wsb), K.stream()))
    else:
        if per_row:
            flags |= pos_shape[1] << STRIDE_SHIFT
        L.check(L.lib.it_b200_attention_kvcache_prompt(BF16, K.ptr(kcd), K.ptr(vcd), K.ptr(qd), K.ptr(kd), K.ptr(vd), K.ptr(pd),
                                                       flags, K.ptr(od), Bn, Hq, Hkv, S, Smax, D, K.stream()))
    K.sync()
    assert torch.equal(got, _bits(od).cpu())
    assert torch.equal(torch.from_numpy(ins[0].copyout_numpy().view(np.int16).copy()), _bits(kcd).cpu())


def test_graph_refuses_fp32_prompt_chunk(K):
    from infinitensor_b200 import backend as B_
    with pytest.raises(RuntimeError, match="fp32"):
        _op_graph(B_, B_.CudaRuntime(0), 1, 1, 2, 2, 4, 16, 128, [1, 4], True)


# ---------------------------------------------------------------- Llama prompt steps
def _argmax_agree(got, ref, tol):
    """argmax equal wherever the oracle's top two logits are further apart than the tolerance allows the error to move them"""
    top2 = np.sort(ref, axis=-1)[..., -2:]
    clear = (top2[..., 1] - top2[..., 0]) > 2 * tol * np.abs(ref).max()
    return np.array_equal(np.argmax(got, -1)[clear], np.argmax(ref, -1)[clear])


def run_prompt_then_decode(cfg, S, p0, decode_steps, cudagraph, tol):
    """prompt step of S tokens at p0 .. p0 + S - 1 (per-row [B, S] positions), then decode steps, on the device and on the
    oracle (tests/llama_oracle.py); every step's logits against the oracle's (rel-to-max error < tol, argmax agreement)"""
    from infinitensor_b200 import backend as B_, graphs as G
    from tests import llama_oracle as L
    rt = B_.CudaRuntime(0)
    rng = np.random.default_rng(3)
    Bn = cfg.batch
    caches = [G.to_storage(rng.standard_normal((Bn, cfg.n_kv, cfg.s_max, cfg.head_dim)).astype(np.float32) * 0.5, cfg.dtype)
              for _ in range(2 * cfg.layers)]

    def step(p, ids, pos, what):
        got, ref = L.llama_step(p, ids, pos, cudagraph)
        err = L.rel_err(got, ref)
        assert np.isfinite(got).all(), f"{what}: non-finite logits"
        assert err < tol, f"{what}: logits rel-to-max error {err:.3e} >= {tol}"
        assert _argmax_agree(got, ref, tol)
        return err

    prompt = L.llama_pair(cfg, seq=S, caches=caches, rt=rt)
    ids = rng.integers(0, cfg.vocab, size=(Bn, S)).astype(np.int64)
    worst = step(prompt, ids, np.broadcast_to(p0 + np.arange(S), (Bn, S)).astype(np.int64).copy(), "prompt step")
    # the appended k rows of layer 0 agree with the oracle's (the projections differ by rounding only)
    L.check_appended_k(prompt, slice(p0, p0 + S), tol)
    assert np.array_equal(prompt.g.k_caches[0].copyout_numpy()[:, :, :p0], caches[0][:, :, :p0])
    if decode_steps:
        # each side continues from its own caches
        dec = L.llama_pair(cfg, caches=L.cache_values(prompt.g), oracle_caches=L.cache_values(prompt.og), rt=rt)
        for i in range(decode_steps):
            ids = rng.integers(0, cfg.vocab, size=(Bn, 1)).astype(np.int64)
            worst = max(worst, step(dec, ids, np.full((Bn, 1), p0 + S + i, np.int64), f"decode step {i}"))
    return worst, prompt.schedule


BF16_TOL = 3e-2  # the bf16 graph tolerance of the decode parity tests (tests/llama_oracle.py)


@pytest.mark.parametrize("cudagraph", [False, True])
def test_tiny_llama_prompt_then_decode(K, cudagraph):
    from infinitensor_b200 import graphs as G
    run_prompt_then_decode(G.LlamaConfig.tiny(), S=16, p0=5, decode_steps=3, cudagraph=cudagraph, tol=BF16_TOL)


@pytest.mark.parametrize("cudagraph", [False, True])
def test_tinyllama_width_prompt_then_decode(K, cudagraph):
    """two TinyLlama-width layers (32 query heads of 64 over 4 KV heads), a 1000-token vocabulary"""
    from infinitensor_b200 import graphs as G
    cfg = G.LlamaConfig(layers=2, d_model=2048, heads=32, kv_heads=4, head_dim=64, ffn=5632, vocab=1000, s_max=256, batch=2)
    run_prompt_then_decode(cfg, S=100, p0=64, decode_steps=3, cudagraph=cudagraph, tol=BF16_TOL)


def test_llama7b_width_prompt_step(K):
    """two Llama-7B-width layers, one 512-token prompt through the fused schedule (MatMulAdd, SiluMul; no decode fusions)"""
    from infinitensor_b200 import graphs as G
    cfg = G.LlamaConfig(layers=2, d_model=4096, heads=32, head_dim=128, ffn=11008, vocab=1000, s_max=1024, batch=1)
    _, sched = run_prompt_then_decode(cfg, S=512, p0=0, decode_steps=0, cudagraph=True, tol=BF16_TOL)
    assert "Single:AttentionKVCache" in sched and not any(s.startswith(("AttentionRope", "MatMulGroup")) for s in sched)
    assert any(s.startswith("MatMulAdd") for s in sched)
