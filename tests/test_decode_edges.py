"""Edges of the Llama decode step that the other parity tests do not reach.

* The decode GEMMs at every row-tile width (M = 1 .. 64 crosses MT = 1 / 2 / 4 of the skinny kernel and NT = 16 / 32 / 64 of the
  wgmma kernel), at the step's own shapes, under the production dispatch and with each kernel pinned, against a float64
  reference with a per-element bound (tests/ref64.py).  FP8 weights at 17..32 rows.
* The residual epilogue as the schedule launches it (full-stride bias, ITB_ACT_ROUND_BEFORE_BIAS | ITB_MATMUL_B_CONST): bit for
  bit MatMul followed by Add.
* The fused RoPE + AttentionKVCache (equal heads and grouped) against RoPE followed by the unfused kernel, bit for bit, with
  per-row RoPE positions, every position dtype and both cache-position rules; the 1024-row batch limit.
* A profiler check that those cases really launch the MT = 2, NT = 32 and RoPE-streaming instantiations.

The CPU self-checks at the top run without a GPU: they show that the float64 bound passes an emulation of the kernels'
arithmetic and fails five plausible kernel bugs.
"""
import re

import numpy as np
import pytest

import oracle
from tests import ref64

F32, F16, BF16 = 1, 10, 16
TILE_K = 64  # k-tile of both decode GEMM kernels


# ====================================================================== CPU: the bound catches real bugs and does not flake
def emulate_gemm(a, w, dt, ktiles_per_split, mutation=None):
    """The decode GEMMs' arithmetic in float32 numpy: fp32 partial products per 64-wide k-tile, one fp32 partial per split,
    the split partials summed in rank order, one rounding to T.  `mutation` injects one kernel bug."""
    m, k = a.shape
    a = np.array(a, np.float32)
    w = np.asarray(w, np.float32)
    if mutation == "row_shift":  # MT = 2 mapping error: rows 16..31 read X one row further on (past M: TMA zero fill)
        a[16:] = np.concatenate([a[17:], np.zeros((1, k), np.float32)])[: m - 16]
    if mutation == "drop_tail":  # the partial last k-tile ignored: the last 8 of K = 4104
        a[:, (k // TILE_K) * TILE_K:] = 0
    ktiles = -(-k // TILE_K)
    partials = []
    for s0 in range(0, ktiles, ktiles_per_split):
        acc = np.zeros((m, w.shape[1]), np.float32)
        for t in range(s0, min(ktiles, s0 + ktiles_per_split)):
            k0, k1 = t * TILE_K, min(k, (t + 1) * TILE_K)
            acc += a[:, k0:k1] @ w[k0:k1]
            if mutation == "lost_k16" and t == 1:  # one k16 slice missing from the 16 x 8 fragment at rows 0..15, cols 8..15
                acc[0:16, 8:16] -= a[0:16, k0 + 32:k0 + 48] @ w[k0 + 32:k0 + 48, 8:16]
        partials.append(oracle.round_to(acc, dt) if mutation == "round_partials" else acc)
    if mutation == "split_twice":
        partials.append(partials[1])
    total = np.zeros_like(partials[0])
    for p in partials:
        total += p
    return oracle.round_to(total, dt)


# (M, K, N, k-tiles per split) as the skinny kernel splits them: 65 k-tiles as 17 / 17 / 17 / 14, and 172 as 4 x 43
EMU_SHAPES = {"ragged": (16, 4104, 4104, 17), "down": (24, 11008, 4096, 43)}
_emu_cache = {}


def _emu_case(name, dt):
    key = (name, dt)
    if key not in _emu_cache:
        m, k, n, per = EMU_SHAPES[name]
        a, w = ref64.activations(m, k, dt, 7), ref64.weights(k, n, dt, 8)
        _emu_cache[key] = (a, w, per) + ref64.product(a, w)
    return _emu_cache[key]


@pytest.mark.parametrize("dt", [BF16, F16])
@pytest.mark.parametrize("name", sorted(EMU_SHAPES))
def test_bound_passes_kernel_arithmetic(name, dt):
    a, w, per, ref, mag = _emu_case(name, dt)
    ref64.assert_within(emulate_gemm(a, w, dt, per), ref, mag, dt, what=f"emulated {name}")


@pytest.mark.parametrize("name,mutation", [("ragged", "lost_k16"), ("down", "lost_k16"), ("down", "row_shift"),
                                           ("ragged", "round_partials"), ("down", "round_partials"),
                                           ("ragged", "split_twice"), ("down", "split_twice"), ("ragged", "drop_tail")])
def test_bound_catches_kernel_bugs(name, mutation):
    """bf16, the coarser type, is where a loose bound would hide a bug; every mutation must leave elements outside it"""
    a, w, per, ref, mag = _emu_case(name, BF16)
    bad = ref64.violations(emulate_gemm(a, w, BF16, per, mutation), ref, mag, BF16)
    assert bad.any(), f"{mutation} on {name} stays inside the bound"


def test_ulp_known_values():
    assert ref64.ulp(np.array([1.0, 1.5, 2.0, -3.0]), BF16).tolist() == [2.0 ** -7, 2.0 ** -7, 2.0 ** -6, 2.0 ** -6]
    assert ref64.ulp(np.array([1.0, 0.0, 2.0 ** -20]), F16).tolist() == [2.0 ** -10, 2.0 ** -24, 2.0 ** -24]
    assert ref64.ulp(np.array([0.0, 2.0 ** -130]), BF16).tolist() == [2.0 ** -133, 2.0 ** -133]


# ====================================================================== GPU fixtures and launchers
@pytest.fixture(scope="module")
def K():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from tests import kernel_harness
    return kernel_harness


GEMM_IMPL = {"": 0, "skinny": 1, "tc": 2, "simt": 3}  # it_b200_matmul_select: "" = the production dispatch


@pytest.fixture
def gemm_impl(request):
    from infinitensor_b200 import _lib
    _lib.lib.it_b200_matmul_select(GEMM_IMPL[request.param], 0)
    yield request.param
    _lib.lib.it_b200_matmul_select(0, 0)


# the decode step's GEMMs (Llama-7B widths): K, output widths, grouped launch
GEMM_CASES = {
    "qkv": (4096, [4096, 4096, 4096], True),  # skinny grouped, unsplit, deep ring
    "o": (4096, [4096], False),                # skinny split-K 4 on the 66 KB ring
    "down": (11008, [4096], False),            # skinny split-K, 43 k-tiles per split
    "ragged": (4104, [4104], False),           # 65 k-tiles as 17/17/17/14, partial last k-tile, 8-column last N tile
    "gateup": (4096, [11008, 11008], True),    # wgmma grouped, 172 tiles
    "logits": (4096, [32000], False),          # wgmma unsplit, 250 tiles
}
M_SWEEP = [1, 8, 16, 17, 24, 31, 32, 33, 48, 64]


class GemmData:
    """device operands at 64 rows and their float64 references, built once per (case, dtype)"""

    def __init__(self):
        self.cache = {}

    def get(self, K, case, dt):
        key = (case, dt)
        if key not in self.cache:
            k, ns, _ = GEMM_CASES[case]
            seed = 100 * (sorted(GEMM_CASES).index(case) + 1)
            x = ref64.activations(ref64.REF_ROWS, k, dt, seed)
            wd, refs = [], []
            for i, n in enumerate(ns):
                w = ref64.weights(k, n, dt, seed + 1 + i)
                refs.append(ref64.product(x, w))
                wd.append(K.dev(w, dt))
                del w
            resid = ref64.activations(ref64.REF_ROWS, ns[0], dt, seed + 9, scale=1.0)
            self.cache[key] = dict(x=K.dev(x, dt), w=wd, refs=refs, ns=ns, k=k, resid=resid, resid_d=K.dev(resid, dt))
        return self.cache[key]


@pytest.fixture(scope="module")
def gemm_data():
    return GemmData()


def run_matmul(K, d, m, dt, act=0, bias=False):
    """C[m, n] = X[:m] . W (+ the first m rows of the [64, n] residual as a full-stride bias) through it_b200_matmul"""
    import torch
    n, k = d["ns"][0], d["k"]
    c = torch.empty((m, n), dtype=K.TORCH_DT[dt], device="cuda")
    b = d["resid_d"] if bias else None
    K.L.check(K.L.lib.it_b200_matmul(dt, K.ptr(d["x"]), K.ptr(d["w"][0]), K.ptr(b), K.ptr(c), 1, m, n, k, m * k, 0, 0, 0,
                                     0, n if bias else 0, 1 if bias else 0, act, None, 0, K.stream()))
    K.sync()
    return K.host(c)


def run_grouped(K, d, m, dt):
    import ctypes
    import torch
    outs = [torch.empty((m, n), dtype=K.TORCH_DT[dt], device="cuda") for n in d["ns"]]
    VP = ctypes.c_void_p
    W = (VP * len(outs))(*[t.data_ptr() for t in d["w"]])
    C = (VP * len(outs))(*[t.data_ptr() for t in outs])
    K.L.check(K.L.lib.it_b200_matmul_grouped(dt, K.ptr(d["x"]), len(outs), W, C, K.L.i32arr(d["ns"]), m, d["k"], K.stream()))
    K.sync()
    return [K.host(o) for o in outs]


# ====================================================================== GPU §2: row-tile sweep against float64
@pytest.mark.gpu
@pytest.mark.parametrize("gemm_impl", ["", "skinny", "tc"], indirect=True)
@pytest.mark.parametrize("case", list(GEMM_CASES))
@pytest.mark.parametrize("dt", [BF16, F16])
def test_gemm_row_tiles_float64(K, gemm_data, gemm_impl, case, dt):
    """M = 1 .. 64 on each decode GEMM: MT = 1 / 2 / 4 of the skinny kernel (10 / 8 / 5-stage unsplit ring, 6 / 4 / 3-stage
    split-K ring), NT = 16 / 32 / 64 of the wgmma kernel (pinned tc on o / down: cluster split-K at NT = 32; pinned skinny on
    logits: 128-wide tiles)"""
    d = gemm_data.get(K, case, dt)
    grouped = GEMM_CASES[case][2]
    for m in M_SWEEP:
        outs = run_grouped(K, d, m, dt) if grouped else [run_matmul(K, d, m, dt)]
        for gi, (got, (ref, mag)) in enumerate(zip(outs, d["refs"])):
            ref64.assert_within(got, ref[:m], mag[:m], dt, what=f"{case} group {gi} M={m} impl={gemm_impl or 'auto'}")


def _fp8_operands(k, n, seed):
    """FP8 E4M3 codes with exponent fields 3..10 (magnitudes 2^-4 .. 3.75 over eight binades) and random signs, and a positive
    per-column scale with the 2^((j mod 5) - 2) column pattern"""
    rng = np.random.default_rng(seed)
    codes = ((rng.integers(3, 11, size=(k, n), dtype=np.uint8) << 3) | rng.integers(0, 8, size=(k, n), dtype=np.uint8)
             | (rng.integers(0, 2, size=(k, n), dtype=np.uint8) << 7))
    scale = (rng.uniform(0.5, 1.0, n) * 0.01 * ref64.col_scale(n)).astype(np.float32)
    return codes.astype(np.uint8), scale


_fp8_cache = {}


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["qkv", "down"])
@pytest.mark.parametrize("dt", [BF16, F16])
def test_fp8_weights_row_tiles_float64(K, case, dt):
    """it_b200_matmul_fp8w at MT = 2 (17..32 rows): q/k/v (three matrices, one launch) and down with the residual fused in, against
    float64 over the dequantised weights e4m3(code) x scale.  With the residual the product is rounded to T before the add
    (MatMul -> Add), which may cost up to one ulp of the product on top of the bound (the third term)."""
    import ctypes
    import torch
    k, ns, _ = GEMM_CASES[case]
    res = case == "down"
    key = (case, dt)
    if key not in _fp8_cache:
        _fp8_cache.clear()
        x = ref64.activations(ref64.REF_ROWS, k, dt, 600)
        qs = [_fp8_operands(k, n, 610 + i) for i, n in enumerate(ns)]
        refs = [ref64.product(x, oracle.e4m3_decode(c).astype(np.float64) * s.astype(np.float64)[None, :]) for c, s in qs]
        resid = ref64.activations(ref64.REF_ROWS, ns[0], dt, 620, scale=1.0) if res else None
        _fp8_cache[key] = (K.dev(x, dt), [K.raw(c) for c, _ in qs], [K.raw(s) for _, s in qs], refs, resid,
                           K.dev(resid, dt) if res else None)
    xd, cd, sd, refs, resid, rd = _fp8_cache[key]
    VP = ctypes.c_void_p
    arr = lambda ts: (VP * len(ts))(*[t.data_ptr() for t in ts])
    for m in (17, 24, 32):
        od = [torch.empty((m, n), dtype=K.TORCH_DT[dt], device="cuda") for n in ns]
        K.L.check(K.L.lib.it_b200_matmul_fp8w(dt, K.ptr(xd), len(ns), arr(cd), arr(sd), arr(od), K.L.i32arr(ns), m, k, K.ptr(rd),
                                              K.stream()))
        K.sync()
        for gi, (o, (ref, mag)) in enumerate(zip(od, refs)):
            ref, mag = ref[:m], mag[:m]
            extra = None
            if res:
                extra = ref64.ulp(ref, dt)
                ref, mag = ref + resid[:m], mag + np.abs(resid[:m])
            ref64.assert_within(K.host(o), ref, mag, dt, what=f"fp8 {case} group {gi} M={m}", extra=extra)


# ====================================================================== GPU §3: the residual epilogue as the schedule calls it
@pytest.mark.gpu
@pytest.mark.parametrize("gemm_impl", ["", "skinny", "tc", "simt"], indirect=True)
@pytest.mark.parametrize("case", ["o", "down", "ragged"])
@pytest.mark.parametrize("dt", [BF16, F16])
def test_residual_epilogue_is_matmul_then_add(K, gemm_data, gemm_impl, case, dt):
    """MatMul -> Add as runMatmul fuses it: the residual as a full [m, n] bias (strides 0, n, 1) with
    ITB_ACT_ROUND_BEFORE_BIAS | ITB_MATMUL_B_CONST equals MatMul followed by the Add kernel bit for bit; requesting the weights
    ahead of the PDL wait (ITB_MATMUL_B_CONST) changes no bit either"""
    d = gemm_data.get(K, case, dt)
    for m in (16, 24, 48):
        plain = run_matmul(K, d, m, dt, act=0)
        early = run_matmul(K, d, m, dt, act=0x200)
        assert np.array_equal(early, plain), f"{case} M={m}: ITB_MATMUL_B_CONST changed the product"
        fused = run_matmul(K, d, m, dt, act=0x300, bias=True)
        two = K.binary("add", early, d["resid"][:m], dt)
        assert np.array_equal(fused, two), \
            f"{case} M={m} impl={gemm_impl or 'auto'}: {np.sum(fused != two)} elements differ, max {np.abs(fused - two).max()}"


# ====================================================================== GPU §4: fused RoPE attention against the unfused kernels
POS_CODE = {"i32": (np.int32, 6), "u32": (np.uint32, 12), "i64": (np.int64, 7)}
# (B, Hq, Hkv, S_max, cache position of row 0)
ATTN_CASES = {
    "llama_layer": (16, 32, 32, 1024, 511),   # the benchmark's layer
    "rows_cross": (64, 8, 8, 128, 100),       # CTA unit ranges cross batch rows: the cos / sin table is rebuilt
    "heads_split": (1, 32, 32, 2048, 2047),   # each head split over CTAs and merged
    "chunk_edges": (3, 5, 5, 128, None),      # per-row positions on chunk edges
    "gqa": (16, 32, 8, 1024, 511),
    "mqa48": (2, 48, 1, 256, 100),
}
ROPE_SPECIAL = [65535, 4095, 1, 0]


def _positions(case, dt):
    B, Hq, Hkv, S, p0 = ATTN_CASES[case]
    if p0 is None:  # chunks of 64 rows (16-bit types) / 32 rows (fp32)
        rows = [63, 64, 65] if dt != F32 else [31, 32, 33]
    else:
        rows = [p0] + [(p0 + 131 * b) % S for b in range(1, B)]
        if B > 1:
            rows[1] = 0
        if B > 2:
            rows[2] = S - 1
    rope = [ROPE_SPECIAL[b] if b < 4 else (2713 * b + 17) % 65536 for b in range(B)]
    return np.array(rows), np.array(rope)


_attn_cache = {}


def _attn_inputs(K, case, dt):
    key = (case, dt)
    if key not in _attn_cache:
        _attn_cache.clear()
        B, Hq, Hkv, S, _ = ATTN_CASES[case]
        rng = np.random.default_rng(700 + sorted(ATTN_CASES).index(case))
        mk = lambda shape: K.dev(oracle.round_to(rng.standard_normal(shape, dtype=np.float32) * np.float32(0.5), dt), dt)
        _attn_cache[key] = [mk((B, Hkv, S, 128)), mk((B, Hkv, S, 128)), mk((B, Hq, 1, 128)), mk((B, Hkv, 1, 128)),
                            mk((B, Hkv, 1, 128))]
    return _attn_cache[key]


def bits(t):
    """a device tensor's raw bits as numpy integers"""
    import torch
    return t.view({2: torch.int16, 4: torch.int32}[t.element_size()]).cpu().numpy()


def attention(K, dt, inputs, Hq, Hkv, pos, pos_code, flags, rope=None, rope_code=None):
    """one AttentionKVCache launch on copies of the caches; RoPE folded in when `rope` (device positions) is given.  G = 1 goes
    through it_b200_attention_kvcache(_rope), G > 1 through it_b200_attention_kvcache_gqa.  Returns (out, k cache, v cache)
    as raw bits."""
    import torch
    kc, vc, q, k, v = inputs
    kc, vc = kc.clone(), vc.clone()
    B, _, S, D = kc.shape
    out = torch.empty_like(q)
    wsb = K.L.lib.it_b200_attention_kvcache_workspace(B, Hq, S, D)
    ws = torch.empty(int(wsb), dtype=torch.uint8, device="cuda")
    lib = K.L.lib
    if Hq != Hkv:
        rc = lib.it_b200_attention_kvcache_gqa(dt, K.ptr(kc), K.ptr(vc), K.ptr(q), K.ptr(k), K.ptr(v), K.ptr(pos), pos_code | flags,
                                               K.ptr(rope), rope_code or 0, K.ptr(out), B, Hq, Hkv, S, D, K.ptr(ws), int(wsb),
                                               K.stream())
    elif rope is not None:
        rc = lib.it_b200_attention_kvcache_rope(dt, K.ptr(kc), K.ptr(vc), K.ptr(q), K.ptr(k), K.ptr(v), K.ptr(pos), pos_code | flags,
                                                K.ptr(rope), rope_code, K.ptr(out), B, Hq, S, D, K.ptr(ws), int(wsb), K.stream())
    else:
        rc = lib.it_b200_attention_kvcache(dt, K.ptr(kc), K.ptr(vc), K.ptr(q), K.ptr(k), K.ptr(v), K.ptr(pos), pos_code | flags,
                                           K.ptr(out), B, Hq, S, D, K.ptr(ws), int(wsb), K.stream())
    K.L.check(rc)
    K.sync()
    return bits(out), bits(kc), bits(vc)


def rope_dev(K, dt, x, rope, rope_code):
    """it_b200_rope (the kernel behind K.rope) on a device [B, H, 1, 128] tensor"""
    import torch
    y = torch.empty_like(x)
    B, H = x.shape[:2]
    K.L.check(K.L.lib.it_b200_rope(dt, K.ptr(rope), rope_code, K.ptr(x), K.ptr(y), B, 1, H * 128, 128, K.stream()))
    K.sync()
    return y


@pytest.mark.gpu
@pytest.mark.parametrize("per_row", [False, True], ids=["pos0", "per_row"])
@pytest.mark.parametrize("dt", [F32, F16, BF16])
@pytest.mark.parametrize("case", list(ATTN_CASES))
def test_fused_rope_attention_is_rope_then_attention(K, case, dt, per_row):
    """RoPE folded into AttentionKVCache gives exactly the bits of RoPE on q and k followed by the unfused kernel: output, k
    cache (the rotated k is appended) and v cache.  RoPE positions differ from row to row and from the cache positions and
    include 0, 1, 4095 and 65535; every position dtype; the cache position as element 0 for all rows (the array still holds
    per-row values, which must be ignored) and with ITB_POS_PER_ROW; ITB_POS_IN_STEP changes nothing.  There is no float64
    RoPE reference: the angle is computed in fp32 on both sides (off by ~4e-3 rad at 65535), and the unfused kernels are pinned to
    the oracle elsewhere."""
    B, Hq, Hkv, S, _ = ATTN_CASES[case]
    inputs = _attn_inputs(K, case, dt)
    rows, rope_pos = _positions(case, dt)
    flags = 0x100 if per_row else 0
    q, k = inputs[2], inputs[3]
    ref = None
    for name, (npdt, code) in POS_CODE.items():
        pos, rope = K.raw(rows.astype(npdt)), K.raw(rope_pos.astype(npdt))
        qr, kr = rope_dev(K, dt, q, rope, code), rope_dev(K, dt, k, rope, code)
        if ref is None:
            ref_q, ref_k = bits(qr), bits(kr)
            ref = attention(K, dt, [inputs[0], inputs[1], qr, kr, inputs[4]], Hq, Hkv, pos, code, flags)
        else:  # the RoPE kernel itself reads every position dtype alike
            assert np.array_equal(bits(qr), ref_q) and np.array_equal(bits(kr), ref_k), f"RoPE with {name} positions"
        got = attention(K, dt, inputs, Hq, Hkv, pos, code, flags, rope=rope, rope_code=code)
        for what, g, r in zip(("out", "k cache", "v cache"), got, ref):
            assert np.array_equal(g, r), f"{what} with {name} positions: {np.sum(g != r)} elements differ"
        if name == "i64":
            got = attention(K, dt, inputs, Hq, Hkv, pos, code, flags | 0x200, rope=rope, rope_code=code)
            for what, g, r in zip(("out", "k cache", "v cache"), got, ref):
                assert np.array_equal(g, r), f"{what} under ITB_POS_IN_STEP: {np.sum(g != r)} elements differ"


def _rnd(shape, seed, dt):
    return oracle.round_to(np.random.default_rng(seed).standard_normal(shape).astype(np.float32) * np.float32(0.5), dt)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F32, F16, BF16])
def test_attention_batch_limit(K, dt):
    """B = 1024 (AS_MAX_B: the per-row position and prefix tables in shared memory) against the oracle, element-0 and per-row
    positions; B = 1025 is refused with a message before anything is written"""
    import torch
    B, H, S = 1024, 1, 64
    kc, vc = _rnd((B, H, S, 128), 28, dt), _rnd((B, H, S, 128), 29, dt)
    q, k, v = _rnd((B, H, 1, 128), 30, dt), _rnd((B, H, 1, 128), 31, dt), _rnd((B, H, 1, 128), 32, dt)
    tol = {F32: 1e-5, F16: 1e-3, BF16: 1e-2}[dt]  # as test_attention_parity (SURVEY 8(c))
    poss = (np.arange(B) * 7 + 3) % S
    for pos in (S - 1, poss):
        kc_ref, vc_ref = kc.copy(), vc.copy()
        if np.ndim(pos):
            ref = np.concatenate([oracle.attention_kvcache(kc_ref[b:b + 1], vc_ref[b:b + 1], q[b:b + 1], k[b:b + 1], v[b:b + 1],
                                                           int(pos[b]), dt) for b in range(B)])
        else:
            ref = oracle.attention_kvcache(kc_ref, vc_ref, q, k, v, pos, dt)
        out, kc_got, vc_got = K.attention_kvcache(kc, vc, q, k, v, pos, dt)
        np.testing.assert_allclose(out.astype(np.float64), ref.astype(np.float64), rtol=tol, atol=tol * 0.05)
        assert np.array_equal(kc_got, kc_ref) and np.array_equal(vc_got, vc_ref)
    B = 1025
    z = lambda shape: torch.full(shape, 0.25, dtype=K.TORCH_DT[dt], device="cuda")
    kcd, vcd, qd, kd, vd = z((B, H, S, 128)), z((B, H, S, 128)), z((B, H, 1, 128)), z((B, H, 1, 128)), z((B, H, 1, 128))
    out = torch.full((B, H, 1, 128), -3.0, dtype=K.TORCH_DT[dt], device="cuda")
    pd = K.raw(np.full(B, 5, np.int64))
    wsb = K.L.lib.it_b200_attention_kvcache_workspace(B, H, S, 128)
    ws = torch.empty(int(wsb), dtype=torch.uint8, device="cuda")
    rc = K.L.lib.it_b200_attention_kvcache(dt, K.ptr(kcd), K.ptr(vcd), K.ptr(qd), K.ptr(kd), K.ptr(vd), K.ptr(pd), 7, K.ptr(out),
                                           B, H, S, 128, K.ptr(ws), int(wsb), K.stream())
    K.sync()
    assert rc != 0 and "batch 1025" in K.L.last_error(), K.L.last_error()
    assert bool((out == -3.0).all()) and bool((kcd == 0.25).all()) and bool((vcd == 0.25).all())


# ====================================================================== GPU §5: the intended instantiations ran
@pytest.mark.gpu
def test_edge_cases_reach_the_intended_kernels(K, gemm_data):
    """Kernel names recorded by torch.profiler (CUDA activity only: CUPTI kernel records, no hardware counters) for one call
    from each group above.  A dispatch change that moves these shapes to other instantiations fails here instead of silently
    dropping the coverage."""
    import ctypes
    import torch
    dt, m = BF16, 24
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        run_matmul(K, gemm_data.get(K, "o", dt), m, dt, act=0x300, bias=True)  # skinny MT = 2, split-K
        run_grouped(K, gemm_data.get(K, "gateup", dt), m, dt)                # wgmma NT = 32, grouped
        k, n = 1024, 512
        x = K.dev(ref64.activations(m, k, dt, 900), dt)
        codes, scale = _fp8_operands(k, n, 901)
        cd, sd = K.raw(codes), K.raw(scale)
        od = torch.empty((m, n), dtype=K.TORCH_DT[dt], device="cuda")
        VP = ctypes.c_void_p
        K.L.check(K.L.lib.it_b200_matmul_fp8w(dt, K.ptr(x), 1, (VP * 1)(cd.data_ptr()), (VP * 1)(sd.data_ptr()),
                                              (VP * 1)(od.data_ptr()), K.L.i32arr([n]), m, k, None, K.stream()))
        inputs = _attn_inputs(K, "chunk_edges", dt)
        rows, rope_pos = _positions("chunk_edges", dt)
        attention(K, dt, inputs, 5, 5, K.raw(rows), 7, 0x100, rope=K.raw(rope_pos), rope_code=7)  # streaming kernel, ROPE
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if "CUDA" in str(e.device_type)}
    if not names:
        pytest.skip("the profiler recorded no CUDA kernel events (CUPTI activity tracing unavailable)")
    want = [r"gemm_skinny_kernel<[^<>]*, 2, 1, false>", r"gemm_skinny_kernel<[^<>]*, 2, 1, true>", r"gemm_tc_kernel<[^<>]*, 32>",
            r"attn_stream_kernel<[^<>]*, true>"]
    missing = [p for p in want if not any(re.search(p, nm) for nm in names)]
    assert not missing, f"not launched: {missing}; kernels seen: {sorted(names)}"
    print("kernels:", *sorted(n for n in names if re.search("gemm_|attn_", n)), sep="\n  ")
