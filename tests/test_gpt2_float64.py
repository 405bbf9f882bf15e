"""The GPT-2 forward's three kernel families against float64: prefill attention (`attention_prefill_kernel`) across score
ranges, tile edges and mask layouts; the Linear layers' GEMM epilogues (`gemm_tc_kernel`: bias, bias -> Gelu / Relu,
+ residual, the split-K reduce-scatter) at GPT-2's shapes; LayerNorm on every `launch_rowop` branch.

The kernel runs a two-pass softmax: pass A keeps an online (max, sum) per 32-column part of every 128-key tile, the four
parts meet once, pass B recomputes the scores and accumulates P.V.  The oracle comparison in test_gpu_kernels.py draws q, k
and v from N(0, 0.7^2), so scores stay within about +-2 and a whole-tensor tolerance of 1e-2 of max|ref| hides a dropped key.
Here (helpers in tests/prefill64.py):

* the reference is the graph's operator chain in float64 with every rounding point rounded straight to T, and the bound is
  per element: ulp_T(|ref|) + 2^-16 sum P|v| plus the cost of the roundings the kernel's fp32 arithmetic leaves ambiguous;
  the share of ambiguous scores must stay <= 1 % per case;
* nine score regimes cycle over the heads: flat, graded peaks arriving late or early, a sink at key 0, a peak on the
  diagonal, peaks just past it that the causal mask must remove, every score near -150, a tent up to +200, and a row whose
  maximum lies in the last key tile's column part 3 while the other parts see far smaller scores;
* v row j is scaled by 2^((j mod 5) - 2) and head h by 2^((h mod 3) - 1), so a key, row or head mix-up changes values by 2x;
* `out` is NaN before every launch and followed by a guard region that must stay untouched; every case runs twice with
  bit-identical output; the strided entry point (tensor-map modes 1 and 2) must equal the dense kernel on materialised copies
  bit for bit;
* rows whose every key is masked (-inf, or f16 sums that all overflow to -inf) are written as 0 (the unfused Softmax writes
  NaN); Skv = 0 writes zeros, Sq = 0 writes nothing, B * H = 65536 is refused without a launch.

The Linear epilogues (helpers in tests/gpt2_64.py) run GPT-2's four Linear layers at M = 128, the MLP pair again at M = 16
... 641 (split 8 down to 4, and unsplit at 641), ragged N = 776 and 2312, Relu and Gelu with and without a residual and
ITB_ACT_ROUND_BEFORE_BIAS, against act(X W + b) [+ r] in float64 with ref64's bound extended by the epilogue's roundings.
LayerNorm runs in fp32, f16 and bf16 at widths 64 ... 12296 (vector, scalar, block with and without the shared-memory row,
and a non-last axis), rows with |mean| / std up to 1e3 (fp32) / 1e2 and constant rows, scale and bias of size 1 and dim,
against float64 with the derived fp32 terms of the mean, the two-pass variance and rsqrtf.  Outputs of both are NaN-filled
and guarded, and every case runs twice with identical bits.

The CPU self-checks at the top run without a GPU: the float64 -> T rounding on known halfway cases, a float32 emulation of
the kernel's order of operations within half the bound (0.49 - 0.5: the output's own rounding, half an ulp, comes
closest), eleven injected kernel bugs that each fail it, and the case list reaching the tile, mask and tensor-map paths
it is meant to; float32 emulations of the split-K epilogue and of LayerNorm within half their bounds; a reduce-scatter row
range off by one, a bias indexed by row, a one-pass variance and a dropped last 16-byte chunk each failing them; split and
unsplit epilogue launches at M > 64 and every launch_rowop branch reached.
"""
import math
import re

import numpy as np
import pytest

from tests import prefill64
from tests import gpt2_64
from tests.prefill64 import Case, Reference
from tests.ref64 import BF16, F16, F32

DTYPES = [F16, BF16]
IDS = ["f16", "bf16"]


# ====================================================================== the GPU case list
# name: (B, H, Sq, Skv, D, mask, scale, regime offset, entry)   entry: "dense" | "qkv" (map mode 1) | "cache" (map mode 2)
DIV, MUL = ("div", None), ("mul", None)
CASES = {
    "gpt2_bench": (1, 12, 128, 128, 64, "causal", DIV, 0, "dense"),
    "gpt2_bench_qkv_view": (1, 12, 128, 128, 64, "causal", DIV, 3, "qkv"),
    "div_sqrt128": (1, 9, 200, 200, 128, "causal", DIV, 1, "dense"),        # sqrt(128) is no power of two: fp32 division
    "mul_inv_sqrt128": (1, 9, 160, 160, 128, "causal", MUL, 2, "dense"),
    "mul_inv_sqrt64": (1, 9, 130, 130, 64, "causal", MUL, 4, "dense"),
    "no_scale": (2, 5, 96, 300, 64, "causal", None, 5, "dense"),              # Sq < Skv: causal offset 204
    "q200_kv72": (2, 5, 200, 72, 128, "pad", DIV, 6, "dense"),               # Skv <= 64 + 8: the second V box half empty
    "kv40": (2, 5, 50, 40, 128, "pad", DIV, 7, "dense"),                     # Skv <= 64: the second V box out of bounds
    "seq1000": (1, 2, 1000, 1000, 128, "causal", MUL, 8, "dense"),
    "seq1024_d64": (1, 2, 1024, 1024, 64, "causal", DIV, 0, "dense"),
    "seq1024_d128": (1, 2, 1024, 1024, 128, "causal", DIV, 2, "dense"),
    "q128_kv2048": (1, 4, 128, 2048, 64, "causal", DIV, 5, "dense"),         # 16 key tiles, causal offset 1920
    "mask_batch": (2, 5, 100, 136, 64, "batch", DIV, 1, "dense"),
    "mask_head": (2, 5, 100, 136, 128, "head", MUL, 3, "dense"),
    "mask_odd_skv": (1, 9, 77, 129, 64, "causal", DIV, 4, "dense"),          # odd row pitch: the scalar mask path
    "mask_head_misaligned": (1, 9, 64, 200, 64, "head_misaligned", DIV, 6, "dense"),
    "mask_transposed": (1, 9, 100, 100, 64, "transposed", DIV, 7, "dense"),
    "mask_neg_inf": (1, 9, 130, 130, 64, "causal_inf", DIV, 8, "dense"),
    "fully_masked_rows": (1, 9, 40, 64, 64, "full", DIV, 0, "dense"),
    "kv_cache_views": (2, 5, 100, 150, 64, "causal", DIV, 2, "cache"),
    "kv_cache_views_d128": (1, 9, 72, 260, 128, "head", DIV, 5, "cache"),
}
for _s in (1, 17, 64, 127, 129, 255, 257):
    CASES[f"tile_edge_{_s}"] = (1, 9, _s, _s, 64 if _s % 2 else 128, "causal", DIV, _s % 9, "dense")

_cases, _refs = {}, {}


def case_of(name):
    if name not in _cases:
        B, H, Sq, Skv, D, mask, scale, off, _ = CASES[name]
        _cases[name] = Case(B, H, Sq, Skv, D, mask, scale, seed=2000 + sorted(CASES).index(name), offset=off)
    return _cases[name]


def ref_of(name, dt):
    if (name, dt) not in _refs:
        _refs[(name, dt)] = Reference(case_of(name), dt)
    return _refs[(name, dt)]


# ====================================================================== CPU: the float64 -> T rounding
def test_rnd_rounds_float64_straight_to_t():
    r = prefill64.rnd
    # halfway cases round to even
    assert r(1 + 2.0 ** -8, BF16) == 1.0 and r(1 + 3 * 2.0 ** -8, BF16) == 1 + 2.0 ** -6
    assert r(1 + 2.0 ** -11, F16) == 1.0 and r(1 + 3 * 2.0 ** -11, F16) == 1 + 2.0 ** -9
    # just above a midpoint: float64 rounds up; through float32 the excess is lost and the tie goes to even
    x = 1 + 2.0 ** -8 + 2.0 ** -40
    assert r(x, BF16) == 1 + 2.0 ** -7
    import oracle
    assert float(oracle.round_to(np.array([x], np.float32), BF16)[0]) == 1.0
    # f16 overflow: s + (-65504) below -65520 is -inf, -65520 itself ties away from the odd 65504
    assert r(-65519.99, F16) == -65504.0 and r(-65520.0, F16) == -np.inf and r(-70000.0, F16) == -np.inf
    assert r(3.4e38, BF16) == np.inf and r(3.39e38, BF16) == 3.3895313892515355e38 and r(-3.0e38, BF16) == prefill64.BIG_NEG[BF16]
    # subnormals, zero, infinities, NaN
    assert r(2.0 ** -25, F16) == 0.0 and r(3 * 2.0 ** -25, F16) == 2.0 ** -23 and r(2.0 ** -134, BF16) == 0.0
    y = r(np.array([0.0, -0.0, np.inf, -np.inf, np.nan]), F16)
    assert y[0] == 0 and y[2] == np.inf and y[3] == -np.inf and np.isnan(y[4])
    # f16 agrees with numpy's float64 -> float16 conversion (which rounds once) on random values across the range
    v = np.random.default_rng(0).standard_normal(200000) * np.exp2(np.random.default_rng(1).uniform(-26, 17, 200000))
    with np.errstate(over="ignore"):
        assert np.array_equal(r(v, F16), v.astype(np.float16).astype(np.float64))


# ====================================================================== CPU: the bound against an emulation of the kernel
EMU_CASES = {
    "causal_3tiles": (1, 9, 360, 360, 64, "causal", DIV, 0),   # last key tile 104 keys, every regime, ÷8 (multiply path)
    "head_5tiles": (1, 9, 72, 520, 128, "head", DIV, 3),      # ÷sqrt(128) (division), per-head mask, causal offset 448
}
_emu = {}


def _emu_case(name, dt):
    if (name, dt) not in _emu:
        B, H, Sq, Skv, D, mask, scale, off = EMU_CASES[name]
        if name not in _emu:
            _emu[name] = Case(B, H, Sq, Skv, D, mask, scale, seed=40 + sorted(EMU_CASES).index(name), offset=off)
        _emu[(name, dt)] = Reference(_emu[name], dt)
    return _emu[name], _emu[(name, dt)]


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
@pytest.mark.parametrize("name", sorted(EMU_CASES))
def test_bound_passes_emulated_kernel(name, dt):
    c, R = _emu_case(name, dt)
    assert set(c.regime.ravel()) == set(prefill64.REGIMES)
    got = prefill64.emulate(c, dt)
    msg = prefill64.report(R.violations(got, scale=0.5), got, R, f"emulated {name} {prefill64.NAMES[dt]} against half the bound")
    assert msg is None, msg
    assert R.share_s() <= 0.01, f"{100 * R.share_s():.2f} % of the scores are ambiguous"


@pytest.mark.parametrize("mutation", prefill64.MUTATIONS)
def test_bound_catches_kernel_bugs(mutation):
    """bf16, the coarser type: each injected bug leaves elements outside the bound on at least one emulated case"""
    seen = []
    for name in sorted(EMU_CASES):
        c, R = _emu_case(name, BF16)
        seen.append(int(R.violations(prefill64.emulate(c, BF16, mutation)).sum()))
    assert any(seen), f"{mutation} stays inside the bound on {sorted(EMU_CASES)}"


def test_inputs_shape_the_scores():
    """the regimes land where they are meant to (scores from the rounded data, after scaling, before the mask)"""
    n = 360  # the last key tile, keys 256 .. 359, reaches column part 3
    c = Case(1, 9, n, n, 64, None, DIV, seed=3)
    x, _ = c.products()
    for h in range(9):
        s = x[0, h] / 8.0
        reg = c.regime[0, h]
        if reg == "neg150":
            assert s.max() < -130
        elif reg == "pos200":
            assert abs(s.max() - 200) < 3 and s.min() < 150
        elif reg == "sink":
            assert (s.argmax(1) == 0).all()
        elif reg == "part3":
            j = s.argmax(1)
            assert (j // 128 == 2).all() and ((j % 128) // 32 == 3).all()
            assert s[:, :256].max() < s.max() - 60 and s[:, 256:352].max() < s.max() - 60
        elif reg in ("diag", "past_diag"):
            # (the flat part's noise, std about 1, rides on the ramp)
            causal = np.where(np.tril(np.ones((n, n), bool)), s, -np.inf)
            assert (np.arange(n) - causal.argmax(1) <= 3).mean() > 0.9
            if reg == "past_diag":
                assert (s[:-1, 1:].diagonal() > s.diagonal()[:-1]).mean() > 0.8
        elif reg == "late":
            assert (s.argmax(1) == round(0.85 * (n - 1))).all()
        elif reg == "flat":
            assert 0.5 < s.std() < 2 and np.abs(s).max() < 10


def _tc_tiles(Sq, Skv):
    return -(-Sq // 128), -(-Skv // 128)


def test_case_list_reaches_the_kernel_paths():
    keys, ragged_q, short_last, scales, paths, modes, part3 = 0, False, False, set(), set(), set(), False
    for name, (B, H, Sq, Skv, D, mask, scale, off, entry) in CASES.items():
        c = case_of(name)
        keys = max(keys, _tc_tiles(Sq, Skv)[1])
        ragged_q |= Sq % 128 != 0 and Sq > 128
        short_last |= Skv > 128 and Skv % 128 != 0 and Skv % 128 < 64
        if scale is None:
            scales.add("none")
        else:
            cv = c.scale_value(F16)
            scales.add("mul" if scale[0] == "mul" or math.frexp(cv)[0] == 0.5 else "div")
        for dt in DTYPES:
            paths |= prefill64.mask_paths(c, dt)
        modes.add({"dense": 0, "qkv": 1, "cache": 2}[entry])
        part3 |= "part3" in set(c.regime.ravel()) and Skv > 128 and (Skv - 1) % 128 >= 96
    assert keys >= 8, keys
    assert ragged_q and short_last
    assert scales == {"none", "mul", "div"}, scales
    assert paths == {"vector", "scalar", "misaligned", "mi0", "mj"}, paths
    assert modes == {0, 1, 2}
    assert part3


# ====================================================================== GPU plumbing
@pytest.fixture(scope="module")
def K():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from tests import kernel_harness
    return kernel_harness


GUARD = 4096
GUARD_BITS = {F32: 0x7FC0BEEF, F16: 0x7E5A, BF16: 0x7E5A}
NAN_BITS = {F32: 0x7FFFFFFF, F16: 0x7FFF, BF16: 0x7FFF}


def guarded(K, n, dt):
    """(integer buffer of n + GUARD elements, its first n as a T view): NaN-filled, a guard pattern after it"""
    import torch
    it = torch.int32 if dt == F32 else torch.int16
    buf = torch.full((n + GUARD,), GUARD_BITS[dt], dtype=it, device="cuda")
    buf[:n] = NAN_BITS[dt]
    return buf, buf[:n].view(K.TORCH_DT[dt])


def guard_ok(buf, n, dt):
    return bool((buf[n:] == GUARD_BITS[dt]).all())


def _dev_mask(K, c, dt):
    store, strides, off, _ = c.mask(dt)
    if store is None:
        return None, (0, 0, 0, 0)
    return K.dev(store.ravel(), dt), strides


def _scale(K, c, dt):
    if c.scale is None:
        return None, 0
    return K.dev(np.array([c.scale_value(dt)], np.float32), dt), int(c.scale[0] == "div")


def run_dense(K, c, dt, q=None, k=None, v=None):
    """the dense entry point; returns (out [B, H, Sq, D] float32, guard intact)"""
    n = c.B * c.H * c.Sq * c.D
    buf, out = guarded(K, n, dt)
    qd = K.dev(c.q if q is None else q, dt)
    kd = K.dev(c.k if k is None else k, dt)
    vd = K.dev(c.v if v is None else v, dt)
    md, (mb, mh, mi, mj) = _dev_mask(K, c, dt)
    sd, div = _scale(K, c, dt)
    K.L.check(K.L.lib.it_b200_attention_prefill(dt, K.ptr(qd), K.ptr(kd), K.ptr(vd), K.ptr(out), c.B, c.H, c.Sq, c.Skv, c.D,
                                                K.ptr(sd), div, K.ptr(md), mb, mh, mi, mj, K.stream()))
    K.sync()
    ok = guard_ok(buf, n, dt)
    return out.float().cpu().numpy().reshape(c.B, c.H, c.Sq, c.D), ok


def run_qkv(K, c, dt):
    """map mode 1: q / k / v as views of one projection output [B, S, 3 H D], out written as [B, S, H D]"""
    import ctypes
    B, H, S, D = c.B, c.H, c.Sq, c.D
    assert c.Sq == c.Skv
    d = H * D
    qkv = np.concatenate([t.transpose(0, 2, 1, 3).reshape(B, S, d) for t in (c.q, c.k, c.v)], axis=2)
    xd = K.dev(qkv, dt)
    n = B * S * d
    buf, out = guarded(K, n, dt)
    md, (mb, mh, mi, mj) = _dev_mask(K, c, dt)
    sd, div = _scale(K, c, dt)
    es, base = xd.element_size(), xd.data_ptr()
    view, ost = K.L.i64arr([S * 3 * d, D, 3 * d]), K.L.i64arr([S * d, D, d])
    K.L.check(K.L.lib.it_b200_attention_prefill_strided(dt, ctypes.c_void_p(base), ctypes.c_void_p(base + d * es),
                                                        ctypes.c_void_p(base + 2 * d * es), K.ptr(out), B, H, S, S, D, view, view,
                                                        view, ost, K.ptr(sd), div, K.ptr(md), mb, mh, mi, mj, K.stream()))
    K.sync()
    ok = guard_ok(buf, n, dt)
    return out.float().cpu().numpy().reshape(B, S, H, D).transpose(0, 2, 1, 3), ok


def run_cache(K, c, dt):
    """map mode 2: k / v as views of [B, H, S_max, D] caches (rows from Skv on NaN), q as a view of a [B, H, Sq + 40, D] buffer
    (rows from Sq on NaN)"""
    B, H, Sq, Skv, D = c.B, c.H, c.Sq, c.Skv, c.D
    smax, qmax = Skv + 72, Sq + 40
    kc = np.full((B, H, smax, D), np.nan, np.float32)
    vc = kc.copy()
    qb = np.full((B, H, qmax, D), np.nan, np.float32)
    kc[:, :, :Skv], vc[:, :, :Skv], qb[:, :, :Sq] = c.k, c.v, c.q
    kd, vd, qd = K.dev(kc, dt), K.dev(vc, dt), K.dev(qb, dt)
    n = B * H * Sq * D
    buf, out = guarded(K, n, dt)
    md, (mb, mh, mi, mj) = _dev_mask(K, c, dt)
    sd, div = _scale(K, c, dt)
    kv = K.L.i64arr([H * smax * D, smax * D, D])
    K.L.check(K.L.lib.it_b200_attention_prefill_strided(dt, K.ptr(qd), K.ptr(kd), K.ptr(vd), K.ptr(out), B, H, Sq, Skv, D,
                                                        K.L.i64arr([H * qmax * D, qmax * D, D]), kv, kv,
                                                        K.L.i64arr([H * Sq * D, Sq * D, D]), K.ptr(sd), div, K.ptr(md), mb, mh,
                                                        mi, mj, K.stream()))
    K.sync()
    ok = guard_ok(buf, n, dt)
    return out.float().cpu().numpy().reshape(B, H, Sq, D), ok


def check_case(K, name):
    entry = CASES[name][-1]
    c = case_of(name)
    fails, stats = [], []
    for dt in DTYPES:
        R = ref_of(name, dt)
        what = f"{name} {prefill64.NAMES[dt]}"
        runner = {"dense": run_dense, "qkv": run_qkv, "cache": run_cache}[entry]
        got, ok = runner(K, c, dt)
        fails += [] if ok else [f"{what}: guard after out written"]
        msg = prefill64.report(R.violations(got), got, R, what)
        if msg:
            bad = R.violations(got)
            b, h, i, _ = (int(t) for t in np.argwhere(bad)[0])
            if not R.dead[b, h, i]:
                kt, part = prefill64.where_max(c, dt, b, h, i)
                msg += f"\n  (first failing row: its maximum score is in key tile {kt}, column part {part}; regime {c.regime[b, h]})"
            fails.append(msg)
        again, _ = runner(K, c, dt)
        if not np.array_equal(again.view(np.int32), got.view(np.int32)):
            fails.append(f"{what}: the second launch differs from the first in {int((again != got).sum())} elements")
        if entry != "dense":
            dense, _ = run_dense(K, c, dt)
            if not np.array_equal(dense.view(np.int32), got.view(np.int32)):
                fails.append(f"{what}: the strided views differ from the dense kernel in {int((dense != got).sum())} elements")
        if R.share_s() > 0.01:
            fails.append(f"{what}: {100 * R.share_s():.2f} % of the scores are ambiguous (> 1 %): the case checks little")
        stats.append(f"{prefill64.NAMES[dt]}: worst |got - ref| / bound {R.ratio(got):.3f}, ambiguous scores "
                     f"{100 * R.share_s():.3f} %, ambiguous P {100 * R.share_p():.2f} %, dead rows {int(R.dead.sum())}")
    print(f"{name}: " + "; ".join(stats))
    assert not fails, "\n".join(fails)


# ====================================================================== GPU: the cases
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_prefill_attention_float64(K, name):
    check_case(K, name)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
def test_prefill_attention_empty_extents(K, dt):
    """Skv = 0: every row has no key and is written as 0.  Sq = 0: nothing is written"""
    c = Case(2, 3, 5, 0, 64, None, DIV, seed=5)
    for runner in (run_dense, run_cache):  # (the strided entry point: map mode 2)
        got, ok = runner(K, c, dt)
        assert ok and np.array_equal(got, np.zeros_like(got)) and not np.signbit(got).any(), runner.__name__
    import torch
    buf = torch.full((GUARD,), GUARD_BITS[dt], dtype=torch.int16, device="cuda")
    qd = K.dev(np.ones((2, 3, 8, 64), np.float32), dt)
    K.L.check(K.L.lib.it_b200_attention_prefill(dt, K.ptr(qd), K.ptr(qd), K.ptr(qd), K.ptr(buf), 2, 3, 0, 8, 64, None, 0, None,
                                                0, 0, 0, 0, K.stream()))
    K.sync()
    assert bool((buf == GUARD_BITS[dt]).all())


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
def test_prefill_attention_grid_limit(K, dt):
    """B * H = 65535 at Sq = Skv = 1: one unmasked key, so out = v bit for bit.  B * H = 65536 is refused before a launch"""
    import torch
    rng = np.random.default_rng(9)
    BH, D = 65535, 64
    v = prefill64.rnd(rng.standard_normal((BH, 1, 1, D)), dt).astype(np.float32)
    q = prefill64.rnd(rng.standard_normal((BH, 1, 1, D)), dt).astype(np.float32)
    qd, vd = K.dev(q, dt), K.dev(v, dt)
    n = BH * D
    buf, out = guarded(K, n, dt)
    K.L.check(K.L.lib.it_b200_attention_prefill(dt, K.ptr(qd), K.ptr(qd), K.ptr(vd), K.ptr(out), 5, BH // 5, 1, 1, D, None, 0,
                                                None, 0, 0, 0, 0, K.stream()))
    K.sync()
    assert guard_ok(buf, n, dt)
    assert np.array_equal(out.float().cpu().numpy().ravel(), v.ravel())
    big = torch.full((65536 * D + GUARD,), GUARD_BITS[dt], dtype=torch.int16, device="cuda")
    qb = torch.zeros((65536 * D,), dtype=K.TORCH_DT[dt], device="cuda")
    rc = K.L.lib.it_b200_attention_prefill(dt, K.ptr(qb), K.ptr(qb), K.ptr(qb), K.ptr(big), 2, 32768, 1, 1, D, None, 0, None, 0,
                                           0, 0, 0, K.stream())
    K.sync()
    assert rc != 0
    assert bool((big == GUARD_BITS[dt]).all())


# ====================================================================== Linear layers: the GEMM epilogues
# name: (M, K, N, act, residual, round before bias, entry)   act 0 none, 1 Relu, 4 Gelu
# entry: "matmul" (it_b200_matmul, production dispatch) | "matmul_tc" (the same, gemm_tc pinned) | "fused" (it_b200_matmul_fused)
LINEAR_CASES = {
    "c_attn": (128, 768, 2304, 0, False, False, "matmul"),
    "attn_c_proj_residual": (128, 768, 768, 0, True, False, "fused"),
    "mlp_c_fc_gelu": (128, 768, 3072, 4, False, False, "fused"),
    "mlp_c_proj_residual": (128, 3072, 768, 0, True, False, "fused"),        # split-K 8, reduce-scatter
    "ragged_n776_gelu_residual": (128, 768, 776, 4, True, False, "fused"),
    "ragged_n2312_relu_residual": (128, 3072, 2312, 1, True, False, "fused"),  # split 6 over 19 column tiles
    "relu": (200, 768, 1024, 1, False, False, "fused"),
    "gelu_residual": (200, 768, 1024, 4, True, False, "fused"),
    "split_gelu_residual": (128, 3072, 768, 4, True, False, "fused"),
    "split_relu": (128, 3072, 768, 1, False, False, "fused"),
    # ITB_ACT_ROUND_BEFORE_BIAS is an it_b200_matmul flag: the wgmma kernel pinned, direct and split epilogue
    "round_before_bias": (128, 768, 768, 0, False, True, "matmul_tc"),
    "split_round_before_bias_relu": (128, 3072, 768, 1, False, True, "matmul_tc"),
}
for _m in (16, 65, 100, 129, 256, 640, 641):  # at 640 five row chunks still split (4 ways); at 641 six do not
    LINEAR_CASES[f"mlp_c_fc_gelu_m{_m}"] = (_m, 768, 3072, 4, False, False, "fused")
    LINEAR_CASES[f"mlp_c_proj_residual_m{_m}"] = (_m, 3072, 768, 0, True, False, "fused")
LINEAR_MMAX = 641
_linear = {}


def linear_of(K_, N):
    """the operands of one (K, N) weight shape at LINEAR_MMAX rows, shared by every case and type"""
    if (K_, N) not in _linear:
        _linear[(K_, N)] = gpt2_64.Linear(LINEAR_MMAX, K_, N, seed=K_ + 7 * N)
    return _linear[(K_, N)]


LINEAR_EMU = (100, 3072, 256)  # split 8 at 16 rows per rank


@pytest.mark.parametrize("dt", DTYPES, ids=IDS)
@pytest.mark.parametrize("act,residual,rb", [(0, True, False), (4, False, False), (4, True, False), (1, True, False),
                                             (1, False, True)])
def test_linear_bound_passes_emulated_epilogue(act, residual, rb, dt):
    M, K_, N = LINEAR_EMU
    L = gpt2_64.Linear(M, K_, N, seed=11)
    ref, bound = gpt2_64.linear_reference(L, M, act, residual, rb, dt)
    got = gpt2_64.emulate_linear(L, M, act, residual, rb, dt)
    assert gpt2_64.tc_split(M, K_, N)[0] == 8
    assert np.all(np.abs(got - ref) <= 0.5 * bound), float(np.nanmax(np.abs(got - ref) / bound))


@pytest.mark.parametrize("mutation", gpt2_64.LINEAR_MUTATIONS)
def test_linear_bound_catches_epilogue_bugs(mutation):
    """a reduce-scatter rank covering rows one past its range, and a bias read by row, each fail the bound (bf16)"""
    M, K_, N = LINEAR_EMU
    L = gpt2_64.Linear(M, K_, N, seed=11)
    for act, residual in ((0, True), (4, False)):
        ref, bound = gpt2_64.linear_reference(L, M, act, residual, False, BF16)
        got = gpt2_64.emulate_linear(L, M, act, residual, False, BF16, mutation)
        assert (~(np.abs(got - ref) <= bound)).any(), (mutation, act, residual)


def test_linear_cases_reach_split_and_unsplit_launches():
    splits = {}
    for name, (M, K_, N, act, res, rb, entry) in LINEAR_CASES.items():
        if entry != "matmul" and M > 64:
            splits.setdefault(gpt2_64.tc_split(M, K_, N)[0] > 1, []).append(name)
    assert set(splits) == {True, False}, splits
    assert gpt2_64.tc_split(128, 3072, 768)[0] == 8 and gpt2_64.tc_split(640, 3072, 768)[0] == 4
    assert gpt2_64.tc_split(641, 3072, 768)[0] == 1


def run_linear(K, name, dt):
    M, K_, N, act, res, rb, entry = LINEAR_CASES[name]
    L = linear_of(K_, N)
    xd, wd, bd = K.dev(L.x[:M], dt), K.dev(L.w, dt), K.dev(L.bias, dt)
    rd = K.dev(L.res[:M], dt) if res else None
    n = M * N
    buf, out = guarded(K, n, dt)
    if entry.startswith("matmul"):
        if entry == "matmul_tc":
            K.L.lib.it_b200_matmul_select(2, 0)
        try:
            rc = K.L.lib.it_b200_matmul(dt, K.ptr(xd), K.ptr(wd), K.ptr(bd), K.ptr(out), 1, M, N, K_, M * K_, 0, 0, 0, 0, 0, 1,
                                        act | (0x100 if rb else 0), None, 0, K.stream())
        finally:
            K.L.lib.it_b200_matmul_select(0, 0)
    else:
        rc = K.L.lib.it_b200_matmul_fused(dt, K.ptr(xd), K.ptr(wd), K.ptr(bd), K.ptr(rd), K.ptr(out), 1, M, N, K_, M * K_, 0, 0,
                                          0, 0, 0, 1, act | 0x200 | (0x100 if rb else 0), K.stream())
    assert rc == 0, f"{name}: rc {rc} (2: the wgmma epilogue did not take the shape)"
    K.sync()
    return out.float().cpu().numpy().reshape(M, N), guard_ok(buf, n, dt)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(LINEAR_CASES))
def test_linear_epilogue_float64(K, name):
    M, K_, N, act, res, rb, entry = LINEAR_CASES[name]
    fails, stats = [], []
    for dt in DTYPES:
        what = f"{name} {prefill64.NAMES[dt]}"
        ref, bound = gpt2_64.linear_reference(linear_of(K_, N), M, act, res, rb, dt)
        got, ok = run_linear(K, name, dt)
        fails += [] if ok else [f"{what}: guard after the output written"]
        bad = ~(np.abs(got - ref) <= bound)
        if bad.any():
            i, j = (int(t) for t in np.argwhere(bad)[0])
            split, rows_per, mpad, _ = gpt2_64.tc_split(M, K_, N)
            fails.append(f"{what}: {int(bad.sum())} of {bad.size} outside the bound; first (row {i}, column {j}): got {got[i, j]!r}, "
                         f"float64 {ref[i, j]!r}, bound {bound[i, j]:.3g}; row chunk {i // mpad}, column tile {j // 128}, "
                         f"split {split} (reduce-scatter rank {(i % mpad) // rows_per})")
        again, _ = run_linear(K, name, dt)
        if not np.array_equal(again.view(np.int32), got.view(np.int32)):
            fails.append(f"{what}: the second launch differs from the first")
        with np.errstate(invalid="ignore"):
            stats.append(f"{prefill64.NAMES[dt]}: worst |got - ref| / bound {float(np.nanmax(np.abs(got - ref) / bound)):.3f}")
    print(f"{name} (split {gpt2_64.tc_split(M, K_, N)[0]}): " + "; ".join(stats))
    assert not fails, "\n".join(fails)


# ====================================================================== LayerNorm
LN_DTYPES = [F32, F16, BF16]
# name: (rows, dim, inner, scale / bias size)   inner > 1: the normalised axis is not the last one (strided_kernel)
LN_CASES = {
    "d768_r128": (128, 768, 1, "dim"),
    "d768_r1": (1, 768, 1, "dim"),
    "d768_r10000_size1": (10000, 768, 1, "one"),
    "d64": (129, 64, 1, "dim"),
    "d200_size1": (129, 200, 1, "one"),
    "d100": (129, 100, 1, "dim"),
    "d770_size1": (129, 770, 1, "one"),
    "d1024": (129, 1024, 1, "dim"),
    "d1032": (129, 1032, 1, "dim"),
    "d4096": (129, 4096, 1, "dim"),
    "d12288": (129, 12288, 1, "dim"),
    "d12296": (129, 12296, 1, "dim"),
    "strided_d100_inner6": (3, 100, 6, "dim"),
    "strided_d768_inner5": (2, 768, 5, "one"),
}
LN_EPS = 1e-5


def ln_inputs(name, dt):
    """(x as the kernel reads it, [outer, dim, inner]; the rows, [outer * inner, dim]; scale; bias)"""
    outer, dim, inner, size = LN_CASES[name]
    seed = sorted(LN_CASES).index(name)
    rows = gpt2_64.ln_rows(outer * inner, dim, dt, seed)
    sc, bi = gpt2_64.ln_params(dim, size, dt, seed + 100)
    x = np.ascontiguousarray(rows.reshape(outer, inner, dim).transpose(0, 2, 1))
    return x, rows, sc, bi


def test_layernorm_cases_reach_every_rowop_branch():
    seen = set()
    for name, (outer, dim, inner, size) in LN_CASES.items():
        for dt in LN_DTYPES:
            seen.add(gpt2_64.rowop_path(dt, dim, inner))
    want = {"strided", "vec1", "vec3", "vec4", "block_cached", "block_uncached"}
    assert want <= seen and any(p.startswith("warp") for p in seen), sorted(seen)
    assert gpt2_64.rowop_path(F32, 768) == "warp32" and gpt2_64.rowop_path(F16, 770) == "warp32"


@pytest.mark.parametrize("dt", LN_DTYPES, ids=["fp32"] + IDS)
@pytest.mark.parametrize("dim", [768, 100, 4096, 12296])
def test_layernorm_bound_passes_emulation(dim, dt):
    path = gpt2_64.rowop_path(dt, dim)
    x = gpt2_64.ln_rows(129, dim, dt, 3)
    sc, bi = gpt2_64.ln_params(dim, "dim", dt, 4)
    ref, bound = gpt2_64.ln_reference(x, sc, bi, LN_EPS, dt, gpt2_64.chain_length(path, dim))
    got = gpt2_64.emulate_ln(x, sc, bi, LN_EPS, dt, path)
    assert np.all(np.abs(got - ref) <= 0.5 * bound), float(np.max(np.abs(got - ref) / bound))


@pytest.mark.parametrize("mutation", gpt2_64.LN_MUTATIONS)
def test_layernorm_bound_catches_bugs(mutation):
    """a one-pass variance E[x^2] - mu^2 and a dropped last 16-byte chunk each fail the bound"""
    for dt in LN_DTYPES:
        path = gpt2_64.rowop_path(dt, 768)
        x = gpt2_64.ln_rows(129, 768, dt, 3)
        sc, bi = gpt2_64.ln_params(768, "dim", dt, 4)
        ref, bound = gpt2_64.ln_reference(x, sc, bi, LN_EPS, dt, gpt2_64.chain_length(path, 768))
        if (~(np.abs(gpt2_64.emulate_ln(x, sc, bi, LN_EPS, dt, path, mutation) - ref) <= bound)).any():
            return
    raise AssertionError(f"{mutation} stays inside the bound in every type")


def run_layernorm(K, name, dt):
    outer, dim, inner, size = LN_CASES[name]
    x, _, sc, bi = ln_inputs(name, dt)
    xd, sd, bd = K.dev(x, dt), K.dev(sc, dt), K.dev(bi, dt)
    n = x.size
    buf, out = guarded(K, n, dt)
    K.L.check(K.L.lib.it_b200_layernorm(dt, K.ptr(xd), K.ptr(sd), K.ptr(bd), K.ptr(out), outer, dim, inner, sd.numel(), bd.numel(),
                                        LN_EPS, K.stream()))
    K.sync()
    y = out.float().cpu().numpy().reshape(outer, dim, inner).transpose(0, 2, 1).reshape(outer * inner, dim)
    return y, guard_ok(buf, n, dt)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(LN_CASES))
def test_layernorm_float64(K, name):
    outer, dim, inner, size = LN_CASES[name]
    fails, stats = [], []
    for dt in LN_DTYPES:
        path = gpt2_64.rowop_path(dt, dim, inner)
        what = f"{name} {prefill64.NAMES.get(dt, 'fp32')} ({path})"
        _, rows, sc, bi = ln_inputs(name, dt)
        ref, bound = gpt2_64.ln_reference(rows, sc, bi, LN_EPS, dt, gpt2_64.chain_length(path, dim))
        got, ok = run_layernorm(K, name, dt)
        fails += [] if ok else [f"{what}: guard after the output written"]
        bad = ~(np.abs(got - ref) <= bound)
        if bad.any():
            r, d = (int(t) for t in np.argwhere(bad)[0])
            fails.append(f"{what}: {int(bad.sum())} of {bad.size} outside the bound; first (row {r}, column {d}, 16-byte chunk "
                         f"{d // 8}): got {got[r, d]!r}, float64 {ref[r, d]!r}, bound {bound[r, d]:.3g}")
        again, _ = run_layernorm(K, name, dt)
        if not np.array_equal(again.view(np.int32), got.view(np.int32)):
            fails.append(f"{what}: the second launch differs from the first")
        with np.errstate(invalid="ignore"):
            stats.append(f"{prefill64.NAMES.get(dt, 'fp32')}: worst |got - ref| / bound {float(np.nanmax(np.abs(got - ref) / bound)):.3f}")
    print(f"{name}: " + "; ".join(stats))
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
def test_softmax_caches_a_12288_row(K):
    """Softmax shares row_block_kernel's shared-memory row with LayerNorm: 12288 floats need the opted-in dynamic limit too"""
    x = np.random.default_rng(5).standard_normal((3, 12288)).astype(np.float32) * 4
    got = K.softmax(x, -1, F32).astype(np.float64)
    e = np.exp(x.astype(np.float64) - x.max(1, keepdims=True))
    ref = e / e.sum(1, keepdims=True)
    assert np.all(np.abs(got - ref) <= 1e-5 * ref + 1e-12), float(np.max(np.abs(got - ref) / ref))


# ====================================================================== GPU: the intended instantiations ran
def profiled_kernel_names():
    """kernel names recorded by torch.profiler (CUDA activity only): prefill attention per head dim and type, an unsplit and a
    split Linear epilogue, LayerNorm on every launch_rowop branch"""
    import torch
    from tests import kernel_harness as K
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for dt in DTYPES:
            for D in (64, 128):
                run_dense(K, Case(1, 2, 130, 130, D, "causal", DIV, seed=7), dt)
            for name in ("attn_c_proj_residual", "mlp_c_proj_residual"):  # unsplit and split gemm_tc
                run_linear(K, name, dt)
        for dt in LN_DTYPES:
            for name in ("d768_r128", "d64", "d100", "d1024", "d4096", "d12296", "strided_d100_inner6"):
                run_layernorm(K, name, dt)
        torch.cuda.synchronize()
    return sorted({e.name for e in prof.events() if "CUDA" in str(e.device_type)})


@pytest.mark.gpu
def test_gpt2_cases_reach_every_instantiation():
    """in a child process, as test_attention_float64.py does (a profiler session in the test process lost the records of a
    later check's first kernels in a full-suite run)"""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = "import json; from tests.test_gpt2_float64 import profiled_kernel_names as f; print(json.dumps(f()))"
    r = subprocess.run([sys.executable, "-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    names = set(json.loads(r.stdout.strip().splitlines()[-1]))
    if not names:
        pytest.skip("the profiler recorded no CUDA kernel events (CUPTI activity tracing unavailable)")
    want = [rf"attention_prefill_kernel<{t}, {d}>" for t in ("__half", "__nv_bfloat16") for d in (64, 128)]
    want += [r"gemm_tc_kernel<__half, 128>", r"gemm_tc_kernel<__nv_bfloat16, 128>"]
    for t in ("__half", "__nv_bfloat16"):
        want += [rf"row_warp_vec_kernel<{t}, {c}, 1>" for c in (1, 3, 4)] + [rf"row_warp_kernel<{t}, 4, 1>"]
    for t in ("float", "__half", "__nv_bfloat16"):
        want += [rf"row_block_kernel<{t}, 1>", rf"strided_kernel<{t}, 1>"]
    want += [r"row_warp_kernel<float, 32, 1>", r"row_warp_kernel<float, 2, 1>"]
    missing = [p for p in want if not any(re.search(p, nm) for nm in names)]
    assert not missing, f"not launched: {missing}; kernels seen: {sorted(n for n in names if 'kernel' in n)}"
