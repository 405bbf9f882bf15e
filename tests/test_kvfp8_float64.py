"""Decode attention over an FP8 E4M3 KV cache (attn_stream_kv8_kernel, attn_gqa_kv8_kernel in attention.cu) against float64 at
large score ranges, across every CTA split and merge, with the append's quantiser at its edges.

The FP8 kernels share the 16-bit kernels' dealing, ring, tickets and merge, with 16 KiB chunks of one-byte codes: 128 rows at
D = 128 and 256 at D = 64.  Here (helpers in tests/kvfp8_64.py, on tests/attn64.py's regimes and dealing model):

* every case cycles nine score regimes over (batch row, query head): attn64's eight, with the scores computed from the decoded
  codes, and "sat", a peak on an appended k row whose large elements lie beyond +-448 * scale, with a saturated v row;
* K scales carry 2^((h mod 5) - 2) and V scales 2^((h mod 3) - 1) on bases 0.7 / 448 and 1.7 / 448, so a scale read from the
  wrong head, K's for V or a query head's for its KV head's changes values by 2x or more;
* every cache row from p on holds NaN codes (0x7F and 0xFF mixed) before the launch (row p is overwritten by the append), and
  `out` and the whole attention workspace are NaN; guard regions after each cache, after `out` and after each scale array
  must stay untouched; the caches are compared byte for byte with row p = quantise of the appended k / v;
* every case runs twice in one stream around three other launches (FP8 streaming and grouped-query splits, a 16-bit split:
  the per-stream tickets are shared by both cache types), and the results must be bit-identical;
* every case also runs with RoPE folded at per-row positions, bit for bit it_b200_rope followed by the unfused launch;
* appended k / v rows made of the quantiser's edges (+-0, ties to even both ways, +-448 s, +-464 s, >= 480 s, +-inf, the
  smallest subnormal and half of it, and T-exact inputs on which a reciprocal multiply would round differently), codes bit
  for bit against kvfp8_oracle.quantise, in both kernels, both T and both widths;
* a failure names the batch row, head, KV head, query group, regime and the CTAs sharing the segment.

The CPU self-checks at the top run without a GPU: a float32 emulation of both kernels' arithmetic passes half the bound, nine
injected slips each fail it, the merge's owner formula inverts the dealing, the case list reaches the dealing states and all
24 FP8 instantiations, and the quantiser edge rows hold every edge class exactly in T.
"""
import re

import numpy as np
import pytest

import oracle
from tests import attn64
from tests import kvfp8_64 as E
from tests import kvfp8_oracle as KV
from tests.attn64 import BF16, F16, Deal

DTYPES = [F16, BF16]
NAMES = {F16: "f16", BF16: "bf16"}


def ch_rows(d):
    return attn64.chunk_rows(BF16, d, kv8=True)


# ====================================================================== the GPU case lists
# name: (D, B, Hq, Hkv, S_max, pos (an int, a per-row list, or a function of the chunk rows CH), regime offset, pos dtype)
STREAM_CASES = {
    "llama7b_step": (128, 16, 32, 32, 1024, 511, 0, np.int64),
    "one_head_p32767": (128, 1, 1, 1, 32768, 32767, 7, np.int64),           # 256 CTAs of one unit
    "one_head_p65535_d64": (64, 1, 1, 1, 65536, 65535, 3, np.int64),        # 256 CTAs of one unit
    "append_only_p3968": (128, 1, 4, 4, 4096, 3968, 1, np.int64),           # 3968 = 31 x 128
    "append_only_p3840_d64": (64, 1, 4, 4, 4096, 3840, 2, np.int64),        # 3840 = 15 x 256
    "units265": (128, 1, 265, 265, 128, 10, 0, np.int64),                   # 265 units: one CTA owns 2
    # 282 units: append-only last chunks alone on a CTA and after a cache chunk on one; int32 positions
    "per_row": (128, 12, 3, 3, 4096, [0, 1, 127, 128, 129, 4095, 2000, 0, 255, 256, 1023, 3072], 5, np.int32),
    "per_row_d64": (64, 12, 3, 3, 8192, [0, 1, 255, 256, 257, 8191, 4000, 0, 511, 512, 2047, 6144], 6, np.int32),
}
for _d in (128, 64):
    _s = "" if _d == 128 else "_d64"
    STREAM_CASES[f"chunk_edge_minus1{_s}"] = (_d, 2, 3, 3, 1024, lambda ch: ch - 1, 2, np.int64)
    STREAM_CASES[f"chunk_edge{_s}"] = (_d, 2, 3, 3, 1024, lambda ch: ch, 3, np.int64)
    STREAM_CASES[f"chunk_edge_plus1{_s}"] = (_d, 2, 3, 3, 1024, lambda ch: ch + 1, 4, np.int64)
    STREAM_CASES[f"pos0{_s}"] = (_d, 3, 5, 5, 256, 0, 0, np.int64)
GQA_SWEEP_G = [2, 4, 8, 16, 17, 24, 32, 33, 40, 64, 80]
GQA_CASES = {
    "llama3_8b_step": (128, 16, 32, 8, 1024, 511, 0, np.int64),
    "mqa_p32767": (128, 1, 8, 1, 32768, 32767, 0, np.int64),
    "mqa_p65535_d64": (64, 1, 8, 1, 65536, 65535, 4, np.int64),
    # 424 units: CTA ranges cross batch rows with different chunk counts
    "per_row": (128, 6, 32, 8, 4096, [0, 128, 4095, 127, 1, 2000], 3, np.int64),
    "per_row_d64": (64, 6, 32, 8, 8192, [0, 256, 8191, 255, 1, 4000], 5, np.int32),
}
for _d in (128, 64):
    _s = "" if _d == 128 else "_d64"
    for _i, _g in enumerate(GQA_SWEEP_G):
        _hkv = 1 + _i % 2
        GQA_CASES[f"G{_g}_Hkv{_hkv}_pCH{_s}"] = (_d, 1, _g * _hkv, _hkv, 1024, lambda ch: ch, _i, np.int64)
        GQA_CASES[f"G{_g}_Hkv{_hkv}_p4095{_s}"] = (_d, 1, _g * _hkv, _hkv, 4096, 4095, _i + 3, np.int64)
ALL_CASES = [("stream", n, c) for n, c in STREAM_CASES.items()] + [("gqa", n, c) for n, c in GQA_CASES.items()]


def positions(spec):
    D, _, _, _, _, pos, _, _ = spec
    return pos(ch_rows(D)) if callable(pos) else pos


def deal_of(spec):
    D, B, Hq, Hkv, S, _, _, _ = spec
    return Deal(BF16, B, Hq, Hkv, S, positions(spec), D, kv8=True)


def kernel_of(spec):
    """(kernel, D, QT) the case runs: QT 0 for the streaming kernel"""
    D, _, Hq, Hkv = spec[:4]
    g = Hq // Hkv
    return ("stream", D, 0) if g == 1 else ("gqa", D, 1 if g <= 16 else 2)


# ====================================================================== CPU: the dealing model and the case list
def test_merge_owner_formula_matches_dealing():
    """cta(u) = ((u + 1) G - 1) / total inverts the forward dealing on every unit of every case, with FP8 chunk rows"""
    for _, name, spec in ALL_CASES:
        d = deal_of(spec)
        u = np.arange(d.total, dtype=np.int64)
        fwd = np.searchsorted(np.asarray(d.u0), u, side="right") - 1
        assert np.array_equal(d.owner(u), fwd), name
        assert all(d.u0[c + 1] > d.u0[c] for c in range(d.ncta)), f"{name}: a CTA without units"


def _reach():
    """the dealing states the case list reaches with FP8 chunk rows (as test_attention_float64 asserts for 16-bit caches)"""
    r = dict(nseg=set(), max_nseg=0, mixed_total=False, append_shared=False, append_alone=False, append_after_cache=False,
             row_cross=False, segs_per_cta=0, qt=set(), nqg2=False, partial_group={})
    for kind, name, spec in ALL_CASES:
        d = deal_of(spec)
        per = [d.u0[c + 1] - d.u0[c] for c in range(d.ncta)]
        r["mixed_total"] |= d.ncta == attn64.GRID_MAX and min(per) == 1 and max(per) == 2
        for b in range(d.B):
            for s in range(d.segs):
                hu0, ctas, chunks = d.segment(b, s)
                r["nseg"].add(min(len(ctas), 3))
                r["max_nseg"] = max(r["max_nseg"], len(ctas))
                if d.pos[b] % d.CH == 0 and d.pos[b] > 0:  # the last chunk holds only the appended row
                    r["append_shared"] |= len(ctas) >= 2
                    r["append_alone"] |= len(ctas) >= 2 and chunks[-1] == [d.nch[b] - 1] and per[ctas[-1]] == 1
                    r["append_after_cache"] |= len(chunks[-1]) >= 2
        for units in d.ctas_units():
            rows = {b for b, _, _ in units}
            r["row_cross"] |= len({int(d.nch[b]) for b in rows}) >= 2
            r["segs_per_cta"] = max(r["segs_per_cta"], len({(b, s) for b, s, _ in units}))
        if kind == "gqa":
            r["qt"].add(d.QT)
            r["nqg2"] |= d.NQG >= 2
            if d.NQG >= 2 and d.grp % d.GP:
                r["partial_group"][d.grp] = True
    return r


def test_case_list_reaches_the_dealing_states():
    r = _reach()
    assert r["nseg"] == {1, 2, 3}, f"whole heads, two-way and >= 3-way splits: {r['nseg']}"
    assert r["max_nseg"] >= 256, f"one head over >= 256 CTAs: {r['max_nseg']}"
    assert r["mixed_total"], "no case with total just above 264 (CTAs owning 2 units and 1)"
    assert r["append_shared"] and r["append_alone"], "an append-only last chunk shared with an earlier CTA / alone on its CTA"
    assert r["append_after_cache"], "an append-only last chunk after a cache chunk of the same head on one CTA"
    assert r["row_cross"], "no CTA range crossing batch rows with different chunk counts"
    assert r["segs_per_cta"] >= 3, "no CTA with >= 3 segments (the 2-stage ring wraps)"
    assert r["qt"] == {1, 2} and r["nqg2"], (r["qt"], r["nqg2"])
    assert {40, 80} <= set(r["partial_group"]), f"partly filled last query group: {sorted(r['partial_group'])}"


def test_case_list_launches_every_instantiation():
    """T x D x {streaming, grouped QT 1, grouped QT 2} x RoPE off / on: every case runs in both T, unfused and folded"""
    kernels = {kernel_of(spec) for _, _, spec in ALL_CASES}
    want = {(k, d, qt) for d in (64, 128) for k, qt in (("stream", 0), ("gqa", 1), ("gqa", 2))}
    assert kernels == want, sorted(want - kernels)
    assert len({(t, k, rope) for t in DTYPES for k in kernels for rope in (False, True)}) == 24


def test_inputs_shape_the_scores():
    """the regimes' scores, computed from the decoded codes, land where they are meant to; NaN codes from row p on"""
    for D, Hq, Hkv in ((128, 9, 9), (64, 18, 2)):
        c = E.Case(2, Hq, Hkv, 1024, D, [700, 300], seed=1)
        g = c.grp
        for b in range(2):
            p = int(c.pos[b])
            assert np.isin(c.kc[b, :, p:], E.NAN_CODES).all() and np.isin(c.vc[b, :, p:], E.NAN_CODES).all()
            assert {0x7F, 0xFF} <= set(np.unique(c.kc[b, :, p:]).tolist())
            assert not np.isin(c.kc[b, :, :p] & 0x7F, [0x7F]).any()
            for h in range(Hq):
                s = c.scores(b, h)
                reg = c.regime[b, h]
                if reg == "neg150":
                    assert s.max() < -125, (D, b, h, s.max())
                elif reg == "pos200":
                    assert abs(s.max() - 200) < 10 and s.min() < E.TENT_FLOOR + 5, (D, b, h, s.max(), s.min())
                elif reg in ("append", "sat"):
                    assert s.argmax() == p and s.max() > 8, (D, b, h, reg, s.argmax(), s.max())
                elif reg == "prev":
                    assert s.argmax() == p - 1, (D, b, h)
                elif reg == "sink":
                    assert s.argmax() == 0, (D, b, h)
                elif reg == "flat":  # (E4M3 rounding of the group's other rows leaks a few units into these scores)
                    assert np.ptp(s) < 8, (D, b, h, np.ptp(s))
            for kv in range(Hkv):  # "sat": the appended rows hold saturated codes (+-448 is code 0x7E / 0xFE)
                if any(c.regime[b, kv * g + r] == "sat" for r in range(g)):
                    ka, va = c.appended()
                    big = np.abs(c.kn[b, kv, 0]) > 448 * c.ksc[kv]
                    assert big.any() and ((ka[b, kv][big] & 0x7F) == 0x7E).all()
                    assert ((va[b, kv] & 0x7F) == 0x7E).any()
        for reg in E.REGIMES:
            assert reg in set(c.regime.ravel()), reg
        # the scales: neighbouring heads' K scales, K against V, differ by >= 2x or by a factor that is not a power of two
        assert np.all(np.abs(np.log2(c.ksc[1:] / c.ksc[:-1])) >= 1)


# ====================================================================== CPU: the bound against an emulation of the kernels
EMU_CASES = {
    # (B, Hq, Hkv, S, D, pos): heads split over 2 - 3 CTAs with 1 - 2 chunks each, append-only last chunks
    "stream": (2, 9, 9, 4096, 128, [4000, 3072]),
    "stream64": (3, 9, 9, 8192, 64, [8000, 4096, 5000]),
    "gqa": (2, 10, 2, 16384, 128, [16000, 9000]),       # G = 5, one tile; 394 units
    "gqa40_64": (1, 40, 1, 40960, 64, 40000),           # G = 40: two tiles, two query groups, the second 8 rows full
}
_emu = {}


def _emu_case(name):
    if name not in _emu:
        B, Hq, Hkv, S, D, pos = EMU_CASES[name]
        c = E.Case(B, Hq, Hkv, S, D, pos, seed=40 + sorted(EMU_CASES).index(name))
        _emu[name] = (c, c.reference())
    return _emu[name]


@pytest.mark.parametrize("dt", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("name", sorted(EMU_CASES))
def test_bound_passes_emulated_kernels_with_margin(name, dt):
    c, refs = _emu_case(name)
    got = E.emulate(c, dt)
    msg = E.report(E.violations(got, refs, dt, c.grp > 1, scale=0.5), got, refs, dt, c.grp > 1, c, c.deal(dt),
                   f"emulated {name} {NAMES[dt]} against half the bound")
    assert msg is None, msg


@pytest.mark.parametrize("mutation,names", [
    ("neighbour_k_scale", ["stream", "gqa"]),
    ("kv_scales_swapped", ["stream", "gqa"]),
    ("v_scale_partials", ["stream", "gqa"]),
    ("scale_by_query_head", ["gqa"]),
    ("unquantised_append", ["stream", "gqa"]),
    ("drop_last_row", ["stream", "gqa"]),
    ("merge_ignore_max", ["stream", "gqa"]),
    ("no_rescale", ["stream", "gqa"]),
    ("round_p_once", ["gqa", "gqa40_64"]),
])
def test_bound_catches_kernel_bugs(mutation, names):
    """bf16: each injected slip (kvfp8_64.MUTATIONS) leaves elements outside the bound on at least one emulated case"""
    seen = []
    for name in names:
        c, refs = _emu_case(name)
        with np.errstate(all="ignore"):
            bad = E.violations(E.emulate(c, BF16, mutation), refs, BF16, c.grp > 1)
        seen.append(int(bad.sum()))
    assert any(seen), f"{mutation} ({E.MUTATIONS[mutation]}) stays inside the bound on {names}"


# ====================================================================== the quantiser's edges
EDGE_POW2 = np.float32(2.0 ** -3)
# not a power of two: fp32(3 / 6.25), so that 3 x 2^k / s lies within an fp32 ulp of the E4M3 midpoint 6.25 x 2^k and the
# correctly rounded division and a multiply by fp32(1 / s) land on different codes for 15 T-exact magnitudes in f16 and bf16
EDGE_S2 = np.float32(3 / 6.25)


def edge_rows(dt, D, rows, s):
    """[rows, D] appended values for a power-of-two scale s (even rows) and a scale that is not one (odd rows, EDGE_S2).  An
    even row k repeats the 15 edge classes and two midpoints (17 values, rotated by k // 2), so that over 17 even rows every
    class falls on every column position mod 16 (a lane's 16 codes, the quantiser's pairs); the midpoints cycle over the rows"""
    classes, mids = E.pow2_edges(s)
    dis = E.disagreeing_inputs(dt, EDGE_S2, n=64)
    out = np.empty((rows, D), np.float32)
    for r in range(rows):
        k = r // 2
        if r % 2 == 0:
            m = mids[(2 * k + np.arange(2)) % mids.size]
            out[r] = np.resize(np.roll(np.concatenate([classes, m]), k), D)
        else:
            out[r] = np.resize(np.roll(dis, 7 * k), D)
    return out


def test_quantiser_edge_rows():
    for dt in DTYPES:
        for D in (64, 128):
            x = edge_rows(dt, D, 48, EDGE_POW2)
            fin = np.isfinite(x)
            assert np.array_equal(oracle.round_to(np.where(fin, x, 0), dt), np.where(fin, x, 0)), "edge values exact in T"
            even = x[0::2] / EDGE_POW2
            for v in (0.0, 448.0, 464.0, 480.0, 2.0 ** 14, np.inf, 2.0 ** -9, 2.0 ** -10):
                for sign in (1, -1):
                    if v == 2.0 ** 14 and sign < 0:
                        continue
                    hit = (even == sign * v) & (np.signbit(even) == (sign < 0))
                    assert {int(c) % 16 for c in np.argwhere(hit)[:, 1]} == set(range(16)), (dt, D, sign * v)
            codes = KV.quantise(x[0::2], EDGE_POW2)
            assert {0x7E, 0xFE, 0x00, 0x80, 0x01, 0x81} <= set(codes.ravel().tolist())
            tie = np.isin(np.abs(even), (KV.DECODE[1:127] + KV.DECODE[0:126]) / 2)
            up = KV.decode(codes)[tie] * np.sign(even[tie]) > np.abs(even[tie])
            assert up.any() and (~up).any(), "ties to even both ways"
            odd = x[1::2]
            assert (KV.quantise(odd, EDGE_S2) != KV.quantise_reciprocal(odd, EDGE_S2)).all(), "inputs the two rules disagree on"


# ====================================================================== GPU plumbing
@pytest.fixture(scope="module")
def K():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from tests import kernel_harness
    return kernel_harness


GUARD = 4096
GUARD_BITS = {"u8": 0xA5, "f32": -7.25, "t": 0x7E5A}
NAN_BITS = 0x7FFF
POS_CODE = {np.int64: 7, np.int32: 6}


class Launch:
    """one FP8 case in one activation type on the device: guarded code caches, scales and out, NaN-filled workspace.
    q / k: the case's (or rotated ones for the unfused half of a RoPE comparison); rope_pos: fold RoPE at these positions."""

    def __init__(self, K, case, dt, pos_dtype=np.int64, q=None, k=None, rope_pos=None):
        import torch
        self.K, self.case, self.dt = K, case, dt
        B, Hq, Hkv, S, D = case.B, case.Hq, case.Hkv, case.S, case.D

        def guarded_u8(x):
            buf = torch.full((x.size + GUARD,), GUARD_BITS["u8"], dtype=torch.uint8, device="cuda")
            buf[:x.size].copy_(torch.from_numpy(np.ascontiguousarray(x).ravel()).cuda())
            return buf

        def guarded_f32(x):
            buf = torch.full((x.size + GUARD,), GUARD_BITS["f32"], dtype=torch.float32, device="cuda")
            buf[:x.size].copy_(torch.from_numpy(np.ascontiguousarray(x, np.float32).ravel()).cuda())
            return buf
        self.kc, self.vc = guarded_u8(case.kc), guarded_u8(case.vc)
        self.ksc, self.vsc = guarded_f32(case.ksc), guarded_f32(case.vsc)
        self.q = K.dev((case.q if q is None else q).reshape(B, Hq, 1, D), dt)
        self.k = K.dev(case.kn if k is None else k, dt)
        self.v = K.dev(case.vn, dt)
        self.out = torch.full((B * Hq * D + GUARD,), GUARD_BITS["t"], dtype=torch.int16, device="cuda")
        self.pos = K.raw(case.pos.astype(pos_dtype))
        self.code = POS_CODE[pos_dtype] | (0x100 if case.per_row else 0)
        self.rope = None if rope_pos is None else K.raw(np.asarray(rope_pos, np.int64))
        self.wsb = int(K.L.lib.it_b200_attention_kvcache_workspace(B, Hq, S, D))
        self.ws = torch.empty(self.wsb // 4 + GUARD, dtype=torch.float32, device="cuda")
        self.deal = case.deal(dt)

    def run(self):
        """fill out / workspace with NaN, launch, return out as float32 [B, Hq, D]"""
        import torch
        K, c = self.K, self.case
        n = c.B * c.Hq * c.D
        self.out[:n].fill_(NAN_BITS)
        self.ws.fill_(float("nan"))
        outv = self.out[:n].view(K.TORCH_DT[self.dt])
        rc = K.L.lib.it_b200_attention_kvcache_fp8(
            self.dt, K.ptr(self.kc), K.ptr(self.vc), K.ptr(self.ksc), K.ptr(self.vsc), K.ptr(self.q), K.ptr(self.k),
            K.ptr(self.v), K.ptr(self.pos), self.code, K.ptr(self.rope), 7, K.ptr(outv), c.B, c.Hq, c.Hkv, c.S, c.D,
            K.ptr(self.ws), self.wsb, K.stream())
        K.L.check(rc)
        K.sync()
        return outv.float().cpu().numpy().reshape(c.B, c.Hq, c.D)

    def caches(self):
        n = self.case.kc.size
        shp = self.case.kc.shape
        return self.kc[:n].cpu().numpy().reshape(shp), self.vc[:n].cpu().numpy().reshape(shp)

    def guard_failures(self, what):
        fails = []
        for name, buf, bits in (("k cache", self.kc, GUARD_BITS["u8"]), ("v cache", self.vc, GUARD_BITS["u8"]),
                                ("k_scale", self.ksc, GUARD_BITS["f32"]), ("v_scale", self.vsc, GUARD_BITS["f32"]),
                                ("out", self.out, GUARD_BITS["t"])):
            if not bool((buf[-GUARD:] == bits).all()):
                fails.append(f"{what}: {name} guard written")
        c = self.case
        for name, buf, want in (("k_scale", self.ksc, c.ksc), ("v_scale", self.vsc, c.vsc)):
            if not np.array_equal(buf[:c.Hkv].cpu().numpy(), want):
                fails.append(f"{what}: {name} changed")
        return fails

    def cache_failures(self, what, want=None):
        """every cache row but p_b byte for byte as before; row p_b = the quantised (rotated) k / v; guards untouched"""
        fails = self.guard_failures(what)
        want = want or self.case.after_append()
        for name, got, w in zip(("k", "v"), self.caches(), want):
            if not np.array_equal(got, w):
                bad = np.argwhere((got != w).any(-1))[:4].tolist()
                fails.append(f"{what}: {name} cache rows differ from the expected codes at (b, kv head, row) {bad}")
        return fails


def rope_dev(K, pos, x, D, dt):
    """it_b200_rope over [B, 1, H * D] with head width D, per-row positions pos [B]"""
    import torch
    B = x.shape[0]
    xd = K.dev(x.reshape(B, 1, -1), dt)
    pd = K.raw(np.asarray(pos, np.int64).reshape(B, 1))
    y = torch.empty_like(xd)
    K.L.check(K.L.lib.it_b200_rope(dt, K.ptr(pd), 7, K.ptr(xd), K.ptr(y), B, 1, xd.shape[-1], D, K.stream()))
    K.sync()
    return K.host(y).reshape(x.shape)


# launched between the two runs of every case on the same stream: an FP8 streaming split, an FP8 grouped-query split and a
# 16-bit split, since the per-stream tickets serve both cache types
INTERPOSERS = [("fp8", (2, 5, 5, 4096, 128, 3000)), ("fp8", (2, 12, 3, 4096, 64, 3000)), ("16", (2, 5, 5, 1024, 700))]
_interposers = {}


def interpose(K, dt):
    """launch the interposers; each must give the bits of its first launch every time"""
    from tests.test_attention_float64 import Launch as Launch16
    fails = []
    for i, (kind, shape) in enumerate(INTERPOSERS):
        key = (i, dt)
        if key not in _interposers:
            if kind == "fp8":
                B, Hq, Hkv, S, D, pos = shape
                ln = Launch(K, E.Case(B, Hq, Hkv, S, D, pos, seed=90 + i), dt)
            else:
                ln = Launch16(K, attn64.Case(*shape, seed=90 + i), dt)
            _interposers[key] = (ln, ln.run())
        ln, first = _interposers[key]
        if not np.array_equal(ln.run().view(np.int32), first.view(np.int32)):
            fails.append(f"interposer {kind} {shape} {NAMES[dt]}: output changed between launches (stale tickets?)")
    return fails


def rope_positions(case):
    return (case.pos * 7 + 3 * np.arange(case.B) + 1) % 100000


def check_rope(K, case, dt, pos_dtype, what):
    """RoPE folded at per-row positions, bit for bit it_b200_rope then the unfused launch (codes and output)"""
    rp = rope_positions(case)
    fused = Launch(K, case, dt, pos_dtype, rope_pos=rp)
    got_f = fused.run()
    qr = rope_dev(K, rp, case.q.reshape(case.B, case.Hq, 1, case.D), case.D, dt).reshape(case.q.shape)
    kr = rope_dev(K, rp, case.kn, case.D, dt)
    unf = Launch(K, case, dt, pos_dtype, q=qr, k=kr)
    got_u = unf.run()
    fails = fused.guard_failures(what + " RoPE folded") + unf.guard_failures(what + " RoPE unfused")
    kf, vf = fused.caches()
    ku, vu = unf.caches()
    if not (np.array_equal(kf, ku) and np.array_equal(vf, vu)):
        fails.append(f"{what}: RoPE folded appends other codes than RoPE + the unfused launch")
    same = got_f.view(np.int32) == got_u.view(np.int32)
    if not same.all():
        b, h, d = np.argwhere(~same)[0]
        fails.append(f"{what}: RoPE folded differs from RoPE + the unfused launch in {int((~same).sum())} elements, first at "
                     f"{fused.deal.where(int(b), int(h))}, column {int(d)}")
    # the rotated append against the host quantiser
    want_k = case.kc.copy()
    kq = KV.quantise(kr[:, :, 0], case.ksc[None, :, None])
    for b in range(case.B):
        want_k[b, :, int(case.pos[b])] = kq[b]
    if not np.array_equal(ku, want_k):
        fails.append(f"{what}: the rotated k row's codes differ from quantise(rope(k))")
    return fails


_cases = {}


def check_case(K, kind, name, spec):
    D, B, Hq, Hkv, S, _, offset, pos_dtype = spec
    key = name
    if key not in _cases:
        _cases.clear()
        case = E.Case(B, Hq, Hkv, S, D, positions(spec), seed=2000 + [n for _, n, _ in ALL_CASES].index(name), offset=offset)
        _cases[key] = (case, case.reference())
    case, refs = _cases[key]
    gqa, fails = kind == "gqa", []
    for dt in DTYPES:
        what = f"{kind} {name} {NAMES[dt]}"
        ln = Launch(K, case, dt, pos_dtype)
        got = ln.run()
        msg = E.report(E.violations(got, refs, dt, gqa), got, refs, dt, gqa, case, ln.deal, what)
        fails += [msg] if msg else []
        fails += ln.cache_failures(what)
        fails += interpose(K, dt)
        again = ln.run()
        if not np.array_equal(again.view(np.int32), got.view(np.int32)):
            fails.append(f"{what}: the second launch differs from the first in {int((again != got).sum())} elements")
        fails += ln.cache_failures(what + " (second launch)")
        del ln
        fails += check_rope(K, case, dt, pos_dtype, what)
    assert not fails, "\n".join(fails)


# ====================================================================== GPU: equal heads (attn_stream_kv8_kernel)
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(STREAM_CASES))
def test_fp8_stream_attention_float64(K, name):
    check_case(K, "stream", name, STREAM_CASES[name])


# ====================================================================== GPU: grouped query heads (attn_gqa_kv8_kernel)
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GQA_CASES))
def test_fp8_gqa_attention_float64(K, name):
    check_case(K, "gqa", name, GQA_CASES[name])


# ====================================================================== GPU: the quantiser's edges in the append
@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("D", [128, 64])
@pytest.mark.parametrize("Hq", [8, 32], ids=["stream", "gqa"])
def test_fp8_append_quantiser_edges(K, Hq, D, dt):
    """appended k and v rows of edge values (edge_rows): power-of-two scales on even KV heads, EDGE_S2 (not a power of two) on
    odd ones; the codes bit for bit kvfp8_oracle.quantise, the output inside the bound"""
    B, Hkv, S = 6, 8, 512
    case = E.Case(B, Hq, Hkv, S, D, [200, 127, 128, 300, 0, 511], seed=77)
    case.ksc[0::2] = EDGE_POW2
    case.vsc[0::2] = EDGE_POW2 * 2
    case.ksc[1::2] = case.vsc[1::2] = EDGE_S2
    rows = edge_rows(dt, D, 2 * B * Hkv, EDGE_POW2)
    # row r of the layout: even ones carry the power-of-two classes, odd ones the disagreeing inputs; head kv takes its parity
    for b in range(B):
        for kv in range(Hkv):
            i = 2 * (b * (Hkv // 2) + kv // 2) + kv % 2
            case.kn[b, kv, 0] = rows[i]
            case.vn[b, kv, 0] = rows[(i + 2) % rows.shape[0]] * (2 if kv % 2 == 0 else 1)
    refs = case.reference()
    ln = Launch(K, case, dt)
    got = ln.run()
    fails = ln.cache_failures(f"edges Hq {Hq} D {D} {NAMES[dt]}")
    msg = E.report(E.violations(got, refs, dt, Hq > Hkv), got, refs, dt, Hq > Hkv, case, ln.deal,
                   f"edges Hq {Hq} D {D} {NAMES[dt]}")
    fails += [msg] if msg else []
    assert not fails, "\n".join(fails)


# ====================================================================== GPU: the intended instantiations ran
def profiled_kernel_names():
    """kernel names recorded by torch.profiler (CUDA activity only) for one small launch per FP8 instantiation"""
    import torch
    from tests import kernel_harness as K
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for dt in DTYPES:
            for D in (128, 64):
                for B, Hq, Hkv in ((2, 3, 3), (2, 8, 2), (1, 24, 1)):  # equal heads; G = 4 (one tile); G = 24 (two tiles)
                    c = E.Case(B, Hq, Hkv, 512, D, 300, seed=7)
                    Launch(K, c, dt).run()
                    Launch(K, c, dt, rope_pos=rope_positions(c)).run()
        torch.cuda.synchronize()
    return sorted({e.name for e in prof.events() if "CUDA" in str(e.device_type)})


@pytest.mark.gpu
def test_fp8_attention_cases_reach_the_intended_kernels():
    """The profiler runs in a child process, as the other profiler checks do: a profiler session in the test process loses
    kernel records of a later one in a full-suite run."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = "import json; from tests.test_kvfp8_float64 import profiled_kernel_names as f; print(json.dumps(f()))"
    r = subprocess.run([sys.executable, "-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    names = set(json.loads(r.stdout.strip().splitlines()[-1]))
    if not names:
        pytest.skip("the profiler recorded no CUDA kernel events (CUPTI activity tracing unavailable)")
    want = []
    for t in ("__half", "__nv_bfloat16"):
        for d in (128, 64):
            for rope in ("false", "true"):
                want += [rf"attn_stream_kv8_kernel<{t}, {d}, 8, 4, {rope}>", rf"attn_gqa_kv8_kernel<{t}, {d}, 1, {rope}>",
                         rf"attn_gqa_kv8_kernel<{t}, {d}, 2, {rope}>"]
    missing = [p for p in want if not any(re.search(p, nm) for nm in names)]
    assert len(want) == 24 and not missing, f"not launched: {missing}; kernels seen: {sorted(n for n in names if 'kv8' in n)}"
