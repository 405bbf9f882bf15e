"""The decode attention kernels (attention.cu) against float64 at large score ranges, across every CTA split and merge.

attn_stream_kernel (query heads = KV heads; the Llama-7B step) and attn_gqa_kernel (grouped-query layers; the Llama-3-8B step)
run a stable online softmax that rescales by the running maximum per chunk, across the two sub-rows of a warp, across the
8 consumer warps and across the CTAs of a head dealt to several of them.  The oracle computes exp(dot / sqrt(128)) without
max subtraction, so tests against it keep scores within about 2 of each other.  Here (helpers in tests/attn64.py):

* every case cycles eight score regimes over (batch row, query head): flat, graded peaks a few units apart with the maximum
  arriving late or early, a sink at row 0, a peak at row pos - 1, a peak on the appended row, every score near -150
  (underflow without max subtraction) and a tent of scores up to +200 (overflow without it);
* V rows are scaled by 2^((j mod 5) - 2) and KV heads by 2^((h mod 3) - 1), so a row or head mix-up changes values by >= 2x;
* every cache row from pos on is NaN before the launch (row pos is overwritten by the append), and so are `out` and the
  whole attention workspace; guard regions after `out` and after each cache must stay untouched; the caches are compared bit
  for bit through an integer view;
* every case runs twice in one stream with two other shapes in between, and the results must be bit-identical (the
  per-head tickets clean themselves up);
* the output is held to the per-element bound of tests/attn64.py; a failure names the batch row, head, KV head and query
  group, and the CTAs sharing the segment.

The CPU self-checks at the top run without a GPU: a float32 emulation of both kernels' arithmetic passes half the bound, seven
injected kernel bugs each fail it, the merge's owner formula agrees with the forward dealing on every unit of every case, and
the case list reaches the dealing states it is meant to reach.
"""
import re

import numpy as np
import pytest

from tests import attn64, ref64
from tests.attn64 import BF16, F16, F32, Case, Deal

DTYPES = [F32, F16, BF16]


# ====================================================================== the GPU case lists
# name: (B, Hq, Hkv, S_max, pos (an int, a per-row list, or a function of the chunk rows CH), regime offset, pos dtype)
STREAM_CASES = {
    "llama7b_step": (16, 32, 32, 1024, 511, 0, np.int64),
    "one_head_p16383": (1, 1, 1, 16384, 16383, 7, np.int64),           # bf16 / f16: 256 CTAs of one unit; fp32: 264
    "append_only_p4032": (1, 4, 4, 4096, 4032, 1, np.int64),           # 4032 % 64 = 4032 % 32 = 0
    "chunk_edge_minus1": (2, 3, 3, 256, lambda ch: ch - 1, 2, np.int64),
    "chunk_edge": (2, 3, 3, 256, lambda ch: ch, 3, np.int64),
    "chunk_edge_plus1": (2, 3, 3, 256, lambda ch: ch + 1, 4, np.int64),
    "pos0": (3, 5, 5, 64, 0, 0, np.int64),
    "units265": (1, 265, 265, 64, 10, 0, np.int64),                    # 265 units: some CTAs own 2, most 1
    # 282 units (f16 / bf16): append-only last chunks alone on a CTA and after a cache chunk on one; int32 positions
    "per_row": (12, 3, 3, 2048, [0, 1, 63, 64, 65, 2047, 1000, 0, 127, 128, 511, 1536], 5, np.int32),
}
GQA_SWEEP_G = [2, 4, 8, 16, 17, 24, 32, 33, 40, 64, 80]
GQA_CASES = {
    "llama3_8b_step": (16, 32, 8, 1024, 511, 0, np.int64),
    "mqa_p16383": (1, 8, 1, 16384, 16383, 0, np.int64),
    # 404 units (f16 / bf16): CTA ranges cross batch rows with different chunk counts
    "per_row": (6, 32, 4, 4096, [0, 64, 4095, 63, 1, 2000], 3, np.int64),
}
for _i, _g in enumerate(GQA_SWEEP_G):
    _hkv = 1 + _i % 2
    GQA_CASES[f"G{_g}_Hkv{_hkv}_p64"] = (1, _g * _hkv, _hkv, 128, 64, _i, np.int64)
    GQA_CASES[f"G{_g}_Hkv{_hkv}_p4095"] = (1, _g * _hkv, _hkv, 4096, 4095, _i + 3, np.int64)
ALL_CASES = [("stream", n, c) for n, c in STREAM_CASES.items()] + [("gqa", n, c) for n, c in GQA_CASES.items()]


def positions(spec, dt):
    B, _, _, _, pos, _, _ = spec
    return pos(attn64.chunk_rows(dt)) if callable(pos) else pos


def deal_of(spec, dt):
    B, Hq, Hkv, S, _, _, _ = spec
    return Deal(dt, B, Hq, Hkv, S, positions(spec, dt))


# ====================================================================== CPU: the dealing model and the case list
def test_merge_owner_formula_matches_dealing():
    """cta(u) = ((u + 1) G - 1) / total, which the merge uses to find the CTAs sharing a head, inverts the forward dealing
    [c total / G, (c + 1) total / G) on every unit of every case"""
    for _, name, spec in ALL_CASES:
        for dt in DTYPES:
            d = deal_of(spec, dt)
            u = np.arange(d.total, dtype=np.int64)
            fwd = np.searchsorted(np.asarray(d.u0), u, side="right") - 1
            assert np.array_equal(d.owner(u), fwd), f"{name} {attn64.NAMES[dt]}"
            assert all(d.u0[c + 1] > d.u0[c] for c in range(d.ncta)), f"{name}: a CTA without units"


def _reach(dt):
    """the dealing states the case list reaches in one dtype"""
    r = dict(nseg=set(), max_nseg=0, mixed_total=False, append_shared=False, append_alone=False, append_after_cache=False,
             row_cross=False, segs_per_cta=0, qt=set(), nqg2=False, partial_group={})
    for kind, name, spec in ALL_CASES:
        d = deal_of(spec, dt)
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


@pytest.mark.parametrize("dt", DTYPES, ids=["fp32", "f16", "bf16"])
def test_case_list_reaches_the_dealing_states(dt):
    r = _reach(dt)
    assert r["nseg"] == {1, 2, 3}, f"whole heads, two-way and >= 3-way splits: {r['nseg']}"
    assert r["max_nseg"] >= 256, f"one head over >= 256 CTAs: {r['max_nseg']}"
    assert r["mixed_total"], "no case with total just above 264 (CTAs owning 2 units and 1)"
    assert r["append_shared"] and r["append_alone"], "an append-only last chunk shared with an earlier CTA / alone on its CTA"
    assert r["append_after_cache"], "an append-only last chunk after a cache chunk of the same head on one CTA"
    assert r["row_cross"], "no CTA range crossing batch rows with different chunk counts"
    assert r["segs_per_cta"] >= 3, "no CTA with >= 3 segments (the 2-stage ring wraps)"
    assert r["qt"] == {1, 2} and r["nqg2"], (r["qt"], r["nqg2"])
    assert {40, 80} <= set(r["partial_group"]), f"partly filled last query group: {sorted(r['partial_group'])}"


def test_ulp_f32_known_values():
    assert ref64.ulp(np.array([1.0, 1.5, 2.0, -3.0, 0.0]), F32).tolist() == [2.0 ** -23, 2.0 ** -23, 2.0 ** -22, 2.0 ** -22,
                                                                             2.0 ** -149]


def test_inputs_shape_the_scores():
    """the regimes' scores, computed from the rounded data, land where they are meant to; the poison starts at row pos"""
    c = Case(2, 8, 2, 256, [200, 97], seed=1)
    kc, vc, kn, _ = c.caches()
    for b in range(2):
        p = int(c.pos[b])
        assert np.isnan(kc[b, :, p:]).all() and np.isnan(vc[b, :, p:]).all() and not np.isnan(kc[b, :, :p]).any()
        assert np.array_equal(kn[b, :, 0], c.kseq[b, :, p])
        for h in range(8):
            s = c.q[b, h].astype(np.float64) @ c.kseq[b, h // 4, :p + 1].T.astype(np.float64) / np.sqrt(128)
            reg = c.regime[b, h]
            if reg == "neg150":
                assert s.max() < -130, s.max()
            elif reg == "pos200":
                assert abs(s.max() - 200) < 3 and s.min() < 200 - 60, (s.max(), s.min())
            elif reg == "append":
                assert s.argmax() == p and s.max() > 17
            elif reg == "prev":
                assert s.argmax() == p - 1
            elif reg == "sink":
                assert s.argmax() == 0
            elif reg == "flat":
                assert np.ptp(s) < 4
    for reg in attn64.REGIMES:
        assert reg in set(c.regime.ravel())


# ====================================================================== CPU: the bound against an emulation of the kernels
EMU_CASES = {
    "stream": (4, 7, 7, 1024, [1000, 1000, 640, 64]),  # 315 bf16 units over 264 CTAs, append-only last chunks, split heads
    "gqa": (2, 10, 2, 1024, [1000, 320]),               # G = 5 (one tile), heads split over 16 / 6 CTAs
    "gqa40": (1, 40, 1, 1024, 700),                     # G = 40: two tiles, two query groups, the second 8 rows full
}
_emu = {}


def _emu_case(name):
    if name not in _emu:
        B, Hq, Hkv, S, pos = EMU_CASES[name]
        c = Case(B, Hq, Hkv, S, pos, seed=40 + sorted(EMU_CASES).index(name))
        _emu[name] = (c, c.reference())
    return _emu[name]


@pytest.mark.parametrize("dt", DTYPES, ids=["fp32", "f16", "bf16"])
@pytest.mark.parametrize("name", sorted(EMU_CASES))
def test_bound_passes_emulated_kernels_with_margin(name, dt):
    c, refs = _emu_case(name)
    got = attn64.emulate(c, dt)
    deal = Deal(dt, c.B, c.Hq, c.Hkv, c.S, c.pos)
    msg = attn64.report(attn64.violations(got, refs, dt, c.grp > 1, scale=0.5), got, refs, dt, c.grp > 1, deal,
                        f"emulated {name} {attn64.NAMES[dt]} against half the bound")
    assert msg is None, msg


@pytest.mark.parametrize("mutation,names", [
    ("round_p_once", ["gqa", "gqa40"]),                 # P rounded once to T before P.V
    ("no_rescale", ["stream", "gqa"]),                  # a later chunk raises the running max, l / acc not rescaled
    ("merge_ignore_max", ["stream", "gqa"]),            # the CTA merge adds partials without their maxima
    ("merge_slot0_max", ["stream", "gqa"]),             # ... rescales to slot 0's maximum
    ("drop_last_row", ["stream", "gqa"]),               # the last valid cache row of the last chunk dropped
    ("append_twice", ["stream", "gqa"]),                # the appended row added twice
    ("kv_mod", ["gqa"]),                                # query head i reads KV head i mod Hkv instead of i / G
    ("merge_skip_last", ["stream", "gqa"]),             # the merge skips the last partial
])
def test_bound_catches_kernel_bugs(mutation, names):
    """bf16, the coarser type: each injected bug leaves elements outside the bound on at least one emulated case"""
    seen = []
    for name in names:
        c, refs = _emu_case(name)
        with np.errstate(all="ignore"):
            bad = attn64.violations(attn64.emulate(c, BF16, mutation), refs, BF16, c.grp > 1)
        seen.append(int(bad.sum()))
    assert any(seen), f"{mutation} stays inside the bound on {names}"


# ====================================================================== GPU plumbing
@pytest.fixture(scope="module")
def K():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from tests import kernel_harness
    return kernel_harness


GUARD = 4096                                   # elements after each buffer
GUARD_BITS = {F32: 0x7FC0BEEF, F16: 0x7E5A, BF16: 0x7E5A}
NAN_BITS = {F32: 0x7FFFFFFF, F16: 0x7FFF, BF16: 0x7FFF}
POS_CODE = {np.int64: 7, np.int32: 6}


def _int(dt):
    import torch
    return torch.int32 if dt == F32 else torch.int16


def guarded(K, x, dt):
    """(buffer, view): x (float32 numpy, NaN allowed) stored as T in the head of a buffer whose tail is a guard pattern"""
    import torch
    buf = torch.full((x.size + GUARD,), GUARD_BITS[dt], dtype=_int(dt), device="cuda")
    view = buf[:x.size].view(K.TORCH_DT[dt]).view(x.shape)
    view.copy_(torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda())
    return buf, view


class Launch:
    """one case in one dtype on the device: guarded caches / out, NaN-filled workspace"""

    def __init__(self, K, case, dt, pos_dtype=np.int64):
        import torch
        self.K, self.case, self.dt = K, case, dt
        kc, vc, kn, vn = case.caches()
        self.kc, self.vc = guarded(K, kc, dt), guarded(K, vc, dt)
        self.q = K.dev(case.q.reshape(case.B, case.Hq, 1, 128), dt)
        self.k, self.v = K.dev(kn, dt), K.dev(vn, dt)
        self.out = guarded(K, np.zeros((case.B, case.Hq, 1, 128), np.float32), dt)
        self.pos = K.raw(case.pos.astype(pos_dtype))
        self.code = POS_CODE[pos_dtype] | (0x100 if case.per_row else 0)
        self.wsb = int(K.L.lib.it_b200_attention_kvcache_workspace(case.B, case.Hq, case.S, 128))
        self.ws = torch.empty(self.wsb // 4, dtype=torch.float32, device="cuda")
        self.before = [t[0][:-GUARD].clone() for t in (self.kc, self.vc)]
        self.deal = Deal(dt, case.B, case.Hq, case.Hkv, case.S, case.pos)

    def run(self):
        """fill out / workspace with NaN, launch, return out as float32 [B, Hq, 128]"""
        K, c = self.K, self.case
        self.out[0][:-GUARD].fill_(NAN_BITS[self.dt])
        self.ws.fill_(float("nan"))
        kcp, vcp, outp = K.ptr(self.kc[1]), K.ptr(self.vc[1]), K.ptr(self.out[1])
        if c.Hq == c.Hkv:
            rc = K.L.lib.it_b200_attention_kvcache(self.dt, kcp, vcp, K.ptr(self.q), K.ptr(self.k), K.ptr(self.v), K.ptr(self.pos),
                                                   self.code, outp, c.B, c.Hq, c.S, 128, K.ptr(self.ws), self.wsb, K.stream())
        else:
            rc = K.L.lib.it_b200_attention_kvcache_gqa(self.dt, kcp, vcp, K.ptr(self.q), K.ptr(self.k), K.ptr(self.v),
                                                       K.ptr(self.pos), self.code, None, 0, outp, c.B, c.Hq, c.Hkv, c.S, 128,
                                                       K.ptr(self.ws), self.wsb, K.stream())
        K.L.check(rc)
        K.sync()
        return self.out[1].float().cpu().numpy().reshape(c.B, c.Hq, 128)

    def cache_failures(self, what):
        """guards untouched; every cache row but pos_b bit for bit as before; row pos_b = the appended k / v bits"""
        fails = []
        for name, (buf, _), before, new in (("k", self.kc, self.before[0], self.k), ("v", self.vc, self.before[1], self.v)):
            n = buf.numel() - GUARD
            if not bool((buf[n:] == GUARD_BITS[self.dt]).all()):
                fails.append(f"{what}: {name} cache guard written")
            want = before.view(self.case.B, self.case.Hkv, self.case.S, 128).clone()
            nb = new.view(_int(self.dt)).view(self.case.B, self.case.Hkv, 128)
            for b in range(self.case.B):
                want[b, :, int(self.case.pos[b])] = nb[b]
            got = buf[:n].view(want.shape)
            if not bool((got == want).all()):
                bad = (got != want).any(-1).nonzero()[:4].tolist()
                fails.append(f"{what}: {name} cache rows differ from the expected bits at (b, kv head, row) {bad}")
        if not bool((self.out[0][-GUARD:] == GUARD_BITS[self.dt]).all()):
            fails.append(f"{what}: out guard written")
        return fails


# two shapes launched between the two runs of every case: split heads in both kernels, on the same stream's tickets
INTERPOSERS = [(2, 5, 5, 1024, 700), (2, 12, 3, 1024, 700)]
_interposers = {}


def interpose(K, dt):
    """launch both interposer shapes; each must give the bits of its first launch every time"""
    fails = []
    for i, (B, Hq, Hkv, S, pos) in enumerate(INTERPOSERS):
        key = (i, dt)
        if key not in _interposers:
            ln = Launch(K, Case(B, Hq, Hkv, S, pos, seed=90 + i), dt)
            _interposers[key] = (ln, ln.run())
        ln, first = _interposers[key]
        again = ln.run()
        if not np.array_equal(again.view(np.int32), first.view(np.int32)):
            fails.append(f"interposer {INTERPOSERS[i]} {attn64.NAMES[dt]}: output changed between launches (stale tickets?)")
    return fails


def check_case(K, kind, name, spec):
    B, Hq, Hkv, S, _, offset, pos_dtype = spec
    refs_by_pos, fails = {}, []
    for dt in DTYPES:
        pos = positions(spec, dt)
        key = str(pos)
        if key not in refs_by_pos:
            case = Case(B, Hq, Hkv, S, pos, seed=1000 + [n for _, n, _ in ALL_CASES].index(name), offset=offset)
            refs_by_pos[key] = (case, case.reference())
        case, refs = refs_by_pos[key]
        ln = Launch(K, case, dt, pos_dtype)
        what = f"{kind} {name} {attn64.NAMES[dt]}"
        got = ln.run()
        msg = attn64.report(attn64.violations(got, refs, dt, kind == "gqa"), got, refs, dt, kind == "gqa", ln.deal, what)
        fails += [msg] if msg else []
        fails += ln.cache_failures(what)
        fails += interpose(K, dt)
        again = ln.run()
        if not np.array_equal(again.view(np.int32), got.view(np.int32)):
            fails.append(f"{what}: the second launch differs from the first in {int((again != got).sum())} elements")
        fails += ln.cache_failures(what + " (second launch)")
        del ln
    assert not fails, "\n".join(fails)


# ====================================================================== GPU: equal heads (attn_stream_kernel)
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(STREAM_CASES))
def test_stream_attention_float64(K, name):
    check_case(K, "stream", name, STREAM_CASES[name])


# ====================================================================== GPU: grouped query heads (attn_gqa_kernel)
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GQA_CASES))
def test_gqa_attention_float64(K, name):
    check_case(K, "gqa", name, GQA_CASES[name])


# ====================================================================== GPU: the intended instantiations ran
def profiled_kernel_names():
    """kernel names recorded by torch.profiler (CUDA activity only) for one small launch per kernel, tile count and dtype"""
    import torch
    from tests import kernel_harness as K
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for dt in DTYPES:
            for B, Hq, Hkv in ((2, 3, 3), (2, 8, 2), (1, 24, 1)):  # equal heads; G = 4 (one tile); G = 24 (two tiles)
                Launch(K, Case(B, Hq, Hkv, 128, 70, seed=7), dt).run()
        torch.cuda.synchronize()
    return sorted({e.name for e in prof.events() if "CUDA" in str(e.device_type)})


@pytest.mark.gpu
def test_attention_cases_reach_the_intended_kernels():
    """The profiler runs in a child process: with this session in the test process, a later profiler check
    (test_decode_edges.py) lost the records of its first kernels in a full-suite run."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = "import json; from tests.test_attention_float64 import profiled_kernel_names as f; print(json.dumps(f()))"
    r = subprocess.run([sys.executable, "-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    names = set(json.loads(r.stdout.strip().splitlines()[-1]))
    if not names:
        pytest.skip("the profiler recorded no CUDA kernel events (CUPTI activity tracing unavailable)")
    want = []
    for t in ("float", "__half", "__nv_bfloat16"):
        want += [rf"attn_stream_kernel<{t}, 8, 4, false>", rf"attn_gqa_kernel<{t}, 1, false>", rf"attn_gqa_kernel<{t}, 2, false>"]
    missing = [p for p in want if not any(re.search(p, nm) for nm in names)]
    assert not missing, f"not launched: {missing}; kernels seen: {sorted(n for n in names if 'attn' in n)}"
