"""The persistent decode kernel (`decode_stack_kernel`, decode_stack.cu) against float64, phase by phase, with per-row
positions and every split (helpers in tests/stack64.py).

Each launch writes every layer's q, k, v, attn_out, x_mid, gate, up and x_out and appends one row to each cache, so every
phase of every layer is checked in float64 from the GPU's own inputs to that phase:

* RMSNorm -> q / k / v and RMSNorm -> gate / up: first layer from x_raw, later ones through the ss hand-over, K > 4096 with the
  norm weight read from global memory; o-proj + residual; Silu.Mul -> down + residual: stack64's per-element bounds;
* RoPE + attention: the appended k row must equal it_b200_rope of the stack's k bit for bit and the v row the stack's v, every
  other cache row is untouched, and the output is held to attn64's bound on q rotated by it_b200_rope.  Layer 0 is launched
  twice: the second time its cache rows below the position are rebuilt along the rotated q of the first launch so the eight
  score regimes of attn64 cycle over (row, head); its q / k / v must not change between the two launches;
* before each launch every output buffer, the whole workspace and every cache row from the position on are NaN; guard regions
  after each output and cache must stay untouched; x_in must be unchanged;
* each case is launched once more after a decode GEMM chain with another phase count (which moves the shared grid-barrier
  generation) and must give the same bits.

The chain shapes of test_gpu_decode_stack.py run under the same bounds, and so do the unfused rmsnorm_kernel and
silu_mul_kernel that the stack replaces.  The CPU self-checks at the top need no GPU: a float32 emulation of the GEMM phases
stays within half the bound, six injected bugs each fail it, the attention merge under the stack's dealing passes and a
skipped partial fails, the merge's owner formula inverts the dealing, and the case list reaches the dealing states it is meant
to reach.
"""
import ctypes
import re
import time

import numpy as np
import pytest

from tests import attn64, ref64, stack64
from tests.ref64 import BF16, F16, F32
from tests.stack64 import GemmDeal, Operand, StackDeal

NAMES = {F32: "fp32", F16: "f16", BF16: "bf16"}
I32, I64 = 6, 7
PER_ROW, IN_STEP = 0x100, 0x200
# ambiguous share of a transformed operand: the first layer's x_raw reduction at K = 4096 is a chain of 133 roundings, a window
# of 141 2^-24 against f16's spacing of 2^-10 .. 2^-11 relative: about 2.4 % of the elements straddle a rounding point
MAX_AMB_SHARE = 0.05

# ====================================================================== the stack cases
# name: dict(B, d, H, ffn, S, pos (int or per-row list), layers, dts, pos_dt, rope: None (= the cache positions) or a list)
PER_ROW_POS = [0, 1, 63, 64, 65, 127, 128, 255, 200, 17, 192, 3, 100, 254, 129, 5]
STACK_CASES = {
    "bench_B16_d4096": dict(B=16, d=4096, H=32, ffn=11008, S=1024, pos=511, layers=2),
    "d5120_global_normw": dict(B=5, d=5120, H=40, ffn=13824, S=256, pos=130, layers=1, dts=[BF16]),
    "tp4_shard_dl1024": dict(B=15, d=4096, H=8, ffn=2752, S=512, pos=320, layers=1),
    "ragged_B7": dict(B=7, d=1024, H=8, ffn=1416, S=1000, pos=999, layers=2),
    "tiny_p0": dict(B=1, d=128, H=1, ffn=136, S=64, pos=0, layers=1),
    "tiny_p63": dict(B=1, d=128, H=1, ffn=136, S=64, pos=63, layers=1),
    "per_row_i64": dict(B=16, d=1024, H=8, ffn=2816, S=256, pos=PER_ROW_POS, layers=1),
    "per_row_i32": dict(B=16, d=1024, H=8, ffn=2816, S=256, pos=PER_ROW_POS, layers=1, pos_dt=I32),
    "per_row_rope_in_step": dict(B=16, d=1024, H=8, ffn=2816, S=256, pos=PER_ROW_POS, layers=1, pos_dt=I32,
                                 rope=[65535, 0, 1, 4095, 30000, 7, 64, 65534, 1000, 2, 12345, 255, 60000, 31, 4096, 9]),
    "four_layers": dict(B=4, d=256, H=2, ffn=704, S=128, pos=100, layers=4),
}
DEFAULTS = dict(dts=[F16, BF16], pos_dt=I64, rope=None)


def spec(name):
    return {**DEFAULTS, **STACK_CASES[name]}


def case_pos(c):
    return np.clip(np.broadcast_to(np.asarray(c["pos"], np.int64), (c["B"],)), 0, c["S"] - 1)


def gemm_phases(c, nctas=stack64.NUM_SMS):
    """the five GEMM-phase shapes of a layer: name -> GemmDeal"""
    d, dl, f = c["d"], c["H"] * 128, c["ffn"]
    return {"qkv": GemmDeal(3, dl, d, nctas), "o": GemmDeal(1, d, dl, nctas), "gate_up": GemmDeal(2, f, d, nctas),
            "down": GemmDeal(1, d, f, nctas)}


# ====================================================================== CPU: dealing model and coverage
def test_pick_split_matches_the_library():
    """stack64.pick_split against the library's own itb::ds_pick_split (a host function, no GPU needed) on every case's
    phases and a sweep of shapes, at 132 and at 114 SMs"""
    from infinitensor_b200 import _lib as L
    fn = L.lib._ZN3itb13ds_pick_splitEiii
    fn.restype, fn.argtypes = ctypes.c_int, [ctypes.c_int] * 3
    shapes = {(g.ntiles, g.kchunks) for n in STACK_CASES for g in gemm_phases(spec(n)).values()}
    shapes |= {(t, k) for t in (1, 2, 3, 7, 32, 86, 96, 131, 132, 133, 264) for k in (1, 2, 3, 16, 17, 64, 80, 172, 216)}
    for nctas in (132, 114):
        bad = [(t, k) for t, k in sorted(shapes) if stack64.pick_split(t, k, nctas) != fn(t, k, nctas)]
        assert not bad, f"{nctas} SMs: {bad[:8]}"
    got = {k: v.S for k, v in gemm_phases(spec("bench_B16_d4096")).items()}
    assert got == {"qkv": 4, "o": 4, "gate_up": 13, "down": 4}, got


def test_owner_formula_inverts_the_stack_dealing():
    for name in STACK_CASES:
        c = spec(name)
        d = StackDeal(c["B"], c["H"], c["S"], case_pos(c))
        u = np.arange(d.total, dtype=np.int64)
        fwd = np.searchsorted(np.asarray(d.u0), u, side="right") - 1
        assert np.array_equal(d.owner(u), fwd), name
        assert all(d.u0[i + 1] > d.u0[i] for i in range(d.ncta)), f"{name}: a CTA without units"


def reach(nctas=stack64.NUM_SMS):
    r = dict(res_S1=set(), res_S2=set(), waves2=False, few_units=False, nseg=set(), row_cross=False, append_only=False)
    for name in STACK_CASES:
        c = spec(name)
        for ph, g in gemm_phases(c, nctas).items():
            if ph in ("o", "down"):
                (r["res_S1"] if g.S == 1 else r["res_S2"]).add(ph)
            r["waves2"] |= g.waves(0) >= 2
            r["few_units"] |= g.nunits < nctas
        d = StackDeal(c["B"], c["H"], c["S"], case_pos(c), nctas)
        for b in range(d.B):
            for s in range(d.segs):
                _, ctas, _ = d.segment(b, s)
                r["nseg"].add(min(len(ctas), 3))
                r["append_only"] |= d.pos[b] > 0 and d.pos[b] % 64 == 0
        for units in d.ctas_units():
            rows = {b for b, _, _ in units}
            r["row_cross"] |= len({int(d.pos[b]) for b in rows}) >= 2
    return r


def test_case_list_reaches_the_dealing_states():
    r = reach()
    assert r["res_S1"] == {"o", "down"} and r["res_S2"] == {"o", "down"}, \
        f"both residual phases unsplit and split (ss_out written by a ticket finisher): {r['res_S1']}, {r['res_S2']}"
    assert r["waves2"] and r["few_units"], "a CTA with >= 2 units in a phase, and a phase with fewer units than SMs"
    assert r["nseg"] == {1, 2, 3}, f"heads on 1, 2 and >= 3 CTAs: {r['nseg']}"
    assert r["row_cross"], "a CTA range crossing batch rows with different positions"
    assert r["append_only"], "an append-only last chunk"


# ====================================================================== CPU: the bound against an emulation of the kernel
def _emu_layer(dt, m, d, f, seed):
    """(inputs, emulated outputs) of one layer's GEMM phases at a small width: rmsnorm (x_raw) -> qkv (grouped), o-proj +
    residual (ss out) -> rmsnorm (ss) -> gate / up -> silu.mul -> down + residual"""
    x = stack64.rows(m, d, dt, seed)
    n1, n2 = stack64.norm_weight(d, dt, seed + 1), stack64.norm_weight(d, dt, seed + 2)
    W = {k: stack64.weights(kk, nn, dt, seed + 3 + i, s, "cpu")
         for i, (k, kk, nn, s) in enumerate([("qkv", d, 3 * 256, 1.0 / np.sqrt(d)), ("o", 256, d, 0.5 / np.sqrt(256)),
                                             ("gu", d, 2 * f, 1.0 / np.sqrt(d)), ("down", f, d, 0.5 / np.sqrt(f))])}
    attn = stack64.rows(m, 256, dt, seed + 9, 0.5)
    return dict(x=x, n1=n1, n2=n2, W={k: v.float().numpy() for k, v in W.items()}, Wt=W, attn=attn)


def emulate_layer(inp, dt, mutation=None):
    x, W = inp["x"], inp["W"]
    e = stack64
    rinv = e.emu_rinv_x_raw(x.astype(np.float32))
    xn = e.emu_rmsnorm(x.astype(np.float32), inp["n1"], rinv, dt, mutation)
    qkv = e.emu_gemm(xn, W["qkv"], 3, dt, mutation=mutation)
    xm = e.emu_gemm(inp["attn"].astype(np.float32), W["o"], 1, dt, epi=1, res=x, mutation=mutation)
    ss = e.emu_ss(xm)
    r2 = e.emu_rinv_ss(e.emu_ss(x.astype(np.float32)) if mutation == "rinv_pre_residual" else ss, x.shape[1], mutation)
    hn = e.emu_rmsnorm(xm, inp["n2"], r2, dt, mutation)
    f = W["gu"].shape[1] // 2
    gu = e.emu_gemm(hn, W["gu"], 2, dt, mutation=mutation)
    mm = e.emu_silu_mul(gu[:, :f], gu[:, f:], dt)
    xo = e.emu_gemm(mm, W["down"], 1, dt, epi=1, res=xm, mutation=mutation)
    return dict(qkv=qkv, x_mid=xm, gu=gu, x_out=xo)


def layer_refs(inp, out, dt):
    """phase references from the emulated layer's own inputs to each phase"""
    e, Wt, d = stack64, inp["Wt"], inp["x"].shape[1]
    f = inp["W"]["gu"].shape[1] // 2
    op1 = e.rmsnorm_operand(inp["x"], inp["n1"], dt, e.chain_length("x_raw", d))
    op4 = e.rmsnorm_operand(out["x_mid"], inp["n2"], dt, e.chain_length("ss", d, nt=-(-d // 128)))
    op5 = e.silu_mul_operand(out["gu"][:, :f], out["gu"][:, f:], dt)
    return dict(qkv=e.store_ref(op1, Wt["qkv"], dt), x_mid=e.residual_ref(Operand(inp["attn"]), Wt["o"], inp["x"], dt),
                gu=e.store_ref(op4, Wt["gu"], dt), x_out=e.residual_ref(op5, Wt["down"], out["x_mid"], dt))


EMU_SHAPES = {"d1024": (5, 1024, 704), "d4160": (3, 4160, 200)}  # rows, d_model, ffn (K > 4096: the global norm weight)
_emu = {}


def _emu_inputs(name, dt):
    if (name, dt) not in _emu:
        m, d, f = EMU_SHAPES[name]
        _emu[(name, dt)] = _emu_layer(dt, m, d, f, seed=11 + sorted(EMU_SHAPES).index(name))
    return _emu[(name, dt)]


@pytest.mark.parametrize("dt", [F16, BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("name", sorted(EMU_SHAPES))
def test_bound_passes_emulated_phases_with_margin(name, dt):
    inp = _emu_inputs(name, dt)
    out = emulate_layer(inp, dt)
    fails = []
    for ph, R in layer_refs(inp, out, dt).items():
        msg = stack64.report(R.violations(out[ph], 0.5), out[ph], R, f"emulated {name} {NAMES[dt]} {ph} against half the bound")
        fails += [msg] if msg else []
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("mutation", stack64.MUTATIONS)
def test_bound_catches_kernel_bugs(mutation):
    """bf16: each injected bug leaves elements outside the bound of some phase (the references use the emulation's own
    inputs to each phase, as the GPU test uses the kernel's)"""
    seen = {}
    for name in sorted(EMU_SHAPES):
        inp = _emu_inputs(name, BF16)
        out = emulate_layer(inp, BF16, mutation)
        for ph, R in layer_refs(inp, out, BF16).items():
            seen[(name, ph)] = int(R.violations(out[ph]).sum())
    assert any(seen.values()), f"{mutation} stays inside the bound: {seen}"


def test_split_rounded_case_has_splits():
    """the mutation split_rounded needs split tiles with several partials in the emulated shapes"""
    assert GemmDeal(1, 1024, 256, stack64.NUM_SMS).S >= 2 and GemmDeal(1, 1024, 704, stack64.NUM_SMS).S >= 2


def _stack_attn_case():
    return attn64.Case(4, 7, 7, 1024, [1000, 1000, 640, 64], seed=40)


@pytest.mark.parametrize("mutation", [None, "merge_skip_last"])
def test_attention_merge_under_the_stack_dealing(monkeypatch, mutation):
    """attn64's float32 emulation of attn_stream_kernel's consumers, dealt over the stack's 132 CTAs (the stack's consumer
    arithmetic is the same, see stack64): within half the bound as is; a skipped CTA partial in the merge fails it"""
    monkeypatch.setattr(attn64, "GRID_MAX", stack64.NUM_SMS)
    c = _stack_attn_case()
    refs = c.reference()
    deal = attn64.Deal(BF16, c.B, c.Hq, c.Hkv, c.S, c.pos)
    sd = StackDeal(c.B, c.Hq, c.S, c.pos)
    assert deal.ncta == sd.ncta and deal.u0 == sd.u0
    with np.errstate(all="ignore"):
        got = attn64.emulate(c, BF16, mutation)
    bad = attn64.violations(got, refs, BF16, False, scale=0.5 if mutation is None else 1.0)
    if mutation is None:
        msg = attn64.report(bad, got, refs, BF16, False, deal, "stack dealing, emulated")
        assert msg is None, msg
    else:
        assert bad.any(), "a skipped CTA partial stays inside the bound"


def test_stale_rope_table_fails_the_bound():
    """a CTA whose segment crosses into a new batch row but keeps the previous row's RoPE table rotates q (and the appended
    k) by the wrong position; the heads it serves leave the attention bound"""
    B, H, p, rpos = 2, 3, [40, 100], np.array([7, 900])
    right, stale = (attn64.Case(B, H, H, 128, p, seed=5) for _ in range(2))
    q = right.q
    right.q = stack64.rope(q, rpos, BF16).astype(np.float32)
    stale.q = right.q.copy()
    stale.q[1] = stack64.rope(q[1:2], rpos[:1], BF16)[0]
    refs = right.reference()
    with np.errstate(all="ignore"):
        assert not attn64.violations(attn64.emulate(right, BF16), refs, BF16, False).any()
        assert attn64.violations(attn64.emulate(stale, BF16), refs, BF16, False)[1].any()


# ====================================================================== GPU plumbing
@pytest.fixture(scope="module")
def K():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from tests import kernel_harness
    return kernel_harness


def _guarded(K, shape, dt):
    from tests.test_attention_float64 import guarded
    return guarded(K, np.zeros(shape, np.float32), dt)


def _bits(t):
    import torch
    return t.contiguous().view(torch.int16).cpu().numpy()


def _interpose(K, dt):
    """a decode GEMM chain of three phases: its launch moves the grid-barrier generation by two"""
    import torch
    from infinitensor_b200 import _lib as L
    x = K.dev(stack64.rows(2, 128, dt, 3), dt)
    ws_ = [K.dev(np.eye(128, dtype=np.float32), dt) for _ in range(3)]
    outs = [torch.empty((2, 128), dtype=K.TORCH_DT[dt], device="cuda") for _ in range(3)]
    VP = ctypes.c_void_p
    arr = lambda v: (VP * len(v))(*v)
    wsb = 8 << 20
    wsp = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    L.check(L.lib.it_b200_decode_gemm_chain(dt, 2, 3, L.i32arr([1, 1, 1]), arr([w.data_ptr() for w in ws_]),
                                            arr([o.data_ptr() for o in outs]), L.i32arr([128] * 3), L.i32arr([128] * 3),
                                            L.i32arr([0] * 3), L.i32arr([0] * 3),
                                            arr([x.data_ptr(), outs[0].data_ptr(), outs[1].data_ptr()]), None, None, None,
                                            VP(wsp.data_ptr()), wsb, K.stream()))
    K.sync()
    assert np.array_equal(K.host(outs[2]), K.host(x)), "interposed chain: identity weights must return x"


class Stack:
    """one stack case in one dtype on the device"""
    OUTS = ["q", "k", "v", "attn_out", "x_mid", "gate", "up", "x_out"]

    def __init__(self, K, c, dt, seed):
        import torch
        from tests.test_attention_float64 import GUARD, GUARD_BITS
        from infinitensor_b200 import _lib as L
        self.K, self.c, self.dt, self.L = K, c, dt, L
        B, d, H, f, S, nl = c["B"], c["d"], c["H"], c["ffn"], c["S"], c["layers"]
        dl = H * 128
        self.dl, self.GUARD, self.GUARD_BITS = dl, GUARD, GUARD_BITS
        self.sms = torch.cuda.get_device_properties(0).multi_processor_count  # the grid the launch deals over
        self.pos = case_pos(c)
        self.pos_raw = np.broadcast_to(np.asarray(c["pos"], np.int64), (B,)).copy()
        self.rope_pos = np.asarray(c["rope"] if c["rope"] is not None else self.pos_raw, np.int64)
        npd = np.int64 if c["pos_dt"] == I64 else np.int32
        self.pos_dev = K.raw(self.pos_raw.astype(npd))
        self.rope_dev = K.raw(self.rope_pos.astype(npd)) if c["rope"] is not None else self.pos_dev
        self.flags = c["pos_dt"] | (PER_ROW if isinstance(c["pos"], list) else 0) | (IN_STEP if c["rope"] is not None else 0)
        TD = K.TORCH_DT[dt]
        dev = "cuda"
        s = seed * 100
        self.x_in = K.dev(stack64.rows(B, d, dt, s), dt)
        self.x_in_bits = _bits(self.x_in)
        self.layers = []
        for li in range(nl):
            t = s + 10 * (li + 1)
            # q, k elements about 2 in rms and cache k rows of rms 2: scores q.k / sqrt(128) of std about 4, spanning tens
            Ly = dict(ln1=stack64.norm_weight(d, dt, t), ln2=stack64.norm_weight(d, dt, t + 1),
                      wq=stack64.weights(d, dl, dt, t + 2, 1.2 / np.sqrt(d), dev),
                      wk=stack64.weights(d, dl, dt, t + 3, 1.2 / np.sqrt(d), dev),
                      wv=stack64.weights(d, dl, dt, t + 4, 0.5 / np.sqrt(d), dev),
                      wo=stack64.weights(dl, d, dt, t + 5, 0.5 / np.sqrt(dl), dev),
                      wg=stack64.weights(d, f, dt, t + 6, 1.0 / np.sqrt(d), dev),
                      wu=stack64.weights(d, f, dt, t + 7, 1.0 / np.sqrt(d), dev),
                      wd=stack64.weights(f, d, dt, t + 8, 0.5 / np.sqrt(f), dev))
            Ly["ln1_dev"], Ly["ln2_dev"] = K.dev(Ly["ln1"], dt), K.dev(Ly["ln2"], dt)
            g = torch.Generator(device=dev).manual_seed(t + 9)
            kc = torch.randn((B, H, S, 128), generator=g, device=dev) * 2.0
            vrow = torch.exp2((torch.arange(S, device=dev) % 5) - 2.0)[None, None, :, None]
            vh = torch.exp2((torch.arange(H, device=dev) % 3) - 1.0)[None, :, None, None]
            vc = torch.randn((B, H, S, 128), generator=g, device=dev) * 0.5 * vrow * vh
            for name, val in (("kc", kc), ("vc", vc)):
                buf = torch.full((B * H * S * 128 + GUARD,), GUARD_BITS[dt], dtype=torch.int16, device=dev)
                view = buf[:-GUARD].view(TD).view(B, H, S, 128)
                view.copy_(val.to(TD))
                Ly[name] = (buf, view)
            for name, w in (("q", dl), ("k", dl), ("v", dl), ("attn_out", dl), ("x_mid", d), ("gate", f), ("up", f), ("x_out", d)):
                Ly[name] = _guarded(K, (B, w), dt)
            self.layers.append(Ly)
        self.wsb = int(L.lib.it_b200_decode_stack_workspace(nl, B, d, H, S, f))
        self.ws = torch.empty(self.wsb // 4, dtype=torch.float32, device=dev)
        self.arr = (L.LlamaLayer * nl)()
        for li, Ly in enumerate(self.layers):
            vals = dict(ln1_w=Ly["ln1_dev"].data_ptr(), wq=Ly["wq"].data_ptr(), wk=Ly["wk"].data_ptr(), wv=Ly["wv"].data_ptr(),
                        wo=Ly["wo"].data_ptr(), ln2_w=Ly["ln2_dev"].data_ptr(), wg=Ly["wg"].data_ptr(), wu=Ly["wu"].data_ptr(),
                        wd=Ly["wd"].data_ptr(), k_cache=Ly["kc"][1].data_ptr(), v_cache=Ly["vc"][1].data_ptr())
            vals.update({n: Ly[n][1].data_ptr() for n in self.OUTS})
            for k_, v_ in vals.items():
                setattr(self.arr[li], k_, v_)
        self.snapshot_caches()

    def snapshot_caches(self):
        """the cache contents every launch must leave in place (rows >= pos are NaN-filled before a launch)"""
        for Ly in self.layers:
            for name in ("kc", "vc"):
                v = Ly[name][1]
                for b in range(self.c["B"]):
                    v[b, :, int(self.pos[b]):].fill_(float("nan"))
            Ly["kc_before"], Ly["vc_before"] = Ly["kc"][0][:-self.GUARD].clone(), Ly["vc"][0][:-self.GUARD].clone()

    def launch(self):
        """NaN-fill, launch, return {layer: {name: float32 [B, w]}} plus the raw bits of every output"""
        import torch
        K, c, L = self.K, self.c, self.L
        for Ly in self.layers:
            for n in self.OUTS:
                Ly[n][0][:-self.GUARD].fill_(0x7FFF)
            for name in ("kc", "vc"):
                Ly[name][0][:-self.GUARD].copy_(Ly[name + "_before"])
        self.ws.fill_(float("nan"))
        L.check(L.lib.it_b200_llama_decode_stack(self.dt, c["layers"], ctypes.cast(self.arr, ctypes.c_void_p), K.ptr(self.x_in),
                                                 K.ptr(self.pos_dev), self.flags, K.ptr(self.rope_dev), c["pos_dt"], c["B"], c["d"],
                                                 c["H"], c["S"], c["ffn"], K.ptr(self.ws), self.wsb, K.stream()))
        K.sync()
        res = [{n: Ly[n][1].float().cpu().numpy() for n in self.OUTS} for Ly in self.layers]
        bits = [{n: _bits(Ly[n][1]) for n in self.OUTS} | {nm: _bits(Ly[nm][0]) for nm in ("kc", "vc")} for Ly in self.layers]
        return res, bits

    def rope(self, x):
        """it_b200_rope of [B, H 128] with the stack's RoPE positions -> [B, H, 128] float32, and the T bits"""
        import torch
        K, B = self.K, self.c["B"]
        xd = K.dev(x, self.dt)
        y = torch.empty_like(xd)
        code = self.c["pos_dt"]
        K.L.check(K.L.lib.it_b200_rope(self.dt, K.ptr(self.rope_dev), code, K.ptr(xd), K.ptr(y), B, 1, self.dl, 128, K.stream()))
        K.sync()
        return K.host(y).reshape(B, -1, 128), _bits(y).reshape(B, -1, 128)

    def rebuild_layer0(self, q0):
        """layer 0's cache k rows below each position set along the rotated q so that attn64's regimes cycle over (row, head)"""
        import torch
        c, dt = self.c, self.dt
        qr, _ = self.rope(q0)
        rng = np.random.default_rng(77)
        Ly = self.layers[0]
        kv = Ly["kc"][1]
        for b in range(c["B"]):
            p = int(self.pos[b])
            if p == 0:
                continue
            z = kv[b, :, :p].float().cpu().numpy().astype(np.float64)
            for h in range(c["H"]):
                q = qr[b, h].astype(np.float64)
                reg = attn64.REGIMES[(b * c["H"] + h) % len(attn64.REGIMES)]
                for j, t in attn64.targets(reg, p, rng).items():
                    if j < p:
                        z[h, j] += (t * np.sqrt(128.0) - q @ z[h, j]) / (q @ q) * q
            kv[b, :, :p].copy_(torch.from_numpy(stack64.rnd(z, dt).astype(np.float32)).to(kv.dtype))
        self.snapshot_caches()

    def cache_host(self, li, name):
        return self.layers[li][name][1].float().cpu().numpy()


def check_guards(st, what):
    fails = []
    for li, Ly in enumerate(st.layers):
        for n in st.OUTS + ["kc", "vc"]:
            if not bool((Ly[n][0][-st.GUARD:] == st.GUARD_BITS[st.dt]).all()):
                fails.append(f"{what}: layer {li} {n} guard written")
    if not np.array_equal(_bits(st.x_in), st.x_in_bits):
        fails.append(f"{what}: x_in changed")
    return fails


def check_phases(st, res, bits, what, stats):
    """every phase of every layer against float64 from the launch's own inputs to it"""
    c, dt = st.c, st.dt
    B, d, H = c["B"], c["d"], c["H"]
    nt = -(-d // 128)
    fails = []

    def hold(R, got, name, op=None):
        r = R.ratio(got)
        stats[name] = max(stats.get(name, 0.0), r)
        if op is not None:
            stats[name + " amb"] = max(stats.get(name + " amb", 0.0), op.share)
            if op.share > MAX_AMB_SHARE:
                fails.append(f"{what} {name}: {100 * op.share:.2f} % of the operand is ambiguous")
        msg = stack64.report(R.violations(got), got, R, f"{what} {name}")
        fails.extend([msg] if msg else [])

    for li, Ly in enumerate(st.layers):
        o = res[li]
        x = st.x_in.float().cpu().numpy() if li == 0 else res[li - 1]["x_out"]
        L1 = stack64.chain_length("x_raw", d) if li == 0 else stack64.chain_length("ss", d, nt=nt)
        op1 = stack64.rmsnorm_operand(x, Ly["ln1"], dt, L1)
        for n, w in (("q", "wq"), ("k", "wk"), ("v", "wv")):
            hold(stack64.store_ref(op1, Ly[w], dt), o[n], f"L{li} rmsnorm->{n}", op1)
        # attention: the appended rows bit for bit, every other row untouched, the output within attn64's bound
        qr, _ = st.rope(o["q"])
        kr, kbits = st.rope(o["k"])
        vbits = bits[li]["v"].reshape(B, H, 128)
        for name, new in (("kc", kbits), ("vc", vbits)):
            want = Ly[name + "_before"].view(B, H, c["S"], 128).cpu().numpy().copy()
            for b in range(B):
                want[b, :, int(st.pos[b])] = new[b]
            got = bits[li][name][:-st.GUARD].reshape(want.shape)
            if not np.array_equal(got, want):
                badr = np.argwhere((got != want).any(-1))[:4].tolist()
                fails.append(f"{what}: layer {li} {name}: rows differ from the expected bits at (b, head, row) {badr}")
        kc, vc = st.cache_host(li, "kc"), st.cache_host(li, "vc")
        case = stack64.AttnInputs(qr, kc, vc, kr, o["v"].reshape(B, H, 128), st.pos)
        refs = case.reference()
        got = o["attn_out"].reshape(B, H, 128)
        with np.errstate(invalid="ignore", divide="ignore"):
            r = float(np.nanmax(np.where(np.isnan(got), np.inf, np.abs(got - refs[0]) / attn64.bound(refs, dt, False))))
        stats["attention"] = max(stats.get("attention", 0.0), r)
        msg = attn64.report(attn64.violations(got, refs, dt, False), got, refs, dt, False,
                            StackDeal(B, H, c["S"], st.pos, st.sms), f"{what} layer {li} attention")
        fails += [msg] if msg else []
        hold(stack64.residual_ref(Operand(o["attn_out"]), Ly["wo"], x, dt), o["x_mid"], f"L{li} o-proj+residual")
        op4 = stack64.rmsnorm_operand(o["x_mid"], Ly["ln2"], dt, stack64.chain_length("ss", d, nt=nt))
        hold(stack64.store_ref(op4, Ly["wg"], dt), o["gate"], f"L{li} rmsnorm->gate", op4)
        hold(stack64.store_ref(op4, Ly["wu"], dt), o["up"], f"L{li} rmsnorm->up", op4)
        op5 = stack64.silu_mul_operand(o["gate"], o["up"], dt)
        hold(stack64.residual_ref(op5, Ly["wd"], o["x_mid"], dt), o["x_out"], f"L{li} silu.mul->down+residual", op5)
    return fails


def _same_bits(a, b):
    return all(np.array_equal(x[n], y[n]) for x, y in zip(a, b) for n in x)


SUMMARY = {}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(STACK_CASES))
def test_decode_stack_float64(K, name):
    c = spec(name)
    fails = []
    for dt in c["dts"]:
        t0 = time.time()
        what = f"{name} {NAMES[dt]}"
        st = Stack(K, c, dt, seed=1 + list(STACK_CASES).index(name))
        res1, bits1 = st.launch()
        fails += check_guards(st, what + " (first launch)")
        st.rebuild_layer0(res1[0]["q"])
        res2, bits2 = st.launch()
        for n in ("q", "k", "v"):
            if not np.array_equal(bits1[0][n], bits2[0][n]):
                fails.append(f"{what}: layer 0 {n} changed between launches (it depends only on x and the weights)")
        fails += check_guards(st, what)
        stats = {}
        fails += check_phases(st, res2, bits2, what, stats)
        _interpose(K, dt)
        _, bits3 = st.launch()
        if not _same_bits(bits2, bits3):
            fails.append(f"{what}: a launch after another program differs from the one before it")
        fails += check_guards(st, what + " (third launch)")
        SUMMARY[what] = {k: round(v, 4) for k, v in stats.items()} | {"wall_s": round(time.time() - t0, 1)}
        print(f"\n{what}: {SUMMARY[what]}")
        del st
    assert not fails, "\n".join(fails)


# ====================================================================== GPU: the chain shapes of test_gpu_decode_stack.py
def _chain(K, dt, rows, phases):
    from tests.test_gpu_decode_stack import chain
    return chain(K, dt, rows, phases)


def _t(w):
    import torch
    return torch.from_numpy(np.asarray(w, np.float32))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [BF16, F16], ids=["bf16", "f16"])
@pytest.mark.parametrize("rows,k,n", [(1, 200, 8), (5, 1000, 136), (5, 200, 8), (1, 1000, 136), (16, 1000, 136)])
def test_chain_single_gemm_float64(K, rows, k, n, dt):
    x = stack64.rows(rows, k, dt, 1, 0.5)
    w = ref64.weights(k, n, dt, 2)
    got = _chain(K, dt, rows, [dict(W=[w], X=x.astype(np.float32))])[0][0]
    R = stack64.store_ref(Operand(x), _t(w), dt)
    msg = stack64.report(R.violations(got), got, R, f"chain {rows}x{k}x{n} {NAMES[dt]}")
    assert msg is None, msg


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [BF16, F16], ids=["bf16", "f16"])
def test_chain_grouped_rmsnorm_and_residual_float64(K, dt):
    rows, d = 16, 1024
    x, nw = stack64.rows(rows, d, dt, 3), stack64.norm_weight(d, dt, 4)
    ws = [ref64.weights(d, d, dt, 5 + i, 0.03) for i in range(3)]
    wo, res = ref64.weights(d, d, dt, 9, 0.03), stack64.rows(rows, d, dt, 10)
    got = _chain(K, dt, rows, [dict(W=ws, X=x.astype(np.float32), xform=1, norm_w=nw.astype(np.float32)),
                               dict(W=[wo], X=("out", 0, 0), epi=1, residual=res.astype(np.float32))])
    op = stack64.rmsnorm_operand(x, nw, dt, stack64.chain_length("x_raw", d))
    fails = []
    for g, w in enumerate(ws):
        R = stack64.store_ref(op, _t(w), dt)
        fails.append(stack64.report(R.violations(got[0][g]), got[0][g], R, f"group {g}"))
    R = stack64.residual_ref(Operand(got[0][0]), _t(wo), res, dt)
    fails.append(stack64.report(R.violations(got[1][0]), got[1][0], R, "residual"))
    assert op.share <= MAX_AMB_SHARE and not any(fails), "\n".join(f for f in fails if f)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [BF16, F16], ids=["bf16", "f16"])
@pytest.mark.parametrize("rows,d,f", [(16, 1024, 2816), (7, 512, 1408), (5, 4096, 11008)])
def test_chain_mlp_half_layer_float64(K, rows, d, f, dt):
    a, x0 = stack64.rows(rows, d, dt, 11, 0.5), stack64.rows(rows, d, dt, 12)
    wo, wg, wu, wd = (ref64.weights(d, d, dt, 13, 0.02), ref64.weights(d, f, dt, 14, 0.02), ref64.weights(d, f, dt, 15, 0.02),
                      ref64.weights(f, d, dt, 16, 0.02))
    nw = stack64.norm_weight(d, dt, 17)
    got = _chain(K, dt, rows, [dict(W=[wo], X=a.astype(np.float32), epi=1, residual=x0.astype(np.float32)),
                               dict(W=[wg, wu], X=("out", 0, 0), xform=1, norm_w=nw.astype(np.float32)),
                               dict(W=[wd], X=("out", 1, 0), X2=("out", 1, 1), xform=2, epi=1, residual=("out", 0, 0))])
    xm, g_, u_, xo = got[0][0], got[1][0], got[1][1], got[2][0]
    fails = []
    R = stack64.residual_ref(Operand(a), _t(wo), x0, dt)
    fails.append(stack64.report(R.violations(xm), xm, R, "o-proj + residual"))
    op = stack64.rmsnorm_operand(xm, nw, dt, stack64.chain_length("ss", d, nt=-(-d // 128)))
    for nm, w, gv in (("gate", wg, g_), ("up", wu, u_)):
        R = stack64.store_ref(op, _t(w), dt)
        fails.append(stack64.report(R.violations(gv), gv, R, nm))
    op5 = stack64.silu_mul_operand(g_, u_, dt)
    R = stack64.residual_ref(op5, _t(wd), xm, dt)
    fails.append(stack64.report(R.violations(xo), xo, R, "down + residual"))
    assert max(op.share, op5.share) <= MAX_AMB_SHARE and not any(fails), "\n".join(f for f in fails if f)


# ====================================================================== GPU: the unfused kernels the stack replaces
def rmsnorm_path(dt, hidden):
    """rmsnorm_impl's choice for aligned pointers: "one" (one vector per thread), "vec" or "scalar", and items per thread"""
    V = 4 if dt == F32 else 8
    threads = 512 if hidden >= 4096 else 256 if hidden >= 1024 else 128
    if hidden % V:
        return "scalar", -(-hidden // threads)
    nv = hidden // V
    return ("one", V) if nv <= threads else ("vec", -(-nv // threads) * V)


RMS_HIDDEN = [4096, 1024, 5120, 1000, 1004, 1001]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F32, F16, BF16], ids=["fp32", "f16", "bf16"])
@pytest.mark.parametrize("hidden", RMS_HIDDEN)
def test_unfused_rmsnorm_float64(K, hidden, dt):
    """every element of it_b200_rmsnorm / _constw equals rnd(rnd(x rinv) w) or, where rinv's fp32 window straddles a rounding
    point, a value between the two ends"""
    x = stack64.rows(24, hidden, dt, hidden) if dt != F32 else \
        np.random.default_rng(hidden).standard_normal((24, hidden)).astype(np.float32) * ref64.row_scale(24)[:, None]
    w = stack64.norm_weight(hidden, dt, hidden + 1)
    path, items = rmsnorm_path(dt, hidden)
    op = stack64.rmsnorm_operand(x, w, dt, stack64.chain_length("block", hidden, items=items))
    fails = []
    for const_w in (False, True):
        got = K.rms_norm(x.astype(np.float32), w.astype(np.float32), dt, const_w)
        bad = op.outside(got)
        if bad.any():
            i, j = np.argwhere(bad)[0]
            fails.append(f"{path} const_w={const_w}: {int(bad.sum())} elements outside; first ({i}, {j}): got {got[i, j]!r}, "
                         f"nominal {op.a[i, j]!r}, candidates {op.lo[i, j]!r} .. {op.hi[i, j]!r}")
    assert not fails and op.share <= (1.0 if dt == F32 else MAX_AMB_SHARE), "\n".join(fails) or f"ambiguous {op.share:.3%}"


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F32, F16, BF16], ids=["fp32", "f16", "bf16"])
@pytest.mark.parametrize("n", [16 * 1024, 16 * 1000 + 5])
def test_unfused_silu_mul_float64(K, n, dt):
    """it_b200_silu_mul, vector loop and scalar tail: rnd(rnd(silu(g)) u) or the other candidate where ambiguous"""
    rng = np.random.default_rng(n)
    g = stack64.rnd(rng.standard_normal(n) * 3.0, dt) if dt != F32 else (rng.standard_normal(n) * 3.0).astype(np.float32)
    u = stack64.rnd(rng.standard_normal(n), dt) if dt != F32 else rng.standard_normal(n).astype(np.float32)
    op = stack64.silu_mul_operand(g, u, dt)
    got = K.silu_mul(np.asarray(g, np.float32), np.asarray(u, np.float32), dt)
    bad = op.outside(got)
    assert not bad.any(), f"{int(bad.sum())} elements outside; first {np.argwhere(bad)[0]}"


# ====================================================================== GPU: the intended kernels ran
def profiled_kernel_names():
    import torch
    from tests import kernel_harness as K
    x = np.random.default_rng(0).standard_normal((4, 5120)).astype(np.float32)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for dt in (F16, BF16):
            st = Stack(K, spec("tiny_p63"), dt, seed=99)
            st.launch()
            for h, cw in ((1024, True), (1024, False), (5120, False)):
                K.rms_norm(x[:, :h], np.ones(h, np.float32), dt, cw)
            K.silu_mul(x[0], x[1], dt)
        torch.cuda.synchronize()
    return sorted({e.name for e in prof.events() if "CUDA" in str(e.device_type)})


@pytest.mark.gpu
def test_decode_stack_cases_reach_the_intended_kernels():
    """in a child process, as test_attention_float64 does: a profiler session in the test process loses records of later ones"""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = "import json; from tests.test_decode_stack_float64 import profiled_kernel_names as f; print(json.dumps(f()))"
    r = subprocess.run([sys.executable, "-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    names = set(json.loads(r.stdout.strip().splitlines()[-1]))
    if not names:
        pytest.skip("the profiler recorded no CUDA kernel events (CUPTI activity tracing unavailable)")
    want = [r"decode_stack_kernel<__half>", r"decode_stack_kernel<__nv_bfloat16>", r"rmsnorm_kernel<.*true, true>",
            r"rmsnorm_kernel<.*true, false>", r"rmsnorm_kernel<.*false, false>", r"silu_mul_kernel"]
    missing = [p for p in want if not any(re.search(p, nm) for nm in names)]
    assert not missing, f"not launched: {missing}; kernels seen: {sorted(names)}"
