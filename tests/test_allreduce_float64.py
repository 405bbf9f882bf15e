"""The tensor-parallel all-reduce + residual + RMSNorm kernel (`allreduce_ll_kernel`, allreduce.cu) against a float32
emulation bit for bit and against float64, at every world size, on one GPU (helpers in tests/ar64.py).

The kernel takes raw peer-workspace pointers and its LL protocol is deterministic, so a world of W ranks runs on one device:
W workspaces, the ranks launched one after another on one stream.  Before a round every slot of every workspace holds NaN
payload carrying the tag its row will look for (the other parity, rows >= M, ranks >= W, each rank's own slot, the slots of
ranks launched earlier), and only the packets of the ranks launched LATER are staged: a rank reads real pushes from the ranks
before it, staged packets from the ones after it, and NaN, at once and without polling, from anywhere a wrong parity, stride
or missing push would send it.  The launch order rotates over the rounds, so every (writer, reader) pair is real in some round.
After a round every workspace must equal the model bit for bit (epoch[row] + 1 for rows < M, the packets of every rank in
slot (e & 1, p, row), nothing else written), the timeout flag must be 0, `out` and `out_norm` must be the same bits on every
rank, guards after them untouched and the inputs unchanged.

* out: bit for bit against ar64.emulate and within ar64.out_ref's float64 bound;
* out_norm: inside operand64.rmsnorm_operand's interval from the kernel's own out, within ar64.norm_bound, and bit for bit equal
  to it_b200_rmsnorm / _constw of the same out where the two kernels' per-thread partitions coincide;
* epochs: zero, per-row epochs of both parities in one launch, sequences of rounds with M and the order varying on the same
  workspaces, and a sequence through the wrap at INT_MAX (the epoch arithmetic is unsigned).

The graph tier runs AllReduceSum -> Add -> RMSNorm through the runtime at world 1 (the fused step, eager and CUDA-graph
replayed; the three separate operators when a one-rank NCCL communicator can be made), and a torchrun tier
(tools/ar_worker.py) runs the same layer on 2, 4 and 8 GPUs through the production IPC mapping when the box has them.
"""
import ctypes
import json
import os
import re
import subprocess
import sys
import time

import numpy as np
import pytest

from tests import ar64
from tests.ar64 import BF16, F16, F32

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT_MAX = 2 ** 31 - 1

# ====================================================================== cases
# name: dict(dt, W, M, H, regime, res, norm, epochs (int or per-row list), ms (M per round; default W rounds of M))
MIXED_EPOCHS = [(r * 5) % 7 for r in range(64)]                     # both parities among the rows of one launch
CASES = {
    "bf16_tp8_M16_H4096": dict(dt=BF16, W=8, M=16, H=4096),                          # the benchmark's TP-8 shape
    "bf16_W2_M16_H4096_cancel": dict(dt=BF16, W=2, M=16, H=4096, regime="cancel"),
    "bf16_W7_M63_H4160_spread": dict(dt=BF16, W=7, M=63, H=4160, regime="spread"),  # nv 520: a ragged second pass
    "bf16_W4_M64_H8192_residual": dict(dt=BF16, W=4, M=64, H=8192, regime="residual_dominates"),   # the 16 KiB row
    "bf16_W3_M1_H8_one_vector": dict(dt=BF16, W=3, M=1, H=8),
    "bf16_W8_M64_H128_nores": dict(dt=BF16, W=8, M=64, H=128, res=False),           # nv 16 < 32
    "bf16_W3_M16_H264_nonorm": dict(dt=BF16, W=3, M=16, H=264, norm=False, regime="spread"),   # nv 33
    "bf16_W4_M16_H3072": dict(dt=BF16, W=4, M=16, H=3072),                           # partitions differ
    "bf16_W2_M63_H5120_huge": dict(dt=BF16, W=2, M=63, H=5120, regime="huge_element"),
    "bf16_W1_M64_H4096_subnormal": dict(dt=BF16, W=1, M=64, H=4096, regime="subnormal"),
    "bf16_W8_M1_H4096_bare": dict(dt=BF16, W=8, M=1, H=4096, res=False, norm=False),
    "bf16_W4_M64_H4096_mixed_epochs": dict(dt=BF16, W=4, M=64, H=4096, epochs=MIXED_EPOCHS),
    "f16_W4_M16_H4096_overflow": dict(dt=F16, W=4, M=16, H=4096, regime="overflow"),
    "f16_W2_M64_H8192_subnormal": dict(dt=F16, W=2, M=64, H=8192, regime="subnormal"),
    "f16_W7_M16_H264_spread": dict(dt=F16, W=7, M=16, H=264, regime="spread"),
    "f16_W1_M1_H8_zero": dict(dt=F16, W=1, M=1, H=8, regime="zero_rows"),
    "f16_W8_M63_H4096_cancel": dict(dt=F16, W=8, M=63, H=4096, regime="cancel", res=False),
    "f16_W3_M16_H5120_huge": dict(dt=F16, W=3, M=16, H=5120, regime="huge_element"),
    "fp32_W2_M16_H2048": dict(dt=F32, W=2, M=16, H=2048),                            # partitions differ
    "fp32_W8_M64_H4096_spread": dict(dt=F32, W=8, M=64, H=4096, regime="spread"),   # the 16 KiB row
    "fp32_W3_M1_H4_one_vector": dict(dt=F32, W=3, M=1, H=4, regime="zero_rows"),
    "fp32_W4_M16_H1000_cancel": dict(dt=F32, W=4, M=16, H=1000, regime="cancel"),
    # sequences on the same workspaces: M and the launch order change every round, rows fall behind and catch up
    "seq_bf16_W4_H4096": dict(dt=BF16, W=4, M=16, H=4096, ms=[16, 64, 1, 63, 16, 40, 64, 5]),
    "seq_f16_W3_H2048_wrap": dict(dt=F16, W=3, M=16, H=2048, epochs=INT_MAX - 2, ms=[8, 16, 3, 16, 16, 9, 16]),
    "seq_bf16_W8_H4096_wrap": dict(dt=BF16, W=8, M=16, H=4096, epochs=INT_MAX - 2, ms=[16, 16, 4, 16, 16, 16]),
    "seq_fp32_W7_H4096": dict(dt=F32, W=7, M=64, H=4096, regime="spread", ms=[64, 2, 64, 33, 64, 64, 1]),
}
DEFAULTS = dict(regime="normal", res=True, norm=True, epochs=0, ms=None)


def spec(name):
    return {**DEFAULTS, **CASES[name]}


def plan(c):
    """[(M, launch order)] per round: the rotations of the ranks, reversed on odd rounds"""
    W = c["W"]
    ms = c["ms"] or [c["M"]] * W
    out = []
    for k, m in enumerate(ms):
        order = [(k + j) % W for j in range(W)]
        out.append((m, order[::-1] if k % 2 else order))
    return out


def epoch_states(c):
    """per round, the uint32 epochs of the launched rows (the model of World.epoch)"""
    e = np.broadcast_to(np.asarray(c["epochs"], np.int64) & 0xFFFFFFFF, (ar64.MAX_ROWS,)).copy()
    states = []
    for m, _ in plan(c):
        states.append(e[:m].copy())
        e[:m] = (e[:m] + 1) & 0xFFFFFFFF
    return states


def seed_of(name, k):
    return 1000 * (1 + sorted(CASES).index(name)) + k


# ====================================================================== CPU: layout, launch rules, coverage
def test_workspace_layout_matches_the_library():
    from infinitensor_b200 import _lib as L
    assert int(L.lib.it_b200_allreduce_workspace_bytes()) == ar64.WS_BYTES
    assert ar64.DATA_OFF == 5120 and ar64.slot_offset(1, 7, 63) + ar64.SLOT_BYTES == ar64.WS_BYTES


def test_partition_rule():
    """where out_norm must equal rmsnorm_kernel's bits: the TP shape and small rows coincide, bf16 3072 and fp32 2048 do not"""
    assert ar64.partitions_coincide(BF16, 4096) and ar64.partitions_coincide(BF16, 264) and ar64.partitions_coincide(F32, 4096)
    assert not ar64.partitions_coincide(BF16, 3072) and not ar64.partitions_coincide(F32, 2048)
    assert ar64.ar_threads(BF16, 264) == 64 and ar64.ar_threads(BF16, 4160) == 512 and ar64.ar_threads(F32, 4) == 32


def test_case_list_reaches():
    seen = dict(W=set(), M=set(), dt=set(), coincide=set(), res=set(), norm=set(), regimes=set())
    order_sensitive = mixed_parity = wrap = 0
    ragged = exact512 = tail = small = False
    for name in CASES:
        c = spec(name)
        dt, H = c["dt"], c["H"]
        nv = ar64.nvec(dt, H)
        seen["W"].add(c["W"])
        seen["dt"].add(dt)
        seen["coincide"].add(ar64.partitions_coincide(dt, H))
        seen["res"].add(c["res"])
        seen["norm"].add(c["norm"])
        seen["regimes"].add(c["regime"])
        ragged |= nv > 512 and nv % 512 != 0
        exact512 |= nv == 512
        tail |= nv % 32 != 0
        small |= nv < 32
        for (m, _), e in zip(plan(c), epoch_states(c)):
            seen["M"].add(m)
            mixed_parity += len(set((e & 1).tolist())) == 2
            wrap += bool(np.any(e == INT_MAX))
        if c["regime"] == "spread" and c["W"] > 1:
            P, _, _ = ar64.inputs(dt, c["W"], plan(c)[0][0], H, c["regime"], seed_of(name, 0), c["res"], c["norm"])
            order_sensitive += ar64.order_sensitive(P)
    assert seen["W"] >= {1, 2, 3, 4, 7, 8} and seen["M"] >= {1, 16, 63, 64} and seen["dt"] == {F32, F16, BF16}, seen
    assert seen["coincide"] == {True, False} and seen["res"] == {True, False} and seen["norm"] == {True, False}, seen
    assert seen["regimes"] == set(ar64.REGIMES), seen["regimes"]
    assert ragged and exact512 and tail and small, "nv > 512 ragged, nv = 512, nv not a multiple of 32, nv < 32"
    assert order_sensitive > 100, f"only {order_sensitive} order-sensitive elements"
    assert mixed_parity >= 3 and wrap >= 2, (mixed_parity, wrap)


# ====================================================================== CPU: the bounds against the emulation
EMU_CASES = {  # small shapes of every regime; name: (dt, W, M, H, regime, res, norm)
    "bf16_normal": (BF16, 4, 5, 4160, "normal", True, True),
    "bf16_cancel": (BF16, 2, 6, 264, "cancel", True, True),
    "bf16_spread": (BF16, 8, 4, 3072, "spread", True, True),
    "bf16_residual": (BF16, 3, 4, 1024, "residual_dominates", True, True),
    "bf16_subnormal": (BF16, 3, 4, 1024, "subnormal", True, True),
    "bf16_huge": (BF16, 2, 4, 512, "huge_element", True, True),
    "f16_overflow": (F16, 4, 4, 1024, "overflow", True, False),
    "f16_subnormal": (F16, 4, 4, 264, "subnormal", False, True),
    "f16_zero": (F16, 2, 6, 136, "zero_rows", True, True),
    "f16_spread": (F16, 7, 4, 4160, "spread", True, True),
    "fp32_spread": (F32, 8, 4, 2048, "spread", True, True),
    "fp32_cancel": (F32, 2, 4, 1000, "cancel", True, True),
    "fp32_nores": (F32, 3, 4, 1028, "normal", False, True),
}
_emu = {}


def emu_case(name):
    if name not in _emu:
        dt, W, M, H, regime, res, norm = EMU_CASES[name]
        _emu[name] = (dt, ar64.inputs(dt, W, M, H, regime, 7 + sorted(EMU_CASES).index(name), res, norm))
    return _emu[name]


def norm_check(out, y, w, dt, scale=1.0):
    """(rows checked, interval failures, norm_bound ratio) over the rows whose out is finite"""
    fin = np.isfinite(out).all(1)
    if not fin.any():
        return fin, np.zeros((0,), bool), 0.0
    op = ar64.norm_operand(out[fin], w, dt)
    R = ar64.norm_bound(out[fin], w, dt)
    return fin, op.outside(y[fin]) | R.violations(y[fin], scale), R.ratio(y[fin])


@pytest.mark.parametrize("name", sorted(EMU_CASES))
def test_emulation_within_half_the_bounds(name):
    dt, (P, R, w) = emu_case(name)
    out, y = ar64.emulate(P, R, w, dt)
    Ro = ar64.out_ref(P, R, dt)
    msg = ar64.report(Ro.violations(out, 0.5), out, Ro, f"{name}: emulated out against half the bound", dt, P.shape[2])
    assert msg is None, msg
    if y is not None:
        fin, bad, r = norm_check(out, y, w, dt, 0.5)
        assert not bad.any(), f"{name}: emulated out_norm outside the interval or half the bound at {np.argwhere(bad)[:4]}"


@pytest.mark.parametrize("mutation", ar64.MUTATIONS)
def test_injected_bugs_fail(mutation):
    """each bug changes out's bits (the GPU check is bit for bit) or leaves out / out_norm outside a float64 bound"""
    caught = {}
    for name in sorted(EMU_CASES):
        dt, (P, R, w) = emu_case(name)
        out, y = ar64.emulate(P, R, w, dt)
        mo, my = ar64.emulate(P, R, w, dt, mutation)
        bits = not np.array_equal(out.view(np.int32), mo.view(np.int32))
        bound = bool(ar64.out_ref(P, R, dt).violations(mo).any())
        nb = False
        if my is not None:
            fin, bad, _ = norm_check(out, my, w, dt)
            nb = bool(bad.any())
        if mutation in ar64.OUT_MUTATIONS:
            caught[name] = bits or bound
        else:
            caught[name] = nb
    assert any(caught.values()), f"{mutation} passes every case: {caught}"


def test_out_bound_alone_catches_gross_bugs():
    """accumulating in T, dropping a rank and dropping the tail fail the float64 bound itself, not just the bit check"""
    for mutation in ("accumulate_in_T", "drop_last_rank", "drop_tail_vector"):
        hits = []
        for name in sorted(EMU_CASES):
            dt, (P, R, w) = emu_case(name)
            mo, _ = ar64.emulate(P, R, w, dt, mutation)
            hits.append(bool(ar64.out_ref(P, R, dt).violations(mo).any()))
        assert any(hits), mutation


# ====================================================================== CPU: argument rejections (before any CUDA call)
def _call(dt=BF16, inp=0x10000, res=0x20000, nw=0x30000, out=0x40000, on=0x50000, M=16, H=4096, peers=None, W=2, rank=0):
    from infinitensor_b200 import _lib as L
    VP = ctypes.c_void_p
    peers = peers if peers is not None else [0x100000 * (p + 1) for p in range(max(W, 1))]
    arr = (VP * max(len(peers), 1))(*[VP(p) if p else None for p in peers])
    v = lambda a: VP(a) if a else None
    return int(L.lib.it_b200_allreduce_fused(dt, v(inp), v(res), v(nw), v(out), v(on), M, H, arr, W, rank, None, None))


@pytest.mark.parametrize("args,what", [
    (dict(M=65), "65 rows"), (dict(H=8200), "a row over 16 KiB"), (dict(H=100), "a row not a multiple of 16 bytes"),
    (dict(dt=F32, H=4100), "an fp32 row over 16 KiB"), (dict(W=0, peers=[0x100000]), "world 0"),
    (dict(W=9, peers=[0x100000] * 9), "world 9"), (dict(rank=2), "rank = world"), (dict(rank=-1), "rank -1"),
    (dict(inp=0x10008), "misaligned in"), (dict(out=0x40004), "misaligned out"), (dict(res=0x20002), "misaligned residual"),
    (dict(nw=0x30008), "misaligned norm weight"), (dict(on=0x50008), "misaligned norm output"),
    (dict(on=0), "norm weight without norm output"), (dict(nw=0), "norm output without norm weight"),
    (dict(peers=[0x100000, 0]), "a NULL peer workspace"), (dict(dt=6), "an integer dtype"),
])
def test_argument_rejections(args, what):
    from infinitensor_b200 import _lib as L
    assert _call(**args) != 0, f"{what} accepted"
    assert "allreduce_fused" in L.last_error(), L.last_error()


def test_zero_rows_is_a_no_op():
    assert _call(M=0, peers=[0, 0]) == 0


# ====================================================================== GPU: the kernel at every world size
@pytest.fixture(scope="module")
def K():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from tests import kernel_harness
    return kernel_harness


def _int_dt(dt):
    import torch
    return torch.int32 if dt == F32 else torch.int16


def _bits(t, dt):
    return t.contiguous().view(_int_dt(dt)).cpu().numpy()


def _guarded(K, n, dt):
    from tests.test_gpt2_float64 import guarded
    return guarded(K, n, dt)


SUMMARY = {}


def _to_T_bits(K, a, dt):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(K.TORCH_DT[dt]).view(_int_dt(dt)).numpy()


def check_round(K, name, c, k, world, m, order, stats):
    """one round of case c: inputs of seed (name, k), launch, every check; returns failure messages"""
    import torch
    from tests.test_gpt2_float64 import GUARD_BITS, guard_ok
    dt, W, H = c["dt"], c["W"], c["H"]
    what = f"{name} round {k} (M {m}, order {order})"
    P, R, w = ar64.inputs(dt, W, m, H, c["regime"], seed_of(name, k), c["res"], c["norm"])
    P_dev = K.dev(P, dt)
    R_dev = K.dev(R, dt) if R is not None else None
    w_dev = K.dev(w, dt) if w is not None else None
    n = m * H
    bufs = [(_guarded(K, n, dt), _guarded(K, n, dt) if w is not None else None) for _ in range(W)]
    outs = [(b[0][1], b[1][1] if b[1] is not None else None) for b in bufs]
    fails = [f"{what}: {f}" for f in world.round(P_dev, R_dev, w_dev, outs, m, H, dt, order)]
    for r, (ob, nb) in enumerate(bufs):
        for buf, nm in ((ob, "out"), (nb, "out_norm")):
            if buf is not None and not guard_ok(buf[0], n, dt):
                fails.append(f"{what}: rank {r} wrote past the end of {nm}")
    got = [(_bits(o, dt).reshape(m, H), _bits(y, dt).reshape(m, H) if y is not None else None) for o, y in outs]
    for r in range(1, W):
        for j, nm in ((0, "out"), (1, "out_norm")):
            if got[r][j] is not None and not np.array_equal(got[r][j], got[0][j]):
                i, col = np.argwhere(got[r][j] != got[0][j])[0]
                fails.append(f"{what}: rank {r}'s {nm} differs from rank 0's at {ar64.describe(dt, H, i, col)}")
    out = outs[0][0].float().cpu().numpy().reshape(m, H)
    emu, _ = ar64.emulate(P, R, w, dt)
    want = _to_T_bits(K, emu, dt).reshape(m, H)
    if not np.array_equal(got[0][0], want):
        bad = got[0][0] != want
        i, col = np.argwhere(bad)[0]
        fails.append(f"{what}: out differs from the fp32 emulation in {int(bad.sum())} elements; first at "
                     f"{ar64.describe(dt, H, i, col)}: got {out[i, col]!r}, emulated {emu[i, col]!r}")
        stats["out_bit_exact"] = False
    Ro = ar64.out_ref(P, R, dt)
    stats["out"] = max(stats.get("out", 0.0), Ro.ratio(out))
    msg = ar64.report(Ro.violations(out), out, Ro, f"{what}: out", dt, H)
    fails += [msg] if msg else []
    if w is not None:
        y = outs[0][1].float().cpu().numpy().reshape(m, H)
        fin, bad, r = norm_check(out, y, w, dt)
        stats["out_norm"] = max(stats.get("out_norm", 0.0), r)
        if bad.any():
            rows = np.flatnonzero(fin)
            i, col = np.argwhere(bad)[0]
            fails.append(f"{what}: out_norm outside the interval / bound in {int(bad.sum())} elements; first at "
                         f"{ar64.describe(dt, H, rows[i], col)}: got {y[rows[i], col]!r}")
        ident = True
        for fn in ("it_b200_rmsnorm", "it_b200_rmsnorm_constw"):
            yr = torch.empty_like(outs[0][0])
            K.L.check(getattr(K.L.lib, fn)(dt, K.ptr(outs[0][0]), K.ptr(w_dev), K.ptr(yr), m, H, K.stream()))
            K.sync()
            rb = _bits(yr, dt).reshape(m, H)
            same = np.array_equal(rb[fin], got[0][1][fin])
            ident &= same
            if not same and ar64.partitions_coincide(dt, H):
                bad = (rb != got[0][1]) & fin[:, None]
                i, col = np.argwhere(bad)[0]
                fails.append(f"{what}: out_norm differs from {fn} of the same out where the partitions coincide, in "
                             f"{int(bad.sum())} elements; first at {ar64.describe(dt, H, i, col)}")
        stats.setdefault("rmsnorm_identical", True)
        stats["rmsnorm_identical"] &= bool(ident)
    return fails


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_allreduce_float64(K, name):
    c = spec(name)
    t0 = time.time()
    world = ar64.World(c["W"], c["epochs"])
    stats = {"out_bit_exact": True}
    fails = []
    for k, (m, order) in enumerate(plan(c)):
        fails += check_round(K, name, c, k, world, m, order, stats)
        if fails:
            break           # the workspaces no longer match the model: a later round could poll for a tag never staged
    if not fails:
        world.check_epochs()
    stats = {k: (round(v, 4) if isinstance(v, float) else v) for k, v in stats.items()}
    stats |= {"coincide": ar64.partitions_coincide(c["dt"], c["H"]), "rounds": world.rounds, "wall_s": round(time.time() - t0, 2)}
    SUMMARY[name] = stats
    print(f"\n{name}: {stats}")
    assert not fails, "\n".join(fails)


# ====================================================================== GPU: through the graph at world 1
def _graph(monkeypatch, dt, M, H, add_order, mask=None, nccl=False):
    """(handler, tensors, schedule) of AllReduceSum -> Add -> RMSNorm(weight) on a world-1 runtime"""
    from infinitensor_b200 import backend as B
    if mask is None:
        monkeypatch.delenv("ITB_FUSION_MASK", raising=False)
    else:
        monkeypatch.setenv("ITB_FUSION_MASK", str(mask))
    rt = B.CudaRuntime(0)
    if nccl:
        rt.init_comm_with_id(B.CudaRuntime.nccl_unique_id(), 1, 0)
    else:
        rt.p2p_import([rt.p2p_export()], 1, 0)
    h = B.GraphHandler(rt)
    x, r, w = h.tensor([M, H], dt), h.tensor([M, H], dt), h.tensor([H], dt)
    x.set_input()
    r.set_input()
    w.set_weight()
    a = h.allReduceSum(x, None)
    s = h.add(a, r, None) if add_order == 0 else h.add(r, a, None)
    y = h.RMSNorm(s, w, None)
    s.set_output()
    y.set_output()
    sched = h.schedule()
    h.data_malloc()
    return rt, h, (x, r, w, s, y), sched


def _graph_steps(h, T, dt, M, H, seed, steps, replay):
    """run `steps` steps with new inputs each; returns the failures and the raw outputs of the last step"""
    from infinitensor_b200 import graphs as G
    x, r, w, s, y = T
    fails, last = [], None
    _, _, wv = ar64.inputs(dt, 1, 1, H, "normal", seed, True, True)
    w.copyin_numpy(G.to_storage(wv, dt))
    for k in range(steps):
        P, R, _ = ar64.inputs(dt, 1, M, H, "normal", seed + 1 + k, True, False)
        x.copyin_numpy(G.to_storage(P[0], dt))
        r.copyin_numpy(G.to_storage(R, dt))
        h.run_with_cudagraph() if replay else h.run()
        so = G.from_storage(s.copyout_numpy(), dt).astype(np.float32)
        yo = G.from_storage(y.copyout_numpy(), dt).astype(np.float32)
        emu, _ = ar64.emulate(P, R, wv, dt)
        if not np.array_equal(so.view(np.int32), emu.view(np.int32)):
            fails.append(f"step {k} ({'replay' if replay else 'eager'}): the Add output differs from the emulation")
        _, bad, _ = norm_check(so, yo, wv, dt)
        if bad.any():
            fails.append(f"step {k} ({'replay' if replay else 'eager'}): the RMSNorm output leaves the bound")
        last = (s.copyout_numpy(), y.copyout_numpy())
    return fails, last


@pytest.mark.gpu
@pytest.mark.parametrize("dt,H", [(BF16, 4096), (F16, 3072), (F32, 2048)], ids=["bf16_4096", "f16_3072", "fp32_2048"])
@pytest.mark.parametrize("add_order", [0, 1], ids=["ar_plus_res", "res_plus_ar"])
def test_graph_fused_world1(K, monkeypatch, dt, H, add_order):
    M = 16
    rt, h, T, sched = _graph(monkeypatch, dt, M, H, add_order)
    assert "AllReduceAddNorm:AllReduceSum+Add+RMSNorm" in sched, sched
    fails, _ = _graph_steps(h, T, dt, M, H, 50 + add_order, 3, replay=False)
    f2, _ = _graph_steps(h, T, dt, M, H, 60 + add_order, 4, replay=True)        # capture, then three replays
    assert rt.cuda_graph_capture_count() >= 1
    assert not fails + f2, "\n".join(fails + f2)


@pytest.mark.gpu
@pytest.mark.parametrize("dt,H", [(BF16, 4096), (F32, 2048)], ids=["bf16_4096", "fp32_2048"])
def test_graph_fallback_world1(K, monkeypatch, dt, H):
    """the three separate operators (one-rank NCCL AllReduceSum, Add, RMSNorm): at M = 65 (too many rows for the fused
    kernel) against the references, and with bit 4 of ITB_FUSION_MASK off at M = 16, bit for bit equal to the fused step
    where the partitions coincide"""
    from infinitensor_b200 import backend as B
    try:
        rt0 = B.CudaRuntime(0)
        rt0.init_comm_with_id(B.CudaRuntime.nccl_unique_id(), 1, 0)
        del rt0
    except Exception as e:  # noqa: BLE001 -- reported as the skip reason
        pytest.skip(f"no one-rank NCCL communicator: {e}")
    _, h, T, _ = _graph(monkeypatch, dt, 65, H, 0, nccl=True)
    fails, _ =_graph_steps(h, T, dt, 65, H, 70, 2, replay=False)
    default = 127 | 256 | 512 | 1024 | 2048
    _, h1, T1, s1 = _graph(monkeypatch, dt, 16, H, 0, mask=default & ~16, nccl=True)
    assert not any(s.startswith("AllReduceAddNorm") for s in s1), s1
    f1, sep = _graph_steps(h1, T1, dt, 16, H, 80, 1, replay=False)
    _, h2, T2, s2 = _graph(monkeypatch, dt, 16, H, 0)
    assert "AllReduceAddNorm:AllReduceSum+Add+RMSNorm" in s2, s2
    f2, fused = _graph_steps(h2, T2, dt, 16, H, 80, 1, replay=False)
    fails += f1 + f2
    assert np.array_equal(sep[0], fused[0]), "the Add output differs between the separate operators and the fused step"
    if ar64.partitions_coincide(dt, H):
        assert np.array_equal(sep[1], fused[1]), "RMSNorm differs between the separate operators and the fused step"
    assert not fails, "\n".join(fails)


# ====================================================================== GPU: real ranks (torchrun, >= 2 devices)
def _ngpu():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 4, 8])
def test_allreduce_real_ranks(tmp_path, world):
    if _ngpu() < max(world, 2):
        pytest.skip(f"needs {world} GPUs, the box has {_ngpu()}")
    out = str(tmp_path / "ar")
    env = dict(os.environ, AR_OUT=out, MASTER_ADDR="127.0.0.1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr",
           "127.0.0.1", "--master-port", str(29630 + world), os.path.join(ROOT, "tools", "ar_worker.py")]
    subprocess.run(cmd, check=True, env=env, cwd=ROOT, timeout=900)
    res = [json.load(open(f"{out}.{r}.json")) for r in range(world)]
    fails = [f for rr in res for f in rr["fails"]]
    for c in res[0]["cases"]:
        assert c["steps"] >= 100 and "AllReduceAddNorm:AllReduceSum+Add+RMSNorm" in c["schedule"], c
    digests = [[c["digest"] for c in rr["cases"]] for rr in res]
    assert all(d == digests[0] for d in digests), "the ranks' outputs differ"
    assert not fails, "\n".join(fails[:20])


# ====================================================================== GPU: the intended kernels ran
def profiled_kernel_names():
    import torch
    from tests import kernel_harness as K
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for dt, H in ((F32, 2048), (F16, 4096), (BF16, 264), (BF16, 4096)):
            world = ar64.World(2)
            P, R, w = ar64.inputs(dt, 2, 2, H, "normal", 3)
            outs = [(K.dev(np.zeros((2, H), np.float32), dt), K.dev(np.zeros((2, H), np.float32), dt)) for _ in range(2)]
            world.round(K.dev(P, dt), K.dev(R, dt), K.dev(w, dt), outs, 2, H, dt, [0, 1])
            for cw in (False, True):
                K.rms_norm(outs[0][0].float().cpu().numpy(), w, dt, cw)
        x = np.ones((2, 5120), np.float32)
        K.rms_norm(x, np.ones(5120, np.float32), BF16)
        torch.cuda.synchronize()
    return sorted({e.name for e in prof.events() if "CUDA" in str(e.device_type)})


@pytest.mark.gpu
def test_allreduce_cases_reach_the_intended_kernels():
    """in a child process, as the other float64 files do: a profiler session in the test process loses records of later ones"""
    code = "import json; from tests.test_allreduce_float64 import profiled_kernel_names as f; print(json.dumps(f()))"
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    names = set(json.loads(r.stdout.strip().splitlines()[-1]))
    if not names:
        pytest.skip("the profiler recorded no CUDA kernel events (CUPTI activity tracing unavailable)")
    want = [r"allreduce_ll_kernel<float>", r"allreduce_ll_kernel<__half>", r"allreduce_ll_kernel<__nv_bfloat16>",
            r"rmsnorm_kernel<.*true, true>", r"rmsnorm_kernel<.*true, false>", r"rmsnorm_kernel<.*false, false>"]
    missing = [p for p in want if not any(re.search(p, nm) for nm in names)]
    assert not missing, f"not launched: {missing}; kernels seen: {sorted(names)}"
