"""Float64 references, a float32 emulation and a one-device harness for the tensor-parallel all-reduce + residual + RMSNorm
kernel (`allreduce_ll_kernel`, allreduce.cu).

The kernel, CTA `row` of rank r, epoch e = epoch[row] of r's own workspace, tag = e + 1 (uint32), parity b = e & 1:
  (1) pushes vector i (16 bytes, words x y z w) of its partial row into slot (b, r, row) of EVERY rank's workspace (its own
      included) as the two LL packets 2i = {x, tag, y, tag} and 2i + 1 = {z, tag, w, tag}: the slot is the row's words
      interleaved with the tag;
  (2) polls slots (b, p, row), p < world, of its own workspace until every tag reads e + 1;
  (3) acc = 0.0f + p_0 + p_1 + ... in rank order (fp32), x = round_t(acc), with a residual x = round_t(r + x); stores x;
  (4) with a norm weight: rinv = rsqrtf(block_sum(ss) / H + 1e-5f), ss the per-thread sums of x^2 over the thread's vectors;
      out_norm = round_t(round_t(x rinv) w);
  (5) epoch[row] = e + 1.

Bounds (u = 2^-24).  The library is built without fast-math, so the fp32 emulation below gives `out` bit for bit.  Against
float64, out = rnd_T(rnd_T(sum p) + r): each rounding to T within ulp_T of its exact value (a whole ulp covers a rounding
that crosses a binade), plus the fp32 chain of W - 1 additions, each within u of a partial sum no larger than sum |p|:
    |out - (sum p + r)| <= (W - 1) u sum|p| + ulp_T(sum p) [+ ulp_T(sum p + r)]
out_norm is held to operand64.rmsnorm_operand's interval from the kernel's own `out` (rinv's fp32 window for a chain of
`items + 10` roundings: the thread's items, then block_sum's two 5-level warp trees), and to a ratio bound `norm_bound`.

Work partition.  The fused kernel runs threads = min(512, roundup32(nv)) per row (nv = H / V vectors of 16 bytes, V = 16 /
sizeof(T)); thread t owns vectors t, t + threads, ...  rmsnorm_kernel (norm.cu) runs 512 threads from H >= 4096, 256 from
H >= 1024, else 128, with the same ownership rule.  The per-thread vector lists, and so every fp32 sum of squares and rinv,
coincide when nv <= both thread counts or the counts are equal; there out_norm must equal it_b200_rmsnorm of `out` bit
for bit (`partitions_coincide`).
"""
import numpy as np

from tests import operand64, ref64
from tests.gpt2_64 import rnd
from tests.ref64 import BF16, F16, F32

U = 2.0 ** -24

# ====================================================================== workspace layout (allreduce.cu)
MAX_WORLD, MAX_ROWS, MAX_ROW_BYTES = 8, 64, 16384
SLOT_BYTES = 2 * MAX_ROW_BYTES                    # LL packets double the row
EPOCH_OFF, FLAGS_OFF = 0, 1024
DATA_OFF = 1024 + 2 * MAX_ROWS * MAX_WORLD * 4
WS_BYTES = DATA_OFF + 2 * MAX_WORLD * MAX_ROWS * SLOT_BYTES
ESIZE = {F32: 4, F16: 2, BF16: 2}
NAMES = {F32: "fp32", F16: "f16", BF16: "bf16"}


def slot_offset(b, rank, row):
    return DATA_OFF + ((b * MAX_WORLD + rank) * MAX_ROWS + row) * SLOT_BYTES


def vec(dt):
    return 16 // ESIZE[dt]


def nvec(dt, H):
    return H // vec(dt)


# ====================================================================== launch rules
def ar_threads(dt, H):
    """it_b200_allreduce_fused: min(512, max(32, roundup32(nv)))"""
    return min(512, max(32, -(-nvec(dt, H) // 32) * 32))


def rms_threads(H):
    """rmsnorm_impl (norm.cu)"""
    return 512 if H >= 4096 else 256 if H >= 1024 else 128


def ar_items(dt, H):
    """elements of the row one thread of the fused kernel squares and adds"""
    return -(-nvec(dt, H) // ar_threads(dt, H)) * vec(dt)


def partitions_coincide(dt, H):
    """vector i belongs to thread i mod threads in both kernels: the same lists iff nv fits both or the counts agree"""
    nv, ta, tr = nvec(dt, H), ar_threads(dt, H), rms_threads(H)
    return nv <= min(ta, tr) or ta == tr


def owner(dt, H, i):
    """(thread, pass) of vector i in the fused kernel"""
    t = ar_threads(dt, H)
    return i % t, i // t


# ====================================================================== float32 emulation
def _f(x):
    return np.asarray(x, np.float64).astype(np.float32)


def _r(x, dt):
    return rnd(np.asarray(x, np.float32).astype(np.float64), dt).astype(np.float32)


MUTATIONS = ["accumulate_in_T", "reversed_rank_order", "residual_before_round", "drop_last_rank", "drop_tail_vector",
             "rinv_pre_residual", "normw_shift_vector", "rinv_neighbour_row", "eps_omitted"]
OUT_MUTATIONS = MUTATIONS[:5]


def _block_sum(ss, threads):
    """block_sum over [rows, threads] per-thread sums: warp butterflies, then one over the warp sums (zero-padded to 32)"""
    m = ss.shape[0]
    nw = -(-threads // 32)
    warps = operand64._xor_tree(ss.reshape(m, nw, 32), 5)
    red = np.zeros((m, 32), np.float32)
    red[:, :nw] = warps
    return operand64._xor_tree(red, 5)


def emu_rinv(x, dt, eps=True):
    """the fused kernel's rinv of the rows x [M, H] (float32, exact in T): per-thread sums in the kernel's order"""
    m, H = x.shape
    V, nv, T = vec(dt), nvec(dt, H), ar_threads(dt, H)
    passes = -(-nv // T)
    xs = np.zeros((m, passes * T * V), np.float32)
    xs[:, :H] = x
    xs = xs.reshape(m, passes, T, V)
    ss = np.zeros((m, T), np.float32)
    for it in range(passes):
        for j in range(V):
            f = xs[:, it, :, j].astype(np.float64)
            ss = _f(ss.astype(np.float64) + f * f)     # fmaf: the product is exact in float64
    tot = _block_sum(ss, T)
    with np.errstate(divide="ignore", over="ignore"):
        return _f(1.0 / np.sqrt(_f(_f(tot / np.float32(H)) + (np.float32(1e-5) if eps else np.float32(0))).astype(np.float64)))


def emulate(P, R, w, dt, mutation=None):
    """(out, out_norm or None) as float32 [M, H] from the partials P [W, M, H], residual R [M, H] or None, weight w [H] or None"""
    P = np.asarray(P, np.float32)
    W, M, H = P.shape
    ranks = list(range(W))
    if mutation == "reversed_rank_order":
        ranks = ranks[::-1]
    if mutation == "drop_last_rank":
        ranks = ranks[:-1]
    acc = np.zeros((M, H), np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        for p in ranks:
            acc = _f(acc.astype(np.float64) + P[p])
            if mutation == "accumulate_in_T":
                acc = _r(acc, dt)
        pre = _r(acc, dt)
        if R is None:
            x = pre
        elif mutation == "residual_before_round":
            x = _r(_f(np.asarray(R, np.float64) + acc), dt)
        else:
            x = _r(_f(np.asarray(R, np.float64) + pre), dt)
        if mutation == "drop_tail_vector":
            nv, T, V = nvec(dt, H), ar_threads(dt, H), vec(dt)
            if nv % T:
                x = x.copy()
                x[:, (nv // T) * T * V:] = np.nan
        if w is None:
            return x, None
        rinv = emu_rinv(pre if mutation == "rinv_pre_residual" else x, dt, eps=mutation != "eps_omitted")
        if mutation == "rinv_neighbour_row":
            rinv = np.roll(rinv, -1)
        ww = np.asarray(w, np.float32)
        if mutation == "normw_shift_vector":
            ww = np.concatenate([ww[vec(dt):], ww[:vec(dt)]])
        y = _r(_f(_r(_f(x.astype(np.float64) * rinv[:, None]), dt).astype(np.float64) * ww), dt)
    return x, y


# ====================================================================== float64 references
class Ref:
    """reference and bound of one output; non-finite references must be matched exactly"""

    def __init__(self, ref, bound, exact):
        self.ref, self.bound, self.exact = ref, bound, exact

    def violations(self, got, scale=1.0):
        got = np.asarray(got, np.float64)
        fin = np.isfinite(self.exact)
        with np.errstate(invalid="ignore"):
            ok = np.where(fin, np.abs(got - self.ref) <= scale * self.bound, got == self.exact)
        return ~ok

    def ratio(self, got):
        got = np.asarray(got, np.float64)
        fin = np.isfinite(self.exact)
        with np.errstate(invalid="ignore"):
            r = np.where(fin, np.abs(got - self.ref) / self.bound, np.where(got == self.exact, 0.0, np.inf))
        r = np.where(np.isnan(r), np.inf, r)
        return float(r.max()) if r.size else 0.0


def out_ref(P, R, dt):
    P = np.asarray(P, np.float64)
    W = P.shape[0]
    s, mag = P.sum(0), np.abs(P).sum(0)
    ref = s if R is None else s + np.asarray(R, np.float64)
    bound = (W - 1) * U * mag + ref64.ulp(s, dt)
    with np.errstate(invalid="ignore", over="ignore"):
        chain = rnd(s, dt) if R is None else rnd(rnd(s, dt) + np.asarray(R, np.float64), dt)
        if R is not None:
            bound = bound + ref64.ulp(ref, dt)
    return Ref(ref, bound, chain)


def norm_chain(dt, H):
    return operand64.chain_length("block", H, items=ar_items(dt, H))


def norm_operand(out, w, dt):
    """operand64's interval operand of rnd(rnd(out rinv) w) for the fused kernel's chain"""
    return operand64.rmsnorm_operand(out, w, dt, norm_chain(dt, out.shape[1]))


def norm_bound(out, w, dt):
    """ref = out rinv w in float64; bound: the two roundings (whole ulps) and rinv's fp32 window carried through w"""
    x, w = np.asarray(out, np.float64), np.asarray(w, np.float64)[None, :]
    y = x * operand64.rinv64(x)
    ref = y * w
    bound = ref64.ulp(ref, dt) + np.abs(w) * (ref64.ulp(y, dt) + operand64.rms_window(norm_chain(dt, x.shape[1])) * np.abs(y))
    return Ref(ref, bound, ref)


# ====================================================================== inputs
REGIMES = ["normal", "cancel", "spread", "residual_dominates", "overflow", "subnormal", "zero_rows", "huge_element"]


def inputs(dt, W, M, H, regime, seed, residual=True, norm=True):
    """(P [W, M, H], R [M, H] or None, w [H] or None) as float32, every value exact in T"""
    rng = np.random.default_rng(seed)
    rs = ref64.row_scale(M)[None, :, None].astype(np.float64)
    g = lambda *s: rng.standard_normal(s)
    P = g(W, M, H) * rs
    R = g(M, H) * ref64.row_scale(M)[:, None] if residual else None
    if regime == "cancel" and W >= 2:
        P[1] = -P[0] + g(M, H) * rs[0] * 2.0 ** -12     # p0 + p1 cancels all but the last few bits
        P[2:] *= 2.0 ** -10
    elif regime == "spread":
        lim = 10 if dt == F16 else 24
        P *= np.exp2(rng.integers(-lim, lim + 1, size=P.shape))
    elif regime == "residual_dominates" and R is not None:
        R *= 2.0 ** 12
    elif regime == "overflow" and dt == F16:
        # sums of same-signed ranks leave f16's range on about a third of the elements; the partials stay finite
        sgn = np.sign(g(1, M, H))
        big = rng.uniform(0.5, 1.0, (1, M, H)) < 0.35
        P = np.where(big, sgn * 60000.0 / max(W - 1, 1) * rng.uniform(0.9, 1.0, (W, M, H)), P)
    elif regime == "subnormal":
        tiny = {F16: 2.0 ** -20, BF16: 2.0 ** -130, F32: 2.0 ** -140}[dt]
        P = g(W, M, H) * tiny
        if R is not None:
            R = g(M, H) * tiny
    elif regime == "zero_rows":
        z = (np.arange(M) % 3) == 0
        P[:, z] = 0.0
        if R is not None:
            R[z] = 0.0
    elif regime == "huge_element":
        huge = {F16: 30000.0, BF16: 2.0 ** 56, F32: 2.0 ** 56}[dt]
        col = rng.integers(0, H, M)
        P[rng.integers(0, W), np.arange(M), col] = huge
    P = rnd(P, dt).astype(np.float32)
    R = None if R is None else rnd(R, dt).astype(np.float32)
    w = operand64.norm_weight(H, dt, seed + 7).astype(np.float32) if norm else None
    return P, R, w


def order_sensitive(P):
    """elements whose fp32 rank-order sum differs from the reverse-order one"""
    P = np.asarray(P, np.float32)
    fwd, rev = np.zeros(P.shape[1:], np.float32), np.zeros(P.shape[1:], np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        for p in range(P.shape[0]):
            fwd = _f(fwd.astype(np.float64) + P[p])
            rev = _f(rev.astype(np.float64) + P[-1 - p])
    return int((fwd != rev).sum())


def describe(dt, H, row, col):
    """rank-independent location of element (row, col): row, vector, owning thread and pass"""
    i = col // vec(dt)
    t, k = owner(dt, H, i)
    return f"row {row}, vector {i} (thread {t}, pass {k}), element {col}"


def report(bad, got, R, what, dt, H, limit=4):
    if not bad.any():
        return None
    got = np.asarray(got, np.float64)
    idx = np.argwhere(bad)
    lines = [f"{what}: {int(bad.sum())} of {bad.size} elements outside the bound"]
    for i, j in idx[:limit]:
        lines.append(f"  {describe(dt, H, i, j)}: got {got[i, j]!r}, float64 {R.ref[i, j]!r}, bound {R.bound[i, j]:.3g}")
    return "\n".join(lines)


# ====================================================================== the one-device harness (torch, on the GPU)
NAN_WORD = 0x7FFF7FFF   # NaN as fp32 and as each 16-bit half, f16 and bf16 alike
EPOCH_PAD, FLAGS_FILL = 0x5A5A5A5A, 0x13579BDF


def i32(v):
    """uint32 -> the int32 with the same bits"""
    v = int(v) & 0xFFFFFFFF
    return v - (1 << 32) if v >= (1 << 31) else v


class World:
    """W comm workspaces on one device, each laid out as allreduce.cu lays it out, and the epoch model"""

    def __init__(self, W, epochs=0):
        import torch
        from infinitensor_b200 import _lib as L
        assert int(L.lib.it_b200_allreduce_workspace_bytes()) == WS_BYTES
        self.W = W
        self.ws = [torch.empty(WS_BYTES // 4, dtype=torch.int32, device="cuda") for _ in range(W)]
        self.epoch = np.broadcast_to(np.asarray(epochs, np.int64) & 0xFFFFFFFF, (MAX_ROWS,)).copy()   # as uint32
        for w in self.ws:
            w[:FLAGS_OFF // 4].fill_(EPOCH_PAD)
            w[FLAGS_OFF // 4:DATA_OFF // 4].fill_(FLAGS_FILL)
            w[:MAX_ROWS].copy_(torch.tensor([i32(e) for e in self.epoch], dtype=torch.int32))
        self.flag = torch.zeros(1, dtype=torch.int32).pin_memory()
        self.rounds = 0

    def data(self, q):
        return self.ws[q][DATA_OFF // 4:].view(2, MAX_WORLD, MAX_ROWS, SLOT_BYTES // 4)

    def check_epochs(self):
        """every workspace's epoch array against the model (the next round's tags come from it)"""
        want = np.array([i32(e) for e in self.epoch], np.int64)
        for q in range(self.W):
            got = self.ws[q][:MAX_ROWS].cpu().numpy().astype(np.int64)
            if not np.array_equal(got, want):
                rows = np.flatnonzero(got != want)[:8].tolist()
                raise AssertionError(f"round {self.rounds}: rank {q}'s epoch[{rows}] = {got[rows].tolist()}, model "
                                     f"{want[rows].tolist()}; the sequence stops here (a wrong tag would make the next round poll)")

    def packets(self, P_dev, M):
        """[W, M, 8 nv] int32: each rank's rows as LL packets with the tag of their row"""
        import torch
        words = P_dev.contiguous().view(torch.int32).view(self.W, M, -1)          # [W, M, 4 nv]
        tag = torch.tensor([i32(self.epoch[r] + 1) for r in range(M)], dtype=torch.int32, device="cuda")
        return torch.stack([words, tag[None, :, None].expand_as(words)], -1).reshape(self.W, M, -1)

    def round(self, P_dev, R_dev, w_dev, outs, M, H, dt, order):
        """poison, stage, launch the W ranks in `order` on one stream; returns the list of failure messages"""
        import ctypes
        import torch
        from infinitensor_b200 import _lib as L
        from tests import kernel_harness as K
        self.check_epochs()
        W, nv = self.W, nvec(dt, H)
        pk = self.packets(P_dev, M)
        b = torch.tensor([int(self.epoch[r] & 1) for r in range(M)], dtype=torch.long, device="cuda")
        rows = torch.arange(M, device="cuda")
        tags_all = torch.tensor([i32(e + 1) for e in self.epoch], dtype=torch.int32, device="cuda")
        pos = {r: k for k, r in enumerate(order)}
        expect = []
        for q in range(W):
            d = self.data(q).view(2, MAX_WORLD, MAX_ROWS, SLOT_BYTES // 8, 2)
            d[..., 0] = NAN_WORD                              # every slot: NaN payload carrying the tag the row looks for
            d[..., 1] = tags_all[None, None, :, None]
            dq = self.data(q)
            for p in range(W):
                if pos[p] > pos[q]:                           # launched later: its packets are staged
                    dq[b, p, rows, :8 * nv] = pk[p]
            e = self.ws[q].clone()
            ed = e[DATA_OFF // 4:].view(2, MAX_WORLD, MAX_ROWS, SLOT_BYTES // 4)
            for p in range(W):
                ed[b, p, rows, :8 * nv] = pk[p]
            e[:M] = torch.tensor([i32(self.epoch[r] + 1) for r in range(M)], dtype=torch.int32, device="cuda")
            expect.append(e)
        before = [t.clone() for t in (P_dev, R_dev, w_dev) if t is not None]
        VP = ctypes.c_void_p
        peers = (VP * W)(*[t.data_ptr() for t in self.ws])
        self.flag.zero_()
        for r in order:
            L.check(L.lib.it_b200_allreduce_fused(dt, VP(P_dev[r].data_ptr()), K.ptr(R_dev), K.ptr(w_dev), VP(outs[r][0].data_ptr()),
                                                  VP(outs[r][1].data_ptr()) if outs[r][1] is not None else None, M, H, peers, W, r,
                                                  VP(self.flag.data_ptr()), K.stream()))
        K.sync()
        fails = []
        if int(self.flag[0]):
            code = int(self.flag[0]) - 1
            fails.append(f"round {self.rounds}: timeout flag raised: rank {code // 16} never saw rank {code % 16}'s packets")
        for q in range(W):
            if not torch.equal(self.ws[q], expect[q]):
                fails.append(self.diff(q, expect[q], dt, H))
        for t0, t in zip(before, [t for t in (P_dev, R_dev, w_dev) if t is not None]):
            if not torch.equal(t0.view(torch.int16 if t.element_size() == 2 else torch.int32),
                               t.view(torch.int16 if t.element_size() == 2 else torch.int32)):
                fails.append(f"round {self.rounds}: an input (in, residual or norm_w) changed")
        for r in range(M):
            self.epoch[r] = (self.epoch[r] + 1) & 0xFFFFFFFF
        self.rounds += 1
        return fails

    def diff(self, q, expect, dt, H):
        got, e = self.ws[q], expect
        bad = (got != e).nonzero().flatten()
        n = int(bad.numel())
        w = int(bad[0]) * 4
        if w < FLAGS_OFF:
            where = f"epoch word {w // 4}" if w // 4 < MAX_ROWS else f"epoch padding word {w // 4}"
        elif w < DATA_OFF:
            where = f"flags word {(w - FLAGS_OFF) // 4}"
        else:
            o = w - DATA_OFF
            slot, within = divmod(o, SLOT_BYTES)
            bb, rest = divmod(slot, MAX_WORLD * MAX_ROWS)
            p, row = divmod(rest, MAX_ROWS)
            i = within // 32
            t, k = owner(dt, H, i) if i < nvec(dt, H) else (None, None)
            where = (f"slot (parity {bb}, rank {p}, row {row}), packet byte {within} = vector {i}"
                     + (f" (thread {t}, pass {k})" if t is not None else " (past the row)"))
        return (f"round {self.rounds}: rank {q}'s workspace differs from the model in {n} words; first at byte {w}: {where}: "
                f"got {int(got[w // 4]) & 0xFFFFFFFF:#010x}, want {int(e[w // 4]) & 0xFFFFFFFF:#010x}")
