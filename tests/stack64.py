"""Float64 references, per-element bounds, work-dealing model and float32 emulation of the persistent decode kernel
(`decode_stack_kernel`, decode_stack.cu), phase by phase.

The stack writes every intermediate of the operator graph (q, k, v before RoPE, attn_out, x_mid, gate, up, x_out) and appends
one row to each cache, so each phase of each layer is checked from the GPU's own inputs to that phase.  Those inputs are
exact in T, so they are exact in float64, errors do not compound across layers and every phase gets its own tight bound.
rnd (gpt2_64.rnd: prefill64.rnd for f16 / bf16) rounds float64 straight to T; u = 2^-24.

* RMSNorm -> GEMM (q/k/v, gate/up).  xn = rnd(rnd(x rinv) w), rinv = 1 / sqrt(mean(x^2) + fp32(1e-5)), out_g = xn . W_g.
  Bound: ref64's ulp_T(|ref|) + 2^-16 S (S = |xn| . |W|) plus AMB_MARGIN sum_{ambiguous k} |c_hi - c_lo| |W_kn|.
* Silu.Mul -> GEMM + residual (down).  m = rnd(rnd(silu(gate)) up); x_out = x_mid + m . Wd, bounded as gpt2_64 bounds its
  residual epilogue: 2^-16 S + ulp_T(m . Wd) (the product rounded to T before the add) + ulp_T(|ref|) + the ambiguity term.
* o-proj + residual.  x_mid = x + attn_out . Wo, the same bound without an ambiguity term (no operand transform).
* RoPE + attention: tests/attn64.py's reference and bound (gqa=False) on q and the appended k rotated by it_b200_rope.  The
  stack's score chain is attn_stream_kernel's: q is scaled by fp32(1/sqrt(128)) (2 roundings), each lane chains 8 products
  in fmaf (EPL = 8 for 2-byte T) and a 4-level xor shuffle tree sums the row's 16 lanes (LPR = 16): 2 + 8 + 4 = 14 roundings
  of partial sums no larger than a_j = sum |q_i k_ji| / sqrt(128), within attn64's C_SCORE = 32.  The online softmax, the
  sub-row / warp folds and the ticket merge of CTA partials follow attn_stream_kernel step for step; only the dealing
  differs (min(units, SMs) CTAs instead of 264), which changes how many partials a head's merge adds, not the error per add.

Ambiguous roundings.  rinv and silu come from fp32 arithmetic, so an element whose exact value lies within the fp32 error
window of a T rounding midpoint may round either way.  As prefill64 does, each path gets a relative window and the element
is ambiguous where rnd at the two ends of the window differ; c_lo / c_hi are the transformed operand at those ends.

* rinv: the sum of squares is a chain of L roundings of a positive sum (relative error <= L u), then the division by K and
  the eps add (1 u each), rsqrtf (<= 2 ulp, 4 u) and the product x * rinv (1 u): |error| <= (L / 2 + 7) u; the window is
  (L + 8) u.  L per path (`chain_length`):
    - the first layer reduces x_raw itself: K / 32 fmaf per lane, then a 5-level warp tree: K / 32 + 5 (also a chain phase
      with no producer phase);
    - the ss hand-over: the epilogue's f * f (1), its warp tree (5), the sum of the 4 quads (3); the next phase's 8 lanes per
      row sum every 8th of the nt tiles (ceil(nt / 8)) and a 3-level xor tree: 12 + ceil(nt / 8);
    - the standalone rmsnorm_kernel's block_sum: the items of one thread, then two 5-level warp trees: items + 10.
* silu(g) = g / (1 + expf(-g)): expf <= 2 ulp (4 u relative to exp(-g)), the add <= 4 u + 1 u relative to 1 + exp(-g), the
  division 1 u: <= 6 u; the window is 8 u.
* The second rounding adds no ambiguity: rnd(x rinv) w and rnd(silu) up are products of two T values, 8 x 8 (bf16) or
  11 x 11 (f16) significant bits, exact in fp32's 24, so rnd of them is rnd of an exact value.
* The ambiguity term is what taking the other side costs, counted twice (AMB_MARGIN, as prefill64) so that an emulation
  flipping some of them is still held to half of the bound.

What the bound cannot see.  silu left unrounded before the multiply changes each m_k by at most half an ulp of silu, of random
sign: at K = 11008 that moves an output by about 2^-9 sqrt(K) rms(m W), the same order as the 2^-16 S accumulation allowance
(2^-16 K mean|m W|), so whether it fails depends on the data, and no test relies on it.

The float32 emulation below follows the kernel's arithmetic (the transforms, fp32 partials per k16 step of each k chunk, the
split partials summed in split order by the ticket finisher, the epilogue roundings, the per-tile sums of squares in the
kernel's order, rinv from them) and stays within half of the bound (test_decode_stack_float64.py checks it).
"""
import numpy as np

from tests import attn64, ref64
from tests.gpt2_64 import rnd
from tests.prefill64 import AMB_MARGIN
from tests.ref64 import BF16, F16

U = 2.0 ** -24
EPS32 = float(np.float32(1e-5))   # the kernels' 0.00001f
SILU_WINDOW = 8 * U
NUM_SMS = 132
NORMW_MAX = 4096                  # DS_NORMW_MAX: a longer norm weight is read from global memory


# ====================================================================== dealing model
def pick_split(ntiles, kchunks, nctas):
    """ds_pick_split: the smallest split S whose wave fill is within 2 % of the best"""
    smax = max(1, min(16, kchunks // 2))
    eff = {}
    for S in range(1, smax + 1):
        waves = -(-(ntiles * S) // nctas)
        per = -(-kchunks // S)
        eff[S] = ntiles * kchunks / (waves * per * nctas)
    best = max(eff.values())
    return next(S for S in range(1, smax + 1) if eff[S] >= best - 0.02)


class GemmDeal:
    """a GEMM phase's units: unit = cta + wave nctas -> (split = unit / ntiles, tile = unit % ntiles), k chunks
    [split kchunks / S, (split + 1) kchunks / S)"""

    def __init__(self, ngroups, N, K, nctas):
        self.tpg = -(-N // 128)
        self.ntiles = ngroups * self.tpg
        self.kchunks = -(-K // 64)
        self.S = pick_split(self.ntiles, self.kchunks, nctas)
        self.nctas = nctas
        self.nunits = self.ntiles * self.S

    def krange(self, sp):
        return sp * self.kchunks // self.S, (sp + 1) * self.kchunks // self.S

    def waves(self, cta):
        return len(range(cta, self.nunits, self.nctas))


class StackDeal(attn64.Deal):
    """the stack's attention dealing: (head, 64-row chunk) units of the batch in equal contiguous ranges over
    min(units, SMs) CTAs (attn_stream_kernel's, with the SM count in place of its 264-CTA grid)"""

    def __init__(self, B, H, S, pos, nctas=NUM_SMS):
        super().__init__(BF16, B, H, H, S, pos)
        self.ncta = min(self.total, nctas)
        self.u0 = [c * self.total // self.ncta for c in range(self.ncta + 1)]


# ====================================================================== inputs (torch, on any device)
def weights(k, n, dt, seed, scale, device):
    """W [k, n] as T: standard normal x scale, column j x 2^((j mod 5) - 2) (ref64's column scaling)"""
    import torch
    g = torch.Generator(device=device).manual_seed(seed)
    w = torch.randn((k, n), generator=g, device=device, dtype=torch.float32) * scale
    return (w * torch.from_numpy(ref64.col_scale(n)).to(device)[None, :]).to({F16: torch.float16, BF16: torch.bfloat16}[dt])


def norm_weight(k, dt, seed):
    """1 + U(-1/4, 1/4), exact in T"""
    return rnd(1.0 + 0.25 * np.random.default_rng(seed).uniform(-1, 1, k), dt)


def rows(m, k, dt, seed, scale=1.0):
    """[m, k]: standard normal x scale, row i x 2^((i mod 7) - 3) (ref64's row scaling), exact in T"""
    x = np.random.default_rng(seed).standard_normal((m, k)) * scale * ref64.row_scale(m)[:, None]
    return rnd(x, dt)


# ====================================================================== float64 products
def gemm64(a, w, amb=None, block=4096):
    """(a . w, |a| . |w|, amb . |w|) as float64 numpy [rows, N]; a, amb: float64 numpy [rows, K]; w: a torch tensor [K, N] on
    any device, converted to float64 block by block of columns"""
    import torch
    dev = w.device
    a64 = torch.from_numpy(np.ascontiguousarray(a, np.float64)).to(dev)
    aa = a64.abs()
    d64 = None if amb is None else torch.from_numpy(np.ascontiguousarray(amb, np.float64)).to(dev)
    n = w.shape[1]
    ref, mag, am = (torch.empty((a.shape[0], n), dtype=torch.float64, device=dev) for _ in range(3))
    am.zero_()
    for j in range(0, n, block):
        wb = w[:, j:j + block].double()
        ref[:, j:j + block] = a64 @ wb
        wa = wb.abs()
        mag[:, j:j + block] = aa @ wa
        if d64 is not None:
            am[:, j:j + block] = d64 @ wa
    return ref.cpu().numpy(), mag.cpu().numpy(), am.cpu().numpy()


# ====================================================================== operand transforms and their ambiguity
def chain_length(path, K, nt=0, items=0):
    """longest chain of fp32 additions in the sum of squares: "x_raw" (a phase with no producer), "ss" (the hand-over from the
    previous residual phase's nt tiles) or "block" (rmsnorm_kernel, `items` per thread)"""
    if path == "x_raw":
        return K // 32 + 5
    if path == "ss":
        return 12 + -(-nt // 8)
    return items + 10


def rms_window(L):
    return (L + 8) * U


class Operand:
    """a GEMM operand: nominal value a; for a transformed one, the values c_lo / c_hi at the two ends of the fp32 window, and
    amb = |c_hi - c_lo| (0 where the rounding is not ambiguous)"""

    def __init__(self, a, lo=None, hi=None):
        self.a = np.asarray(a, np.float64)
        self.lo = self.a if lo is None else lo
        self.hi = self.a if hi is None else hi
        self.amb = np.abs(self.hi - self.lo)
        self.n_amb = int((self.amb > 0).sum())

    @property
    def share(self):
        return self.n_amb / max(self.a.size, 1)

    def outside(self, got):
        """elements of a kernel's transformed operand outside [min(c_lo, c_hi), max(c_lo, c_hi)]"""
        got = np.asarray(got, np.float64)
        return ~((got >= np.minimum(self.lo, self.hi)) & (got <= np.maximum(self.lo, self.hi)))


def _two_sided(y, window, tail, dt):
    """Operand tail(rnd(y)) when y carries a relative error up to `window`"""
    return Operand(tail(rnd(y, dt)), tail(rnd(y * (1 - window), dt)), tail(rnd(y * (1 + window), dt)))


def rinv64(x):
    x = np.asarray(x, np.float64)
    return 1.0 / np.sqrt((x * x).mean(1, keepdims=True) + EPS32)


def rmsnorm_operand(x, w, dt, L):
    """xn = rnd(rnd(x rinv) w) with rinv's window for a chain of L roundings"""
    x, w = np.asarray(x, np.float64), np.asarray(w, np.float64)
    return _two_sided(x * rinv64(x), rms_window(L), lambda r: rnd(r * w[None, :], dt), dt)


def silu64(g):
    g = np.asarray(g, np.float64)
    return g / (1.0 + np.exp(-g))


def silu_mul_operand(g, u, dt):
    """m = rnd(rnd(silu(g)) u)"""
    u = np.asarray(u, np.float64)
    return _two_sided(silu64(g), SILU_WINDOW, lambda r: rnd(r * u, dt), dt)


# ====================================================================== phase references
class PhaseRef:
    """reference and bound [rows, N] of one GEMM output"""

    def __init__(self, ref, bound):
        self.ref, self.bound = ref, bound

    def ratio(self, got):
        got = np.asarray(got, np.float64)
        r = np.abs(got - self.ref) / self.bound
        return float(np.max(np.where(np.isnan(r), np.inf, r))) if r.size else 0.0

    def violations(self, got, scale=1.0):
        return ~(np.abs(np.asarray(got, np.float64) - self.ref) <= scale * self.bound)


def store_ref(op, w, dt):
    """out = op.a . W rounded to T once"""
    ref, mag, am = gemm64(op.a, w, op.amb)
    return PhaseRef(ref, ref64.ulp(ref, dt) + ref64.ACC_SLACK * mag + AMB_MARGIN * am)


def residual_ref(op, w, res, dt):
    """out = rnd(res + rnd(op.a . W)): the product rounded as the separate MatMul stores it, then the Add"""
    acc, mag, am = gemm64(op.a, w, op.amb)
    ref = acc + np.asarray(res, np.float64)
    return PhaseRef(ref, ref64.ACC_SLACK * mag + ref64.ulp(acc, dt) + ref64.ulp(ref, dt) + AMB_MARGIN * am)


def report(bad, got, R, what, limit=4):
    if not bad.any():
        return None
    got = np.asarray(got, np.float64)
    idx = np.argwhere(bad)
    lines = [f"{what}: {int(bad.sum())} of {bad.size} elements outside the bound (worst "
             f"{float(np.max(np.where(bad, np.abs(got - R.ref) / R.bound, 0))):.3g}x)"]
    for i, j in idx[:limit]:
        lines.append(f"  row {i}, column {j} (tile {j // 128}): got {got[i, j]!r}, float64 {R.ref[i, j]!r}, "
                     f"bound {R.bound[i, j]:.3g}")
    lines.append(f"  rows with errors {sorted(set(idx[:, 0].tolist()))[:16]}, columns {sorted(set(idx[:, 1].tolist()))[:16]}")
    return "\n".join(lines)


# ====================================================================== RoPE in T (it_b200_rope's arithmetic)
def rope(x, pos, dt):
    """x [B, H, 128] rotated by per-row positions: each product rounded to T, then the difference / sum"""
    x = np.asarray(x, np.float64)
    c = np.arange(64)
    freq = (np.asarray(pos, np.float32)[:, None] * np.power(np.float32(10000.0), -(2.0 * c) / 128.0).astype(np.float32))
    cs = rnd(np.cos(freq.astype(np.float32).astype(np.float64)), dt)[:, None, :]
    sn = rnd(np.sin(freq.astype(np.float32).astype(np.float64)), dt)[:, None, :]
    lo, hi = x[..., :64], x[..., 64:]
    r32 = lambda v: rnd(np.asarray(v, np.float32).astype(np.float64), dt)
    return np.concatenate([r32(rnd(lo * cs, dt) - rnd(hi * sn, dt)), r32(rnd(hi * cs, dt) + rnd(lo * sn, dt))], -1)


class AttnInputs(attn64.Case):
    """an attention problem given by its tensors: q [B, H, 128] (rotated), cache rows kc / vc [B, H, >= max pos, 128] below each
    row's position, the appended kn / vn [B, H, 128]"""

    def __init__(self, q, kc, vc, kn, vn, pos):
        B, H = q.shape[:2]
        self.B, self.Hq, self.Hkv, self.grp = B, H, H, 1
        self.pos = np.asarray(pos, np.int64)
        self.S = int(self.pos.max()) + 1
        self.per_row = True
        self.q = np.asarray(q, np.float32)
        self.kseq = np.full((B, H, self.S, 128), np.nan, np.float32)
        self.vseq = np.full_like(self.kseq, np.nan)
        for b in range(B):
            p = int(self.pos[b])
            self.kseq[b, :, :p], self.vseq[b, :, :p] = kc[b, :, :p], vc[b, :, :p]
            self.kseq[b, :, p], self.vseq[b, :, p] = kn[b], vn[b]


# ====================================================================== float32 emulation of the GEMM phases
def _f(x):
    return np.asarray(x, np.float64).astype(np.float32)


def _r(x, dt):
    """round_t<T> of a float32 value"""
    return rnd(np.asarray(x, np.float32).astype(np.float64), dt).astype(np.float32)


def _xor_tree(v, levels):
    """lane 0 of a __shfl_xor_sync butterfly over the last axis (2^levels lanes)"""
    v = np.asarray(v, np.float32)
    n = v.shape[-1]
    o = n // 2
    while o:
        v = _f(v + v[..., np.arange(n) ^ o])
        o //= 2
    return v[..., 0]


MUTATIONS = ["ss_drop_tile", "rinv_pre_residual", "normw_shift8", "split_rounded", "lost_k16", "rinv_row_shift"]


def emu_rinv_x_raw(x):
    """the transform warps' own reduction of x_raw: lane i sums vectors i, i + 32, ... (8 fmaf each), then a warp tree"""
    m, K = x.shape
    xs = np.zeros((m, -(-K // 256) * 256), np.float32)
    xs[:, :K] = x
    lanes = xs.reshape(m, -1, 32, 8)  # [row, round, lane, j]: element (round 32 + lane) 8 + j
    s = np.zeros((m, 32), np.float32)
    for it in range(lanes.shape[1]):
        for j in range(8):
            f = lanes[:, it, :, j].astype(np.float64)
            s = _f(s + f * f)
    tot = _xor_tree(s, 5)
    return _f(1.0 / np.sqrt(_f(_f(tot / np.float32(K)) + np.float32(1e-5)).astype(np.float64)))


def emu_ss(y):
    """per-tile sums of squares the residual epilogue writes: [ntiles, rows]; columns past N count 0"""
    m, N = y.shape
    nt = -(-N // 128)
    yp = np.zeros((m, nt * 128), np.float32)
    yp[:, :N] = y
    sq = _f(yp.astype(np.float64) ** 2).reshape(m, nt, 4, 32)
    w = _xor_tree(sq, 5)                                     # [m, nt, 4]
    t = _f(_f(_f(w[..., 0] + w[..., 1]) + w[..., 2]) + w[..., 3])
    return t.T                                               # [nt, m]


def emu_rinv_ss(ss, K, mutation=None):
    nt, m = ss.shape
    if mutation == "ss_drop_tile":
        ss = ss.copy()
        ss[0] = 0
    part = np.zeros((m, 8), np.float32)
    for c8 in range(8):
        for tt in range(c8, nt, 8):
            part[:, c8] = _f(part[:, c8] + ss[tt])
    tot = _xor_tree(part, 3)
    return _f(1.0 / np.sqrt(_f(_f(tot / np.float32(K)) + np.float32(1e-5)).astype(np.float64)))


def emu_rmsnorm(x, w, rinv, dt, mutation=None):
    K = x.shape[1]
    if mutation == "rinv_row_shift":
        rinv = np.roll(rinv, -1)
    ww = np.asarray(w, np.float32)
    if mutation == "normw_shift8" and K > NORMW_MAX:
        ww = np.concatenate([ww[8:], np.zeros(8, np.float32)])
    return _r(_f(_r(_f(x * rinv[:, None]), dt).astype(np.float64) * ww), dt)


def emu_silu_mul(g, u, dt):
    g64 = np.asarray(g, np.float32)
    with np.errstate(over="ignore"):
        e = np.exp(-g64.astype(np.float64)).astype(np.float32)
    s = _f(g64.astype(np.float64) / _f(1.0 + e).astype(np.float64))
    return _r(_f(_r(s, dt).astype(np.float64) * u), dt)


def emu_gemm(a, w, ngroups, dt, epi=0, res=None, nctas=NUM_SMS, mutation=None):
    """one GEMM phase: out [rows, ngroups N] from the T operand a [rows, K] and W = the groups' weights side by side [K, ngroups N]
    (float32); fp32 partial tiles per k16 step of each unit's k chunks, the splits summed in split order, the epilogue."""
    m, K = a.shape
    N = w.shape[1] // ngroups
    d = GemmDeal(ngroups, N, K, nctas)
    a64 = np.zeros((m, d.kchunks * 64))
    a64[:, :K] = a
    out = np.empty((m, ngroups * N), np.float32)
    for tile in range(d.ntiles):
        g, n0 = divmod(tile, d.tpg)
        cols = np.arange(n0 * 128, min(N, n0 * 128 + 128))
        wt = np.zeros((d.kchunks * 64, len(cols)))
        wt[:K] = w[:, g * N + cols]
        f = np.zeros((m, len(cols)), np.float32)
        for sp in range(d.S):
            kb, ke = d.krange(sp)
            p = np.zeros((m, len(cols)), np.float32)
            for kc in range(kb, ke):
                for kk in range(4):
                    k0 = kc * 64 + kk * 16
                    prod = a64[:, k0:k0 + 16] @ wt[k0:k0 + 16]
                    if mutation == "lost_k16" and kc == kb and kk == 2:
                        prod[:, :64] = 0                          # one k16 step lost in the first m64 half
                    p = _f(p + prod)
            if mutation == "split_rounded" and d.S > 1:
                p = _r(p, dt)
            f = _f(f + p)
        if epi == 0:
            out[:, g * N + cols] = _r(f, dt)
        else:
            out[:, g * N + cols] = _r(_f(np.asarray(res, np.float32)[:, cols] + _r(f, dt)), dt)
    return out
