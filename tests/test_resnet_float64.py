"""The ResNet-50 kernels at the benchmark's batch of 64 against float64, element by element.

The element-level conv tests elsewhere run shapes on which no CTA of the persistent implicit-GEMM kernel reaches a third tile,
so the state it carries from tile to tile (TMA ring slot and phase, the parked-accumulator parity, the per-warp residual slab
ring with parity (q / 4) & 1, the residual prefetch cursor running 3 slabs ahead, the BatchNorm reload when the filter tile
changes) is never exercised there.  Here:

* A. every distinct conv of ResNet-50 at N = 64, 224^2, with the epilogue the schedule gives it, f16 and bf16, the 3x3 filters
  repacked for all banks by one it_b200_conv_repack_filters call and read with workspace_bytes < 0 as the runtime does; stage-1
  and stage-4 c3 also with NCHW output and residual;
* B. a tile-walk sweep: 131 .. 2245 tiles (one tile to 17 per CTA, +-1), and filter tiles that do not divide the 132 CTAs;
* C. the stem at (64, 3, 224, 224) and at a size whose blocks are cut on both sides;
* D. the batched filter repack over 30 banks (two launches), bit for bit, and a conv reading it against the self-repacking call;
* E. the NHWC 3x3 max pool and global average pool at the benchmark's shapes; F. the classifier GEMM with its bias;
* G. a profiler check that these cases launch the kernels the ResNet-50 step runs.

Inputs are exact in f16, bf16 and float64: input channel c scaled by 2^((c mod 7) - 3), filter f by 2^((f mod 5) - 2), so a
channel or filter mix-up changes values by at least 2x.  With ref = conv64(x, w) and S = conv64(|x|, |w|):

    plain conv:  |got - ref| <= ulp_T(|ref|) + 2^-16 S                            (tests/ref64.py: fp32 sums, K <= 4608)
    fused tail:  y64 = relu(a64 ref + b64 + r),  a64 = scale / sqrt(var + eps),  b64 = bias - mean a64  (float64 from the fp32
                 parameters);  |got - y64| <= ulp_T(|y64|) + |a64| 2^-16 S + 2^-20 (|a64 ref| + |mean a64| + |bias| + |r|)

The last term covers the fp32 epilogue: a and b are rounded in fp32 (b = fma(-mean, a, bias) may cancel, hence |mean a| + |bias|
rather than |b|), the fma and the residual add each round once in fp32.  ReLU does not enlarge a difference.  Every output is
filled with a NaN pattern before the launch (an unwritten element fails the bound) and followed by a guard region that must stay
untouched (the TMA store must clip the ragged last pixel tile).  A failure names the element and its place in the kernel's walk:
tile t, CTA t % grid, iteration t // grid.

The CPU self-checks at the top run without a GPU: a float32 emulation of conv_nhwc_kernel's arithmetic passes the bound, and six
plausible kernel bugs each fail it; the case list is checked to reach the tile-walk states above.
"""
import re

import numpy as np
import pytest
import torch

import oracle
from tests import ref64

F16, BF16 = 10, 16
DTYPES = [F16, BF16]
TORCH_DT = {F16: torch.float16, BF16: torch.bfloat16}
SMS = 132                   # persistent grid of the implicit-GEMM conv: min(tiles, 132)
BM, FT = 128, 64            # pixels x filters per output tile
STEM_BLOCK, STEM_CTAS_MAX = 16, 2 * SMS
TAIL_SLACK = 2.0 ** -20
NAN16 = 0x7FFF              # a NaN in both f16 and bf16
EPS = 1e-5


# ====================================================================== inputs and bounds (torch, CPU or GPU)
def exact(shape, seed, scale, dim=None, period=7, offset=3, device="cuda"):
    """standard normal x scale, the slice i along `dim` x 2^((i mod period) - offset), rounded to bf16, |v| < 2^-14 zeroed: every
    value is then exact in f16 as well (asserted), so one float64 reference serves both types"""
    g = torch.Generator(device=device).manual_seed(seed)
    v = torch.randn(shape, generator=g, device=device, dtype=torch.float32) * scale
    if dim is not None:
        s = torch.exp2((torch.arange(shape[dim], device=device) % period).float() - offset)
        v = v * s.view([-1 if d == dim else 1 for d in range(len(shape))])
    v = v.to(torch.bfloat16).float()
    v = torch.where(v.abs() < 2.0 ** -14, torch.zeros_like(v), v)
    assert torch.equal(v.to(torch.float16).float(), v) and torch.equal(v.to(torch.bfloat16).float(), v)
    return v


def batchnorm_params(f, seed, device="cuda"):
    g = torch.Generator(device=device).manual_seed(seed)
    u = lambda: torch.rand(f, generator=g, device=device) + 0.5
    mean = torch.randn(f, generator=g, device=device) * 0.1
    var, scale = u(), u()
    bias = torch.randn(f, generator=g, device=device) * 0.1
    return mean, var, scale, bias


def ulp_t(x, dt):
    """ref64.ulp on a torch tensor (float64)"""
    emin, mant = (-126, 7) if dt == BF16 else (-14, 10)
    _, ex = torch.frexp(x.abs())
    e = torch.where(x != 0, ex - 1, torch.full_like(ex, emin)).clamp(min=emin)
    return torch.exp2((e - mant).double())


def tail_reference(ref, S, bn=None, resid=None, relu=False):
    """(y64, bound) of the plain conv (bn None) or the fused tail; ref, S [M, F] float64, resid [M, F] or None"""
    if bn is None:
        return ref, ref64.ACC_SLACK * S
    mean, var, scale, bias = [v.double() for v in bn]
    a = scale / torch.sqrt(var + float(np.float32(EPS)))
    b = bias - mean * a
    y = ref * a + b
    tail = (ref * a).abs() + (mean * a).abs() + bias.abs()
    if resid is not None:
        r = resid.double()
        y = y + r
        tail = tail + r.abs()
    if relu:
        y = y.clamp(min=0)
    return y, a.abs() * ref64.ACC_SLACK * S + TAIL_SLACK * tail


def violations(got, y64, extra, dt):
    """boolean mask of the elements of `got` (T, any device) outside ulp_T(|y64|) + extra; NaN is outside"""
    return ~((got.double() - y64).abs() <= ulp_t(y64, dt) + extra)


# ====================================================================== tile-walk geometry (the launchers' formulas)
def conv_out(h, r, s, p):
    return (h + 2 * p - r) // s + 1


class Walk:
    """the implicit-GEMM conv's walk: M = N*P pixels in 128-pixel tiles, filter tiles of 64, tile t = mt * tiles_f + ft, CTA
    t % grid at iteration t // grid"""

    def __init__(self, n, oh, ow, f):
        self.N, self.OH, self.OW, self.F = n, oh, ow, f
        self.P, self.M = oh * ow, n * oh * ow
        self.tiles_m, self.tiles_f = -(-self.M // BM), -(-f // FT)
        self.tiles = self.tiles_m * self.tiles_f
        self.grid = min(self.tiles, SMS)
        self.min_per_cta = self.tiles // self.grid
        self.ragged = self.M % BM != 0
        # a tile whose first and last pixel belong to different images
        self.straddles = any((mt * BM) // self.P != (min(self.M, mt * BM + BM) - 1) // self.P for mt in range(min(self.tiles_m, 64)))

    def where(self, m, f):
        n, p = divmod(int(m), self.P)
        t = (int(m) // BM) * self.tiles_f + int(f) // FT
        return (f"pixel {int(m)} (image {n}, oh {p // self.OW}, ow {p % self.OW}), filter {int(f)}: tile {t} of {self.tiles}, "
                f"CTA {t % self.grid}, iteration {t // self.grid}")

    def ctas(self):
        return [list(range(b, self.tiles, self.grid)) for b in range(self.grid)]


def stem_grid(c, h, w, r, s, ph, pw, sh, sw, n):
    """(blocks, grid) of conv_stem_kernel: 16 x 16 output blocks, up to 2 CTAs per SM by shared memory"""
    oh, ow = conv_out(h, r, sh, ph), conv_out(w, s, sw, pw)
    blocks = n * -(-oh // STEM_BLOCK) * -(-ow // STEM_BLOCK)
    s4 = -(-s // 4) * 4
    wpitch = r * s4 * 4 + 8
    smem = 64 * wpitch * 2 + 64 * 8 + 8 * 32 * 144 + ((STEM_BLOCK - 1) * sh + r) * ((STEM_BLOCK - 1) * sw + s4) * 8
    per_sm = max(1, min(2, 220 * 1024 // (smem + 1024)))
    return blocks, min(blocks, SMS * per_sm)


def report(bad, got, y64, walk_where, what, limit=6):
    """an assertion message naming the first violations (indices into [M, F]) and their place in the walk"""
    nbad = int(bad.sum())
    if not nbad:
        return None
    idx = bad.nonzero()[:limit].tolist()
    lines = [f"{what}: {nbad} of {bad.numel()} elements outside the bound"]
    for m, f in idx:
        lines.append(f"  {walk_where(m, f)}: got {float(got[m, f])!r}, float64 {float(y64[m, f])!r}")
    return "\n".join(lines)


# ====================================================================== CPU: emulation of conv_nhwc_kernel's arithmetic
def im2col(x, r_, s_, p, st, mutation=None):
    """x [N, H, W, C] -> A [M, R*S, C] (zero padding); mutations as the TMA im2col box could get them wrong"""
    n_, h, w, c = x.shape
    oh, ow = conv_out(h, r_, st, p), conv_out(w, s_, st, p)
    m = np.arange(n_ * oh * ow)
    img, pp = np.divmod(m, oh * ow)
    yy, xx = np.divmod(pp, ow)
    if mutation == "straddle":  # the tile's later image read from the image of its first pixel
        img = (m // BM * BM) // (oh * ow)
    a = np.zeros((m.size, r_ * s_, c), np.float32)
    for r in range(r_):
        for s in range(s_):
            ih, iw = yy * st - p + r, xx * st - p + s
            if mutation == "edge_pad":  # left border: the edge pixel instead of the zero fill
                iw = np.maximum(iw, 0)
            ok = (ih >= 0) & (ih < h) & (iw >= 0) & (iw < w)
            a[ok, r * s_ + s] = x[img[ok], ih[ok], iw[ok]]
    return a, (n_, oh, ow)


def emulate_conv(x, w, p, st, dt, bn, resid, relu, mutation=None):
    """conv_nhwc_kernel's arithmetic in float32 numpy: k = filter tap x 64-channel chunk x k16, one fp32 product sum per k16
    step added into fp32 running sums; the epilogue fma(acc, a, b) with a = scale * rsqrt(var + eps), b = fma(-mean, a, bias),
    + residual, ReLU, all in fp32, one rounding to T.  `mutation` injects one kernel bug."""
    f_, c, r_, s_ = w.shape
    a, out_shape = im2col(x, r_, s_, p, st, mutation)
    walk = Walk(*out_shape, f_)
    m, rs, cp = a.shape[0], r_ * s_, -(-c // 64) * 64
    ap = np.zeros((m, rs, cp), np.float32)
    ap[:, :, :c] = a
    wp = np.zeros((f_, rs, cp), np.float32)
    wp[:, :, :c] = w.reshape(f_, c, rs).transpose(0, 2, 1)
    if mutation == "cp_stride":  # channels 64..71 of tap rs read from tap rs + 1
        wp[:, :-1, 64:72] = wp[:, 1:, 64:72].copy()
        wp[:, -1, 64:72] = 0
    acc = np.zeros((m, f_), np.float32)
    upper = (np.arange(m) % BM) >= 64
    for t in range(rs):
        for c0 in range(0, cp, 64):
            for kk in range(4):
                k0 = c0 + 16 * kk
                part = ap[:, t, k0:k0 + 16] @ wp[:, t, k0:k0 + 16].T
                if mutation == "lost_k16" and t == rs // 2 and c0 == 0 and kk == 1:  # the second wgmma of one k16 step
                    part[upper] = 0
                acc += part
    if bn is None:
        return oracle.round_to(acc, dt), walk
    mean, var, scale, bias = [np.asarray(v, np.float32) for v in bn]
    av = (scale * (np.float32(1) / np.sqrt(var + np.float32(EPS)))).astype(np.float32)
    bv = (-mean.astype(np.float64) * av + bias).astype(np.float32)
    pad_f = walk.tiles_f * FT
    a_t = np.ones((walk.tiles_m * BM, pad_f), np.float32)
    b_t = np.zeros_like(a_t)
    r_t = np.zeros_like(a_t)
    a_ext, b_ext = np.ones(pad_f, np.float32), np.zeros(pad_f, np.float32)
    a_ext[:f_], b_ext[:f_] = av, bv
    r_pad = np.zeros_like(a_t)
    if resid is not None:
        r_pad[:m, :f_] = resid
    blk = lambda t: (slice((t // walk.tiles_f) * BM, (t // walk.tiles_f + 1) * BM), slice((t % walk.tiles_f) * FT, (t % walk.tiles_f + 1) * FT))
    for tiles in walk.ctas():
        for i, t in enumerate(tiles):
            rows, cols = blk(t)
            ft = t % walk.tiles_f
            if mutation == "stale_bn" and i > 0:  # bn_sm kept from the CTA's previous tile
                ft = tiles[i - 1] % walk.tiles_f
            a_t[rows, cols], b_t[rows, cols] = a_ext[ft * FT:(ft + 1) * FT], b_ext[ft * FT:(ft + 1) * FT]
            src = tiles[i - 4] if mutation == "stale_residual" and i >= 4 else t  # ring buffer q % 4 reused before its load landed
            r_t[rows, cols] = r_pad[blk(src)]
    y = (acc.astype(np.float64) * a_t[:m, :f_] + b_t[:m, :f_]).astype(np.float32)
    if resid is not None:
        y = y + r_t[:m, :f_]
    if relu:
        y = np.maximum(y, np.float32(0))
    return oracle.round_to(y, dt), walk


# (N, H, W, C, F, R, pad, stride): 3x3 s1 (two pixel tiles, the first straddling three images), 3x3 s2, 1x1, and a 1x1 walk
# with 680 tiles over 5 filter tiles (5 to 6 tiles per CTA, the filter tile changing at every step of each CTA's walk)
EMU_SHAPES = {"3x3s1": (3, 9, 7, 72, 80, 3, 1, 1), "3x3s2": (3, 9, 7, 72, 80, 3, 1, 2), "1x1": (3, 9, 7, 72, 80, 1, 0, 1),
              "walk": (3, 75, 77, 72, 312, 1, 0, 1)}
_emu_cache = {}


def _emu_case(name):
    if name not in _emu_cache:
        n, h, w, c, f, r, p, st = EMU_SHAPES[name]
        x = exact((n, h, w, c), 11, 1.0, dim=3, device="cpu")
        wt = exact((f, c, r, r), 12, 1.0 / np.sqrt(c * r * r), dim=0, period=5, offset=2, device="cpu")
        a, _ = im2col(x.numpy(), r, r, p, st)
        ref = a.reshape(a.shape[0], -1).astype(np.float64) @ wt.numpy().transpose(0, 2, 3, 1).reshape(f, -1).T.astype(np.float64)
        mag = np.abs(a.reshape(a.shape[0], -1)).astype(np.float64) @ np.abs(wt.numpy().transpose(0, 2, 3, 1).reshape(f, -1)).T
        bn = batchnorm_params(f, 13, device="cpu")
        resid = exact((a.shape[0], f), 14, 1.0, device="cpu")
        _emu_cache[name] = (x.numpy(), wt.numpy(), p, st, torch.from_numpy(ref), torch.from_numpy(mag), bn, resid)
    return _emu_cache[name]


def _emu_violations(name, dt, fused, mutation=None):
    x, w, p, st, ref, mag, bn, resid = _emu_case(name)
    got, _ = emulate_conv(x, w, p, st, dt, [v.numpy() for v in bn] if fused else None, resid.numpy() if fused else None, fused,
                          mutation)
    y64, extra = tail_reference(ref, mag, bn if fused else None, resid if fused else None, fused)
    return violations(torch.from_numpy(got), y64, extra, dt)


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("name", sorted(EMU_SHAPES))
def test_bound_passes_conv_arithmetic(name, dt):
    for fused in (False, True):
        bad = _emu_violations(name, dt, fused)
        assert not bad.any(), f"emulated {name} fused={fused}: {int(bad.sum())} elements outside the bound"


@pytest.mark.parametrize("name,mutation", [("3x3s1", "lost_k16"), ("1x1", "lost_k16"), ("3x3s1", "edge_pad"),
                                           ("3x3s2", "edge_pad"), ("3x3s1", "straddle"), ("walk", "stale_residual"),
                                           ("walk", "stale_bn"), ("3x3s1", "cp_stride"), ("3x3s2", "cp_stride")])
def test_bound_catches_conv_bugs(name, mutation):
    """bf16, the coarser type: each injected bug leaves elements outside the fused-tail bound"""
    assert _emu_violations(name, BF16, True, mutation).any(), f"{mutation} on {name} stays inside the bound"


def test_ulp_matches_ref64():
    x = np.array([0.0, 2.0 ** -30, 2.0 ** -14, 2.0 ** -13 * 1.5, 1.0, -1.75, 3.0, 65504.0, 2.0 ** -130, 1e30])
    for dt in DTYPES:
        assert np.array_equal(ulp_t(torch.from_numpy(x), dt).numpy(), ref64.ulp(x, dt))


def test_exact_inputs_scale_channels_and_filters():
    """the same draw with and without the per-slice powers of two: every value that survives both is scaled exactly"""
    for shape, dim, period, offset in [((2, 3, 3, 14), 3, 7, 3), ((10, 4, 3, 3), 0, 5, 2)]:
        plain = exact(shape, 1, 0.05, device="cpu")
        scaled = exact(shape, 1, 0.05, dim=dim, period=period, offset=offset, device="cpu")
        s = torch.exp2((torch.arange(shape[dim]) % period).float() - offset).view([-1 if d == dim else 1 for d in range(len(shape))])
        both = (plain != 0) & (scaled != 0)
        assert both.float().mean() > 0.9 and torch.equal(scaled[both], (plain * s)[both])
        assert torch.all((scaled == 0) | (scaled.abs() >= 2.0 ** -14))


# ====================================================================== the GPU case lists
def _resnet50_convs():
    """every distinct conv of ResNet-50 (v1.5: stride on the 3x3) at N = 64, 224^2: (name, C, H, F, R, stride, epilogue);
    epilogue "relu" = BN + ReLU, "res" = BN + residual + ReLU, "bn" = BN only"""
    cases = [("s1.c1", 64, 56, 64, 1, 1, "relu"), ("s1.c1b", 256, 56, 64, 1, 1, "relu"), ("s1.c2", 64, 56, 64, 3, 1, "relu"),
             ("s1.c3", 64, 56, 256, 1, 1, "res"), ("s1.down", 64, 56, 256, 1, 1, "bn")]
    for k, (w, h) in enumerate([(128, 56), (256, 28), (512, 14)], start=2):
        cases += [(f"s{k}.c1", 2 * w, h, w, 1, 1, "relu"), (f"s{k}.c2", w, h, w, 3, 2, "relu"), (f"s{k}.c3", w, h // 2, 4 * w, 1, 1, "res"),
                  (f"s{k}.down", 2 * w, h, 4 * w, 1, 2, "bn"), (f"s{k}.c1b", 4 * w, h // 2, w, 1, 1, "relu"),
                  (f"s{k}.c2b", w, h // 2, w, 3, 1, "relu")]
    return cases


BATCH = 64
RESNET_CONVS = _resnet50_convs()
NCHW_TOO = {"s1.c3", "s4.c3"}
# B: 1x1, C = 64, 8x8 images (two per tile), + residual + ReLU: (N, F).  131 .. 2245 tiles = one to 17 per CTA, +-1; then
# 5 and 32 filter tiles (neither divides 132) at 9 tiles per CTA
SWEEP = [(2 * t, 64) for t in (131, 132, 133, 528, 1188, 1189, 2245)] + [(480, 320), (76, 2048)]
STEM_CASES = [(64, 224, 224), (200, 61, 53)]  # (N, H, W): 3 channels, 64 filters 7x7 s2 p3, BN + ReLU


def _conv_walks():
    """(name, walk, has residual, dtypes) of every implicit-GEMM conv case"""
    out = []
    for name, c, h, f, r, st, epi in RESNET_CONVS:
        oh = conv_out(h, r, st, r // 2)
        out.append((name, Walk(BATCH, oh, oh, f), epi == "res", DTYPES))
    for n, f in SWEEP:
        out.append((f"sweep N={n} F={f}", Walk(n, 8, 8, f), True, DTYPES))
    return out


def test_case_list_reaches_the_tile_walk_states():
    walks = _conv_walks()
    assert len(RESNET_CONVS) == 23
    for dt in DTYPES:  # a residual slab ring that flips its parity twice: 9 slabs per warp, one per tile
        assert any(res and dt in dts and w.min_per_cta >= 9 for _, w, res, dts in walks), dt
    assert any(SMS % w.tiles_f and w.tiles >= 2 * w.grid for _, w, _, _ in walks), "no filter-tile change along a walk"
    assert any(w.ragged for _, w, _, _ in walks), "no ragged last pixel tile"
    assert any(w.straddles for _, w, _, _ in walks), "no tile straddling two images"
    assert {w.tiles for _, w, _, _ in walks} >= {131, 132, 133, 528, 1188, 1189, 2245}
    s1c3 = dict((nm, w) for nm, w, _, _ in walks)["s1.c3"]
    assert s1c3.tiles == 6272 and s1c3.min_per_cta == 47
    blocks, grid = stem_grid(3, 224, 224, 7, 7, 3, 3, 2, 2, 64)
    assert blocks == 3136 and grid <= STEM_CTAS_MAX and blocks // grid >= 4


# ====================================================================== GPU plumbing
@pytest.fixture(scope="module")
def K():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from tests import kernel_harness
    return kernel_harness


def guarded(n, dt, guard):
    """n elements of T filled with a NaN pattern, followed by `guard` more that nothing may write"""
    return torch.full((n + guard,), NAN16, dtype=torch.int16, device="cuda").view(TORCH_DT[dt])


def assert_guard(buf, n, what):
    g = buf[n:].view(torch.int16)
    assert bool((g == NAN16).all()), f"{what}: {int((g != NAN16).sum())} elements written past the end of the output"


def conv64(x_nchw, w, stride, pad):
    """(ref, S) in float64 as [N, OH, OW, F]"""
    x, wd = x_nchw.double(), w.double()
    ref = torch.nn.functional.conv2d(x, wd, stride=stride, padding=pad)
    mag = torch.nn.functional.conv2d(x.abs(), wd.abs(), stride=stride, padding=pad)
    return ref.permute(0, 2, 3, 1).contiguous(), mag.permute(0, 2, 3, 1).contiguous()


def pin_reference(x_nchw, w, stride, pad, ref, mag, pixels):
    """the float64 reference at a few output pixels (all filters) against numpy float64 on the CPU"""
    n_, c, h, wd = x_nchw.shape
    f, _, r_, s_ = w.shape
    _, oh_, ow_, _ = ref.shape
    w64 = w.double().cpu().numpy()
    for m in pixels:
        n, p = divmod(int(m), oh_ * ow_)
        oh, ow = divmod(p, ow_)
        xi = np.pad(x_nchw[n].double().cpu().numpy(), ((0, 0), (pad, pad), (pad, pad)))
        patch = xi[:, oh * stride:oh * stride + r_, ow * stride:ow * stride + s_]
        want = np.einsum("crs,fcrs->f", patch, w64)
        want_mag = np.einsum("crs,fcrs->f", np.abs(patch), np.abs(w64))
        got, got_mag = ref[n, oh, ow].cpu().numpy(), mag[n, oh, ow].cpu().numpy()
        assert np.all(np.abs(got - want) <= 2.0 ** -40 * want_mag) and np.allclose(got_mag, want_mag, rtol=2.0 ** -40, atol=0), \
            f"float64 reference at pixel {int(m)}"


def sample_pixels(walk):
    """the first tile, a tile straddling two images (if any), the ragged last tile"""
    px = [0, 1, 64, min(walk.M, BM) - 1]
    if walk.P % BM:
        s = (walk.P // BM) * BM  # the tile holding the last pixels of image 0 and the first of image 1
        px += [s, walk.P - 1, min(walk.M - 1, walk.P)]
    px += [(walk.tiles_m - 1) * BM, walk.M - 1]
    return sorted(set(px))


def run_conv(K, dt, x, w, walk, r, st, pad, bn, resid, relu, y_nhwc, repacked=None, workspace=True):
    """one it_b200_conv2d_nhwc launch into a NaN-filled, guarded output; x [N, H, W, C] in T.  `repacked`: (buffer, bytes) from
    it_b200_conv_repack_filters, passed with workspace_bytes < 0.  Returns the output as [M, F] (a view for NCHW output)."""
    n_, h, wd, c = x.shape
    f = w.shape[0]
    n = walk.M * f
    buf = guarded(n, dt, BM * f + 64)
    if repacked is not None:
        ws, wsb = repacked[0], -repacked[1]
    elif r > 1 and workspace:
        wsb = int(K.L.lib.it_b200_conv2d_nhwc_workspace(dt, c, f, r, r))
        ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    else:
        ws, wsb = None, 0
    ms = [K.ptr(v) for v in bn] if bn is not None else [None] * 4
    K.L.check(K.L.lib.it_b200_conv2d_nhwc(dt, K.ptr(x), K.ptr(w), K.ptr(buf), int(y_nhwc), n_, c, h, wd, f, r, r, pad, pad, st, st,
                                          1, 1, *ms, EPS, K.ptr(resid), int(relu), K.ptr(ws), wsb, K.stream()))
    K.sync()
    assert_guard(buf, n, f"conv N={n_} C={c} {h}x{wd} F={f} {r}x{r} s{st}")
    y = buf[:n]
    return y.view(walk.M, f) if y_nhwc else y.view(walk.N, f, walk.P).permute(0, 2, 1).reshape(walk.M, f)


def repack(K, dt, banks):
    """one it_b200_conv_repack_filters call over `banks` (device [F, C, R, S] in T); each destination NaN-filled and guarded.
    Returns [(buffer, bytes)]"""
    import ctypes
    VP = ctypes.c_void_p
    outs = []
    for w in banks:
        f, c, r, s = w.shape
        nbytes = int(K.L.lib.it_b200_conv2d_nhwc_workspace(dt, c, f, r, s))
        outs.append((guarded(nbytes // 2, dt, 256), nbytes))
    K.L.check(K.L.lib.it_b200_conv_repack_filters(dt, len(banks), (VP * len(banks))(*[w.data_ptr() for w in banks]),
                                                  (VP * len(banks))(*[o.data_ptr() for o, _ in outs]),
                                                  K.L.i32arr([w.shape[0] for w in banks]), K.L.i32arr([w.shape[1] for w in banks]),
                                                  K.L.i32arr([w.shape[2] for w in banks]), K.L.i32arr([w.shape[3] for w in banks]),
                                                  K.stream()))
    K.sync()
    for i, (o, nbytes) in enumerate(outs):
        assert_guard(o, nbytes // 2, f"repack bank {i}")
    return outs


def _seed(name):
    return 1000 + 10 * sorted(c[0] for c in RESNET_CONVS).index(name)


class ResnetData:
    """the filters of every ResNet-50 conv (exact, float32 on the device) and, per dtype, the 3x3 banks repacked by ONE
    it_b200_conv_repack_filters call, as the runtime does at the start of a step"""

    def __init__(self, K):
        self.w = {}
        for name, c, _, f, r, _, _ in RESNET_CONVS:
            self.w[name] = exact((f, c, r, r), _seed(name) + 1, 1.0 / np.sqrt(c * r * r), dim=0, period=5, offset=2)
        self.wt, self.packed = {}, {}
        for dt in DTYPES:
            for name in self.w:
                self.wt[name, dt] = self.w[name].to(TORCH_DT[dt])
            names = [c[0] for c in RESNET_CONVS if c[4] == 3]
            for name, out in zip(names, repack(K, dt, [self.wt[nm, dt] for nm in names])):
                self.packed[name, dt] = out


@pytest.fixture(scope="module")
def resnet(K):
    return ResnetData(K)


def check_conv(dt, walk, got, y64, extra, what):
    msg = report(violations(got, y64, extra, dt), got, y64, walk.where, f"{what} {'bf16' if dt == BF16 else 'f16'}")
    return [msg] if msg else []


# ====================================================================== GPU A: every ResNet-50 conv at N = 64
@pytest.mark.gpu
@pytest.mark.parametrize("case", RESNET_CONVS, ids=[c[0] for c in RESNET_CONVS])
def test_resnet50_conv_float64(K, resnet, case):
    name, c, h, f, r, st, epi = case
    pad = r // 2
    oh = conv_out(h, r, st, pad)
    walk = Walk(BATCH, oh, oh, f)
    seed = _seed(name)
    x = exact((BATCH, h, h, c), seed, 1.0, dim=3)
    bn = batchnorm_params(f, seed + 2)
    resid = exact((walk.M, f), seed + 3, 1.0) if epi == "res" else None
    relu = epi != "bn"
    x_nchw = x.permute(0, 3, 1, 2)
    ref, mag = conv64(x_nchw, resnet.w[name], st, pad)
    pin_reference(x_nchw, resnet.w[name], st, pad, ref, mag, sample_pixels(walk))
    ref, mag = ref.view(walk.M, f), mag.view(walk.M, f)
    del x_nchw
    y64, extra = tail_reference(ref, mag, bn, resid, relu)
    del ref, mag
    fails = []
    for dt in DTYPES:
        xt = x.to(TORCH_DT[dt])
        rt = resid.to(TORCH_DT[dt]) if resid is not None else None
        got = run_conv(K, dt, xt, resnet.wt[name, dt], walk, r, st, pad, bn, rt, relu, True, resnet.packed.get((name, dt)))
        fails += check_conv(dt, walk, got, y64, extra, f"{name} NHWC")
        if name in NCHW_TOO:  # NCHW output and residual ([N, F, OH, OW]), for a consumer outside the NHWC domain
            rn = rt.view(BATCH, walk.P, f).permute(0, 2, 1).contiguous() if rt is not None else None
            got = run_conv(K, dt, xt, resnet.wt[name, dt], walk, r, st, pad, bn, rn, relu, False, resnet.packed.get((name, dt)))
            fails += check_conv(dt, walk, got, y64, extra, f"{name} NCHW")
    assert not fails, "\n".join(fails)


# ====================================================================== GPU B: tile-walk sweep
@pytest.mark.gpu
@pytest.mark.parametrize("n,f", SWEEP, ids=[f"N{n}-F{f}" for n, f in SWEEP])
def test_conv_tile_walk_float64(K, n, f):
    walk = Walk(n, 8, 8, f)
    seed = 3000 + n + f
    x = exact((n, 8, 8, 64), seed, 1.0, dim=3)
    w = exact((f, 64, 1, 1), seed + 1, 0.125, dim=0, period=5, offset=2)
    bn = batchnorm_params(f, seed + 2)
    resid = exact((walk.M, f), seed + 3, 1.0)
    ref = x.view(walk.M, 64).double() @ w.view(f, 64).double().T
    mag = x.view(walk.M, 64).double().abs() @ w.view(f, 64).double().abs().T
    y64, extra = tail_reference(ref, mag, bn, resid, True)
    fails = []
    for dt in DTYPES:
        got = run_conv(K, dt, x.to(TORCH_DT[dt]), w.to(TORCH_DT[dt]), walk, 1, 1, 0, bn, resid.to(TORCH_DT[dt]), True, True)
        fails += check_conv(dt, walk, got, y64, extra, f"1x1 N={n} F={f} ({walk.tiles} tiles)")
    assert not fails, "\n".join(fails)


# ====================================================================== GPU C: the stem
def run_stem(K, dt, x, w, bn):
    n_, c, h, wd = x.shape
    f = w.shape[0]
    oh, ow = conv_out(h, 7, 2, 3), conv_out(wd, 7, 2, 3)
    n = n_ * oh * ow * f
    buf = guarded(n, dt, 16 * 16 * f)
    assert K.L.lib.it_b200_conv2d_stem_supported(dt, c, f, 7, 7, 3, 3, 2, 2, 1, 1, 1) == 1
    K.L.check(K.L.lib.it_b200_conv2d_stem(dt, K.ptr(x), K.ptr(w), K.ptr(buf), n_, c, h, wd, f, 7, 7, 3, 3, 2, 2,
                                          *[K.ptr(v) for v in bn], EPS, 1, K.stream()))
    K.sync()
    assert_guard(buf, n, f"stem {tuple(x.shape)}")
    return buf[:n].view(n_ * oh * ow, f)


@pytest.mark.gpu
@pytest.mark.parametrize("n,h,w", STEM_CASES, ids=[f"{n}x{h}x{w}" for n, h, w in STEM_CASES])
def test_stem_float64(K, n, h, w):
    seed = 4000 + n
    x = exact((n, 3, h, w), seed, 1.0, dim=1)
    wt = exact((64, 3, 7, 7), seed + 1, 1.0 / np.sqrt(147), dim=0, period=5, offset=2)
    bn = batchnorm_params(64, seed + 2)
    ref, mag = conv64(x, wt, 2, 3)
    oh, ow = ref.shape[1:3]
    blocks, grid = stem_grid(3, h, w, 7, 7, 3, 3, 2, 2, n)
    tw_, th_ = -(-ow // STEM_BLOCK), -(-oh // STEM_BLOCK)

    def where(m, f):
        img, p = divmod(m, oh * ow)
        y, xx = divmod(p, ow)
        b = (img * th_ + y // STEM_BLOCK) * tw_ + xx // STEM_BLOCK
        return f"image {img}, oh {y}, ow {xx}, filter {f}: block {b} of {blocks}, CTA {b % grid}, iteration {b // grid}"

    pin_reference(x, wt, 2, 3, ref, mag, [0, ow - 1, oh * ow - 1, n * oh * ow - 1])
    y64, extra = tail_reference(ref.view(-1, 64), mag.view(-1, 64), bn, None, True)
    fails = []
    for dt in DTYPES:
        got = run_stem(K, dt, x.to(TORCH_DT[dt]), wt.to(TORCH_DT[dt]), bn)
        msg = report(violations(got, y64, extra, dt), got, y64, where, f"stem {n}x3x{h}x{w} {dt}")
        fails += [msg] if msg else []
    assert not fails, "\n".join(fails)


# ====================================================================== GPU D: the batched filter repack
# 30 banks (two launches, the second with 6): 3x3 at C = 24, 72, 256 and the ResNet widths, and 3x5, 5x5, 1x7 banks
REPACK_BANKS = [(64, 64, 3, 3), (128, 128, 3, 3), (256, 256, 3, 3), (512, 512, 3, 3), (40, 24, 3, 5), (304, 72, 3, 3),
                (8, 24, 5, 5), (64, 72, 1, 7), (16, 256, 3, 3), (24, 72, 5, 5)] * 3


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
def test_repack_filters_batch_bit_exact(K, dt):
    banks = [exact(s, 5000 + i, 0.5).to(TORCH_DT[dt]) for i, s in enumerate(REPACK_BANKS)]
    outs = repack(K, dt, banks)
    for i, ((f, c, r, s), w, (o, nbytes)) in enumerate(zip(REPACK_BANKS, banks, outs)):
        cp = -(-c // 64) * 64
        want = np.zeros((f, r * s, cp), np.int16)
        want[:, :, :c] = w.view(torch.int16).cpu().numpy().reshape(f, c, r * s).transpose(0, 2, 1)
        got = o[:nbytes // 2].view(torch.int16).cpu().numpy().reshape(f, r * s, cp)
        assert np.array_equal(got, want), f"bank {i} {(f, c, r, s)}: {np.sum(got != want)} elements differ"
    # a conv reading the repacked filters (workspace_bytes < 0) equals the call that repacks its own, bit for bit
    for i in (5, 4, 9):
        f, c, r, s = REPACK_BANKS[i]
        if r != s:
            continue  # run_conv takes square filters; the 3x5 bank's layout is checked above
        x = exact((3, 19, 13, c), 5100 + i, 1.0, dim=3).to(TORCH_DT[dt])
        bn = batchnorm_params(f, 5200 + i)
        walk = Walk(3, conv_out(19, r, 1, r // 2), conv_out(13, r, 1, r // 2), f)
        own = run_conv(K, dt, x, banks[i], walk, r, 1, r // 2, bn, None, True, True)
        pre = run_conv(K, dt, x, banks[i], walk, r, 1, r // 2, bn, None, True, True, repacked=outs[i])
        assert torch.equal(own.view(torch.int16), pre.view(torch.int16)), f"bank {i}: pre-repacked filters change the conv"


# ====================================================================== GPU E: NHWC pools at the benchmark's shapes
def run_pool(K, dt, x, is_max, k, st, pad, oh, ow):
    n_, h, w, c = x.shape
    n = n_ * oh * ow * c
    buf = guarded(n, dt, 4096)
    K.L.check(K.L.lib.it_b200_pool2d_nhwc(dt, int(is_max), K.ptr(x), K.ptr(buf), n_, c, h, w, k[0], k[1], 1, 1, pad, pad, st, st,
                                          oh, ow, K.stream()))
    K.sync()
    assert_guard(buf, n, "pool")
    return buf[:n].view(n_, oh, ow, c)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
def test_pools_nhwc_float64(K, dt):
    """3x3 s2 p1 max pool on (64, 64, 112, 112): bit for bit the max over the valid taps (padding never wins, the inputs are
    half negative); global average pool on (64, 2048, 7, 7): ulp_T(|ref|) + 2^-16 mean|x|"""
    x = exact((64, 112, 112, 64), 6000, 1.0, dim=3)
    got = run_pool(K, dt, x.to(TORCH_DT[dt]), True, (3, 3), 2, 1, 56, 56)
    want = torch.nn.functional.max_pool2d(x.permute(0, 3, 1, 2).double(), 3, 2, 1).permute(0, 2, 3, 1)
    bad = got.double() != want
    assert not bad.any(), f"max pool: {int(bad.sum())} elements differ, first at (n, oh, ow, c) {bad.nonzero()[0].tolist()}"
    x = exact((64, 7, 7, 2048), 6001, 1.0, dim=3)
    got = run_pool(K, dt, x.to(TORCH_DT[dt]), False, (7, 7), 1, 0, 1, 1).view(64, 2048)
    x64 = x.double().view(64, 49, 2048)
    ref = x64.mean(1)
    bad = violations(got, ref, ref64.ACC_SLACK * x64.abs().mean(1), dt)
    assert not bad.any(), f"global average pool: {int(bad.sum())} elements outside the bound, first (n, c) {bad.nonzero()[0].tolist()}"


# ====================================================================== GPU F: the classifier
@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
def test_classifier_float64(K, dt):
    """(64 x 2048) . (1000 x 2048)^T + bias through it_b200_matmul with transB, the ref64 bound with the bias in the sum"""
    m, k, n = 64, 2048, 1000
    x = ref64.activations(m, k, dt, 7000)
    w = ref64.weights(k, n, dt, 7001)
    bias = oracle.round_to(np.random.default_rng(7002).standard_normal(n).astype(np.float32) * np.float32(0.5), dt)
    ref, mag = ref64.product(x, w)
    c = torch.empty((m, n), dtype=TORCH_DT[dt], device="cuda")
    K.L.check(K.L.lib.it_b200_matmul(dt, K.ptr(K.dev(x, dt)), K.ptr(K.dev(np.ascontiguousarray(w.T), dt)), K.ptr(K.dev(bias, dt)),
                                     K.ptr(c), 1, m, n, k, m * k, 0, 0, 1, 0, 0, 1, 0, None, 0, K.stream()))
    K.sync()
    ref64.assert_within(K.host(c), ref + bias[None, :], mag + np.abs(bias)[None, :], dt, what=f"classifier {dt}")


# ====================================================================== GPU G: the intended kernels ran
def profiled_kernel_names():
    """kernel names recorded by torch.profiler (CUDA activity only) for one small call of each kind above"""
    from tests import kernel_harness as K
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for dt in DTYPES:
            x = exact((2, 8, 8, 64), 8000, 1.0, dim=3).to(TORCH_DT[dt])
            w = exact((64, 64, 3, 3), 8001, 0.05).to(TORCH_DT[dt])
            packed = repack(K, dt, [w])
            run_conv(K, dt, x, w, Walk(2, 8, 8, 64), 3, 1, 1, None, None, False, True, packed[0])
        dt = F16
        run_stem(K, dt, exact((1, 3, 32, 32), 8002, 1.0).to(TORCH_DT[dt]), exact((64, 3, 7, 7), 8003, 0.1).to(TORCH_DT[dt]),
                 batchnorm_params(64, 8004))
        run_pool(K, dt, exact((1, 16, 16, 64), 8005, 1.0).to(TORCH_DT[dt]), True, (3, 3), 2, 1, 8, 8)
        run_pool(K, dt, exact((2, 7, 7, 256), 8006, 1.0).to(TORCH_DT[dt]), False, (7, 7), 1, 0, 1, 1)
        torch.cuda.synchronize()
    return sorted({e.name for e in prof.events() if "CUDA" in str(e.device_type)})


@pytest.mark.gpu
def test_resnet_cases_reach_the_intended_kernels(K):
    """in a child process, as the other float64 files do: a profiler session earlier in the test process can lose the
    records of a later one's first kernels"""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = "import json; from tests.test_resnet_float64 import profiled_kernel_names as f; print(json.dumps(f()))"
    r = subprocess.run([sys.executable, "-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    names = set(json.loads(r.stdout.strip().splitlines()[-1]))
    if not names:
        pytest.skip("the profiler recorded no CUDA kernel events (CUPTI activity tracing unavailable)")
    want = [r"conv_nhwc_kernel<__half", r"conv_nhwc_kernel<__nv_bfloat16", r"conv_stem_kernel<", r"repack_filters_batch_kernel<",
            r"pool2d_nhwc3x3_kernel<", r"global_avgpool_nhwc_kernel<"]
    missing = [p for p in want if not any(re.search(p, nm) for nm in names)]
    assert not missing, f"not launched: {missing}; kernels seen: {sorted(names)}"
