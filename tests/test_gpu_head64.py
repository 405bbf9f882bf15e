"""Decode attention at head width 64 on the GPU: both kernels (query heads = KV heads, and grouped-query) against the
oracle rule at 1/sqrt(64), the folded RoPE against RoPE(dim_head 64) + the unfused kernel, a float64 per-element bound
over the score regimes and CTA splits of tests/attn64.py, and whole TinyLlama-shape and GPT-2 decode graphs."""
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import oracle
from tests import attn64
from tests.llama_oracle import attention_kvcache_d, run_llama_parity

F32, F16, BF16 = 1, 10, 16
D = 64
TOL = {F32: 1e-5, F16: 1e-3, BF16: 1e-2}  # as test_gpu_gqa
POS_IN_STEP, POS_PER_ROW = 0x200, 0x100


@pytest.fixture(scope="module")
def K():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from tests import kernel_harness
    return kernel_harness


def rnd(shape, seed, dt, scale=0.5):
    return oracle.round_to(np.random.default_rng(seed).standard_normal(shape).astype(np.float32) * np.float32(scale), dt)


def close(got, exp, rel, abs_):
    np.testing.assert_allclose(np.asarray(got, np.float64).ravel(), np.asarray(exp, np.float64).ravel(), rtol=rel, atol=abs_)


def launch(K, kc, vc, q, k, v, pos, dt, flags=0, rope_pos=None):
    """one it_b200_attention_kvcache_gqa launch (Hq == Hkv runs the streaming kernel); returns (out, k cache, v cache)"""
    import torch
    L = K.L
    kcd, vcd = K.dev(kc, dt), K.dev(vc, dt)
    qd, kd, vd = K.dev(q, dt), K.dev(k, dt), K.dev(v, dt)
    B, Hkv, Smax, Dh = kc.shape
    Hq = q.shape[1]
    if np.ndim(pos) > 0:
        flags |= POS_PER_ROW
    pd = K.raw(np.atleast_1d(np.asarray(pos)).astype(np.int64))
    rp = None if rope_pos is None else K.raw(np.asarray(rope_pos, np.int64))
    out = torch.empty_like(qd)
    wsb = L.lib.it_b200_attention_kvcache_workspace(B, Hq, Smax, Dh)
    ws = torch.empty(max(int(wsb), 16), dtype=torch.uint8, device="cuda")
    L.check(L.lib.it_b200_attention_kvcache_gqa(dt, K.ptr(kcd), K.ptr(vcd), K.ptr(qd), K.ptr(kd), K.ptr(vd), K.ptr(pd), 7 | flags,
                                                K.ptr(rp), 7, K.ptr(out), B, Hq, Hkv, Smax, Dh, K.ptr(ws), int(wsb), K.stream()))
    K.sync()
    return K.host(out), K.host(kcd), K.host(vcd)


def inputs(B, Hq, Hkv, S, dt):
    kc, vc = rnd((B, Hkv, S, D), 28, dt), rnd((B, Hkv, S, D), 29, dt)
    q, k, v = rnd((B, Hq, 1, D), 30, dt), rnd((B, Hkv, 1, D), 31, dt), rnd((B, Hkv, 1, D), 32, dt)
    return kc, vc, q, k, v


# G = 1 (streaming kernel), G in {2, 4, 8, 32, 48} (one query tile up to G = 16, two above); contexts shorter than, equal to
# and longer than one 128-row chunk (64 rows for fp32), up to a whole 4096-row head
SHAPES = [(2, 8, 8, 256, 0), (7, 5, 5, 300, 129), (16, 12, 12, 1024, 511), (1, 1, 1, 4096, 4095), (2, 8, 4, 256, 37),
          (4, 16, 4, 512, 257), (16, 32, 4, 1024, 511), (1, 32, 1, 2048, 2047), (2, 48, 1, 256, 100), (3, 24, 3, 384, 128)]


@pytest.mark.parametrize("dt", [F32, F16, BF16])
@pytest.mark.parametrize("B,Hq,Hkv,S,pos", SHAPES)
def test_head64_attention_parity(K, B, Hq, Hkv, S, pos, dt):
    kc, vc, q, k, v = inputs(B, Hq, Hkv, S, dt)
    kc_ref, vc_ref = kc.copy(), vc.copy()
    ref = attention_kvcache_d(kc_ref, vc_ref, q, k, v, pos, dt)
    out, kc_got, vc_got = launch(K, kc, vc, q, k, v, pos, dt)
    close(out, ref, TOL[dt], TOL[dt] * 0.05)
    assert np.array_equal(kc_got, kc_ref) and np.array_equal(vc_got, vc_ref)  # append is bit-exact, rest untouched


@pytest.mark.parametrize("dt", [F32, F16, BF16])
@pytest.mark.parametrize("B,Hq,Hkv,S,poss", [(4, 8, 8, 256, [0, 37, 255, 128]), (3, 32, 4, 512, [511, 0, 130]),
                                             (5, 48, 1, 256, [200, 1, 255, 0, 129]), (16, 12, 12, 1024, None)])
def test_head64_attention_per_row_positions(K, B, Hq, Hkv, S, poss, dt):
    """ITB_POS_PER_ROW; ITB_POS_IN_STEP must not change a bit"""
    if poss is None:
        poss = np.random.default_rng(5).integers(0, S, size=B).tolist()
    kc, vc, q, k, v = inputs(B, Hq, Hkv, S, dt)
    kc_ref, vc_ref = kc.copy(), vc.copy()
    ref = attention_kvcache_d(kc_ref, vc_ref, q, k, v, poss, dt)
    out, kc_got, vc_got = launch(K, kc, vc, q, k, v, poss, dt)
    close(out, ref, TOL[dt], TOL[dt] * 0.05)
    assert np.array_equal(kc_got, kc_ref) and np.array_equal(vc_got, vc_ref)
    out2, kc2, vc2 = launch(K, kc, vc, q, k, v, poss, dt, flags=POS_IN_STEP)
    assert np.array_equal(out2, out) and np.array_equal(kc2, kc_got) and np.array_equal(vc2, vc_got)


def _rope64(K, dt, x, rope):
    """it_b200_rope with dim_head 64 on a device [B, H, 1, 64] tensor"""
    import torch
    y = torch.empty_like(x)
    B, H = x.shape[:2]
    K.L.check(K.L.lib.it_b200_rope(dt, K.ptr(rope), 7, K.ptr(x), K.ptr(y), B, 1, H * D, D, K.stream()))
    K.sync()
    return y


@pytest.mark.parametrize("dt", [F32, F16, BF16])
@pytest.mark.parametrize("B,Hq,Hkv,S,pos", [(3, 12, 12, 512, 257), (16, 32, 4, 1024, 511), (2, 48, 1, 256, 100),
                                           (4, 8, 8, 256, [0, 37, 255, 128])])
def test_head64_rope_folded_is_rope_then_attention(K, B, Hq, Hkv, S, pos, dt):
    """RoPE folded into the attention kernel gives exactly the bits of RoPE(dim_head 64) on q and k followed by the unfused
    kernel: output, k cache (the rotated k is appended) and v cache; RoPE positions differ per row and include 0 and 65535"""
    kc, vc, q, k, v = inputs(B, Hq, Hkv, S, dt)
    rope = np.array([(65535 if b == 1 else 3 * b + 7) if b else 0 for b in range(B)], np.int64)
    rd = K.raw(rope)
    qr = K.host(_rope64(K, dt, K.dev(q, dt), rd))
    kr = K.host(_rope64(K, dt, K.dev(k, dt), rd))
    ref = launch(K, kc, vc, qr, kr, v, pos, dt)
    got = launch(K, kc, vc, q, k, v, pos, dt, rope_pos=rope)
    for what, g, r in zip(("out", "k cache", "v cache"), got, ref):
        assert np.array_equal(g, r), f"{what}: {np.sum(g != r)} elements differ"


# ====================================================================== float64 per-element bound (tests/attn64.py's method)
class Case64:
    """attn64.Case at D = 64: q [B, Hq, 64], kseq / vseq [B, Hkv, S, 64], row pos_b the appended k / v; score regimes cycle
    over (batch row, query head)"""

    def __init__(self, B, Hq, Hkv, S, pos, seed, offset=0):
        self.B, self.Hq, self.Hkv, self.S, self.grp = B, Hq, Hkv, S, Hq // Hkv
        self.pos = np.clip(np.broadcast_to(np.asarray(pos, np.int64), (B,)), 0, S - 1)
        self.per_row = np.ndim(pos) > 0
        rng = np.random.default_rng(seed)
        g = self.grp
        self.q = np.empty((B, Hq, D), np.float32)
        self.kseq = np.full((B, Hkv, S, D), np.nan, np.float32)
        self.vseq = np.full((B, Hkv, S, D), np.nan, np.float32)
        self.regime = np.empty((B, Hq), object)
        vrow = np.exp2((np.arange(S) % 5) - 2.0)
        for b in range(B):
            n = int(self.pos[b]) + 1
            for kv in range(Hkv):
                qo, _ = np.linalg.qr(rng.standard_normal((D, g)))
                qg = attn64.exact(qo.T * math.sqrt(16.0)).astype(np.float64)  # |q|^2 = 16, as N(0, 0.5^2) draws of 64
                z = rng.standard_normal((n, D)) * 0.5
                kk = z.copy()
                for r in range(g):
                    h = kv * g + r
                    reg = attn64.REGIMES[(b * Hq + h + offset) % len(attn64.REGIMES)]
                    self.regime[b, h] = reg
                    for j, t in attn64.targets(reg, n - 1, rng).items():
                        kk[j] += (t * math.sqrt(D) - qg[r] @ z[j]) / (qg[r] @ qg[r]) * qg[r]
                self.q[b, kv * g:(kv + 1) * g] = qg
                self.kseq[b, kv, :n] = attn64.exact(kk)
                vv = rng.standard_normal((n, D)) * 0.5 * vrow[:n, None] * 2.0 ** ((kv % 3) - 1)
                self.vseq[b, kv, :n] = attn64.exact(vv)

    def caches(self):
        kc, vc = self.kseq.copy(), self.vseq.copy()
        kn = np.empty((self.B, self.Hkv, 1, D), np.float32)
        vn = np.empty_like(kn)
        for b in range(self.B):
            p = int(self.pos[b])
            kn[b, :, 0], vn[b, :, 0] = self.kseq[b, :, p], self.vseq[b, :, p]
            kc[b, :, p:] = np.nan
            vc[b, :, p:] = np.nan
        return kc, vc, kn, vn

    def reference(self, mutation=None, dt=F32):
        """float64 (ref, sum w|v|, sum w a |v - ref|, sum |v| / L), each [B, Hq, 64].  `mutation` builds instead the output of
        a kernel with one bug (what the bound must catch):
          scale128       the 128-wide kernel's 1/sqrt(128) kept at D = 64
          drop_append    the appended row left out of the softmax
          scores_in_t    q.k rounded to the storage type before the scale (the fp32 score is what the kernels keep)
          round_p_once   every weight rounded once to the storage type before P.V (no hi + lo split)"""
        sc = 1.0 / math.sqrt(128 if mutation == "scale128" else D)
        out = [np.empty((self.B, self.Hq, D)) for _ in range(4)]
        for b in range(self.B):
            n = int(self.pos[b]) + (0 if mutation == "drop_append" and self.pos[b] > 0 else 1)
            for kv in range(self.Hkv):
                hs = slice(kv * self.grp, (kv + 1) * self.grp)
                q = self.q[b, hs].astype(np.float64)
                k = self.kseq[b, kv, :n].astype(np.float64)
                v = self.vseq[b, kv, :n].astype(np.float64)
                dot = q @ k.T
                if mutation == "scores_in_t":
                    dot = oracle.round_to(dot.astype(np.float32), dt).astype(np.float64)
                s = dot * sc
                a = np.abs(q) @ np.abs(k).T * sc
                e = np.exp(s - s.max(1, keepdims=True))
                L = e.sum(1, keepdims=True)
                if mutation == "round_p_once":
                    e = oracle.round_to(e.astype(np.float32), dt).astype(np.float64)
                w = e / L
                ref = w @ v
                out[0][b, hs], out[1][b, hs] = ref, w @ np.abs(v)
                out[2][b, hs] = [(w[r] * a[r]) @ np.abs(v - ref[r]) for r in range(self.grp)]
                out[3][b, hs] = np.abs(v).sum(0)[None, :] / L
        return out


def _ctas_per_head(B, Hq, Hkv, S, pos, dt):
    """how many CTAs share each segment under the kernels' dealing at D = 64 (chunks of 16 KiB: 128 rows, fp32 64)"""
    ch = 16384 // (D * (4 if dt == F32 else 2))
    grp = Hq // Hkv
    segs = Hq if grp == 1 else Hkv * -(-grp // (16 if grp <= 16 else 32))
    posv = np.clip(np.broadcast_to(np.asarray(pos, np.int64), (B,)), 0, S - 1)
    nch = posv // ch + 1
    pre = np.concatenate([[0], np.cumsum(segs * nch)])
    total = int(pre[-1])
    ncta = min(total, B * segs * (S // ch + 1), attn64.GRID_MAX)
    shares = []
    for b in range(B):
        for s in range(segs):
            u0 = int(pre[b]) + s * int(nch[b])
            first, last = ((u0 + 1) * ncta - 1) // total, ((u0 + int(nch[b])) * ncta - 1) // total
            shares.append(last - first + 1)
    return shares


# one head over 128 (256 for fp32) CTAs; heads split two or three ways; whole heads; per-row positions; grouped-query with one
# and two query tiles, a group split over CTAs
F64_CASES = {
    "one_head_16k": (1, 1, 1, 16384, 16383),
    "gpt2_rows": (2, 12, 12, 4096, [4095, 1000]),
    "many_heads": (16, 12, 12, 512, 511),
    "ragged": (5, 4, 4, 2048, [0, 127, 128, 2047, 700]),
    "tinyllama_g8": (16, 32, 4, 1024, 511),
    "g8_split": (1, 8, 1, 8192, 8191),
    "g48_two_tiles": (3, 48, 1, 2048, [2047, 5, 1000]),
}


@pytest.mark.parametrize("dt", [F32, F16, BF16])
@pytest.mark.parametrize("case", list(F64_CASES))
def test_head64_attention_float64_bound(K, case, dt):
    B, Hq, Hkv, S, pos = F64_CASES[case]
    cs = Case64(B, Hq, Hkv, S, pos, seed=11)
    kc, vc, kn, vn = cs.caches()
    q = cs.q.reshape(B, Hq, 1, D)
    out, kc_got, vc_got = launch(K, kc, vc, q, kn, vn, pos, dt)
    got = out.reshape(B, Hq, D)
    refs = cs.reference()
    gqa = Hq != Hkv
    bad = attn64.violations(got, refs, dt, gqa)
    assert not bad.any(), f"{case}: {int(bad.sum())} of {bad.size} elements outside the float64 bound"
    for b in range(B):  # the append, bit for bit
        p = int(cs.pos[b])
        assert np.array_equal(kc_got[b, :, p], kn[b, :, 0]) and np.array_equal(vc_got[b, :, p], vn[b, :, 0])
    shares = _ctas_per_head(B, Hq, Hkv, S, pos, dt)
    if case in ("one_head_16k", "g8_split"):
        assert max(shares) >= 64  # the merge of many CTA partials is exercised
    # injected bugs the bound must catch (Case64.reference): the gross ones everywhere they apply; a score rounded to a 16-bit
    # type (2^-9 / 2^-12 of |s|) wherever several heads give it room to show; a weight rounded once to bf16 (2^-9)
    muts = ["scale128"] + (["drop_append"] if any(r == "append" for r in cs.regime.ravel()) else [])
    muts += (["scores_in_t"] if dt != F32 and B * Hq > 1 else []) + (["round_p_once"] if dt == BF16 else [])
    for m in muts:
        assert attn64.violations(cs.reference(m, dt)[0], refs, dt, gqa).any(), f"{case}: the bound misses {m}"


# ====================================================================== graphs
@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("mode", ["fused_cudagraph", "fused", "unfused"])
def test_tinyllama_graph_parity(dtype, mode):
    """two TinyLlama-width layers (32 query heads of 64 over 4 KV heads, ffn 5632) at B 16 against the oracle, positions
    127 and 128 (the second crosses the 128-row chunk boundary)"""
    from infinitensor_b200 import graphs as G
    cfg = G.LlamaConfig.tinyllama_1b(batch=16, s_max=256, dtype=dtype, layers=2)
    cfg.vocab = 2048
    env = {"ITB_NO_FUSION": "1"} if mode == "unfused" else None
    _, _, sched = run_llama_parity(cfg, pos=127, steps=2, cudagraph=mode == "fused_cudagraph", env=env)
    if mode != "unfused":
        assert sum(s.startswith("AttentionRope") for s in sched) == cfg.layers


def test_gpt2_decode_matches_forward():
    """GPT-2-width layers (12 heads of 64) at B 16: 136 decode steps from an empty cache, CUDA-graph replayed, reproduce the
    rows of build_gpt2's forward (prefill attention kernel) over the same tokens, past the 128-row chunk boundary"""
    from infinitensor_b200 import backend as B, graphs as G
    T = 136
    cfg = G.GPT2Config(layers=2, d_model=768, heads=12, ffn=3072, vocab=2048, n_pos=256, seq=T, batch=16, dtype=F16,
                       lm_head=True)
    rng = np.random.default_rng(7)
    ids = rng.integers(0, cfg.vocab, size=(cfg.batch, T)).astype(np.int64)
    rt = B.CudaRuntime(0)
    fh = B.GraphHandler(rt)
    fg = G.build_gpt2(fh, cfg)
    fh.data_malloc()
    G.fill_gpt2_weights_host(fg)
    fg.input_ids.copyin_numpy(ids)
    fg.position_ids.copyin_numpy(np.broadcast_to(np.arange(T, dtype=np.int64), (cfg.batch, T)).copy())
    fh.run()
    ref = G.from_storage(fg.out.copyout_numpy(), F16).astype(np.float64)  # [B, T, vocab]
    dh = B.GraphHandler(rt)
    dg = G.build_gpt2_decode(dh, cfg, 256)
    dh.data_malloc()
    G.fill_gpt2_weights_host(dg)
    for c in dg.k_caches + dg.v_caches:
        c.copyin_numpy(np.zeros(c.shape(), np.float16))
    worst = 0.0
    for t in range(T):
        dg.input_ids.copyin_numpy(ids[:, t:t + 1])
        dg.position_ids.copyin_numpy(np.full((cfg.batch, 1), t, np.int64))
        dh.run_with_cudagraph()
        got = G.from_storage(dg.out.copyout_numpy(), F16).astype(np.float64)[:, 0]
        err = np.abs(got - ref[:, t]).max() / np.abs(ref[:, t]).max()
        worst = max(worst, err)
        assert err < 2e-2, f"token {t}: rel-to-max error {err:.3e}"
    print(f"gpt2 decode vs forward: worst rel-to-max {worst:.3e}")
