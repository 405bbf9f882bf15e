"""GPU parity of the persistent decode kernel (decode_stack.cu) through the C-ABI: chains of wgmma skinny GEMM phases
with the RMSNorm / Silu*Mul operand transforms and the residual epilogue, and the whole decoder-layer stack, against the
CPU oracle composed from the same operator sequence the graph executes (SURVEY 8(a) rows a1, a3, a6-a9).
Tolerances: SURVEY 8(c) -- GEMM abs <= 2^-8 (bf16) / 2^-11 (fp16) * sqrt(K) * max|a| * max|b|, end-to-end rel-to-max."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F16, BF16 = 10, 16
EPS = {F16: 2.0 ** -11, BF16: 2.0 ** -8}


@pytest.fixture(scope="module")
def K():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from tests import kernel_harness
    return kernel_harness


def rnd(shape, seed, dt, scale=1.0):
    import oracle
    return oracle.round_to(np.random.default_rng(seed).standard_normal(shape).astype(np.float32) * np.float32(scale), dt)


def chain(K, dt, rows, phases):
    """phases: list of dicts {W: [arrays], X, X2, residual, norm_w, xform, epi}; X may be an int = index of an earlier
    phase's output tensor (('out', phase, group)).  Returns the list of per-phase output lists (float32 numpy)."""
    import torch
    from infinitensor_b200 import _lib as L
    dev = K.dev
    outs_dev, keep = [], []
    Wp, Op, ng, npg, Ks, xf, ep, Xp, X2p, Rp, Np = [], [], [], [], [], [], [], [], [], [], []

    def resolve(v):
        if v is None:
            return None
        if isinstance(v, tuple):
            return outs_dev[v[1]][v[2]]
        t = dev(v, dt)
        keep.append(t)
        return t
    for ph in phases:
        ws = [dev(w, dt) for w in ph["W"]]
        keep += ws
        k, n = ph["W"][0].shape
        os_ = [torch.zeros((rows, n), dtype=K.TORCH_DT[dt], device="cuda") for _ in ws]
        outs_dev.append(os_)
        Wp += [w.data_ptr() for w in ws]
        Op += [o.data_ptr() for o in os_]
        ng.append(len(ws)); npg.append(n); Ks.append(k); xf.append(ph.get("xform", 0)); ep.append(ph.get("epi", 0))
        x, x2, r, nw = resolve(ph["X"]), resolve(ph.get("X2")), resolve(ph.get("residual")), resolve(ph.get("norm_w"))
        Xp.append(x.data_ptr()); X2p.append(x2.data_ptr() if x2 is not None else None)
        Rp.append(r.data_ptr() if r is not None else None); Np.append(nw.data_ptr() if nw is not None else None)
    ws_bytes = 64 << 20
    wsb = torch.zeros(ws_bytes, dtype=torch.uint8, device="cuda")
    VP = ctypes.c_void_p
    arr = lambda v: (VP * len(v))(*v)
    for _ in range(2):  # second launch: self-cleaning tickets, cached program
        L.check(L.lib.it_b200_decode_gemm_chain(dt, rows, len(phases), L.i32arr(ng), arr(Wp), arr(Op), L.i32arr(npg), L.i32arr(Ks),
                                                L.i32arr(xf), L.i32arr(ep), arr(Xp), arr(X2p), arr(Rp), arr(Np),
                                                VP(wsb.data_ptr()), ws_bytes, K.stream()))
        K.sync()
    return [[K.host(o) for o in os_] for os_ in outs_dev]


def gemm_tol(dt, k, amax, bmax):
    return EPS[dt] * np.sqrt(k) * amax * bmax + 1e-6


@pytest.mark.parametrize("dt", [BF16, F16])
@pytest.mark.parametrize("rows,k,n", [(16, 4096, 4096), (16, 512, 1024), (5, 4096, 11008), (16, 11008, 4096), (16, 4096, 32000),
                                      (1, 64, 128), (16, 1000, 136), (16, 200, 8)])
def test_chain_single_gemm(K, rows, k, n, dt):
    import oracle
    x, w = rnd((rows, k), 1, dt, 0.5), rnd((k, n), 2, dt, 0.05)
    got = chain(K, dt, rows, [dict(W=[w], X=x)])[0][0]
    ref = oracle.matmul(x, w, None, False, False, dt)
    assert np.abs(got - ref).max() <= 2 * EPS[dt] * np.abs(ref).max() + gemm_tol(dt, k, np.abs(x).max(), np.abs(w).max())


@pytest.mark.parametrize("dt", [BF16, F16])
def test_chain_grouped_rmsnorm_and_residual(K, dt):
    """[RMSNorm ->] three weight matrices sharing X (q/k/v shape), then a residual-epilogue GEMM on one of the outputs."""
    import oracle
    rows, d = 16, 1024
    x, nw = rnd((rows, d), 3, dt, 1.0), rnd((d,), 4, dt, 0.1) + 1
    nw = oracle.round_to(nw, dt)
    ws = [rnd((d, d), 5 + i, dt, 0.03) for i in range(3)]
    wo, res = rnd((d, d), 9, dt, 0.03), rnd((rows, d), 10, dt, 1.0)
    got = chain(K, dt, rows, [dict(W=ws, X=x, xform=1, norm_w=nw),
                              dict(W=[wo], X=("out", 0, 0), epi=1, residual=res)])
    xn = oracle.rms_norm(x, nw, dt)
    refs = [oracle.matmul(xn, w, None, False, False, dt) for w in ws]
    for g_, r_ in zip(got[0], refs):
        assert np.abs(g_ - r_).max() <= 2 * EPS[dt] * np.abs(r_).max() + gemm_tol(dt, d, np.abs(xn).max(), 0.15)
    o = oracle.matmul(refs[0], wo, None, False, False, dt)
    ref2 = oracle.binary("add", res, o, dt)
    assert np.abs(got[1][0] - ref2).max() <= 4 * EPS[dt] * np.abs(ref2).max() + gemm_tol(dt, d, np.abs(refs[0]).max(), 0.15)


@pytest.mark.parametrize("dt", [BF16])
@pytest.mark.parametrize("rows,d,f", [(16, 1024, 2816), (16, 4096, 11008), (7, 512, 1408)])
def test_chain_mlp_half_layer(K, rows, d, f, dt):
    """o-proj + residual -> [RMSNorm from the epilogue's per-tile sums of squares] gate / up -> [Silu * Mul] down + residual:
    three grid barriers, both operand transforms, the ss hand-over between phases."""
    import oracle
    a, x0 = rnd((rows, d), 11, dt, 0.5), rnd((rows, d), 12, dt, 1.0)
    wo, wg, wu, wd = rnd((d, d), 13, dt, 0.02), rnd((d, f), 14, dt, 0.02), rnd((d, f), 15, dt, 0.02), rnd((f, d), 16, dt, 0.02)
    nw = oracle.round_to(rnd((d,), 17, dt, 0.1) + 1, dt)
    got = chain(K, dt, rows, [dict(W=[wo], X=a, epi=1, residual=x0),
                              dict(W=[wg, wu], X=("out", 0, 0), xform=1, norm_w=nw),
                              dict(W=[wd], X=("out", 1, 0), X2=("out", 1, 1), xform=2, epi=1, residual=("out", 0, 0))])
    x1 = oracle.binary("add", x0, oracle.matmul(a, wo, None, False, False, dt), dt)
    hn = oracle.rms_norm(x1, nw, dt)
    g_, u_ = oracle.matmul(hn, wg, None, False, False, dt), oracle.matmul(hn, wu, None, False, False, dt)
    m = oracle.binary("mul", oracle.unary("silu", g_, dt), u_, dt)
    x2 = oracle.binary("add", x1, oracle.matmul(m, wd, None, False, False, dt), dt)
    rel = lambda got_, ref_: np.abs(got_ - ref_).max() / np.abs(ref_).max()
    assert rel(got[0][0], x1) < 2e-2 and rel(got[1][0], g_) < 3e-2 and rel(got[1][1], u_) < 3e-2
    assert rel(got[2][0], x2) < 3e-2


@pytest.mark.parametrize("dt", [BF16, F16])
@pytest.mark.parametrize("B,layers,d,H,f,S,pos", [(16, 2, 512, 4, 1408, 128, 37), (4, 1, 256, 2, 512, 64, 0), (16, 2, 1024, 8, 2816, 256, [3, 200, 64, 0, 255, 17, 128, 90, 1, 2, 3, 4, 5, 6, 7, 8]),
                                                  (16, 1, 4096, 32, 11008, 1024, 511)])
def test_llama_decode_stack_vs_oracle(K, B, layers, d, H, f, S, pos, dt):
    """The whole persistent kernel against the CPU oracle executing the operator graph (graphs.build_llama_decode): the
    residual stream leaving the last layer, every appended cache row bit-exact."""
    import torch
    from infinitensor_b200 import _lib as L, graphs as G
    from oracle.graph_oracle import OracleHandler
    assert d == H * 128
    cfg = G.LlamaConfig(layers=layers, d_model=d, heads=H, head_dim=128, ffn=f, vocab=64, s_max=S, batch=B, dtype=dt)
    oh = OracleHandler()
    g = G.build_llama_decode(oh, cfg)
    G.fill_llama_weights_host(g)
    caches = []
    for li in range(layers):
        kc, vc = G.llama_cache_values(cfg, li, "k"), G.llama_cache_values(cfg, li, "v")
        g.k_caches[li].copyin_numpy(G.to_storage(kc, dt)); g.v_caches[li].copyin_numpy(G.to_storage(vc, dt))
        caches.append((g.k_caches[li].f32().copy(), g.v_caches[li].f32().copy()))
    per_row = isinstance(pos, list)
    posv = np.asarray(pos if per_row else [pos] * B, np.int64).reshape(B, 1)
    if per_row:
        pytest.skip("per-row positions: covered through the graph API")  # the graph builder has no per-row switch yet
    ids = (np.arange(B, dtype=np.int64).reshape(-1, 1) * 5 + 1) % cfg.vocab
    g.input_ids.copyin_numpy(ids); g.position_ids.copyin_numpy(posv)
    oh.run()
    final_norm_op = oh.ops[-2]
    x_ref = np.asarray(final_norm_op[1][0].f32()).reshape(B, d)
    x0 = np.asarray(oh.ops[0][2][0].f32()).reshape(B, d)   # embedding rows = the stack's input

    dev, TD = K.dev, K.TORCH_DT[dt]
    keep = []
    def W(name):
        t = dev(g.weights[name][0].f32(), dt); keep.append(t); return t.data_ptr()
    def buf(*shape):
        t = torch.zeros(shape, dtype=TD, device="cuda"); keep.append(t); return t
    arr = (L.LlamaLayer * layers)()
    kcs, vcs, xouts = [], [], []
    for li in range(layers):
        p = f"l{li}."
        kc, vc = dev(caches[li][0], dt), dev(caches[li][1], dt)
        kcs.append(kc); vcs.append(vc)
        xo = buf(B, d); xouts.append(xo)
        vals = dict(ln1_w=W(p + "ln1"), wq=W(p + "wq"), wk=W(p + "wk"), wv=W(p + "wv"), wo=W(p + "wo"), ln2_w=W(p + "ln2"),
                    wg=W(p + "wg"), wu=W(p + "wu"), wd=W(p + "wd"), k_cache=kc.data_ptr(), v_cache=vc.data_ptr(),
                    q=buf(B, d).data_ptr(), k=buf(B, d).data_ptr(), v=buf(B, d).data_ptr(), attn_out=buf(B, d).data_ptr(),
                    x_mid=buf(B, d).data_ptr(), gate=buf(B, f).data_ptr(), up=buf(B, f).data_ptr(), x_out=xo.data_ptr())
        for k_, v_ in vals.items():
            setattr(arr[li], k_, v_)
    xin = dev(x0, dt)
    pd = K.raw(posv)
    wsb = int(L.lib.it_b200_decode_stack_workspace(layers, B, d, H, S, f))
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    L.check(L.lib.it_b200_llama_decode_stack(dt, layers, ctypes.cast(arr, ctypes.c_void_p), K.ptr(xin), K.ptr(pd), 7, K.ptr(pd), 7,
                                             B, d, H, S, f, K.ptr(ws), wsb, K.stream()))
    K.sync()
    got = K.host(xouts[-1])
    err = np.abs(got - x_ref).max() / np.abs(x_ref).max()
    assert err < (3e-2 if dt == BF16 else 4e-3), f"rel-to-max {err:.3e}"
    # appended rows: the rotated k and v of this step, everything else untouched
    for li in range(layers):
        kref, vref = np.asarray(g.k_caches[li].f32()), np.asarray(g.v_caches[li].f32())
        kg, vg = K.host(kcs[li]), K.host(vcs[li])
        p0 = int(posv[0, 0])
        mask = np.ones(kref.shape, bool); mask[:, :, p0, :] = False
        assert np.array_equal(kg[mask], kref[mask]) and np.array_equal(vg[mask], vref[mask])
        assert np.abs(kg[:, :, p0] - kref[:, :, p0]).max() <= 8 * EPS[dt] * np.abs(kref[:, :, p0]).max()
        assert np.abs(vg[:, :, p0] - vref[:, :, p0]).max() <= 8 * EPS[dt] * np.abs(vref[:, :, p0]).max()
