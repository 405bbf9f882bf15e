"""Launch accounting: it_b200_launch_count() is the launches-per-step figure bench.py reports, so every C-ABI launcher must count
exactly the kernels it puts on the stream.

* GPU: one warmed-up call of each launcher family inside one torch.profiler session (in a child process, as the float64 files
  run their profiler checks); per call, the change in it_b200_launch_count() equals the kernel records the profiler saw
  (memset / memcpy records excluded).  Calls are separated by a marker fill kernel, so the records split by call.
* CPU: every launch in csrc/kernels goes through itb::launch (common.cuh), which sets the launch attributes, opts in the
  shared memory and counts: no other file launches, opts in or counts by hand."""
import ctypes
import json
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNELS = os.path.join(ROOT, "infinitensor_b200", "csrc", "kernels")
F32, F16, BF16, I64 = 1, 10, 16, 7


def test_launches_only_through_the_launcher():
    bad = []
    for f in sorted(os.listdir(KERNELS)):
        if f in ("common.cuh", "support.cu") or not f.endswith((".cu", ".cuh")):
            continue
        for i, line in enumerate(open(os.path.join(KERNELS, f)), 1):
            if re.search(r"cudaLaunchKernelEx|cudaLaunchConfig_t|cudaFuncSetAttribute|count_launch|<<<", line):
                bad.append(f"{f}:{i}: {line.strip()}")
    assert not bad, "launch by hand outside common.cuh / support.cu:\n" + "\n".join(bad)


def launcher_calls():
    """[(family, call)]: each call issues one C-ABI launch on buffers allocated here, and returns its rc"""
    import torch
    from infinitensor_b200 import _lib as L
    lib, keep = L.lib, []
    VP = ctypes.c_void_p
    st = lambda: VP(torch.cuda.current_stream().cuda_stream)

    def t(shape, dt=F32, fill=0.5):
        x = torch.full(shape, fill, dtype={F32: torch.float32, F16: torch.float16, BF16: torch.bfloat16}[dt], device="cuda")
        keep.append(x)
        return x

    def u8(n, fill=0x38):
        x = torch.full((n,), fill, dtype=torch.uint8, device="cuda")
        keep.append(x)
        return x

    def i64(vals):
        x = torch.tensor(vals, dtype=torch.int64, device="cuda")
        keep.append(x)
        return x

    p = lambda x: VP(x.data_ptr()) if x is not None else None
    arr = lambda xs: (VP * len(xs))(*[x.data_ptr() if x is not None else 0 for x in xs])
    i64a, i32a = L.i64arr, L.i32arr
    calls = []

    def add(name):
        return lambda f: calls.append((name, f))

    x, y = t((64, 64)), t((64, 64))
    add("unary")(lambda: lib.it_b200_unary(0, F32, p(x), p(y), 4096, st()))
    add("binary")(lambda: lib.it_b200_binary(0, F32, p(x), p(x), p(y), 2, i64a([64, 64]), i64a([64, 1]), i64a([64, 1]), st()))
    h = t((64, 64), F16)
    add("cast")(lambda: lib.it_b200_cast(F32, F16, p(x), p(h), 4096, st()))
    c = u8(4096, 1)
    add("where")(lambda: lib.it_b200_where(4, p(c), p(x), p(x), p(y), 2, i64a([64, 64]), i64a([64, 1]), i64a([64, 1]),
                                           i64a([64, 1]), st()))
    add("expand")(lambda: lib.it_b200_expand(4, p(x), p(y), 2, i64a([64, 64]), i64a([0, 1]), st()))
    add("copy")(lambda: lib.it_b200_copy(p(x), p(y), 4096 * 4, st()))
    add("transpose")(lambda: lib.it_b200_transpose(4, p(x), p(y), 2, i64a([32, 128]), i32a([1, 0]), st()))
    parts = [t((4, 2)) for _ in range(40)]
    joined = t((4, 80))
    add("concat (40 parts: two launches)")(lambda: lib.it_b200_concat(4, 40, arr(parts), i64a([2] * 40), p(joined), 4, 1, st()))
    add("split")(lambda: lib.it_b200_split(4, 3, arr(parts[:3]), i64a([2] * 3), p(joined), 4, 1, st()))
    idx = i64([3, 0, 7, 1, 5])
    add("gather")(lambda: lib.it_b200_gather(4, I64, p(x), p(idx), p(y), 1, 64, 64, 5, st()))
    add("pad_slice")(lambda: lib.it_b200_pad_slice(4, p(x), p(y), 2, i64a([64, 64]), i64a([16, 16]), i64a([1, 1]), i64a([2, 2]),
                                                   st()))
    add("reduce")(lambda: lib.it_b200_reduce(F32, 1, p(x), p(y), 3, i64a([8, 16, 32]), i32a([0, 1, 0]), st()))
    img, pooled = t((2, 4, 16, 16)), t((2, 4, 8, 8))
    add("pool2d")(lambda: lib.it_b200_pool2d(F32, 1, p(img), p(pooled), 2, 4, 16, 16, 3, 3, 1, 1, 1, 1, 2, 2, 8, 8, st()))
    nhwc, nhwc_out = t((2, 8, 8, 16), F16), t((2, 4, 4, 16), F16)
    add("pool2d_nhwc 3x3")(lambda: lib.it_b200_pool2d_nhwc(F16, 1, p(nhwc), p(nhwc_out), 2, 16, 8, 8, 3, 3, 1, 1, 1, 1, 2, 2, 4, 4,
                                                           st()))
    add("pool2d_nhwc global average")(lambda: lib.it_b200_pool2d_nhwc(F16, 0, p(nhwc), p(nhwc_out), 2, 16, 8, 8, 8, 8, 1, 1, 0, 0, 1,
                                                                      1, 1, 1, st()))
    bn = [t((4,), F32, v) for v in (0.1, 1.0, 1.5, 0.2)]
    bn_out = t((2, 4, 16, 16))
    add("batchnorm")(lambda: lib.it_b200_batchnorm(F32, p(img), *[p(v) for v in bn], p(bn_out), 2, 4, 256, 1e-5, st()))
    rows, rows_out = t((4, 12288)), t((4, 12288))
    add("softmax (row in shared memory)")(lambda: lib.it_b200_softmax(F32, p(rows), p(rows_out), 4, 12288, 1, st()))
    ln_w = t((768,))
    add("layernorm")(lambda: lib.it_b200_layernorm(F32, p(rows), p(ln_w), p(ln_w), p(rows_out), 8, 768, 1, 768, 768, 1e-5, st()))
    hb, hb_out, wb = t((4, 4096), BF16), t((4, 4096), BF16), t((4096,), BF16)
    add("rmsnorm")(lambda: lib.it_b200_rmsnorm(BF16, p(hb), p(wb), p(hb_out), 4, 4096, st()))
    pos = i64([5, 9, 11, 300])
    add("rope")(lambda: lib.it_b200_rope(BF16, p(pos), I64, p(hb), p(hb_out), 4, 1, 4096, 128, st()))
    add("silu_mul")(lambda: lib.it_b200_silu_mul(BF16, p(hb), p(hb), p(hb_out), 4 * 4096, st()))

    m, n, k = 16, 256, 512
    a, w, cm = t((128, k), BF16), t((k, n), BF16), t((128, n), BF16)
    for impl, kname in ((1, "skinny"), (2, "wgmma"), (3, "simt")):
        def pinned(impl=impl):
            lib.it_b200_matmul_select(impl, 0)
            try:
                return lib.it_b200_matmul(BF16, p(a), p(w), None, p(cm), 1, m, n, k, m * k, k * n, 0, 0, 0, 0, 0, 0, None, 0, st())
            finally:
                lib.it_b200_matmul_select(0, 0)
        add(f"matmul pinned to {kname}")(pinned)
    ws3, cs3 = [t((k, n), BF16) for _ in range(3)], [t((m, n), BF16) for _ in range(3)]
    add("matmul_grouped")(lambda: lib.it_b200_matmul_grouped(BF16, p(a), 3, arr(ws3), arr(cs3), i32a([n] * 3), m, k, st()))
    bias = t((n,), BF16)
    add("matmul_fused")(lambda: lib.it_b200_matmul_fused(BF16, p(a), p(w), p(bias), None, p(cm), 1, 128, n, k, 128 * k, 0, 0, 0, 0, 0,
                                                         1, 1 | 0x200, st()))
    w8, s8 = u8(k * n), t((n,), F32, 0.01)
    add("matmul_fp8w")(lambda: lib.it_b200_matmul_fp8w(BF16, p(a), 1, arr([w8]), arr([s8]), arr([cm]), i32a([n]), m, k, None, st()))
    w4, s4 = u8(n * k // 2, 0x98), t((n, k // 32), BF16, 0.01)
    for rows_m in (16, 128):
        nb = i32a([n])
        wsb = int(lib.it_b200_matmul_nbits_workspace(BF16, rows_m, k, 1, nb))
        ws4 = u8(max(wsb, 16))
        add(f"matmul_nbits m={rows_m}")(lambda rows_m=rows_m, nb=nb, wsb=wsb, ws4=ws4: lib.it_b200_matmul_nbits(
            BF16, p(a), 1, arr([w4]), arr([s4]), None, arr([cm]), nb, rows_m, k, 32, None, p(ws4), wsb, st()))

    # convs: the folded im2col GEMM with padded filters (im2col, pad, GEMM), the implicit-GEMM kernel with its repack, the stem
    cx, cw, cy = t((2, 3, 16, 16), F16), t((16, 3, 7, 7), F16), t((2, 16, 8, 8), F16)
    conv = (2, 3, 16, 16, 16, 7, 7, 3, 3, 2, 2, 1, 1, 1)
    cwsb = int(lib.it_b200_conv2d_workspace(F16, *conv))
    cws = u8(max(cwsb, 16))
    add("conv2d")(lambda: lib.it_b200_conv2d(F16, p(cx), p(cw), p(cy), *conv, p(cws), cwsb, st()))
    cbn = [t((16,), F32, v) for v in (0.1, 1.0, 1.5, 0.2)]
    add("conv2d_fused")(lambda: lib.it_b200_conv2d_fused(F16, p(cx), p(cw), p(cy), *conv, *[p(v) for v in cbn], 1e-5, None, 1, p(cws),
                                                         cwsb, st()))
    nx, nw, ny = t((2, 8, 8, 16), F16), t((16, 16, 3, 3), F16), t((2, 8, 8, 16), F16)
    nwsb = int(lib.it_b200_conv2d_nhwc_workspace(F16, 16, 16, 3, 3))
    nws = u8(max(nwsb, 16))
    add("conv2d_nhwc (repack and conv)")(lambda: lib.it_b200_conv2d_nhwc(
        F16, p(nx), p(nw), p(ny), 1, 2, 16, 8, 8, 16, 3, 3, 1, 1, 1, 1, 1, 1, *[p(v) for v in cbn], 1e-5, None, 1, p(nws), nwsb, st()))
    sx, sw, sy = t((2, 3, 32, 32), F16), t((64, 3, 7, 7), F16), t((2, 16, 16, 64), F16)
    add("conv2d_stem")(lambda: lib.it_b200_conv2d_stem(F16, p(sx), p(sw), p(sy), 2, 3, 32, 32, 64, 7, 7, 3, 3, 2, 2,
                                                       *[None] * 4, 1e-5, 0, st()))
    add("conv_repack_filters")(lambda: lib.it_b200_conv_repack_filters(F16, 1, arr([nw]), arr([nws]), i32a([16]), i32a([16]),
                                                                       i32a([3]), i32a([3]), st()))

    B, H, S, D = 2, 2, 64, 64
    qkv, att = t((B, S, 3 * H * D), BF16, 0.1), t((B, S, H * D), BF16)
    q3 = [t((B, H, S, D), BF16, 0.1) for _ in range(3)]
    add("attention_prefill")(lambda: lib.it_b200_attention_prefill(BF16, *[p(v) for v in q3], p(att), B, H, S, S, D, None, 0, None,
                                                                   0, 0, 0, 0, st()))
    es, d = 2, H * D
    view, ost = i64a([S * 3 * d, D, 3 * d]), i64a([S * d, D, d])
    add("attention_prefill_strided")(lambda: lib.it_b200_attention_prefill_strided(
        BF16, VP(qkv.data_ptr()), VP(qkv.data_ptr() + d * es), VP(qkv.data_ptr() + 2 * d * es), p(att), B, H, S, S, D, view, view, view,
        ost, None, 0, None, 0, 0, 0, 0, st()))

    Bk, Hq, Hkv, Smax, Dk = 2, 8, 2, 256, 128
    kc, vc = t((Bk, Hq, Smax, Dk), BF16, 0.1), t((Bk, Hq, Smax, Dk), BF16, 0.1)
    qd, kd, od = t((Bk, Hq, 1, Dk), BF16, 0.1), t((Bk, Hq, 1, Dk), BF16, 0.1), t((Bk, Hq, 1, Dk), BF16)
    p0 = i64([100])
    kwsb = int(lib.it_b200_attention_kvcache_workspace(Bk, Hq, Smax, Dk))
    kws = u8(kwsb)
    add("attention_kvcache")(lambda: lib.it_b200_attention_kvcache(BF16, p(kc), p(vc), p(qd), p(kd), p(kd), p(p0), I64, p(od), Bk, Hq,
                                                                   Smax, Dk, p(kws), kwsb, st()))
    add("attention_kvcache_gqa")(lambda: lib.it_b200_attention_kvcache_gqa(BF16, p(kc), p(vc), p(qd), p(kd), p(kd), p(p0), I64, None,
                                                                           0, p(od), Bk, Hq, Hkv, Smax, Dk, p(kws), kwsb, st()))
    k8, v8, sc8 = u8(Bk * Hkv * Smax * Dk), u8(Bk * Hkv * Smax * Dk), t((Hq,), F32, 0.01)
    add("attention_kvcache_fp8")(lambda: lib.it_b200_attention_kvcache_fp8(BF16, p(k8), p(v8), p(sc8), p(sc8), p(qd), p(kd), p(kd),
                                                                           p(p0), I64, None, 0, p(od), Bk, Hq, Hkv, Smax, Dk, p(kws),
                                                                           kwsb, st()))
    Sp = 65
    qp, kp, op = t((Bk, Hq, Sp, Dk), BF16, 0.1), t((Bk, Hkv, Sp, Dk), BF16, 0.1), t((Bk, Hq, Sp, Dk), BF16)
    add("attention_kvcache_prompt (append and attention)")(lambda: lib.it_b200_attention_kvcache_prompt(
        BF16, p(kc), p(vc), p(qp), p(kp), p(kp), p(p0), I64, p(op), Bk, Hq, Hkv, Sp, Smax, Dk, st()))
    return calls, keep


def counted_and_profiled():
    """{family: [launches counted, kernel records profiled]} for one warmed-up call of each family"""
    import torch
    from infinitensor_b200 import _lib as L
    calls, keep = launcher_calls()
    for name, f in calls:
        assert f() == 0, f"{name}: {L.last_error()}"
    torch.cuda.synchronize()
    mark = torch.zeros(1, device="cuda")
    counted = []
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for i, (name, f) in enumerate(calls):
            mark.fill_(i)
            torch.cuda.synchronize()
            n0 = L.lib.it_b200_launch_count()
            assert f() == 0, f"{name}: {L.last_error()}"
            counted.append(L.lib.it_b200_launch_count() - n0)
            torch.cuda.synchronize()
        mark.fill_(len(calls))
        torch.cuda.synchronize()
    kernels = sorted((e.time_range.start, e.name) for e in prof.events()
                     if "CUDA" in str(e.device_type) and not e.name.startswith(("Memset", "Memcpy")))
    seen = []
    for _, kname in kernels:
        if "FillFunctor" in kname:
            seen.append(0)
        elif seen:
            seen[-1] += 1
    if not kernels:
        return {}
    assert len(seen) == len(calls) + 1, f"{len(seen)} markers for {len(calls)} calls"
    return {name: [counted[i], seen[i]] for i, (name, _) in enumerate(calls)}


@pytest.mark.gpu
def test_launch_count_matches_profiled_kernels():
    code = ("import json; from tests.test_launch_accounting import counted_and_profiled as f; print(json.dumps(f()))")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    if not got:
        pytest.skip("the profiler recorded no CUDA kernel events (CUPTI activity tracing unavailable)")
    wrong = {name: cp for name, cp in got.items() if cp[0] != cp[1]}
    assert not wrong, f"[launches counted, kernels profiled] differ: {wrong}"
    assert all(cp[1] >= 1 for cp in got.values()), got
