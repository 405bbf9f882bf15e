#!/usr/bin/env python
"""Micro-benchmark of the decode GEMM kernels through the C-ABI (CUDA events, rotating weights >> L2).
   python tools/gemm_bench.py [impl ...]      impl in {skinny, tc}"""
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from infinitensor_b200 import _lib as L

SHAPES = [(16, 4096, 4096), (16, 4096, 11008), (16, 11008, 4096), (16, 4096, 32000), (16, 4096, 12288), (16, 4096, 22016)]


def run(impl, m, k, n, reps=40, nbuf=12):
    nbuf = max(2, min(nbuf, int(1.5e9 / (k * n * 2))))
    if impl == "cublas":  # what the reference's matmulCublas dispatches to (matmul.cc:141-168), through torch.matmul
        ws = [torch.randn(k, n, device="cuda", dtype=torch.bfloat16) * 0.02 for _ in range(nbuf)]
        x = torch.randn(m, k, device="cuda", dtype=torch.bfloat16)
        y = torch.empty(m, n, device="cuda", dtype=torch.bfloat16)
        for i in range(nbuf):
            torch.matmul(x, ws[i], out=y)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(reps):
            torch.matmul(x, ws[i % nbuf], out=y)
        e1.record()
        e1.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / reps
        return us, (k * n + m * (k + n)) * 2 / 1e9 / (us * 1e-6)
    L.lib.it_b200_matmul_select({"skinny": 1, "tc": 2, "simt": 3}[impl], 0)
    ws = [torch.randn(k, n, device="cuda", dtype=torch.bfloat16) * 0.02 for _ in range(nbuf)]
    x = torch.randn(m, k, device="cuda", dtype=torch.bfloat16)
    y = torch.empty(m, n, device="cuda", dtype=torch.bfloat16)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def go(i):
        L.check(L.lib.it_b200_matmul(16, ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(ws[i % nbuf].data_ptr()), None,
                                     ctypes.c_void_p(y.data_ptr()), 1, m, n, k, m * k, 0, 0, 0, 0, 0, 0, 0x200, None, 0, st))
    for i in range(nbuf):
        go(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(reps):
        go(i)
    e1.record()
    e1.synchronize()
    L.lib.it_b200_matmul_select(0, 0)
    us = e0.elapsed_time(e1) * 1e3 / reps
    gb = (k * n + m * (k + n)) * 2 / 1e9
    return us, gb / (us * 1e-6)


if __name__ == "__main__":
    if os.environ.get("GEMM_BENCH_SHAPES"):  # "m,k,n;m,k,n;..."
        SHAPES = [tuple(int(v) for v in t.split(",")) for t in os.environ["GEMM_BENCH_SHAPES"].split(";")]
    impls = sys.argv[1:] or ["skinny", "tc"]
    print(f"{'shape':>22s} " + " ".join(f"{i:>22s}" for i in impls))
    for (m, k, n) in SHAPES:
        row = []
        for impl in impls:
            us, gbs = run(impl, m, k, n)
            row.append(f"{us:8.2f} us {gbs:7.0f} GB/s")
        print(f"{str((m, k, n)):>22s} " + " ".join(f"{r:>22s}" for r in row), flush=True)
