#!/usr/bin/env python
"""Grouped-query decode attention on the GPU: kernel timing over KV head counts, and a Llama-3-8B-shape decode step.

  python tools/gqa_bench.py [--iters 100] [--steps 50] [--warmup 10] [--no-step] [--head-dim {64,128}]
                            [--model {llama3_8b,tinyllama_1b}]

Kernel: B 16, Hq 32, Hkv in {32, 8, 4, 1}, (S_max, p) in {(1024, 511), (4096, 4095)}, bf16, head width --head-dim, RoPE
folded off.  Launches are timed with CUDA events and rotate over enough cache buffers (>= 6, >= 256 MB in all) that the caches
are not L2-resident.  Algorithmic bytes: the K and V rows read (B Hkv 2 p D e), the appended rows (B Hkv 2 D e) and q / out
(B Hq 2 D e).  At --head-dim 64 the run also times, back to back, the streaming kernel at B 16, H 64, D 64 and at B 16, H 32,
D 128 (S_max 4096, p 4095): the same bytes, so the GB/s ratio is what the narrower rows cost.
Step: LlamaConfig.<model>() at p 511, CUDA-graph replay; the roofline is graphs.LlamaConfig.algorithmic_bytes over the
H100 SXM data-sheet 3.35 TB/s -- a bound computed from the shapes, not a measurement.  The card's name, power limit and
SM clock are printed from the same run."""
import argparse
import ctypes
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from infinitensor_b200 import _lib as L

HBM = 3.35e12  # bytes/s, H100 SXM data sheet
BF16 = 16


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "nvidia-smi unavailable"


def kernel_bytes(B, Hq, Hkv, p, e=2, D=128):
    return B * Hkv * 2 * p * D * e + B * Hkv * 2 * D * e + B * Hq * 2 * D * e


def time_kernel(B, Hq, Hkv, S, p, iters, D=128):
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    set_bytes = 2 * B * Hkv * S * D * 2
    nbuf = max(6, -(-(256 << 20) // set_bytes))
    caches = [(torch.randn(B, Hkv, S, D, device="cuda").bfloat16(), torch.randn(B, Hkv, S, D, device="cuda").bfloat16())
              for _ in range(nbuf)]
    q = torch.randn(B, Hq, 1, D, device="cuda").bfloat16()
    k = torch.randn(B, Hkv, 1, D, device="cuda").bfloat16()
    v = torch.randn(B, Hkv, 1, D, device="cuda").bfloat16()
    out = torch.empty_like(q)
    pos = torch.tensor([p], dtype=torch.int64, device="cuda")
    wsb = L.lib.it_b200_attention_kvcache_workspace(B, Hq, S, D)
    ws = torch.empty(max(int(wsb), 16), dtype=torch.uint8, device="cuda")
    P = lambda t: ctypes.c_void_p(t.data_ptr())

    def launch(i):
        kc, vc = caches[i % nbuf]
        L.check(L.lib.it_b200_attention_kvcache_gqa(BF16, P(kc), P(vc), P(q), P(k), P(v), P(pos), 7, None, 7, P(out), B, Hq,
                                                    Hkv, S, D, P(ws), int(wsb), st))

    for i in range(2 * nbuf):
        launch(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        launch(i)
    e1.record()
    e1.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / iters
    del caches
    torch.cuda.empty_cache()
    return us, nbuf


def time_step(steps, warmup, pos=511, model="llama3_8b"):
    from infinitensor_b200 import backend as B
    from infinitensor_b200 import graphs as G
    cfg = getattr(G.LlamaConfig, model)()
    rt = B.CudaRuntime(0)
    h = B.GraphHandler(rt)
    g = G.build_llama_decode(h, cfg)
    h.data_malloc()
    gen = torch.Generator(device="cuda")
    ts = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def fill(t, std, mean, seed):
        gen.manual_seed(seed)
        tmp = torch.empty(t.shape(), dtype=torch.bfloat16, device="cuda").normal_(mean, std, generator=gen)
        L.check(L.lib.it_b200_copy(ctypes.c_void_p(tmp.data_ptr()), ctypes.c_void_p(t.device_ptr()), t.nbytes(), ts))
        torch.cuda.current_stream().synchronize()

    for i, (name, (t, shape, kind, shard)) in enumerate(g.weights.items()):
        fill(t, 0.02, 1.0 if kind == "norm" else 0.0, 1000 + i)
    for li in range(cfg.layers):
        fill(g.k_caches[li], 0.5, 0.0, 5000 + li)
        fill(g.v_caches[li], 0.5, 0.0, 7000 + li)
    g.input_ids.copyin_numpy(np.random.default_rng(1).integers(0, cfg.vocab, size=(cfg.batch, 1)).astype(np.int64))
    g.position_ids.copyin_numpy(np.full((cfg.batch, 1), pos, np.int64))
    for _ in range(max(warmup, 3)):
        h.run_with_cudagraph()
    stream = torch.cuda.ExternalStream(rt.stream())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(stream)
    for _ in range(steps):
        h.launch_cudagraph_async()
    e1.record(stream)
    e1.synchronize()
    ms = e0.elapsed_time(e1) / steps
    byts = cfg.algorithmic_bytes(pos)
    sched = h.schedule()
    return cfg, ms, byts, sched


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--no-step", action="store_true")
    ap.add_argument("--head-dim", type=int, choices=(64, 128), default=128)
    ap.add_argument("--model", choices=("llama3_8b", "tinyllama_1b"), default="llama3_8b")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "gqa_bench needs a GPU"
    D = a.head_dim
    print(f"card: {card()}")
    print(f"{'B':>3} {'Hq':>3} {'Hkv':>3} {'D':>3} {'S_max':>5} {'p':>5} {'bufs':>4} {'us':>9} {'MB':>9} {'GB/s':>8} "
          f"{'of 3.35TB/s':>11}")
    res = {}

    def row(B, Hq, Hkv, S, p, d):
        us, nbuf = time_kernel(B, Hq, Hkv, S, p, a.iters, d)
        byts = kernel_bytes(B, Hq, Hkv, p, D=d)
        gbs = byts / us / 1e3
        print(f"{B:>3} {Hq:>3} {Hkv:>3} {d:>3} {S:>5} {p:>5} {nbuf:>4} {us:>9.2f} {byts / 1e6:>9.2f} {gbs:>8.1f} "
              f"{gbs * 1e9 / HBM:>10.1%}")
        return us, gbs

    for S, p in ((1024, 511), (4096, 4095)):
        for Hkv in (32, 8, 4, 1):
            res[(S, Hkv)] = row(16, 32, Hkv, S, p, D)
    print(f"p 511: Hkv 8 / Hkv 32 time = {res[(1024, 8)][0] / res[(1024, 32)][0]:.3f}; "
          f"p 4095: Hkv 8 / Hkv 32 GB/s = {res[(4096, 8)][1] / res[(4096, 32)][1]:.3f}")
    if D == 64:
        narrow, wide = row(16, 64, 64, 4096, 4095, 64), row(16, 32, 32, 4096, 4095, 128)
        print(f"same bytes, D 64 (H 64) / D 128 (H 32) GB/s = {narrow[1] / wide[1]:.3f}")
    if not a.no_step:
        cfg, ms, byts, sched = time_step(a.steps, a.warmup, model=a.model)
        print(f"{a.model} step (B {cfg.batch}, p 511, {cfg.layers} layers, {cfg.heads} q / {cfg.n_kv} kv heads of "
              f"{cfg.head_dim}, bf16, "
              f"CUDA graph, {a.steps} steps): {ms:.3f} ms/step, {cfg.batch / ms * 1e3:.0f} tok/s; algorithmic bytes "
              f"{byts / 1e9:.2f} GB -> bound {byts / HBM * 1e3:.2f} ms at 3.35 TB/s = {byts / HBM * 1e3 / ms:.1%} of roofline; "
              f"{sum(s.startswith('AttentionRope') for s in sched)} AttentionRope steps")
    print(f"card: {card()}")


if __name__ == "__main__":
    main()
