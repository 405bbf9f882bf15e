#!/usr/bin/env python
"""FP8 E4M3 KV cache against the 16-bit cache on the GPU: decode attention kernel time and whole Llama decode steps.

  python tools/kvfp8_bench.py [--iters 100] [--steps 30] [--warmup 5] [--no-step]

Kernel: B 16, Hq 32, Hkv in {32, 8, 4, 1}, (S_max, p) in {(1024, 511), (4096, 4095)}, D 128, bf16 activations, RoPE off;
it_b200_attention_kvcache_gqa on a bf16 cache and it_b200_attention_kvcache_fp8 on an FP8 cache, timed alternately in the
same run with CUDA events over enough cache buffers (>= 6, >= 256 MB in all) that the caches are not L2-resident.
Algorithmic bytes: the K and V rows read and appended at e bytes per element (2, or 1 for FP8), q / out at 2, and the two
4-byte scales per KV head.  GB/s is those bytes over kernel time.
Steps: LlamaConfig.llama3_8b() at p 511 and a Llama-7B shape at S_max 4096, p 4095, B 16, each with the 16-bit and the FP8
cache, CUDA-graph replay; the roofline is LlamaConfig.algorithmic_bytes over the H100 SXM data-sheet 3.35 TB/s -- a bound
computed from the shapes, not a measurement.  The card's name, power limit and SM clock are printed from the same run."""
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
D = 128


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "nvidia-smi unavailable"


def kernel_bytes(B, Hq, Hkv, p, fp8):
    e = 1 if fp8 else 2
    return B * Hkv * 2 * (p + 1) * D * e + B * Hq * 2 * D * 2 + B * Hkv * 2 * D * 2 + (Hkv * 8 if fp8 else 0)


def fp8_codes(shape, std=0.5):
    """random cache codes (values N(0, std^2) / scale, scale 4 std / 448)"""
    x = torch.randn(shape, device="cuda") * (448.0 / 4.0)
    return x.to(torch.float8_e4m3fn).view(torch.uint8)


class Kernel:
    def __init__(self, B, Hq, Hkv, S, p, fp8):
        self.B, self.Hq, self.Hkv, self.S, self.fp8 = B, Hq, Hkv, S, fp8
        e = 1 if fp8 else 2
        set_bytes = 2 * B * Hkv * S * D * e
        self.nbuf = max(6, -(-(256 << 20) // set_bytes))
        mk = (lambda: fp8_codes((B, Hkv, S, D))) if fp8 else (lambda: torch.randn(B, Hkv, S, D, device="cuda").bfloat16())
        self.caches = [(mk(), mk()) for _ in range(self.nbuf)]
        self.scales = torch.full((Hkv,), 2.0 / 448.0, device="cuda")
        self.q = torch.randn(B, Hq, 1, D, device="cuda").bfloat16()
        self.k = torch.randn(B, Hkv, 1, D, device="cuda").bfloat16()
        self.v = torch.randn(B, Hkv, 1, D, device="cuda").bfloat16()
        self.out = torch.empty_like(self.q)
        self.pos = torch.tensor([p], dtype=torch.int64, device="cuda")
        self.wsb = int(L.lib.it_b200_attention_kvcache_workspace(B, Hq, S, D))
        self.ws = torch.empty(max(self.wsb, 16), dtype=torch.uint8, device="cuda")
        self.st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def launch(self, i):
        P = lambda t: ctypes.c_void_p(t.data_ptr())
        kc, vc = self.caches[i % self.nbuf]
        if self.fp8:
            L.check(L.lib.it_b200_attention_kvcache_fp8(BF16, P(kc), P(vc), P(self.scales), P(self.scales), P(self.q), P(self.k),
                                                        P(self.v), P(self.pos), 7, None, 7, P(self.out), self.B, self.Hq, self.Hkv,
                                                        self.S, D, P(self.ws), self.wsb, self.st))
        else:
            L.check(L.lib.it_b200_attention_kvcache_gqa(BF16, P(kc), P(vc), P(self.q), P(self.k), P(self.v), P(self.pos), 7, None,
                                                        7, P(self.out), self.B, self.Hq, self.Hkv, self.S, D, P(self.ws), self.wsb,
                                                        self.st))

    def time(self, iters):
        for i in range(2 * self.nbuf):
            self.launch(i)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(iters):
            self.launch(i)
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) * 1e3 / iters


def time_step(cfg, steps, warmup, pos):
    from infinitensor_b200 import backend as B
    from infinitensor_b200 import graphs as G
    rt = B.CudaRuntime(0)
    h = B.GraphHandler(rt)
    g = G.build_llama_decode(h, cfg)
    h.data_malloc()
    gen = torch.Generator(device="cuda")
    ts = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def upload(t, tmp):
        assert tmp.numel() * tmp.element_size() == t.nbytes()
        L.check(L.lib.it_b200_copy(ctypes.c_void_p(tmp.data_ptr()), ctypes.c_void_p(t.device_ptr()), t.nbytes(), ts))
        torch.cuda.current_stream().synchronize()

    for i, (name, (t, shape, kind, shard)) in enumerate(g.weights.items()):
        gen.manual_seed(1000 + i)
        if kind == "kv_scale":
            upload(t, torch.full(t.shape(), 2.0 / 448.0, device="cuda"))
        else:
            upload(t, torch.empty(t.shape(), dtype=torch.bfloat16, device="cuda").normal_(1.0 if kind == "norm" else 0.0, 0.02,
                                                                                          generator=gen))
    for c in g.k_caches + g.v_caches:
        upload(c, fp8_codes(c.shape()) if cfg.kv_fp8 else torch.randn(c.shape(), device="cuda").bfloat16() * 0.5)
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
    sched = h.schedule()
    del g, h, rt
    torch.cuda.empty_cache()
    return ms, cfg.algorithmic_bytes(pos), sched


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no-step", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "kvfp8_bench needs a GPU"
    print(f"card: {card()}")
    print(f"{'B':>3} {'Hq':>3} {'Hkv':>3} {'S_max':>5} {'p':>5} | {'bf16 us':>9} {'GB/s':>7} | {'fp8 us':>9} {'GB/s':>7} | "
          f"{'fp8/bf16 time':>13}")
    for S, p in ((1024, 511), (4096, 4095)):
        for Hkv in (32, 8, 4, 1):
            ks = {fp8: Kernel(16, 32, Hkv, S, p, fp8) for fp8 in (False, True)}
            t = {False: [], True: []}
            for _ in range(3):  # alternate the two caches
                for fp8 in (False, True):
                    t[fp8].append(ks[fp8].time(a.iters))
            us = {f: float(np.median(v)) for f, v in t.items()}
            gbs = {f: kernel_bytes(16, 32, Hkv, p, f) / us[f] / 1e3 for f in us}
            print(f"{16:>3} {32:>3} {Hkv:>3} {S:>5} {p:>5} | {us[False]:>9.2f} {gbs[False]:>7.0f} | {us[True]:>9.2f} "
                  f"{gbs[True]:>7.0f} | {us[True] / us[False]:>13.3f}")
            del ks
            torch.cuda.empty_cache()
    if not a.no_step:
        from infinitensor_b200 import graphs as G
        shapes = [("llama3_8b p 511", lambda f: G.LlamaConfig.llama3_8b(kv_fp8=f), 511),
                  ("llama-7b S_max 4096 p 4095", lambda f: G.LlamaConfig(s_max=4096, batch=16, kv_fp8=f), 4095)]
        for name, mk, pos in shapes:
            for fp8 in (False, True):
                cfg = mk(fp8)
                ms, byts, sched = time_step(cfg, a.steps, a.warmup, pos)
                print(f"{name} (B {cfg.batch}, {cfg.layers} layers, {cfg.heads} q / {cfg.n_kv} kv heads, bf16, "
                      f"{'FP8' if fp8 else 'bf16'} cache, CUDA graph, {a.steps} steps): {ms:.3f} ms/step, "
                      f"{cfg.batch / ms * 1e3:.0f} tok/s; algorithmic bytes {byts / 1e9:.2f} GB -> bound "
                      f"{byts / HBM * 1e3:.2f} ms at 3.35 TB/s = {byts / HBM * 1e3 / ms:.1%} of roofline; "
                      f"{sum(s.startswith('AttentionRope') for s in sched)} AttentionRope steps")
    print(f"card: {card()}")


if __name__ == "__main__":
    main()
