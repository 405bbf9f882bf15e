#!/usr/bin/env python
"""4-bit weights (MatMulNBits, block 128) against 16-bit and FP8 weights on the GPU: the decode GEMMs and whole Llama decode steps.

  python tools/w4_bench.py [--iters 200] [--steps 50] [--warmup 10] [--no-step]

GEMMs: the Llama-7B decode shapes at M = 16 rows, bf16 activations -- q/k/v (three 4096 x 4096 matrices, one grouped launch), o
(4096 x 4096, residual fused), gate/up (two 4096 x 11008, grouped), down (11008 x 4096, residual fused), logits (4096 x 32000).
Each runs as bf16 weights (it_b200_matmul / _grouped, the production dispatch), FP8 E4M3 weights with column scales
(it_b200_matmul_fp8w) and int4 codes with one bf16 scale per 128 weights (it_b200_matmul_nbits), timed alternately in the same
run with CUDA events over enough weight copies (>= 256 MB in all) that the weights are not L2-resident.  Algorithmic bytes: the
weights at 2 / 1 / 0.5 bytes per element, their scales, X, C and the residual; GB/s is those bytes over kernel time.
Steps: Llama-7B shape (B 16, p 511, S_max 1024) with bf16, FP8 and int4 weights, and the Llama-3-8B shape with bf16 and int4
weights, CUDA-graph replay, the variants of one shape alternated; the roofline is LlamaConfig.algorithmic_bytes over the H100 SXM
data-sheet 3.35 TB/s -- a bound computed from the shapes, not a measurement.  The card's name, power limit and SM clock are
printed from the same run, and the logits of every step are checked finite."""
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
BF16, F32 = 16, 1
M = 16
BS = 128
B_CONST = 0x200  # ITB_MATMUL_B_CONST
ROUND_BEFORE_BIAS = 0x100  # ITB_ACT_ROUND_BEFORE_BIAS
VP = ctypes.c_void_p
GEMMS = [("q/k/v", 4096, [4096, 4096, 4096], False), ("o", 4096, [4096], True), ("gate/up", 4096, [11008, 11008], False),
         ("down", 11008, [4096], True), ("logits", 4096, [32000], False)]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "nvidia-smi unavailable"


def P(t):
    return VP(t.data_ptr()) if t is not None else None


def fp8_codes(shape, std=0.5):
    return (torch.randn(shape, device="cuda") * (448.0 / 4.0 * std)).to(torch.float8_e4m3fn).view(torch.uint8)


class Gemm:
    """one decode GEMM (1..3 matrices sharing X) in one weight format: 'bf16', 'fp8' or 'int4'"""

    def __init__(self, K, Ns, res, fmt):
        self.K, self.Ns, self.fmt = K, Ns, fmt
        self.x = torch.randn(M, K, device="cuda").bfloat16()
        self.c = [torch.empty(M, N, device="cuda", dtype=torch.bfloat16) for N in Ns]
        self.r = torch.randn(M, Ns[0], device="cuda").bfloat16() if res else None

        def one_set():
            if fmt == "bf16":
                return [(torch.randn(K, N, device="cuda").bfloat16() * 0.02, None) for N in Ns]
            if fmt == "fp8":
                return [(fp8_codes((K, N)), torch.full((N,), 0.02 / 112.0, device="cuda")) for N in Ns]
            return [(torch.randint(0, 256, (N, K // BS, BS // 2), dtype=torch.uint8, device="cuda"),
                     torch.full((N * K // BS,), 0.004, device="cuda").bfloat16()) for N in Ns]
        wb = {"bf16": 2.0, "fp8": 1.0, "int4": 0.5}[fmt]
        sb = {"bf16": 0, "fp8": 4 * sum(Ns), "int4": 2 * sum(Ns) * K // BS}[fmt]
        set_bytes = int(wb * K * sum(Ns)) + sb
        self.nbuf = max(2, -(-(256 << 20) // set_bytes))
        self.sets = [one_set() for _ in range(self.nbuf)]
        self.bytes = set_bytes + 2 * M * K + 2 * M * sum(Ns) + (2 * M * Ns[0] if res else 0)
        self.st = VP(torch.cuda.current_stream().cuda_stream)
        self.Narr = L.i32arr(Ns)
        self.Carr = (VP * len(Ns))(*[c.data_ptr() for c in self.c])

    def launch(self, i):
        ws = self.sets[i % self.nbuf]
        g = len(self.Ns)
        Warr = (VP * g)(*[w.data_ptr() for w, _ in ws])
        if self.fmt == "bf16":
            if g > 1:
                L.check(L.lib.it_b200_matmul_grouped(BF16, P(self.x), g, Warr, self.Carr, self.Narr, M, self.K, self.st))
            else:
                N = self.Ns[0]
                act = B_CONST | (ROUND_BEFORE_BIAS if self.r is not None else 0)
                L.check(L.lib.it_b200_matmul(BF16, P(self.x), VP(ws[0][0].data_ptr()), P(self.r), P(self.c[0]), 1, M, N, self.K,
                                             M * self.K, 0, 0, 0, 0, N if self.r is not None else 0, 1 if self.r is not None else 0,
                                             act, None, 0, self.st))
        elif self.fmt == "fp8":
            Sarr = (VP * g)(*[s.data_ptr() for _, s in ws])
            L.check(L.lib.it_b200_matmul_fp8w(BF16, P(self.x), g, Warr, Sarr, self.Carr, self.Narr, M, self.K, P(self.r), self.st))
        else:
            Sarr = (VP * g)(*[s.data_ptr() for _, s in ws])
            L.check(L.lib.it_b200_matmul_nbits(BF16, P(self.x), g, Warr, Sarr, None, self.Carr, self.Narr, M, self.K, BS, P(self.r),
                                               None, 0, self.st))

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
        assert all(torch.isfinite(c.float()).all() for c in self.c), "non-finite GEMM output"
        return e0.elapsed_time(e1) * 1e3 / iters


class Step:
    """a decode-step graph with synthetic weights, replayed as a CUDA graph"""

    def __init__(self, cfg, pos):
        from infinitensor_b200 import backend as B
        from infinitensor_b200 import graphs as G
        self.cfg, self.pos = cfg, pos
        self.rt = B.CudaRuntime(0)
        self.h = B.GraphHandler(self.rt)
        self.g = G.build_llama_decode(self.h, cfg)
        self.h.data_malloc()
        gen = torch.Generator(device="cuda")
        ts = VP(torch.cuda.current_stream().cuda_stream)

        def upload(t, tmp):
            assert tmp.numel() * tmp.element_size() == t.nbytes()
            L.check(L.lib.it_b200_copy(VP(tmp.data_ptr()), VP(t.device_ptr()), t.nbytes(), ts))
            torch.cuda.current_stream().synchronize()

        for i, (name, (t, shape, kind, shard)) in enumerate(self.g.weights.items()):
            gen.manual_seed(1000 + i)
            if kind == "proj_fp8":
                upload(t, fp8_codes(t.shape()))
            elif kind == "proj_int4":
                upload(t, torch.randint(0, 256, t.shape(), dtype=torch.uint8, device="cuda", generator=gen))
            elif kind == "scale":  # FP8 column scales (f32) or int4 block scales (bf16)
                upload(t, torch.full(t.shape(), 0.02 / 112.0, device="cuda") if t.dtype() == F32 else
                       torch.full(t.shape(), 0.004, device="cuda").bfloat16())
            else:
                upload(t, torch.empty(t.shape(), dtype=torch.bfloat16, device="cuda").normal_(1.0 if kind == "norm" else 0.0, 0.02,
                                                                                              generator=gen))
        for c in self.g.k_caches + self.g.v_caches:
            upload(c, torch.randn(c.shape(), device="cuda").bfloat16() * 0.5)
        self.g.input_ids.copyin_numpy(np.random.default_rng(1).integers(0, cfg.vocab, size=(cfg.batch, 1)).astype(np.int64))
        self.g.position_ids.copyin_numpy(np.full((cfg.batch, 1), pos, np.int64))
        self.stream = torch.cuda.ExternalStream(self.rt.stream())

    def time(self, steps, warmup):
        for _ in range(max(warmup, 3)):
            self.h.run_with_cudagraph()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(self.stream)
        for _ in range(steps):
            self.h.launch_cudagraph_async()
        e1.record(self.stream)
        e1.synchronize()
        from infinitensor_b200 import graphs as G
        assert np.isfinite(G.from_storage(self.g.logits.copyout_numpy(), self.cfg.dtype)).all(), "non-finite logits"
        return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-step", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "w4_bench needs a GPU"
    print(f"card: {card()}")
    fmts = ("bf16", "fp8", "int4")
    print(f"M = {M}, bf16 activations, int4 block {BS}; median of {a.rounds} alternated rounds of {a.iters} launches")
    print(f"{'GEMM':>8} {'K':>6} {'N':>17} | " + " | ".join(f"{f + ' us':>9} {'GB/s':>6}" for f in fmts) + " | int4/bf16 time")
    for name, K, Ns, res in GEMMS:
        gs = {f: Gemm(K, Ns, res, f) for f in fmts}
        t = {f: [] for f in fmts}
        for _ in range(a.rounds):
            for f in fmts:
                t[f].append(gs[f].time(a.iters))
        us = {f: float(np.median(v)) for f, v in t.items()}
        cols = " | ".join(f"{us[f]:>9.2f} {gs[f].bytes / us[f] / 1e3:>6.0f}" for f in fmts)
        print(f"{name:>8} {K:>6} {'x'.join(map(str, Ns)):>17} | {cols} | {us['int4'] / us['bf16']:.3f}")
        del gs
        torch.cuda.empty_cache()
    if not a.no_step:
        from infinitensor_b200 import graphs as G
        shapes = [("llama-7b p 511", lambda **kw: G.LlamaConfig(batch=16, **kw), ("bf16", "fp8", "int4")),
                  ("llama3_8b p 511", lambda **kw: G.LlamaConfig.llama3_8b(**kw), ("bf16", "int4"))]
        for name, mk, variants in shapes:
            kws = {"bf16": {}, "fp8": {"fp8_weights": True}, "int4": {"int4_block": BS}}
            steps = {v: Step(mk(**kws[v]), 511) for v in variants}
            t = {v: [] for v in variants}
            for _ in range(a.rounds):
                for v in variants:
                    t[v].append(steps[v].time(a.steps, a.warmup))
            for v in variants:
                cfg = steps[v].cfg
                ms = float(np.median(t[v]))
                byts = cfg.algorithmic_bytes(511)
                print(f"{name} (B {cfg.batch}, {cfg.layers} layers, {v} weights, CUDA graph, {a.steps} steps x {a.rounds} rounds, "
                      f"logits finite): {ms:.3f} ms/step (rounds {', '.join(f'{x:.3f}' for x in t[v])}), "
                      f"{cfg.batch / ms * 1e3:.0f} tok/s; algorithmic bytes {byts / 1e9:.2f} GB -> bound {byts / HBM * 1e3:.2f} ms "
                      f"at 3.35 TB/s = {byts / HBM * 1e3 / ms:.1%} of roofline")
            del steps
            torch.cuda.empty_cache()
    print(f"card: {card()}")


if __name__ == "__main__":
    main()
