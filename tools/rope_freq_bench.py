#!/usr/bin/env python
"""Decode step of Llama-3.1-8B (RoPE from an inv_freq table) against the Llama-3-8B shape (base-10000 RoPE) on the GPU.

  python tools/rope_freq_bench.py [--steps 50] [--warmup 10] [--rounds 5] [--batch 16] [--pos 511]

Both graphs are built once in one process (bf16, S_max 1024) and timed alternately, --rounds times each, as whole steps of
CUDA-graph replay between two CUDA events.  The two graphs differ only in their RoPE: llama31_8b's folded RoPE reads a
64-entry f32 table where llama3_8b's computes powf(10000, -2c / 128) once per CTA cos / sin table.  The card's name, power
limit and SM clock are printed from the same run."""
import argparse
import ctypes
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from infinitensor_b200 import _lib as L
from tools.gqa_bench import card


def build(model, batch, pos):
    from infinitensor_b200 import backend as B
    from infinitensor_b200 import graphs as G
    cfg = getattr(G.LlamaConfig, model)(batch=batch)
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
        if kind == "inv_freq":
            t.copyin_numpy(G.rope_inv_freq(cfg.head_dim, cfg.rope_theta, cfg.rope_scaling))
        else:
            fill(t, 0.02, 1.0 if kind == "norm" else 0.0, 1000 + i)
    for li in range(cfg.layers):
        fill(g.k_caches[li], 0.5, 0.0, 5000 + li)
        fill(g.v_caches[li], 0.5, 0.0, 7000 + li)
    g.input_ids.copyin_numpy(np.random.default_rng(1).integers(0, cfg.vocab, size=(cfg.batch, 1)).astype(np.int64))
    g.position_ids.copyin_numpy(np.full((cfg.batch, 1), pos, np.int64))
    return rt, h, g


def time_steps(rt, h, steps):
    stream = torch.cuda.ExternalStream(rt.stream())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(stream)
    for _ in range(steps):
        h.launch_cudagraph_async()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--pos", type=int, default=511)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "rope_freq_bench needs a GPU"
    print(f"card: {card()}")
    models = ("llama3_8b", "llama31_8b")
    built = {m: build(m, a.batch, a.pos) for m in models}
    for m in models:
        rt, h, g = built[m]
        for _ in range(max(a.warmup, 3)):
            h.run_with_cudagraph()
        sched = h.schedule()
        print(f"{m}: {sum(s.startswith('AttentionRope') for s in sched)} AttentionRope steps of {len(sched)}")
    ms = {m: [] for m in models}
    for _ in range(a.rounds):
        for m in models:
            rt, h, _ = built[m]
            ms[m].append(time_steps(rt, h, a.steps))
    for m in models:
        v = ms[m]
        print(f"{m:>11}: B {a.batch} p {a.pos}  ms/step " + " ".join(f"{x:.4f}" for x in v) +
              f"  median {statistics.median(v):.4f}  tok/s {a.batch * 1e3 / statistics.median(v):.1f}")
    r = statistics.median(ms["llama31_8b"]) / statistics.median(ms["llama3_8b"])
    print(f"llama31_8b / llama3_8b median step time: {r:.4f}")


if __name__ == "__main__":
    main()
