"""Prompt prefill into the KV cache on one GPU: the AttentionKVCache prompt kernels alone, and a whole Llama-7B-shape prompt
step against the decode-step loop it replaces.

  python tools/prompt_bench.py [--iters N] [--layers L] [--skip-step]

1. it_b200_attention_kvcache_prompt (the append launch + the causal attention launch), bf16, B = 1, Hq = 32, D = 128, Hkv in
   {32, 8}: S = 512 and 2048 at p = 0, S = 512 at p = 1536, and S = 16 at p = 4000 (a short chunk at long context: few CTAs).
   CUDA events around `iters` back-to-back calls; TFLOP/s on the algorithmic FLOPs 4 D sum_i (p + i + 1) per query head
   (Q K^T and P V over the causal rows only).
2. Llama-7B shape (32 layers, d 4096, 32 heads of 128, ffn 11008, vocab 32000), B = 1: one prompt step of 512 tokens by
   CUDA-graph replay, and 512 replays of the B = 1 decode graph (positions 0 .. 511), the way a prompt is fed without a prompt
   step.  Synthetic weights drawn on the device.
Prints one JSON line per measurement, with the card's name and power limit read in the same run.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BF16, I64 = 16, 7


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[0] if q.stdout else "unavailable"}


def attention_flops(S, p, D, Hq):
    return 4.0 * D * Hq * sum(p + i + 1 for i in range(S))


def bench_kernel(L, Hkv, S, p, iters, Hq=32, D=128, S_max=4096):
    import torch
    g = torch.Generator(device="cuda").manual_seed(0)
    mk = lambda *s: torch.empty(s, dtype=torch.bfloat16, device="cuda").normal_(0, 0.5, generator=g)  # noqa: E731
    kc, vc = mk(1, Hkv, S_max, D), mk(1, Hkv, S_max, D)
    q, k, v = mk(1, Hq, S, D), mk(1, Hkv, S, D), mk(1, Hkv, S, D)
    out = torch.empty_like(q)
    pos = torch.tensor([p], dtype=torch.int64, device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731

    def call():
        L.check(L.lib.it_b200_attention_kvcache_prompt(BF16, P(kc), P(vc), P(q), P(k), P(v), P(pos), I64, P(out), 1, Hq, Hkv, S,
                                                       S_max, D, st))
    for _ in range(10):
        call()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        call()
    e1.record()
    e1.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / iters
    fl = attention_flops(S, p, D, Hq)
    return {"what": "attention_kvcache_prompt (append + attention)", "dtype": "bf16", "B": 1, "Hq": Hq, "Hkv": Hkv, "D": D, "S": S,
            "p": p, "us": round(us, 2), "tflops": round(fl / us / 1e6, 1), "iters": iters}


def bench_step(L, layers, iters_prompt, S=512):
    import torch
    from infinitensor_b200 import backend as B, graphs as G
    cfg = G.LlamaConfig(layers=layers, batch=1, s_max=1024)
    rt = B.CudaRuntime(0)
    gen = torch.Generator(device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def fill(t, std, mean, seed):
        gen.manual_seed(seed)
        tmp = torch.empty(list(t.shape()), dtype=torch.bfloat16, device="cuda").normal_(mean, std, generator=gen)
        L.check(L.lib.it_b200_copy(ctypes.c_void_p(tmp.data_ptr()), ctypes.c_void_p(t.device_ptr()), t.nbytes(), st))
        torch.cuda.current_stream().synchronize()

    def graph(seq):
        h = B.GraphHandler(rt)
        g = G.build_llama_decode(h, cfg, seq=seq)
        h.data_malloc()
        for i, (name, (t, shape, kind, shard)) in enumerate(g.weights.items()):
            fill(t, 0.02, 1.0 if kind == "norm" else 0.0, 1000 + i)
        for li in range(cfg.layers):
            fill(g.k_caches[li], 0.5, 0.0, 5000 + li)
            fill(g.v_caches[li], 0.5, 0.0, 7000 + li)
        return h, g

    ids = np.random.default_rng(1).integers(0, cfg.vocab, size=(1, S)).astype(np.int64)
    hp, gp = graph(S)
    gp.input_ids.copyin_numpy(ids)
    gp.position_ids.copyin_numpy(np.arange(S, dtype=np.int64)[None])
    for _ in range(3):
        hp.run_with_cudagraph()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters_prompt):
        hp.run_with_cudagraph()
    e1.record()
    e1.synchronize()
    prompt_ms = e0.elapsed_time(e1) / iters_prompt
    del hp, gp
    torch.cuda.empty_cache()

    hd, gd = graph(1)
    gd.input_ids.copyin_numpy(ids[:, :1])
    gd.position_ids.copyin_numpy(np.zeros((1, 1), np.int64))
    for _ in range(3):
        hd.run_with_cudagraph()
    torch.cuda.synchronize()
    # the positions change every step: copied in before each replay, as a token-by-token prompt feed must
    e0.record()
    for i in range(S):
        gd.input_ids.copyin_numpy(ids[:, i:i + 1])
        gd.position_ids.copyin_numpy(np.full((1, 1), i, np.int64))
        hd.run_with_cudagraph()
    e1.record()
    e1.synchronize()
    loop_ms = e0.elapsed_time(e1)
    return {"what": f"Llama-7B shape ({layers} layers), B 1, {S}-token prompt", "prompt_step_ms": round(prompt_ms, 2),
            "decode_loop_ms": round(loop_ms, 1), "decode_step_ms": round(loop_ms / S, 3), "speedup": round(loop_ms / prompt_ms, 1),
            "prompt_step_iters": iters_prompt}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--skip-step", action="store_true")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "prompt_bench needs a GPU"
    from infinitensor_b200 import _lib as L
    info = card()
    print(json.dumps(info), flush=True)
    for Hkv in (32, 8):
        for S, p in ((512, 0), (2048, 0), (512, 1536), (16, 4000)):
            print(json.dumps(bench_kernel(L, Hkv, S, p, args.iters)), flush=True)
    if not args.skip_step:
        print(json.dumps(bench_step(L, args.layers, 10)), flush=True)


if __name__ == "__main__":
    main()
