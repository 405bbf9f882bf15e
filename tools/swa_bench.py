#!/usr/bin/env python
"""Sliding-window attention against no window on one GPU.

  python tools/swa_bench.py [--iters 200] [--steps 30] [--rounds 5] [--layers 32] [--skip-step]

1. Decode attention, B 8, 32 query heads over 8 KV heads of 128, S_max 16384, p 16383: it_b200_attention_kvcache_window with
   window 4096 against window 0, bf16 and FP8 caches.  CUDA events around `iters` back-to-back calls, alternated `rounds`
   times; GB/s on the algorithmic bytes (the K / V rows read, min(p + 1, W) per head with a window, p + 1 without, plus q,
   the appended row and the output).
2. A whole Mistral-7B-v0.1 decode step (mistral_7b_v01, B 8, S_max 16384, p 16383) against the same graph without its
   window, both built in one process and replayed alternately as CUDA graphs.  Synthetic weights drawn on the device.
3. The prompt attention (it_b200_attention_kvcache_prompt_window: append + attention), B 1, S 8192 at p 0, window 4096
   against none; TFLOP/s on the algorithmic FLOPs 4 D Hq sum_i min(i + 1, W).
Prints one JSON line per measurement, and the card's name and power limit read in the same run.
"""
import argparse
import ctypes
import dataclasses
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

F16, BF16, F32, I64 = 10, 16, 1, 7


def events_ms(fn, iters, stream=None):
    """ms per call of fn, from CUDA events on the stream its work goes to (default: torch's current stream)"""
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(stream)
    for _ in range(iters):
        fn()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def alternate(fns, iters, rounds, streams=None):
    """median ms per call of each fn, timed in alternation"""
    streams = streams or {}
    for k, f in fns.items():
        events_ms(f, 3, streams.get(k))
    ms = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            ms[k].append(events_ms(f, iters, streams.get(k)))
    return {k: statistics.median(v) for k, v in ms.items()}


def decode_kernel(a, fp8):
    import torch
    from infinitensor_b200 import _lib as L
    B, Hq, Hkv, S, D, p, W = 8, 32, 8, 16384, 128, 16383, 4096
    bf = torch.bfloat16
    if fp8:
        kc = torch.randint(0, 0x7E, (B, Hkv, S, D), dtype=torch.uint8, device="cuda")
        vc = torch.randint(0, 0x7E, (B, Hkv, S, D), dtype=torch.uint8, device="cuda")
        sc = [torch.full((Hkv,), 0.01, dtype=torch.float32, device="cuda") for _ in range(2)]
    else:
        kc, vc = (torch.randn((B, Hkv, S, D), dtype=bf, device="cuda") * 0.5 for _ in range(2))
        sc = [None, None]
    q, k, v = torch.randn((B, Hq, 1, D), dtype=bf, device="cuda"), *(torch.randn((B, Hkv, 1, D), dtype=bf, device="cuda") for _ in range(2))
    out = torch.empty_like(q)
    pos = torch.full((B,), p, dtype=torch.int64, device="cuda")
    wsb = int(L.lib.it_b200_attention_kvcache_workspace(B, Hq, S, D))
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())

    def call(window):
        return lambda: L.check(L.lib.it_b200_attention_kvcache_window(BF16, P(kc), P(vc), P(sc[0]), P(sc[1]), P(q), P(k), P(v), None,
                                                                      0, None, F32, 0, window, P(pos), I64, P(out), B, Hq, Hkv, S,
                                                                      D, P(ws), wsb, st))
    ms = alternate({W: call(W), 0: call(0)}, a.iters, a.rounds)
    elt = 1 if fp8 else 2
    for w, t in ms.items():
        rows = min(p + 1, W) if w else p + 1
        nbytes = 2 * B * Hkv * rows * D * elt + (2 * B * Hq + 2 * B * Hkv) * D * 2
        print(json.dumps({"what": "decode_attention", "cache": "fp8" if fp8 else "bf16", "B": B, "Hq": Hq, "Hkv": Hkv, "p": p,
                          "window": w, "us": round(t * 1e3, 2), "GBps": round(nbytes / (t * 1e-3) / 1e9, 1)}))
    print(json.dumps({"what": "decode_attention_ratio", "cache": "fp8" if fp8 else "bf16", "unwindowed_over_windowed": round(ms[0] / ms[W], 3)}))


def whole_step(a):
    import torch
    from infinitensor_b200 import _lib as L
    from infinitensor_b200 import backend as Bk
    from infinitensor_b200 import graphs as G
    base = G.LlamaConfig.mistral_7b_v01(batch=8, s_max=16384, layers=a.layers)
    built = {}
    for name, cfg in (("window", base), ("none", dataclasses.replace(base, sliding_window=None))):
        rt = Bk.CudaRuntime(0)
        h = Bk.GraphHandler(rt)
        g = G.build_llama_decode(h, cfg)
        h.data_malloc()
        gen = torch.Generator(device="cuda")
        ts = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

        def fill(t, std, mean, seed):
            gen.manual_seed(seed)
            tmp = torch.empty(t.shape(), dtype=torch.bfloat16, device="cuda").normal_(mean, std, generator=gen)
            L.check(L.lib.it_b200_copy(ctypes.c_void_p(tmp.data_ptr()), ctypes.c_void_p(t.device_ptr()), t.nbytes(), ts))
            torch.cuda.current_stream().synchronize()
        for i, (_, (t, _, kind, _)) in enumerate(g.weights.items()):
            fill(t, 0.02, 1.0 if kind == "norm" else 0.0, 1000 + i)
        for li in range(cfg.layers):
            fill(g.k_caches[li], 0.5, 0.0, 5000 + li)
            fill(g.v_caches[li], 0.5, 0.0, 7000 + li)
        g.input_ids.copyin_numpy(np.random.default_rng(1).integers(0, cfg.vocab, size=(cfg.batch, 1)).astype(np.int64))
        g.position_ids.copyin_numpy(np.full((cfg.batch, 1), 16383, np.int64))
        for _ in range(3):
            h.run_with_cudagraph()
        built[name] = (rt, h, cfg)

    def step(name):
        rt, h, _ = built[name]
        return lambda: h.launch_cudagraph_async()
    # graph replays run on each runtime's own stream
    ms = alternate({n: step(n) for n in built}, a.steps, a.rounds,
                   {n: torch.cuda.ExternalStream(built[n][0].stream()) for n in built})
    for n, t in ms.items():
        cfg = built[n][2]
        nbytes = cfg.algorithmic_bytes(16383)
        print(json.dumps({"what": "mistral_7b_v01_step", "layers": cfg.layers, "B": cfg.batch, "p": 16383,
                          "window": cfg.sliding_window or 0, "ms": round(t, 4), "tok_s": round(cfg.batch * 1e3 / t, 1),
                          "GBps_algorithmic": round(nbytes / (t * 1e-3) / 1e9, 1)}))
    print(json.dumps({"what": "mistral_7b_v01_step_ratio", "unwindowed_over_windowed": round(ms["none"] / ms["window"], 3)}))


def prompt(a):
    import torch
    from infinitensor_b200 import _lib as L
    B, Hq, Hkv, S, D, W = 1, 32, 8, 8192, 128, 4096
    bf = torch.bfloat16
    kc, vc = (torch.zeros((B, Hkv, S, D), dtype=bf, device="cuda") for _ in range(2))
    q = torch.randn((B, Hq, S, D), dtype=bf, device="cuda")
    k, v = (torch.randn((B, Hkv, S, D), dtype=bf, device="cuda") for _ in range(2))
    out = torch.empty_like(q)
    pos = torch.zeros((B,), dtype=torch.int64, device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda t: ctypes.c_void_p(t.data_ptr())

    def call(window):
        return lambda: L.check(L.lib.it_b200_attention_kvcache_prompt_window(BF16, P(kc), P(vc), P(q), P(k), P(v), P(pos), I64, P(out),
                                                                             B, Hq, Hkv, S, S, D, window, st))
    ms = alternate({W: call(W), 0: call(0)}, max(a.iters // 20, 5), a.rounds)
    for w, t in ms.items():
        flops = 4.0 * D * Hq * sum(min(i + 1, w) if w else i + 1 for i in range(S))
        print(json.dumps({"what": "prompt_attention", "B": B, "Hq": Hq, "Hkv": Hkv, "S": S, "window": w, "ms": round(t, 4),
                          "TFLOPs": round(flops / (t * 1e-3) / 1e12, 1)}))
    print(json.dumps({"what": "prompt_attention_ratio", "unwindowed_over_windowed": round(ms[0] / ms[W], 3)}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--skip-step", action="store_true")
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "swa_bench needs a GPU"
    from tools.prompt_bench import card
    print(json.dumps({"card": card()}))
    decode_kernel(a, fp8=False)
    decode_kernel(a, fp8=True)
    prompt(a)
    if not a.skip_step:
        whole_step(a)


if __name__ == "__main__":
    main()
