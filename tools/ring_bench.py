#!/usr/bin/env python
"""The rolling KV cache against a linear windowed cache on one GPU.

  python tools/ring_bench.py [--iters 200] [--steps 30] [--rounds 5] [--layers 32] [--skip-step]

1. Decode attention, B 8, 32 query heads over 8 KV heads of 128, window 4096, p 16383: it_b200_attention_kvcache_window over
   a 4608-row ring (ITB_POS_RING) against a 16384-row linear cache, bf16 and FP8 caches.  CUDA events around `iters`
   back-to-back calls, alternated `rounds` times; GB/s on the algorithmic bytes (the same for both).
2. A whole mistral_7b_v01(rolling_cache=True) decode step, B 32 at p 32767 on a 4608-row ring, replayed as a CUDA graph:
   ms / step, tok/s, and the cache bytes allocated against those a linear cache would need (which do not fit an 80 GB card).
3. 512-token prompt chunks (append + attention) through a 4608-row ring at p 32256 against the linear windowed chunk at the
   same key-tile offsets, B 1, 32 / 8 heads of 128, window 4096.
Prints one JSON line per measurement, and the card's name and power limit read in the same run.
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.swa_bench import alternate  # noqa: E402

F32, BF16, I64, RING = 1, 16, 7, 0x400


def decode_kernel(a, fp8):
    import torch
    from infinitensor_b200 import _lib as L
    B, Hq, Hkv, D, p, W = 8, 32, 8, 128, 16383, 4096
    P = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    q = torch.randn((B, Hq, 1, D), dtype=torch.bfloat16, device="cuda")
    k, v = (torch.randn((B, Hkv, 1, D), dtype=torch.bfloat16, device="cuda") for _ in range(2))
    out = torch.empty_like(q)
    pos = torch.full((B,), p, dtype=torch.int64, device="cuda")
    sc = [torch.full((Hkv,), 0.01, dtype=torch.float32, device="cuda") for _ in range(2)] if fp8 else [None, None]
    calls = {}
    for name, S, flags in (("ring", 4608, RING), ("linear", 16384, 0)):
        if fp8:
            kc, vc = (torch.randint(0, 0x7E, (B, Hkv, S, D), dtype=torch.uint8, device="cuda") for _ in range(2))
        else:
            kc, vc = (torch.randn((B, Hkv, S, D), dtype=torch.bfloat16, device="cuda") * 0.5 for _ in range(2))
        wsb = int(L.lib.it_b200_attention_kvcache_workspace(B, Hq, S, D))
        ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")

        def call(kc=kc, vc=vc, ws=ws, wsb=wsb, S=S, flags=flags):
            L.check(L.lib.it_b200_attention_kvcache_window(BF16, P(kc), P(vc), P(sc[0]), P(sc[1]), P(q), P(k), P(v), None, 0, None,
                                                           F32, 0, W, P(pos), I64 | flags, P(out), B, Hq, Hkv, S, D, P(ws), wsb, st))
        calls[name] = call
    ms = alternate(calls, a.iters, a.rounds)
    elt = 1 if fp8 else 2
    nbytes = 2 * B * Hkv * W * D * elt + (2 * B * Hq + 2 * B * Hkv) * D * 2
    for n, t in ms.items():
        print(json.dumps({"what": "decode_attention", "cache": "fp8" if fp8 else "bf16", "layout": n, "B": B, "p": p, "window": W,
                          "us": round(t * 1e3, 2), "GBps": round(nbytes / (t * 1e-3) / 1e9, 1)}))
    print(json.dumps({"what": "decode_attention_ratio", "cache": "fp8" if fp8 else "bf16", "ring_over_linear": round(ms["ring"] / ms["linear"], 4)}))


def whole_step(a):
    import numpy as np
    import torch
    from infinitensor_b200 import _lib as L
    from infinitensor_b200 import backend as Bk
    from infinitensor_b200 import graphs as G
    cfg = G.LlamaConfig.mistral_7b_v01(batch=32, s_max=4608, layers=a.layers, rolling_cache=True)
    p = 32767
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
        del tmp
    for i, (_, (t, _, kind, _)) in enumerate(g.weights.items()):
        fill(t, 0.02, 1.0 if kind == "norm" else 0.0, 1000 + i)
    for li in range(cfg.layers):
        fill(g.k_caches[li], 0.5, 0.0, 5000 + li)
        fill(g.v_caches[li], 0.5, 0.0, 7000 + li)
    g.input_ids.copyin_numpy(np.random.default_rng(1).integers(0, cfg.vocab, size=(cfg.batch, 1)).astype(np.int64))
    g.position_ids.copyin_numpy(np.full((cfg.batch, 1), p, np.int64))
    for _ in range(3):
        h.run_with_cudagraph()
    ms = alternate({"ring": lambda: h.launch_cudagraph_async()}, a.steps, a.rounds,
                   {"ring": torch.cuda.ExternalStream(rt.stream())})["ring"]
    row = 2 * cfg.layers * cfg.n_kv * cfg.head_dim * 2  # bytes of one cached token, k and v of every layer
    logits = g.logits.copyout_numpy()
    print(json.dumps({"what": "mistral_7b_v01_ring_step", "layers": cfg.layers, "B": cfg.batch, "p": p, "ring_rows": cfg.s_max,
                      "ms": round(ms, 4), "tok_s": round(cfg.batch * 1e3 / ms, 1),
                      "GBps_algorithmic": round(cfg.algorithmic_bytes(p) / (ms * 1e-3) / 1e9, 1),
                      "cache_bytes_allocated": sum(t.nbytes() for t in g.k_caches + g.v_caches),
                      "linear_cache_bytes_needed": row * cfg.batch * (p + 1),
                      "logits_finite": bool(np.isfinite(G.from_storage(logits, cfg.dtype)).all())}))


def prompt(a):
    import torch
    from infinitensor_b200 import _lib as L
    B, Hq, Hkv, S, D, W = 1, 32, 8, 512, 128, 4096
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    q = torch.randn((B, Hq, S, D), dtype=torch.bfloat16, device="cuda")
    k, v = (torch.randn((B, Hkv, S, D), dtype=torch.bfloat16, device="cuda") for _ in range(2))
    out = torch.empty_like(q)
    calls = {}
    # the ring at p 32256 and the linear cache at p 4608: the same offsets in their key tiles, the same window lengths
    for name, S_max, p, flags in (("ring", 4608, 32256, RING), ("linear", 8192, 4608, 0)):
        kc, vc = (torch.randn((B, Hkv, S_max, D), dtype=torch.bfloat16, device="cuda") for _ in range(2))
        pos = torch.full((B,), p, dtype=torch.int64, device="cuda")

        def call(kc=kc, vc=vc, pos=pos, S_max=S_max, flags=flags):
            L.check(L.lib.it_b200_attention_kvcache_prompt_window(BF16, P(kc), P(vc), P(q), P(k), P(v), P(pos), I64 | flags, P(out),
                                                                  B, Hq, Hkv, S, S_max, D, W, st))
        calls[name] = call
    ms = alternate(calls, max(a.iters // 4, 10), a.rounds)
    flops = 4.0 * D * Hq * sum(min(4608 + i + 1, W) for i in range(S))
    for n, t in ms.items():
        print(json.dumps({"what": "prompt_chunk", "layout": n, "B": B, "S": S, "window": W, "ms": round(t, 4),
                          "TFLOPs": round(flops / (t * 1e-3) / 1e12, 1)}))
    print(json.dumps({"what": "prompt_chunk_ratio", "ring_over_linear": round(ms["ring"] / ms["linear"], 4)}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--skip-step", action="store_true")
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "ring_bench needs a GPU"
    from tools.prompt_bench import card
    print(json.dumps({"card": card()}))
    decode_kernel(a, fp8=False)
    decode_kernel(a, fp8=True)
    prompt(a)
    if not a.skip_step:
        whole_step(a)


if __name__ == "__main__":
    main()
