#!/usr/bin/env python
"""Small single-process workloads for ncu captures (profiles/r02_*):  python tools/ncu_targets.py llama|prefill|resnet
   llama   : one eager pass of a 1-layer BASELINE-width Llama decode graph (q/k/v group, attention, o, gate/up group, down, logits GEMMs)
   prefill : GPT-2's attention block shape through attention_prefill_kernel
   resnet  : ResNet-50 B = 64 fp16, two eager passes"""
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

what = sys.argv[1] if len(sys.argv) > 1 else "llama"
from infinitensor_b200 import backend as B, graphs as G, _lib as L


def llama(layers):
    cfg = G.LlamaConfig(layers=layers)
    rt = B.CudaRuntime(0)
    h = B.GraphHandler(rt)
    g = G.build_llama_decode(h, cfg)
    h.data_malloc()
    ts = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    gen = torch.Generator(device="cuda")
    for i, (name, (t, shape, kind, shard)) in enumerate(g.weights.items()):
        gen.manual_seed(i)
        tmp = torch.empty(t.shape(), dtype=torch.bfloat16, device="cuda").normal_(1.0 if kind == "norm" else 0.0, 0.02, generator=gen)
        L.check(L.lib.it_b200_copy(ctypes.c_void_p(tmp.data_ptr()), ctypes.c_void_p(t.device_ptr()), t.nbytes(), ts))
        torch.cuda.synchronize()
    g.input_ids.copyin_numpy(np.arange(cfg.batch, dtype=np.int64).reshape(-1, 1))
    g.position_ids.copyin_numpy(np.full((cfg.batch, 1), 511, np.int64))
    for _ in range(3):
        h.run()


if what == "llama":
    llama(1)
elif what == "prefill":
    q, k, v = (torch.randn(1, 12, 128, 64, device="cuda").half() for _ in range(3))
    out = torch.zeros_like(q)
    scale = torch.tensor([8.0], device="cuda").half()
    mask = torch.triu(torch.full((128, 128), -65504.0, device="cuda"), 1).half().contiguous()
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    for _ in range(3):
        L.check(L.lib.it_b200_attention_prefill(10, P(q), P(k), P(v), P(out), 1, 12, 128, 128, 64, P(scale), 1, P(mask), 0, 0, 128, 1,
                                                ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
else:
    cfg = G.ResNetConfig()
    rt = B.CudaRuntime(0)
    h = B.GraphHandler(rt)
    g = G.build_resnet50(h, cfg)
    h.data_malloc()
    G.fill_resnet_weights_host(g)
    x = np.random.default_rng(3).standard_normal((cfg.batch, 3, cfg.image, cfg.image)).astype(np.float32)
    g.input.copyin_numpy(G.to_storage(x, cfg.dtype))
    h.run()
    h.run()
