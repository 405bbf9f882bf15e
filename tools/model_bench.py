#!/usr/bin/env python
"""Whole-graph timings of the two non-headline BASELINE configs (parity-test cases, not bench lines):
   C2 GPT-2-small (B=1, S=128, fp16) and C4 ResNet-50 (B=64, fp16), CUDA-graph replay, device-timed;
   gpt2-decode: one GPT-2-small KV-cache decode step (B 16, p 511, fp16, with the tied LM head), ms / step and its share of
   the GPT2Config.algorithmic_bytes bound at the HBM peak.  The card's name, power limit and SM clock are printed with each.
   python tools/model_bench.py [gpt2] [gpt2-decode] [resnet] [--batch N]"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from gqa_bench import card  # noqa: E402 (tools/ is this script's directory)
from infinitensor_b200 import backend as B, graphs as G

_PEAKS_PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
# peaks measured on the card when MEASURED_PEAKS.json exists; else the H100 SXM data sheet (HBM3 3.35 TB/s, dense bf16 989 TFLOP/s)
PEAKS = json.load(open(_PEAKS_PATH)) if os.path.exists(_PEAKS_PATH) else {"hbm_gbs": 3350.0, "bf16_tflops": 989.0}


def timed(h, rt, reps, warm=5):
    if os.environ.get("MB_PROFILE"):  # under ncu: two eager passes, no graph replay
        h.run()
        h.run()
        return 1.0, 0
    for _ in range(warm):
        h.run_with_cudagraph()
    h.sync()
    l0 = rt.kernel_launches()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    st = torch.cuda.ExternalStream(rt.stream())
    with torch.cuda.stream(st):
        e0.record()
        for _ in range(reps):
            h.launch_cudagraph_async()
        e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps, (rt.kernel_launches() - l0) // max(reps, 1)


def gpt2():
    cfg = G.GPT2Config()
    rt = B.CudaRuntime(0)
    h = B.GraphHandler(rt)
    g = G.build_gpt2(h, cfg)
    h.data_malloc()
    G.fill_gpt2_weights_host(g)
    ids = np.random.default_rng(1).integers(0, cfg.vocab, size=(cfg.batch, cfg.seq)).astype(np.int64)
    pos = np.arange(cfg.seq, dtype=np.int64).reshape(1, -1).repeat(cfg.batch, 0)
    g.input_ids.copyin_numpy(ids)
    g.position_ids.copyin_numpy(pos)
    ms, _ = timed(h, rt, 50)
    steps = h.schedule()
    wbytes = (12 * 7087872 + 50257 * 768 + 1024 * 768) * 2
    print(json.dumps({"config": "C2 gpt2-small B=1 S=128 fp16 (no LM head, as the reference exports it)", "ms_per_forward": round(ms, 4),
                      "tokens_per_s": round(cfg.batch * cfg.seq / ms * 1e3, 1), "scheduled_steps": len(steps),
                      "weight_bytes": wbytes, "hbm_floor_ms": round(wbytes / PEAKS["hbm_gbs"] / 1e6, 4)}))


def gpt2_decode(batch=16, pos=511):
    cfg = G.GPT2Config(batch=batch, lm_head=True)
    rt = B.CudaRuntime(0)
    h = B.GraphHandler(rt)
    g = G.build_gpt2_decode(h, cfg, 1024)
    h.data_malloc()
    G.fill_gpt2_weights_host(g)
    rng = np.random.default_rng(2)
    for c in g.k_caches + g.v_caches:
        c.copyin_numpy((rng.standard_normal(c.shape(), dtype=np.float32) * 0.5).astype(np.float16))
    g.input_ids.copyin_numpy(rng.integers(0, cfg.vocab, size=(batch, 1)).astype(np.int64))
    g.position_ids.copyin_numpy(np.full((batch, 1), pos, np.int64))
    ms, launches = timed(h, rt, 100)
    byts = cfg.algorithmic_bytes(pos)
    floor = byts / PEAKS["hbm_gbs"] / 1e6
    print(json.dumps({"config": f"gpt2-small decode step B={batch} p={pos} fp16 (tied LM head)", "ms_per_step": round(ms, 4),
                      "tokens_per_s": round(batch / ms * 1e3, 1), "algorithmic_bytes": byts, "hbm_floor_ms": round(floor, 4),
                      "frac_of_bound": round(floor / ms, 4), "launches_per_step": launches,
                      "scheduled_steps": len(h.schedule()), "card": card()}))


def resnet(batch):
    cfg = G.ResNetConfig(batch=batch)
    rt = B.CudaRuntime(0)
    h = B.GraphHandler(rt)
    g = G.build_resnet50(h, cfg)
    h.data_malloc()
    G.fill_resnet_weights_host(g)
    x = np.random.default_rng(3).standard_normal((cfg.batch, 3, cfg.image, cfg.image)).astype(np.float32)
    g.input.copyin_numpy(G.to_storage(x, cfg.dtype))
    ms, _ = timed(h, rt, 10, warm=3)
    flop = 2 * 4.09e9 * batch
    tf = flop / ms / 1e9
    out = G.from_storage(g.out.copyout_numpy(), cfg.dtype)
    print(json.dumps({"config": f"C4 resnet50 B={batch} fp16", "ms_per_batch": round(ms, 3),
                      "images_per_s": round(batch / ms * 1e3, 1), "tflops": round(tf, 1),
                      "frac_of_measured_dense_peak": round(tf / PEAKS["bf16_tflops"], 4),
                      "scheduled_steps": len(h.schedule()), "finite": bool(np.isfinite(out).all())}))


if __name__ == "__main__":
    args = [a for a in sys.argv[1:] if not a.startswith("--")] or ["gpt2", "resnet"]
    batch = 64
    if "--batch" in sys.argv:
        batch = int(sys.argv[sys.argv.index("--batch") + 1])
    if "gpt2" in args:
        gpt2()
    if "gpt2-decode" in args:
        gpt2_decode()
    if "resnet" in args:
        resnet(batch)
