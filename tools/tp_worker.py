#!/usr/bin/env python
"""One rank of a tensor-parallel parity run (launched by torchrun from tests/test_gpu_multi.py):
builds the sharded tiny Llama decode graph on this rank's GPU, runs it with (a) the fused NVLink one-shot
all-reduce + residual + RMSNorm kernel and (b) in-graph NCCL all-reduce, and saves the logits."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist

from infinitensor_b200 import backend as B
from infinitensor_b200 import graphs as G


def run(mode, cfg, rank, world, local):
    os.environ["ITB_FUSION_MASK"] = "31" if mode == "p2p" else "15"
    rt = B.CudaRuntime(local)
    box = [B.CudaRuntime.nccl_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(box, src=0)
    rt.init_comm_with_id(box[0], world, rank)
    if mode == "p2p":
        handles = [None] * world
        dist.all_gather_object(handles, rt.p2p_export())
        rt.p2p_import(handles, world, rank)
    h = B.GraphHandler(rt)
    g = G.build_llama_decode(h, cfg, world, rank)
    sched = h.schedule()
    h.data_malloc()
    G.fill_llama_weights_host(g, world, rank)
    for li in range(cfg.layers):
        g.k_caches[li].copyin_numpy(G.to_storage(G.llama_cache_values(cfg, li, "k", world, rank), cfg.dtype))
        g.v_caches[li].copyin_numpy(G.to_storage(G.llama_cache_values(cfg, li, "v", world, rank), cfg.dtype))
    outs = []
    for step in range(3):
        g.input_ids.copyin_numpy((np.arange(cfg.batch, dtype=np.int64).reshape(-1, 1) * 7 + step) % cfg.vocab)
        g.position_ids.copyin_numpy(np.full((cfg.batch, 1), 9 + step, np.int64))
        h.run_with_cudagraph()
        outs.append(G.from_storage(g.logits.copyout_numpy(), cfg.dtype).copy())
    dist.barrier()
    return sched, np.stack(outs)


def main():
    dist.init_process_group("nccl")
    rank, world = dist.get_rank(), dist.get_world_size()
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dtype = int(os.environ.get("TP_DTYPE", "16"))
    kv = os.environ.get("TP_KV_HEADS")  # grouped-query attention: KV heads of the unsharded model
    cfg = G.LlamaConfig(layers=2, d_model=1024, heads=8, head_dim=128, ffn=2816, vocab=2048, s_max=64, batch=16, dtype=dtype,
                        kv_heads=int(kv) if kv else None)
    out = os.environ["TP_OUT"]
    for mode in ("p2p", "nccl"):
        sched, logits = run(mode, cfg, rank, world, local)
        np.save(f"{out}.{mode}.{rank}.npy", logits)
        if rank == 0:
            with open(f"{out}.{mode}.sched", "w") as f:
                f.write("\n".join(sched))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
