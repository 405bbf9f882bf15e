#!/usr/bin/env python
"""One rank of the all-reduce float64 run on real GPUs (launched by torchrun from tests/test_allreduce_float64.py).

Builds AllReduceSum -> Add(residual) -> RMSNorm(weight) on this rank's GPU with the comm workspaces mapped through the
production cudaIpc exchange, so the step runs as the fused one-shot kernel with every rank live.  Every rank derives the
whole world's partials from one seed per step and feeds its own, so each rank can check its outputs against the same
references as the one-device tests (tests/ar64.py): the Add output bit for bit against the fp32 emulation and within the
float64 bound, the RMSNorm output within its interval and bound.  Runs eager steps, then CUDA-graph replays, every step with
new inputs, and writes {cases: [...], fails: [...]} to $AR_OUT.<rank>.json."""
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist

from infinitensor_b200 import backend as B
from infinitensor_b200 import graphs as G
from tests import ar64
from tests.ar64 import BF16, F16, F32

CASES = [(BF16, 16, 4096), (F16, 64, 2048), (F32, 7, 4096)]   # (dtype, tokens, hidden)
EAGER, REPLAYS = 40, 60
REGIMES = ["normal", "spread", "cancel", "residual_dominates"]


def run_case(dt, M, H, rank, world, local):
    rt = B.CudaRuntime(local)
    handles = [None] * world
    dist.all_gather_object(handles, rt.p2p_export())
    rt.p2p_import(handles, world, rank)
    h = B.GraphHandler(rt)
    x, r, w = h.tensor([M, H], dt), h.tensor([M, H], dt), h.tensor([H], dt)
    x.set_input()
    r.set_input()
    w.set_weight()
    s = h.add(h.allReduceSum(x, None), r, None)
    y = h.RMSNorm(s, w, None)
    s.set_output()
    y.set_output()
    sched = h.schedule()
    h.data_malloc()
    _, _, wv = ar64.inputs(dt, 1, 1, H, "normal", 99)
    w.copyin_numpy(G.to_storage(wv, dt))
    fails, digest = [], hashlib.sha256()
    what = f"rank {rank}/{world} {ar64.NAMES[dt]} M {M} H {H}"
    for step in range(EAGER + REPLAYS):
        P, R, _ = ar64.inputs(dt, world, M, H, REGIMES[step % len(REGIMES)], 1000 * dt + step, True, False)
        x.copyin_numpy(G.to_storage(P[rank], dt))
        r.copyin_numpy(G.to_storage(R, dt))
        dist.barrier()
        if step < EAGER:
            h.run()
        else:
            h.run_with_cudagraph()
        sb, yb = s.copyout_numpy(), y.copyout_numpy()
        digest.update(sb.tobytes())
        digest.update(yb.tobytes())
        so = G.from_storage(sb, dt).astype(np.float32)
        yo = G.from_storage(yb, dt).astype(np.float32)
        emu, _ = ar64.emulate(P, R, wv, dt)
        if not np.array_equal(so.view(np.int32), emu.view(np.int32)):
            i, j = np.argwhere(so.view(np.int32) != emu.view(np.int32))[0]
            fails.append(f"{what} step {step}: out differs from the emulation at {ar64.describe(dt, H, i, j)}")
        Ro = ar64.out_ref(P, R, dt)
        if Ro.violations(so).any():
            fails.append(f"{what} step {step}: out outside the float64 bound")
        fin = np.isfinite(so).all(1)
        op, Rn = ar64.norm_operand(so[fin], wv, dt), ar64.norm_bound(so[fin], wv, dt)
        if (op.outside(yo[fin]) | Rn.violations(yo[fin])).any():
            fails.append(f"{what} step {step}: out_norm outside its interval / bound")
    dist.barrier()
    return dict(case=f"{ar64.NAMES[dt]}_M{M}_H{H}", steps=EAGER + REPLAYS, schedule=sched, digest=digest.hexdigest()), fails


def main():
    dist.init_process_group("nccl")
    rank, world = dist.get_rank(), dist.get_world_size()
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    cases, fails = [], []
    for dt, M, H in CASES:
        c, f = run_case(dt, M, H, rank, world, local)
        cases.append(c)
        fails += f
    with open(f"{os.environ['AR_OUT']}.{rank}.json", "w") as fh:
        json.dump(dict(cases=cases, fails=fails), fh)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
