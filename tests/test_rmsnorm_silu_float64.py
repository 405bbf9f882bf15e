"""The unfused rmsnorm_kernel (it_b200_rmsnorm / _constw, every path) and silu_mul_kernel against float64 (helpers in
tests/operand64.py): every stored element must equal the float64 value rounded as the kernel rounds it or, where the fp32
arithmetic before the rounding leaves it ambiguous, lie between the two candidates.
"""
import re

import numpy as np
import pytest

from tests import operand64, ref64
from tests.ref64 import BF16, F16, F32

# ambiguous share of an f16 / bf16 RMSNorm operand: the longest chain here (hidden 5120, 16 items per thread + 10) gives a
# window of 34 2^-24 against f16's spacing of 2^-10 .. 2^-11 relative: under 1 % of the elements straddle a rounding point
MAX_AMB_SHARE = 0.05


@pytest.fixture(scope="module")
def K():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from tests import kernel_harness
    return kernel_harness


def rmsnorm_path(dt, hidden):
    """rmsnorm_impl's choice for aligned pointers: "one" (one vector per thread), "vec" or "scalar", and items per thread"""
    V = 4 if dt == F32 else 8
    threads = 512 if hidden >= 4096 else 256 if hidden >= 1024 else 128
    if hidden % V:
        return "scalar", -(-hidden // threads)
    nv = hidden // V
    return ("one", V) if nv <= threads else ("vec", -(-nv // threads) * V)


RMS_HIDDEN = [4096, 1024, 5120, 1000, 1004, 1001]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F32, F16, BF16], ids=["fp32", "f16", "bf16"])
@pytest.mark.parametrize("hidden", RMS_HIDDEN)
def test_unfused_rmsnorm_float64(K, hidden, dt):
    """every element of it_b200_rmsnorm / _constw equals rnd(rnd(x rinv) w) or, where rinv's fp32 window straddles a rounding
    point, a value between the two ends"""
    x = operand64.rows(24, hidden, dt, hidden) if dt != F32 else \
        np.random.default_rng(hidden).standard_normal((24, hidden)).astype(np.float32) * ref64.row_scale(24)[:, None]
    w = operand64.norm_weight(hidden, dt, hidden + 1)
    path, items = rmsnorm_path(dt, hidden)
    op = operand64.rmsnorm_operand(x, w, dt, operand64.chain_length("block", hidden, items=items))
    fails = []
    for const_w in (False, True):
        got = K.rms_norm(x.astype(np.float32), w.astype(np.float32), dt, const_w)
        bad = op.outside(got)
        if bad.any():
            i, j = np.argwhere(bad)[0]
            fails.append(f"{path} const_w={const_w}: {int(bad.sum())} elements outside; first ({i}, {j}): got {got[i, j]!r}, "
                         f"nominal {op.a[i, j]!r}, candidates {op.lo[i, j]!r} .. {op.hi[i, j]!r}")
    assert not fails and op.share <= (1.0 if dt == F32 else MAX_AMB_SHARE), "\n".join(fails) or f"ambiguous {op.share:.3%}"


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F32, F16, BF16], ids=["fp32", "f16", "bf16"])
@pytest.mark.parametrize("n", [16 * 1024, 16 * 1000 + 5])
def test_unfused_silu_mul_float64(K, n, dt):
    """it_b200_silu_mul, vector loop and scalar tail: rnd(rnd(silu(g)) u) or the other candidate where ambiguous"""
    rng = np.random.default_rng(n)
    g = operand64.rnd(rng.standard_normal(n) * 3.0, dt) if dt != F32 else (rng.standard_normal(n) * 3.0).astype(np.float32)
    u = operand64.rnd(rng.standard_normal(n), dt) if dt != F32 else rng.standard_normal(n).astype(np.float32)
    op = operand64.silu_mul_operand(g, u, dt)
    got = K.silu_mul(np.asarray(g, np.float32), np.asarray(u, np.float32), dt)
    bad = op.outside(got)
    assert not bad.any(), f"{int(bad.sum())} elements outside; first {np.argwhere(bad)[0]}"


# ====================================================================== GPU: the intended kernels ran
def profiled_kernel_names():
    import torch
    from tests import kernel_harness as K
    x = np.random.default_rng(0).standard_normal((4, 5120)).astype(np.float32)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for dt in (F16, BF16):
            for h, cw in ((1024, True), (1024, False), (5120, False)):
                K.rms_norm(x[:, :h], np.ones(h, np.float32), dt, cw)
            K.silu_mul(x[0], x[1], dt)
        torch.cuda.synchronize()
    return sorted({e.name for e in prof.events() if "CUDA" in str(e.device_type)})


@pytest.mark.gpu
def test_unfused_cases_reach_the_intended_kernels():
    """in a child process, as test_attention_float64 does: a profiler session in the test process loses records of later ones"""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = "import json; from tests.test_rmsnorm_silu_float64 import profiled_kernel_names as f; print(json.dumps(f()))"
    r = subprocess.run([sys.executable, "-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    names = set(json.loads(r.stdout.strip().splitlines()[-1]))
    if not names:
        pytest.skip("the profiler recorded no CUDA kernel events (CUPTI activity tracing unavailable)")
    want = [r"rmsnorm_kernel<.*true, true>", r"rmsnorm_kernel<.*true, false>", r"rmsnorm_kernel<.*false, false>", r"silu_mul_kernel"]
    missing = [p for p in want if not any(re.search(p, nm) for nm in names)]
    assert not missing, f"not launched: {missing}; kernels seen: {sorted(names)}"
