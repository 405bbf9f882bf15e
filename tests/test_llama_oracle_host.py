"""CPU tier for the graph oracle of tests/llama_oracle.py: one step of every Llama decode variant build_llama_decode accepts,
each feature combined with every other, runs on it."""
import itertools

import numpy as np
import pytest

F32, F16, BF16 = 1, 10, 16

# (G, D, FP8 cache, int4 weights, seq); an FP8 cache takes one token per step
VARIANTS = [v for v in itertools.product((1, 2), (128, 64), (False, True), (False, True), (1, 4)) if not (v[2] and v[4] > 1)]


@pytest.mark.parametrize("G_,D,kv_fp8,int4,seq", VARIANTS)
def test_every_variant_runs_on_the_oracle(G_, D, kv_fp8, int4, seq):
    from infinitensor_b200 import graphs as G
    from tests.llama_oracle import oracle_graph
    heads = 256 // D
    cfg = G.LlamaConfig(layers=1, d_model=256, heads=heads, kv_heads=heads // G_, head_dim=D, ffn=256, vocab=64, s_max=16,
                        batch=2, dtype=BF16, kv_fp8=kv_fp8, int4_block=32 if int4 else 0)
    oh, og = oracle_graph(cfg, seq)
    og.input_ids.copyin_numpy(np.arange(2 * seq, dtype=np.int64).reshape(2, seq) * 7 % cfg.vocab)
    og.position_ids.copyin_numpy(np.broadcast_to(3 + np.arange(seq), (2, seq)).astype(np.int64).copy())
    oh.run()
    logits = og.logits.f32()
    assert logits.shape == (2, seq, cfg.vocab) and np.isfinite(logits).all()
