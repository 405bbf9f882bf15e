"""smoke(): one tiny Llama-shape decode step on cuda:0 through the public graph API, CUDA-graph replayed,
checked against the CPU oracle executing the same graph description."""


def run():
    from infinitensor_b200 import graphs as G
    from tests.llama_oracle import run_llama_parity
    worst, launches, _ = run_llama_parity(G.LlamaConfig.tiny(dtype=16, layers=2, batch=4), pos=5, steps=2)
    assert launches > 0
    print(f"smoke ok: tiny Llama decode (bf16, 2 layers, CUDA graph replay) max rel err {worst:.3e}, "
          f"{launches} kernel launches")
