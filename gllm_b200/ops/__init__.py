"""Op namespace.

`gllm_b200.ops.ref`   — pure-PyTorch oracle (CPU-capable; tests + CPU plumbing).
`gllm_b200.ops.sm100` — the product: hand-written sm_90a kernels.
`gllm_b200.ops.cpu`   — CPU stand-ins of the sampler ops, with the sm100 signatures, over the oracle.

CUDA tensors always run sm100; there is no silent fallback — if the kernel library cannot be loaded on a GPU box,
importing the ops raises.
"""
