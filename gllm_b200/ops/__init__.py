"""Op namespace.

`gllm_b200.ops.ref`   — pure-PyTorch oracle (CPU-capable; tests + CPU plumbing).
`gllm_b200.ops.sm100` — the product: hand-written sm_90a kernels.
`gllm_b200.ops.cpu`   — CPU stand-ins of the ops the model and the sampler call, with the sm100 signatures.

Model code takes one table per device, `table(device)`, and calls it with the same arguments on either. CUDA devices
always run sm100; there is no silent fallback — if the kernel library cannot be loaded on a GPU box, the first op
raises.
"""
import torch

from gllm_b200.ops import cpu, sm100


def table(device):
    """The op table of `device`: `ops.sm100` on a CUDA device, `ops.cpu` otherwise."""
    return sm100 if torch.device(device).type == "cuda" else cpu
