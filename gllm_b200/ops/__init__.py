"""Op namespace.

`gllm_b200.ops.ref`   — pure-PyTorch oracle (CPU-capable; tests + CPU plumbing).
`gllm_b200.ops.sm100` — the product: hand-written sm_90a kernels.

`backend()` picks sm100 whenever a CUDA device is present; there is no silent fallback —
if the kernel library cannot be loaded on a GPU box, importing the ops raises.
"""
from __future__ import annotations

import os

import torch

_forced = os.environ.get("GLLM_B200_BACKEND", "")


def backend() -> str:
    if _forced:
        return _forced
    return "sm100" if torch.cuda.is_available() else "ref"


def use_sm100(t: torch.Tensor | None = None) -> bool:
    if t is not None and not t.is_cuda:
        return False
    return backend() == "sm100"
