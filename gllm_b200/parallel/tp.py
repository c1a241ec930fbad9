"""Tensor-parallel execution strategies for a decoder block.

The model code never calls a collective directly. It asks a `TPComm` to run the two Megatron
patterns of a block:

    col_linear(x, w, b)                         column-parallel GEMM   (QKV, gate/up)
    row_linear_add_norm(x, w, res, nw, eps)     row-parallel GEMM -> sum over ranks -> residual add
                                                -> RMSNorm  (O-proj / down-proj + the next norm)

`TPComm`       : tp == 1, or the NCCL baseline (GEMM -> all_reduce -> fused add+norm — exactly the
                 reference's sequence, gllm/layers/linear.py:247-250; this is the "ref-mode" used as
                 correctness oracle and measured baseline, and the gloo path for CPU tests).
`FusedTPComm`  : (parallel/fused.py) the product path — token-sharded activations, GEMM ⊕
                 reduce-scatter and all-gather ⊕ GEMM over NVLink peer memory.
"""
from __future__ import annotations

from typing import Callable, Optional

import torch

from gllm_b200 import ops as _ops
from gllm_b200.parallel import state as ps


class TPComm:
    fused = False

    def __init__(self, ops):
        self.ops = ops     # op table of this rank's device (`gllm_b200.ops.table`)
        st = ps.get_state()
        self.tp_size = st.tp_size
        self.tp_rank = st.tp_rank

    # hooks the runner calls around a forward pass (used by the fused implementation)
    def begin_forward(self, num_tokens: int):
        pass

    def first_norm(self, x: torch.Tensor, norm_w: torch.Tensor, eps: float):
        """Embedding output -> (normed block input, residual stream)."""
        h, _ = self.ops.rmsnorm(x, norm_w, eps)
        return h, x

    def materialize(self, h: torch.Tensor) -> torch.Tensor:
        """Make `h` safe to read by kernels that are not collective-aware (no-op here)."""
        return h

    def stage_exit(self, residual: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
        """Residual stream in the replicated [T, H] form a pipeline stage boundary ships (no-op here)."""
        return residual

    def col_linear(self, x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
        return self.ops.linear(x, w, bias)

    def col_linear_silu_mul(self, x: torch.Tensor, w_interleaved: torch.Tensor) -> torch.Tensor:
        return self.ops.linear_silu_mul(x, w_interleaved)

    def all_reduce(self, x: torch.Tensor) -> torch.Tensor:
        return ps.tp_all_reduce(x)

    def reduce_add_norm(self, partial: torch.Tensor, residual: Optional[torch.Tensor], norm_w: torch.Tensor,
                        eps: float):
        """sum partial over TP ranks; residual += sum; return (rmsnorm(residual), residual)."""
        if self.tp_size > 1:
            ps.tp_all_reduce(partial)
        if residual is None:
            normed, _ = self.ops.rmsnorm(partial, norm_w, eps)
            return normed, partial
        return self.ops.rmsnorm(partial, norm_w, eps, residual)

    def moe_add_norm(self, block, h: torch.Tensor, residual: Optional[torch.Tensor], norm_w: torch.Tensor,
                     eps: float):
        """MoE block (TP-partial output) + reduce + residual add + next RMSNorm. The fused strategy
        overrides this with the all-to-all dispatch/combine form for EP models."""
        partial = block(self.materialize(h), self)
        return self.reduce_add_norm(partial, residual, norm_w, eps)

    def row_linear_add_norm(self, x: torch.Tensor, w: torch.Tensor, residual: Optional[torch.Tensor],
                            norm_w: torch.Tensor, eps: float, bias: Optional[torch.Tensor] = None,
                            delta: Optional[Callable[[torch.Tensor], None]] = None):
        """`delta(partial)` (LoRA) adds to this rank's partial GEMM output in place, before the sum over ranks."""
        # bias is added once (rank 0) like the reference (gllm/layers/linear.py:230-258)
        partial = self.ops.linear(x, w, bias if self.tp_rank == 0 else None)
        if delta is not None:
            delta(partial)
        return self.reduce_add_norm(partial, residual, norm_w, eps)

    def row_linear(self, x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None,
                   delta: Optional[Callable[[torch.Tensor], None]] = None) -> torch.Tensor:
        out = self.ops.linear(x, w, bias if self.tp_rank == 0 else None)
        if delta is not None:
            delta(out)
        return self.all_reduce(out)

    def gather_logits(self, local_logits: torch.Tensor, vocab_size: int) -> torch.Tensor:
        """[B, Vp/tp] per rank -> [B, V] (reference: vocab_parallel_embedding.py:423-435)."""
        if self.tp_size == 1:
            return local_logits[:, :vocab_size]
        return ps.tp_all_gather_last_dim(local_logits)[:, :vocab_size]


def make_tp_comm(device, fused: bool = False, **kw) -> TPComm:
    st = ps.get_state()
    if fused and st.tp_size > 1 and torch.cuda.is_available():
        from gllm_b200.parallel.fused import FusedTPComm
        return FusedTPComm(device=device, **kw)
    return TPComm(_ops.table(device))
