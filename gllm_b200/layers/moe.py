"""Mixture-of-experts block: router -> top-k -> experts (EP or TP sharded) [+ shared expert].

Reference: gllm/layers/moe/fused_moe_triton/layer.py:197-369 (FusedMoE), gllm/models/qwen2_moe.py:35-89,
gllm/models/mixtral.py:28-54. Sharding follows the reference: with EP (default when tp > 1) every
rank holds `E / ep` whole experts (contiguous block, remainder on the last rank); without EP every
rank holds all experts with `intermediate / tp` columns. The block returns the *partial* sum over
this rank's experts; the caller reduces it over the TP group together with the following
residual-add + RMSNorm (`TPComm.reduce_add_norm`).

On CUDA the experts run as one grouped wgmma GEMM pair over expert-sorted token slots
(csrc/moe/); the all-to-all dispatch/combine variant lives in parallel/fused.py.
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import nn

from gllm_b200 import ops
from gllm_b200.models import weight_utils as wu
from gllm_b200.ops import ref
from gllm_b200.parallel import state as ps


def _param(*shape, dtype, device):
    return nn.Parameter(torch.empty(shape, dtype=dtype, device=device), requires_grad=False)


class FusedMoE(nn.Module):
    def __init__(self, num_experts: int, top_k: int, hidden: int, intermediate: int, dtype, device,
                 renormalize: bool = True, use_ep: Optional[bool] = None, scoring: str = "softmax",
                 n_group: int = 0, topk_group: int = 0, routed_scaling: float = 1.0, bias_correction: bool = False,
                 quant: Optional[str] = None):
        super().__init__()
        self.ops = ops.table(device)
        self.quant = quant if (quant == "fp8" and hidden % 128 == 0) else None
        st = ps.get_state()
        self.num_experts, self.top_k, self.hidden = num_experts, top_k, hidden
        self.renormalize, self.scoring = renormalize, scoring
        self.n_group, self.topk_group, self.routed_scaling = n_group, topk_group, routed_scaling
        self.tp_size, self.tp_rank = st.tp_size, st.tp_rank
        self.use_ep = (st.ep_size > 1) if use_ep is None else (use_ep and st.tp_size > 1)
        if self.use_ep:
            self.e_start, self.e_local = wu.expert_range(num_experts, st.ep_rank, st.ep_size)
            self.inter = intermediate
            emap = torch.full((num_experts,), -1, dtype=torch.int32)
            emap[self.e_start:self.e_start + self.e_local] = torch.arange(self.e_local, dtype=torch.int32)
            self.register_buffer("expert_map", emap.to(device), persistent=False)
        else:
            self.e_start, self.e_local = 0, num_experts
            assert intermediate % st.tp_size == 0
            self.inter = intermediate // st.tp_size
            self.expert_map = None
        self.router_w = _param(num_experts, hidden, dtype=dtype, device=device)
        self.e_bias = _param(num_experts, dtype=torch.float32, device=device) if bias_correction else None
        if self.quant == "fp8" and self.inter % 128 != 0:
            self.quant = None
        if self.quant == "fp8":
            # block-scaled e4m3 experts (reference: Fp8MoEMethod, fused_moe_triton/layer.py:99-194); scales are
            # kept per 64 weight rows so an interleaved [64 gate | 64 up] GEMM tile can carry two block scales
            f8 = torch.float8_e4m3fn
            self.w13 = nn.Parameter(torch.zeros(self.e_local, 2 * self.inter, hidden, dtype=f8, device=device),
                                    requires_grad=False)
            self.w2 = nn.Parameter(torch.zeros(self.e_local, hidden, self.inter, dtype=f8, device=device),
                                   requires_grad=False)
            self.w13_ws = nn.Parameter(torch.ones(self.e_local, 2 * self.inter // 64, hidden // 128,
                                                  dtype=torch.float32, device=device), requires_grad=False)
            self.w2_ws = nn.Parameter(torch.ones(self.e_local, hidden // 64, self.inter // 128,
                                                 dtype=torch.float32, device=device), requires_grad=False)
        else:
            self.w13 = _param(self.e_local, 2 * self.inter, hidden, dtype=dtype, device=device)
            self.w2 = _param(self.e_local, hidden, self.inter, dtype=dtype, device=device)

    # -- routing ----------------------------------------------------------------------------------
    def process_weights(self):
        """The wgmma GEMM wants N % 8 == 0: expert counts like 60 (Qwen1.5-MoE) get a zero-padded router
        weight, built once after loading (before CUDA-graph capture); the logits are sliced back to E columns."""
        if self.num_experts % 8 != 0:
            e_pad = (self.num_experts + 7) // 8 * 8
            old = getattr(self, "_router_pad", None)
            if old is None:
                old = torch.zeros(e_pad, self.hidden, dtype=self.router_w.dtype, device=self.router_w.device)
                self._router_pad = old
            old[: self.num_experts].copy_(self.router_w.data)

    def _router_logits(self, h: torch.Tensor) -> torch.Tensor:
        if self.num_experts % 8 != 0:
            if getattr(self, "_router_pad", None) is None:
                assert not (torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()), \
                    "call model.process_weights() before capture"
                self.process_weights()
            return self.ops.linear(h, self._router_pad)[:, : self.num_experts]
        return self.ops.linear(h, self.router_w)

    def route(self, h: torch.Tensor):
        logits = self._router_logits(h)
        if self.n_group > 0:
            return self.ops.grouped_topk(logits, self.top_k, self.renormalize, self.n_group, self.topk_group,
                                         self.scoring, self.e_bias, self.routed_scaling)
        return self.ops.topk_softmax(logits, self.top_k, self.renormalize)

    def forward(self, h: torch.Tensor, tpc=None) -> torch.Tensor:
        w, ids = self.route(h)
        if self.quant == "fp8":
            return self.ops.fused_experts_fp8(h, self.w13, self.w13_ws, self.w2, self.w2_ws, w, ids, self.expert_map)
        return self.ops.fused_experts(h, self.w13, self.w2, w, ids, self.expert_map)

    # -- weights ----------------------------------------------------------------------------------
    def load_expert(self, global_e: int, gate: torch.Tensor, up: torch.Tensor, down: torch.Tensor):
        """HF per-expert tensors gate/up [I, H], down [H, I]."""
        if not (self.e_start <= global_e < self.e_start + self.e_local):
            return
        le = global_e - self.e_start
        if self.use_ep or self.tp_size == 1:
            gu = torch.cat([gate, up], dim=0)
        else:
            gu = wu.shard_gate_up(gate, up, self.tp_rank, self.tp_size)
            down = wu.shard_cols(down, self.tp_rank, self.tp_size)
        # w13: gate/up rows interleaved as the grouped GEMM's SiLU-gate epilogue reads them (fp8: I % 128 == 0)
        if self.quant == "fp8":
            q13, s13 = _block_quant_rows64(gu)
            q2, s2 = _block_quant_rows64(down)
            self.w13.data[le].copy_(ref.interleave_gate_up(q13.view(torch.uint8), 64).view(torch.float8_e4m3fn))
            self.w13_ws.data[le].copy_(ref.interleave_gate_up(s13, 1))
            self.w2.data[le].copy_(q2)
            self.w2_ws.data[le].copy_(s2)
            return
        self.w13.data[le].copy_(ref.interleave_gate_up(gu, ref.moe_gate_up_block(self.inter)))
        self.w2.data[le].copy_(down)


def _block_quant_rows64(w: torch.Tensor):
    """[N, K] -> (e4m3 [N, K], fp32 scales [N/64, K/128]): `weight_utils.fp8_block_quant` with the scales
    repeated per 64-row half block, so that an interleaved [64 gate | 64 up] GEMM tile carries two block scales."""
    q, sc = wu.fp8_block_quant(w)
    return q, sc.repeat_interleave(2, 0)[: (w.shape[0] + 63) // 64]


class SparseMoeBlock(nn.Module):
    """Router + routed experts + optional (sigmoid-gated) shared expert; returns a TP-partial sum."""

    def __init__(self, spec, layer_id: int, device):
        super().__init__()
        from gllm_b200.models.decoder import DenseMLP
        m = spec.moe
        self.experts = FusedMoE(m.num_experts, m.top_k, spec.hidden_size, m.intermediate_size, spec.dtype, device,
                                renormalize=m.norm_topk_prob, scoring=m.scoring, n_group=m.n_group,
                                topk_group=m.topk_group, routed_scaling=m.routed_scaling,
                                bias_correction=m.has_bias_correction, quant=getattr(spec, "quant", None))
        self.shared = None
        self.shared_gate_w = None
        if m.shared_intermediate_size > 0:
            self.shared = DenseMLP(spec.hidden_size, m.shared_intermediate_size, spec.dtype, device, spec=spec)
            if m.shared_gate:
                self.shared_gate_w = _param(1, spec.hidden_size, dtype=spec.dtype, device=device)

    def forward(self, h: torch.Tensor, tpc) -> torch.Tensor:
        out = self.experts(h, tpc)
        if self.shared is not None:
            # partial (un-reduced) shared-expert output: reduced together with the routed experts —
            # the reference double-reduces here on Qwen2-MoE (SURVEY §2.2 C23); we do it once.
            s = self.experts.ops.linear(self.shared.act(h, tpc), self.shared.down_weight())
            if self.shared_gate_w is not None:
                g = torch.sigmoid(torch.nn.functional.linear(h.float(), self.shared_gate_w.float()))
                s = (s.float() * g).to(s.dtype)
            out = out + s
        return out

    def load_weights(self, reader, pre: str, nm: dict):
        ex = self.experts
        ex.router_w.data.copy_(reader.get(pre + nm["router"]))
        if ex.e_bias is not None and "router_bias" in nm and reader.has(pre + nm["router_bias"]):
            ex.e_bias.data.copy_(reader.get(pre + nm["router_bias"]).float())
        fused_name = nm.get("experts_fused_gate_up", "mlp.experts.gate_up_proj")
        first_expert = pre + nm["expert"].format(e=ex.e_start) + nm["e_gate"]
        if not reader.has(first_expert) and reader.has(pre + fused_name):
            # fused expert tensors: Qwen3-VL-MoE stores [E, H, 2I] / [E, I, H] (transposed);
            # transformers>=5 in-memory layout is [E, 2I, H] / [E, H, I]
            gu = reader.get(pre + fused_name)
            dn = reader.get(pre + nm.get("experts_fused_down", "mlp.experts.down_proj"))
            transposed = gu.shape[1] == ex.hidden and gu.shape[2] != ex.hidden
            for e in range(ex.e_start, ex.e_start + ex.e_local):
                if transposed:
                    inter = gu.shape[-1] // 2
                    g = gu[e, :, :inter].t().contiguous()
                    u = gu[e, :, inter:].t().contiguous()
                    d = dn[e].t().contiguous()
                else:
                    inter = gu.shape[1] // 2
                    g, u, d = gu[e, :inter], gu[e, inter:], dn[e]
                ex.load_expert(e, g, u, d)
        else:
            for e in range(ex.e_start, ex.e_start + ex.e_local):
                ep = pre + nm["expert"].format(e=e)
                ex.load_expert(e, reader.get(ep + nm["e_gate"]), reader.get(ep + nm["e_up"]),
                               reader.get(ep + nm["e_down"]))
        if self.shared is not None:
            sp = pre + nm["shared"]
            tp, tr = ex.tp_size, ex.tp_rank
            gate, up = reader.get(sp + "gate_proj.weight"), reader.get(sp + "up_proj.weight")
            self.shared.set_gate_up(wu.shard_gate_up(gate, up, tr, tp))
            from gllm_b200.models.decoder import _store_linear
            _store_linear(self.shared.down_w, self.shared.down_ws,
                          wu.shard_cols(reader.get(sp + "down_proj.weight"), tr, tp))
            if self.shared_gate_w is not None:
                self.shared_gate_w.data.copy_(reader.get(pre + nm["shared_gate"]))


def make_moe_block(spec, layer_id: int, device):
    return SparseMoeBlock(spec, layer_id, device)
