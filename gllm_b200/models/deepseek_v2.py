"""DeepSeek-V2 / V3 / R1 (and Moonlight / Kimi-K2, same architecture): MLA attention + DeepSeek MoE
(reference: gllm/models/deepseek_v2.py:61-548, gllm/layers/attention.py:65-492).

MLA here stores the *latent* KV cache — `[kv_c (kv_lora_rank, RMS-normed) | k_pe (rope dims, rotated)]`
per token, one "head", replicated on every TP rank (like the reference's MLA `Segment`,
gllm/memory_manager.py:38-42) — and q heads are split over TP. Routing uses the group-limited top-k
kernel (sigmoid + bias-corrected `noaux_tc` for V3), experts run through the grouped wgmma GEMMs,
shared experts are an ordinary gated MLP whose partial output is reduced together with the routed one.

On sm_90a the attention runs in the *absorbed* form: q_nope·W_UK per head (batched wgmma GEMM over strided
views, written straight into the 576-wide query), fused RoPE + latent-cache write, split-KV multi-query attention
over the paged latent cache (csrc/attn/mla_attention.cu), then out_lat·W_UV per head (the same batched GEMM,
written in the [T, heads·v] layout o_proj reads). No cuBLAS and no host synchronisation on that path, so decode
batches run inside CUDA graphs (SURVEY §2.3 K11/K13). The CPU / odd-shape path below evaluates the *expanded* form
with PyTorch ops per sequence (the numerical oracle of the GPU path).
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F
from torch import nn

from gllm_b200 import ops
from gllm_b200.layers.moe import SparseMoeBlock
from gllm_b200.layers.rotary import build_rope
from gllm_b200.models import weight_utils as wu
from gllm_b200.models.decoder import (CausalLM, DenseMLP, ModelSpec, MoESpec, _linear_params, _param, _qw,
                                      _store_linear)
from gllm_b200.models.registry import _dtype
from gllm_b200.ops import ref
from gllm_b200.parallel import state as ps
from gllm_b200.parallel.tp import TPComm


class MLAAttention(nn.Module):
    def __init__(self, spec: ModelSpec, layer_id: int, rope, device):
        super().__init__()
        x = spec.extra
        st = ps.get_state()
        tp = st.tp_size
        self.ops = ops.table(device)
        self.layer_id = layer_id
        self.tp, self.tr = tp, st.tp_rank
        self.num_heads = spec.num_heads // tp
        self.nope, self.rope_dim, self.v_dim = x["qk_nope_head_dim"], x["qk_rope_head_dim"], x["v_head_dim"]
        self.qk_dim = self.nope + self.rope_dim
        self.kv_lora, self.q_lora = x["kv_lora_rank"], x.get("q_lora_rank")
        self.rope = rope
        self.eps = spec.rms_eps
        self.scaling = self.qk_dim ** -0.5 * rope.attn_mscale
        h, dt = spec.hidden_size, spec.dtype
        # The projections follow the checkpoint's quantisation (fp8 block-scaled for V3 / R1: (weight, scale_inv)
        # pairs on the UTCQMMA GEMM — reference plumbs quant_config into them, gllm/models/deepseek_v2.py:280-440).
        # kv_b_proj stays bf16: it is only ever used absorbed, as the per-head W_UK / W_UV operands.
        if self.q_lora:
            self.q_a_w, self.q_a_ws = _linear_params(self.q_lora, h, spec, device)
            self.q_a_norm_w = _param(self.q_lora, dtype=dt, device=device, fill=1.0)
            self.q_b_w, self.q_b_ws = _linear_params(self.num_heads * self.qk_dim, self.q_lora, spec, device)
        else:
            self.q_w, self.q_ws = _linear_params(self.num_heads * self.qk_dim, h, spec, device)
        self.kv_a_w, self.kv_a_ws = _linear_params(self.kv_lora + self.rope_dim, h, spec, device)
        self.kv_a_norm_w = _param(self.kv_lora, dtype=dt, device=device, fill=1.0)
        self.kv_b_w = _param(self.num_heads * (self.nope + self.v_dim), self.kv_lora, dtype=dt, device=device)
        self.o_w, self.o_ws = _linear_params(h, self.num_heads * self.v_dim, spec, device)
        self.o_b = None
        # attributes the generic runner looks at
        self.num_kv_heads = 1
        self.head_dim = self.kv_lora + self.rope_dim

    def forward(self, inp, h: torch.Tensor, kv_cache, tpc: TPComm) -> torch.Tensor:
        t = h.shape[0]
        hl = self.num_heads
        h = tpc.materialize(h)
        if self.q_lora:
            qa, _ = self.ops.rmsnorm(self.ops.linear(h, _qw(self.q_a_w, self.q_a_ws)), self.q_a_norm_w, self.eps)
            q = self.ops.linear(qa, _qw(self.q_b_w, self.q_b_ws))
        else:
            q = self.ops.linear(h, _qw(self.q_w, self.q_ws))
        q = q.view(t, hl, self.qk_dim)
        kv_a = self.ops.linear(h, _qw(self.kv_a_w, self.kv_a_ws))
        kv_c, _ = self.ops.rmsnorm(kv_a[:, : self.kv_lora].contiguous(), self.kv_a_norm_w, self.eps)
        if kv_cache is None:
            return q[:, :, : self.v_dim].reshape(t, hl * self.v_dim).contiguous()
        cache = kv_cache.k_cache[self.layer_id]
        # the absorbed kernels need kv_lora 512 / rope 64: the expanded form below serves every other shape
        if self.ops is ops.sm100 and self.kv_lora == 512 and self.rope_dim == 64:
            return self._forward_absorbed(inp, q, kv_c, kv_a[:, self.kv_lora:], cache)
        k_pe = kv_a[:, self.kv_lora:].contiguous().view(t, 1, self.rope_dim)
        q_pe = q[:, :, self.nope:].contiguous()
        # GPT-J style (interleaved) rotary on the rope dims only; oracle op (strided sub-views)
        ref.rope_kv_write(q_pe, k_pe, None, inp.positions, self.rope.cos_sin, self.rope_dim, False, None, None,
                          self.eps, None, None, None)
        latent = torch.cat([kv_c, k_pe.view(t, self.rope_dim)], dim=-1).view(t, 1, self.head_dim)
        ref.write_kv_cache(latent, None, cache, None, inp.slot_mapping)
        q = torch.cat([q[:, :, : self.nope], q_pe], dim=-1)
        out = torch.empty(t, hl, self.v_dim, dtype=h.dtype, device=h.device)
        qsl = inp.query_start_loc.tolist()
        sls = inp.seq_lens.tolist()
        for s in range(inp.num_seqs):
            q0, q1 = qsl[s], qsl[s + 1]
            ql, sl = q1 - q0, sls[s]
            if ql <= 0:
                continue
            lat = ref.gather_kv(cache, inp.block_table[s], sl)[:, 0]  # [L, 576]
            kvb = F.linear(lat[:, : self.kv_lora], self.kv_b_w).view(sl, hl, self.nope + self.v_dim)
            k = torch.cat([kvb[:, :, : self.nope], lat[:, None, self.kv_lora:].expand(sl, hl, self.rope_dim)], dim=-1)
            v = kvb[:, :, self.nope:]
            att = torch.einsum("qhd,khd->hqk", q[q0:q1].float(), k.float()) * self.scaling
            qi = torch.arange(ql, device=h.device).view(ql, 1) + (sl - ql)
            kj = torch.arange(sl, device=h.device).view(1, sl)
            att = att.masked_fill((kj > qi).unsqueeze(0), float("-inf"))
            out[q0:q1] = torch.einsum("hqk,khd->qhd", torch.softmax(att, -1), v.float()).to(h.dtype)
        return out.view(t, hl * self.v_dim)

    def process_weights(self):
        """W_UK [hl, nope, 512] and W_UV [hl, 512, v] views of kv_b_proj, made contiguous once, eagerly, after
        the weights are final and BEFORE any CUDA-graph capture (tensors created inside a capture only get
        their contents when the graph replays). Reference: MLAAttention.process_weights,
        gllm/layers/attention.py:106-127."""
        if not self.kv_b_w.is_cuda:
            return
        kvb = self.kv_b_w.data.view(self.num_heads, self.nope + self.v_dim, self.kv_lora)
        # both in the [batch, N, K] (nn.Linear) layout the batched GEMM reads:
        #   q_lat[:, h] = q_nope[:, h] @ W_UK[h]      -> weight [512 (N), nope (K)] = W_UK[h]^T
        #   out[:, h]   = out_lat[:, h] @ W_UV[h]^T   -> weight [v (N), 512 (K)]    = kv_b rows of the value part
        w_uk_nk, w_uv_nk = kvb[:, : self.nope, :].transpose(1, 2), kvb[:, self.nope:, :]
        old = getattr(self, "_w_abs", None)
        if old is not None:   # keep the addresses: captured CUDA graphs point at these tensors
            old[0].copy_(w_uk_nk)
            old[1].copy_(w_uv_nk)
        else:
            self._w_abs = (w_uk_nk.contiguous(), w_uv_nk.contiguous())

    def _absorbed_weights(self):
        if getattr(self, "_w_abs", None) is None:
            assert not torch.cuda.is_current_stream_capturing(), "call model.process_weights() before capture"
            self.process_weights()
        return self._w_abs

    def _forward_absorbed(self, inp, q, kv_c, k_pe, cache):
        """sm_90a path: multi-query attention over the latent cache (csrc/attn/mla_attention.cu). No host
        synchronisation, so decode batches run inside CUDA graphs."""
        t, hl = q.shape[0], self.num_heads
        w_uk, w_uv = self._absorbed_weights()
        q_full = torch.empty(t, hl, 576, dtype=q.dtype, device=q.device)
        self.ops.gemm_batched(q[:, :, : self.nope], w_uk, q_full[:, :, :512])   # per head: q_nope · W_UK
        self.ops.mla_rope_cache(q[:, :, self.nope:], q_full, k_pe, kv_c, self.rope.cos_sin, inp.positions,
                                inp.slot_mapping, cache)
        splits = self.ops.mla_splits(t, hl)
        out_lat = self.ops.mla_attention(q_full, cache, inp.block_table, inp.tok_seq, inp.positions, self.scaling,
                                         splits=splits)
        out = torch.empty(t, hl, self.v_dim, dtype=q.dtype, device=q.device)
        self.ops.gemm_batched(out_lat, w_uv, out)                               # per head: out_lat · W_UV
        return out.view(t, hl * self.v_dim)


class DeepseekDecoderLayer(nn.Module):
    def __init__(self, spec: ModelSpec, layer_id: int, local_id: int, rope, device):
        super().__init__()
        self.spec, self.layer_id, self.local_id = spec, layer_id, local_id
        dt, h = spec.dtype, spec.hidden_size
        self.input_norm_w = _param(h, dtype=dt, device=device, fill=1.0)
        self.post_norm_w = _param(h, dtype=dt, device=device, fill=1.0)
        self.attn = MLAAttention(spec, local_id, rope, device)
        self.is_moe = spec.is_moe_layer(layer_id)
        self.mlp = SparseMoeBlock(spec, layer_id, device) if self.is_moe else \
            DenseMLP(h, spec.intermediate_size, dt, device, spec=spec)

    def forward(self, inp, h, residual, kv_cache, tpc: TPComm, next_norm_w):
        eps = self.spec.rms_eps
        a = self.attn(inp, h, kv_cache, tpc)
        h, residual = tpc.row_linear_add_norm(a, _qw(self.attn.o_w, self.attn.o_ws), residual, self.post_norm_w, eps)
        if self.is_moe:
            partial = self.mlp(tpc.materialize(h), tpc)
            if next_norm_w is None:
                return tpc.all_reduce(partial), residual
            return tpc.reduce_add_norm(partial, residual, next_norm_w, eps)
        act = self.mlp.act(h, tpc)
        if next_norm_w is None:
            return tpc.row_linear(act, self.mlp.down_weight()), residual
        return tpc.row_linear_add_norm(act, self.mlp.down_weight(), residual, next_norm_w, eps)


class DeepseekForCausalLM(CausalLM):
    def __init__(self, spec: ModelSpec, device="cpu"):
        # build the generic skeleton with zero layers, then install MLA layers
        nn.Module.__init__(self)
        self.spec = spec
        st = ps.get_state()
        self.device = torch.device(device)
        self.ops = ops.table(device)
        self.layers_range = ps.get_pp_layers(spec.num_layers)
        self.is_first, self.is_last = ps.is_first_pp_rank(), ps.is_last_pp_rank()
        self.tp_size, self.tp_rank = st.tp_size, st.tp_rank
        x = spec.extra
        self.rope = build_rope(x["qk_rope_head_dim"], spec.max_position, spec.rope_theta, spec.rope_scaling,
                               x["qk_rope_head_dim"], False, device=device)
        dt, h = spec.dtype, spec.hidden_size
        self.vocab_padded = wu.pad_vocab(spec.vocab_size, self.tp_size)
        self.vocab_per_rank = self.vocab_padded // self.tp_size
        self.vocab_start = self.tp_rank * self.vocab_per_rank
        need_embed = self.is_first or (spec.tie_word_embeddings and self.is_last)
        self.embed_w = _param(self.vocab_per_rank, h, dtype=dt, device=device) if need_embed else None
        self.layers = nn.ModuleList([DeepseekDecoderLayer(spec, gid, lid, self.rope, device)
                                     for lid, gid in enumerate(self.layers_range)])
        if self.is_last:
            self.final_norm_w = _param(h, dtype=dt, device=device, fill=1.0)
            self.lm_head_w = self.embed_w if spec.tie_word_embeddings else _param(self.vocab_per_rank, h, dtype=dt,
                                                                                   device=device)
        else:
            self.final_norm_w = self.lm_head_w = None
        self.kv_latent_dim = x["kv_lora_rank"] + x["qk_rope_head_dim"]

    @property
    def num_kv_heads(self): return 1

    @property
    def head_dim(self): return self.kv_latent_dim

    def _load_attention(self, reader, pre, nm, at: MLAAttention):
        tp, tr = self.tp_size, self.tp_rank
        p = pre + "self_attn."
        if at.q_lora:
            _store_linear(at.q_a_w, at.q_a_ws, reader.get(p + "q_a_proj.weight"))
            at.q_a_norm_w.data.copy_(reader.get(p + "q_a_layernorm.weight"))
            _store_linear(at.q_b_w, at.q_b_ws, wu.shard_rows(reader.get(p + "q_b_proj.weight"), tr, tp))
        else:
            _store_linear(at.q_w, at.q_ws, wu.shard_rows(reader.get(p + "q_proj.weight"), tr, tp))
        _store_linear(at.kv_a_w, at.kv_a_ws, reader.get(p + "kv_a_proj_with_mqa.weight"))
        at.kv_a_norm_w.data.copy_(reader.get(p + "kv_a_layernorm.weight"))
        at.kv_b_w.data.copy_(wu.shard_rows(reader.get(p + "kv_b_proj.weight"), tr, tp))
        _store_linear(at.o_w, at.o_ws, wu.shard_cols(reader.get(p + "o_proj.weight"), tr, tp))


def spec_deepseek(cfg) -> ModelSpec:
    heads = cfg["num_attention_heads"]
    moe = None
    moe_layers = None
    if cfg.get("n_routed_experts"):
        is_v3_arch = "V3" in (cfg.get("architectures") or [""])[0]
        v3 = cfg.get("topk_method") == "noaux_tc" or (is_v3_arch and cfg.get("topk_method") is None)
        if is_v3_arch and cfg.get("scoring_func") is None:
            cfg["scoring_func"] = "sigmoid"  # transformers >= 5 configs drop the field; V3 is always sigmoid
        n_shared = cfg.get("n_shared_experts") or 0
        moe = MoESpec(num_experts=cfg["n_routed_experts"], top_k=cfg["num_experts_per_tok"],
                      intermediate_size=cfg["moe_intermediate_size"], norm_topk_prob=bool(cfg.get("norm_topk_prob", False)),
                      shared_intermediate_size=cfg["moe_intermediate_size"] * n_shared, shared_gate=False,
                      scoring=cfg.get("scoring_func", "softmax"), n_group=cfg.get("n_group") or 1,
                      topk_group=cfg.get("topk_group") or 1, routed_scaling=cfg.get("routed_scaling_factor", 1.0),
                      has_bias_correction=v3)
        first_dense, freq = cfg.get("first_k_dense_replace", 0), cfg.get("moe_layer_freq", 1)
        moe_layers = [i for i in range(cfg["num_hidden_layers"]) if i >= first_dense and i % freq == 0]
    rope_scaling = cfg.get("rope_scaling") or None
    rp = cfg.get("rope_parameters")
    rope_theta = cfg.get("rope_theta", 10000.0)
    if rp:
        rope_theta = rp.get("rope_theta", rope_theta)
        if rp.get("rope_type", "default") != "default":
            rope_scaling = dict(rp)
    spec = ModelSpec(
        arch="deepseek", hidden_size=cfg["hidden_size"], num_layers=cfg["num_hidden_layers"], num_heads=heads,
        num_kv_heads=heads, head_dim=cfg["kv_lora_rank"] + cfg["qk_rope_head_dim"],
        intermediate_size=cfg["intermediate_size"], vocab_size=cfg["vocab_size"],
        rms_eps=cfg.get("rms_norm_eps", 1e-6), tie_word_embeddings=bool(cfg.get("tie_word_embeddings", False)),
        max_position=cfg.get("max_position_embeddings", 4096), rope_theta=rope_theta,
        rope_scaling=dict(rope_scaling) if rope_scaling else None, moe=moe, moe_layers=moe_layers, dtype=_dtype(cfg),
        use_mla=True, eos_token_id=cfg.get("eos_token_id"))
    spec.extra = {k: cfg.get(k) for k in ("q_lora_rank", "kv_lora_rank", "qk_nope_head_dim", "qk_rope_head_dim",
                                          "v_head_dim")}
    spec.names = {"shared": "mlp.shared_experts.", "router_bias": "mlp.gate.e_score_correction_bias"}
    qc = cfg.get("quantization_config") or {}
    if qc.get("quant_method") == "fp8" and list(qc.get("weight_block_size") or []) == [128, 128]:
        # routed experts, MLA projections (q_a / q_b / kv_a / o) and dense / shared MLPs stay block-scaled e4m3 as in
        # the checkpoint; kv_b_proj is de-quantised once into the bf16 W_UK / W_UV absorption operands
        spec.quant = "fp8"
    return spec


def build_deepseek(cfg, device):
    if cfg.get("kv_lora_rank") is None:
        raise NotImplementedError("non-MLA DeepSeek checkpoints are not supported")
    return DeepseekForCausalLM(spec_deepseek(cfg), device)
