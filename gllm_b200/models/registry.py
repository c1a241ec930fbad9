"""HF architecture name -> ModelSpec / model builder (reference table: gllm/model_loader.py:117-146).

Supported `architectures[0]` values:
  LlamaForCausalLM, Qwen2ForCausalLM, Qwen3ForCausalLM, Qwen2MoeForCausalLM, Qwen3MoeForCausalLM,
  MixtralForCausalLM, ChatGLMModel / ChatGLMForConditionalGeneration, DeepseekV2ForCausalLM,
  DeepseekV3ForCausalLM, Qwen2_5_VLForConditionalGeneration, Qwen3VLForConditionalGeneration,
  Qwen3VLMoeForConditionalGeneration.
"""
from __future__ import annotations

from typing import Callable, Dict

import torch

from gllm_b200.models import weight_utils as wu
from gllm_b200.models.decoder import CausalLM, ModelSpec, MoESpec

_DTYPES = {"bfloat16": torch.bfloat16, "float16": torch.float16, "float32": torch.float32,
           torch.bfloat16: torch.bfloat16, torch.float16: torch.float16, torch.float32: torch.float32}


class HFConfig(dict):
    """config.json as an attribute dict (nested dicts become HFConfig too)."""

    def __getattr__(self, k):
        try:
            v = self[k]
        except KeyError as e:
            raise AttributeError(k) from e
        return HFConfig(v) if isinstance(v, dict) and not isinstance(v, HFConfig) else v

    def __setattr__(self, k, v):
        self[k] = v


def _dtype(cfg) -> torch.dtype:
    d = cfg.get("torch_dtype", cfg.get("dtype", "bfloat16"))
    return _DTYPES.get(d, torch.bfloat16)


def _base_spec(cfg: HFConfig, arch: str, **kw) -> ModelSpec:
    heads = cfg["num_attention_heads"]
    hidden = cfg["hidden_size"]
    rope_scaling = cfg.get("rope_scaling") or None
    rope_theta = cfg.get("rope_theta", 10000.0)
    rp = cfg.get("rope_parameters")
    if rp:  # transformers >= 5 style
        rope_theta = rp.get("rope_theta", rope_theta)
        if rp.get("rope_type", "default") != "default" or "mrope_section" in rp:
            rope_scaling = dict(rp)
    spec = ModelSpec(
        arch=arch, hidden_size=hidden, num_layers=cfg["num_hidden_layers"], num_heads=heads,
        num_kv_heads=cfg.get("num_key_value_heads", heads) or heads,
        head_dim=cfg.get("head_dim") or hidden // heads,
        intermediate_size=cfg.get("intermediate_size", 0), vocab_size=cfg["vocab_size"],
        rms_eps=cfg.get("rms_norm_eps", 1e-6), tie_word_embeddings=bool(cfg.get("tie_word_embeddings", False)),
        max_position=cfg.get("max_position_embeddings", 8192), rope_theta=rope_theta,
        rope_scaling=dict(rope_scaling) if rope_scaling else None, dtype=_dtype(cfg),
        eos_token_id=cfg.get("eos_token_id"))
    qc = cfg.get("quantization_config") or {}
    if qc.get("quant_method") == "fp8" and list(qc.get("weight_block_size") or []) == [128, 128]:
        spec.quant = "fp8"
    spec.w4 = wu.w4_config(qc)
    if spec.w4 is not None:
        spec.quant = spec.w4.method
        if spec.dtype == torch.float16:    # every kernel here is bf16: fp16 tensors are rounded to bf16 once, at load
            spec.dtype = torch.bfloat16
    for k, v in kw.items():
        setattr(spec, k, v)
    return spec


def spec_llama(cfg):
    return _base_spec(cfg, "llama", qkv_bias=bool(cfg.get("attention_bias", False)),
                      o_bias=bool(cfg.get("attention_bias", False)))


def spec_qwen2(cfg):
    return _base_spec(cfg, "qwen2", qkv_bias=True)


def spec_qwen3(cfg):
    return _base_spec(cfg, "qwen3", qkv_bias=bool(cfg.get("attention_bias", False)), qk_norm=True)


def _moe_layers(cfg, n_layers):
    only = set(cfg.get("mlp_only_layers", []) or [])
    step = cfg.get("decoder_sparse_step", 1) or 1
    return [i for i in range(n_layers) if i not in only and (i + 1) % step == 0]


def spec_qwen2_moe(cfg):
    spec = spec_qwen2(cfg)
    spec.arch = "qwen2_moe"
    spec.moe = MoESpec(num_experts=cfg.get("num_experts") or cfg["num_local_experts"],
                       top_k=cfg["num_experts_per_tok"],
                       intermediate_size=cfg["moe_intermediate_size"],
                       norm_topk_prob=bool(cfg.get("norm_topk_prob", False)),
                       shared_intermediate_size=cfg.get("shared_expert_intermediate_size", 0) or 0,
                       shared_gate=True)
    spec.moe_layers = _moe_layers(cfg, spec.num_layers)
    return spec


def spec_qwen3_moe(cfg):
    spec = spec_qwen3(cfg)
    spec.arch = "qwen3_moe"
    spec.moe = MoESpec(num_experts=cfg.get("num_experts") or cfg["num_local_experts"],
                       top_k=cfg["num_experts_per_tok"],
                       intermediate_size=cfg["moe_intermediate_size"],
                       norm_topk_prob=bool(cfg.get("norm_topk_prob", True)))
    spec.moe_layers = _moe_layers(cfg, spec.num_layers)
    return spec


def spec_mixtral(cfg):
    spec = _base_spec(cfg, "mixtral")
    spec.moe = MoESpec(num_experts=cfg["num_local_experts"], top_k=cfg["num_experts_per_tok"],
                       intermediate_size=cfg["intermediate_size"], norm_topk_prob=True)
    spec.names = {"router": "block_sparse_moe.gate.weight", "expert": "block_sparse_moe.experts.{e}.",
                  "e_gate": "w1.weight", "e_up": "w3.weight", "e_down": "w2.weight"}
    return spec


def spec_chatglm(cfg):
    heads = cfg["num_attention_heads"]
    hidden = cfg["hidden_size"]
    head_dim = cfg.get("kv_channels", hidden // heads)
    mq = cfg.get("multi_query_attention", False)
    spec = ModelSpec(
        arch="chatglm", hidden_size=hidden, num_layers=cfg["num_layers"], num_heads=heads,
        num_kv_heads=cfg.get("multi_query_group_num", heads) if mq else heads, head_dim=head_dim,
        intermediate_size=cfg["ffn_hidden_size"], vocab_size=cfg.get("padded_vocab_size", cfg.get("vocab_size")),
        rms_eps=cfg.get("layernorm_epsilon", 1e-5), qkv_bias=bool(cfg.get("add_qkv_bias", False)),
        max_position=cfg.get("seq_length", 8192), rope_theta=10000.0 * cfg.get("rope_ratio", 1.0),
        rot_dim=head_dim // 2, rope_neox=False, dtype=_dtype(cfg), eos_token_id=cfg.get("eos_token_id"))
    spec.names = {
        "embed": "transformer.embedding.word_embeddings.weight",
        "final_norm": "transformer.encoder.final_layernorm.weight",
        "lm_head": "transformer.output_layer.weight",
        "layer": "transformer.encoder.layers.{i}.",
        "qkv_fused": "self_attention.query_key_value", "o": "self_attention.dense",
        "gate_up_fused": "mlp.dense_h_to_4h", "down": "mlp.dense_4h_to_h",
    }
    return spec


def _build_decoder(spec_fn):
    def build(cfg, device):
        from gllm_b200.layers.moe import make_moe_block
        return CausalLM(spec_fn(cfg), device, moe_factory=make_moe_block)
    return build


def _build_deepseek(cfg, device):
    from gllm_b200.models.deepseek_v2 import build_deepseek
    return build_deepseek(cfg, device)


def _build_qwen2_5_vl(cfg, device):
    from gllm_b200.models.qwen2_5_vl import build_qwen2_5_vl
    return build_qwen2_5_vl(cfg, device)


def _build_qwen3_vl(cfg, device):
    from gllm_b200.models.qwen3_vl import build_qwen3_vl
    return build_qwen3_vl(cfg, device)


ARCHITECTURES: Dict[str, Callable] = {
    "LlamaForCausalLM": _build_decoder(spec_llama),
    "MistralForCausalLM": _build_decoder(spec_llama),
    "Qwen2ForCausalLM": _build_decoder(spec_qwen2),
    "Qwen3ForCausalLM": _build_decoder(spec_qwen3),
    "Qwen2MoeForCausalLM": _build_decoder(spec_qwen2_moe),
    "Qwen3MoeForCausalLM": _build_decoder(spec_qwen3_moe),
    "MixtralForCausalLM": _build_decoder(spec_mixtral),
    "ChatGLMModel": _build_decoder(spec_chatglm),
    "ChatGLMForConditionalGeneration": _build_decoder(spec_chatglm),
    "DeepseekV2ForCausalLM": _build_deepseek,
    "DeepseekV3ForCausalLM": _build_deepseek,
    "Qwen2_5_VLForConditionalGeneration": _build_qwen2_5_vl,
    "Qwen3VLForConditionalGeneration": _build_qwen3_vl,
    "Qwen3VLMoeForConditionalGeneration": _build_qwen3_vl,
}


def build_model(cfg: HFConfig, device):
    arch = cfg["architectures"][0]
    if arch not in ARCHITECTURES:
        raise ValueError(f"unsupported architecture {arch}; supported: {sorted(ARCHITECTURES)}")
    if wu.w4_config(cfg.get("quantization_config") or {}) is not None and arch not in wu.W4_ARCHITECTURES:
        raise ValueError(f"4-bit AWQ / GPTQ weights are not supported for {arch} (supported: "
                         f"{', '.join(wu.W4_ARCHITECTURES)})")
    return ARCHITECTURES[arch](cfg, device)
