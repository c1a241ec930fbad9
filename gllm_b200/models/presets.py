"""Built-in HF `config.json` equivalents for the benchmark models, so `--load-format dummy` runs
need no checkpoint directory (there is no network in the build/bench environment).
Use as `model_path="preset:qwen3-8b"`. Shapes follow the public HF configs (SURVEY Appendix A).
"""
PRESETS = {
    "qwen3-8b": {
        "architectures": ["Qwen3ForCausalLM"], "hidden_size": 4096, "num_hidden_layers": 36,
        "num_attention_heads": 32, "num_key_value_heads": 8, "head_dim": 128, "intermediate_size": 12288,
        "vocab_size": 151936, "rms_norm_eps": 1e-6, "rope_theta": 1000000.0, "max_position_embeddings": 40960,
        "tie_word_embeddings": False, "attention_bias": False, "torch_dtype": "bfloat16",
        "eos_token_id": 151645, "bos_token_id": 151643,
    },
    "qwen3-0.6b": {
        "architectures": ["Qwen3ForCausalLM"], "hidden_size": 1024, "num_hidden_layers": 28,
        "num_attention_heads": 16, "num_key_value_heads": 8, "head_dim": 128, "intermediate_size": 3072,
        "vocab_size": 151936, "rms_norm_eps": 1e-6, "rope_theta": 1000000.0, "max_position_embeddings": 40960,
        "tie_word_embeddings": True, "attention_bias": False, "torch_dtype": "bfloat16", "eos_token_id": 151645,
    },
    "llama-2-7b": {
        "architectures": ["LlamaForCausalLM"], "hidden_size": 4096, "num_hidden_layers": 32,
        "num_attention_heads": 32, "num_key_value_heads": 32, "intermediate_size": 11008, "vocab_size": 32000,
        "rms_norm_eps": 1e-5, "rope_theta": 10000.0, "max_position_embeddings": 4096,
        "tie_word_embeddings": False, "torch_dtype": "bfloat16", "eos_token_id": 2, "bos_token_id": 1,
    },
    "llama-3-70b": {
        "architectures": ["LlamaForCausalLM"], "hidden_size": 8192, "num_hidden_layers": 80,
        "num_attention_heads": 64, "num_key_value_heads": 8, "intermediate_size": 28672, "vocab_size": 128256,
        "rms_norm_eps": 1e-5, "rope_theta": 500000.0, "max_position_embeddings": 8192,
        "tie_word_embeddings": False, "torch_dtype": "bfloat16", "eos_token_id": 128001, "bos_token_id": 128000,
    },
    "mixtral-8x7b": {
        "architectures": ["MixtralForCausalLM"], "hidden_size": 4096, "num_hidden_layers": 32,
        "num_attention_heads": 32, "num_key_value_heads": 8, "intermediate_size": 14336, "vocab_size": 32000,
        "rms_norm_eps": 1e-5, "rope_theta": 1000000.0, "max_position_embeddings": 32768,
        "num_local_experts": 8, "num_experts_per_tok": 2, "tie_word_embeddings": False,
        "torch_dtype": "bfloat16", "eos_token_id": 2, "bos_token_id": 1,
    },
    "qwen3-30b-a3b": {
        "architectures": ["Qwen3MoeForCausalLM"], "hidden_size": 2048, "num_hidden_layers": 48,
        "num_attention_heads": 32, "num_key_value_heads": 4, "head_dim": 128, "intermediate_size": 6144,
        "moe_intermediate_size": 768, "num_experts": 128, "num_experts_per_tok": 8, "norm_topk_prob": True,
        "decoder_sparse_step": 1, "mlp_only_layers": [], "vocab_size": 151936, "rms_norm_eps": 1e-6,
        "rope_theta": 1000000.0, "max_position_embeddings": 40960, "tie_word_embeddings": False,
        "torch_dtype": "bfloat16", "eos_token_id": 151645,
    },
    "deepseek-v3": {
        "architectures": ["DeepseekV3ForCausalLM"], "hidden_size": 7168, "num_hidden_layers": 61,
        "num_attention_heads": 128, "num_key_value_heads": 128, "intermediate_size": 18432,
        "moe_intermediate_size": 2048, "n_routed_experts": 256, "n_shared_experts": 1, "num_experts_per_tok": 8,
        "n_group": 8, "topk_group": 4, "topk_method": "noaux_tc", "scoring_func": "sigmoid",
        "norm_topk_prob": True, "routed_scaling_factor": 2.5, "first_k_dense_replace": 3, "moe_layer_freq": 1,
        "q_lora_rank": 1536, "kv_lora_rank": 512, "qk_nope_head_dim": 128, "qk_rope_head_dim": 64,
        "v_head_dim": 128, "vocab_size": 129280, "rms_norm_eps": 1e-6, "rope_theta": 10000.0,
        "max_position_embeddings": 163840,
        "rope_scaling": {"type": "yarn", "factor": 40, "original_max_position_embeddings": 4096,
                         "beta_fast": 32, "beta_slow": 1, "mscale": 1.0, "mscale_all_dim": 1.0},
        "tie_word_embeddings": False, "torch_dtype": "bfloat16", "eos_token_id": 1, "bos_token_id": 0,
        "quantization_config": {"quant_method": "fp8", "activation_scheme": "dynamic", "fmt": "e4m3",
                                "weight_block_size": [128, 128]},
    },
}
# 4-bit AWQ builds of the public shapes (group 128, fp16 scales); with dummy weights they need no files
_AWQ = {"quant_method": "awq", "bits": 4, "group_size": 128, "zero_point": True, "version": "gemm"}
PRESETS["qwen3-8b-awq"] = dict(PRESETS["qwen3-8b"], torch_dtype="float16", quantization_config=dict(_AWQ))
PRESETS["llama-3-70b-awq"] = dict(PRESETS["llama-3-70b"], torch_dtype="float16", quantization_config=dict(_AWQ))


def tiny(arch: str = "Qwen3ForCausalLM", **over):
    """A very small random-init config of the given family for tests."""
    cfg = {
        "architectures": [arch], "hidden_size": 128, "num_hidden_layers": 2, "num_attention_heads": 4,
        "num_key_value_heads": 2, "head_dim": 32, "intermediate_size": 256, "vocab_size": 512,
        "rms_norm_eps": 1e-6, "rope_theta": 10000.0, "max_position_embeddings": 512,
        "tie_word_embeddings": False, "torch_dtype": "float32", "eos_token_id": 1,
    }
    cfg.update(over)
    return cfg
