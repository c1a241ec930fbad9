"""End-to-end on the GPU: the engine (sm_100a kernels, CUDA graphs) must reproduce the CPU oracle
path's greedy tokens on a small random model."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _cfg():
    from gllm_b200.models.presets import tiny
    return tiny("Qwen3ForCausalLM", hidden_size=256, num_hidden_layers=3, num_attention_heads=4,
                num_key_value_heads=2, head_dim=64, intermediate_size=512, vocab_size=1024, torch_dtype="bfloat16")


def _gen(device, graphs, prompts, out_len, state=None):
    from gllm_b200 import LLM
    llm = LLM(_cfg(), load_format="dummy", maxp=128, maxd=64, max_cuda_graph_bs=8, num_gpu_pages=256,
              num_cpu_pages=256, model_max_length=512, log_stats=False, device=device,
              disable_cuda_graph=not graphs)
    model = llm.worker.runner.model
    if state is not None:
        for (n, p), (_, q) in zip(model.named_parameters(), state):
            p.data.copy_(q.to(p.device))
    outs = llm.generate(tokens=prompts, output_lens=[out_len] * len(prompts), ignore_eos=True)
    toks = [s.token_ids[len(p):] for s, p in zip(outs, prompts)]
    params = [(n, p.detach().cpu().clone()) for n, p in model.named_parameters()]
    logits_stats = llm.worker.runner.stats.copy()
    llm.shutdown()
    return toks, params, logits_stats


def test_gpu_matches_cpu_oracle():
    torch.manual_seed(0)
    prompts = [[5, 9, 100, 7], list(range(20, 190)), [77] * 33, [3, 1, 4, 1, 5, 9, 2, 6]]
    cpu_toks, params, _ = _gen("cpu", False, prompts, 6)
    gpu_toks, _, st = _gen("cuda", True, prompts, 6, state=params)
    assert st["graph_steps"] > 0, "CUDA graphs were not used for decode"
    # bf16 kernels vs fp32-accumulated oracle: allow rare argmax flips after the first tokens
    agree = sum(a == b for x, y in zip(cpu_toks, gpu_toks) for a, b in zip(x, y))
    total = sum(len(x) for x in cpu_toks)
    assert [x[0] for x in cpu_toks] == [y[0] for y in gpu_toks], (cpu_toks, gpu_toks)
    # once a near-tie flips, the rest of that sequence differs: require most sequences to match fully
    same_seqs = sum(x == y for x, y in zip(cpu_toks, gpu_toks))
    assert same_seqs >= len(prompts) // 2 and agree / total >= 0.6, (cpu_toks, gpu_toks)


def test_graph_and_eager_agree():
    prompts = [[5, 9, 100, 7], list(range(20, 150)), [77] * 33]
    t1, params, _ = _gen("cuda", False, prompts, 8)
    t2, _, st = _gen("cuda", True, prompts, 8, state=params)
    assert st["graph_steps"] > 0
    assert t1 == t2


def test_qwen3_vl_gpu_matches_cpu_engine():
    """Qwen3-VL (vision tower, interleaved M-RoPE kernel path, DeepStack) on the GPU vs the fp32 CPU engine."""
    import numpy as np
    from gllm_b200 import LLM
    img, vstart = 290, 292
    cfg = {"architectures": ["Qwen3VLForConditionalGeneration"], "image_token_id": img, "video_token_id": 291,
           "vision_start_token_id": vstart, "tie_word_embeddings": False,
           "text_config": dict(hidden_size=256, num_hidden_layers=4, num_attention_heads=4, num_key_value_heads=2,
                               head_dim=64, intermediate_size=512, vocab_size=512, max_position_embeddings=512,
                               rms_norm_eps=1e-6, eos_token_id=1,
                               rope_parameters={"rope_type": "default", "mrope_section": [12, 10, 10],
                                                "mrope_interleaved": True, "rope_theta": 10000.0}),
           "vision_config": dict(depth=3, hidden_size=64, num_heads=2, intermediate_size=128, out_hidden_size=256,
                                 patch_size=16, spatial_merge_size=2, temporal_patch_size=2,
                                 num_position_embeddings=16, deepstack_visual_indexes=[0, 1], in_channels=3)}
    grids = [(1, 4, 6)]
    g = torch.Generator().manual_seed(0)
    pix = torch.randn(24, 3 * 2 * 16 * 16, generator=g).numpy()
    ids = [5, 17, 99, vstart] + [img] * 6 + [7, 8, 45, 46]
    mm = {"pixel_values": pix, "image_grid_thw": np.asarray(grids)}
    outs, params = {}, None
    cfg["torch_dtype"] = "bfloat16"
    for dev in ("cpu", "cuda"):
        torch.manual_seed(11)
        llm = LLM(cfg, load_format="dummy", device=dev, maxp=64, maxd=16, model_max_length=256, log_stats=False,
                  num_cpu_pages=64, num_gpu_pages=64, max_cuda_graph_bs=4)
        model = llm.worker.runner.model
        if params is None:
            params = [(n, p.detach().cpu().clone()) for n, p in model.named_parameters()]
        else:
            for (n, p), (_, q) in zip(model.named_parameters(), params):
                p.data.copy_(q.to(p.device))
        o = llm.generate(tokens=[ids, ids[:3]], output_lens=[6, 6], ignore_eos=True, mm_contents=[mm, None])
        outs[dev] = [s.token_ids[-6:] for s in o]
        llm.shutdown()
    # bf16 kernels vs the PyTorch oracle path on a random model: the first generated tokens must agree
    assert [x[0] for x in outs["cpu"]] == [x[0] for x in outs["cuda"]], outs


def test_deepseek_mla_gpu_matches_cpu_engine():
    """DeepSeek-V3 style model (MLA latent cache 512+64, grouped top-k MoE with a shared expert): the sm_100a
    absorbed-MLA kernel path with CUDA graphs vs the PyTorch expanded-form oracle on the CPU."""
    from gllm_b200 import LLM
    cfg = {"architectures": ["DeepseekV3ForCausalLM"], "hidden_size": 256, "intermediate_size": 512,
           "moe_intermediate_size": 128, "num_hidden_layers": 3, "num_attention_heads": 8, "num_key_value_heads": 8,
           "n_routed_experts": 8, "n_shared_experts": 1, "num_experts_per_tok": 2, "n_group": 2, "topk_group": 1,
           "first_k_dense_replace": 1, "routed_scaling_factor": 2.5, "norm_topk_prob": True, "q_lora_rank": 128,
           "kv_lora_rank": 512, "qk_nope_head_dim": 128, "qk_rope_head_dim": 64, "v_head_dim": 128,
           "vocab_size": 1024, "max_position_embeddings": 512, "eos_token_id": 1, "rms_norm_eps": 1e-6,
           "rope_theta": 10000.0, "torch_dtype": "bfloat16", "scoring_func": "sigmoid", "topk_method": "noaux_tc"}
    prompts = [[5, 9, 100, 7], list(range(20, 150)), [77] * 33]
    outs, params, stats = {}, None, None
    for dev in ("cpu", "cuda"):
        torch.manual_seed(21)
        llm = LLM(cfg, load_format="dummy", device=dev, maxp=64, maxd=16, model_max_length=256, log_stats=False,
                  num_cpu_pages=64, num_gpu_pages=64, max_cuda_graph_bs=4)
        model = llm.worker.runner.model
        if params is None:
            params = [(n, p.detach().cpu().clone()) for n, p in model.named_parameters()]
        else:
            for (n, p), (_, q) in zip(model.named_parameters(), params):
                p.data.copy_(q.to(p.device))
            model.process_weights()
        o = llm.generate(tokens=prompts, output_lens=[6] * len(prompts), ignore_eos=True)
        outs[dev] = [s.token_ids[-6:] for s in o]
        stats = dict(llm.worker.runner.stats)
        llm.shutdown()
    assert stats["graph_steps"] > 0, "MLA decode did not run inside CUDA graphs"
    assert [x[0] for x in outs["cpu"]] == [x[0] for x in outs["cuda"]], outs
    # decode steps (CUDA graphs on the GPU) must agree too on most sequences (bf16 near-ties may flip late tokens)
    assert sum(a == b for a, b in zip(outs["cpu"], outs["cuda"])) >= 2, outs


def _family_cfgs():
    from gllm_b200.models.presets import tiny
    base = dict(hidden_size=256, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2, head_dim=64,
                intermediate_size=512, vocab_size=1024, torch_dtype="bfloat16")
    return {
        "llama": tiny("LlamaForCausalLM", **base),
        "qwen2-bias-tied": tiny("Qwen2ForCausalLM", **{**base, "tie_word_embeddings": True}),
        "mixtral": tiny("MixtralForCausalLM", **{**base, "intermediate_size": 256, "num_local_experts": 4,
                                                  "num_experts_per_tok": 2}),
        "qwen3-moe": tiny("Qwen3MoeForCausalLM", **{**base, "moe_intermediate_size": 128, "num_experts": 8,
                                                    "num_experts_per_tok": 2, "decoder_sparse_step": 1,
                                                    "mlp_only_layers": [], "norm_topk_prob": True}),
        "qwen2-moe-shared": tiny("Qwen2MoeForCausalLM", **{**base, "moe_intermediate_size": 128, "num_experts": 4,
                                                           "num_experts_per_tok": 2, "decoder_sparse_step": 1,
                                                           "mlp_only_layers": [],
                                                           "shared_expert_intermediate_size": 256}),
        "chatglm": {"architectures": ["ChatGLMModel"], "hidden_size": 256, "num_layers": 2, "num_attention_heads": 4,
                    "multi_query_attention": True, "multi_query_group_num": 2, "kv_channels": 64,
                    "ffn_hidden_size": 512, "padded_vocab_size": 1024, "layernorm_epsilon": 1e-5,
                    "add_qkv_bias": True, "seq_length": 512, "torch_dtype": "bfloat16", "eos_token_id": 1},
    }


@pytest.mark.parametrize("family", ["llama", "qwen2-bias-tied", "mixtral", "qwen3-moe", "qwen2-moe-shared", "chatglm"])
def test_model_families_gpu_match_cpu_engine_on_verbatim_weights(family):
    """Every decoder family through the GPU engine (native kernels + CUDA graphs) vs the CPU oracle engine with
    the same weights, copied verbatim: both engines store the same weight layout."""
    from gllm_b200 import LLM
    cfg = _family_cfgs()[family]
    prompts = [[5, 9, 100, 7], list(range(20, 120)), [77] * 33]
    outs, params = {}, None
    for dev in ("cpu", "cuda"):
        torch.manual_seed(31)
        llm = LLM(cfg, load_format="dummy", device=dev, maxp=64, maxd=16, model_max_length=256, log_stats=False,
                  num_cpu_pages=64, num_gpu_pages=64, max_cuda_graph_bs=4)
        model = llm.worker.runner.model
        if params is None:
            params = [(n, p.detach().cpu().clone()) for n, p in model.named_parameters()]
        else:
            for (n, p), (_, q) in zip(model.named_parameters(), params):
                p.data.copy_(q.to(p.device))
            model.process_weights()
        o = llm.generate(tokens=prompts, output_lens=[5] * len(prompts), ignore_eos=True)
        outs[dev] = [s.token_ids[-5:] for s in o]
        if dev == "cuda":
            assert llm.worker.runner.stats["graph_steps"] > 0
        llm.shutdown()
    assert [x[0] for x in outs["cpu"]] == [x[0] for x in outs["cuda"]], outs
    assert sum(a == b for a, b in zip(outs["cpu"], outs["cuda"])) >= 2, outs
