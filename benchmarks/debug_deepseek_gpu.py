"""Layer-by-layer CPU vs GPU comparison of a tiny DeepSeek model (debug aid)."""
import os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gllm_b200 import LLM
from gllm_b200.models import deepseek_v2 as ds

cfg = {"architectures": ["DeepseekV3ForCausalLM"], "hidden_size": 256, "intermediate_size": 512,
       "moe_intermediate_size": 128, "num_hidden_layers": 3, "num_attention_heads": 8, "num_key_value_heads": 8,
       "n_routed_experts": 8, "n_shared_experts": 1, "num_experts_per_tok": 2, "n_group": 2, "topk_group": 1,
       "first_k_dense_replace": 1, "routed_scaling_factor": 2.5, "norm_topk_prob": True, "q_lora_rank": 128,
       "kv_lora_rank": 512, "qk_nope_head_dim": 128, "qk_rope_head_dim": 64, "v_head_dim": 128,
       "vocab_size": 1024, "max_position_embeddings": 512, "eos_token_id": 1, "rms_norm_eps": 1e-6,
       "rope_theta": 10000.0, "torch_dtype": "bfloat16", "scoring_func": "sigmoid", "topk_method": "noaux_tc"}
rec = {}
orig_attn = ds.MLAAttention.forward
orig_layer = ds.DeepseekDecoderLayer.forward
def attn_fwd(self, inp, h, kv_cache, tpc):
    out = orig_attn(self, inp, h, kv_cache, tpc)
    if kv_cache is not None and not (out.is_cuda and torch.cuda.is_current_stream_capturing()):
        rec.setdefault(CUR[0], []).append((f"L{self.layer_id}.attn", out.detach().float().cpu()))
    return out
def layer_fwd(self, inp, h, residual, kv_cache, tpc, next_norm_w):
    o = orig_layer(self, inp, h, residual, kv_cache, tpc, next_norm_w)
    if kv_cache is not None and not (o[0].is_cuda and torch.cuda.is_current_stream_capturing()):
        rec.setdefault(CUR[0], []).append((f"L{self.layer_id}.out_h", o[0].detach().float().cpu()))
    return o
ds.MLAAttention.forward = attn_fwd
ds.DeepseekDecoderLayer.forward = layer_fwd
CUR = ["cpu"]
VARIANTS = {
    "multi_seq_short": dict(prompts=[[5, 9, 100, 7], [77] * 33, list(range(20, 50))], graphs=False),
    "one_long_chunked": dict(prompts=[list(range(20, 150))], graphs=False),
    "one_short_graphs": dict(prompts=[[5, 9, 100, 7]], graphs=True),
}
for vname, v in VARIANTS.items():
    params = None
    res = {}
    for dev in ("cpu", "cuda"):
        CUR[0] = dev
        torch.manual_seed(21)
        llm = LLM(cfg, load_format="dummy", device=dev, maxp=64, maxd=16, model_max_length=256, log_stats=False,
                  num_cpu_pages=64, num_gpu_pages=64, disable_cuda_graph=not v["graphs"], max_cuda_graph_bs=4)
        model = llm.worker.runner.model
        if params is None:
            params = [(n, p.detach().cpu().clone()) for n, p in model.named_parameters()]
        else:
            for (n, p), (n2, q) in zip(model.named_parameters(), params):
                p.data.copy_(q.to(p.device))
            model.process_weights()
        rec[dev] = []
        o = llm.generate(tokens=v["prompts"], output_lens=[4] * len(v["prompts"]), ignore_eos=True)
        res[dev] = [s_.token_ids[-4:] for s_ in o]
        llm.shutdown()
    print(vname, "cpu", res["cpu"], "cuda", res["cuda"], flush=True)
    for (n1, a), (n2, b) in list(zip(rec["cpu"], rec["cuda"]))[:6]:
        if a.shape == b.shape:
            print(f"   {n1:14s} rel err {((a - b).norm() / (a.norm() + 1e-9)).item():.4f}")
