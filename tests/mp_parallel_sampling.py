"""Parallel sampling in a multi-process engine (TP / PP over gloo on the CPU, NCCL on GPUs).

usage: mp_parallel_sampling.py <pp> <tp> <out_json> [cpu|cuda]
Runs greedy requests once with n = 1 and once with n = 3 (page size 4: prompts ending on, just after and just
before a page boundary) and makes rank 0 write the generated tokens and the number of KV pages copied, so the test
can check that every choice equals the n = 1 continuation on every rank layout.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PROMPTS = [[5, 17, 99, 200, 3, 45, 7, 8], [9] * 13, list(range(20, 31)), list(range(40, 90))]


def main():
    pp, tp, out = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3]
    device = sys.argv[4] if len(sys.argv) > 4 else "cpu"
    import torch
    from gllm_b200 import LLM
    from gllm_b200.models.presets import tiny
    cpu = device == "cpu"
    cfg = tiny("Qwen3ForCausalLM", num_hidden_layers=4, vocab_size=777,
               **({} if cpu else dict(hidden_size=256, head_dim=64, torch_dtype="bfloat16")))
    torch.manual_seed(0)
    dev_kw = dict(device="cpu", num_cpu_pages=256) if cpu else dict(num_gpu_pages=512, max_cuda_graph_bs=16)
    llm = LLM(cfg, load_format="dummy", pp_size=pp, tp_size=tp, maxp=32, maxd=16, page_size=4 if cpu else 16,
              model_max_length=256, log_stats=False, launch_mode="inproc", seed=0,
              async_schedule=os.environ.get("GLLM_TEST_ASYNC") == "1", **dev_kw)
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from shard_util import load_global_weights
    load_global_weights(llm.worker.runner.model, cfg, seed=123)
    kw = dict(output_lens=[8] * len(PROMPTS), ignore_eos=True, top_k=1)
    single = llm.generate(tokens=PROMPTS, **kw)
    many = llm.generate(tokens=PROMPTS, n=3, **kw)
    if int(os.environ.get("RANK", "0")) == 0:
        with open(out, "w") as f:
            json.dump({"single": [s.token_ids[s.prompt_len:] for s in single],
                       "many": [s.token_ids[s.prompt_len:] for s in many],
                       "copied": llm.worker.runner.stats.get("kv_copy_pages", 0)}, f)
    llm.shutdown()
    if torch.distributed.is_initialized():
        torch.distributed.barrier()
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
