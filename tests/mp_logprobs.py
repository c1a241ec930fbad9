"""Multi-process log-prob check: run under torchrun with WORLD_SIZE = pp*tp ranks (directly for one process).
usage: mp_logprobs.py <pp> <tp> <out_json> [cpu|cuda]
Rank 0 writes, per request, [generated tokens, output_logprobs]. The vocabulary (777) is not a multiple of the shard
padding, so the last TP rank's logits shard ends with padding columns."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    pp, tp, out = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3]
    device = sys.argv[4] if len(sys.argv) > 4 else "cpu"
    from gllm_b200 import LLM
    from gllm_b200.models.presets import tiny
    cpu = device == "cpu"
    cfg = tiny("Qwen3ForCausalLM", num_hidden_layers=4, vocab_size=777,
               **({} if cpu else dict(hidden_size=256, head_dim=64, torch_dtype="bfloat16")))
    torch.manual_seed(0)
    dev_kw = dict(device="cpu", num_cpu_pages=128) if cpu else dict(num_gpu_pages=256, max_cuda_graph_bs=8)
    llm = LLM(cfg, load_format="dummy", pp_size=pp, tp_size=tp, maxp=48, maxd=16, model_max_length=256,
              log_stats=False, launch_mode="inproc", seed=0, async_schedule=os.environ.get("GLLM_TEST_ASYNC") == "1",
              **dev_kw)
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from shard_util import load_global_weights
    load_global_weights(llm.worker.runner.model, cfg, seed=123)
    prompts = [[5, 17, 99, 200, 3, 45, 7], [9] * 40, list(range(20, 120)), [300, 301]]
    # greedy and sampled rows, with and without log-probs, in one batch
    seqs = llm.generate(tokens=prompts, output_lens=[8] * 4, ignore_eos=True, temperature=[0.0, 0.8, 0.0, 0.0],
                        top_k=[1, 8, 1, 1], logprobs=[5, 3, None, 20])
    if int(os.environ.get("RANK", "0")) == 0:
        with open(out, "w") as f:
            json.dump([[s.token_ids[len(p):], s.output_logprobs] for s, p in zip(seqs, prompts)], f)
    llm.shutdown()
    if torch.distributed.is_initialized():
        torch.distributed.barrier()
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
