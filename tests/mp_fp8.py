"""Multi-process W8A8 check: run under torchrun with WORLD_SIZE = pp*tp ranks (directly for one process).
usage: mp_fp8.py <pp> <tp> <out> <model dir> <device: cpu | cuda>
Every rank saves (its tokens, its [(sequence ids, logits)]) to <out>.<rank> with torch.save: the first rank returns
the tokens, the ranks of the last stage hold the logits."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PROMPTS = [[5, 17, 99, 200, 3, 45, 7], [9] * 40, list(range(20, 120)), [300, 301], [8] * 30]


def main():
    pp, tp, out, d, device = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3], sys.argv[4], sys.argv[5]
    os.environ["GLLM_KEEP_LOGITS"] = "1"
    from gllm_b200 import LLM
    kw = dict(num_cpu_pages=128) if device == "cpu" else dict(num_gpu_pages=256, max_cuda_graph_bs=8)
    llm = LLM(d, device=device, pp_size=pp, tp_size=tp, maxp=24, maxd=16, model_max_length=256, log_stats=False,
              launch_mode="inproc", seed=0, tp_mode="nccl", **kw)
    seqs = llm.generate(tokens=PROMPTS, output_lens=[6] * len(PROMPTS), ignore_eos=True)
    log = [(i, lg.float().cpu().clone()) for i, lg in llm.worker.runner.logit_log]
    torch.save(([s.token_ids for s in seqs], log), f"{out}.{os.environ.get('RANK', '0')}")
    llm.shutdown()
    if torch.distributed.is_initialized():
        torch.distributed.barrier()
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
