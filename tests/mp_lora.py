"""Multi-process multi-LoRA check: run under torchrun with WORLD_SIZE = pp*tp ranks (directly for one process).
usage: mp_lora.py <pp> <tp> <out_json> <model dir with adapters a/ and b/>
Rank 0 writes the token ids of a batch mixing adapter a, adapter b and base requests (chunked: maxp = 24)."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    pp, tp, out, d = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3], sys.argv[4]
    from gllm_b200 import LLM
    llm = LLM(d, device="cpu", num_cpu_pages=128, pp_size=pp, tp_size=tp, maxp=24, maxd=16, model_max_length=256,
              log_stats=False, launch_mode="inproc", seed=0, tp_mode="nccl",
              lora_modules={"a": os.path.join(d, "a"), "b": os.path.join(d, "b")}, max_lora_rank=16)
    prompts = [[5, 17, 99, 200, 3, 45, 7], [9] * 40, list(range(20, 120)), [300, 301], [8] * 30]
    seqs = llm.generate(tokens=prompts, output_lens=[6] * 5, ignore_eos=True, lora=["a", "b", None, "b", "a"])
    if int(os.environ.get("RANK", "0")) == 0:
        with open(out, "w") as f:
            json.dump([s.token_ids for s in seqs], f)
    llm.shutdown()
    if torch.distributed.is_initialized():
        torch.distributed.barrier()
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
