"""Sampler streams of the tiny CPU model: run under torchrun with WORLD_SIZE = tp ranks (directly for one process).

usage: mp_sampler_streams.py <tp> <out_json>
Rank 0 writes, per returned sequence, [generated tokens, output_logprobs] for a greedy batch with log-probs and then
a mixed batch: unseeded temperature / top-k / top-p rows, a repetition penalty, frequency / presence penalties with
logit_bias, seeded rows, log-probs and n = 3. Unseeded rows draw from the engine's seeded CPU generator, so the file
pins the CPU random streams exactly (`tests/golden/sampler_cpu_streams.json`)."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PROMPTS = [[5, 17, 99, 200, 3, 45, 7], [9] * 40, list(range(20, 120)), [300, 301], [1, 2, 3, 4, 5, 6],
           [600, 7, 600, 7, 600], [42] * 9, [11, 12, 13]]
MIXED = [
    dict(temperature=0.9, top_k=0, top_p=1.0),                                                     # full vocabulary
    dict(temperature=0.8, top_k=20, top_p=0.9),                                                    # top-k + top-p
    dict(temperature=0.7, top_k=50, top_p=1.0, repetition_penalty=1.3),
    dict(temperature=0.8, top_k=0, top_p=1.0, frequency_penalty=0.5, presence_penalty=0.3,
         logit_bias={7: 3.0, 11: -100.0}),
    dict(temperature=0.8, top_k=20, top_p=1.0, seed=1234),
    dict(temperature=1.0, top_k=0, top_p=0.95, seed=77, frequency_penalty=0.2),
    dict(temperature=0.0, top_k=1, top_p=1.0, logprobs=5),
    dict(temperature=0.8, top_k=8, top_p=1.0, logprobs=3, n=3),
]


def main():
    tp, out = int(sys.argv[1]), sys.argv[2]
    import torch
    from gllm_b200 import LLM
    from gllm_b200.models.presets import tiny
    cfg = tiny("Qwen3ForCausalLM", num_hidden_layers=4, vocab_size=777)
    torch.manual_seed(0)
    llm = LLM(cfg, load_format="dummy", tp_size=tp, maxp=48, maxd=16, model_max_length=256, log_stats=False,
              launch_mode="inproc", seed=0, async_schedule=os.environ.get("GLLM_TEST_ASYNC") == "1", device="cpu",
              num_cpu_pages=256)
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from shard_util import load_global_weights
    load_global_weights(llm.worker.runner.model, cfg, seed=123)
    greedy = llm.generate(tokens=PROMPTS[:3], output_lens=[6] * 3, ignore_eos=True, temperature=0.0, top_k=1,
                          logprobs=[2, None, 4])
    keys = ("temperature", "top_k", "top_p", "repetition_penalty", "frequency_penalty", "presence_penalty",
            "logit_bias", "seed", "logprobs", "n")
    kw = {k: [p.get(k) for p in MIXED] for k in keys}
    kw["repetition_penalty"] = [p.get("repetition_penalty", 1.0) for p in MIXED]
    mixed = llm.generate(tokens=PROMPTS, output_lens=[8] * len(PROMPTS), ignore_eos=True, **kw)
    if int(os.environ.get("RANK", "0")) == 0:
        with open(out, "w") as f:
            json.dump([[s.token_ids[s.prompt_len:], s.output_logprobs] for s in greedy + mixed], f)
    llm.shutdown()
    if torch.distributed.is_initialized():
        torch.distributed.barrier()
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
