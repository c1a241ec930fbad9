"""Cost of the per-request sampling parameters on the GPU (csrc/sample/sampler.cu: the bias row read by the sampler,
the seeded race, bias_account_kernel).

    python benchmarks/sampling_params_bench.py [--skip-kernels] [--skip-e2e] [--num-prompts 500] [--rounds 2]

1. Kernel time with CUDA events at V = 151936 bf16 logits (Qwen3's vocabulary), E rows in {1, 32, 256}: "plain"
   (top-k 50, no new parameter), "seeded" (top-k 50, every row seeded), "biased" (top-k 50, every row with a bias row,
   plus the accounting kernel), on the plain sampler and on the vocab-parallel pair (vp_candidates + vp_final, one
   shard).
2. End to end: the bench.py workload (Qwen3-8B dummy weights, ShareGPT-shaped lengths, greedy, prefix caching on),
   no request using the parameters vs every request with frequency_penalty = presence_penalty = 0.5, alternated in
   one process.
Prints one JSON line per measurement, each with the GPU name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, plim = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": plim}
    except Exception as e:  # noqa: BLE001
        return {"gpu": None, "power_limit": None, "error": repr(e)}


def kernels(info: dict, iters: int = 100):
    import torch
    from gllm_b200.ops import sm100
    v = 151936
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    logits = (torch.randn(256, v, device=dev, generator=g) * 3).bfloat16()
    bias = torch.zeros(257, v, device=dev)
    out_seen = torch.zeros(257, (v + 31) // 32, dtype=torch.int32, device=dev)
    for e in (1, 32, 256):
        x = logits[:e]
        temp = torch.full((e,), 0.8, device=dev)
        top_k = torch.full((e,), 50, dtype=torch.int32, device=dev)
        top_p = torch.ones(e, device=dev)
        step = torch.zeros(1, dtype=torch.int64, device=dev)
        seeds = torch.arange(e, dtype=torch.int64, device=dev)
        pos = torch.full((e,), 100, dtype=torch.int32, device=dev)
        bslot = torch.arange(1, e + 1, dtype=torch.int32, device=dev)
        fp = torch.full((e,), 0.5, device=dev)
        cases = {"plain": {}, "seeded": dict(seeds=seeds, seed_pos=pos), "biased": dict(bias=bias, bias_slot=bslot)}
        for name, kw in cases.items():
            for route in ("plain", "vocab_parallel"):
                def run():
                    if route == "plain":
                        tok = sm100.sample(x, temp, top_k, top_p, seed=1, step=step, **kw)
                    else:
                        rec = sm100.vp_candidates(x, v, v, 256, temp, top_k, top_p, seed=1, step=step, **kw)
                        tok = sm100.vp_final(rec.unsqueeze(0), 256, v, top_k, top_p, seed=1, step=step,
                                             seeds=kw.get("seeds"), seed_pos=kw.get("seed_pos"))
                    if name == "biased":
                        sm100.bias_account(bias, out_seen, bslot, tok, fp, fp)
                for _ in range(10):
                    run()
                torch.cuda.synchronize()
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                for _ in range(iters):
                    run()
                t1.record()
                torch.cuda.synchronize()
                us = t0.elapsed_time(t1) * 1e3 / iters
                print(json.dumps({"kind": "kernel", "case": name, "route": route, "E": e, "V": v, "dtype": "bf16",
                                  "top_k": 50, "us": round(us, 2), **info}), flush=True)


def e2e(info: dict, num_prompts: int, rounds: int):
    import torch
    from bench import synth_requests
    from gllm_b200 import LLM
    llm = LLM("preset:qwen3-8b", load_format="dummy", maxp=4096, maxd=1024, max_cuda_graph_bs=512,
              enable_prefix_caching=True, gpu_memory_util=0.9, model_max_length=2048 + 16, log_stats=False,
              launch_mode="inproc", seed=0)
    vocab = llm.loader.config["vocab_size"]
    _, out_lens = synth_requests(num_prompts, vocab, 0)
    total_out = sum(out_lens)
    pass_idx = [0]

    def one(pen):
        prompts = synth_requests(num_prompts, vocab, 0, pass_idx[0])[0]    # fresh ids: no cross-pass cache hits
        pass_idx[0] += 1
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        llm.generate(tokens=prompts, output_lens=out_lens, ignore_eos=True, top_k=1, temperature=0.0,
                     frequency_penalty=pen, presence_penalty=pen)
        torch.cuda.synchronize()
        return total_out / (time.perf_counter() - t0)

    one(None)             # warm-up: both shapes of the step
    one(0.5)
    res = {"none": [], "penalties": []}
    for _ in range(rounds):
        res["none"].append(round(one(None), 1))
        res["penalties"].append(round(one(0.5), 1))
    mean = {k: sum(v) / len(v) for k, v in res.items()}
    print(json.dumps({"kind": "e2e", "model": "qwen3-8b (dummy weights)", "num_prompts": num_prompts,
                      "output_tokens_per_pass": total_out, "output_tok_per_s": res,
                      "overhead": round(1 - mean["penalties"] / mean["none"], 4),
                      "feed_steps": llm.worker.runner.stats.get("feed_steps", 0), **info}), flush=True)
    llm.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-kernels", action="store_true")
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--num-prompts", type=int, default=500)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this benchmark measures the GPU; there is no CPU fallback"
    info = gpu_info()
    if not args.skip_kernels:
        kernels(info)
    if not args.skip_e2e:
        e2e(info, args.num_prompts, args.rounds)


if __name__ == "__main__":
    main()
