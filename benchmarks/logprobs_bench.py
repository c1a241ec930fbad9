"""Cost of token log-probabilities on the GPU (csrc/sample/sampler.cu: logprobs_shard_kernel + logprobs_final_kernel).

    python benchmarks/logprobs_bench.py [--skip-kernels] [--skip-e2e] [--num-prompts 500] [--rounds 2]

1. Kernel time of shard + final with CUDA events at V = 151936 bf16 logits (Qwen3's vocabulary), E requesting rows
   in {1, 32, 256} and N in {0, 5, 20}; the unique bytes each row reads (its V bf16 logits) and the share of the H100
   SXM data-sheet HBM3 bandwidth (3.35 TB/s) that rate would be. The kernel re-reads the row from L2 on later passes.
2. End to end: the bench.py workload (Qwen3-8B dummy weights, ShareGPT-shaped lengths, greedy, prefix caching on),
   every request without log-probs vs every request with top_logprobs = 5, alternated in one process.
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

HBM_BYTES_PER_S = 3.35e12


def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, plim = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": plim}
    except Exception as e:  # noqa: BLE001
        return {"gpu": None, "power_limit": None, "error": repr(e)}


def kernels(info: dict, iters: int = 200):
    import torch
    from gllm_b200.ops import sm100
    v = 151936
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    logits = (torch.randn(256, v, device=dev, generator=g) * 3).bfloat16()
    toks = logits.float().argmax(-1).to(torch.int32)
    for e in (1, 32, 256):
        rows = torch.arange(e, dtype=torch.int32, device=dev)
        for n in (0, 5, 20):
            def run():
                rec = sm100.logprobs_shard(logits, v, n, toks, rows)
                return sm100.logprobs_final(rec.unsqueeze(0), n)
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
            row_bytes = v * 2
            rate = e * row_bytes / (us * 1e-6)
            print(json.dumps({"kind": "kernel", "E": e, "N": n, "V": v, "dtype": "bf16", "us": round(us, 2),
                              "bytes_read_per_row": row_bytes, "unique_bytes_per_s": round(rate / 1e9, 1),
                              "share_of_hbm_peak": round(rate / HBM_BYTES_PER_S, 4), **info}), flush=True)


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

    def one(lp):
        prompts = synth_requests(num_prompts, vocab, 0, pass_idx[0])[0]    # fresh ids: no cross-pass cache hits
        pass_idx[0] += 1
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        seqs = llm.generate(tokens=prompts, output_lens=out_lens, ignore_eos=True, top_k=1, temperature=0.0,
                            logprobs=lp)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if lp is not None:
            assert all(len(s.output_logprobs) == s.num_output_tokens for s in seqs)
        return total_out / dt

    one(None)             # warm-up: both shapes of the step
    one(5)
    res = {"none": [], "top5": []}
    for _ in range(rounds):
        res["none"].append(round(one(None), 1))
        res["top5"].append(round(one(5), 1))
    mean = {k: sum(v) / len(v) for k, v in res.items()}
    print(json.dumps({"kind": "e2e", "model": "qwen3-8b (dummy weights)", "num_prompts": num_prompts,
                      "output_tokens_per_pass": total_out, "output_tok_per_s": res,
                      "overhead": round(1 - mean["top5"] / mean["none"], 4),
                      "logprob_rows": llm.worker.runner.stats.get("logprob_rows", 0), **info}), flush=True)
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
