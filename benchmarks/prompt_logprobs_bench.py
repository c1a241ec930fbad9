"""Prompt log-probabilities (scoring) on one GPU: what a scored prompt token costs.

    python benchmarks/prompt_logprobs_bench.py [--part all|kernels|engine] [--engine-requests 24] [--rounds 3]

1. Kernels, per LM-head tile of R rows at V = 151936 (Qwen3) and tp shard widths 1 and 2: the tile's LM-head GEMM
   (H = 4096), then each records pass on the tile the GEMM just wrote (as the engine runs them), for N = 0, 1, 5:
   prompt_logprobs_shard_kernel (one pass, N <= 1) against logprobs_shard_kernel. A records pass is timed as
   (GEMM + pass) - GEMM over a rotation of 8 distinct tiles; bytes/s counts one read of the tile's logits.
2. Engine scoring throughput, Qwen3-8B with dummy weights: requests of 512-2048 prompt tokens and one output token,
   with prompt_logprobs = 0, = 1 and without, alternated in one process; prompt tokens per second.
Prints one JSON line per measurement, the card's name and power limit first (read in the same run).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

V, H = 151936, 4096


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def _time(fn, iters: int) -> float:
    """ms per call, CUDA events around `iters` calls after a warm-up."""
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def kernels():
    from gllm_b200.ops import sm100
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    for tp in (1, 2):
        per = -(-V // tp)
        per = (per + 127) // 128 * 128
        w = (torch.randn(per, H, device=dev, generator=g) * 0.02).to(torch.bfloat16)
        for r in (64, 128, 256):
            xs = [torch.randn(r, H, device=dev, generator=g).to(torch.bfloat16) for _ in range(8)]
            buf = torch.empty(r, per, dtype=torch.bfloat16, device=dev)
            targets = torch.randint(0, min(per, V), (r,), device=dev, generator=g, dtype=torch.int32)
            valid = min(per, V)
            state = {"i": 0}

            def gemm():
                state["i"] = (state["i"] + 1) % len(xs)
                sm100.linear(xs[state["i"]], w, out=buf)

            t_gemm = _time(gemm, 80)
            flops = 2.0 * r * H * per
            print(json.dumps({"what": "lm_head_tile", "tp": tp, "rows": r, "shard_cols": per, "ms": round(t_gemm, 4),
                              "tflops": round(flops / t_gemm / 1e9, 1)}), flush=True)
            nbytes = r * valid * 2
            for n in (0, 1, 5):
                arms = {"logprobs_shard": lambda n=n: sm100.logprobs_shard(buf, valid, n, targets)}
                if n <= 1:
                    arms["prompt_logprobs_shard"] = lambda n=n: sm100.prompt_logprobs_shard(buf, valid, n, targets)
                for name, rec in arms.items():
                    def both(rec=rec):
                        gemm()
                        rec()
                    t = _time(both, 80) - t_gemm
                    alone = _time(rec, 80)
                    print(json.dumps({"what": "records", "kernel": name, "tp": tp, "rows": r, "N": n,
                                      "ms_after_gemm": round(t, 4), "ms_alone": round(alone, 4),
                                      "GB_per_s_after_gemm": round(nbytes / max(t, 1e-6) / 1e6, 1)}), flush=True)
            del xs, buf
        del w
        torch.cuda.empty_cache()


def engine(num_requests: int, rounds: int):
    from gllm_b200 import LLM
    import random
    rnd = random.Random(0)
    llm = LLM("preset:qwen3-8b", load_format="dummy", maxp=4096, maxd=256, gpu_memory_util=0.85,
              model_max_length=2048 + 16, log_stats=False, seed=0, enable_prefix_caching=False)
    vocab = 151936
    prompts = [[rnd.randrange(vocab) for _ in range(rnd.randint(512, 2048))] for _ in range(num_requests)]
    ntok = sum(len(p) for p in prompts)
    arms = [None, 0, 1]
    llm.generate(tokens=prompts[:4], output_lens=[1] * 4, ignore_eos=True, prompt_logprobs=1)   # warm-up
    res = {str(a): [] for a in arms}
    for _ in range(rounds):
        for a in arms:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            llm.generate(tokens=prompts, output_lens=[1] * len(prompts), ignore_eos=True, prompt_logprobs=a)
            torch.cuda.synchronize()
            res[str(a)].append(ntok / (time.perf_counter() - t0))
    llm.shutdown()
    for a, v in res.items():
        print(json.dumps({"what": "engine_scoring", "model": "qwen3-8b dummy", "prompt_logprobs": a,
                          "requests": num_requests, "prompt_tokens": ntok,
                          "prompt_tok_per_s": [round(x) for x in v]}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--engine-requests", type=int, default=24)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--part", default="all", choices=["all", "kernels", "engine"])
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    print(json.dumps({"card": _card()}), flush=True)
    if args.part != "engine":
        kernels()
    if args.part != "kernels":
        engine(args.engine_requests, args.rounds)


if __name__ == "__main__":
    main()
