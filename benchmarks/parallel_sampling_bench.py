"""Parallel sampling (`n` choices per request) on the GPU.

    python benchmarks/parallel_sampling_bench.py [--skip-kernels] [--skip-e2e] [--num-prompts 64] [--n 8]
                                                 [--prompt-len 2048] [--output-len 256] [--rounds 1]

1. Kernel: `kv_copy_pages` (csrc/elemwise/kv_copy.cu) with CUDA events over many back-to-back launches, for Qwen3-8B
   cache shapes (36 layers, K and V, 8 KV heads of 128, 16-token pages: 72 tensors of 32 KiB pages) at 1, 8 and 64
   pairs: the launch alone, whose achieved GB/s counts every byte read and written, and the front-end call the engine
   makes (host checks and staging of the pairs included).
2. Engine: Qwen3-8B with dummy weights, `--num-prompts` prompts of `--prompt-len` random tokens, `--n` choices each,
   `--output-len` output tokens, temperature 1. The same sequences as `n` duplicated n = 1 requests, with prefix
   caching off and on. The arms alternate in one process (the engine's memory manager is swapped between passes, while
   it is idle). Reports output tok/s, prefill tokens computed and the peak number of KV pages in use.
Prints one JSON line per measurement, each with the GPU name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import random
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


def kernels(info: dict, iters: int = 200):
    import torch
    from gllm_b200.ops import sm100
    from gllm_b200.ops.ref import kv_cache_shape
    layers, pages = 36, 2048
    shape = kv_cache_shape(pages, 8, 128, 16)
    tensors = [torch.zeros(shape, dtype=torch.bfloat16, device="cuda") for _ in range(2 * layers)]
    page_bytes = tensors[0][0].numel() * 2
    bases = torch.tensor([t.data_ptr() for t in tensors], dtype=torch.int64, device="cuda")
    for n in (1, 8, 64):
        pairs = [(i, pages // 2 + i) for i in range(n)]
        dev_pairs = torch.tensor(pairs, dtype=torch.int32, device="cuda")
        res = {}
        # "kernel": the launch alone (pairs already on the device); "call": the engine's front end, which also checks
        # the pairs on the host and stages them to the device
        for what, fn in (("kernel", lambda: sm100.launch_kv_copy_pages(tensors, bases, dev_pairs)),
                         ("call", lambda: sm100.kv_copy_pages(tensors, pairs))):
            for _ in range(10):
                fn()
            torch.cuda.synchronize()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(iters):
                fn()
            t1.record()
            torch.cuda.synchronize()
            res[what] = t0.elapsed_time(t1) * 1e3 / iters
        moved = 2 * n * len(tensors) * page_bytes          # read + write
        print(json.dumps({"kind": "kernel", "op": "kv_copy_pages", "pairs": n, "tensors": len(tensors),
                          "page_bytes": page_bytes, "bytes_moved": moved, "kernel_us": round(res["kernel"], 2),
                          "kernel_GB_per_s": round(moved / res["kernel"] / 1e3, 1),
                          "call_us": round(res["call"], 2), **info}), flush=True)
    del tensors
    torch.cuda.empty_cache()


def e2e(info: dict, num_prompts: int, n: int, prompt_len: int, output_len: int, rounds: int):
    import torch
    from gllm_b200 import LLM
    from gllm_b200.memory_manager import MemoryManager, PrefixMemoryManager
    llm = LLM("preset:qwen3-8b", load_format="dummy", maxp=8192, maxd=1024, max_cuda_graph_bs=512,
              enable_prefix_caching=False, gpu_memory_util=0.9, model_max_length=prompt_len + output_len + 16,
              log_stats=False, launch_mode="inproc", seed=0)
    w = llm.worker
    sch, runner = w.scheduler, w.runner
    vocab = llm.loader.config["vocab_size"]
    usage = {"prefill": 0, "min_free": 1 << 30}
    step0, sched0 = runner.step, sch.schedule_once

    def step(batch, *a, **k):
        usage["prefill"] += batch.num_tokens - batch.num_decode_seqs
        return step0(batch, *a, **k)

    def schedule_once():
        out = sched0()
        usage["min_free"] = min(usage["min_free"], w.mm.get_num_free_pages())
        return out
    runner.step, sch.schedule_once = step, schedule_once
    pass_idx = [0]

    def one(arm):
        prefix = arm == "duplicated_prefix_on"
        if isinstance(w.mm, PrefixMemoryManager) != prefix:      # idle: every page is free
            w.mm = (PrefixMemoryManager if prefix else MemoryManager)(w.mm.num_pages, w.mm.page_size,
                                                                       reserve_dummy_page=True)
            sch.mm = w.mm
        rng = random.Random(pass_idx[0])                          # fresh prompts: no cross-pass cache hits
        pass_idx[0] += 1
        prompts = [[rng.randrange(vocab) for _ in range(prompt_len)] for _ in range(num_prompts)]
        kw = dict(ignore_eos=True, temperature=1.0, top_k=0, top_p=1.0)
        usage["prefill"], usage["min_free"] = 0, w.mm.get_num_free_pages()
        pre0 = sch.num_preempt_seqs
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if arm == "n":
            outs = llm.generate(tokens=prompts, output_lens=[output_len] * num_prompts, n=n, **kw)
        else:
            outs = llm.generate(tokens=[p for p in prompts for _ in range(n)],
                                output_lens=[output_len] * (num_prompts * n), **kw)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        total = sum(s.num_output_tokens for s in outs)
        return {"output_tok_per_s": round(total / dt, 1), "seconds": round(dt, 2), "output_tokens": total,
                "prefill_tokens": usage["prefill"], "peak_kv_pages": w.mm.usable_pages - usage["min_free"],
                "preempted": sch.num_preempt_seqs - pre0}

    arms = ["n", "duplicated_prefix_off", "duplicated_prefix_on"]
    saved = num_prompts
    num_prompts = max(1, saved // 8)             # warm-up: every arm, a smaller pass
    for arm in arms:
        one(arm)
    num_prompts = saved
    for r in range(rounds):
        for arm in arms:
            res = one(arm)
            print(json.dumps({"kind": "e2e", "arm": arm, "round": r, "model": "qwen3-8b (dummy weights)",
                              "prompts": num_prompts, "n": n, "prompt_len": prompt_len, "output_len": output_len,
                              "kv_pages": w.mm.usable_pages, "page_size": w.mm.page_size, **res, **info}),
                  flush=True)
    llm.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-kernels", action="store_true")
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--num-prompts", type=int, default=64)
    ap.add_argument("--n", type=int, default=8)
    ap.add_argument("--prompt-len", type=int, default=2048)
    ap.add_argument("--output-len", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=1)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this benchmark measures the GPU; there is no CPU fallback"
    info = gpu_info()
    if not args.skip_kernels:
        kernels(info)
    if not args.skip_e2e:
        e2e(info, args.num_prompts, args.n, args.prompt_len, args.output_len, args.rounds)


if __name__ == "__main__":
    main()
