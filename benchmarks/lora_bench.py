"""Multi-LoRA on one GPU: what the adapter kernels cost, and the serving overhead of adapters.

    python benchmarks/lora_bench.py [--part all|kernels|engine] [--num-prompts 500] [--rounds 2]

1. Kernels at Qwen3-8B shapes (H 4096, q/k/v 4096/1024/1024, I 12288), tp 1: lora_shrink and lora_expand_add for
   the q/k/v, o and down projections and lora_expand_silu_mul for gate/up, for T in {1, 8, 32, 256, 2048, 8192} token
   rows, rank r in {16, 64}, and the rows spread round-robin over 1 or 4 adapters. Bytes are the minimum the kernel
   must move (each active adapter's A or B once, x or y read / written once, U in fp32); FLOPs are 2·T·M·K (shrink) and
   2·T·N·r (expand). Device time of 50 launches captured in one CUDA graph, as decode replays them.
2. Engine: output tokens/s on the bench.py workload (Qwen3-8B with dummy weights, 500 ShareGPT-shaped requests,
   greedy, CUDA graphs, prefix caching) in three arms alternated in one process: base model only, every request on
   one rank-16 adapter, requests spread over four rank-16 adapters.
Prints one JSON line per measurement, the card's name and power limit first (read in the same run).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

H, Q, KV, INTER = 4096, 4096, 1024, 12288


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def _time(fn, iters: int = 50) -> float:
    """Device ms per call: `iters` calls captured in one CUDA graph (as decode runs them), replayed under events, so
    the Python and ctypes cost of an eager call (tens of µs) does not hide the kernel time at small T."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn()
    g.replay()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    g.replay()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def _csr(t: int, n_adapters: int):
    import numpy as np
    from gllm_b200.input_data import InputData
    inp = InputData(t, 1, 1, "cuda")
    inp.set_lora(n_adapters)
    inp._flip = 1
    inp._load_lora((np.arange(t) % n_adapters).astype(np.int32))
    torch.cuda.synchronize()
    return inp._lora[0][1], inp._lora[1][1], inp._lora[2][1][:t], inp.lora_groups


def kernels():
    from gllm_b200.ops import sm100
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    # (name, K, module widths of the output)
    mods = [("qkv", H, [Q, KV, KV]), ("o", Q, [H]), ("down", INTER, [H])]
    for r in (16, 64):
        for n_ad in (1, 4):
            for t in (1, 8, 32, 256, 2048, 8192):
                csr = _csr(t, n_ad)
                active = min(n_ad, t)
                for name, k, widths in mods:
                    m, n = len(widths) * r, sum(widths)
                    x = torch.randn(t, k, device=dev, generator=g).to(torch.bfloat16)
                    A = (torch.randn(n_ad, m, k, device=dev, generator=g) * 0.05).to(torch.bfloat16)
                    B = (torch.randn(n_ad, n, r, device=dev, generator=g) * 0.05).to(torch.bfloat16)
                    y = torch.randn(t, n, device=dev, generator=g).to(torch.bfloat16)
                    bounds = [0]
                    for w in widths:
                        bounds.append(bounds[-1] + w)
                    u = sm100.lora_shrink(x, A, *csr)
                    ms_s = _time(lambda: sm100.lora_shrink(x, A, *csr))
                    ms_e = _time(lambda: sm100.lora_expand_add(y, u, B, bounds, *csr))
                    by_s = active * m * k * 2 + t * k * 2 + t * m * 4
                    by_e = active * n * r * 2 + t * n * 4 + t * m * 4
                    for op, ms, by, fl in (("shrink", ms_s, by_s, 2 * t * m * k), ("expand_add", ms_e, by_e,
                                                                                  2 * t * n * r)):
                        print(json.dumps({"kernel": f"lora_{op}", "module": name, "T": t, "r": r, "adapters": n_ad,
                                          "ms": round(ms, 4), "bytes": by, "flops": fl,
                                          "TB/s": round(by / ms / 1e9, 3), "TFLOP/s": round(fl / ms / 1e9, 2)}),
                              flush=True)
                # gate/up: shrink (m = 2) then the fused expand + SiLU-gate
                x = torch.randn(t, H, device=dev, generator=g).to(torch.bfloat16)
                A = (torch.randn(n_ad, 2 * r, H, device=dev, generator=g) * 0.05).to(torch.bfloat16)
                B = (torch.randn(n_ad, 2 * INTER, r, device=dev, generator=g) * 0.05).to(torch.bfloat16)
                pre = torch.randn(t, 2 * INTER, device=dev, generator=g).to(torch.bfloat16)
                u = sm100.lora_shrink(x, A, *csr)
                ms = _time(lambda: sm100.lora_expand_silu_mul(pre, u, B, *csr))
                by = active * 2 * INTER * r * 2 + t * 2 * INTER * 2 + t * INTER * 2 + t * 2 * r * 4
                fl = 2 * t * 2 * INTER * r
                print(json.dumps({"kernel": "lora_expand_silu_mul", "module": "gate_up", "T": t, "r": r,
                                  "adapters": n_ad, "ms": round(ms, 4), "bytes": by, "flops": fl,
                                  "TB/s": round(by / ms / 1e9, 3), "TFLOP/s": round(fl / ms / 1e9, 2)}), flush=True)


def engine(num_prompts: int, rounds: int):
    from bench import synth_requests
    from gllm_b200 import LLM
    from gllm_b200.models.presets import PRESETS
    from lora_util import write_adapter
    cfg = dict(PRESETS["qwen3-8b"])
    tmp = tempfile.mkdtemp(prefix="gllm_lora_bench_")
    mods = {}
    for i in range(4):
        p = os.path.join(tmp, f"a{i}")
        write_adapter(p, cfg, r=16, alpha=32, seed=i, std=0.01)
        mods[f"a{i}"] = p
    llm = LLM("preset:qwen3-8b", load_format="dummy", maxp=4096, maxd=1024, max_cuda_graph_bs=512,
              enable_prefix_caching=True, gpu_memory_util=0.9, model_max_length=2048 + 16, log_stats=False,
              launch_mode="inproc", seed=0, lora_modules=mods, max_lora_rank=16)
    vocab = llm.loader.config["vocab_size"]
    _, out_lens = synth_requests(num_prompts, vocab, 0)
    arms = {"base": None, "one_adapter": "a0", "four_adapters": [f"a{i % 4}" for i in range(num_prompts)]}
    k = 0
    for rnd in range(rounds + 1):        # round 0 warms every arm up
        for arm, lora in arms.items():
            k += 1
            prompts, _ = synth_requests(num_prompts, vocab, 0, k)     # fresh ids: no prefix-cache hits across passes
            st = llm.worker.runner.stats
            g0, l0 = st["graph_steps"], st.get("lora_graph_steps", 0)
            torch.cuda.synchronize()
            t0 = time.time()
            llm.generate(tokens=prompts, output_lens=out_lens, ignore_eos=True, top_k=1, temperature=0.0, lora=lora)
            torch.cuda.synchronize()
            dt = time.time() - t0
            if rnd:
                print(json.dumps({"engine": arm, "round": rnd, "output_tok_s": round(sum(out_lens) / dt, 1),
                                  "seconds": round(dt, 2), "graph_steps": st["graph_steps"] - g0,
                                  "lora_graph_steps": st.get("lora_graph_steps", 0) - l0}), flush=True)
    llm.shutdown()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--part", default="all", choices=["all", "kernels", "engine"])
    ap.add_argument("--num-prompts", type=int, default=500)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "lora_bench measures on the GPU"
    print(json.dumps({"card": _card()}), flush=True)
    if args.part in ("all", "kernels"):
        kernels()
    if args.part in ("all", "engine"):
        engine(args.num_prompts, args.rounds)


if __name__ == "__main__":
    main()
