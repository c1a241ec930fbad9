"""4-bit weights (AWQ / GPTQ) on one GPU: what the W4A16 GEMM costs against the bf16 GEMM, and what int4 weights give
the engine.

    python benchmarks/w4a16_bench.py [--part all|kernels|engine|70b] [--num-prompts 500]

1. Kernels: every projection of Qwen3-8B and Llama-3-70B at tp 1 and 2 (N, K), M in {1, 8, 32, 64, 256, 1024,
   8192} token rows, group 128, fp16 scales: `ops.sm100.linear_w4a16` against `ops.sm100.linear` on a bf16 weight of
   the same shape. Bytes are the minimum each kernel must move (int4 codes, fp16 scales and uint8 zeros or the bf16
   weight, x read and y written once in bf16); FLOPs are 2·M·N·K. Device time of 20 launches captured in one CUDA
   graph, replayed under events.
2. Engine: output tokens/s of `preset:qwen3-8b` and `preset:qwen3-8b-awq` (dummy weights) on the bench.py workload
   (500 ShareGPT-shaped requests, greedy, CUDA graphs), then decode at 1, 8 and 32 concurrent requests of 256 output
   tokens (prompts of 128 tokens). The two models run one after the other, each in a child process of this script
   (an engine does not return all of its device memory at shutdown).
3. `preset:llama-3-70b-awq` on one GPU: GB of weights, KV pages, and output tokens/s at 32 concurrent requests.
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {   # projection -> (N, K) at tp 1; column-parallel ones split N, row-parallel ones split K
    "qwen3-8b": {"qkv": (6144, 4096, "col"), "o": (4096, 4096, "row"), "gate_up": (24576, 4096, "col"),
                 "down": (4096, 12288, "row")},
    "llama-3-70b": {"qkv": (10240, 8192, "col"), "o": (8192, 8192, "row"), "gate_up": (57344, 8192, "col"),
                    "down": (8192, 28672, "row")},
}
MS = (1, 8, 32, 64, 256, 1024, 8192)


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def _time(fn, iters: int = 20) -> float:
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


def kernels():
    from gllm_b200.ops import ref, sm100
    dev = torch.device("cuda")
    gen = torch.Generator(device=dev).manual_seed(0)
    for model, mods in SHAPES.items():
        for tp in (1, 2):
            for name, (n, k, kind) in mods.items():
                n, k = (n // tp, k) if kind == "col" else (n, k // tp)
                g = k // 128
                packed = torch.randint(-2 ** 31, 2 ** 31 - 1, (n, k // 8), dtype=torch.int32, device=dev,
                                       generator=gen)
                w4 = ref.Int4Weight(packed, torch.full((g, n), 0.004, dtype=torch.float16, device=dev),
                                    torch.full((g, n), 8, dtype=torch.uint8, device=dev), 128, k)
                wb = (torch.randn(n, k, device=dev, generator=gen) * 0.02).to(torch.bfloat16)
                for m in MS:
                    x = torch.randn(m, k, device=dev, generator=gen).to(torch.bfloat16)
                    y = torch.empty(m, n, dtype=torch.bfloat16, device=dev)
                    ms4 = _time(lambda: sm100.linear_w4a16(x, w4, out=y))
                    ms16 = _time(lambda: sm100.linear(x, wb, out=y))
                    io = 2 * m * k + 2 * m * n
                    b4, b16 = n * k // 2 + g * n * 3 + io, 2 * n * k + io
                    fl = 2 * m * n * k
                    print(json.dumps({"kernel": "w4a16", "model": model, "tp": tp, "proj": name, "N": n, "K": k,
                                      "M": m, "w4_us": round(ms4 * 1e3, 2), "bf16_us": round(ms16 * 1e3, 2),
                                      "speedup": round(ms16 / ms4, 2),
                                      "w4_TB/s": round(b4 / ms4 / 1e9, 3), "bf16_TB/s": round(b16 / ms16 / 1e9, 3),
                                      "w4_TFLOP/s": round(fl / ms4 / 1e9, 1),
                                      "bf16_TFLOP/s": round(fl / ms16 / 1e9, 1)}), flush=True)


def _llm(model, **kw):
    from gllm_b200 import LLM
    args = dict(load_format="dummy", maxp=4096, maxd=1024, max_cuda_graph_bs=512, enable_prefix_caching=True,
                gpu_memory_util=0.9, model_max_length=2048 + 16, log_stats=False, launch_mode="inproc", seed=0)
    args.update(kw)
    return LLM(model, **args)


def _gen(llm, prompts, out_lens):
    torch.cuda.synchronize()
    t0 = time.time()
    llm.generate(tokens=prompts, output_lens=out_lens, ignore_eos=True, top_k=1, temperature=0.0)
    torch.cuda.synchronize()
    return time.time() - t0


def engine(num_prompts: int, model: str):
    from bench import synth_requests
    llm = _llm(model)
    vocab = llm.loader.config["vocab_size"]
    _, out_lens = synth_requests(num_prompts, vocab, 0)
    for k in range(3):           # pass 0 warms up
        prompts, _ = synth_requests(num_prompts, vocab, 0, k + 1)
        dt = _gen(llm, prompts, out_lens)
        if k:
            print(json.dumps({"engine": model, "workload": "bench.py", "pass": k,
                              "output_tok_s": round(sum(out_lens) / dt, 1), "seconds": round(dt, 2)}), flush=True)
    g = torch.Generator().manual_seed(1)
    for conc in (1, 8, 32):
        prompts = [torch.randint(10, vocab - 10, (128,), generator=g).tolist() for _ in range(conc)]
        _gen(llm, prompts, [16] * conc)
        dt = _gen(llm, prompts, [256] * conc)
        print(json.dumps({"engine": model, "workload": "decode", "concurrent": conc, "output_tokens": 256,
                          "output_tok_s": round(256 * conc / dt, 1), "seconds": round(dt, 2)}), flush=True)
    llm.shutdown()


def llama70b():
    llm = _llm("preset:llama-3-70b-awq", max_cuda_graph_bs=64, maxd=64)
    runner = llm.worker.runner
    gb = sum(p.numel() * p.element_size() for p in runner.model.parameters()) / 2 ** 30
    vocab = llm.loader.config["vocab_size"]
    g = torch.Generator().manual_seed(2)
    prompts = [torch.randint(10, vocab - 10, (128,), generator=g).tolist() for _ in range(32)]
    _gen(llm, prompts, [16] * 32)
    dt = _gen(llm, prompts, [256] * 32)
    print(json.dumps({"engine": "preset:llama-3-70b-awq", "weights_GB": round(gb, 2), "kv_pages": runner.num_pages,
                      "page_size": runner.page_size, "concurrent": 32, "output_tokens": 256,
                      "output_tok_s": round(256 * 32 / dt, 1), "seconds": round(dt, 2)}), flush=True)
    llm.shutdown()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--part", default="all", choices=["all", "kernels", "engine", "70b"])
    ap.add_argument("--num-prompts", type=int, default=500)
    ap.add_argument("--model", default=None, help="engine part: this model only, in this process")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "w4a16_bench measures on the GPU"
    if not args.model:
        print(json.dumps({"card": _card()}), flush=True)
    if args.part in ("all", "kernels"):
        kernels()
    if args.part == "engine" and args.model:
        engine(args.num_prompts, args.model)
    elif args.part in ("all", "engine"):
        for model in ("preset:qwen3-8b", "preset:qwen3-8b-awq"):
            subprocess.run([sys.executable, os.path.abspath(__file__), "--part", "engine", "--model", model,
                            "--num-prompts", str(args.num_prompts)], check=True)
    if args.part in ("all", "70b"):
        llama70b()


if __name__ == "__main__":
    main()
