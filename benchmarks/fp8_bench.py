"""FP8 W8A8 (per-channel weights, per-token activations) on one GPU: what the W8A8 GEMMs cost against the bf16 GEMM and
the block-scaled FP8 GEMM, where the decode kernel should hand over to the prefill kernel, and what FP8 gives the
engine.

    python benchmarks/fp8_bench.py [--part all|kernels|switch|engine] [--num-prompts 500] [--rounds 2]

1. Kernels: every projection of Qwen3-8B and Llama-3-70B at tp 1 and 2 (N, K), M in {1, 8, 32, 64, 256, 1024, 8192}:
   `ops.sm100.linear_fp8` (per-token quantiser + GEMM) against `ops.sm100.linear` on a bf16 weight and
   `ops.sm100.linear_fp8_block` (its own per-group quantiser + GEMM) on the same shape, and the per-token quantiser
   alone. Bytes are the minimum the W8A8 path must move (e4m3 weight, fp32 scales, x read in bf16, y written in bf16);
   FLOPs are 2·M·N·K, against 1,979 TFLOP/s dense FP8. Device time of 20 launches captured in one CUDA graph, replayed
   under events.
2. Switch: the decode (swap-AB split-K) and the prefill (persistent wgmma) W8A8 kernels at M in 16..128 on the same
   shapes, to place `sm100._FP8_SMALLM_MAX`.
3. Engine: output tokens/s of `preset:qwen3-8b` in bf16 and with `quantization="fp8"` (dummy weights) on the bench.py
   workload, then decode at 1, 8 and 32 concurrent requests of 256 output tokens, and GB of weights and KV pages of
   each arm. The arms alternate, each in a child process of this script (an engine does not return all of its device
   memory at shutdown), `--rounds` times.
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
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))

from w4a16_bench import MS, SHAPES, _card, _gen, _llm, _time  # noqa: E402

FP8_PEAK_TFLOPS = 1979.0


def _shapes():
    for model, mods in SHAPES.items():
        for tp in (1, 2):
            for name, (n, k, kind) in mods.items():
                yield model, tp, name, *((n // tp, k) if kind == "col" else (n, k // tp))


def _weights(n, k, gen, dev):
    from gllm_b200.ops import ref
    codes = (torch.randn(n, k, device=dev, generator=gen) * 100).clamp(-448, 448).to(torch.float8_e4m3fn)
    w8 = ref.Fp8Weight(codes, torch.full((n,), 2e-4, device=dev))
    wb = (torch.randn(n, k, device=dev, generator=gen) * 0.02).to(torch.bfloat16)
    ws_block = torch.full((-(-n // 128), k // 128), 2e-4, device=dev)
    return w8, wb, ws_block


def kernels():
    from gllm_b200.ops import sm100
    dev = torch.device("cuda")
    gen = torch.Generator(device=dev).manual_seed(0)
    for model, tp, name, n, k in _shapes():
        w8, wb, wsb = _weights(n, k, gen, dev)
        for m in MS:
            x = torch.randn(m, k, device=dev, generator=gen).to(torch.bfloat16)
            y = torch.empty(m, n, dtype=torch.bfloat16, device=dev)
            t8 = _time(lambda: sm100.linear_fp8(x, w8, out=y))
            t16 = _time(lambda: sm100.linear(x, wb, out=y))
            tb = _time(lambda: sm100.linear_fp8_block(x, w8.codes, wsb, out=y))
            tq = _time(lambda: sm100.fp8_quant_token(x))
            b8 = n * k + 4 * n + 2 * m * k + 2 * m * n
            fl = 2 * m * n * k
            print(json.dumps({"kernel": "w8a8", "model": model, "tp": tp, "proj": name, "N": n, "K": k, "M": m,
                              "fp8_us": round(t8 * 1e3, 2), "bf16_us": round(t16 * 1e3, 2),
                              "block_us": round(tb * 1e3, 2), "quant_us": round(tq * 1e3, 2),
                              "vs_bf16": round(t16 / t8, 2), "vs_block": round(tb / t8, 2),
                              "fp8_TB/s": round(b8 / t8 / 1e9, 3),
                              "fp8_TFLOP/s": round(fl / t8 / 1e9, 1),
                              "fp8_share_of_1979": round(fl / t8 / 1e9 / FP8_PEAK_TFLOPS, 3)}), flush=True)
        del w8, wb, wsb


def switch():
    from gllm_b200.ops import sm100
    dev = torch.device("cuda")
    gen = torch.Generator(device=dev).manual_seed(1)
    keep = sm100._FP8_SMALLM_MAX
    for model, tp, name, n, k in _shapes():
        w8, _, _ = _weights(n, k, gen, dev)
        for m in (16, 32, 48, 64, 96, 128):
            x = torch.randn(m, k, device=dev, generator=gen).to(torch.bfloat16)
            y = torch.empty(m, n, dtype=torch.bfloat16, device=dev)
            t = {}
            for arm, lim in (("small", 128), ("large", 0)):
                sm100._FP8_SMALLM_MAX = lim
                t[arm] = _time(lambda: sm100.linear_fp8(x, w8, out=y))
            sm100._FP8_SMALLM_MAX = keep
            print(json.dumps({"switch": "w8a8", "model": model, "tp": tp, "proj": name, "N": n, "K": k, "M": m,
                              "small_us": round(t["small"] * 1e3, 2), "large_us": round(t["large"] * 1e3, 2)}),
                  flush=True)


def engine(num_prompts: int, arm: str):
    from bench import synth_requests
    kw = {"quantization": "fp8"} if arm == "fp8" else {}
    llm = _llm("preset:qwen3-8b", **kw)
    runner = llm.worker.runner
    gb = sum(p.numel() * p.element_size() for p in runner.model.parameters()) / 2 ** 30
    print(json.dumps({"engine": arm, "weights_GB": round(gb, 2), "kv_pages": runner.num_pages,
                      "page_size": runner.page_size}), flush=True)
    vocab = llm.loader.config["vocab_size"]
    _, out_lens = synth_requests(num_prompts, vocab, 0)
    for k in range(3):           # pass 0 warms up
        prompts, _ = synth_requests(num_prompts, vocab, 0, k + 1)
        dt = _gen(llm, prompts, out_lens)
        if k:
            print(json.dumps({"engine": arm, "workload": "bench.py", "pass": k,
                              "output_tok_s": round(sum(out_lens) / dt, 1), "seconds": round(dt, 2)}), flush=True)
    g = torch.Generator().manual_seed(1)
    for conc in (1, 8, 32):
        prompts = [torch.randint(10, vocab - 10, (128,), generator=g).tolist() for _ in range(conc)]
        _gen(llm, prompts, [16] * conc)
        dt = _gen(llm, prompts, [256] * conc)
        print(json.dumps({"engine": arm, "workload": "decode", "concurrent": conc, "output_tokens": 256,
                          "output_tok_s": round(256 * conc / dt, 1), "seconds": round(dt, 2)}), flush=True)
    llm.shutdown()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--part", default="all", choices=["all", "kernels", "switch", "engine"])
    ap.add_argument("--num-prompts", type=int, default=500)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--arm", default=None, choices=["bf16", "fp8"], help="engine part: this arm only, in this process")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "fp8_bench measures on the GPU"
    if not args.arm:
        print(json.dumps({"card": _card()}), flush=True)
    if args.part in ("all", "kernels"):
        kernels()
    if args.part in ("all", "switch"):
        switch()
    if args.part == "engine" and args.arm:
        engine(args.num_prompts, args.arm)
    elif args.part in ("all", "engine"):
        for _ in range(args.rounds):
            for arm in ("bf16", "fp8"):
                subprocess.run([sys.executable, os.path.abspath(__file__), "--part", "engine", "--arm", arm,
                                "--num-prompts", str(args.num_prompts)], check=True)


if __name__ == "__main__":
    main()
