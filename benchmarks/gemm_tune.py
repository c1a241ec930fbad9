"""Sweep (BN, split-K) for the decode-sized GEMMs of Qwen3-8B and print the best configuration per shape next
to what the built-in cost model picks (CUDA-event timing, L2 flushed between iterations).

    python benchmarks/gemm_tune.py
"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from benchmarks.kernel_bench import timeit  # noqa: E402
from gllm_b200.ops import lib as _lib, ref, sm100  # noqa: E402


def main():
    L = _lib.load()
    H, I, QKV = 4096, 12288, 6144
    for m in (64, 128, 256, 384, 512):
        for n, k, name, silu in ((QKV, H, "qkv", False), (H, H, "o", False), (2 * I, H, "gate_up", True),
                                 (H, I, "down", False)):
            x = (torch.randn(m, k, device="cuda") * 0.1).bfloat16()
            w = (torch.randn(n, k, device="cuda") * 0.1).bfloat16()
            res = {}
            for bn in ((256,) if silu else (256, 128, 64)):
                for split in (1, 2, 4, 8):
                    sm100._FORCE_BN = bn
                    L.gllm_gemm_tune(split if split > 1 else 0, 0 if split == 1 else 100000)
                    fn = (lambda: sm100.linear_silu_mul(x, w)) if silu else (lambda: sm100.linear(x, w))
                    res[f"{bn}x{split}"] = round(timeit(fn, iters=12, warmup=3) * 1e3, 1)
            sm100._FORCE_BN = 0
            L.gllm_gemm_tune(0, 512)
            fn = (lambda: sm100.linear_silu_mul(x, w)) if silu else (lambda: sm100.linear(x, w))
            auto = round(timeit(fn, iters=12, warmup=3) * 1e3, 1)
            out = torch.empty(m, n, device="cuda", dtype=torch.bfloat16)
            cublas = round(timeit(lambda: torch.matmul(x, w.t(), out=out), iters=12, warmup=3) * 1e3, 1)
            best = min(res, key=res.get)
            print(json.dumps({"M": m, "case": name, "auto_us": auto, "best": best, "best_us": res[best],
                              "cublas_us": cublas, "all": res}), flush=True)


if __name__ == "__main__":
    main()
