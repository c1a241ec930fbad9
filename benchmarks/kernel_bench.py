"""Micro-benchmarks of the sm_90a kernels against their rooflines (CUDA-event timing, L2 flushed
between iterations). Prints one JSON line per case; cuBLAS / flash-attn numbers are printed only
as context for the same shapes.

    python benchmarks/kernel_bench.py [gemm|attn|all]
"""
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gllm_b200.ops import ref, sm100  # noqa: E402

PEAKS = {"hbm_gbs": 6491.8, "bf16_tflops": 1732.9}
try:
    PEAKS.update(json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                             "MEASURED_PEAKS.json"))))
except Exception:  # noqa: BLE001
    pass

_flush = None


def flush_l2():
    global _flush
    if _flush is None:
        _flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    _flush.zero_()


def timeit(fn, iters=20, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush_l2()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def bench_gemm():
    H, I, QKV, V = 4096, 12288, 6144, 151936
    shapes = []
    max_m = int(os.environ.get("KB_MAX_M", "8192"))
    for m in (16, 64, 128, 256, 384, 512, 1024, 2048, 4096, 8192):
        if m > max_m:
            continue
        shapes += [(m, QKV, H, "qkv"), (m, H, H, "o"), (m, 2 * I, H, "gate_up"), (m, H, I, "down")]
    shapes += [(256, V, H, "lm_head")] + ([(8192, 8192, 8192, "square")] if max_m >= 8192 else [])
    for m, n, k, name in shapes:
        x = (torch.randn(m, k, device="cuda") * 0.1).bfloat16()
        w = (torch.randn(n, k, device="cuda") * 0.1).bfloat16()
        out = torch.empty(m, n, device="cuda", dtype=torch.bfloat16)
        ms = timeit(lambda: sm100.linear(x, w, out=out))
        ms_cublas = timeit(lambda: torch.matmul(x, w.t(), out=out))
        flops = 2.0 * m * n * k
        byts = 2.0 * (m * k + n * k + m * n)
        tf = flops / ms / 1e9
        gbs = byts / ms / 1e6
        roof_ms = max(flops / (PEAKS["bf16_tflops"] * 1e9), byts / (PEAKS["hbm_gbs"] * 1e6))
        print(json.dumps({"kernel": "gemm_bf16", "case": name, "M": m, "N": n, "K": k, "ms": round(ms, 4),
                          "tflops": round(tf, 1), "gbs": round(gbs, 1), "frac_of_measured_roofline": round(roof_ms / ms, 3),
                          "cublas_ms": round(ms_cublas, 4)}), flush=True)


def bench_attn():
    hq, hkv, d, page = 32, 8, 128, 16
    for b, ctx in ((1, 4096), (32, 1024), (256, 512), (256, 1024), (512, 1024)):
        n_pages = b * ((ctx + page - 1) // page) + 1
        shape = ref.kv_cache_shape(n_pages, hkv, d, page)
        kc = torch.randn(shape, device="cuda").bfloat16()
        vc = torch.randn(shape, device="cuda").bfloat16()
        bt = torch.arange(b * (ctx // page), device="cuda", dtype=torch.int32).view(b, -1).contiguous()
        sl = torch.full((b,), ctx, device="cuda", dtype=torch.int32)
        qsl = torch.arange(b + 1, device="cuda", dtype=torch.int32)
        q = torch.randn(b, hq * d, device="cuda").bfloat16()
        out = torch.empty_like(q)
        scale = 1 / math.sqrt(d)
        ms = timeit(lambda: sm100.paged_attention(q, kc, vc, bt, sl, qsl, scale, hq, d, b, b, 1, ctx, out=out))
        byts = 2.0 * b * ctx * hkv * d * 2
        print(json.dumps({"kernel": "attn_decode", "B": b, "ctx": ctx, "ms": round(ms, 4),
                          "gbs": round(byts / ms / 1e6, 1),
                          "frac_of_measured_hbm": round(byts / ms / 1e6 / PEAKS["hbm_gbs"], 3)}), flush=True)
    for b, ql in ((1, 8192), (8, 1024), (16, 512)):
        n_pages = b * (ql // page) + 1
        shape = ref.kv_cache_shape(n_pages, hkv, d, page)
        kc = torch.randn(shape, device="cuda").bfloat16()
        vc = torch.randn(shape, device="cuda").bfloat16()
        bt = torch.arange(b * (ql // page), device="cuda", dtype=torch.int32).view(b, -1).contiguous()
        sl = torch.full((b,), ql, device="cuda", dtype=torch.int32)
        qsl = (torch.arange(b + 1, device="cuda", dtype=torch.int32) * ql).contiguous()
        q = torch.randn(b * ql, hq * d, device="cuda").bfloat16()
        out = torch.empty_like(q)
        scale = 1 / math.sqrt(d)
        flops = 4.0 * b * hq * d * ql * ql / 2
        variants = [("mma.sync", False, 0)]
        if os.environ.get("KB_ATTN_TC", "0") == "1":      # wgmma kernel, both KV tile sizes
            variants += [("wgmma", True, 128), ("wgmma", True, 64)]
        for name, tc, kvt in variants:
            sm100.ATTN_TC, sm100.ATTN_TC_KV = tc, (kvt or 128)
            ms = timeit(lambda: sm100.paged_attention(q, kc, vc, bt, sl, qsl, scale, hq, d, 0, b, ql, ql, out=out),
                        iters=10)
            print(json.dumps({"kernel": "attn_prefill", "impl": name, "kv_tile": kvt, "B": b, "q_len": ql,
                              "ms": round(ms, 4), "tflops": round(flops / ms / 1e9, 1),
                              "frac_of_measured_bf16": round(flops / ms / 1e9 / PEAKS["bf16_tflops"], 3)}), flush=True)
        sm100.ATTN_TC = False


def bench_mla():
    """DeepSeek MLA decode over the latent cache: bytes = latent rows read once per 16-head group."""
    page = 16
    for b, ctx, heads in ((64, 4096, 16), (256, 2048, 16), (32, 4096, 128)):
        n_pages = b * (ctx // page) + 1
        cache = (torch.randn(n_pages, 1, 9, page, 64, device="cuda") * 0.3).bfloat16()
        bt = torch.arange(b * (ctx // page), device="cuda", dtype=torch.int32).view(b, -1).contiguous()
        pos = torch.full((b,), ctx - 1, device="cuda", dtype=torch.int32)
        q = (torch.randn(b, heads, 576, device="cuda") * 0.3).bfloat16()
        ms = timeit(lambda: sm100.mla_attention(q, cache, bt, None, pos, 192 ** -0.5), iters=10)
        groups = (heads + 15) // 16
        byts = 1.0 * b * ctx * 576 * 2 * groups
        flops = 2.0 * b * ctx * heads * (576 + 512)
        print(json.dumps({"kernel": "mla_decode", "B": b, "ctx": ctx, "heads": heads, "ms": round(ms, 4),
                          "gbs_incl_group_rereads": round(byts / ms / 1e6, 1), "tflops": round(flops / ms / 1e9, 1),
                          "unique_latent_gbs": round(byts / groups / ms / 1e6, 1)}), flush=True)


if __name__ == "__main__":
    what = sys.argv[1] if len(sys.argv) > 1 else "all"
    if what in ("gemm", "all"):
        bench_gemm()
    if what in ("attn", "all"):
        bench_attn()
    if what in ("mla", "all"):
        bench_mla()
