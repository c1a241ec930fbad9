"""ctypes binding to the in-tree sm_90a kernel library.

The library is `gllm_b200/_C/libgllm_b200.so`, built by `gllm_b200.build` with plain
nvcc (`-gencode arch=compute_90a,code=sm_90a`). It exposes a flat C ABI; every entry
point takes raw device pointers plus the CUDA stream handle and returns 0 on success.

On a GPU box a missing library is a hard error (we never silently fall back to PyTorch
on the product path); on a CPU box `available()` is False and callers use the torch
reference ops in `gllm_b200.ops.ref`.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_float, c_int, c_int64, c_uint32, c_uint64, c_void_p
from typing import Optional

import torch

_LIB = None
_LIB_ERR = None

LIB_PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "_C",
                        "libgllm_b200.so")

MAX_PEERS = 8   # kMaxPeers / kMaxTp / kMaxEp in csrc (gemm_bf16.cu, comm/tp_fused.cu, comm/ep_a2a.cu)


class GemmComm(ctypes.Structure):
    """Mirror of `GemmComm` in csrc/gemm/gemm_bf16.cu."""

    _fields_ = [
        ("a_ready", c_void_p),
        ("a_expected", c_void_p),
        ("m_rot", c_int),
        ("rs_world", c_int),
        ("rs_rank", c_int),
        ("rows_per_rank", c_int),
        ("rs_inc", c_uint32),
        ("peer_out", c_void_p * MAX_PEERS),
        ("peer_cnt", c_void_p * MAX_PEERS),
        ("rs_bcast", c_int),
    ]


class ReduceNormArgs(ctypes.Structure):
    """Mirror of `ReduceNormArgs` in csrc/comm/tp_fused.cu."""
    _fields_ = [
        ("stage", c_void_p), ("cnt", c_void_p), ("n_tiles", c_uint32 * MAX_PEERS), ("local_x", c_void_p),
        ("local_ld", c_int64), ("residual", c_void_p), ("residual_in", c_int), ("norm_w", c_void_p),
        ("ag_peers", c_void_p * MAX_PEERS), ("flag_peers", c_void_p * MAX_PEERS), ("unnormed_out", c_void_p),
        ("st", c_void_p), ("parity", c_int), ("ag_idx", c_int), ("tp", c_int), ("rank", c_int),
        ("rows_per_rank", c_int), ("rows_valid", c_int), ("H", c_int), ("eps", c_float), ("T", c_int),
        ("bcast", c_int), ("push_x", c_void_p), ("push_ld", c_int64), ("stage_peers", c_void_p * MAX_PEERS),
        ("cnt_peers", c_void_p * MAX_PEERS),
    ]


class LLArgs(ctypes.Structure):
    """Mirror of `LLArgs` in csrc/comm/tp_fused.cu (one-shot LL all-reduce + add + RMSNorm)."""
    _fields_ = [("x", c_void_p), ("ldx", c_int64), ("residual", c_void_p), ("residual_in", c_int),
                ("norm_w", c_void_p), ("out", c_void_p), ("ll_peers", c_void_p * MAX_PEERS), ("st", c_void_p),
                ("tp", c_int), ("rank", c_int), ("T", c_int), ("H", c_int), ("row_cap", c_int), ("eps", c_float)]


class NvlsArgs(ctypes.Structure):
    """Mirror of `NvlsArgs` in csrc/comm/tp_fused.cu (in-switch multimem all-reduce + add + RMSNorm)."""
    _fields_ = [("x", c_void_p), ("ldx", c_int64), ("residual", c_void_p), ("residual_in", c_int),
                ("norm_w", c_void_p), ("out", c_void_p), ("buf_local", c_void_p), ("buf_mc", c_void_p),
                ("flags_mc", c_void_p), ("flags_local", c_void_p), ("st", c_void_p),
                ("tp", c_int), ("rank", c_int), ("T", c_int), ("H", c_int), ("row_cap", c_int), ("eps", c_float)]


class EpArgs(ctypes.Structure):
    """Mirror of `EpArgs` in csrc/comm/ep_a2a.cu."""
    _fields_ = [("recv_x", c_void_p * MAX_PEERS), ("recv_e", c_void_p * MAX_PEERS),
                ("recv_src", c_void_p * MAX_PEERS), ("ctrl", c_void_p * MAX_PEERS), ("comb", c_void_p * MAX_PEERS),
                ("state", c_void_p), ("ep", c_int), ("rank", c_int), ("experts_per_rank", c_int), ("top_k", c_int),
                ("H", c_int), ("r_max", c_int)]


# Parameter types of every `GLLM_EXPORT int gllm_*(...)` in csrc (each returns an int).
# tests/test_abi_cpu.py holds this table to the C prototypes.
P, I, L, F, U64 = c_void_p, c_int, c_int64, c_float, c_uint64
ABI = {
    "gllm_gemm_bf16": [P, L, P, L, P, L, I, I, I, P, I, I, POINTER(GemmComm), P, L, P, I, P],
    "gllm_gemm_bf16_tiles_covering": [I, I, I, I, I, I, I, L, I],
    "gllm_gemm_tune": [I, I],
    "gllm_gemm_bf16_batched": [P, L, L, P, P, L, L, I, I, I, I, P],
    "gllm_gemm_smallm": [P, L, P, L, P, L, I, I, I, P, I, I, P, L, P, P],
    "gllm_gemm_w4a16": [P, L, P, P, P, I, I, P, L, I, I, I, P, I, P, L, P, L, P],
    "gllm_rmsnorm": [P, P, P, P, P, I, I, L, F, P],
    "gllm_silu_and_mul": [P, P, I, I, L, P],
    "gllm_embedding": [P, P, P, I, I, I, I, P],
    "gllm_gather_rows": [P, P, P, I, I, P],
    "gllm_kv_copy_pages": [P, I, L, P, I, P],
    "gllm_rope_kv_write": [P, L, L, I, P, L, L, I, P, L, L, P, P, P, I, I, I, I, P, P, F, P, P, I, I, I, L, P],
    "gllm_attn_decode": [P, L, P, P, P, L, P, P, P, P, I, I, I, I, I, I, I, I, F, P, P],
    "gllm_attn_prefill": [P, L, P, P, P, L, P, P, P, I, I, I, I, I, I, I, I, F, P],
    "gllm_attn_prefill_tc": [P, L, P, P, P, L, P, P, P, I, I, I, I, I, I, I, I, F, I, P],
    "gllm_mla_attention": [P, P, P, L, P, P, P, P, P, I, I, I, I, I, F, P],
    "gllm_mla_rope_cache": [P, L, L, I, P, P, L, P, L, P, P, P, P, I, I, P],
    "gllm_sample": [P, I, L, P, I, I, P, P, P, P, P, I, P, U64, P, P, I, P, L, P, P, P, P],
    "gllm_mark_seen": [P, I, P, P, I, P],
    "gllm_vp_candidates": [P, I, L, P, I, I, I, I, P, P, P, P, P, I, P, U64, P, I, P, L, P, P, P, P],
    "gllm_vp_final": [P, I, I, I, I, P, P, U64, P, P, P, P, P],
    "gllm_bias_account": [P, L, P, I, P, P, P, P, I, P],
    "gllm_bias_rebuild": [P, L, P, I, I, I, P, P, P, P, P, P, P, P],
    "gllm_logprobs_shard": [P, I, L, I, I, I, P, P, P, I, P],
    "gllm_logprobs_final": [P, I, I, I, P, P],
    "gllm_prompt_logprobs_shard": [P, I, L, I, I, I, P, P, I, P],
    "gllm_moe_topk_softmax": [P, L, P, P, I, I, I, I, P],
    "gllm_moe_grouped_topk": [P, L, P, P, P, I, I, I, I, I, I, I, F, P],
    "gllm_moe_align_gather": [P, P, I, I, I, P, P, I, P, P, L, P, I, P, P],
    "gllm_moe_grouped_gemm": [P, L, P, P, L, I, I, I, I, P, P, I, P, P],
    "gllm_moe_combine": [P, P, P, P, I, I, I, P],
    "gllm_fp8_quant_group": [P, L, P, P, I, I, P],
    "gllm_moe_grouped_gemm_fp8": [P, P, P, P, P, L, I, I, I, I, P, P, I, P],
    "gllm_gemm_fp8_block": [P, P, P, P, P, L, I, I, I, P, P],
    "gllm_fp8_quant_token": [P, L, P, P, P, I, I, P],
    "gllm_gemm_fp8_w8a8": [P, P, P, P, P, L, I, I, I, P, P],
    "gllm_gemm_fp8_smallm": [P, P, P, P, P, L, I, I, I, P, I, P, L, P, P],
    "gllm_lora_shrink": [P, L, P, P, P, I, I, I, P, P, P, I, I, P],
    "gllm_lora_expand_add": [P, L, P, P, L, I, I, I, I, I, I, P, P, P, I, P],
    "gllm_lora_expand_silu_mul": [P, L, P, L, P, P, L, I, I, I, P, P, P, I, P],
    # fused tensor / expert parallelism (parallel/fused.py)
    "gllm_rs_reduce_norm": [POINTER(ReduceNormArgs), P],
    "gllm_push_partial_rows": [P, L, I, I, I, I, P, P, P],
    "gllm_wait_ag_flags": [P, P, I, I, P],
    "gllm_tp_state_bytes": [],
    "gllm_ll_allreduce_norm": [POINTER(LLArgs), P],
    "gllm_nvls_allreduce_norm": [POINTER(NvlsArgs), P],
    "gllm_ep_state_bytes": [],
    "gllm_ep_dispatch": [POINTER(EpArgs), P, L, P, I, P],
    "gllm_ep_row_dest": [POINTER(EpArgs), P, P, I, P],
    "gllm_ep_combine": [POINTER(EpArgs), P, P, I, P],
    # micro-benchmark (benchmarks/tma_stream_bench.py)
    "gllm_bench_tma_stream": [P, L, L, L, I, I, I, I, I, P, P],
}


def _declare(lib):
    for name, argtypes in ABI.items():
        fn = getattr(lib, name, None)
        if fn is None:
            raise RuntimeError(f"{LIB_PATH} has no entry point {name}: the library is stale, rebuild it with "
                               f"`python -m gllm_b200.build`")
        fn.argtypes = argtypes
        fn.restype = c_int


def load():
    global _LIB, _LIB_ERR
    if _LIB is not None:
        return _LIB
    if _LIB_ERR is not None:
        raise _LIB_ERR
    try:
        if not os.path.exists(LIB_PATH):
            # safety net: build in-tree on first use when a toolchain is present (takes about a minute); a box
            # without nvcc gets the loud error — there is no PyTorch fallback on the GPU path
            try:
                from gllm_b200 import build as _build
                _build.build()
            except Exception as be:  # noqa: BLE001
                raise FileNotFoundError(
                    f"{LIB_PATH} not found and the in-tree build failed ({be}) — run `python -m gllm_b200.build` "
                    f"(or __graft_entry__.build())") from be
        lib = ctypes.CDLL(LIB_PATH)
        _declare(lib)
        _LIB = lib
        return lib
    except Exception as e:  # noqa: BLE001
        _LIB_ERR = e
        raise


def available() -> bool:
    """True iff a CUDA device is present (then the library MUST load)."""
    if not torch.cuda.is_available():
        return False
    load()
    return True


def stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def check(rc: int, what: str):
    if rc != 0:
        raise RuntimeError(f"gllm_b200 kernel launch failed: {what} (rc={rc})")


def _p(t: Optional[torch.Tensor]):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


_launch_count = 0


def launches() -> int:
    """Number of kernel launches issued through this module (bench.py `gpu_launches`)."""
    return _launch_count


def _count(n=1):
    global _launch_count
    _launch_count += n


def launch(name: str, *args, n: int = 1):
    """Call entry point `name` with `args` and the current stream, raise on a non-zero return and count `n` kernel
    launches (a front-end that runs several entry points as one block charges the block on its last call)."""
    global _launch_count
    rc = getattr(load(), name)(*args, stream_ptr())
    if rc != 0:
        check(rc, name)
    _launch_count += n
