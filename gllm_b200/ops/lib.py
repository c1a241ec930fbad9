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

import torch

_LIB = None
_LIB_ERR = None

LIB_PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "_C",
                        "libgllm_b200.so")

MAX_PEERS = 8


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


def _declare(lib):
    def sig(name, argtypes, restype=c_int):
        fn = getattr(lib, name, None)
        if fn is None:
            return
        fn.argtypes = argtypes
        fn.restype = restype

    P, I, L, F, U = c_void_p, c_int, c_int64, c_float, c_uint32
    sig("gllm_gemm_bf16", [P, L, P, L, P, L, I, I, I, P, I, I, POINTER(GemmComm), P, L, P, I, P])
    sig("gllm_gemm_bf16_tiles_covering", [I, I, I, I, I, I, I, L, I])
    sig("gllm_gemm_tune", [I, I])
    sig("gllm_gemm_bf16_batched", [P, L, L, P, P, L, L, I, I, I, I, P])
    sig("gllm_gemm_smallm", [P, L, P, L, P, L, I, I, I, P, I, I, P, L, P, P])
    sig("gllm_gemm_w4a16", [P, L, P, P, P, I, I, P, L, I, I, I, P, I, P, L, P, L, P])
    sig("gllm_rmsnorm", [P, P, P, P, P, I, I, L, F, P])
    sig("gllm_silu_and_mul", [P, P, I, I, L, P])
    sig("gllm_embedding", [P, P, P, I, I, I, I, P])
    sig("gllm_gather_rows", [P, P, P, I, I, P])
    sig("gllm_kv_copy_pages", [P, I, L, P, I, P])
    sig("gllm_rope_kv_write",
        [P, L, L, I, P, L, L, I, P, L, L, P, P, P, I, I, I, I, P, P, F, P, P, I, I, I, L, P])
    sig("gllm_attn_decode", [P, L, P, P, P, L, P, P, P, P, I, I, I, I, I, I, I, I, F, P, P])
    sig("gllm_attn_prefill", [P, L, P, P, P, L, P, P, P, I, I, I, I, I, I, I, I, F, P])
    sig("gllm_attn_prefill_tc", [P, L, P, P, P, L, P, P, P, I, I, I, I, I, I, I, I, F, I, P])
    sig("gllm_mla_attention", [P, P, P, L, P, P, P, P, P, I, I, I, I, I, F, P])
    sig("gllm_mla_rope_cache", [P, L, L, I, P, P, L, P, L, P, P, P, P, I, I, P])
    sig("gllm_sample", [P, I, L, P, I, I, P, P, P, P, P, I, P, c_uint64, P, P, I, P, L, P, P, P, P])
    sig("gllm_mark_seen", [P, I, P, P, I, P])
    sig("gllm_vp_candidates", [P, I, L, P, I, I, I, I, P, P, P, P, P, I, P, c_uint64, P, I, P, L, P, P, P, P])
    sig("gllm_vp_final", [P, I, I, I, I, P, P, c_uint64, P, P, P, P, P])
    sig("gllm_bias_account", [P, L, P, I, P, P, P, P, I, P])
    sig("gllm_bias_rebuild", [P, L, P, I, I, I, P, P, P, P, P, P, P, P])
    sig("gllm_logprobs_shard", [P, I, L, I, I, I, P, P, P, I, P])
    sig("gllm_logprobs_final", [P, I, I, I, P, P])
    sig("gllm_prompt_logprobs_shard", [P, I, L, I, I, I, P, P, I, P])
    sig("gllm_moe_topk_softmax", [P, L, P, P, I, I, I, I, P])
    sig("gllm_moe_grouped_topk", [P, L, P, P, P, I, I, I, I, I, I, I, F, P])
    sig("gllm_moe_align_gather", [P, P, I, I, I, P, P, I, P, P, L, P, I, P, P])
    sig("gllm_moe_grouped_gemm", [P, L, P, P, L, I, I, I, I, P, P, I, P, P])
    sig("gllm_moe_combine", [P, P, P, P, I, I, I, P])
    sig("gllm_fp8_quant_group", [P, L, P, P, I, I, P])
    sig("gllm_moe_grouped_gemm_fp8", [P, P, P, P, P, L, I, I, I, I, P, P, I, P])
    sig("gllm_gemm_fp8_block", [P, P, P, P, P, L, I, I, I, P, P])
    sig("gllm_lora_shrink", [P, L, P, P, P, I, I, I, P, P, P, I, I, P])
    sig("gllm_lora_expand_add", [P, L, P, P, L, I, I, I, I, I, I, P, P, P, I, P])
    sig("gllm_lora_expand_silu_mul", [P, L, P, L, P, P, L, I, I, I, P, P, P, I, P])


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
