"""MoE front-ends: routing kernels + grouped wgmma expert GEMMs (csrc/moe/, csrc/gemm/).

fused_experts pipeline (reference: gllm/layers/moe/fused_moe_triton/fused_moe.py:768-972):
    align+gather (expert-sorted 128-row tiles) -> grouped GEMM1 with SiLU-gate epilogue
    -> grouped GEMM2 -> combine (routing weights, sum over top-k)
No host synchronisation anywhere: tile counts stay on the device, buffers are sized for the worst
case (T*k + E_local*127 rows), so the block is CUDA-graph capturable.
"""
from __future__ import annotations

from typing import Optional

import torch

from gllm_b200.ops import lib as _lib
from gllm_b200.ops.lib import check, stream_ptr
from gllm_b200.ops.sm100 import _count, _p

_BF16 = torch.bfloat16
_ws = {}
_retired = []


def _buf(key, shape, dtype, device, zero=False):
    k = (key, device)
    t = _ws.get(k)
    n = 1
    for s in shape:
        n *= s
    if t is None or t.numel() < n or t.dtype != dtype:
        if t is not None:
            _retired.append(t)     # a CUDA graph captured earlier may still point at the outgrown buffer
        t = (torch.zeros if zero else torch.empty)(max(n, 1), dtype=dtype, device=device)
        _ws[k] = t
    return t[:n].view(*shape)


def topk_softmax(logits: torch.Tensor, top_k: int, renormalize: bool):
    assert logits.dtype == _BF16 and logits.stride(1) == 1
    t, e = logits.shape
    w = torch.empty(t, top_k, dtype=torch.float32, device=logits.device)
    ids = torch.empty(t, top_k, dtype=torch.int32, device=logits.device)
    L = _lib.load()
    check(L.gllm_moe_topk_softmax(_p(logits), logits.stride(0), _p(w), _p(ids), t, e, top_k, int(renormalize),
                                  stream_ptr()), "moe_topk_softmax")
    _count()
    return w, ids


def grouped_topk(logits: torch.Tensor, top_k: int, renormalize: bool, n_group: int, topk_group: int,
                 scoring: str = "softmax", bias: Optional[torch.Tensor] = None, routed_scaling: float = 1.0):
    assert logits.dtype == _BF16 and logits.stride(1) == 1
    t, e = logits.shape
    w = torch.empty(t, top_k, dtype=torch.float32, device=logits.device)
    ids = torch.empty(t, top_k, dtype=torch.int32, device=logits.device)
    if bias is not None:
        assert bias.dtype == torch.float32
    L = _lib.load()
    check(L.gllm_moe_grouped_topk(_p(logits), logits.stride(0), _p(bias), _p(w), _p(ids), t, e, top_k, n_group,
                                  topk_group, int(renormalize), int(scoring == "sigmoid"), float(routed_scaling),
                                  stream_ptr()), "moe_grouped_topk")
    _count()
    return w, ids


def fused_experts(x: torch.Tensor, w13: torch.Tensor, w2: torch.Tensor, topk_w: Optional[torch.Tensor],
                  topk_ids: torch.Tensor, expert_map: Optional[torch.Tensor] = None,
                  out: Optional[torch.Tensor] = None, n_valid: Optional[torch.Tensor] = None,
                  row_dest_fn=None) -> Optional[torch.Tensor]:
    """x [T,H]; w13 [E_local, 2I, H] (gate/up rows interleaved per 64); w2 [E_local, H, I]; ids global.

    `n_valid` (device int32 scalar): only the first n_valid rows of x are live (EP receive pool).
    `row_dest_fn(slot_pos, rows)` -> int64 [rows] device table: GEMM2's epilogue then stores every output
    row straight to that address (peer memory) and the local combine is skipped (returns None)."""
    assert x.dtype == _BF16 and x.stride(1) == 1 and w13.is_contiguous() and w2.is_contiguous()
    t, h = x.shape
    e_local, two_i, _ = w13.shape
    inter = two_i // 2
    assert inter % 64 == 0, "the SiLU-gate epilogue reads gate/up rows interleaved per 64"
    k = topk_ids.shape[1]
    dev = x.device
    if out is None and row_dest_fn is None:
        out = torch.empty(t, h, dtype=_BF16, device=dev)
    if t == 0:
        return out
    max_tiles = (t * k + 127) // 128 + e_local
    rows = max_tiles * 128
    meta = _buf("meta", (2 + 3 * e_local + 1,), torch.int32, dev)
    tile_expert = _buf("tile_expert", (max_tiles,), torch.int32, dev)
    slot_pos = _buf("slot_pos", (t * k,), torch.int32, dev)
    xs = _buf("xs", (rows, h), _BF16, dev, zero=True)
    hbuf = _buf("h", (rows, inter), _BF16, dev)
    L = _lib.load()
    st = stream_ptr()
    check(L.gllm_moe_align_gather(_p(topk_ids), _p(expert_map), t, k, e_local, _p(meta), _p(tile_expert), max_tiles,
                                  _p(slot_pos), _p(x), x.stride(0), _p(xs), h, _p(n_valid), st), "moe_align_gather")
    check(L.gllm_moe_grouped_gemm(_p(xs), h, _p(w13), _p(hbuf), inter, max_tiles, two_i, h, e_local,
                                  _p(tile_expert), _p(meta), 1, None, st), "moe_grouped_gemm1")
    if row_dest_fn is not None:
        row_dest = row_dest_fn(slot_pos, rows)
        check(L.gllm_moe_grouped_gemm(_p(hbuf), inter, _p(w2), _p(hbuf), h, max_tiles, h, inter, e_local,
                                      _p(tile_expert), _p(meta), 0, _p(row_dest), st), "moe_grouped_gemm2_push")
        _count(6)
        return None
    ybuf = _buf("y", (rows, h), _BF16, dev)
    check(L.gllm_moe_grouped_gemm(_p(hbuf), inter, _p(w2), _p(ybuf), h, max_tiles, h, inter, e_local,
                                  _p(tile_expert), _p(meta), 0, None, st), "moe_grouped_gemm2")
    check(L.gllm_moe_combine(_p(ybuf), _p(slot_pos), _p(topk_w), _p(out), t, k, h, st), "moe_combine")
    _count(7)
    return out


def fused_experts_fp8(x: torch.Tensor, w13: torch.Tensor, w13_s: torch.Tensor, w2: torch.Tensor, w2_s: torch.Tensor,
                      topk_w: torch.Tensor, topk_ids: torch.Tensor, expert_map: Optional[torch.Tensor] = None,
                      out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Block-scaled fp8 experts (DeepSeek-V3 / Qwen3-FP8 checkpoints; reference: Fp8MoEMethod,
    gllm/layers/moe/fused_moe_triton/layer.py:99-194). w13 [E_local, 2I, H] e4m3 with gate/up rows interleaved
    per 64, w13_s fp32 [E_local, 2I/64, H/128]; w2 [E_local, H, I] e4m3, w2_s [E_local, H/64, I/128].
    align+gather (bf16) -> per-token-group quant -> grouped fp8 GEMM1 (SiLU gate) -> quant -> grouped fp8
    GEMM2 -> combine."""
    assert x.dtype == _BF16 and x.stride(1) == 1 and w13.dtype == torch.float8_e4m3fn
    t, h = x.shape
    e_local, two_i, _ = w13.shape
    inter = two_i // 2
    k = topk_ids.shape[1]
    dev = x.device
    if out is None:
        out = torch.empty(t, h, dtype=_BF16, device=dev)
    if t == 0:
        return out
    max_tiles = (t * k + 127) // 128 + e_local
    rows = max_tiles * 128
    meta = _buf("meta", (2 + 3 * e_local + 1,), torch.int32, dev)
    tile_expert = _buf("tile_expert", (max_tiles,), torch.int32, dev)
    slot_pos = _buf("slot_pos", (t * k,), torch.int32, dev)
    xs = _buf("xs", (rows, h), _BF16, dev, zero=True)
    xs8 = _buf("xs8", (rows, h), torch.uint8, dev)
    xs_s = _buf("xs_s", (h // 128, rows), torch.float32, dev)
    hbuf = _buf("h", (rows, inter), _BF16, dev)
    h8 = _buf("h8", (rows, inter), torch.uint8, dev)
    h_s = _buf("h_s", (inter // 128, rows), torch.float32, dev)
    ybuf = _buf("y", (rows, h), _BF16, dev)
    L = _lib.load()
    st = stream_ptr()
    check(L.gllm_moe_align_gather(_p(topk_ids), _p(expert_map), t, k, e_local, _p(meta), _p(tile_expert), max_tiles,
                                  _p(slot_pos), _p(x), x.stride(0), _p(xs), h, None, st), "moe_align_gather")
    check(L.gllm_fp8_quant_group(_p(xs), h, _p(xs8), _p(xs_s), rows, h, st), "fp8_quant(xs)")
    check(L.gllm_moe_grouped_gemm_fp8(_p(xs8), _p(xs_s), _p(w13), _p(w13_s), _p(hbuf), inter, max_tiles, two_i, h,
                                      e_local, _p(tile_expert), _p(meta), 1, st), "moe_grouped_gemm_fp8(1)")
    check(L.gllm_fp8_quant_group(_p(hbuf), inter, _p(h8), _p(h_s), rows, inter, st), "fp8_quant(h)")
    check(L.gllm_moe_grouped_gemm_fp8(_p(h8), _p(h_s), _p(w2), _p(w2_s), _p(ybuf), h, max_tiles, h, inter, e_local,
                                      _p(tile_expert), _p(meta), 0, st), "moe_grouped_gemm_fp8(2)")
    check(L.gllm_moe_combine(_p(ybuf), _p(slot_pos), _p(topk_w), _p(out), t, k, h, st), "moe_combine")
    _count(9)
    return out
