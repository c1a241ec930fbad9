"""Python front-ends of the hand-written sm_90a kernels (ctypes -> libgllm_b200.so).

Each function validates shapes/dtypes, allocates the output and launches on the current
CUDA stream. No fallback: if the library is missing on a GPU box this raises.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional

import torch

from gllm_b200.ops import lib as _lib
from gllm_b200.ops.lib import GemmComm, check, stream_ptr
from gllm_b200.ops.ref import Int4Weight

_BF16 = torch.bfloat16
NUM_SMS = 132   # H100 SXM


def _p(t: Optional[torch.Tensor]):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


_launch_count = 0


def launches() -> int:
    """Number of kernel launches issued through this module (bench.py `gpu_launches`)."""
    return _launch_count


def _count(n=1):
    global _launch_count
    _launch_count += n


# ----------------------------------------------------------------------------------------------
# GEMM
# ----------------------------------------------------------------------------------------------
_FORCE_BN = int(os.environ.get("GLLM_GEMM_BN", "0"))
_SMALLM_MAX = int(os.environ.get("GLLM_GEMM_SMALLM_MAX", "32"))   # M <= this -> swap-AB split-K kernel
_FORCE_SPLIT = int(os.environ.get("GLLM_GEMM_SPLIT", "0"))
_SMALLM_WS_FLOATS = 24 << 20   # fp32 partial-sum workspace shared by the swap-AB and the split-K kernels
_SPLITK_MAX_TILES = 4096
_smallm_ws = {}


def _smallm_workspace(device):
    ws = _smallm_ws.get(device)
    if ws is None:
        ws = (torch.empty(_SMALLM_WS_FLOATS, dtype=torch.float32, device=device),
              torch.zeros(8192, dtype=torch.int32, device=device),
              torch.zeros(2 * _SPLITK_MAX_TILES, dtype=torch.int32, device=device))
        _smallm_ws[device] = ws
    return ws


def _linear_smallm(x, w, bias, out, silu: bool):
    m, k = x.shape
    n = w.shape[0]
    ws, cnt, _ = _smallm_workspace(x.device)
    L = _lib.load()
    rc = L.gllm_gemm_smallm(_p(x), x.stride(0), _p(w), w.stride(0), _p(out), out.stride(0), m, n, k, _p(bias),
                            1 if silu else 0, _FORCE_SPLIT, _p(ws), ws.numel(), _p(cnt), stream_ptr())
    check(rc, "gemm_smallm")
    _count()
    return out


def linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None,
           out: Optional[torch.Tensor] = None, comm: Optional[GemmComm] = None, epi: int = 0) -> torch.Tensor:
    """y = x @ w.T (+ bias). x [M, K] (row stride arbitrary, unit inner stride), w [N, K], (e4m3, scale_inv) or an
    `Int4Weight`."""
    if isinstance(w, Int4Weight):
        return linear_w4a16(x, w, bias, out=out)
    if isinstance(w, tuple):
        return linear_fp8_block(x, w[0], w[1], bias, out=out)
    assert x.dtype == _BF16 and w.dtype == _BF16, (x.dtype, w.dtype)
    assert x.dim() == 2 and w.dim() == 2 and x.shape[1] == w.shape[1], (x.shape, w.shape)
    assert x.stride(1) == 1 and w.stride(1) == 1
    m, k = x.shape
    n = w.shape[0]
    n_out = n // 2 if epi == 1 else n
    if out is None:
        out = torch.empty(m, n_out, dtype=_BF16, device=x.device)
    else:
        assert out.shape == (m, n_out) and out.stride(1) == 1
    if m == 0:
        return out
    if comm is None and epi == 0 and _FORCE_BN == 0 and (m <= _SMALLM_MAX or (m <= 64 and k >= 8192)):
        return _linear_smallm(x, w, bias, out, False)
    L = _lib.load()
    ws, _, tcnt = _smallm_workspace(x.device)
    rc = L.gllm_gemm_bf16(_p(x), x.stride(0), _p(w), w.stride(0), _p(out), out.stride(0), m, n, k, _p(bias),
                          epi, _FORCE_BN, ctypes.byref(comm) if comm is not None else None, _p(ws),
                          ws.numel() * 4, _p(tcnt), _SPLITK_MAX_TILES, stream_ptr())
    check(rc, "gemm_bf16")
    _count()
    return out


def linear_silu_mul(x: torch.Tensor, w_interleaved: torch.Tensor, out: Optional[torch.Tensor] = None,
                    comm: Optional[GemmComm] = None):
    """Fused gate/up projection + SiLU-gate epilogue; weight rows interleaved per 128
    (see ops.ref.interleave_gate_up): BN=256 tiles == [128 gate | 128 up] (the 128-wide tile is
    SMEM-bandwidth bound: 934 us vs 534 us for the Qwen3-8B gate/up GEMM at M=4096)."""
    assert x.dtype == _BF16 and w_interleaved.dtype == _BF16
    m, k = x.shape
    n = w_interleaved.shape[0]
    if out is None:
        out = torch.empty(m, n // 2, dtype=_BF16, device=x.device)
    if m == 0:
        return out
    if m <= _SMALLM_MAX and _FORCE_BN == 0 and comm is None:
        return _linear_smallm(x, w_interleaved, None, out, True)
    L = _lib.load()
    ws, _, tcnt = _smallm_workspace(x.device)
    rc = L.gllm_gemm_bf16(_p(x), x.stride(0), _p(w_interleaved), w_interleaved.stride(0), _p(out),
                          out.stride(0), m, n, k, None, 1, 256,
                          ctypes.byref(comm) if comm is not None else None, _p(ws), ws.numel() * 4, _p(tcnt),
                          _SPLITK_MAX_TILES, stream_ptr())
    check(rc, "gemm_bf16(silu)")
    _count()
    return out


_W4_FORCE_SPLIT = int(os.environ.get("GLLM_W4_SPLIT", "0"))


def linear_w4a16(x: torch.Tensor, w: Int4Weight, bias: Optional[torch.Tensor] = None,
                 out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """y = x @ W.T (+ bias) with W the de-quantised int4 weight of `w` (csrc/gemm/gemm_w4a16.cu), x bf16 [M, K] (row
    stride a multiple of 8, unit inner stride). Split-K partials use the small-M workspace (allocated before graph
    capture) and are reduced in a fixed order."""
    assert isinstance(w, Int4Weight) and w.packed.dtype == torch.int32 and w.zeros.dtype == torch.uint8
    assert w.scales.dtype in (torch.float16, _BF16) and w.packed.is_contiguous() and w.scales.is_contiguous()
    assert x.dtype == _BF16 and x.dim() == 2 and x.stride(1) == 1 and x.shape[1] == w.in_features, (x.shape,
                                                                                                   w.in_features)
    assert x.data_ptr() % 16 == 0 and x.stride(0) % 8 == 0, "TMA needs 16-byte aligned rows"
    m, k = x.shape
    n = w.out_features
    if out is None:
        out = torch.empty(m, n, dtype=_BF16, device=x.device)
    else:
        assert out.shape == (m, n) and out.stride(1) == 1 and out.dtype == _BF16
    if m == 0:
        return out
    ws, _, tcnt = _smallm_workspace(x.device)
    L = _lib.load()
    rc = L.gllm_gemm_w4a16(_p(x), x.stride(0), _p(w.packed), _p(w.scales), _p(w.zeros),
                           1 if w.scales.dtype == _BF16 else 0, w.group_size, _p(out), out.stride(0), m, n, k,
                           _p(bias), _W4_FORCE_SPLIT, _p(ws), ws.numel(), _p(tcnt), tcnt.numel(), stream_ptr())
    check(rc, "gemm_w4a16")
    _count()
    return out


# ----------------------------------------------------------------------------------------------
# norm / activation / embedding
# ----------------------------------------------------------------------------------------------
def rmsnorm(x: torch.Tensor, w: torch.Tensor, eps: float, residual: Optional[torch.Tensor] = None,
            out: Optional[torch.Tensor] = None, residual_out: Optional[torch.Tensor] = None):
    assert x.dtype == _BF16 and x.dim() == 2 and x.stride(1) == 1
    t, h = x.shape
    if out is None:
        out = torch.empty(t, h, dtype=_BF16, device=x.device)
    if residual is not None:
        assert residual.is_contiguous()
        if residual_out is None:
            residual_out = residual  # in place, like the reference's fused_add_rms_norm
    L = _lib.load()
    rc = L.gllm_rmsnorm(_p(x), _p(residual), _p(w), _p(out), _p(residual_out), t, h, x.stride(0), float(eps),
                        stream_ptr())
    check(rc, "rmsnorm")
    _count()
    return out, residual_out


def silu_and_mul(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    assert x.dtype == _BF16 and x.dim() == 2 and x.stride(1) == 1
    t, two_i = x.shape
    i = two_i // 2
    if out is None:
        out = torch.empty(t, i, dtype=_BF16, device=x.device)
    L = _lib.load()
    check(L.gllm_silu_and_mul(_p(x), _p(out), t, i, x.stride(0), stream_ptr()), "silu_and_mul")
    _count()
    return out


def embedding(ids: torch.Tensor, table: torch.Tensor, vocab_start: int = 0, vocab_end: Optional[int] = None,
              out: Optional[torch.Tensor] = None):
    assert ids.dtype == torch.int32 and table.dtype == _BF16 and table.is_contiguous()
    t = ids.shape[0]
    h = table.shape[1]
    vocab_end = vocab_start + table.shape[0] if vocab_end is None else vocab_end
    if out is None:
        out = torch.empty(t, h, dtype=_BF16, device=table.device)
    L = _lib.load()
    check(L.gllm_embedding(_p(ids), _p(table), _p(out), t, h, vocab_start, vocab_end, stream_ptr()), "embedding")
    _count()
    return out


def gather_rows(src: torch.Tensor, idx: torch.Tensor, out: Optional[torch.Tensor] = None):
    assert src.dtype == _BF16 and src.is_contiguous() and idx.dtype == torch.int32
    n, h = idx.shape[0], src.shape[1]
    if out is None:
        out = torch.empty(n, h, dtype=_BF16, device=src.device)
    L = _lib.load()
    check(L.gllm_gather_rows(_p(src), _p(idx), _p(out), n, h, stream_ptr()), "gather_rows")
    _count()
    return out


# ----------------------------------------------------------------------------------------------
# rope + kv write
# ----------------------------------------------------------------------------------------------
def rope_kv_write(q: torch.Tensor, k: torch.Tensor, v: Optional[torch.Tensor], positions: torch.Tensor,
                  cos_sin: Optional[torch.Tensor], rot_dim: int, neox: bool,
                  q_norm_w: Optional[torch.Tensor], k_norm_w: Optional[torch.Tensor], eps: float,
                  k_cache: Optional[torch.Tensor], v_cache: Optional[torch.Tensor],
                  slots: Optional[torch.Tensor], mrope_section=None):
    """q [T,Hq,D], k [T,Hkv,D], v [T,Hkv,D] strided views (unit inner stride); in place."""
    assert q.dtype == _BF16 and q.stride(2) == 1 and k.stride(2) == 1
    t, hq, d = q.shape
    hkv = k.shape[1]
    if t == 0:
        return
    page_size = k_cache.shape[3] if k_cache is not None else 16
    if cos_sin is not None:
        assert cos_sin.dtype == torch.float32 and cos_sin.is_contiguous()
    assert positions.dtype == torch.int32
    sec0 = sec1 = 0
    pos_stride = 0
    if mrope_section is not None and positions.dim() == 2:
        # chunked [T|H|W] sections (Qwen2.5-VL) or, flagged by a 4th entry "interleaved", THWTHW.. (Qwen3-VL)
        if len(mrope_section) > 3 and mrope_section[3]:
            sec0, sec1 = -int(mrope_section[1]), int(mrope_section[2])
        else:
            sec0, sec1 = int(mrope_section[0]), int(mrope_section[1])
        assert positions.stride(1) == 1
        pos_stride = positions.stride(0)
    elif positions.dim() == 2:
        positions = positions[0]
    L = _lib.load()
    rc = L.gllm_rope_kv_write(
        _p(q), q.stride(0), q.stride(1), hq, _p(k), k.stride(0), k.stride(1), hkv,
        _p(v), v.stride(0) if v is not None else 0, v.stride(1) if v is not None else 0,
        _p(q_norm_w), _p(k_norm_w), _p(cos_sin), d, rot_dim if cos_sin is not None else 0, 1 if neox else 0, t,
        _p(positions), _p(slots), float(eps), _p(k_cache), _p(v_cache), sec0, sec1, page_size, pos_stride,
        stream_ptr())
    check(rc, "rope_kv_write")
    _count()


# ----------------------------------------------------------------------------------------------
# paged attention
# ----------------------------------------------------------------------------------------------
_attn_ws = {}
_FUSED_MERGE = os.environ.get("GLLM_ATTN_FUSED_MERGE", "0") == "1"
# wgmma prefill attention (csrc/attn/prefill_attention_tc.cu) is the default prefill kernel; GLLM_ATTN_TC=0 selects
# the mma.sync kernel, which also serves the shapes outside the wgmma kernel's envelope. ATTN_TC_KV = keys per
# pipeline stage (64 or 128). Module attributes so tests / benches can flip them.
ATTN_TC = os.environ.get("GLLM_ATTN_TC", "1") == "1"
ATTN_TC_KV = int(os.environ.get("GLLM_ATTN_TC_KV", "64"))


def decode_splits(num_seqs: int, num_kv_heads: int, num_q_heads: int, max_seq_len: int) -> int:
    g = num_q_heads // num_kv_heads
    gp = max(d for d in range(1, min(g, 16) + 1) if g % d == 0)
    ctas = num_seqs * num_kv_heads * (g // gp)
    target = 4 * NUM_SMS
    s = max(1, min(16, -(-target // max(ctas, 1))))
    max_tiles = max(1, -(-max_seq_len // 64))
    return max(1, min(s, max_tiles))


_retired = []   # outgrown workspaces stay alive: CUDA graphs captured earlier may still point at them


def _workspace(device, n_floats: int, tag: str) -> torch.Tensor:
    key = (device, tag)
    ws = _attn_ws.get(key)
    if ws is None or ws.numel() < n_floats:
        if ws is not None:
            _retired.append(ws)
        ws = torch.empty(max(n_floats, 1 << 20), dtype=torch.float32, device=device)
        _attn_ws[key] = ws
    return ws


def _split_counters(device, n: int) -> torch.Tensor:
    """Zero-at-rest arrival counters of the split-KV decode kernel (the last split CTA merges in-kernel)."""
    key = (device, "split_cnt")
    c = _attn_ws.get(key)
    if c is None or c.numel() < n:
        if c is not None:
            _retired.append(c)
        c = torch.zeros(max(n, 1 << 16), dtype=torch.int32, device=device)
        _attn_ws[key] = c
    return c


def reserve_attn_workspace(device, max_seqs: int, num_q_heads: int, head_dim: int, max_splits: int = 16):
    """Pre-size the split-KV workspace (call before CUDA-graph capture so pointers stay fixed)."""
    _workspace(device, max_seqs * num_q_heads * max_splits * head_dim, "part_o")
    _workspace(device, max_seqs * num_q_heads * max_splits, "part_lse")
    _split_counters(device, max_seqs * num_q_heads)
    if head_dim == 576:      # MLA latent attention: its own split-KV partials
        _mla_workspace(device, num_q_heads)


def paged_attention(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, block_table: torch.Tensor,
                    seq_lens: torch.Tensor, query_start_loc: torch.Tensor, scale: float, num_q_heads: int,
                    head_dim: int, num_decode_seqs: int, num_seqs: int, max_q_len: int, max_seq_len: int,
                    out: Optional[torch.Tensor] = None, splits: Optional[int] = None) -> torch.Tensor:
    """Mixed batch, decode sequences first (one token each), then prefill chunks.
    q [T, Hq*D] (row stride arbitrary); caches [pages, Hkv, D/64, page, 64]."""
    assert q.dtype == _BF16 and q.stride(1) == 1
    t = q.shape[0]
    hq, d = num_q_heads, head_dim
    pages, hkv, nslab, page_size, w = k_cache.shape
    assert w == 64 and nslab * 64 == d, "sm100 attention needs head_dim % 64 == 0"
    assert block_table.dtype == torch.int32 and seq_lens.dtype == torch.int32
    if out is None:
        out = torch.empty(t, hq * d, dtype=_BF16, device=q.device)
    L = _lib.load()
    st = stream_ptr()
    max_blocks = block_table.shape[1]
    if num_decode_seqs > 0:
        if splits is None:
            splits = decode_splits(num_decode_seqs, hkv, hq, max_seq_len)
        part_o = part_lse = None
        split_cnt = None
        if splits > 1:
            part_o = _workspace(q.device, num_decode_seqs * hq * splits * d, "part_o")
            part_lse = _workspace(q.device, num_decode_seqs * hq * splits, "part_lse")
            if _FUSED_MERGE:   # last split CTA merges in-kernel; measured 4 % slower end to end than the
                split_cnt = _split_counters(q.device, num_decode_seqs * hq)   # PDL-launched merge kernel
        rc = L.gllm_attn_decode(_p(q), q.stride(0), _p(out), _p(k_cache), _p(v_cache), pages, _p(block_table),
                                _p(seq_lens), _p(part_o), _p(part_lse), num_decode_seqs, 0, max_blocks, hq, hkv, d,
                                page_size, splits, float(scale), _p(split_cnt), st)
        check(rc, "attn_decode")
        _count(1 if (splits == 1 or split_cnt is not None) else 2)
    n_prefill = num_seqs - num_decode_seqs
    if n_prefill > 0:
        assert query_start_loc.dtype == torch.int32
        rc = 2
        if ATTN_TC:
            rc = L.gllm_attn_prefill_tc(_p(q), q.stride(0), _p(out), _p(k_cache), _p(v_cache), pages, _p(block_table),
                                        _p(seq_lens), _p(query_start_loc), n_prefill, num_decode_seqs, max_q_len,
                                        max_blocks, hq, hkv, d, page_size, float(scale), ATTN_TC_KV, st)
            if rc != 2:                     # 2 = shape outside the wgmma kernel's envelope -> mma.sync kernel
                check(rc, "attn_prefill_tc")
                _count()
                return out
        rc = L.gllm_attn_prefill(_p(q), q.stride(0), _p(out), _p(k_cache), _p(v_cache), pages, _p(block_table),
                                 _p(seq_lens), _p(query_start_loc), n_prefill, num_decode_seqs, max_q_len,
                                 max_blocks, hq, hkv, d, page_size, float(scale), st)
        check(rc, "attn_prefill")
        _count()
    return out


def gemm_batched(a: torch.Tensor, w: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out[:, b, :] = a[:, b, :] @ w[b].T for every batch entry b, on the wgmma GEMM's batched mode
    (csrc/gemm/gemm_bf16.cu): a [T, B, K] and out [T, B, N] may be strided views (last dim contiguous) — the operand
    is read through a 3-D TMA map and the result written in place, no transposing copies; w [B, N, K] contiguous.
    MLA weight absorption (per-head q_nope·W_UK and out_lat·W_UV) runs on this instead of a cuBLAS bmm."""
    t, b, k = a.shape
    n = w.shape[1]
    assert w.shape == (b, n, k) and w.is_contiguous() and out.shape == (t, b, n)
    assert a.dtype == _BF16 and w.dtype == _BF16 and out.dtype == _BF16
    assert a.stride(2) == 1 and out.stride(2) == 1
    L = _lib.load()
    rc = L.gllm_gemm_bf16_batched(_p(a), a.stride(0), a.stride(1), _p(w), _p(out), out.stride(0), out.stride(1),
                                  t, b, n, k, stream_ptr())
    check(rc, "gemm_bf16_batched")
    _count()
    return out


# ----------------------------------------------------------------------------------------------
# sampling
# ----------------------------------------------------------------------------------------------
def sample(logits: torch.Tensor, temperature=None, top_k=None, top_p=None, rep_penalty=None,
           seen_bits: Optional[torch.Tensor] = None, slot_idx: Optional[torch.Tensor] = None, seed: int = 0,
           step: Optional[torch.Tensor] = None,
           out: Optional[torch.Tensor] = None, out_max: Optional[torch.Tensor] = None,
           vocab_offset: int = 0, bias: Optional[torch.Tensor] = None, bias_slot: Optional[torch.Tensor] = None,
           seeds: Optional[torch.Tensor] = None, seed_pos: Optional[torch.Tensor] = None) -> torch.Tensor:
    """logits [B, V] bf16/fp32; per-row params fp32/int32 tensors or None. seen_bits: uint32/int32
    bitmask [B, ceil(V/32)] of tokens subject to the repetition penalty. bias: fp32 [slots, >= V_full] additive rows
    (frequency / presence penalties, logit_bias) indexed by token id, bias_slot: int32 [B] row of each batch row (-1:
    none). seeds: int64 [B] request seeds, seed_pos: int32 [B] position of the token being produced (-1: unseeded
    row, keyed by `seed` + `step` and the batch row)."""
    assert logits.dim() == 2 and logits.stride(1) == 1
    b, v = logits.shape
    dtype = 0 if logits.dtype == _BF16 else 1
    assert logits.dtype in (_BF16, torch.float32)
    if out is None:
        out = torch.empty(b, dtype=torch.int32, device=logits.device)
    seen_words = seen_bits.shape[1] if seen_bits is not None else 0
    L = _lib.load()
    rc = L.gllm_sample(_p(logits), dtype, logits.stride(0), _p(out), b, v, _p(temperature), _p(top_k), _p(top_p),
                       _p(rep_penalty), _p(seen_bits), seen_words, _p(slot_idx),
                       ctypes.c_uint64(seed & ((1 << 64) - 1)),
                       _p(step), _p(out_max), vocab_offset, *_bias_seed_args(bias, bias_slot, seeds, seed_pos),
                       stream_ptr())
    check(rc, "sample")
    _count()
    return out


def _bias_seed_args(bias, bias_slot, seeds, seed_pos):
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.stride(1) == 1 and bias_slot.dtype == torch.int32
    if seeds is not None:
        assert seeds.dtype == torch.int64 and seed_pos.dtype == torch.int32
    return (_p(bias), bias.stride(0) if bias is not None else 0, _p(bias_slot if bias is not None else None),
            _p(seeds), _p(seed_pos if seeds is not None else None))


def vp_candidates(shard: torch.Tensor, valid: int, v_full: int, c: int, temperature=None, top_k=None, top_p=None,
                  rep_penalty=None, seen_bits: Optional[torch.Tensor] = None,
                  slot_idx: Optional[torch.Tensor] = None, seed: int = 0, step: Optional[torch.Tensor] = None,
                  vocab_offset: int = 0, bias: Optional[torch.Tensor] = None,
                  bias_slot: Optional[torch.Tensor] = None, seeds: Optional[torch.Tensor] = None,
                  seed_pos: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Vocab-parallel sampling, stage 1 (csrc/sample/sampler.cu): this rank's per-row record [B, 2c+4] fp32 — its c
    best candidates (value, token id), (max, sum exp) of the shard, and the shard's race winner for unfiltered rows.
    `valid`: columns of `shard` that are real vocabulary entries (the last rank's shard ends with padding)."""
    assert shard.dim() == 2 and shard.stride(1) == 1 and shard.dtype in (_BF16, torch.float32)
    b = shard.shape[0]
    out = torch.empty(b, 2 * c + 4, dtype=torch.float32, device=shard.device)
    seen_words = seen_bits.shape[1] if seen_bits is not None else 0
    L = _lib.load()
    rc = L.gllm_vp_candidates(_p(shard), 0 if shard.dtype == _BF16 else 1, shard.stride(0), _p(out), b, valid, v_full,
                              c, _p(temperature), _p(top_k), _p(top_p), _p(rep_penalty), _p(seen_bits), seen_words,
                              _p(slot_idx), ctypes.c_uint64(seed & ((1 << 64) - 1)), _p(step), vocab_offset,
                              *_bias_seed_args(bias, bias_slot, seeds, seed_pos), stream_ptr())
    check(rc, "vp_candidates")
    _count()
    return out


def vp_final(gathered: torch.Tensor, c: int, v_full: int, top_k=None, top_p=None, seed: int = 0,
             step: Optional[torch.Tensor] = None, seeds: Optional[torch.Tensor] = None,
             seed_pos: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Vocab-parallel sampling, stage 2: `gathered` [tp, B, 2c+4] (all ranks' stage-1 records) -> tokens [B]."""
    tp, b, w = gathered.shape
    assert w == 2 * c + 4 and gathered.is_contiguous() and gathered.dtype == torch.float32
    out = torch.empty(b, dtype=torch.int32, device=gathered.device)
    L = _lib.load()
    rc = L.gllm_vp_final(_p(gathered), tp, b, c, v_full, _p(top_k), _p(top_p),
                         ctypes.c_uint64(seed & ((1 << 64) - 1)), _p(step), _p(out),
                         *_bias_seed_args(None, None, seeds, seed_pos)[3:], stream_ptr())
    check(rc, "vp_final")
    _count()
    return out


MAX_LOGPROBS = 20


def logprobs_shard(logits: torch.Tensor, valid: int, n: int, tokens: torch.Tensor,
                   rows: Optional[torch.Tensor] = None, vocab_offset: int = 0) -> torch.Tensor:
    """Log-probabilities, stage 1 (csrc/sample/sampler.cu:logprobs_shard_kernel): per requesting row a record
    [E, 2n+3] fp32 — this shard's n largest raw logits and their token ids, the shard's (max, sum exp) and the raw logit
    of the sampled token if this shard holds it. `logits` [B, >= valid] bf16/fp32 (this rank's vocab shard, or the full
    row); `valid` real vocabulary columns; `tokens` int32 [B] sampled tokens; `rows` int32 [E] logits row of each
    requesting row (None: all B rows)."""
    assert logits.dim() == 2 and logits.stride(1) == 1 and logits.dtype in (_BF16, torch.float32)
    assert 0 <= n <= MAX_LOGPROBS and tokens.dtype == torch.int32 and tokens.is_contiguous()
    assert rows is None or (rows.dtype == torch.int32 and rows.is_contiguous())
    e = logits.shape[0] if rows is None else rows.numel()
    out = torch.empty(e, 2 * n + 3, dtype=torch.float32, device=logits.device)
    L = _lib.load()
    rc = L.gllm_logprobs_shard(_p(logits), 0 if logits.dtype == _BF16 else 1, logits.stride(0), e, valid, n, _p(rows),
                               _p(tokens), _p(out), vocab_offset, stream_ptr())
    check(rc, "logprobs_shard")
    _count()
    return out


def prompt_logprobs_shard(logits: torch.Tensor, valid: int, n: int, targets: torch.Tensor, vocab_offset: int = 0,
                          out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Prompt log-probabilities, stage 1 for n in {0, 1} (csrc/sample/sampler.cu:prompt_logprobs_shard_kernel): one
    pass over each row of `logits` [Q, >= valid] bf16/fp32, scored against `targets` int32 [Q]; the same [Q, 2n+3]
    record as `logprobs_shard` (written into `out` when given)."""
    assert logits.dim() == 2 and logits.stride(1) == 1 and logits.dtype in (_BF16, torch.float32)
    assert n in (0, 1) and targets.dtype == torch.int32 and targets.is_contiguous()
    q = logits.shape[0]
    assert targets.numel() == q
    if out is None:
        out = torch.empty(q, 2 * n + 3, dtype=torch.float32, device=logits.device)
    assert out.shape == (q, 2 * n + 3) and out.is_contiguous() and out.dtype == torch.float32
    L = _lib.load()
    rc = L.gllm_prompt_logprobs_shard(_p(logits), 0 if logits.dtype == _BF16 else 1, logits.stride(0), q, valid, n,
                                      _p(targets), _p(out), vocab_offset, stream_ptr())
    check(rc, "prompt_logprobs_shard")
    _count()
    return out


def logprobs_final(gathered: torch.Tensor, n: int) -> torch.Tensor:
    """Log-probabilities, stage 2: `gathered` [tp, E, 2n+3] (every rank's stage-1 records) -> [E, 1 + 2n] fp32: the
    sampled token's log-prob, then n x (token id bit-cast to float, log-prob), largest logit first, ties to the lower
    id; id -1 / -inf past the real vocabulary."""
    tp, e, w = gathered.shape
    assert w == 2 * n + 3 and gathered.is_contiguous() and gathered.dtype == torch.float32
    out = torch.empty(e, 1 + 2 * n, dtype=torch.float32, device=gathered.device)
    L = _lib.load()
    check(L.gllm_logprobs_final(_p(gathered), tp, e, n, _p(out), stream_ptr()), "logprobs_final")
    _count()
    return out


def bias_account(bias: torch.Tensor, out_seen: torch.Tensor, bias_slot: torch.Tensor, tokens: torch.Tensor,
                 freq: torch.Tensor, pres: torch.Tensor):
    """Charge each emitting row's sampled token to its bias row (csrc/sample/sampler.cu:bias_account_kernel):
    bias[slot, tok] -= freq (+ pres the first time), out_seen bit set. bias_slot int32 [E] (-1: no row)."""
    e = bias_slot.numel()
    assert tokens.dtype == torch.int32 and tokens.numel() >= e and bias_slot.dtype == torch.int32
    assert freq.dtype == torch.float32 and pres.dtype == torch.float32 and bias.stride(1) == 1
    L = _lib.load()
    check(L.gllm_bias_account(_p(bias), bias.stride(0), _p(out_seen), out_seen.shape[1], _p(bias_slot), _p(tokens),
                              _p(freq), _p(pres), e, stream_ptr()), "bias_account")
    _count()


def bias_rebuild(bias: torch.Tensor, out_seen: torch.Tensor, v: int, slots: torch.Tensor, pen: torch.Tensor,
                 lb_off: torch.Tensor, lb_ids: torch.Tensor, lb_vals: torch.Tensor, out_off: torch.Tensor,
                 out_toks: torch.Tensor):
    """Rebuild the bias rows of (re)assigned slots (bias_rebuild_kernel): clear, scatter logit_bias, replay the counts
    of the output tokens in order. pen fp32 [R, 2] (frequency, presence); *_off int32 [R + 1] offsets."""
    r = slots.numel()
    for t, dt in ((slots, torch.int32), (pen, torch.float32), (lb_off, torch.int32), (lb_ids, torch.int32),
                  (lb_vals, torch.float32), (out_off, torch.int32), (out_toks, torch.int32)):
        assert t.dtype == dt and t.is_contiguous()
    L = _lib.load()
    check(L.gllm_bias_rebuild(_p(bias), bias.stride(0), _p(out_seen), out_seen.shape[1], v, r, _p(slots), _p(pen),
                              _p(lb_off), _p(lb_ids), _p(lb_vals), _p(out_off), _p(out_toks), stream_ptr()),
          "bias_rebuild")
    _count()


_kv_bases = {}


def kv_copy_pages(tensors, pairs, dummy_page: Optional[int] = None):
    """For every page-major KV-cache tensor of this rank (K and V of each layer, or the MLA latent): page dst := page
    src for each (src, dst) in `pairs`, in one launch (csrc/elemwise/kv_copy.cu). The pairs are checked on the host
    first (`ref.check_copy_pairs`). The device array of layer base pointers is built once per set of tensors."""
    if len(pairs) == 0:
        return
    from gllm_b200.ops.ref import check_copy_pairs
    t0 = tensors[0]
    check_copy_pairs(pairs, t0.shape[0], dummy_page)
    for t in tensors:
        assert t.is_cuda and t.is_contiguous() and t.shape == t0.shape and t.dtype == t0.dtype
        assert t.data_ptr() % 16 == 0
    key = tuple(t.data_ptr() for t in tensors)
    bases = _kv_bases.get(key)
    if bases is None:
        bases = torch.tensor(list(key), dtype=torch.int64).to(t0.device)
        _kv_bases[key] = bases
    # (pinned staging: a copy from pageable memory would make the host wait for the work queued before it)
    host = torch.tensor([[int(s), int(d)] for s, d in pairs], dtype=torch.int32).pin_memory()
    launch_kv_copy_pages(tensors, bases, host.to(t0.device, non_blocking=True))


def launch_kv_copy_pages(tensors, bases: torch.Tensor, dev_pairs: torch.Tensor):
    """The launch alone: `bases` int64 [len(tensors)] and `dev_pairs` int32 [n, 2] already on the device and checked."""
    t0 = tensors[0]
    L = _lib.load()
    check(L.gllm_kv_copy_pages(_p(bases), len(tensors), t0[0].numel() * t0.element_size(), _p(dev_pairs),
                               dev_pairs.shape[0], stream_ptr()), "kv_copy_pages")
    _count()


def mark_seen(seen_bits: torch.Tensor, rows: torch.Tensor, tokens: torch.Tensor):
    assert rows.dtype == torch.int32 and tokens.dtype == torch.int32
    L = _lib.load()
    check(L.gllm_mark_seen(_p(seen_bits), seen_bits.shape[1], _p(rows), _p(tokens), rows.numel(), stream_ptr()),
          "mark_seen")
    _count()


# ----------------------------------------------------------------------------------------------
# fp8 block-scaled GEMM (DeepSeek-V3 / Qwen3-FP8 checkpoints)
# ----------------------------------------------------------------------------------------------
def fp8_quant_group(x: torch.Tensor):
    """bf16 [M, K] -> (e4m3 [M, K], fp32 scales [K/128, M]) — dynamic per-token-group(128) quantisation."""
    assert x.dtype == _BF16 and x.dim() == 2 and x.stride(1) == 1 and x.shape[1] % 128 == 0
    m, k = x.shape
    q = torch.empty(m, k, dtype=torch.float8_e4m3fn, device=x.device)
    s = torch.empty(k // 128, m, dtype=torch.float32, device=x.device)
    L = _lib.load()
    check(L.gllm_fp8_quant_group(_p(x), x.stride(0), _p(q), _p(s), m, k, stream_ptr()), "fp8_quant_group")
    _count()
    return q, s


def linear_fp8_block(x: torch.Tensor, w8: torch.Tensor, w_scale_inv: torch.Tensor,
                     bias: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x bf16 [M,K]; w8 e4m3 [N,K]; w_scale_inv fp32 [ceil(N/128), K/128] -> bf16 [M,N]."""
    assert w8.dtype == torch.float8_e4m3fn and w8.is_contiguous() and w_scale_inv.dtype == torch.float32
    assert w_scale_inv.is_contiguous()
    m, k = x.shape
    n = w8.shape[0]
    if out is None:
        out = torch.empty(m, n, dtype=_BF16, device=x.device)
    if m == 0:
        return out
    xq, xs = fp8_quant_group(x)
    L = _lib.load()
    check(L.gllm_gemm_fp8_block(_p(xq), _p(xs), _p(w8), _p(w_scale_inv), _p(out), out.stride(0), m, n, k, _p(bias),
                                stream_ptr()), "gemm_fp8_block")
    _count()
    return out


# ----------------------------------------------------------------------------------------------
# multi-head latent attention (DeepSeek): absorbed MQA over the paged latent cache
# ----------------------------------------------------------------------------------------------
def mla_splits(tokens: int, heads: int) -> int:
    """KV splits so that a decode batch still fills the machine (one CTA = 16 heads of one token)."""
    ctas = max(1, tokens * ((heads + 15) // 16))
    return max(1, min(16, 296 // ctas))


def _mla_workspace(device, heads: int):
    """Split-KV partials of the MLA kernel, allocated ONCE per device (never re-allocated: CUDA graphs captured
    earlier keep writing to it — a lazily grown buffer was freed under them and a later replay faulted). Capacity:
    a forward splits only while tokens * ceil(heads/16) * splits <= 296 CTAs (`mla_splits`), i.e. at most
    296 * 16 (token, head, split) rows, or 16 splits of one token's heads."""
    key = ("mla_ws", torch.device(device))
    ws = _attn_ws.get(key)
    rows = max(296 * 16, 16 * heads)
    if ws is None or ws[1].numel() < rows:
        assert not (torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()), \
            "reserve_attn_workspace() must run before CUDA-graph capture"
        ws = (torch.empty(rows * 512, dtype=torch.float32, device=device),
              torch.empty(rows, dtype=torch.float32, device=device))
        _attn_ws[key] = ws
    return ws


def mla_rope_cache(q_pe: torch.Tensor, q_full: torch.Tensor, k_pe: torch.Tensor, kv_c: torch.Tensor,
                   cos_sin: torch.Tensor, positions: torch.Tensor, slots: torch.Tensor, cache: torch.Tensor):
    """q_pe [T,H,64] (strided view), q_full [T,H,576] (rope part written), k_pe [T,64], kv_c [T,512];
    latent row -> cache [pages,1,9,page,64] at `slots`."""
    t, h, r = q_pe.shape
    assert r == 64 and q_pe.stride(2) == 1 and k_pe.stride(-1) == 1 and kv_c.stride(1) == 1 and kv_c.shape[1] == 512
    assert q_full.is_contiguous() and q_full.shape == (t, h, 576) and cos_sin.dtype == torch.float32
    if positions.dim() == 2:
        positions = positions[0]
    L = _lib.load()
    check(L.gllm_mla_rope_cache(_p(q_pe), q_pe.stride(0), q_pe.stride(1), h, _p(q_full), _p(k_pe), k_pe.stride(0),
                                _p(kv_c), kv_c.stride(0), _p(cos_sin), _p(positions), _p(slots), _p(cache),
                                cache.shape[3], t, stream_ptr()), "mla_rope_cache")
    _count()


def mla_attention(q_full: torch.Tensor, cache: torch.Tensor, block_table: torch.Tensor,
                  tok_seq: Optional[torch.Tensor], positions: torch.Tensor, scale: float,
                  splits: Optional[int] = None) -> torch.Tensor:
    """q_full [T,H,576] bf16 -> out_lat [T,H,512]; every token attends to keys [0, position]."""
    t, h, d = q_full.shape
    assert d == 576 and q_full.is_contiguous() and q_full.dtype == _BF16
    pages, hkv, nslab, page_size, w = cache.shape
    assert hkv == 1 and nslab == 9 and w == 64
    if positions.dim() == 2:
        positions = positions[0]
    if splits is None:
        splits = mla_splits(t, h)
    out = torch.empty(t, h, 512, dtype=_BF16, device=q_full.device)
    part_o = part_lse = None
    if splits > 1:
        if t * h * splits > max(296 * 16, 16 * h):
            splits = max(1, max(296 * 16, 16 * h) // (t * h))      # caller-forced split beyond the workspace
    if splits > 1:
        part_o, part_lse = _mla_workspace(q_full.device, h)
        assert t * h * splits <= part_lse.numel()
    L = _lib.load()
    check(L.gllm_mla_attention(_p(q_full), _p(out), _p(cache), pages, _p(block_table), _p(tok_seq), _p(positions),
                               _p(part_o), _p(part_lse), t, block_table.shape[1], h, page_size, splits, float(scale),
                               stream_ptr()), "mla_attention")
    _count(2 if splits > 1 else 1)
    return out


# ----------------------------------------------------------------------------------------------
# multi-LoRA (csrc/lora/lora.cu); slots / row_off / rows: the batch CSR (see ops.ref.lora_shrink)
# ----------------------------------------------------------------------------------------------
def lora_k_splits(t: int, k: int, m: int) -> int:
    """K-slices per shrink tile: enough CTAs to spread A over the SMs when few row tiles exist (decode)."""
    tiles = ((m + 63) // 64) * ((t + 63) // 64)
    return max(1, min(k // 128, (2 * NUM_SMS + tiles - 1) // tiles))


def lora_shrink(x: torch.Tensor, A: torch.Tensor, slots: torch.Tensor, row_off: torch.Tensor, rows: torch.Tensor,
                num_groups: int) -> torch.Tensor:
    """U [T, M] fp32 = x [T, K] · A[slot] [M, K]ᵀ per adapter group; 0 for rows without an adapter. `rows` lists every
    one of the T rows. Deterministic: K-sliced partial sums are added in a fixed order."""
    assert x.dtype == _BF16 and A.dtype == _BF16 and A.is_contiguous() and x.stride(1) == 1
    t, k = x.shape
    m = A.shape[1]
    assert rows.shape[0] == t, (rows.shape, t)
    u = torch.empty(t, m, dtype=torch.float32, device=x.device)
    splits = lora_k_splits(t, k, m)
    ws = torch.empty(splits * t * m, dtype=torch.float32, device=x.device) if splits > 1 else None
    L = _lib.load()
    check(L.gllm_lora_shrink(_p(x), x.stride(0), _p(A), _p(u), _p(ws), t, k, m, _p(slots), _p(row_off), _p(rows),
                             num_groups, splits, stream_ptr()), "lora_shrink")
    _count(2 if splits > 1 and num_groups > 0 else 1)
    return u


def lora_expand_add(y: torch.Tensor, u: torch.Tensor, B: torch.Tensor, bounds, slots: torch.Tensor,
                    row_off: torch.Tensor, rows: torch.Tensor, num_groups: int) -> torch.Tensor:
    """y [T, N] += U_m · B_m[slot]ᵀ in place; `bounds` = column offsets of the (up to three) modules, ending at N."""
    assert y.dtype == _BF16 and y.stride(1) == 1 and B.dtype == _BF16 and B.is_contiguous()
    assert u.dtype == torch.float32 and u.stride(1) == 1 and len(bounds) in (2, 3, 4) and bounds[-1] == y.shape[1]
    n, r = B.shape[1], B.shape[2]
    nb = list(bounds[1:-1]) + [n, n]
    L = _lib.load()
    check(L.gllm_lora_expand_add(_p(u), u.stride(0), _p(B), _p(y), y.stride(0), y.shape[0], n, r, nb[0], nb[1],
                                 (len(bounds) - 1) * r, _p(slots), _p(row_off), _p(rows), num_groups, stream_ptr()),
          "lora_expand_add")
    _count()
    return y


def lora_expand_silu_mul(pre: torch.Tensor, u: torch.Tensor, B: torch.Tensor, slots: torch.Tensor,
                         row_off: torch.Tensor, rows: torch.Tensor, num_groups: int) -> torch.Tensor:
    """SiLU(gate + dg) · (up + du) [T, I] from the 128-interleaved gate/up pre-activations pre [T, 2I]."""
    assert pre.dtype == _BF16 and pre.stride(1) == 1 and B.dtype == _BF16 and B.is_contiguous()
    t, two_i = pre.shape
    r = B.shape[2]
    out = torch.empty(t, two_i // 2, dtype=_BF16, device=pre.device)
    L = _lib.load()
    check(L.gllm_lora_expand_silu_mul(_p(pre), pre.stride(0), _p(u), u.stride(0), _p(B), _p(out), out.stride(0), t,
                                      two_i // 2, r, _p(slots), _p(row_off), _p(rows), num_groups, stream_ptr()),
          "lora_expand_silu_mul")
    _count()
    return out


# the MoE front-ends, so that a model module sees one table (sm100_moe imports _count and _p, defined above)
from gllm_b200.ops.sm100_moe import fused_experts, fused_experts_fp8, grouped_topk, topk_softmax  # noqa: E402,F401
