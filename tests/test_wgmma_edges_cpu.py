"""The element-wise comparators of tests/test_wgmma_edges_gpu.py have teeth: on the CPU, a float64 result rounded to
bf16 (with and without fp32 summation-order noise) passes, and emulated kernels carrying one known slip each are
rejected. Where the global `_rel_err` limits of tests/test_kernels_gpu.py (6e-3 for the GEMMs, 1e-2 for the FP8 GEMM
and attention) would have accepted the slipped output, the test says so and asserts it: that is the gap the
element-wise bounds close.
"""
import math

import pytest
import torch

from test_attn_tc_model_cpu import emulate_prefill_tc
from test_kernels_gpu import _rel_err
from test_wgmma_edges_gpu import (attn_oracle, attn_report, edge_seqs, fp8_oracle, gemm_oracle, gemm_report,
                                  make_paged_batch, q_view, set_monotone, tc_group_pack)


# ----------------------------------------------------------------------------------------------------------------
# bf16 GEMM
# ----------------------------------------------------------------------------------------------------------------
def _gemm_inputs(m, n, k, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(m, k, generator=g) * 0.5).bfloat16()
    w = (torch.randn(n, k, generator=g) * 0.05).bfloat16()
    b = torch.randn(n, generator=g).bfloat16()
    return x, w, b


def _kblock_partials(x, w, kb=64):
    """fp32 partial products of every 64-wide K block (the last one is the K tail): [ceil(K/64), M, N]."""
    k = x.shape[1]
    return torch.stack([x[:, i:i + kb].float() @ w[:, i:i + kb].float().t() for i in range(0, k, kb)])


def _emulated_gemm(parts, bias, reverse=False):
    """fp32 sum of the K-block partials (in either order), fp32 bias add, bf16 rounding."""
    acc = torch.zeros_like(parts[0])
    for p in (parts.flip(0) if reverse else parts):
        acc = acc + p
    if bias is not None:
        acc = acc + bias.float()
    return acc.bfloat16()


@pytest.mark.parametrize("m,n,k", [(65, 264, 200), (129, 136, 3424), (1, 1032, 8)])
def test_gemm_bound_accepts_correct_results(m, n, k):
    x, w, b = _gemm_inputs(m, n, k, m + n + k)
    y64, bound = gemm_oracle(x, w, b)
    assert gemm_report(y64.bfloat16(), y64, bound) is None
    parts = _kblock_partials(x, w)
    for reverse in (False, True):
        assert gemm_report(_emulated_gemm(parts, b, reverse), y64, bound) is None


def test_gemm_rejects_one_dropped_k_block():
    """One 64-wide K block missing from one 128x128 tile: rejected, and the report names the tile."""
    m, n, k = 256, 4096, 1024
    x, w, b = _gemm_inputs(m, n, k, 1)
    y64, bound = gemm_oracle(x, w, b)
    parts = _kblock_partials(x, w)
    parts[5, 128:256, 1024:1152] = 0
    y = _emulated_gemm(parts, b)
    rep = gemm_report(y, y64, bound)
    assert rep is not None and "tile m1 n8" in rep, rep


def test_gemm_rejects_ignored_k_tail():
    """The last 8-wide K block (K = 3424 = 53 x 64 + 32) dropped everywhere."""
    m, n, k = 64, 1024, 3424
    x, w, b = _gemm_inputs(m, n, k, 2)
    y64, bound = gemm_oracle(x, w, b)
    parts = _kblock_partials(x, w)
    parts[-1] = 0
    assert gemm_report(_emulated_gemm(parts, b), y64, bound) is not None


def test_gemm_rejects_zeroed_columns_of_the_last_partial_n_tile():
    """8 columns of the last, partial N tile zeroed, at a vocabulary-sized N (151936 = 593.5 tiles of 256): the
    global error (about 7e-3) passes the old 1e-2 limit of the attention / SiLU tests."""
    m, n, k = 5, 151936, 64
    x, w, b = _gemm_inputs(m, n, k, 3)
    y64, bound = gemm_oracle(x, w, None)
    y = _emulated_gemm(_kblock_partials(x, w), None)
    y[:, n - 8:] = 0
    rep = gemm_report(y, y64, bound, tile=(128, 256))
    assert rep is not None and "n593" in rep, rep
    assert _rel_err(y, y64) < 1e-2


def test_gemm_rejects_missing_bias_on_the_last_partial_n_tile():
    """No bias on the 8 columns of the last, partial N tile."""
    m, n, k = 64, 8200, 512
    x, w, b = _gemm_inputs(m, n, k, 4)
    y64, bound = gemm_oracle(x, w, b)
    parts = _kblock_partials(x, w)
    y = _emulated_gemm(parts, b)
    y[:, 8192:] = _emulated_gemm(parts[:, :, 8192:], None)
    assert gemm_report(y, y64, bound) is not None


# ----------------------------------------------------------------------------------------------------------------
# FP8 block GEMM
# ----------------------------------------------------------------------------------------------------------------
def _fp8_inputs(m, n, k, seed, spread, rows_per_scale=128):
    """e4m3 activations / weights with fp32 scales; `spread` = max |e| of the 2^e factor of every weight block and
    activation cell (0 = the near-uniform scales of tests/test_kernels_gpu.py)."""
    g = torch.Generator().manual_seed(seed)
    kb = k // 128
    xq = (torch.randn(m, k, generator=g) * 100).clamp(-448, 448).to(torch.float8_e4m3fn)
    wq = (torch.randn(n, k, generator=g) * 100).clamp(-448, 448).to(torch.float8_e4m3fn)
    e_x = torch.randint(-spread, spread + 1, (kb, m), generator=g).double()
    e_w = torch.randint(-spread, spread + 1, ((n + rows_per_scale - 1) // rows_per_scale, kb), generator=g).double()
    xs = (torch.pow(2.0, e_x) * 0.7 / 448 * (1 + 0.01 * torch.rand(kb, m, generator=g))).float()
    ws = (torch.pow(2.0, e_w) * 0.05 / 448 * (1 + 0.01 * torch.rand(e_w.shape, generator=g))).float()
    return xq, xs, wq, ws


def _emulated_fp8(xq, xs, wq, ws, rows_per_scale=128):
    """fp32 per-block partials, promoted in fp32 as acc += part * (a_s * w_s), bf16 rounding."""
    m, k = xq.shape
    n = wq.shape[0]
    sw = ws.repeat_interleave(rows_per_scale, 0)[:n]
    acc = torch.zeros(m, n)
    for j in range(k // 128):
        part = xq[:, 128 * j:128 * (j + 1)].float() @ wq[:, 128 * j:128 * (j + 1)].float().t()
        acc = acc + part * (xs[j].view(m, 1) * sw[:, j].view(1, n))
    return acc.bfloat16()


def test_fp8_bound_accepts_correct_results():
    xq, xs, wq, ws = _fp8_inputs(129, 576, 512, 5, spread=8)
    y64, bound = fp8_oracle(xq, xs, wq, ws)
    assert gemm_report(y64.bfloat16(), y64, bound) is None
    assert gemm_report(_emulated_fp8(xq, xs, wq, ws), y64, bound) is None


def test_fp8_rejects_two_swapped_weight_block_scales():
    """Two weight-block scales of one N block swapped. With near-uniform block scales (the old test's inputs) the
    swap passes the old 1e-2 limit, and no comparator can see it; with 2^e scales it is far off, and the bound
    rejects it."""
    for spread in (0, 8):
        xq, xs, wq, ws = _fp8_inputs(129, 576, 512, 6, spread)
        ws_bad = ws.clone()
        ws_bad[0, 0], ws_bad[0, 1] = ws[0, 1], ws[0, 0]
        y64, bound = fp8_oracle(xq, xs, wq, ws)
        y = _emulated_fp8(xq, xs, wq, ws_bad)
        if spread == 0:
            assert _rel_err(y, y64) < 1e-2
        else:
            assert not 0.5 <= float(ws[0, 0] / ws[0, 1]) <= 2.0
            rep = gemm_report(y, y64, bound)
            assert rep is not None and "n0" in rep, rep


def test_fp8_rejects_gate_scale_used_for_the_up_half():
    """Grouped MoE tile [64 gate | 64 up] with one scale row per 64 weight rows: sw_hi := sw in one tile."""
    xq, xs, wq, ws = _fp8_inputs(128, 256, 256, 7, spread=6, rows_per_scale=64)
    ws[1] = ws[0] * 64                                   # the up half of tile 0 scaled 2^6 above its gate half
    y64, bound = fp8_oracle(xq, xs, wq, ws, w_rows_per_scale=64)
    assert gemm_report(_emulated_fp8(xq, xs, wq, ws, 64), y64, bound) is None
    ws_bad = ws.clone()
    ws_bad[1] = ws[0]
    rep = gemm_report(_emulated_fp8(xq, xs, wq, ws_bad, 64), y64, bound)
    assert rep is not None and "n0" in rep, rep


# ----------------------------------------------------------------------------------------------------------------
# prefill attention (the kernel's algorithm, emulated by tests/test_attn_tc_model_cpu.py)
# ----------------------------------------------------------------------------------------------------------------
def _attn(hq, hkv, d, seqs, nd, monotone=False, kv_tile=64, page=16, mutation=None, seed=0):
    b = make_paged_batch(seqs, hq, hkv, d, page, seed=seed, device="cpu", nd=nd)
    if monotone:
        set_monotone(b)
    q = q_view(b).contiguous()
    scale = 1.0 / math.sqrt(d)
    o64, pv = attn_oracle(q, b["kc"], b["vc"], b["bt"], b["sl"], b["qsl"], hq, d, scale)
    o = emulate_prefill_tc(q, b["kc"], b["vc"], b["bt"], b["sl"], b["qsl"], hq, hkv, d, page, scale, kv_tile,
                           seq_offset=nd, mutation=mutation)
    t0 = int(b["qsl"][nd])                                # the decode rows are not this kernel's
    qsl = b["qsl"][nd:] - t0
    gp = tc_group_pack(hq // hkv)
    rep = attn_report(o[t0:], o64[t0:], pv[t0:], qsl, hq, d, gp)
    return rep, _rel_err(o[t0:], o64[t0:].reshape(o[t0:].shape))


_SEQS = [(0, 1), (40, 1), (0, 200), (130, 129), (64, 70)]


@pytest.mark.parametrize("monotone", [False, True])
def test_attention_bound_accepts_correct_results(monotone):
    """bf16(o64) and the emulated kernel (fp32 S, bf16 P, online softmax) both pass."""
    seqs, nd = edge_seqs(32, 16, kv_tiles=(64,), nd=2)
    b = make_paged_batch(seqs[:14], 8, 2, 64, 16, seed=1, device="cpu", nd=nd)
    if monotone:
        set_monotone(b)
    q = q_view(b)
    o64, pv = attn_oracle(q, b["kc"], b["vc"], b["bt"], b["sl"], b["qsl"], 8, 64, 0.125)
    assert attn_report(o64.reshape(q.shape).bfloat16(), o64, pv, b["qsl"], 8, 64) is None
    rep, _ = _attn(8, 2, 64, _SEQS, 2, monotone=monotone)
    assert rep is None, rep


def test_attention_rejects_causal_leak_in_one_query_tile():
    """The first query tile (32 tokens) of a 1000-token chunk behind 1000 cached keys sees one key past its horizon.
    With random, nearly flat scores each of its rows moves by about 1/1000 of |v|: the old global 1e-2 limit and the
    per-row bound both pass that, which is why the GPU tests use monotone keys. There the leaked key carries the row's
    largest score, and the bound rejects the leak and names the query tile."""
    seqs = [(0, 1), (40, 1), (1000, 1000)]
    rep, old = _attn(8, 2, 64, seqs, 2, mutation="horizon+1")
    assert old < 1e-2
    rep, _ = _attn(8, 2, 64, seqs, 2, monotone=True, mutation="horizon+1")
    assert rep is not None and "query tile 0" in rep, rep


def test_attention_rejects_skipped_alpha_rescale():
    """O not rescaled when the row max moves, with random scores and with monotone keys (the max moves on every KV
    tile)."""
    for monotone in (False, True):
        rep, _ = _attn(8, 2, 64, _SEQS, 2, monotone=monotone, mutation="no_alpha")
        assert rep is not None, rep


def test_attention_rejects_head_base_off_by_one_group():
    """G = 12 (GP = 4, three row blocks per KV head): every block's head base one group too high, so the last block
    of each KV head computes the next KV head's first query heads with the wrong keys."""
    rep, _ = _attn(24, 2, 64, _SEQS, 2, mutation="hbase+1")
    assert rep is not None, rep
