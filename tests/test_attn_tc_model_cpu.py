"""Executable specification of csrc/attn/prefill_attention_tc.cu: the kernel's per-CTA algorithm — grid mapping,
GQA row packing, causal horizon, tile loop, diagonal-tile masking, online softmax with a bf16 P and an O rescaled
only when a row max moved, final normalisation — transcribed line by line into torch and compared with the fp32
oracle (`ops/ref.py`). The kernel itself cannot run on this GPU-less box; this pins down the arithmetic it has to
reproduce, so that on-GPU bring-up only has to deal with the hardware side (descriptors, barriers).
"""
import math

import pytest
import torch

from gllm_b200.ops import ref
from test_kernels_gpu import _make_paged        # the GPU test's paged-input builder (runs on CPU tensors too)

ROWS = 128


def emulate_prefill_tc(q, kc, vc, bt, seq_lens, q_start, hq, hkv, d, page, scale, kv_tile, seq_offset=0,
                       mutation=None):
    """`mutation` injects one known slip, for showing that a comparator rejects it (tests/test_wgmma_edges_cpu.py):
    'horizon+1'  query tile 0 of every sequence sees one key past its causal horizon,
    'no_alpha'   O is not rescaled when a row max moves,
    'hbase+1'    the head base of every row block is one group too high (wrapping into the next KV head's heads)."""
    assert mutation in (None, "horizon+1", "no_alpha", "hbase+1"), mutation
    t = q.shape[0]
    out = torch.zeros(t, hq, d)
    qf = q.view(t, hq, d).float()
    g_all = hq // hkv
    gp = next(x for x in range(min(g_all, ROWS), 0, -1) if g_all % x == 0 and ROWS % x == 0)
    scale_log2 = scale * 1.4426950408889634
    toks_per_tile = ROWS // gp
    num_seqs = seq_lens.shape[0] - seq_offset
    max_q = int((q_start[1:] - q_start[:-1]).max())
    for by in range(num_seqs):                                              # blockIdx.y
        seq = by + seq_offset
        q_begin, q_len = int(q_start[seq]), int(q_start[seq + 1] - q_start[seq])
        seq_len = int(seq_lens[seq])
        ctx_len = seq_len - q_len
        n_qtiles = (q_len + toks_per_tile - 1) // toks_per_tile
        for bx in range((max_q + toks_per_tile - 1) // toks_per_tile):       # blockIdx.x
            if bx >= n_qtiles:
                continue
            qt = n_qtiles - 1 - bx
            tok_base = qt * toks_per_tile
            last_tok = min(tok_base + toks_per_tile, q_len) - 1
            leak = 1 if mutation == "horizon+1" and qt == 0 else 0
            kv_end = ctx_len + last_tok + 1 + leak
            n_tiles = (kv_end + kv_tile - 1) // kv_tile
            last_page = (seq_len - 1) // page
            for bz in range(hkv * (g_all // gp)):                           # blockIdx.z
                kvh = bz // (g_all // gp)
                hbase = kvh * g_all + (bz % (g_all // gp) + (mutation == "hbase+1")) * gp
                rows = torch.arange(ROWS)
                tok = tok_base + rows // gp
                head = (hbase + rows % gp) % hq
                row_ok = tok < q_len
                qrows = torch.zeros(ROWS, d)
                qrows[row_ok] = qf[q_begin + tok[row_ok], head[row_ok]]
                lim = ctx_len + tok + leak
                m_run = torch.full((ROWS,), -math.inf)
                l_run = torch.zeros(ROWS)
                o = torch.zeros(ROWS, d)
                for tile in range(n_tiles):
                    # producer: pages of this tile, clamped to the last page of the sequence
                    kt, vt = torch.zeros(kv_tile, d), torch.zeros(kv_tile, d)
                    for j in range(kv_tile // page):
                        pi = min(tile * (kv_tile // page) + j, last_page)
                        pg = int(bt[seq, pi])
                        kt[j * page:(j + 1) * page] = kc[pg, kvh].permute(1, 0, 2).reshape(page, d).float()
                        vt[j * page:(j + 1) * page] = vc[pg, kvh].permute(1, 0, 2).reshape(page, d).float()
                    s = qrows @ kt.t()                                       # S = Q K^T (fp32 accumulate)
                    key0 = tile * kv_tile
                    keys = key0 + torch.arange(kv_tile)
                    need_mask = key0 + kv_tile - 1 > ctx_len + tok_base + leak
                    vis = keys.view(1, -1) <= lim.view(-1, 1) if need_mask else torch.ones(ROWS, kv_tile, dtype=torch.bool)
                    mx = torch.where(vis, s, torch.tensor(-math.inf)).max(dim=1).values
                    m_new = torch.maximum(m_run, mx * scale_log2)
                    m_use = torch.where(torch.isinf(m_new) & (m_new < 0), torch.zeros(()), m_new)
                    alpha = torch.exp2(m_run - m_use)
                    m_run = m_new
                    p = torch.exp2(s * scale_log2 - m_use.view(-1, 1))
                    p = torch.where(vis, p, torch.zeros(()))
                    l_run = l_run * alpha + p.sum(dim=1)
                    if tile > 0 and mutation != "no_alpha":
                        o = o * alpha.view(-1, 1)       # (the kernel skips this when every alpha of the warp is 1)
                    o = o + p.bfloat16().float() @ vt                        # P is rounded to bf16 for the MMA
                inv = torch.where(l_run > 0, 1.0 / l_run, torch.zeros(()))
                res = o * inv.view(-1, 1)
                out[q_begin + tok[row_ok], head[row_ok]] = res[row_ok]
    return out.view(t, hq * d)


@pytest.mark.parametrize("kv_tile", [128, 64])
@pytest.mark.parametrize("hq,hkv,d", [(8, 2, 128), (4, 4, 64), (14, 2, 128)])
def test_tc_prefill_algorithm_matches_oracle(hq, hkv, d, kv_tile):
    seq_lens = [7, 130, 40, 300, 129, 64, 257]
    q_lens = [1, 1, 40, 100, 129, 3, 257]
    nd = 2                                                     # two leading decode rows are not this kernel's job
    q, kc, vc, bt, sl, qsl = _make_paged(seq_lens, q_lens, hq, hkv, d, 16, "cpu", seed=1)
    scale = 1.0 / math.sqrt(d)
    want = ref.paged_attention(q, kc, vc, bt, sl, qsl, scale, hq, d).float()
    got = emulate_prefill_tc(q, kc, vc, bt, sl, qsl, hq, hkv, d, 16, scale, kv_tile, seq_offset=nd)
    t0 = int(qsl[nd])
    err = (got[t0:] - want[t0:]).norm() / want[t0:].norm()
    assert torch.isfinite(got).all() and err < 1e-2, float(err)
