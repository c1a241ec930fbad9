"""The comparators of tests/test_decode_edges_gpu.py have teeth: on the CPU, small torch emulations of the split-KV
decode kernel (+ LSE merge), the MLA latent kernel and the NeoX RoPE lane shuffle pass unmutated, and each known slip
(wrong head-group base, a dropped KV tile, an empty split's -inf LSE read as 0, a warp-local softmax max, a rotary
partner one lane off, one key read past seq_len) is rejected.
"""
import math

import pytest
import torch

from gllm_b200.ops import ref
from test_decode_edges_gpu import (MLA_SCALE, decode_gp, elem_report, make_mla_batch, mla_oracle, mla_report,
                                   rope_oracle, set_mla_monotone)
from test_wgmma_edges_gpu import attn_oracle, attn_report, make_paged_batch, q_view, set_monotone

LOG2E = 1.4426950408889634


# ----------------------------------------------------------------------------------------------------------------
# emulated kernels
# ----------------------------------------------------------------------------------------------------------------
def merge_splits(part_o, lse, mutation=None):
    """attn_merge_kernel / the in-kernel merge: softmax of the splits' log2 LSEs; an empty split (LSE -inf) has
    weight 0 ('empty_lse_zero': its -inf read as 0, weight 2^(0 - m))."""
    m = lse.amax(-1, keepdim=True)
    empty = lse == -math.inf
    w = torch.where(empty, torch.zeros_like(lse), torch.exp2(lse - m))
    if mutation == "empty_lse_zero":
        w = torch.where(empty, torch.exp2(-m).expand_as(lse), w)
    return ((w.unsqueeze(-1) * part_o).sum(-2) / w.sum(-1, keepdim=True)).bfloat16()


def emulate_decode(b, splits, scale, mutation=None):
    """attn_decode_kernel's algorithm: one CTA per (KV head x head group, sequence, split); CTA x serves heads
    hbase .. hbase + GP - 1 with hbase = kvh G + (x % groups_per_kv) GP; split s takes 64-key tiles
    [s tps, (s + 1) tps); fp32 scores in the log2 domain, bf16 P, per-split (O / l, LSE). Heads no CTA writes stay
    NaN. Mutations: 'hbase+1' (head-group base one group high), 'drop_tile' (split 0 drops its last tile),
    'past_seq_len' (the key at index seq_len is not masked), 'empty_lse_zero' (see merge_splits)."""
    q, kc, vc, bt, sl = q_view(b), b["kc"], b["vc"], b["bt"], b["sl"]
    hq, hkv, d = b["hq"], b["hkv"], b["d"]
    t = q.shape[0]
    g = hq // hkv
    gp = decode_gp(g)
    gpk = g // gp
    qf = q.float().view(t, hq, d)
    part_o = torch.full((t, hq, splits, d), math.nan)
    lse = torch.full((t, hq, splits), math.nan)
    for seq in range(t):
        n = int(sl[seq])
        n_tiles = -(-n // 64)
        tps = -(-n_tiles // splits)
        lim = n + 1 if mutation == "past_seq_len" else n
        kk = ref.gather_kv(kc, bt[seq], lim).float()
        vv = ref.gather_kv(vc, bt[seq], lim).float()
        for x in range(hkv * gpk):
            kvh = x // gpk
            hbase = kvh * g + (x % gpk + (1 if mutation == "hbase+1" else 0)) * gp
            heads = [h for h in range(hbase, hbase + gp) if h < hq]
            for sp in range(splits):
                tb = min(sp * tps, n_tiles)
                te = min(tb + tps, n_tiles)
                if mutation == "drop_tile" and sp == 0 and te > tb:
                    te -= 1
                k0, k1 = tb * 64, min(te * 64, lim)
                if k1 <= k0:
                    part_o[seq, heads, sp] = 0.0
                    lse[seq, heads, sp] = -math.inf
                    continue
                s = qf[seq, heads] @ kk[k0:k1, kvh].t() * (scale * LOG2E)
                m = s.amax(-1, keepdim=True)
                p = torch.exp2(s - m)
                l_ = p.sum(-1, keepdim=True)
                part_o[seq, heads, sp] = (p.bfloat16().float() @ vv[k0:k1, kvh]) / l_
                lse[seq, heads, sp] = (m + torch.log2(l_)).squeeze(-1)
    if splits == 1:
        return part_o[:, :, 0].bfloat16()
    return merge_splits(part_o, lse, mutation)


def emulate_mla(b, scale, splits, mutation=None):
    """mla_attn_kernel's algorithm: one CTA per (16-head block, token, split); per 64-key tile the four warps score
    16 keys each (fp32, log2 domain), exchange their row maxima so every warp uses the tile max, write bf16 P, and
    warp w accumulates value columns [128 w, 128 w + 128) with its own alpha; per-warp row sums l are added at the
    end. 'no_xwarp_max': each warp keeps its own running max (P of different warps on different scales)."""
    q, cache, bt = b["q"], b["kc"], b["bt"]
    ts, pos = b["tok_seq"].tolist(), b["pos"].tolist()
    t, h, _ = q.shape
    part_o = torch.full((t, h, splits, 512), math.nan)
    lse = torch.full((t, h, splits), math.nan)
    for i in range(t):
        n = pos[i] + 1
        lat = ref.gather_kv(cache, bt[ts[i]], n)[:, 0].float()
        n_tiles = -(-n // 64)
        tps = -(-n_tiles // splits)
        for hb in range(0, h, 16):
            rows = list(range(hb, min(hb + 16, h)))
            r = len(rows)
            qq = q[i, rows].float()
            for sp in range(splits):
                tb = min(sp * tps, n_tiles)
                te = min(tb + tps, n_tiles)
                o = torch.zeros(r, 4, 128)
                m_run = torch.full((4, r), -math.inf)
                l_run = torch.zeros(4, r)
                for tile in range(tb, te):
                    keys = torch.zeros(64, 576)
                    k0, k1 = tile * 64, min(tile * 64 + 64, n)
                    keys[: k1 - k0] = lat[k0:k1]
                    s = qq @ keys.t() * (scale * LOG2E)
                    s[:, k1 - k0:] = -math.inf
                    s = s.view(r, 4, 16)
                    mx = s.amax(-1).t()                                          # [warp, row]
                    m_tile = mx if mutation == "no_xwarp_max" else mx.amax(0, keepdim=True).expand(4, r)
                    m_new = torch.maximum(m_run, m_tile)
                    m_use = torch.where(m_new == -math.inf, torch.zeros_like(m_new), m_new)
                    alpha = torch.exp2(m_run - m_use)
                    m_run = m_new
                    l_run = l_run * alpha
                    p = torch.exp2(s - m_use.t().unsqueeze(-1))                  # keys of warp w use warp w's max
                    l_run = l_run + p.sum(-1).t()
                    pv = p.reshape(r, 64).bfloat16().float() @ keys[:, :512]
                    o = o * alpha.t().unsqueeze(-1) + pv.view(r, 4, 128)
                l_all = l_run.sum(0)
                if te > tb:
                    part_o[i, rows, sp] = o.reshape(r, 512) / l_all.unsqueeze(-1)
                    lse[i, rows, sp] = m_run[0] + torch.log2(l_all)
                else:
                    part_o[i, rows, sp] = 0.0
                    lse[i, rows, sp] = -math.inf
    if splits == 1:
        return part_o[:, :, 0].bfloat16()
    return merge_splits(part_o, lse)


def emulate_rope_neox(x, cos, sin, rot, mutation=None):
    """rope_kv_kernel's NeoX path: D = 32 C, lane L holds elements [L C, L C + C) and takes its partner's values by a
    shuffle from lane L +- (rot / 2) / C; lanes at or past rot keep their values. fp32 math, bf16 output.
    'partner+1': the shuffle source one lane high."""
    t, h, d = x.shape
    c_ = d // 32
    half = rot // 2
    dl = half // c_
    lane = torch.arange(32)
    lo = lane * c_ < half
    src = torch.where(lo, lane + dl, lane - dl) + (1 if mutation == "partner+1" else 0)
    xl = x.float().view(t, h, 32, c_)
    y = xl[:, :, src % 32]
    i = (lane.view(32, 1) * c_ + torch.arange(c_).view(1, c_)) % half                  # [32, C]
    c, s = cos.float()[:, i].unsqueeze(1), sin.float()[:, i].unsqueeze(1)                # [t, 1, 32, C]
    lo_, in_rot = lo.view(32, 1), (lane * c_ < rot).view(32, 1)
    out = torch.where(in_rot, torch.where(lo_, xl * c - y * s, xl * c + y * s), xl)
    return out.reshape(t, h, d).bfloat16()


# ----------------------------------------------------------------------------------------------------------------
# GQA split-KV decode
# ----------------------------------------------------------------------------------------------------------------
LENS = [1, 7, 16, 17, 63, 64, 65, 129, 300]


def _decode(g, splits, monotone=False, mutation=None, lens=LENS, d=64, seed=0):
    hkv = 2
    b = make_paged_batch([(n - 1, 1) for n in lens], g * hkv, hkv, d, 16, seed=seed, device="cpu", nd=len(lens))
    if monotone:
        set_monotone(b)
    scale = 1.0 / math.sqrt(d)
    o64, pv = attn_oracle(q_view(b), b["kc"], b["vc"], b["bt"], b["sl"], b["qsl"], b["hq"], d, scale)
    o = emulate_decode(b, splits, scale, mutation)
    return attn_report(o, o64, pv, b["qsl"], b["hq"], d, decode_gp(g)), (o64, pv, b)


@pytest.mark.parametrize("splits", [1, 3, 16])
@pytest.mark.parametrize("monotone", [False, True])
def test_decode_bound_accepts_correct_results(splits, monotone):
    """G = 20 (two head groups per KV head), empty splits at 16: the emulated kernel and bf16(o64) both pass."""
    rep, (o64, pv, b) = _decode(20, splits, monotone)
    assert rep is None, rep
    assert attn_report(o64.bfloat16(), o64, pv, b["qsl"], b["hq"], b["d"]) is None


@pytest.mark.parametrize("g", [20, 24, 32])
def test_decode_rejects_head_group_base_off_by_one(g):
    """G > 16: every CTA's head base one group high, so a KV head's last group computes the next KV head's heads
    with the wrong keys and the first group's heads are never written."""
    rep, _ = _decode(g, 1, mutation="hbase+1")
    assert rep is not None and "head 0" in rep, rep


@pytest.mark.parametrize("monotone", [False, True])
def test_decode_rejects_dropped_split_tile(monotone):
    """Split 0 of every sequence drops its last 64-key tile (with random scores too)."""
    rep, _ = _decode(8, 3, monotone, mutation="drop_tile")
    assert rep is not None, rep


def test_decode_rejects_empty_split_lse_read_as_zero():
    """Short sequences across 16 splits: 15 empty splits whose -inf LSE, read as 0, dilutes the one real split."""
    rep, _ = _decode(8, 16, mutation="empty_lse_zero")
    assert rep is not None, rep


def test_decode_rejects_one_key_past_seq_len():
    """The key at index seq_len (a POISON slot, on the next page when seq_len is a page multiple) unmasked: with
    monotone keys it carries the row's largest score."""
    rep, _ = _decode(8, 3, True, mutation="past_seq_len")
    assert rep is not None, rep


# ----------------------------------------------------------------------------------------------------------------
# MLA latent attention
# ----------------------------------------------------------------------------------------------------------------
def _mla(splits, monotone=False, mutation=None, h=20, seqs=None):
    seqs = seqs or [(n - 1, 1) for n in (1, 15, 16, 17, 63, 64, 65, 129, 300)]
    b = make_mla_batch(seqs, h, 16, seed=3, device="cpu")
    scale = set_mla_monotone(b) if monotone else MLA_SCALE
    o64, pv = mla_oracle(b["q"], b["kc"], b["bt"], b["tok_seq"], b["pos"], scale)
    o = emulate_mla(b, scale, splits, mutation)
    return mla_report(o, o64, pv, b["tok_seq"], b["pos"]), (o64, pv, b)


@pytest.mark.parametrize("splits", [1, 3])
@pytest.mark.parametrize("monotone", [False, True])
def test_mla_bound_accepts_correct_results(splits, monotone):
    """H = 20 (a partial 16-head block), the emulated kernel and bf16(o64) both pass; a mixed batch too."""
    rep, (o64, pv, b) = _mla(splits, monotone)
    assert rep is None, rep
    assert mla_report(o64.bfloat16(), o64, pv, b["tok_seq"], b["pos"]) is None
    rep, _ = _mla(splits, monotone, seqs=[(0, 1), (63, 1), (0, 65), (64, 30)], h=16)
    assert rep is None, rep


def test_mla_rejects_warp_local_max():
    """Monotone scores put every tile's max in the last warp's keys: a warp that skips the max exchange scales its
    P (and its value columns) differently from the others."""
    rep, _ = _mla(1, True, mutation="no_xwarp_max")
    assert rep is not None, rep


# ----------------------------------------------------------------------------------------------------------------
# NeoX partial rotary
# ----------------------------------------------------------------------------------------------------------------
def _rope(d, rot, mutation=None):
    g = torch.Generator().manual_seed(d + rot)
    t, h = 13, 3
    x = (torch.randn(t, h, d, generator=g) * 2).bfloat16()
    pos = torch.randint(0, 4096, (t,), generator=g)
    cs = ref.build_cos_sin_cache(rot, 4096, 10000.0)[pos]
    cos, sin = cs[:, : rot // 2], cs[:, rot // 2:]
    y64, bound = rope_oracle(x, cos, sin, rot, True)
    return elem_report(emulate_rope_neox(x, cos, sin, rot, mutation), y64, bound), (y64, bound)


@pytest.mark.parametrize("d,rot", [(64, 64), (64, 16), (128, 128), (128, 64), (128, 32), (256, 64)])
def test_rope_bound_accepts_the_lane_shuffle(d, rot):
    rep, (y64, bound) = _rope(d, rot)
    assert rep is None, rep
    assert elem_report(y64.bfloat16(), y64, bound) is None


@pytest.mark.parametrize("d,rot", [(128, 64), (128, 32), (256, 64)])
def test_rope_rejects_partner_one_lane_off(d, rot):
    rep, _ = _rope(d, rot, mutation="partner+1")
    assert rep is not None, rep
