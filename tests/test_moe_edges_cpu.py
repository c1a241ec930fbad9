"""The MoE comparators of tests/test_moe_edges_gpu.py have teeth: on the CPU, correctly rounded results and emulated
correct kernels pass, and emulated kernels carrying one known slip each are rejected. Where the limits of the older
tests in tests/test_kernels_gpu.py (a dense `allclose` of the routing, a global `_rel_err` of 2e-2 for the whole
block) would have accepted the slipped output, the test says so and asserts it.
"""
import torch

from test_kernels_gpu import _rel_err
from test_moe_edges_gpu import (EDGE_COUNTS, align_oracle, align_report, block_oracle, combine_oracle,
                                grid_logits, grouped_topk_oracle, ids_with_counts, route_report, tie_rows,
                                topk_softmax_oracle)
from test_wgmma_edges_gpu import gemm_report
from gllm_b200.ops import ref


# ----------------------------------------------------------------------------------------------------------------
# routing
# ----------------------------------------------------------------------------------------------------------------
def _vpt(e):
    v = (e + 31) // 32
    return next(x for x in (1, 2, 4, 8, 16) if v <= x)


def port_grouped_topk(logits, bias, k, renorm, n_group, topk_group, scoring, scaling, fixed):
    """Lane-level fp32 port of grouped_topk_kernel: expert e = lane * V + i. fixed=False is the kernel before group
    scoring was made per expert (lanes_per_group = epg / V lanes merge their top-2 with a butterfly and the group of
    lane l is (l V) / epg), fixed=True the per-group full-warp merge."""
    t, e = logits.shape
    v = _vpt(e)
    epg = e // n_group
    lanes = torch.arange(32)
    eid = lanes.view(32, 1) * v + torch.arange(v).view(1, v)
    pad = eid >= e
    ws, ids = torch.zeros(t, k), torch.zeros(t, k, dtype=torch.int32)
    for r in range(t):
        x = torch.full((32, v), -float("inf"))
        x[~pad] = logits[r].float()[eid[~pad]]
        if scoring == "sigmoid":
            sc = torch.where(pad, torch.zeros(()), torch.sigmoid(x))
        else:
            ex = torch.where(pad, torch.zeros(()), torch.exp(x - x.max()))
            sc = ex / ex.sum()
        b = torch.zeros(32, v) if bias is None else torch.where(pad, torch.zeros(()), bias.float()[eid.clamp_max(e - 1)])
        sel = torch.where(pad, torch.full((), -float("inf")), sc + b)
        top2 = sel.sort(-1, descending=True)[0][:, :2] if v > 1 else torch.cat([sel, torch.full((32, 1), -float("inf"))], 1)
        if fixed:
            grp = torch.where(pad, torch.full_like(eid, -1), eid // epg)
            gs = torch.empty(n_group)
            for g in range(n_group):
                s = sel[grp == g].sort(descending=True)[0]
                gs[g] = s[0] + s[1] if bias is not None else s[0]
            better = torch.tensor([int(((gs > gs[g]) | ((gs == gs[g]) & (torch.arange(n_group) < g))).sum())
                                   for g in range(n_group)])
            on = better < topk_group
            ok = ~pad & on[(eid // epg).clamp_max(n_group - 1)]
        else:
            lpg = max(1, epg // v)
            t1, t2 = top2[:, 0].clone(), top2[:, 1].clone()
            o = 1
            while o < lpg:
                o1, o2 = t1[lanes ^ o], t2[lanes ^ o]
                n1 = torch.where(o1 > t1, o1, t1)
                n2 = torch.where(o1 > t1, torch.maximum(t1, o2), torch.maximum(t2, o1))
                t1, t2 = n1, n2
                o <<= 1
            gscore = t1 + t2 if bias is not None else t1
            my_group = lanes * v // epg
            better = torch.zeros(32, dtype=torch.long)
            for g in range(n_group):
                gsv = gscore[(g * epg) // v]
                better += ((gsv > gscore) | ((gsv == gscore) & (g < my_group))).long()
            ok = (lanes.view(32, 1) * v < e) & (better < topk_group).view(32, 1) & ~pad
        key = torch.where(ok, sel, torch.full((), -float("inf"))).flatten()
        flat_sc = sc.flatten()
        for j in range(k):
            best = key.max()
            bi = int(torch.nonzero(key == best)[0])          # equal keys: lower id first
            ids[r, j] = bi
            ws[r, j] = flat_sc[bi]
            key[bi] = -float("inf")
    if renorm:
        ws = ws / (ws.sum(-1, keepdim=True) + 1e-20)
    return ws * scaling, ids


def _dense(ids, w, e):
    return torch.zeros(ids.shape[0], e).scatter(1, ids.long(), w.float())


def _old_routing_allclose(ids, w, ids_r, w_r, e, atol=5e-3, rtol=2e-2):
    """The comparison of tests/test_kernels_gpu.py: routing weights scattered densely by id, allclose."""
    return torch.allclose(_dense(ids, w, e), _dense(ids_r, w_r, e), atol=atol, rtol=rtol)


def test_routing_accepts_correct_results():
    """The oracle's ids with fp32-rounded weights, and the fixed lane-level port, pass on grid, tie and underflow
    rows."""
    g = torch.Generator().manual_seed(0)
    x = torch.cat([grid_logits(64, 160, g), tie_rows(160, 6, 8)])
    orc = grouped_topk_oracle(x, 6, True, 8, 3, "softmax", None, 16.0)
    assert route_report(orc["ids"], orc["weights"](orc["ids"])[0].float(), orc, "oracle") is None
    w, ids = port_grouped_topk(x, None, 6, True, 8, 3, "softmax", 16.0, fixed=True)
    assert route_report(ids, w, orc, "fixed port") is None
    x = torch.cat([grid_logits(64, 128, g), tie_rows(128, 8, 1)])
    orc = topk_softmax_oracle(x, 8, True)
    w = torch.softmax(x.float(), -1).gather(1, orc["ids"])
    assert route_report(orc["ids"], w / w.sum(-1, keepdim=True), orc, "fp32 softmax") is None


def test_routing_rejects_the_old_group_assignment():
    """The kernel before this fix, ported lane by lane: at E = 160 (8 groups of 20, DeepSeek-V2) and E = 96 (4 groups
    of 24) most tokens get another expert set. At E = 256 with 8 groups, the only grouped shape the old test tried,
    the port is exact, so that test could not see it."""
    g = torch.Generator().manual_seed(1)
    for e, k, ng, tg in ((160, 6, 8, 3), (96, 4, 4, 2)):
        x = grid_logits(64, e, g)
        orc = grouped_topk_oracle(x, k, True, ng, tg, "softmax", None, 1.0)
        w, ids = port_grouped_topk(x, None, k, True, ng, tg, "softmax", 1.0, fixed=False)
        rep = route_report(ids, w, orc, f"E={e}")
        assert rep is not None and "chose other experts" in rep, rep
        assert int(rep.split(": ")[1].split(" of")[0]) > 16, rep
    b = grid_logits(1, 256, g)[0].float() / 64
    x = grid_logits(64, 256, g)
    orc = grouped_topk_oracle(x, 8, True, 8, 4, "sigmoid", b, 2.5)
    w, ids = port_grouped_topk(x, b, 8, True, 8, 4, "sigmoid", 2.5, fixed=False)
    assert route_report(ids, w, orc, "E=256") is None


def test_routing_rejects_ties_broken_toward_the_higher_id():
    """A tie inside the top-k taken in the wrong order: the old dense allclose cannot see a reordering (the dense
    scatter is the same), the id comparison rejects it. A tie at the top-k boundary resolved to the higher id is
    rejected as well."""
    x = torch.full((1, 64), -2.0)
    x[0, [7, 40]] = 3.0                                   # tied first place
    x[0, [1, 9, 33]] = 1.0                                # tie across the boundary of K = 4: ids 1, 9 in, 33 out
    x = x.bfloat16()
    orc = topk_softmax_oracle(x, 4, True)
    assert orc["ids"].tolist() == [[7, 40, 1, 9]]
    w_ok = orc["weights"](orc["ids"])[0].float()
    swapped = torch.tensor([[40, 7, 1, 9]])
    w_sw = orc["weights"](swapped)[0].float()
    assert _old_routing_allclose(swapped, w_sw, orc["ids"], w_ok, 64)
    rep = route_report(swapped, w_sw, orc, "swapped tie")
    assert rep is not None and "token 0, slot 0" in rep, rep
    high = torch.tensor([[7, 40, 9, 33]])
    rep = route_report(high, orc["weights"](high)[0].float(), orc, "boundary tie to the higher id")
    assert rep is not None and "slot 2" in rep, rep


def test_routing_rejects_a_weight_off_by_1e_4():
    """A weight 1e-4 relative off (a wrong renorm sum, a dropped exp correction) passes the old allclose
    (rtol 2e-2) and fails the per-element bound."""
    g = torch.Generator().manual_seed(3)
    x = grid_logits(32, 128, g)
    orc = topk_softmax_oracle(x, 8, True)
    w = orc["weights"](orc["ids"])[0].float()
    w_bad = w.clone()
    w_bad[5, 3] *= 1 + 1e-4
    assert _old_routing_allclose(orc["ids"], w_bad, orc["ids"], w, 128)
    rep = route_report(orc["ids"], w_bad, orc, "w")
    assert rep is not None and "worst token 5, slot 3" in rep, rep


# ----------------------------------------------------------------------------------------------------------------
# align + gather
# ----------------------------------------------------------------------------------------------------------------
def emulate_align(ids, expert_map, e_local, x, n_live, slip=None):
    """Python align + gather with the kernel's outputs: meta, tile_expert (-1 past the live tiles), slot_pos (slots
    of an expert in slot order; the kernel's order is arbitrary, any bijection passes), xs (NaN elsewhere)."""
    t, k = ids.shape
    h = x.shape[1]
    loc, counts, off = align_oracle(ids, expert_map, n_live, e_local)
    max_tiles = (t * k + 127) // 128 + e_local
    nt = int(off[-1]) // 128
    meta = torch.cat([torch.tensor([nt, int(off[-1])]), counts, counts, off]).to(torch.int32)
    te = torch.full((max_tiles,), -1, dtype=torch.int32)
    te[:nt] = torch.repeat_interleave(torch.arange(e_local), (off[1:] - off[:-1]) // 128).to(torch.int32)
    pos = torch.full((t * k,), -1, dtype=torch.int32)
    for e in range(e_local):
        s = torch.nonzero(loc == e).flatten()
        pos[s] = (off[e] + torch.arange(s.numel())).to(torch.int32)
    if slip == "slot_pos+1":                 # the last slot of the expert with 129 rows moves to the next row
        e = EDGE_COUNTS.index(129)
        s = int(torch.nonzero(loc == e).flatten()[-1])
        pos[s] += 1
    if slip == "tile_expert+1":
        te[1:nt] = te[:nt - 1].clone()
    xs = torch.full((max_tiles * 128, h), 0x7FC1, dtype=torch.int16).view(torch.bfloat16)
    live = pos >= 0
    xs[pos[live].long()] = x[torch.nonzero(live).flatten() // k]
    return dict(meta=meta, tile_expert=te, slot_pos=pos, xs=xs, max_tiles=max_tiles, k=k)


def _align_case():
    g = torch.Generator().manual_seed(4)
    ids = ids_with_counts(EDGE_COUNTS, 2, g)
    x = (torch.randn(ids.shape[0], 64, generator=g) * 0.5).bfloat16()
    return ids, x


def test_align_accepts_correct_results():
    ids, x = _align_case()
    a = emulate_align(ids, None, len(EDGE_COUNTS), x, ids.numel())
    assert align_report(a, ids, None, len(EDGE_COUNTS), x, ids.numel()) is None
    emap = torch.full((len(EDGE_COUNTS),), -1, dtype=torch.int32)
    emap[::2] = torch.arange(5, dtype=torch.int32)
    a = emulate_align(ids, emap, 5, x, 700)
    assert align_report(a, ids, emap, 5, x, 700) is None


def test_align_rejects_slot_pos_off_by_one_row():
    """One slot one row further down its segment (into the padding): the copy lands there and the real row stays
    empty. Nothing in the older tests checked the align step."""
    ids, x = _align_case()
    a = emulate_align(ids, None, len(EDGE_COUNTS), x, ids.numel(), slip="slot_pos+1")
    rep = align_report(a, ids, None, len(EDGE_COUNTS), x, ids.numel())
    assert rep is not None and "outside its segment" in rep, rep


def test_align_rejects_tile_expert_shifted_by_one_tile():
    ids, x = _align_case()
    a = emulate_align(ids, None, len(EDGE_COUNTS), x, ids.numel(), slip="tile_expert+1")
    rep = align_report(a, ids, None, len(EDGE_COUNTS), x, ids.numel())
    assert rep is not None and "tile_expert[3] = 0, want 2" in rep, rep     # tiles 0..2 hold expert 0's 257 rows


# ----------------------------------------------------------------------------------------------------------------
# combine and the whole block
# ----------------------------------------------------------------------------------------------------------------
def test_combine_rejects_a_dropped_routing_weight():
    g = torch.Generator().manual_seed(5)
    t, k, h = 50, 4, 64
    y = (torch.randn(t * k + 28, h, generator=g)).bfloat16()
    pos = torch.randperm(t * k, generator=g).to(torch.int32)
    pos[3 * k:4 * k] = -1                                   # token 3: every expert remote -> exactly 0
    w = torch.rand(t, k, generator=g) + 0.1
    o64, bound = combine_oracle(y, pos, w, t, k)
    yy = y.float()[pos.long().clamp_min(0)].view(t, k, h) * (pos >= 0).view(t, k, 1)
    good = (w.view(t, k, 1) * yy).sum(1).bfloat16()
    assert gemm_report(good, o64, bound) is None
    assert bool((good[3] == 0).all())
    bad = yy.sum(1).bfloat16()
    assert gemm_report(bad, o64, bound) is not None


def _emulated_block(x, w13, w2, tw, ids, drop_rows_of=None):
    """fp32 fused_experts (bf16 h and y, fp32 combine); drop_rows_of=e zeroes the rows of expert e's last partial
    tile (a kernel that rounds the tile count down)."""
    t, k = ids.shape
    inter = w13.shape[1] // 2
    out = torch.zeros(t, x.shape[1])
    for e in range(w13.shape[0]):
        tok, slot = torch.where(ids.long() == e)
        if tok.numel() == 0:
            continue
        gu = x[tok].float() @ w13[e].float().t()
        hh = (torch.nn.functional.silu(gu[:, :inter]) * gu[:, inter:]).bfloat16()
        y = (hh.float() @ w2[e].float().t()).bfloat16().float()
        if drop_rows_of == e:
            y[tok.numel() // 128 * 128:] = 0
        out.index_add_(0, tok, y * tw[tok, slot].unsqueeze(-1))
    return out.bfloat16()


def test_block_rejects_a_dropped_last_partial_tile():
    """Expert 0 gets 129 slots; a kernel that drops its last, one-row tile loses one slot of one token. The old
    global limit (2e-2 against ref.fused_experts) accepts that; the element-wise block bound names the token."""
    g = torch.Generator().manual_seed(6)
    t, e, k, h, inter = 1000, 64, 6, 256, 128
    logits = torch.randn(t, e, generator=g).bfloat16()
    tw, ids = ref.topk_softmax(logits, k, True)
    flat = ids.flatten().clone()
    n0 = int((flat == 0).sum())
    assert n0 < 129
    flat[torch.nonzero(flat != 0).flatten()[:129 - n0]] = 0     # expert 0 gets exactly 129 slots
    ids = flat.view(t, k)
    x = (torch.randn(t, h, generator=g) * 0.5).bfloat16()
    w13 = (torch.randn(e, 2 * inter, h, generator=g) * 0.05).bfloat16()
    w2 = (torch.randn(e, h, inter, generator=g) * 0.05).bfloat16()
    o64, bound, _, _ = block_oracle(x, w13, w2, tw, ids)
    assert gemm_report(_emulated_block(x, w13, w2, tw, ids), o64, bound) is None
    bad = _emulated_block(x, w13, w2, tw, ids, drop_rows_of=0)
    rep = gemm_report(bad, o64, bound)
    tok = int(torch.where(ids.long() == 0)[0][-1])
    assert rep is not None and f"worst at row {tok}," in rep, rep
    assert _rel_err(bad, ref.fused_experts(x, w13, w2, tw, ids)) < 2e-2
