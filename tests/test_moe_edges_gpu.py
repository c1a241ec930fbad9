"""Element-wise edge tests of the MoE path (csrc/moe/moe_routing.cu, the grouped modes of gemm_bf16.cu and
gemm_fp8_block.cu, ops/sm100_moe.py) against float64 oracles (`pytest -m gpu`, one H100).

Routing ids must equal a float64 oracle that breaks ties the kernel's way (equal keys: lower expert id first; equal
group scores: lower group first), except in rows where two distinct float64 keys lie within the kernel's derived
error of each other; such rows are counted and must be rare. Weights, align metadata, gathered rows, every GEMM
stage, the combine and the whole block are checked element by element against bounds derived from the kernel's
arithmetic (constants below); a failure names the worst token, expert, row or tile.
tests/test_moe_edges_cpu.py shows on emulated kernels that these comparators reject the slips they are meant for.

The oracles and comparators work on CPU tensors too: the CPU module imports them.
"""
import math

import pytest
import torch

from gllm_b200.ops import ref
from test_wgmma_edges_gpu import GEMM_C, U_BF16, U_FP32, _worst, fp8_oracle, gemm_oracle, gemm_report, \
    silu_gate_oracle

pytestmark = pytest.mark.gpu

# ----------------------------------------------------------------------------------------------------------------
# routing error model (the library is built with --use_fast_math)
# ----------------------------------------------------------------------------------------------------------------
# __expf(d): at most 2 + floor(|1.173 d|) ulp (CUDA C++ Programming Guide, table of intrinsic functions). One ulp of
#   a normal fp32 value y is at most 2^-23 |y|. Results below 2^-126 are flushed to zero (-ftz), an absolute error of
#   at most TINY on a value the kernels then divide by a sum >= 1 (softmax) or multiply into a sigmoid <= 1.
ULP_REL = 2.0 ** -23
TINY = 2.0 ** -126
# x / y and 1 / y compile to the approximate division (__fdividef / rcp.approx): at most 2 ulp for the operand
#   ranges here (Programming Guide: 2 ulp for 2^-126 <= |y| <= 2^126).
DIV_REL = 2 * ULP_REL
# The routing bounds below add the first-order relative errors of every rounding step; ROUTE_C = 2 covers the
#   second-order products of those terms (each is below 1e-4, so their products are below 1e-8 of the value) and
#   gives a factor 2 of slack on the __expf figure.
ROUTE_C = 2.0
# An absolute floor for weights whose exact value underflows fp32: w64 < 2^-100 while the kernel gives 0.
W_ABS = 2.0 ** -100


def expf_rel(d):
    """Relative error bound of __expf(d) (see ULP_REL)."""
    return (2.0 + torch.floor(1.173 * d.abs())) * ULP_REL


def _stable_order(key):
    """Expert order by descending key, equal keys in ascending index (the kernels' tie rule)."""
    return torch.sort(-key, dim=-1, stable=True)[1]


def _near_tie(key, kerr, order, n):
    """bool [T]: among sorted positions 0..n, two neighbours differ, but by no more than their error bounds (the
    kernel may order them either way)."""
    n = min(n, key.shape[1] - 1)
    ks, es = key.gather(1, order[:, :n + 1]), kerr.gather(1, order[:, :n + 1])
    diff = ks[:, :-1] - ks[:, 1:]
    return ((diff > 0) & (diff <= es[:, :-1] + es[:, 1:])).any(-1)


def _softmax64(x):
    """float64 softmax of the exact logits and the relative errors of the kernel's exp values and of its fp32 sum:
    v = __expf(x - max) (x - max is exact for bf16 inputs), sum = E fp32 adds of the v (recursive or butterfly
    summation: at most E u of the sum of |terms|) plus the exp errors of its terms."""
    e = x.shape[1]
    d = x - x.max(-1, keepdim=True)[0]
    v = torch.exp(d)
    s = v.sum(-1, keepdim=True)
    rel_v = expf_rel(d) + TINY / v.clamp_min(1e-300)
    rel_s = (v / s * expf_rel(d)).sum(-1, keepdim=True) + e * U_FP32 + e * TINY
    return v / s, v, rel_v, rel_s


def topk_softmax_oracle(logits, k, renorm):
    """float64 oracle of gllm_moe_topk_softmax. Returns dict(ids [T, k] int64, amb bool [T], weights(ids) ->
    (w64, bound)). The kernel ranks v = __expf(x - max); weights are v * (1 / sum) (one approximate reciprocal,
    one multiply), renormalised by w / wsum (K fp32 adds, one approximate division)."""
    x = logits.double()
    p, v, rel_v, rel_s = _softmax64(x)
    order = _stable_order(p)
    kerr = p * rel_v
    rel_w = rel_v + rel_s + DIV_REL + U_FP32

    def weights(ids):
        ids = ids.long()
        w64, rel = p.gather(1, ids), rel_w.gather(1, ids)
        if renorm:
            ws = w64.sum(-1, keepdim=True)
            rel = rel + rel.max(-1, keepdim=True)[0] + k * U_FP32 + DIV_REL
            w64 = w64 / ws
        return w64, ROUTE_C * rel * w64.abs() + W_ABS

    return dict(ids=order[:, :k], amb=_near_tie(p, kerr, order, k), weights=weights, key=p, kerr=kerr)


def grouped_topk_oracle(logits, k, renorm, n_group, topk_group, scoring, bias, scaling):
    """float64 oracle of gllm_moe_grouped_topk with the kernel's tie rules.
    scores: softmax  sc = __expf(x - max) / sum        (exp, sum and one approximate division)
            sigmoid  sc = 1 / (1 + __expf(-x))          (exp of -x, one add, one approximate reciprocal)
    keys sel = sc + bias (one fp32 add); group score = sum of the top-2 keys (bias) or the max key, one more add.
    Weights: sc of the chosen experts, / (wsum + 1e-20) when renormalised (K adds, one division), * scaling."""
    x = logits.double()
    t, e = x.shape
    if scoring == "softmax":
        sc, _, rel_v, rel_s = _softmax64(x)
        rel_sc = rel_v + rel_s + DIV_REL
    else:
        sc = torch.sigmoid(x)
        rel_sc = expf_rel(x) + U_FP32 + DIV_REL
    sel = sc + (bias.double().view(1, e) if bias is not None else 0.0)
    kerr = sc * rel_sc + TINY + U_FP32 * sel.abs()
    epg = e // n_group
    grp, gerr = sel.view(t, n_group, epg), kerr.view(t, n_group, epg)
    o = _stable_order(grp)[:, :, :2]
    top, terr = grp.gather(2, o), gerr.gather(2, o)
    if bias is not None:
        gs = top[:, :, 0] + top[:, :, 1]
        gse = terr[:, :, 0] + terr[:, :, 1] + U_FP32 * gs.abs()
    else:
        gs, gse = top[:, :, 0], terr[:, :, 0]
    gorder = _stable_order(gs)
    tg = min(topk_group, n_group)
    amb = torch.zeros(t, dtype=torch.bool, device=x.device)
    if tg < n_group:
        a, b = gorder[:, tg - 1:tg], gorder[:, tg:tg + 1]
        diff = (gs.gather(1, a) - gs.gather(1, b)).squeeze(1)
        amb |= (diff > 0) & (diff <= (gse.gather(1, a) + gse.gather(1, b)).squeeze(1))
    on = torch.zeros(t, n_group, dtype=torch.bool, device=x.device).scatter(1, gorder[:, :tg], True)
    masked = sel.masked_fill(~on.repeat_interleave(epg, 1), -math.inf)
    order = _stable_order(masked)
    amb |= _near_tie(masked, kerr, order, k)

    def weights(ids):
        ids = ids.long()
        w64, rel = sc.gather(1, ids), rel_sc.gather(1, ids)
        if renorm:
            ws = w64.sum(-1, keepdim=True)
            rel = rel + rel.max(-1, keepdim=True)[0] + k * U_FP32 + DIV_REL + 1e-20 / ws
            w64 = w64 / ws
        return w64 * scaling, ROUTE_C * (rel + U_FP32) * (w64 * scaling).abs() + W_ABS

    return dict(ids=order[:, :k], amb=amb, weights=weights, key=masked, kerr=kerr)


def route_report(ids, w, orc, what, max_amb=0.0):
    """None when the kernel's ids equal the oracle's on every row without a near-tie, near-tie rows are at most a
    max_amb fraction, ids are distinct and in range, and every weight is within its bound; else a message naming the
    worst token and slot."""
    ids, w = ids.cpu().long(), w.cpu()
    want, amb = orc["ids"].cpu(), orc["amb"].cpu()
    t, k = ids.shape
    e = orc["key"].shape[1]
    msgs = []
    bad_rows = torch.nonzero((ids != want).any(-1) & ~amb).flatten()
    if bad_rows.numel():
        r = int(bad_rows[0])
        j = int(torch.nonzero(ids[r] != want[r])[0])
        msgs.append(f"{what}: {bad_rows.numel()} of {t} tokens chose other experts than the oracle; first token {r}, "
                    f"slot {j}: expert {int(ids[r, j])} instead of {int(want[r, j])} (kernel {ids[r].tolist()}, "
                    f"oracle {want[r].tolist()})")
    srt = ids.sort(-1)[0]
    broken = ((ids < 0) | (ids >= e)).any(-1) | (srt[:, 1:] == srt[:, :-1]).any(-1)
    if broken.any():
        r = int(torch.nonzero(broken)[0])
        msgs.append(f"{what}: token {r} has ids out of range or repeated: {ids[r].tolist()}")
    n_amb = int(amb.sum())
    if n_amb > max_amb * t:
        msgs.append(f"{what}: {n_amb} of {t} tokens have near-tied keys (allowed {max_amb * t:.0f})")
    if not broken.any():
        w64, bound = orc["weights"](ids.to(orc["key"].device))
        n_bad, idx = _worst((w.double() - w64.cpu()).abs(), bound.cpu())
        if n_bad:
            r, j = idx
            msgs.append(f"{what}: {n_bad} weights outside the bound; worst token {r}, slot {j} (expert "
                        f"{int(ids[r, j])}): got {float(w[r, j]):.9g}, want {float(w64[r, j]):.9g}, bound "
                        f"{float(bound[r, j]):.3g}")
    return "\n".join(msgs) or None


# ----------------------------------------------------------------------------------------------------------------
# routing inputs
# ----------------------------------------------------------------------------------------------------------------
def grid_logits(t, e, gen):
    """Logits on a 2^-4 grid, |x| <= 8 (exact in bf16): distinct softmax keys differ by e^(1/16) - 1 = 6 %, distinct
    sigmoid keys by at least 2e-5 near |x| = 8, far beyond the derived bounds (about 3e-6 there)."""
    return (torch.randint(-128, 129, (t, e), generator=gen).double() / 16).bfloat16()


def grid_bias(e, gen, period=None):
    """Correction bias on a 2^-6 grid (|b| <= 1/8); `period` repeats the first `period` values."""
    b = torch.randint(-8, 9, (period or e,), generator=gen).float() / 64
    return b.repeat(e // b.numel()) if period else b


def tie_rows(e, k, n_group):
    """Rows with exact ties: a top-k boundary inside a tie of three, duplicated keys inside every group, all groups
    equal (the lower groups win), and underflow (one logit +60, three at +55, the rest -60: under softmax the -60
    experts' scores are 0 in fp32 and the kernel takes them by lowest id)."""
    epg = e // n_group
    rows = []
    r = torch.full((e,), -4.0)
    for j in range(k - 1):
        r[(j * 37 + 5) % e] = 4.0 - j / 16
    tied = [i for i in (e - 1, e // 2 + 1, 1, e // 3) if r[i] == -4.0][:3]
    r[tied] = 2.0
    rows.append(r)
    g = torch.Generator().manual_seed(e + k)
    r = grid_logits(1, e, g)[0].float()
    r.view(n_group, epg)[:, 1] = r.view(n_group, epg)[:, 0]
    rows.append(r)
    r = grid_logits(1, epg, g)[0].float().repeat(n_group)
    rows.append(r)
    r = torch.full((e,), -60.0)
    r[e // 2] = 60.0
    r[[3 % e, (e - 2) % e, (e // 3 + 1) % e]] = 55.0
    rows.append(r)
    return torch.stack(rows).bfloat16()


# (name, E, K, renorm, n_group, topk_group, scoring, bias, scaling); n_group None = topk_softmax
ROUTING = [
    ("mixtral", 8, 2, True, None, None, None, False, 1.0),
    ("qwen1.5-moe", 60, 4, False, None, None, None, False, 1.0),
    ("qwen2-57b", 64, 8, False, None, None, None, False, 1.0),
    ("qwen3-30b-a3b", 128, 8, True, None, None, None, False, 1.0),
    ("e512-k32", 512, 32, True, None, None, None, False, 1.0),
    ("deepseek-v2-lite", 64, 6, False, 1, 1, "softmax", False, 1.0),
    ("deepseek-v2", 160, 6, False, 8, 3, "softmax", False, 16.0),
    ("e96-4-2", 96, 4, True, 4, 2, "softmax", False, 1.0),
    ("deepseek-v3", 256, 8, True, 8, 4, "sigmoid", True, 2.5),
    ("kimi-k2", 384, 8, True, 1, 1, "sigmoid", True, 2.827),
    ("e512-g32", 512, 32, True, 32, 8, "sigmoid", True, 1.0),
]


def _dev():
    return torch.device("cuda:0")


def _route(cfg, logits, bias):
    """Runs the kernel and the oracle on the same logits (any strided view)."""
    from gllm_b200.ops import sm100_moe
    _, e, k, renorm, ng, tg, scoring, _, scaling = cfg
    if ng is None:
        w, ids = sm100_moe.topk_softmax(logits, k, renorm)
        orc = topk_softmax_oracle(logits, k, renorm)
    else:
        w, ids = sm100_moe.grouped_topk(logits, k, renorm, ng, tg, scoring, bias, scaling)
        orc = grouped_topk_oracle(logits, k, renorm, ng, tg, scoring, bias, scaling)
    torch.cuda.synchronize()
    return ids, w, orc


def _routing_inputs(cfg, t, seed, kind):
    name, e, k, _, ng, _, _, use_bias, _ = cfg
    g = torch.Generator().manual_seed(seed)
    if kind == "grid":
        x = grid_logits(t, e, g)
        b = grid_bias(e, g) if use_bias else None
    elif kind == "ties":
        x = tie_rows(e, k, ng or 1)
        b = grid_bias(e, g, period=e // (ng or 1)) if use_bias else None
    else:
        x = torch.randn(t, e, generator=g).bfloat16()
        b = (torch.randn(e, generator=g) * 0.1).float() if use_bias else None
    x = x.to(_dev())
    if e == 60:                       # FusedMoE._router_logits passes a [:, :E] view of a 64-wide buffer
        buf = torch.randn(x.shape[0], 64, device=_dev()).bfloat16()
        buf[:, :60] = x
        x = buf[:, :60]
    return x, (b.to(_dev()) if b is not None else None)


@pytest.mark.parametrize("cfg", ROUTING, ids=[c[0] for c in ROUTING])
def test_routing_grid_logits(cfg):
    """Grid logits (distinct keys far apart, some exactly tied): ids exactly as the oracle's, weights in bound. Under
    sigmoid + bias a sum of two keys (a group score) can still fall within the bound of another: at most 1 % of
    the rows may be near-tied."""
    x, b = _routing_inputs(cfg, 512, cfg[1], "grid")
    ids, w, orc = _route(cfg, x, b)
    rep = route_report(ids, w, orc, f"{cfg[0]} grid", max_amb=0.01)
    assert rep is None, rep


@pytest.mark.parametrize("cfg", ROUTING, ids=[c[0] for c in ROUTING])
def test_routing_exact_ties_and_underflow(cfg):
    """Exact ties at the top-k boundary, inside groups and between whole groups, and underflowed scores."""
    x, b = _routing_inputs(cfg, 0, cfg[1] + 1, "ties")
    ids, w, orc = _route(cfg, x, b)
    rep = route_report(ids, w, orc, f"{cfg[0]} ties")
    assert rep is None, rep


@pytest.mark.parametrize("cfg", ROUTING, ids=[c[0] for c in ROUTING])
def test_routing_random_bf16(cfg):
    """Plain random bf16 logits: either order is accepted only where the float64 keys are within the bound; such
    rows must stay under 2 %."""
    x, b = _routing_inputs(cfg, 1024, cfg[1] + 2, "random")
    ids, w, orc = _route(cfg, x, b)
    rep = route_report(ids, w, orc, f"{cfg[0]} random", max_amb=0.02)
    assert rep is None, rep


@pytest.mark.parametrize("t", [1, 3001])
@pytest.mark.parametrize("name", ["e512-k32", "e512-g32"])
def test_routing_token_extremes(name, t):
    """One token, and enough tokens for hundreds of 8-warp blocks with a partial last block."""
    cfg = next(c for c in ROUTING if c[0] == name)
    x, b = _routing_inputs(cfg, t, t + 100, "grid")
    ids, w, orc = _route(cfg, x, b)
    rep = route_report(ids, w, orc, f"{name} T={t}", max_amb=0.02)
    assert rep is None, rep


def test_routing_rejects_unsupported_shapes():
    """Shapes the routing kernels cannot do return an error before any launch (buffers are large enough that a
    launch could not fault either)."""
    from gllm_b200.ops import lib, sm100
    L = lib.load()
    p = sm100._p
    st = lib.stream_ptr()
    x = torch.zeros(1, 512, dtype=torch.bfloat16, device=_dev())
    w = torch.zeros(1, 64, dtype=torch.float32, device=_dev())
    ids = torch.zeros(1, 64, dtype=torch.int32, device=_dev())
    bias = torch.zeros(512, dtype=torch.float32, device=_dev())
    assert L.gllm_moe_topk_softmax(p(x), 512, p(w), p(ids), 1, 4, 5, 1, st) != 0            # K > E
    assert L.gllm_moe_topk_softmax(p(x), 512, p(w), p(ids), 1, 513, 8, 1, st) != 0          # E > 512
    assert L.gllm_moe_topk_softmax(p(x), 512, p(w), p(ids), 1, 64, 33, 1, st) != 0          # K > 32
    gt = L.gllm_moe_grouped_topk
    assert gt(p(x), 512, p(bias), p(w), p(ids), 1, 4, 5, 1, 1, 1, 1, 1.0, st) != 0          # K > E
    assert gt(p(x), 512, p(bias), p(w), p(ids), 1, 64, 8, 64, 8, 1, 1, 1.0, st) != 0        # 64 groups
    assert gt(p(x), 512, p(bias), p(w), p(ids), 1, 96, 8, 5, 2, 1, 1, 1.0, st) != 0         # E % groups
    assert gt(p(x), 512, p(bias), p(w), p(ids), 1, 64, 8, 8, 0, 1, 1, 1.0, st) != 0         # no group
    assert gt(p(x), 512, p(bias), p(w), p(ids), 1, 64, 9, 8, 1, 1, 1, 1.0, st) != 0         # K > experts in groups
    # and what it can do is accepted (no launch: T = 0 returns first, so the shape check runs for T > 0 only)
    for e, k, ng, tg in ((160, 6, 8, 3), (96, 4, 4, 2), (512, 32, 32, 8), (384, 8, 1, 1), (64, 8, 8, 1)):
        assert gt(p(x), 512, p(bias), p(w), p(ids), 1, e, k, ng, tg, 1, 1, 1.0, st) == 0, (e, ng)
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------------------------
# align + gather
# ----------------------------------------------------------------------------------------------------------------
POISON_BITS = 0x7FC1   # a quiet NaN in bf16: rows the kernel must not write keep exactly these bits


def align_oracle(ids, expert_map, n_live, e_local):
    """Per slot: the local expert (-1 remote or dead), the per-expert counts and the 128-row padded offsets."""
    loc = ids.long().flatten().cpu()
    if expert_map is not None:
        loc = expert_map.long().cpu()[loc]
    live = torch.arange(loc.numel()) < n_live
    loc = torch.where(live & (loc >= 0) & (loc < e_local), loc, torch.full_like(loc, -1))
    counts = torch.bincount(loc[loc >= 0], minlength=e_local)
    off = torch.cat([torch.zeros(1, dtype=torch.long), ((counts + 127) // 128 * 128).cumsum(0)])
    return loc, counts, off


def run_align(ids, expert_map, e_local, x, n_valid=None):
    """gllm_moe_align_gather on test-owned buffers, in the order fused_experts passes them; stale garbage in meta /
    tile_expert / slot_pos and NaN (POISON_BITS) in every xs row."""
    from gllm_b200.ops import lib, sm100
    L = lib.load()
    p = sm100._p
    t, k = ids.shape
    h = x.shape[1]
    max_tiles = (t * k + 127) // 128 + e_local
    dev = x.device
    meta = torch.full((2 + 3 * e_local + 1,), 12345, dtype=torch.int32, device=dev)
    tile_expert = torch.full((max_tiles,), 777, dtype=torch.int32, device=dev)
    slot_pos = torch.full((t * k,), 999999, dtype=torch.int32, device=dev)
    xs = torch.full((max_tiles * 128, h), POISON_BITS, dtype=torch.int16, device=dev).view(torch.bfloat16)
    rc = L.gllm_moe_align_gather(p(ids), p(expert_map), t, k, e_local, p(meta), p(tile_expert), max_tiles,
                                 p(slot_pos), p(x), x.stride(0), p(xs), h, p(n_valid), lib.stream_ptr())
    assert rc == 0
    torch.cuda.synchronize()
    return dict(meta=meta, tile_expert=tile_expert, slot_pos=slot_pos, xs=xs, max_tiles=max_tiles, k=k)


def align_report(a, ids, expert_map, e_local, x, n_live):
    """Exact checks of the align step; None or a message naming the expert, tile or slot."""
    loc, counts, off = align_oracle(ids, expert_map, n_live, e_local)
    meta, te, pos = a["meta"].cpu().long(), a["tile_expert"].cpu().long(), a["slot_pos"].cpu().long()
    k, max_tiles = a["k"], a["max_tiles"]
    e = e_local
    nt = int(off[-1]) // 128
    if int(meta[0]) != nt or int(meta[1]) != int(off[-1]):
        return f"align: num_tiles {int(meta[0])} / rows {int(meta[1])}, want {nt} / {int(off[-1])}"
    for name, got, want in (("count", meta[2:2 + e], counts), ("cursor", meta[2 + e:2 + 2 * e], counts),
                            ("offset", meta[2 + 2 * e:3 + 3 * e], off)):
        if not torch.equal(got, want):
            j = int(torch.nonzero(got != want)[0])
            return f"align: {name} of expert {j} is {int(got[j])}, want {int(want[j])}"
    want_te = torch.full((max_tiles,), -1, dtype=torch.long)
    want_te[:nt] = torch.repeat_interleave(torch.arange(e), (off[1:] - off[:-1]) // 128)
    if not torch.equal(te, want_te):
        j = int(torch.nonzero(te != want_te)[0])
        return f"align: tile_expert[{j}] = {int(te[j])}, want {int(want_te[j])} (live tiles {nt}, max {max_tiles})"
    dead = loc < 0
    if (pos[dead] != -1).any():
        s = int(torch.nonzero(dead & (pos != -1))[0])
        return f"align: slot {s} (remote or dead) has slot_pos {int(pos[s])}, want -1"
    lo, hi = off[loc.clamp_min(0)], off[loc.clamp_min(0)] + counts[loc.clamp_min(0)]
    out = ~dead & ((pos < lo) | (pos >= hi))
    if out.any():
        s = int(torch.nonzero(out)[0])
        return (f"align: slot {s} (expert {int(loc[s])}) at row {int(pos[s])}, outside its segment "
                f"[{int(lo[s])}, {int(hi[s])})")
    live_pos = pos[~dead]
    if live_pos.unique().numel() != live_pos.numel():
        return "align: two live slots share a row"
    xs_bits = a["xs"].view(torch.int16).cpu()
    x_bits = x.contiguous().view(torch.int16).cpu()
    slots = torch.nonzero(~dead).flatten()
    diff = (xs_bits[pos[slots]] != x_bits[slots // k]).any(-1)
    if diff.any():
        s = int(slots[torch.nonzero(diff)[0]])
        return f"align: row {int(pos[s])} (slot {s}, token {s // k}) is not a bitwise copy of x[{s // k}]"
    untouched = torch.ones(xs_bits.shape[0], dtype=torch.bool)
    untouched[live_pos] = False
    if (xs_bits[untouched] != POISON_BITS).any():
        r = int(torch.nonzero((xs_bits != POISON_BITS).any(-1) & untouched)[0])
        return f"align: padding row {r} (tile {r // 128}) was written"
    return None


def ids_with_counts(counts, k, gen):
    """Slot ids [T, k] (T = sum / k) whose local-expert histogram is exactly `counts`, in random slot order."""
    flat = torch.repeat_interleave(torch.arange(len(counts)), torch.tensor(counts))
    assert flat.numel() % k == 0
    flat = flat[torch.randperm(flat.numel(), generator=gen)]
    return flat.view(-1, k).to(torch.int32)


EDGE_COUNTS = [257, 0, 1, 128, 129, 127, 255, 256, 0, 3]


def _x(t, h, gen, ld=None):
    buf = (torch.randn(t, ld or h, generator=gen) * 0.5).bfloat16().to(_dev())
    return buf[:, :h]


@pytest.mark.parametrize("case", ["edge_counts", "one_expert", "e_local_1", "half_remote", "n_valid",
                                  "strided_x"])
def test_align_gather(case):
    """Counts, padded offsets, tile_expert (-1 past the live tiles), slot_pos (a bijection onto each expert's
    segment, -1 for remote / dead slots) and bitwise row copies; rows the kernel should not write keep NaN."""
    g = torch.Generator().manual_seed(len(case))
    emap, n_valid, n_live, ld = None, None, None, None
    h = 1000
    if case == "edge_counts":
        e_local, ids = len(EDGE_COUNTS), ids_with_counts(EDGE_COUNTS, 2, g)
    elif case == "one_expert":
        e_local, ids = 8, torch.full((300, 2), 5, dtype=torch.int32)
    elif case == "e_local_1":
        e_local, ids = 1, torch.zeros(257, 1, dtype=torch.int32)
    elif case == "half_remote":
        # 16 global experts, the odd ones remote; local ids reversed so a missing map lookup is visible
        e_local = 8
        ids = torch.stack([torch.randperm(16, generator=g)[:4] for _ in range(300)]).to(torch.int32)
        emap = torch.full((16,), -1, dtype=torch.int32)
        emap[0::2] = torch.arange(7, -1, -1, dtype=torch.int32)
        emap = emap.to(_dev())
    elif case == "n_valid":
        # only the first 300 of 512 slots are live; the dead ones hold in-range ids of one expert, so a missing
        # n_valid check miscounts instead of faulting
        e_local = 8
        ids = torch.randint(0, 8, (512, 1), generator=g).to(torch.int32)
        ids[300:] = 3
        n_live = 300
        n_valid = torch.tensor([300], dtype=torch.int32, device=_dev())
    else:
        e_local, ids, ld = 8, torch.randint(0, 8, (333, 2), generator=g).to(torch.int32), h + 64
    ids = ids.to(_dev())
    x = _x(ids.shape[0], h, g, ld)
    a = run_align(ids, emap, e_local, x, n_valid)
    rep = align_report(a, ids, emap, e_local, x, ids.numel() if n_live is None else n_live)
    assert rep is None, f"{case}: {rep}"


def test_align_gather_rejects_unsupported_shapes():
    """E_local > 1024 (the offsets kernel's fixed shared array), H % 8 != 0, a misaligned x or row stride (the
    16-byte row copy): an error code, no launch."""
    from gllm_b200.ops import lib, sm100
    L = lib.load()
    p = sm100._p
    st = lib.stream_ptr()
    dev = _dev()
    ids = torch.zeros(4, 1, dtype=torch.int32, device=dev)
    meta = torch.zeros(2 + 3 * 1025 + 1, dtype=torch.int32, device=dev)
    te = torch.zeros(1100, dtype=torch.int32, device=dev)
    sp = torch.zeros(4, dtype=torch.int32, device=dev)
    x = torch.zeros(4, 1040, dtype=torch.bfloat16, device=dev)
    xs = torch.zeros(1100 * 128 * 16, dtype=torch.bfloat16, device=dev)
    f = L.gllm_moe_align_gather
    assert f(p(ids), None, 4, 1, 1025, p(meta), p(te), 1026, p(sp), p(x), 1040, p(xs), 8, None, st) != 0
    assert f(p(ids), None, 4, 1, 8, p(meta), p(te), 9, p(sp), p(x), 1040, p(xs), 1001, None, st) != 0
    assert f(p(ids), None, 4, 1, 8, p(meta), p(te), 9, p(sp), p(x[:, 1:]), 1040, p(xs), 1000, None, st) != 0
    assert f(p(ids), None, 4, 1, 8, p(meta), p(te), 9, p(sp), p(x), 1036, p(xs), 1000, None, st) != 0
    assert f(p(ids), None, 4, 1, 8, p(meta), p(te), 9, p(sp), p(x), 1040, p(xs[1:]), 1000, None, st) != 0
    assert f(p(ids), None, 4, 1, 1024, p(meta), p(te), 1025, p(sp), p(x), 1040, p(xs), 1000, None, st) == 0
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------------------------
# grouped GEMMs and the combine, stage by stage on the kernel's own inputs
# ----------------------------------------------------------------------------------------------------------------
def combine_oracle(y, slot_pos, w, t, k):
    """float64 out[t] = sum_j w[t, j] y[pos[t, j]] on the kernel's bf16 y, and its bound: K fp32 multiply-adds
    (2 K u of sum |w y|, covering an unfused multiply and add per step) plus the bf16 rounding of the result."""
    pos = slot_pos.long().view(t, k)
    yy = y.double()[pos.clamp_min(0)] * (pos >= 0).unsqueeze(-1)
    ww = w.double().view(t, k, 1)
    o64 = (ww * yy).sum(1)
    mag = (ww.abs() * yy.abs()).sum(1)
    return o64, U_BF16 * o64.abs() + 2 * k * U_FP32 * mag


def _weights(e_local, inter, h, gen, fp8=False):
    w13 = torch.randn(e_local, 2 * inter, h, generator=gen) * 0.05
    w2 = torch.randn(e_local, h, inter, generator=gen) * 0.05
    if fp8:   # gate and up halves of every expert on block scales far apart, and experts 2^e apart
        w13[:, :inter] *= 2.0 ** -6
        w13[:, inter:] *= 2.0 ** 6
        w13 *= torch.pow(2.0, torch.arange(e_local) % 5 - 2.0).view(-1, 1, 1)
    return w13.bfloat16().to(_dev()), w2.bfloat16().to(_dev())


def _slots_of(loc, e):
    return torch.nonzero(loc == e).flatten()


def stage_reports(a, loc, x, w13, w2, hbuf, ybuf, out, tw, e_local, inter, k, t, emap_all_remote=None):
    """Per-expert element-wise checks of GEMM1 (SiLU gate), GEMM2 and the combine on the kernel's own inputs."""
    reps = []
    pos = a["slot_pos"].cpu().long()
    xs = a["xs"]
    for e in range(e_local):
        s = _slots_of(loc, e)
        if s.numel() == 0:
            continue
        rows = pos[s].to(x.device)
        o64, b1 = silu_gate_oracle(xs[rows], w13[e, :inter], w13[e, inter:])
        r = gemm_report(hbuf[rows], o64, b1, what=f"GEMM1 (SiLU gate) expert {e}")
        if r:
            reps.append(r + f" (rows count the expert's slots in slot order; its first is xs row {int(rows[0])})")
        y64, b2 = gemm_oracle(hbuf[rows], w2[e])
        r = gemm_report(ybuf[rows], y64, b2, what=f"GEMM2 expert {e}")
        if r:
            reps.append(r)
    live = hbuf[pos[pos >= 0].to(x.device)]
    if not torch.isfinite(live.float()).all():
        reps.append("a live row of h is not finite: a tile mixed in a padding row")
    o64, b3 = combine_oracle(ybuf, a["slot_pos"], tw, t, k)
    r = gemm_report(out, o64, b3, what="combine")
    if r:
        reps.append(r.replace("row", "token", 1))
    if emap_all_remote is not None and emap_all_remote.numel():
        nz = out[emap_all_remote].view(torch.int16) != 0
        if nz.any():
            reps.append(f"combine: token {int(emap_all_remote[torch.nonzero(nz.any(-1))[0]])} has no local expert "
                        f"but a non-zero output")
    return reps


STAGE_CASES = [   # (name, T, K, E, E_local, H, inter)
    ("edge_counts", None, 2, 10, 10, 1000, 64),
    ("h1000_i192", 77, 2, 8, 8, 1000, 192),
    ("ep_half_i768", 200, 4, 16, 8, 512, 768),
]


def _stage_inputs(name, t, k, e, e_local, h, gen):
    emap = None
    if name == "edge_counts":
        ids = ids_with_counts(EDGE_COUNTS, k, gen)
        t = ids.shape[0]
    else:
        logits = torch.randn(t, e, generator=gen).bfloat16()
        _, ids = ref.topk_softmax(logits, k, True)
    if e_local < e:
        emap = torch.full((e,), -1, dtype=torch.int32)
        emap[1::2] = torch.arange(e_local, dtype=torch.int32)
        ids[:3] = torch.tensor([0, 2, 4, 6][:k], dtype=torch.int32)        # tokens 0..2: every expert remote
        emap = emap.to(_dev())
    tw = torch.rand(t, k, generator=gen).float() + 0.1
    return ids.to(_dev()), tw.to(_dev()), emap, t


@pytest.mark.parametrize("case", STAGE_CASES, ids=[c[0] for c in STAGE_CASES])
def test_grouped_bf16_stages(case):
    """align -> GEMM1 (SiLU gate on the 64-interleaved slab) -> GEMM2 -> combine through the library with NaN in
    every padding row of xs: each stage against its float64 oracle on the previous stage's kernel output. H = 1000
    puts a K tail in GEMM1 and an N tail in GEMM2; per-expert counts cover 0, 1, 127..129, 255..257."""
    from gllm_b200.ops import lib, sm100
    name, t, k, e, e_local, h, inter = case
    g = torch.Generator().manual_seed(h + inter)
    ids, tw, emap, t = _stage_inputs(name, t, k, e, e_local, h, g)
    x = _x(t, h, g)
    w13, w2 = _weights(e_local, inter, h, g)
    w13_il = torch.stack([ref.interleave_gate_up(w13[j], 64) for j in range(e_local)]).contiguous()
    a = run_align(ids, emap, e_local, x)
    rep = align_report(a, ids, emap, e_local, x, ids.numel())
    assert rep is None, rep
    L, p, st = lib.load(), sm100._p, lib.stream_ptr()
    rows = a["max_tiles"] * 128
    hbuf = torch.empty(rows, inter, dtype=torch.bfloat16, device=_dev())
    ybuf = torch.empty(rows, h, dtype=torch.bfloat16, device=_dev())
    out = torch.empty(t, h, dtype=torch.bfloat16, device=_dev())
    assert L.gllm_moe_grouped_gemm(p(a["xs"]), h, p(w13_il), p(hbuf), inter, a["max_tiles"], 2 * inter, h, e_local,
                                   p(a["tile_expert"]), p(a["meta"]), 1, None, st) == 0
    assert L.gllm_moe_grouped_gemm(p(hbuf), inter, p(w2), p(ybuf), h, a["max_tiles"], h, inter, e_local,
                                   p(a["tile_expert"]), p(a["meta"]), 0, None, st) == 0
    assert L.gllm_moe_combine(p(ybuf), p(a["slot_pos"]), p(tw), p(out), t, k, h, st) == 0
    torch.cuda.synchronize()
    loc, _, _ = align_oracle(ids, emap, ids.numel(), e_local)
    remote = torch.nonzero((loc.view(t, k) < 0).all(-1)).flatten().to(_dev())
    reps = stage_reports(a, loc, x, w13, w2, hbuf, ybuf, out, tw, e_local, inter, k, t, remote)
    assert not reps, "\n".join(reps)


def _fp8_weights(w13, w2):
    """Per expert: 128x128 block quantisation with one scale row per 64 weight rows (as the checkpoint loader does),
    gate/up interleaved per 64 for the kernel; returns (kernel q13, s13, q2, s2) and the plain (q13, s13)."""
    from gllm_b200.layers.moe import _block_quant_rows64
    q13, s13, q2, s2, pq13, ps13 = [], [], [], [], [], []
    for i in range(w13.shape[0]):
        a, sa = _block_quant_rows64(w13[i])
        b, sb = _block_quant_rows64(w2[i])
        pq13.append(a)
        ps13.append(sa)
        q13.append(ref.interleave_gate_up(a.view(torch.uint8), 64).view(torch.float8_e4m3fn))
        s13.append(ref.interleave_gate_up(sa, 1))
        q2.append(b)
        s2.append(sb)
    st = lambda v: torch.stack(v).contiguous()  # noqa: E731
    return st(q13), st(s13), st(q2), st(s2), pq13, ps13


def silu_compose(g64, eg, u64, eu):
    """silu(g) u and its bound from the bounds of g and u (the same propagation as silu_gate_oracle)."""
    s = g64 * torch.sigmoid(g64)
    o64 = s * u64
    return o64, (U_BF16 + 2.0 ** -16) * o64.abs() + 1.1 * eg * (u64.abs() + eu) + s.abs() * eu


def _scales_report(xin, s, rows, what):
    """Activation scales of the quantiser must equal amax / 448 exactly on the live rows."""
    amax = xin[rows].float().view(rows.numel(), -1, 128).abs().amax(-1).clamp_min(1e-10)
    got = s[:, rows].t()
    want = amax / 448.0
    if torch.equal(got, want):
        return None
    r, gi = [int(i) for i in torch.nonzero(got != want)[0]]
    return f"{what}: scale of row {int(rows[r])}, group {gi} is {float(got[r, gi])!r}, want {float(want[r, gi])!r}"


@pytest.mark.parametrize("t,k,e,inter", [(300, 2, 6, 128), (129, 4, 8, 256)])
def test_grouped_fp8_stages(t, k, e, inter):
    """Block-scaled fp8 experts stage by stage: scales equal amax / 448; GEMM1 (SiLU gate, gate and up halves on
    scales 2^12 apart, experts on scales 2^e apart) and GEMM2 through fp8_oracle with one scale row per 64 weight
    rows and per-expert scale slabs; the combine on the kernel's y. Padding rows of xs hold NaN."""
    from gllm_b200.ops import lib, sm100
    g = torch.Generator().manual_seed(t + inter)
    h = 512
    logits = torch.randn(t, e, generator=g).bfloat16()
    _, ids = ref.topk_softmax(logits, k, True)
    ids = ids.to(_dev())
    tw = (torch.rand(t, k, generator=g).float() + 0.1).to(_dev())
    x = _x(t, h, g)
    w13, w2 = _weights(e, inter, h, g, fp8=True)
    q13, s13, q2, s2, pq13, ps13 = _fp8_weights(w13, w2)
    a = run_align(ids, None, e, x)
    L, p, st = lib.load(), sm100._p, lib.stream_ptr()
    mt = a["max_tiles"]
    rows = mt * 128
    xs8 = torch.empty(rows, h, dtype=torch.uint8, device=_dev())
    xs_s = torch.empty(h // 128, rows, dtype=torch.float32, device=_dev())
    hbuf = torch.empty(rows, inter, dtype=torch.bfloat16, device=_dev())
    h8 = torch.empty(rows, inter, dtype=torch.uint8, device=_dev())
    h_s = torch.empty(inter // 128, rows, dtype=torch.float32, device=_dev())
    ybuf = torch.empty(rows, h, dtype=torch.bfloat16, device=_dev())
    out = torch.empty(t, h, dtype=torch.bfloat16, device=_dev())
    te, meta = p(a["tile_expert"]), p(a["meta"])
    assert L.gllm_fp8_quant_group(p(a["xs"]), h, p(xs8), p(xs_s), rows, h, st) == 0
    assert L.gllm_moe_grouped_gemm_fp8(p(xs8), p(xs_s), p(q13), p(s13), p(hbuf), inter, mt, 2 * inter, h, e, te,
                                       meta, 1, st) == 0
    assert L.gllm_fp8_quant_group(p(hbuf), inter, p(h8), p(h_s), rows, inter, st) == 0
    assert L.gllm_moe_grouped_gemm_fp8(p(h8), p(h_s), p(q2), p(s2), p(ybuf), h, mt, h, inter, e, te, meta, 0,
                                       st) == 0
    assert L.gllm_moe_combine(p(ybuf), p(a["slot_pos"]), p(tw), p(out), t, k, h, st) == 0
    torch.cuda.synchronize()
    loc, _, _ = align_oracle(ids, None, ids.numel(), e)
    pos = a["slot_pos"].cpu().long()
    live = pos[pos >= 0].to(_dev())
    reps = [r for r in (_scales_report(a["xs"], xs_s, live, "quant(xs)"), _scales_report(hbuf, h_s, live, "quant(h)"))
            if r]
    xq, hq = xs8.view(torch.float8_e4m3fn), h8.view(torch.float8_e4m3fn)
    ni = inter // 64
    for j in range(e):
        s = _slots_of(loc, j)
        if s.numel() == 0:
            continue
        r_ = pos[s].to(_dev())
        g64, eg = fp8_oracle(xq[r_], xs_s[:, r_], pq13[j][:inter], ps13[j][:ni], w_rows_per_scale=64)
        u64, eu = fp8_oracle(xq[r_], xs_s[:, r_], pq13[j][inter:], ps13[j][ni:], w_rows_per_scale=64)
        o64, b1 = silu_compose(g64, eg, u64, eu)
        r = gemm_report(hbuf[r_], o64, b1, what=f"fp8 GEMM1 (SiLU gate) expert {j}")
        if r:
            reps.append(r)
        y64, b2 = fp8_oracle(hq[r_], h_s[:, r_], q2[j], s2[j], w_rows_per_scale=64)
        r = gemm_report(ybuf[r_], y64, b2, what=f"fp8 GEMM2 expert {j}")
        if r:
            reps.append(r)
    if not torch.isfinite(ybuf[live].float()).all():
        reps.append("a live row of y is not finite: a tile mixed in a padding row")
    o64, b3 = combine_oracle(ybuf, a["slot_pos"], tw, t, k)
    r = gemm_report(out, o64, b3, what="fp8 combine")
    if r:
        reps.append(r)
    assert not reps, "\n".join(reps)


# ----------------------------------------------------------------------------------------------------------------
# the whole block
# ----------------------------------------------------------------------------------------------------------------
def block_oracle(x, w13, w2, tw, ids, expert_map=None):
    """float64 oracle of fused_experts per (token, slot) and per token, with the bound carried through the stages:
    GEMM1 + SiLU (silu_gate_oracle, bf16 rounding of h included) -> |w2| err_h + the GEMM2 bound on |h| + err_h ->
    the combine (|w| err_y, K multiply-adds, bf16 rounding). Returns (out64, bound [T, H], y64, err_y [T, K, H])."""
    t, k = ids.shape
    h = x.shape[1]
    inter = w13.shape[1] // 2
    loc = ids.long()
    if expert_map is not None:
        loc = expert_map.long()[loc]
    y64 = torch.zeros(t, k, h, dtype=torch.float64, device=x.device)
    ey = torch.zeros_like(y64)
    for e in range(w13.shape[0]):
        tok, slot = torch.where(loc == e)
        if tok.numel() == 0:
            continue
        o64, b1 = silu_gate_oracle(x[tok], w13[e, :inter], w13[e, inter:])
        w2a = w2[e].double().abs()
        yy = o64 @ w2[e].double().t()
        prop = b1 @ w2a.t()
        y64[tok, slot] = yy
        ey[tok, slot] = U_BF16 * (yy.abs() + prop) + prop + GEMM_C * inter * U_FP32 * ((o64.abs() + b1) @ w2a.t())
    w = tw.double().unsqueeze(-1) if tw is not None else torch.ones(t, k, 1, dtype=torch.float64, device=x.device)
    out64 = (w * y64).sum(1)
    mag = (w.abs() * (y64.abs() + ey)).sum(1)
    bound = (w.abs() * ey).sum(1) + U_BF16 * (out64.abs() + (w.abs() * ey).sum(1)) + 2 * k * U_FP32 * mag
    return out64, bound, y64, ey


@pytest.mark.parametrize("t,e,k,h,inter,ep", [(5, 8, 2, 256, 64, False), (300, 8, 2, 1000, 192, False),
                                               (200, 16, 4, 512, 768, True), (1000, 64, 6, 256, 128, False)])
def test_fused_experts_block(t, e, k, h, inter, ep):
    """sm100_moe.fused_experts against the float64 block oracle, element by element."""
    from gllm_b200.ops import sm100_moe
    g = torch.Generator().manual_seed(t + e + inter)
    e_local = e // 2 if ep else e
    x = _x(t, h, g)
    w13, w2 = _weights(e_local, inter, h, g)
    logits = torch.randn(t, e, generator=g).bfloat16().to(_dev())
    tw, ids = sm100_moe.topk_softmax(logits, k, True)
    emap = None
    if ep:
        emap = torch.full((e,), -1, dtype=torch.int32, device=_dev())
        emap[e // 2:] = torch.arange(e_local, dtype=torch.int32, device=_dev())
    w13_il = torch.stack([ref.interleave_gate_up(w13[j], 64) for j in range(e_local)]).contiguous()
    out = sm100_moe.fused_experts(x, w13_il, w2, tw, ids, emap)
    torch.cuda.synchronize()
    o64, bound, _, _ = block_oracle(x, w13, w2, tw, ids, emap)
    rep = gemm_report(out, o64, bound, what=f"fused_experts T={t} E={e} K={k} H={h} I={inter}")
    assert rep is None, rep.replace("row", "token", 1)


def test_fused_experts_fp8_block():
    """fused_experts_fp8 against the float64 oracle of the de-quantised weights and un-quantised activations: the
    e4m3 rounding of x and h (3 significand bits: at most 2^-4 relative, subnormal steps 2^-10 of the group
    scale) is carried through the stages like the bf16 block bound, with the fp8 accumulation term of FP8_ACC."""
    from test_wgmma_edges_gpu import FP8_ACC
    from gllm_b200.ops import sm100_moe
    g = torch.Generator().manual_seed(9)
    t, e, k, h, inter = 150, 8, 2, 512, 256
    x = _x(t, h, g)
    w13, w2 = _weights(e, inter, h, g, fp8=True)
    q13, s13, q2, s2, pq13, ps13 = _fp8_weights(w13, w2)
    logits = torch.randn(t, e, generator=g).bfloat16().to(_dev())
    tw, ids = sm100_moe.topk_softmax(logits, k, True)
    out = sm100_moe.fused_experts_fp8(x, q13, s13, q2, s2, tw, ids)
    torch.cuda.synchronize()
    Q = 2.0 ** -4 + 2.0 ** -22          # e4m3 rounding of a / s (a * (1 / s) in the kernel)

    def deq(q, s):
        return q.double() * s.double().repeat_interleave(64, 0).repeat_interleave(128, 1)

    def qerr(a):                        # bound of |a - dq(q(a))| per element: 2^-4 |a| + 2^-10 * group scale
        sc = a.double().view(a.shape[0], -1, 128).abs().amax(-1, keepdim=True) / 448
        return (Q * a.double().abs().view(a.shape[0], -1, 128) + 2.0 ** -10 * sc).view(a.shape)

    loc = ids.long()
    out64 = torch.zeros(t, h, dtype=torch.float64, device=_dev())
    err = torch.zeros_like(out64)
    for j in range(e):
        tok, slot = torch.where(loc == j)
        if tok.numel() == 0:
            continue
        wd, w2d = deq(pq13[j], ps13[j]), deq(q2[j], s2[j])
        xa = x[tok].double()
        ex = qerr(x[tok])
        gu = xa @ wd.t()
        mag = (xa.abs() + ex) @ wd.abs().t()
        egu = ex @ wd.abs().t() + (FP8_ACC + (h // 128 + 2) * U_FP32) * mag
        o64, b1 = silu_compose(gu[:, :inter], egu[:, :inter], gu[:, inter:], egu[:, inter:])
        eh = b1 + qerr(o64.float().bfloat16()) + Q * b1
        yy = o64 @ w2d.t()
        m2 = (o64.abs() + eh) @ w2d.abs().t()
        ey = eh @ w2d.abs().t() + (FP8_ACC + (inter // 128 + 2) * U_FP32) * m2 + U_BF16 * (yy.abs() + m2)
        wv = tw[tok, slot].double().unsqueeze(-1)
        out64.index_add_(0, tok, wv * yy)
        err.index_add_(0, tok, wv.abs() * ey + 2 * k * U_FP32 * wv.abs() * (yy.abs() + ey))
    bound = err + U_BF16 * (out64.abs() + err)
    rep = gemm_report(out, out64, bound, what="fused_experts_fp8")
    assert rep is None, rep.replace("row", "token", 1)


def test_ep_push_path():
    """The parallel/fused.py call shape on one GPU: top-1 local ids, no routing weight, n_valid live rows of the
    receive pool, and row_dest_fn mapping every live slot's row to an address in a sentinel-filled tensor (0 for
    padding rows). Each live slot's output lands at its address; nothing else changes."""
    from gllm_b200.ops import sm100_moe
    g = torch.Generator().manual_seed(21)
    r_max, n_live, e_local, h, inter = 700, 517, 4, 512, 128
    x = _x(r_max, h, g)
    w13, w2 = _weights(e_local, inter, h, g)
    w13_il = torch.stack([ref.interleave_gate_up(w13[j], 64) for j in range(e_local)]).contiguous()
    ids = torch.randint(0, e_local, (r_max, 1), generator=g).to(torch.int32)
    ids[:260] = 2                                            # expert 2 gets more than two tiles
    ids[n_live:] = 1                                         # dead slots: in range, must not be computed
    ids = ids.to(_dev())
    n_valid = torch.tensor([n_live], dtype=torch.int32, device=_dev())
    dest = torch.full((r_max + 8, h), SENTINEL, dtype=torch.bfloat16, device=_dev())
    perm = torch.randperm(r_max + 8, generator=g)[:r_max].to(_dev())   # slot s -> dest row perm[s]
    seen = {}

    def row_dest_fn(slot_pos, rows):
        rd = torch.zeros(rows, dtype=torch.int64, device=_dev())
        live = slot_pos[:r_max] >= 0
        s = torch.nonzero(live).flatten()
        rd[slot_pos[s].long()] = dest.data_ptr() + perm[s] * dest.stride(0) * dest.element_size()
        seen["slot_pos"] = slot_pos
        return rd

    assert sm100_moe.fused_experts(x, w13_il, w2, None, ids, None, n_valid=n_valid, row_dest_fn=row_dest_fn) is None
    torch.cuda.synchronize()
    sp = seen["slot_pos"][:r_max].cpu()
    assert bool((sp[n_live:] == -1).all()) and bool((sp[:n_live] >= 0).all()), "slot_pos of live / dead slots"
    _, bound, y64, ey = block_oracle(x[:n_live], w13, w2, None, ids[:n_live])
    got = dest[perm[:n_live]]
    rep = gemm_report(got, y64[:, 0], bound, what="EP push")
    assert rep is None, rep.replace("row", "slot", 1)
    untouched = torch.ones(r_max + 8, dtype=torch.bool, device=_dev())
    untouched[perm[:n_live]] = False
    assert bool((dest[untouched] == SENTINEL).all()), "rows written outside the live slots' addresses"


SENTINEL = -3.0


# ----------------------------------------------------------------------------------------------------------------
# CUDA graphs and determinism
# ----------------------------------------------------------------------------------------------------------------
def test_fused_experts_cuda_graph():
    """Capture fused_experts at a fixed T, replay it under other routings (an expert going from 0 tokens to 257);
    every replay equals an eager call bit for bit (rows are independent, the combine sums in slot order). An eager
    call at a larger T then grows the workspace and retires the captured buffers: a further replay still matches."""
    from gllm_b200.ops import sm100_moe
    g = torch.Generator().manual_seed(33)
    t, e, k, h, inter = 160, 8, 2, 512, 128
    w13, w2 = _weights(e, inter, h, g)
    w13_il = torch.stack([ref.interleave_gate_up(w13[j], 64) for j in range(e)]).contiguous()

    def routing(seed, hot=None, cold=None):
        gg = torch.Generator().manual_seed(seed)
        x = _x(t, h, gg).contiguous()
        tw = (torch.rand(t, k, generator=gg) + 0.1).float()
        if hot is not None:       # slot order: 257 slots of `hot`, the rest spread over the others
            rest = [i for i in range(e) if i != hot]
            flat = torch.tensor([hot] * 257 + [rest[i % len(rest)] for i in range(t * k - 257)])
            ids = flat[torch.randperm(t * k, generator=gg)].view(t, k).to(torch.int32)
        else:
            choices = [i for i in range(e) if i != cold]
            ids = torch.tensor(choices)[torch.randint(0, len(choices), (t, k), generator=gg)].to(torch.int32)
        return x, tw.to(_dev()), ids.to(_dev())

    xa, twa, idsa = routing(1, cold=3)
    x_s, tw_s, ids_s = xa.clone(), twa.clone(), idsa.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            sm100_moe.fused_experts(x_s, w13_il, w2, tw_s, ids_s)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out_s = sm100_moe.fused_experts(x_s, w13_il, w2, tw_s, ids_s)

    def replay_matches(inputs, what):
        x, tw, ids = inputs
        x_s.copy_(x)
        tw_s.copy_(tw)
        ids_s.copy_(ids)
        graph.replay()
        got = out_s.clone()
        want = sm100_moe.fused_experts(x, w13_il, w2, tw, ids)
        torch.cuda.synchronize()
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), f"{what}: replay differs from eager"
        return want, x, tw, ids

    replay_matches((xa, twa, idsa), "routing A (expert 3 empty)")
    want, x, tw, ids = replay_matches(routing(2, hot=3), "routing B (expert 3 has 257 slots)")
    o64, bound, _, _ = block_oracle(x, w13, w2, tw, ids)
    rep = gemm_report(want, o64, bound, what="eager B")
    assert rep is None, rep
    big = routing(3)
    xb = _x(4 * t, h, g)
    sm100_moe.fused_experts(xb, w13_il, w2, big[1].repeat(4, 1), big[2].repeat(4, 1))   # grows _ws
    torch.cuda.synchronize()
    replay_matches(routing(4, hot=5), "routing C after the workspace grew")
