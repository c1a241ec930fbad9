"""Element-wise edge tests of the wgmma kernels (persistent bf16 GEMM, swap-AB small-M GEMM, block-scaled FP8 GEMM,
prefill flash attention) and of the split-KV decode kernel, against float64 oracles (`pytest -m gpu`, one H100).

Every comparison is element by element against an error bound derived from the kernel's arithmetic (constants
below), so a fault confined to one tile, row or column fails with its coordinates instead of vanishing in a global
norm. The inputs are built so that each known class of slip (K tail, partial N tile, mis-indexed block scale, causal
leak, skipped softmax rescale, wrong GQA head base, reads past a sequence's last key) moves the output far beyond
rounding; tests/test_wgmma_edges_cpu.py shows on emulated kernels that these bounds reject such slips.

The oracles and comparators work on CPU tensors too: the CPU module imports them.
"""
import math

import pytest
import torch

from gllm_b200.ops import ref

pytestmark = pytest.mark.gpu

U_BF16 = 2.0 ** -8   # unit roundoff of bf16 (8-bit significand, round to nearest)
U_FP32 = 2.0 ** -24  # unit roundoff of fp32

# bf16 GEMM:  |y - y64| <= 2^-8 |y64| + GEMM_C * K * 2^-24 * (|x| |w|^T)[row, col]
#   2^-8 |y64|: the bf16 rounding of the fp32 result (bias included).
#   K * 2^-24 * (|x||w|^T): fp32 accumulation of K exact bf16 x bf16 products; recursive summation errs by at most
#   (K - 1) u sum|x_k w_k| with u = 2^-24 for round-to-nearest adds.
#   GEMM_C = 4: x2 because the tensor core aligns and truncates addends rather than rounding them (u = 2^-23), x2 for
#   the split-K partial sums (at most 8 more fp32 adds), the bias add and the second rounding of fp32 -> bf16.
GEMM_C = 4.0

# FP8 block GEMM: the same shape of bound per 128-deep K block, on the dequantised magnitudes:
#   |y - y64| <= 2^-8 |y64| + (FP8_ACC + (K/128 + 2) 2^-24) * sum_kb |a_s w_s| (|a8| |w8|^T)_kb
#   Hopper's e4m3 wgmma accumulates with fewer bits than fp32 (not documented), so FP8_ACC is calibrated on the GPU:
#   test_fp8_accumulation_factor measures the worst (|y - y64| - 2^-8 |y64|) / magnitude over correct outputs and
#   requires FP8_ACC >= 4x that. Measured on an H100 80GB HBM3 at a 700 W power limit: 7.5e-4 with all-positive
#   products, 2.4e-5 with mixed signs (M = N = 256, K = 1024); 2^-8 = 3.9e-3 >= 4 x 7.5e-4.
#   The (K/128 + 2) 2^-24 term is the fp32 promotion acc += part * (a_s * w_s).
FP8_ACC = 2.0 ** -8

# Attention, per (token, head) row: |o - o64| <= ATTN_C 2^-9 (P |V|) + 2^-9 |o64|, P the exact float64 probabilities.
#   The kernels round P to bf16 for the P.V MMA: sum_j |p~_j - p_j| |v_j| <= 2^-8 (P|V|) = 2 * 2^-9 (P|V|).
#   ATTN_C = 4 doubles that for the fp32 errors of S = QK^T (tensor-core accumulation over d), exp2f, the row sum l
#   and the O accumulation. 2^-9 |o64| plus the P term (|o64| <= P|V|) covers the bf16 rounding of the output.
ATTN_C = 4.0


def _dev():
    return torch.device("cuda:0")


def _sm100():
    from gllm_b200.ops import sm100
    return sm100


# ----------------------------------------------------------------------------------------------------------------
# oracles and comparators
# ----------------------------------------------------------------------------------------------------------------
def _worst(err, bound):
    """(number of violations, index of the worst one by err / bound); NaN counts as a violation."""
    bad = ~(err <= bound)
    n_bad = int(bad.sum())
    if n_bad == 0:
        return 0, None
    ratio = torch.where(bad, err / bound.clamp_min(1e-300), torch.zeros_like(err))
    ratio = torch.where(torch.isnan(err), torch.full_like(err, math.inf), ratio)
    flat = int(torch.argmax(ratio.reshape(-1)))
    return n_bad, tuple(int(i) for i in torch.unravel_index(torch.tensor(flat), err.shape))


def gemm_acc_bound(x, w):
    """Accumulation part of the bf16 GEMM bound, GEMM_C K 2^-24 (|x| |w|^T), float64 [M, N]."""
    return GEMM_C * x.shape[1] * U_FP32 * (x.double().abs() @ w.double().abs().t())


def gemm_oracle(x, w, bias=None):
    """float64 y = x w^T (+ bias) of the exact bf16 inputs, and the element-wise bound of a correct kernel."""
    y64 = x.double() @ w.double().t()
    if bias is not None:
        y64 = y64 + bias.double()
    return y64, U_BF16 * y64.abs() + gemm_acc_bound(x, w)


def silu_gate_oracle(x, w_gate, w_up):
    """float64 silu(x w_gate^T) * (x w_up^T) and its bound: the accumulation errors eg, eu of the two products
    propagate through silu (|silu'| <= 1.1) and the product; __expf adds ~2^-21 relative, taken as 2^-16 |o|."""
    g64, u64 = x.double() @ w_gate.double().t(), x.double() @ w_up.double().t()
    eg, eu = gemm_acc_bound(x, w_gate), gemm_acc_bound(x, w_up)
    s = g64 * torch.sigmoid(g64)
    o64 = s * u64
    return o64, (U_BF16 + 2.0 ** -16) * o64.abs() + 1.1 * eg * (u64.abs() + eu) + s.abs() * eu


def fp8_oracle(xq, xs, wq, ws, bias=None, w_rows_per_scale=128):
    """float64 block-scaled GEMM of the exact kernel inputs: xq e4m3 [M, K], xs fp32 [K/128, M] (the quantiser's
    output), wq e4m3 [N, K], ws fp32 [ceil(N / w_rows_per_scale), K/128]. Returns (y64, bound)."""
    m, k = xq.shape
    n = wq.shape[0]
    kb = k // 128
    a = xq.double().view(m, kb, 128)
    b = wq.double().view(n, kb, 128)
    part = torch.einsum("mkc,nkc->kmn", a, b)
    mag = torch.einsum("mkc,nkc->kmn", a.abs(), b.abs())
    sw = ws.double().repeat_interleave(w_rows_per_scale, 0)[:n].t()            # [kb, N]
    s = xs.double()[:, :, None] * sw[:, None, :]                               # [kb, M, N]
    y64 = (part * s).sum(0)
    if bias is not None:
        y64 = y64 + bias.double()
    m_abs = (mag * s.abs()).sum(0)
    return y64, U_BF16 * y64.abs() + (FP8_ACC + (kb + 2) * U_FP32) * m_abs


def gemm_report(y, y64, bound, tile=(128, 128), what="gemm"):
    """None when every element of y is within bound of y64, else a message naming the worst (row, col) and tile."""
    err = (y.double() - y64).abs()
    n_bad, idx = _worst(err, bound)
    if n_bad == 0:
        return None
    r, c = idx
    return (f"{what}: {n_bad} of {err.numel()} elements outside the bound; worst at row {r}, col {c} "
            f"(tile m{r // tile[0]} n{c // tile[1]} of {tile[0]}x{tile[1]}): got {float(y[r, c]):.6g}, "
            f"want {float(y64[r, c]):.6g}, |err| {float(err[r, c]):.3g} > bound {float(bound[r, c]):.3g}")


def attn_oracle(q, kc, vc, bt, seq_lens, q_start, hq, d, scale, head_chunk=8):
    """float64 causal paged attention of the exact bf16 inputs. Returns (o64, pv) [T, Hq, D]: the output and
    P |V| with P the float64 probabilities. Query i of a sequence sits at position seq_len - q_len + i."""
    t = q.shape[0]
    hkv = kc.shape[1]
    g = hq // hkv
    o64 = torch.zeros(t, hq, d, dtype=torch.float64, device=q.device)
    pv = torch.zeros_like(o64)
    qsl, sl = q_start.tolist(), seq_lens.tolist()
    for s in range(len(sl)):
        q0, q1 = qsl[s], qsl[s + 1]
        ql, n = q1 - q0, sl[s]
        if ql <= 0:
            continue
        kk = ref.gather_kv(kc, bt[s], n).double()
        vv = ref.gather_kv(vc, bt[s], n).double()
        qq = q[q0:q1].reshape(ql, hq, d).double()
        pos = torch.arange(ql, device=q.device) + (n - ql)
        mask = torch.arange(n, device=q.device).view(1, n) > pos.view(ql, 1)
        for h0 in range(0, hq, head_chunk):
            h1 = min(hq, h0 + head_chunk)
            kvi = torch.arange(h0, h1, device=q.device) // g
            logits = torch.einsum("qhd,khd->hqk", qq[:, h0:h1], kk[:, kvi]) * scale
            p = torch.softmax(logits.masked_fill(mask.unsqueeze(0), -math.inf), dim=-1)
            o64[q0:q1, h0:h1] = torch.einsum("hqk,khd->qhd", p, vv[:, kvi])
            pv[q0:q1, h0:h1] = torch.einsum("hqk,khd->qhd", p, vv[:, kvi].abs())
    return o64, pv


def tc_group_pack(g):
    """Heads per 128-row block of the wgmma prefill kernel (GP): the largest divisor of G that divides 128."""
    return next(x for x in range(min(g, 128), 0, -1) if g % x == 0 and 128 % x == 0)


def attn_report(o, o64, pv, q_start, hq, d, gp=1, what="attention"):
    """None when every (token, head) row is within the attention bound, else the worst (sequence, token, head) with
    its query tile (128/GP tokens per tile) and head group."""
    t = o64.shape[0]
    err = (o.reshape(t, hq, d).double() - o64).abs()
    bound = ATTN_C * 2.0 ** -9 * pv + 2.0 ** -9 * o64.abs()
    n_bad, idx = _worst(err, bound)
    if n_bad == 0:
        return None
    row, h, c = idx
    qsl = q_start.tolist()
    seq = max(i for i in range(len(qsl) - 1) if qsl[i] <= row)
    tok = row - qsl[seq]
    return (f"{what}: {n_bad} of {err.numel()} values outside the bound; worst at sequence {seq}, token {tok}, "
            f"head {h}, dim {c} (query tile {tok // (128 // gp)}, head group {h // gp}): "
            f"got {float(o.reshape(t, hq, d)[row, h, c]):.6g}, want {float(o64[row, h, c]):.6g}, "
            f"|err| {float(err[row, h, c]):.3g} > bound {float(bound[row, h, c]):.3g}")


# ----------------------------------------------------------------------------------------------------------------
# inputs
# ----------------------------------------------------------------------------------------------------------------
POISON = 1.0e4   # large but finite: the KV cache is zero-initialised, finite memory


def _pow2(shape, gen, lo=-8, hi=8):
    return torch.pow(2.0, torch.randint(lo, hi + 1, shape, generator=gen).double()).float()


def scatter_seq(cache, bt_row, page, vals):
    """Write vals [L, Hkv, D] as the first L keys of the sequence whose block-table row is bt_row."""
    n, hkv, d = vals.shape
    idx = torch.arange(n, device=cache.device)
    pages = bt_row.to(cache.device)[idx // page].long()
    cache[pages, :, :, idx % page, :] = vals.view(n, hkv, d // 64, 64).to(cache)


def make_paged_batch(seqs, hq, hkv, d, page, seed, device, nd=0, q_scale=0.5, kv_scale=0.5):
    """seqs: [(context_len, q_len)], the first nd of them decode sequences (q_len 1). Random bf16 q/k/v; q is the strided view
    qkv[:, :hq*d] of a fused projection output. Cache slots past each sequence's last key and three pages that no
    block table lists hold POISON; block-table padding points at one of those pages (a valid index)."""
    g = torch.Generator().manual_seed(seed)
    seq_lens = [c + ql for c, ql in seqs]
    q_lens = [ql for _, ql in seqs]
    npg = [(s + page - 1) // page for s in seq_lens]
    n_pages = sum(npg) + 3
    perm = torch.randperm(n_pages, generator=g).tolist()
    unlisted = perm[sum(npg):]
    max_blocks = max(npg) + 1
    bt = torch.full((len(seqs), max_blocks), unlisted[0], dtype=torch.int32)
    c = 0
    for i, n in enumerate(npg):
        bt[i, :n] = torch.tensor(perm[c:c + n], dtype=torch.int32)
        c += n
    shape = ref.kv_cache_shape(n_pages, hkv, d, page)
    kc = (torch.randn(shape, generator=g) * kv_scale).bfloat16()
    vc = (torch.randn(shape, generator=g) * kv_scale).bfloat16()
    t = sum(q_lens)
    qkv = (torch.randn(t, (hq + 2 * hkv) * d, generator=g) * q_scale).bfloat16()
    qsl = torch.tensor([0] + torch.tensor(q_lens).cumsum(0).tolist(), dtype=torch.int32)
    b = dict(qkv=qkv.to(device), kc=kc.to(device), vc=vc.to(device), bt=bt.to(device),
             sl=torch.tensor(seq_lens, dtype=torch.int32, device=device), qsl=qsl.to(device),
             seqs=list(seqs), nd=nd, hq=hq, hkv=hkv, d=d, page=page, unlisted=unlisted)
    poison_tail(b)
    return b


def poison_tail(b):
    """(Re)write POISON into the slots past every sequence's last key and into the unlisted pages."""
    page = b["page"]
    for cache in (b["kc"], b["vc"]):
        cache[b["unlisted"]] = POISON
        for i, s in enumerate(b["sl"].tolist()):
            if s % page:
                cache[int(b["bt"][i, s // page]), :, :, s % page:, :] = POISON


def q_view(b):
    return b["qkv"][:, : b["hq"] * b["d"]]


def set_monotone(b, lam=0.25):
    """Scores that rise with key position: key j carries (j // 256, j % 256) in dims 0, 1 and zeros elsewhere, every
    query of head h carries (256 s_h, s_h), so q.k = s_h j exactly. s_h * scale = lam * (1, 1.5, 2)[h % 3] per key:
    every query's best visible key is its own position, any causal leak lands on a larger score, and the running
    max moves on every KV tile."""
    hq, hkv, d, page = b["hq"], b["hkv"], b["d"], b["page"]
    scale = 1.0 / math.sqrt(d)
    for i, s in enumerate(b["sl"].tolist()):
        j = torch.arange(s, dtype=torch.float32)
        kv = torch.zeros(s, hkv, d)
        kv[:, :, 0] = (j // 256).view(s, 1)
        kv[:, :, 1] = (j % 256).view(s, 1)
        scatter_seq(b["kc"], b["bt"][i], page, kv)
    q = torch.zeros(b["qkv"].shape[0], hq, d)
    for h in range(hq):
        sh = float(torch.tensor(lam * (1.0, 1.5, 2.0)[h % 3] / scale).bfloat16())
        q[:, h, 0], q[:, h, 1] = 256.0 * sh, sh
    b["qkv"][:, : hq * d] = q.view(-1, hq * d).to(b["qkv"])
    poison_tail(b)


def set_peaked(b, seed):
    """Peaked logits: queries q = 0.6 z + c_kvh share a direction per KV head, keys are N(0, 1) except key 0 of every
    sequence (a sink) = beta c_kvh; with scale = 20 / sqrt(1.36 d) the scaled logits have a spread of about 20
    (extremes near +-80 over a few thousand keys) and the sink sits near +30."""
    g = torch.Generator().manual_seed(seed)
    hq, hkv, d, page = b["hq"], b["hkv"], b["d"], b["page"]
    scale = 20.0 / math.sqrt(1.36 * d)
    c = torch.randn(hkv, d, generator=g)
    t = b["qkv"].shape[0]
    q = 0.6 * torch.randn(t, hq, d, generator=g) + c.repeat_interleave(hq // hkv, 0).view(1, hq, d)
    b["qkv"][:, : hq * d] = q.view(t, hq * d).to(b["qkv"])
    for i, s in enumerate(b["sl"].tolist()):
        k = torch.randn(s, hkv, d, generator=g)
        k[0] = c * (30.0 / (scale * d))
        scatter_seq(b["kc"], b["bt"][i], page, k)
    poison_tail(b)
    return scale


def edge_seqs(tpt, page, kv_tiles=(64, 128), nd=2):
    """(context, q_len) pairs around the query tile (tpt tokens), the KV tiles and page multiples, each at -1, 0, +1,
    behind nd decode sequences. Returns (pairs, nd)."""
    pairs = [(0, 1), (76, 1)][:nd]
    qls = sorted({x for x in (1, tpt - 1, tpt, tpt + 1) if x > 0})
    ctxs = sorted({0} | {kv + e for kv in kv_tiles for e in (-1, 0, 1)})
    body = [(c, ql) for ql in qls for c in ctxs]
    body += [(s - ql, ql) for ql in (tpt, tpt + 1) for s in (2 * page - 1, 2 * page, 2 * page + 1) if s >= ql]
    for p in body:
        if p not in pairs[nd:]:
            pairs.append(p)
    return pairs, nd


def run_attention(kind, b, monkeypatch, scale=None, splits=None):
    """kind: 'tc64' / 'tc128' (wgmma kernel with that KV tile) or 'mma' (the mma.sync kernel)."""
    sm100 = _sm100()
    monkeypatch.setattr(sm100, "ATTN_TC", kind != "mma")
    if kind != "mma":
        monkeypatch.setattr(sm100, "ATTN_TC_KV", int(kind[2:]))
    seqs, nd = b["seqs"], b["nd"]
    max_q = max(ql for _, ql in seqs[nd:]) if nd < len(seqs) else 1
    scale = scale if scale is not None else 1.0 / math.sqrt(b["d"])
    o = sm100.paged_attention(q_view(b), b["kc"], b["vc"], b["bt"], b["sl"], b["qsl"], scale, b["hq"], b["d"], nd,
                              len(seqs), max_q, int(b["sl"].max()), splits=splits)
    torch.cuda.synchronize()
    return o


def _attn_case(b, kinds, monkeypatch, scale=None):
    scale = scale if scale is not None else 1.0 / math.sqrt(b["d"])
    o64, pv = attn_oracle(q_view(b), b["kc"], b["vc"], b["bt"], b["sl"], b["qsl"], b["hq"], b["d"], scale)
    gp = tc_group_pack(b["hq"] // b["hkv"])
    reps = []
    for kind in kinds:
        o = run_attention(kind, b, monkeypatch, scale)
        assert torch.isfinite(o.float()).all(), kind
        r = attn_report(o, o64, pv, b["qsl"], b["hq"], b["d"], gp, what=kind)
        if r:
            reps.append(r)
    assert not reps, "\n".join(reps)


# ----------------------------------------------------------------------------------------------------------------
# GEMM fixtures / helpers
# ----------------------------------------------------------------------------------------------------------------
SENTINEL = -3.0


@pytest.fixture
def gemm_tune():
    """Forces a split-K factor / split-K M ceiling through gllm_gemm_tune; afterwards the library goes back to the
    defaults it derives from the environment (-1 = read GLLM_GEMM_FORCE_SPLITK / GLLM_GEMM_SPLITK_MAX_M again)."""
    from gllm_b200.ops import lib
    L = lib.load()

    def tune(force_split, max_split_m=512):
        assert L.gllm_gemm_tune(int(force_split), int(max_split_m)) == 0

    yield tune
    L.gllm_gemm_tune(-1, -1)


def _rand(shape, scale, gen):
    return (torch.randn(*shape, generator=gen) * scale).bfloat16().to(_dev())


def _strided_x(m, k, gen, scale=0.5):
    """[M, K] activation with row stride K + 24 (a column slice of a wider buffer)."""
    return _rand((m, k + 24), scale, gen)[:, :k]


def _guarded_out(m, n, ldc_pad=24):
    """[M, N] output view inside a sentinel-filled [M + 2, N + ldc_pad] buffer (16-byte aligned start)."""
    big = torch.full((m + 2, n + ldc_pad), SENTINEL, dtype=torch.bfloat16, device=_dev())
    return big, big[1:m + 1, 8:8 + n]


def _outside_untouched(big, m, n):
    mask = torch.ones(big.shape, dtype=torch.bool, device=big.device)
    mask[1:m + 1, 8:8 + n] = False
    bits = big.view(torch.int16)[mask]
    want = torch.tensor(SENTINEL, dtype=torch.bfloat16).view(torch.int16).item()
    bad = int((bits != want).sum())
    return bad == 0, f"{bad} bf16 values written outside the [{m}, {n}] output view"


def _interleave_gu(w, block=128):
    return ref.interleave_gate_up(w, block)


# ----------------------------------------------------------------------------------------------------------------
# persistent bf16 GEMM (gemm_bf16.cu)
# ----------------------------------------------------------------------------------------------------------------
M_EDGES = [1, 63, 64, 65, 127, 128, 129, 255, 257, 1000]
K_EDGES = [8, 16, 56, 72, 136, 200, 3424, 4104]
N_EDGES = [(n, bn) for n in (8, 24, 40, 72, 136, 264) for bn in (32, 64, 128, 256)] + \
          [(3 * bn + s, bn) for bn in (32, 64, 128, 256) for s in (-8, 8)]


def _linear_checked(sm100, x, w, bias, tile, what):
    m, n = x.shape[0], w.shape[0]
    big, out = _guarded_out(m, n)
    y = sm100.linear(x, w, bias, out=out)
    torch.cuda.synchronize()
    assert y.data_ptr() == out.data_ptr()
    ok, msg = _outside_untouched(big, m, n)
    assert ok, f"{what}: {msg}"
    y64, bound = gemm_oracle(x, w, bias)
    return gemm_report(out, y64, bound, tile, what)


@pytest.mark.parametrize("bn", [128, 64])
@pytest.mark.parametrize("m", M_EDGES)
def test_bf16_gemm_m_edges(m, bn, monkeypatch):
    """Every M tile edge, strided x, bias, sentinel-guarded strided out; N = 264 and K = 136 have tails too."""
    sm100 = _sm100()
    monkeypatch.setattr(sm100, "_FORCE_BN", bn)
    g = torch.Generator().manual_seed(m * 7 + bn)
    n, k = 264, 136
    x, w, b = _strided_x(m, k, g), _rand((n, k), 0.05, g), _rand((n,), 1.0, g)
    rep = _linear_checked(sm100, x, w, b, (128, bn), f"gemm_bf16 M={m} BN={bn}")
    assert rep is None, rep


@pytest.mark.parametrize("n,bn", N_EDGES)
def test_bf16_gemm_n_edges(n, bn, monkeypatch):
    """N at every BN edge (partial last N tile: stores and bias guarded by col < N), M = 129, K = 200 (tail 8)."""
    sm100 = _sm100()
    monkeypatch.setattr(sm100, "_FORCE_BN", bn)
    g = torch.Generator().manual_seed(n * 3 + bn)
    m, k = 129, 200
    x, w, b = _strided_x(m, k, g), _rand((n, k), 0.05, g), _rand((n,), 1.0, g)
    rep = _linear_checked(sm100, x, w, b, (128, bn), f"gemm_bf16 N={n} BN={bn}")
    assert rep is None, rep


@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("k", K_EDGES)
def test_bf16_gemm_k_edges(k, bias, gemm_tune):
    """K tails (TMA zero fill of the last 64-wide block; K < 64 is a box wider than the tensor), with the
    split-K choice of the cost model and with split-K off."""
    sm100 = _sm100()
    g = torch.Generator().manual_seed(k * 2 + bias)
    m, n = 200, 264
    x, w = _strided_x(m, k, g), _rand((n, k), 0.05, g)
    b = _rand((n,), 1.0, g) if bias else None
    reps = [_linear_checked(sm100, x, w, b, (128, 128), f"gemm_bf16 K={k} (auto split)")]
    gemm_tune(0, 0)                                                # split-K off
    reps.append(_linear_checked(sm100, x, w, b, (128, 128), f"gemm_bf16 K={k} (no split)"))
    reps = [r for r in reps if r]
    assert not reps, "\n".join(reps)


def _silu_checked(sm100, x, w, tile, what):
    m, i = x.shape[0], w.shape[0] // 2
    big, out = _guarded_out(m, i)
    sm100.linear_silu_mul(x, _interleave_gu(w), out=out)
    torch.cuda.synchronize()
    ok, msg = _outside_untouched(big, m, i)
    assert ok, f"{what}: {msg}"
    o64, bound = silu_gate_oracle(x, w[:i], w[i:])
    return gemm_report(out, o64, bound, tile, what)


@pytest.mark.parametrize("m,k", [(1, 200), (77, 3424), (200, 72), (300, 4104)])
def test_bf16_gemm_silu_k_tail(m, k, monkeypatch):
    """SiLU-gate epilogue (BN = 256 tiles = [128 gate | 128 up]) with a K tail."""
    sm100 = _sm100()
    monkeypatch.setattr(sm100, "_FORCE_BN", 256)                 # through gemm_bf16 even for small M
    g = torch.Generator().manual_seed(m + k)
    x, w = _strided_x(m, k, g), _rand((2 * 384, k), 0.05, g)
    rep = _silu_checked(sm100, x, w, (128, 128), f"gemm_bf16 silu M={m} K={k}")
    assert rep is None, rep


def _split_used(m, n, k, epi, bn):
    from gllm_b200.ops import lib
    sm100 = _sm100()
    units = lib.load().gllm_gemm_bf16_tiles_covering(m, n, k, epi, bn, 0, m, sm100._SMALLM_WS_FLOATS * 4,
                                                     sm100._SPLITK_MAX_TILES)
    return units // (((m + 127) // 128) * ((n + bn - 1) // bn))


@pytest.mark.parametrize("bn,split,epi", [(256, 2, 0), (256, 4, 0), (256, 8, 0), (128, 2, 0), (128, 4, 0), (64, 2, 0),
                                          (256, 2, 1), (256, 4, 1), (256, 8, 1)])
@pytest.mark.parametrize("m", [1, 200])
def test_bf16_gemm_forced_splitk(m, bn, split, epi, gemm_tune, monkeypatch):
    """Every legal split-K factor per tile width; K = 3424 = 53.5 k-blocks, so the last slice is short and ends in
    the K tail (split 8: 7 + ... + 5 blocks)."""
    sm100 = _sm100()
    monkeypatch.setattr(sm100, "_FORCE_BN", bn)
    gemm_tune(split)
    g = torch.Generator().manual_seed(m + bn + split + epi)
    k = 3424
    if epi == 0:
        n = 1032
        assert _split_used(m, n, k, 0, bn) == split
        x, w, b = _strided_x(m, k, g), _rand((n, k), 0.05, g), _rand((n,), 1.0, g)
        rep = _linear_checked(sm100, x, w, b, (128, bn), f"gemm_bf16 split={split} BN={bn}")
    else:
        i = 640
        assert _split_used(m, 2 * i, k, 1, 256) == split
        x, w = _strided_x(m, k, g), _rand((2 * i, k), 0.05, g)
        rep = _silu_checked(sm100, x, w, (128, 128), f"gemm_bf16 silu split={split}")
    assert rep is None, rep


def test_bf16_gemm_splitk_counters_rearm(gemm_tune, monkeypatch):
    """Split-K tile counters re-arm themselves: shape A, then B (other tile count), then A again, bitwise equal."""
    sm100 = _sm100()
    monkeypatch.setattr(sm100, "_FORCE_BN", 256)
    gemm_tune(4)
    g = torch.Generator().manual_seed(5)
    xa, wa = _rand((64, 3424), 0.5, g), _rand((1024, 3424), 0.05, g)
    xb, wb = _rand((300, 4104), 0.5, g), _rand((264, 4104), 0.05, g)
    assert _split_used(64, 1024, 3424, 0, 256) == 4 and _split_used(300, 264, 4104, 0, 256) == 4
    ya1 = sm100.linear(xa, wa).clone()
    yb = sm100.linear(xb, wb)
    ya2 = sm100.linear(xa, wa)
    torch.cuda.synchronize()
    assert torch.equal(ya1, ya2)
    for y, x, w, what in ((ya1, xa, wa, "A"), (yb, xb, wb, "B")):
        y64, bound = gemm_oracle(x, w)
        rep = gemm_report(y, y64, bound, what=f"gemm_bf16 re-arm {what}")
        assert rep is None, rep


@pytest.mark.parametrize("k", [72, 200])
@pytest.mark.parametrize("t", [1, 130, 257])
def test_gemm_batched_tails(t, k):
    """Batched mode: T not a multiple of 128, K tail, strided operand and strided sentinel-guarded output."""
    sm100 = _sm100()
    g = torch.Generator().manual_seed(t + k)
    b, n = 3, 136
    a = _rand((t, b, k + 8), 0.5, g)[:, :, :k]
    w = _rand((b, n, k), 0.1, g)
    out_full = torch.full((t, b, n + 8), SENTINEL, dtype=torch.bfloat16, device=_dev())
    out = out_full[:, :, :n]
    sm100.gemm_batched(a, w, out)
    torch.cuda.synchronize()
    assert bool((out_full[:, :, n:] == SENTINEL).all()), "written outside the output view"
    reps = []
    for j in range(b):
        y64, bound = gemm_oracle(a[:, j], w[j])
        reps.append(gemm_report(out[:, j], y64, bound, what=f"gemm_batched T={t} K={k} batch {j}"))
    reps = [r for r in reps if r]
    assert not reps, "\n".join(reps)


# ----------------------------------------------------------------------------------------------------------------
# swap-AB small-M GEMM (gemm_bf16_smallm.cu)
# ----------------------------------------------------------------------------------------------------------------
SMALLM_M = [1, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256]


def _token_tile(m):
    return next(bt for bt in (16, 32, 64, 128, 256) if m <= bt)


@pytest.mark.parametrize("split", [0, 1, 3])
@pytest.mark.parametrize("m", SMALLM_M)
def test_smallm_m_edges(m, split, monkeypatch):
    """Every token-tile edge; N = 1000 (partial weight tile), K = 3424 (tail), bias, forced splits (1 = the direct
    store epilogue, 3 = the last-arriver reduction)."""
    sm100 = _sm100()
    monkeypatch.setattr(sm100, "_SMALLM_MAX", 256)
    monkeypatch.setattr(sm100, "_FORCE_SPLIT", split)
    g = torch.Generator().manual_seed(m * 5 + split)
    n, k = 1000, 3424
    x, w, b = _strided_x(m, k, g), _rand((n, k), 0.05, g), _rand((n,), 1.0, g)
    rep = _linear_checked(sm100, x, w, b, (_token_tile(m), 128), f"gemm_smallm M={m} split={split}")
    assert rep is None, rep


@pytest.mark.parametrize("split", [0, 2])
@pytest.mark.parametrize("k", K_EDGES)
def test_smallm_k_edges(k, split, monkeypatch):
    sm100 = _sm100()
    monkeypatch.setattr(sm100, "_SMALLM_MAX", 256)
    monkeypatch.setattr(sm100, "_FORCE_SPLIT", split)
    g = torch.Generator().manual_seed(k + split)
    m, n = 17, 264
    x, w, b = _strided_x(m, k, g), _rand((n, k), 0.05, g), _rand((n,), 1.0, g)
    rep = _linear_checked(sm100, x, w, b, (32, 128), f"gemm_smallm K={k} split={split}")
    assert rep is None, rep


@pytest.mark.parametrize("split", [0, 2])
@pytest.mark.parametrize("m", [1, 17, 64, 200])
def test_smallm_silu_k_tail(m, split, monkeypatch):
    sm100 = _sm100()
    monkeypatch.setattr(sm100, "_SMALLM_MAX", 256)
    monkeypatch.setattr(sm100, "_FORCE_SPLIT", split)
    g = torch.Generator().manual_seed(m + 31 * split)
    x, w = _strided_x(m, 3424, g), _rand((2 * 384, 3424), 0.05, g)
    rep = _silu_checked(sm100, x, w, (_token_tile(m), 128), f"gemm_smallm silu M={m} split={split}")
    assert rep is None, rep


def test_smallm_counters_rearm(monkeypatch):
    """Shape A, B, A through the split reduction: the per-tile arrival counters reset themselves."""
    sm100 = _sm100()
    monkeypatch.setattr(sm100, "_SMALLM_MAX", 256)
    monkeypatch.setattr(sm100, "_FORCE_SPLIT", 3)
    g = torch.Generator().manual_seed(9)
    xa, wa = _rand((17, 3424), 0.5, g), _rand((1000, 3424), 0.05, g)
    xb, wb = _rand((129, 4104), 0.5, g), _rand((264, 4104), 0.05, g)
    ya1 = sm100.linear(xa, wa).clone()
    yb = sm100.linear(xb, wb)
    ya2 = sm100.linear(xa, wa)
    torch.cuda.synchronize()
    assert torch.equal(ya1, ya2)
    y64, bound = gemm_oracle(xb, wb)
    rep = gemm_report(yb, y64, bound, what="gemm_smallm re-arm B")
    assert rep is None, rep


@pytest.mark.parametrize("m", [33, 64])
def test_smallm_production_routing(m, monkeypatch):
    """With _SMALLM_MAX at its default, linear() sends m <= 64 and k >= 8192 to the small-M kernel."""
    sm100 = _sm100()
    calls = []
    orig = sm100._linear_smallm

    def spy(*a, **kw):
        calls.append(a[0].shape)
        return orig(*a, **kw)

    monkeypatch.setattr(sm100, "_linear_smallm", spy)
    g = torch.Generator().manual_seed(m)
    k, n = 8200, 264
    x, w, b = _strided_x(m, k, g), _rand((n, k), 0.05, g), _rand((n,), 1.0, g)
    rep = _linear_checked(sm100, x, w, b, (64, 128), f"linear M={m} K={k}")
    assert calls, "not routed to the small-M kernel"
    assert rep is None, rep


@pytest.mark.parametrize("m", [1, 16, 200])
def test_linear_rejects_unaligned_n_and_ldc(m):
    """N and the output row stride must be multiples of 8 on both GEMM paths (16-byte / 8-byte vector stores):
    linear() fails cleanly, before any launch, whatever M selects."""
    sm100 = _sm100()
    g = torch.Generator().manual_seed(m)
    x = _rand((m, 64), 0.5, g)
    with pytest.raises(RuntimeError, match="launch failed"):
        sm100.linear(x, _rand((1001, 64), 0.05, g))
    big = torch.zeros(m, 1004, dtype=torch.bfloat16, device=_dev())
    with pytest.raises(RuntimeError, match="launch failed"):
        sm100.linear(x, _rand((1000, 64), 0.05, g), out=big[:, :1000])
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------------------------
# block-scaled FP8 GEMM and the activation quantiser (gemm_fp8_block.cu)
# ----------------------------------------------------------------------------------------------------------------
def _scaled_activations(m, k, gen):
    """bf16 [M, K] whose (row, 128-group) cells are scaled by 2^e, e in [-8, 8]; one all-zero row (when M > 1) and
    one all-zero group in every other row."""
    x = torch.randn(m, k // 128, 128, generator=gen) * _pow2((m, k // 128, 1), gen)
    if m > 1:
        x[m // 2] = 0
    x[::2, 1] = 0
    return x.reshape(m, k).bfloat16().to(_dev())


def _block_scaled_weight(n, k, gen):
    """e4m3 [N, K] + fp32 scale_inv [ceil(N/128), K/128]; every 128x128 block scaled by 2^e, e in [-8, 8]."""
    nb, kb = (n + 127) // 128, k // 128
    w = torch.randn(nb, 128, kb, 128, generator=gen) * 0.05 * _pow2((nb, 1, kb, 1), gen)
    s_inv = (w.abs().amax(dim=(1, 3)) / 448.0).clamp_min(1e-12)
    w8 = (w / s_inv.view(nb, 1, kb, 1)).view(nb * 128, k)[:n].to(torch.float8_e4m3fn)
    return w8.contiguous().to(_dev()), s_inv.contiguous().to(_dev())


def _e4m3_ordinal(q):
    b = q.view(torch.uint8).to(torch.int16)
    mag = b & 0x7F
    return torch.where((b & 0x80) != 0, -mag, mag)


@pytest.mark.parametrize("m", [1, 129, 300])
def test_fp8_quantiser(m):
    """Scales equal amax / 448 exactly (IEEE division). Codes may differ from x / s by one e4m3 step: the kernel
    multiplies by 1/s, which differs from x / s in the last fp32 bit and can cross an e4m3 rounding boundary."""
    sm100 = _sm100()
    g = torch.Generator().manual_seed(m)
    k = 512
    x = _scaled_activations(m, k, g)
    q, s = sm100.fp8_quant_group(x)
    torch.cuda.synchronize()
    amax = x.float().view(m, k // 128, 128).abs().amax(-1).clamp_min(1e-10)
    want = (amax / 448.0).t()
    if not torch.equal(s, want):
        g_, r_ = [int(i) for i in torch.nonzero(s != want)[0]]
        raise AssertionError(f"{int((s != want).sum())} scales differ from amax/448; first at row {r_}, group {g_}: "
                             f"{float(s[g_, r_])!r} vs {float(want[g_, r_])!r}")
    q_ref = (x.float().view(m, k // 128, 128) / want.t().unsqueeze(-1)).clamp(-448, 448)
    q_ref = q_ref.reshape(m, k).to(torch.float8_e4m3fn)
    step = (_e4m3_ordinal(q) - _e4m3_ordinal(q_ref)).abs()
    assert int(step.max()) <= 1, f"code off by {int(step.max())} e4m3 steps at {torch.nonzero(step > 1)[0].tolist()}"
    zero = x.float().abs().amax(-1) == 0
    assert bool((q.float()[zero] == 0).all()) and torch.isfinite(s).all()


@pytest.mark.parametrize("m,n", [(1, 576), (129, 192), (129, 576), (300, 1024), (64, 256)])
def test_fp8_gemm_block_scales(m, n):
    """Block scales spanning 2^-8 .. 2^8 per weight block and per activation cell, so any mis-indexed scale (w_s
    transposed, a_s with the wrong pitch) is off by orders of magnitude; the oracle gets the kernel's own quantiser
    output, so the comparison is exact arithmetic up to the bound. Zero rows give bias only, zero groups no NaN."""
    sm100 = _sm100()
    g = torch.Generator().manual_seed(m * 11 + n)
    k = 512
    x = _scaled_activations(m, k, g)
    w8, s_inv = _block_scaled_weight(n, k, g)
    b = _rand((n,), 1.0, g)
    big, out = _guarded_out(m, n)
    sm100.linear_fp8_block(x, w8, s_inv, b, out=out)
    xq, xs = sm100.fp8_quant_group(x)
    torch.cuda.synchronize()
    ok, msg = _outside_untouched(big, m, n)
    assert ok, msg
    assert torch.isfinite(out.float()).all()
    y64, bound = fp8_oracle(xq, xs, w8, s_inv, b)
    rep = gemm_report(out, y64, bound, what=f"gemm_fp8_block M={m} N={n}")
    assert rep is None, rep
    if m > 1:
        assert torch.equal(out[m // 2], b), "an all-zero row must give exactly the bias"


def fp8_acc_excess(y, y64, m_abs):
    """Worst (|y - y64| - 2^-8 |y64|) / magnitude: the accumulation error the FP8_ACC term has to cover."""
    return float(((y.double() - y64).abs() - U_BF16 * y64.abs()).clamp_min(0).div(m_abs.clamp_min(1e-300)).max())


def test_fp8_accumulation_factor():
    """FP8_ACC is at least 4x the worst accumulation error measured on correct outputs: all-positive products (the
    error adds up, nothing cancels) and mixed signs (the output is small next to the magnitudes)."""
    sm100 = _sm100()
    g = torch.Generator().manual_seed(123)
    m, n, k = 256, 256, 1024
    measured = {}
    for positive in (True, False):
        x = torch.randn(m, k, generator=g)
        w = torch.randn(n, k, generator=g) * 0.05
        if positive:
            x, w = x.abs(), w.abs()
        x = x.bfloat16().to(_dev())
        nb, kb = n // 128, k // 128
        s_inv = (w.view(nb, 128, kb, 128).abs().amax(dim=(1, 3)) / 448.0)
        w8 = (w.view(nb, 128, kb, 128) / s_inv.view(nb, 1, kb, 1)).view(n, k).to(torch.float8_e4m3fn)
        w8, s_inv = w8.to(_dev()), s_inv.to(_dev())
        y = sm100.linear_fp8_block(x, w8, s_inv)
        xq, xs = sm100.fp8_quant_group(x)
        torch.cuda.synchronize()
        y64, _ = fp8_oracle(xq, xs, w8, s_inv)
        m_abs = (fp8_oracle(xq.float().abs().to(torch.float8_e4m3fn), xs, w8.float().abs().to(torch.float8_e4m3fn),
                            s_inv)[0])
        measured["all-positive" if positive else "mixed-sign"] = fp8_acc_excess(y, y64, m_abs)
    worst = max(measured.values())
    print(f"fp8 accumulation excess: {measured}, FP8_ACC {FP8_ACC:.3g}")
    assert 4 * worst <= FP8_ACC, f"measured {worst:.3g}: FP8_ACC {FP8_ACC:.3g} is less than 4x"


def test_moe_fp8_gate_up_scales_differ():
    """Grouped fp8 expert GEMMs on [64 gate | 64 up] tiles whose two halves carry block scales 2^12 apart: reading the
    gate scale for the up half (or the reverse) scales half of every intermediate by 2^+-12. Per token row against
    the de-quantised oracle (both activation quantisations emulated)."""
    from gllm_b200.layers.moe import _block_quant_rows64
    from gllm_b200.ops import sm100_moe
    g = torch.Generator().manual_seed(77)
    dev = _dev()
    t, e, k, h, inter = 200, 4, 2, 256, 128
    x = (torch.randn(t, h, generator=g) * 0.5).bfloat16().to(dev)
    w13 = torch.randn(e, 2 * inter, h, generator=g) * 0.05
    w13[:, :inter] *= 2.0 ** -6                                   # gate rows
    w13[:, inter:] *= 2.0 ** 6                                    # up rows
    w13 = w13.bfloat16().to(dev)
    w2 = (torch.randn(e, h, inter, generator=g) * 0.05).bfloat16().to(dev)
    logits = torch.randn(t, e, generator=g).bfloat16().to(dev)
    tw, ids = sm100_moe.topk_softmax(logits, k, True)
    q13, s13, q2, s2, d13, d2 = [], [], [], [], [], []
    for i in range(e):
        a, sa = _block_quant_rows64(w13[i])
        b, sb = _block_quant_rows64(w2[i])
        assert float(sa[2:].min()) > 2.0 ** 10 * float(sa[:2].max())   # up-half scales >> gate-half scales
        d13.append(a.double() * sa.double().repeat_interleave(64, 0).repeat_interleave(128, 1))
        d2.append(b.double() * sb.double().repeat_interleave(64, 0).repeat_interleave(128, 1))
        q13.append(ref.interleave_gate_up(a.view(torch.uint8), 64).view(torch.float8_e4m3fn))
        s13.append(ref.interleave_gate_up(sa, 1))
        q2.append(b)
        s2.append(sb)
    out = sm100_moe.fused_experts_fp8(x, torch.stack(q13), torch.stack(s13).contiguous(), torch.stack(q2),
                                      torch.stack(s2).contiguous(), tw, ids)
    torch.cuda.synchronize()

    def qdq(a):
        q, sc = ref.fp8_quant_group(a, 128)
        return (q.double().reshape(a.shape[0], -1, 128) * sc.double().unsqueeze(-1)).reshape(a.shape)

    want = torch.zeros(t, h, dtype=torch.float64, device=dev)
    for i in range(e):
        tok, slot = torch.where(ids.long() == i)
        if tok.numel() == 0:
            continue
        hg = qdq(x[tok]) @ d13[i].t()
        hd = (torch.nn.functional.silu(hg[:, :inter]) * hg[:, inter:]).bfloat16()
        want.index_add_(0, tok, (qdq(hd) @ d2[i].t()) * tw[tok, slot].double().unsqueeze(-1))
    assert torch.isfinite(out.float()).all()
    row_err = (out.double() - want).norm(dim=1) / want.norm(dim=1)
    worst = int(row_err.argmax())
    # e4m3 quantisation of the bf16 intermediate is re-done here with torch's x / s: some codes differ by one step
    assert float(row_err.max()) < 6e-2, f"token {worst}: relative error {float(row_err[worst]):.3g}"


# ----------------------------------------------------------------------------------------------------------------
# prefill attention (prefill_attention_tc.cu, mma.sync fallback in paged_attention.cu) and split-KV decode
# ----------------------------------------------------------------------------------------------------------------
ALL_KINDS = ("tc64", "tc128", "mma")


@pytest.mark.parametrize("g", [1, 2, 3, 4, 5, 6, 7, 8, 12, 16])
@pytest.mark.parametrize("d", [64, 128])
def test_prefill_gqa_edges(d, g, monkeypatch):
    """Every GQA ratio (GP = 1, 2, 4, 8 or 16 heads per row block; G = 6 / 12 put several blocks on one KV head),
    q_len / context / seq_len at -1, 0, +1 around the query tile, both KV tiles and page multiples; decode sequences
    in front, strided q, poisoned cache tails and unlisted pages."""
    hkv = 2
    seqs, nd = edge_seqs(128 // tc_group_pack(g), 16)
    b = make_paged_batch(seqs, g * hkv, hkv, d, 16, seed=g * 100 + d, device=_dev(), nd=nd)
    _attn_case(b, ALL_KINDS, monkeypatch)


@pytest.mark.parametrize("kv", [64, 128])
@pytest.mark.parametrize("page", [8, 16, 32, 64, 128])
def test_prefill_page_sizes(page, kv, monkeypatch):
    """Page size x KV tile (G = 12: GP = 4, three row blocks per KV head). Pages larger than the KV tile (128 with a
    64-key tile) must still give the right answer; the mma.sync kernel and the decode kernel take pages up to 64."""
    hq, hkv, d = 24, 2, 128
    seqs, nd = edge_seqs(32, page, nd=2 if page <= 64 else 0)
    b = make_paged_batch(seqs, hq, hkv, d, page, seed=page + kv, device=_dev(), nd=nd)
    kinds = [f"tc{kv}"] + (["mma"] if page <= 64 and kv == 64 else [])
    _attn_case(b, kinds, monkeypatch)


@pytest.mark.parametrize("g", [1, 6])
def test_prefill_monotone_keys(g, monkeypatch):
    """Scores rising with key position: a causal leak of one key or a skipped O rescale (alpha) moves a row far
    beyond the bound; the running max changes on every KV tile."""
    hkv = 2
    seqs = [(0, 1), (300, 1), (0, 300), (130, 129), (1000, 77), (64, 64), (0, 1), (127, 129)]
    b = make_paged_batch(seqs, g * hkv, hkv, 128, 16, seed=g, device=_dev(), nd=2)
    set_monotone(b)
    _attn_case(b, ALL_KINDS, monkeypatch)


def test_prefill_peaked_logits(monkeypatch):
    """A sink key near +30 and scaled logits out to about +-80: finite, within the bound."""
    seqs = [(0, 1), (500, 1), (0, 257), (2000, 100), (31, 33)]
    b = make_paged_batch(seqs, 8, 2, 128, 16, seed=3, device=_dev(), nd=2)
    scale = set_peaked(b, seed=4)
    _attn_case(b, ALL_KINDS, monkeypatch, scale=scale)


@pytest.mark.parametrize("content", ["random", "monotone"])
def test_prefill_long_context(content, monkeypatch):
    """Contexts past 4096 keys with a short last chunk (and one chunk just over a query tile)."""
    seqs = [(4100, 37), (4095, 130), (4097, 1)]
    b = make_paged_batch(seqs, 16, 2, 128, 16, seed=11, device=_dev())
    if content == "monotone":
        set_monotone(b, lam=0.05)
    _attn_case(b, ALL_KINDS, monkeypatch)


@pytest.mark.parametrize("splits", [None, 1, 3])
@pytest.mark.parametrize("page", [8, 32, 64])
def test_decode_split_kv(page, splits, monkeypatch):
    """Split-KV decode kernel (+ merge), per-row bound, poisoned tails / unlisted pages, lengths at page +-1."""
    seqs = [(c, 1) for c in (0, 6, 7, 8, 30, 31, 32, 62, 63, 64, 299, 2048)]
    b = make_paged_batch(seqs, 32, 4, 128, page, seed=page, device=_dev(), nd=len(seqs))
    scale = 1.0 / math.sqrt(128)
    o = run_attention("tc64", b, monkeypatch, splits=splits)
    assert torch.isfinite(o.float()).all()
    o64, pv = attn_oracle(q_view(b), b["kc"], b["vc"], b["bt"], b["sl"], b["qsl"], 32, 128, scale)
    rep = attn_report(o, o64, pv, b["qsl"], 32, 128, what=f"decode page={page} splits={splits}")
    assert rep is None, rep
