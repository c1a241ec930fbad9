"""Element-wise edge tests of the decode path against float64 oracles (`pytest -m gpu`, one H100): the split-KV GQA
decode kernel with both split merges (the merge kernel and the in-kernel last-arriver merge), the same kernel under
CUDA-graph replay, D = 256 mixed batches, MLA latent attention, and the two KV-cache writers (`rope_kv_write`,
`mla_rope_cache`).

Attention outputs are compared per (token, head) row with the bound of tests/test_wgmma_edges_gpu.py; outputs are
pre-filled with NaN so a row no CTA writes fails too. The writers are compared element by element, the cache bit for
bit: written slots against the kernel's own q/k output (or the exact input), every other slot against a snapshot.
tests/test_decode_edges_cpu.py shows on emulated kernels that these comparators reject the slips they are meant to
catch.
"""
import math

import pytest
import torch

from gllm_b200.ops import ref
from test_wgmma_edges_gpu import (ATTN_C, POISON, U_BF16, U_FP32, _worst, attn_oracle, attn_report, edge_seqs,
                                  make_paged_batch, poison_tail, q_view, scatter_seq, set_monotone, set_peaked)

pytestmark = pytest.mark.gpu


def _dev():
    return torch.device("cuda:0")


def _sm100():
    from gllm_b200.ops import sm100
    return sm100


# ----------------------------------------------------------------------------------------------------------------
# GQA decode: helpers
# ----------------------------------------------------------------------------------------------------------------
def decode_gp(g):
    """Query heads per decode CTA (GP): the largest divisor of G that is at most 16; G / GP CTAs share a KV head."""
    return max(x for x in range(1, min(g, 16) + 1) if g % x == 0)


def decode_lengths(page):
    """seq_len at 1, page -1 / 0 / +1, the 64-key tile +-1, two tiles +-1 and one long context."""
    return sorted({1, page - 1, page, page + 1, 63, 64, 65, 127, 129, 4097})


def decode_batch(lengths, g, d, page, seed, hkv=2, device=None):
    seqs = [(n - 1, 1) for n in lengths]
    return make_paged_batch(seqs, g * hkv, hkv, d, page, seed=seed, device=device or _dev(), nd=len(seqs))


def split_counters():
    """The arrival counters of the in-kernel split merge (only present once the fused merge has run)."""
    return [v for k, v in _sm100()._attn_ws.items() if k[1] == "split_cnt"]


def assert_counters_at_rest():
    for c in split_counters():
        n = int((c != 0).sum())
        assert n == 0, f"{n} split-merge arrival counters left armed (first at {int(torch.nonzero(c)[0])})"


def nan_out(t, hq, d):
    return torch.full((t, hq * d), math.nan, dtype=torch.bfloat16, device=_dev())


def run_decode(b, splits, scale=None, out=None):
    """All sequences of b are decode sequences; returns the output (NaN-filled before the call)."""
    sm100 = _sm100()
    n, hq, d = len(b["seqs"]), b["hq"], b["d"]
    scale = scale if scale is not None else 1.0 / math.sqrt(d)
    out = nan_out(n, hq, d) if out is None else out
    sm100.paged_attention(q_view(b), b["kc"], b["vc"], b["bt"], b["sl"], b["qsl"], scale, hq, d, n, n, 1,
                          int(b["sl"].max()), out=out, splits=splits)
    torch.cuda.synchronize()
    assert_counters_at_rest()
    return out


def decode_report(b, o, splits, scale=None, what="decode"):
    """attn_report per (sequence, head) row, plus the worst sequence's length and how its KV tiles split."""
    hq, d = b["hq"], b["d"]
    scale = scale if scale is not None else 1.0 / math.sqrt(d)
    o64, pv = attn_oracle(q_view(b), b["kc"], b["vc"], b["bt"], b["sl"], b["qsl"], hq, d, scale)
    rep = attn_report(o, o64, pv, b["qsl"], hq, d, decode_gp(hq // b["hkv"]), what=what)
    if rep is None:
        return None
    seq = int(rep.split("worst at sequence ")[1].split(",")[0])
    n = int(b["sl"][seq])
    tiles = -(-n // 64)
    s = splits if splits is not None else _sm100().decode_splits(len(b["seqs"]), b["hkv"], hq, int(b["sl"].max()))
    tps = -(-tiles // s)
    return rep + f" [seq_len {n}: {tiles} KV tiles, {s} splits of {tps} tiles]"


def _decode_case(b, splits, content, seed, what):
    scale = None
    if content == "monotone":
        set_monotone(b)
    elif content == "peaked":
        scale = set_peaked(b, seed)
    o = run_decode(b, splits, scale)
    return decode_report(b, o, splits, scale, what=f"{what} {content}")


# ----------------------------------------------------------------------------------------------------------------
# 1. GQA decode matrix
# ----------------------------------------------------------------------------------------------------------------
G_ALL = [1, 2, 3, 5, 6, 7, 8, 12, 16, 20, 24, 32]


@pytest.mark.parametrize("g", G_ALL)
def test_decode_gqa_ratios(g):
    """Every GQA ratio at D = 128, page 16: GP in {1, 2, 3, 5, 6, 7, 8, 12, 16, 10}, and G = 20 / 24 / 32 put two
    head groups on one KV head (the kvh / hbase mapping). Random, monotone and peaked content."""
    reps = []
    for i, content in enumerate(("random", "monotone", "peaked")):
        b = decode_batch(decode_lengths(16), g, 128, 16, seed=g * 10 + i)
        reps.append(_decode_case(b, None, content, g + i, f"decode G={g}"))
    reps = [r for r in reps if r]
    assert not reps, "\n".join(reps)


@pytest.mark.parametrize("g", [6, 24])
@pytest.mark.parametrize("page", [8, 16, 32, 64])
@pytest.mark.parametrize("d", [64, 128, 256])
def test_decode_dims_pages(d, page, g):
    """Every head dim x page size, at one G <= 16 (GP 6) and one G > 16 (GP 12, two groups per KV head)."""
    b = decode_batch(decode_lengths(page), g, d, page, seed=d + page + g)
    rep = _decode_case(b, None, "random", 0, f"decode D={d} page={page} G={g}")
    assert rep is None, rep


# ----------------------------------------------------------------------------------------------------------------
# 2. split counts, both merge paths
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fused", [False, True], ids=["merge_kernel", "fused_merge"])
@pytest.mark.parametrize("splits", [1, 2, 3, 16, None])
@pytest.mark.parametrize("d", [64, 128, 256])
def test_decode_splits(d, splits, fused, monkeypatch):
    """Every split count at every head dim (G = 20: two head groups per KV head), random and monotone content.
    Lengths below 64 x splits leave splits empty (LSE -inf). The fused merge must leave its counters at zero."""
    monkeypatch.setattr(_sm100(), "_FUSED_MERGE", fused)
    reps = []
    for i, content in enumerate(("random", "monotone")):
        b = decode_batch(decode_lengths(16), 20, d, 16, seed=d * 3 + (splits or 0) + i)
        reps.append(_decode_case(b, splits, content, i, f"decode D={d} splits={splits} fused={fused}"))
    reps = [r for r in reps if r]
    assert not reps, "\n".join(reps)


def test_fused_merge_rearms_across_calls(monkeypatch):
    """Back-to-back calls that change the batch size, the GQA ratio and the split count: a counter left armed by
    one call would make the next call's merge fire early (or never). Each output against the oracle, and the first
    batch again, bit for bit."""
    monkeypatch.setattr(_sm100(), "_FUSED_MERGE", True)
    a = decode_batch([4097, 1, 65, 129, 700, 64, 2, 300, 63, 1000, 17, 4000], 24, 128, 16, seed=1)
    bb = decode_batch([129, 3000, 1, 64, 65], 8, 128, 16, seed=2)
    c = decode_batch([2049, 5, 4097, 128, 33, 1, 640], 20, 128, 32, seed=3)
    plan = [(a, 3), (bb, 16), (c, 2), (bb, 5), (a, 16), (c, 16), (a, 3)]
    reps, first = [], None
    for i, (b, s) in enumerate(plan):
        o = run_decode(b, s)
        reps.append(decode_report(b, o, s, what=f"call {i} (bs={len(b['seqs'])}, splits={s})"))
        if i == 0:
            first = o.clone()
    assert torch.equal(o, first), "the first batch gave a different result when repeated"
    reps = [r for r in reps if r]
    assert not reps, "\n".join(reps)


# ----------------------------------------------------------------------------------------------------------------
# 3. CUDA-graph replay
# ----------------------------------------------------------------------------------------------------------------
def _capture(fn):
    """Warm up on a side stream, then capture fn() (as the model runner does); returns (graph, fn's result)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        res = fn()
    torch.cuda.synchronize()
    return g, res


class _Static:
    """Fixed-address q / cache / block-table / seq_lens buffers that batches are copied into between replays.
    Pages a batch does not use hold POISON; the last page is the graph-padding dummy page (random content)."""

    def __init__(self, bs, hq, hkv, d, page, n_pages, max_blocks):
        dev = _dev()
        self.hq, self.hkv, self.d, self.page, self.n_pages = hq, hkv, d, page, n_pages
        self.dummy = n_pages - 1
        self.qkv = torch.zeros(bs, (hq + 2 * hkv) * d, dtype=torch.bfloat16, device=dev)
        shape = ref.kv_cache_shape(n_pages, hkv, d, page)
        self.kc = torch.zeros(shape, dtype=torch.bfloat16, device=dev)
        self.vc = torch.zeros(shape, dtype=torch.bfloat16, device=dev)
        self.bt = torch.zeros(bs, max_blocks, dtype=torch.int32, device=dev)
        self.sl = torch.ones(bs, dtype=torch.int32, device=dev)
        self.qsl = torch.arange(bs + 1, dtype=torch.int32, device=dev)

    def load(self, b, rows=None, pad_rows=()):
        """Copy batch b in. rows: the rows taken from b (default all); pad_rows: rows laid out as graph padding
        (seq_len 1 on the dummy page, only block-table column 0 rewritten, the rest left stale)."""
        rows = list(range(len(b["seqs"]))) if rows is None else rows
        np_ = b["kc"].shape[0]
        assert np_ < self.dummy
        for cache, src in ((self.kc, b["kc"]), (self.vc, b["vc"])):
            cache.fill_(POISON)
            cache[:np_].copy_(src)
            cache[self.dummy].copy_(torch.randn(cache[self.dummy].shape, device=cache.device) * 0.5)
        self.qkv.copy_(b["qkv"])
        for r in rows:
            self.bt[r].fill_(b["unlisted"][0])
            self.bt[r, : b["bt"].shape[1]].copy_(b["bt"][r])
            self.sl[r] = b["sl"][r]
        for r in pad_rows:
            self.bt[r, 0] = self.dummy
            self.sl[r] = 1

    def batch(self, seqs):
        return dict(qkv=self.qkv, kc=self.kc, vc=self.vc, bt=self.bt, sl=self.sl, qsl=self.qsl, seqs=seqs,
                    nd=len(seqs), hq=self.hq, hkv=self.hkv, d=self.d, page=self.page)


GRAPH_BS = 8
GRAPH_CAPTURE = [100, 200, 300, 64, 65, 129, 1, 17]
GRAPH_LONG = [4097, 3000, 2049, 1025, 4096, 513, 65, 4000]      # longer than anything seen at capture
GRAPH_SHORT = [1, 2, 3, 5, 8, 17, 33, 64]                       # one KV tile each: 15 of 16 splits empty
GRAPH_PADDED = [700, 1, 129, 64, 4097]                          # + 3 padding rows


@pytest.mark.parametrize("fused", [False, True], ids=["merge_kernel", "fused_merge"])
def test_decode_graph_replay(fused, monkeypatch):
    """paged_attention captured the way capture_graphs does it (workspace reserved first, splits from
    decode_splits(bs, Hkv, Hq, 32768)), then replayed with the static buffers rewritten in place: longer contexts
    than at capture, much shorter ones, and a batch padded like pad_for_graph. Every replay checked per row."""
    sm100 = _sm100()
    monkeypatch.setattr(sm100, "_FUSED_MERGE", fused)
    hq, hkv, d, page, bs = 48, 2, 128, 16, GRAPH_BS
    sm100.reserve_attn_workspace(_dev(), bs, hq, d)
    splits = sm100.decode_splits(bs, hkv, hq, 32768)
    assert splits == 16
    st = _Static(bs, hq, hkv, d, page, n_pages=bs * (4097 // page + 2) + 8, max_blocks=4097 // page + 2)
    b0 = decode_batch(GRAPH_CAPTURE, hq // hkv, d, page, seed=0, hkv=hkv)
    st.load(b0)
    out = nan_out(bs, hq, d)
    scale = 1.0 / math.sqrt(d)

    def fn():
        return sm100.paged_attention(q_view(st.batch([])), st.kc, st.vc, st.bt, st.sl, st.qsl, scale, hq, d, bs, bs,
                                     1, 32768, out=out, splits=splits)

    graph, _ = _capture(fn)
    assert_counters_at_rest()
    reps = [decode_report(st.batch(b0["seqs"]), out, splits, what="capture")]
    cases = [("longer", GRAPH_LONG, None), ("shorter", GRAPH_SHORT, None),
             ("padded", GRAPH_PADDED + [1] * (bs - len(GRAPH_PADDED)), range(len(GRAPH_PADDED), bs))]
    for i, (name, lens, pad) in enumerate(cases):
        b = decode_batch(lens, hq // hkv, d, page, seed=i + 1, hkv=hkv)
        if name != "shorter":
            set_monotone(b)
        if pad is None:
            st.load(b)
        else:
            st.load(b, rows=range(len(GRAPH_PADDED)), pad_rows=pad)
        out.fill_(math.nan)
        graph.replay()
        torch.cuda.synchronize()
        assert_counters_at_rest()
        reps.append(decode_report(st.batch(b["seqs"]), out, splits, what=f"replay {name}"))
    reps = [r for r in reps if r]
    assert not reps, "\n".join(reps)


# ----------------------------------------------------------------------------------------------------------------
# 4. D = 256 mixed batch (the wgmma prefill kernel declines it; the mma.sync kernel serves the prefill chunks)
# ----------------------------------------------------------------------------------------------------------------
def _prefill_gp(g):
    return max(x for x in range(1, min(g, 64) + 1) if g % x == 0 and 64 % x == 0)


@pytest.mark.parametrize("g", [1, 5, 20])
def test_d256_mixed_batch(g, monkeypatch):
    """Decode rows then prefill chunks at D = 256: q_len / context around the mma.sync query tile and the KV tile,
    per row against the oracle, through the default route (wgmma first) and with the mma.sync kernel forced."""
    from gllm_b200.ops import lib
    sm100 = _sm100()
    hkv, d, page = 2, 256, 16
    seqs, nd = edge_seqs(64 // _prefill_gp(g), page, kv_tiles=(64,), nd=2)
    b = make_paged_batch(seqs, g * hkv, hkv, d, page, seed=g, device=_dev(), nd=nd)
    n = len(seqs)
    max_q = max(ql for _, ql in seqs[nd:])
    scale = 1.0 / math.sqrt(d)
    rc = lib.load().gllm_attn_prefill_tc(
        sm100._p(q_view(b)), q_view(b).stride(0), sm100._p(nan_out(q_view(b).shape[0], g * hkv, d)), sm100._p(b["kc"]), sm100._p(b["vc"]),
        b["kc"].shape[0], sm100._p(b["bt"]), sm100._p(b["sl"]), sm100._p(b["qsl"]), n - nd, nd, max_q,
        b["bt"].shape[1], g * hkv, hkv, d, page, float(scale), 64, sm100.stream_ptr())
    assert rc == 2, f"the wgmma prefill kernel accepted D = 256 (rc {rc})"
    o64, pv = attn_oracle(q_view(b), b["kc"], b["vc"], b["bt"], b["sl"], b["qsl"], g * hkv, d, scale)
    reps = []
    for tc in (True, False):
        monkeypatch.setattr(sm100, "ATTN_TC", tc)
        out = nan_out(q_view(b).shape[0], g * hkv, d)
        sm100.paged_attention(q_view(b), b["kc"], b["vc"], b["bt"], b["sl"], b["qsl"], scale, g * hkv, d, nd, n,
                              max_q, int(b["sl"].max()), out=out)
        torch.cuda.synchronize()
        reps.append(attn_report(out, o64, pv, b["qsl"], g * hkv, d, _prefill_gp(g),
                                what=f"D=256 G={g} ATTN_TC={tc}"))
    reps = [r for r in reps if r]
    assert not reps, "\n".join(reps)


# ----------------------------------------------------------------------------------------------------------------
# 5. MLA latent attention
# ----------------------------------------------------------------------------------------------------------------
# The bound is attn_report's: |o - o64| <= ATTN_C 2^-9 (P |V|) + 2^-9 |o64| per (token, head) row.
#   Does ATTN_C = 4 still cover S = q . latent accumulated over k = 576 instead of D <= 256? Half of ATTN_C pays for
#   the bf16 P; the other 2 x 2^-9 (P|V|) = 2^-8 (P|V|) must cover the logit errors delta_j, which move o by at most
#   2 max|delta| (P|V|), plus the fp32 row sum l and the O accumulation (n 2^-24 relative each, 2^-11 together at
#   n = 4100 keys). So max|delta| <= (2^-8 - 2^-11) / 2 = 7 x 2^-12. With the GEMMs' worst case for the fp32
#   tensor-core sum (GEMM_C k 2^-24 = 4 k 2^-24 of A = scale sum_i |q_i lat_i|), that holds for A <= 12.4 at
#   k = 576 (A <= 56 at D = 128): the bound is 4.5 times tighter on A. Products that are exactly zero add nothing,
#   so k counts the nonzero products only. The inputs below keep inside it:
#     random  : q ~ 0.3 N(0,1), latent ~ 0.5 N(0,1), scale 192^-0.5: A = 0.072 x 576 x 0.3 x 0.5 x 2/pi = 4;
#     monotone: two nonzero products of small integers per key, summed exactly (delta = 0);
#     peaked  : the scores live on the 64 rope columns (q's first 512 columns are zero): k = 64 nonzero products,
#               for which the same budget admits A <= 112 (A is about 100 for a typical key here).
#   ATTN_C therefore covers MLA as it is; no constant was changed for it.
MLA_SCALE = 192 ** -0.5


def make_mla_batch(seqs, h, page, seed, device=None, q_scale=0.3, lat_scale=0.5):
    """seqs: [(context, q_len)]; the tokens of sequence s sit at positions context .. context + q_len - 1 and
    attend to keys [0, position]. Random bf16 q [T, H, 576] and latent cache [pages, 1, 9, page, 64]; slots past
    every sequence's last key and three unlisted pages hold POISON, block-table padding points at one of them."""
    device = device or _dev()
    b = make_paged_batch([(c, ql) for c, ql in seqs], 1, 1, 576, page, seed=seed, device=device,
                         q_scale=q_scale, kv_scale=lat_scale)
    g = torch.Generator().manual_seed(seed + 7)
    b["vc"] = b["kc"]                             # one latent cache: poison_tail writes it (twice)
    t = sum(ql for _, ql in seqs)
    b["q"] = (torch.randn(t, h, 576, generator=g) * q_scale).bfloat16().to(device)
    b["h"] = h
    b["tok_seq"] = torch.tensor(sum(([i] * ql for i, (_, ql) in enumerate(seqs)), []), dtype=torch.int32,
                                device=device)
    b["pos"] = torch.tensor(sum((list(range(c, c + ql)) for c, ql in seqs), []), dtype=torch.int32, device=device)
    poison_tail(b)
    return b


def mla_decode_batch(lengths, h, page, seed):
    return make_mla_batch([(n - 1, 1) for n in lengths], h, page, seed)


def _mla_rows(b, s):
    """The latent rows [0, seq_len) of sequence s as float32 on the CPU [n, 576], and n."""
    n = int(b["sl"][s])
    return ref.gather_kv(b["kc"], b["bt"][s], n)[:, 0].float().cpu(), n


def set_mla_monotone(b, lam=0.25):
    """Scores rising with key position on the rope columns: latent j carries (j // 256, j % 256) in columns 512, 513
    and zeros in the other rope columns (its 512 value columns stay random); head h's q is zero except
    (256 s_h, s_h) there, so q . latent_j = s_h j exactly with s_h * scale = lam * (1, 1.5, 2)[h % 3]. The tile max
    sits in the last warp's 16 keys of every tile, so a warp that skipped the shared max would use its own."""
    h = b["h"]
    for s in range(len(b["seqs"])):
        rows, n = _mla_rows(b, s)
        j = torch.arange(n, dtype=torch.float32)
        rows[:, 512:] = 0
        rows[:, 512], rows[:, 513] = j // 256, j % 256
        scatter_seq(b["kc"], b["bt"][s], b["page"], rows.view(n, 1, 576))
    q = torch.zeros(b["q"].shape)
    for hh in range(h):
        sh = float(torch.tensor(lam * (1.0, 1.5, 2.0)[hh % 3] / MLA_SCALE).bfloat16())
        q[:, hh, 512], q[:, hh, 513] = 256.0 * sh, sh
    b["q"].copy_(q.bfloat16())
    poison_tail(b)
    return MLA_SCALE


def set_mla_peaked(b, seed):
    """Peaked logits on the rope columns: q's 512 latent columns are zero, its rope part 0.6 z + c (c shared by all
    heads); the keys' rope parts are N(0, 1) except key 0 of every sequence (a sink), c 30 / (scale 64), whose
    scaled logit sits near +30. scale = 20 / sqrt(1.36 x 64): logits spread about 20, extremes near +-80."""
    g = torch.Generator().manual_seed(seed)
    scale = 20.0 / math.sqrt(1.36 * 64)
    c = torch.randn(64, generator=g)
    t, h = b["q"].shape[:2]
    q = torch.zeros(t, h, 576)
    q[:, :, 512:] = 0.6 * torch.randn(t, h, 64, generator=g) + c
    b["q"].copy_(q.bfloat16())
    for s in range(len(b["seqs"])):
        rows, n = _mla_rows(b, s)
        rows[:, 512:] = torch.randn(n, 64, generator=g)
        rows[0, 512:] = c * (30.0 / (scale * 64))
        scatter_seq(b["kc"], b["bt"][s], b["page"], rows.view(n, 1, 576))
    poison_tail(b)
    return scale


def mla_oracle(q, cache, bt, tok_seq, positions, scale, head_chunk=32):
    """float64 MLA of the exact bf16 inputs: token i of block-table row tok_seq[i] (i when None) attends to latent
    rows [0, positions[i]]; keys are the 576-wide rows, values their first 512 columns. Returns (o64, P |V|)
    [T, H, 512]."""
    t, h, _ = q.shape
    o64 = torch.zeros(t, h, 512, dtype=torch.float64, device=q.device)
    pv = torch.zeros_like(o64)
    seqs = tok_seq.tolist() if tok_seq is not None else list(range(t))
    pos = positions.tolist()
    groups = {}
    for i, s in enumerate(seqs):
        groups.setdefault(s, []).append(i)
    for s, toks in groups.items():
        n = max(pos[i] for i in toks) + 1
        lat = ref.gather_kv(cache, bt[s], n)[:, 0].double()                  # [n, 576]
        v = lat[:, :512]
        ti = torch.tensor(toks, device=q.device)
        mask = torch.arange(n, device=q.device).view(1, n) > torch.tensor([pos[i] for i in toks],
                                                                           device=q.device).view(-1, 1)
        for h0 in range(0, h, head_chunk):
            h1 = min(h, h0 + head_chunk)
            logits = torch.einsum("thc,kc->thk", q[ti, h0:h1].double(), lat) * scale
            p = torch.softmax(logits.masked_fill(mask.unsqueeze(1), -math.inf), dim=-1)
            o64[ti, h0:h1] = p @ v
            pv[ti, h0:h1] = p @ v.abs()
    return o64, pv


def mla_report(o, o64, pv, tok_seq, positions, what="mla"):
    """None when every (token, head) row is within the attention bound, else the worst token (its sequence and
    position), head (and its 16-head CTA block) and value column (and the warp that owns it)."""
    err = (o.double() - o64).abs()
    bound = ATTN_C * 2.0 ** -9 * pv + 2.0 ** -9 * o64.abs()
    n_bad, idx = _worst(err, bound)
    if n_bad == 0:
        return None
    i, h, c = idx
    s = int(tok_seq[i]) if tok_seq is not None else i
    return (f"{what}: {n_bad} of {err.numel()} values outside the bound; worst at token {i} (sequence {s}, "
            f"position {int(positions[i])}), head {h} (16-head block {h // 16}), col {c} (value warp {c // 128}): "
            f"got {float(o[i, h, c]):.6g}, want {float(o64[i, h, c]):.6g}, |err| {float(err[i, h, c]):.3g} > "
            f"bound {float(bound[i, h, c]):.3g}")


def run_mla(b, splits, scale=MLA_SCALE, tok_seq=True):
    sm100 = _sm100()
    ts = b["tok_seq"] if tok_seq else None
    o = sm100.mla_attention(b["q"], b["kc"], b["bt"], ts, b["pos"], scale, splits=splits)
    torch.cuda.synchronize()
    return o


def mla_case(b, splits, scale=MLA_SCALE, what="mla", tok_seq=True):
    o = run_mla(b, splits, scale, tok_seq)
    o64, pv = mla_oracle(b["q"], b["kc"], b["bt"], b["tok_seq"], b["pos"], scale)
    return mla_report(o, o64, pv, b["tok_seq"], b["pos"], what=what)


def mla_lengths(page):
    """kv_len at 1 (position 0), page -1 / 0 / +1, the 64-key tile +-1, two tiles +-1 and 4100."""
    return sorted({1, page - 1, page, page + 1, 63, 64, 65, 127, 128, 129, 4100})


@pytest.mark.parametrize("h", [8, 16, 20, 40, 64, 128])
def test_mla_heads(h):
    """Head counts of one to eight 16-head blocks, 20 and 40 with a partial last block; random and monotone
    content; decode tokens without tok_seq (the token index is the block-table row)."""
    reps = []
    for i, content in enumerate(("random", "monotone")):
        b = mla_decode_batch(mla_lengths(16), h, 16, seed=h + i)
        scale = set_mla_monotone(b) if content == "monotone" else MLA_SCALE
        reps.append(mla_case(b, None, scale, what=f"mla H={h} {content}", tok_seq=False))
    reps = [r for r in reps if r]
    assert not reps, "\n".join(reps)


@pytest.mark.parametrize("splits", [1, 2, 3, 16, None])
@pytest.mark.parametrize("page", [8, 16, 32, 64])
def test_mla_pages_splits(page, splits):
    """Every page size x split count (H = 20), random and monotone content; lengths below 64 x splits leave splits
    empty; poisoned tails and unlisted pages."""
    reps = []
    for i, content in enumerate(("random", "monotone")):
        b = mla_decode_batch(mla_lengths(page), 20, page, seed=page * 7 + (splits or 0) + i)
        scale = set_mla_monotone(b) if content == "monotone" else MLA_SCALE
        reps.append(mla_case(b, splits, scale, what=f"mla page={page} splits={splits} {content}"))
    reps = [r for r in reps if r]
    assert not reps, "\n".join(reps)


@pytest.mark.parametrize("h", [16, 40])
def test_mla_peaked(h):
    """A sink key near +30 and scaled logits out to about +-80 on the rope columns."""
    b = mla_decode_batch(mla_lengths(32), h, 32, seed=5)
    scale = set_mla_peaked(b, seed=6)
    rep = mla_case(b, None, scale, what=f"mla peaked H={h}")
    assert rep is None, rep


def test_mla_forced_split_clamp():
    """A caller-forced split count that the workspace cannot hold (3 tokens x 128 heads x 16 splits > 296 x 16
    rows) is clamped (to 12) instead of overrunning the partials."""
    t, h, splits = 3, 128, 16
    cap = max(296 * 16, 16 * h)
    assert t * h * splits > cap and cap // (t * h) == 12
    b = mla_decode_batch([4100, 1, 769], h, 16, seed=9)
    set_mla_monotone(b, lam=0.05)
    rep = mla_case(b, splits, what="mla forced splits=16")
    assert rep is None, rep


@pytest.mark.parametrize("splits", [None, 3])
def test_mla_mixed_batch(splits):
    """Decode tokens, then prefill chunks with prefix context (tok_seq selects the block-table row; every token
    attends to its own causal prefix), at tile and page edges."""
    seqs = [(0, 1), (4099, 1), (63, 1), (0, 65), (64, 64), (127, 3), (1000, 130), (15, 17), (4000, 40)]
    reps = []
    for i, content in enumerate(("random", "monotone")):
        b = make_mla_batch(seqs, 16, 16, seed=11 + i)
        scale = set_mla_monotone(b, lam=0.05) if content == "monotone" else MLA_SCALE
        reps.append(mla_case(b, splits, scale, what=f"mla mixed splits={splits} {content}"))
    reps = [r for r in reps if r]
    assert not reps, "\n".join(reps)


def test_mla_graph_replay():
    """mla_attention captured with splits from mla_splits(bs, H) and replayed with q, block table and positions
    rewritten in place: longer contexts, shorter ones, a pad_for_graph layout (position 0 on the dummy page)."""
    sm100 = _sm100()
    h, page, bs = 20, 16, GRAPH_BS
    sm100.reserve_attn_workspace(_dev(), bs, h, 576)
    splits = sm100.mla_splits(bs, h)
    assert splits == 16
    max_blocks = 4097 // page + 2
    st = _Static(bs, 1, 1, 576, page, n_pages=bs * max_blocks + 8, max_blocks=max_blocks)
    q = torch.zeros(bs, h, 576, dtype=torch.bfloat16, device=_dev())
    pos = torch.zeros(bs, dtype=torch.int32, device=_dev())

    def load(b, rows=None, pad_rows=()):
        st.load(b, rows, pad_rows)
        q.copy_(b["q"])
        pos.copy_(st.sl - 1)

    def fn():
        return sm100.mla_attention(q, st.kc, st.bt, None, pos, MLA_SCALE, splits=splits)

    load(mla_decode_batch(GRAPH_CAPTURE, h, page, seed=0))
    graph, out = _capture(fn)
    reps = []
    cases = [("longer", GRAPH_LONG, None), ("shorter", GRAPH_SHORT, None),
             ("padded", GRAPH_PADDED + [1] * (bs - len(GRAPH_PADDED)), range(len(GRAPH_PADDED), bs))]
    for i, (name, lens, pad) in enumerate(cases):
        b = mla_decode_batch(lens, h, page, seed=i + 1)
        if name != "shorter":
            set_mla_monotone(b)
        if pad is None:
            load(b)
        else:
            load(b, rows=range(len(GRAPH_PADDED)), pad_rows=pad)
        out.fill_(math.nan)
        graph.replay()
        torch.cuda.synchronize()
        o64, pv = mla_oracle(q, st.kc, st.bt, None, pos, MLA_SCALE)
        reps.append(mla_report(out, o64, pv, None, pos, what=f"mla replay {name}"))
    reps = [r for r in reps if r]
    assert not reps, "\n".join(reps)


# ----------------------------------------------------------------------------------------------------------------
# 6. KV-cache writers
# ----------------------------------------------------------------------------------------------------------------
def rope_pairs(d, rot, neox):
    """(first, second) element index of every rotary pair i < rot / 2: NeoX pairs (i, i + rot/2), GPT-J (2i, 2i+1)."""
    i = torch.arange(rot // 2)
    return (i, i + rot // 2) if neox else (2 * i, 2 * i + 1)


def rope_oracle(x, cos, sin, rot, neox, x_step=None):
    """float64 rotation of x [T, H, D] (exact bf16 inputs, or the bf16 normed values) with cos / sin [T, rot/2]
    (the fp32 table's values). Returns (y64, bound): one bf16 rounding of the fp32 rotation, whose error is at most
    4 x 2^-24 (|a c| + |b s|) per element; x_step [T, H, D] (optional) is how far the kernel's input may sit from x
    (one bf16 step where the kernel rounds its own normed value), carried through |c| and |s|. The bound is
    U_BF16 |y64| + 2 (rotation error + carried input step): twice the error before the final rounding covers it."""
    x = x.double()
    a_i, b_i = rope_pairs(x.shape[-1], rot, neox)
    y = x.clone()
    c, s = cos.double().unsqueeze(1), sin.double().unsqueeze(1)
    a, b = x[..., a_i], x[..., b_i]
    y[..., a_i] = a * c - b * s
    y[..., b_i] = b * c + a * s
    e = torch.zeros_like(x)
    e[..., a_i] = 4 * U_FP32 * (a.abs() * c.abs() + b.abs() * s.abs())
    e[..., b_i] = e[..., a_i]
    if x_step is not None:
        st = x_step.double()
        carried = st.clone()
        sa, sb = st[..., a_i], st[..., b_i]
        carried[..., a_i] = sa * c.abs() + sb * s.abs()
        carried[..., b_i] = sb * c.abs() + sa * s.abs()
        e = e + carried
    return y, U_BF16 * y.abs() + 2 * e


def elem_report(y, y64, bound, names=("token", "head", "dim"), what="rope"):
    err = (y.double() - y64).abs()
    n_bad, idx = _worst(err, bound)
    if n_bad == 0:
        return None
    where = ", ".join(f"{n} {i}" for n, i in zip(names, idx))
    return (f"{what}: {n_bad} of {err.numel()} values outside the bound; worst at {where}: got {float(y[idx]):.6g}, "
            f"want {float(y64[idx]):.6g}, |err| {float(err[idx]):.3g} > bound {float(bound[idx]):.3g}")


def cache_rows(cache, slots):
    """[n, Hkv, D] rows of the paged cache at the given slots (all >= 0)."""
    page = cache.shape[3]
    s = slots.long()
    rows = cache[s // page, :, :, s % page, :]                             # [n, Hkv, D/64, 64]
    return rows.reshape(rows.shape[0], rows.shape[1], -1)


def untouched_report(cache, snap, slots, what):
    """Every (page, offset) slot not in `slots` (>= 0 entries) is bit-identical to the snapshot."""
    page = cache.shape[3]
    mask = torch.ones(cache.shape[0], page, dtype=torch.bool, device=cache.device)
    s = slots[slots >= 0].long()
    mask[s // page, s % page] = False
    a = cache.view(torch.int16).permute(0, 3, 1, 2, 4)[mask]
    b = snap.view(torch.int16).permute(0, 3, 1, 2, 4)[mask]
    bad = int((a != b).flatten(1).any(1).sum())
    return None if bad == 0 else f"{what}: {bad} cache slots outside `slots` were modified"


def _slots_for(t, n_pages, page, gen, skip=(1, 5)):
    """t distinct random slots, spread over the pages; the tokens in `skip` get -1 (no cache write)."""
    slots = torch.randperm(n_pages * page, generator=gen)[:t].to(torch.int32)
    for i in skip:
        if i < t:
            slots[i] = -1
    return slots


def _bits_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


@pytest.mark.parametrize("page", [8, 16, 32, 64])
def test_mla_rope_cache(page):
    """Inputs strided as the DeepSeek layer passes them: q_pe = q[:, :, nope:], k_pe and kv_c column views of the
    kv_a projection output. Rope outputs against a float64 interleaved-pair rotation, c_kv copied bit for bit,
    tokens with slot -1 write nothing, every other cache slot and q_full's latent columns unchanged."""
    sm100 = _sm100()
    dev = _dev()
    g = torch.Generator().manual_seed(page)
    t, h, qk_dim, nope, n_pages, max_pos = 37, 16, 192, 128, 40, 8192
    q = (torch.randn(t, h, qk_dim, generator=g) * 2).bfloat16().to(dev)
    kv_a = (torch.randn(t, 576, generator=g) * 2).bfloat16().to(dev)
    kv_c, k_pe = kv_a[:, :512], kv_a[:, 512:]
    pos = torch.randint(0, max_pos, (t,), generator=g, dtype=torch.int32)
    pos[0], pos[2] = 0, max_pos - 1
    slots = _slots_for(t, n_pages, page, g).to(dev)
    pos = pos.to(dev)
    cs = ref.build_cos_sin_cache(64, max_pos, 10000.0).to(dev)
    cache = (torch.randn(n_pages, 1, 9, page, 64, generator=g)).bfloat16().to(dev)
    snap = cache.clone()
    q_full = torch.randn(t, h, 576, generator=g).bfloat16().to(dev)
    q_snap = q_full.clone()
    sm100.mla_rope_cache(q[:, :, nope:], q_full, k_pe, kv_c, cs, pos, slots, cache)
    torch.cuda.synchronize()
    cos, sin = cs[pos.long(), :32], cs[pos.long(), 32:]
    reps = []
    y64, bound = rope_oracle(q[:, :, nope:], cos, sin, 64, False)
    reps.append(elem_report(q_full[:, :, 512:], y64, bound, what="q rope"))
    if not _bits_equal(q_full[:, :, :512], q_snap[:, :, :512]):
        reps.append("q_full's latent columns [0, 512) were modified")
    ok = slots >= 0
    rows = cache_rows(cache, slots[ok])[:, 0]                                # [n, 576]
    if not _bits_equal(rows[:, :512], kv_c[ok]):
        bad = torch.nonzero((rows[:, :512].view(torch.int16) != kv_c[ok].view(torch.int16)).any(1))[0].item()
        reps.append(f"c_kv not copied bit-exactly (first at written token {bad})")
    k64, kb = rope_oracle(k_pe.view(t, 1, 64), cos, sin, 64, False)
    reps.append(elem_report(rows[:, 512:].view(-1, 1, 64), k64[ok], kb[ok], what="cached k_pe rope"))
    reps.append(untouched_report(cache, snap, slots, "mla cache"))
    reps = [r for r in reps if r]
    assert not reps, "\n".join(reps)


ROPE_CASES = [(d, rot, neox, norm) for d in (64, 128, 256) for neox in (True, False)
              for rot in (d, d // 2, d // 4) for norm in (False, True)]


def _norm_bf16(x, w, eps):
    """The kernel's normed value as the oracle sees it: x rsqrt(mean x^2 + eps) w in float64, rounded to bf16,
    and the step (one bf16 ulp) by which the kernel's own fp32 rounding may differ from it."""
    x64 = x.double()
    xn = x64 * torch.rsqrt(x64.pow(2).mean(-1, keepdim=True) + eps) * w.double()
    xb = xn.bfloat16()
    return xb, xb.double().abs() * 2.0 ** -7


def rope_kv_case(t, hq, hkv, d, rot, neox, norm, page, seed, mrope=None, with_slots=True):
    sm100 = _sm100()
    dev = _dev()
    g = torch.Generator().manual_seed(seed)
    n_pages, max_pos, eps = 24, 4096, 1e-6
    width = (hq + 2 * hkv) * d
    buf = (torch.randn(t, width + 64, generator=g) * 2).bfloat16().to(dev)  # 64 guard columns per row
    snap_buf = buf.clone()
    q = buf[:, : hq * d].view(t, hq, d)
    k = buf[:, hq * d: (hq + hkv) * d].view(t, hkv, d)
    v = buf[:, (hq + hkv) * d: width].view(t, hkv, d)
    if mrope is None:
        pos = torch.randint(0, max_pos, (t,), generator=g, dtype=torch.int32)
        pos[0] = max_pos - 1
        pos_d = pos.to(dev)
    else:
        full = torch.randint(0, max_pos, (3, t + 24), generator=g, dtype=torch.int32)
        pos_d = full.to(dev)[:, :t]                                  # a view of a [3, max_tokens] buffer
        pos = full[:, :t]
    slots = _slots_for(t, n_pages, page, g).to(dev) if with_slots else None
    cs = ref.build_cos_sin_cache(rot, max_pos, 10000.0).to(dev)
    qn = (1 + 0.2 * torch.randn(d, generator=g)).bfloat16().to(dev) if norm else None
    kn = (1 + 0.2 * torch.randn(d, generator=g)).bfloat16().to(dev) if norm else None
    shape = ref.kv_cache_shape(n_pages, hkv, d, page)
    kc = torch.randn(shape, generator=g).bfloat16().to(dev)
    vc = torch.randn(shape, generator=g).bfloat16().to(dev)
    kc_snap, vc_snap = kc.clone(), vc.clone()
    q_in, k_in = q.clone(), k.clone()
    sm100.rope_kv_write(q, k, v, pos_d, cs, rot, neox, qn, kn, eps, kc if with_slots else None,
                        vc if with_slots else None, slots, mrope_section=mrope)
    torch.cuda.synchronize()

    # cos / sin per (token, pair): the position row of the pair's M-RoPE section
    half = rot // 2
    if mrope is None:
        p_pair = pos.long().view(t, 1).expand(t, half)
    else:
        axis = torch.zeros(half, dtype=torch.long)
        i = torch.arange(half)
        if len(mrope) > 3 and mrope[3]:
            axis[(i % 3 == 1) & (i < 3 * mrope[1])] = 1
            axis[(i % 3 == 2) & (i < 3 * mrope[2])] = 2
        else:
            axis[mrope[0]: mrope[0] + mrope[1]] = 1
            axis[mrope[0] + mrope[1]:] = 2
        p_pair = pos.long()[axis, :].t()                              # [t, half]
    csc = cs.cpu()
    cos = torch.gather(csc[p_pair], 2, torch.arange(half).view(1, half, 1).expand(t, half, 1))[..., 0]
    sin = torch.gather(csc[p_pair], 2, (half + torch.arange(half)).view(1, half, 1).expand(t, half, 1))[..., 0]
    cos, sin = cos.to(dev), sin.to(dev)

    reps = []
    for name, x_in, out, w in (("q", q_in, q, qn), ("k", k_in, k, kn)):
        step = None
        if w is not None:
            x_in, step = _norm_bf16(x_in, w, eps)
        y64, bound = rope_oracle(x_in, cos, sin, rot, neox, step)
        reps.append(elem_report(out, y64, bound, what=f"{name} rope"))
    what = f"D={d} rot={rot} neox={neox} norm={norm} page={page} Hq={hq} Hkv={hkv}"
    if not _bits_equal(buf[:, (hq + hkv) * d:], snap_buf[:, (hq + hkv) * d:]):
        reps.append("written outside q / k (v or the guard columns changed)")
    if with_slots:
        ok = slots >= 0
        if not _bits_equal(cache_rows(kc, slots[ok]), k[ok]):
            reps.append("k cache rows differ from the kernel's k output")
        if not _bits_equal(cache_rows(vc, slots[ok]), v[ok]):
            reps.append("v cache rows are not bit-exact copies of v")
        reps.append(untouched_report(kc, kc_snap, slots, "k cache"))
        reps.append(untouched_report(vc, vc_snap, slots, "v cache"))
    reps = [f"{what}: {r}" for r in reps if r]
    assert not reps, "\n".join(reps)


@pytest.mark.parametrize("d,rot,neox,norm", ROPE_CASES)
def test_rope_kv_write_elementwise(d, rot, neox, norm):
    """NeoX and GPT-J, full and partial rotary (rot = D, D/2, D/4: the NeoX partner sits rot/2 elements and rot/2C
    lanes away), with and without q/k-norm, at D = 64 / 128 / 256, page sizes 8 .. 64 in turn."""
    page = (8, 16, 32, 64)[(d // 64 + rot + norm) % 4]
    rope_kv_case(29, 8, 2, d, rot, neox, norm, page, seed=d + rot + 3 * neox + norm)


@pytest.mark.parametrize("mrope", [[16, 24, 24], [24, 20, 20, 1]], ids=["chunked", "interleaved"])
@pytest.mark.parametrize("norm", [False, True])
def test_rope_kv_write_mrope(mrope, norm):
    """M-RoPE, chunked [T|H|W] sections (Qwen2.5-VL) and interleaved THW (Qwen3-VL), positions a strided view."""
    rope_kv_case(33, 4, 2, 128, 128, True, norm, 16, seed=7 + norm, mrope=mrope)


@pytest.mark.parametrize("hq,hkv,with_slots", [(1, 1, True), (1, 1, False), (2, 1, False)])
@pytest.mark.parametrize("neox", [True, False])
def test_rope_kv_write_few_heads(hq, hkv, with_slots, neox):
    """Fewer than four heads in total (Hq + Hkv (+ Hkv with a V write) < 4): fewer warps per block than usual."""
    rope_kv_case(9, hq, hkv, 128, 64, neox, True, 8, seed=hq + 2 * with_slots + neox, with_slots=with_slots)
