"""sm_90a kernels vs the PyTorch fp32 oracle (runs on an H100: `pytest -m gpu`)."""
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from gllm_b200.ops import ref


def _dev():
    return torch.device("cuda:0")


def _rel_err(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


@pytest.mark.parametrize("m,n,k", [(128, 256, 64), (1, 512, 128), (37, 384, 192), (256, 6144, 4096),
                                   (1000, 4096, 4096), (2048, 24576, 4096), (5, 151936, 1024),
                                   (130, 72, 320)])
@pytest.mark.parametrize("bn", [0, 32, 64, 128, 256])
def test_gemm_bf16(m, n, k, bn, monkeypatch):
    from gllm_b200.ops import sm100
    if bn and m * n * k > 2e10:
        pytest.skip("big shape only with auto tile")
    monkeypatch.setattr(sm100, "_FORCE_BN", bn)
    torch.manual_seed(0)
    x = (torch.randn(m, k, device=_dev()) * 0.5).bfloat16()
    w = (torch.randn(n, k, device=_dev()) * 0.05).bfloat16()
    y = sm100.linear(x, w)
    torch.cuda.synchronize()
    yr = x.float() @ w.float().t()
    assert _rel_err(y, yr) < 6e-3, _rel_err(y, yr)
    assert torch.isfinite(y.float()).all()


def test_gemm_bias_and_strided():
    from gllm_b200.ops import sm100
    torch.manual_seed(1)
    m, n, k = 300, 1024, 512
    big = (torch.randn(m, k * 2, device=_dev()) * 0.5).bfloat16()
    x = big[:, :k]  # row stride 2k
    w = (torch.randn(n, k, device=_dev()) * 0.05).bfloat16()
    b = torch.randn(n, device=_dev()).bfloat16()
    y = sm100.linear(x, w, b)
    yr = x.float() @ w.float().t() + b.float()
    assert _rel_err(y, yr) < 6e-3


def test_gemm_silu_mul():
    from gllm_b200.ops import sm100
    torch.manual_seed(2)
    m, i, k = 200, 1024, 512
    x = (torch.randn(m, k, device=_dev()) * 0.5).bfloat16()
    w = (torch.randn(2 * i, k, device=_dev()) * 0.05).bfloat16()
    wi = ref.interleave_gate_up(w, 128)
    y = sm100.linear_silu_mul(x, wi)
    h = x.float() @ w.float().t()
    yr = torch.nn.functional.silu(h[:, :i]) * h[:, i:]
    assert _rel_err(y, yr) < 1e-2
    # and the oracle's own interleaved path agrees
    assert _rel_err(ref.linear_silu_mul(x, wi, 128), yr) < 1e-2


@pytest.mark.parametrize("t,h", [(1, 4096), (7, 1024), (300, 4096), (64, 8192), (3, 7168), (2, 16384)])
@pytest.mark.parametrize("add", [False, True])
def test_rmsnorm(t, h, add):
    from gllm_b200.ops import sm100
    torch.manual_seed(3)
    x = torch.randn(t, h, device=_dev()).bfloat16()
    w = (1 + 0.1 * torch.randn(h, device=_dev())).bfloat16()
    r = torch.randn(t, h, device=_dev()).bfloat16() if add else None
    o_ref, r_ref = ref.rmsnorm(x, w, 1e-6, r.clone() if add else None)
    o, r_out = sm100.rmsnorm(x, w, 1e-6, r.clone() if add else None)
    assert _rel_err(o, o_ref) < 5e-3
    if add:
        assert _rel_err(r_out, r_ref) < 1e-3


def test_silu_and_mul():
    from gllm_b200.ops import sm100
    x = torch.randn(77, 2 * 1536, device=_dev()).bfloat16()
    assert _rel_err(sm100.silu_and_mul(x), ref.silu_and_mul(x)) < 5e-3


def test_embedding_and_gather():
    from gllm_b200.ops import sm100
    table = torch.randn(1000, 512, device=_dev()).bfloat16()
    ids = torch.randint(0, 2000, (333,), device=_dev(), dtype=torch.int32)
    o = sm100.embedding(ids, table, 500, 1500)
    o_ref = ref.embedding(ids, table, 500, 1500)
    assert torch.equal(o, o_ref)
    idx = torch.randint(0, 1000, (50,), device=_dev(), dtype=torch.int32)
    assert torch.equal(sm100.gather_rows(table, idx), table[idx.long()])


@pytest.mark.parametrize("d,rot,neox,qk_norm", [(128, 128, True, True), (128, 128, True, False),
                                                (64, 64, True, False), (128, 64, False, False),
                                                (256, 256, True, True)])
def test_rope_kv_write(d, rot, neox, qk_norm):
    from gllm_b200.ops import sm100
    torch.manual_seed(4)
    t, hq, hkv, page, pages = 83, 8, 2, 16, 32
    qkv = torch.randn(t, (hq + 2 * hkv) * d, device=_dev()).bfloat16()
    qkv_ref = qkv.clone()
    pos = torch.randint(0, 500, (t,), device=_dev(), dtype=torch.int32)
    slots = torch.randperm(pages * page, device=_dev())[:t].to(torch.int32)
    slots[5] = -1
    cs = ref.build_cos_sin_cache(rot, 512, 10000.0).to(_dev())
    qn = (1 + 0.1 * torch.randn(d, device=_dev())).bfloat16() if qk_norm else None
    kn = (1 + 0.1 * torch.randn(d, device=_dev())).bfloat16() if qk_norm else None
    shape = ref.kv_cache_shape(pages, hkv, d, page)
    kc, vc = torch.zeros(shape, device=_dev(), dtype=torch.bfloat16), torch.zeros(shape, device=_dev(), dtype=torch.bfloat16)
    kc_r, vc_r = kc.clone(), vc.clone()

    def views(buf):
        q = buf[:, : hq * d].view(t, hq, d)
        k = buf[:, hq * d: (hq + hkv) * d].view(t, hkv, d)
        v = buf[:, (hq + hkv) * d:].view(t, hkv, d)
        return q, k, v

    q, k, v = views(qkv)
    sm100.rope_kv_write(q, k, v, pos, cs, rot, neox, qn, kn, 1e-6, kc, vc, slots)
    qr, kr, vr = views(qkv_ref)
    ref.rope_kv_write(qr, kr, vr, pos, cs, rot, neox, qn, kn, 1e-6, kc_r, vc_r, slots)
    assert _rel_err(qkv, qkv_ref) < 8e-3
    assert _rel_err(kc, kc_r) < 8e-3
    assert torch.equal(vc, vc_r)


@pytest.mark.parametrize("sec", [[16, 24, 24], [24, 20, 20, 1]])   # chunked (Qwen2.5-VL) / interleaved (Qwen3-VL)
@pytest.mark.parametrize("strided", [False, True])
def test_rope_mrope(sec, strided):
    from gllm_b200.ops import sm100
    torch.manual_seed(5)
    t, hq, hkv, d = 40, 4, 2, 128
    q = torch.randn(t, hq, d, device=_dev()).bfloat16()
    k = torch.randn(t, hkv, d, device=_dev()).bfloat16()
    q_r, k_r = q.clone(), k.clone()
    pos = torch.randint(0, 300, (3, t + 24), device=_dev(), dtype=torch.int32)
    pos = pos[:, :t] if strided else pos[:, :t].contiguous()   # the runner passes a view of a [3, max_tokens] buffer
    cs = ref.build_cos_sin_cache(d, 512, 1e6).to(_dev())
    sm100.rope_kv_write(q, k, None, pos, cs, d, True, None, None, 1e-6, None, None, None, mrope_section=sec)
    ref.rope_kv_write(q_r, k_r, None, pos, cs, d, True, None, None, 1e-6, None, None, None, mrope_section=sec)
    assert _rel_err(q, q_r) < 8e-3 and _rel_err(k, k_r) < 8e-3


def _make_paged(seq_lens, q_lens, hq, hkv, d, page, device, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    b = len(seq_lens)
    max_blocks = max((s + page - 1) // page for s in seq_lens) + 1
    n_pages = sum((s + page - 1) // page for s in seq_lens) + 3
    perm = torch.randperm(n_pages, generator=g).tolist()
    bt = torch.zeros(b, max_blocks, dtype=torch.int32)
    c = 0
    for i, s in enumerate(seq_lens):
        n = (s + page - 1) // page
        bt[i, :n] = torch.tensor(perm[c:c + n], dtype=torch.int32)
        c += n
    shape = ref.kv_cache_shape(n_pages, hkv, d, page)
    kc = (torch.randn(shape, generator=g) * 0.5).bfloat16().to(device)
    vc = (torch.randn(shape, generator=g) * 0.5).bfloat16().to(device)
    t = sum(q_lens)
    q = (torch.randn(t, hq * d, generator=g) * 0.5).bfloat16().to(device)
    qsl = torch.tensor([0] + list(torch.tensor(q_lens).cumsum(0)), dtype=torch.int32, device=device)
    sl = torch.tensor(seq_lens, dtype=torch.int32, device=device)
    return q, kc, vc, bt.to(device), sl, qsl


@pytest.mark.parametrize("hq,hkv,d", [(32, 8, 128), (8, 8, 128), (28, 4, 128), (16, 2, 64), (8, 1, 128)])
@pytest.mark.parametrize("splits", [None, 1, 4])
def test_attn_decode(hq, hkv, d, splits):
    from gllm_b200.ops import sm100
    seq_lens = [1, 5, 16, 17, 63, 64, 65, 200, 1000, 333]
    q_lens = [1] * len(seq_lens)
    q, kc, vc, bt, sl, qsl = _make_paged(seq_lens, q_lens, hq, hkv, d, 16, _dev())
    scale = 1.0 / math.sqrt(d)
    o = sm100.paged_attention(q, kc, vc, bt, sl, qsl, scale, hq, d, len(seq_lens), len(seq_lens), 1,
                              max(seq_lens), splits=splits)
    torch.cuda.synchronize()
    o_ref = ref.paged_attention(q, kc, vc, bt, sl, qsl, scale, hq, d)
    assert torch.isfinite(o.float()).all()
    assert _rel_err(o, o_ref) < 1e-2, _rel_err(o, o_ref)


@pytest.mark.parametrize("hq,hkv,d", [(32, 8, 128), (8, 8, 128), (28, 4, 128), (16, 2, 64)])
def test_attn_prefill_and_mixed(hq, hkv, d, monkeypatch):
    from gllm_b200.ops import sm100
    monkeypatch.setattr(sm100, "ATTN_TC", False)     # the mma.sync kernel (fallback for shapes outside the wgmma one)
    # decode seqs first, then prefill chunks (some with prefix/chunk context)
    seq_lens = [7, 130, 40, 300, 129, 64, 1024]
    q_lens = [1, 1, 40, 100, 129, 3, 513]
    nd = 2
    q, kc, vc, bt, sl, qsl = _make_paged(seq_lens, q_lens, hq, hkv, d, 16, _dev(), seed=1)
    scale = 1.0 / math.sqrt(d)
    o = sm100.paged_attention(q, kc, vc, bt, sl, qsl, scale, hq, d, nd, len(seq_lens), max(q_lens), max(seq_lens))
    torch.cuda.synchronize()
    o_ref = ref.paged_attention(q, kc, vc, bt, sl, qsl, scale, hq, d)
    assert torch.isfinite(o.float()).all()
    assert _rel_err(o, o_ref) < 1e-2, _rel_err(o, o_ref)


@pytest.mark.parametrize("kv_tile", [128, 64])
@pytest.mark.parametrize("hq,hkv,d", [(32, 8, 128), (8, 8, 128), (28, 4, 128), (16, 2, 64)])
def test_prefill_attention_tc(hq, hkv, d, kv_tile, monkeypatch):
    """wgmma prefill kernel vs the fp32 oracle: ragged chunks, prefix context, page-boundary cases."""
    from gllm_b200.ops import sm100
    monkeypatch.setattr(sm100, "ATTN_TC", True)
    monkeypatch.setattr(sm100, "ATTN_TC_KV", kv_tile)
    seq_lens = [7, 130, 40, 300, 129, 64, 1024, 257]
    q_lens = [1, 1, 40, 100, 129, 3, 513, 257]
    nd = 2
    q, kc, vc, bt, sl, qsl = _make_paged(seq_lens, q_lens, hq, hkv, d, 16, _dev(), seed=1)
    scale = 1.0 / math.sqrt(d)
    o = sm100.paged_attention(q, kc, vc, bt, sl, qsl, scale, hq, d, nd, len(seq_lens), max(q_lens), max(seq_lens))
    torch.cuda.synchronize()
    o_ref = ref.paged_attention(q, kc, vc, bt, sl, qsl, scale, hq, d)
    assert torch.isfinite(o.float()).all()
    assert _rel_err(o, o_ref) < 1e-2, _rel_err(o, o_ref)


def test_sampler_greedy_and_filter():
    from gllm_b200.ops import sm100
    torch.manual_seed(6)
    b, v = 33, 151936
    logits = (torch.randn(b, v, device=_dev()) * 3).bfloat16()
    tok = sm100.sample(logits)
    assert torch.equal(tok.long(), logits.float().argmax(-1))
    # temperature/top-k/top-p: every drawn token must lie in the oracle's support. fp32 logits so
    # that ties (which the kernel keeps, the sort-based oracle breaks arbitrarily) are improbable;
    # the oracle gets a hair more top-p mass to absorb x*(1/T) vs x/T rounding at the boundary.
    logits = torch.randn(b, v, device=_dev()) * 3
    temp = torch.full((b,), 0.8, device=_dev())
    tk = torch.full((b,), 50, device=_dev(), dtype=torch.int32)
    tp = torch.full((b,), 0.9, device=_dev())
    probs = ref.sample_filter(logits, temp, tk + 1, tp + 1e-3)
    for s in range(3):
        tok = sm100.sample(logits, temp, tk, tp, seed=123 + s)
        p_tok = probs.gather(1, tok.long().view(-1, 1))
        assert (p_tok > 0).all()
    # top-p only (no top-k) and top-k only
    tok = sm100.sample(logits, temp, torch.full((b,), -1, device=_dev(), dtype=torch.int32), tp, seed=5)
    probs = ref.sample_filter(logits, temp, None, tp + 1e-3)
    assert (probs.gather(1, tok.long().view(-1, 1)) > 0).all()
    tok = sm100.sample(logits, temp, tk, None, seed=6)
    probs = ref.sample_filter(logits, temp, tk + 1, None)
    assert (probs.gather(1, tok.long().view(-1, 1)) > 0).all()


def test_sampler_distribution():
    from gllm_b200.ops import sm100
    torch.manual_seed(7)
    v = 64
    row = torch.randn(v, device=_dev()) * 2
    n = 20000
    logits = row.unsqueeze(0).repeat(n, 1).contiguous()
    temp = torch.full((n,), 1.3, device=_dev())
    tk = torch.full((n,), 20, device=_dev(), dtype=torch.int32)
    tp = torch.full((n,), 0.85, device=_dev())
    probs = ref.sample_filter(logits[:1], temp[:1], tk[:1], tp[:1])[0]
    tok = sm100.sample(logits, temp, tk, tp, seed=99)
    emp = torch.bincount(tok.long(), minlength=v).float() / n
    assert (emp[probs == 0] == 0).all()
    assert (emp - probs).abs().max().item() < 0.02


@pytest.mark.parametrize("t", [1, 64, 300])
@pytest.mark.parametrize("b,n,k", [(16, 512, 128), (16, 128, 512), (3, 256, 192)])
def test_gemm_batched_strided_views(t, b, n, k):
    """Batched mode of the wgmma GEMM (MLA weight absorption, K13): strided [T, B, K] operand through a 3-D TMA
    map, result written into a strided [T, B, N] view, vs an fp32 einsum."""
    from gllm_b200.ops import sm100
    torch.manual_seed(t + n)
    dev = _dev()
    a_full = (torch.randn(t, b, k + 64, device=dev) * 0.5).bfloat16()     # the operand is a column slice
    w = (torch.randn(b, n, k, device=dev) * 0.1).bfloat16()
    out_full = torch.full((t, b, n + 64), 7.0, device=dev, dtype=torch.bfloat16)
    a, out = a_full[:, :, :k], out_full[:, :, :n]
    sm100.gemm_batched(a, w, out)
    torch.cuda.synchronize()
    ref_o = torch.einsum("tbk,bnk->tbn", a.float(), w.float())
    assert _rel_err(out, ref_o) < 1e-2, _rel_err(out, ref_o)
    assert bool((out_full[:, :, n:] == 7.0).all())                         # nothing written outside the view


@pytest.mark.parametrize("tp", [2, 8])
def test_vocab_parallel_sampling_equals_the_full_vocab_kernel(tp):
    """SURVEY §2.4 X4: vp_candidates_kernel on each vocab shard + vp_final_kernel on the gathered records draw the
    SAME token as sample_kernel on the full [B, V] row (the race's random numbers are keyed by token id) for greedy,
    top-k, top-k + top-p, nucleus-only, penalised and unfiltered rows — without ever holding the full logits."""
    from gllm_b200.ops import sm100
    torch.manual_seed(11)
    dev = _dev()
    v_full = 151936
    per = (v_full + tp - 1) // tp
    per = (per + 127) // 128 * 128                     # shards are padded: the last one ends with dead columns
    b = 24
    logits = torch.randn(b, tp * per, device=dev) * 3
    logits[:, v_full:] = 50.0                          # padding columns must never win
    base = torch.tensor([1, 20, 50, 200, 0, 0], dtype=torch.int32)
    top_k = base.repeat(b // 6).to(dev)
    top_k = torch.where(top_k <= 0, torch.full_like(top_k, v_full), top_k)
    top_p = torch.tensor([1.0, 0.9, 1.0, 0.8, 0.3, 1.0]).repeat(b // 6).to(dev)
    temp = torch.tensor([0.0, 0.7, 1.0, 1.2, 0.6, 1.0]).repeat(b // 6).to(dev)
    pen = torch.tensor([1.0, 1.3, 1.0, 1.1, 1.0, 1.2]).repeat(b // 6).to(dev)
    seen = torch.randint(-2 ** 31, 2 ** 31 - 1, (b, (tp * per + 31) // 32), dtype=torch.int64, device=dev).to(torch.int32)
    slots = torch.arange(b, dtype=torch.int32, device=dev)
    step = torch.tensor([5], dtype=torch.int64, device=dev)
    full = sm100.sample(logits[:, :v_full].contiguous(), temp, top_k, top_p, pen, seen, slots, seed=77, step=step)
    c = 256
    recs = []
    for r in range(tp):
        lo = r * per
        valid = max(0, min(per, v_full - lo))
        recs.append(sm100.vp_candidates(logits[:, lo:lo + per], valid, v_full, c, temp, top_k, top_p, pen, seen, slots,
                                        seed=77, step=step, vocab_offset=lo))
    toks = sm100.vp_final(torch.stack(recs).contiguous(), c, v_full, top_k, top_p, seed=77, step=step)
    torch.cuda.synchronize()
    assert int(toks.max()) < v_full
    assert torch.equal(toks, full), (toks.tolist(), full.tolist())
    # record hygiene: every shard returns its true top candidates and softmax statistics
    x = ref.apply_penalty_temperature(logits[:, :per], temp, None, None)
    rec0 = recs[0]
    row = 2                                            # top_k 50, no penalty on this row
    got = torch.sort(rec0[row, :50], descending=True).values
    want = torch.topk(logits[row, :per] / temp[row].clamp_min(1e-5), 50).values
    assert torch.allclose(got, want, rtol=1e-5, atol=1e-5)


def test_sampler_rep_penalty():
    from gllm_b200.ops import sm100
    torch.manual_seed(8)
    b, v = 4, 1000
    logits = torch.randn(b, v, device=_dev())
    seen = torch.zeros(b, (v + 31) // 32, dtype=torch.int32, device=_dev())
    top = logits.argmax(-1).to(torch.int32)
    rows = torch.arange(b, device=_dev(), dtype=torch.int32)
    sm100.mark_seen(seen, rows, top)
    pen = torch.full((b,), 50.0, device=_dev())
    tok = sm100.sample(logits, rep_penalty=pen, seen_bits=seen)
    mask = torch.zeros(b, v, dtype=torch.bool, device=_dev())
    mask[rows.long(), top.long()] = True
    exp = ref.sample(logits, rep_penalty=pen, seen_mask=mask)
    assert torch.equal(tok, exp)


@pytest.mark.parametrize("m", [1, 16, 17, 64, 100, 255, 256])
@pytest.mark.parametrize("n,k", [(4096, 4096), (6144, 4096), (4096, 12288), (1000, 512), (152064, 1024)])
@pytest.mark.parametrize("split", [0, 1, 3])
def test_gemm_smallm(m, n, k, split, monkeypatch):
    """swap-AB split-K decode GEMM (bias, forced splits, ragged N)."""
    from gllm_b200.ops import sm100
    monkeypatch.setattr(sm100, "_FORCE_SPLIT", split)
    monkeypatch.setattr(sm100, "_SMALLM_MAX", 256)
    torch.manual_seed(m + n)
    x = (torch.randn(m, k, device=_dev()) * 0.5).bfloat16()
    w = (torch.randn(n, k, device=_dev()) * 0.05).bfloat16()
    b = torch.randn(n, device=_dev()).bfloat16()
    for bias in (None, b):
        y = sm100.linear(x, w, bias)
        yr = x.float() @ w.float().t() + (bias.float() if bias is not None else 0)
        assert _rel_err(y, yr) < 6e-3, _rel_err(y, yr)
    # back-to-back launches reuse the workspace/counters
    y2 = sm100.linear(x, w, None)
    assert torch.equal(y2, sm100.linear(x, w, None))


@pytest.mark.parametrize("m", [3, 64, 200])
@pytest.mark.parametrize("split", [0, 1, 2])
def test_gemm_smallm_silu(m, split, monkeypatch):
    from gllm_b200.ops import sm100
    monkeypatch.setattr(sm100, "_FORCE_SPLIT", split)
    monkeypatch.setattr(sm100, "_SMALLM_MAX", 256)
    torch.manual_seed(m)
    i, k = 1536, 1024
    x = (torch.randn(m, k, device=_dev()) * 0.5).bfloat16()
    w = (torch.randn(2 * i, k, device=_dev()) * 0.05).bfloat16()
    y = sm100.linear_silu_mul(x, ref.interleave_gate_up(w, 128))
    h = x.float() @ w.float().t()
    yr = torch.nn.functional.silu(h[:, :i]) * h[:, i:]
    assert _rel_err(y, yr) < 1e-2


@pytest.mark.parametrize("e,k,renorm", [(8, 2, True), (60, 4, False), (128, 8, True), (256, 8, True)])
def test_moe_topk_softmax(e, k, renorm):
    from gllm_b200.ops import sm100_moe
    torch.manual_seed(e)
    logits = torch.randn(77, e, device=_dev()).bfloat16()
    w, ids = sm100_moe.topk_softmax(logits, k, renorm)
    w_r, ids_r = ref.topk_softmax(logits, k, renorm)
    # compare as sets per row (tie order may differ), weights by id
    dense = torch.zeros(77, e, device=_dev()).scatter(1, ids.long(), w)
    dense_r = torch.zeros(77, e, device=_dev()).scatter(1, ids_r.long(), w_r)
    assert torch.allclose(dense, dense_r, atol=2e-3, rtol=1e-2)


@pytest.mark.parametrize("scoring,bias", [("sigmoid", True), ("softmax", False)])
def test_moe_grouped_topk(scoring, bias):
    from gllm_b200.ops import sm100_moe
    torch.manual_seed(11)
    t, e, k, g, tg = 93, 256, 8, 8, 4
    logits = torch.randn(t, e, device=_dev()).bfloat16()
    b = (torch.randn(e, device=_dev()) * 0.1).float() if bias else None
    w, ids = sm100_moe.grouped_topk(logits, k, True, g, tg, scoring, b, 2.5)
    w_r, ids_r = ref.grouped_topk(logits, k, True, g, tg, scoring, b, 2.5)
    dense = torch.zeros(t, e, device=_dev()).scatter(1, ids.long(), w)
    dense_r = torch.zeros(t, e, device=_dev()).scatter(1, ids_r.long(), w_r)
    assert torch.allclose(dense, dense_r, atol=5e-3, rtol=2e-2)


@pytest.mark.parametrize("t,e,k,h,i,ep", [(5, 8, 2, 256, 512, False), (300, 8, 2, 512, 1024, False),
                                          (200, 16, 4, 256, 256, True), (1000, 64, 6, 256, 128, False)])
def test_moe_fused_experts(t, e, k, h, i, ep):
    from gllm_b200.ops import sm100_moe
    torch.manual_seed(t + e)
    x = (torch.randn(t, h, device=_dev()) * 0.5).bfloat16()
    e_local = e // 2 if ep else e
    w13 = (torch.randn(e_local, 2 * i, h, device=_dev()) * 0.05).bfloat16()
    w2 = (torch.randn(e_local, h, i, device=_dev()) * 0.05).bfloat16()
    logits = torch.randn(t, e, device=_dev()).bfloat16()
    w, ids = ref.topk_softmax(logits, k, True)
    emap = None
    if ep:
        emap = torch.full((e,), -1, dtype=torch.int32, device=_dev())
        emap[e // 2:] = torch.arange(e_local, dtype=torch.int32, device=_dev())
    w13_il = torch.stack([ref.interleave_gate_up(w13[j], 64) for j in range(e_local)])
    y = sm100_moe.fused_experts(x, w13_il, w2, w, ids, emap)
    y_ref = ref.fused_experts(x, w13, w2, w, ids, emap)
    assert torch.isfinite(y.float()).all()
    assert _rel_err(y, y_ref) < 2e-2, _rel_err(y, y_ref)


@pytest.mark.parametrize("m,n,k", [(1, 256, 128), (77, 1536, 512), (300, 4096, 7168), (1024, 2048, 2048),
                                   (64, 576, 7168)])      # 576 = kv_a_proj_with_mqa (MLA): N not a multiple of 128
def test_gemm_fp8_block(m, n, k):
    from gllm_b200.ops import sm100
    torch.manual_seed(m)
    x = (torch.randn(m, k, device=_dev()) * 0.7).bfloat16()
    w = torch.randn(n, k, device=_dev()) * 0.05
    # block-quantise the weight like an HF fp8 checkpoint: per 128x128 block scale_inv = amax / 448
    nb, kb = (n + 127) // 128, k // 128
    wp = torch.zeros(nb * 128, k, device=_dev())
    wp[:n] = w
    blocks = wp.view(nb, 128, kb, 128)
    s_inv = (blocks.abs().amax(dim=(1, 3)) / 448.0).clamp_min(1e-8)
    w8 = (blocks / s_inv.view(nb, 1, kb, 1)).view(nb * 128, k)[:n].to(torch.float8_e4m3fn).contiguous()
    b = torch.randn(n, device=_dev()).bfloat16()
    y = sm100.linear_fp8_block(x, w8, s_inv.contiguous(), b)
    y_ref = ref.linear_fp8_block(x, w8, s_inv, b)
    assert _rel_err(y, y_ref) < 1e-2, _rel_err(y, y_ref)
    # and the quantiser alone
    q, s = sm100.fp8_quant_group(x)
    q_r, s_r = ref.fp8_quant_group(x)
    assert torch.allclose(s.t(), s_r, rtol=1e-5)
    assert _rel_err(q.float(), q_r.float()) < 3e-2


@pytest.mark.parametrize("m", [64, 128, 200, 256, 384, 512])
@pytest.mark.parametrize("n,k", [(4096, 4096), (4096, 12288), (6144, 4096), (1000, 1536)])
def test_gemm_splitk_decode_shapes(m, n, k):
    """Decode-sized M takes the wide-tile split-K path (fp32 partials, last-arriver sum): exact shape sweep,
    bias, and back-to-back launches (tile counters re-arm themselves)."""
    from gllm_b200.ops import sm100
    torch.manual_seed(m + n + k)
    x = (torch.randn(m, k, device=_dev()) * 0.5).bfloat16()
    w = (torch.randn(n, k, device=_dev()) * 0.05).bfloat16()
    b = torch.randn(n, device=_dev()).bfloat16()
    for bias in (None, b):
        y = sm100.linear(x, w, bias)
        yr = x.float() @ w.float().t() + (bias.float() if bias is not None else 0)
        assert _rel_err(y, yr) < 6e-3, _rel_err(y, yr)
    y2 = sm100.linear(x, w, None)
    for _ in range(3):
        assert torch.equal(y2, sm100.linear(x, w, None))   # deterministic slice-ordered reduction


@pytest.mark.parametrize("m", [64, 256, 384])
def test_gemm_splitk_silu(m):
    from gllm_b200.ops import sm100
    torch.manual_seed(m)
    i, k = 12288, 4096
    x = (torch.randn(m, k, device=_dev()) * 0.5).bfloat16()
    w = (torch.randn(2 * i, k, device=_dev()) * 0.02).bfloat16()
    y = sm100.linear_silu_mul(x, ref.interleave_gate_up(w, 128))
    h = x.float() @ w.float().t()
    yr = torch.nn.functional.silu(h[:, :i]) * h[:, i:]
    assert _rel_err(y, yr) < 1e-2


def _mla_ref(q_full, cache, bt, tok_seq, positions, scale):
    t, h, _ = q_full.shape
    out = torch.zeros(t, h, 512, dtype=torch.float32, device=q_full.device)
    for i in range(t):
        s = int(tok_seq[i]) if tok_seq is not None else i
        n = int(positions[i]) + 1
        lat = ref.gather_kv(cache, bt[s], n)[:, 0].float()          # [n, 576]
        att = torch.softmax((q_full[i].float() @ lat.t()) * scale, dim=-1)
        out[i] = att @ lat[:, :512]
    return out


@pytest.mark.parametrize("heads", [16, 8, 40])
@pytest.mark.parametrize("splits", [1, 3, None])
def test_mla_attention_decode(heads, splits):
    from gllm_b200.ops import sm100
    torch.manual_seed(7)
    page, b = 16, 5
    lens = [1, 63, 64, 300, 777]
    max_blocks = max((n + page - 1) // page for n in lens) + 1
    n_pages = sum((n + page - 1) // page for n in lens) + 2
    cache = (torch.randn(n_pages, 1, 9, page, 64, device=_dev()) * 0.5).bfloat16()
    perm = torch.randperm(n_pages)[: n_pages - 1].tolist()
    bt = torch.zeros(b, max_blocks, dtype=torch.int32)
    c = 0
    for i, n in enumerate(lens):
        k = (n + page - 1) // page
        bt[i, :k] = torch.tensor(perm[c:c + k], dtype=torch.int32)
        c += k
    bt = bt.to(_dev())
    q = (torch.randn(b, heads, 576, device=_dev()) * 0.3).bfloat16()
    pos = torch.tensor([n - 1 for n in lens], dtype=torch.int32, device=_dev())
    scale = 192 ** -0.5
    out = sm100.mla_attention(q, cache, bt, None, pos, scale, splits=splits)
    want = _mla_ref(q, cache, bt, None, pos, scale)
    assert _rel_err(out, want) < 1.5e-2, _rel_err(out, want)


def test_mla_attention_prefill_tokens_and_rope_cache():
    """Mixed batch: every token attends to its own causal prefix (tok_seq / positions); plus the fused
    rope + latent-cache write against the PyTorch oracle ops."""
    from gllm_b200.ops import sm100
    torch.manual_seed(8)
    page, heads = 16, 16
    q_lens, ctx = [40, 1, 70], [0, 130, 25]          # new tokens / already cached tokens per sequence
    b = len(q_lens)
    tot = [q + c for q, c in zip(q_lens, ctx)]
    max_blocks = max((n + page - 1) // page for n in tot) + 1
    n_pages = sum((n + page - 1) // page for n in tot) + 1
    cache = (torch.randn(n_pages, 1, 9, page, 64, device=_dev()) * 0.5).bfloat16()
    bt = torch.zeros(b, max_blocks, dtype=torch.int32)
    c = 0
    for i, n in enumerate(tot):
        k = (n + page - 1) // page
        bt[i, :k] = torch.arange(c, c + k, dtype=torch.int32)
        c += k
    tok_seq = torch.tensor(sum(([i] * q for i, q in enumerate(q_lens)), []), dtype=torch.int32)
    pos = torch.tensor(sum((list(range(cx, cx + q)) for q, cx in zip(q_lens, ctx)), []), dtype=torch.int32)
    t = int(tok_seq.numel())
    slots = torch.tensor([int(bt[s, p // page]) * page + p % page for s, p in zip(tok_seq.tolist(), pos.tolist())],
                         dtype=torch.int32)
    bt, tok_seq, pos, slots = bt.to(_dev()), tok_seq.to(_dev()), pos.to(_dev()), slots.to(_dev())
    # ---- rope + cache write ----
    qk_dim, nope = 192, 128
    qp = (torch.randn(t, heads, qk_dim, device=_dev()) * 0.5).bfloat16()
    kv_a = (torch.randn(t, 576, device=_dev()) * 0.5).bfloat16()
    kv_c = kv_a[:, :512].contiguous()
    cs = ref.build_cos_sin_cache(64, 512, 10000.0).to(_dev())
    q_full = torch.zeros(t, heads, 576, dtype=torch.bfloat16, device=_dev())
    cache2 = cache.clone()
    sm100.mla_rope_cache(qp[:, :, nope:], q_full, kv_a[:, 512:], kv_c, cs, pos, slots, cache2)
    q_pe = qp[:, :, nope:].contiguous()
    k_pe = kv_a[:, 512:].contiguous().view(t, 1, 64)
    ref.rope_kv_write(q_pe, k_pe, None, pos, cs, 64, False, None, None, 1e-6, None, None, None)
    cache_ref = cache.clone()
    ref.write_kv_cache(torch.cat([kv_c, k_pe.view(t, 64)], -1).view(t, 1, 576), None, cache_ref, None, slots)
    assert _rel_err(q_full[:, :, 512:], q_pe) < 8e-3
    assert _rel_err(cache2, cache_ref) < 8e-3
    # ---- attention over the freshly written cache ----
    q_full[:, :, :512] = (torch.randn(t, heads, 512, device=_dev()) * 0.3).bfloat16()
    scale = 192 ** -0.5
    out = sm100.mla_attention(q_full, cache2, bt, tok_seq, pos, scale)
    want = _mla_ref(q_full, cache2, bt, tok_seq, pos, scale)
    assert _rel_err(out, want) < 1.5e-2, _rel_err(out, want)


@pytest.mark.parametrize("t,e,k", [(77, 4, 2), (300, 8, 2), (5, 8, 4)])
def test_moe_fused_experts_fp8(t, e, k):
    """Grouped block-scaled fp8 expert GEMMs (SiLU-gate epilogue on interleaved tiles with per-64-row scales)
    against the de-quantised bf16 oracle."""
    from gllm_b200.layers.moe import _block_quant_rows64
    from gllm_b200.ops import sm100_moe
    torch.manual_seed(t + e)
    h, inter = 512, 256
    x = (torch.randn(t, h, device=_dev()) * 0.5).bfloat16()
    w13 = (torch.randn(e, 2 * inter, h, device=_dev()) * 0.05).bfloat16()
    w2 = (torch.randn(e, h, inter, device=_dev()) * 0.05).bfloat16()
    logits = torch.randn(t, e, device=_dev()).bfloat16()
    tw, ids = sm100_moe.topk_softmax(logits, k, True)
    q13, s13, q2, s2, d13, d2 = [], [], [], [], [], []
    for i in range(e):
        a, sa = _block_quant_rows64(w13[i])
        b, sb = _block_quant_rows64(w2[i])
        d13.append((a.float() * sa.repeat_interleave(64, 0).repeat_interleave(128, 1)).bfloat16())
        d2.append((b.float() * sb.repeat_interleave(64, 0).repeat_interleave(128, 1)).bfloat16())
        q13.append(ref.interleave_gate_up(a.view(torch.uint8), 64).view(torch.float8_e4m3fn))
        s13.append(ref.interleave_gate_up(sa, 1))
        q2.append(b)
        s2.append(sb)
    out = sm100_moe.fused_experts_fp8(x, torch.stack(q13), torch.stack(s13).contiguous(), torch.stack(q2),
                                      torch.stack(s2).contiguous(), tw, ids)
    def qdq(a):   # dynamic per-token-group(128) activation quantisation, as the kernel path does
        q, sc = ref.fp8_quant_group(a, 128)
        return (q.float().reshape(a.shape[0], -1, 128) * sc.unsqueeze(-1)).reshape(a.shape).to(a.dtype)

    want = torch.zeros(t, h, dtype=torch.float32, device=_dev())
    for i in range(e):
        tok, slot = torch.where(ids.long() == i)
        if tok.numel() == 0:
            continue
        hd = ref.silu_and_mul(torch.nn.functional.linear(qdq(x[tok]), d13[i]))
        ye = torch.nn.functional.linear(qdq(hd), d2[i]).float()
        want.index_add_(0, tok, ye * tw[tok, slot].float().unsqueeze(-1))
    # (bf16 rounding of the intermediate moves some values across e4m3 rounding boundaries: ~1.8 % measured)
    assert _rel_err(out, want) < 2.5e-2, _rel_err(out, want)
    # and within quantisation noise of the un-quantised-activation oracle
    assert _rel_err(out, ref.fused_experts(x, torch.stack(d13), torch.stack(d2), tw, ids)) < 8e-2
