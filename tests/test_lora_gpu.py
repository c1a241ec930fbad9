"""Multi-LoRA on the GPU: the three sm_90a kernels element by element against a float64 oracle, and the engine at
real width (H = 4096) against merged weights and across eager / CUDA-graph execution.

Error bounds (u = 2^-24, the fp32 unit roundoff; a bf16 rounding has relative error <= 2^-8 after round-to-nearest):
- lora_shrink: U = Σ_k x_k·a_k over K bf16 products, each exact in fp32, summed in fp32 (tensor-core k16 steps, then
  a fixed-order sum across K slices). Any summation order gives |U - U64| <= K·u·Σ_k |x_k·a_k|; we check 2·K·u·Σ|x||a| + 1e-30.
- lora_expand_add: y' = bf16(y + Σ_k u_k·b_k) with an fp32 sum over r: |y' - exact| <= 2^-8·|exact| +
  (r + 1)·u·(|y| + Σ|u||b|)·(1 + 2^-8), checked with 2·r instead of r + 1.
- lora_expand_silu_mul: out = bf16(SiLU(g + dg)·(v + dv)); the fp32 deltas carry e = 2·(r + 1)·u·(|pre| + Σ|u||b|),
  which SiLU (|SiLU'| <= 1.1) and the product propagate, plus the fast-math exp (relative error < 2^-20):
  |out - exact| <= 2^-8·|exact| + 1.1·e_g·|v + dv| + |SiLU(g + dg)|·e_v + 2^-19·|exact|.
Rows without an adapter must come out of lora_expand_add bit for bit unchanged, and every kernel gives the same bits
on every call, eager or replayed from a CUDA graph.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
BF = 2.0 ** -8


def _csr(slot: torch.Tensor, n_adapters: int):
    """Per-row adapter slot (-1: none) -> (slots, row_off, rows, S) like InputData._load_lora."""
    import numpy as np
    from gllm_b200.input_data import InputData
    inp = InputData(max(slot.numel(), 1), 1, 1, "cuda")
    inp.set_lora(n_adapters)
    inp._flip = 1
    inp._load_lora(slot.cpu().numpy().astype(np.int32))
    torch.cuda.synchronize()
    l1 = inp._lora
    return l1[0][1], l1[1][1], l1[2][1][: slot.numel()], inp.lora_groups


def _pattern(kind: str, t: int, n_adapters: int, g):
    if kind == "none":
        return torch.full((t,), -1, dtype=torch.int32)
    if kind == "one":
        return torch.zeros(t, dtype=torch.int32)
    s = torch.randint(-1, 3, (t,), generator=g, dtype=torch.int32)   # three adapters interleaved with base rows
    return s


# (name, K, module column widths) at Qwen3-8B (H 4096, 32 q / 8 kv heads of 128, I 12288) tp 1 and 2, plus odd sizes
SHAPES = [("qkv_tp1", 4096, [4096, 1024, 1024]), ("qkv_tp2", 4096, [2048, 512, 512]),
          ("o_tp1", 4096, [4096]), ("o_tp2", 2048, [4096]), ("down_tp1", 12288, [4096]), ("down_tp2", 6144, [4096]),
          ("gate_up_plain", 4096, [1000, 1000]), ("odd", 1000, [300, 72, 72])]
TS = [1, 3, 32, 64, 65, 257, 4099]
RANKS = [8, 16, 64]
PATTERNS = ["none", "one", "three"]


def _inputs(t, k, widths, r, kind, seed):
    g = torch.Generator().manual_seed(seed)
    n_ad = 3
    m = len(widths)
    x = (torch.randn(t, k, generator=g) * 0.5).to(torch.bfloat16).cuda()
    A = (torch.randn(n_ad, m * r, k, generator=g) * 0.05).to(torch.bfloat16).cuda()
    B = (torch.randn(n_ad, sum(widths), r, generator=g) * 0.05).to(torch.bfloat16).cuda()
    y = (torch.randn(t, sum(widths), generator=g)).to(torch.bfloat16).cuda()
    slot = _pattern(kind, t, n_ad, g)
    return x, A, B, y, slot


def _u64(x, A, slot, m_cols):
    u = torch.zeros(x.shape[0], m_cols, dtype=torch.float64, device=x.device)
    mag = torch.zeros_like(u)
    s = slot.cuda().long()
    for a in range(A.shape[0]):
        rows = (s == a).nonzero().flatten()
        if rows.numel():
            xa = x[rows].double()
            u[rows] = xa @ A[a].double().t()
            mag[rows] = xa.abs() @ A[a].double().abs().t()
    return u, mag


@pytest.mark.parametrize("kind", PATTERNS)
@pytest.mark.parametrize("r", RANKS)
@pytest.mark.parametrize("t", TS)
@pytest.mark.parametrize("name,k,widths", SHAPES)
def test_shrink_and_expand_add_match_float64(name, k, widths, t, r, kind):
    from gllm_b200.ops import sm100
    x, A, B, y, slot = _inputs(t, k, widths, r, kind, seed=t * 131 + r * 7 + len(name))
    csr = _csr(slot, 3)
    u = sm100.lora_shrink(x, A, *csr)
    u64, umag = _u64(x, A, slot, A.shape[1])
    err = (u.double() - u64).abs()
    bound = 2 * k * U32 * umag + 1e-30
    bad = (err > bound) | torch.isnan(u)
    assert not bad.any(), f"shrink {name} t={t} r={r} {kind}: row {bad.nonzero()[0].tolist()}"
    # expand-add from the kernel's own U (so the check isolates the expand arithmetic)
    bounds = [0]
    for w in widths:
        bounds.append(bounds[-1] + w)
    y0 = y.clone()
    sm100.lora_expand_add(y, u, B, bounds, *csr)
    s = slot.cuda().long()
    exact = y0.double().clone()
    mag = y0.double().abs()
    for a in range(3):
        rows = (s == a).nonzero().flatten()
        if not rows.numel():
            continue
        for mi in range(len(widths)):
            c0, c1 = bounds[mi], bounds[mi + 1]
            ua = u[rows][:, mi * r:(mi + 1) * r].double()
            bb = B[a, c0:c1].double()
            exact[rows[:, None], torch.arange(c0, c1, device="cuda")[None]] += ua @ bb.t()
            mag[rows[:, None], torch.arange(c0, c1, device="cuda")[None]] += ua.abs() @ bb.abs().t()
    err = (y.double() - exact).abs()
    bound = BF * exact.abs() + 2 * (r + 1) * U32 * mag * (1 + BF) + 1e-30
    bad = (err > bound) | torch.isnan(y)
    assert not bad.any(), f"expand {name} t={t} r={r} {kind}: at {bad.nonzero()[0].tolist()}"
    # rows without an adapter are untouched bit for bit
    base = (s < 0).nonzero().flatten()
    assert torch.equal(y[base], y0[base])


@pytest.mark.parametrize("kind", PATTERNS)
@pytest.mark.parametrize("r", RANKS)
@pytest.mark.parametrize("t", TS)
@pytest.mark.parametrize("inter", [12288, 6144, 384])
def test_expand_silu_mul_matches_float64(inter, t, r, kind):
    from gllm_b200.ops import sm100
    g = torch.Generator().manual_seed(t * 17 + r + inter)
    n_ad = 3
    pre = torch.randn(t, 2 * inter, generator=g).to(torch.bfloat16).cuda()
    u = (torch.randn(t, 2 * r, generator=g) * 0.5).cuda()
    B = (torch.randn(n_ad, 2 * inter, r, generator=g) * 0.1).to(torch.bfloat16).cuda()
    slot = _pattern(kind, t, n_ad, g)
    csr = _csr(slot, n_ad)
    out = sm100.lora_expand_silu_mul(pre, u, B, *csr)
    s = slot.cuda().long()
    gate_col = (torch.arange(2 * inter, device="cuda") % 256) < 128
    d = torch.zeros(t, 2 * inter, dtype=torch.float64, device="cuda")
    dm = torch.zeros_like(d)
    for a in range(n_ad):
        rows = (s == a).nonzero().flatten()
        if rows.numel():
            bb = B[a].double()
            ug, uu = u[rows, :r].double(), u[rows, r:].double()
            d[rows] = torch.where(gate_col, ug @ bb.t(), uu @ bb.t())
            dm[rows] = torch.where(gate_col, ug.abs() @ bb.abs().t(), uu.abs() @ bb.abs().t())
    full = pre.double() + d
    e = 2 * (r + 1) * U32 * (pre.double().abs() + dm)
    shp = (t, inter // 128, 2, 128)
    full, e = full.reshape(shp), e.reshape(shp)
    gv, vv, eg, ev = full[:, :, 0], full[:, :, 1], e[:, :, 0], e[:, :, 1]
    silu = gv / (1 + torch.exp(-gv))
    exact = (silu * vv).reshape(t, inter)
    bound = (BF + 2.0 ** -19) * exact.abs() + (1.1 * eg * vv.abs() + silu.abs() * ev).reshape(t, inter) + 1e-30
    err = (out.double() - exact).abs()
    bad = (err > bound) | torch.isnan(out)
    assert not bad.any(), f"silu_mul I={inter} t={t} r={r} {kind}: at {bad.nonzero()[0].tolist()}"


@pytest.mark.parametrize("t", [3, 64, 257, 4099])
def test_kernels_are_deterministic_eager_and_in_graphs(t):
    """Same inputs -> the same bits: twice eagerly and once replayed from a CUDA graph (the K-sliced shrink sums its
    partials in a fixed order, so a decode step gives the same logits on every run)."""
    from gllm_b200.ops import sm100
    x, A, B, y, slot = _inputs(t, 4096, [4096, 1024, 1024], 16, "three", seed=t)
    csr = _csr(slot, 3)
    bounds = [0, 4096, 5120, 6144]
    pre = torch.randn(t, 2 * 384, generator=torch.Generator().manual_seed(t)).to(torch.bfloat16).cuda()
    B2 = B[:, :768].contiguous()

    def run():
        u = sm100.lora_shrink(x, A, *csr)
        yy = y.clone()
        sm100.lora_expand_add(yy, u, B, bounds, *csr)
        return u, yy, sm100.lora_expand_silu_mul(pre, u[:, :32].contiguous(), B2, *csr)

    first, second = run(), run()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        graphed = run()
    g.replay()
    torch.cuda.synchronize()
    for a, b, c in zip(first, second, graphed):
        assert torch.equal(a, b) and torch.equal(a, c)


# ---------------------------------------------------------------------------------------------------------------
# engine at real width
# ---------------------------------------------------------------------------------------------------------------
_CFG = dict(hidden_size=4096, num_hidden_layers=2, num_attention_heads=32, num_key_value_heads=8, head_dim=128,
            intermediate_size=12288, vocab_size=2048, torch_dtype="bfloat16", max_position_embeddings=1024)
PROMPTS = [list(range(10, 80)), [5, 9, 100, 7], [77] * 33, list(range(300, 420))]


def _engine(tmp, monkeypatch, **kw):
    from gllm_b200 import LLM
    from gllm_b200.models.presets import tiny
    from lora_util import write_adapter
    monkeypatch.setenv("GLLM_KEEP_LOGITS", "1")
    cfg = tiny("Qwen3ForCausalLM", **_CFG)
    w = write_adapter(str(tmp / "a"), cfg, r=16, alpha=32, seed=1, std=0.05)
    write_adapter(str(tmp / "b"), cfg, r=8, alpha=8, seed=2, std=0.05)
    llm = LLM(cfg, load_format="dummy", maxp=256, maxd=32, max_cuda_graph_bs=8, num_gpu_pages=512,
              model_max_length=1024, log_stats=False, seed=0, enable_prefix_caching=False,
              lora_modules={"a": str(tmp / "a"), "b": str(tmp / "b")}, max_lora_rank=16, **kw)
    return llm, w


def _all_logits(llm):
    """seq id -> its logits rows in step order, from the runner's logit log."""
    out = {}
    for ids, lg in llm.worker.runner.logit_log:
        for i, sid in enumerate(ids):
            out.setdefault(sid, []).append(lg[i].double())
    return out


def _first_logits(llm):
    """seq id -> logits row of its first sampled token (the prefill), from the runner's logit log."""
    out = {}
    for ids, lg in llm.worker.runner.logit_log:
        for i, sid in enumerate(ids):
            out.setdefault(sid, lg[i].double())
    return out


def test_engine_adapter_matches_merged_weights(tmp_path, monkeypatch):
    """Adapter "a" on every prompt vs the base model with W + s·B·A merged into its bf16 weights (same engine, same
    dummy weights). The merged weights are rounded to bf16 once more and the adapter path rounds q/k/v, o and down
    outputs once more, so the prefill logits agree to a relative L2 error of 2 % (measured well below that)."""
    from gllm_b200.ops import ref
    llm, w = _engine(tmp_path, monkeypatch, disable_cuda_graph=True)
    s = 32 / 16
    runner = llm.worker.runner
    outs = llm.generate(tokens=PROMPTS, output_lens=[1] * len(PROMPTS), ignore_eos=True, lora="a")
    got = _first_logits(llm)
    got = [got[o.seq_id] for o in outs]
    runner.logit_log.clear()
    with torch.no_grad():
        for layer in runner.model.layers:
            li = layer.layer_id
            dq, dk, dv = (s * (w[(li, m)][1].double() @ w[(li, m)][0].double()) for m in ("q", "k", "v"))
            at, mlp = layer.attn, layer.mlp
            at.qkv_w.copy_((at.qkv_w.double() + torch.cat([dq, dk, dv]).cuda()).to(at.qkv_w.dtype))
            at.o_w.copy_((at.o_w.double() + (s * w[(li, "o")][1].double() @ w[(li, "o")][0].double()).cuda())
                         .to(at.o_w.dtype))
            gu = torch.cat([s * w[(li, m)][1].double() @ w[(li, m)][0].double() for m in ("gate", "up")])
            mlp.gate_up_w.copy_((mlp.gate_up_w.double() + ref.interleave_gate_up(gu, 128).cuda())
                                .to(mlp.gate_up_w.dtype))
            mlp.down_w.copy_((mlp.down_w.double() + (s * w[(li, "down")][1].double() @ w[(li, "down")][0].double())
                              .cuda()).to(mlp.down_w.dtype))
    base = llm.generate(tokens=PROMPTS, output_lens=[1] * len(PROMPTS), ignore_eos=True)
    want = _first_logits(llm)
    want = [want[o.seq_id] for o in base]
    llm.shutdown()
    for i, (a, b) in enumerate(zip(got, want)):
        rel = (a - b).norm() / b.norm()
        assert rel < 2e-2, (i, float(rel))


def test_engine_graphs_replay_adapter_decode_like_eager(tmp_path, monkeypatch):
    """Mixed batches (adapter a, adapter b, base) decode through the LoRA graph set and agree with eager execution;
    once the adapter requests finish, the base requests replay the plain graphs."""
    lora = ["a", "b", None, "a"]
    lens = [6, 6, 14, 6]
    logs = []
    for eager in (True, False):
        llm, _ = _engine(tmp_path, monkeypatch, disable_cuda_graph=eager)
        outs = llm.generate(tokens=PROMPTS, output_lens=lens, ignore_eos=True, lora=lora)
        st = dict(llm.worker.runner.stats)
        logs.append(([o.token_ids for o in outs], _all_logits(llm), [o.seq_id for o in outs], st))
        llm.shutdown()
    (te, le, ie, se), (tg, lg, ig, sg) = logs
    assert se["graph_steps"] == 0 and sg.get("lora_graph_steps", 0) > 0
    assert sg["graph_steps"] > sg["lora_graph_steps"]      # base-only decode steps replayed the plain graphs
    # every generated token's logits row agrees while the greedy tokens do (the same kernels run in both modes, so
    # the rows are expected bit for bit equal; a near-tie flip would end the comparison of that request)
    compared = 0
    for i, (a, b, x, y, p, n) in enumerate(zip(ie, ig, te, tg, PROMPTS, lens)):
        assert len(le[a]) >= n and len(lg[b]) >= n, (i, len(le[a]), len(lg[b]), n)
        for j in range(n):
            rel = float((le[a][j] - lg[b][j]).norm() / le[a][j].norm())
            assert rel < 1e-2, (i, j, rel)
            compared += 1
            if x[len(p) + j] != y[len(p) + j]:
                break
    assert compared > len(PROMPTS) * 3, compared
