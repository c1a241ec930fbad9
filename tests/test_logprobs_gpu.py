"""Token log-probabilities on the GPU: logprobs_shard_kernel + logprobs_final_kernel (csrc/sample/sampler.cu) element
by element against a float64 oracle built from the exact logits the kernel read, vocab-parallel equivalence, and the
engine with CUDA graphs and async lookahead.

Error bound of one reported log-prob lp = x - lse, lse = m + log z, z = sum_i exp(x_i - m), all in fp32:
  * exp (fast-math __expf): at most (2 + 1.173 |t|) ulp for exp(t), so term i carries a relative error of
    (2 + 1.173 |x_i - m|) * 2^-23; over the row this is sum_i e_i (2 + 1.173 |x_i - m|) 2^-23 / z, computed per row
    from the float64 terms e_i (plus the same for the tp per-shard rescales exp(m_r - gm) in the final kernel);
  * the fp32 sum: a thread adds ceil(V_shard / 1024) terms, a 32-lane shuffle tree and a 32-warp tree add 10 levels,
    the final kernel adds tp shard sums: relative error <= (ceil(V_shard / 1024) + 10 + tp) * 2^-24 to first order;
  * __logf(z), z in [1, V]: absolute error <= max(2^-21.41, 3 ulp(log z));
  * lse = m + log z and x - lse: one fp32 rounding each, <= 2^-24 (|lse| + |lp|).
A relative error r of z is an absolute error r of log z. The sum of these terms (times 1.25 for second-order terms)
is about 2e-5 at V = 151936 with logits of magnitude 10; the token ids are compared exactly (ordering raw logits
involves no arithmetic).
"""
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MAX_LOGPROBS = 20
ULP23, ULP24 = 2.0 ** -23, 2.0 ** -24


def _dev():
    return torch.device("cuda")


def _oracle(x64: np.ndarray, n: int):
    """float64 log_softmax of one row, and its n best token ids by (logit desc, id asc)."""
    m = x64.max()
    t = x64 - m
    e = np.exp(t)
    z = e.sum()
    lp = t - math.log(z)
    order = np.lexsort((np.arange(x64.size), -x64))[:n]
    return lp, order, m, z, e, t


def _bound(x64, lp64, m, z, e, t, shard_len: int, tp: int, shard_max=None) -> np.ndarray:
    fin = np.isfinite(t)
    exp_rel = float((e[fin] * (2 + 1.173 * np.abs(t[fin]))).sum() * ULP23 / z)
    if shard_max is not None:       # the final kernel rescales each shard sum with exp(m_r - gm)
        exp_rel += float(sum((2 + 1.173 * abs(mr - m)) for mr in shard_max if np.isfinite(mr)) * ULP23)
    sum_rel = (math.ceil(shard_len / 1024) + 10 + tp) * ULP24
    logz = math.log(z)
    log_abs = max(2.0 ** -21.41, 3 * ULP24 * 2 * max(abs(logz), 1e-30))
    lse = m + logz
    return 1.25 * (exp_rel + sum_rel + log_abs + ULP24 * (abs(lse) + np.abs(lp64))) + 1e-7


def _logits(b: int, v: int, pad: int, dtype, seed: int):
    """[b, v + pad] rows: random and adversarial; the `pad` trailing columns are huge and must be ignored."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, v + pad, generator=g) * 3
    x[:, v:] = 1e4
    n_tie = min(40, v)
    if b > 1:   # ties around the N-th place: a few clear winners, then a block of equal logits
        idx = torch.randperm(v, generator=g)[: n_tie + 3]
        x[1, idx[:3]] = 12.0
        x[1, idx[3:]] = 9.0
    if b > 2:
        x[2, 123 % v] = 60.0                 # one peaked logit
    if b > 3:
        x[3, :v] = 0.5                       # all equal
    if b > 4:
        x[4, : v : 3] = float("-inf")        # -inf and huge negative logits
        x[4, 1 : v : 5] = -1e30
    if b > 6:
        x[6, :v] = torch.arange(v, dtype=torch.float32) % 7      # many ties everywhere
    return x.to(dtype).to(_dev())


def _check(out: torch.Tensor, logits: torch.Tensor, v: int, n: int, toks: torch.Tensor, rows, tp: int = 1,
           shard_len: int = None, what: str = ""):
    """Every reported element against the float64 oracle; the message names the worst row and token."""
    out = out.cpu()
    vals, ids = out.numpy(), out.view(torch.int32).numpy()
    x_all = logits[:, :v].double().cpu().numpy()
    toks = toks.cpu().numpy()
    shard_len = shard_len or v
    worst = (0.0, None)
    for j, r in enumerate(rows):
        x64 = x_all[r]
        lp64, order, m, z, e, t = _oracle(x64, n)
        per = shard_len
        smax = [x64[k * per:(k + 1) * per].max() if k * per < v else -np.inf for k in range(tp)] if tp > 1 else None
        bnd = _bound(x64, lp64, m, z, e, t, shard_len, tp, smax)
        k = min(n, v)
        got_ids = ids[j, 1:1 + 2 * n:2]
        assert list(got_ids[:k]) == list(order[:k]), \
            f"{what}: row {r}: top-{n} ids {list(got_ids[:k])} != oracle {list(order[:k])}"
        assert (got_ids[k:] == -1).all(), f"{what}: row {r}: slots past the vocabulary {got_ids[k:]}"
        checks = [(int(toks[r]), float(vals[j, 0]), "sampled")] + \
                 [(int(order[i]), float(vals[j, 2 + 2 * i]), f"top{i}") for i in range(k)]
        for tok, got, kind in checks:
            want = lp64[tok]
            if not np.isfinite(want):
                assert got == want or (want < 0 and got < -1e30), f"{what}: row {r} {kind} token {tok}: {got} vs {want}"
                continue
            err = abs(got - want)
            ratio = err / bnd[tok]
            if ratio > worst[0]:
                worst = (ratio, (r, tok, kind, got, want, bnd[tok]))
    assert worst[0] <= 1.0, f"{what}: worst row {worst[1][0]} token {worst[1][1]} ({worst[1][2]}): " \
                            f"got {worst[1][3]:.8g}, float64 {worst[1][4]:.8g}, bound {worst[1][5]:.3g}"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("n", [0, 1, 5, 20])
@pytest.mark.parametrize("v", [151936, 1001, 13])
def test_logprobs_kernels_match_float64_oracle(v, n, dtype):
    from gllm_b200.ops import sm100
    b = 12
    logits = _logits(b, v, 64, dtype, seed=v + n)
    x = logits[:, :v].float()
    toks = x.argmax(-1).to(torch.int32)                  # greedy rows: lowest id among equal maxima
    toks[5] = int(x[5].argmin())                         # a sampled token deep in the tail
    toks[7] = (toks[7] + 17) % v
    rows = [0, 1, 2, 3, 4, 5, 6, 7, 9, 11]               # rows 8 and 10 do not ask
    rec = sm100.logprobs_shard(logits, v, n, toks, torch.tensor(rows, dtype=torch.int32, device=_dev()))
    out = sm100.logprobs_final(rec.unsqueeze(0), n)
    torch.cuda.synchronize()
    assert out.shape == (len(rows), 1 + 2 * n)
    _check(out, logits, v, n, toks, rows, what=f"V={v} N={n} {dtype}")
    if n:   # a greedy row reports its sampled token first
        ids = out.cpu().view(torch.int32)
        for j, r in enumerate(rows):
            if r not in (5, 7):
                assert int(ids[j, 1]) == int(toks[r]), (r, int(ids[j, 1]), int(toks[r]))


@pytest.mark.parametrize("tp,v", [(2, 151936), (8, 151936), (8, 300)])
@pytest.mark.parametrize("n", [1, 20])
def test_vocab_parallel_logprobs_equal_single_rank(tp, v, n):
    """Shards of one padded matrix (the last shard ends with padding; at V = 300, tp = 8 the shards from the third on
    are only padding): the gathered records give the same ids as tp = 1 and log-probs within the bound."""
    from gllm_b200.ops import sm100
    per = (v + tp - 1) // tp
    per = (per + 127) // 128 * 128
    b = 12
    logits = _logits(b, v, tp * per - v, torch.bfloat16, seed=tp * 7 + n)
    toks = logits[:, :v].float().argmax(-1).to(torch.int32)
    toks[5] = int(logits[5, :v].float().argmin())
    rows_l = [0, 1, 2, 3, 4, 5, 6, 9]
    rows = torch.tensor(rows_l, dtype=torch.int32, device=_dev())
    single = sm100.logprobs_final(sm100.logprobs_shard(logits, v, n, toks, rows).unsqueeze(0), n)
    recs = []
    for r in range(tp):
        lo = r * per
        valid = max(0, min(per, v - lo))
        recs.append(sm100.logprobs_shard(logits[:, lo:lo + per], valid, n, toks, rows, vocab_offset=lo))
    out = sm100.logprobs_final(torch.stack(recs).contiguous(), n)
    torch.cuda.synchronize()
    assert torch.equal(out.cpu().view(torch.int32)[:, 1::2], single.cpu().view(torch.int32)[:, 1::2])
    _check(out, logits, v, n, toks, rows_l, tp=tp, shard_len=per, what=f"tp={tp} V={v} N={n}")


def _engine_cfg():
    from gllm_b200.models.presets import tiny
    return tiny("Qwen3ForCausalLM", hidden_size=256, num_hidden_layers=3, num_attention_heads=4,
                num_key_value_heads=2, head_dim=64, intermediate_size=512, vocab_size=1024, torch_dtype="bfloat16")


def test_engine_logprobs_match_the_kept_logits(monkeypatch):
    """CUDA graphs and async lookahead on, greedy and sampled requests with and without log-probs in one batch: every
    reported log-prob equals log_softmax of that step's logits, a greedy row's first entry is its token, and the
    tokens equal those of the same run without log-probs."""
    from gllm_b200 import LLM
    monkeypatch.setenv("GLLM_KEEP_LOGITS", "1")
    prompts = [[5, 9, 100, 7], list(range(20, 190)), [77] * 33, [3, 1, 4, 1, 5, 9, 2, 6]]
    kw = dict(ignore_eos=True, output_lens=[12] * 4, temperature=[0.0, 0.0, 0.8, 0.0], top_k=[1, 1, 8, 1])
    res = {}
    for lp in (None, [5, None, 3, 20]):
        torch.manual_seed(0)
        llm = LLM(_engine_cfg(), load_format="dummy", maxp=128, maxd=64, max_cuda_graph_bs=8, num_gpu_pages=256,
                  model_max_length=512, log_stats=False, seed=0, async_schedule=True)
        outs = llm.generate(tokens=prompts, logprobs=lp, **kw)
        runner = llm.worker.runner
        assert runner.stats["graph_steps"] > 0
        per_seq = {s.seq_id: [] for s in outs}
        for ids, lg in runner.logit_log:
            for row, sid in enumerate(ids):
                if sid in per_seq:
                    per_seq[sid].append(lg[row])
        res[lp is None] = ([s.token_ids[len(p):] for s, p in zip(outs, prompts)], outs, per_seq)
        llm.shutdown()
    toks0 = res[True][0]
    toks1, outs, per_seq = res[False]
    assert toks0 == toks1
    for i, s in enumerate(outs):
        want_n = [5, None, 3, 20][i]
        if want_n is None:
            assert s.output_logprobs == []
            continue
        assert len(s.output_logprobs) == s.num_output_tokens == 12
        for j, (chosen, top) in enumerate(s.output_logprobs):
            x64 = per_seq[s.seq_id][j].double().numpy()
            lp64, order, m, z, e, t = _oracle(x64, want_n)
            bnd = _bound(x64, lp64, m, z, e, t, x64.size, 1)
            tok = toks1[i][j]
            assert abs(chosen - lp64[tok]) <= bnd[tok], (i, j, tok, chosen, lp64[tok])
            assert [a for a, _ in top] == list(order), (i, j)
            for a, val in top:
                assert abs(val - lp64[a]) <= bnd[a], (i, j, a, val, lp64[a])
            if i != 2:
                assert top[0][0] == tok and top[0][1] == chosen


def test_tp2_engine_logprobs_equal_tp1():
    """Vocab-parallel log-prob records across two GPUs (NCCL all-gather) reproduce the single-GPU log-probs."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import json
    import subprocess
    import sys
    import tempfile
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = os.path.join(root, "tests", "mp_logprobs.py")
    outs = {}
    with tempfile.TemporaryDirectory() as d:
        for tp in (1, 2):
            out = os.path.join(d, f"tp{tp}.json")
            cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={tp}",
                   "--master-addr", "127.0.0.1", "--master-port", str(29990 + tp), script, "1", str(tp), out, "cuda"]
            r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=root,
                               env=dict(os.environ, PYTHONPATH=root))
            assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
            outs[tp] = json.load(open(out))
    # bf16 activations reduced across two GPUs round differently from one GPU: compare while the tokens agree (later
    # steps run on different inputs), with a tolerance for that rounding rather than for the log-prob kernels
    for (ta, la), (tb, lb) in zip(outs[1], outs[2]):
        for j in range(len(ta)):
            assert abs(la[j][0] - lb[j][0]) < 5e-2, (j, la[j][0], lb[j][0])
            if ta[j] != tb[j]:
                break
