"""Per-request `seed`, `frequency_penalty`, `presence_penalty` and `logit_bias` on the GPU: the sampler kernels
(csrc/sample/sampler.cu) against a float64 oracle built from the exact logits they read, the bias-row accounting
bit for bit against an fp32 numpy replay, the seeded race's distribution, and the engine with CUDA graphs and async
lookahead against the oracle replayed on its kept logits.

Rounding bounds used below (all fp32, --use_fast_math):
  * bias row: logit_bias_j (exact in fp32), then one fp32 subtraction per generated occurrence of j (of f, or of
    fl(f + p) the first time): each rounds once, |err| <= 2^-24 |partial|, so over c_j occurrences
    |err(b_j)| <= 2^-24 (c_j + 1) (|lb_j| + c_j (|f| + |p|));
  * x + b_j: one more rounding, 2^-24 |x + b_j|; times inv_temp = 1 (temperature 1) is exact;
  * greedy: the kernel's argmax may differ from the float64 argmax only when the two values lie within the sum of
    their bounds (bnd below doubles the terms for second-order slack);
  * seeded draw: t = fl(x2 * fl(1 / T)) (fast-math reciprocal: 2 ulp) gives |err(t)| <= 2^-22 |t| + err(x2) / T;
    the score (t - m) - __logf(e), e = -__logf(u), adds 2^-24 |t - m| for the subtraction, __logf's absolute error
    2^-21.41 (plus 2 ulp of |log u|) divided by e for e, and 2^-21.41 + 2 ulp for log e.
"""
import os

import numpy as np
import pytest
import torch

import mp_sampling_params as mp

pytestmark = pytest.mark.gpu

U24, U22 = 2.0 ** -24, 2.0 ** -22
LOGF_ABS = 2.0 ** -21.41


def _dev():
    return torch.device("cuda")


def _rows(b, v, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, v, generator=g) * 3
    x[1, 7 % v] = 40.0                         # peaked
    x[2, :] = 0.5                              # all equal
    x[3, ::3] = float("-inf")                  # -inf entries
    x[4, :] = torch.arange(v, dtype=torch.float32) % 5       # ties everywhere
    return x.to(dtype)


def _bias_spec(b, v, seed):
    """Per row: (f, p, {token: logit_bias}, output tokens with repeats); both signs."""
    rng = np.random.default_rng(seed)
    specs = []
    for r in range(b):
        f = float(np.float32(rng.uniform(-2, 2)))
        p = float(np.float32(rng.uniform(-2, 2)))
        ids = rng.choice(v, size=min(v, 6), replace=False).tolist()
        lb = {int(i): float(np.float32(rng.uniform(-100, 100) if k % 2 else rng.uniform(-5, 5)))
              for k, i in enumerate(ids)}
        outs = rng.integers(0, min(v, 20), size=int(rng.integers(0, 30))).tolist()
        specs.append((f, p, lb, outs))
    return specs


def _numpy_bias(v, f, p, lb, outs):
    """fp32 numpy replay of bias_rebuild_kernel / bias_account_kernel."""
    row = np.zeros(v, dtype=np.float32)
    for t, b in lb.items():
        row[t] = np.float32(b)
    f32, p32 = np.float32(f), np.float32(p)
    seen = set()
    for t in outs:
        row[t] = row[t] - ((f32 + p32) if t not in seen else f32)
        seen.add(t)
    return row


def _rebuild(bias, out_seen, v, slots, specs):
    from gllm_b200.ops import sm100
    lb_off, lb_ids, lb_vals, out_off, out_toks = [0], [], [], [0], []
    for f, p, lb, outs in specs:
        lb_ids += list(lb)
        lb_vals += list(lb.values())
        lb_off.append(len(lb_ids))
        out_toks += outs
        out_off.append(len(out_toks))
    d = _dev()
    i32 = lambda a: torch.tensor(a, dtype=torch.int32, device=d)   # noqa: E731
    sm100.bias_rebuild(bias, out_seen, v, i32(slots),
                       torch.tensor([[f, p] for f, p, _, _ in specs], dtype=torch.float32, device=d),
                       i32(lb_off), i32(lb_ids), torch.tensor(lb_vals, dtype=torch.float32, device=d), i32(out_off),
                       i32(out_toks))


def _exact_x2(x64, v, f, p, lb, outs):
    b = np.zeros(v)
    for t, val in lb.items():
        b[t] = val
    for t, c in zip(*np.unique(np.asarray(outs, dtype=np.int64), return_counts=True)) if outs else []:
        b[t] -= f * c + p
    return x64 + b


def _bias_bound(x64, v, f, p, lb, outs):
    c = np.bincount(np.asarray(outs, dtype=np.int64), minlength=v)[:v] if outs else np.zeros(v)
    lbv = np.zeros(v)
    for t, val in lb.items():
        lbv[t] = abs(val)
    b_abs = lbv + c * (abs(f) + abs(p))
    xa = np.where(np.isfinite(x64), np.abs(x64), 0.0)
    return 2 * U24 * ((c + 1) * b_abs + xa + b_abs)


# ------------------------------------------------------------------------------------------------
# 1. greedy with bias
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("v", [151936, 1001, 13])
def test_greedy_with_bias_is_the_argmax_of_x2(v, dtype):
    from gllm_b200.ops import sm100
    b = 10
    x = _rows(b, v, dtype, seed=v)
    specs = _bias_spec(b, v, seed=v + 1)
    slots = [2 * r + 1 for r in range(b)]
    bias = torch.full((2 * b + 1, v), 7.0, device=_dev())          # stale contents: the rebuild clears them
    out_seen = torch.full((2 * b + 1, (v + 31) // 32), -1, dtype=torch.int32, device=_dev())
    _rebuild(bias, out_seen, v, slots, specs)
    bslot = torch.tensor(slots, dtype=torch.int32, device=_dev())
    bslot[5] = -1                                                  # a row without a bias row
    tok = sm100.sample(x.to(_dev()), top_k=torch.ones(b, dtype=torch.int32, device=_dev()), bias=bias,
                       bias_slot=bslot).cpu().numpy()
    x64 = x.float().double().numpy()
    near = 0
    for r in range(b):
        f, p, lb, outs = specs[r] if r != 5 else (0.0, 0.0, {}, [])
        x2 = _exact_x2(x64[r], v, f, p, lb, outs)
        want = int(np.lexsort((np.arange(v), -x2))[0])
        if int(tok[r]) != want:
            bnd = _bias_bound(x64[r], v, f, p, lb, outs)
            got = int(tok[r])
            assert x2[want] - x2[got] <= bnd[want] + bnd[got], (r, got, want, x2[want], x2[got])
            near += 1
    assert near <= 1, near


# ------------------------------------------------------------------------------------------------
# 2. seeded draw
# ------------------------------------------------------------------------------------------------
def _race_bound(t, m, u, temp):
    e = -np.log(u.astype(np.float64))
    loge = np.abs(np.log(u.astype(np.float64)))
    return (U22 * np.abs(t) + 2 * U24 * (np.abs(t) + abs(m)) + (LOGF_ABS + 2 * U24 * loge) / e + LOGF_ABS
            + 2 * U24 * np.abs(np.log(e))) * 2


def _seeded_oracle(x2, temp, top_k, seed, pos):
    from gllm_b200.ops import ref
    t = x2 / temp
    s = mp.race_scores(t, seed, pos, top_k)
    want = int(np.lexsort((np.arange(t.size), -s))[0])
    u = ref.race_uniform(seed, pos, np.arange(t.size))
    m = t[np.isfinite(s)].max()
    return s, want, _race_bound(t, m, u, temp)


@pytest.mark.parametrize("v", [151936, 1001])
def test_seeded_draw_follows_the_port_and_is_batch_invariant(v):
    from gllm_b200.ops import sm100
    b = 16
    d = _dev()
    x = _rows(b, v, torch.bfloat16, seed=3 * v).to(d)
    temp = torch.full((b,), 0.7, device=d)
    top_k = torch.tensor([0 if r % 2 else 50 for r in range(b)], dtype=torch.int32, device=d)
    top_p = torch.ones(b, device=d)
    seeds = torch.tensor([1000 + r if r != 6 else -(2 ** 63) for r in range(b)], dtype=torch.int64, device=d)
    pos = torch.tensor([r * 17 if r not in (4, 9) else -1 for r in range(b)], dtype=torch.int32, device=d)
    step = torch.zeros(1, dtype=torch.int64, device=d)
    tok = sm100.sample(x, temp, top_k, top_p, seed=5, step=step, seeds=seeds, seed_pos=pos).cpu().numpy()
    x64 = x.float().double().cpu().numpy()
    near = 0
    for r in range(b):
        if int(pos[r]) < 0:
            continue
        s, want, bnd = _seeded_oracle(x64[r], 0.7, int(top_k[r]), int(seeds[r]), int(pos[r]))
        got = int(tok[r])
        if got != want:
            assert s[want] - s[got] <= bnd[want] + bnd[got], (r, got, want)
            near += 1
    assert near <= 1
    # the same row at other rows, batch sizes and step counters: the same token
    for r in range(b):
        if int(pos[r]) < 0:
            continue
        for nb, at, stp in ((1, 0, 0), (5, 3, 7), (33, 20, 12345)):
            xs = x[r:r + 1].repeat(nb, 1).contiguous()
            z = lambda t: t[r:r + 1].repeat(nb).contiguous()       # noqa: E731
            stp_t = torch.full((1,), stp, dtype=torch.int64, device=d)
            t2 = sm100.sample(xs, z(temp), z(top_k), z(top_p), seed=stp * 31, step=stp_t, seeds=z(seeds),
                              seed_pos=z(pos)).cpu()
            assert int(t2[at]) == int(tok[r]), (r, nb, at, stp)
    # unseeded rows: bit-identical to a call without the new arguments
    plain = sm100.sample(x, temp, top_k, top_p, seed=5, step=step).cpu().numpy()
    for r in (4, 9):
        assert plain[r] == tok[r]
    none = torch.full((b,), -1, dtype=torch.int32, device=d)
    assert np.array_equal(sm100.sample(x, temp, top_k, top_p, seed=5, step=step, seeds=seeds, seed_pos=none)
                          .cpu().numpy(), plain)


# ------------------------------------------------------------------------------------------------
# 3. vocab parallel
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tp,v", [(2, 151936), (8, 151936), (8, 300)])
def test_vocab_parallel_equals_plain_for_seeded_and_biased_rows(tp, v):
    from gllm_b200.ops import sm100
    d = _dev()
    b = 12
    per = (v + tp - 1) // tp
    per = (per + 127) // 128 * 128                     # at V = 300, tp = 8 the shards from the third on are padding
    x = torch.zeros(b, tp * per, dtype=torch.bfloat16, device=d)
    x[:, :v] = _rows(b, v, torch.bfloat16, seed=tp + v).to(d)
    x[:, v:] = 1e4
    specs = _bias_spec(b, v, seed=tp)
    bias = torch.zeros(b + 1, v, device=d)
    out_seen = torch.zeros(b + 1, (v + 31) // 32, dtype=torch.int32, device=d)
    _rebuild(bias, out_seen, v, list(range(1, b + 1)), specs)
    bslot = torch.tensor([r + 1 if r % 3 else -1 for r in range(b)], dtype=torch.int32, device=d)
    temp = torch.full((b,), 0.9, device=d)
    top_k = torch.tensor([[0, 50, 256, 1][r % 4] for r in range(b)], dtype=torch.int32, device=d)
    top_p = torch.ones(b, device=d)
    seeds = torch.arange(b, dtype=torch.int64, device=d) * 977
    pos = torch.tensor([r if r % 5 else -1 for r in range(b)], dtype=torch.int32, device=d)
    step = torch.full((1,), 3, dtype=torch.int64, device=d)
    kw = dict(bias=bias, bias_slot=bslot, seeds=seeds, seed_pos=pos)
    full = sm100.sample(x[:, :v].contiguous(), temp, top_k, top_p, seed=77, step=step, **kw)
    c = min(256, per)
    recs = []
    for r in range(tp):
        lo = r * per
        valid = max(0, min(per, v - lo))
        recs.append(sm100.vp_candidates(x[:, lo:lo + per], valid, v, c, temp, top_k, top_p, seed=77, step=step,
                                        vocab_offset=lo, **kw))
    toks = sm100.vp_final(torch.stack(recs).contiguous(), c, v, top_k, top_p, seed=77, step=step, seeds=seeds,
                          seed_pos=pos)
    assert torch.equal(toks.cpu(), full.cpu()), (toks.cpu().tolist(), full.cpu().tolist())


# ------------------------------------------------------------------------------------------------
# 4. distribution of the seeded race
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("route", ["plain", "vp2"])
@pytest.mark.parametrize("filt", ["unfiltered", "topk5_topp08"])
def test_seeded_draws_follow_the_filtered_distribution(route, filt):
    """4096 fixed seeds over one logits row: chi-square against ref.sample_filter's probabilities (deterministic:
    the seeds are fixed)."""
    from scipy.stats import chisquare
    from gllm_b200.ops import ref, sm100
    d = _dev()
    n, v = 4096, 13
    row = torch.tensor([1.0, 0.2, -0.5, 2.0, 0.0, 1.5, -1.0, 0.7, 0.3, -2.0, 1.1, 0.9, -0.2])
    x = row.repeat(n, 1).to(d)
    temp = torch.full((n,), 0.8, device=d)
    k, p = (0, 1.0) if filt == "unfiltered" else (5, 0.8)
    top_k = torch.full((n,), k, dtype=torch.int32, device=d)
    top_p = torch.full((n,), p, device=d)
    seeds = torch.arange(n, dtype=torch.int64, device=d) * 7919 + 3
    pos = torch.full((n,), 11, dtype=torch.int32, device=d)
    if route == "plain":
        tok = sm100.sample(x, temp, top_k, top_p, seeds=seeds, seed_pos=pos)
    else:
        recs = [sm100.vp_candidates(x[:, lo:lo + 7].contiguous(), min(7, v - lo), v, 7, temp, top_k, top_p,
                                    vocab_offset=lo, seeds=seeds, seed_pos=pos) for lo in (0, 7)]
        tok = sm100.vp_final(torch.stack(recs).contiguous(), 7, v, top_k, top_p, seeds=seeds, seed_pos=pos)
    cnt = np.bincount(tok.cpu().numpy(), minlength=v)
    probs = ref.sample_filter(row[None].double(), torch.tensor([0.8]), torch.tensor([k if k else v]),
                              torch.tensor([p]))[0].numpy()
    assert cnt[probs == 0].sum() == 0, (cnt, probs)
    live = probs > 0
    expect = probs[live].astype(np.float64)
    expect = expect / expect.sum() * n
    expect *= cnt[live].sum() / expect.sum()          # (scipy checks both sums agree to 1.5e-8)
    _, pval = chisquare(cnt[live], expect)
    assert pval > 1e-3, (pval, cnt, probs * n)


# ------------------------------------------------------------------------------------------------
# 5. accounting
# ------------------------------------------------------------------------------------------------
def test_accounting_and_rebuild_equal_the_fp32_replay():
    from gllm_b200.ops import sm100
    d = _dev()
    v = 1001
    specs = [(0.5, 0.25, {3: 1.0, 900: -100.0}, []), (-1.3, 2.0, {}, []), (0.1, -0.7, {5: 0.3}, [])]
    slots = [4, 1, 7]
    bias = torch.zeros(8, v, device=d)
    out_seen = torch.zeros(8, (v + 31) // 32, dtype=torch.int32, device=d)
    _rebuild(bias, out_seen, v, slots, specs)
    rng = np.random.default_rng(0)
    emitted = [[] for _ in slots]
    bslot = torch.tensor(slots + [-1], dtype=torch.int32, device=d)          # a fourth row without a bias row
    freq = torch.tensor([s[0] for s in specs] + [0.0], device=d)
    pres = torch.tensor([s[1] for s in specs] + [0.0], device=d)
    for step in range(40):
        toks = rng.integers(0, 40, size=4).astype(np.int32)
        sm100.bias_account(bias, out_seen, bslot, torch.from_numpy(toks).to(d), freq, pres)
        for i in range(3):
            emitted[i].append(int(toks[i]))
    # "preemption" of the second row: its slot is rebuilt from the outputs so far, into another slot
    _rebuild(bias, out_seen, v, [2], [(specs[1][0], specs[1][1], specs[1][2], emitted[1])])
    torch.cuda.synchronize()
    got, seen = bias.cpu().numpy(), out_seen.cpu().numpy()
    for i, (f, p, lb, _) in enumerate(specs):
        want = _numpy_bias(v, f, p, lb, emitted[i])
        assert np.array_equal(got[slots[i]], want), i
        bits = np.unpackbits(seen[slots[i]].view(np.uint8), bitorder="little")[:v]
        assert set(np.nonzero(bits)[0].tolist()) == set(emitted[i])
    assert np.array_equal(got[2], got[1]) and np.array_equal(seen[2], seen[1])
    assert not got[0].any() and not got[3].any()


# ------------------------------------------------------------------------------------------------
# 6. engine
# ------------------------------------------------------------------------------------------------
def _engine_cfg():
    from gllm_b200.models.presets import tiny
    return tiny("Qwen3ForCausalLM", hidden_size=256, num_hidden_layers=3, num_attention_heads=4,
                num_key_value_heads=2, head_dim=64, intermediate_size=512, vocab_size=1024, torch_dtype="bfloat16")


def _llm(**kw):
    from gllm_b200 import LLM
    torch.manual_seed(0)
    return LLM(_engine_cfg(), load_format="dummy", maxp=128, maxd=64, max_cuda_graph_bs=8, num_gpu_pages=256,
               model_max_length=512, log_stats=False, seed=0, async_schedule=True, **kw)


def _per_seq(runner, outs):
    per = {s.seq_id: [] for s in outs}
    for ids, lg in runner.logit_log:
        for row, sid in enumerate(ids):
            if sid in per:
                per[sid].append(lg[row].double().numpy())
    return per


def _tol_gpu(x, s, want, tok):
    # the bounds of the module docstring for |x2| <= 64, c_j <= 16 and an exponential variate e >= 2^-10 (smaller
    # ones win their race by far more than this): about 1.5e-5, doubled
    return 3e-5


PROMPTS = [[5, 9, 100, 7], list(range(20, 190)), [77] * 33, [3, 1, 4, 1, 5, 9, 2, 6]]


def test_engine_follows_the_oracle_with_graphs_and_lookahead(monkeypatch):
    monkeypatch.setenv("GLLM_KEEP_LOGITS", "1")
    ps = [dict(mp.MIXED[0]), dict(mp.MIXED[1]), dict(mp.MIXED[2]), dict(mp.MIXED[3])]
    llm = _llm()
    outs = llm.generate(tokens=PROMPTS, output_lens=[16, 16, 16, 4], ignore_eos=True, top_p=1.0,
                        **{k: [p.get(k, 1.0 if k == "repetition_penalty" else None) for p in ps]
                           for k in ("temperature", "top_k", "seed", "frequency_penalty", "presence_penalty",
                                     "logit_bias", "repetition_penalty")})
    runner = llm.worker.runner
    assert runner.stats["graph_steps"] > 0 and runner.stats.get("feed_steps", 0) > 0
    per = _per_seq(runner, outs)
    llm.shutdown()
    near = 0
    for s, pr, p in zip(outs, PROMPTS, ps):
        toks = s.token_ids[len(pr):]
        assert len(per[s.seq_id]) == len(toks)
        near += mp.replay(pr, toks, per[s.seq_id], p, _tol_gpu)
    assert near <= 2
    assert 100 not in outs[0].token_ids[len(PROMPTS[0]):]


def test_seeded_requests_in_reverse_order_give_the_same_tokens(monkeypatch):
    monkeypatch.setenv("GLLM_KEEP_LOGITS", "1")
    prompts = [[5, 9, 100, 7], [3, 1, 4, 1, 5, 9, 2, 6], [77] * 33, [8, 8, 8]]
    kw = dict(temperature=0.9, top_k=[0, 30, 0, 5], seed=[11, 22, 33, 44], frequency_penalty=[0.3, 0.0, 0.3, 0.0],
              logit_bias=[None, {5: 2.0}, None, None])
    res = []
    for order in ([0, 1, 2, 3], [3, 2, 1, 0]):
        llm = _llm()
        outs = llm.generate(tokens=[prompts[i] for i in order], output_lens=[8] * 4, ignore_eos=True,
                            **{k: ([v[i] for i in order] if isinstance(v, list) else v) for k, v in kw.items()})
        per = _per_seq(llm.worker.runner, outs)
        res.append({order[j]: (s.token_ids[len(prompts[order[j]]):], per[s.seq_id]) for j, s in enumerate(outs)})
        llm.shutdown()
    for i in range(4):
        (ta, la), (tb, lb) = res[0][i], res[1][i]
        assert np.array_equal(la[0], lb[0])          # one prefill step: bitwise equal logits in either order
        for j in range(len(ta)):
            if not np.array_equal(la[j], lb[j]):
                break                                # (later steps ran in other batches: compare while equal)
            assert ta[j] == tb[j], (i, j)


def test_run_without_the_new_parameters_matches_the_parent_engine():
    """Tokens of a run that uses none of the new parameters, against those the engine produced before they existed
    (tests/golden/sampling_params_plain_tokens.json, same inputs on an H100)."""
    import json
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "tests", "golden", "sampling_params_plain_tokens.json")) as f:
        want = json.load(f)
    assert plain_run_tokens() == want


def plain_run_tokens():
    """Greedy and sampled requests, CUDA graphs and lookahead, no new parameter (also run by the golden's recipe)."""
    llm = _llm()
    outs = llm.generate(tokens=PROMPTS, output_lens=[12] * 4, ignore_eos=True, temperature=[0.0, 0.8, 0.7, 0.0],
                        top_k=[1, 8, 0, 1], repetition_penalty=[1.0, 1.0, 1.0, 1.2])
    toks = [s.token_ids[len(p):] for s, p in zip(outs, PROMPTS)]
    llm.shutdown()
    return toks


# ------------------------------------------------------------------------------------------------
# 7. TP2
# ------------------------------------------------------------------------------------------------
def test_tp2_engine_follows_the_oracle():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import json
    import subprocess
    import sys
    import tempfile
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with tempfile.TemporaryDirectory() as d:
        out = os.path.join(d, "tp2.json")
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
               "--master-addr", "127.0.0.1", "--master-port", "29971", os.path.join(root, "tests",
                                                                                  "mp_sampling_params.py"),
               "1", "2", out, "cuda"]
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=root,
                           env=dict(os.environ, PYTHONPATH=root))
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
        got = json.load(open(out))
    near = 0
    for i, (prompt, outs, steps) in enumerate(got):
        near += mp.replay(prompt, outs, steps, mp.MIXED[i], _tol_gpu)
    assert near <= 2
