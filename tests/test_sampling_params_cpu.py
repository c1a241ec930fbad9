"""Per-request `seed`, `frequency_penalty`, `presence_penalty` and `logit_bias` on the CPU: the seeded race port, the
wire format and the incremental decode path, the engine against a manual HuggingFace loop applying the formula,
TP2 / PP2 over gloo, batch-order invariance of seeded requests, and the OpenAI API (400s, fields reaching the
`Sequence`)."""
from conftest import scratch_dir
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import mp_sampling_params as mp  # noqa: E402


# ------------------------------------------------------------------------------------------------
# seeded race
# ------------------------------------------------------------------------------------------------
def test_race_uniform_is_the_kernel_stream():
    """Values of csrc/sample/sampler.cu:rand_exp's uniform, computed by its C expression on uint32 arithmetic."""
    from gllm_b200.ops import ref
    got = ref.race_uniform(0, 0, [0, 1, 151935, 4294967295])
    want = np.array([0.327775508, 0.0363021195, 0.0802614987, 0.672565103], dtype=np.float32)
    assert np.array_equal(got, want), got
    got = ref.race_uniform(0, 5, [0, 1, 151935, 4294967295])
    assert np.array_equal(got, np.array([0.780790567, 0.155373007, 0.778117895, 0.45351842], dtype=np.float32))
    u = ref.race_uniform(-7, 123, np.arange(100000))
    assert u.dtype == np.float32 and (u > 0).all() and (u < 1).all() and abs(float(u.mean()) - 0.5) < 0.01


def test_ref_sample_seeded_rows_are_batch_invariant():
    from gllm_b200.ops import ref
    torch.manual_seed(0)
    x = torch.randn(6, 50) * 2
    t = torch.full((6,), 0.9)
    k = torch.tensor([10, 50, 10, 5, 50, 10], dtype=torch.int32)
    p = torch.ones(6)
    seeds = torch.tensor([11, 0, 11, 42, 7, 11], dtype=torch.int64)
    pos = torch.tensor([3, -1, 3, 9, 0, 4], dtype=torch.int32)
    a = ref.sample(x, t, k, p, generator=torch.Generator().manual_seed(1), seeds=seeds, seed_pos=pos)
    perm = [5, 4, 3, 2, 1, 0]
    b = ref.sample(x[perm], t[perm], k[perm], p[perm], generator=torch.Generator().manual_seed(99), seeds=seeds[perm],
                   seed_pos=pos[perm])
    for i, j in enumerate(perm):
        if int(pos[j]) >= 0:
            assert int(b[i]) == int(a[j])


def test_ref_bias_rebuild_equals_token_by_token_accounting():
    from gllm_b200.ops import ref
    v = 70
    b1, s1 = torch.zeros(3, v), torch.zeros(3, (v + 31) // 32, dtype=torch.int32)
    b2, s2 = b1.clone(), s1.clone()
    outs = [5, 69, 5, 33, 5, 69, 0]
    ref.bias_rebuild(b1, s1, 2, 0.3, -0.7, [5, 40], [1.5, -100.0], [])
    for t in outs:
        ref.bias_account_one(b1, s1, 2, t, 0.3, -0.7)
    ref.bias_rebuild(b2, s2, 2, 0.3, -0.7, [5, 40], [1.5, -100.0], outs)
    assert torch.equal(b1, b2) and torch.equal(s1, s2)
    want = np.zeros(v, dtype=np.float32)
    want[5], want[40] = 1.5, -100.0
    f, p = np.float32(0.3), np.float32(-0.7)
    seen = set()
    for t in outs:
        want[t] = want[t] - ((f + p) if t not in seen else f)
        seen.add(t)
    assert np.array_equal(b1[2].numpy(), want)
    assert set(np.nonzero(np.unpackbits(s1[2].numpy().view(np.uint8), bitorder="little"))[0].tolist()) == seen


# ------------------------------------------------------------------------------------------------
# wire format, incremental decode path
# ------------------------------------------------------------------------------------------------
def _seq(sid, prompt, outs, **kw):
    from gllm_b200.sequence import Sequence
    s = Sequence(sid, prompt, [], **kw)
    s.token_ids += outs
    s.page_table = [sid * 4 + i for i in range(4)]
    s.computed_token_num = s.scheduled_token_num = len(s.token_ids) - 1
    return s


def test_wire_round_trip_of_the_new_fields():
    from gllm_b200.engine.comm import Comm
    from gllm_b200.input_data import build_batch
    from gllm_b200.scheduler import ScheduledSeq
    seqs = [_seq(1, [3, 4, 5], [], seed=-9, frequency_penalty=0.5, logit_bias={2: 1.0, 9: -3.0}),
            _seq(2, [7, 8], [], top_k=1), _seq(3, [1, 2, 3, 4], [], presence_penalty=-1.5, seed=2 ** 63 - 1)]
    for i, s in enumerate(seqs):
        s.slot, s.slot_fresh = (i + 1 if s.has_bias_row else 0), s.has_bias_row
        s.computed_token_num = s.scheduled_token_num = 0
    b = build_batch([ScheduledSeq(s, 0, len(s)) for s in seqs], 16, 100)
    assert b.need_bias and b.bias_slot.tolist() == [1, -1, 3] and b.seed_pos.tolist() == [3, -1, 4]
    assert b.seed.tolist() == [-9, 0, 2 ** 63 - 1] and b.rb_slots.tolist() == [1, 3]
    assert b.rb_lb_ids.tolist() == [2, 9] and b.rb_lb_off.tolist() == [0, 2, 2] and b.rb_out_off.tolist() == [0, 0, 0]
    got = Comm._decode_batch(memoryview(Comm._encode_batch(b)))
    assert got.need_bias
    for n in ("freq_pen", "pres_pen", "bias_slot", "seed", "seed_pos", "rb_slots", "rb_pen", "rb_lb_off", "rb_lb_ids",
              "rb_lb_vals", "rb_out_off", "rb_out_toks"):
        a, g = getattr(b, n), getattr(got, n)
        assert a.dtype == g.dtype and a.shape == g.shape and np.array_equal(a, g), n
    # a batch without the features sends the header it always sent
    plain = build_batch([ScheduledSeq(_seq(4, [1, 2], []), 0, 2)], 16, 100)
    hdr, _ = plain.to_wire()
    assert len(hdr["scalars"]) == 8 and not any(n in ("seed", "bias_slot") for n, *_ in hdr["arrays"])
    assert not Comm._decode_batch(memoryview(Comm._encode_batch(plain))).need_bias


def test_decode_fast_path_carries_the_rows():
    from gllm_b200.input_data import build_batch
    from gllm_b200.scheduler import ScheduledSeq
    seqs = [_seq(1, [3, 4, 5], [10, 11], seed=5, frequency_penalty=0.5), _seq(2, [7, 8], [12]),
            _seq(3, [1, 2, 3, 4], [13, 14], logit_bias={1: 2.0})]
    for i, s in enumerate(seqs):
        s.slot = i + 1 if s.has_bias_row else 0
    ents = [ScheduledSeq(s, len(s) - 1, 1) for s in seqs]
    prev = build_batch(ents, 16, 100)
    assert prev.seed_pos.tolist() == [5, -1, -1] and prev.bias_slot.tolist() == [1, -1, 3]
    for s, t in zip(seqs, (20, 21, 22)):
        s.append(t)
    order = [2, 0, 1]
    nxt = build_batch([ScheduledSeq(seqs[i], len(seqs[i]) - 1, 1) for i in order], 16, 100, prev=prev)
    assert nxt.seq_ids == [3, 1, 2]            # the incremental path
    assert nxt.seed_pos.tolist() == [-1, 6, -1] and nxt.seed.tolist() == [0, 5, 0]
    assert nxt.bias_slot.tolist() == [3, 1, -1] and nxt.freq_pen.tolist() == [0.0, 0.5, 0.0] and nxt.need_bias
    assert nxt.rb_slots is None
    # the rows using the features finished: the batch is what it would be without them
    s2 = seqs[1]
    s2.append(30)
    last = build_batch([ScheduledSeq(s2, len(s2) - 1, 1)], 16, 100, prev=nxt)
    assert last.seq_ids == [2] and last.seed is None and last.seed_pos is None and not last.need_bias
    assert last.bias_slot is None


# ------------------------------------------------------------------------------------------------
# engine vs a manual HuggingFace loop
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hf_model():
    transformers = pytest.importorskip("transformers")
    torch.manual_seed(3)
    cfg = transformers.Qwen3Config(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4,
                                   num_key_value_heads=2, head_dim=32, vocab_size=512, max_position_embeddings=512,
                                   eos_token_id=1, tie_word_embeddings=False)
    m = transformers.Qwen3ForCausalLM(cfg).eval().float()
    d = scratch_dir("gllm_b200_sp_")
    m.save_pretrained(d, safe_serialization=True)
    return m, d


def _engine(path, **kw):
    from gllm_b200 import LLM
    args = dict(maxp=64, maxd=64, page_size=16, num_cpu_pages=96, model_max_length=320, log_stats=False)
    args.update(kw)
    return LLM(path, **args)


GREEDY = [dict(logit_bias={7: 4.0, 11: -100.0}), dict(frequency_penalty=1.5, presence_penalty=0.5),
          dict(repetition_penalty=1.3, frequency_penalty=0.8), dict(presence_penalty=2.0, logit_bias={3: 1.0}),
          dict(frequency_penalty=-0.5), {}]


def _hf_greedy(m, prompt, n, p):
    """Manual greedy loop applying the formula in fp32 on HuggingFace logits."""
    toks = list(prompt)
    for _ in range(n):
        with torch.no_grad():
            x = m(torch.tensor([toks])).logits[0, -1].float()
        outs = toks[len(prompt):]
        rep = p.get("repetition_penalty", 1.0)
        if rep != 1.0:
            seen = torch.zeros(x.numel(), dtype=torch.bool)
            seen[torch.tensor(sorted(set(toks)))] = True
            x = torch.where(seen, torch.where(x > 0, x / rep, x * rep), x)
        bias = torch.zeros_like(x)
        for t, b in (p.get("logit_bias") or {}).items():
            bias[t] = b
        f, pr = torch.tensor(p.get("frequency_penalty", 0.0)), torch.tensor(p.get("presence_penalty", 0.0))
        seen_out = set()
        for t in outs:
            bias[t] = bias[t] - ((f + pr) if t not in seen_out else f)
            seen_out.add(t)
        toks.append(int((x + bias).argmax()))
    return toks[len(prompt):]


@pytest.mark.parametrize("case", ["default", "prefix_cache_tiny_chunks", "preemption", "sync"])
def test_engine_matches_manual_hf_loop(hf_model, case):
    m, d = hf_model
    kw, prompts, n_out = {}, [[5, 17, 99, 200, 3, 45, 7], [9] * 40, list(range(20, 150)), [300, 301],
                              [7, 7, 7, 3], [40, 41, 42]], 10
    if case == "prefix_cache_tiny_chunks":
        kw = dict(maxp=24, enable_prefix_caching=True)
    elif case == "preemption":
        kw = dict(schedule_method="token_throttling", num_cpu_pages=10, kvthresh=0.0, maxp=32, maxd=8,
                  enable_prefix_caching=False)
        prompts, n_out = [[3 + i, 9, 27, 81, 5] * 4 for i in range(6)], 24
    elif case == "sync":
        kw = dict(async_schedule=False)
    ps = GREEDY[:len(prompts)]
    llm = _engine(d, **kw)
    if case == "prefix_cache_tiny_chunks":
        llm.generate(tokens=prompts, output_lens=[1] * len(prompts), ignore_eos=True)
    outs = llm.generate(tokens=prompts, output_lens=[n_out] * len(prompts), ignore_eos=True, top_k=1,
                        **{k: [p.get(k, 1.0 if k == "repetition_penalty" else None) for p in ps]
                           for k in ("repetition_penalty", "frequency_penalty", "presence_penalty", "logit_bias")})
    if case == "preemption":
        assert llm.worker.scheduler.num_preempt_seqs > 0
    if case == "prefix_cache_tiny_chunks":
        assert any(s.num_cached_tokens > 0 for s in outs)
    llm.shutdown()
    for s, pr, p in zip(outs, prompts, ps):
        assert s.token_ids[len(pr):] == _hf_greedy(m, pr, n_out, p), p
    # the bias visibly acts: token 11 is banned, token 7 favoured
    assert 11 not in outs[0].token_ids[len(prompts[0]):]


# ------------------------------------------------------------------------------------------------
# batch-order invariance of seeded requests
# ------------------------------------------------------------------------------------------------
def test_seeded_requests_in_reverse_order_give_the_same_tokens(monkeypatch):
    from gllm_b200 import LLM
    from gllm_b200.models.presets import tiny
    monkeypatch.setenv("GLLM_KEEP_LOGITS", "1")
    cfg = tiny("Qwen3ForCausalLM", num_hidden_layers=2, vocab_size=300)
    prompts = [[5, 9, 100, 7], [3, 1, 4, 1, 5, 9], [77] * 12, [8, 8]]
    kw = dict(temperature=0.9, top_k=[0, 30, 0, 5], seed=[11, 22, 33, 44], frequency_penalty=0.3,
              output_lens=[1, 1, 1, 1], ignore_eos=True)
    res = []
    for order in ([0, 1, 2, 3], [3, 2, 1, 0]):
        torch.manual_seed(0)
        llm = LLM(cfg, load_format="dummy", device="cpu", num_cpu_pages=64, maxp=64, maxd=16, model_max_length=128,
                  log_stats=False, seed=0)
        outs = llm.generate(tokens=[prompts[i] for i in order],
                            **{k: ([v[i] for i in order] if isinstance(v, list) and k != "output_lens" else v)
                               for k, v in kw.items()})
        lg = {order[j]: llm.worker.runner.logit_log[0][1][j] for j in range(4)}
        res.append(({order[j]: s.token_ids[len(s.token_ids) - 1] for j, s in enumerate(outs)}, lg))
        llm.shutdown()
    (ta, la), (tb, lb) = res
    for i in range(4):
        assert torch.equal(la[i], lb[i])       # one prefill step: the same logits whatever the row
    assert ta == tb


# ------------------------------------------------------------------------------------------------
# TP2 / PP2 over gloo
# ------------------------------------------------------------------------------------------------
def _run(pp, tp, port, async_on=False):
    out = os.path.join(scratch_dir("gllm_b200_sp_"), "sp.json")
    env = dict(os.environ, PYTHONPATH=ROOT, GLLM_B200_LOG="WARNING", GLLM_TEST_ASYNC="1" if async_on else "0")
    script = os.path.join(ROOT, "tests", "mp_sampling_params.py")
    if pp * tp == 1:
        cmd = [sys.executable, script, "1", "1", out]
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={pp * tp}",
               "--master-addr", "127.0.0.1", "--master-port", str(port), script, str(pp), str(tp), out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, env=env, cwd=ROOT)
    assert r.returncode == 0 and os.path.exists(out), r.stdout[-2000:] + r.stderr[-3000:]
    with open(out) as f:
        return json.load(f)


def _tol_cpu(x, s, want, tok):
    return 1e-4 * (1.0 + abs(float(s[want])))     # fp32 evaluation of the same formula


@pytest.fixture(scope="module")
def single_sp():
    return _run(1, 1, 0)


@pytest.mark.parametrize("pp,tp,port,async_on", [(1, 1, 0, False), (1, 2, 29781, False), (2, 1, 29791, False),
                                                 (1, 2, 29801, True)])
def test_multiprocess_engine_follows_the_oracle(single_sp, pp, tp, port, async_on):
    """Every token against the oracle replayed on the kept logits (TP: the gathered logits; the last shard ends with
    padding). Under PP2 the driver holds no logits: its greedy and seeded rows must equal the single-process run."""
    got = single_sp if pp * tp == 1 else _run(pp, tp, port, async_on)
    for i, (prompt, outs, steps) in enumerate(got):
        assert len(outs) == 8
        if pp > 1:
            if i != 2:
                assert outs == single_sp[i][1], i
            continue
        assert len(steps) == 8
        mp.replay(prompt, outs, steps, mp.MIXED[i], _tol_cpu)
    assert 100 not in got[0][1]


# ------------------------------------------------------------------------------------------------
# OpenAI API
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def client():
    pytest.importorskip("fastapi")
    pytest.importorskip("transformers")
    from fastapi.testclient import TestClient
    from gllm_b200.engine.async_llm_engine import AsyncLLM
    from gllm_b200.entrypoints.api_server import build_app
    from test_api_cpu import _make_model_dir
    engine = AsyncLLM(_make_model_dir(), maxp=64, maxd=16, num_cpu_pages=64, model_max_length=128, log_stats=False)
    made = []
    orig = engine.allocate_seq

    def spy(*a, **k):
        s = orig(*a, **k)
        made.append(s)
        return s
    engine.allocate_seq = spy
    with TestClient(build_app(engine)) as c:
        yield c, made
    engine.shutdown()


CHAT = {"messages": [{"role": "user", "content": "hello how are you ?"}], "max_tokens": 4, "ignore_eos": True}
COMPL = {"prompt": "hello world how are you", "max_tokens": 4, "ignore_eos": True}
PARAMS = {"seed": -123456789012, "frequency_penalty": 0.25, "presence_penalty": -1.0,
          "logit_bias": {"5": 3.0, "007": -100, "9": 0.5}}


@pytest.mark.parametrize("url,base", [("/v1/chat/completions", CHAT), ("/v1/completions", COMPL)])
@pytest.mark.parametrize("stream", [False, True])
def test_api_fields_reach_the_sequence(client, url, base, stream):
    c, made = client
    n0 = len(made)
    body = dict(base, stream=stream, **PARAMS)
    if stream:
        with c.stream("POST", url, json=body) as r:
            assert r.status_code == 200
            raw = "".join(r.iter_text())
        assert raw.rstrip().endswith("data: [DONE]")
    else:
        r = c.post(url, json=body)
        assert r.status_code == 200, r.text
    s = made[n0]
    assert s.seed == -123456789012 and s.frequency_penalty == 0.25 and s.presence_penalty == -1.0
    assert s.logit_bias == {5: 3.0, 7: -100.0, 9: 0.5}
    assert 7 not in s.token_ids[s.prompt_len:]


@pytest.mark.parametrize("bad", [{"frequency_penalty": 2.5}, {"presence_penalty": -2.01},
                                 {"frequency_penalty": float("inf")}, {"logit_bias": {"x": 1.0}},
                                 {"logit_bias": {"1.5": 1.0}}, {"logit_bias": {"-1": 1.0}},
                                 {"logit_bias": {"100000": 1.0}}, {"logit_bias": {"3": 101.0}},
                                 {"logit_bias": {"3": float("nan")}},
                                 {"logit_bias": {str(i): 1.0 for i in range(1025)}}, {"seed": 2 ** 63},
                                 {"seed": -2 ** 63 - 1}])
@pytest.mark.parametrize("url,base", [("/v1/chat/completions", CHAT), ("/v1/completions", COMPL)])
def test_api_rejects_out_of_range_parameters(client, url, base, bad):
    c, made = client
    n0 = len(made)
    body = json.dumps(dict(base, **bad), allow_nan=True)
    r = c.post(url, content=body, headers={"content-type": "application/json"})
    assert r.status_code == 400, (bad, r.status_code, r.text)
    assert len(made) == n0


def test_offline_api_validates_and_picks_per_request(hf_model):
    _, d = hf_model
    llm = _engine(d)
    with pytest.raises(ValueError):
        llm.generate(tokens=[[1, 2, 3]], output_lens=[2], logit_bias={600: 1.0})
    with pytest.raises(ValueError):
        llm.generate(tokens=[[1, 2, 3]], output_lens=[2], frequency_penalty=3.0)
    outs = llm.generate(tokens=[[1, 2, 3], [4, 5]], output_lens=[3, 3], ignore_eos=True,
                        logit_bias={9: 100.0}, seed=[1, None], presence_penalty=[0.0, 0.5])
    llm.shutdown()
    assert all(s.logit_bias == {9: 100.0} for s in outs)        # a dict is one value for all requests
    assert [s.seed for s in outs] == [1, None] and [s.presence_penalty for s in outs] == [0.0, 0.5]
    assert outs[0].token_ids[3:] == [9, 9, 9]
