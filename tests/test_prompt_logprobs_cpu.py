"""Prompt log-probabilities on the CPU: the PyTorch model of the one-pass kernel against float64 log_softmax, the
engine against HuggingFace's log_softmax over the prompt (chunking, prefix caching, preemption, sync scheduling,
parallel sampling, mixed batches), TP2 / PP2 over gloo, the OpenAI completions `echo` API, and the wire format of
batches in which no row asks."""
from conftest import scratch_dir
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "batch_wire_no_prompt_logprobs.pkl")


# ------------------------------------------------------------------------------------------------
# oracle of prompt_logprobs_shard_kernel
# ------------------------------------------------------------------------------------------------
def _decode(out: torch.Tensor, n: int):
    ids = out.view(torch.int32)
    return out[:, 0], ids[:, 1:1 + 2 * n:2], out[:, 2:2 + 2 * n:2]


def _adversarial_rows(v: int, pad: int) -> torch.Tensor:
    torch.manual_seed(0)
    x = torch.randn(6, v + pad) * 3
    x[:, v:] = 1e4                              # huge padding columns: never read
    x[1, :v] = 2.0                              # all equal: the lowest id wins
    x[2, :v] = torch.randn(v).clamp(-3, 3)
    x[2, [9, 40, v - 1]] = 7.0                  # a three-way tie at the top
    x[3, ::3] = float("-inf")                   # -inf logits, the target among them
    x[4, :v] = float("-inf")
    x[4, v - 2] = 0.5                           # one finite logit, in the last shard
    return x


@pytest.mark.parametrize("tp", [1, 3])
@pytest.mark.parametrize("n", [0, 1])
def test_ref_prompt_logprobs_match_float64_log_softmax(tp, n):
    from gllm_b200.ops import ref
    v, pad = 101, 60
    x = _adversarial_rows(v, pad)
    targets = torch.tensor([0, 100, 40, 3, v - 2, 55], dtype=torch.int32)
    per = -(-(v + pad) // tp)
    assert tp == 1 or (tp - 1) * per >= v     # with 3 shards the last one is padding only
    recs = [ref.prompt_logprobs_shard(x[:, r * per:(r + 1) * per], max(0, min(per, v - r * per)), n, targets,
                                      vocab_offset=r * per) for r in range(tp)]
    chosen, ids, lps = _decode(ref.logprobs_final(torch.stack(recs), n), n)
    want = torch.log_softmax(x[:, :v].double(), -1)
    for r in range(x.shape[0]):
        w = float(want[r, int(targets[r])])
        assert abs(float(chosen[r]) - w) < 1e-5 or float(chosen[r]) == w == float("-inf"), (r, chosen[r], w)
        if n:
            top = min(range(v), key=lambda i: (-float(x[r, i]), i))
            assert int(ids[r, 0]) == top, (r, int(ids[r, 0]), top)
            assert abs(float(lps[r, 0]) - float(want[r, top])) < 1e-5
    if n:
        assert int(ids[1, 0]) == 0 and int(ids[2, 0]) == 9 and int(ids[4, 0]) == v - 2
    # the records are logprobs_shard's for the same targets
    full = ref.logprobs_shard(x, v, n, targets)
    assert torch.equal(ref.prompt_logprobs_shard(x, v, n, targets), full)


# ------------------------------------------------------------------------------------------------
# engine vs HuggingFace
# ------------------------------------------------------------------------------------------------
# maxp = 24 chunks: 25 tokens end a chunk at P - 1, 48 at P; the others cross several chunks
PROMPTS = [[5, 17, 99, 200, 3, 45, 7], list(range(30, 55)), [9] * 48, list(range(20, 150)), [300, 301, 7]]
ASK = [5, 0, 1, 20, 1]


@pytest.fixture(scope="module")
def hf_model():
    transformers = pytest.importorskip("transformers")
    torch.manual_seed(3)
    cfg = transformers.Qwen3Config(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4,
                                   num_key_value_heads=2, head_dim=32, vocab_size=512, max_position_embeddings=512,
                                   eos_token_id=1, tie_word_embeddings=False)
    m = transformers.Qwen3ForCausalLM(cfg).eval().float()
    d = scratch_dir("gllm_b200_plp_")
    m.save_pretrained(d, safe_serialization=True)
    return m, d


def _engine(path, **kw):
    from gllm_b200 import LLM
    args = dict(maxp=64, maxd=64, page_size=16, num_cpu_pages=96, model_max_length=320, log_stats=False)
    args.update(kw)
    return LLM(path, **args)


def _check_prompt_entries(m, prompt, entries, n):
    assert len(entries) == len(prompt) and entries[0] is None
    with torch.no_grad():
        want = torch.log_softmax(m(torch.tensor([prompt])).logits[0].double(), -1)
    for i in range(1, len(prompt)):
        chosen, top = entries[i]
        w = want[i - 1]
        assert abs(chosen - float(w[prompt[i]])) < 2e-4, (i, chosen, float(w[prompt[i]]))
        assert len(top) == n
        assert [t for t, _ in top] == sorted(range(w.numel()), key=lambda t: (-float(w[t]), t))[:n], i
        for t, v in top:
            assert abs(v - float(w[t])) < 2e-4


@pytest.mark.parametrize("case", ["default", "tiny_chunks", "prefix_cache", "preemption", "sync"])
def test_engine_prompt_logprobs_match_hf_log_softmax(hf_model, case):
    m, d = hf_model
    kw, prompts, ask, n_out = {}, PROMPTS, ASK, 4
    if case == "tiny_chunks":
        kw = dict(maxp=24)
    elif case == "prefix_cache":
        kw = dict(maxp=24, enable_prefix_caching=True)
    elif case == "preemption":
        kw = dict(schedule_method="token_throttling", num_cpu_pages=10, kvthresh=0.0, maxp=32, maxd=8,
                  enable_prefix_caching=False)
        prompts, n_out = [[3 + i, 9, 27, 81, 5] * 4 for i in range(6)], 24
        ask = [1, 5, 0, 20, 1, 3]
    elif case == "sync":
        kw = dict(async_schedule=False)
    llm = _engine(d, **kw)
    plain = llm.generate(tokens=prompts, output_lens=[n_out] * len(prompts), ignore_eos=True)
    if case == "prefix_cache":      # the same prompts are cached now: asking requests take no hits, others do
        again = llm.generate(tokens=prompts, output_lens=[1] * len(prompts), ignore_eos=True)
        assert any(s.num_cached_tokens > 0 for s in again)
    outs = llm.generate(tokens=prompts, output_lens=[n_out] * len(prompts), ignore_eos=True, prompt_logprobs=ask)
    if case == "preemption":
        assert llm.worker.scheduler.num_preempt_seqs > 0
    if case == "prefix_cache":
        assert all(s.num_cached_tokens == 0 for s in outs)
        later = llm.generate(tokens=prompts, output_lens=[1] * len(prompts), ignore_eos=True)
        assert any(s.num_cached_tokens > 0 for s in later)      # their pages were published
    llm.shutdown()
    assert [s.token_ids for s in outs] == [s.token_ids for s in plain]     # asking changes no token
    for s, p, n in zip(outs, prompts, ask):
        assert s.output_logprobs == []
        _check_prompt_entries(m, p, s.prompt_logprobs, n)


def test_parallel_sampling_length_one_and_mixed_requests(hf_model):
    m, d = hf_model
    prompts = [[5, 17, 99, 200, 3, 45, 7, 8, 9], [42], list(range(60, 100)), [11, 12, 13]]
    llm = _engine(d, maxp=24)
    plain = llm.generate(tokens=prompts, output_lens=[5] * 4, ignore_eos=True)
    outs = llm.generate(tokens=prompts, output_lens=[5] * 4, ignore_eos=True, prompt_logprobs=[2, 3, None, 0],
                        logprobs=[None, None, 1, None])
    choices = llm.generate(tokens=[prompts[0]], output_lens=[5], ignore_eos=True, prompt_logprobs=5, n=3,
                           temperature=1.0, top_k=20, seed=7)
    stats = dict(llm.worker.runner.stats)
    llm.shutdown()
    assert [s.token_ids for s in outs] == [s.token_ids for s in plain]
    assert outs[1].prompt_logprobs == [None]           # a prompt of one token: nothing to score
    assert outs[2].prompt_logprobs == [] and len(outs[2].output_logprobs) == 5
    _check_prompt_entries(m, prompts[0], outs[0].prompt_logprobs, 2)
    _check_prompt_entries(m, prompts[3], outs[3].prompt_logprobs, 0)
    assert len(choices) == 3
    _check_prompt_entries(m, prompts[0], choices[0].prompt_logprobs, 5)
    assert all(c.prompt_logprobs == choices[0].prompt_logprobs for c in choices)
    # rows asked: 8 + 0 + 0 + 2 for the mixed batch, then 8 once for the three choices (one prefill)
    assert stats["prompt_logprob_rows"] == 8 + 2 + 8


def test_preempted_choices_do_not_score_the_prompt_again(hf_model):
    """n = 3 under token_throttling with a tiny KV pool: choices are preempted and recompute their prompts, but the
    prompt is scored once, by the parent's prefill, and every choice's list has exactly P entries."""
    m, d = hf_model
    prompts = [[3 + i, 9, 27, 81, 5] * 4 for i in range(2)]
    llm = _engine(d, schedule_method="token_throttling", num_cpu_pages=10, kvthresh=0.0, maxp=32, maxd=8,
                  enable_prefix_caching=False)
    outs = llm.generate(tokens=prompts, output_lens=[24] * 2, ignore_eos=True, prompt_logprobs=1, n=3)
    stats, preempted = dict(llm.worker.runner.stats), llm.worker.scheduler.num_preempt_seqs
    llm.shutdown()
    assert preempted > 0
    assert stats["prompt_logprob_rows"] == sum(len(p) - 1 for p in prompts)
    for j, s in enumerate(outs):
        p = prompts[j // 3]
        assert len(s.prompt_logprobs) == len(p)
        _check_prompt_entries(m, p, s.prompt_logprobs, 1)


def test_generate_rejects_bad_prompt_logprobs(hf_model):
    _, d = hf_model
    llm = _engine(d)
    for bad in (21, -1, 2.5, True):
        with pytest.raises(ValueError):
            llm.generate(tokens=[[5, 6]], output_lens=[2], prompt_logprobs=bad)
    with pytest.raises(ValueError):
        llm.allocate_seq([5, 6], prompt_logprobs=1, mm_contents={"pixel_values": torch.zeros(1)})
    llm.shutdown()


# ------------------------------------------------------------------------------------------------
# TP2 / PP2 over gloo
# ------------------------------------------------------------------------------------------------
def _run(pp, tp, port, async_on=False):
    out = os.path.join(scratch_dir("gllm_b200_plp_"), "plp.json")
    env = dict(os.environ, PYTHONPATH=ROOT, GLLM_B200_LOG="WARNING", GLLM_TEST_ASYNC="1" if async_on else "0")
    script = os.path.join(ROOT, "tests", "mp_prompt_logprobs.py")
    if pp * tp == 1:
        cmd = [sys.executable, script, "1", "1", out]
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={pp * tp}",
               "--master-addr", "127.0.0.1", "--master-port", str(port), script, str(pp), str(tp), out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, env=env, cwd=ROOT)
    assert r.returncode == 0 and os.path.exists(out), r.stdout[-2000:] + r.stderr[-3000:]
    with open(out) as f:
        return json.load(f)


@pytest.mark.parametrize("pp,tp,port,async_on", [(1, 2, 29921, False), (2, 1, 29931, False), (1, 2, 29941, True)])
def test_multiprocess_prompt_logprobs_equal_single_process(pp, tp, port, async_on):
    """Records of vocab shards (the last one ends with padding) all-gathered across TP ranks, and a PP2 output rank
    sending the prompt entries to the driver: the same entries as one process."""
    single, got = _run(1, 1, 0), _run(pp, tp, port, async_on)
    for (ta, la), (tb, lb) in zip(single, got):
        assert ta == tb and len(la) == len(lb) and la[0] is None and lb[0] is None
        for ea, eb in zip(la[1:], lb[1:]):
            assert abs(ea[0] - eb[0]) < 1e-4
            assert [t for t, _ in ea[1]] == [t for t, _ in eb[1]]
            assert all(abs(x - y) < 1e-4 for (_, x), (_, y) in zip(ea[1], eb[1]))


# ------------------------------------------------------------------------------------------------
# wire format: a batch where no row asks is what it was before prompt log-probs
# ------------------------------------------------------------------------------------------------
def _wire_batches():
    from gllm_b200.input_data import build_batch
    from gllm_b200.scheduler import ScheduledSeq
    from gllm_b200.sequence import Sequence
    seqs = [Sequence(i, list(range(3 + i, 40 + 7 * i)), [1], temperature=1.0, top_k=5, logprobs=[-1, 2, 0][i])
            for i in range(3)]
    for k, s in enumerate(seqs):
        s.page_table = [10 * k + j for j in range(8)]
        s.slot = k
    out = []
    entries = [ScheduledSeq(seqs[0], 0, 20), ScheduledSeq(seqs[1], 0, len(seqs[1])),
               ScheduledSeq(seqs[2], 5, len(seqs[2]) - 5)]
    out.append(build_batch(entries, 16, 512, batch_id=3))
    for s in seqs:
        s.append(7)
    dec = [ScheduledSeq(s, len(s) - 1, 1) for s in seqs]
    out.append(build_batch(dec, 16, 512, batch_id=4))
    return [b.to_wire() for b in out]


def _canonical(wire):
    """(header, bytes of every array section): the alignment gaps between sections are left uninitialised."""
    hdr, bufs = wire
    blob = bufs[0]
    return hdr, [bytes(blob[off:off + int(np.prod(shape)) * np.dtype(dt).itemsize])
                 for _, dt, shape, off in hdr["arrays"]]


def test_wire_of_batches_without_prompt_rows_is_unchanged():
    with open(GOLDEN, "rb") as f:
        want = pickle.load(f)
    got = [_canonical(w) for w in _wire_batches()]
    assert got == want


def test_wire_round_trip_carries_prompt_rows():
    from gllm_b200.input_data import BatchArrays, build_batch
    from gllm_b200.scheduler import ScheduledSeq
    from gllm_b200.sequence import Sequence
    s = Sequence(0, list(range(10, 40)), [1], prompt_logprobs=3)
    t = Sequence(1, list(range(50, 60)), [1])
    s.page_table, t.page_table = [0, 1], [2]
    b = build_batch([ScheduledSeq(t, 0, 10), ScheduledSeq(s, 0, 12)], 16, 512)
    assert b.plp_rows.tolist() == list(range(10, 22)) and b.plp_targets.tolist() == list(range(11, 23))
    assert b.plp_n == 3 and s.plp_cursor == 12
    r = BatchArrays.from_wire(*b.to_wire())
    assert np.array_equal(r.plp_rows, b.plp_rows) and np.array_equal(r.plp_targets, b.plp_targets) and r.plp_n == 3
    # the final chunk stops at P - 1; a recompute from 0 (preemption) asks for nothing again
    b2 = build_batch([ScheduledSeq(s, 12, 18)], 16, 512)
    assert b2.plp_rows.tolist() == list(range(0, 17)) and s.plp_cursor == 29 and not s.plp_pending
    assert build_batch([ScheduledSeq(s, 0, 30)], 16, 512).plp_rows is None


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
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_api_cpu import _make_model_dir
    engine = AsyncLLM(_make_model_dir(), maxp=64, maxd=16, num_cpu_pages=64, model_max_length=128, log_stats=False)
    with TestClient(build_app(engine)) as c:
        yield c, engine
    engine.shutdown()


def _sse(c, url, body):
    with c.stream("POST", url, json=dict(body, stream=True)) as r:
        assert r.status_code == 200
        raw = "".join(r.iter_text())
    events = [e for e in raw.split("\n\n") if e]
    assert events[-1] == "data: [DONE]"
    return [json.loads(e[6:]) for e in events[:-1]]


PROMPT = "hello world how are you"
ECHO = {"prompt": PROMPT, "max_tokens": 4, "ignore_eos": True, "top_k": 1, "echo": True}


def _merged(chunks, i=0):
    out = {k: [] for k in ("tokens", "token_logprobs", "top_logprobs", "text_offset")}
    for ch in chunks:
        c = ch["choices"][0]
        if c["index"] == i and c["logprobs"]:
            for k in out:
                out[k] += c["logprobs"][k]
    return out


def test_completion_echo_with_logprobs(client):
    c, engine = client
    plain = c.post("/v1/completions", json=dict(ECHO, echo=False, logprobs=2)).json()["choices"][0]
    body = c.post("/v1/completions", json=dict(ECHO, logprobs=2)).json()
    ch = body["choices"][0]
    p = len(engine.encode(PROMPT))
    assert ch["text"] == PROMPT + plain["text"]
    lp = ch["logprobs"]
    assert len(lp["tokens"]) == p + 4 and body["usage"] == {"prompt_tokens": p, "completion_tokens": 4,
                                                            "total_tokens": p + 4}
    assert lp["token_logprobs"][0] is None and lp["top_logprobs"][0] is None
    assert all(x <= 0 for x in lp["token_logprobs"][1:]) and all(len(t) <= 2 for t in lp["top_logprobs"][1:])
    assert lp["tokens"][p:] == plain["logprobs"]["tokens"] and lp["token_logprobs"][p:] == \
        plain["logprobs"]["token_logprobs"]
    # text_offset runs from 0 across prompt and completion
    offs, acc = [], 0
    for t in lp["tokens"]:
        offs.append(acc)
        acc += len(t)
    assert lp["text_offset"] == offs
    # streamed: the first chunk carries the prompt text and entries, then the generated ones follow
    chunks = _sse(c, "/v1/completions", dict(ECHO, logprobs=2))
    assert chunks[0]["choices"][0]["text"] == PROMPT and len(chunks[0]["choices"][0]["logprobs"]["tokens"]) == p
    assert "".join(x["choices"][0]["text"] for x in chunks) == ch["text"]
    assert _merged(chunks) == lp
    assert chunks[-1]["usage"]["completion_tokens"] == 4


def test_completion_echo_token_ids_without_logprobs_and_max_tokens_zero(client):
    c, engine = client
    ids = engine.encode(PROMPT)
    r = c.post("/v1/completions", json=dict(ECHO, prompt=ids)).json()["choices"][0]
    assert r["text"].startswith(engine.tokenizer.decode(ids)) and r["logprobs"] is None
    for stream in (False, True):
        body = dict(ECHO, prompt=ids, max_tokens=0, logprobs=1)
        if stream:
            chunks = _sse(c, "/v1/completions", body)
            text = "".join(x["choices"][0]["text"] for x in chunks)
            lp, fin, usage = _merged(chunks), chunks[-1]["choices"][0]["finish_reason"], chunks[-1]["usage"]
        else:
            out = c.post("/v1/completions", json=body).json()
            text, lp = out["choices"][0]["text"], out["choices"][0]["logprobs"]
            fin, usage = out["choices"][0]["finish_reason"], out["usage"]
        assert text == engine.tokenizer.decode(ids) and fin == "length"
        assert usage["completion_tokens"] == 0 and usage["prompt_tokens"] == len(ids)
        assert len(lp["tokens"]) == len(ids) and lp["token_logprobs"][0] is None
        assert all(len(t) == 1 for t in lp["top_logprobs"][1:])


def test_completion_echo_with_two_choices(client):
    c, engine = client
    p = len(engine.encode(PROMPT))
    body = c.post("/v1/completions", json=dict(ECHO, logprobs=1, n=2, temperature=1.0, top_k=20, seed=3)).json()
    assert [ch["index"] for ch in body["choices"]] == [0, 1]
    heads = [ch["logprobs"]["token_logprobs"][:p] for ch in body["choices"]]
    assert heads[0] == heads[1] and heads[0][0] is None
    assert all(ch["text"].startswith(PROMPT) for ch in body["choices"])
    chunks = _sse(c, "/v1/completions", dict(ECHO, logprobs=1, n=2, temperature=1.0, top_k=20, seed=3))
    for i in range(2):
        first = [x for x in chunks if x["choices"][0]["index"] == i][0]
        assert first["choices"][0]["text"] == PROMPT and len(first["choices"][0]["logprobs"]["tokens"]) == p


def test_prompt_logprobs_validation_is_400(client):
    c, engine = client
    for body in [dict(ECHO, max_tokens=0, echo=False), dict(ECHO, logprobs=1, prompt_logprobs=21),
                 dict(ECHO, logprobs=1, prompt_logprobs=-1), dict(ECHO, prompt_logprobs=1),
                 dict(ECHO, echo=False, logprobs=1, prompt_logprobs=1)]:
        r = c.post("/v1/completions", json=body)
        assert r.status_code == 400 and r.json()["object"] == "error", (body, r.text)


def test_prompt_logprobs_field_sets_the_prompt_n(client):
    c, engine = client
    lp = c.post("/v1/completions", json=dict(ECHO, logprobs=1, prompt_logprobs=4)).json()["choices"][0]["logprobs"]
    p = len(engine.encode(PROMPT))
    assert all(len(t) == 4 for t in lp["top_logprobs"][1:p]) and all(len(t) == 1 for t in lp["top_logprobs"][p:])


def test_chat_is_unchanged(client):
    c, engine = client
    msg = {"messages": [{"role": "user", "content": "hello"}], "max_tokens": 3, "ignore_eos": True, "top_k": 1,
           "logprobs": True, "top_logprobs": 2, "echo": True}
    a = c.post("/v1/chat/completions", json=msg).json()
    b = c.post("/v1/chat/completions", json={k: v for k, v in msg.items() if k != "echo"}).json()
    for r in (a, b):
        del r["id"], r["created"]
    assert a == b and set(a["choices"][0]) == {"index", "message", "logprobs", "finish_reason"}
