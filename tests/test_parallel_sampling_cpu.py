"""Parallel sampling (`n` choices per request) on the CPU: the `kv_copy_pages` oracle, greedy parity with a manual
HuggingFace loop across prefix caching, lookahead, page-boundary prompt lengths, preemption, TP2 and PP2 over gloo,
one prefill per request, page reference counts under random request streams, and the OpenAI API."""
from conftest import scratch_dir
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------
# kv_copy_pages oracle
# ------------------------------------------------------------------------------------------------
def test_ref_kv_copy_pages_equals_an_indexing_copy():
    from gllm_b200.ops import ref
    g = torch.Generator().manual_seed(0)
    tensors = [torch.randn(12, 2, 2, 4, 64, generator=g).to(torch.bfloat16) for _ in range(5)]
    want = [t.clone() for t in tensors]
    pairs = [(3, 7), (0, 1), (3, 10)]
    for w in want:
        for s, d in pairs:
            w[d] = w[s]
    ref.kv_copy_pages(tensors, pairs, dummy_page=11)
    for t, w in zip(tensors, want):
        assert torch.equal(t, w)


@pytest.mark.parametrize("pairs", [[(1, 2), (3, 2)], [(1, 2), (2, 4)], [(1, 11)], [(11, 3)], [(1, 12)], [(-1, 3)]])
def test_copy_pairs_are_checked_on_the_host(pairs):
    from gllm_b200.ops import ref
    t = torch.zeros(12, 1, 1, 4, 64)
    with pytest.raises(ValueError):
        ref.kv_copy_pages([t], pairs, dummy_page=11)


# ------------------------------------------------------------------------------------------------
# engine vs a manual HuggingFace greedy loop
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hf_model():
    transformers = pytest.importorskip("transformers")
    torch.manual_seed(5)
    cfg = transformers.Qwen3Config(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4,
                                   num_key_value_heads=2, head_dim=32, vocab_size=512, max_position_embeddings=512,
                                   eos_token_id=1, tie_word_embeddings=False)
    m = transformers.Qwen3ForCausalLM(cfg).eval().float()
    d = scratch_dir("gllm_b200_ps_")
    m.save_pretrained(d, safe_serialization=True)
    return m, d


def _hf_greedy(m, prompt, n):
    toks = list(prompt)
    for _ in range(n):
        with torch.no_grad():
            toks.append(int(m(torch.tensor([toks])).logits[0, -1].float().argmax()))
    return toks[len(prompt):]


def _engine(path, **kw):
    from gllm_b200 import LLM
    args = dict(maxp=64, maxd=64, page_size=4, num_cpu_pages=128, model_max_length=320, log_stats=False)
    args.update(kw)
    return LLM(path, **args)


# P mod 4 = 0, 1, 3 (page size 4) and a prompt longer than one chunk
PROMPTS = [[5, 17, 99, 200, 3, 45, 7, 8], [9] * 13, list(range(20, 31)), list(range(40, 110))]


@pytest.mark.parametrize("prefix,async_on", [(False, True), (False, False), (True, True), (True, False)])
def test_greedy_choices_equal_the_hf_continuation(hf_model, prefix, async_on):
    m, d = hf_model
    n_out = 7
    llm = _engine(d, enable_prefix_caching=prefix, async_schedule=async_on, maxp=32)
    one = llm.generate(tokens=PROMPTS, output_lens=[n_out] * 4, ignore_eos=True, top_k=1)
    many = llm.generate(tokens=PROMPTS, output_lens=[n_out] * 4, ignore_eos=True, top_k=1, n=3)
    mm = llm.worker.mm
    copied = llm.worker.runner.stats.get("kv_copy_pages", 0)
    free, usable, used_ids = mm.get_num_free_pages(), mm.usable_pages, llm.id_allocator.get_num_used_ids()
    llm.shutdown()
    assert len(many) == 12
    for j, pr in enumerate(PROMPTS):
        want = _hf_greedy(m, pr, n_out)
        assert one[j].token_ids[len(pr):] == want, j
        for i in range(3):
            s = many[3 * j + i]
            assert s.token_ids[:len(pr)] == pr and s.token_ids[len(pr):] == want, (j, i)
    # the three prompts that end inside a page copied it for each of their two extra choices
    assert copied == 2 * sum(1 for p in PROMPTS if len(p) % 4)
    if not prefix:
        assert free == usable
    assert used_ids == 0


def test_prefill_once(hf_model):
    _, d = hf_model
    llm = _engine(d, enable_prefix_caching=False)
    p = list(range(30, 67))
    t0 = llm.worker.runner.stats["tokens"]
    outs = llm.generate(tokens=[p], output_lens=[1], ignore_eos=True, top_k=1, n=4)
    computed = llm.worker.runner.stats["tokens"] - t0
    llm.shutdown()
    assert len(outs) == 4 and computed == len(p)       # not 4 * len(p)


@pytest.mark.parametrize("case", ["siblings", "parent"])
def test_preemption_follows_the_oracle(hf_model, case):
    """A pool small enough that decoding choices get preempted and are recomputed from scratch. `parent`: one
    request, so the choice that gets preempted first is the parent itself, after its fan-out."""
    m, d = hf_model
    kw = dict(schedule_method="token_throttling", num_cpu_pages=14, kvthresh=0.0, maxp=32, maxd=8,
              enable_prefix_caching=False)
    if case == "siblings":
        prompts, n, n_out = [[3 + i, 9, 27, 81, 5] * 2 + [i] for i in range(3)], 3, 14
    else:
        prompts, n, n_out = [[3, 9, 27, 81, 5, 7] * 3], 4, 20
    llm = _engine(d, **kw)
    outs = llm.generate(tokens=prompts, output_lens=[n_out] * len(prompts), ignore_eos=True, top_k=1, n=n)
    preempted = llm.worker.scheduler.num_preempt_seqs
    free, usable = llm.worker.mm.get_num_free_pages(), llm.worker.mm.usable_pages
    llm.shutdown()
    assert preempted > 0 and free == usable
    for j, pr in enumerate(prompts):
        want = _hf_greedy(m, pr, n_out)
        for i in range(n):
            assert outs[n * j + i].token_ids[len(pr):] == want, (j, i)


def test_seeded_choices_draw_as_single_requests_with_seed_plus_i(hf_model):
    """Choice i of a request seeded with s draws its first token exactly as an n = 1 request seeded with s + i."""
    _, d = hf_model
    p = [5, 17, 99, 200, 3]
    llm = _engine(d)
    many = llm.generate(tokens=[p], output_lens=[1], ignore_eos=True, temperature=1.5, top_k=0, top_p=1.0, n=6,
                        seed=2 ** 63 - 3)
    single = llm.generate(tokens=[p] * 6, output_lens=[1] * 6, ignore_eos=True, temperature=1.5, top_k=0, top_p=1.0,
                          seed=[2 ** 63 - 3, 2 ** 63 - 2, 2 ** 63 - 1, -2 ** 63, -2 ** 63 + 1, -2 ** 63 + 2])
    llm.shutdown()
    assert [s.seed for s in many] == [s.seed for s in single]
    assert [s.token_ids[-1] for s in many] == [s.token_ids[-1] for s in single]
    assert len({s.token_ids[-1] for s in many}) > 1


def test_offline_api_validates_n(hf_model):
    _, d = hf_model
    llm = _engine(d, maxp=16)
    for bad in (0, 129, 17, -1, 2.5, True, "3"):
        with pytest.raises(ValueError):
            llm.generate(tokens=[[1, 2, 3]], output_lens=[2], n=bad)
    with pytest.raises(ValueError):
        llm.allocate_choices([1, 2, 3], 2, mm_contents={"pixel_values": None})
    outs = llm.generate(tokens=[[1, 2, 3], [4, 5]], output_lens=[2, 3], ignore_eos=True, n=[2, None])
    used = llm.id_allocator.get_num_used_ids()
    llm.shutdown()
    assert [len(s.token_ids) for s in outs] == [5, 5, 5] and used == 0


# ------------------------------------------------------------------------------------------------
# TP2 / PP2 over gloo
# ------------------------------------------------------------------------------------------------
def _run(pp, tp, port, async_on):
    out = os.path.join(scratch_dir("gllm_b200_ps_"), "ps.json")
    env = dict(os.environ, PYTHONPATH=ROOT, GLLM_B200_LOG="WARNING", GLLM_TEST_ASYNC="1" if async_on else "0")
    script = os.path.join(ROOT, "tests", "mp_parallel_sampling.py")
    if pp * tp == 1:
        cmd = [sys.executable, script, "1", "1", out]
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={pp * tp}",
               "--master-addr", "127.0.0.1", "--master-port", str(port), script, str(pp), str(tp), out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, env=env, cwd=ROOT)
    assert r.returncode == 0 and os.path.exists(out), r.stdout[-2000:] + r.stderr[-3000:]
    with open(out) as f:
        return json.load(f)


@pytest.mark.parametrize("pp,tp,port,async_on", [(1, 2, 29831, False), (2, 1, 29841, False), (1, 2, 29851, True)])
def test_multiprocess_greedy_choices_equal_n1(pp, tp, port, async_on):
    got = _run(pp, tp, port, async_on)
    assert got["single"] and len(got["many"]) == 3 * len(got["single"])
    for j, want in enumerate(got["single"]):
        for i in range(3):
            assert got["many"][3 * j + i] == want, (j, i)
    assert got["copied"] > 0


# ------------------------------------------------------------------------------------------------
# page reference counts under random request streams
# ------------------------------------------------------------------------------------------------
def _check_pages(mm, live):
    holders = {}
    for s in live:
        assert len(set(s.page_table)) == len(s.page_table)
        for p in s.page_table:
            holders[p] = holders.get(p, 0) + 1
    if mm.dummy_page is not None:
        holders[mm.dummy_page] = holders.get(mm.dummy_page, 0) + 1
    for p in range(mm.num_pages):
        assert mm.page_ref[p] == holders.get(p, 0), (p, mm.page_ref[p], holders.get(p, 0))
        assert mm.id_allocator.is_free(p) == (mm.page_ref[p] == 0), p


hypothesis = pytest.importorskip("hypothesis")
from hypothesis import HealthCheck, given, settings, strategies as st  # noqa: E402


@settings(max_examples=40, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.too_slow])
@given(seed=st.integers(0, 10 ** 6), n_req=st.integers(1, 10), pages=st.integers(12, 40), prefix=st.booleans(),
       method=st.sampled_from(["chunked_prefill", "token_throttling"]), maxp=st.sampled_from([8, 16, 64]),
       abort_rate=st.sampled_from([0.0, 0.15]), pp=st.sampled_from([1, 2]), page=st.sampled_from([2, 4]))
def test_random_streams_keep_page_refcounts(seed, n_req, pages, prefix, method, maxp, abort_rate, pp, page):
    from gllm_b200.memory_manager import MemoryManager, PrefixMemoryManager
    from gllm_b200.scheduler import Scheduler
    from gllm_b200.sequence import Sequence
    rng = random.Random(seed)
    mm = (PrefixMemoryManager if prefix else MemoryManager)(pages, page, reserve_dummy_page=True)
    cap = 6 if method == "token_throttling" else maxp
    sch = Scheduler(mm, pp_size=pp, world_size=pp, schedule_method=method, maxd=6, maxp=maxp, minp=4, iterp=2,
                    kvthresh=0.0, page_size=page, log=False, max_seqs=cap)
    stems = [[rng.randrange(50) for _ in range(rng.randrange(2, 12))] for _ in range(3)]
    heads, everyone, sid = [], [], 0
    for _ in range(n_req):
        stem = rng.choice(stems)
        toks = stem[:rng.randrange(1, len(stem) + 1)] + [rng.randrange(50) for _ in range(rng.randrange(0, 5))]
        k = rng.randrange(1, min(4, cap) + 1)
        out = rng.randrange(1, 7)
        if k * ((len(toks) + out + page - 1) // page) > pages - 1:
            continue
        choices = [Sequence(sid + i, toks, [2], output_len=out, ignore_eos=True) for i in range(k)]
        sid += k
        choices[0].forks = choices[1:]
        heads.append(choices[0])
        everyone += choices
    pending = list(heads)
    freed, produced, inflight = [], {}, []
    for _ in range(2000):
        if pending and rng.random() < 0.5:
            k = rng.randrange(1, len(pending) + 1)
            sch.add_new_requests(pending[:k])
            del pending[:k]
        if abort_rate and rng.random() < abort_rate and everyone:
            sch.add_abort_ids([rng.choice(everyone).seq_id])
            o = sch.check_abort_seqs()
            if o is not None:
                freed += o.free_ids
        batch = sch.schedule_once()
        _check_pages(mm, everyone)
        if batch:
            rows = sum(1 for e in batch if e.emits) + sum(len(e.forks or ()) for e in batch)
            assert rows <= cap
            for e in batch:
                for s in e.forks or ():
                    assert s.page_table[:len(e.seq.token_ids) // page] == \
                        e.seq.page_table[:len(e.seq.token_ids) // page]
            inflight.append(batch)
        if inflight and (len(inflight) == pp or not batch):
            done = inflight.pop(0)
            rows = sum(1 for e in done if e.emits) + sum(len(e.forks or ()) for e in done)
            sch.add_next_tokens([rng.randrange(3, 50) for _ in range(rows)])
            o = sch.process_output()
            freed += o.free_ids
            for s, t in zip(o.act_schedule_ids, o.next_tokens):
                produced.setdefault(s, []).append(t)
            _check_pages(mm, everyone)
        if not pending and not sch.has_work():
            break
    assert not sch.has_work() and not pending, "engine did not drain"
    assert sorted(freed) == sorted(s.seq_id for s in everyone)          # every id reported exactly once
    for s in everyone:
        assert not s.page_table
        if not s.is_abort:
            assert len(produced.get(s.seq_id, [])) == s.output_len
    assert mm.get_num_free_pages() == mm.usable_pages
    _check_pages(mm, [])


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
    with TestClient(build_app(engine)) as c:
        yield c, engine
    engine.shutdown()


CHAT = {"messages": [{"role": "user", "content": "hello how are you ?"}], "max_tokens": 4, "ignore_eos": True,
        "temperature": 1.0, "top_k": 0, "seed": 3}
COMPL = {"prompt": "hello world how are you", "max_tokens": 4, "ignore_eos": True, "temperature": 1.0, "top_k": 0,
         "seed": 3}


def _events(raw):
    out = []
    for block in raw.split("\n\n"):
        if block.startswith("data: ") and block != "data: [DONE]":
            out.append(json.loads(block[6:]))
    return out


@pytest.mark.parametrize("url,base,chat", [("/v1/chat/completions", CHAT, True), ("/v1/completions", COMPL, False)])
def test_api_n3_non_stream(client, url, base, chat):
    c, _ = client
    lp = {"logprobs": True, "top_logprobs": 2} if chat else {"logprobs": 2}
    body = dict(base, n=3, max_tokens=5, **lp)
    r = c.post(url, json=body)
    assert r.status_code == 200, r.text
    js = r.json()
    assert [ch["index"] for ch in js["choices"]] == [0, 1, 2]
    assert all(ch["finish_reason"] == "length" for ch in js["choices"])
    u = js["usage"]
    assert u["completion_tokens"] == 15 and u["total_tokens"] == u["prompt_tokens"] + 15
    assert u["prompt_tokens"] == (5 if not chat else u["prompt_tokens"]) and u["prompt_tokens"] < 15
    for ch in js["choices"]:
        n_lp = len(ch["logprobs"]["content"]) if chat else len(ch["logprobs"]["tokens"])
        assert n_lp == 5
    # choice 0 is the n = 1 request with the same seed
    one = c.post(url, json=dict(base, max_tokens=5, **lp)).json()
    key = (lambda ch: ch["message"]["content"]) if chat else (lambda ch: ch["text"])
    assert key(one["choices"][0]) == key(js["choices"][0])
    if chat:     # (the values may differ in the last bits: the second request hits the prefix cache)
        toks = [[e["token"] for e in o["choices"][0]["logprobs"]["content"]] for o in (one, js)]
    else:
        toks = [o["choices"][0]["logprobs"]["tokens"] for o in (one, js)]
    assert toks[0] == toks[1]


@pytest.mark.parametrize("url,base,chat", [("/v1/chat/completions", CHAT, True), ("/v1/completions", COMPL, False)])
def test_api_n3_stream(client, url, base, chat):
    c, _ = client
    lp = {"logprobs": True, "top_logprobs": 1} if chat else {"logprobs": 1}
    body = dict(base, n=3, stream=True, stop=None, **lp)
    body["max_tokens"] = 3
    with c.stream("POST", url, json=body) as r:
        assert r.status_code == 200
        raw = "".join(r.iter_text())
    assert raw.rstrip().endswith("data: [DONE]")
    ev = _events(raw)
    assert all(len(e["choices"]) == 1 for e in ev)
    finishes = [e for e in ev if e["choices"][0].get("finish_reason")]
    assert sorted(e["choices"][0]["index"] for e in finishes) == [0, 1, 2]
    assert all(e["choices"][0]["finish_reason"] == "length" for e in finishes)
    assert finishes[-1] is ev[-1] and ev[-1]["usage"]["completion_tokens"] == 9
    assert all(e.get("usage") is None for e in ev[:-1])
    assert len({e["id"] for e in ev}) == 1
    for i in range(3):
        mine = [e for e in ev if e["choices"][0]["index"] == i and not e["choices"][0].get("finish_reason")]
        if chat:
            assert mine[0]["choices"][0]["delta"]["role"] == "assistant"
            assert sum(len(e["choices"][0]["logprobs"]["content"]) for e in mine) == 3
        else:
            assert sum(len(e["choices"][0]["logprobs"]["tokens"]) for e in mine) == 3


@pytest.mark.parametrize("bad", [0, 129, -3, 65])
@pytest.mark.parametrize("url,base", [("/v1/chat/completions", CHAT), ("/v1/completions", COMPL)])
def test_api_rejects_bad_n(client, url, base, bad):
    c, engine = client
    used = engine.id_allocator.get_num_used_ids()
    r = c.post(url, json=dict(base, n=bad))
    assert r.status_code == 400, r.text
    assert engine.id_allocator.get_num_used_ids() == used


def test_api_rejects_n_with_an_image():
    pytest.importorskip("fastapi")
    from fastapi.testclient import TestClient
    from gllm_b200.entrypoints import api_server

    class _Loader:
        use_mm = True
        config = {"vocab_size": 100}

    class _Cfg:
        max_running_seqs = 64

    class _Engine:
        loader, cfg, failed, tokenizer = _Loader(), _Cfg(), None, None

        def check_seq_length(self, *_):
            return True

    calls = []

    async def _add(*a, **k):
        calls.append(k)
        raise AssertionError("must not be reached")
    eng = _Engine()
    eng.add_requests_async = _add
    import gllm_b200.models.multimodal as mmod
    saved, saved_llm = mmod.encode_mm, api_server.llm
    mmod.encode_mm = lambda llm, messages: ([1, 2, 3], {"pixel_values": torch.zeros(1)})
    try:
        with TestClient(api_server.build_app(eng)) as c:
            body = {"messages": [{"role": "user", "content": [{"type": "image_url", "image_url": {"url": "x"}}]}],
                    "n": 2}
            r = c.post("/v1/chat/completions", json=body)
    finally:
        mmod.encode_mm = saved
        api_server.llm = saved_llm      # build_app binds the module's engine: give the other tests theirs back
    assert r.status_code == 400 and "multimodal" in r.text and not calls


def test_api_disconnect_frees_every_choice(client):
    c, engine = client
    used = engine.id_allocator.get_num_used_ids()
    body = dict(CHAT, n=4, stream=True, max_tokens=60)
    with c.stream("POST", "/v1/chat/completions", json=body) as r:
        assert r.status_code == 200, r.read()
        for _ in r.iter_lines():
            break       # leave after the first event: the client disconnects
    import time
    t0 = time.time()
    while engine.id_allocator.get_num_used_ids() != used and time.time() - t0 < 30:
        time.sleep(0.05)
    assert engine.id_allocator.get_num_used_ids() == used
    assert engine.worker.mm.get_num_free_pages() == engine.worker.mm.usable_pages


@pytest.mark.parametrize("url,base", [("/v1/chat/completions", CHAT), ("/v1/completions", COMPL)])
@pytest.mark.parametrize("stream", [False, True])
def test_api_n1_keeps_the_single_choice_shape(client, url, base, stream):
    c, _ = client
    shapes = []
    for extra in ({}, {"n": 1}):
        body = dict(base, stream=stream, **extra)
        if stream:
            with c.stream("POST", url, json=body) as r:
                raw = "".join(r.iter_text())
            shapes.append([_shape(e) for e in _events(raw)])
        else:
            shapes.append(_shape(c.post(url, json=body).json()))
    assert shapes[0] == shapes[1]


def _shape(js):
    """Keys and value types, recursively (ids, timestamps and texts may differ)."""
    if isinstance(js, dict):
        return {k: _shape(v) for k, v in js.items()}
    if isinstance(js, list):
        return [_shape(v) for v in js]
    return type(js).__name__


def test_metrics_count_requests_not_choices(client):
    c, engine = client
    m0 = dict(engine.metrics)
    r = c.post("/v1/completions", json=dict(COMPL, n=5, max_tokens=2))
    assert r.status_code == 200
    m1 = engine.metrics
    assert m1["requests_total"] - m0["requests_total"] == 1
    assert m1["requests_finished"] - m0["requests_finished"] == 1
    assert m1["prompt_tokens_total"] - m0["prompt_tokens_total"] == 5
    assert m1["generation_tokens_total"] - m0["generation_tokens_total"] == 10
