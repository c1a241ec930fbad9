"""Token log-probabilities on the CPU: the PyTorch oracle of the log-prob kernels, the engine against HuggingFace's
log_softmax, TP2 / PP2 over gloo, and the OpenAI API shapes (chat `logprobs` / `top_logprobs`, completions
`logprobs`)."""
from conftest import scratch_dir
import asyncio
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------
# oracle
# ------------------------------------------------------------------------------------------------
def _decode(out: torch.Tensor, n: int):
    ids = out.view(torch.int32)
    return out[:, 0], ids[:, 1:1 + 2 * n:2], out[:, 2:2 + 2 * n:2]


@pytest.mark.parametrize("tp", [1, 3])
def test_ref_logprobs_match_float64_log_softmax(tp):
    from gllm_b200.ops import ref
    torch.manual_seed(0)
    v, pad, n = 101, 27, 6
    x = torch.randn(5, v + pad) * 3
    x[:, v:] = 1e3                           # padding columns: ignored
    x[1, :] = 2.0                            # all equal: ids 0..n-1
    x[2, :v] = torch.randn(v).clamp(-3, 3)
    x[2, [7, 40, 90]] = 5.0
    x[2, [3, 50, 60, 99]] = 4.0              # a tie cut at the n-th place: lower ids win
    x[3, ::4] = float("-inf")
    toks = torch.tensor([0, 100, 60, 1, 55], dtype=torch.int32)
    rows = torch.tensor([0, 1, 2, 3], dtype=torch.int32)     # row 4 does not ask
    per = -(-(v + pad) // tp)
    recs = [ref.logprobs_shard(x[:, r * per:(r + 1) * per], max(0, min(per, v - r * per)), n, toks, rows,
                               vocab_offset=r * per) for r in range(tp)]
    chosen, ids, lps = _decode(ref.logprobs_final(torch.stack(recs), n), n)
    want = torch.log_softmax(x[:, :v].double(), -1)
    for j, r in enumerate(rows.tolist()):
        order = sorted(range(v), key=lambda i: (-float(x[r, i]), i))[:n]
        assert ids[j].tolist() == order, (r, ids[j].tolist(), order)
        assert torch.allclose(lps[j].double(), want[r, order], atol=1e-5)
        assert abs(float(chosen[j]) - float(want[r, int(toks[r])])) < 1e-5 or \
            (float(chosen[j]) == float(want[r, int(toks[r])]) == float("-inf"))
    assert ids[2].tolist()[:5] == [7, 40, 90, 3, 50]
    # fewer real tokens than n: empty slots carry id -1
    small = ref.logprobs_final(ref.logprobs_shard(x[:, :4], 4, n, torch.zeros(5, dtype=torch.int32))[None], n)
    assert (_decode(small, n)[1][:, 4:] == -1).all() and torch.isinf(_decode(small, n)[2][:, 4:]).all()


# ------------------------------------------------------------------------------------------------
# engine vs HuggingFace
# ------------------------------------------------------------------------------------------------
PROMPTS = [[5, 17, 99, 200, 3, 45, 7], [9] * 40, list(range(20, 150)), [300, 301]]
ASK = [5, None, 20, 0]


@pytest.fixture(scope="module")
def hf_model():
    transformers = pytest.importorskip("transformers")
    torch.manual_seed(3)
    cfg = transformers.Qwen3Config(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4,
                                   num_key_value_heads=2, head_dim=32, vocab_size=512, max_position_embeddings=512,
                                   eos_token_id=1, tie_word_embeddings=False)
    m = transformers.Qwen3ForCausalLM(cfg).eval().float()
    d = scratch_dir("gllm_b200_lp_")
    m.save_pretrained(d, safe_serialization=True)
    return m, d


def _engine(path, **kw):
    from gllm_b200 import LLM
    args = dict(maxp=64, maxd=64, page_size=16, num_cpu_pages=96, model_max_length=320, log_stats=False)
    args.update(kw)
    return LLM(path, **args)


@pytest.mark.parametrize("case", ["default", "prefix_cache_tiny_chunks", "preemption", "sync"])
def test_engine_logprobs_match_hf_log_softmax(hf_model, case):
    m, d = hf_model
    kw, prompts, n_out = {}, PROMPTS, 10
    if case == "prefix_cache_tiny_chunks":
        kw = dict(maxp=24, enable_prefix_caching=True)
    elif case == "preemption":
        kw = dict(schedule_method="token_throttling", num_cpu_pages=10, kvthresh=0.0, maxp=32, maxd=8,
                  enable_prefix_caching=False)
        prompts, n_out = [[3 + i, 9, 27, 81, 5] * 4 for i in range(6)], 24
    elif case == "sync":
        kw = dict(async_schedule=False)
    ask = (ASK * 2)[:len(prompts)]
    llm = _engine(d, **kw)
    plain = llm.generate(tokens=prompts, output_lens=[n_out] * len(prompts), ignore_eos=True)
    plain = [s.token_ids[len(p):] for s, p in zip(plain, prompts)]
    if case == "prefix_cache_tiny_chunks":     # the same prompts again: served from the prefix cache
        assert llm.generate(tokens=prompts, output_lens=[1] * len(prompts), ignore_eos=True)
    outs = llm.generate(tokens=prompts, output_lens=[n_out] * len(prompts), ignore_eos=True, logprobs=ask)
    if case == "preemption":
        assert llm.worker.scheduler.num_preempt_seqs > 0
    if case == "prefix_cache_tiny_chunks":
        assert any(s.num_cached_tokens > 0 for s in outs)
    llm.shutdown()
    assert [s.token_ids[len(p):] for s, p in zip(outs, prompts)] == plain   # asking changes no token
    for s, p, n in zip(outs, prompts, ask):
        if n is None:
            assert s.output_logprobs == []
            continue
        assert len(s.output_logprobs) == s.num_output_tokens == n_out
        with torch.no_grad():
            lg = m(torch.tensor([s.token_ids[:-1]])).logits[0, len(p) - 1:].double()
        want = torch.log_softmax(lg, -1)
        for j, (chosen, top) in enumerate(s.output_logprobs):
            tok = s.token_ids[len(p) + j]
            assert abs(chosen - float(want[j, tok])) < 2e-4, (j, chosen, float(want[j, tok]))
            assert len(top) == n
            if n:
                assert top[0] == (tok, chosen)                                 # greedy: the sampled token first
            for t, v in top:
                assert abs(v - float(want[j, t])) < 2e-4
            if n:   # the n most likely (HF's n-th value within fp32 noise of the last reported)
                assert float(torch.topk(want[j], n).values[-1]) <= top[-1][1] + 2e-4


# ------------------------------------------------------------------------------------------------
# TP2 / PP2 over gloo
# ------------------------------------------------------------------------------------------------
def _run(pp, tp, port, async_on=False):
    out = os.path.join(scratch_dir("gllm_b200_lp_"), "lp.json")
    env = dict(os.environ, PYTHONPATH=ROOT, GLLM_B200_LOG="WARNING", GLLM_TEST_ASYNC="1" if async_on else "0")
    script = os.path.join(ROOT, "tests", "mp_logprobs.py")
    if pp * tp == 1:
        cmd = [sys.executable, script, "1", "1", out]
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={pp * tp}",
               "--master-addr", "127.0.0.1", "--master-port", str(port), script, str(pp), str(tp), out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, env=env, cwd=ROOT)
    assert r.returncode == 0 and os.path.exists(out), r.stdout[-2000:] + r.stderr[-3000:]
    with open(out) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def single_lp():
    return _run(1, 1, 0)


@pytest.mark.parametrize("pp,tp,port,async_on", [(1, 2, 29881, False), (2, 1, 29891, False), (1, 2, 29901, True)])
def test_multiprocess_logprobs_equal_single_process(single_lp, pp, tp, port, async_on):
    """Vocab-parallel records gathered across TP ranks (the last shard ends with padding), and the output rank of a
    PP2 pipeline sending tokens + log-probs to the driver: the greedy rows equal the single-process log-probs. The
    sampled row (its random draws differ per layout) must come back complete."""
    got = _run(pp, tp, port, async_on)
    for i, ((ta, la), (tb, lb)) in enumerate(zip(single_lp, got)):
        n = [5, 3, None, 20][i]
        assert len(lb) == (0 if n is None else 8) and all(len(e[1]) == n for e in lb)
        if i == 1:
            continue
        assert ta == tb
        for ea, eb in zip(la, lb):
            assert abs(ea[0] - eb[0]) < 1e-4
            assert [t for t, _ in ea[1]] == [t for t, _ in eb[1]]
            assert all(abs(x - y) < 1e-4 for (_, x), (_, y) in zip(ea[1], eb[1]))


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


CHAT = {"messages": [{"role": "user", "content": "hello how are you ?"}], "max_tokens": 6, "ignore_eos": True,
        "top_k": 1, "logprobs": True, "top_logprobs": 5}
COMPL = {"prompt": "hello world how are you", "max_tokens": 6, "ignore_eos": True, "top_k": 1, "logprobs": 5}


def test_chat_logprobs_shape_and_streaming(client):
    c, engine = client
    body = c.post("/v1/chat/completions", json=CHAT).json()
    content = body["choices"][0]["logprobs"]["content"]
    assert len(content) == body["usage"]["completion_tokens"] == 6
    for e in content:
        assert set(e) == {"token", "logprob", "bytes", "top_logprobs"} and len(e["top_logprobs"]) == 5
        assert e["bytes"] == list(e["token"].encode()) and e["logprob"] <= 0
        assert e["top_logprobs"][0]["token"] == e["token"] and e["top_logprobs"][0]["logprob"] == e["logprob"]
        assert set(e["top_logprobs"][0]) == {"token", "logprob", "bytes"}
    chunks = _sse(c, "/v1/chat/completions", CHAT)
    streamed = [e for ch in chunks for e in ((ch["choices"][0].get("logprobs") or {}).get("content") or [])]
    assert streamed == content
    assert "".join(ch["choices"][0]["delta"].get("content") or "" for ch in chunks) == \
        body["choices"][0]["message"]["content"]
    # logprobs without alternatives
    e0 = c.post("/v1/chat/completions", json=dict(CHAT, top_logprobs=0)).json()["choices"][0]["logprobs"]["content"]
    assert len(e0) == 6 and all(e["top_logprobs"] == [] for e in e0)


def test_completion_logprobs_shape_and_streaming(client):
    c, engine = client
    body = c.post("/v1/completions", json=COMPL).json()
    lp = body["choices"][0]["logprobs"]
    assert set(lp) == {"tokens", "token_logprobs", "top_logprobs", "text_offset"}
    assert len(lp["tokens"]) == len(lp["token_logprobs"]) == len(lp["top_logprobs"]) == len(lp["text_offset"]) == \
        body["usage"]["completion_tokens"] == 6
    assert all(len(t) <= 5 and lp["tokens"][i] in t for i, t in enumerate(lp["top_logprobs"]))
    assert lp["text_offset"][0] == 0 and lp["text_offset"] == sorted(lp["text_offset"])
    chunks = _sse(c, "/v1/completions", COMPL)
    merged = {k: [] for k in lp}
    for ch in chunks:
        part = ch["choices"][0]["logprobs"]
        if part:
            for k in merged:
                merged[k] += part[k]
    assert merged == lp
    assert chunks[-1]["usage"]["completion_tokens"] == 6


def test_stop_string_cuts_logprob_entries(client):
    c, engine = client
    full = c.post("/v1/completions", json=dict(COMPL, max_tokens=12)).json()["choices"][0]
    words = full["text"].split()
    stop = " " + words[3] + " "
    r = c.post("/v1/completions", json=dict(COMPL, max_tokens=12, stop=[stop])).json()
    n = len(r["choices"][0]["logprobs"]["tokens"])
    assert r["choices"][0]["finish_reason"] == "stop" and 4 <= n < 12
    assert r["choices"][0]["logprobs"]["tokens"] == full["logprobs"]["tokens"][:n]     # up to the stop's last token
    chunks = _sse(c, "/v1/completions", dict(COMPL, max_tokens=12, stop=[stop]))
    assert sum(len((ch["choices"][0]["logprobs"] or {}).get("tokens", [])) for ch in chunks) == n


def test_logprobs_validation_is_400(client):
    c, engine = client
    msgs = CHAT["messages"]
    for url, body in [("/v1/chat/completions", {"messages": msgs, "logprobs": True, "top_logprobs": 21}),
                      ("/v1/chat/completions", {"messages": msgs, "logprobs": True, "top_logprobs": -1}),
                      ("/v1/chat/completions", {"messages": msgs, "top_logprobs": 3}),
                      ("/v1/completions", {"prompt": "hello", "logprobs": 21}),
                      ("/v1/completions", {"prompt": "hello", "logprobs": -1})]:
        r = c.post(url, json=dict(body, max_tokens=2))
        assert r.status_code == 400 and r.json()["object"] == "error", (url, body, r.text)


def test_requests_without_logprobs_keep_the_old_shape(client):
    c, engine = client
    r = c.post("/v1/completions", json={"prompt": "hello world", "max_tokens": 3, "ignore_eos": True}).json()
    assert r["choices"][0]["logprobs"] is None
    r = c.post("/v1/chat/completions", json={"messages": CHAT["messages"], "max_tokens": 3, "ignore_eos": True}).json()
    assert r["choices"][0]["logprobs"] is None
    chunks = _sse(c, "/v1/chat/completions", {"messages": CHAT["messages"], "max_tokens": 3, "ignore_eos": True})
    assert all("logprobs" not in ch["choices"][0] for ch in chunks)
    chunks = _sse(c, "/v1/completions", {"prompt": "hello", "max_tokens": 3, "ignore_eos": True})
    assert all(ch["choices"][0]["logprobs"] is None for ch in chunks)


def test_stream_delivers_entries_with_the_text_that_releases_them():
    """An entry whose token text is held back (a stop-string prefix) leaves with the delta that releases the text;
    entries of tokens without text leave at the end."""
    from gllm_b200.engine.async_llm_engine import AsyncStream

    async def drain(parts, stop):
        st = AsyncStream(None, stop, logprobs=True)
        for i, p in enumerate(parts):
            st.add_logprobs([i])
            if p is not None:
                st.put(p)
        st.finish("length")
        return [(str(x), x.logprobs) async for x in st]

    assert asyncio.run(drain(["ab", "c<", "/x", "y"], ["</s>"])) == [("ab", [0]), ("c", []), ("</x", [1, 2]),
                                                                            ("y", [3])]
    # the token that completes the stop string is reported with the tokens whose text it cut
    assert asyncio.run(drain(["ab", "c<", "/s", ">zz"], ["</s>"])) == [("ab", [0]), ("c", []), ("", [1, 2, 3])]
    assert asyncio.run(drain(["ab", None, "cd"], None)) == [("ab", [0]), ("cd", [1, 2])]
    assert asyncio.run(drain(["ab", None], None)) == [("ab", [0]), ("", [1])]


def test_generate_rejects_out_of_range_logprobs(hf_model):
    _, d = hf_model
    llm = _engine(d)
    with pytest.raises(ValueError):
        llm.generate(tokens=[[5, 6]], output_lens=[2], logprobs=21)
    llm.shutdown()
