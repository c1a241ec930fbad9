"""Parallel sampling (`n` choices per request) on the GPU: `kv_copy_pages` (csrc/elemwise/kv_copy.cu) element by
element, greedy choices with CUDA graphs and lookahead (the shared prompt pages and the copied partial page must give
every choice bitwise the same logits), seeded sampled choices with penalties and logit_bias against the sampling
oracle, and TP2."""
import os

import numpy as np
import pytest
import torch

import mp_sampling_params as mp

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------
# 1. kv_copy_pages
# ------------------------------------------------------------------------------------------------
def _random_bits(shape, gen):
    """bf16 tensor with uniformly random bit patterns (NaNs and infinities included): a copy must move the bits."""
    raw = torch.randint(-2 ** 15, 2 ** 15, shape, dtype=torch.int32, generator=gen).to(torch.int16)
    return raw.view(torch.bfloat16).cuda()


@pytest.mark.parametrize("kind", ["kv", "mla"])
@pytest.mark.parametrize("n_pairs", [1, 8, 64])
def test_kv_copy_pages_bitwise(kind, n_pairs):
    from gllm_b200.ops import sm100
    from gllm_b200.ops.ref import kv_cache_shape
    gen = torch.Generator().manual_seed(n_pairs)
    pages, layers = 160, 5
    if kind == "kv":        # Qwen3-8B per rank: 8 KV heads of 128, 16-token pages; K and V per layer
        shape = kv_cache_shape(pages, 8, 128, 16)
        tensors = [_random_bits(shape, gen) for _ in range(2 * layers)]
    else:                   # DeepSeek-V2 latent: 512 + 64, one "head"
        shape = kv_cache_shape(pages, 1, 576, 16)
        tensors = [_random_bits(shape, gen) for _ in range(layers)]
    dummy = pages - 1
    perm = torch.randperm(pages - 1, generator=gen).tolist()
    dst = perm[:n_pairs - 1] + [pages - 2] if (pages - 2) not in perm[:n_pairs - 1] else perm[:n_pairs]
    rest = [p for p in range(pages - 1) if p not in dst]
    src = [rest[i % len(rest)] for i in range(n_pairs)]      # a src may be copied to several dst pages
    pairs = list(zip(src, dst))
    before = [t.clone() for t in tensors]
    sm100.kv_copy_pages(tensors, pairs, dummy_page=dummy)
    torch.cuda.synchronize()
    dset = set(dst)
    keep = torch.tensor([p for p in range(pages) if p not in dset], device="cuda")
    for li, (t, b) in enumerate(zip(tensors, before)):
        tv, bv = t.view(torch.int16), b.view(torch.int16)
        for s, d in pairs:
            assert torch.equal(tv[d], bv[s]), (li, s, d)
        assert torch.equal(tv[keep], bv[keep]), li           # every page not named as a dst is unchanged
    assert (pages - 2) in dset


@pytest.mark.parametrize("pairs", [[(1, 2), (3, 2)], [(1, 2), (2, 4)], [(1, 15)], [(15, 3)], [(1, 16)]])
def test_kv_copy_pages_rejects_bad_pairs_before_launch(pairs):
    from gllm_b200.ops import sm100
    t = torch.zeros(16, 1, 2, 16, 64, dtype=torch.bfloat16, device="cuda")
    n0 = sm100.launches()
    with pytest.raises(ValueError):
        sm100.kv_copy_pages([t], pairs, dummy_page=15)
    assert sm100.launches() == n0


# ------------------------------------------------------------------------------------------------
# 2. engine
# ------------------------------------------------------------------------------------------------
def _engine_cfg():
    from gllm_b200.models.presets import tiny
    return tiny("Qwen3ForCausalLM", hidden_size=256, num_hidden_layers=3, num_attention_heads=4,
                num_key_value_heads=2, head_dim=64, intermediate_size=512, vocab_size=1024, torch_dtype="bfloat16")


def _llm(**kw):
    from gllm_b200 import LLM
    torch.manual_seed(0)
    return LLM(_engine_cfg(), load_format="dummy", maxp=128, maxd=64, max_cuda_graph_bs=8, num_gpu_pages=256,
               model_max_length=512, log_stats=False, seed=0, async_schedule=True, enable_prefix_caching=False, **kw)


def _per_seq(runner, outs):
    per = {s.seq_id: [] for s in outs}
    for ids, lg in runner.logit_log:
        for row, sid in enumerate(ids):
            if sid in per:
                per[sid].append(lg[row].numpy())
    return per


# P mod 16 = 1, 15 and 0 (16-token pages)
PROMPTS = [list(range(20, 53)), [77] * 31, [3, 1, 4, 1, 5, 9, 2, 6] * 4]


@pytest.mark.parametrize("prompt", PROMPTS, ids=["p33", "p31", "p32"])
def test_greedy_choices_have_bitwise_equal_logits(monkeypatch, prompt):
    monkeypatch.setenv("GLLM_KEEP_LOGITS", "1")
    n_out = 24
    llm = _llm()
    one = llm.generate(tokens=[prompt], output_lens=[n_out], ignore_eos=True, top_k=1)
    many = llm.generate(tokens=[prompt, prompt], output_lens=[n_out] * 2, ignore_eos=True, top_k=1, n=4)
    runner = llm.worker.runner
    assert runner.stats["graph_steps"] > 0 and runner.stats.get("feed_steps", 0) > 0
    copied = runner.stats.get("kv_copy_pages", 0)
    per = _per_seq(runner, one + many)
    llm.shutdown()
    assert copied == (6 if len(prompt) % 16 else 0)
    base = one[0]
    for r in range(2):
        ch = many[4 * r: 4 * r + 4]
        rows = [per[s.seq_id] for s in ch]
        assert all(len(x) == n_out for x in rows)
        for i in range(1, 4):
            assert np.array_equal(rows[i][0], rows[0][0])           # first tokens: one logits row
            for j in range(n_out):                                  # the forks decode side by side in every step
                assert np.array_equal(rows[i][j], rows[1][j]), (r, i, j)
            assert ch[i].token_ids == ch[1].token_ids
        # choice 0 runs its steps in other batches than the forks (its first decode step rides on the lookahead):
        # its tokens equal theirs, and the n = 1 run's, as long as the logits agree bitwise
        for other in (ch[1], base):
            lo = per[other.seq_id]
            for j in range(n_out):
                if not np.array_equal(rows[0][j], lo[j]):
                    break
                assert ch[0].token_ids[len(prompt) + j] == other.token_ids[len(prompt) + j], (r, j)


def _tol_gpu(x, s, want, tok):
    return 3e-5      # as in test_sampling_params_gpu.py


def test_seeded_choices_follow_the_oracle(monkeypatch):
    monkeypatch.setenv("GLLM_KEEP_LOGITS", "1")
    prompt = list(range(20, 61))
    p = dict(temperature=0.8, top_k=20, frequency_penalty=0.5, presence_penalty=0.3, logit_bias={7: 3.0, 100: -100.0})
    seed = 2 ** 63 - 2
    llm = _llm()
    outs = llm.generate(tokens=[prompt], output_lens=[16], ignore_eos=True, top_p=1.0, n=4, seed=seed, **p)
    per = _per_seq(llm.worker.runner, outs)
    llm.shutdown()
    first = [per[s.seq_id][0] for s in outs]
    assert all(np.array_equal(f, first[0]) for f in first[1:])
    near = 0
    for i, s in enumerate(outs):
        assert s.seed == mp_seed(seed, i)
        toks = s.token_ids[len(prompt):]
        assert len(per[s.seq_id]) == len(toks) == 16
        near += mp.replay(prompt, toks, [x.astype(np.float64) for x in per[s.seq_id]], dict(p, seed=s.seed),
                          _tol_gpu)
        assert 100 not in toks
    assert near <= 2
    assert len({tuple(s.token_ids) for s in outs}) > 1


def mp_seed(seed, i):
    return (seed + i + 2 ** 63) % 2 ** 64 - 2 ** 63


def test_tp2_greedy_choices_equal_n1():
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
               "--master-addr", "127.0.0.1", "--master-port", "29981",
               os.path.join(root, "tests", "mp_parallel_sampling.py"), "1", "2", out, "cuda"]
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=root,
                           env=dict(os.environ, PYTHONPATH=root, GLLM_TEST_ASYNC="1"))
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
        got = json.load(open(out))
    for j in range(len(got["single"])):
        ch = got["many"][3 * j: 3 * j + 3]
        assert ch[1] == ch[2], j                      # the forks decode side by side: bitwise the same logits
        assert ch[0][0] == ch[1][0], j                # first tokens: one logits row
    assert got["copied"] > 0
