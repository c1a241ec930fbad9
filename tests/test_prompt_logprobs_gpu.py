"""Prompt log-probabilities on the GPU: prompt_logprobs_shard_kernel (csrc/sample/sampler.cu) element by element
against a float64 oracle built from the exact logits it read, against logprobs_shard_kernel, through
logprobs_final_kernel with tp-way records, and the engine's prefill scoring against its own decode log-probs.

Error bound of one reported log-prob lp = x - lse, lse = m + log z, z = sum_i exp(x_i - m), all in fp32. The terms of
tests/test_logprobs_gpu.py, with the one-pass kernel's online rescaling added:
  * exp (fast-math __expf) of term i: at most (2 + 1.173 |x_i - m_run|) ulp, with m_run <= m the running max when the
    term was added, so |x_i - m_run| <= |t_i|, t_i = x_i - m;
  * rescales: the partial sum holding term i is multiplied by exp(m_old - m_new) each time the running max grows,
    each an error of (2 + 1.173 |m_old - m_new|) ulp; the increases add up to at most m - x_i = |t_i|, and a term
    sees at most K in-thread rescales, 5 warp-shuffle merges and 1 merge across the 16 warps. K = ceil(V_shard /
    (512 * 8)) on a row that starts 16-byte aligned (one rescale per 8-wide vector), K = ceil(V_shard / 512) on any
    other row (the scalar path: one per element). So term i carries (2 (K + 7) + 2.346 |t_i|) * 2^-23 relatively;
    over the row the sum of e_i times that,
    divided by z (computed per row from the float64 terms e_i), plus the tp per-shard rescales of the final kernel;
  * the fp32 sum: a thread adds ceil(V_shard / 512) terms (8 at a time), 5 shuffle levels, 16 warp partials, then
    tp shard sums: relative error <= (ceil(V_shard / 512) + 8 + 5 + 16 + tp) * 2^-24 to first order;
  * __logf(z), lse = m + log z and x - lse: as in tests/test_logprobs_gpu.py.
Token ids are compared exactly: the running argmax involves no arithmetic.
"""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_logprobs_gpu import _logits, _oracle  # noqa: E402

pytestmark = pytest.mark.gpu

ULP23, ULP24 = 2.0 ** -23, 2.0 ** -24


def _bound(lp64, m, z, e, t, shard_len: int, tp: int, shard_max=None, aligned: bool = True) -> np.ndarray:
    fin = np.isfinite(t)
    k = math.ceil(shard_len / (512 * 8) if aligned else shard_len / 512) + 6
    exp_rel = float((e[fin] * (2 * (k + 1) + 2.346 * np.abs(t[fin]))).sum() * ULP23 / z)
    if shard_max is not None:
        exp_rel += float(sum((2 + 1.173 * abs(mr - m)) for mr in shard_max if np.isfinite(mr)) * ULP23)
    sum_rel = (math.ceil(shard_len / 512) + 8 + 5 + 16 + tp) * ULP24
    logz = math.log(z)
    log_abs = max(2.0 ** -21.41, 3 * ULP24 * 2 * max(abs(logz), 1e-30))
    lse = m + logz
    return 1.25 * (exp_rel + sum_rel + log_abs + ULP24 * (abs(lse) + np.abs(lp64))) + 1e-7


def _check(out, logits, v, n, targets, tp=1, per=None, what=""):
    out = out.cpu()
    vals, ids = out.numpy(), out.view(torch.int32).numpy()
    x_all = logits[:, :v].double().cpu().numpy()
    targets = targets.cpu().numpy()
    per = per or v
    row_bytes = logits.stride(0) * logits.element_size()
    base = logits.data_ptr()
    worst = (0.0, None)
    for r in range(x_all.shape[0]):
        # every shard of the row starts at a multiple of `per` columns: aligned iff the row and a shard step are
        aligned = (base + r * row_bytes) % 16 == 0 and (tp == 1 or per * logits.element_size() % 16 == 0)
        x64 = x_all[r]
        lp64, order, m, z, e, t = _oracle(x64, max(n, 1))
        smax = [x64[k * per:(k + 1) * per].max() if k * per < v else -np.inf for k in range(tp)] if tp > 1 else None
        bnd = _bound(lp64, m, z, e, t, per, tp, smax, aligned)
        checks = [(int(targets[r]), float(vals[r, 0]), "target")]
        if n:
            assert int(ids[r, 1]) == int(order[0]), f"{what}: row {r}: top-1 id {int(ids[r, 1])} != {int(order[0])}"
            checks.append((int(order[0]), float(vals[r, 2]), "top1"))
        for tok, got, kind in checks:
            want = lp64[tok]
            if not np.isfinite(want):
                assert got == want or (want < 0 and got < -1e30), f"{what}: row {r} {kind} {tok}: {got} vs {want}"
                continue
            ratio = abs(got - want) / bnd[tok]
            if ratio > worst[0]:
                worst = (ratio, (r, tok, kind, got, want, bnd[tok]))
    assert worst[0] <= 1.0, f"{what}: worst row {worst[1][0]} token {worst[1][1]} ({worst[1][2]}): " \
                            f"got {worst[1][3]:.8g}, float64 {worst[1][4]:.8g}, bound {worst[1][5]:.3g}"


def _targets(logits, v, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(0, v, (logits.shape[0],), generator=g, dtype=torch.int32)
    t[0] = int(logits[0, :v].float().argmax())
    if logits.shape[0] > 4:
        t[4] = 0                                  # an -inf logit (row 4 has -inf at every third column)
    return t.to(logits.device)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("n", [0, 1])
@pytest.mark.parametrize("v,pad", [(151936, 64), (1001, 0), (1001, 7)])
def test_prompt_kernel_matches_float64_oracle_and_logprobs_shard(v, pad, n, dtype):
    """V = 151936 with 16-byte rows; V = 1001 with rows of odd length (most rows unaligned: the scalar path) and
    with padding columns."""
    from gllm_b200.ops import sm100
    logits = _logits(12, v, pad, dtype, seed=v + 3 * n + pad)
    targets = _targets(logits, v, seed=v + n)
    rec = sm100.prompt_logprobs_shard(logits, v, n, targets)
    out = sm100.logprobs_final(rec.unsqueeze(0), n)
    old = sm100.logprobs_final(sm100.logprobs_shard(logits, v, n, targets).unsqueeze(0), n)
    torch.cuda.synchronize()
    _check(out, logits, v, n, targets, what=f"V={v} pad={pad} N={n} {dtype}")
    if n:   # the same top-1 id as the multi-pass kernel
        assert torch.equal(out.cpu().view(torch.int32)[:, 1], old.cpu().view(torch.int32)[:, 1])


@pytest.mark.parametrize("tp,v", [(2, 151936), (8, 151936), (8, 300)])
@pytest.mark.parametrize("n", [0, 1])
def test_vocab_parallel_prompt_records_equal_single_shard(tp, v, n):
    """Shards of one padded matrix (the last shard ends with padding; at V = 300, tp = 8 the shards from the third on
    are only padding): tp-way records through logprobs_final give the single-shard ids and log-probs within the
    bound."""
    from gllm_b200.ops import sm100
    per = (v + tp - 1) // tp
    per = (per + 127) // 128 * 128
    logits = _logits(12, v, tp * per - v, torch.bfloat16, seed=tp * 11 + n)
    targets = _targets(logits, v, seed=tp + n)
    single = sm100.logprobs_final(sm100.prompt_logprobs_shard(logits, v, n, targets).unsqueeze(0), n)
    recs = [sm100.prompt_logprobs_shard(logits[:, r * per:(r + 1) * per], max(0, min(per, v - r * per)), n, targets,
                                        vocab_offset=r * per) for r in range(tp)]
    out = sm100.logprobs_final(torch.stack(recs).contiguous(), n)
    torch.cuda.synchronize()
    if n:
        assert torch.equal(out.cpu().view(torch.int32)[:, 1], single.cpu().view(torch.int32)[:, 1])
    _check(out, logits, v, n, targets, tp=tp, per=per, what=f"tp={tp} V={v} N={n}")


def test_engine_prefill_scoring_matches_decode_logprobs(monkeypatch):
    """CUDA graphs and async lookahead on: generate K tokens greedily with logprobs = 5, then resubmit prompt +
    generated tokens with prompt_logprobs = 5 (maxp = 48 and 16-row LM-head tiles: several chunks, several tiles per
    chunk). At the generated positions the prefill entries match the decode ones: bf16 prefill and decode kernels
    round differently, so the log-probs agree within 5e-2 and the top ids wherever neighbouring log-probs differ
    by more than that."""
    from gllm_b200 import LLM
    from gllm_b200.model_runner import ModelRunner
    from gllm_b200.models.presets import tiny
    monkeypatch.setattr(ModelRunner, "PLP_TILE_ROWS", 16)
    cfg = tiny("Qwen3ForCausalLM", hidden_size=256, num_hidden_layers=3, num_attention_heads=4,
               num_key_value_heads=2, head_dim=64, intermediate_size=512, vocab_size=1024, torch_dtype="bfloat16")
    torch.manual_seed(0)
    llm = LLM(cfg, load_format="dummy", maxp=48, maxd=32, max_cuda_graph_bs=8, num_gpu_pages=256,
              model_max_length=512, log_stats=False, seed=0, async_schedule=True)
    prompts = [list(range(20, 190)), [5, 9, 100, 7], [77] * 33]
    k = 12
    gen = llm.generate(tokens=prompts, output_lens=[k] * 3, ignore_eos=True, logprobs=5)
    assert llm.worker.runner.stats["graph_steps"] > 0
    again = llm.generate(tokens=[s.token_ids for s in gen], output_lens=[1] * 3, ignore_eos=True, prompt_logprobs=5)
    assert llm.worker.runner.plp_tile_rows() == 16
    llm.shutdown()
    for s, r, p in zip(gen, again, prompts):
        assert len(r.prompt_logprobs) == len(p) + k and r.prompt_logprobs[0] is None
        for i in range(k):
            dec, pre = s.output_logprobs[i], r.prompt_logprobs[len(p) + i]
            assert abs(dec[0] - pre[0]) < 5e-2, (i, dec[0], pre[0])
            for j, ((ta, la), (tb, lb)) in enumerate(zip(dec[1], pre[1])):
                assert abs(la - lb) < 5e-2, (i, j, la, lb)
                if j + 1 == len(dec[1]):
                    break       # (the gap to the sixth most likely token is not reported)
                gaps = [abs(la - dec[1][q][1]) for q in (j - 1, j + 1) if q >= 0]
                if all(g > 5e-2 for g in gaps):
                    assert ta == tb, (i, j, ta, tb)


def test_bench_without_prompt_logprobs_is_unchanged(tmp_path):
    """`bench.py --gpus 1 --steps 3 --warmup 3` (no request asks for prompt log-probs) generates the same tokens and
    issues the same kernel launches and device-to-host bytes per step as the engine before the feature, recorded on an
    H100 in tests/golden/bench_no_prompt_logprobs.json."""
    import hashlib
    import json
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "tests", "golden", "bench_no_prompt_logprobs.json")) as f:
        want = json.load(f)
    r = subprocess.run([sys.executable, "bench.py", "--gpus", "1", "--steps", "3", "--warmup", "3", "--dump-outputs",
                        str(tmp_path)], cwd=root, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    got = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1])
    assert got["gpu_launches"] == want["gpu_launches"]
    assert got["e2e"]["d2h_bytes_per_step"] == want["d2h_bytes_per_step"]
    toks = np.load(tmp_path / "output_token_ids.npy")
    lens = np.load(tmp_path / "output_lens.npy")
    assert toks.size == want["num_output_tokens"]
    assert hashlib.sha256(np.ascontiguousarray(toks).tobytes()).hexdigest() == want["output_token_ids_sha256"]
    assert hashlib.sha256(np.ascontiguousarray(lens).tobytes()).hexdigest() == want["output_lens_sha256"]
