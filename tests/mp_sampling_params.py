"""Per-request sampling parameters (`seed`, `frequency_penalty`, `presence_penalty`, `logit_bias`): the replay oracle
shared by the CPU and GPU tests, and a multi-process engine run.

usage: mp_sampling_params.py <pp> <tp> <out_json> [cpu|cuda]
Runs the engine with GLLM_KEEP_LOGITS=1 (every rank keeps the gathered last-token logits of every step) on a mixed
batch and makes rank 0 write, per request, its prompt, parameters, generated tokens and the kept logits of each
step, so the test can replay the oracle on exactly what the sampler read. The vocabulary (777) is not a multiple of
the shard padding, so the last TP rank's logits shard ends with padding columns.
"""
import json
import os
import sys
from collections import Counter

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# (temperature, top_k, repetition_penalty, seed, frequency_penalty, presence_penalty, logit_bias)
MIXED = [
    dict(temperature=0.0, top_k=1, logit_bias={7: 5.0, 100: -100.0, 3: 2.5}),                 # greedy + bias
    dict(temperature=0.8, top_k=20, seed=1234, frequency_penalty=0.5, presence_penalty=0.5),  # seeded sampled
    dict(temperature=0.8, top_k=8),                                                            # plain unseeded
    dict(temperature=0.0, top_k=1, repetition_penalty=1.3, frequency_penalty=0.7),           # rep + frequency
]


def x2_row(x, prompt, outs, p):
    """float64 x2 of one step (see entrypoints/protocol.py): repetition penalty over prompt + output, then
    - f * c_j - p * [c_j > 0] + logit_bias_j, with c_j the counts among the generated tokens `outs`."""
    x = np.asarray(x, dtype=np.float64).copy()
    rep = p.get("repetition_penalty", 1.0)
    if rep != 1.0:
        seen = np.zeros(x.size, dtype=bool)
        seen[list(set(prompt) | set(outs))] = True
        x = np.where(seen, np.where(x > 0, x / rep, x * rep), x)
    f, pr = p.get("frequency_penalty", 0.0), p.get("presence_penalty", 0.0)
    for tok, c in Counter(outs).items():
        x[tok] -= f * c + pr
    for tok, b in (p.get("logit_bias") or {}).items():
        x[int(tok)] += b
    return x


def race_scores(t, seed, pos, top_k):
    """float64 exponential-race scores of a seeded row over its top-k survivors (ties at the threshold survive, as
    in the kernel); -inf elsewhere."""
    from gllm_b200.ops import ref
    v = t.size
    keep = np.isfinite(t)
    if 0 < top_k < v:
        thr = np.sort(t)[::-1][top_k - 1]
        keep &= t >= thr
    u = ref.race_uniform(seed, pos, np.arange(v)).astype(np.float64)
    e = -np.log(u)
    m = t[keep].max()
    return np.where(keep, (t - m) - np.log(e), -np.inf)


def replay(prompt, outs, steps, p, tol):
    """Check every generated token against the oracle on the kept logits `steps[j]`. Greedy and seeded rows: the
    oracle's choice, except where the oracle's best and the engine's token lie within `tol(...)` of each other (a
    near-tie inside the fp32 rounding bound); unseeded sampled rows: a top-k survivor. Returns the near-tie count."""
    near = 0
    for j, tok in enumerate(outs):
        x = x2_row(steps[j], prompt, outs[:j], p)
        if p.get("top_k", 1) == 1:
            s = x
        elif p.get("seed") is not None:
            s = race_scores(x / p["temperature"], p["seed"], len(prompt) + j, p["top_k"])
        else:
            t = x / p["temperature"]
            thr = np.sort(t)[::-1][p["top_k"] - 1]
            assert t[tok] >= thr, (j, tok, "not a top-k survivor")
            continue
        want = int(np.lexsort((np.arange(s.size), -s))[0])
        if tok != want:
            assert s[want] - s[tok] <= tol(x, s, want, tok), (j, tok, want, float(s[want]), float(s[tok]))
            near += 1
    return near


def main():
    pp, tp, out = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3]
    device = sys.argv[4] if len(sys.argv) > 4 else "cpu"
    os.environ["GLLM_KEEP_LOGITS"] = "1"
    import torch
    from gllm_b200 import LLM
    from gllm_b200.models.presets import tiny
    cpu = device == "cpu"
    cfg = tiny("Qwen3ForCausalLM", num_hidden_layers=4, vocab_size=777,
               **({} if cpu else dict(hidden_size=256, head_dim=64, torch_dtype="bfloat16")))
    torch.manual_seed(0)
    dev_kw = dict(device="cpu", num_cpu_pages=128) if cpu else dict(num_gpu_pages=256, max_cuda_graph_bs=8)
    llm = LLM(cfg, load_format="dummy", pp_size=pp, tp_size=tp, maxp=48, maxd=16, model_max_length=256,
              log_stats=False, launch_mode="inproc", seed=0, async_schedule=os.environ.get("GLLM_TEST_ASYNC") == "1",
              **dev_kw)
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from shard_util import load_global_weights
    load_global_weights(llm.worker.runner.model, cfg, seed=123)
    prompts = [[5, 17, 99, 200, 3, 45, 7], [9] * 40, list(range(20, 120)), [300, 301]]
    kw = {k: [p.get(k) for p in MIXED] for k in ("temperature", "top_k", "seed", "frequency_penalty",
                                                  "presence_penalty", "logit_bias")}
    kw["repetition_penalty"] = [p.get("repetition_penalty", 1.0) for p in MIXED]
    kw["top_p"] = 1.0         # (the oracle has no top-p; the engine's default comes from the generation config)
    seqs = llm.generate(tokens=prompts, output_lens=[8] * 4, ignore_eos=True, **kw)
    runner = llm.worker.runner
    if int(os.environ.get("RANK", "0")) == 0:
        per = {s.seq_id: [] for s in seqs}
        for ids, lg in runner.logit_log:
            for row, sid in enumerate(ids):
                if sid in per:
                    per[sid].append(lg[row].tolist())
        with open(out, "w") as f:
            json.dump([[p, s.token_ids[len(p):], per[s.seq_id]] for s, p in zip(seqs, prompts)], f)
    llm.shutdown()
    if torch.distributed.is_initialized():
        torch.distributed.barrier()
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
