"""The FP8 W8A8 kernels on the GPU: the per-token quantiser bit for bit against `ops.ref`, both GEMMs (swap-AB split-K
for decode, persistent wgmma for prefill) through identity rows and against float64 on the same quantised operands,
the same bits eager and under CUDA-graph replay, and the engine at Qwen3-8B width with graphs, LoRA and TP."""
import os
import subprocess
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from fp8_util import random_codes, write_channel  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _weight(n, k, gen, static=None):
    from gllm_b200.ops import ref
    scale = torch.rand(n, generator=gen) * 3e-4 + 1e-4
    return ref.Fp8Weight(random_codes(n, k, gen).cuda(), scale.float().cuda(),
                         None if static is None else torch.tensor(static, dtype=torch.float32).cuda())


@pytest.fixture(params=["small", "large"])
def kernel(request, monkeypatch):
    """Route every M through one of the two GEMMs."""
    from gllm_b200.ops import sm100
    monkeypatch.setattr(sm100, "_FP8_SMALLM_MAX", 128 if request.param == "small" else 0)
    return request.param


# ---------------------------------------------------------------------------------------------------------------
# quantiser
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [1, 3, 64, 257, 8192])
@pytest.mark.parametrize("k", [4096, 1040, 1000, 4097])
@pytest.mark.parametrize("static", [None, 0.01])
def test_quantiser_matches_ref_bit_for_bit(m, k, static):
    from gllm_b200.ops import ref, sm100
    gen = torch.Generator().manual_seed(m * 7 + k)
    base = torch.randn(m, k + 24, generator=gen) * torch.logspace(-6, 2, m).view(m, 1)
    base[:, 5] = 0.0
    if m > 2:
        base[2] = 0.0                          # all-zero row
    x = base.to(torch.bfloat16).cuda()[:, 8:8 + k]    # strided rows (16-byte aligned only when k % 8 == 0)
    s_in = None if static is None else torch.tensor(static, dtype=torch.float32).cuda()
    q, s = sm100.fp8_quant_token(x, s_in)
    rq, rs = ref.fp8_quant_token(x.cpu(), None if s_in is None else s_in.cpu())
    assert torch.equal(s.cpu(), rs)
    assert torch.equal(q.cpu().view(torch.uint8), rq.view(torch.uint8))


# ---------------------------------------------------------------------------------------------------------------
# GEMMs
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [1, 16, 100, 128])
@pytest.mark.parametrize("n,k", [(200, 272), (136, 1040), (264, 4096)])
def test_identity_rows_return_the_scaled_codes_bit_for_bit(kernel, m, n, k):
    """x row i = 448 at column k_i, zero elsewhere: s_x = 1 and acc = 448 · w_q[n, k_i] exactly, so the output is
    bf16(448 · w_q · s_w) across tile edges in N and K."""
    from gllm_b200.ops import sm100
    gen = torch.Generator().manual_seed(m + n + k)
    w = _weight(n, k, gen)
    cols = torch.randint(0, k, (m,), generator=gen)
    cols[0] = k - 1
    x = torch.zeros(m, k, dtype=torch.bfloat16)
    x[torch.arange(m), cols] = 448.0
    y = sm100.linear_fp8(x.cuda(), w)
    want = (448.0 * w.codes.cpu().float()[:, cols].t() * w.scale.cpu()).to(torch.bfloat16)
    assert torch.equal(y.cpu(), want)


def _reference(x, w, bias):
    """float64 of the kernel's definition on the same quantised operands."""
    from gllm_b200.ops import ref
    xq, xs = ref.fp8_quant_token(x.cpu(), None if w.input_scale is None else w.input_scale.cpu())
    terms = xq.double().abs() @ w.codes.cpu().double().abs().t()
    acc = xq.double() @ w.codes.cpu().double().t()
    sc = xs.double()[:, None] * w.scale.cpu().double()[None, :]
    y = acc * sc + (bias.cpu().double() if bias is not None else 0.0)
    # bf16 rounding of the output, plus the fp32 sums (K terms, each promoted every 128) of the accumulator
    tol = y.abs() * 2.0 ** -8 + terms * sc * x.shape[1] * 2.0 ** -24 + 1e-30
    return y, tol


def _check(y, x, w, bias):
    ref64, tol = _reference(x, w, bias)
    err = (y.cpu().double() - ref64).abs()
    assert bool((err <= tol).all()), float((err / tol).max())


@pytest.mark.parametrize("m", [1, 5, 16, 17, 32, 33, 64, 65, 100, 128])
@pytest.mark.parametrize("split", [0, 1, 3])
def test_small_m_kernel_against_float64(m, split, monkeypatch):
    from gllm_b200.ops import sm100
    monkeypatch.setattr(sm100, "_FP8_SMALLM_MAX", 128)
    monkeypatch.setattr(sm100, "_FORCE_SPLIT", split)
    gen = torch.Generator().manual_seed(m * 3 + split)
    n, k = 328, 1040
    w = _weight(n, k, gen)
    x = (torch.randn(m, k, generator=gen)).to(torch.bfloat16).cuda()
    bias = (torch.randn(n, generator=gen) * 0.1).to(torch.bfloat16).cuda()
    _check(sm100.linear_fp8(x, w, bias), x, w, bias)
    _check(sm100.linear_fp8(x, w), x, w, None)


@pytest.mark.parametrize("m", [1, 65, 129, 300, 1000, 4096])
def test_large_m_kernel_against_float64(m, monkeypatch):
    from gllm_b200.ops import sm100
    monkeypatch.setattr(sm100, "_FP8_SMALLM_MAX", 0)
    gen = torch.Generator().manual_seed(m)
    n, k = 392, 1040
    w = _weight(n, k, gen)
    x = (torch.randn(m, k, generator=gen) * 2).to(torch.bfloat16).cuda()
    bias = (torch.randn(n, generator=gen) * 0.1).to(torch.bfloat16).cuda()
    _check(sm100.linear_fp8(x, w, bias), x, w, bias)


@pytest.mark.parametrize("m", [1, 24, 200])
def test_strided_x_out_view_and_static_scale(kernel, m):
    from gllm_b200.ops import sm100
    gen = torch.Generator().manual_seed(40 + m)
    n, k = 256, 2048
    w = _weight(n, k, gen, static=0.02)
    wide = (torch.randn(m, k + 512, generator=gen)).to(torch.bfloat16).cuda()
    x = wide[:, 256:256 + k]
    out = torch.full((m, n + 64), 7.0, dtype=torch.bfloat16, device="cuda")
    y = sm100.linear_fp8(x, w, out=out[:, 32:32 + n])
    assert y.data_ptr() == out[:, 32:].data_ptr()
    assert bool((out[:, :32] == 7).all()) and bool((out[:, 32 + n:] == 7).all())
    _check(y, x, w, None)


@pytest.mark.parametrize("n,k", [(6144, 4096), (4096, 4096), (24576, 4096), (4096, 12288), (10240, 8192),
                                 (8192, 14336)])
def test_model_shapes_against_float64(n, k):
    """Qwen3-8B and Llama-3-70B projections (tp 1 / 2) at decode and prefill sizes."""
    from gllm_b200.ops import sm100
    gen = torch.Generator().manual_seed(n + k)
    w = _weight(n, k, gen)
    for m in (1, 32, 64, 256):
        x = torch.randn(m, k, generator=gen).to(torch.bfloat16).cuda()
        _check(sm100.linear_fp8(x, w), x, w, None)


def test_same_bits_eager_and_graph_replay():
    from gllm_b200.ops import sm100
    gen = torch.Generator().manual_seed(11)
    ws = [_weight(6144, 4096, gen), _weight(4096, 12288, gen)]
    xs = [torch.randn(m, w.codes.shape[1], generator=gen).to(torch.bfloat16).cuda()
          for w in ws for m in (1, 7, 32, 100, 300)]

    def run():
        return [sm100.linear_fp8(x, ws[i // 5]) for i, x in enumerate(xs)]

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
    g.replay()
    torch.cuda.synchronize()
    for a, b, c in zip(first, second, graphed):
        assert torch.equal(a, b) and torch.equal(a, c)


# ---------------------------------------------------------------------------------------------------------------
# engine at Qwen3-8B width
# ---------------------------------------------------------------------------------------------------------------
_CFG = dict(hidden_size=4096, num_hidden_layers=2, num_attention_heads=32, num_key_value_heads=8, head_dim=128,
            intermediate_size=12288, vocab_size=2048, torch_dtype="bfloat16", max_position_embeddings=1024)
PROMPTS = [list(range(10, 80)), [5, 9, 100, 7], [77] * 33, list(range(300, 420))]


def _engine(device="cuda", **kw):
    from gllm_b200 import LLM
    from gllm_b200.models.presets import tiny
    args = dict(load_format="dummy", maxp=256, maxd=32, max_cuda_graph_bs=8, model_max_length=1024, log_stats=False,
                seed=0, enable_prefix_caching=False, quantization="fp8", device=device)
    args.update(dict(num_gpu_pages=512) if device == "cuda" else dict(num_cpu_pages=96))
    args.update(kw)
    return LLM(tiny("Qwen3ForCausalLM", **_CFG), **args)


def _logits(llm):
    out = {}
    for ids, lg in llm.worker.runner.logit_log:
        for i, sid in enumerate(ids):
            out.setdefault(sid, []).append(lg[i].double())
    return out


def test_engine_first_step_logits_against_the_cpu_oracle(monkeypatch):
    """Prefill logits of the FP8 engine against the CPU engine on the same parameters, whose W8A8 linears are
    `ref.linear_fp8` (the same quantiser, an exact sum) and whose other ops are fp32 oracles. Where the two engines'
    bf16 activations differ in the last bit, an element can round to the neighbouring e4m3 code (1/16 apart), and the
    random dummy layers carry that on. Bound: relative L2 error 0.15; measured 0.058 to 0.088 on an H100."""
    monkeypatch.setenv("GLLM_KEEP_LOGITS", "1")
    g = _engine(disable_cuda_graph=True)
    c = _engine(device="cpu")
    with torch.no_grad():
        cp = dict(c.worker.runner.model.named_parameters())
        for name, p in g.worker.runner.model.named_parameters():
            cp[name].copy_(p.cpu())
    res = []
    for llm in (g, c):
        outs = llm.generate(tokens=PROMPTS, output_lens=[1] * len(PROMPTS), ignore_eos=True)
        lg = _logits(llm)
        res.append([lg[o.seq_id][0] for o in outs])
        llm.shutdown()
    rels = [float((a - b).norm() / b.norm()) for a, b in zip(*res)]
    print("relative L2 error per prompt:", rels)
    assert max(rels) < 0.15, rels


def test_engine_graphs_decode_like_eager(monkeypatch):
    monkeypatch.setenv("GLLM_KEEP_LOGITS", "1")
    lens = [6, 10, 14, 6]
    logs = []
    for eager in (True, False):
        llm = _engine(disable_cuda_graph=eager)
        outs = llm.generate(tokens=PROMPTS, output_lens=lens, ignore_eos=True)
        logs.append(([o.token_ids for o in outs], dict(llm.worker.runner.stats)))
        llm.shutdown()
    (te, se), (tg, sg) = logs
    assert se["graph_steps"] == 0 and sg["graph_steps"] > 0
    assert te == tg


def test_lora_adapter_on_fp8_base_decodes_through_the_lora_graphs(tmp_path):
    from lora_util import write_adapter
    from gllm_b200.models.presets import tiny
    cfg = tiny("Qwen3ForCausalLM", **_CFG)
    write_adapter(str(tmp_path / "a"), cfg, r=16, alpha=32, seed=1, std=0.05)
    toks = []
    for eager in (True, False):
        llm = _engine(disable_cuda_graph=eager, lora_modules={"a": str(tmp_path / "a")}, max_lora_rank=16)
        outs = llm.generate(tokens=PROMPTS, output_lens=[8] * 4, ignore_eos=True, lora=["a", None, "a", None])
        st = dict(llm.worker.runner.stats)
        toks.append([o.token_ids for o in outs])
        llm.shutdown()
    assert st.get("lora_graph_steps", 0) > 0
    assert toks[0] == toks[1]


def test_checkpoint_engine_pp1_on_the_gpu(tmp_path):
    """A compressed-tensors channel checkpoint through the GPU engine, eager, with the tokens of the CPU engine."""
    from gllm_b200.models.presets import tiny
    cfg = tiny("Qwen3ForCausalLM", hidden_size=512, num_hidden_layers=2, num_attention_heads=8, num_key_value_heads=2,
               head_dim=128, intermediate_size=1024, torch_dtype="bfloat16")
    write_channel(str(tmp_path / "m"), cfg, seed=6)
    out = str(tmp_path / "o")
    env = dict(os.environ, PYTHONPATH=ROOT, GLLM_B200_LOG="WARNING")
    for dev in ("cuda", "cpu"):
        subprocess.run([sys.executable, os.path.join(ROOT, "tests", "mp_fp8.py"), "1", "1", out + dev,
                        str(tmp_path / "m"), dev], env=env, check=True, timeout=600, cwd=ROOT)
    g, c = torch.load(out + "cuda.0"), torch.load(out + "cpu.0")
    x, y = g[1][0][1], c[1][0][1]
    assert float((x - y).norm() / y.norm()) < 0.15


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_tp2_runs(monkeypatch):
    """TP 2 (each rank its own dummy weights): both GEMMs and the NCCL fallback of the fused TP path run."""
    monkeypatch.setenv("GLLM_KEEP_LOGITS", "1")
    llm = _engine(tp_size=2)
    outs = llm.generate(tokens=PROMPTS, output_lens=[8] * 4, ignore_eos=True)
    assert all(len(o.token_ids) == len(p) + 8 for o, p in zip(outs, PROMPTS))
    assert all(bool(torch.isfinite(lg).all()) for _, lg in llm.worker.runner.logit_log)
    llm.shutdown()
