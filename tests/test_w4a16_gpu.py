"""The W4A16 GEMM (csrc/gemm/gemm_w4a16.cu) on the GPU: the de-quantised weight bit for bit through identity rows,
random GEMMs against float64, identical bits eager and under CUDA-graph replay, and the engine at real width against
the same engine running the de-quantised bf16 weights, with CUDA graphs, LoRA adapters and TP."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from w4a16_util import module_tensors, quant_config, random_module  # noqa: E402

pytestmark = pytest.mark.gpu

GROUPS = (32, 64, 128, -1)


def _handle(codes, zeros, scales, group):
    from gllm_b200.ops import ref
    n, k = codes.shape
    p, s, z = ref.w4a16_pack(codes, zeros, scales)
    return ref.Int4Weight(p.cuda(), s.cuda(), z.cuda(), group if group > 0 else k, k)


def _dequant(codes, zeros, scales, group):
    from gllm_b200.ops import ref
    return ref.w4a16_dequant(codes, zeros, scales, group if group > 0 else codes.shape[1], torch.bfloat16)


def _through_checkpoint(method, codes, zeros, scales, group, fmt="gptq"):
    """The module written in `method`'s packing and read back by the loader (`CheckpointReader.get_w4`)."""
    from gllm_b200.models import weight_utils as wu
    t = module_tensors(method, "m", codes, zeros, scales, group, fmt)
    cfg = wu.w4_config(quant_config(method, group, fmt))
    w = wu.CheckpointReader.from_state_dict(t).get_w4("m", cfg)
    return w.codes, w.zeros, w.scales


@pytest.mark.parametrize("group", GROUPS)
@pytest.mark.parametrize("sdt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("method", ["awq", "gptq"])
def test_identity_rows_return_the_dequantised_weight_bit_for_bit(group, sdt, method):
    from gllm_b200.ops import sm100
    gen = torch.Generator().manual_seed(7)
    n, k = 264, 512
    fmt = "gptq_v2" if method == "gptq" else "gptq"
    codes, zeros, scales = random_module(n, k, group, gen, sdt, 0, 15)
    # extreme codes, zeros and scales: q = 0 / 15, z = 0 / 15 (16 through a v1 GPTQ checkpoint below), the largest
    # fp16 scale and subnormal fp16 scales
    codes[:8] = 0
    codes[8:16] = 15
    zeros[16:24] = 0
    zeros[24:32] = 15
    scales[32:40] = 65504.0 if sdt == torch.float16 else 3.0e38 / 16
    scales[40:48] = 2.0 ** -24 if sdt == torch.float16 else 2.0 ** -120
    scales[48:56] = 6.1e-5
    c, z, s = _through_checkpoint(method, codes, zeros, scales, group, fmt)
    assert torch.equal(c, codes) and torch.equal(z, zeros) and torch.equal(s, scales)
    want = _dequant(codes, zeros, scales, group)
    w = _handle(codes, zeros, scales, group)
    for rows in (torch.arange(k), torch.arange(0, k, 37)):
        x = torch.eye(k, dtype=torch.bfloat16)[rows].cuda()
        y = sm100.linear_w4a16(x, w)
        assert torch.equal(y.t().cpu(), want[:, rows]), (group, sdt, method)
    if method == "gptq":     # v1: stored z - 1, so z = 16 is representable
        zeros[56:64] = 16
        zeros[64:72] = 1
        c, z, s = _through_checkpoint("gptq", codes, torch.clamp(zeros, min=1), scales, group, "gptq")
        want = _dequant(c, z, s, group)
        y = sm100.linear_w4a16(torch.eye(k, dtype=torch.bfloat16).cuda(), _handle(c, z, s, group))
        assert torch.equal(y.t().cpu(), want)


def _bound_check(x, wd, bias, y):
    x64, w64 = x.double().cpu(), wd.double()
    y64 = x64 @ w64.t()
    if bias is not None:
        y64 = y64 + bias.double().cpu()
    k = x.shape[1]
    tol = 2.0 ** -8 * y64.abs() + 2 * k * 2.0 ** -24 * (x64.abs() @ w64.abs().t())
    err = (y.double().cpu() - y64).abs()
    assert bool((err <= tol).all()), float((err - tol).max())


MS = [1, 3, 15, 16, 17, 31, 32, 33, 63, 64, 65, 255, 256, 257, 1000, 4099, 8193]


@pytest.mark.parametrize("m", MS)
def test_random_gemm_against_float64(m):
    from gllm_b200.ops import sm100
    gen = torch.Generator().manual_seed(m)
    for n, k, group in ((392, 544, 32), (1024, 4096, 128), (136, 96, 32), (520, 1024, -1)):
        codes, zeros, scales = random_module(n, k, group, gen)
        w = _handle(codes, zeros, scales, group)
        wd = _dequant(codes, zeros, scales, group)
        x = (torch.randn(m, k, generator=gen) * 0.5).to(torch.bfloat16).cuda()
        bias = (torch.randn(n, generator=gen) * 0.1).to(torch.bfloat16).cuda()
        _bound_check(x, wd, None, sm100.linear_w4a16(x, w))
        _bound_check(x, wd, bias, sm100.linear_w4a16(x, w, bias))


# projections of Qwen3-8B and Llama-3-70B at tp 1 and 2: (N, K)
SHAPES = {"qwen3-8b": [(6144, 4096), (4096, 4096), (24576, 4096), (4096, 12288)],
          "llama-3-70b": [(10240, 8192), (8192, 8192), (57344, 8192), (8192, 28672)]}


@pytest.mark.parametrize("model", sorted(SHAPES))
@pytest.mark.parametrize("tp", [1, 2])
def test_model_shapes_against_float64(model, tp):
    from gllm_b200.ops import sm100
    gen = torch.Generator().manual_seed(tp)
    for i, (n, k) in enumerate(SHAPES[model]):
        n, k = (n // tp, k) if i != 1 and i != 3 else (n, k // tp)
        codes, zeros, scales = random_module(n, k, 128, gen)
        w = _handle(codes, zeros, scales, 128)
        wd = _dequant(codes, zeros, scales, 128)
        for m in (1, 32, 300):
            x = (torch.randn(m, k, generator=gen) * 0.5).to(torch.bfloat16).cuda()
            _bound_check(x, wd, None, sm100.linear_w4a16(x, w))


def test_strided_x_and_out_view():
    from gllm_b200.ops import sm100
    gen = torch.Generator().manual_seed(5)
    n, k = 200, 256
    codes, zeros, scales = random_module(n, k, 64, gen)
    w = _handle(codes, zeros, scales, 64)
    wd = _dequant(codes, zeros, scales, 64)
    for m in (5, 70, 600):
        big = (torch.randn(m, k + 64, generator=gen) * 0.5).to(torch.bfloat16).cuda()
        x = big[:, 64:]                                    # row stride k + 64
        out = torch.full((m, n + 24), 7.0, dtype=torch.bfloat16, device="cuda")
        view = out[:, 8:8 + n]
        y = sm100.linear_w4a16(x, w, out=view)
        assert y.data_ptr() == view.data_ptr()
        _bound_check(x, wd, None, view)
        assert bool((out[:, :8] == 7).all()) and bool((out[:, 8 + n:] == 7).all())
        assert torch.equal(sm100.linear(x, w), view)      # `linear` dispatches on the handle


def test_same_bits_eager_and_graph_replay():
    from gllm_b200.ops import sm100
    gen = torch.Generator().manual_seed(11)
    ws = []
    for n, k, g in ((4096, 12288, 128), (1024, 4096, 32)):
        ws.append(_handle(*random_module(n, k, g, gen), g))
    xs = [(torch.randn(m, 12288, generator=gen)).to(torch.bfloat16).cuda() for m in (1, 7, 32, 200)]
    xs2 = [(torch.randn(m, 4096, generator=gen)).to(torch.bfloat16).cuda() for m in (1, 7, 32, 200)]

    def run():
        return [sm100.linear_w4a16(x, ws[0]) for x in xs] + [sm100.linear_w4a16(x, ws[1]) for x in xs2]

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
# engine at real width
# ---------------------------------------------------------------------------------------------------------------
_CFG = dict(hidden_size=4096, num_hidden_layers=2, num_attention_heads=32, num_key_value_heads=8, head_dim=128,
            intermediate_size=12288, vocab_size=2048, torch_dtype="float16", max_position_embeddings=1024)
PROMPTS = [list(range(10, 80)), [5, 9, 100, 7], [77] * 33, list(range(300, 420))]


def _engine(quant=True, **kw):
    from gllm_b200 import LLM
    from gllm_b200.models.presets import tiny
    cfg = tiny("Qwen3ForCausalLM", **_CFG)
    if quant:
        cfg["quantization_config"] = quant_config("awq", 128)
    else:
        cfg["torch_dtype"] = "bfloat16"
    args = dict(load_format="dummy", maxp=256, maxd=32, max_cuda_graph_bs=8, num_gpu_pages=512,
                model_max_length=1024, log_stats=False, seed=0, enable_prefix_caching=False)
    args.update(kw)
    return LLM(cfg, **args)


def _logits(llm):
    out = {}
    for ids, lg in llm.worker.runner.logit_log:
        for i, sid in enumerate(ids):
            out.setdefault(sid, []).append(lg[i].double())
    return out


def test_engine_matches_dequantised_bf16_weights(monkeypatch):
    """Prefill logits of the W4A16 engine against a bf16 engine holding the de-quantised weights (and the same
    embeddings, norms and LM head). Both multiply the same bf16 W; only the GEMMs' summation orders differ. Bound:
    relative L2 error 1e-2; measured 2.2e-3 to 3.1e-3 on an H100."""
    from gllm_b200.ops import ref
    monkeypatch.setenv("GLLM_KEEP_LOGITS", "1")
    q = _engine(disable_cuda_graph=True)
    d = _engine(quant=False, disable_cuda_graph=True)
    qm, dm = q.worker.runner.model, d.worker.runner.model
    with torch.no_grad():
        qp = dict(qm.named_parameters())
        for name, p in dm.named_parameters():
            if name in qp and qp[name].dtype == p.dtype and qp[name].shape == p.shape:
                p.copy_(qp[name])
        from gllm_b200.models.decoder import _qw

        def dq(w, s):
            return ref.w4a16_dequant(*ref.w4a16_unpack(_qw(w, s)), s.group_size, torch.bfloat16).cuda()
        for lq, ld in zip(qm.layers, dm.layers):
            ld.attn.qkv_w.copy_(dq(lq.attn.qkv_w, lq.attn.qkv_ws))
            ld.attn.o_w.copy_(dq(lq.attn.o_w, lq.attn.o_ws))
            ld.mlp.gate_up_w.copy_(ref.interleave_gate_up(dq(lq.mlp.gate_up_w, lq.mlp.gate_up_ws), 128))
            ld.mlp.down_w.copy_(dq(lq.mlp.down_w, lq.mlp.down_ws))
    res = []
    for llm in (q, d):
        outs = llm.generate(tokens=PROMPTS, output_lens=[1] * len(PROMPTS), ignore_eos=True)
        lg = _logits(llm)
        res.append([lg[o.seq_id][0] for o in outs])
        llm.shutdown()
    rels = [float((a - b).norm() / b.norm()) for a, b in zip(*res)]
    print("relative L2 error per prompt:", rels)
    assert max(rels) < 1e-2, rels


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


def test_lora_adapter_on_int4_base_decodes_through_the_lora_graphs(tmp_path):
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


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_tp2_gives_the_tokens_of_tp1():
    res = []
    for tp in (1, 2):
        llm = _engine(tp_size=tp)
        outs = llm.generate(tokens=PROMPTS, output_lens=[8] * 4, ignore_eos=True)
        res.append([o.token_ids for o in outs])
        llm.shutdown()
    assert res[0] == res[1]
