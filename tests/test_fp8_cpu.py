"""FP8 W8A8 checkpoints on the CPU: each format loads to the checkpoint's codes and expanded scales (per TP shard),
every refusal, the per-token quantiser's known answers, and the engine across formats, online quantisation, PP / TP
over gloo and LoRA adapters."""
from conftest import scratch_dir
import inspect
import os
import subprocess
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from fp8_util import (E4M3, ct_config, hf_config, online_rule, write_channel, write_online_pair,  # noqa: E402
                      write_tensor_pair)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _tiny(arch="Qwen3ForCausalLM", layers=2, **kw):
    from gllm_b200.models.presets import tiny
    return tiny(arch, num_hidden_layers=layers, **kw)


def _build(cfg, tp=1, rank=0, monkeypatch=None):
    from gllm_b200.models import registry
    from gllm_b200.parallel import state as ps
    if tp > 1:
        monkeypatch.setattr(ps.get_state(), "tp_size", tp)
        monkeypatch.setattr(ps.get_state(), "tp_rank", rank)
    return registry.build_model(registry.HFConfig(cfg), "cpu")


# ---------------------------------------------------------------------------------------------------------------
# formats: codes byte for byte, scales expanded, per TP shard
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ["hf-tensor", "ct-tensor", "ct-channel", "ct-channel-bf16", "hf-static"])
@pytest.mark.parametrize("tp", [1, 2])
def test_each_format_loads_codes_and_scales_exactly(fmt, tp, monkeypatch):
    from gllm_b200.models import weight_utils as wu
    from gllm_b200.models.decoder import _qw
    cfg = _tiny("LlamaForCausalLM", layers=1)
    d = scratch_dir("gllm_b200_fp8_")
    if fmt == "ct-channel":
        mods = write_channel(os.path.join(d, "m"), cfg, seed=1)
        path = os.path.join(d, "m")
    elif fmt == "ct-channel-bf16":
        mods = write_channel(os.path.join(d, "m"), cfg, seed=1, scale_dtype=torch.bfloat16)
        mods = {k: (c, s.bfloat16().float(), i) for k, (c, s, i) in mods.items()}
        path = os.path.join(d, "m")
    else:
        mods = write_tensor_pair(os.path.join(d, "hf"), os.path.join(d, "ct"), cfg, seed=1, static=fmt == "hf-static")
        path = os.path.join(d, "ct" if fmt == "ct-tensor" else "hf")
    import json
    with open(os.path.join(path, "config.json")) as f:
        full_cfg = json.load(f)
    h, nh, nkv = cfg["hidden_size"], cfg["num_attention_heads"], cfg["num_key_value_heads"]
    hd = h // nh

    def full(m):
        codes, s, ins = mods["model.layers.0." + m]
        return codes, s.float().reshape(-1).expand(codes.shape[0]), ins

    for r in range(tp):
        model = _build(full_cfg, tp, r, monkeypatch)
        model.load_weights(wu.CheckpointReader(path))
        at, mlp = model.layers[0].attn, model.layers[0].mlp
        q, k, v = (full(f"self_attn.{x}_proj") for x in "qkv")
        want_codes = wu.shard_qkv(q[0], k[0], v[0], nh, nkv, hd, r, tp)
        want_scale = wu.shard_qkv(q[1], k[1], v[1], nh, nkv, hd, r, tp)
        hq = _qw(at.qkv_w, at.qkv_ws)
        assert torch.equal(hq.codes.view(torch.uint8), want_codes.view(torch.uint8))
        assert torch.equal(hq.scale, want_scale)
        if fmt == "hf-static":
            assert torch.equal(hq.input_scale, torch.stack([q[2], k[2], v[2]]).max())
        else:
            assert hq.input_scale is None
        g, u = full("mlp.gate_proj"), full("mlp.up_proj")
        hg = _qw(mlp.gate_up_w, mlp.gate_up_ws)
        assert torch.equal(hg.codes.view(torch.uint8), wu.shard_gate_up(g[0], u[0], r, tp).view(torch.uint8))
        assert torch.equal(hg.scale, wu.shard_gate_up(g[1], u[1], r, tp))
        for hnd, (codes, s, _) in ((_qw(at.o_w, at.o_ws), full("self_attn.o_proj")),
                                   (mlp.down_weight(), full("mlp.down_proj"))):
            assert torch.equal(hnd.codes.view(torch.uint8), wu.shard_cols(codes, r, tp).view(torch.uint8))
            assert torch.equal(hnd.scale, s)      # row-parallel: every output channel's full scale


def test_per_tensor_checkpoint_serves_the_right_weights():
    """The regression: a per-tensor HF fp8 checkpoint used to load its raw e4m3 codes as bf16 weights (|w| up to
    448) and ignore `weight_scale`. The de-quantised weights now equal the originals to within e4m3 rounding."""
    from gllm_b200.models import weight_utils as wu
    from gllm_b200.models.decoder import _qw
    from w4a16_util import MODS, shapes
    cfg = _tiny("LlamaForCausalLM", layers=1, quantization_config=hf_config())
    gen = torch.Generator().manual_seed(0)
    sd, orig = {}, {}
    for m, (n, k) in shapes(cfg).items():
        w = torch.randn(n, k, generator=gen) * 0.02
        s = w.abs().amax() / 448
        name = "model.layers.0." + MODS[m]
        sd[name + ".weight"] = (w / s).to(E4M3)
        sd[name + ".weight_scale"] = s.reshape(())
        orig[m] = w
    h, v = cfg["hidden_size"], cfg["vocab_size"]
    for n in ("model.layers.0.input_layernorm.weight", "model.layers.0.post_attention_layernorm.weight",
              "model.norm.weight"):
        sd[n] = torch.ones(h)
    sd["model.embed_tokens.weight"] = sd["lm_head.weight"] = torch.randn(v, h) * 0.02
    model = _build(cfg)
    assert model.spec.quant == "w8a8"
    model.load_weights(wu.CheckpointReader.from_state_dict(sd))
    hq = _qw(model.layers[0].attn.qkv_w, model.layers[0].attn.qkv_ws)
    wq = hq.codes.float() * hq.scale[:, None]
    nq = orig["q"].shape[0]
    assert float(wq[:nq].abs().max()) < 0.1
    # e4m3 keeps 3 mantissa bits: relative error <= 2^-4, plus the subnormal step (2^-9 · s) near zero
    s = orig["q"].abs().amax() / 448
    assert bool(((wq[:nq] - orig["q"]).abs() <= orig["q"].abs() / 16 + s * 2 ** -10).all())


# ---------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------
_W = {"num_bits": 8, "type": "float", "symmetric": True, "strategy": "channel", "dynamic": False}


@pytest.mark.parametrize("qc,match", [
    (ct_config(input_activations=None), "weight-only"),
    (ct_config(weights=dict(_W, strategy="group", group_size=128)), "strategy='group'"),
    (ct_config(weights=dict(_W, strategy="block", block_structure=[128, 128])), "strategy='block'"),
    (ct_config(weights=dict(_W, num_bits=4, type="int")), "not 8-bit"),
    (ct_config(weights=dict(_W, symmetric=False)), "not 8-bit symmetric"),
    (dict(ct_config(), ignore=["lm_head", "model.layers.0.mlp.down_proj"]), "ignore"),
    (dict(ct_config(), format="pack-quantized"), "format"),
    (ct_config(input_activations={"num_bits": 8, "type": "float", "strategy": "token", "dynamic": False}),
     "strategy='token'"),
    (ct_config(input_activations={"num_bits": 8, "type": "float", "strategy": "group", "dynamic": True}),
     "strategy='group'"),
    (dict(ct_config(), config_groups={}), "config groups"),
    (dict(hf_config(), activation_scheme="weird"), "activation_scheme"),
    (dict(hf_config(), ignored_layers=["model.layers.1.self_attn.q_proj"]), "ignore"),
])
def test_unsupported_fp8_configs_are_refused(qc, match):
    from gllm_b200.models import registry
    with pytest.raises(ValueError, match=match):
        registry.build_model(registry.HFConfig(_tiny(quantization_config=qc)), "cpu")


def test_lm_head_in_the_ignore_list_and_a_kv_cache_scheme_are_accepted():
    from gllm_b200.models import registry
    qc = dict(ct_config(), kv_cache_scheme={"num_bits": 8, "type": "float", "strategy": "tensor"})
    assert registry.build_model(registry.HFConfig(_tiny(quantization_config=qc)), "cpu").spec.quant == "w8a8"


@pytest.mark.parametrize("arch", ["MixtralForCausalLM", "Qwen2MoeForCausalLM", "Qwen3MoeForCausalLM",
                                  "DeepseekV3ForCausalLM", "ChatGLMModel", "Qwen2_5_VLForConditionalGeneration"])
@pytest.mark.parametrize("how", ["checkpoint", "online"])
def test_other_architectures_are_refused(arch, how):
    from gllm_b200.models import registry
    cfg = _tiny(arch) if how == "online" else _tiny(arch, quantization_config=ct_config())
    if how == "online":
        cfg[registry.QUANTIZATION_KEY] = "fp8"
    with pytest.raises(ValueError, match=arch):
        registry.build_model(registry.HFConfig(cfg), "cpu")


@pytest.mark.parametrize("qc", [ct_config(), {"quant_method": "awq", "bits": 4, "group_size": 64},
                                {"quant_method": "fp8", "weight_block_size": [128, 128]}])
def test_online_quantisation_of_a_quantised_checkpoint_is_refused(qc):
    from gllm_b200 import LLM
    with pytest.raises(ValueError, match="quantization='fp8' needs an unquantised checkpoint"):
        LLM(_tiny(quantization_config=qc), device="cpu", quantization="fp8", log_stats=False)


def test_unknown_quantization_option_is_refused():
    from gllm_b200 import LLM
    with pytest.raises(ValueError, match="quantization='int8'"):
        LLM(_tiny(), device="cpu", quantization="int8", log_stats=False)


def test_e5m2_weights_are_refused():
    from gllm_b200.models import weight_utils as wu
    sd = {"m.weight": torch.zeros(16, 32, dtype=torch.float8_e5m2), "m.weight_scale": torch.ones(16, 1)}
    with pytest.raises(ValueError, match="e4m3"):
        wu.CheckpointReader.from_state_dict(sd).get_w8("m", wu.w8_config(ct_config()))


def test_block_scaled_fp8_is_unchanged():
    from gllm_b200.models import registry
    qc = {"quant_method": "fp8", "weight_block_size": [128, 128], "activation_scheme": "dynamic"}
    cfg = _tiny(hidden_size=256, intermediate_size=512, quantization_config=qc)
    m = registry.build_model(registry.HFConfig(cfg), "cpu")
    assert m.spec.quant == "fp8" and m.spec.w8 is None
    assert isinstance(m.layers[0].attn.qkv_ws, torch.nn.Parameter)


# ---------------------------------------------------------------------------------------------------------------
# the per-token quantiser and the op tables
# ---------------------------------------------------------------------------------------------------------------
def test_fp8_quant_token_known_answers():
    from gllm_b200.ops import ref
    x = torch.zeros(5, 24, dtype=torch.bfloat16)
    x[1, 3], x[1, 7] = 448.0, -224.0                   # amax exactly 448: scale 1, codes exact
    x[2, 0], x[2, 1] = 1.0, 2.0 ** -10                 # 2^-10 · 448 = 0.4375 = 7 · 2^-4: a normal e4m3 (2^-2 · 1.75)
    x[3, 0], x[3, 1] = 448.0, 2.0 ** -7                # scale 1: 2^-7 is subnormal in e4m3 (min normal 2^-6)
    x[4, 0], x[4, 1] = 448.0, 2.0 ** -11               # below half the smallest subnormal (2^-9): rounds to 0
    q, s = ref.fp8_quant_token(x)
    assert s.dtype == torch.float32 and q.dtype == E4M3
    assert float(s[0]) == (torch.tensor(1e-10) / 448).item() and not q[0].float().any()
    assert float(s[1]) == 1.0 and float(q[1, 3]) == 448.0 and float(q[1, 7]) == -224.0
    assert float(q[2, 0]) == 448.0 and float(q[2, 1]) == 0.4375
    assert float(q[3, 1]) == 2.0 ** -7 and q[3, 1].view(torch.uint8).item() == 0x04   # subnormal code 4 · 2^-9
    assert float(q[4, 1]) == 0.0
    # static: x / s, clamped to +-448
    xs = torch.tensor([[1.0, -1000.0, 0.5, 3.0]], dtype=torch.bfloat16)
    q, s = ref.fp8_quant_token(xs, torch.tensor(0.5))
    assert float(s[0]) == 0.5 and q.float().tolist() == [[2.0, -448.0, 1.0, 6.0]]
    # the GEMM of the identity row: 448 · w_q · s_w
    w = ref.Fp8Weight(torch.tensor([[1.0, -2.0], [0.5, 448.0]]).to(E4M3), torch.tensor([0.25, 2.0 ** -9]))
    y = ref.linear_fp8(torch.tensor([[448.0, 0.0]], dtype=torch.bfloat16), w)
    assert y.float().tolist() == [[448.0 * 0.25, 448.0 * 0.5 * 2.0 ** -9]]


def test_cpu_stand_ins_have_the_kernel_signatures():
    from gllm_b200.ops import cpu, sm100
    for name in ("linear_fp8", "fp8_quant_token"):
        assert inspect.signature(getattr(cpu, name)) == inspect.signature(getattr(sm100, name))


def test_dummy_weights_have_the_intended_spread():
    from gllm_b200.models import registry
    from gllm_b200.models.decoder import _qw
    cfg = _tiny(hidden_size=512, intermediate_size=1024, num_attention_heads=8, num_key_value_heads=2, head_dim=64)
    cfg[registry.QUANTIZATION_KEY] = "fp8"
    model = registry.build_model(registry.HFConfig(cfg), "cpu")
    model.init_dummy()
    for hnd in (_qw(model.layers[0].attn.qkv_w, model.layers[0].attn.qkv_ws), model.layers[1].mlp.down_weight()):
        wd = hnd.codes.float() * hnd.scale[:, None]
        assert abs(float(wd.std()) - 0.02) < 0.002, float(wd.std())


def test_online_rule():
    from gllm_b200.ops import ref
    w = torch.tensor([[0.0, 0.0], [1.0, -3.0], [1e-3, 2e-3]], dtype=torch.bfloat16)
    codes, s = ref.fp8_channel_quant(w)
    c2, s2 = online_rule(w)
    assert torch.equal(codes.view(torch.uint8), c2.view(torch.uint8)) and torch.equal(s, s2)
    assert float(s[0]) == (torch.tensor(1e-12) / 448).item() and float(codes[1, 1]) == -448.0


# ---------------------------------------------------------------------------------------------------------------
# the engine
# ---------------------------------------------------------------------------------------------------------------
PROMPTS = [[5, 17, 99, 200, 3, 45, 7], [9] * 40, list(range(20, 150)), [300, 301]]


def _run(path, monkeypatch, lora_modules=None, lora=None, **kw):
    from gllm_b200 import LLM
    monkeypatch.setenv("GLLM_KEEP_LOGITS", "1")
    llm = LLM(path, device="cpu", num_cpu_pages=96, maxp=64, maxd=16, model_max_length=320, log_stats=False,
              lora_modules=lora_modules, max_lora_rank=16, **kw)
    outs = llm.generate(tokens=PROMPTS, output_lens=[6] * len(PROMPTS), ignore_eos=True, lora=lora)
    logits = [(ids, lg.clone()) for ids, lg in llm.worker.runner.logit_log]
    llm.shutdown()
    return [o.token_ids for o in outs], logits


def _same(a, b):
    assert a[0] == b[0]
    assert len(a[1]) == len(b[1]) and all(x[0] == y[0] and torch.equal(x[1], y[1]) for x, y in zip(a[1], b[1]))


@pytest.mark.parametrize("arch,static", [("LlamaForCausalLM", False), ("Qwen2ForCausalLM", True),
                                         ("Qwen3ForCausalLM", False)])
def test_hf_per_tensor_and_compressed_tensors_tensor_give_identical_logits(arch, static, monkeypatch):
    d = scratch_dir("gllm_b200_fp8_")
    write_tensor_pair(os.path.join(d, "hf"), os.path.join(d, "ct"), _tiny(arch), seed=2, static=static)
    a = _run(os.path.join(d, "hf"), monkeypatch)
    _same(a, _run(os.path.join(d, "ct"), monkeypatch))
    assert all(bool(torch.isfinite(x[1]).all()) for x in a[1])


def test_online_quantisation_equals_the_channel_checkpoint_of_the_rule(monkeypatch):
    d = scratch_dir("gllm_b200_fp8_")
    write_online_pair(os.path.join(d, "bf16"), os.path.join(d, "ct"), _tiny("Qwen3ForCausalLM"), seed=3)
    online = _run(os.path.join(d, "bf16"), monkeypatch, quantization="fp8")
    _same(online, _run(os.path.join(d, "ct"), monkeypatch))
    # and it is a different model from the bf16 one, close to it
    plain = _run(os.path.join(d, "bf16"), monkeypatch)
    x, y = online[1][0][1], plain[1][0][1]
    assert not torch.equal(x, y) and float((x - y).norm() / y.norm()) < 0.1


def test_lora_on_the_fp8_base(monkeypatch):
    """Adapters on an FP8 base: the online-quantised base and the equivalent channel checkpoint give the same logits
    with the adapter, bit for bit; a base-only request in the same batch gets the base model's logits, bit for bit;
    an adapter request gets different ones."""
    from lora_util import write_adapter
    d = scratch_dir("gllm_b200_fp8_")
    cfg = _tiny("Qwen3ForCausalLM")
    write_online_pair(os.path.join(d, "bf16"), os.path.join(d, "ct"), cfg, seed=4)
    a = os.path.join(d, "a")
    write_adapter(a, cfg, r=8, alpha=16, seed=5)
    lora = ["a", None, "a", "a"]
    t_online, l_online = _run(os.path.join(d, "bf16"), monkeypatch, {"a": a}, lora, quantization="fp8")
    t_ct, l_ct = _run(os.path.join(d, "ct"), monkeypatch, {"a": a}, lora)
    _same((t_online, l_online), (t_ct, l_ct))
    _, base = _run(os.path.join(d, "ct"), monkeypatch)
    # the base-only request gives the base model's logits, bit for bit, with adapters in the batch
    assert torch.equal(l_ct[0][1][1], base[0][1][1])
    assert not torch.equal(l_ct[0][1][0], base[0][1][0])


def _mp(pp, tp, port, d):
    out = os.path.join(scratch_dir("gllm_b200_fp8_mp_"), "out")
    env = dict(os.environ, PYTHONPATH=ROOT, GLLM_B200_LOG="WARNING")
    script = os.path.join(ROOT, "tests", "mp_fp8.py")
    if pp * tp == 1:
        cmd = [sys.executable, script, "1", "1", out, d, "cpu"]
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={pp * tp}",
               "--master-addr", "127.0.0.1", "--master-port", str(port), script, str(pp), str(tp), out, d, "cpu"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    ranks = [torch.load(f"{out}.{r}") for r in range(pp * tp)]
    return next(t for t, _ in ranks if t), next(lg for _, lg in ranks if lg)


def _rows(res):
    """Every logits row of a run, in a fixed order (PP regroups the steps' rows)."""
    x = torch.cat([lg for _, lg in res[1]])
    return x[torch.argsort(x.double().sum(1))]


def test_pp2_and_tp2_against_tp1():
    """PP 2 changes no GEMM: the tokens of PP 1, and its logits up to the CPU stand-ins of the unquantised ops, whose
    fp32 sums depend on how PP groups the rows. TP 2 quantises each rank's half of the o / down inputs with that
    half's own per-token scale: close to TP 1, not identical."""
    d = scratch_dir("gllm_b200_fp8_")
    write_channel(os.path.join(d, "m"), _tiny("Qwen3ForCausalLM", layers=4), seed=6)
    one = _mp(1, 1, 0, os.path.join(d, "m"))
    pp2 = _mp(2, 1, 29961, os.path.join(d, "m"))
    assert pp2[0] == one[0]
    assert float((_rows(pp2) - _rows(one)).abs().max()) < 1e-5
    tp2 = _mp(1, 2, 29951, os.path.join(d, "m"))
    x, y = tp2[1][0][1], one[1][0][1]
    assert float((x - y).norm() / y.norm()) < 0.05
