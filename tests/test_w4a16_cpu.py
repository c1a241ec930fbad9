"""4-bit AWQ / GPTQ checkpoints on the CPU: the formats' nibble orders, the loader's repack into the device layout and
its TP shards, every refusal, the op tables, and the engine on a W4A16 checkpoint against the engine on the same
model with de-quantised weights (bit for bit), with TP2 / PP2 over gloo and with LoRA adapters."""
from conftest import scratch_dir
import inspect
import json
import os
import subprocess
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from w4a16_util import (module_tensors, pack_awq, pack_gptq_cols, pack_gptq_rows, quant_config,  # noqa: E402
                        random_module, write_pair)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORD = torch.tensor([[0x76543210]], dtype=torch.int32)


# ---------------------------------------------------------------------------------------------------------------
# formats
# ---------------------------------------------------------------------------------------------------------------
def test_known_answer_nibble_orders():
    from gllm_b200.models import weight_utils as wu
    assert wu.unpack_awq(WORD).tolist() == [[0, 4, 1, 5, 2, 6, 3, 7]]
    assert wu.unpack_gptq_rows(WORD)[:, 0].tolist() == list(range(8))
    assert (wu.unpack_gptq_cols(WORD).int() + 1).tolist() == [list(range(1, 9))]
    # the test's own writers invert them
    codes = torch.arange(8, dtype=torch.uint8).view(1, 8)
    assert pack_awq(codes).tolist() == [[0x75316420]]
    assert pack_gptq_rows(codes.t()).tolist() == [[0x76543210]]
    assert pack_gptq_cols(codes).tolist() == [[0x76543210]]


@pytest.mark.parametrize("method,fmt,sym", [("awq", "gptq", False), ("gptq", "gptq", False),
                                            ("gptq", "gptq_v2", False), ("gptq", "gptq", True)])
def test_reader_decodes_each_format(method, fmt, sym):
    from gllm_b200.models import weight_utils as wu
    gen = torch.Generator().manual_seed(1)
    lo, hi = (1, 16) if (method, fmt) == ("gptq", "gptq") else (0, 15)
    codes, zeros, scales = random_module(48, 256, 64, gen, torch.bfloat16, lo, hi)
    if sym:
        zeros.fill_(8)      # symmetric GPTQ: stored 7 in a v1 checkpoint
    t = module_tensors(method, "m", codes, zeros, scales, 64, fmt)
    if sym:
        assert (t["m.qzeros"] == 0x77777777).all()
    w = wu.CheckpointReader.from_state_dict(t).get_w4("m", wu.w4_config(quant_config(method, 64, fmt, sym)))
    assert torch.equal(w.codes, codes) and torch.equal(w.zeros, zeros) and torch.equal(w.scales, scales)


@pytest.mark.parametrize("group", [32, 64, 128, -1])
@pytest.mark.parametrize("tp", [1, 2, 4])
def test_repacked_shards_unpack_to_exact_slices(group, tp):
    """Device layout after shard + repack -> exactly this rank's slice of the checkpoint's codes, zeros and scales,
    for a column-parallel (rows) and a row-parallel (columns) linear."""
    from gllm_b200.models import weight_utils as wu
    from gllm_b200.ops import ref
    gen = torch.Generator().manual_seed(group + tp)
    n, k = 320, 1024
    full = wu.W4Tensor(*random_module(n, k, group, gen))
    g = k if group == -1 else group
    full_wd = ref.w4a16_dequant(full.codes, full.zeros, full.scales, g, torch.float32)
    for r in range(tp):
        r0, r1, c0, c1 = r * n // tp, (r + 1) * n // tp, r * k // tp, (r + 1) * k // tp
        col = wu.W4Tensor(*(wu.shard_rows(t, r, tp) for t in (full.codes, full.zeros, full.scales)))
        for w, rows, cols in ((wu.shard_cols_w4(full, r, tp), slice(0, n), (c0, c1)), (col, slice(r0, r1), (0, k))):
            kk = cols[1] - cols[0]
            h = ref.Int4Weight(*ref.w4a16_pack(w.codes, w.zeros, w.scales), g if group > 0 else kk, kk)
            codes, zeros, scales = ref.w4a16_unpack(h)
            assert torch.equal(codes, full.codes[rows, cols[0]:cols[1]])
            gs = slice(0, 1) if group == -1 else slice(cols[0] // g, cols[1] // g)
            assert torch.equal(zeros, full.zeros[rows, gs]) and torch.equal(scales, full.scales[rows, gs])
            wd = ref.w4a16_dequant(codes, zeros, scales, h.group_size, torch.float32)
            assert torch.equal(wd, full_wd[rows, cols[0]:cols[1]])


# ---------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("change,match", [
    ({"bits": 8}, "bits=8"),
    ({"version": "gemv"}, "version"),
    ({"zero_point": False}, "zero_point"),
    ({"quant_method": "gptq", "desc_act": True}, "desc_act"),
    ({"quant_method": "compressed-tensors"}, "compressed-tensors"),
    ({"quant_method": "bitsandbytes"}, "bitsandbytes"),
    ({"modules_to_not_convert": ["model.layers.0.mlp.down_proj"]}, "modules_to_not_convert"),
    ({"group_size": 96}, "group_size"),
    ({"quant_method": "gptq", "checkpoint_format": "marlin"}, "checkpoint_format"),
])
def test_unsupported_configs_are_refused(change, match):
    from gllm_b200.models import registry
    from gllm_b200.models.presets import tiny
    cfg = tiny("Qwen3ForCausalLM", quantization_config=dict(quant_config("awq", 64), **change))
    with pytest.raises(ValueError, match=match):
        registry.build_model(registry.HFConfig(cfg), "cpu")


@pytest.mark.parametrize("arch", ["MixtralForCausalLM", "Qwen2MoeForCausalLM", "Qwen3MoeForCausalLM",
                                  "DeepseekV3ForCausalLM", "ChatGLMModel", "Qwen2_5_VLForConditionalGeneration"])
def test_other_architectures_are_refused(arch):
    from gllm_b200.models import registry
    from gllm_b200.models.presets import tiny
    cfg = tiny(arch, quantization_config=quant_config("awq", 64))
    with pytest.raises(ValueError, match=arch):
        registry.build_model(registry.HFConfig(cfg), "cpu")


def test_act_order_g_idx_is_refused():
    from gllm_b200.models import weight_utils as wu
    gen = torch.Generator().manual_seed(2)
    t = module_tensors("gptq", "m", *random_module(16, 128, 32, gen, z_lo=1, z_hi=16), 32)
    t["m.g_idx"] = t["m.g_idx"].flip(0)
    with pytest.raises(ValueError, match="g_idx"):
        wu.CheckpointReader.from_state_dict(t).get_w4("m", wu.w4_config(quant_config("gptq", 32)))


def test_row_parallel_width_not_a_multiple_of_the_group_is_refused(monkeypatch):
    """tiny: o_proj K = 4 heads x 32 = 128, so at tp 2 each rank holds 64 columns: not a multiple of g = 128."""
    from gllm_b200.models import registry
    from gllm_b200.models.presets import tiny
    from gllm_b200.parallel import state as ps
    monkeypatch.setattr(ps.get_state(), "tp_size", 2)
    cfg = tiny("Qwen3ForCausalLM", quantization_config=quant_config("awq", 128))
    with pytest.raises(ValueError, match="not a multiple of group_size 128"):
        registry.build_model(registry.HFConfig(cfg), "cpu")


def test_cpu_stand_in_has_the_kernel_signature():
    from gllm_b200.ops import cpu, sm100
    assert inspect.signature(cpu.linear_w4a16) == inspect.signature(sm100.linear_w4a16)


def test_awq_preset_builds_with_the_dummy_weight_spread():
    from gllm_b200.models import registry
    from gllm_b200.models.decoder import _qw
    from gllm_b200.models.presets import PRESETS
    from gllm_b200.ops import ref
    cfg = dict(PRESETS["qwen3-8b-awq"], num_hidden_layers=1, vocab_size=1024)
    model = registry.build_model(registry.HFConfig(cfg), "cpu")
    assert model.spec.quant == "awq" and model.spec.dtype == torch.bfloat16
    model.init_dummy()
    at = model.layers[0].attn
    h = _qw(at.qkv_w, at.qkv_ws)
    assert h.scales.dtype == torch.float16 and h.packed.shape == (6144, 4096 // 8)
    wd = ref.w4a16_dequant(*ref.w4a16_unpack(h), h.group_size, torch.float32)
    assert abs(float(wd.std()) - 0.02) < 0.002, float(wd.std())


# ---------------------------------------------------------------------------------------------------------------
# the engine: W4A16 checkpoint == the de-quantised checkpoint, bit for bit
# ---------------------------------------------------------------------------------------------------------------
PROMPTS = [[5, 17, 99, 200, 3, 45, 7], [9] * 40, list(range(20, 150)), [300, 301]]


def _pair(arch, method, group, fmt="gptq", layers=2, seed=0):
    from gllm_b200.models.presets import tiny
    d = scratch_dir("gllm_b200_w4_")
    cfg = tiny(arch, num_hidden_layers=layers)
    write_pair(os.path.join(d, "q"), os.path.join(d, "d"), cfg, method, group, seed=seed, fmt=fmt)
    return os.path.join(d, "q"), os.path.join(d, "d"), cfg


def _run(path, monkeypatch, lora_modules=None, lora=None):
    from gllm_b200 import LLM
    monkeypatch.setenv("GLLM_KEEP_LOGITS", "1")
    llm = LLM(path, device="cpu", num_cpu_pages=96, maxp=64, maxd=16, model_max_length=320, log_stats=False,
              lora_modules=lora_modules, max_lora_rank=16)
    outs = llm.generate(tokens=PROMPTS, output_lens=[6] * len(PROMPTS), ignore_eos=True, lora=lora)
    logits = [(ids, lg.clone()) for ids, lg in llm.worker.runner.logit_log]
    llm.shutdown()
    return [o.token_ids for o in outs], logits


@pytest.mark.parametrize("arch,method,group,fmt", [
    ("LlamaForCausalLM", "awq", 128, "gptq"),
    ("Qwen2ForCausalLM", "awq", 32, "gptq"),
    ("Qwen3ForCausalLM", "awq", -1, "gptq"),
    ("LlamaForCausalLM", "gptq", 64, "gptq"),
    ("Qwen2ForCausalLM", "gptq", 128, "gptq_v2"),
    ("Qwen3ForCausalLM", "gptq", 32, "gptq"),
])
def test_engine_matches_the_dequantised_checkpoint_bit_for_bit(arch, method, group, fmt, monkeypatch):
    q, d, _ = _pair(arch, method, group, fmt)
    tq, lq = _run(q, monkeypatch)
    td, ld = _run(d, monkeypatch)
    assert tq == td
    assert len(lq) == len(ld) and all(a[0] == b[0] and torch.equal(a[1], b[1]) for a, b in zip(lq, ld))


def test_lora_on_the_int4_base_equals_lora_on_the_dequantised_base(monkeypatch):
    from lora_util import write_adapter
    q, d, cfg = _pair("Qwen3ForCausalLM", "awq", 64, seed=4)
    a = os.path.join(os.path.dirname(q), "a")
    write_adapter(a, cfg, r=8, alpha=16, seed=5)
    lora = ["a", None, "a", "a"]
    tq, lq = _run(q, monkeypatch, {"a": a}, lora)
    td, ld = _run(d, monkeypatch, {"a": a}, lora)
    assert tq == td
    assert all(torch.equal(x[1], y[1]) for x, y in zip(lq, ld))


def _mp(pp, tp, port, d):
    out = os.path.join(scratch_dir("gllm_b200_w4_mp_"), "out.json")
    env = dict(os.environ, PYTHONPATH=ROOT, GLLM_B200_LOG="WARNING")
    script = os.path.join(ROOT, "tests", "mp_lora.py")
    if pp * tp == 1:
        cmd = [sys.executable, script, "1", "1", out, d]
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={pp * tp}",
               "--master-addr", "127.0.0.1", "--master-port", str(port), script, str(pp), str(tp), out, d]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, env=env, cwd=ROOT)
    assert r.returncode == 0 and os.path.exists(out), r.stdout[-2000:] + r.stderr[-3000:]
    with open(out) as f:
        return json.load(f)


def test_tp2_and_pp2_give_the_tokens_of_tp1():
    """A GPTQ checkpoint (group 32, so the row-parallel shards keep whole groups) with two adapters, through
    tests/mp_lora.py: mixed adapter / base batches under chunked prefill."""
    from lora_util import write_adapter
    q, _, cfg = _pair("Qwen3ForCausalLM", "gptq", 32, layers=4, seed=6)
    write_adapter(os.path.join(q, "a"), cfg, r=8, alpha=16, seed=31)
    write_adapter(os.path.join(q, "b"), cfg, r=16, alpha=16, seed=32, mods=("k", "o", "gate", "up"))
    one = _mp(1, 1, 0, q)
    assert _mp(1, 2, 29971, q) == one
    assert _mp(2, 1, 29981, q) == one
