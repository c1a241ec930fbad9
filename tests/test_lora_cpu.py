"""Multi-LoRA on the CPU: the PEFT loader (scale, padding, TP shards, refusals), greedy tokens against HuggingFace
models with the adapter merged into their weights (fp32), mixed adapter / base batches under every scheduling
feature, the prefix cache, TP2 / PP2 over gloo, and the OpenAI `model` routing."""
from conftest import scratch_dir
import json
import math
import os
import subprocess
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from lora_util import merged, scale_of, write_adapter  # noqa: E402

transformers = pytest.importorskip("transformers")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _qwen3(seed=0, layers=2):
    from transformers import Qwen3Config, Qwen3ForCausalLM
    torch.manual_seed(seed)
    cfg = Qwen3Config(hidden_size=128, intermediate_size=256, num_hidden_layers=layers, num_attention_heads=4,
                      num_key_value_heads=2, head_dim=32, vocab_size=512, max_position_embeddings=512, eos_token_id=1)
    return Qwen3ForCausalLM(cfg).eval().float()


def _save(model):
    d = scratch_dir("gllm_b200_lora_")
    model.save_pretrained(d, safe_serialization=True)
    return d


def _hf_greedy(model, prompt, n):
    with torch.no_grad():
        out = model.generate(torch.tensor([prompt]), max_new_tokens=n, do_sample=False, eos_token_id=None,
                             pad_token_id=0)
    return out[0, len(prompt):].tolist()


def _engine(path, lora_modules, **kw):
    from gllm_b200 import LLM
    args = dict(maxp=64, maxd=64, page_size=16, num_cpu_pages=96, model_max_length=320, log_stats=False,
                lora_modules=lora_modules, max_lora_rank=16)
    args.update(kw)
    return LLM(path, **args)


PROMPTS = [[5, 17, 99, 200, 3, 45, 7], [9] * 40, list(range(20, 150)), [300, 301]]


# ---------------------------------------------------------------------------------------------------------------
# loader
# ---------------------------------------------------------------------------------------------------------------
def _spec():
    from gllm_b200.models.decoder import ModelSpec
    return ModelSpec(arch="Qwen3ForCausalLM", hidden_size=128, num_layers=2, num_heads=4, num_kv_heads=2, head_dim=32,
                     intermediate_size=256, vocab_size=512, dtype=torch.float32)


_HF = dict(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2,
           head_dim=32)


@pytest.mark.parametrize("rslora", [False, True])
def test_loader_folds_scale_into_b_and_pads_to_max_rank(rslora):
    from gllm_b200.lora import load_adapter
    d = scratch_dir("gllm_b200_lora_")
    w = write_adapter(d, _HF, r=8, alpha=24, seed=3, rslora=rslora, default_segment=rslora)
    got = load_adapter(d, _spec(), 16)
    s = 24 / math.sqrt(8) if rslora else 24 / 8
    assert set(got) == set(w)
    for key, (a, b) in w.items():
        ga, gb = got[key]
        assert ga.shape == (16, a.shape[1]) and gb.shape == (b.shape[0], 16)
        assert torch.equal(ga[:8], a) and not ga[8:].any() and not gb[:, 8:].any()
        assert torch.allclose(gb[:, :8], b * s, rtol=1e-6, atol=0)


def _refuse(match, **kw):
    from gllm_b200.lora import load_adapter
    d = scratch_dir("gllm_b200_lora_")
    write_adapter(d, _HF, **kw)
    with pytest.raises(ValueError, match=match):
        load_adapter(d, _spec(), 16)


def test_loader_refusals():
    _refuse("DoRA", config_extra={"use_dora": True})
    _refuse("modules_to_save", config_extra={"modules_to_save": ["lm_head"]})
    _refuse("bias", config_extra={"bias": "all"})
    _refuse("fan_in_fan_out", config_extra={"fan_in_fan_out": True})
    _refuse("embed_tokens", config_extra={"target_modules": ["q_proj", "embed_tokens"]})
    _refuse("lm_head", config_extra={"target_modules": ["lm_head"]})
    _refuse("exceeds max_lora_rank", r=24)
    _refuse("has 2 layers", layers=[0, 2])
    _refuse("no self_attn.gate_proj", tensors_extra={
        "base_model.model.model.layers.0.self_attn.gate_proj.lora_A.weight": torch.zeros(8, 128)})
    _refuse("not a lora_A / lora_B", tensors_extra={"base_model.model.lm_head.lora_A.weight": torch.zeros(8, 128)})
    _refuse("has shape", tensors_extra={
        "base_model.model.model.layers.1.mlp.down_proj.lora_A.weight": torch.zeros(8, 128)}, mods=("q",))
    from gllm_b200.lora import adapter_ids, check_max_rank
    with pytest.raises(ValueError, match="max_lora_rank"):
        check_max_rank(128)
    d = scratch_dir("gllm_b200_lora_")
    write_adapter(d, _HF)
    with pytest.raises(ValueError, match="Qwen3MoeForCausalLM"):
        adapter_ids("Qwen3MoeForCausalLM", {"a": d}, 16)
    with pytest.raises(ValueError, match="DeepseekV3ForCausalLM"):
        adapter_ids("DeepseekV3ForCausalLM", {"a": d}, 16)


def test_engine_refuses_moe_architecture():
    from gllm_b200 import LLM
    from gllm_b200.models.presets import tiny
    d = scratch_dir("gllm_b200_lora_")
    write_adapter(d, _HF)
    cfg = tiny("Qwen3MoeForCausalLM", num_experts=4, num_experts_per_tok=2, moe_intermediate_size=64)
    with pytest.raises(ValueError, match="not supported for Qwen3MoeForCausalLM"):
        LLM(cfg, load_format="dummy", lora_modules={"a": d}, num_cpu_pages=32, log_stats=False)


class _Obj:
    def __init__(self, **kw):
        self.__dict__.update(kw)


@pytest.mark.parametrize("fused_act", [True, False])
def test_tp2_shards_are_slices_of_the_merged_delta(fused_act):
    """Each rank's B_r·A_r equals this rank's slice of s·B·A: rows of q/k/v and gate/up (interleaved per 128 for the
    fused SiLU-gate layout), columns of o and down."""
    from gllm_b200.lora import LoraStore
    from gllm_b200.models import weight_utils as wu
    from gllm_b200.ops import ref
    spec = _spec()
    d = scratch_dir("gllm_b200_lora_")
    w = write_adapter(d, _HF, r=8, alpha=16, seed=5)
    s = scale_of(8, 16)
    delta = {k: s * b @ a for k, (a, b) in w.items()}
    for tr in range(2):
        inter = 128
        layers = [_Obj(layer_id=i, attn=_Obj(q_size=64, kv_size=32), mlp=_Obj(inter=inter, fused_act=fused_act),
                       lora=None) for i in range(2)]
        model = _Obj(spec=spec, tp_size=2, tp_rank=tr, layers=layers)
        LoraStore({"a": d}, 16, model, "cpu")
        for lay in layers:
            t, li = lay.lora.t, lay.layer_id
            # q/k/v: column m of U is module m's A; B rows of this rank
            a3 = t["qkv_A"][0].reshape(3, 16, -1)
            b = t["qkv_B"][0]
            got = torch.cat([b[:64] @ a3[0], b[64:96] @ a3[1], b[96:] @ a3[2]])
            want = wu.shard_qkv(delta[(li, "q")], delta[(li, "k")], delta[(li, "v")], 4, 2, 32, tr, 2)
            assert torch.allclose(got, want, atol=1e-6)
            a2 = t["gate_up_A"][0].reshape(2, 16, -1)
            gu = wu.shard_gate_up(delta[(li, "gate")], delta[(li, "up")], tr, 2)
            if fused_act:
                gu = ref.interleave_gate_up(gu, 128)
            bb = t["gate_up_B"][0]
            gate_row = ((torch.arange(2 * inter) % 256) < 128) if fused_act else (torch.arange(2 * inter) < inter)
            got = torch.where(gate_row[:, None], bb @ a2[0], bb @ a2[1])
            assert torch.allclose(got, gu, atol=1e-6)
            for mod in ("o", "down"):
                got = t[mod + "_B"][0] @ t[mod + "_A"][0]
                assert torch.allclose(got, wu.shard_cols(delta[(li, mod)], tr, 2), atol=1e-6)


# ---------------------------------------------------------------------------------------------------------------
# against HF with merged weights
# ---------------------------------------------------------------------------------------------------------------
def _models():
    from transformers import LlamaConfig, LlamaForCausalLM, Qwen2Config, Qwen2ForCausalLM
    torch.manual_seed(1)
    llama = LlamaForCausalLM(LlamaConfig(hidden_size=128, intermediate_size=192, num_hidden_layers=2,
                                         num_attention_heads=4, num_key_value_heads=2, vocab_size=512,
                                         max_position_embeddings=512, eos_token_id=1)).eval().float()
    torch.manual_seed(2)
    qwen2 = Qwen2ForCausalLM(Qwen2Config(hidden_size=128, intermediate_size=256, num_hidden_layers=2,
                                         num_attention_heads=4, num_key_value_heads=2, vocab_size=512,
                                         max_position_embeddings=512, eos_token_id=1)).eval().float()
    for n, p in qwen2.named_parameters():
        if n.endswith("bias"):
            torch.nn.init.normal_(p, std=0.5)
    return {"qwen3": _qwen3(), "llama": llama, "qwen2": qwen2}


@pytest.mark.parametrize("arch", ["qwen3", "llama", "qwen2"])
def test_greedy_tokens_and_logprobs_match_hf_merged(arch):
    m = _models()[arch]
    d = _save(m)
    cfg = m.config.to_dict()
    ad = os.path.join(d, "adapter")
    w = write_adapter(ad, cfg, r=8, alpha=16, seed=11, rslora=arch == "llama")
    ref_model = merged(m, w, scale_of(8, 16, rslora=arch == "llama"))
    llm = _engine(d, {"ad": ad})
    outs = llm.generate(tokens=PROMPTS, output_lens=[10] * 4, ignore_eos=True, lora="ad", logprobs=0)
    for p, s in zip(PROMPTS, outs):
        assert s.token_ids[len(p):] == _hf_greedy(ref_model, p, 10), (arch, len(p))
        with torch.no_grad():
            lp = torch.log_softmax(ref_model(torch.tensor([s.token_ids])).logits[0].double(), -1)
        for i, (got, _) in enumerate(s.output_logprobs):
            want = float(lp[len(p) - 1 + i, s.token_ids[len(p) + i]])
            assert abs(got - want) < 1e-3, (arch, i, got, want)
    base = llm.generate(tokens=PROMPTS[:1], output_lens=[10], ignore_eos=True)
    assert base[0].token_ids[len(PROMPTS[0]):] == _hf_greedy(m, PROMPTS[0], 10)
    llm.shutdown()


# ---------------------------------------------------------------------------------------------------------------
# mixed batches
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def two_adapters():
    m = _qwen3(seed=7)
    d = _save(m)
    cfg = m.config.to_dict()
    write_adapter(os.path.join(d, "a"), cfg, r=8, alpha=16, seed=21)
    write_adapter(os.path.join(d, "b"), cfg, r=16, alpha=8, seed=22, mods=("q", "v", "down"))
    return d, {"a": os.path.join(d, "a"), "b": os.path.join(d, "b")}


MIX = [[5, 17, 99, 200, 3, 45, 7], list(range(20, 150)), [9] * 40, list(range(200, 260)), [300, 301], [7] * 19]
MIX_LORA = ["a", "b", None, "a", "b", None]


def _solo(d, mods):
    llm = _engine(d, mods, enable_prefix_caching=False)
    out = []
    for p, name in zip(MIX, MIX_LORA):
        s = llm.generate(tokens=[p], output_lens=[24], ignore_eos=True, lora=name, logprobs=0)[0]
        out.append(s.token_ids)
    llm.shutdown()
    return out


@pytest.fixture(scope="module")
def solo(two_adapters):
    return _solo(*two_adapters)


@pytest.mark.parametrize("case", ["plain", "chunked", "preempt", "sync", "n2", "plp"])
def test_mixed_batch_equals_solo_runs(two_adapters, solo, case):
    d, mods = two_adapters
    kw = dict(enable_prefix_caching=False)
    gen = dict(output_lens=[24] * len(MIX), ignore_eos=True, lora=MIX_LORA)
    if case == "chunked":
        kw.update(maxp=16)
    elif case == "preempt":
        kw.update(schedule_method="token_throttling", num_cpu_pages=12, kvthresh=0.0, maxp=32, maxd=8)
    elif case == "sync":
        kw.update(async_schedule=False)
    elif case == "n2":
        gen.update(n=2, temperature=0.0)
    elif case == "plp":
        gen.update(prompt_logprobs=1)
    llm = _engine(d, mods, **kw)
    outs = llm.generate(tokens=MIX, **gen)
    if case == "preempt":
        assert llm.worker.scheduler.num_preempt_seqs > 0
    llm.shutdown()
    per = 2 if case == "n2" else 1
    for i, want in enumerate(solo):
        for j in range(per):
            assert outs[i * per + j].token_ids == want, (case, i, j, MIX_LORA[i])
    if case == "plp":
        for s in outs:
            assert len(s.prompt_logprobs) == s.prompt_len


def test_prefix_cache_is_keyed_by_adapter(two_adapters, solo):
    d, mods = two_adapters
    llm = _engine(d, mods, enable_prefix_caching=True)
    p = MIX[1]
    mm = llm.worker.mm
    base = llm.generate(tokens=[p], output_lens=[24], ignore_eos=True)[0]
    h0 = mm.num_hit_pages
    a1 = llm.generate(tokens=[p], output_lens=[24], ignore_eos=True, lora="b")[0]
    assert mm.num_hit_pages == h0 and a1.num_cached_tokens == 0       # no hit on the base model's pages
    a2 = llm.generate(tokens=[p], output_lens=[24], ignore_eos=True, lora="b")[0]
    assert mm.num_hit_pages > h0 and a2.num_cached_tokens > 0          # the same adapter hits its own pages
    c = llm.generate(tokens=[p], output_lens=[24], ignore_eos=True, lora="a")[0]
    assert c.num_cached_tokens == 0                                     # ... and no other adapter's
    llm.shutdown()
    assert a1.token_ids == a2.token_ids == solo[1]
    assert base.token_ids != a1.token_ids
    cold = _engine(d, mods, enable_prefix_caching=False)
    assert cold.generate(tokens=[p], output_lens=[24], ignore_eos=True)[0].token_ids == base.token_ids
    assert cold.generate(tokens=[p], output_lens=[24], ignore_eos=True, lora="a")[0].token_ids == c.token_ids
    cold.shutdown()


def test_unknown_adapter_is_a_value_error(two_adapters):
    d, mods = two_adapters
    llm = _engine(d, mods)
    with pytest.raises(ValueError, match="unknown LoRA adapter"):
        llm.generate(tokens=MIX[:1], output_lens=[2], lora="zzz")
    llm.shutdown()
    plain = _engine(d, None)
    with pytest.raises(ValueError, match="without lora_modules"):
        plain.generate(tokens=MIX[:1], output_lens=[2], lora="a")
    plain.shutdown()


def test_batch_without_adapter_rows_has_no_lora_fields(two_adapters):
    from gllm_b200.input_data import BatchArrays
    d, mods = two_adapters
    llm = _engine(d, mods)
    seen = []
    runner = llm.worker.runner
    orig = runner.step

    def spy(batch, *a, **k):
        seen.append(batch)
        return orig(batch, *a, **k)
    runner.step = spy
    llm.generate(tokens=MIX[:2], output_lens=[3, 3], ignore_eos=True)
    llm.generate(tokens=MIX[:2], output_lens=[3, 3], ignore_eos=True, lora=["a", None])
    llm.shutdown()
    base = [b for b in seen if b.lora_slot is None]
    lora = [b for b in seen if b.lora_slot is not None]
    assert base and lora
    for b in base:
        hdr, _ = b.to_wire()
        assert "lora_slot" not in [a[0] for a in hdr["arrays"]]
    for b in lora:
        assert b.lora_slot.shape == (b.num_tokens,)
        back = BatchArrays.from_wire(*b.to_wire())
        assert (back.lora_slot == b.lora_slot).all()


# ---------------------------------------------------------------------------------------------------------------
# TP2 / PP2 over gloo
# ---------------------------------------------------------------------------------------------------------------
def _mp(pp, tp, port, d):
    out = os.path.join(scratch_dir("gllm_b200_lora_mp_"), "out.json")
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
    m = _qwen3(seed=9, layers=4)
    d = _save(m)
    cfg = m.config.to_dict()
    write_adapter(os.path.join(d, "a"), cfg, r=8, alpha=16, seed=31)
    write_adapter(os.path.join(d, "b"), cfg, r=16, alpha=16, seed=32, mods=("k", "o", "gate", "up"))
    one = _mp(1, 1, 0, d)
    assert _mp(1, 2, 29951, d) == one
    assert _mp(2, 1, 29961, d) == one


# ---------------------------------------------------------------------------------------------------------------
# OpenAI API
# ---------------------------------------------------------------------------------------------------------------
def _api_dir():
    from tokenizers import Tokenizer, models, pre_tokenizers
    from transformers import LlamaConfig, LlamaForCausalLM, PreTrainedTokenizerFast
    torch.manual_seed(0)
    words = ["<unk>", "<s>", "</s>", "<|user|>", "<|assistant|>"] + [f"w{i}" for i in range(200)] + ["hello", "world"]
    tok = Tokenizer(models.WordLevel({w: i for i, w in enumerate(words)}, unk_token="<unk>"))
    tok.pre_tokenizer = pre_tokenizers.Whitespace()
    fast = PreTrainedTokenizerFast(tokenizer_object=tok, unk_token="<unk>", bos_token="<s>", eos_token="</s>")
    fast.chat_template = "{% for m in messages %}<|{{ m['role'] }}|> {{ m['content'] }} {% endfor %}" \
                         "{% if add_generation_prompt %}<|assistant|> {% endif %}"
    cfg = LlamaConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=2,
                      num_key_value_heads=2, vocab_size=len(words), max_position_embeddings=256, eos_token_id=2)
    d = scratch_dir("gllm_b200_lora_api_")
    LlamaForCausalLM(cfg).eval().float().save_pretrained(d, safe_serialization=True)
    fast.save_pretrained(d)
    write_adapter(os.path.join(d, "ad"), cfg.to_dict(), r=8, alpha=32, seed=41, std=0.3)
    return d


def test_api_model_routing_and_models_list():
    pytest.importorskip("fastapi")
    from fastapi.testclient import TestClient
    from gllm_b200.engine.async_llm_engine import AsyncLLM
    from gllm_b200.entrypoints.api_server import build_app, make_parser, parse_lora_modules
    d = _api_dir()
    args = make_parser().parse_args(["--model-path", d, "--lora-modules", f"ad={d}/ad", "--max-lora-rank", "8"])
    assert parse_lora_modules(args.lora_modules) == {"ad": f"{d}/ad"} and args.max_lora_rank == 8
    body = {"prompt": "hello world w1 w2 w3", "max_tokens": 8, "temperature": 0, "top_k": 1, "ignore_eos": True}
    chat = {"messages": [{"role": "user", "content": "hello w5 w6"}], "max_tokens": 6, "temperature": 0, "top_k": 1,
            "ignore_eos": True}
    for with_lora in (False, True):
        eng = AsyncLLM(d, maxp=64, maxd=16, num_cpu_pages=64, model_max_length=128, log_stats=False,
                       lora_modules={"ad": f"{d}/ad"} if with_lora else None, max_lora_rank=8)
        with TestClient(build_app(eng)) as c:
            cards = c.get("/v1/models").json()["data"]
            base_text = c.post("/v1/completions", json={**body, "model": d}).json()["choices"][0]["text"]
            other = c.post("/v1/completions", json={**body, "model": "nope"})
            if not with_lora:
                assert [x["id"] for x in cards] == [d]
                assert other.status_code == 200 and other.json()["choices"][0]["text"] == base_text
                plain = base_text
            else:
                assert [x["id"] for x in cards] == [d, "ad"]
                assert cards[1]["root"] == f"{d}/ad" and cards[1]["parent"] == d
                assert base_text == plain
                assert other.status_code == 404 and other.json()["code"] == "model_not_found"
                assert c.post("/v1/chat/completions", json={**chat, "model": "nope"}).status_code == 404
                ad = c.post("/v1/completions", json={**body, "model": "ad"}).json()["choices"][0]["text"]
                assert ad != base_text
                # streamed: the same text
                r = c.post("/v1/completions", json={**body, "model": "ad", "stream": True})
                chunks = [json.loads(ln[6:]) for ln in r.text.splitlines()
                          if ln.startswith("data: ") and ln != "data: [DONE]"]
                assert "".join(ch["choices"][0]["text"] for ch in chunks if ch["choices"]) == ad
                cb = c.post("/v1/chat/completions", json={**chat, "model": "ad"}).json()
                cs = c.post("/v1/chat/completions", json={**chat, "model": "ad", "stream": True})
                parts = [json.loads(ln[6:]) for ln in cs.text.splitlines()
                         if ln.startswith("data: ") and ln != "data: [DONE]"]
                txt = "".join(p["choices"][0]["delta"].get("content") or "" for p in parts if p["choices"])
                assert txt == cb["choices"][0]["message"]["content"]
        eng.shutdown()
