"""FP8 W8A8 checkpoint writers for tests: the seven projections of a dense decoder as e4m3 codes with per-tensor or
per-channel scales, in the HF `fp8` and the `compressed-tensors` layouts, and a 16-bit checkpoint next to the
`compressed-tensors` channel checkpoint that the online rule makes of it. The rules are written here from the formats'
definitions, independently of the package's readers:
  HF fp8 (per-tensor): `<m>.weight` e4m3 [N, K], `<m>.weight_scale` fp32 [], `<m>.input_scale` fp32 [] when static;
  compressed-tensors: `<m>.weight` e4m3 [N, K], `<m>.weight_scale` [N, 1] (channel) or [1] (tensor);
  online: s[n] = max(amax_k |w[n, k]|, 1e-12) / 448, codes = e4m3_rn(w / s)."""
import json
import os

import torch

from w4a16_util import MODS, shapes

E4M3 = torch.float8_e4m3fn


def random_codes(n, k, gen):
    """e4m3 [N, K] spread over the whole range (std about 100, |q| <= 448)."""
    return (torch.randn(n, k, generator=gen) * 100.0).clamp(-448.0, 448.0).to(E4M3)


def online_rule(w):
    wf = w.float()
    s = torch.clamp(wf.abs().amax(1), min=1e-12) / 448.0
    return torch.clamp(wf / s[:, None], -448.0, 448.0).to(E4M3), s


def hf_config(static=False):
    return {"quant_method": "fp8", "activation_scheme": "static" if static else "dynamic"}


def ct_config(strategy="channel", static=False, **group_changes):
    act = {"num_bits": 8, "type": "float", "symmetric": True, "strategy": "tensor" if static else "token",
           "dynamic": not static}
    grp = {"targets": ["Linear"], "input_activations": act,
           "weights": {"num_bits": 8, "type": "float", "symmetric": True, "strategy": strategy, "dynamic": False}}
    grp.update(group_changes)
    return {"quant_method": "compressed-tensors", "format": "float-quantized", "config_groups": {"group_0": grp},
            "ignore": ["lm_head"]}


def _common(cfg, gen, dtype):
    h, v = cfg["hidden_size"], cfg["vocab_size"]
    d = cfg.get("head_dim") or h // cfg["num_attention_heads"]
    arch = cfg["architectures"][0]
    t = {"model.embed_tokens.weight": torch.randn(v, h, generator=gen) * 0.5,
         "model.norm.weight": 1 + 0.1 * torch.randn(h, generator=gen),
         "lm_head.weight": torch.randn(v, h, generator=gen) * 0.05}
    for li in range(cfg["num_hidden_layers"]):
        pre = f"model.layers.{li}."
        t[pre + "input_layernorm.weight"] = 1 + 0.1 * torch.randn(h, generator=gen)
        t[pre + "post_attention_layernorm.weight"] = 1 + 0.1 * torch.randn(h, generator=gen)
        if arch == "Qwen3ForCausalLM":
            t[pre + "self_attn.q_norm.weight"] = 1 + 0.1 * torch.randn(d, generator=gen)
            t[pre + "self_attn.k_norm.weight"] = 1 + 0.1 * torch.randn(d, generator=gen)
        if arch == "Qwen2ForCausalLM":
            for m in ("q", "k", "v"):
                t[pre + MODS[m] + ".bias"] = 0.1 * torch.randn(shapes(cfg)[m][0], generator=gen)
    return {k: x.to(dtype) for k, x in t.items()}


def _save(path, cfg, tensors, qc):
    from safetensors.torch import save_file
    os.makedirs(path, exist_ok=True)
    c = dict(cfg)
    if qc is not None:
        c["quantization_config"] = qc
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(c, f)
    save_file({k: t.contiguous() for k, t in tensors.items()}, os.path.join(path, "model.safetensors"))


def modules(cfg, gen, per_channel, static):
    """{checkpoint module name: (codes, scale fp32 [N] or [], input_scale fp32 [] or None)}"""
    out = {}
    for li in range(cfg["num_hidden_layers"]):
        for m, (n, k) in shapes(cfg).items():
            codes = random_codes(n, k, gen)
            scale = (torch.rand(n if per_channel else (), generator=gen) * 3e-4 + 1e-4).float()
            ins = (torch.rand((), generator=gen) * 0.01 + 0.005).float() if static else None
            out[f"model.layers.{li}." + MODS[m]] = (codes, scale, ins)
    return out


def write_tensor_pair(hf_dir, ct_dir, cfg, seed=0, static=False):
    """The same per-tensor codes and scales as an HF `fp8` and a compressed-tensors `tensor` checkpoint."""
    gen = torch.Generator().manual_seed(seed)
    common = _common(cfg, gen, torch.bfloat16)
    hf, ct = dict(common), dict(common)
    mods = modules(cfg, gen, False, static)
    for name, (codes, scale, ins) in mods.items():
        hf[name + ".weight"], ct[name + ".weight"] = codes, codes
        hf[name + ".weight_scale"], ct[name + ".weight_scale"] = scale.reshape(()), scale.reshape(1)
        if static:
            hf[name + ".input_scale"], ct[name + ".input_scale"] = ins.reshape(()), ins.reshape(1)
    _save(hf_dir, cfg, hf, hf_config(static))
    _save(ct_dir, cfg, ct, ct_config("tensor", static))
    return mods


def write_channel(ct_dir, cfg, seed=0, scale_dtype=torch.float32):
    gen = torch.Generator().manual_seed(seed)
    t = _common(cfg, gen, torch.bfloat16)
    mods = modules(cfg, gen, True, False)
    for name, (codes, scale, _) in mods.items():
        t[name + ".weight"] = codes
        t[name + ".weight_scale"] = scale.to(scale_dtype).reshape(-1, 1)
    _save(ct_dir, cfg, t, ct_config("channel"))
    return mods


def write_online_pair(bf16_dir, ct_dir, cfg, seed=0):
    """A bf16 checkpoint, and the compressed-tensors `channel` checkpoint the online rule makes of it."""
    gen = torch.Generator().manual_seed(seed)
    common = _common(cfg, gen, torch.bfloat16)
    dense, ct = dict(common), dict(common)
    for li in range(cfg["num_hidden_layers"]):
        for m, (n, k) in shapes(cfg).items():
            name = f"model.layers.{li}." + MODS[m]
            w = (torch.randn(n, k, generator=gen) * 0.02).to(torch.bfloat16)
            codes, s = online_rule(w)
            dense[name + ".weight"] = w
            ct[name + ".weight"], ct[name + ".weight_scale"] = codes, s.reshape(-1, 1)
    _save(bf16_dir, cfg, dense, None)
    _save(ct_dir, cfg, ct, ct_config("channel"))
