"""PEFT-format LoRA adapters with random non-zero A and B for tests (PEFT itself starts B at zero), and the merged
reference model W + s·B·A."""
import copy
import json
import math
import os

import torch

MODS = ("q", "k", "v", "o", "gate", "up", "down")
_PARENT = {"q": "self_attn", "k": "self_attn", "v": "self_attn", "o": "self_attn",
           "gate": "mlp", "up": "mlp", "down": "mlp"}


def shapes(cfg):
    h, i = cfg["hidden_size"], cfg["intermediate_size"]
    d = cfg.get("head_dim") or h // cfg["num_attention_heads"]
    q, kv = cfg["num_attention_heads"] * d, cfg["num_key_value_heads"] * d
    return {"q": (q, h), "k": (kv, h), "v": (kv, h), "o": (h, q), "gate": (i, h), "up": (i, h), "down": (h, i)}


def write_adapter(path, cfg, r=8, alpha=16, seed=0, mods=MODS, layers=None, rslora=False, std=0.05,
                  default_segment=False, config_extra=None, tensors_extra=None):
    """Write a PEFT adapter directory for the HF config dict `cfg` -> {(layer, module): (A [r, K], B [N, r])}."""
    from safetensors.torch import save_file
    os.makedirs(path, exist_ok=True)
    g = torch.Generator().manual_seed(seed)
    sh = shapes(cfg)
    layers = range(cfg["num_hidden_layers"]) if layers is None else layers
    weights, tensors = {}, {}
    seg = ".default" if default_segment else ""
    for li in layers:
        for m in mods:
            n, k = sh[m]
            a = torch.randn(r, k, generator=g) * std
            b = torch.randn(n, r, generator=g) * std
            weights[(li, m)] = (a, b)
            pre = f"base_model.model.model.layers.{li}.{_PARENT[m]}.{m}_proj.lora_"
            tensors[pre + "A" + seg + ".weight"] = a.contiguous()
            tensors[pre + "B" + seg + ".weight"] = b.contiguous()
    tensors.update(tensors_extra or {})
    conf = {"peft_type": "LORA", "r": r, "lora_alpha": alpha, "use_rslora": rslora, "bias": "none",
            "target_modules": [m + "_proj" for m in mods], "fan_in_fan_out": False, "use_dora": False,
            "modules_to_save": None}
    conf.update(config_extra or {})
    with open(os.path.join(path, "adapter_config.json"), "w") as f:
        json.dump(conf, f)
    save_file(tensors, os.path.join(path, "adapter_model.safetensors"))
    return weights


def scale_of(r, alpha, rslora=False):
    return alpha / math.sqrt(r) if rslora else alpha / r


def merged(model, weights, scale):
    """A copy of the HF model with W + scale·B·A in every adapted projection."""
    m = copy.deepcopy(model)
    with torch.no_grad():
        for (li, mod), (a, b) in weights.items():
            lin = getattr(getattr(m.model.layers[li], _PARENT[mod]), mod + "_proj")
            lin.weight += scale * (b.double() @ a.double()).to(lin.weight.dtype)
    return m
