"""Multi-LoRA serving: PEFT adapters loaded at engine start and applied per request in one batch.

An adapter is a PEFT directory (`adapter_config.json` + `adapter_model.safetensors`) with low-rank factors
A [r, K] and B [N, r] for some of the seven projections of the dense decoder (q, k, v, o, gate, up, down). A row of
a batch that uses adapter `a` computes y = x·Wᵀ + (x·A_aᵀ)·(s·B_a)ᵀ, with s = alpha / r (alpha / sqrt(r) with
rsLoRA). The scale is folded into B in fp32 before the cast to the model dtype, and every adapter is zero-padded to
the engine's `max_lora_rank` so one rank runs everywhere.

Device store (`LoraStore`): per layer and input group the adapters are stacked, A [L, m·R, K_local] and
B [L, N_local, R] for the m modules that read the same input (q/k/v: 3, gate/up: 2, o and down: 1). Sharding follows
the base weights: column-parallel q/k/v and gate/up keep A whole and take this rank's rows of B (gate/up B also in
the 128-row interleave of the fused SiLU-gate GEMM); row-parallel o and down take this rank's columns of A and keep B
whole, so the sum over ranks of each rank's partial delta is the full delta and no extra collective is needed.

Adapter ids: 0 is the base model, adapter i (in `lora_modules` order) has id i + 1 and device slot i.
"""
from __future__ import annotations

import json
import math
import os
import re
from typing import Dict, List, Optional, Tuple

import torch

from gllm_b200 import ops
from gllm_b200.models import weight_utils as wu
from gllm_b200.ops import ref

SUPPORTED_ARCHITECTURES = ("LlamaForCausalLM", "MistralForCausalLM", "Qwen2ForCausalLM", "Qwen3ForCausalLM")
MAX_LORA_RANK = 64
MODULES = ("q", "k", "v", "o", "gate", "up", "down")
_KEY = re.compile(r"^base_model\.model\.model\.layers\.(\d+)\.(self_attn|mlp)\.(q|k|v|o|gate|up|down)_proj"
                  r"\.lora_([AB])(?:\.default)?\.weight$")
_PARENT = {"q": "self_attn", "k": "self_attn", "v": "self_attn", "o": "self_attn",
           "gate": "mlp", "up": "mlp", "down": "mlp"}


def check_max_rank(max_lora_rank) -> int:
    if isinstance(max_lora_rank, bool) or not isinstance(max_lora_rank, int) or \
            not 8 <= max_lora_rank <= MAX_LORA_RANK or max_lora_rank % 8:
        raise ValueError(f"max_lora_rank must be a multiple of 8 in [8, {MAX_LORA_RANK}], got {max_lora_rank!r}")
    return max_lora_rank


def adapter_ids(architecture: str, lora_modules: Optional[Dict[str, str]], max_lora_rank: int) -> Dict[str, int]:
    """Validate the engine's adapter set before any weight is loaded -> {name: adapter id}."""
    if not lora_modules:
        return {}
    check_max_rank(max_lora_rank)
    if architecture not in SUPPORTED_ARCHITECTURES:
        raise ValueError(f"LoRA adapters are not supported for {architecture}: only the dense decoders "
                         f"{', '.join(SUPPORTED_ARCHITECTURES)}")
    ids = {}
    for i, (name, path) in enumerate(lora_modules.items()):
        if not isinstance(name, str) or not name:
            raise ValueError(f"LoRA adapter names must be non-empty strings, got {name!r}")
        read_config(path, max_lora_rank)
        ids[name] = i + 1
    return ids


def read_config(path: str, max_lora_rank: int) -> Tuple[int, float]:
    """-> (r, scale) of the PEFT adapter at `path`; ValueError for what this engine cannot serve."""
    f = os.path.join(path, "adapter_config.json")
    if not os.path.isfile(f):
        raise ValueError(f"{path}: no adapter_config.json")
    with open(f) as fh:
        cfg = json.load(fh)
    if cfg.get("use_dora"):
        raise ValueError(f"{path}: DoRA adapters (use_dora) are not supported")
    if cfg.get("modules_to_save"):
        raise ValueError(f"{path}: modules_to_save ({cfg['modules_to_save']}) is not supported")
    if cfg.get("bias", "none") != "none":
        raise ValueError(f"{path}: bias={cfg['bias']!r} is not supported (only 'none')")
    if cfg.get("fan_in_fan_out"):
        raise ValueError(f"{path}: fan_in_fan_out adapters are not supported")
    targets = cfg.get("target_modules") or []
    if isinstance(targets, str):
        targets = [] if targets == "all-linear" else [targets]
    for t in targets:
        if t.removesuffix("_proj") not in MODULES:
            raise ValueError(f"{path}: target module {t!r} is not supported (only the q/k/v/o/gate/up/down "
                             f"projections; not embeddings or lm_head)")
    r = int(cfg.get("r", 0))
    if r <= 0:
        raise ValueError(f"{path}: rank r={r} must be positive")
    if r > max_lora_rank:
        raise ValueError(f"{path}: rank r={r} exceeds max_lora_rank={max_lora_rank}")
    alpha = float(cfg.get("lora_alpha", r))
    scale = alpha / math.sqrt(r) if cfg.get("use_rslora") else alpha / r
    return r, scale


def module_shapes(spec) -> Dict[str, Tuple[int, int]]:
    """Full (unsharded) (N, K) of each projection."""
    h, d, i = spec.hidden_size, spec.head_dim, spec.intermediate_size
    q, kv = spec.num_heads * d, spec.num_kv_heads * d
    return {"q": (q, h), "k": (kv, h), "v": (kv, h), "o": (h, q), "gate": (i, h), "up": (i, h), "down": (h, i)}


def load_adapter(path: str, spec, max_lora_rank: int) -> Dict[Tuple[int, str], Tuple[torch.Tensor, torch.Tensor]]:
    """{(layer, module): (A fp32 [R, K], s·B fp32 [N, R])}, zero-padded to R = max_lora_rank."""
    r, scale = read_config(path, max_lora_rank)
    f = os.path.join(path, "adapter_model.safetensors")
    if not os.path.isfile(f):
        raise ValueError(f"{path}: no adapter_model.safetensors")
    from safetensors.torch import load_file
    tensors = load_file(f)
    shapes = module_shapes(spec)
    parts: Dict[Tuple[int, str], Dict[str, torch.Tensor]] = {}
    for key, t in tensors.items():
        m = _KEY.match(key)
        if m is None:
            raise ValueError(f"{path}: tensor {key!r} is not a lora_A / lora_B weight of a q/k/v/o/gate/up/down "
                             f"projection of a decoder layer")
        layer, parent, mod, ab = int(m.group(1)), m.group(2), m.group(3), m.group(4)
        if parent != _PARENT[mod]:
            raise ValueError(f"{path}: {key!r}: the model has no {parent}.{mod}_proj")
        if layer >= spec.num_layers:
            raise ValueError(f"{path}: {key!r}: the model has {spec.num_layers} layers")
        n, k = shapes[mod]
        want = (r, k) if ab == "A" else (n, r)
        if tuple(t.shape) != want:
            raise ValueError(f"{path}: {key!r} has shape {tuple(t.shape)}, expected {want} (r={r})")
        parts.setdefault((layer, mod), {})[ab] = t
    out = {}
    for (layer, mod), ab in parts.items():
        if set(ab) != {"A", "B"}:
            raise ValueError(f"{path}: layer {layer} {mod}_proj has lora_{next(iter(ab))} but not its partner")
        n, k = shapes[mod]
        a = torch.zeros(max_lora_rank, k, dtype=torch.float32)
        b = torch.zeros(n, max_lora_rank, dtype=torch.float32)
        a[:r] = ab["A"].float()
        b[:, :r] = ab["B"].float() * scale
        out[(layer, mod)] = (a, b)
    return out


class LoraLayer:
    """One decoder layer's stacked adapter weights on this rank, and the three ways the forward applies them."""

    def __init__(self, tensors: Dict[str, torch.Tensor], bounds: Dict[str, List[int]], fused_act: bool, device):
        self.t = tensors           # "<group>_A" [L, m·R, K_local], "<group>_B" [L, N_local, R]
        self.bounds = bounds       # group -> column offsets of its modules in the output
        self.fused_act = fused_act
        self.ops = ops.table(device)

    def add(self, group: str, csr, x: torch.Tensor, y: torch.Tensor):
        """y += delta of `group` (qkv, gate_up, o, down) for the adapter rows of input x, in place. `csr`: the batch's
        (slots, row offsets, rows, number of groups), `InputData.lora`."""
        u = self.ops.lora_shrink(x, self.t[group + "_A"], *csr)
        self.ops.lora_expand_add(y, u, self.t[group + "_B"], self.bounds[group], *csr)

    def silu_mul(self, csr, x: torch.Tensor, pre: torch.Tensor) -> torch.Tensor:
        """Interleaved gate/up pre-activations of the fused-act layout -> SiLU(gate + dg) · (up + du)."""
        u = self.ops.lora_shrink(x, self.t["gate_up_A"], *csr)
        return self.ops.lora_expand_silu_mul(pre, u, self.t["gate_up_B"], *csr)


class LoraStore:
    """Every adapter of the engine, resident on this rank's device for this pipeline stage's layers."""

    def __init__(self, lora_modules: Dict[str, str], max_lora_rank: int, model, device):
        spec = model.spec
        self.names = list(lora_modules)
        self.num_adapters = len(self.names)
        self.rank = max_lora_rank
        R = max_lora_rank
        tp, tr = model.tp_size, model.tp_rank
        d = spec.head_dim
        adapters = [load_adapter(lora_modules[n], spec, R) for n in self.names]
        shapes = module_shapes(spec)
        dt = spec.dtype
        self.nbytes = 0

        def pair(ad, layer, mod):
            if (layer, mod) in ad:
                return ad[(layer, mod)]
            n, k = shapes[mod]
            return torch.zeros(R, k), torch.zeros(n, R)

        for layer in model.layers:
            lid = layer.layer_id
            at, mlp = layer.attn, layer.mlp
            t = {k: [] for k in ("qkv_A", "qkv_B", "o_A", "o_B", "gate_up_A", "gate_up_B", "down_A", "down_B")}
            for ad in adapters:
                (aq, bq), (ak, bk), (av, bv) = (pair(ad, lid, m) for m in ("q", "k", "v"))
                t["qkv_A"].append(torch.cat([aq, ak, av]))
                t["qkv_B"].append(wu.shard_qkv(bq, bk, bv, spec.num_heads, spec.num_kv_heads, d, tr, tp))
                ao, bo = pair(ad, lid, "o")
                t["o_A"].append(wu.shard_cols(ao, tr, tp))
                t["o_B"].append(bo)
                (ag, bg), (au, bu) = pair(ad, lid, "gate"), pair(ad, lid, "up")
                t["gate_up_A"].append(torch.cat([ag, au]))
                b = wu.shard_gate_up(bg, bu, tr, tp)
                t["gate_up_B"].append(ref.interleave_gate_up(b, 128) if mlp.fused_act else b)
                adn, bdn = pair(ad, lid, "down")
                t["down_A"].append(wu.shard_cols(adn, tr, tp))
                t["down_B"].append(bdn)
            stacked = {k: torch.stack(v).to(device=device, dtype=dt).contiguous() for k, v in t.items()}
            self.nbytes += sum(x.numel() * x.element_size() for x in stacked.values())
            qs, kvs, inter = at.q_size, at.kv_size, mlp.inter
            bounds = {"qkv": [0, qs, qs + kvs, qs + 2 * kvs], "gate_up": [0, inter, 2 * inter],
                      "o": [0, spec.hidden_size], "down": [0, spec.hidden_size]}
            layer.lora = LoraLayer(stacked, bounds, mlp.fused_act, device)
