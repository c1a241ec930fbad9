"""TP/EP/PP weight sharding helpers (reference: gllm/models/weight_utils.py:6-84) + a lazy
checkpoint reader that only touches the tensors (and row ranges) a rank actually needs — the
reference loads the whole checkpoint into host RAM on every worker (gllm/model_loader.py:41-85).
"""
from __future__ import annotations

import glob
import json
import os
from dataclasses import dataclass
from typing import Dict, List, Optional

import torch


# ------------------------------------------------------------------------------------------------
# pure sharding functions (also used by the round-trip tests)
# ------------------------------------------------------------------------------------------------
def shard_rows(w: torch.Tensor, rank: int, size: int) -> torch.Tensor:
    n = w.shape[0]
    assert n % size == 0, (n, size)
    s = n // size
    return w[rank * s:(rank + 1) * s]


def shard_cols(w: torch.Tensor, rank: int, size: int) -> torch.Tensor:
    n = w.shape[1]
    assert n % size == 0, (n, size)
    s = n // size
    return w[:, rank * s:(rank + 1) * s]


def kv_head_range(num_kv_heads: int, tp_rank: int, tp_size: int):
    """KV heads are split across TP ranks, or replicated when tp_size > num_kv_heads
    (reference: gllm/layers/linear.py:396-468)."""
    if num_kv_heads >= tp_size:
        assert num_kv_heads % tp_size == 0
        n = num_kv_heads // tp_size
        return tp_rank * n, n
    assert tp_size % num_kv_heads == 0
    return tp_rank // (tp_size // num_kv_heads), 1


def shard_qkv(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, num_heads: int, num_kv_heads: int,
              head_dim: int, tp_rank: int, tp_size: int) -> torch.Tensor:
    """HF q/k/v ([heads*D, H] or [heads*D] for biases) -> fused per-rank [(hq + 2 hkv)*D, ...]."""
    hq = num_heads // tp_size
    kv0, nkv = kv_head_range(num_kv_heads, tp_rank, tp_size)
    qs = q[tp_rank * hq * head_dim:(tp_rank + 1) * hq * head_dim]
    ks = k[kv0 * head_dim:(kv0 + nkv) * head_dim]
    vs = v[kv0 * head_dim:(kv0 + nkv) * head_dim]
    return torch.cat([qs, ks, vs], dim=0)


def shard_gate_up(gate: torch.Tensor, up: torch.Tensor, tp_rank: int, tp_size: int) -> torch.Tensor:
    return torch.cat([shard_rows(gate, tp_rank, tp_size), shard_rows(up, tp_rank, tp_size)], dim=0)


def pad_vocab(vocab_size: int, tp_size: int, multiple: int = 64) -> int:
    m = multiple * tp_size
    return (vocab_size + m - 1) // m * m


def shard_vocab(w: torch.Tensor, tp_rank: int, tp_size: int, multiple: int = 64) -> torch.Tensor:
    """Rows [V, H] -> this rank's padded vocab shard [Vp/tp, H] (zero padded)."""
    v, h = w.shape
    vp = pad_vocab(v, tp_size, multiple)
    per = vp // tp_size
    a, b = tp_rank * per, min((tp_rank + 1) * per, v)
    out = torch.zeros(per, h, dtype=w.dtype)
    if b > a:
        out[: b - a] = w[a:b]
    return out


def expert_range(num_experts: int, ep_rank: int, ep_size: int):
    """Contiguous block per rank, remainder to the last rank
    (reference: gllm/layers/moe/fused_moe_triton/layer.py:326-369)."""
    per = num_experts // ep_size
    start = ep_rank * per
    n = per if ep_rank < ep_size - 1 else num_experts - start
    return start, n


def fp8_block_quant(w: torch.Tensor):
    """[N, K] -> (e4m3 [N, K], fp32 scale_inv [ceil(N/128), ceil(K/128)]): 128x128 block quantisation, scale_inv =
    amax / 448 per block. Re-quantising the de-quantised tensor of an fp8 checkpoint is lossless as long as the
    blocks stay aligned (shard boundaries on block boundaries: head_dim 128, intermediate % 128 == 0)."""
    w = w.float()
    n, k = w.shape
    nb, kb = (n + 127) // 128, (k + 127) // 128
    wp = torch.zeros(nb * 128, kb * 128, dtype=torch.float32, device=w.device)
    wp[:n, :k] = w
    blk = wp.view(nb, 128, kb, 128)
    sc = (blk.abs().amax(dim=(1, 3)) / 448.0).clamp_min(1e-12)
    q = (blk / sc.view(nb, 1, kb, 1)).view(nb * 128, kb * 128)[:n, :k].to(torch.float8_e4m3fn)
    return q, sc


# ------------------------------------------------------------------------------------------------
# 4-bit AWQ / GPTQ checkpoints
# ------------------------------------------------------------------------------------------------
W4_MODULES = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")
W4_ARCHITECTURES = ("LlamaForCausalLM", "MistralForCausalLM", "Qwen2ForCausalLM", "Qwen3ForCausalLM")
AWQ_ORDER = (0, 2, 4, 6, 1, 3, 5, 7)   # AWQ: nibble i of a word holds column 8 c + AWQ_ORDER[i]


@dataclass
class W4Config:
    """A validated AWQ / GPTQ `quantization_config`: 4-bit codes, `group_size` input columns per scale (-1: the whole
    unsharded K), and `zero_offset` added to the stored zero points (1 for GPTQ v1 checkpoints)."""
    method: str
    group_size: int
    zero_offset: int = 0


def w4_config(qc: dict) -> Optional[W4Config]:
    """Parse `quantization_config`: None for an unquantised or fp8 checkpoint, a `W4Config` for a supported AWQ /
    GPTQ one; anything else raises ValueError naming the cause."""
    method = str(qc.get("quant_method", "")).lower() if qc else ""
    if method in ("", "fp8", "compressed-tensors"):
        return None
    if method not in ("awq", "gptq"):
        raise ValueError(f"quantization method {method!r} is not supported (supported: fp8, awq, gptq)")
    bits = qc.get("bits", qc.get("w_bit", 4))
    if bits != 4:
        raise ValueError(f"{method}: bits={bits} is not supported (only 4-bit weights)")
    g = qc.get("group_size", qc.get("q_group_size", 128))
    if g not in (32, 64, 128, -1):
        raise ValueError(f"{method}: group_size={g} is not supported (32, 64, 128 or -1)")
    skip = [m for m in (qc.get("modules_to_not_convert") or []) if any(p in m for p in W4_MODULES)]
    if skip:
        raise ValueError(f"{method}: modules_to_not_convert names quantised projections {skip}")
    if method == "awq":
        version = str(qc.get("version", "gemm")).lower()
        if version != "gemm":
            raise ValueError(f"awq: version={version!r} is not supported (only 'gemm')")
        if not qc.get("zero_point", True):
            raise ValueError("awq: zero_point=false is not supported")
        return W4Config("awq", g)
    if qc.get("desc_act", False):
        raise ValueError("gptq: desc_act=true (act-order) is not supported")
    fmt = qc.get("checkpoint_format", "gptq")
    if fmt not in ("gptq", "gptq_v2"):
        raise ValueError(f"gptq: checkpoint_format={fmt!r} is not supported ('gptq' or 'gptq_v2')")
    return W4Config("gptq", g, 1 if fmt == "gptq" else 0)


@dataclass
class W4Tensor:
    """One quantised linear in checkpoint orientation, whatever the format: codes uint8 [N, K], zeros uint8 [N, G]
    (with the format's offset applied), scales fp16/bf16 [N, G]."""
    codes: torch.Tensor
    zeros: torch.Tensor
    scales: torch.Tensor


def _nibbles(words: torch.Tensor) -> torch.Tensor:
    """int32 [..., W] -> uint8 [..., W, 8]: nibble i of each word at index i."""
    w = words.to(torch.int64) & 0xFFFFFFFF
    return ((w.unsqueeze(-1) >> (4 * torch.arange(8))) & 0xF).to(torch.uint8)


def unpack_awq(packed: torch.Tensor) -> torch.Tensor:
    """AWQ int32 [R, C/8] packed along columns -> uint8 [R, C]."""
    nib = _nibbles(packed)
    inv = torch.tensor([AWQ_ORDER.index(j) for j in range(8)])
    return nib[..., inv].reshape(packed.shape[0], -1)


def unpack_gptq_rows(packed: torch.Tensor) -> torch.Tensor:
    """GPTQ qweight int32 [K/8, N] packed along rows -> uint8 [K, N]."""
    return _nibbles(packed).permute(0, 2, 1).reshape(-1, packed.shape[1])


def unpack_gptq_cols(packed: torch.Tensor) -> torch.Tensor:
    """GPTQ qzeros int32 [G, N/8] packed along columns -> uint8 [G, N]."""
    return _nibbles(packed).reshape(packed.shape[0], -1)


def shard_cols_w4(w: W4Tensor, rank: int, size: int) -> W4Tensor:
    """Row-parallel shard of a quantised linear: this rank's K columns and their groups (with one group over the
    whole K, every rank keeps its zeros and scales)."""
    one = w.zeros.shape[1] == 1 and w.codes.shape[1] > 1
    return W4Tensor(shard_cols(w.codes, rank, size), w.zeros if one else shard_cols(w.zeros, rank, size),
                    w.scales if one else shard_cols(w.scales, rank, size))


# ------------------------------------------------------------------------------------------------
# FP8 W8A8 checkpoints: per-channel / per-tensor e4m3 weights, per-token or static e4m3 activations
# ------------------------------------------------------------------------------------------------
@dataclass
class W8Config:
    """A validated W8A8 configuration. `method`: "fp8" (HF per-tensor), "compressed-tensors" or "fp8-online" (a 16-bit
    checkpoint quantised per output channel at load); `static`: the checkpoint holds per-tensor `input_scale`s."""
    method: str
    static: bool = False


def w8_config(qc: dict, quantization: Optional[str] = None) -> Optional[W8Config]:
    """Parse `quantization_config` (and the engine's `quantization` option) into a `W8Config`: None when the checkpoint
    is not a per-channel / per-tensor FP8 one; a ValueError naming the cause for an FP8 configuration this engine
    cannot serve exactly."""
    method = str(qc.get("quant_method", "")).lower() if qc else ""
    if quantization is not None:
        if quantization != "fp8":
            raise ValueError(f"quantization={quantization!r} is not supported (None or 'fp8')")
        if qc:
            raise ValueError(f"quantization='fp8' needs an unquantised checkpoint; this one has a quantization_config "
                             f"({method or qc})")
        return W8Config("fp8-online")
    if method == "fp8":
        if qc.get("weight_block_size") is not None:     # block-scaled: de-quantised by `CheckpointReader.get`
            return None
        scheme = str(qc.get("activation_scheme", "dynamic")).lower()
        if scheme not in ("dynamic", "static"):
            raise ValueError(f"fp8: activation_scheme={scheme!r} is not supported ('dynamic' or 'static')")
        _check_ignore("fp8", qc.get("ignored_layers") or qc.get("modules_to_not_convert") or [])
        return W8Config("fp8", scheme == "static")
    if method != "compressed-tensors":
        return None
    fmt = qc.get("format")
    if fmt not in ("float-quantized", "naive-quantized"):
        raise ValueError(f"compressed-tensors: format={fmt!r} is not supported ('float-quantized' or "
                         f"'naive-quantized')")
    groups = qc.get("config_groups") or {}
    if len(groups) != 1:
        raise ValueError(f"compressed-tensors: {len(groups)} config groups (exactly one, targeting Linear)")
    grp = next(iter(groups.values()))
    if list(grp.get("targets") or []) != ["Linear"]:
        raise ValueError(f"compressed-tensors: targets={grp.get('targets')} is not supported (['Linear'])")
    w, a = grp.get("weights") or {}, grp.get("input_activations")
    if (w.get("num_bits"), str(w.get("type")), bool(w.get("symmetric", True))) != (8, "float", True):
        raise ValueError(f"compressed-tensors: weights {w} are not 8-bit symmetric float")
    if w.get("strategy") not in ("channel", "tensor"):
        raise ValueError(f"compressed-tensors: weight strategy={w.get('strategy')!r} is not supported ('channel' or "
                         f"'tensor')")
    if w.get("dynamic", False):
        raise ValueError("compressed-tensors: dynamic weight scales are not supported")
    if a is None:
        raise ValueError("compressed-tensors: weight-only FP8 (input_activations: null) is not supported")
    if (a.get("num_bits"), str(a.get("type"))) != (8, "float"):
        raise ValueError(f"compressed-tensors: input activations {a} are not 8-bit float")
    act = (a.get("strategy"), bool(a.get("dynamic")))
    if act not in (("token", True), ("tensor", False)):
        raise ValueError(f"compressed-tensors: input activation strategy={act[0]!r}, dynamic={act[1]} is not "
                         f"supported (token and dynamic, or tensor and static)")
    _check_ignore("compressed-tensors", qc.get("ignore") or [])
    if qc.get("kv_cache_scheme"):
        from gllm_b200.utils.logging import logger
        logger.info("compressed-tensors: kv_cache_scheme is ignored, the KV cache stays bf16")
    return W8Config("compressed-tensors", act == ("tensor", False))


def _check_ignore(method: str, names):
    skip = [m for m in names if any(p in m for p in W4_MODULES)]
    if skip:
        raise ValueError(f"{method}: the ignore list names quantised projections {skip}")


@dataclass
class W8Tensor:
    """One W8A8 linear in checkpoint orientation: codes e4m3 [N, K], scale fp32 [N] (per-tensor scales expanded to
    their rows), input_scale fp32 scalar tensor (static activations) or None."""
    codes: torch.Tensor
    scale: torch.Tensor
    input_scale: Optional[torch.Tensor] = None


def fuse_w8(parts, fuse) -> W8Tensor:
    """The W8Tensor of linears fused into one GEMM: `fuse` applied to their codes and to their scales (each keeps its
    rows' scale); the static input scale is the largest of theirs."""
    ins = [p.input_scale for p in parts]
    return W8Tensor(fuse(*(p.codes for p in parts)), fuse(*(p.scale for p in parts)),
                    None if ins[0] is None else torch.stack([t.reshape(()) for t in ins]).max())


def shard_cols_w8(w: W8Tensor, rank: int, size: int) -> W8Tensor:
    """Row-parallel shard: this rank's K columns, every output channel's full scale."""
    return W8Tensor(shard_cols(w.codes, rank, size), w.scale, w.input_scale)


# ------------------------------------------------------------------------------------------------
# checkpoint reader
# ------------------------------------------------------------------------------------------------
class CheckpointReader:
    """Maps tensor name -> file for a HuggingFace directory (`*.safetensors`, else `*.bin`) and
    reads tensors on demand. `prefixes` lets VL checkpoints resolve `model.` ->
    `model.language_model.` etc. (reference: weight_utils.get_tensor_from_dict)."""

    def __init__(self, path: str):
        self.path = path
        self._files: Dict[str, str] = {}
        self._handles = {}
        self._bin: Dict[str, torch.Tensor] = {}
        st = sorted(glob.glob(os.path.join(path, "*.safetensors")))
        if st:
            idx = os.path.join(path, "model.safetensors.index.json")
            if os.path.exists(idx):
                with open(idx) as f:
                    for k, v in json.load(f)["weight_map"].items():
                        self._files[k] = os.path.join(path, v)
            else:
                from safetensors import safe_open
                for fpath in st:
                    with safe_open(fpath, "pt", device="cpu") as f:
                        for k in f.keys():
                            self._files[k] = fpath
        else:
            for fpath in sorted(glob.glob(os.path.join(path, "*.bin"))):
                sd = torch.load(fpath, map_location="cpu", weights_only=True)
                self._bin.update(sd)

    @classmethod
    def from_state_dict(cls, sd: Dict[str, torch.Tensor]) -> "CheckpointReader":
        r = cls.__new__(cls)
        r.path, r._files, r._handles, r._bin = "<memory>", {}, {}, dict(sd)
        return r

    def keys(self):
        return list(self._files.keys()) + list(self._bin.keys())

    _ALIASES = (("model.", "model.language_model."), ("visual.", "model.visual."),
                ("lm_head.", "model.lm_head."), ("model.", "language_model.model."),
                ("lm_head.", "language_model.lm_head."))

    def resolve(self, name: str) -> Optional[str]:
        if name in self._files or name in self._bin:
            return name
        for a, b in self._ALIASES:
            if name.startswith(a):
                alt = b + name[len(a):]
                if alt in self._files or alt in self._bin:
                    return alt
        return None

    def has(self, name: str) -> bool:
        return self.resolve(name) is not None

    def _handle(self, fpath: str):
        h = self._handles.get(fpath)
        if h is None:
            from safetensors import safe_open
            h = safe_open(fpath, "pt", device="cpu")
            self._handles[fpath] = h
        return h

    def get_raw(self, name: str) -> torch.Tensor:
        key = self.resolve(name)
        if key is None:
            raise KeyError(f"tensor {name} not found in checkpoint {self.path}")
        if key in self._bin:
            return self._bin[key]
        return self._handle(self._files[key]).get_tensor(key)

    def get(self, name: str) -> torch.Tensor:
        """Tensor by name. Block-quantised fp8 weights (`<name>` e4m3 + `<name>_scale_inv` fp32 per
        128x128 block — DeepSeek-V3 / Qwen3-FP8 checkpoints, reference: gllm/layers/linear.py:68-112)
        are de-quantised to bf16 here unless the caller asks for the raw pair via `get_fp8`."""
        t = self.get_raw(name)
        if t.dtype in (torch.float8_e4m3fn, torch.float8_e5m2) and self.has(name + "_scale_inv"):
            s = self.get_raw(name + "_scale_inv").float()
            n, k = t.shape
            bn, bk = -(-n // s.shape[0]), -(-k // s.shape[1])
            full = s.repeat_interleave(bn, 0)[:n].repeat_interleave(bk, 1)[:, :k]
            return (t.float() * full).to(torch.bfloat16)
        return t

    def is_fp8(self, name: str) -> bool:
        key = self.resolve(name)
        if key is None or not self.has(name + "_scale_inv"):
            return False
        return self.get_raw(name).dtype == torch.float8_e4m3fn

    def get_fp8(self, name: str):
        """(e4m3 weight, fp32 scale_inv [ceil(N/128), ceil(K/128)])"""
        return self.get_raw(name), self.get_raw(name + "_scale_inv").float()

    def get_w4(self, module: str, cfg: W4Config) -> W4Tensor:
        """`<module>.qweight / .qzeros / .scales (/ .g_idx)` of an AWQ or GPTQ checkpoint -> `W4Tensor`."""
        qw, qz = self.get_raw(module + ".qweight"), self.get_raw(module + ".qzeros")
        scales = self.get_raw(module + ".scales")
        if cfg.method == "awq":
            codes = unpack_awq(qw).t()
            zeros = unpack_awq(qz)
        else:
            codes = unpack_gptq_rows(qw).t()
            zeros = unpack_gptq_cols(qz).to(torch.int32) + cfg.zero_offset
            k = codes.shape[1]
            if self.has(module + ".g_idx"):
                g_idx = self.get_raw(module + ".g_idx").to(torch.int64)
                want = torch.arange(k) // cfg.group_size if cfg.group_size > 0 else torch.zeros(k, dtype=torch.int64)
                if not torch.equal(g_idx, want):
                    raise ValueError(f"{module}: g_idx is not k // group_size (act-order GPTQ is not supported)")
        n, k = codes.shape
        groups = 1 if cfg.group_size == -1 else k // cfg.group_size
        if scales.shape != (groups, n) or zeros.shape != (groups, n) or scales.dtype not in (torch.float16,
                                                                                              torch.bfloat16):
            raise ValueError(f"{module}: scales {tuple(scales.shape)} {scales.dtype} / zeros {tuple(zeros.shape)} do "
                             f"not match {cfg.method} codes [{n}, {k}] with group_size {cfg.group_size}")
        return W4Tensor(codes.contiguous(), zeros.t().to(torch.uint8).contiguous(), scales.t().contiguous())

    def get_w8(self, module: str, cfg: W8Config) -> W8Tensor:
        """`<module>.weight` (+ `.weight_scale`, `.input_scale`) of a W8A8 checkpoint -> `W8Tensor`, codes byte for
        byte; for `quantization="fp8"` the 16-bit weight quantised per output channel (`ref.fp8_channel_quant`)."""
        w = self.get_raw(module + ".weight")
        if cfg.method == "fp8-online":
            from gllm_b200.ops.ref import fp8_channel_quant
            return W8Tensor(*fp8_channel_quant(w))
        if w.dtype != torch.float8_e4m3fn:
            raise ValueError(f"{module}.weight is {w.dtype}: {cfg.method} W8A8 needs e4m3 weights")
        n = w.shape[0]
        s = self.get_raw(module + ".weight_scale")
        if s.dtype not in (torch.float32, torch.bfloat16, torch.float16) or s.numel() not in (1, n):
            raise ValueError(f"{module}.weight_scale {tuple(s.shape)} {s.dtype}: expected one fp32 / bf16 scale per "
                             f"tensor or per output channel ({n})")
        scale = s.float().reshape(-1).expand(n).contiguous()
        ins = None
        if cfg.static:
            i = self.get_raw(module + ".input_scale")
            if i.numel() != 1:
                raise ValueError(f"{module}.input_scale {tuple(i.shape)}: a static activation scale is one scalar")
            ins = i.float().reshape(())
        return W8Tensor(w.contiguous(), scale, ins)

    def get_rows(self, name: str, start: int, end: int) -> torch.Tensor:
        key = self.resolve(name)
        if key is None:
            raise KeyError(f"tensor {name} not found in checkpoint {self.path}")
        if key in self._bin:
            return self._bin[key][start:end]
        return self._handle(self._files[key]).get_slice(key)[start:end]

    def get_cols(self, name: str, start: int, end: int) -> torch.Tensor:
        key = self.resolve(name)
        if key is None:
            raise KeyError(f"tensor {name} not found in checkpoint {self.path}")
        if key in self._bin:
            return self._bin[key][:, start:end]
        return self._handle(self._files[key]).get_slice(key)[:, start:end]
