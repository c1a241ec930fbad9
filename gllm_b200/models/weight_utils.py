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
    if method in ("", "fp8"):
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
