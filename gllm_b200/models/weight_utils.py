"""TP/EP/PP weight sharding helpers (reference: gllm/models/weight_utils.py:6-84) + a lazy
checkpoint reader that only touches the tensors (and row ranges) a rank actually needs — the
reference loads the whole checkpoint into host RAM on every worker (gllm/model_loader.py:41-85).
"""
from __future__ import annotations

import glob
import json
import os
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
