"""AWQ / GPTQ checkpoint writers for tests: random int4 codes, zero points and 16-bit scales for the seven projections
of a dense decoder, written in each format's packing, next to the same model with the de-quantised weights. The
nibble orders here are written from the formats' definitions, independently of the package's readers:
  AWQ qweight [K, N/8] and qzeros [G, N/8]: nibble i of word [r, c] holds column 8 c + [0, 2, 4, 6, 1, 3, 5, 7][i];
  GPTQ qweight [K/8, N]: nibble i of word [r, n] holds row 8 r + i; GPTQ qzeros [G, N/8]: column 8 c + i, and a v1
  checkpoint ("gptq") stores z - 1."""
import json
import os

import torch

AWQ_ORDER = [0, 2, 4, 6, 1, 3, 5, 7]
MODS = {"q": "self_attn.q_proj", "k": "self_attn.k_proj", "v": "self_attn.v_proj", "o": "self_attn.o_proj",
        "gate": "mlp.gate_proj", "up": "mlp.up_proj", "down": "mlp.down_proj"}


def _word(nibbles):
    """8 ints in [0, 15] (nibble 0 first) -> one int32 word."""
    v = sum(int(x) << (4 * i) for i, x in enumerate(nibbles))
    return v - (1 << 32) if v >= 1 << 31 else v


def _pack(t: torch.Tensor, dim: int, order=range(8)) -> torch.Tensor:
    """uint8 codes -> int32 words packing 8 entries of `dim`: nibble i holds entry 8 c + order[i]."""
    t = t.to(torch.int64)
    if dim == 0:
        return _pack(t.t(), 1, order).t().contiguous()
    r, c = t.shape
    g = t.view(r, c // 8, 8)[:, :, list(order)]
    w = (g << (4 * torch.arange(8))).sum(-1)
    return torch.where(w >= 1 << 31, w - (1 << 32), w).to(torch.int32)


def pack_awq(codes_kn: torch.Tensor) -> torch.Tensor:
    return _pack(codes_kn, 1, AWQ_ORDER)


def pack_gptq_rows(codes_kn: torch.Tensor) -> torch.Tensor:
    return _pack(codes_kn, 0)


def pack_gptq_cols(zeros_gn: torch.Tensor) -> torch.Tensor:
    return _pack(zeros_gn, 1)


def shapes(cfg):
    h, i = cfg["hidden_size"], cfg["intermediate_size"]
    d = cfg.get("head_dim") or h // cfg["num_attention_heads"]
    q, kv = cfg["num_attention_heads"] * d, cfg["num_key_value_heads"] * d
    return {"q": (q, h), "k": (kv, h), "v": (kv, h), "o": (h, q), "gate": (i, h), "up": (i, h), "down": (h, i)}


def dequant(codes_nk, zeros_ng, scales_ng, group, dtype):
    """W [N, K] = dtype(fp32(s) · (q − z)), computed here in float64 (exact) and rounded once."""
    k = codes_nk.shape[1]
    gi = torch.arange(k) // group if group > 0 else torch.zeros(k, dtype=torch.long)
    w = scales_ng.double()[:, gi] * (codes_nk.double() - zeros_ng.double()[:, gi])
    return w.to(dtype)


def random_module(n, k, group, gen, scale_dtype=torch.float16, z_lo=0, z_hi=15):
    """Random codes [N, K], zeros [N, G] in [z_lo, z_hi] and scales [N, G] (weight std about 0.05)."""
    g = 1 if group == -1 else k // group
    codes = torch.randint(0, 16, (n, k), generator=gen, dtype=torch.uint8)
    zeros = torch.randint(z_lo, z_hi + 1, (n, g), generator=gen, dtype=torch.uint8)
    scales = (torch.rand(n, g, generator=gen) * 0.02 + 0.005).to(scale_dtype)
    return codes, zeros, scales


def quant_config(method, group, fmt="gptq", sym=False):
    if method == "awq":
        return {"quant_method": "awq", "bits": 4, "group_size": group, "zero_point": True, "version": "gemm"}
    return {"quant_method": "gptq", "bits": 4, "group_size": group, "desc_act": False, "sym": sym,
            "checkpoint_format": fmt}


def module_tensors(method, name, codes, zeros, scales, group, fmt="gptq", g_idx=True):
    """The checkpoint tensors of one quantised module `name` (codes [N, K], zeros [N, G], scales [N, G])."""
    out = {name + ".scales": scales.t().contiguous()}
    if method == "awq":
        out[name + ".qweight"] = pack_awq(codes.t().contiguous())
        out[name + ".qzeros"] = pack_awq(zeros.t().contiguous())
    else:
        z = zeros.t().to(torch.int64) - (1 if fmt == "gptq" else 0)
        assert int(z.min()) >= 0 and int(z.max()) <= 15
        out[name + ".qweight"] = pack_gptq_rows(codes.t().contiguous())
        out[name + ".qzeros"] = pack_gptq_cols(z.to(torch.uint8))
        if g_idx:
            k = codes.shape[1]
            out[name + ".g_idx"] = (torch.arange(k) // group if group > 0 else torch.zeros(k, dtype=torch.long)).to(
                torch.int32)
    return out


def write_pair(qdir, ddir, cfg, method, group, seed=0, fmt="gptq", sym=False, scale_dtype=torch.float16):
    """Write a W4A16 checkpoint of the HF config dict `cfg` to `qdir` and the same model with de-quantised weights (in
    the model dtype) to `ddir`. Unquantised tensors (embeddings, norms, biases, LM head) are the same in both."""
    from safetensors.torch import save_file
    dtype = {"float32": torch.float32, "bfloat16": torch.bfloat16, "float16": torch.float16}[cfg["torch_dtype"]]
    gen = torch.Generator().manual_seed(seed)
    h, v = cfg["hidden_size"], cfg["vocab_size"]
    arch = cfg["architectures"][0]
    dense, quant = {}, {}
    common = {"model.embed_tokens.weight": torch.randn(v, h, generator=gen) * 0.5,
              "model.norm.weight": 1 + 0.1 * torch.randn(h, generator=gen),
              "lm_head.weight": torch.randn(v, h, generator=gen) * 0.05}
    d = cfg.get("head_dim") or h // cfg["num_attention_heads"]
    z_lo = 1 if (method == "gptq" and fmt == "gptq") else 0
    z_hi = 16 if (method == "gptq" and fmt == "gptq") else 15
    for li in range(cfg["num_hidden_layers"]):
        pre = f"model.layers.{li}."
        common[pre + "input_layernorm.weight"] = 1 + 0.1 * torch.randn(h, generator=gen)
        common[pre + "post_attention_layernorm.weight"] = 1 + 0.1 * torch.randn(h, generator=gen)
        if arch == "Qwen3ForCausalLM":
            common[pre + "self_attn.q_norm.weight"] = 1 + 0.1 * torch.randn(d, generator=gen)
            common[pre + "self_attn.k_norm.weight"] = 1 + 0.1 * torch.randn(d, generator=gen)
        if arch == "Qwen2ForCausalLM":
            for m in ("q", "k", "v"):
                common[pre + MODS[m] + ".bias"] = 0.1 * torch.randn(shapes(cfg)[m][0], generator=gen)
        for m, (n, k) in shapes(cfg).items():
            codes, zeros, scales = random_module(n, k, group, gen, scale_dtype, z_lo, z_hi)
            if sym and method == "gptq":
                zeros.fill_(8)
            name = pre + MODS[m]
            quant.update(module_tensors(method, name, codes, zeros, scales, group, fmt))
            dense[name + ".weight"] = dequant(codes, zeros, scales, group, dtype)
    common = {k: t.to(dtype) for k, t in common.items()}
    for path, tensors, qc in ((qdir, {**common, **quant}, quant_config(method, group, fmt, sym)),
                              (ddir, {**common, **dense}, None)):
        os.makedirs(path, exist_ok=True)
        c = dict(cfg)
        if qc is not None:
            c["quantization_config"] = qc
        with open(os.path.join(path, "config.json"), "w") as f:
            json.dump(c, f)
        save_file({k: t.contiguous() for k, t in tensors.items()}, os.path.join(path, "model.safetensors"))
