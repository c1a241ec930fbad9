"""Pure-PyTorch reference implementations of every op (CPU-capable).

These are the correctness oracle for the sm_90a kernels (tests compare against them in
fp32) and the execution path for the CPU plumbing tests (BASELINE config #1: scheduler +
paged-KV on CPU). They are NOT a product path: on a GPU box the engine always runs the
hand-written kernels in `gllm_b200.ops.sm100`.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F


def kv_slab(head_dim: int) -> int:
    """Width of the innermost KV-cache slab (64 on the product path)."""
    return 64 if head_dim % 64 == 0 else head_dim


def kv_cache_shape(num_pages: int, num_kv_heads: int, head_dim: int, page_size: int):
    w = kv_slab(head_dim)
    return (num_pages, num_kv_heads, head_dim // w, page_size, w)


def check_copy_pairs(pairs, num_pages: int, dummy_page: Optional[int] = None):
    """Validate (src, dst) page pairs of `kv_copy_pages` on the host: every page in [0, num_pages), the dst pages
    distinct, no dst page also a src page (the copies of one launch run in any order), neither the dummy page."""
    src = [int(s) for s, _ in pairs]
    dst = [int(d) for _, d in pairs]
    for p in src + dst:
        if not 0 <= p < num_pages:
            raise ValueError(f"kv_copy_pages: page {p} outside [0, {num_pages})")
        if dummy_page is not None and p == dummy_page:
            raise ValueError("kv_copy_pages: the dummy page is neither copied nor overwritten")
    if len(set(dst)) != len(dst):
        raise ValueError("kv_copy_pages: dst pages must be distinct")
    if set(dst) & set(src):
        raise ValueError("kv_copy_pages: a dst page is also a src page")


def kv_copy_pages(tensors, pairs, dummy_page: Optional[int] = None):
    """PyTorch model of csrc/elemwise/kv_copy.cu: for every page-major cache tensor, page dst := page src."""
    if len(pairs) == 0:
        return
    check_copy_pairs(pairs, tensors[0].shape[0], dummy_page)
    src = torch.tensor([int(s) for s, _ in pairs], dtype=torch.long)
    dst = torch.tensor([int(d) for _, d in pairs], dtype=torch.long)
    for t in tensors:
        t[dst.to(t.device)] = t[src.to(t.device)]


# ----------------------------------------------------------------------------------------------
# dense ops
# ----------------------------------------------------------------------------------------------
def rmsnorm(x: torch.Tensor, w: torch.Tensor, eps: float, residual: Optional[torch.Tensor] = None):
    """Returns (normed, new_residual). new_residual is None when residual is None."""
    if residual is not None:
        r = (x.float() + residual.float()).to(x.dtype)
        xf = r.float()
    else:
        r = None
        xf = x.float()
    var = xf.pow(2).mean(-1, keepdim=True)
    out = (xf * torch.rsqrt(var + eps) * w.float()).to(x.dtype)
    return out, r


def linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    return F.linear(x, w, bias)


def silu_and_mul(x: torch.Tensor) -> torch.Tensor:
    d = x.shape[-1] // 2
    return (F.silu(x[..., :d].float()) * x[..., d:].float()).to(x.dtype)


def interleave_gate_up(w: torch.Tensor, block: int = 128) -> torch.Tensor:
    """[2I, K] (gate rows then up rows) -> per-`block` interleaved layout used by the fused
    SiLU-gate GEMM epilogue: tile j = [gate[j*b:(j+1)*b]; up[j*b:(j+1)*b]]."""
    two_i, k = w.shape
    i = two_i // 2
    assert i % block == 0, (i, block)
    g = w[:i].reshape(i // block, block, k)
    u = w[i:].reshape(i // block, block, k)
    return torch.cat([g, u], dim=1).reshape(two_i, k).contiguous()


def moe_gate_up_block(inter: int) -> int:
    """Rows per gate / up block of the MoE experts' w13 [E, 2I, H]: 64, the SiLU-gate tile of the grouped GEMM (which
    needs I % 64 == 0); any other I, which only the CPU runs, keeps one block: the plain [gate; up] layout."""
    return 64 if inter % 64 == 0 else inter


def linear_silu_mul(x: torch.Tensor, w_interleaved: torch.Tensor, block: int = 128) -> torch.Tensor:
    y = F.linear(x, w_interleaved)
    t, two_i = y.shape
    y = y.reshape(t, two_i // (2 * block), 2, block)
    return (F.silu(y[:, :, 0].float()) * y[:, :, 1].float()).to(x.dtype).reshape(t, two_i // 2)


def embedding(ids: torch.Tensor, table: torch.Tensor, vocab_start: int = 0, vocab_end: Optional[int] = None):
    vocab_end = table.shape[0] + vocab_start if vocab_end is None else vocab_end
    mask = (ids >= vocab_start) & (ids < vocab_end)
    local = torch.where(mask, ids - vocab_start, torch.zeros_like(ids)).long()
    out = F.embedding(local, table)
    out = out * mask.unsqueeze(-1).to(out.dtype)
    return out


# ----------------------------------------------------------------------------------------------
# rope + kv cache write
# ----------------------------------------------------------------------------------------------
def build_cos_sin_cache(rot_dim: int, max_pos: int, base: float, inv_freq: Optional[torch.Tensor] = None,
                        mscale: float = 1.0) -> torch.Tensor:
    """fp32 [max_pos, rot_dim]: cos | sin."""
    if inv_freq is None:
        inv_freq = 1.0 / (base ** (torch.arange(0, rot_dim, 2, dtype=torch.float32) / rot_dim))
    t = torch.arange(max_pos, dtype=torch.float32)
    freqs = torch.outer(t, inv_freq.float())
    return torch.cat([freqs.cos() * mscale, freqs.sin() * mscale], dim=-1).contiguous()


def _rope_one(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, rot: int, neox: bool) -> torch.Tensor:
    # x [T, H, D] fp32; cos/sin [T, rot/2]
    xr, xp = x[..., :rot], x[..., rot:]
    c, s = cos.unsqueeze(1), sin.unsqueeze(1)
    if neox:
        x1, x2 = xr[..., : rot // 2], xr[..., rot // 2:]
        o = torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], dim=-1)
    else:
        x1, x2 = xr[..., 0::2], xr[..., 1::2]
        o = torch.stack([x1 * c - x2 * s, x2 * c + x1 * s], dim=-1).flatten(-2)
    return torch.cat([o, xp], dim=-1)


def write_kv_cache(k: torch.Tensor, v: Optional[torch.Tensor], k_cache: torch.Tensor,
                   v_cache: Optional[torch.Tensor], slots: torch.Tensor):
    """k/v [T, Hkv, D]; caches [pages, Hkv, D/W, page, W]; slots [T] (negative = skip)."""
    pages, hkv, nslab, page_size, w = k_cache.shape
    valid = slots >= 0
    if not bool(valid.all()):
        k, slots_v = k[valid], slots[valid]
        v = v[valid] if v is not None else None
    else:
        slots_v = slots
    page = (slots_v // page_size).long()
    off = (slots_v % page_size).long()
    t = k.shape[0]
    k_cache[page, :, :, off, :] = k.reshape(t, hkv, nslab, w).to(k_cache.dtype)
    if v is not None and v_cache is not None:
        v_cache[page, :, :, off, :] = v.reshape(t, hkv, nslab, w).to(v_cache.dtype)


def rope_kv_write(q: torch.Tensor, k: torch.Tensor, v: Optional[torch.Tensor], positions: torch.Tensor,
                  cos_sin: Optional[torch.Tensor], rot_dim: int, neox: bool,
                  q_norm_w: Optional[torch.Tensor], k_norm_w: Optional[torch.Tensor], eps: float,
                  k_cache: Optional[torch.Tensor], v_cache: Optional[torch.Tensor],
                  slots: Optional[torch.Tensor], mrope_section=None):
    """In place on q [T,Hq,D] and k [T,Hkv,D] (views allowed): optional per-head RMSNorm, RoPE,
    then K/V scatter into the paged cache."""
    dt = q.dtype
    qf, kf = q.float(), k.float()
    if q_norm_w is not None:
        qf = (qf * torch.rsqrt(qf.pow(2).mean(-1, keepdim=True) + eps) * q_norm_w.float()).to(dt).float()
    if k_norm_w is not None:
        kf = (kf * torch.rsqrt(kf.pow(2).mean(-1, keepdim=True) + eps) * k_norm_w.float()).to(dt).float()
    if rot_dim > 0 and cos_sin is not None:
        half = rot_dim // 2
        if mrope_section is not None and positions.dim() == 2:
            # positions [3, T]; pair index i picks the section's position row
            sec = torch.zeros(half, dtype=torch.long, device=positions.device)
            if len(mrope_section) > 3 and mrope_section[3]:   # interleaved THWTHW.. (Qwen3-VL)
                sec[1:mrope_section[1] * 3:3] = 1
                sec[2:mrope_section[2] * 3:3] = 2
            else:
                s0, s1 = mrope_section[0], mrope_section[1]
                sec[s0:s0 + s1] = 1
                sec[s0 + s1:] = 2
            cs = cos_sin.to(positions.device)[positions.long()]  # [3, T, rot]
            idx = sec.view(1, 1, half).expand(1, positions.shape[1], half)
            cos = torch.gather(cs[..., :half], 0, idx)[0]
            sin = torch.gather(cs[..., half:], 0, idx)[0]
        else:
            pos = positions if positions.dim() == 1 else positions[0]
            cs = cos_sin.to(pos.device)[pos.long()]
            cos, sin = cs[..., :half], cs[..., half:]
        qf = _rope_one(qf, cos, sin, rot_dim, neox)
        kf = _rope_one(kf, cos, sin, rot_dim, neox)
    q.copy_(qf.to(dt))
    k.copy_(kf.to(dt))
    if k_cache is not None and slots is not None:
        write_kv_cache(k, v, k_cache, v_cache, slots)


# ----------------------------------------------------------------------------------------------
# paged attention
# ----------------------------------------------------------------------------------------------
def gather_kv(cache: torch.Tensor, block_row: torch.Tensor, seq_len: int) -> torch.Tensor:
    """-> [seq_len, Hkv, D]"""
    pages, hkv, nslab, page_size, w = cache.shape
    n_pages = (seq_len + page_size - 1) // page_size
    blk = cache[block_row[:n_pages].long()]  # [n, Hkv, nslab, page, W]
    blk = blk.permute(0, 3, 1, 2, 4).reshape(n_pages * page_size, hkv, nslab * w)
    return blk[:seq_len]


def paged_attention(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, block_table: torch.Tensor,
                    seq_lens: torch.Tensor, query_start_loc: torch.Tensor, scale: float,
                    num_q_heads: int, head_dim: int) -> torch.Tensor:
    """q [T, Hq*D] -> out [T, Hq*D]. Causal with context offset (chunked prefill / prefix cache):
    query i of a sequence sits at absolute position (seq_len - q_len + i)."""
    t = q.shape[0]
    hq, d = num_q_heads, head_dim
    hkv = k_cache.shape[1]
    g = hq // hkv
    out = torch.zeros(t, hq * d, dtype=q.dtype, device=q.device)
    qsl = query_start_loc.tolist()
    sl = seq_lens.tolist()
    for s in range(len(sl)):
        q0, q1 = qsl[s], qsl[s + 1]
        ql = q1 - q0
        if ql <= 0:
            continue
        kk = gather_kv(k_cache, block_table[s], sl[s]).float()  # [L, Hkv, D]
        vv = gather_kv(v_cache, block_table[s], sl[s]).float()
        qq = q[q0:q1].reshape(ql, hq, d).float()
        kk = kk.repeat_interleave(g, dim=1)
        vv = vv.repeat_interleave(g, dim=1)
        att = torch.einsum("qhd,khd->hqk", qq, kk) * scale
        ctx = sl[s] - ql
        qi = torch.arange(ql, device=q.device).view(ql, 1) + ctx
        kj = torch.arange(sl[s], device=q.device).view(1, sl[s])
        att = att.masked_fill((kj > qi).unsqueeze(0), float("-inf"))
        p = torch.softmax(att, dim=-1)
        o = torch.einsum("hqk,khd->qhd", p, vv)
        out[q0:q1] = o.reshape(ql, hq * d).to(q.dtype)
    return out


def varlen_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, cu_seqlens: torch.Tensor,
                     scale: float, causal: bool) -> torch.Tensor:
    """Non-paged varlen attention (ViT towers, MLA prefill). q [T,H,Dq] k [T,Hk,Dq] v [T,Hk,Dv]."""
    out = torch.empty(q.shape[0], q.shape[1], v.shape[-1], dtype=q.dtype, device=q.device)
    cs = cu_seqlens.tolist()
    g = q.shape[1] // k.shape[1]
    for i in range(len(cs) - 1):
        a, b = cs[i], cs[i + 1]
        if b <= a:
            continue
        qq, kk, vv = q[a:b].float(), k[a:b].float(), v[a:b].float()
        if g > 1:
            kk, vv = kk.repeat_interleave(g, 1), vv.repeat_interleave(g, 1)
        att = torch.einsum("qhd,khd->hqk", qq, kk) * scale
        if causal:
            n = b - a
            m = torch.triu(torch.ones(n, n, dtype=torch.bool, device=q.device), 1)
            att = att.masked_fill(m.unsqueeze(0), float("-inf"))
        out[a:b] = torch.einsum("hqk,khd->qhd", torch.softmax(att, -1), vv).to(q.dtype)
    return out


# ----------------------------------------------------------------------------------------------
# sampling
# ----------------------------------------------------------------------------------------------
_M32 = 0xFFFFFFFF


def _hash_u32(x):
    """csrc/sample/sampler.cu:hash_u32 on uint64 numpy arrays holding uint32 values (products wrap mod 2^64, whose
    low 32 bits are the uint32 product)."""
    x = x ^ (x >> 16)
    x = (x * 0x7feb352d) & _M32
    x = x ^ (x >> 15)
    x = (x * 0x846ca68b) & _M32
    return x ^ (x >> 16)


def race_uniform(seed: int, row: int, tokens) -> "np.ndarray":
    """Bit-exact port of the uniform inside csrc/sample/sampler.cu:rand_exp — u in (0, 1), float32, for the
    exponential race keyed (seed, row, token id). A seeded request row uses (its seed, position of the token being
    produced); the kernel's exponential variate is -log(u) (fast-math log, so that part agrees to rounding only)."""
    import numpy as np
    seed = int(seed) & ((1 << 64) - 1)
    lo, hi = seed & _M32, seed >> 32
    t = np.asarray(tokens, dtype=np.int64).astype(np.uint64) & _M32
    a = _hash_u32(np.asarray([(int(row) * 0x9E3779B9 + 0x85ebca6b) & _M32], dtype=np.uint64))
    h = _hash_u32((t + ((hi * 0xc2b2ae35) & _M32)) & _M32)
    h = _hash_u32(np.uint64(lo) ^ a ^ h)
    h = _hash_u32(h ^ 0x27d4eb2f)
    return (((h >> 8).astype(np.float32) + np.float32(0.5)) * np.float32(1.0 / 16777216.0)).astype(np.float32)


def race_exp(seed: int, row: int, tokens) -> torch.Tensor:
    """Exponential variates of the seeded race (float32): -log of `race_uniform`."""
    return -torch.log(torch.from_numpy(race_uniform(seed, row, tokens)))


def _seeded_exp(probs_shape, generator, seeds, seed_pos, tokens=None) -> torch.Tensor:
    """Exp(1) variates [B, n]: from `generator` for unseeded rows, from the seeded race for rows with seed_pos >= 0
    (`tokens` [B, n] token id of each column; default: the column index)."""
    b, n = probs_shape
    g = torch.empty(b, n).exponential_(1.0, generator=generator)
    if seeds is not None:
        for r in range(b):
            pos = int(seed_pos[r])
            if pos >= 0:
                tk = tokens[r].cpu().numpy() if tokens is not None else range(n)
                g[r] = race_exp(int(seeds[r]), pos, list(tk))
    return g


def apply_penalty_temperature(logits: torch.Tensor, temperature, rep_penalty, seen_mask, bias=None) -> torch.Tensor:
    """`bias`: optional dense fp32 [B, V] additive term (frequency / presence penalties and logit_bias), added after
    the repetition penalty and before the temperature, as the kernel does."""
    x = logits.float().clone()
    if rep_penalty is not None and seen_mask is not None:
        pen = rep_penalty.view(-1, 1).float()
        x = torch.where(seen_mask, torch.where(x > 0, x / pen, x * pen), x)
    if bias is not None:
        x = x + bias.float()
    if temperature is not None:
        t = temperature.float().clone()
        t[t <= 1e-5] = 1.0
        x = x / t.view(-1, 1)
    return x


def sample_filter(logits: torch.Tensor, temperature=None, top_k=None, top_p=None, rep_penalty=None,
                  seen_mask=None, bias=None) -> torch.Tensor:
    """Returns the filtered probability distribution [B, V] the sampler draws from
    (reference semantics: gllm/layers/sampler.py:22-54)."""
    x = apply_penalty_temperature(logits, temperature, rep_penalty, seen_mask, bias)
    b, v = x.shape
    if top_k is not None:
        k = top_k.clone().long()
        k[(k <= 0) | (k > v)] = v
        srt, _ = torch.sort(x, dim=-1, descending=True)
        thr = srt.gather(1, (k - 1).view(-1, 1))
        x = x.masked_fill(x < thr, float("-inf"))
    if top_p is not None:
        probs = torch.softmax(x, dim=-1)
        sp, si = torch.sort(probs, dim=-1, descending=True)
        cum = sp.cumsum(-1)
        # keep the smallest prefix whose mass reaches top_p
        drop = (cum - sp) >= top_p.view(-1, 1).float()
        drop_orig = torch.zeros_like(drop).scatter(1, si, drop)
        x = x.masked_fill(drop_orig, float("-inf"))
    return torch.softmax(x, dim=-1)


def sample(logits: torch.Tensor, temperature=None, top_k=None, top_p=None, rep_penalty=None,
           seen_mask=None, generator: Optional[torch.Generator] = None, bias=None, seeds=None,
           seed_pos=None) -> torch.Tensor:
    """`seeds` / `seed_pos` (int64 / int32 [B]): rows with seed_pos >= 0 draw from the seeded race (`race_exp`), so
    their token depends on their logits alone, whatever the batch."""
    b, v = logits.shape
    greedy = top_k is None or bool((top_k == 1).all())
    if greedy:
        x = apply_penalty_temperature(logits, temperature, rep_penalty, seen_mask, bias)
        return x.argmax(-1).to(torch.int32)
    probs = sample_filter(logits, temperature, top_k, top_p, rep_penalty, seen_mask, bias)
    g = _seeded_exp(probs.shape, generator, seeds, seed_pos)
    tok = (probs / g).argmax(-1)
    # rows with top_k == 1 are exactly greedy
    return tok.to(torch.int32)


def vp_candidates(shard: torch.Tensor, valid: int, v_full: int, c: int, temperature=None, top_k=None, top_p=None,
                  rep_penalty=None, seen_mask=None, race_exp: Optional[torch.Tensor] = None,
                  vocab_offset: int = 0, bias=None) -> torch.Tensor:
    """PyTorch model of csrc/sample/sampler.cu:vp_candidates_kernel — per-row record [B, 2c+4]: the shard's c best
    candidates after penalty / temperature (values, then token ids bit-cast to float), shard max, shard sum-exp, and
    for unfiltered rows the shard's exponential-race winner (score relative to the shard max, token id).
    `seen_mask` / `race_exp` / `bias` are [B, valid] slices for this shard."""
    b = shard.shape[0]
    out = torch.full((b, 2 * c + 4), float("-inf"), dtype=torch.float32)
    out[:, c:2 * c] = 0.0
    out[:, 2 * c + 1] = 0.0
    out[:, 2 * c + 3] = 0.0
    if valid <= 0:
        return out
    x = apply_penalty_temperature(shard[:, :valid], temperature, rep_penalty, seen_mask, bias)
    m = x.max(dim=-1).values
    out[:, 2 * c] = m
    out[:, 2 * c + 1] = torch.exp(x - m.view(-1, 1)).sum(-1)
    ck = min(c, valid)
    vals, idx = torch.topk(x, ck, dim=-1)
    out[:, :ck] = vals
    out[:, c:c + ck] = (idx + vocab_offset).to(torch.int32).view(torch.float32)
    k = top_k.long() if top_k is not None else torch.ones(b, dtype=torch.long)
    k = torch.where((k <= 0) | (k > v_full), torch.full_like(k, v_full), k)
    p = top_p.float() if top_p is not None else torch.ones(b)
    free = (k >= v_full) & (p >= 1.0)
    if bool(free.any()) and race_exp is not None:
        score = (x - m.view(-1, 1)) - torch.log(race_exp[:, :valid])
        best, bi = score.max(dim=-1)
        out[free, 2 * c + 2] = best[free]
        out[free, 2 * c + 3] = (bi[free] + vocab_offset).to(torch.int32).view(torch.float32)
    return out


def vp_final(gathered: torch.Tensor, c: int, v_full: int, top_k=None, top_p=None,
             generator: Optional[torch.Generator] = None, seeds=None, seed_pos=None) -> torch.Tensor:
    """PyTorch model of vp_final_kernel: finish top-k / top-p / draw on the gathered candidates [tp, B, 2c+4] with
    the exact global normalisation (the mass of non-candidate tokens is known from the per-shard sum-exp)."""
    tp, b, _ = gathered.shape
    vals = gathered[:, :, :c].permute(1, 0, 2).reshape(b, tp * c)
    toks = gathered[:, :, c:2 * c].contiguous().view(torch.int32).permute(1, 0, 2).reshape(b, tp * c).long()
    ms, zs = gathered[:, :, 2 * c], gathered[:, :, 2 * c + 1]
    gm = ms.max(dim=0).values
    gz = (zs * torch.exp(torch.where(zs > 0, ms - gm.view(1, -1), torch.zeros_like(ms)))).sum(0)
    n = tp * c
    k = top_k.long() if top_k is not None else torch.ones(b, dtype=torch.long)
    k = torch.where((k <= 0) | (k > v_full), torch.full_like(k, v_full), k)
    p = top_p.float() if top_p is not None else torch.ones(b)
    out = torch.zeros(b, dtype=torch.int32)
    e_all = torch.empty(b, n).exponential_(1.0, generator=generator)
    for r in range(b):
        seeded = seeds is not None and int(seed_pos[r]) >= 0
        if k[r] >= v_full and p[r] >= 1.0:
            sc = gathered[:, r, 2 * c + 2] + (ms[:, r] - gm[r])
            out[r] = gathered[int(sc.argmax()), r, 2 * c + 3].view(torch.int32)
            continue
        x, t = vals[r], toks[r]
        order = torch.argsort(x, descending=True, stable=True)
        x, t = x[order], t[order]
        e_r = race_exp(int(seeds[r]), int(seed_pos[r]), t.tolist()) if seeded else e_all[r]
        kk = int(min(k[r], n))
        if kk == 1:
            out[r] = t[0]
            continue
        prob = torch.exp(x - gm[r])
        keep = torch.zeros(n, dtype=torch.bool)
        keep[:kk] = True
        keep &= x >= x[kk - 1]
        keep |= (x == x[kk - 1]) & (x > float("-inf"))      # ties at the threshold survive (as in the kernel)
        mass = prob[keep].sum() if kk < v_full else gz[r]
        if p[r] < 1.0:
            cum = torch.cumsum(torch.where(keep, prob, torch.zeros_like(prob)), 0)
            keep &= (cum - prob) < p[r] * mass
        keep &= x > float("-inf")
        score = torch.where(keep, torch.log(prob) - torch.log(e_r), torch.full_like(prob, float("-inf")))
        out[r] = t[int(score.argmax())]
    return out


def bias_rebuild(bias: torch.Tensor, out_seen: torch.Tensor, slot: int, freq: float, pres: float, lb_ids, lb_vals,
                 out_toks):
    """PyTorch model of bias_rebuild_kernel for one slot: clear, scatter logit_bias, replay the output tokens' counts
    in order with the fp32 operations of bias_account."""
    bias[slot] = 0.0
    out_seen[slot] = 0
    if len(lb_ids):
        bias[slot, torch.as_tensor(lb_ids, dtype=torch.long)] = torch.as_tensor(lb_vals, dtype=torch.float32)
    for tok in out_toks:
        bias_account_one(bias, out_seen, slot, int(tok), freq, pres)


def bias_account_one(bias: torch.Tensor, out_seen: torch.Tensor, slot: int, tok: int, freq: float, pres: float):
    """PyTorch model of bias_account_kernel for one row: bias[slot, tok] -= f (+ p on the first occurrence)."""
    w, bit = tok >> 5, 1 << (tok & 31)
    word = int(out_seen[slot, w]) & _M32
    first = (word & bit) == 0
    new = word | bit
    out_seen[slot, w] = new - (1 << 32) if new >= 1 << 31 else new     # int32 storage of the uint32 word
    f, p = torch.tensor(freq, dtype=torch.float32), torch.tensor(pres, dtype=torch.float32)
    bias[slot, tok] = bias[slot, tok] - ((f + p) if first else f)


LP_NO_TOKEN = 0x7fffffff   # token id of an empty candidate slot in a log-prob record


def logprobs_shard(logits: torch.Tensor, valid: int, n: int, tokens: torch.Tensor,
                   rows: Optional[torch.Tensor] = None, vocab_offset: int = 0) -> torch.Tensor:
    """PyTorch model of csrc/sample/sampler.cu:logprobs_shard_kernel — per requesting row a record [E, 2n+3]: the
    shard's n largest raw logits (lower token id first on ties), their token ids bit-cast to float, shard max, shard
    sum-exp, and the raw logit of the sampled token if this shard holds it (-inf otherwise)."""
    x_all = logits if rows is None else logits[rows.long()]
    toks = tokens if rows is None else tokens[rows.long()]
    e = x_all.shape[0]
    out = torch.full((e, 2 * n + 3), float("-inf"), dtype=torch.float32, device=logits.device)
    ids = out.view(torch.int32)
    ids[:, n:2 * n] = LP_NO_TOKEN
    out[:, 2 * n + 1] = 0.0
    if valid <= 0 or e == 0:
        return out
    x = x_all[:, :valid].float()
    m = x.max(dim=-1).values
    finite = m > float("-inf")
    out[:, 2 * n] = m
    out[:, 2 * n + 1] = torch.where(finite, torch.exp(x - torch.where(finite, m, 0.0).view(-1, 1)).sum(-1), 0.0)
    local = toks.long() - vocab_offset
    mine = (local >= 0) & (local < valid)
    chosen = x.gather(1, local.clamp(0, valid - 1).view(-1, 1))[:, 0]
    out[:, 2 * n + 2] = torch.where(mine, chosen, float("-inf"))
    k = min(n, valid)
    if k:
        vals, idx = torch.sort(x, dim=-1, descending=True, stable=True)
        out[:, :k] = vals[:, :k]
        ids[:, n:n + k] = (idx[:, :k] + vocab_offset).to(torch.int32)
    return out


def prompt_logprobs_shard(logits: torch.Tensor, valid: int, n: int, targets: torch.Tensor, vocab_offset: int = 0,
                          out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """PyTorch model of csrc/sample/sampler.cu:prompt_logprobs_shard_kernel (n in {0, 1}): row q of `logits` scored
    against targets[q], in logprobs_shard's record layout — [argmax logit, its token id (lowest on ties)] when n = 1,
    then shard max, shard sum-exp and the target's raw logit (-inf when another shard holds it)."""
    assert n in (0, 1)
    rec = logprobs_shard(logits, valid, n, targets, vocab_offset=vocab_offset)
    if out is not None:
        return out.copy_(rec)
    return rec


def logprobs_final(gathered: torch.Tensor, n: int) -> torch.Tensor:
    """PyTorch model of logprobs_final_kernel: [tp, E, 2n+3] records -> [E, 1 + 2n] = sampled token's log-prob, then
    n x (token id bit-cast to float, log-prob) by logit, ties to the lower id; id -1 / -inf past the vocabulary."""
    tp, e, _ = gathered.shape
    ms, zs, ch = gathered[:, :, 2 * n], gathered[:, :, 2 * n + 1], gathered[:, :, 2 * n + 2]
    gm = ms.max(dim=0).values
    gz = (zs * torch.exp(torch.where(zs > 0, ms - gm.view(1, -1), torch.zeros_like(ms)))).sum(0)
    lse = gm + torch.log(gz)
    out = torch.empty(e, 1 + 2 * n, dtype=torch.float32, device=gathered.device)
    out[:, 0] = ch.max(dim=0).values - lse
    if n:
        vals = gathered[:, :, :n].permute(1, 0, 2).reshape(e, tp * n)
        toks = gathered[:, :, n:2 * n].contiguous().view(torch.int32).permute(1, 0, 2).reshape(e, tp * n)
        o1 = torch.argsort(toks, dim=1, stable=True)                  # token ascending, then logit descending (stable)
        vals, toks = vals.gather(1, o1), toks.gather(1, o1)
        o2 = torch.argsort(vals, dim=1, descending=True, stable=True)[:, :n]
        vals, toks = vals.gather(1, o2), toks.gather(1, o2)
        real = toks != LP_NO_TOKEN
        out.view(torch.int32)[:, 1::2] = torch.where(real, toks, torch.full_like(toks, -1))
        out[:, 2::2] = torch.where(real, vals - lse.view(-1, 1), torch.full_like(vals, float("-inf")))
    return out


# ----------------------------------------------------------------------------------------------
# MoE
# ----------------------------------------------------------------------------------------------
def topk_softmax(logits: torch.Tensor, top_k: int, renormalize: bool):
    probs = torch.softmax(logits.float(), dim=-1)
    w, ids = torch.topk(probs, top_k, dim=-1)
    if renormalize:
        w = w / w.sum(-1, keepdim=True)
    return w, ids.to(torch.int32)


def grouped_topk(logits: torch.Tensor, top_k: int, renormalize: bool, n_group: int, topk_group: int,
                 scoring: str = "softmax", bias: Optional[torch.Tensor] = None, routed_scaling: float = 1.0):
    """DeepSeek group-limited routing (reference: gllm/layers/moe/topk.py:87-138)."""
    x = logits.float()
    scores = torch.softmax(x, -1) if scoring == "softmax" else torch.sigmoid(x)
    t, e = scores.shape
    sel = scores + bias.float().view(1, -1) if bias is not None else scores
    grp = sel.view(t, n_group, e // n_group)
    if bias is not None:
        gscore = grp.topk(2, dim=-1)[0].sum(-1)
    else:
        gscore = grp.max(-1)[0]
    gidx = gscore.topk(topk_group, dim=-1)[1]
    gmask = torch.zeros_like(gscore).scatter(1, gidx, 1.0)
    mask = gmask.unsqueeze(-1).expand(t, n_group, e // n_group).reshape(t, e)
    masked = sel.masked_fill(mask == 0, float("-inf"))
    ids = masked.topk(top_k, dim=-1)[1]
    w = scores.gather(1, ids)
    if renormalize:
        w = w / (w.sum(-1, keepdim=True) + 1e-20)
    return w * routed_scaling, ids.to(torch.int32)


def fused_experts(x: torch.Tensor, w13: torch.Tensor, w2: torch.Tensor, topk_w: torch.Tensor,
                  topk_ids: torch.Tensor, expert_map: Optional[torch.Tensor] = None,
                  block: Optional[int] = None) -> torch.Tensor:
    """x [T,H]; w13 [E_local, 2I, H] (gate rows then up rows, or with `block` interleaved per `block` rows, see
    interleave_gate_up); w2 [E_local, H, I]; ids are GLOBAL expert ids, expert_map maps global -> local (or -1).
    Non-local experts contribute zero (reference EP semantics)."""
    t, h = x.shape
    out = torch.zeros(t, h, dtype=torch.float32, device=x.device)
    e_local = w13.shape[0]
    ids = topk_ids.long()
    if expert_map is not None:
        ids = expert_map.to(ids.device)[ids].long()
    for e in range(e_local):
        tok, slot = torch.where(ids == e)
        if tok.numel() == 0:
            continue
        xe = x[tok]
        hdn = silu_and_mul(F.linear(xe, w13[e])) if block is None else linear_silu_mul(xe, w13[e], block)
        ye = F.linear(hdn, w2[e]).float()
        out.index_add_(0, tok, ye * topk_w[tok, slot].float().unsqueeze(-1))
    return out.to(x.dtype)


# ----------------------------------------------------------------------------------------------
# fp8 block quantisation (reference semantics: gllm/layers/quantization/fp8.py)
# ----------------------------------------------------------------------------------------------
FP8_MAX = 448.0


def fp8_quant_group(x: torch.Tensor, group: int = 128):
    """Dynamic per-token-group quantisation -> (e4m3 tensor, fp32 scales [T, K/group])."""
    t, k = x.shape
    xg = x.float().reshape(t, k // group, group)
    amax = xg.abs().amax(-1).clamp_min(1e-10)
    scale = amax / FP8_MAX
    q = (xg / scale.unsqueeze(-1)).clamp(-FP8_MAX, FP8_MAX).to(torch.float8_e4m3fn)
    return q.reshape(t, k), scale


def fp8_block_dequant(w: torch.Tensor, scale_inv: torch.Tensor, block: int = 128) -> torch.Tensor:
    n, k = w.shape
    s = scale_inv.float().repeat_interleave(block, 0)[:n].repeat_interleave(block, 1)[:, :k]
    return w.float() * s


def linear_fp8_block(x: torch.Tensor, w: torch.Tensor, w_scale_inv: torch.Tensor,
                     bias: Optional[torch.Tensor] = None, block: int = 128) -> torch.Tensor:
    xq, xs = fp8_quant_group(x, block)
    xd = (xq.float().reshape(x.shape[0], -1, block) * xs.unsqueeze(-1)).reshape(x.shape[0], -1)
    wd = fp8_block_dequant(w, w_scale_inv, block)
    y = xd @ wd.t()
    if bias is not None:
        y = y + bias.float()
    return y.to(x.dtype)


def merge_attn_states(o1: torch.Tensor, lse1: torch.Tensor, o2: torch.Tensor, lse2: torch.Tensor):
    """LSE-weighted merge of two partial attention results. o [T,H,D], lse [T,H] (natural log)."""
    m = torch.maximum(lse1, lse2)
    w1, w2 = torch.exp(lse1 - m), torch.exp(lse2 - m)
    den = w1 + w2
    o = (o1.float() * (w1 / den).unsqueeze(-1) + o2.float() * (w2 / den).unsqueeze(-1)).to(o1.dtype)
    return o, m + torch.log(den)


# ----------------------------------------------------------------------------------------------
# multi-LoRA (csrc/lora/lora.cu). Rows are grouped per adapter by the batch CSR: slots [S], row_off [S + 1] and
# rows [T] (the adapter groups first, then the rows without an adapter).
# ----------------------------------------------------------------------------------------------
def _lora_groups(slots, row_off, rows):
    off = row_off.tolist()
    for g, s in enumerate(slots.tolist()):
        if off[g + 1] > off[g]:
            yield s, rows[off[g]:off[g + 1]].long()


def lora_shrink(x: torch.Tensor, A: torch.Tensor, slots, row_off, rows) -> torch.Tensor:
    """U [T, M] fp32 = x [T, K] · A[slot(row)] [M, K]ᵀ for every row of an adapter group, 0 for the others."""
    u = torch.zeros(x.shape[0], A.shape[1], dtype=torch.float32, device=x.device)
    for s, r in _lora_groups(slots, row_off, rows):
        u[r] = x[r].float() @ A[s].float().t()
    return u


def lora_delta(u: torch.Tensor, B: torch.Tensor, bounds, slots, row_off, rows) -> torch.Tensor:
    """fp32 [T, N] delta: column n of module m (bounds[m] <= n < bounds[m + 1]) is U[:, m·r : (m+1)·r] · B[slot, n]."""
    r = B.shape[2]
    d = torch.zeros(u.shape[0], B.shape[1], dtype=torch.float32, device=u.device)
    for s, rr in _lora_groups(slots, row_off, rows):
        for m in range(len(bounds) - 1):
            a, b = bounds[m], bounds[m + 1]
            d[rr, a:b] = u[rr, m * r:(m + 1) * r] @ B[s, a:b].float().t()
    return d


def lora_expand_add(y: torch.Tensor, u: torch.Tensor, B: torch.Tensor, bounds, slots, row_off, rows) -> torch.Tensor:
    """y [T, N] += delta (fp32 sum, one rounding to y's dtype), in place."""
    y.copy_((y.float() + lora_delta(u, B, bounds, slots, row_off, rows)).to(y.dtype))
    return y


def lora_expand_silu_mul(pre: torch.Tensor, u: torch.Tensor, B: torch.Tensor, slots, row_off, rows,
                         block: int = 128) -> torch.Tensor:
    """pre [T, 2I] gate/up pre-activations interleaved per `block` rows (see interleave_gate_up), u [T, 2r] (gate's
    shrink then up's), B [L, 2I, r] interleaved like the weight -> SiLU(gate + dg) · (up + du) [T, I]."""
    t, two_i = pre.shape
    r = B.shape[2]
    gate_col = (torch.arange(two_i, device=pre.device) % (2 * block)) < block
    d = torch.zeros(t, two_i, dtype=torch.float32, device=pre.device)
    for s, rr in _lora_groups(slots, row_off, rows):
        d[rr] = torch.where(gate_col, u[rr, :r] @ B[s].float().t(), u[rr, r:2 * r] @ B[s].float().t())
    y = (pre.float() + d).reshape(t, two_i // (2 * block), 2, block)
    return (F.silu(y[:, :, 0]) * y[:, :, 1]).to(pre.dtype).reshape(t, two_i // 2)


# ----------------------------------------------------------------------------------------------
# W4A16: int4 weights with 16-bit group scales and uint8 zero points (AWQ / GPTQ checkpoints)
# ----------------------------------------------------------------------------------------------
class Int4Weight:
    """Weight handle of a W4A16 linear, in the device layout of csrc/gemm/gemm_w4a16.cu (the same on every device):
    `packed` int32 [round_up(N, 16), round_up(K, 128) / 8], `scales` fp16/bf16 [G, N], `zeros` uint8
    [G, round_up(N, 16)], with G = ceil(K / group_size). `group_size` >= K means one group. Not a tuple: the linear
    ops send tuples to the fp8 block GEMM."""
    __slots__ = ("packed", "scales", "zeros", "group_size", "in_features")

    def __init__(self, packed, scales, zeros, group_size: int, in_features: int):
        self.packed, self.scales, self.zeros = packed, scales, zeros
        self.group_size, self.in_features = int(group_size), int(in_features)

    @property
    def out_features(self) -> int:
        return self.scales.shape[1]


W4_BLOCK_K = 128


def _w4_fragment_index():
    """[256 words, 8 nibbles] -> (row, k) index (row * 128 + k) inside one 16-row x 128-k block of the device layout:
    word p = 128 h + 4 lane + j holds lane's m64k16 A fragment of k-step 4 h + j; nibble e is fragment element e, at
    row lane / 4 (+ 8 for e = 2, 3, 6, 7) and column 2 (lane % 4) + e % 2 (+ 8 for e >= 4)."""
    p = torch.arange(256).view(256, 1)
    e = torch.arange(8).view(1, 8)
    h, lane, j = p // 128, (p // 4) % 32, p % 4
    row = lane // 4 + 8 * ((e // 2) % 2)
    col = 16 * (4 * h + j) + 2 * (lane % 4) + e % 2 + 8 * (e // 4)
    return row * W4_BLOCK_K + col


_W4_IDX = _w4_fragment_index()


def w4a16_pack(codes: torch.Tensor, zeros: torch.Tensor, scales: torch.Tensor):
    """Checkpoint orientation -> device layout. codes uint8 [N, K] in [0, 15], zeros uint8 [N, G], scales 16-bit
    [N, G] -> (packed, scales [G, N], zeros [G, Np]); see `Int4Weight`."""
    n, k = codes.shape
    np_, kp = -(-n // 16) * 16, -(-k // W4_BLOCK_K) * W4_BLOCK_K
    c = torch.zeros(np_, kp, dtype=torch.int64)
    c[:n, :k] = codes.to(torch.int64)
    blocks = c.view(np_ // 16, 16, kp // W4_BLOCK_K, W4_BLOCK_K).permute(0, 2, 1, 3).reshape(
        np_ // 16, kp // W4_BLOCK_K, 16 * W4_BLOCK_K)
    nib = blocks[:, :, _W4_IDX.view(-1)].view(np_ // 16, kp // W4_BLOCK_K, 256, 8)
    words = (nib << (4 * torch.arange(8))).sum(-1)
    words = torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32)
    packed = words.view(np_ // 16, kp // W4_BLOCK_K, 16, 16).permute(0, 2, 1, 3).reshape(np_, kp // 8)
    z = torch.zeros(zeros.shape[1], np_, dtype=torch.uint8)
    z[:, :n] = zeros.t()
    return packed.contiguous(), scales.t().contiguous(), z


def w4a16_unpack(w: Int4Weight):
    """Device layout -> checkpoint orientation: (codes uint8 [N, K], zeros uint8 [N, G], scales [N, G])."""
    packed = w.packed.cpu()
    np_, kw = packed.shape
    kp = kw * 8
    words = packed.view(np_ // 16, 16, kp // W4_BLOCK_K, 16).permute(0, 2, 1, 3).reshape(
        np_ // 16, kp // W4_BLOCK_K, 256, 1).to(torch.int64) & 0xFFFFFFFF
    nib = (words >> (4 * torch.arange(8))) & 0xF
    blocks = torch.empty(np_ // 16, kp // W4_BLOCK_K, 16 * W4_BLOCK_K, dtype=torch.int64)
    blocks[:, :, _W4_IDX.view(-1)] = nib.view(np_ // 16, kp // W4_BLOCK_K, 2048)
    codes = blocks.view(np_ // 16, kp // W4_BLOCK_K, 16, W4_BLOCK_K).permute(0, 2, 1, 3).reshape(np_, kp)
    n, k = w.out_features, w.in_features
    return (codes[:n, :k].to(torch.uint8), w.zeros.cpu()[:, :n].t().contiguous(),
            w.scales.cpu().t().contiguous())


def w4a16_dequant(codes: torch.Tensor, zeros: torch.Tensor, scales: torch.Tensor, group_size: int,
                  dtype: torch.dtype) -> torch.Tensor:
    """W [N, K] = dtype( fp32(s) · (q − z) ): exact in fp32 (a 16-bit scale has at most 11 significant bits and
    |q − z| <= 16), rounded once. Column k uses group k // group_size (one group if group_size >= K)."""
    k = codes.shape[1]
    gi = torch.arange(k) // group_size if group_size < k else torch.zeros(k, dtype=torch.long)
    q = codes.to(torch.float32)
    z = zeros.to(torch.float32)[:, gi]
    s = scales.to(torch.float32)[:, gi]
    return (s * (q - z)).to(dtype)


def linear_w4a16(x: torch.Tensor, w: Int4Weight, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    codes, zeros, scales = w4a16_unpack(w)
    wd = w4a16_dequant(codes, zeros, scales, w.group_size, x.dtype).to(x.device)
    return linear(x, wd, bias)
