"""CPU stand-ins for the sampler ops of `ops.sm100`, with the same signatures and the same device-state formats:
seen-token bitmask rows plus a slot index, per-slot bias rows plus a slot, and an RNG keyed by `seed` plus the step
counter. Each stand-in converts that state to the dense arguments of its `ops.ref` oracle. This is the CPU plumbing
path only; it never stands in for a missing kernel on a GPU.
"""
from __future__ import annotations

from typing import Optional

import torch

from gllm_b200.ops import ref
from gllm_b200.ops.ref import (kv_copy_pages, logprobs_final, logprobs_shard,  # noqa: F401  (sm100 signatures)
                               prompt_logprobs_shard)
from gllm_b200.parallel import state as ps


def _generator(seed: int, step: Optional[torch.Tensor], salt: int = 0) -> torch.Generator:
    """Unseeded rows' random stream: one generator per step, keyed by the engine seed and the step counter."""
    return torch.Generator().manual_seed(seed + (int(step) if step is not None else 0) + salt)


def _seen_mask(seen_bits: Optional[torch.Tensor], slot_idx, lo: int, hi: int) -> Optional[torch.Tensor]:
    """Dense bool [B, hi - lo] over token ids [lo, hi) of the bitmask rows `seen_bits[slot_idx]`."""
    if seen_bits is None:
        return None
    rows = seen_bits[slot_idx.long()]
    bits = (rows.unsqueeze(-1) >> torch.arange(32, dtype=torch.int32)) & 1
    return bits.reshape(rows.shape[0], -1)[:, lo:hi].bool()


def _dense_bias(bias: Optional[torch.Tensor], bias_slot, lo: int, hi: int) -> Optional[torch.Tensor]:
    """fp32 [B, hi - lo] over token ids [lo, hi) of each batch row's bias row (zeros where it has none)."""
    if bias is None or bias_slot is None:
        return None
    rows = bias[bias_slot.clamp(min=0).long(), lo:hi].clone()
    rows[bias_slot < 0] = 0.0
    return rows


def sample(logits: torch.Tensor, temperature=None, top_k=None, top_p=None, rep_penalty=None,
           seen_bits: Optional[torch.Tensor] = None, slot_idx: Optional[torch.Tensor] = None, seed: int = 0,
           step: Optional[torch.Tensor] = None,
           out: Optional[torch.Tensor] = None, out_max: Optional[torch.Tensor] = None,
           vocab_offset: int = 0, bias: Optional[torch.Tensor] = None, bias_slot: Optional[torch.Tensor] = None,
           seeds: Optional[torch.Tensor] = None, seed_pos: Optional[torch.Tensor] = None) -> torch.Tensor:
    lo, hi = vocab_offset, vocab_offset + logits.shape[1]
    if out_max is not None:     # greedy argmax of a vocab shard, with the winning value
        val, idx = logits.float().max(dim=1)
        out_max.copy_(val)
        tok = (idx + lo).to(torch.int32)
    else:
        tok = ref.sample(logits, temperature, top_k, top_p, rep_penalty, _seen_mask(seen_bits, slot_idx, lo, hi),
                         generator=_generator(seed, step), bias=_dense_bias(bias, bias_slot, lo, hi), seeds=seeds,
                         seed_pos=seed_pos) + lo
    if out is not None:
        return out.copy_(tok)
    return tok


def vp_candidates(shard: torch.Tensor, valid: int, v_full: int, c: int, temperature=None, top_k=None, top_p=None,
                  rep_penalty=None, seen_bits: Optional[torch.Tensor] = None,
                  slot_idx: Optional[torch.Tensor] = None, seed: int = 0, step: Optional[torch.Tensor] = None,
                  vocab_offset: int = 0, bias: Optional[torch.Tensor] = None,
                  bias_slot: Optional[torch.Tensor] = None, seeds: Optional[torch.Tensor] = None,
                  seed_pos: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Unseeded rows race on one draw over the whole padded vocabulary [B, per * tp] (every rank draws the same
    block and keeps its own columns); seeded rows on the kernel's stream keyed by token id."""
    e, per = shard.shape
    hi = vocab_offset + max(valid, 0)
    race = torch.empty(e, per * ps.get_tp_size()).exponential_(1.0, generator=_generator(seed, step))
    race = race[:, vocab_offset:hi]
    if seeds is not None:
        for r in torch.nonzero(seed_pos >= 0)[:, 0].tolist():
            race[r] = ref.race_exp(int(seeds[r]), int(seed_pos[r]), range(vocab_offset, hi))
    return ref.vp_candidates(shard, valid, v_full, c, temperature, top_k, top_p, rep_penalty,
                             _seen_mask(seen_bits, slot_idx, vocab_offset, hi), race,
                             vocab_offset=vocab_offset, bias=_dense_bias(bias, bias_slot, vocab_offset, hi))


def vp_final(gathered: torch.Tensor, c: int, v_full: int, top_k=None, top_p=None, seed: int = 0,
             step: Optional[torch.Tensor] = None, seeds: Optional[torch.Tensor] = None,
             seed_pos: Optional[torch.Tensor] = None) -> torch.Tensor:
    return ref.vp_final(gathered, c, v_full, top_k, top_p, generator=_generator(seed, step, 0x5bd1), seeds=seeds,
                        seed_pos=seed_pos)


def mark_seen(seen_bits: torch.Tensor, rows: torch.Tensor, tokens: torch.Tensor):
    word = (tokens >> 5).long()
    bit = (torch.ones_like(tokens) << (tokens & 31)).to(torch.int32)
    for rw, wd, bt in zip(rows.tolist(), word.tolist(), bit.tolist()):
        seen_bits[rw, wd] |= bt


def bias_account(bias: torch.Tensor, out_seen: torch.Tensor, bias_slot: torch.Tensor, tokens: torch.Tensor,
                 freq: torch.Tensor, pres: torch.Tensor):
    for r, (slot, tok) in enumerate(zip(bias_slot.tolist(), tokens.tolist())):
        if slot >= 0:
            ref.bias_account_one(bias, out_seen, slot, int(tok), float(freq[r]), float(pres[r]))


def bias_rebuild(bias: torch.Tensor, out_seen: torch.Tensor, v: int, slots: torch.Tensor, pen: torch.Tensor,
                 lb_off: torch.Tensor, lb_ids: torch.Tensor, lb_vals: torch.Tensor, out_off: torch.Tensor,
                 out_toks: torch.Tensor):
    lo, oo = lb_off.tolist(), out_off.tolist()
    for r, slot in enumerate(slots.tolist()):
        ref.bias_rebuild(bias, out_seen, slot, float(pen[r, 0]), float(pen[r, 1]), lb_ids[lo[r]:lo[r + 1]],
                         lb_vals[lo[r]:lo[r + 1]], out_toks[oo[r]:oo[r + 1]].tolist())
