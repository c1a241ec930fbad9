"""Token sampling on the last pipeline stage: the per-slot device state of the sampling parameters and the flow from
one step's logits to its tokens and log-probabilities, on the op table of the device (`ops.table`)."""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from gllm_b200 import ops
from gllm_b200.input_data import BatchArrays, InputData
from gllm_b200.parallel import state as ps


def _all_gather(x: torch.Tensor) -> torch.Tensor:
    """[tp, *x.shape]: `x` of every TP rank, in rank order."""
    import torch.distributed as dist
    st = ps.get_state()
    out = torch.empty(st.tp_size, *x.shape, dtype=x.dtype, device=x.device)
    dist.all_gather_into_tensor(out.view(st.tp_size * x.shape[0], *x.shape[1:]), x, group=st.tp_group)
    return out


class Sampler:
    VP_CANDIDATES = 256   # per rank and row; top_k <= this is exact (csrc/sample/sampler.cu)

    def __init__(self, device: torch.device, vocab_size: int, seed: int, inp: InputData, stats: dict,
                 vocab_parallel: bool):
        """`vocab_parallel`: the logits are this TP rank's vocab shard, and no rank ever gathers the [E, V] logits."""
        self.ops = ops.table(device)
        self.device, self.vocab_size, self.seed, self.inp, self.stats = device, vocab_size, seed, inp, stats
        self.vocab_parallel = vocab_parallel
        self.seen_bits = None    # int32 [slots, ceil(V/32)]: prompt + output tokens under the repetition penalty
        self.bias_rows = None    # fp32 [slots, V]: frequency / presence penalties + logit_bias
        self.out_seen = None     # int32 [slots, ceil(V/32)]: tokens each slot's sequence has generated
        # steps that drew random numbers (greedy-only batches do not count): keys the unseeded rows' streams
        self.step_counter = torch.zeros(1, dtype=torch.int64, device=device)

    def sample(self, batch: BatchArrays, logits: torch.Tensor):
        """-> (tokens [E] on the logits' device, log-prob records [E_lp, 1 + 2N] or None when no row asked). `logits`
        [E, V] or, vocab-parallel, this rank's shard [E, Vp/tp]."""
        inp, e = self.inp, logits.shape[0]
        bias = self._bias(batch) if batch.need_bias else None
        if self.vocab_parallel and batch.plain_greedy:
            toks = self._vp_greedy(logits)
            return toks, self._logprobs(batch, logits, toks)
        seen = self._mark_seen(batch) if batch.need_penalty else None
        # (rep_penalty, seen_bits, slot_idx) arguments of the sampling ops
        pen = (inp.rep_penalty[:e], seen, inp.state_slot[:e]) if seen is not None else (None, None, None)
        if not batch.all_greedy:
            self.step_counter += 1
        if self.vocab_parallel:
            toks = self._vp_sample(logits, pen, bias)
        elif batch.plain_greedy:
            toks = self.ops.sample(logits)
        else:
            seeds, spos = inp.seeds
            toks = self.ops.sample(logits, inp.temperature[:e], inp.top_k[:e], inp.top_p[:e], *pen,
                                   seed=self.seed, step=self.step_counter, bias=bias, bias_slot=inp.bias_slot,
                                   seeds=seeds, seed_pos=spos)
        if batch.need_bias:
            # charged on the device: the host never sends per-step tokens, so these rows stay eligible for lookahead
            # and the incremental decode path
            self.ops.bias_account(self.bias_rows, self.out_seen, inp.bias_slot, toks.to(torch.int32).contiguous(),
                                  inp.freq_pen, inp.pres_pen)
        return toks, self._logprobs(batch, logits, toks)

    # -- per-slot state ----------------------------------------------------------------------------
    def _grown(self, t: Optional[torch.Tensor], rows: int, cols: int, dtype) -> torch.Tensor:
        """`t` with at least `rows` rows, one per slot: grown (never shrunk) to cover the largest slot handed out —
        every rank sees the same slots."""
        if t is not None and t.shape[0] >= rows:
            return t
        new = torch.zeros(max(rows, 65 if t is None else 2 * t.shape[0]), cols, dtype=dtype, device=self.device)
        if t is not None:
            new[: t.shape[0]] = t
        return new

    def _mark_seen(self, batch: BatchArrays) -> torch.Tensor:
        """The seen-token bitmask (row 0: no penalty state), with this step's cleared slots and new prompt tokens."""
        rows = int(batch.state_slot.max()) + 1 if len(batch.state_slot) else 1
        self.seen_bits = seen = self._grown(self.seen_bits, rows, (self.vocab_size + 31) // 32, torch.int32)
        dev = self.device
        if batch.clear_slots is not None:
            seen[torch.from_numpy(batch.clear_slots).to(dev).long()] = 0
        if batch.seen_rows is not None:
            self.ops.mark_seen(seen, torch.from_numpy(batch.seen_rows).to(dev),
                               torch.from_numpy(batch.seen_tokens).to(dev))
        return seen

    def _bias(self, batch: BatchArrays) -> torch.Tensor:
        """The bias rows, with the slots (re)assigned this step rebuilt: cleared, logit_bias scattered, the counts of
        the outputs known so far replayed. About V * 4.125 bytes per slot (594 KiB at V = 151936), not part of the
        KV-cache sizing."""
        rows, v = int(batch.bias_slot.max()) + 1, self.vocab_size
        self.bias_rows = self._grown(self.bias_rows, rows, v, torch.float32)
        self.out_seen = self._grown(self.out_seen, rows, (v + 31) // 32, torch.int32)
        if batch.rb_slots is not None:
            t = [torch.from_numpy(np.ascontiguousarray(a)).to(self.device) for a in
                 (batch.rb_slots, batch.rb_pen, batch.rb_lb_off, batch.rb_lb_ids, batch.rb_lb_vals, batch.rb_out_off,
                  batch.rb_out_toks)]
            self.ops.bias_rebuild(self.bias_rows, self.out_seen, v, *t)
        return self.bias_rows

    # -- vocab-parallel ----------------------------------------------------------------------------
    def _shard(self, per: int):
        """(token id of column 0, real vocabulary columns) of this rank's shard: the last one ends with padding."""
        r0 = ps.get_tp_rank() * per
        return r0, max(0, min(per, self.vocab_size - r0))

    def _vp_sample(self, shard: torch.Tensor, pen: tuple, bias: Optional[torch.Tensor]) -> torch.Tensor:
        """Vocab-parallel top-k / top-p / penalty sampling (SURVEY §2.4 X4): every rank reduces its vocab shard to
        a [E, 2C+4] record (C best candidates, softmax statistics, race winner), the ranks all-gather the records —
        ~2 KB per row and rank instead of V/tp logits — and finish on the tp x C candidates with the exact global
        normalisation. The [E, V] logits are never materialised (the reference all-gathers them and sorts the full
        vocabulary: gllm/layers/vocab_parallel_embedding.py:423-435, gllm/layers/sampler.py:8-54)."""
        inp = self.inp
        e, per = shard.shape
        r0, valid = self._shard(per)
        c = min(self.VP_CANDIDATES, per)
        seeds, spos = inp.seeds
        rec = self.ops.vp_candidates(shard, valid, self.vocab_size, c, inp.temperature[:e], inp.top_k[:e],
                                     inp.top_p[:e], *pen, seed=self.seed, step=self.step_counter,
                                     vocab_offset=r0, bias=bias, bias_slot=inp.bias_slot, seeds=seeds, seed_pos=spos)
        allr = _all_gather(rec)
        self.stats["vp_sample_steps"] = self.stats.get("vp_sample_steps", 0) + 1
        return self.ops.vp_final(allr, c, self.vocab_size, inp.top_k[:e], inp.top_p[:e], seed=self.seed,
                                 step=self.step_counter, seeds=seeds, seed_pos=spos)

    def _vp_greedy(self, shard: torch.Tensor) -> torch.Tensor:
        """Vocab-parallel greedy sampling (SURVEY §2.4 X4): every rank takes the argmax of its own vocab shard
        with the sampler kernel, the ranks exchange (value, global index) pairs — 8 bytes per row instead of the
        [E, V] logits — and pick the winner (lowest rank on ties == lowest token id)."""
        e, per = shard.shape
        r0, valid = self._shard(per)
        pack = torch.empty(e, 2, dtype=torch.float32, device=shard.device)
        if valid > 0:
            val = torch.empty(e, dtype=torch.float32, device=shard.device)
            idx = self.ops.sample(shard[:, :valid], out_max=val, vocab_offset=r0)
            pack[:, 0] = val
            pack[:, 1] = idx.float()   # token ids < 2^24 are exact in fp32
        else:
            pack[:, 0] = float("-inf")
            pack[:, 1] = 0
        allp = _all_gather(pack)
        best = allp[:, :, 0].argmax(dim=0, keepdim=True)
        return allp[:, :, 1].gather(0, best)[0].to(torch.int32)

    # -- log-probabilities -------------------------------------------------------------------------
    def _logprobs(self, batch: BatchArrays, logits: torch.Tensor, toks: torch.Tensor) -> Optional[torch.Tensor]:
        """Log-probabilities of the raw model distribution for the emitting rows that asked (csrc/sample/sampler.cu:
        logprobs_shard_kernel / logprobs_final_kernel), after the tokens are chosen. Vocab-parallel, every TP rank
        reduces its shard to [E_lp, 2N+3] records and the ranks all-gather them (every rank decides from the batch
        alone, so all of them join the collective). None when no row asked: then the step launches, exchanges and
        copies nothing more than without this feature."""
        lpn = batch.logprobs_n
        if lpn is None:
            return None
        want = np.nonzero(lpn >= 0)[0].astype(np.int32)
        if want.size == 0:
            return None
        n = int(lpn[want].max())
        rows = torch.from_numpy(want).to(logits.device)
        toks = toks.to(torch.int32).contiguous()
        off, valid = self._shard(logits.shape[1]) if self.vocab_parallel else (0, self.vocab_size)
        rec = self.ops.logprobs_shard(logits, valid, n, toks, rows, vocab_offset=off)
        allr = _all_gather(rec) if self.vocab_parallel else rec.unsqueeze(0)
        self.stats["logprob_rows"] = self.stats.get("logprob_rows", 0) + len(want)
        return self.ops.logprobs_final(allr, n)

    def prompt_logprobs(self, batch: BatchArrays, hidden: torch.Tensor, lm_head, tile_rows: int) -> torch.Tensor:
        """Log-probabilities of the batch's prompt rows, each scored against its target (the next prompt token) ->
        fp32 [Q, 1 + 2N], logprobs_final's layout. The rows' final-normed hidden states go through the LM head
        (`lm_head(rows, out)` -> [R, Vp/tp]) `tile_rows` at a time into one reused buffer, and each tile is reduced to
        records right after its GEMM, while it is in L2 (csrc/sample/sampler.cu: prompt_logprobs_shard_kernel, one
        pass, for N <= 1; logprobs_shard_kernel for N > 1). The TP ranks all-gather the records of all tiles once."""
        dev, n = hidden.device, batch.plp_n
        rows, targets = self.inp.plp
        q = rows.numel()
        rec = torch.empty(q, 2 * n + 3, dtype=torch.float32, device=dev)
        buf = None
        for a in range(0, q, tile_rows):
            b = min(q, a + tile_rows)
            x = self.ops.gather_rows(hidden.contiguous(), rows[a:b])
            logits = lm_head(x, None if buf is None else buf[: b - a])
            if buf is None:
                buf = logits
            off, valid = self._shard(logits.shape[1])
            if n <= 1:
                self.ops.prompt_logprobs_shard(logits, valid, n, targets[a:b], vocab_offset=off, out=rec[a:b])
            else:
                rec[a:b] = self.ops.logprobs_shard(logits, valid, n, targets[a:b], vocab_offset=off)
        allr = _all_gather(rec) if ps.get_tp_size() > 1 else rec.unsqueeze(0)
        self.stats["prompt_logprob_rows"] = self.stats.get("prompt_logprob_rows", 0) + q
        return self.ops.logprobs_final(allr, n)
