"""Continuous-batching scheduler with three policies (reference: gllm/scheduler.py:16-355):

  * ``chunked_prefill``  — Sarathi-style: one token budget `maxp`; decode first, rest to prefill.
  * ``split_pd``         — prefill-priority: decode budget is zeroed while prefills wait and KV
                           headroom exists.
  * ``token_throttling`` — gLLM (SC'25): prefill budget throttled by KV utilisation (UT) and by
                           the amount of waiting work spread over `iterp` iterations (WT); decode
                           budget = all running decode seqs balanced over the `pp_size`
                           micro-batches in flight.

Invariants kept from the reference: at most `pp_size` micro-batches in flight; each batch is
**decode sequences first, then prefill chunks**; preemption = free KV + recompute; a sequence
emits a token only once its whole prompt is computed.

The budget computations are exposed as pure functions so they can be unit-tested against the
formulas without an engine.
"""
from __future__ import annotations

import random
import time
from collections import deque
from dataclasses import dataclass, field
from typing import Deque, List, Optional

from gllm_b200.memory_manager import MemoryManager, PrefixMemoryManager
from gllm_b200.sequence import Sequence
from gllm_b200.utils.logging import logger


# ------------------------------------------------------------------------------------------------
# pure budget functions
# ------------------------------------------------------------------------------------------------
def balanced_decode_budget(num_total_decode_seqs: int, pp_size: int, maxd: int, rnd: Optional[int] = None) -> int:
    """⌊(#running decode seqs + U[0,pp)) / pp⌋ capped by maxd (gllm/scheduler.py:192-203)."""
    if num_total_decode_seqs < pp_size:
        budget = 1
    else:
        r = random.randint(0, pp_size - 1) if rnd is None else rnd
        budget = (num_total_decode_seqs + r) // pp_size
    return min(maxd, budget)


def kv_headroom_tokens(num_free_pages: int, num_kvthresh_pages: int, page_size: int) -> int:
    return page_size * max(num_free_pages - num_kvthresh_pages, 0)


def throttled_prefill_budget(headroom_tokens: int, world_size: int, free_ratio: float, kvthresh: float,
                             maxp: int, minp: int, iterp: int, num_wait_seqs: int, num_wait_tokens: int) -> int:
    """Token-throttling prefill budget #P (gllm/scheduler.py:299-320)."""
    budget = headroom_tokens
    if world_size > 1 and budget != 0:
        ratio = max((free_ratio - kvthresh) / (1 - kvthresh), 0.0)
        budget = min(round(ratio * maxp), budget)  # UT
        if num_wait_seqs > 1:  # WT
            budget = min(max(num_wait_tokens // iterp, minp), budget)
    else:
        budget = min(maxp, budget)
    return budget


PLACEHOLDER = -1  # token id of a position whose value is still being sampled on the device (lookahead step)


class ScheduledSeq:
    """One entry of a micro-batch: compute tokens [start, start + n) of `seq`."""
    __slots__ = ("seq", "start", "n", "emits", "is_decode", "forks", "kv_copy", "plp")

    def __init__(self, seq: Sequence, start: int, n: int):
        self.seq, self.start, self.n = seq, start, n
        # A token is sampled only when the chunk reaches the end of everything known so far. (After a
        # preemption the recomputed "prompt" includes the tokens generated before; the reference's
        # `computed_token_num >= prompt_len` test would emit early on a chunked recompute.)
        self.emits = start + n >= len(seq.token_ids)
        self.is_decode = n == 1 and self.emits and start >= seq.prompt_len
        # parallel sampling: the other choices whose first tokens are drawn from this entry's last logits row (one
        # extra sampled row each, after every entry's own row) and the (src, dst) page copies that give each of them
        # the partial last prompt page. None for every other entry.
        self.forks: Optional[List[Sequence]] = None
        self.kv_copy: Optional[List[tuple]] = None
        # prompt log-probabilities: how many prompt rows this entry carries (set when its batch is built)
        self.plp = 0

    def __repr__(self):
        return f"ScheduledSeq(id={self.seq.seq_id}, start={self.start}, n={self.n})"


@dataclass
class SchedulerOutput:
    """What rank 0 tells the front-end after a batch finished (mirrors IPCPackage fields)."""
    act_schedule_ids: List[int] = field(default_factory=list)
    next_tokens: List[int] = field(default_factory=list)
    free_ids: List[int] = field(default_factory=list)
    # aligned with next_tokens when some row of the batch asked for log-probs (entry None for rows that did not),
    # None otherwise
    next_logprobs: Optional[list] = None
    # prompt log-probabilities delivered by the batch: seq id -> its next entries in prompt order; None when none
    prompt_logprobs: Optional[dict] = None


class Scheduler:
    def __init__(self, memory_manager: MemoryManager, pp_size: int = 1, world_size: int = 1,
                 schedule_method: str = "chunked_prefill", maxd: int = 2048, maxp: int = 2048, minp: int = 32,
                 iterp: int = 8, kvthresh: float = 0.05, page_size: int = 16, log: bool = True,
                 max_seqs: Optional[int] = None):
        assert schedule_method in ("chunked_prefill", "split_pd", "token_throttling"), schedule_method
        self.mm = memory_manager
        self.pp_size = pp_size
        self.world_size = world_size
        self.schedule_method = schedule_method
        self.maxd, self.maxp, self.minp, self.iterp = maxd, maxp, minp, iterp
        self.kvthresh = kvthresh
        self.page_size = page_size
        # capacity of the runner's per-sequence buffers (config.max_running_seqs): a micro-batch never holds more
        # sequences. With token_throttling that capacity is maxd (as in the reference, model_runner.py:67-71) while a
        # batch is decode rows PLUS prefill rows — without this cap a full decode batch plus one prompt overflows.
        self.max_seqs = max_seqs
        self.num_kvthresh_pages = int(kvthresh * self.mm.get_num_free_pages())
        self.seqs_to_prefill: Deque[Sequence] = deque()
        self.seqs_to_decode: Deque[Sequence] = deque()
        self.batch_running: Deque[List[ScheduledSeq]] = deque()
        self.next_tokens_queue: Deque[List[int]] = deque()
        self.next_logprobs_queue: Deque[Optional[list]] = deque()   # one entry per next_tokens_queue entry
        self.next_plp_queue: Deque[Optional[list]] = deque()        # prompt log-prob rows, likewise
        self.abort_ids = set()
        self.on_preempt = None      # callback(seq): the owner releases per-sequence device state
        self.num_preempt_seqs = 0
        self._log_preempt_at = 10
        self.num_wait_tokens = 0
        self.log = log
        self.log_time = 0.0
        self.last_stats = {}

    # -- inputs -----------------------------------------------------------------------------------
    def add_new_requests(self, seqs: List[Sequence]):
        cap = (self.mm.num_pages - (1 if getattr(self.mm, "dummy_page", None) is not None else 0)) * self.page_size
        # prefill may only use the pages above the kvthresh reserve (kv_headroom_tokens), decode may use all of them
        prompt_cap = cap - self.num_kvthresh_pages * self.page_size
        for seq in seqs:
            if len(seq) + 1 > prompt_cap:
                # the prompt alone can never be resident: it would wait in the queue forever
                logger.error("request %d: prompt of %d tokens but the KV cache can hold %d during prefill: rejected",
                             seq.seq_id, len(seq), prompt_cap)
                self.abort_ids.add(seq.seq_id)
            elif len(seq) + seq.output_len > cap:
                # alone in the pool it would still outgrow it and be preempted/recomputed forever: cap the length
                logger.warning("request %d: output capped to %d tokens (KV cache holds %d tokens)", seq.seq_id,
                               cap - len(seq), cap)
                seq.output_len = cap - len(seq)
            for sib in seq.forks:
                sib.output_len = min(sib.output_len, max(cap - len(seq), 1))
        self.seqs_to_prefill.extend(seqs)

    def add_abort_ids(self, ids):
        self.abort_ids.update(ids)

    def add_next_tokens(self, next_tokens: List[int], next_logprobs: Optional[list] = None,
                        prompt_logprobs: Optional[list] = None):
        """`next_logprobs`: None, or one entry per emitting row (None where the row did not ask). `prompt_logprobs`:
        None, or one entry per prompt log-prob row of the batch, in entry order (`ScheduledSeq.plp` rows each)."""
        self.next_tokens_queue.append(next_tokens)
        self.next_logprobs_queue.append(next_logprobs)
        self.next_plp_queue.append(prompt_logprobs)

    def set_log(self, log: bool):
        self.log = log

    # -- state ------------------------------------------------------------------------------------
    def has_work(self) -> bool:
        return bool(self.seqs_to_decode or self.seqs_to_prefill or self.batch_running)

    def get_num_decode_seqs(self) -> int:
        # reference counts every seq of every in-flight batch (gllm/scheduler.py:64-68)
        return len(self.seqs_to_decode) + sum(len(b) for b in self.batch_running)

    def update_num_wait_tokens(self):
        self.num_wait_tokens = sum(len(s) - s.scheduled_token_num for s in self.seqs_to_prefill)

    # -- outputs ----------------------------------------------------------------------------------
    def process_output(self) -> Optional[SchedulerOutput]:
        if not self.next_tokens_queue:
            return None
        batch = self.batch_running.popleft()
        next_tokens = self.next_tokens_queue.popleft()
        next_logprobs = self.next_logprobs_queue.popleft()
        plp = self.next_plp_queue.popleft()
        out = SchedulerOutput()
        if next_logprobs is not None:
            out.next_logprobs = []
        if plp is not None:
            out.prompt_logprobs = {}
            j = 0
            for ent in batch:
                if ent.plp:
                    seq = ent.seq
                    if not (seq.zombie or seq.is_abort):
                        n = seq.prompt_logprobs_n       # (the batch reports its largest N for every row)
                        out.prompt_logprobs.setdefault(seq.seq_id, []).extend(
                            (lp, top[:n]) for lp, top in plp[j:j + ent.plp])
                    j += ent.plp
        prefix, ps = isinstance(self.mm, PrefixMemoryManager), self.page_size
        if any(ent.forks for ent in batch):
            self._process_forks(batch, next_tokens, next_logprobs, out)
        k = 0  # next_tokens holds one token per *emitting* entry, in batch order
        for ent in batch:
            seq = ent.seq
            if ent.emits:
                k += 1
            if seq.zombie:
                # finished (or aborted) while this lookahead step was already in flight: its token is
                # discarded, its pages can go now unless yet another step still references them
                if not self._in_flight(seq):
                    seq.zombie = False
                    if seq.page_table:
                        self.mm.free(seq)
                continue
            if seq.is_abort:
                # whoever flagged it (check_abort_seqs) took it out of the queues; be robust against a flag set
                # elsewhere: a freed sequence left at the head of seqs_to_prefill would be scheduled again on an
                # empty page table
                self._drop_from_queues(seq)
                self.mm.publish_computed(seq)
                out.free_ids.append(seq.seq_id)     # exactly once: the zombie branch above never reports
                if self._in_flight(seq):
                    seq.zombie = True
                else:
                    self.mm.free(seq)
                self.abort_ids.discard(seq.seq_id)
                continue
            done = ent.start + ent.n
            if done > seq.computed_token_num:
                seq.computed_token_num = done
            if prefix and done // ps > seq.published:      # (hot loop: a page completes once per `ps` decode steps)
                self.mm.publish_computed(seq)
            if ent.emits:
                tok = int(next_tokens[k - 1])
                out.act_schedule_ids.append(seq.seq_id)
                out.next_tokens.append(tok)
                if next_logprobs is not None:
                    out.next_logprobs.append(next_logprobs[k - 1])
                ahead = seq.pending == ent.start + ent.n   # a lookahead step already follows this one
                if ahead:
                    seq.token_ids[seq.pending] = tok
                    seq.pending = -1
                else:
                    seq.append(tok)
                # == seq.is_finish (inlined: this loop runs once per sequence per step; the prompt is computed
                # whenever an entry emits)
                if (not seq.ignore_eos and tok in seq.finish_tokens) or \
                        len(seq.token_ids) - seq.prompt_len >= seq.output_len:
                    out.free_ids.append(seq.seq_id)
                    if ahead:
                        seq.zombie = True
                    else:
                        self.mm.free(seq)
                elif not ahead:
                    self.seqs_to_decode.appendleft(seq)
            # else: unfinished prefill — its continuation is already at the head of seqs_to_prefill
        return out

    def _process_forks(self, batch, next_tokens, next_logprobs, out: SchedulerOutput):
        """The extra rows of a fan-out follow every entry's own row: hand token i to choice i. Runs before the
        entries' own tokens, so it is done before the parent can be freed (it may finish on its first token)."""
        k = sum(1 for ent in batch if ent.emits)
        for ent in batch:
            for sib in ent.forks or ():
                tok = int(next_tokens[k])
                lp = next_logprobs[k] if next_logprobs is not None else None
                k += 1
                if sib.is_abort or sib.seq_id in self.abort_ids:
                    sib.is_abort = True
                    self.mm.free(sib)
                    out.free_ids.append(sib.seq_id)
                    self.abort_ids.discard(sib.seq_id)
                    continue
                sib.append(tok)
                out.act_schedule_ids.append(sib.seq_id)
                out.next_tokens.append(tok)
                if next_logprobs is not None:
                    out.next_logprobs.append(lp)
                if (not sib.ignore_eos and tok in sib.finish_tokens) or \
                        len(sib.token_ids) - sib.prompt_len >= sib.output_len:
                    out.free_ids.append(sib.seq_id)
                    self.mm.free(sib)
                else:
                    self.seqs_to_decode.appendleft(sib)

    def _fan_out(self, ent: "ScheduledSeq"):
        """The final prompt chunk of a sequence with forks is scheduled (its pages are allocated): every fork takes
        the F full prompt pages (shared, reference counted: nobody writes them again) and, when the prompt ends
        inside a page, a fresh page that the device fills with a copy of page F right after this batch's forward."""
        seq, ps = ent.seq, self.page_size
        p = len(seq.token_ids)
        full = p // ps
        pairs = []
        for sib in seq.forks:
            sib.page_table = [self.mm.share_page(pg) for pg in seq.page_table[:full]]
            if p % ps:
                dst = self.mm.allocate_page()
                sib.page_table.append(dst)
                pairs.append((seq.page_table[full], dst))
            sib.computed_token_num = sib.scheduled_token_num = p
            sib.published = full     # the shared pages are the parent's to publish
            # the parent's prefill scores the prompt for every choice: a fork's recompute after a preemption must not
            # ask for those rows again
            sib.plp_cursor = max(sib.plp_cursor, sib.prompt_len - 1)
        ent.forks, ent.kv_copy = seq.forks, (pairs or None)
        seq.forks = []

    def _abort_forks(self, seq: Sequence, everything: bool, out: SchedulerOutput):
        """Forks still waiting with their parent (before its fan-out): drop the aborted ones, or all of them."""
        for sib in list(seq.forks):
            if everything or sib.seq_id in self.abort_ids:
                seq.forks.remove(sib)
                sib.is_abort = True
                out.free_ids.append(sib.seq_id)
                self.abort_ids.discard(sib.seq_id)

    def _in_flight(self, seq: Sequence) -> bool:
        return any(e.seq is seq for b in self.batch_running for e in b)

    def _drop_from_queues(self, seq: Sequence):
        for q in (self.seqs_to_prefill, self.seqs_to_decode):
            try:
                q.remove(seq)
            except ValueError:
                pass

    def schedule_lookahead(self) -> Optional[List["ScheduledSeq"]]:
        """Asynchronous scheduling: while the single in-flight decode batch is still running, schedule the decode
        step that follows it. The input token of every row is not known on the host yet — the sequence gets a
        PLACEHOLDER and the runner feeds the value from the previous step's device-side sampler output — so the
        GPU never waits for the host's output processing / scheduling / batch building. Returns None whenever the
        assumptions do not hold (more runnable sequences than one batch, penalties, split_pd, no KV headroom, ...),
        in which case the caller simply waits for the in-flight batch as before."""
        if self.pp_size != 1 or len(self.batch_running) != 1 or self.seqs_to_decode or self.next_tokens_queue or \
                self.abort_ids or self.schedule_method == "split_pd":
            return None
        base = self.batch_running[0]
        cont = []
        ps = self.page_size
        need = 0
        for ent in base:
            seq = ent.seq
            if not ent.emits:
                continue   # unfinished prefill chunk: its continuation is ordinary prefill work (tokens known)
            if seq.pending >= 0 or seq.repetition_penalty != 1.0 or seq.mm_state:
                return None
            if seq.is_abort or seq.zombie:
                continue
            if len(seq.token_ids) + 1 - seq.prompt_len >= seq.output_len:
                continue   # finishes by length with the token of the in-flight step
            cont.append(seq)
            if (len(seq.token_ids) + 1 + ps - 1) // ps > len(seq.page_table):
                need += 1
        if len(cont) > min(self.maxd, self.maxp) or self.mm.get_num_free_pages() < need + self.num_kvthresh_pages:
            return None
        if not cont and not self.seqs_to_prefill:
            return None
        entries = []
        for seq in reversed(cont):   # process_output re-queues head-first, so the next step sees the reverse order
            idx = len(seq.token_ids)
            seq.token_ids.append(PLACEHOLDER)
            seq.pending = idx
            seq.scheduled_token_num = idx + 1
            entries.append(ScheduledSeq(seq, idx, 1))
        self.mm.pre_allocate_page([e.seq for e in entries])
        n_prefill = 0
        if self.seqs_to_prefill:
            # new / continuing prompts ride along exactly as in the synchronous policies (their tokens are known)
            headroom = kv_headroom_tokens(self.mm.get_num_free_pages(), self.num_kvthresh_pages, self.page_size)
            if self.schedule_method == "token_throttling":
                if self.world_size > 1 and headroom != 0:
                    self.update_num_wait_tokens()
                budget = throttled_prefill_budget(headroom, self.world_size, self.mm.get_memory_free(), self.kvthresh,
                                                  self.maxp, self.minp, self.iterp, len(self.seqs_to_prefill),
                                                  self.num_wait_tokens)
            else:
                budget = min(self.maxp - len(entries), headroom)
            room = None if self.max_seqs is None else max(self.max_seqs - len(entries), 0)
            prefill_batch, n_prefill = self.schedule_prefill_batch(budget, room)
            entries = entries + prefill_batch
        if not entries:
            return None
        self._log_status(len(cont), n_prefill, len(cont))
        self.batch_running.append(entries)
        return entries

    def check_abort_seqs(self) -> Optional[SchedulerOutput]:
        if not self.abort_ids:
            return None
        out = SchedulerOutput()
        inflight = {id(e.seq) for b in self.batch_running for e in b}
        for q in (self.seqs_to_prefill, self.seqs_to_decode):
            for seq in list(q):
                if seq.forks:
                    self._abort_forks(seq, seq.seq_id in self.abort_ids, out)
                if seq.seq_id in self.abort_ids:
                    q.remove(seq)
                    seq.is_abort = True
                    if id(seq) in inflight:
                        continue  # a chunk is still in flight: freed when that batch returns
                    out.free_ids.append(seq.seq_id)
                    self.mm.free(seq)
                    self.abort_ids.discard(seq.seq_id)
        live = set()
        for batch in self.batch_running:
            for ent in batch:
                if ent.seq.seq_id in self.abort_ids:
                    ent.seq.is_abort = True
                    live.add(ent.seq.seq_id)
                for sib in ent.forks or ():      # fanned out in flight: freed when that batch returns
                    if sib.seq_id in self.abort_ids:
                        live.add(sib.seq_id)
        # an abort that matches nothing alive (the sequence finished just before, or was never admitted) must not
        # linger: it would disable lookahead scheduling for good and hit a later request that re-uses the id
        self.abort_ids &= live
        return out if out.free_ids else None

    # -- scheduling -------------------------------------------------------------------------------
    def can_schedule(self) -> bool:
        return bool(self.seqs_to_decode or self.seqs_to_prefill) and len(self.batch_running) < self.pp_size

    def schedule_once(self) -> List["ScheduledSeq"]:
        if not self.can_schedule():
            return []
        seqs = self._schedule()
        if not seqs and not self.batch_running and not self.seqs_to_decode and self._break_prefill_stall():
            seqs = self._schedule()
        if seqs:
            self.batch_running.append(seqs)
        return seqs

    def _schedule(self) -> List["ScheduledSeq"]:
        return self.token_throttling() if self.schedule_method == "token_throttling" else self.chunked_prefill()

    def _break_prefill_stall(self) -> bool:
        """Nothing is running, nothing could be scheduled, yet sequences are waiting: every free page is gone to
        partially prefilled sequences (preempted sequences re-enter at the head of the queue, in front of a
        half-prefilled one, so several of them can end up holding pages) and nobody can advance. Give back the
        pages of waiting sequences from the tail of the queue — they are recomputed later — until the head has
        room again. Returns whether anything was freed."""
        if len(self.seqs_to_prefill) < 2:
            return False
        head, freed = self.seqs_to_prefill[0], False
        for seq in reversed(self.seqs_to_prefill):
            if seq is head:
                break
            if seq.page_table:
                self.mm.free(seq)
                seq.preempt()
                if self.on_preempt is not None:
                    self.on_preempt(seq)
                self.num_preempt_seqs += 1
                freed = True
                if self.mm.get_num_free_pages() > self.num_kvthresh_pages:
                    break
        return freed

    def check_preempt(self, num_pages_to_allocate: int):
        preempted = []
        while self.mm.get_num_free_pages() < num_pages_to_allocate and self.seqs_to_decode:
            seq = self.seqs_to_decode.popleft()
            self.mm.free(seq)
            seq.preempt()
            if self.on_preempt is not None:
                self.on_preempt(seq)
            preempted.append(seq)
        if preempted:
            self.seqs_to_prefill.extendleft(preempted)
            self.num_preempt_seqs += len(preempted)
            if self.num_preempt_seqs >= self._log_preempt_at:
                self._log_preempt_at *= 2
                logger.warning("#Preempted seqs: %d, try increasing --kvthresh or performance will be poor!",
                               self.num_preempt_seqs)

    def schedule_decode_batch(self, budget: int) -> List["ScheduledSeq"]:
        self.check_preempt(min(budget, len(self.seqs_to_decode)))
        batch = []
        seqs = []
        for _ in range(budget):
            if not self.seqs_to_decode:
                break
            seq = self.seqs_to_decode.popleft()
            start = seq.computed_token_num
            seq.scheduled_token_num = start + 1
            batch.append(ScheduledSeq(seq, start, 1))
            seqs.append(seq)
        self.mm.pre_allocate_page(seqs)
        return batch

    def schedule_prefill_batch(self, budget: int, room: Optional[int] = None):
        """`room`: how many more sequences the micro-batch may take (None = unlimited)."""
        batch: List[ScheduledSeq] = []
        n_tokens = 0
        fork_rows = 0    # extra sampled rows of the fan-outs in this batch (each takes a sequence slot of the runner)
        while self.seqs_to_prefill and budget > 0 and (room is None or len(batch) + fork_rows < room):
            seq = self.seqs_to_prefill[0]
            if isinstance(self.mm, PrefixMemoryManager) and seq.scheduled_token_num == 0 and not seq.page_table:
                self.mm.pre_allocate_computed_page([seq])
            start = seq.scheduled_token_num
            remaining = len(seq) - start
            take = min(remaining, budget)
            seq.scheduled_token_num = start + take
            fan = seq.forks if take == remaining else None
            need = self.mm.pages_needed(seq)
            if fan:
                need += len(fan) if len(seq) % self.page_size else 0
                if room is not None and len(batch) + fork_rows + 1 + len(fan) > room:
                    seq.scheduled_token_num = start
                    break  # no room for the choices' rows in this batch: the chunk waits
            if need > self.mm.get_num_free_pages():
                seq.scheduled_token_num = start
                break  # no KV room right now
            self.mm.pre_allocate_page([seq])
            n_tokens += take
            budget -= take
            ent = ScheduledSeq(seq, start, take)
            if fan:
                self._fan_out(ent)
                fork_rows += len(ent.forks)
            batch.append(ent)
            if take == remaining:
                self.seqs_to_prefill.popleft()
            # else: unfinished prefill stays at the queue head and continues with its next chunk —
            # possibly while this one is still in flight when pp_size > 1 (the reference deep-copies
            # the sequence for that, gllm/scheduler.py:226-231)
        return batch, n_tokens

    def chunked_prefill(self) -> List["ScheduledSeq"]:
        budget = self.maxp
        num_total_decode = self.get_num_decode_seqs()
        decode_budget = min(balanced_decode_budget(num_total_decode, self.pp_size, self.maxd), budget)
        # split_pd: prefill has priority while there is KV headroom for it. (Strictly positive headroom: with
        # free pages == threshold neither phase would be scheduled and the engine would stall.)
        if self.schedule_method == "split_pd" and self.seqs_to_prefill and \
                kv_headroom_tokens(self.mm.get_num_free_pages(), self.num_kvthresh_pages, self.page_size) > 0:
            decode_budget = 0
        decode_batch = self.schedule_decode_batch(decode_budget)
        budget -= len(decode_batch)
        budget = min(budget, kv_headroom_tokens(self.mm.get_num_free_pages(), self.num_kvthresh_pages,
                                                 self.page_size))
        room = None if self.max_seqs is None else max(self.max_seqs - len(decode_batch), 0)
        prefill_batch, n_prefill = self.schedule_prefill_batch(budget, room)
        self._log_status(num_total_decode, n_prefill, len(decode_batch))
        return decode_batch + prefill_batch

    def token_throttling(self) -> List["ScheduledSeq"]:
        headroom = kv_headroom_tokens(self.mm.get_num_free_pages(), self.num_kvthresh_pages, self.page_size)
        if self.world_size > 1 and headroom != 0:
            self.update_num_wait_tokens()
        budget = throttled_prefill_budget(headroom, self.world_size, self.mm.get_memory_free(), self.kvthresh,
                                          self.maxp, self.minp, self.iterp, len(self.seqs_to_prefill),
                                          self.num_wait_tokens)
        num_total_decode = self.get_num_decode_seqs()
        decode_budget = balanced_decode_budget(num_total_decode, self.pp_size, self.maxd)
        room = None if self.max_seqs is None else \
            max(self.max_seqs - min(decode_budget, len(self.seqs_to_decode)), 0)     # decode rows come first
        prefill_batch, n_prefill = self.schedule_prefill_batch(budget, room)
        decode_batch = self.schedule_decode_batch(decode_budget)
        self._log_status(num_total_decode, n_prefill, len(decode_batch))
        return decode_batch + prefill_batch

    def _log_status(self, num_run: int, n_prefill: int, n_decode: int):
        self.last_stats = {"wait": len(self.seqs_to_prefill), "run": num_run, "prefill_tokens": n_prefill,
                           "decode_seqs": n_decode, "memory_util": self.mm.get_memory_util(),
                           "cache_hit_rate": self.mm.get_cache_hit_rate(), "preempted": self.num_preempt_seqs}
        if self.log and time.time() - self.log_time > 1:
            self.log_time = time.time()
            msg = "#wait: %4d #run: %4d #prefill: %4d #decode: %4d memory_util: %5.2f %%" % (
                len(self.seqs_to_prefill), num_run, n_prefill, n_decode, self.mm.get_memory_util())
            if isinstance(self.mm, PrefixMemoryManager):
                msg += " cache_hit_rate: %5.2f %%" % self.mm.get_cache_hit_rate()
            logger.info(msg)
