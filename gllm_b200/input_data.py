"""Batch -> tensors (reference: gllm/input_data.py).

The driver rank turns a scheduled micro-batch (decode entries first, then prefill chunks) into
one flat `BatchArrays` bundle of int32/float32 numpy arrays. That bundle is (a) copied into
persistent pinned staging + persistent device buffers (stable addresses for CUDA graphs) and
(b) shipped verbatim to every other rank, which therefore needs neither the Sequence objects nor
a Python rebuild of the batch (the reference re-runs the per-token Python loops on every rank,
gllm/worker.py:131-136).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch


class _DtypeCache(dict):
    def __missing__(self, key):
        self[key] = np.dtype(key)
        return self[key]


_WIRE_DTYPES = _DtypeCache()


@dataclass
class BatchArrays:
    """Host-side description of one micro-batch. All arrays are contiguous numpy."""
    tokens: np.ndarray            # int32 [T]
    positions: np.ndarray         # int32 [T] or [3, T] (M-RoPE)
    slot_mapping: np.ndarray      # int32 [T]
    block_table: np.ndarray       # int32 [B, max_blocks_in_batch]
    seq_lens: np.ndarray          # int32 [B]   KV length after this step
    query_start_loc: np.ndarray   # int32 [B + 1]
    logits_idx: np.ndarray        # int32 [E]   rows whose logits are needed (last token of emitting seqs)
    emit_seq: np.ndarray          # int32 [E]   index into the batch of each emitting seq
    temperature: np.ndarray       # float32 [E]
    top_k: np.ndarray             # int32 [E]
    top_p: np.ndarray             # float32 [E]
    rep_penalty: np.ndarray       # float32 [E]
    state_slot: np.ndarray        # int32 [E]   row in the persistent per-sequence device state
    num_decode_seqs: int = 0
    num_seqs: int = 0
    num_tokens: int = 0
    max_q_len: int = 0
    max_seq_len: int = 0
    all_greedy: bool = True
    need_penalty: bool = False
    # prompt tokens that must be marked in the repetition-penalty bitmask this step
    seen_rows: Optional[np.ndarray] = None   # int32 [P] state_slot per token
    seen_tokens: Optional[np.ndarray] = None  # int32 [P]
    clear_slots: Optional[np.ndarray] = None  # int32: bitmask rows to zero first (slot re-use)
    batch_id: int = 0
    mm: Optional[dict] = None  # multimodal payload (pixel values, grids) for the first stage
    # lookahead (async scheduling): row i takes its input token from element feed_src[i] of the PREVIOUS step's
    # device-side sampler output instead of `tokens[i]` (which holds a placeholder)
    feed_src: Optional[np.ndarray] = None
    # int32 [E]: top alternatives whose log-probs each emitting row wants (-1: none); None when no row asks
    logprobs_n: Optional[np.ndarray] = None
    # frequency / presence penalties and logit_bias (None unless `need_bias`): per emitting row the penalties and the
    # slot of its bias row on the device (-1: none)
    need_bias: bool = False
    freq_pen: Optional[np.ndarray] = None    # float32 [E]
    pres_pen: Optional[np.ndarray] = None    # float32 [E]
    bias_slot: Optional[np.ndarray] = None   # int32 [E]
    # bias rows to rebuild first (slot (re)assigned): slot, (frequency, presence), the request's logit_bias entries and
    # the output tokens generated so far, concatenated with [R + 1] offsets
    rb_slots: Optional[np.ndarray] = None    # int32 [R]
    rb_pen: Optional[np.ndarray] = None      # float32 [R, 2]
    rb_lb_off: Optional[np.ndarray] = None   # int32 [R + 1]
    rb_lb_ids: Optional[np.ndarray] = None   # int32
    rb_lb_vals: Optional[np.ndarray] = None  # float32
    rb_out_off: Optional[np.ndarray] = None  # int32 [R + 1]
    rb_out_toks: Optional[np.ndarray] = None  # int32
    # seeded rows (None when no row has a seed): request seed and position of the token being produced (-1: unseeded)
    seed: Optional[np.ndarray] = None        # int64 [E]
    seed_pos: Optional[np.ndarray] = None    # int32 [E]
    # parallel sampling: (src, dst) KV pages every rank copies for its own layers right after this batch's forward
    # (the partial last prompt page of a request that fans out into several choices); None when there is none
    kv_copy: Optional[np.ndarray] = None     # int32 [C, 2]
    # prompt log-probabilities: rows (in the batch's token order) whose logits score the next prompt token, that
    # token, and the largest N any of them asks for; None / -1 when no row asks
    plp_rows: Optional[np.ndarray] = None    # int32 [Q]
    plp_targets: Optional[np.ndarray] = None  # int32 [Q]
    plp_n: int = -1
    # multi-LoRA: adapter slot of every token row (-1: base model); None when no row uses an adapter
    lora_slot: Optional[np.ndarray] = None   # int32 [T]
    emit_ids: Optional[list] = None  # driver-local: sequence id per EMITTING entry (order of the sampler output)
    seq_ids: Optional[list] = None  # driver-local: sequence id per row (incremental decode batches); not sent
    pt_gens: Optional[list] = None  # driver-local: Sequence.pt_gen per row when the block table rows were written
    seq_index: Optional[dict] = None  # driver-local: seq id -> row (built lazily by the next batch)

    def is_decode_only(self) -> bool:
        return self.num_decode_seqs == self.num_seqs

    @property
    def plain_greedy(self) -> bool:
        """Every emitting row takes the argmax of its raw logits: no penalty, bias or sampling parameter to apply."""
        return self.all_greedy and not self.need_penalty and not self.need_bias

    def to_wire(self):
        """(header dict, [one contiguous buffer]) for zero-copy IPC: every array is packed into a single blob
        (16-byte aligned sections) so a batch costs two zmq frames per peer instead of one per array."""
        names = ["tokens", "positions", "slot_mapping", "block_table", "seq_lens", "query_start_loc",
                 "logits_idx", "emit_seq", "temperature", "top_k", "top_p", "rep_penalty", "state_slot"]
        opt = ["seen_rows", "seen_tokens", "clear_slots", "feed_src", "logprobs_n", "freq_pen", "pres_pen",
               "bias_slot", "rb_slots", "rb_pen", "rb_lb_off", "rb_lb_ids", "rb_lb_vals", "rb_out_off", "rb_out_toks",
               "seed", "seed_pos", "kv_copy", "plp_rows", "plp_targets", "lora_slot"]
        scalars = (self.num_decode_seqs, self.num_seqs, self.num_tokens, self.max_q_len, self.max_seq_len,
                   self.all_greedy, self.need_penalty, self.batch_id)
        if self.need_bias:      # (only then: a batch without the feature sends the header it always sent)
            scalars += (True,)
        hdr = {"scalars": scalars, "arrays": [], "mm": self.mm}
        if self.plp_rows is not None:
            hdr["plp_n"] = self.plp_n
        parts, off = [], 0
        for n in names + opt:
            a = getattr(self, n)
            if a is None:
                continue
            a = np.ascontiguousarray(a)
            hdr["arrays"].append((n, a.dtype.str, a.shape, off))
            parts.append(a)
            off += (a.nbytes + 15) // 16 * 16
        blob = np.empty(max(off, 16), dtype=np.uint8)
        for (_, _, _, o), a in zip(hdr["arrays"], parts):
            blob[o:o + a.nbytes] = a.reshape(-1).view(np.uint8)
        return hdr, [blob]

    @staticmethod
    def from_wire(hdr, bufs) -> "BatchArrays":
        kw = {}
        blob = bufs[0]
        for n, dt, shape, off in hdr["arrays"]:
            if len(shape) == 1:     # (hot path on every peer every step: no np.prod / reshape for 1-D arrays)
                kw[n] = np.frombuffer(blob, dtype=_WIRE_DTYPES[dt], count=shape[0], offset=off)
            else:
                kw[n] = np.frombuffer(blob, dtype=_WIRE_DTYPES[dt], count=math.prod(shape), offset=off).reshape(shape)
        s = hdr["scalars"]
        return BatchArrays(**kw, num_decode_seqs=s[0], num_seqs=s[1], num_tokens=s[2], max_q_len=s[3],
                           max_seq_len=s[4], all_greedy=s[5], need_penalty=s[6], batch_id=s[7], mm=hdr.get("mm"),
                           need_bias=len(s) > 8 and s[8], plp_n=hdr.get("plp_n", -1))


def _page_array(seq) -> np.ndarray:
    """numpy view of the page table; converting the Python list every step costs O(pages) per sequence, so the
    mirror is rebuilt only when the table changed length (every `page_size` tokens) or was reset."""
    pt = seq.pt_np
    n = len(seq.page_table)
    if pt is None or pt.shape[0] != n or (n and (pt[0] != seq.page_table[0] or pt[-1] != seq.page_table[-1])):
        pt = np.asarray(seq.page_table, dtype=np.int32)
        seq.pt_np = pt
    return pt


def _build_decode_fast(entries, page_size: int, batch_id: int, prev: "BatchArrays") -> Optional["BatchArrays"]:
    """Steady-state decode: the same sequences as the previous micro-batch, one new token each. Everything is
    derived from the previous arrays with vectorised numpy (new arrays, never in place: zero-copy zmq sends may
    still reference the old ones); only rows that crossed a page boundary touch their Python page table."""
    b = len(entries)
    # (a SUBSET of the previous rows is fine too: sequences finish all the time and the survivors keep decoding)
    if prev is None or prev.seq_ids is None or b > prev.num_seqs or prev.num_decode_seqs != prev.num_seqs \
            or prev.need_penalty or prev.mm is not None or prev.positions.ndim != 1:
        return None
    # the scheduler re-queues finished-step sequences head-first, so the row order flips between iterations:
    # map every entry to its row in the previous batch
    where = prev.seq_index
    if where is None:
        where = {sid: i for i, sid in enumerate(prev.seq_ids)}
        prev.seq_index = where
    try:   # one pass over the entries: (previous row, position, token, seq id)
        data = [(where[e.seq.seq_id], e.start, e.seq.token_ids[e.start], e.seq.seq_id, e.seq.pt_gen)
                if e.n == 1 and e.emits else None for e in entries]
        arr = np.array(data, dtype=np.int64)
    except (KeyError, TypeError, ValueError):
        return None
    if arr.ndim != 2:
        return None
    perm = arr[:, 0]
    starts = arr[:, 1].astype(np.int32)
    tokens = arr[:, 2].astype(np.int32)
    ids = arr[:, 3].tolist()
    gens = arr[:, 4].tolist()
    if not np.array_equal(starts, prev.positions[perm] + 1):
        return None
    # a sequence that was preempted and whose recompute ends in a 1-token tail looks like a decode row, but its
    # page table was rebuilt (other physical pages, e.g. prefix-cache hits): the previous block-table row is stale
    if prev.pt_gens is None or [prev.pt_gens[i] for i in perm.tolist()] != gens:
        return None
    blk = starts // page_size
    bt = prev.block_table[perm]              # fancy indexing: a new array
    width = int(blk.max()) + 1
    if width > bt.shape[1]:
        bt = np.concatenate([bt, np.zeros((b, width - bt.shape[1]), dtype=np.int32)], axis=1)
    for i in np.nonzero(starts % page_size == 0)[0]:      # first token of a fresh page
        bt[i, blk[i]] = entries[i].seq.page_table[blk[i]]
    rows = np.arange(b, dtype=np.int32)
    slots = bt[rows, blk] * page_size + starts % page_size
    seq_lens = starts + 1
    feed = perm.astype(np.int32) if (tokens < 0).any() else None   # lookahead rows: token still on the device
    lp_n = prev.logprobs_n[perm] if prev.logprobs_n is not None else None
    if lp_n is not None and not (lp_n >= 0).any():
        lp_n = None        # the rows that asked have finished: the batch is what it would be without the feature
    bias = {}
    if prev.need_bias:
        if any(e.seq.slot_fresh for e in entries):
            return None    # a bias row to rebuild: the full path sends it
        bslot = prev.bias_slot[perm]
        if (bslot >= 0).any():
            bias = dict(need_bias=True, bias_slot=bslot, freq_pen=prev.freq_pen[perm], pres_pen=prev.pres_pen[perm])
    lora = prev.lora_slot[perm] if prev.lora_slot is not None else None
    if lora is not None and not (lora >= 0).any():
        lora = None        # the adapter rows have finished
    seed = seed_pos = None
    if prev.seed_pos is not None:
        seed_pos = prev.seed_pos[perm]
        if (seed_pos >= 0).any():
            seed, seed_pos = prev.seed[perm], np.where(seed_pos >= 0, seed_pos + 1, -1).astype(np.int32)
        else:
            seed_pos = None
    return BatchArrays(feed_src=feed,
        tokens=tokens, positions=starts, slot_mapping=slots.astype(np.int32), block_table=bt, seq_lens=seq_lens,
        query_start_loc=prev.query_start_loc[:b + 1], logits_idx=prev.logits_idx[:b], emit_seq=prev.emit_seq[:b],
        temperature=prev.temperature[perm], top_k=prev.top_k[perm], top_p=prev.top_p[perm],
        rep_penalty=prev.rep_penalty[perm], state_slot=prev.state_slot[perm],
        logprobs_n=lp_n, num_decode_seqs=b, num_seqs=b, num_tokens=b, max_q_len=1,
        max_seq_len=int(seq_lens.max()), all_greedy=prev.all_greedy, need_penalty=False, batch_id=batch_id,
        seq_ids=ids, emit_ids=ids, pt_gens=gens, seed=seed, seed_pos=seed_pos, lora_slot=lora, **bias)


def _bias_fields(freq_pen, pres_pen, bias_slot, rb_slots, rb_pen, rb_lb_off, rb_lb_ids, rb_lb_vals, rb_out_off,
                 rb_out_toks) -> dict:
    out = dict(need_bias=True, freq_pen=np.asarray(freq_pen, dtype=np.float32),
               pres_pen=np.asarray(pres_pen, dtype=np.float32), bias_slot=np.asarray(bias_slot, dtype=np.int32))
    if rb_slots:
        out.update(rb_slots=np.asarray(rb_slots, dtype=np.int32), rb_pen=np.asarray(rb_pen, dtype=np.float32),
                   rb_lb_off=np.asarray(rb_lb_off, dtype=np.int32), rb_lb_ids=np.asarray(rb_lb_ids, dtype=np.int32),
                   rb_lb_vals=np.asarray(rb_lb_vals, dtype=np.float32),
                   rb_out_off=np.asarray(rb_out_off, dtype=np.int32),
                   rb_out_toks=np.asarray(rb_out_toks, dtype=np.int32))
    return out


def build_batch(entries, page_size: int, vocab_size: int, batch_id: int = 0, mrope: bool = False,
                prev: Optional["BatchArrays"] = None) -> BatchArrays:
    """entries: List[ScheduledSeq], decode entries first (scheduler invariant). `prev` (the previous
    micro-batch of this engine) enables the incremental decode fast path."""
    b = len(entries)
    if prev is not None and not mrope and b:
        fast = _build_decode_fast(entries, page_size, batch_id, prev)
        if fast is not None:
            return fast
    n_dec = 0
    for e in entries:
        if e.is_decode:
            n_dec += 1
        else:
            break
    q_lens = np.fromiter((e.n for e in entries), dtype=np.int32, count=b)
    starts = np.fromiter((e.start for e in entries), dtype=np.int32, count=b)
    seq_lens = starts + q_lens
    qsl = np.zeros(b + 1, dtype=np.int32)
    np.cumsum(q_lens, out=qsl[1:])
    t = int(qsl[-1])
    tokens = np.empty(t, dtype=np.int32)
    positions = np.empty((3, t) if mrope else t, dtype=np.int32)
    slots = np.empty(t, dtype=np.int32)
    max_blocks = int((seq_lens.max() + page_size - 1) // page_size) if b else 1
    block_table = np.zeros((b, max_blocks), dtype=np.int32)

    emit_seq, logits_idx = [], []
    temperature, top_k, top_p, rep_pen, state_slot = [], [], [], [], []
    seen_rows, seen_tokens, clear_slots = [], [], []
    logprobs_n, want_logprobs = [], False
    all_greedy, need_penalty = True, False
    freq_pen, pres_pen, bias_slot, need_bias = [], [], [], False
    rb_slots, rb_pen, rb_lb_ids, rb_lb_vals, rb_out_toks, rb_lb_off, rb_out_off = [], [], [], [], [], [0], [0]
    seeds, seed_pos, want_seed = [], [], False
    emit_rows, fork_rows, kv_copy = [], [], []   # (entry, logits row, sequence, end of its known tokens)
    plp_rows, plp_targets, plp_n = [], [], -1
    for i, e in enumerate(entries):
        seq = e.seq
        pt = _page_array(seq)
        npg = (int(seq_lens[i]) + page_size - 1) // page_size
        block_table[i, :npg] = pt[:npg]
        a, z = int(qsl[i]), int(qsl[i + 1])
        s0 = e.start
        if e.n == 1:
            tokens[a] = seq.token_ids[s0]
            if mrope:
                positions[:, a] = (s0 + seq.mrope_delta) if (not seq.mm_state or s0 >= seq.prompt_len) \
                    else seq.mm_state["positions"][:, s0]
            else:
                positions[a] = s0
            slots[a] = pt[s0 // page_size] * page_size + s0 % page_size
        else:
            tokens[a:z] = seq.token_ids[s0:s0 + e.n]
            pos = np.arange(s0, s0 + e.n, dtype=np.int32)
            if mrope:
                from gllm_b200.models.multimodal import seq_positions
                positions[:, a:z] = seq_positions(seq, s0, e.n)
            else:
                positions[a:z] = pos
            slots[a:z] = pt[pos // page_size] * page_size + pos % page_size
        if seq.prompt_logprobs_n >= 0 and not e.is_decode:
            # prompt positions [lo, hi) score tokens lo + 1 .. hi; position P - 1 is the sampled row. The cursor makes
            # every position go out once, whatever the chunking or a recompute after preemption.
            lo, hi = max(s0, seq.plp_cursor), min(s0 + e.n, seq.prompt_len - 1)
            if hi > lo:
                assert lo == seq.plp_cursor, (seq.seq_id, s0, seq.plp_cursor)
                plp_rows.append(np.arange(a + lo - s0, a + hi - s0, dtype=np.int32))
                plp_targets.append(np.asarray(seq.token_ids[lo + 1:hi + 1], dtype=np.int32))
                plp_n = max(plp_n, seq.prompt_logprobs_n)
                seq.plp_cursor = hi
                e.plp = hi - lo
        if e.emits:
            emit_rows.append((i, z - 1, seq, s0 + e.n))
            for sib in e.forks or ():        # parallel sampling: the other choices draw from the same logits row
                fork_rows.append((i, z - 1, sib, s0 + e.n))
            if e.kv_copy:
                kv_copy.extend(e.kv_copy)
    emit_ids = []
    for i, row, seq, end in emit_rows + fork_rows:
        emit_seq.append(i)
        emit_ids.append(seq.seq_id)
        logits_idx.append(row)
        temperature.append(seq.temperature)
        k = seq.top_k
        top_k.append(vocab_size if (k is None or k <= 0 or k > vocab_size) else k)
        top_p.append(seq.top_p)
        rep_pen.append(seq.repetition_penalty)
        state_slot.append(seq.slot)
        logprobs_n.append(seq.logprobs)
        if seq.logprobs >= 0:
            want_logprobs = True
        if top_k[-1] != 1:
            all_greedy = False
        # the state row was just (re)assigned — first emission, or first one after a preemption: its contents are
        # rebuilt from everything known so far
        fresh = seq.slot_fresh
        seq.slot_fresh = False
        if seq.seed is not None:
            want_seed = True
            seeds.append(seq.seed)
            seed_pos.append(end)               # index of the token this step produces
        else:
            seeds.append(0)
            seed_pos.append(-1)
        if seq.has_bias_row:
            need_bias = True
            bias_slot.append(seq.slot)
            freq_pen.append(seq.frequency_penalty)
            pres_pen.append(seq.presence_penalty)
            if fresh:
                rb_slots.append(seq.slot)
                rb_pen.append((seq.frequency_penalty, seq.presence_penalty))
                lb = seq.logit_bias or {}
                rb_lb_ids.extend(lb.keys())
                rb_lb_vals.extend(lb.values())
                rb_lb_off.append(len(rb_lb_ids))
                rb_out_toks.extend(seq.token_ids[seq.prompt_len:end])
                rb_out_off.append(len(rb_out_toks))
        else:
            bias_slot.append(-1)
            freq_pen.append(0.0)
            pres_pen.append(0.0)
        if seq.repetition_penalty != 1.0:
            need_penalty = True
            if fresh:
                # everything known so far (prompt and the tokens generated before) becomes "seen"
                clear_slots.append(seq.slot)
                seen_rows.append(np.full(end, seq.slot, dtype=np.int32))
                seen_tokens.append(np.asarray(seq.token_ids[:end], dtype=np.int32))
            else:
                n = entries[i].n
                seen_rows.append(np.full(n, seq.slot, dtype=np.int32))
                seen_tokens.append(np.asarray(seq.token_ids[end - n:end], dtype=np.int32))
    lora_slot = None
    if any(e.seq.lora_id for e in entries):
        lora_slot = np.repeat(np.fromiter((e.seq.lora_id - 1 for e in entries), dtype=np.int32, count=b), q_lens)
    mm = None
    if mrope:
        from gllm_b200.models.multimodal import batch_mm_payload
        mm = batch_mm_payload(entries, qsl)
    return BatchArrays(
        tokens=tokens, positions=positions, slot_mapping=slots, block_table=block_table, seq_lens=seq_lens,
        query_start_loc=qsl, logits_idx=np.asarray(logits_idx, dtype=np.int32),
        emit_seq=np.asarray(emit_seq, dtype=np.int32), temperature=np.asarray(temperature, dtype=np.float32),
        top_k=np.asarray(top_k, dtype=np.int32), top_p=np.asarray(top_p, dtype=np.float32),
        rep_penalty=np.asarray(rep_pen, dtype=np.float32), state_slot=np.asarray(state_slot, dtype=np.int32),
        num_decode_seqs=n_dec, num_seqs=b, num_tokens=t, max_q_len=int(q_lens.max()) if b else 0,
        max_seq_len=int(seq_lens.max()) if b else 0, all_greedy=all_greedy, need_penalty=need_penalty,
        seen_rows=np.concatenate(seen_rows) if seen_rows else None,
        seen_tokens=np.concatenate(seen_tokens) if seen_tokens else None,
        clear_slots=np.asarray(clear_slots, dtype=np.int32) if clear_slots else None, batch_id=batch_id, mm=mm,
        logprobs_n=np.asarray(logprobs_n, dtype=np.int32) if want_logprobs else None,
        seed=np.asarray(seeds, dtype=np.int64) if want_seed else None,
        seed_pos=np.asarray(seed_pos, dtype=np.int32) if want_seed else None,
        kv_copy=np.asarray(kv_copy, dtype=np.int32).reshape(-1, 2) if kv_copy else None,
        plp_rows=np.concatenate(plp_rows) if plp_rows else None,
        plp_targets=np.concatenate(plp_targets) if plp_rows else None, plp_n=plp_n, lora_slot=lora_slot,
        **(_bias_fields(freq_pen, pres_pen, bias_slot, rb_slots, rb_pen, rb_lb_off, rb_lb_ids, rb_lb_vals, rb_out_off,
                        rb_out_toks) if need_bias else {}),
        seq_ids=[e.seq.seq_id for e in entries] if n_dec == b else None,
        pt_gens=[e.seq.pt_gen for e in entries] if n_dec == b else None,
        emit_ids=emit_ids)


class InputData:
    """Persistent device-side batch state (stable addresses => CUDA-graph friendly).

    One instance per worker. `load(batch)` copies a `BatchArrays` into pinned staging and then
    into the device buffers with a single non-blocking H2D per array.
    """

    def __init__(self, max_tokens: int, max_seqs: int, max_blocks: int, device, mrope: bool = False):
        self.device = torch.device(device)
        self.max_tokens, self.max_seqs, self.max_blocks = max_tokens, max_seqs, max_blocks
        self.mrope = mrope
        pin = self.device.type == "cuda"
        i32, f32 = torch.int32, torch.float32

        def buf(shape, dtype):
            # TWO pinned staging buffers per array, alternated every step: with asynchronous scheduling the host
            # assembles step N+1 while the H2D copies of step N may still be queued behind step N-1's kernels
            hosts = [torch.zeros(shape, dtype=dtype, pin_memory=pin) for _ in range(2)]
            return ([(h, h.numpy()) for h in hosts], torch.zeros(shape, dtype=dtype, device=self.device))

        self._flip = 0

        self._tokens = buf((max_tokens,), i32)
        self._positions = buf((3, max_tokens) if mrope else (max_tokens,), i32)
        self._slots = buf((max_tokens,), i32)
        self._block_table = buf((max_seqs, max_blocks), i32)
        self._seq_lens = buf((max_seqs,), i32)
        self._qsl = buf((max_seqs + 1,), i32)
        self._logits_idx = buf((max_seqs,), i32)
        self._temperature = buf((max_seqs,), f32)
        self._top_k = buf((max_seqs,), i32)
        self._top_p = buf((max_seqs,), f32)
        self._rep_penalty = buf((max_seqs,), f32)
        self._state_slot = buf((max_seqs,), i32)
        self._tok_seq = buf((max_tokens,), i32)
        self._feed = buf((max_seqs,), i32)
        self._freq_pen = buf((max_seqs,), f32)
        self._pres_pen = buf((max_seqs,), f32)
        self._bias_slot = buf((max_seqs,), i32)
        self._seed = buf((max_seqs,), torch.int64)
        self._seed_pos = buf((max_seqs,), i32)
        self._buf = buf
        self._plp = None   # (rows, targets) of prompt log-prob rows: allocated by the first batch that has them
        self.lora_adapters = 0   # number of adapters the engine serves (`set_lora`)
        self.lora_groups = 0     # adapter groups of the loaded batch (the graph capture pins it to lora_adapters)
        self._lora_h2d = 0
        self.need_tok_seq = False  # MLA attention wants token -> sequence for mixed / prefill batches
        self.batch: Optional[BatchArrays] = None
        self.num_tokens = self.num_seqs = self.num_decode_seqs = self.num_emit = 0
        self.max_q_len = self.max_seq_len = 0
        self.padded_tokens = 0  # > 0 when padded to a CUDA-graph bucket
        self.decode_splits = None  # None: pick per batch (eager); int: fixed (CUDA graphs)

    def set_lora(self, num_adapters: int):
        """Allocate the per-batch adapter CSR (see csrc/lora/lora.cu): slots [L], row_off [L + 1], rows [T]."""
        self.lora_adapters = num_adapters
        self._lora = (self._buf((num_adapters,), torch.int32), self._buf((num_adapters + 1,), torch.int32),
                      self._buf((self.max_tokens,), torch.int32))

    def _load_lora(self, lora_slot: np.ndarray):
        """Group the token rows by adapter: the S active slots in increasing order, then the rows without one. row_off
        is padded to L + 1 entries with the end of the adapter rows, so a kernel launched for L groups (CUDA graphs)
        sees the extra groups empty."""
        n_ad = self.lora_adapters
        key = np.where(lora_slot < 0, n_ad, lora_slot)
        rows = np.argsort(key, kind="stable").astype(np.int32)
        counts = np.bincount(key, minlength=n_ad + 1)[:n_ad]
        slots = np.nonzero(counts)[0].astype(np.int32)
        off = np.empty(n_ad + 1, dtype=np.int32)
        off[0] = 0
        np.cumsum(counts[slots], out=off[1:slots.shape[0] + 1])
        off[slots.shape[0] + 1:] = off[slots.shape[0]]
        self.lora_groups = int(slots.shape[0])
        if slots.shape[0]:
            self._put(self._lora[0], slots)
        self._put(self._lora[1], off)
        self._put(self._lora[2], rows)
        self._lora_h2d = slots.nbytes + off.nbytes + rows.nbytes

    def _put(self, pair, arr: np.ndarray):
        """numpy array -> this step's pinned staging buffer (plain numpy store through a shared-memory view: no
        tensor wrapping per array) -> one non-blocking H2D copy."""
        stages, dev = pair
        host, host_np = stages[self._flip]
        if arr.ndim == 1:
            n = arr.shape[0]
            host_np[:n] = arr
            dev[:n].copy_(host[:n], non_blocking=True)
        else:
            r, c = arr.shape
            host_np[:r, :c] = arr
            dev[:r, :c].copy_(host[:r, :c], non_blocking=True)

    def load(self, batch: BatchArrays):
        assert batch.num_tokens <= self.max_tokens, (batch.num_tokens, self.max_tokens)
        assert batch.num_seqs <= self.max_seqs, (batch.num_seqs, self.max_seqs)
        assert batch.block_table.shape[1] <= self.max_blocks
        self.batch = batch
        self._flip ^= 1
        self.num_tokens, self.num_seqs = batch.num_tokens, batch.num_seqs
        self.num_decode_seqs = batch.num_decode_seqs
        self.num_emit = int(batch.logits_idx.shape[0])
        self.max_q_len, self.max_seq_len = batch.max_q_len, batch.max_seq_len
        self.padded_tokens = 0
        self._put(self._tokens, batch.tokens)
        if self.mrope:
            pos = batch.positions if batch.positions.ndim == 2 else np.broadcast_to(batch.positions, (3, batch.num_tokens))
            self._put(self._positions, pos)
        else:
            self._put(self._positions, batch.positions if batch.positions.ndim == 1 else batch.positions[0])
        self._put(self._slots, batch.slot_mapping)
        if self.need_tok_seq and not batch.is_decode_only():
            qsl = batch.query_start_loc
            self._put(self._tok_seq, np.repeat(np.arange(batch.num_seqs, dtype=np.int32), np.diff(qsl)))
        if batch.feed_src is not None:
            self._put(self._feed, batch.feed_src)
        if batch.plp_rows is not None:
            if self._plp is None:
                self._plp = (self._buf((self.max_tokens,), torch.int32), self._buf((self.max_tokens,), torch.int32))
            self._put(self._plp[0], batch.plp_rows)
            self._put(self._plp[1], batch.plp_targets)
        if batch.lora_slot is not None:
            self._load_lora(batch.lora_slot)
        self._put(self._block_table, batch.block_table)
        self._put(self._seq_lens, batch.seq_lens)
        self._put(self._qsl, batch.query_start_loc)
        if self.num_emit:
            self._put(self._logits_idx, batch.logits_idx)
            # the greedy argmax path of the sm_90a sampler reads none of these
            if not (self.device.type == "cuda" and batch.plain_greedy):
                self._put(self._temperature, batch.temperature)
                self._put(self._top_k, batch.top_k)
                self._put(self._top_p, batch.top_p)
                self._put(self._rep_penalty, batch.rep_penalty)
                self._put(self._state_slot, batch.state_slot)
            # per-request sampling parameters: staged only when some row uses them
            if batch.need_bias:
                self._put(self._freq_pen, batch.freq_pen)
                self._put(self._pres_pen, batch.pres_pen)
                self._put(self._bias_slot, batch.bias_slot)
            if batch.seed is not None:
                self._put(self._seed, batch.seed)
                self._put(self._seed_pos, batch.seed_pos)

    def apply_feed(self, prev_tokens_out: torch.Tensor):
        """Lookahead step: the input tokens are the previous step's sampled tokens, still on the device."""
        b = self.batch.feed_src.shape[0]
        idx = self._feed[1][:b]
        self._tokens[1][:b].copy_(prev_tokens_out.index_select(0, idx.long() if prev_tokens_out.device.type == "cpu"
                                                               else idx))

    def pad_for_graph(self, bucket: int, dummy_slot: int, dummy_page: int):
        """Pad a decode-only batch of B seqs to `bucket` seqs: dummy rows attend to one dummy token
        and write their K/V into the reserved dummy page (reference: input_data.py:319-367)."""
        b = self.num_seqs
        assert self.num_decode_seqs == b and bucket >= b
        if bucket == b:
            self.padded_tokens = b
            return
        n = bucket - b
        self._tokens[1][b:bucket].zero_()
        if self.mrope:
            self._positions[1][:, b:bucket].zero_()
        else:
            self._positions[1][b:bucket].zero_()
        self._slots[1][b:bucket].fill_(dummy_slot)
        self._block_table[1][b:bucket, 0].fill_(dummy_page)
        self._seq_lens[1][b:bucket].fill_(1)
        self._qsl[1][b:bucket + 1].copy_(torch.arange(b, bucket + 1, dtype=torch.int32, device=self.device))
        if self.batch.lora_slot is not None:     # padding rows: no adapter (the last CSR group runs them as base rows)
            self._lora[2][1][b:bucket].copy_(torch.arange(b, bucket, dtype=torch.int32, device=self.device))
        self.padded_tokens = bucket

    # -- views ------------------------------------------------------------------------------------
    def _n_tok(self):
        return self.padded_tokens or self.num_tokens

    def _n_seq(self):
        return self.padded_tokens or self.num_seqs

    @property
    def tokens(self): return self._tokens[1][: self._n_tok()]

    @property
    def positions(self):
        return self._positions[1][:, : self._n_tok()] if self.mrope else self._positions[1][: self._n_tok()]

    @property
    def slot_mapping(self): return self._slots[1][: self._n_tok()]

    @property
    def tok_seq(self):
        """token -> sequence row, or None when every sequence has exactly one token (decode)."""
        if self.padded_tokens or self.num_decode_seqs == self.num_seqs:
            return None
        return self._tok_seq[1][: self.num_tokens]

    @property
    def block_table(self): return self._block_table[1][: self._n_seq()]

    @property
    def seq_lens(self): return self._seq_lens[1][: self._n_seq()]

    @property
    def query_start_loc(self): return self._qsl[1][: self._n_seq() + 1]

    @property
    def logits_idx(self): return self._logits_idx[1][: self.num_emit]

    @property
    def temperature(self): return self._temperature[1][: self.num_emit]

    @property
    def top_k(self): return self._top_k[1][: self.num_emit]

    @property
    def top_p(self): return self._top_p[1][: self.num_emit]

    @property
    def rep_penalty(self): return self._rep_penalty[1][: self.num_emit]

    @property
    def state_slot(self): return self._state_slot[1][: self.num_emit]

    @property
    def freq_pen(self): return self._freq_pen[1][: self.num_emit]

    @property
    def pres_pen(self): return self._pres_pen[1][: self.num_emit]

    @property
    def bias_slot(self):
        """int32 [E] bias row of each emitting row (-1: none), or None when no row of the batch has one."""
        return self._bias_slot[1][: self.num_emit] if self.batch is not None and self.batch.need_bias else None

    @property
    def lora(self):
        """(slots, row_off, rows, number of groups) of the batch's adapter CSR, or None when no row uses an adapter."""
        if self.batch is None or self.batch.lora_slot is None:
            return None
        l1 = self._lora
        return l1[0][1], l1[1][1], l1[2][1][: self._n_tok()], self.lora_groups

    @property
    def plp(self):
        """(int32 rows [Q], int32 targets [Q]) of the batch's prompt log-prob rows on the device."""
        q = self.batch.plp_rows.shape[0]
        return self._plp[0][1][:q], self._plp[1][1][:q]

    @property
    def seeds(self):
        """(int64 seeds [E], int32 positions [E]) of a batch with seeded rows, else (None, None)."""
        if self.batch is None or self.batch.seed is None:
            return None, None
        return self._seed[1][: self.num_emit], self._seed_pos[1][: self.num_emit]

    def h2d_bytes(self) -> int:
        b = self.batch
        if b is None:
            return 0
        tot = 0
        for a in (b.tokens, b.positions, b.slot_mapping, b.block_table, b.seq_lens, b.query_start_loc,
                  b.logits_idx, b.temperature, b.top_k, b.top_p, b.rep_penalty, b.state_slot):
            tot += a.nbytes
        for a in (b.freq_pen, b.pres_pen, b.bias_slot, b.seed, b.seed_pos, b.plp_rows, b.plp_targets):
            if a is not None:
                tot += a.nbytes
        if b.lora_slot is not None:
            tot += self._lora_h2d
        return tot
