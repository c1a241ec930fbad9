"""Per-request state (reference: gllm/sequence.py:8-98)."""
from __future__ import annotations

from typing import Dict, List, Optional


class Sequence:
    __slots__ = ("seq_id", "token_ids", "prompt_len", "page_table", "prompt", "output", "ignore_eos",
                 "finish_tokens", "output_len", "cur_length", "temperature", "top_p", "top_k",
                 "repetition_penalty", "computed_token_num", "scheduled_token_num", "is_abort",
                 "mm_contents", "page_hashes", "num_cached_tokens", "arrival_time", "first_token_time",
                 "finish_time", "slot", "mrope_delta", "mm_state", "pt_np", "pending", "zombie", "pt_gen", "published",
                 "slot_fresh", "logprobs", "output_logprobs", "seed", "frequency_penalty", "presence_penalty",
                 "logit_bias", "forks", "prompt_logprobs_n", "plp_cursor", "prompt_logprobs")

    def __init__(self, seq_id: int, token_ids: List[int], finish_tokens: List[int],
                 output_len: Optional[int] = None, ignore_eos: bool = False, temperature: float = 0.6,
                 top_p: float = 0.9, top_k: int = 10, repetition_penalty: float = 1.0, mm_contents=None,
                 logprobs: int = -1, seed: Optional[int] = None, frequency_penalty: float = 0.0,
                 presence_penalty: float = 0.0, logit_bias: Optional[Dict[int, float]] = None,
                 prompt_logprobs: int = -1):
        self.seq_id = seq_id
        self.token_ids: List[int] = list(token_ids)
        self.prompt_len = len(self.token_ids)
        self.page_table: List[int] = []
        self.page_hashes: List[int] = []  # chained hash per *full* page (prefix cache)
        self.prompt = ""
        self.output = ""
        self.ignore_eos = ignore_eos
        self.finish_tokens = list(finish_tokens)
        self.output_len = 4096 if output_len is None else output_len
        self.cur_length = self.prompt_len  # detokeniser cursor
        self.temperature = temperature
        self.top_p = top_p
        self.top_k = top_k
        self.repetition_penalty = repetition_penalty
        # log-probabilities: how many top alternatives to report per generated token (-1: none), and one entry
        # (sampled token's log-prob, [(token, log-prob), ...]) per generated token, filled by the front-end
        self.logprobs = logprobs
        self.output_logprobs: list = []
        # prompt log-probabilities (scoring): how many top alternatives to report per prompt token (-1: none); the
        # driver's cursor, the next prompt position whose row has been requested from the model (a recompute after a
        # preemption never asks twice); and the front-end's list, one entry per prompt token (None for the first)
        self.prompt_logprobs_n = prompt_logprobs
        self.plp_cursor = 0
        self.prompt_logprobs: list = [None] if prompt_logprobs >= 0 else []
        # OpenAI sampling parameters: a seeded request draws from a stream keyed by (seed, token position), so its
        # tokens depend on its logits alone; the penalties and logit_bias form an additive row on the device
        # (`has_bias_row`), subtracted per generated occurrence / added per token id before the temperature
        self.seed = seed
        self.frequency_penalty = frequency_penalty
        self.presence_penalty = presence_penalty
        self.logit_bias = logit_bias or None
        # computed_token_num : tokens whose KV is computed AND whose batch has returned
        # scheduled_token_num: tokens covered by chunks scheduled so far (returned or in flight);
        #                      with pp_size > 1 several chunks of one prompt can be in flight
        self.computed_token_num = 0
        self.scheduled_token_num = 0
        self.num_cached_tokens = 0
        self.is_abort = False
        self.mm_contents = mm_contents
        self.arrival_time = 0.0
        self.first_token_time = 0.0
        self.finish_time = 0.0
        self.published = 0   # leading pages of page_table already offered to the prefix cache
        self.slot_fresh = False  # penalty state row just (re)assigned: rebuild its contents at the next emission
        self.slot = -1  # row in the persistent per-sequence device state (penalty bitmask, ...)
        self.mrope_delta = 0
        self.pt_np = None  # numpy mirror of page_table (rebuilt only when its length changes)
        self.pt_gen = 0    # bumped whenever the page table is rebuilt from scratch (preemption): rows derived from
                           # an earlier table (incremental batch assembly) are stale then
        self.pending = -1    # index of a placeholder token reserved by a lookahead step (async scheduling)
        self.zombie = False  # finished while a lookahead step was already in flight: pages freed when it returns
        self.mm_state = None
        # parallel sampling (`n` > 1): the other choices of this request. They travel with this sequence (choice 0)
        # and are not scheduled on their own: when its final prompt chunk is scheduled they take its full prompt
        # pages, a copy of its partial last page, and first tokens drawn from its last logits row. Emptied then.
        self.forks: List["Sequence"] = []

    @property
    def plp_pending(self) -> bool:
        """Some prompt log-prob row has not been requested yet: the prompt's hidden states are still needed."""
        return self.prompt_logprobs_n >= 0 and self.plp_cursor < self.prompt_len - 1

    @property
    def has_bias_row(self) -> bool:
        return self.frequency_penalty != 0.0 or self.presence_penalty != 0.0 or bool(self.logit_bias)

    def __len__(self):
        return len(self.token_ids)

    def __getitem__(self, key):
        return self.token_ids[key]

    def append(self, token_id: int):
        self.token_ids.append(token_id)

    @property
    def computed_prompt(self) -> bool:
        return self.computed_token_num >= self.prompt_len

    @property
    def seq_len(self) -> int:
        """KV length once every scheduled chunk has run."""
        return self.scheduled_token_num

    @property
    def num_output_tokens(self) -> int:
        return len(self.token_ids) - self.prompt_len

    @property
    def is_finish(self) -> bool:
        return self.computed_prompt and (
            (not self.ignore_eos and self.token_ids[-1] in self.finish_tokens)
            or len(self.token_ids) - self.prompt_len >= self.output_len)

    def preempt(self):
        """Drop KV; the sequence will be recomputed from scratch (prompt + generated so far)."""
        self.computed_token_num = 0
        self.scheduled_token_num = 0
        self.page_table = []
        self.pt_np = None
        self.pt_gen += 1
        self.page_hashes = []
        self.published = 0
        if self.mm_state:
            self.mm_state["sent"] = False  # the vision embeddings must be recomputed too

    @property
    def known_len(self) -> int:
        """Number of tokens whose values are known on the host (a trailing lookahead placeholder is not)."""
        return len(self.token_ids) - (1 if self.pending >= 0 else 0)

    def detokenize_inc(self, tokenizer, end: Optional[int] = None) -> str:
        """Incremental detokenisation of the tokens up to `end` (default: every known token); holds back while the
        tail decodes to U+FFFD."""
        end = self.known_len if end is None else end
        if self.cur_length >= end:
            return ""
        prev = tokenizer.decode(self.token_ids[self.cur_length - 1: self.cur_length + 1],
                                skip_special_tokens=True) if self.cur_length > 0 else ""
        added_space = " " if " " in prev.strip() else ""
        delta = tokenizer.decode(self.token_ids[self.cur_length:end], skip_special_tokens=True)
        if delta.endswith("�"):
            return ""
        if len(delta) > 0 and delta[0] != " ":
            delta = added_space + delta
        self.cur_length = end
        return delta
