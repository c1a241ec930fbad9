"""Paged KV-cache bookkeeping + storage (reference: gllm/memory_manager.py).

Differences from the reference, by design:
  * storage layout is `[pages, Hkv, D/64, page_size, 64]` per layer (TMA-friendly slabs, see
    csrc/elemwise/rope_kv.cu) instead of `[pages, page_size, Hkv, D]`;
  * prefix-cache page keys are *chained* hashes — key(page i) = hash((key(page i-1), tokens of
    page i)) — O(page_size) per page instead of re-hashing the whole prefix
    (gllm/memory_manager.py:205-208);
  * re-acquiring a specific cached page is O(1) (`IDAllocator`);
  * only the driver rank owns a manager; peers receive ready-made block tables.
Behaviour kept: freed pages go to the tail of the free list, a page's hash is evicted when the
page is handed out again, decode-generated full pages are registered, cache granularity is full
pages, a reserved dummy page absorbs CUDA-graph padding writes.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from gllm_b200.id_allocator import IDAllocator
from gllm_b200.ops.ref import kv_cache_shape
from gllm_b200.sequence import Sequence


class KVCache:
    """Device storage: per-layer K and V tensors (or one latent tensor per layer for MLA)."""

    def __init__(self, num_layers: int, num_pages: int, page_size: int, kv_head_num: int, kv_head_dim: int,
                 dtype: torch.dtype, device, use_mla: bool = False):
        self.num_layers, self.num_pages, self.page_size = num_layers, num_pages, page_size
        self.kv_head_num, self.kv_head_dim, self.use_mla = kv_head_num, kv_head_dim, use_mla
        heads = 1 if use_mla else kv_head_num
        shape = kv_cache_shape(num_pages, heads, kv_head_dim, page_size)
        # zero-init: masked / padded positions must hold finite values (attention multiplies them by 0)
        self.k_cache = [torch.zeros(shape, dtype=dtype, device=device) for _ in range(num_layers)]
        self.v_cache = [] if use_mla else [torch.zeros(shape, dtype=dtype, device=device) for _ in range(num_layers)]

    @staticmethod
    def bytes_per_page(num_layers, page_size, kv_head_num, kv_head_dim, dtype_bytes, use_mla=False) -> int:
        if use_mla:
            return num_layers * page_size * kv_head_dim * dtype_bytes
        return 2 * num_layers * page_size * kv_head_num * kv_head_dim * dtype_bytes


class MemoryManager:
    def __init__(self, num_pages: int, page_size: int, reserve_dummy_page: bool = False):
        self.num_pages = num_pages
        self.page_size = page_size
        self.id_allocator = IDAllocator(0, num_pages - 1)
        # the LAST page is the dummy page (CUDA-graph padding rows read/write it)
        self.dummy_page: Optional[int] = self.id_allocator.allocate(num_pages - 1) if reserve_dummy_page else None
        self.usable_pages = num_pages - (1 if reserve_dummy_page else 0)
        # page tables holding each page: several sequences share pages (prefix-cache hits, the prompt pages of the
        # choices of a parallel-sampling request); a page returns to the free list when the last one lets go
        self.page_ref: List[int] = [0] * num_pages
        if self.dummy_page is not None:
            self.page_ref[self.dummy_page] = 1

    # -- page accounting ------------------------------------------------------------------------
    def allocate_page(self) -> int:
        page = self.id_allocator.allocate()
        self.page_ref[page] += 1
        return page

    def share_page(self, page: int) -> int:
        """One more page table holds `page` (already held by another one)."""
        assert self.page_ref[page] > 0, page
        self.page_ref[page] += 1
        return page

    def free_page(self, page: int):
        assert self.page_ref[page] > 0, page
        self.page_ref[page] -= 1
        if self.page_ref[page] == 0:
            self.id_allocator.free(page)

    def pages_needed(self, seq: Sequence) -> int:
        return max(0, (seq.seq_len + self.page_size - 1) // self.page_size - len(seq.page_table))

    def pre_allocate_page(self, seqs: List[Sequence]):
        for seq in seqs:
            for _ in range(self.pages_needed(seq)):
                seq.page_table.append(self.allocate_page())

    def free(self, seq: Sequence):
        for page in seq.page_table:
            self.free_page(page)
        seq.page_table = []
        seq.pt_np = None
        seq.pt_gen += 1
        seq.page_hashes = []
        seq.published = 0

    def publish_computed(self, seq: Sequence):
        """Hook called when a chunk of `seq` has returned (computed_token_num advanced); the prefix cache publishes
        the pages that became complete."""

    def get_num_free_pages(self) -> int:
        return self.id_allocator.get_num_free_ids()

    def get_memory_util(self) -> float:
        return round(100.0 * self.id_allocator.get_num_used_ids() / max(self.id_allocator.size, 1), 2)

    def get_memory_free(self) -> float:
        return self.get_num_free_pages() / max(self.num_pages, 1)

    def get_cache_hit_rate(self) -> float:
        return 0.0


class PrefixMemoryManager(MemoryManager):
    """Adds a hash -> page map (automatic prefix caching); cached pages are shared through `page_ref`."""

    def __init__(self, num_pages: int, page_size: int, reserve_dummy_page: bool = False):
        super().__init__(num_pages, page_size, reserve_dummy_page)
        self.hash2page: Dict[int, int] = {}
        self.page2hash: List[Optional[int]] = [None] * num_pages
        self.num_allocated_pages = 0
        self.num_hit_pages = 0

    # -- hashing --------------------------------------------------------------------------------
    def _extend_hashes(self, seq: Sequence, upto_pages: int):
        """Make seq.page_hashes cover the first `upto_pages` full pages."""
        ps = self.page_size
        hs = seq.page_hashes
        toks = seq.token_ids
        while len(hs) < upto_pages:
            i = len(hs)
            # multimodal prompts share placeholder ids: salt the chain with a digest of the pixels
            if hs:
                prev = hs[-1]
            else:
                prev = 0x9E3779B97F4A7C15 ^ ((seq.mm_state or {}).get("salt", 0))
                if seq.lora_id:    # an adapter's KV differs from the base model's and every other adapter's
                    prev = hash((prev, -1, seq.lora_id))
            hs.append(hash((prev, tuple(toks[i * ps:(i + 1) * ps]))))

    # -- allocation -----------------------------------------------------------------------------
    def allocate_page(self, page_hash: Optional[int] = None) -> int:
        page = self.id_allocator.allocate()
        old = self.page2hash[page]
        if old is not None:
            if self.hash2page.get(old) == page:
                del self.hash2page[old]
            self.page2hash[page] = None
        if page_hash is not None and page_hash not in self.hash2page:
            self.page2hash[page] = page_hash
            self.hash2page[page_hash] = page
        self.page_ref[page] += 1
        return page

    def pre_allocate_computed_page(self, seqs: List[Sequence]):
        """First touch of a sequence: reuse cached full pages of its prefix."""
        ps = self.page_size
        for seq in seqs:
            assert len(seq.page_table) == 0
            n_tok = len(seq.token_ids)
            num_page = (n_tok + ps - 1) // ps
            if not seq.computed_prompt:
                self.num_allocated_pages += num_page
            full = n_tok // ps
            # never serve the *whole* prompt from cache: the last token must be computed to get logits
            if full * ps == n_tok:
                full -= 1
            if seq.plp_pending:
                full = 0     # prompt log-probs need the hidden state of every prompt position: no hits
            self._extend_hashes(seq, max(full, 0))
            for i in range(max(full, 0)):
                page = self.hash2page.get(seq.page_hashes[i])
                if page is None:
                    break
                self.id_allocator.allocate(page)  # O(1) removal from the free list if it was free
                self.page_ref[page] += 1
                seq.page_table.append(page)
                seq.computed_token_num += ps
                seq.scheduled_token_num += ps
                self.num_hit_pages += 1
            seq.num_cached_tokens = seq.computed_token_num
            seq.published = len(seq.page_table)

    def publish_computed(self, seq: Sequence):
        """A page becomes a cache entry only once its KV has been written: called when a chunk returns, with
        `computed_token_num` covering it. (Registering at allocation — as the reference does,
        gllm/memory_manager.py:150-203 — lets an aborted / stall-broken / preempted sequence leave hashes behind
        for pages it never filled; the next request with the same prefix would then attend to garbage.)"""
        ps = self.page_size
        full = min(seq.computed_token_num // ps, len(seq.page_table))
        if full <= seq.published:
            return
        self._extend_hashes(seq, full)
        for i in range(seq.published, full):
            h, page = seq.page_hashes[i], seq.page_table[i]
            if h not in self.hash2page and self.page2hash[page] is None:
                self.page2hash[page] = h
                self.hash2page[h] = page
        seq.published = full

    def get_cache_hit_rate(self) -> float:
        if self.num_allocated_pages == 0:
            return 0.0
        return round(100.0 * self.num_hit_pages / self.num_allocated_pages, 2)
