"""Worker-side model execution (reference: gllm/model_runner.py:165-478).

Owns: this rank's model slice, the paged KV cache, the persistent `InputData`, static PP
activation buffers, CUDA graphs for decode-only batches, and the `Sampler`.

    runner.init()                                  load / profile / size KV / capture graphs
    runner.step(batch, hidden=None, residual=None) one micro-batch through this stage

`step` returns a `StepResult`: sampled tokens on the last stage (device tensor + pinned host
copy issued asynchronously), or the (hidden, residual) views to ship to the next stage.
"""
from __future__ import annotations

import os
import time
from dataclasses import dataclass
from typing import Dict, List, Optional

import numpy as np
import torch

from gllm_b200.config import EngineConfig, capture_sizes
from gllm_b200.input_data import BatchArrays, InputData
from gllm_b200.memory_manager import KVCache
from gllm_b200.model_loader import ModelLoader
from gllm_b200.parallel import state as ps
from gllm_b200.parallel.tp import make_tp_comm
from gllm_b200.sampler import Sampler
from gllm_b200.utils.logging import logger


@dataclass
class StepResult:
    tokens: Optional[torch.Tensor] = None          # int32 [E] device
    tokens_host: Optional[torch.Tensor] = None     # pinned copy (valid after `event.synchronize()`)
    event: Optional[object] = None
    hidden: Optional[torch.Tensor] = None
    residual: Optional[torch.Tensor] = None
    num_emit: int = 0
    # log-probabilities (only when some emitting row asked): fp32 [E_lp, 1 + 2N] for the asking rows in emit order,
    # its pinned copy (same event as tokens_host) and the int32 [E] request (-1: none) per emitting row
    logprobs: Optional[torch.Tensor] = None
    logprobs_host: Optional[torch.Tensor] = None
    logprobs_n: Optional[np.ndarray] = None
    # prompt log-probabilities (only when the batch has prompt rows): fp32 [Q, 1 + 2N] in the batch's prompt-row order
    # and its pinned copy (same event)
    prompt_logprobs: Optional[torch.Tensor] = None
    prompt_logprobs_host: Optional[torch.Tensor] = None

    def tokens_list(self) -> List[int]:
        if self.tokens is None:
            return []
        if self.event is not None:
            self.event.synchronize()
            return self.tokens_host[: self.num_emit].tolist()
        return self.tokens[: self.num_emit].tolist()

    def logprobs_list(self) -> Optional[list]:
        """None when no row asked; else per emitting row None or (sampled token's log-prob, [(token, log-prob), ...]
        with the row's N most likely tokens, largest first)."""
        if self.logprobs_n is None:
            return None
        lp = self.logprobs
        if self.event is not None:
            self.event.synchronize()
            lp = self.logprobs_host[: lp.numel()].view(lp.shape)
        vals = lp.cpu().numpy()
        ids = vals.view(np.int32)
        out, j = [], 0
        for n in self.logprobs_n[: self.num_emit].tolist():
            if n < 0:
                out.append(None)
                continue
            out.append(_entry(vals, ids, j, n))
            j += 1
        return out

    def prompt_logprobs_list(self) -> Optional[list]:
        """None when the batch had no prompt rows; else per prompt row (target token's log-prob, [(token, log-prob),
        ...] with the batch's N most likely tokens, largest first)."""
        lp = self.prompt_logprobs
        if lp is None:
            return None
        if self.event is not None:
            self.event.synchronize()
            lp = self.prompt_logprobs_host[: lp.numel()].view(lp.shape)
        vals = lp.cpu().numpy()
        ids = vals.view(np.int32)
        n = (lp.shape[1] - 1) // 2
        return [_entry(vals, ids, j, n) for j in range(lp.shape[0])]


def _entry(vals: np.ndarray, ids: np.ndarray, j: int, n: int):
    """(chosen log-prob, [(token, log-prob)] of the n most likely) from row j of a logprobs_final result."""
    top = [(int(ids[j, 1 + 2 * i]), float(vals[j, 2 + 2 * i])) for i in range(n) if ids[j, 1 + 2 * i] >= 0]
    return float(vals[j, 0]), top


class ModelRunner:
    def __init__(self, cfg: EngineConfig, loader: Optional[ModelLoader] = None):
        self.cfg = cfg
        self.loader = loader or ModelLoader(cfg.model_path, cfg.load_format)
        self.page_size = cfg.page_size
        self.max_num_batched_tokens = cfg.max_num_batched_tokens
        self.max_running_seqs = cfg.max_running_seqs
        self.model_max_length = self.resolve_model_max_length(cfg.model_max_length)
        self.capture_sizes = [] if cfg.disable_cuda_graph else capture_sizes(
            min(cfg.max_cuda_graph_bs, self.max_running_seqs))
        self.model = None
        self.kv_cache: Optional[KVCache] = None
        self.input_data: Optional[InputData] = None
        self.tpc = None
        self.graphs: Dict[int, object] = {}
        self.num_pages = 0
        self.device = None
        self.sampler: Optional[Sampler] = None
        self.stats = {"steps": 0, "graph_steps": 0, "tokens": 0, "h2d_bytes": 0, "d2h_bytes": 0,
                      "graph_kernel_launches": 0, "gpu_ms": 0.0}
        self.graph_kernels: Dict[int, int] = {}
        self.time_steps = False   # bench: bracket every step with CUDA events
        self._step_events = []

    def resolve_model_max_length(self, model_max_length):
        if model_max_length is None:
            gl = self.loader.generation_config.get("max_length", 20)
            if gl != 20:
                model_max_length = gl
        if model_max_length is None:
            model_max_length = min(self.loader.config.get("max_position_embeddings", 8192), 8192)
        return int(model_max_length)

    # -------------------------------------------------------------------------------------------
    def init(self, device: str, progress=None):
        cfg = self.cfg
        self.device = torch.device(device)
        is_cuda = self.device.type == "cuda"
        if is_cuda:
            torch.cuda.set_device(self.device)
        t0 = time.time()
        self.model = self.loader.load_model(self.device, progress)
        self.spec = self.model.spec
        want_fused = cfg.tp_mode == "fused" and cfg.tp_size > 1 and is_cuda
        why_not = "fp8 block-scaled linears" if getattr(self.spec, "quant", None) is not None else \
            "DeepStack (Qwen3-VL) feature injection" if getattr(self.model, "num_deepstack", 0) else None
        if want_fused and why_not:
            logger.warning("tp_mode=fused is not available with %s: tensor-parallel collectives run on NCCL", why_not)
        self.tpc = make_tp_comm(fused=(want_fused and why_not is None),
                                max_tokens=self.max_num_batched_tokens,
                                hidden_size=self.spec.hidden_size, dtype=self.spec.dtype, device=self.device) \
            if cfg.tp_size > 1 else make_tp_comm(False)
        max_blocks = (self.model_max_length + self.page_size - 1) // self.page_size + 1
        mrope = self.model.rope.mrope_section is not None if hasattr(self.model, "rope") else False
        self.input_data = InputData(self.max_num_batched_tokens, max(self.max_running_seqs, 1), max_blocks,
                                    self.device, mrope=mrope)
        self.input_data.need_tok_seq = bool(self.loader.use_mla)
        # test hook (tests/mp_tp_check.py): keep the full last-token logits of every step, per emitting sequence id
        self.keep_logits = os.environ.get("GLLM_KEEP_LOGITS", "0") == "1"
        self.logit_log = []
        # vocab-parallel sampling: the forward (and its CUDA graphs) ends at this rank's logits shard
        self.sampler = Sampler(self.device, self.spec.vocab_size, cfg.seed, self.input_data, self.stats,
                               vocab_parallel=cfg.tp_size > 1 and os.environ.get("GLLM_VP_SAMPLE", "1") != "0")
        h, dt = self.spec.hidden_size, self.spec.dtype
        if not ps.is_first_pp_rank():
            self.input_hidden = torch.zeros(self.max_num_batched_tokens, h, dtype=dt, device=self.device)
            self.input_residual = torch.zeros(self.max_num_batched_tokens, h, dtype=dt, device=self.device)
        if ps.is_last_pp_rank():
            pin = is_cuda
            self.tokens_out = torch.zeros(max(self.max_running_seqs, 1), dtype=torch.int32, device=self.device)
            # two pinned result buffers: with async scheduling the next step's D2H copy may land before the host
            # has read the previous step's tokens
            self._tokens_host2 = [torch.zeros(max(self.max_running_seqs, 1), dtype=torch.int32, pin_memory=pin)
                                  for _ in range(2)]
            self._host_flip = 0
            self.tokens_host = self._tokens_host2[0]
            self._lp_host2 = None        # pinned log-prob result buffers, allocated on the first request that asks
            self._plp_host2 = None       # the same for prompt log-probs
        self._plp = None                 # this step's prompt log-prob result, from the forward to the sampling
        logger.info("model loaded in %.1fs", time.time() - t0)
        self.profile_run()
        self.num_pages = self.compute_num_pages()
        kvh, kvd = self.kv_shape()
        self.kv_cache = KVCache(self.model.num_layers, self.num_pages, self.page_size, kvh, kvd, dt, self.device,
                                use_mla=self.loader.use_mla)
        if is_cuda and not cfg.disable_cuda_graph:
            self.capture_graphs()
        return self

    def kv_shape(self):
        if self.loader.use_mla:
            return 1, self.model.kv_latent_dim
        return self.model.num_kv_heads, self.model.head_dim

    def profile_run(self):
        """Peak-activation probe: max tokens through the model without a KV cache."""
        if self.device.type != "cuda":
            return
        t = self.max_num_batched_tokens
        n = max(1, min(self.max_running_seqs, t))
        batch = _dummy_batch(t, n, self.page_size, self.input_data.max_blocks)
        torch.cuda.synchronize()
        hidden = residual = None
        if not ps.is_first_pp_rank():     # later stages start from the previous stage's (hidden, residual)
            hidden, residual = self.input_hidden[:t], self.input_residual[:t]
        self._forward(batch, hidden, residual, use_kv=False)
        torch.cuda.synchronize()

    def compute_num_pages(self) -> int:
        cfg = self.cfg
        kvh, kvd = self.kv_shape()
        per_page = KVCache.bytes_per_page(self.model.num_layers, self.page_size, kvh, kvd,
                                          torch.empty(0, dtype=self.spec.dtype).element_size(), self.loader.use_mla)
        if self.device.type != "cuda":
            num = cfg.num_cpu_pages
        elif cfg.num_gpu_pages is not None:
            num = cfg.num_gpu_pages
        else:
            torch.cuda.empty_cache()
            free, _ = torch.cuda.mem_get_info(self.device)
            num = int((free // max(per_page, 1)) * cfg.gpu_memory_util)
        if ps.get_world_size() > 1 and torch.distributed.is_initialized():
            all_n = [None] * ps.get_world_size()
            torch.distributed.all_gather_object(all_n, num)
            num = min(all_n)
        logger.info("KV cache: %d pages (%d tokens/page), %.2f KB/token, %.2f GB total", num, self.page_size,
                    per_page / 1024 / self.page_size, num * per_page / 2 ** 30)
        assert num >= 4, "not enough memory for the KV cache"
        return num

    # -------------------------------------------------------------------------------------------
    def _forward(self, batch: BatchArrays, hidden, residual, use_kv=True):
        inp = self.input_data
        inp.load(batch)
        return self._forward_loaded(hidden, residual, use_kv)

    def _forward_loaded(self, hidden, residual, use_kv=True, all_rows=False, recv_tiles=None):
        inp = self.input_data
        kv = self.kv_cache if use_kv else None
        self.tpc.begin_forward(inp.padded_tokens or inp.num_tokens)
        if recv_tiles is not None:
            h, r = self.model(inp, kv, self.tpc, hidden, residual, recv_tiles=recv_tiles)
        else:
            h, r = self.model(inp, kv, self.tpc, hidden, residual)
        if ps.is_last_pp_rank():
            vp = self.sampler.vocab_parallel
            h = self.tpc.materialize(h)
            if not all_rows and inp.batch is not None and inp.batch.plp_rows is not None:
                # before the sampled rows' logits: the step's logits footprint stays within one [R, Vp/tp] tile or
                # the [E, Vp/tp] logits, both covered by the profile run
                self._plp = self.sampler.prompt_logprobs(inp.batch, h, self.model.lm_head, self.plp_tile_rows())
            return self.model.compute_logits(inp, h, self.tpc, all_rows=all_rows, local=vp), None
        return h, r

    # prompt rows per LM-head tile. Measured on H100 at V = 151936, tp 1 and 2 (benchmarks/prompt_logprobs_bench.py,
    # README): 256-row tiles cost half as much per row as 128-row ones in the GEMM, and the one-pass records kernel
    # still reads a tile right after its GEMM at 1.5-3.5 TB/s (tp 2 - tp 1; partly from L2). Capped by
    # max_running_seqs, so a tile is never wider than the [max_running_seqs, Vp/tp] logits the profile run
    # materialises.
    PLP_TILE_ROWS = 256

    def plp_tile_rows(self) -> int:
        return max(1, min(self.PLP_TILE_ROWS, self.max_running_seqs))

    def capture_graphs(self):
        """Decode-only batches replay a CUDA graph per power-of-two bucket (forward -> logits)."""
        inp = self.input_data
        self.graph_pool = None
        self.graph_logits: Dict[int, torch.Tensor] = {}
        self.graph_hidden: Dict[int, tuple] = {}
        from gllm_b200.ops import sm100
        kvh, _ = self.kv_shape()
        sm100.reserve_attn_workspace(self.device, max(self.capture_sizes or [1]), self.model.layers[0].attn.num_heads
                                     if len(self.model.layers) else 1, self.model.head_dim)
        dummy_page = self.num_pages - 1
        t0 = time.time()
        for bs in self.capture_sizes:
            batch = _dummy_batch(bs, bs, self.page_size, inp.max_blocks, page=dummy_page, decode=True)
            inp.load(batch)
            inp.padded_tokens = bs
            inp.decode_splits = sm100.decode_splits(bs, max(kvh, 1), self.model.layers[0].attn.num_heads
                                                    if len(self.model.layers) else 1, self.model_max_length)
            hid = res = None
            if not ps.is_first_pp_rank():
                hid, res = self.input_hidden[:bs], self.input_residual[:bs]
            # warm-up on a side stream, then capture
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for _ in range(2):
                    self._forward_loaded(hid, res, all_rows=True)
            torch.cuda.current_stream().wait_stream(s)
            g = torch.cuda.CUDAGraph()
            n0 = sm100.launches()
            with torch.cuda.graph(g, pool=self.graph_pool):
                out, r = self._forward_loaded(hid, res, all_rows=True)
            self.graph_kernels[bs] = sm100.launches() - n0
            self.graph_pool = self.graph_pool or g.pool()
            self.graphs[bs] = (g, inp.decode_splits)
            if ps.is_last_pp_rank():
                self.graph_logits[bs] = out
            else:
                self.graph_hidden[bs] = (out, r)
        inp.decode_splits = None
        inp.padded_tokens = 0
        torch.cuda.synchronize()
        if ps.get_world_size() > 1 and torch.distributed.is_initialized():
            torch.distributed.barrier()
        logger.info("captured %d CUDA graphs (buckets %s) in %.1fs", len(self.graphs), self.capture_sizes,
                    time.time() - t0)

    # -------------------------------------------------------------------------------------------
    def step(self, batch: BatchArrays, hidden: Optional[torch.Tensor] = None,
             residual: Optional[torch.Tensor] = None, recv_tiles=None) -> StepResult:
        inp = self.input_data
        self.stats["steps"] += 1
        self.stats["tokens"] += batch.num_tokens
        bucket = None
        # (a fan-out batch has more sampled rows than sequences: the graphs produce one logits row per sequence)
        if self.graphs and batch.is_decode_only() and batch.num_seqs <= self.capture_sizes[0] and \
                batch.logits_idx.shape[0] == batch.num_seqs:
            bucket = min(b for b in self.graphs if b >= batch.num_seqs)
        inp.load(batch)
        if batch.feed_src is not None:
            inp.apply_feed(self.tokens_out)
            self.stats["feed_steps"] = self.stats.get("feed_steps", 0) + 1     # lookahead steps
        self.stats["h2d_bytes"] += inp.h2d_bytes()
        if self.time_steps and self.device.type == "cuda":
            ev0 = torch.cuda.Event(enable_timing=True)
            ev0.record()
        try:
            res = self._step_loaded(batch, bucket, hidden, residual, recv_tiles)
            if batch.kv_copy is not None:
                self.copy_pages(batch.kv_copy)
            return res
        finally:
            if self.time_steps and self.device.type == "cuda":
                ev1 = torch.cuda.Event(enable_timing=True)
                ev1.record()
                kind = f"graph{bucket}" if bucket is not None else \
                    ("decode_eager" if batch.is_decode_only() else "prefill")
                self._step_events.append((ev0, ev1, kind, batch.num_tokens))

    def copy_pages(self, pairs):
        """Parallel sampling: page dst := page src in every KV-cache tensor of this rank (its layers, its KV heads), in
        stream order after the forward that wrote the src pages."""
        kv = self.kv_cache
        self.sampler.ops.kv_copy_pages(kv.k_cache + kv.v_cache, pairs.tolist(), dummy_page=self.num_pages - 1)
        self.stats["kv_copy_pages"] = self.stats.get("kv_copy_pages", 0) + len(pairs)

    def gpu_busy_ms(self) -> float:
        """Sum of per-step device time (CUDA events around forward + sampling); resets the log."""
        if self._step_events:
            self._step_events[-1][1].synchronize()
        tot = 0.0
        self.busy_by_kind = {}        # kind -> [steps, device ms, tokens] of the log just consumed
        for a, b, kind, ntok in self._step_events:
            ms = a.elapsed_time(b)
            tot += ms
            acc = self.busy_by_kind.setdefault(kind, [0, 0.0, 0])
            acc[0] += 1
            acc[1] += ms
            acc[2] += ntok
        self._step_events = []
        return tot

    def _step_loaded(self, batch, bucket, hidden, residual, recv_tiles=None) -> StepResult:
        inp = self.input_data
        if bucket is not None and recv_tiles:
            for _, _, works in recv_tiles:  # graphs read the static input buffers: need every tile
                for w in works:
                    w.wait()
            recv_tiles = None
        if bucket is not None:
            assert batch.plp_rows is None, "a decode-only batch carries no prompt rows"
            g, splits = self.graphs[bucket]
            inp.pad_for_graph(bucket, (self.num_pages - 1) * self.page_size, self.num_pages - 1)
            g.replay()
            self.stats["graph_steps"] += 1
            self.stats["graph_kernel_launches"] += self.graph_kernels.get(bucket, 0)
            inp.padded_tokens = 0
            if ps.is_last_pp_rank():
                logits = self.graph_logits[bucket][: batch.num_seqs]
                return self._sample(batch, logits)
            h, r = self.graph_hidden[bucket]
            return StepResult(hidden=h[: batch.num_tokens], residual=r[: batch.num_tokens])
        out, r = self._forward_loaded(hidden, residual, recv_tiles=recv_tiles)
        if ps.is_last_pp_rank():
            return self._sample(batch, out)
        return StepResult(hidden=out, residual=r)

    def _sample(self, batch: BatchArrays, logits: torch.Tensor) -> StepResult:
        e = logits.shape[0]
        plp, self._plp = self._plp, None
        if e == 0:
            if plp is None:
                return StepResult(tokens=self.tokens_out[:0], num_emit=0)
            return self._finish_sample(self.tokens_out[:0], 0, None, plp)
        if self.keep_logits:
            full = self.tpc.gather_logits(logits, self.spec.vocab_size) if self.sampler.vocab_parallel else logits
            self.logit_log.append((list(batch.emit_ids or []), full[:e, : self.spec.vocab_size].float().cpu()))
        toks, logprobs = self.sampler.sample(batch, logits)
        return self._finish_sample(toks, e, logprobs, plp)

    def _finish_sample(self, toks: torch.Tensor, e: int, logprobs: Optional[torch.Tensor] = None,
                       plp: Optional[torch.Tensor] = None) -> StepResult:
        self.tokens_out[:e].copy_(toks)
        # (CPU: no async D2H copy — snapshot the values, a lookahead step may overwrite tokens_out before the
        # scheduler reads them)
        res = StepResult(tokens=self.tokens_out if self.device.type == "cuda" else self.tokens_out[:e].clone(),
                         num_emit=e)
        if logprobs is not None:
            res.logprobs, res.logprobs_n = logprobs, self.input_data.batch.logprobs_n[:e]
        res.prompt_logprobs = plp
        if self.device.type == "cuda":
            self._host_flip ^= 1
            self.tokens_host = self._tokens_host2[self._host_flip]
            self.tokens_host[:e].copy_(self.tokens_out[:e], non_blocking=True)
            self.stats["d2h_bytes"] += 4 * e
            if logprobs is not None:
                # two pinned buffers, flipped with tokens_host: a lookahead step's copy may land before the host has
                # read this one
                if self._lp_host2 is None:
                    from gllm_b200.ops.sm100 import MAX_LOGPROBS
                    size = max(self.max_running_seqs, 1) * (1 + 2 * MAX_LOGPROBS)
                    self._lp_host2 = [torch.zeros(size, dtype=torch.float32, pin_memory=True) for _ in range(2)]
                host = self._lp_host2[self._host_flip]
                host[: logprobs.numel()].copy_(logprobs.view(-1), non_blocking=True)
                res.logprobs_host = host
                self.stats["d2h_bytes"] += 4 * logprobs.numel()
            if plp is not None:
                if self._plp_host2 is None:
                    from gllm_b200.ops.sm100 import MAX_LOGPROBS
                    size = self.max_num_batched_tokens * (1 + 2 * MAX_LOGPROBS)
                    self._plp_host2 = [torch.zeros(size, dtype=torch.float32, pin_memory=True) for _ in range(2)]
                host = self._plp_host2[self._host_flip]
                host[: plp.numel()].copy_(plp.view(-1), non_blocking=True)
                res.prompt_logprobs_host = host
                self.stats["d2h_bytes"] += 4 * plp.numel()
            ev = torch.cuda.Event()
            ev.record()
            res.tokens_host, res.event = self.tokens_host, ev
        return res

    def close(self):
        if self.device is not None and torch.device(self.device).type == "cuda":
            torch.cuda.synchronize()
        self.graphs.clear()
        tpc, self.tpc = self.tpc, None
        if tpc is not None and hasattr(tpc, "close"):
            tpc.close()


def _dummy_batch(num_tokens: int, num_seqs: int, page_size: int, max_blocks: int, page: int = 0,
                 decode: bool = False) -> BatchArrays:
    """Synthetic batch for the memory probe / graph capture: `num_seqs` sequences sharing the
    tokens evenly (decode=True: one token each, KV length 1 on `page`)."""
    if decode:
        q = np.ones(num_seqs, dtype=np.int32)
    else:
        q = np.full(num_seqs, num_tokens // num_seqs, dtype=np.int32)
        q[: num_tokens - int(q.sum())] += 1
    qsl = np.zeros(num_seqs + 1, dtype=np.int32)
    np.cumsum(q, out=qsl[1:])
    t = int(qsl[-1])
    nb = min(max_blocks, max(1, (int(q.max()) + page_size - 1) // page_size))
    bt = np.full((num_seqs, nb), page, dtype=np.int32)
    pos = np.concatenate([np.arange(n, dtype=np.int32) for n in q]) if t else np.zeros(0, np.int32)
    e = num_seqs
    return BatchArrays(
        tokens=np.zeros(t, np.int32), positions=pos, slot_mapping=np.full(t, -1 if not decode else page * page_size, np.int32),
        block_table=bt, seq_lens=q.copy(), query_start_loc=qsl, logits_idx=(qsl[1:] - 1).astype(np.int32),
        emit_seq=np.arange(e, dtype=np.int32), temperature=np.ones(e, np.float32), top_k=np.ones(e, np.int32),
        top_p=np.ones(e, np.float32), rep_penalty=np.ones(e, np.float32), state_slot=np.zeros(e, np.int32),
        num_decode_seqs=num_seqs if decode else 0, num_seqs=num_seqs, num_tokens=t, max_q_len=int(q.max()),
        max_seq_len=int(q.max()), all_greedy=True, need_penalty=False)
