"""Engine front-end `LLM` (reference: gllm/llm_engine.py:19-430).

Owns the tokenizer, sequence ids and the running map; talks to the driver worker either
  * in-process (`launch_mode="inproc"`: world_size == 1, or one process per GPU started by an
    external launcher such as torchrun — then rank 0 is front-end + driver and the other ranks
    serve inside `generate()` until the driver tells them to stop), or
  * over ZeroMQ to `pp x tp` spawned worker processes (`launch_mode="normal"`, and
    `master` / `slave` for multi-node — same protocol as the reference).

Public surface kept: `LLM(model_path, **kwargs)`, `generate(prompts=|tokens=, output_lens=,
temperature=, top_p=, top_k=)`, `chat()`, `add_requests()`, `schedule()`,
`start_profile()/stop_profile()`.
"""
from __future__ import annotations

import os
import sys
import threading
import time
from typing import Dict, List, Optional

import torch
import torch.multiprocessing as mp

from gllm_b200.config import EngineConfig
from gllm_b200.engine.comm import Comm, IPCPackage, ipc_base
from gllm_b200.engine.worker import Worker, run_worker
from gllm_b200.id_allocator import IDAllocator
from gllm_b200.model_loader import ModelLoader
from gllm_b200.parallel import state as ps
from gllm_b200.sequence import Sequence

MAX_LOGPROBS = 20   # most likely tokens reported per generated token (csrc/sample/sampler.cu: kMaxLogprobs)
# logit_bias entries per request: this engine's own cap (one scatter per entry when the bias row is rebuilt)
MAX_LOGIT_BIAS = 1024
MAX_N = 128         # choices per request (parallel sampling, OpenAI `n`)


def check_n(n, max_running_seqs: int, multimodal: bool = False) -> int:
    """Validate OpenAI `n` -> the number of choices. None means 1. Raises ValueError: n must be an integer in
    [1, MAX_N] and at most the engine's max_running_seqs (all first tokens are drawn in one batch); n > 1 with
    multimodal input is not supported."""
    if n is None:
        return 1
    if isinstance(n, bool) or not isinstance(n, int) and not (isinstance(n, float) and n.is_integer()):
        raise ValueError("n must be an integer")
    n = int(n)
    if not 1 <= n <= min(MAX_N, max_running_seqs):
        raise ValueError(f"n must be in [1, {min(MAX_N, max_running_seqs)}]")
    if n > 1 and multimodal:
        raise ValueError("n > 1 is not supported with multimodal input")
    return n


def check_prompt_logprobs(prompt_logprobs, multimodal: bool = False) -> int:
    """Validate `prompt_logprobs` -> N, or -1 for None (no prompt log-probs). Raises ValueError: N must be an integer
    in [0, MAX_LOGPROBS]; multimodal input is refused (image placeholder tokens make no sensible targets)."""
    if prompt_logprobs is None:
        return -1
    if isinstance(prompt_logprobs, bool) or not isinstance(prompt_logprobs, int) or \
            not 0 <= prompt_logprobs <= MAX_LOGPROBS:
        raise ValueError(f"prompt_logprobs must be an integer in [0, {MAX_LOGPROBS}]")
    if multimodal:
        raise ValueError("prompt_logprobs is not supported with multimodal input")
    return prompt_logprobs


def choice_seed(seed: Optional[int], i: int) -> Optional[int]:
    """Seed of choice i of a request seeded with `seed`: seed + i, wrapped to a signed 64-bit int."""
    if seed is None:
        return None
    return (seed + i + 2 ** 63) % 2 ** 64 - 2 ** 63


def check_sampling_params(seed=None, frequency_penalty=None, presence_penalty=None, logit_bias=None,
                          vocab_size=None):
    """Validate and normalise the OpenAI sampling parameters -> (seed or None, frequency_penalty, presence_penalty,
    {token id: bias} or None). Raises ValueError: penalties must be finite and in [-2, 2]; logit_bias takes at most
    MAX_LOGIT_BIAS entries whose keys parse as ints in [0, vocab_size) and whose values are finite and in
    [-100, 100] (a key given twice, e.g. "7" and "07", keeps the last value); seed must fit a signed 64-bit int."""
    import math
    out = []
    for name, v in (("frequency_penalty", frequency_penalty), ("presence_penalty", presence_penalty)):
        v = 0.0 if v is None else float(v)
        if not (math.isfinite(v) and -2.0 <= v <= 2.0):
            raise ValueError(f"{name} must be a finite number in [-2, 2]")
        out.append(v)
    if seed is not None:
        if isinstance(seed, bool) or int(seed) != seed or not -2 ** 63 <= int(seed) < 2 ** 63:
            raise ValueError("seed must be an integer that fits in a signed 64-bit int")
        seed = int(seed)
    lb = None
    if logit_bias:
        if len(logit_bias) > MAX_LOGIT_BIAS:
            raise ValueError(f"logit_bias takes at most {MAX_LOGIT_BIAS} entries")
        if vocab_size is None:
            raise ValueError("logit_bias needs a model with a known vocabulary size")
        lb = {}
        for k, v in logit_bias.items():
            try:
                tok = int(k)
            except (TypeError, ValueError):
                raise ValueError(f"logit_bias key {k!r} is not a token id") from None
            if not 0 <= tok < vocab_size:
                raise ValueError(f"logit_bias key {k!r} must be a token id in [0, {vocab_size})")
            try:
                val = float(v)
            except (TypeError, ValueError):
                raise ValueError(f"logit_bias value for {k!r} is not a number") from None
            if not (math.isfinite(val) and -100.0 <= val <= 100.0):
                raise ValueError(f"logit_bias value for {k!r} must be a finite number in [-100, 100]")
            lb[tok] = val
    return seed, out[0], out[1], lb
from gllm_b200.utils.logging import logger


def _env_rank():
    return int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0")), \
        int(os.environ.get("WORLD_SIZE", "1"))


def load_tokenizer(path):
    if not isinstance(path, str) or path.startswith("preset:") or not os.path.isdir(path):
        return None
    try:
        from transformers import AutoTokenizer
        return AutoTokenizer.from_pretrained(path, trust_remote_code=True)
    except Exception as e:  # noqa: BLE001
        logger.warning("no tokenizer loaded from %s (%s): token-id API only", path, e)
        return None


class LLM:
    _instances = 0      # engines created by this process (names the ipc endpoints of each one)

    def __init__(self, model_path, host=None, master_addr="127.0.0.1", master_port=8001, zmq_port_base=8002,
                 launch_mode="normal", worker_ranks=None, load_format="auto", gpu_memory_util=0.9, page_size=16,
                 maxd=2048, maxp=2048, minp=32, iterp=8, kvthresh=0.05, enable_prefix_caching=True, pp_size=1,
                 tp_size=1, use_ep=True, assigned_layers=None, use_async_worker=False, async_schedule=True,
                 use_thinking=True,
                 schedule_method="chunked_prefill", disable_cuda_graph=False, max_cuda_graph_bs=32,
                 model_max_length=None, mm_processor_min_pixels=None, mm_processor_max_pixels=None, **extra):
        if isinstance(assigned_layers, str):
            assigned_layers = [int(x) for x in assigned_layers.split(",")]
        if isinstance(worker_ranks, str):
            worker_ranks = [int(x) for x in worker_ranks.split(",")]
        from gllm_b200.utils import resolve_model_path
        model_path = resolve_model_path(model_path)      # HF repo id -> local snapshot (under a file lock)
        self.cfg = EngineConfig(
            model_path=model_path, load_format=load_format, host=host or "0.0.0.0", master_addr=master_addr,
            master_port=master_port, zmq_port_base=zmq_port_base, launch_mode=launch_mode,
            worker_ranks=worker_ranks, gpu_memory_util=gpu_memory_util, page_size=page_size, maxd=maxd, maxp=maxp,
            minp=minp, iterp=iterp, kvthresh=kvthresh, enable_prefix_caching=enable_prefix_caching,
            pp_size=pp_size, tp_size=tp_size, use_ep=use_ep, assigned_layers=assigned_layers,
            use_async_worker=use_async_worker, async_schedule=async_schedule, use_thinking=use_thinking,
            schedule_method=schedule_method,
            disable_cuda_graph=disable_cuda_graph, max_cuda_graph_bs=max_cuda_graph_bs,
            model_max_length=model_max_length, mm_processor_min_pixels=mm_processor_min_pixels,
            mm_processor_max_pixels=mm_processor_max_pixels, **extra)
        cfg = self.cfg
        self.loader = ModelLoader(cfg.model_path, cfg.load_format, cfg.quantization)
        from gllm_b200.lora import adapter_ids
        # multi-LoRA: adapter name -> id (0 is the base model), validated before any worker starts
        self.lora_ids: Dict[str, int] = adapter_ids(self.loader.architecture, cfg.lora_modules, cfg.max_lora_rank)
        self.tokenizer = load_tokenizer(cfg.tokenizer_path or cfg.model_path)
        self.finish_tokens = self.loader.eos_token_ids()
        gen = self.loader.generation_config
        self.default_temperature = gen.get("temperature", 0.6)
        self.default_top_p = gen.get("top_p", 0.9)
        self.default_repetition_penalty = gen.get("repetition_penalty", 1.0)
        self.id_allocator = IDAllocator(0, 99999)
        self.running_maps: Dict[int, Sequence] = {}
        self.wait_lists: List[Sequence] = []
        self.abort_ids: List[int] = []
        self.control_cmds: List[tuple] = []
        self._inbox_lock = threading.Lock()
        self.finished: List[Sequence] = []
        self.last_stats: dict = {}
        self.worker: Optional[Worker] = None
        self.comm: Optional[Comm] = None
        self.procs = []
        self.mp_alive = None
        self.env_rank, self.env_local_rank, env_world = _env_rank()
        self.is_external = env_world > 1 and env_world == cfg.world_size and launch_mode in ("normal", "inproc")
        if self.is_external:
            cfg.launch_mode = "inproc"
            cfg.master_addr = os.environ.get("MASTER_ADDR", cfg.master_addr)
            cfg.master_port = int(os.environ.get("MASTER_PORT", cfg.master_port)) + 1
        elif cfg.world_size == 1 and launch_mode in ("normal", "inproc"):
            cfg.launch_mode = "inproc"
        self.model_max_length = None
        self._init_workers()

    # -------------------------------------------------------------------------------------------
    # start-up
    # -------------------------------------------------------------------------------------------
    def _init_workers(self):
        cfg = self.cfg
        if cfg.launch_mode == "inproc":
            rank, local_rank = (self.env_rank, self.env_local_rank) if self.is_external else (0, 0)
            comm = None
            if cfg.world_size > 1:
                # one set of ipc endpoints per engine INSTANCE: ranks create their engines in lockstep, so the counter
                # agrees across ranks. Re-using the file names of a previous engine of this process is unsafe — zmq
                # closes sockets asynchronously and a listener unlinks its ipc file when it finally goes away, which
                # can be after the next engine has bound the same path (its peers then never hear from the driver).
                LLM._instances += 1
                base = ipc_base(f"p{cfg.master_port}_{LLM._instances}")
                comm = Comm(base, rank, cfg.world_size, (cfg.pp_size - 1) * cfg.tp_size, frontend=False)
                comm.sock_fe_in = comm.sock_fe_out = None
            self.worker = Worker(cfg, rank, local_rank, comm=_NoFrontend(comm) if comm else None,
                                 loader=self.loader)
            self.worker.init()
            if cfg.world_size > 1:
                torch.distributed.barrier()
            self.model_max_length = self.worker.runner.model_max_length
            return
        # spawned workers + zmq front-end
        ctx = mp.get_context("spawn")
        base = ipc_base()
        multi_node = cfg.launch_mode in ("master", "slave")
        ranks = cfg.worker_ranks if cfg.worker_ranks is not None else list(range(cfg.world_size))
        self.mp_alive = ctx.Array("i", [0] * len(ranks))
        self.mp_progress = ctx.Array("i", [0] * (2 * len(ranks)))
        out_rank = (cfg.pp_size - 1) * cfg.tp_size
        for local_rank, rank in enumerate(ranks):
            comm = Comm(base, rank, cfg.world_size, out_rank, frontend=False,
                        tcp_host=cfg.host if multi_node else None, port_base=cfg.zmq_port_base,
                        master_addr=cfg.master_addr)
            w = Worker(cfg, rank, local_rank, comm=comm, loader=None, mp_alive=self.mp_alive,
                       mp_progress=self.mp_progress)
            p = ctx.Process(target=run_worker, args=(w,), daemon=True)
            p.start()
            self.procs.append(p)
        if cfg.launch_mode != "slave":
            self.comm = Comm(base, -1, cfg.world_size, out_rank, frontend=True,
                             tcp_host=cfg.host if multi_node else None, port_base=cfg.zmq_port_base,
                             master_addr=cfg.master_addr).init()
        self._wait_workers()
        from gllm_b200.model_runner import ModelRunner
        self.model_max_length = ModelRunner(cfg, self.loader).model_max_length

    def _wait_workers(self):
        t0 = time.time()
        while True:
            self.check_worker_alive()
            if all(v == 1 for v in self.mp_alive):
                break
            time.sleep(0.05)
        logger.info("all workers ready in %.1fs", time.time() - t0)

    def check_worker_alive(self):
        if self.mp_alive is not None and any(v == -1 for v in self.mp_alive):
            logger.error("a worker died — shutting down")
            self.shutdown()
            sys.exit(1)
        for p in self.procs:
            if not p.is_alive() and p.exitcode not in (0, None):
                logger.error("worker process exited with code %s", p.exitcode)
                sys.exit(1)

    @property
    def is_driver_process(self) -> bool:
        return self.worker is None or self.worker.rank == 0

    # -------------------------------------------------------------------------------------------
    # requests
    # -------------------------------------------------------------------------------------------
    def encode(self, prompt: str, chat: bool = False, messages=None) -> List[int]:
        assert self.tokenizer is not None, "no tokenizer: pass token ids"
        if chat or messages is not None:
            msgs = messages if messages is not None else [{"role": "user", "content": prompt}]
            try:
                ids = self.tokenizer.apply_chat_template(msgs, add_generation_prompt=True, tokenize=True,
                                                         enable_thinking=self.cfg.use_thinking)
            except TypeError:
                ids = self.tokenizer.apply_chat_template(msgs, add_generation_prompt=True, tokenize=True)
            if hasattr(ids, "keys"):  # transformers >= 5 returns a BatchEncoding
                ids = ids["input_ids"]
            if len(ids) and isinstance(ids[0], (list, tuple)):
                ids = ids[0]
            return list(ids)
        return list(self.tokenizer.encode(prompt))

    def check_seq_length(self, token_ids: List[int], output_len: Optional[int]) -> bool:
        """Reject prompts that cannot fit (reference: gllm/llm_engine.py:293-303)."""
        max_len = self.model_max_length
        if len(token_ids) >= max_len:
            return False
        if output_len is not None and len(token_ids) + output_len > max_len:
            return False
        return True

    def allocate_seq(self, token_ids: List[int], output_len=None, ignore_eos=False, temperature=None, top_p=None,
                     top_k=None, repetition_penalty=None, mm_contents=None, logprobs=None, seed=None,
                     frequency_penalty=None, presence_penalty=None, logit_bias=None, prompt_logprobs=None,
                     lora=None) -> Sequence:
        """Defaults: temperature/top_p/repetition_penalty from generation_config, top_k = 1
        (greedy) unless given (reference: gllm/llm_engine.py:305-337). `logprobs`: None (no log-probs) or the number
        N in [0, MAX_LOGPROBS] of most likely tokens to report next to every generated token's log-prob.
        `prompt_logprobs`: likewise for every prompt token after the first (`Sequence.prompt_logprobs`).
        `seed`, `frequency_penalty`, `presence_penalty`, `logit_bias`: OpenAI semantics, validated by
        `check_sampling_params` (see entrypoints/protocol.py for the formula). `lora`: None (the base model) or the
        name of one of the engine's `lora_modules`."""
        lora_id = self.lora_id(lora)
        if logprobs is not None and not 0 <= int(logprobs) <= MAX_LOGPROBS:
            raise ValueError(f"logprobs must be in [0, {MAX_LOGPROBS}]")
        plp = check_prompt_logprobs(prompt_logprobs, bool(mm_contents))
        seed, frequency_penalty, presence_penalty, logit_bias = check_sampling_params(
            seed, frequency_penalty, presence_penalty, logit_bias, self.loader.config.get("vocab_size"))
        if len(token_ids) == 0:
            raise ValueError("empty prompt: there is no position to sample the first token from")
        vocab = self.loader.config.get("vocab_size")
        if vocab is not None and (min(token_ids) < 0 or max(token_ids) >= vocab):
            raise ValueError(f"token ids must be in [0, {vocab}) (the embedding lookup would fault on the device)")
        with self._inbox_lock:      # ids are freed by the tick thread (`_apply`)
            sid = self.id_allocator.allocate()
        seq = Sequence(sid, token_ids, self.finish_tokens, output_len, ignore_eos,
                       self.default_temperature if temperature is None else temperature,
                       self.default_top_p if top_p is None else top_p,
                       1 if top_k is None else top_k,
                       self.default_repetition_penalty if repetition_penalty is None else repetition_penalty,
                       mm_contents, -1 if logprobs is None else int(logprobs), seed, frequency_penalty,
                       presence_penalty, logit_bias, plp, lora_id)
        if output_len is None:
            seq.output_len = min(4096, self.model_max_length - len(token_ids))
        if mm_contents:
            from gllm_b200.models.multimodal import MMInfo, prepare_mm_sequence
            prepare_mm_sequence(seq, MMInfo.from_config(self.loader.config))
        seq.arrival_time = time.time()
        return seq

    def allocate_choices(self, token_ids: List[int], n=None, output_len=None, ignore_eos=False, temperature=None,
                         top_p=None, top_k=None, repetition_penalty=None, mm_contents=None, logprobs=None, seed=None,
                         frequency_penalty=None, presence_penalty=None, logit_bias=None,
                         prompt_logprobs=None, lora=None) -> List[Sequence]:
        """The `n` choices of one request (parallel sampling; see `check_n`): choice 0 is the request as `allocate_seq`
        makes it, choices 1..n-1 are its forks (`Sequence.forks`): the prompt is prefilled once and every choice draws
        its first token from the same logits row, then continues on its own. With a seed, choice i uses seed + i.
        Only choice 0 goes to `add_requests`; the forks travel with it. The prompt's log-probs are computed once: every
        choice holds the same `prompt_logprobs` list."""
        k = check_n(n, self.cfg.max_running_seqs, bool(mm_contents))
        seqs = []
        try:
            for i in range(k):
                seqs.append(self.allocate_seq(token_ids, output_len, ignore_eos, temperature, top_p, top_k,
                                              repetition_penalty, mm_contents, logprobs,
                                              choice_seed(seed, i) if i else seed, frequency_penalty, presence_penalty,
                                              logit_bias, prompt_logprobs, lora))
        except Exception:
            with self._inbox_lock:
                for s in seqs:
                    self.id_allocator.free(s.seq_id)
            raise
        seqs[0].forks = seqs[1:]
        for s in seqs[1:]:
            s.prompt_logprobs = seqs[0].prompt_logprobs
        return seqs

    def lora_id(self, name) -> int:
        """Adapter id of `name` (None: 0, the base model); ValueError for a name the engine does not serve."""
        if name is None:
            return 0
        if name not in self.lora_ids:
            raise ValueError(f"unknown LoRA adapter {name!r}" + (
                f" (this engine serves {', '.join(self.lora_ids)})" if self.lora_ids else
                " (this engine was started without lora_modules)"))
        return self.lora_ids[name]

    # The three inboxes below are filled from request handlers (event-loop thread of the API server) while the
    # engine tick runs in a worker thread: every append and the swap in `_send` hold `_inbox_lock`, so a request
    # can never land in a list the tick has already shipped (the reference has this race, SURVEY §5.2).
    def add_requests(self, seqs: List[Sequence]):
        with self._inbox_lock:
            self.wait_lists.extend(seqs)

    def abort(self, seq_ids: List[int]):
        with self._inbox_lock:
            self.abort_ids.extend(seq_ids)

    # -------------------------------------------------------------------------------------------
    # engine tick
    # -------------------------------------------------------------------------------------------
    def _send(self):
        if not (self.wait_lists or self.abort_ids or self.control_cmds):
            return
        with self._inbox_lock:
            wait, self.wait_lists = self.wait_lists, []
            aborts, self.abort_ids = self.abort_ids, []
            cmds, self.control_cmds = self.control_cmds, []
        for seq in wait:
            self.running_maps[seq.seq_id] = seq
            for sib in seq.forks:
                self.running_maps[sib.seq_id] = sib
        if cmds:
            for cmd in cmds[:-1]:
                self._post(IPCPackage(control_cmd=cmd))
            pkg = IPCPackage(schedule_lists=wait, abort_ids=aborts, control_cmd=cmds[-1])
        else:
            pkg = IPCPackage(schedule_lists=wait, abort_ids=aborts)
        self._post(pkg)

    def _post(self, pkg: IPCPackage):
        if self.worker is not None:
            self.worker.frontend_in.append(pkg)
        else:
            self.comm.send_frontend(pkg)

    def _recv(self) -> List[IPCPackage]:
        if self.worker is not None:
            out = list(self.worker.frontend_out)
            self.worker.frontend_out.clear()
            return out
        return self.comm.recv_frontend()

    def _apply(self, pkg: IPCPackage, on_token=None):
        now = time.time()
        inproc = self.worker is not None
        lps = pkg.next_logprobs
        for sid, entries in (pkg.prompt_logprobs or {}).items():
            seq = self.running_maps.get(sid)
            if seq is not None:
                seq.prompt_logprobs.extend(entries)     # (shared by the choices of a request)
        for i, (sid, tok) in enumerate(zip(pkg.act_schedule_ids, pkg.next_tokens)):
            seq = self.running_maps.get(sid)
            if seq is None:
                continue
            if not inproc:
                seq.append(tok)  # in-proc: the scheduler already appended to the shared object
            if lps is not None and lps[i] is not None:
                seq.output_logprobs.append(lps[i])   # only here: the scheduler never touches output_logprobs
            if seq.first_token_time == 0.0:
                seq.first_token_time = now
            if on_token is not None:
                on_token(seq, tok)
        for sid in pkg.free_ids:
            seq = self.running_maps.pop(sid, None)
            if seq is None:
                continue        # already released (a duplicate report must not free the id twice)
            seq.finish_time = now
            self.finished.append(seq)
            with self._inbox_lock:
                self.id_allocator.free(sid)
        if pkg.stats:
            self.last_stats = pkg.stats

    def schedule(self, on_token=None) -> bool:
        """One front-end tick: push new requests, advance the in-proc engine, collect outputs."""
        self.check_worker_alive()
        self._send()
        did = False
        if self.worker is not None:
            did = self.worker.step()
        for pkg in self._recv():
            self._apply(pkg, on_token)
            did = True
        return did

    # -------------------------------------------------------------------------------------------
    # offline API
    # -------------------------------------------------------------------------------------------
    def generate(self, prompts: Optional[List[str]] = None, tokens: Optional[List[List[int]]] = None,
                 output_lens: Optional[List[int]] = None, temperature=None, top_p=None, top_k=None,
                 repetition_penalty=None, ignore_eos: bool = False, progress: bool = False,
                 mm_contents: Optional[List[Optional[dict]]] = None, logprobs=None, seed=None,
                 frequency_penalty=None, presence_penalty=None, logit_bias=None, n=None,
                 prompt_logprobs=None, lora=None) -> List[Sequence]:
        """Batch generation; returns the finished `Sequence`s in request order with `.prompt`,
        `.output`, `.token_ids` (reference: gllm/llm_engine.py:343-378). `mm_contents[i]` (VL models) is
        the processor output of request i: pixel_values / image_grid_thw [/ pixel_values_videos ...].
        `logprobs` (None or N in [0, 20], one value or one per request): every generated token gets an entry
        (its log-prob, [(token, log-prob) of the N most likely tokens]) in `.output_logprobs`, under the raw model
        distribution (log_softmax of the logits, before penalty / temperature / top-k / top-p).
        `seed`, `frequency_penalty`, `presence_penalty`, `logit_bias` ({token id: bias}): OpenAI sampling parameters,
        one value or one per request like the others (a dict is one value for all requests).
        `n` (parallel sampling, one value or one per request): request j gives n_j choices, returned consecutively in
        choice order; the prompt is prefilled once (see `allocate_choices`).
        `prompt_logprobs` (None or N in [0, 20], one value or one per request): `.prompt_logprobs` gets one entry per
        prompt token — None for the first, then (its log-prob given the tokens before it, [(token, log-prob) of the N
        most likely tokens at that position]), under the same distribution as `logprobs`; [] when not asked. Not
        available with multimodal input. Such a request takes no prefix-cache hits (it needs every prompt position's
        hidden state); it still publishes its pages for later requests.
        `lora` (multi-LoRA): None for the base model or the name of one of the engine's `lora_modules`; one value or
        a list with one name or None per request. Requests on different adapters run in the same batches."""
        if self.worker is not None and self.worker.rank != 0:
            return self._serve_until_stop()
        if tokens is None:
            assert prompts is not None
            tokens = [self.encode(p) for p in prompts]
        seqs, heads = [], []
        for i, toks in enumerate(tokens):
            ol = output_lens[i] if output_lens is not None else None
            if not self.check_seq_length(toks, ol):
                raise ValueError(f"request {i}: prompt ({len(toks)}) + output ({ol}) exceeds the model max length "
                                 f"{self.model_max_length}")
            def pick(v):            # sampling parameters: one value for all requests, or one per request
                return v[i] if isinstance(v, (list, tuple)) else v
            choices = self.allocate_choices(toks, pick(n), ol, ignore_eos, pick(temperature), pick(top_p), pick(top_k),
                                            pick(repetition_penalty),
                                            mm_contents[i] if mm_contents is not None else None, pick(logprobs),
                                            pick(seed), pick(frequency_penalty), pick(presence_penalty),
                                            pick(logit_bias), pick(prompt_logprobs), pick(lora))
            heads.append(choices[0])
            seqs.extend(choices)
        n = len(seqs)
        self.add_requests(heads)
        base = len(self.finished)
        bar = None
        if progress:
            from tqdm import tqdm
            bar = tqdm(total=n)
        done = 0
        while len(self.finished) - base < n:
            self.schedule()
            if bar is not None and len(self.finished) - base != done:
                bar.update(len(self.finished) - base - done)
                done = len(self.finished) - base
        if bar is not None:
            bar.close()
        del self.finished[base:]
        if self.is_external:
            self._stop_peers()
        if self.tokenizer is not None:
            for s in seqs:
                s.prompt = self.tokenizer.decode(s.token_ids[: s.prompt_len], skip_special_tokens=True)
                s.output = self.tokenizer.decode(s.token_ids[s.prompt_len:], skip_special_tokens=True)
        return seqs

    def _serve_until_stop(self):
        """Non-driver rank under an external launcher: run the worker loop until the driver stops us."""
        w = self.worker
        w.stop = False
        idle = 0
        parent = os.getppid()
        while not w.stop:
            if w.step():
                idle = 0
            else:
                idle += 1
                if idle > 5000:
                    time.sleep(0.0001)
                    if idle % 20000 == 0 and os.getppid() != parent:
                        # the launcher (torchrun) is gone without taking us down — e.g. it was SIGKILLed by a test
                        # harness timeout: an orphaned rank must not keep spinning (and holding its GPU) forever
                        logger.error("launcher process %d disappeared: rank exits", parent)
                        raise SystemExit(1)
        return []

    def _stop_peers(self):
        if self.worker is not None and self.worker.comm is not None:
            self.worker.comm.broadcast_control(("stop",))
            torch.cuda.synchronize() if torch.cuda.is_available() else None

    def chat(self):
        """Interactive console chat (reference: gllm/llm_engine.py:380-430)."""
        assert self.tokenizer is not None
        history = []
        print("type \\quit to exit, \\clear to reset the conversation")
        while True:
            try:
                prompt = input(">>> ")
            except EOFError:
                break
            if prompt.strip() == "\\quit":
                break
            if prompt.strip() == "\\clear":
                history = []
                continue
            history.append({"role": "user", "content": prompt})
            toks = self.encode(None, messages=history)
            seq = self.allocate_seq(toks)
            self.add_requests([seq])
            text = []

            def on_token(s, tok):
                delta = s.detokenize_inc(self.tokenizer)
                text.append(delta)
                print(delta, end="", flush=True)

            base = len(self.finished)
            while len(self.finished) == base:
                self.schedule(on_token)
            del self.finished[base:]
            print()
            from gllm_b200.utils.chat import process_response
            _, history = process_response((self.loader.config.get("architectures") or [""])[0], "".join(text), history)

    # -------------------------------------------------------------------------------------------
    def send_control_command(self, cmd: tuple):
        with self._inbox_lock:
            self.control_cmds.append(cmd)

    def start_profile(self):
        self.send_control_command(("start_profile",))

    def stop_profile(self):
        self.send_control_command(("stop_profile",))

    def shutdown(self):
        if self.worker is not None:
            self.worker.shutdown()
        comm, self.comm = self.comm, None
        if comm is not None:
            try:
                if self.worker is None:
                    comm.send_frontend(IPCPackage(control_cmd=("stop",)))
                    time.sleep(0.05)
            except Exception:  # noqa: BLE001
                pass
        for p in self.procs:
            p.join(timeout=2)
            if p.is_alive():
                p.terminate()
        self.procs = []
        if comm is not None:
            # after the workers are gone nobody is left to re-create the ipc files, so the front-end removes all of
            # them — except under an external launcher (torchrun): there every rank is alive and cleans up its own
            # endpoints; a rank that is already building its next engine must not lose the sockets it just bound
            comm.close(unlink_all=not self.is_external)

    def close(self):
        """Full teardown for an orderly process exit: stop the workers, then release device-side state that other
        ranks map (CUDA graphs first — they reference the peers' buffers —, then the symmetric-memory handles).
        Collective when tp > 1: every rank calls it, peers still alive."""
        worker = self.worker
        world = self.is_external and torch_dist_ready()
        if world:
            import torch.distributed as dist
            dist.barrier()          # nobody tears sockets down while a peer is still serving
        self.shutdown()
        runner = getattr(worker, "runner", None) if worker is not None else None
        if runner is not None:
            runner.close()
        if world:
            dist.barrier()          # ... and nobody builds the next engine before everyone has let go of this one

    def __del__(self):
        try:
            self.shutdown()
        except Exception:  # noqa: BLE001
            pass


def torch_dist_ready() -> bool:
    try:
        import torch.distributed as dist
        return dist.is_available() and dist.is_initialized()
    except Exception:  # noqa: BLE001
        return False


class _NoFrontend:
    """Comm wrapper for the in-proc driver: peers/tokens channels only, no front-end sockets."""

    def __init__(self, comm: Comm):
        self._c = comm
        self.frontend = False
        self.sock_fe_out = None

    def init(self):
        c = self._c
        import zmq
        from gllm_b200.engine.comm import make_socket
        P, L = zmq.PUSH, zmq.PULL
        c.ctx = zmq.Context.instance()
        ring = c.use_shm_ring()
        if ring:
            c.init_ring()
        if c.rank == 0:
            for r in range(1, c.world_size if not ring else 1):
                c.batch_out.append(make_socket(c.ctx, P, c._addr("batch", r), bind=False))
            if c.output_rank != 0:
                c.tok_in = make_socket(c.ctx, L, c._addr("tok"), bind=True)
        else:
            if not ring:
                c.batch_in = make_socket(c.ctx, L, c._addr("batch", c.rank), bind=True)
            if c.rank == c.output_rank:
                c.tok_out = make_socket(c.ctx, P, c._addr("tok"), bind=False)
        return self

    def recv_frontend(self):
        return []

    def __getattr__(self, k):
        return getattr(self._c, k)
