"""Worker runtime: one process (or the caller's process, in-proc mode) per GPU
(reference: gllm/worker.py:29-265).

Roles, by rank (`rank = pp_rank * tp + tp_rank`):
  * driver (rank 0)      — owns the Scheduler + paged-KV bookkeeping; every spin: aborts, front-end
                           requests, returned tokens, schedule one micro-batch (≤ pp_size in
                           flight), broadcast it, run its own stage, post-process outputs.
  * stage-0 TP peers     — receive the micro-batch arrays, run the same stage.
  * later stages         — receive the arrays + the PP activations (NCCL p2p), run their stage;
                           the output rank (first TP rank of the last stage) samples and returns
                           the tokens to the driver.

`Worker.step()` performs one non-blocking iteration of the role loop and reports whether it did
any work, so the same class serves the spawned busy-loop (`run_worker`), the in-process engine
(`LLM` drives `step()`), and the tests.
"""
from __future__ import annotations

import os
import time
import traceback
from collections import deque
from typing import Deque, List, Optional

import numpy as np
import torch

from gllm_b200.config import EngineConfig
from gllm_b200.engine.comm import Comm, IPCPackage
from gllm_b200.engine.profiler import ProfilerMixin
from gllm_b200.id_allocator import IDAllocator
from gllm_b200.input_data import BatchArrays, build_batch
from gllm_b200.memory_manager import MemoryManager, PrefixMemoryManager
from gllm_b200.model_loader import ModelLoader
from gllm_b200.model_runner import ModelRunner, StepResult
from gllm_b200.parallel import state as ps
from gllm_b200.scheduler import Scheduler, SchedulerOutput
from gllm_b200.utils import logging as glog
from gllm_b200.utils.logging import logger


class Worker(ProfilerMixin):
    def __init__(self, cfg: EngineConfig, rank: int, local_rank: int, comm: Optional[Comm] = None,
                 loader: Optional[ModelLoader] = None, mp_alive=None, mp_progress=None):
        self.cfg = cfg
        self.rank, self.local_rank = rank, local_rank
        self.comm = comm
        self.loader = loader
        self.mp_alive, self.mp_progress = mp_alive, mp_progress
        self.runner: Optional[ModelRunner] = None
        self.scheduler: Optional[Scheduler] = None
        self.phase_stats = {f"{p}_step_{k}": 0 for p in ("prefill", "decode") for k in ("seconds", "count", "tokens")}
        self.pending: Deque = deque()          # driver: (batch_id, StepResult) whose tokens are not read yet
        self.peer_batches: Deque[BatchArrays] = deque()
        self.inflight_sends: Deque = deque()   # keep isend handles alive (reference drops them)
        self.batch_counter = 0
        self.frontend_out: Deque[IPCPackage] = deque()  # in-proc front-end mailbox
        self.frontend_in: Deque[IPCPackage] = deque()
        self.stop = False
        self._seq_slots = {}                   # seq_id -> row of the penalty / bias state it holds
        self._free_slots = []                  # rows given back (row 0 = "no penalty state")
        self._num_slots = 1
        self._penalty_seen = False
        self.init_profiler()

    # -------------------------------------------------------------------------------------------
    def init(self):
        cfg = self.cfg
        if ps.get_state().initialized is False or ps.get_world_size() != cfg.world_size:
            ps.init_dist(cfg.pp_size, cfg.tp_size, self.rank, self.local_rank, cfg.master_addr, cfg.master_port,
                         use_ep=cfg.use_ep, assigned_layers=cfg.assigned_layers)
        glog.set_prefix(f"rank{self.rank} pp{ps.get_pp_rank()} tp{ps.get_tp_rank()}")
        device = cfg.resolved_device(self.local_rank)
        if self.comm is not None:
            self.comm.init()
        self.runner = ModelRunner(cfg, self.loader)
        self.runner.init(device, progress=self._progress)
        if self.rank == 0:
            mm_cls = PrefixMemoryManager if cfg.enable_prefix_caching else MemoryManager
            self.mm = mm_cls(self.runner.num_pages, cfg.page_size, reserve_dummy_page=True)
            self.scheduler = Scheduler(self.mm, pp_size=cfg.pp_size, world_size=cfg.world_size,
                                       schedule_method=cfg.schedule_method, maxd=cfg.maxd, maxp=cfg.maxp,
                                       minp=cfg.minp, iterp=cfg.iterp, kvthresh=cfg.kvthresh,
                                       page_size=cfg.page_size, log=cfg.log_stats,
                                       max_seqs=cfg.max_running_seqs)
            self.scheduler.on_preempt = self._release_slot
        if self.mp_alive is not None:
            self.mp_alive[self.local_rank] = 1
        return self

    def _progress(self, done: int, total: int):
        if self.mp_progress is not None:
            self.mp_progress[self.local_rank * 2] = done
            self.mp_progress[self.local_rank * 2 + 1] = total

    # -------------------------------------------------------------------------------------------
    # driver
    # -------------------------------------------------------------------------------------------
    def _recv_frontend(self) -> bool:
        pkgs = list(self.frontend_in)
        self.frontend_in.clear()
        if self.comm is not None:
            pkgs += self.comm.recv_frontend()
        for pkg in pkgs:
            if pkg.schedule_lists:
                for seq in pkg.schedule_lists:
                    for s in [seq] + seq.forks:
                        s.slot = 0      # penalty state rows are assigned at the first emission (`_assign_slots`)
                        if s.repetition_penalty != 1.0 or s.has_bias_row:
                            self._penalty_seen = True
                self.scheduler.add_new_requests(pkg.schedule_lists)
            if pkg.abort_ids:
                self.scheduler.add_abort_ids(pkg.abort_ids)
            if pkg.control_cmd is not None:
                self.handle_control(pkg.control_cmd, broadcast=True)
        return bool(pkgs)

    def _to_frontend(self, out: SchedulerOutput):
        pkg = IPCPackage(act_schedule_ids=out.act_schedule_ids, next_tokens=out.next_tokens,
                         next_logprobs=out.next_logprobs, free_ids=out.free_ids)
        if self.scheduler is not None:
            pkg.stats = dict(self.scheduler.last_stats)
            pkg.stats.update(self.phase_stats)
        if self.comm is not None and self.comm.sock_fe_out is not None and not self.comm.frontend:
            self.comm.send_frontend(pkg)
        else:
            self.frontend_out.append(pkg)

    def run_driver(self) -> bool:
        did = False
        sch = self.scheduler
        out = sch.check_abort_seqs()
        if out is not None:
            self._free_finished_slots(out)
            self._to_frontend(out)
            did = True
        did |= self._recv_frontend()
        # tokens coming back from the output rank (pp > 1 or tp-only with output rank != 0)
        if self.comm is not None:
            for batch_id, toks, lps in self.comm.recv_tokens():
                sch.add_next_tokens(toks, lps)
                did = True
        if self.cfg.async_schedule and len(self.pending) == 1:
            # async scheduling: queue the NEXT decode step behind the one still running on the GPU, before its
            # tokens are back (the runner feeds them device-side); falls through when the conditions do not hold
            look = sch.schedule_lookahead()
            if look:
                did = True
                self._launch(look)
        keep = 1 if (self.cfg.async_schedule and len(self.pending) == 2) else 0   # the step queued just now
        # tokens of our own finished micro-batches
        while len(self.pending) > keep:
            bid, res, t0, phase, ntok = self.pending[0]
            if res.event is not None and not res.event.query():
                break
            self.pending.popleft()
            # per-phase step accounting for /metrics: launch -> tokens-ready wall time of this micro-batch
            self.phase_stats[phase + "_step_seconds"] += time.perf_counter() - t0
            self.phase_stats[phase + "_step_count"] += 1
            self.phase_stats[phase + "_step_tokens"] += ntok
            sch.add_next_tokens(res.tokens_list(), res.logprobs_list())
            did = True
        while True:
            out = sch.process_output()
            if out is None:
                break
            self._free_finished_slots(out)
            self._to_frontend(out)
            did = True
        # schedule + run one micro-batch
        entries = sch.schedule_once()
        if entries:
            did = True
            self._launch(entries)
        return did

    def _assign_slots(self, entries):
        """Penalty state (the per-sequence seen-token bitmask and the frequency / presence / logit_bias row on the
        device) is held only by sequences that are sampling: a row is assigned when a sequence first emits and
        returned when it finishes, is aborted or is preempted — never by waiting requests, whose number is unbounded.
        The pool grows on demand (the runner grows the device tensors to match), so this cannot fail on the request
        path."""
        if not self._penalty_seen:
            return          # no request with a penalty or logit_bias has arrived yet: nothing to scan per step
        for e in entries:
            if not e.emits:
                continue
            for seq in [e.seq] + (e.forks or []):     # (forks: the other choices of a fan-out, first emission)
                if (seq.repetition_penalty != 1.0 or seq.has_bias_row) and seq.slot <= 0:
                    if self._free_slots:
                        seq.slot = self._free_slots.pop()
                    else:
                        seq.slot = self._num_slots
                        self._num_slots += 1
                    seq.slot_fresh = True
                    self._seq_slots[seq.seq_id] = seq.slot

    def _release_slot(self, seq):
        slot = self._seq_slots.pop(seq.seq_id, 0)
        if slot > 0:
            self._free_slots.append(slot)
        seq.slot = 0

    def _launch(self, entries):
        self.batch_counter += 1
        t0 = time.perf_counter()
        self._assign_slots(entries)
        batch = build_batch(entries, self.cfg.page_size, self.runner.spec.vocab_size, self.batch_counter,
                            mrope=self.runner.input_data.mrope, prev=getattr(self, "_last_batch", None))
        if batch.feed_src is None and entries[0].seq.pending == entries[0].start:
            # lookahead batch that did not take the incremental path (mixed base batch): the leading decode rows
            # take their tokens from the previous step's sampler output, indexed in its emit order
            import numpy as np
            where = {sid: i for i, sid in enumerate(self._last_batch.emit_ids)}
            batch.feed_src = np.asarray([where[e.seq.seq_id] for e in entries if e.seq.pending == e.start],
                                        dtype=np.int32)
        self._last_batch = batch if self.cfg.pp_size == 1 else None   # PP interleaves micro-batches
        if self.comm is not None:
            self.comm.send_batch(batch)
        res = self.runner.step(batch)
        if ps.is_last_pp_rank():
            if ps.is_output_rank():
                phase = "decode" if batch.num_decode_seqs == batch.num_seqs else "prefill"
                self.pending.append((batch.batch_id, res, t0, phase, batch.num_tokens))
        else:
            self._pp_send(res)

    def _free_finished_slots(self, out: SchedulerOutput):
        for sid in out.free_ids:
            slot = self._seq_slots.pop(sid, 0)
            if slot > 0:
                self._free_slots.append(slot)

    # -------------------------------------------------------------------------------------------
    # peers
    # -------------------------------------------------------------------------------------------
    def _drain_peer_msgs(self, block_ms: int = 0) -> bool:
        got = False
        while True:
            msg = self.comm.recv_batch(block_ms if not got else 0)
            if msg is None:
                break
            got = True
            kind, payload = msg
            if kind == "batch":
                self.peer_batches.append(payload)
            elif kind == "control":
                self.handle_control(payload, broadcast=False)
        return got

    def run_peer(self) -> bool:
        did = self._drain_peer_msgs()
        self._reap_sends()
        if not self.peer_batches:
            return did
        batch = self.peer_batches.popleft()
        hidden = residual = None
        if not ps.is_first_pp_rank():
            t = batch.num_tokens
            hidden, residual = self.runner.input_hidden[:t], self.runner.input_residual[:t]
            # tile-streamed receive: all irecvs are posted now, the compute stream waits per tile
            tiles = ps.pp_recv_tiled([hidden, residual] if self.runner.model.ret_residual else [hidden])
        else:
            tiles = None
        res = self.runner.step(batch, hidden, residual, recv_tiles=tiles)
        if ps.is_last_pp_rank():
            if ps.is_output_rank():
                self.comm.send_tokens(batch.batch_id, res.tokens_list(), res.logprobs_list())
        else:
            self._pp_send(res)
        return True

    def _pp_send(self, res: StepResult):
        tensors = [res.hidden, res.residual] if self.runner.model.ret_residual else [res.hidden]
        # clone: the static output buffers are overwritten by the next micro-batch while the send is
        # still in flight (latent race in the reference, SURVEY §5.2)
        tensors = [t.clone() for t in tensors]
        handles = ps.pp_send_tiled(tensors)
        self.inflight_sends.append((handles, tensors))

    def _reap_sends(self):
        while self.inflight_sends and all(h.is_completed() for h in self.inflight_sends[0][0]):
            self.inflight_sends.popleft()

    # -------------------------------------------------------------------------------------------
    def handle_control(self, cmd: tuple, broadcast: bool):
        name = cmd[0]
        if broadcast and self.comm is not None:
            self.comm.broadcast_control(cmd)
        if name == "start_profile":
            self.start_profile(cmd[1] if len(cmd) > 1 else None)
        elif name == "stop_profile":
            self.stop_profile()
        elif name == "stop":
            self.stop = True

    def _maybe_inject_fault(self):
        """`GLLM_FAULT_INJECT=<rank>:<step>` kills this worker once it has run <step> engine steps — exercises the
        fail-stop contract (worker marks itself dead, the front-end exits non-zero) in tests."""
        spec = os.environ.get("GLLM_FAULT_INJECT")
        if not spec or self.runner is None:
            return
        r, n = spec.split(":")
        if int(r) == self.rank and self.runner.stats["steps"] >= int(n):
            raise RuntimeError(f"fault injected on rank {self.rank} after {n} steps (GLLM_FAULT_INJECT)")

    def step(self) -> bool:
        self._maybe_inject_fault()
        self._reap_sends()
        if self.rank == 0:
            return self.run_driver()
        return self.run_peer()

    def shutdown(self):
        try:
            if self.comm is not None:
                self.comm.close()
        finally:
            pass


async def _run_worker_async(worker: Worker):
    """`--use-async-worker`: the same role loop as a coroutine that yields to the event loop between engine
    iterations, so control-plane coroutines (profiler control, health probes) can interleave
    (reference: gllm/async_worker.py:6-63)."""
    import asyncio
    idle = 0
    while not worker.stop:
        if worker.step():
            idle = 0
            await asyncio.sleep(0)
        else:
            idle += 1
            await asyncio.sleep(0.0002 if idle > 2000 else 0)


def run_worker(worker: Worker):
    """Entry point of a spawned worker process (reference: gllm/worker.py:252-265)."""
    try:
        worker.init()
        if getattr(worker.cfg, "use_async_worker", False):
            import asyncio
            asyncio.run(_run_worker_async(worker))
            return
        idle = 0
        while not worker.stop:
            if worker.step():
                idle = 0
            else:
                idle += 1
                if idle > 2000:
                    time.sleep(0.0002)  # back off instead of a pure busy-poll
    except KeyboardInterrupt:
        pass
    except Exception:  # noqa: BLE001
        logger.error("worker %d died:\n%s", worker.rank, traceback.format_exc())
        if worker.mp_alive is not None:
            worker.mp_alive[worker.local_rank] = -1
        raise
    finally:
        worker.shutdown()
        ps.destroy()
