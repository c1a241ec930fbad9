"""asyncio front-end for the HTTP server (reference: gllm/async_llm_engine.py:11-109).

One `AsyncStream` per request (an asyncio.Queue of text deltas); a single background task ticks the
engine (`LLM.schedule`) in a worker thread so the event loop stays responsive, detokenises new
tokens incrementally, and aborts requests whose client disconnected.
"""
from __future__ import annotations

import asyncio
import time
from typing import Dict, List, Optional

from gllm_b200.engine.llm_engine import LLM
from gllm_b200.utils.logging import logger


class Histogram:
    """Cumulative-bucket latency histogram in the Prometheus exposition layout (seconds)."""

    def __init__(self, bounds):
        self.bounds = tuple(bounds)
        self.counts = [0] * (len(self.bounds) + 1)
        self.sum = 0.0
        self.count = 0

    def observe(self, v: float):
        self.sum += v
        self.count += 1
        for i, b in enumerate(self.bounds):
            if v <= b:
                self.counts[i] += 1
                return
        self.counts[-1] += 1

    def lines(self, name: str) -> List[str]:
        out, acc = [f"# TYPE {name} histogram"], 0
        for b, c in zip(self.bounds, self.counts):
            acc += c
            out.append(f'{name}_bucket{{le="{b:g}"}} {acc}')
        out.append(f'{name}_bucket{{le="+Inf"}} {self.count}')
        out.append(f"{name}_sum {self.sum:.6f}")
        out.append(f"{name}_count {self.count}")
        return out


TTFT_BUCKETS = (0.005, 0.01, 0.02, 0.04, 0.06, 0.08, 0.1, 0.25, 0.5, 0.75, 1.0, 2.5, 5.0, 7.5, 10.0, 30.0)
TPOT_BUCKETS = (0.002, 0.004, 0.006, 0.008, 0.01, 0.015, 0.02, 0.03, 0.04, 0.05, 0.075, 0.1, 0.2, 0.5, 1.0)
E2E_BUCKETS = (0.1, 0.25, 0.5, 1.0, 2.5, 5.0, 10.0, 20.0, 40.0, 60.0, 120.0, 300.0)


class Delta(str):
    """A text delta of a stream that asked for log-probs: `logprobs` lists the entries (token, log-prob,
    [(token, log-prob), ...]) of the tokens whose text this delta releases (the text may be empty)."""
    logprobs: list = []


class AsyncStream:
    def __init__(self, raw_request=None, stop=None, logprobs: bool = False):
        self.stop = [x for x in ([stop] if isinstance(stop, str) else list(stop or [])) if x]
        self._held = ""
        # log-probs: [text end offset (None until the token's text is put), entry] not delivered yet; an entry leaves
        # with the delta that releases the last character of its token's text
        self._lp: Optional[list] = [] if logprobs else None
        self._text_total = 0     # characters put so far (held ones included)
        self._released = 0       # characters delivered
        self.lp_count = 0        # generated tokens whose entry was added
        self.logprobs_out: list = []   # entries drained by LLM.collect
        self.stop_hit = False
        self._queue: asyncio.Queue = asyncio.Queue()
        self._finished = False
        self._raw_request = raw_request
        self.prompt_tokens = 0
        self.completion_tokens = 0
        self.finish_reason: Optional[str] = None
        self.created = time.time()
        self.first_token_time: Optional[float] = None
        self.seq_id = -1
        self.aborted = False     # an abort id was sent for this request (front-end side state only)
        self.group: Optional[list] = None   # parallel sampling: the streams of all choices of the request
        # prompt log-probs: the request's entries (None for the first token), filled before the first delta is put
        self.prompt_logprobs: list = []

    def put(self, item: str):
        """Queue a text delta. With stop strings (OpenAI `stop`; not honoured by the reference) the text that could
        still turn into a stop string is held back; on a hit the text before it is delivered, the stream ends with
        finish_reason "stop" and `stop_hit` tells the engine to abort the request."""
        if self._finished:
            return
        if self._lp is not None:          # the text of the tokens added since the last put ends here
            self._text_total += len(item)
            for rec in self._lp:
                if rec[0] is None:
                    rec[0] = self._text_total
        if not self.stop:
            self._out(item)
            return
        buf = self._held + item
        cut = min((i for i in (buf.find(s) for s in self.stop) if i >= 0), default=-1)
        if cut >= 0:
            self._held = ""
            if cut or self._lp:
                self._out(buf[:cut], everything=True)   # the latest token completed the stop string
            self.stop_hit = True
            self.finish("stop")
            return
        hold = 0      # longest suffix of buf that is a proper prefix of some stop string
        for s in self.stop:
            for k in range(min(len(s) - 1, len(buf)), hold, -1):
                if buf.endswith(s[:k]):
                    hold = k
                    break
        if len(buf) > hold:
            self._out(buf[:len(buf) - hold])
        elif self._lp:
            self._out("")
        self._held = buf[len(buf) - hold:] if hold else ""

    def add_logprobs(self, entries: list):
        """Entries of tokens whose text the next `put` carries (or a later one, while it is held back)."""
        if self._lp is not None and not self._finished:
            self._lp.extend([None, e] for e in entries)

    @property
    def want_logprobs(self) -> bool:
        return self._lp is not None

    def _out(self, text: str, everything: bool = False):
        if self._lp is None:
            self._queue.put_nowait(text)
            return
        self._released += len(text)
        done = [r for r in self._lp if everything or (r[0] is not None and r[0] <= self._released)]
        if done:
            self._lp = [r for r in self._lp if not (everything or (r[0] is not None and r[0] <= self._released))]
        if text or done:
            d = Delta(text)
            d.logprobs = [r[1] for r in done]
            self._queue.put_nowait(d)

    def finish(self, reason: str = "stop"):
        if not self._finished:
            if self._held:                     # generation ended while a possible stop prefix was held back
                self._out(self._held, everything=True)
                self._held = ""
            elif self._lp:                     # entries whose text never came (held U+FFFD tail, empty token text)
                self._out("", everything=True)
            self.finish_reason = reason
            self._queue.put_nowait(StopAsyncIteration())
            self._finished = True

    @property
    def finished(self) -> bool:
        return self._finished

    def __aiter__(self):
        return self

    async def __anext__(self):
        item = await self._queue.get()
        if isinstance(item, Exception):
            raise item
        return item

    async def is_disconnected(self) -> bool:
        if self._raw_request is None:
            return False
        try:
            return await self._raw_request.is_disconnected()
        except Exception:  # noqa: BLE001
            return False


class AsyncLLM(LLM):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.async_streams: Dict[int, AsyncStream] = {}
        self._task: Optional[asyncio.Task] = None
        self._pending_tokens: List = []
        self.failed: Optional[str] = None      # set when the engine loop died: the server answers 500 from then on
        self.metrics = {"requests_total": 0, "requests_finished": 0, "requests_aborted": 0,
                        "prompt_tokens_total": 0, "generation_tokens_total": 0, "ttft_sum": 0.0, "ttft_count": 0}
        self.hist = {"ttft": Histogram(TTFT_BUCKETS), "tpot": Histogram(TPOT_BUCKETS),
                     "e2e": Histogram(E2E_BUCKETS)}

    async def add_requests_async(self, raw_request, token_ids: List[int], output_len=None, ignore_eos=False,
                                 temperature=None, top_p=None, top_k=None, repetition_penalty=None,
                                 mm_contents=None, stop=None, logprobs=None, seed=None, frequency_penalty=None,
                                 presence_penalty=None, logit_bias=None, n=None, prompt_logprobs=None, lora=None):
        """`logprobs`: None, or N in [0, 20] — every text delta of the stream is then a `Delta` carrying the
        log-prob entries of the tokens whose text it releases (see `LLM.generate`). `seed`, `frequency_penalty`,
        `presence_penalty`, `logit_bias`: see `LLM.allocate_seq` (ValueError when out of range).
        Returns the request's `AsyncStream`; with `n` given (parallel sampling, see `LLM.allocate_choices`) a list of
        one stream per choice, in choice order. A stop string ends only its own choice. `prompt_logprobs`: see
        `LLM.generate`; every stream's `prompt_logprobs` is the request's list, complete before its first delta."""
        seqs = self.allocate_choices(token_ids, n, output_len, ignore_eos, temperature, top_p, top_k,
                                     repetition_penalty, mm_contents, logprobs, seed, frequency_penalty,
                                     presence_penalty, logit_bias, prompt_logprobs, lora)
        streams = []
        for seq in seqs:
            stream = AsyncStream(raw_request, stop, logprobs=logprobs is not None)
            stream.prompt_tokens = len(token_ids)
            stream.seq_id = seq.seq_id
            stream.prompt_logprobs = seq.prompt_logprobs
            self.async_streams[seq.seq_id] = stream
            streams.append(stream)
        if len(streams) > 1:
            for st in streams:
                st.group = streams
        self.metrics["requests_total"] += 1          # requests, not choices
        self.metrics["prompt_tokens_total"] += len(token_ids)
        self.add_requests(seqs[:1])
        if self._task is None and self.failed is None:
            self.start_schedule_engine()
        return streams if n is not None else streams[0]

    def abort_stream(self, stream: AsyncStream):
        """Client went away: abort the request so its KV pages are freed (reference:
        async_llm_engine.py:93-97 polls `is_disconnected` from the engine task; here the request's own
        task reports it, which also works under ASGI test transports)."""
        # Only the abort id is sent: the Sequence object is shared with the in-proc scheduler, which must be the
        # one to take it out of its queues before flagging it (a flag set from here while a prefill chunk was in
        # flight left a freed sequence at the head of the prefill queue and took the engine down).
        live = [st for st in (stream.group or [stream]) if not st.aborted and not st.finished]
        if live:           # every choice of the request
            for st in live:
                st.aborted = True
            self.abort([st.seq_id for st in live])
            self.metrics["requests_aborted"] += 1

    async def collect(self, stream: AsyncStream) -> str:
        """Drain a stream to a string, aborting the request if the client disconnects meanwhile."""
        text = ""
        while True:
            try:
                item = await asyncio.wait_for(stream.__anext__(), timeout=0.5)
                text += item
                if isinstance(item, Delta):
                    stream.logprobs_out.extend(item.logprobs)
            except StopAsyncIteration:
                return text
            except asyncio.TimeoutError:
                if await stream.is_disconnected():
                    self.abort_stream(stream)
                    return text

    def _on_token(self, seq, tok):
        self._pending_tokens.append(seq)

    def _tick(self) -> bool:
        return self.schedule(self._on_token)

    def _deliver(self):
        seen = set()
        for seq in self._pending_tokens:
            if id(seq) in seen:
                continue
            seen.add(id(seq))
            st = self.async_streams.get(seq.seq_id)
            if st is None:
                continue
            if st.first_token_time is None:
                st.first_token_time = time.time()
                if st.group is None or all(o.first_token_time is None for o in st.group if o is not st):
                    self.metrics["ttft_sum"] += st.first_token_time - st.created     # once per request
                    self.metrics["ttft_count"] += 1
                    self.hist["ttft"].observe(st.first_token_time - st.created)
            st.completion_tokens = seq.num_output_tokens
            if st.want_logprobs:
                self._deliver_with_logprobs(seq, st)
            elif self.tokenizer is not None:
                delta = seq.detokenize_inc(self.tokenizer)
                if delta:
                    st.put(delta)
            else:
                st.put(" ".join(str(t) for t in seq.token_ids[seq.cur_length:seq.known_len]) + " ")
                seq.cur_length = seq.known_len
            if st.stop_hit and not st.aborted:      # a stop string completed: stop generating for this request
                st.aborted = True
                self.abort([seq.seq_id])
        self._pending_tokens = []
        self._finish_streams()

    def _deliver_with_logprobs(self, seq, st: AsyncStream):
        """Token by token, so that each log-prob entry leaves with the delta that releases its token's text."""
        end, lps = seq.known_len, seq.output_logprobs
        while st.lp_count < len(lps) and not st.finished:
            j = seq.prompt_len + st.lp_count
            if j >= end:
                break
            chosen, top = lps[st.lp_count]
            st.add_logprobs([(seq.token_ids[j], chosen, top)])
            st.lp_count += 1
            if self.tokenizer is not None:
                before = seq.cur_length
                delta = seq.detokenize_inc(self.tokenizer, j + 1)
                if seq.cur_length != before:
                    st.put(delta)
            else:
                st.put(f"{seq.token_ids[j]} ")
                seq.cur_length = j + 1

    def _finish_streams(self):
        for seq in self.finished:
            st = self.async_streams.pop(seq.seq_id, None)
            if st is not None:
                st.completion_tokens = seq.num_output_tokens
                self.metrics["generation_tokens_total"] += seq.num_output_tokens
                now = time.time()
                # a request with several choices counts once, when its last choice ends
                if st.group is None or all(o.finished for o in st.group if o is not st):
                    self.metrics["requests_finished"] += 1
                    self.hist["e2e"].observe(now - st.created)
                if st.first_token_time is not None and seq.num_output_tokens > 1:
                    self.hist["tpot"].observe((now - st.first_token_time) / (seq.num_output_tokens - 1))
                reason = "length" if seq.num_output_tokens >= seq.output_len else "stop"
                if st.stop_hit:
                    reason = "stop"
                elif st.aborted or seq.is_abort:
                    reason = "abort"
                st.finish(reason)
        self.finished = []

    async def _loop(self):
        loop = asyncio.get_running_loop()
        idle = 0
        while True:
            did = await loop.run_in_executor(None, self._tick)
            self._deliver()
            if did or self.running_maps or self.wait_lists:
                idle = 0
                await asyncio.sleep(0)
            else:
                idle += 1
                await asyncio.sleep(0.001 if idle < 1000 else 0.01)

    def start_schedule_engine(self):
        self._task = asyncio.get_event_loop().create_task(self._loop())

        def _done(task):
            try:
                task.result()
            except asyncio.CancelledError:
                logger.info("engine loop cancelled")
            except Exception as e:  # noqa: BLE001
                logger.error("engine background task failed: %r", e, exc_info=e)
                # fail-stop: release every waiting client instead of hanging them
                self.failed = repr(e)
                for st in list(self.async_streams.values()):
                    st._queue.put_nowait(RuntimeError(f"engine failure: {e!r}"))
                self.async_streams.clear()
                self._task = None
        self._task.add_done_callback(_done)


# name used by the reference (gllm/async_llm_engine.py:56)
PipeAsyncLLM = AsyncLLM
