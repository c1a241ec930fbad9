"""OpenAI-compatible HTTP server (reference: gllm/entrypoints/api_server.py:36-322).

    python -m gllm_b200.entrypoints.api_server --model-path <hf dir | preset:name> [--tp 8 --pp 1 ...]

Routes kept from the reference: GET /v1/models, POST /v1/chat/completions, POST /v1/completions,
POST /start_profile, POST /stop_profile. Added: GET /health, GET /metrics (Prometheus text),
POST /tokenize, POST /detokenize; `usage` is filled in (the reference always returns zeros).
Streaming = server-sent events `data: {json}\\n\\n` ... `data: [DONE]\\n\\n`; a client disconnect
aborts the request and frees its KV pages.
"""
from __future__ import annotations

import argparse
import asyncio
from http import HTTPStatus
from typing import List, Optional

from fastapi import Request  # module level: FastAPI resolves the (string) annotations of the handlers here

from gllm_b200.entrypoints.protocol import (ChatCompletionRequest, ChatCompletionResponse,
                                            ChatCompletionResponseChoice, ChatCompletionResponseStreamChoice,
                                            ChatCompletionStreamResponse, ChatMessage, CompletionRequest,
                                            CompletionResponse, CompletionResponseChoice,
                                            CompletionResponseStreamChoice, CompletionStreamResponse, DeltaMessage,
                                            DetokenizeRequest, DetokenizeResponse, ErrorResponse, ModelCard, ModelList,
                                            ModelPermission, TokenizeRequest, TokenizeResponse, UsageInfo)
from gllm_b200.utils.logging import logger

llm = None  # AsyncLLM, set by build_app / main


def _error(msg: str, status=HTTPStatus.BAD_REQUEST):
    from fastapi.responses import JSONResponse
    return JSONResponse(ErrorResponse(message=msg, type="BadRequestError", code=status.value).model_dump(),
                        status_code=status.value)


def _validate_sampling(request):
    if request.temperature is not None and request.temperature < 0:
        return "temperature must be >= 0"
    if request.top_p is not None and not 0.0 < request.top_p <= 1.0:
        return "top_p must be in (0, 1]"
    if request.repetition_penalty is not None and request.repetition_penalty <= 0:
        return "repetition_penalty must be > 0"
    return None


MAX_LOGPROBS = 20


def _validate_logprobs(request, chat: bool):
    if chat:
        n = request.top_logprobs or 0
        if not 0 <= n <= MAX_LOGPROBS:
            return f"top_logprobs must be in [0, {MAX_LOGPROBS}]"
        if n > 0 and not request.logprobs:
            return "top_logprobs requires logprobs to be true"
        return None
    if request.logprobs is not None and not 0 <= request.logprobs <= MAX_LOGPROBS:
        return f"logprobs must be in [0, {MAX_LOGPROBS}]"
    return None


def _validate_prompt_logprobs(request):
    """`prompt_logprobs` sets the N of the echoed prompt's entries: without `echo` and `logprobs` there is nowhere to
    report them, so it is refused rather than ignored."""
    from gllm_b200.engine.llm_engine import check_prompt_logprobs
    try:
        check_prompt_logprobs(request.prompt_logprobs)
    except ValueError as e:
        return str(e)
    if request.prompt_logprobs is not None and not (request.echo and request.logprobs is not None):
        return "prompt_logprobs needs echo: true and logprobs"
    return None


def _check_params(request, multimodal: bool = False):
    """-> (error message or None, kwargs of the OpenAI sampling parameters for add_requests_async). `n` is passed
    only when it is above 1, so an n = 1 request takes exactly the path it took before parallel sampling."""
    from gllm_b200.engine.llm_engine import check_n, check_sampling_params
    try:
        seed, f, p, lb = check_sampling_params(request.seed, request.frequency_penalty, request.presence_penalty,
                                               request.logit_bias, llm.loader.config.get("vocab_size"))
        n = check_n(request.n, llm.cfg.max_running_seqs, multimodal)
    except (ValueError, TypeError) as e:
        return str(e), None
    out = dict(seed=seed, frequency_penalty=f, presence_penalty=p, logit_bias=lb)
    if n > 1:
        out["n"] = n
    return None, out


def _token_str(tok: int) -> str:
    return llm.tokenizer.decode([tok]) if llm.tokenizer is not None else f"token_id:{tok}"


def _lp_num(lp: float) -> float:
    return max(lp, -9999.0)      # JSON has no -inf (a token whose logit is -inf)


def _chat_logprobs(entries):
    """OpenAI chat shape: {"content": [{token, logprob, bytes, top_logprobs: [{token, logprob, bytes}]}]}."""
    def one(tok, lp):
        s = _token_str(tok)
        return {"token": s, "logprob": _lp_num(lp), "bytes": list(s.encode("utf-8"))}
    return {"content": [dict(one(tok, lp), top_logprobs=[one(t, v) for t, v in top]) for tok, lp, top in entries]}


def _completion_logprobs(entries, offset: int = 0):
    """Legacy completions shape {tokens, token_logprobs, top_logprobs: [{token: logprob}], text_offset}; `offset` is
    the text offset of the first entry. Returns (logprobs, offset after the last entry). An entry (tok, None, None) is
    the first prompt token, which nothing predicts: null log-prob and null alternatives."""
    out = {"tokens": [], "token_logprobs": [], "top_logprobs": [], "text_offset": []}
    for tok, lp, top in entries:
        s = _token_str(tok)
        out["tokens"].append(s)
        out["token_logprobs"].append(None if lp is None else _lp_num(lp))
        out["top_logprobs"].append(None if top is None else {_token_str(t): _lp_num(v) for t, v in top})
        out["text_offset"].append(offset)
        offset += len(s)
    return out, offset


def _prompt_entries(token_ids, prompt_logprobs):
    """Completion-shaped entries (token, log-prob, alternatives) of the prompt: the first token has none."""
    return [(token_ids[0], None, None)] + [(t, lp, top) for t, (lp, top) in zip(token_ids[1:], prompt_logprobs[1:])]


def _prompt_text(prompt, token_ids) -> str:
    if isinstance(prompt, str):
        return prompt
    if isinstance(prompt, list) and prompt and isinstance(prompt[0], str):
        return prompt[0]
    if llm.tokenizer is not None:
        return llm.tokenizer.decode(token_ids)
    return "".join(_token_str(t) for t in token_ids)


def _validate(token_ids, output_len, vocab_size=None):
    """-> error message or None. An empty prompt or a token id outside the vocabulary would take the whole engine
    down (there is no row to sample from / the embedding lookup faults), so they are refused at the door."""
    if not token_ids:
        return "the prompt is empty"
    if output_len is not None and output_len < 1:
        return "max_tokens must be at least 1"
    if vocab_size is not None and (min(token_ids) < 0 or max(token_ids) >= vocab_size):
        return f"token ids must be in [0, {vocab_size})"
    if not llm.check_seq_length(token_ids, output_len):
        return "seq length exceeds max model length"
    return None


def _usage(streams) -> UsageInfo:
    """The prompt counts once; the completion tokens of every choice (parallel sampling) add up."""
    done = sum(st.completion_tokens for st in streams)
    return UsageInfo(prompt_tokens=streams[0].prompt_tokens, completion_tokens=done,
                     total_tokens=streams[0].prompt_tokens + done)


async def _merge(streams):
    """Interleave the deltas of the choices' streams as they come: yields (choice index, delta), and
    (choice index, None) when that choice has ended."""
    q: asyncio.Queue = asyncio.Queue()

    async def pump(i, st):
        try:
            async for d in st:
                await q.put((i, d))
        except Exception as e:  # noqa: BLE001 (engine failure: re-raised in the consumer)
            await q.put((i, e))
            return
        await q.put((i, None))
    tasks = [asyncio.get_running_loop().create_task(pump(i, st)) for i, st in enumerate(streams)]
    left = len(streams)
    try:
        while left:
            i, d = await q.get()
            if isinstance(d, Exception):
                raise d
            if d is None:
                left -= 1
            yield i, d
    finally:
        for t in tasks:
            t.cancel()


# ------------------------------------------------------------------------------------------------
# response generators (reference: serving_chat.py / serving_completions.py)
# ------------------------------------------------------------------------------------------------
async def chat_completion_generator(streams, request) -> ChatCompletionResponse:
    texts = await asyncio.gather(*(llm.collect(st) for st in streams))
    choices = []
    for i, (st, text) in enumerate(zip(streams, texts)):
        choice = ChatCompletionResponseChoice(index=i, message=ChatMessage(role="assistant", content=text),
                                              finish_reason=st.finish_reason)
        if st.want_logprobs:
            choice.logprobs = _chat_logprobs(st.logprobs_out)
        choices.append(choice)
    return ChatCompletionResponse(choices=choices, usage=_usage(streams), model=request.model)


async def chat_completion_stream_generator(streams, request):
    """`streams`: one per choice. One choice per chunk, with its index; every choice ends with its own finish chunk,
    and the last of those carries the usage of the whole request (with one choice: today's single-choice stream)."""
    rid = None
    first = [True] * len(streams)
    left = len(streams)
    try:
        async for i, delta in _merge(streams):
            st = streams[i]
            if delta is None:
                left -= 1
                chunk = ChatCompletionStreamResponse(
                    choices=[ChatCompletionResponseStreamChoice(index=i, delta=DeltaMessage(),
                                                                finish_reason=st.finish_reason or "stop")],
                    model=request.model, usage=_usage(streams) if left == 0 else None)
            else:
                dm = DeltaMessage(role="assistant", content=delta) if first[i] else DeltaMessage(content=delta)
                first[i] = False
                chunk = ChatCompletionStreamResponse(
                    choices=[ChatCompletionResponseStreamChoice(index=i, delta=dm)], model=request.model)
                if st.want_logprobs:
                    chunk.choices[0].logprobs = _chat_logprobs(delta.logprobs)
            if rid is None:
                rid = chunk.id
            chunk.id = rid
            yield f"data: {chunk.model_dump_json(exclude_none=True)}\n\n"
    finally:
        llm.abort_stream(streams[0])  # every choice; no-op unless the client disconnected mid-stream
    yield "data: [DONE]\n\n"


async def completion_generator(streams, request, echo=None) -> CompletionResponse:
    """`echo`: None, or (prompt text, prompt token ids) to put in front of every choice."""
    texts = await asyncio.gather(*(llm.collect(st) for st in streams))
    choices = []
    for i, (st, text) in enumerate(zip(streams, texts)):
        gen = st.logprobs_out
        if echo is not None and request.max_tokens == 0:
            text, gen, st.completion_tokens, st.finish_reason = "", [], 0, "length"   # the sampled token is dropped
        choice = CompletionResponseChoice(index=i, text=text if echo is None else echo[0] + text,
                                          finish_reason=st.finish_reason)
        if st.want_logprobs:
            pre = _prompt_entries(echo[1], st.prompt_logprobs) if echo is not None else []
            choice.logprobs = _completion_logprobs(pre + gen)[0]
        choices.append(choice)
    return CompletionResponse(choices=choices, model=request.model, usage=_usage(streams))


async def completion_stream_generator(streams, request, echo=None):
    """`echo`: None, or (prompt text, prompt token ids): the first chunk of each choice carries the prompt text (and
    its log-prob entries), before any generated text."""
    rid = None
    offset = [0] * len(streams)
    left = len(streams)
    echoed = [echo is None] * len(streams)
    drop = echo is not None and request.max_tokens == 0     # the engine's one sampled token is not part of the answer
    try:
        async for i, delta in _merge(streams):
            st = streams[i]
            if not echoed[i]:
                echoed[i] = True
                chunk = CompletionStreamResponse(choices=[CompletionResponseStreamChoice(index=i, text=echo[0])],
                                                 model=request.model)
                if st.want_logprobs:
                    chunk.choices[0].logprobs, offset[i] = _completion_logprobs(
                        _prompt_entries(echo[1], st.prompt_logprobs), offset[i])
                rid = rid or chunk.id
                chunk.id = rid
                yield f"data: {chunk.model_dump_json(exclude_unset=False)}\n\n"
            if drop:
                if delta is not None:
                    continue
                st.completion_tokens, st.finish_reason = 0, "length"
            if delta is None:
                left -= 1
                chunk = CompletionStreamResponse(
                    choices=[CompletionResponseStreamChoice(index=i, text="", finish_reason=st.finish_reason or "stop")],
                    model=request.model, usage=_usage(streams) if left == 0 else None)
            else:
                chunk = CompletionStreamResponse(choices=[CompletionResponseStreamChoice(index=i, text=delta)],
                                                 model=request.model)
                if st.want_logprobs:
                    chunk.choices[0].logprobs, offset[i] = _completion_logprobs(delta.logprobs, offset[i])
            if rid is None:
                rid = chunk.id
            chunk.id = rid
            yield f"data: {chunk.model_dump_json(exclude_unset=False)}\n\n"
    finally:
        llm.abort_stream(streams[0])  # every choice; no-op unless the client disconnected mid-stream
    yield "data: [DONE]\n\n"


# ------------------------------------------------------------------------------------------------
def _encode_prompt(prompt) -> List[int]:
    if isinstance(prompt, str):
        return llm.encode(prompt)
    if isinstance(prompt, list) and prompt and isinstance(prompt[0], int):
        return list(prompt)
    if isinstance(prompt, list) and prompt and isinstance(prompt[0], list):
        return list(prompt[0])
    if isinstance(prompt, list) and prompt and isinstance(prompt[0], str):
        return llm.encode(prompt[0])
    raise ValueError("unsupported prompt type")


def build_app(engine):
    """FastAPI app bound to an AsyncLLM (also used by the tests with fastapi.testclient)."""
    import fastapi
    from fastapi.responses import JSONResponse, PlainTextResponse, StreamingResponse
    global llm
    llm = engine
    app = fastapi.FastAPI(title="gllm_b200")
    async def _in_thread(fn, *a, **kw):
        return await asyncio.get_running_loop().run_in_executor(None, lambda: fn(*a, **kw))

    @app.get("/health")
    async def health():
        llm.check_worker_alive()
        if llm.failed:
            return JSONResponse({"status": "engine failure", "detail": llm.failed}, status_code=500)
        return JSONResponse({"status": "ok"})

    @app.get("/metrics")
    async def metrics():
        m, s = llm.metrics, llm.last_stats or {}
        lines = [
            "# TYPE gllm_requests_total counter", f"gllm_requests_total {m['requests_total']}",
            "# TYPE gllm_requests_finished_total counter", f"gllm_requests_finished_total {m['requests_finished']}",
            "# TYPE gllm_requests_aborted_total counter", f"gllm_requests_aborted_total {m['requests_aborted']}",
            "# TYPE gllm_prompt_tokens_total counter", f"gllm_prompt_tokens_total {m['prompt_tokens_total']}",
            "# TYPE gllm_generation_tokens_total counter", f"gllm_generation_tokens_total {m['generation_tokens_total']}",
            *llm.hist["ttft"].lines("gllm_time_to_first_token_seconds"),
            *llm.hist["tpot"].lines("gllm_time_per_output_token_seconds"),
            *llm.hist["e2e"].lines("gllm_e2e_request_latency_seconds"),
            "# TYPE gllm_num_requests_running gauge", f"gllm_num_requests_running {len(llm.running_maps)}",
            "# TYPE gllm_num_requests_waiting gauge", f"gllm_num_requests_waiting {s.get('wait', 0)}",
            "# TYPE gllm_kv_cache_usage_perc gauge", f"gllm_kv_cache_usage_perc {s.get('memory_util', 0.0)}",
            "# TYPE gllm_prefix_cache_hit_rate gauge", f"gllm_prefix_cache_hit_rate {s.get('cache_hit_rate', 0.0)}",
            "# TYPE gllm_num_preemptions_total counter", f"gllm_num_preemptions_total {s.get('preempted', 0)}",
        ]
        # per-phase step accounting from the driver worker (launch -> tokens-ready time of every micro-batch;
        # a batch that carries any prefill chunk counts as prefill)
        for key, kind in (("seconds", "seconds"), ("count", "iterations"), ("tokens", "tokens")):
            lines.append(f"# TYPE gllm_step_{kind}_total counter")
            for ph in ("prefill", "decode"):
                lines.append(f'gllm_step_{kind}_total{{phase="{ph}"}} {s.get(f"{ph}_step_{key}", 0):.6g}')
        return PlainTextResponse("\n".join(lines) + "\n")

    @app.get("/v1/models")
    async def show_available_models():
        name = str(llm.cfg.model_path)
        models = ModelList(data=[ModelCard(id=name, root=name, max_model_len=llm.model_max_length,
                                           permission=[ModelPermission()])])
        return JSONResponse(content=models.model_dump())

    @app.post("/v1/chat/completions")
    async def create_chat_completion(request: ChatCompletionRequest, raw_request: Request):
        mm_contents = None
        try:
            if llm.loader.use_mm:
                from gllm_b200.models.multimodal import encode_mm
                token_ids, mm_contents = await _in_thread(encode_mm, llm, request.messages)
            else:
                token_ids = await _in_thread(llm.encode, None, True, request.messages)
        except Exception as e:  # noqa: BLE001
            return _error(f"cannot encode messages: {e}")
        bad, params = _check_params(request, multimodal=bool(mm_contents))
        bad = bad or _validate_sampling(request) or _validate_logprobs(request, chat=True) or \
            _validate(token_ids, request.output_len(), llm.loader.config.get("vocab_size"))
        if bad:
            return _error(bad)
        if llm.failed:
            return _error(f"engine is down: {llm.failed}", HTTPStatus.INTERNAL_SERVER_ERROR)
        stream = await llm.add_requests_async(raw_request, token_ids, request.output_len(), request.ignore_eos,
                                              request.temperature, request.top_p, request.top_k,
                                              request.repetition_penalty, mm_contents, stop=request.stop,
                                              logprobs=(request.top_logprobs or 0) if request.logprobs else None,
                                              **params)
        streams = stream if "n" in params else [stream]
        if request.stream:
            return StreamingResponse(chat_completion_stream_generator(streams, request),
                                     media_type="text/event-stream")
        return JSONResponse(content=(await chat_completion_generator(streams, request)).model_dump())

    @app.post("/v1/completions")
    async def create_completion(request: CompletionRequest, raw_request: Request):
        try:
            token_ids = await _in_thread(_encode_prompt, request.prompt)
        except Exception as e:  # noqa: BLE001
            return _error(f"cannot encode prompt: {e}")
        bad, params = _check_params(request)
        # `max_tokens: 0` (scoring the prompt alone) is served with echo: one token is sampled and dropped
        max_tokens = 1 if request.echo and request.max_tokens == 0 else request.max_tokens
        bad = bad or _validate_sampling(request) or _validate_logprobs(request, chat=False) or \
            _validate_prompt_logprobs(request) or \
            _validate(token_ids, max_tokens, llm.loader.config.get("vocab_size"))
        if bad:
            return _error(bad)
        if llm.failed:
            return _error(f"engine is down: {llm.failed}", HTTPStatus.INTERNAL_SERVER_ERROR)
        if request.echo and request.logprobs is not None:
            params["prompt_logprobs"] = request.logprobs if request.prompt_logprobs is None else \
                request.prompt_logprobs
        stream = await llm.add_requests_async(raw_request, token_ids, max_tokens, request.ignore_eos,
                                              request.temperature, request.top_p, request.top_k,
                                              request.repetition_penalty, stop=request.stop,
                                              logprobs=request.logprobs, **params)
        streams = stream if "n" in params else [stream]
        echo = (await _in_thread(_prompt_text, request.prompt, token_ids), token_ids) if request.echo else None
        if request.stream:
            return StreamingResponse(completion_stream_generator(streams, request, echo),
                                     media_type="text/event-stream")
        return JSONResponse(content=(await completion_generator(streams, request, echo)).model_dump())

    @app.post("/tokenize")
    async def tokenize(request: TokenizeRequest):
        toks = llm.encode(request.prompt) if request.prompt is not None else llm.encode(None, True, request.messages)
        return JSONResponse(TokenizeResponse(count=len(toks), max_model_len=llm.model_max_length,
                                             tokens=toks).model_dump())

    @app.post("/detokenize")
    async def detokenize(request: DetokenizeRequest):
        return JSONResponse(DetokenizeResponse(prompt=llm.tokenizer.decode(request.tokens)).model_dump())

    @app.post("/start_profile")
    async def start_profile():
        llm.start_profile()
        return JSONResponse(content={"message": "Profiler started", "success": True})

    @app.post("/stop_profile")
    async def stop_profile():
        llm.stop_profile()
        return JSONResponse(content={"message": "Profiler stopped", "success": True})

    return app


def make_parser() -> argparse.ArgumentParser:
    """CLI surface of the reference (gllm/entrypoints/api_server.py:134-278)."""
    p = argparse.ArgumentParser(description="gllm_b200 OpenAI-compatible server")
    p.add_argument("--host", type=str, default="0.0.0.0")
    p.add_argument("--port", type=int, default=8000)
    p.add_argument("--master-addr", type=str, default="0.0.0.0")
    p.add_argument("--master-port", type=int, default=8001)
    p.add_argument("--zmq-port-base", type=int, default=8002)
    p.add_argument("--model-path", type=str, required=True, help="local HF directory or preset:<name>")
    p.add_argument("--load-format", type=str, choices=["auto", "dummy"], default="auto")
    p.add_argument("--disable-thinking", action="store_true")
    p.add_argument("--model-max-length", type=int, default=None)
    p.add_argument("--use-async-worker", action="store_true")
    p.add_argument("--async-schedule", action=argparse.BooleanOptionalAction, default=True,
                   help="queue the next decode step before the previous step's tokens are back on the host "
                        "(default on; --no-async-schedule for the strictly synchronous loop)")
    p.add_argument("--gpu-memory-util", type=float, default=0.9)
    p.add_argument("--enable-prefix-caching", action="store_true")
    p.add_argument("--page-size", type=int, default=16)
    p.add_argument("--disable-cuda-graph", action="store_true")
    p.add_argument("--max-cuda-graph-bs", type=int, default=512)
    p.add_argument("--pp", type=int, default=1)
    p.add_argument("--tp", type=int, default=1)
    p.add_argument("--disable-ep", action="store_true")
    p.add_argument("--assigned-layers", type=str, default=None, help="e.g. 16,16,17,15")
    p.add_argument("--maxd", type=int, default=2048)
    p.add_argument("--maxp", type=int, default=8192)
    p.add_argument("--minp", type=int, default=32)
    p.add_argument("--iterp", type=int, default=8)
    p.add_argument("--kvthresh", type=float, default=0.05)
    p.add_argument("--schedule-method", type=str, default="chunked_prefill",
                   choices=["split_pd", "chunked_prefill", "token_throttling"])
    p.add_argument("--launch-mode", type=str, default="normal", choices=["normal", "master", "slave"])
    p.add_argument("--ranks", type=str, default=None, help="comma separated global ranks hosted by this node")
    p.add_argument("--mm-processor-min-pixels", type=int, default=None)
    p.add_argument("--mm-processor-max-pixels", type=int, default=None)
    p.add_argument("--tp-mode", type=str, default="fused", choices=["fused", "nccl"])
    return p


def engine_kwargs(args) -> dict:
    return dict(model_path=args.model_path, host=args.host, master_addr=args.master_addr,
                master_port=args.master_port, zmq_port_base=args.zmq_port_base, launch_mode=args.launch_mode,
                worker_ranks=args.ranks, load_format=args.load_format, gpu_memory_util=args.gpu_memory_util,
                page_size=args.page_size, maxd=args.maxd, maxp=args.maxp, minp=args.minp, iterp=args.iterp,
                kvthresh=args.kvthresh, enable_prefix_caching=args.enable_prefix_caching, pp_size=args.pp,
                tp_size=args.tp, use_ep=not args.disable_ep, assigned_layers=args.assigned_layers,
                use_async_worker=args.use_async_worker, async_schedule=args.async_schedule,
                use_thinking=not args.disable_thinking,
                schedule_method=args.schedule_method, disable_cuda_graph=args.disable_cuda_graph,
                max_cuda_graph_bs=args.max_cuda_graph_bs, model_max_length=args.model_max_length,
                mm_processor_min_pixels=args.mm_processor_min_pixels,
                mm_processor_max_pixels=args.mm_processor_max_pixels, tp_mode=args.tp_mode)


async def run_server(app, host: str, port: int):
    import uvicorn
    server = uvicorn.Server(uvicorn.Config(app, port=port, host=host, log_level="warning"))
    task = asyncio.get_running_loop().create_task(server.serve())
    try:
        await task
    except asyncio.CancelledError:
        await server.shutdown()


def main(argv: Optional[List[str]] = None):
    args = make_parser().parse_args(argv)
    from gllm_b200.engine.async_llm_engine import AsyncLLM
    kw = engine_kwargs(args)
    engine = AsyncLLM(kw.pop("model_path"), **kw)
    if args.launch_mode == "slave":
        # a slave node only hosts workers (reference: api_server.py:312-322)
        logger.info("slave node: hosting ranks %s", args.ranks)
        for p in engine.procs:
            p.join()
        return
    app = build_app(engine)
    logger.info("serving on http://%s:%d", args.host, args.port)
    asyncio.run(run_server(app, args.host, args.port))


if __name__ == "__main__":
    main()
