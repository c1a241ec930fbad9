"""OpenAI-compatible request / response schemas (pydantic v2).

Written against the public OpenAI API shape; field coverage follows what the reference accepts
(gllm/entrypoints/protocol.py:165-716) plus a filled `usage`. Unknown request fields are ignored
rather than rejected so stock OpenAI clients work unchanged.

Log-probabilities (chat `logprobs` + `top_logprobs`, completions `logprobs: N`) are those of the raw model
distribution: log_softmax in fp32 of the logits the LM head produced, over the real vocabulary, before repetition
penalty, temperature, top-k and top-p. So they do not depend on the sampling parameters, and the sampled token's
log-prob is reported under that distribution even when it was drawn with a temperature or a filter. Every generated
token gets its log-prob and the N most likely tokens (0 <= N <= 20), ordered by logit, ties to the lower token id; for
a greedy request the first of them is the sampled token when it uses no penalty or bias. Token strings are `tokenizer.decode([id])` (`bytes`: its UTF-8 encoding), or "token_id:<id>" without a
tokenizer. A log-prob of -inf is reported as -9999.0. Out-of-range `top_logprobs` / `logprobs`, or `top_logprobs > 0` without `logprobs`, is a 400.

`frequency_penalty`, `presence_penalty` and `logit_bias` follow OpenAI's formula. For a generated token, with x the
raw LM-head logit of token j:

    x1 = repetition_penalty(x)            # multiplicative, over prompt + output, as before
    x2 = x1 - frequency_penalty * c_j - presence_penalty * [c_j > 0] + logit_bias_j
    t  = x2 / temperature                 # then top-k -> top-p -> draw

c_j counts the occurrences of token j among the tokens this request has generated so far (prompt tokens do not
count). A greedy request (top_k == 1) takes the argmax of x2, ties to the lower token id. `seed`: a seeded request
keys its random draw by (seed, index in the sequence of the token being produced, token id), so given the same logits
it draws the same token whatever the batch, its row in it, the engine's step count, CUDA graphs, lookahead, preemption
or the tensor-parallel degree; without a seed the draw comes from the engine's own stream. A 400 answers: a penalty
outside [-2, 2] or not finite; a logit_bias key that is not an int in [0, vocab_size), a value outside [-100, 100] or
not finite, or more than 1024 entries (this engine's own cap); a seed that does not fit a signed 64-bit int.

Completions `echo: true` puts the prompt text in front of each choice's `text` (a token-id prompt is decoded). With
`logprobs: N` as well, `tokens` / `token_logprobs` / `top_logprobs` / `text_offset` start with the prompt's entries,
under the same distribution and with the same N (`prompt_logprobs: M` sets another N for the prompt; it is a 400
without `echo: true` and `logprobs`, which are where the entries are reported): the first prompt
token has `token_logprobs[0] = null` and `top_logprobs[0] = null`, and `text_offset` runs from 0 across prompt and
completion. When streaming, the first chunk of each choice carries the echoed prompt and its entries. `max_tokens: 0`
is accepted only with `echo: true`: the response is the echoed prompt (and its entries) with `finish_reason: "length"`
and `usage.completion_tokens = 0`; the engine still samples one token internally and drops it. A request with prompt
log-probs takes no prefix-cache hits. `prompt_logprobs` outside [0, 20] is a 400. Chat completions have no prompt
log-probs.

Multi-LoRA: a server started with `--lora-modules name=path ...` serves each PEFT adapter next to the base model. In
chat and completions, a `model` equal to an adapter name runs the request with that adapter; the base model's id (or
no `model`) runs the base model; any other `model` is a 404 with `code: "model_not_found"`. `/v1/models` lists the
base model, then one card per adapter with `root` = its path and `parent` = the base model's id. Without adapters,
`model` is not looked at and every response is what it was before.

`n` asks for n independent choices of one request (parallel sampling). The prompt is prefilled once, its full KV
pages are shared by the choices and its partial last page is copied on the device; every choice draws its first token
from the same logits row, then continues as a sequence of its own with its own stop handling, `finish_reason` and
logprobs. `choices[i].index` is i. `usage.prompt_tokens` counts the prompt once, `completion_tokens` is summed over the
choices. When streaming, every chunk carries one choice with its index, each choice ends with its own finish chunk and
the last finish chunk carries `usage`. With `seed = s`, choice i draws as an n = 1 request seeded with s + i would
(wrapping in signed 64-bit). A stop string ends only its own choice; a client disconnect aborts all of them. `n` must
be an integer in [1, 128] and at most the engine's max_running_seqs, and n > 1 is refused with multimodal input (400).
`n = 1` (or absent) gives exactly the single-choice response. `best_of` is ignored.
"""
from __future__ import annotations

import time
import uuid
from typing import Any, Dict, List, Literal, Optional, Union

from pydantic import BaseModel, ConfigDict, Field


def _rid(prefix: str) -> str:
    return f"{prefix}-{uuid.uuid4().hex}"


class OpenAIBase(BaseModel):
    model_config = ConfigDict(extra="allow")


class ErrorResponse(OpenAIBase):
    object: str = "error"
    message: str
    type: str
    param: Optional[str] = None
    code: int


class ModelPermission(OpenAIBase):
    id: str = Field(default_factory=lambda: _rid("modelperm"))
    object: str = "model_permission"
    created: int = Field(default_factory=lambda: int(time.time()))
    allow_create_engine: bool = False
    allow_sampling: bool = True
    allow_logprobs: bool = True
    allow_search_indices: bool = False
    allow_view: bool = True
    allow_fine_tuning: bool = False
    organization: str = "*"
    group: Optional[str] = None
    is_blocking: bool = False


class ModelCard(OpenAIBase):
    id: str
    object: str = "model"
    created: int = Field(default_factory=lambda: int(time.time()))
    owned_by: str = "gllm_b200"
    root: Optional[str] = None
    parent: Optional[str] = None
    max_model_len: Optional[int] = None
    permission: List[ModelPermission] = Field(default_factory=list)


class ModelList(OpenAIBase):
    object: str = "list"
    data: List[ModelCard] = Field(default_factory=list)


class UsageInfo(OpenAIBase):
    prompt_tokens: int = 0
    total_tokens: int = 0
    completion_tokens: Optional[int] = 0


class StreamOptions(OpenAIBase):
    include_usage: Optional[bool] = True
    continuous_usage_stats: Optional[bool] = False


class _SamplingMixin(OpenAIBase):
    temperature: Optional[float] = None
    top_p: Optional[float] = None
    top_k: Optional[int] = None
    repetition_penalty: Optional[float] = None
    ignore_eos: bool = False
    stream: Optional[bool] = False
    stream_options: Optional[StreamOptions] = None
    n: Optional[int] = 1
    seed: Optional[int] = None
    stop: Optional[Union[str, List[str]]] = None
    frequency_penalty: Optional[float] = 0.0
    presence_penalty: Optional[float] = 0.0
    logit_bias: Optional[Dict[str, float]] = None
    user: Optional[str] = None


class ChatCompletionRequest(_SamplingMixin):
    messages: List[Dict[str, Any]]
    model: Optional[str] = None
    max_tokens: Optional[int] = None
    max_completion_tokens: Optional[int] = None
    logprobs: Optional[bool] = False
    top_logprobs: Optional[int] = 0
    tools: Optional[List[Dict[str, Any]]] = None
    tool_choice: Optional[Union[str, Dict[str, Any]]] = None
    response_format: Optional[Dict[str, Any]] = None
    chat_template_kwargs: Optional[Dict[str, Any]] = None

    def output_len(self) -> Optional[int]:
        return self.max_completion_tokens if self.max_completion_tokens is not None else self.max_tokens


class CompletionRequest(_SamplingMixin):
    model: Optional[str] = None
    prompt: Union[str, List[str], List[int], List[List[int]]]
    max_tokens: Optional[int] = 16
    echo: Optional[bool] = False
    logprobs: Optional[int] = None
    prompt_logprobs: Optional[int] = None
    suffix: Optional[str] = None
    best_of: Optional[int] = None


class ChatMessage(OpenAIBase):
    role: str
    content: Optional[str] = None
    reasoning_content: Optional[str] = None
    tool_calls: List[Dict[str, Any]] = Field(default_factory=list)


class ChatCompletionResponseChoice(OpenAIBase):
    index: int
    message: ChatMessage
    logprobs: Optional[Any] = None
    finish_reason: Optional[str] = "stop"


class ChatCompletionResponse(OpenAIBase):
    id: str = Field(default_factory=lambda: _rid("chatcmpl"))
    object: Literal["chat.completion"] = "chat.completion"
    created: int = Field(default_factory=lambda: int(time.time()))
    model: Optional[str] = None
    choices: List[ChatCompletionResponseChoice]
    usage: UsageInfo


class DeltaMessage(OpenAIBase):
    role: Optional[str] = None
    content: Optional[str] = None
    reasoning_content: Optional[str] = None
    tool_calls: List[Dict[str, Any]] = Field(default_factory=list)


class ChatCompletionResponseStreamChoice(OpenAIBase):
    index: int
    delta: DeltaMessage
    logprobs: Optional[Any] = None
    finish_reason: Optional[str] = None


class ChatCompletionStreamResponse(OpenAIBase):
    id: str = Field(default_factory=lambda: _rid("chatcmpl"))
    object: Literal["chat.completion.chunk"] = "chat.completion.chunk"
    created: int = Field(default_factory=lambda: int(time.time()))
    model: Optional[str] = None
    choices: List[ChatCompletionResponseStreamChoice]
    usage: Optional[UsageInfo] = None


class CompletionResponseChoice(OpenAIBase):
    index: int
    text: str
    logprobs: Optional[Any] = None
    finish_reason: Optional[str] = "stop"


class CompletionResponse(OpenAIBase):
    id: str = Field(default_factory=lambda: _rid("cmpl"))
    object: str = "text_completion"
    created: int = Field(default_factory=lambda: int(time.time()))
    model: Optional[str] = None
    choices: List[CompletionResponseChoice]
    usage: UsageInfo


class CompletionResponseStreamChoice(OpenAIBase):
    index: int
    text: str
    logprobs: Optional[Any] = None
    finish_reason: Optional[str] = None


class CompletionStreamResponse(OpenAIBase):
    id: str = Field(default_factory=lambda: _rid("cmpl"))
    object: str = "text_completion"
    created: int = Field(default_factory=lambda: int(time.time()))
    model: Optional[str] = None
    choices: List[CompletionResponseStreamChoice]
    usage: Optional[UsageInfo] = None


class TokenizeRequest(OpenAIBase):
    model: Optional[str] = None
    prompt: Optional[str] = None
    messages: Optional[List[Dict[str, Any]]] = None
    add_special_tokens: bool = True


class TokenizeResponse(OpenAIBase):
    count: int
    max_model_len: int
    tokens: List[int]


class DetokenizeRequest(OpenAIBase):
    model: Optional[str] = None
    tokens: List[int]


class DetokenizeResponse(OpenAIBase):
    prompt: str
