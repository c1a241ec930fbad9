"""gllm_b200 — a Hopper (H100 / sm_90a) native LLM serving engine.

Public API mirrors the reference engine (`gllm/__init__.py:1-3`):

    from gllm_b200 import LLM
"""
__version__ = "0.1.0"


def __getattr__(name):
    if name == "LLM":
        from gllm_b200.engine.llm_engine import LLM

        return LLM
    if name == "AsyncLLM":
        from gllm_b200.engine.async_llm_engine import AsyncLLM

        return AsyncLLM
    raise AttributeError(name)
