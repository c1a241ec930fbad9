"""Small framework helpers (reference: gllm/utils/__init__.py — thread-pool offload, pinned H2D copies, the
download lock, numeric helpers; the custom-op registration and FlashAttention-version probing of the reference
have no counterpart here: every kernel is an in-tree C ABI symbol).
"""
from __future__ import annotations

import asyncio
import functools
import hashlib
import os
import tempfile
import uuid
from typing import Awaitable, Callable, Optional, TypeVar

import torch

T = TypeVar("T")


def make_async(fn: Callable[..., T], executor=None) -> Callable[..., Awaitable[T]]:
    """Run a blocking callable on the loop's thread pool so the event loop keeps serving
    (reference: utils/__init__.py:44-57)."""

    @functools.wraps(fn)
    def wrapper(*args, **kwargs):
        loop = asyncio.get_running_loop()
        return loop.run_in_executor(executor, functools.partial(fn, *args, **kwargs))

    return wrapper


def random_uuid() -> str:
    return uuid.uuid4().hex


def async_tensor_h2d(data, dtype: torch.dtype, device, pin_memory: Optional[bool] = None) -> torch.Tensor:
    """Host list / array -> device tensor through a pinned staging buffer and a non-blocking copy
    (reference: utils/__init__.py:64-72)."""
    device = torch.device(device)
    if pin_memory is None:
        pin_memory = device.type == "cuda"
    host = torch.tensor(data, dtype=dtype, pin_memory=pin_memory)
    return host.to(device, non_blocking=True)


def round_up(x: int, y: int) -> int:
    return (x + y - 1) // y * y


def round_down(x: int, y: int) -> int:
    return x // y * y


def cdiv(a: int, b: int) -> int:
    return -(-a // b)


def dtype_bytes(dtype: torch.dtype) -> int:
    return torch.empty(0, dtype=dtype).element_size()


def device_capability(index: int = 0) -> Optional[int]:
    """Compute capability as major*10 + minor (90 on H100), None without a CUDA device."""
    if not torch.cuda.is_available():
        return None
    major, minor = torch.cuda.get_device_capability(index)
    return major * 10 + minor


def clamp_overflow(x: torch.Tensor, margin: float = 1000.0) -> torch.Tensor:
    """fp16 safety net for activations that overflowed (used by the vision towers when they run in fp16;
    reference: utils/__init__.py:261-268). A no-op when every value is finite."""
    if x.dtype == torch.float16 and not torch.isfinite(x).all():
        lim = torch.finfo(x.dtype).max - margin
        x = torch.nan_to_num(x, nan=0.0, posinf=lim, neginf=-lim).clamp_(-lim, lim)
    return x


# ---------------------------------------------------------------------------------------------------------
# model path resolution: local directory, preset:<name>, dict config, or a HuggingFace repo id
# ---------------------------------------------------------------------------------------------------------
def _lock_path(name: str, cache_dir: Optional[str] = None) -> str:
    root = cache_dir or os.environ.get("GLLM_B200_LOCK_DIR") or tempfile.gettempdir()
    os.makedirs(root, exist_ok=True)
    digest = hashlib.sha256(name.encode()).hexdigest()[:16]
    return os.path.join(root, f"gllm_b200_{digest}.lock")


def download_lock(name: str, cache_dir: Optional[str] = None):
    """Inter-process lock keyed on the model name: the front-end and every spawned worker resolve the same
    repo id, only one of them downloads (reference: utils/__init__.py:95-105)."""
    import filelock
    return filelock.FileLock(_lock_path(name, cache_dir), mode=0o666)


def resolve_model_path(model_path, cache_dir: Optional[str] = None, _download=None):
    """Map what the user passed as `model_path` to something the loader can open.

    dict configs, `preset:<name>` and existing directories are returned unchanged; anything else is treated as
    a HuggingFace repo id and fetched with `huggingface_hub.snapshot_download` (weights, config, tokenizer)
    under `download_lock` (reference: model_loader.py:41-85 downloads in every worker under a file lock)."""
    if not isinstance(model_path, str) or model_path.startswith("preset:") or os.path.isdir(model_path):
        return model_path
    if os.path.sep in model_path and model_path.count("/") != 1:
        raise FileNotFoundError(f"model path {model_path!r} does not exist")
    if _download is None:
        from huggingface_hub import snapshot_download as _download
    with download_lock(model_path, cache_dir):
        return _download(model_path, cache_dir=cache_dir,
                         allow_patterns=["*.safetensors", "*.bin", "*.json", "*.txt", "*.model", "*.tiktoken",
                                         "*.jinja"])
