"""Engine configuration: one dataclass carrying every public knob of the reference CLI / `LLM`
constructor (gllm/llm_engine.py:19-49, gllm/entrypoints/api_server.py:134-278)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional


@dataclass
class EngineConfig:
    model_path: object = None                 # local HF dir | "preset:<name>" | config dict
    load_format: str = "auto"                 # auto | dummy
    host: str = "0.0.0.0"
    master_addr: str = "127.0.0.1"
    master_port: int = 8001
    zmq_port_base: int = 8002
    launch_mode: str = "normal"               # normal | master | slave | inproc
    worker_ranks: Optional[List[int]] = None
    gpu_memory_util: float = 0.9
    page_size: int = 16
    maxd: int = 2048
    maxp: int = 2048
    minp: int = 32
    iterp: int = 8
    kvthresh: float = 0.05
    enable_prefix_caching: bool = True
    pp_size: int = 1
    tp_size: int = 1
    use_ep: bool = True
    assigned_layers: Optional[List[int]] = None
    use_async_worker: bool = False
    async_schedule: bool = True               # lookahead decode scheduling (next step queued before tokens return)
    use_thinking: bool = True
    schedule_method: str = "chunked_prefill"  # split_pd | chunked_prefill | token_throttling
    disable_cuda_graph: bool = False
    max_cuda_graph_bs: int = 32
    model_max_length: Optional[int] = None
    mm_processor_min_pixels: Optional[int] = None
    mm_processor_max_pixels: Optional[int] = None
    # --- additions of this engine ---
    device: Optional[str] = None              # None: cuda if available else cpu
    tp_mode: str = "fused"                    # fused (NVLink kernels) | nccl (baseline / oracle)
    num_cpu_pages: int = 512                  # KV pages when running on CPU
    num_gpu_pages: Optional[int] = None       # override the memory-derived page count
    seed: int = 0
    log_stats: bool = True
    tokenizer_path: Optional[str] = None
    lora_modules: Optional[Dict[str, str]] = None   # multi-LoRA: adapter name -> PEFT directory (gllm_b200/lora.py)
    max_lora_rank: int = 16                           # every adapter is zero-padded to this rank (<= 64)

    @property
    def world_size(self) -> int:
        return self.pp_size * self.tp_size

    @property
    def max_num_batched_tokens(self) -> int:
        # reference: gllm/model_runner.py:61-65
        return self.maxp if self.schedule_method in ("chunked_prefill", "split_pd") else self.maxp + self.maxd

    @property
    def max_running_seqs(self) -> int:
        # reference: gllm/model_runner.py:67-71
        return self.maxp if self.schedule_method in ("chunked_prefill", "split_pd") else self.maxd

    def resolved_device(self, local_rank: int = 0) -> str:
        import torch
        if self.device:
            return self.device if (":" in self.device or self.device == "cpu") else f"{self.device}:{local_rank}"
        return f"cuda:{local_rank}" if torch.cuda.is_available() else "cpu"


def capture_sizes(max_bs: int) -> List[int]:
    """Power-of-two CUDA-graph buckets up to max_bs, descending; max_bs itself is always a bucket
    (reference: gllm/model_runner.py:145-163)."""
    if max_bs <= 0:
        return []
    sizes, s = [], 1
    while s <= max_bs:
        sizes.append(s)
        s *= 2
    if sizes[-1] != max_bs:
        sizes.append(max_bs)
    return list(reversed(sizes))
