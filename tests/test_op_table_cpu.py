"""The model forward and the sampler call one op table per device (`gllm_b200.ops.table`) with the same arguments on
either: every op they call has the same signature in the kernel table and in its CPU stand-ins. Importing `ops.sm100`
loads no library, so this runs without a GPU."""
import inspect

import pytest
import torch

from gllm_b200 import ops
from gllm_b200.ops import cpu, sm100

MODEL_OPS = ["linear", "linear_silu_mul", "linear_fp8_block", "rmsnorm", "silu_and_mul", "embedding", "gather_rows",
             "rope_kv_write", "paged_attention", "lora_shrink", "lora_expand_add", "lora_expand_silu_mul",
             "topk_softmax", "grouped_topk", "fused_experts", "fused_experts_fp8"]
SAMPLER_OPS = ["sample", "vp_candidates", "vp_final", "mark_seen", "bias_account", "bias_rebuild", "logprobs_shard",
               "prompt_logprobs_shard", "logprobs_final", "kv_copy_pages"]


@pytest.mark.parametrize("name", MODEL_OPS + SAMPLER_OPS)
def test_cpu_stand_in_has_the_kernel_signature(name):
    assert inspect.signature(getattr(cpu, name)) == inspect.signature(getattr(sm100, name))


def test_table_per_device():
    assert ops.table(torch.device("cpu")) is ops.cpu
    assert ops.table("cpu") is ops.cpu
    assert ops.table(torch.device("cuda", 0)) is ops.sm100
