"""Device-directed op entry points used by the model code.

CUDA tensors always run the hand-written sm_90a kernels (`ops.sm100`); CPU tensors run the
PyTorch oracle (`ops.ref`) — that is the CPU plumbing/test path only, never a GPU fallback.
"""
from __future__ import annotations

from gllm_b200.ops import ref


def _sm():
    from gllm_b200.ops import sm100
    return sm100


def linear(x, w, bias=None, out=None):
    if isinstance(w, tuple):  # (e4m3 weight, fp32 block scale_inv): block-scaled fp8 GEMM
        if x.is_cuda:
            return _sm().linear_fp8_block(x, w[0], w[1], bias, out=out)
        return ref.linear_fp8_block(x, w[0], w[1], bias)
    if x.is_cuda:
        return _sm().linear(x, w, bias, out=out)
    return ref.linear(x, w, bias)


def linear_silu_mul(x, w_interleaved):
    if x.is_cuda:
        return _sm().linear_silu_mul(x, w_interleaved)
    return ref.linear_silu_mul(x, w_interleaved)


def rmsnorm(x, w, eps, residual=None, out=None):
    """-> (normed, residual_out). With `residual`, computes residual += x first (in place on GPU)."""
    if x.is_cuda:
        return _sm().rmsnorm(x, w, eps, residual, out=out)
    o, r = ref.rmsnorm(x, w, eps, residual)
    if out is not None:
        out.copy_(o)
        o = out
    if residual is not None:
        residual.copy_(r)  # same in-place contract as the GPU kernel
        r = residual
    return o, r


def silu_and_mul(x):
    if x.is_cuda:
        return _sm().silu_and_mul(x)
    return ref.silu_and_mul(x)


def embedding(ids, table, vocab_start=0, vocab_end=None):
    if table.is_cuda:
        return _sm().embedding(ids, table, vocab_start, vocab_end)
    return ref.embedding(ids, table, vocab_start, vocab_end)


def gather_rows(src, idx):
    if src.is_cuda:
        return _sm().gather_rows(src.contiguous(), idx)
    return src[idx.long()]


def rope_kv_write(q, k, v, positions, cos_sin, rot_dim, neox, q_norm_w, k_norm_w, eps, k_cache, v_cache, slots,
                  mrope_section=None):
    if q.is_cuda:
        return _sm().rope_kv_write(q, k, v, positions, cos_sin, rot_dim, neox, q_norm_w, k_norm_w, eps, k_cache,
                                   v_cache, slots, mrope_section)
    return ref.rope_kv_write(q, k, v, positions, cos_sin, rot_dim, neox, q_norm_w, k_norm_w, eps, k_cache,
                             v_cache, slots, mrope_section)


def paged_attention(q, k_cache, v_cache, inp, scale, num_q_heads, head_dim):
    """`inp` is the worker's InputData (device batch state)."""
    if q.is_cuda:
        return _sm().paged_attention(q, k_cache, v_cache, inp.block_table, inp.seq_lens, inp.query_start_loc, scale,
                                     num_q_heads, head_dim, inp.padded_tokens or inp.num_decode_seqs,
                                     inp.padded_tokens or inp.num_seqs, inp.max_q_len, inp.max_seq_len,
                                     splits=inp.decode_splits)
    return ref.paged_attention(q, k_cache, v_cache, inp.block_table, inp.seq_lens, inp.query_start_loc, scale,
                               num_q_heads, head_dim)



def lora_shrink(x, A, csr):
    """`csr` = (slots, row_off, rows, number of groups) of the batch (InputData.lora)."""
    if x.is_cuda:
        return _sm().lora_shrink(x, A, *csr)
    return ref.lora_shrink(x, A, *csr[:3])


def lora_expand_add(y, u, B, bounds, csr):
    if y.is_cuda:
        return _sm().lora_expand_add(y, u, B, bounds, *csr)
    return ref.lora_expand_add(y, u, B, bounds, *csr[:3])


def lora_expand_silu_mul(pre, u, B, csr):
    if pre.is_cuda:
        return _sm().lora_expand_silu_mul(pre, u, B, *csr)
    return ref.lora_expand_silu_mul(pre, u, B, *csr[:3])
