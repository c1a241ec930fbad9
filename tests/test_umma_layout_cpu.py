"""Address arithmetic of the wgmma prefill attention kernel (csrc/attn/prefill_attention_tc.cu), checked on the
CPU against the canonical wgmma shared-memory layouts (CuTe `mma_traits_sm90_gmma.hpp`: SW128 K-major
`((8,m),(T,2)):((8T,SBO),(1,T))`, SW128 MN-major `((T,8,m),(8,k)):((1,T,LBO),(8T,SBO))`, T = 8 bf16 per 16 bytes)
and the 128-byte TMA swizzle. The K-major half of this model is what the GPU-validated GEMM relies on; the test's
purpose is to catch slips in slab strides, LBO / SBO / K-advance and the hand-written swizzled stores before any
GPU time is spent on the kernel.
"""
import numpy as np
import pytest

ELEM = 2                      # bf16


def swz(addr: int) -> int:
    """128-byte swizzle on absolute shared-memory byte addresses: 16-byte chunk index ^= row-in-atom."""
    return addr ^ (((addr >> 7) & 7) << 4)


def tma_box_store(smem, dst, box):
    """cp.async.bulk.tensor with SWIZZLE_128B: box[rows][64] bf16, inner dimension = one 128-byte line."""
    rows, cols = box.shape
    assert cols == 64 and dst % 1024 == 0
    for r in range(rows):
        for c in range(cols):
            a = swz(dst + r * 128 + c * ELEM)
            smem[a // ELEM] = box[r, c]


def kmajor_elem(smem, start, sbo, mn, k):
    """Operand element (mn, k) of ONE MMA (k < 16) for a K-major SW128 descriptor with start address `start`."""
    a = start + (mn % 8) * 128 + (mn // 8) * sbo + k * ELEM
    return smem[swz(a) // ELEM]


def mnmajor_elem(smem, start, lbo, sbo, mn, k):
    """Operand element (mn, k) for an MN-major SW128 descriptor: 64 mn-values per 128-byte line, next 64 at LBO;
    8 k-rows are 8 consecutive lines, the next 8 at SBO."""
    a = start + (mn % 64) * ELEM + (mn // 64) * lbo + (k % 8) * 128 + (k // 8) * sbo
    return smem[swz(a) // ELEM]


def a_tile_off(row, c):
    """prefill_attention_tc.cu: byte offset of (row, 16-byte chunk c) in a [c / 8][128 rows][128 B] operand tile."""
    return (c >> 3) * (128 * 128) + row * 128 + (((c & 7) ^ (row & 7)) << 4)


@pytest.mark.parametrize("D,KV,page", [(128, 128, 16), (128, 64, 16), (64, 128, 8), (64, 64, 32)])
def test_kv_tiles_assembled_by_tma_match_both_operand_forms(D, KV, page):
    rng = np.random.default_rng(0)
    K = rng.integers(1, 60000, size=(KV, D)).astype(np.int64)       # logical tile [key][d], unique-ish values
    V = rng.integers(1, 60000, size=(KV, D)).astype(np.int64)
    tile_bytes = KV * D * ELEM
    smem = np.zeros(2 * tile_bytes // ELEM, dtype=np.int64)
    sk, sv = 0, tile_bytes
    # producer: one TMA box per (page, 64-wide slab) at  slab * (KV*128) + j * (page*128)
    for j in range(KV // page):
        for sl in range(D // 64):
            off = sl * (KV * 128) + j * (page * 128)
            tma_box_store(smem, sk + off, K[j * page:(j + 1) * page, sl * 64:(sl + 1) * 64])
            tma_box_store(smem, sv + off, V[j * page:(j + 1) * page, sl * 64:(sl + 1) * 64])
    # S = Q K^T: B operand = K tile, K-major, N = keys; per slab kd and k-step kk the start address advances 32 B
    for kd in range(D // 64):
        for kk in range(4):
            start = sk + kd * (KV * 128) + kk * 32
            for n in (0, 1, 7, 8, 9, KV // 2, KV - 1):
                for k in range(16):
                    assert kmajor_elem(smem, start, 1024, n, k) == K[n, kd * 64 + kk * 16 + k]
    # O += P V: B operand = V tile, MN-major, N = d (two 64-wide slabs via LBO), K = keys; 2048 B per 16-key step
    lbo, sbo = KV * 128, 1024
    for kstep in range(KV // 16):
        start = sv + kstep * 2048
        for n in (0, 1, 63, 64 % D, D - 1):
            for k in range(16):
                assert mnmajor_elem(smem, start, lbo, sbo, n, k) == V[kstep * 16 + k, n]


@pytest.mark.parametrize("cols", [64, 128])
def test_hand_swizzled_q_and_p_stores_form_a_kmajor_operand(cols):
    """Q (cols = D) is written by the MMA warpgroups, 16 bytes at a time, with `a_tile_off`; the same layout with
    cols = KV is the K-major form of any 128-row operand tile."""
    rng = np.random.default_rng(1)
    A = rng.integers(1, 60000, size=(128, cols)).astype(np.int64)
    smem = np.zeros(128 * cols, dtype=np.int64)
    for row in range(128):
        for c in range(cols // 8):
            base = a_tile_off(row, c)
            for e in range(8):
                smem[(base + e * ELEM) // ELEM] = A[row, c * 8 + e]
    for ks in range(cols // 64):                 # one descriptor per 64-column slab, 32 B per 16-column k-step
        for kk in range(4):
            start = ks * (128 * 128) + kk * 32
            for m in (0, 5, 8, 77, 127):
                for k in range(16):
                    assert kmajor_elem(smem, start, 1024, m, k) == A[m, ks * 64 + kk * 16 + k]
