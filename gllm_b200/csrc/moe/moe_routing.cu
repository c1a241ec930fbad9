// MoE routing + token permutation kernels for sm_90a.
//
//   topk_softmax      softmax over experts + top-k (+renorm)            (ref: vLLM _moe_C.topk_softmax,
//                                                                         gllm/layers/moe/topk.py:141-171)
//   grouped_topk      DeepSeek group-limited routing (sigmoid/softmax scores, bias correction, top
//                     groups by sum of top-2 / max, renorm, scaling)     (gllm/layers/moe/topk.py:29-138)
//   moe_align         counting sort of the (token, k) slots by LOCAL expert into 128-row tiles:
//                     expert_count -> padded offsets -> per-tile expert id, slot -> row position
//                     (ref: moe_align_block_size, gllm/layers/moe/moe_align_block_size.py:10-78)
//   moe_gather        xs[row] = x[token(row)]  (rows of padding are zero)
//   moe_combine       out[t] = sum_j w[t,j] * y[pos[t,j]]   (ref: moe_sum, fused with the routing weight)
//
// The expert GEMMs themselves are the wgmma kernel in gemm/gemm_bf16.cu running in grouped mode
// (per-M-tile expert id selects the weight slab; the tile count is read from device memory so the
// whole MoE block is CUDA-graph capturable without a host sync).
#include "../common/host_utils.h"
#include "../common/ptx.cuh"

namespace b200 {

static constexpr int kTileM = 128;

// ---------------------------------------------------------------------------------------------
// top-k softmax: one warp per token, E <= 512
// ---------------------------------------------------------------------------------------------
template <int VPT>  // values per lane, E <= 32 * VPT
__global__ void topk_softmax_kernel(const __nv_bfloat16* __restrict__ logits, int64_t ld, float* __restrict__ w_out,
                                    int32_t* __restrict__ id_out, int T, int E, int K, int renorm) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= T) return;
  const __nv_bfloat16* row = logits + static_cast<size_t>(warp) * ld;
  float v[VPT];
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int e = lane + i * 32;
    v[i] = e < E ? __bfloat162float(row[e]) : -INFINITY;
    mx = fmaxf(mx, v[i]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    v[i] = (lane + i * 32 < E) ? __expf(v[i] - mx) : 0.f;
    sum += v[i];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float inv = 1.f / sum;
  float wsum = 0.f;
  float my_w = 0.f;
  int my_id = 0;
  for (int k = 0; k < K; ++k) {
    float best = -1.f;
    int bi = 0x7fffffff;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int e = lane + i * 32;
      if (v[i] > best) { best = v[i]; bi = e; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if ((bi & 31) == lane) v[bi >> 5] = -1.f;  // remove the winner
    if (lane == k) { my_w = best * inv; my_id = bi; }
    wsum += best * inv;
  }
  if (lane < K) {
    w_out[static_cast<size_t>(warp) * K + lane] = renorm ? my_w / wsum : my_w;
    id_out[static_cast<size_t>(warp) * K + lane] = my_id;
  }
}

// ---------------------------------------------------------------------------------------------
// grouped top-k (DeepSeek): one warp per token, E <= 512, groups <= 32, any E % n_group == 0
// ---------------------------------------------------------------------------------------------
template <int VPT>
__global__ void grouped_topk_kernel(const __nv_bfloat16* __restrict__ logits, int64_t ld, const float* __restrict__ bias,
                                    float* __restrict__ w_out, int32_t* __restrict__ id_out, int T, int E, int K,
                                    int n_group, int topk_group, int renorm, int sigmoid, float scaling) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= T) return;
  const __nv_bfloat16* row = logits + static_cast<size_t>(warp) * ld;
  // expert e = lane * VPT + i
  float sc[VPT], sel[VPT];
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int e = lane * VPT + i;
    sc[i] = e < E ? __bfloat162float(row[e]) : -INFINITY;
    mx = fmaxf(mx, sc[i]);
  }
  if (sigmoid) {
#pragma unroll
    for (int i = 0; i < VPT; ++i) sc[i] = (lane * VPT + i < E) ? 1.f / (1.f + __expf(-sc[i])) : 0.f;
  } else {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) { sc[i] = (lane * VPT + i < E) ? __expf(sc[i] - mx) : 0.f; sum += sc[i]; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
#pragma unroll
    for (int i = 0; i < VPT; ++i) sc[i] /= sum;
  }
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int e = lane * VPT + i;
    sel[i] = e < E ? sc[i] + (bias != nullptr ? bias[e] : 0.f) : -INFINITY;
  }
  // group score: sum of the top-2 keys (bias-corrected) or the max key. A group need not fall on whole lanes
  // (E = 160, 8 groups: 20 experts per group, 8 per lane), so for every group each lane takes the top-2 of its own
  // experts of that group and a full-warp butterfly merges them; lane g keeps the score of group g.
  const int epg = E / n_group;            // experts per group
  int grp[VPT];                           // group of each of my experts (-1: padding)
#pragma unroll
  for (int i = 0; i < VPT; ++i) grp[i] = lane * VPT + i < E ? (lane * VPT + i) / epg : -1;
  float my_gscore = -INFINITY;
  for (int g = 0; g < n_group; ++g) {
    float t1 = -INFINITY, t2 = -INFINITY;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      if (grp[i] == g) {
        if (sel[i] > t1) { t2 = t1; t1 = sel[i]; } else if (sel[i] > t2) { t2 = sel[i]; }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float o1 = __shfl_xor_sync(0xffffffffu, t1, o), o2 = __shfl_xor_sync(0xffffffffu, t2, o);
      if (o1 > t1) { t2 = fmaxf(t1, o2); t1 = o1; } else { t2 = fmaxf(t2, o1); }
    }
    if (lane == g) my_gscore = (bias != nullptr) ? t1 + t2 : t1;
  }
  // lane g < n_group: rank of group g = number of groups with a strictly better score (ties: lower index wins)
  int better = 0;
  for (int g = 0; g < n_group; ++g) {
    const float gs = __shfl_sync(0xffffffffu, my_gscore, g);
    if (gs > my_gscore || (gs == my_gscore && g < lane)) ++better;
  }
  const unsigned group_on = __ballot_sync(0xffffffffu, lane < n_group && better < topk_group);
  // the group mask applies per expert
#pragma unroll
  for (int i = 0; i < VPT; ++i) if (grp[i] < 0 || !((group_on >> grp[i]) & 1u)) sel[i] = -INFINITY;
  float wsum = 0.f, my_w = 0.f;
  int my_id = 0;
  for (int k = 0; k < K; ++k) {
    float best = -INFINITY, bw = 0.f;
    int bi = 0x7fffffff;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      if (sel[i] > best) { best = sel[i]; bi = lane * VPT + i; bw = sc[i]; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const float ow = __shfl_xor_sync(0xffffffffu, bw, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; bw = ow; }
    }
    if (bi / VPT == lane) sel[bi % VPT] = -INFINITY;
    if (lane == k) { my_w = bw; my_id = bi; }
    wsum += bw;
  }
  if (lane < K) {
    const float w = renorm ? my_w / (wsum + 1e-20f) : my_w;
    w_out[static_cast<size_t>(warp) * K + lane] = w * scaling;
    id_out[static_cast<size_t>(warp) * K + lane] = my_id;
  }
}

// ---------------------------------------------------------------------------------------------
// align: slots -> expert-sorted, 128-row padded tiles
// meta layout (int32): [0] num_tiles, [1] num_rows_padded, [2..2+E) counts, [2+E .. 2+2E) cursors,
//                      [2+2E .. 2+3E+1) padded offsets
// ---------------------------------------------------------------------------------------------
// n_valid (optional device scalar): only the first *n_valid slots are live (EP receive pool, comm/ep_a2a.cu)
__global__ void moe_count_kernel(const int32_t* __restrict__ ids, const int32_t* __restrict__ expert_map, int n_slots,
                                 int E_local, int32_t* __restrict__ meta, const int32_t* __restrict__ n_valid) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_slots || (n_valid != nullptr && i >= *n_valid)) return;
  int e = ids[i];
  if (expert_map != nullptr) e = expert_map[e];
  if (e >= 0 && e < E_local) atomicAdd(&meta[2 + e], 1);
}

__global__ void moe_offsets_kernel(int32_t* __restrict__ meta, int32_t* __restrict__ tile_expert, int E_local,
                                   int max_tiles) {
  // single thread block; E_local <= 1024
  __shared__ int s_off[1025];
  if (threadIdx.x == 0) {
    int off = 0;
    for (int e = 0; e < E_local; ++e) {
      s_off[e] = off;
      off += (meta[2 + e] + kTileM - 1) / kTileM * kTileM;
    }
    s_off[E_local] = off;
    meta[0] = off / kTileM;
    meta[1] = off;
  }
  __syncthreads();
  for (int e = threadIdx.x; e <= E_local; e += blockDim.x) meta[2 + 2 * E_local + e] = s_off[e];
  for (int e = threadIdx.x; e < E_local; e += blockDim.x) {
    meta[2 + E_local + e] = 0;  // cursors
    for (int t = s_off[e] / kTileM; t < s_off[e + 1] / kTileM; ++t) tile_expert[t] = e;
  }
  const int nt = s_off[E_local] / kTileM;
  for (int t = nt + threadIdx.x; t < max_tiles; t += blockDim.x) tile_expert[t] = -1;
}

// one warp per slot: claim a row in the expert's segment, copy the token row there
__global__ void moe_scatter_gather_kernel(const int32_t* __restrict__ ids, const int32_t* __restrict__ expert_map,
                                          int n_slots, int top_k, int E_local, int32_t* __restrict__ meta,
                                          int32_t* __restrict__ slot_pos, const __nv_bfloat16* __restrict__ x,
                                          int64_t ldx, __nv_bfloat16* __restrict__ xs, int H,
                                          const int32_t* __restrict__ n_valid) {
  const int slot = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (slot >= n_slots) return;
  int e = (n_valid != nullptr && slot >= *n_valid) ? -1 : ids[slot];
  if (expert_map != nullptr && e >= 0) e = expert_map[e];
  int pos = -1;
  if (e >= 0 && e < E_local) {
    if (lane == 0) pos = meta[2 + 2 * E_local + e] + atomicAdd(&meta[2 + E_local + e], 1);
    pos = __shfl_sync(0xffffffffu, pos, 0);
    const __nv_bfloat16* src = x + static_cast<size_t>(slot / top_k) * ldx;
    __nv_bfloat16* dst = xs + static_cast<size_t>(pos) * H;
    for (int i = lane * 8; i < H; i += 256) *reinterpret_cast<uint4*>(dst + i) = *reinterpret_cast<const uint4*>(src + i);
  }
  if (lane == 0) slot_pos[slot] = pos;
}

__global__ void moe_combine_kernel(const __nv_bfloat16* __restrict__ y, const int32_t* __restrict__ slot_pos,
                                   const float* __restrict__ w, __nv_bfloat16* __restrict__ out, int top_k, int H) {
  const int t = blockIdx.x;
  for (int i = threadIdx.x * 8; i < H; i += blockDim.x * 8) {
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int j = 0; j < top_k; ++j) {
      const int pos = slot_pos[t * top_k + j];
      if (pos < 0) continue;  // expert lives on another rank
      const float wt = w[t * top_k + j];
      const uint4 v = *reinterpret_cast<const uint4*>(y + static_cast<size_t>(pos) * H + i);
      const float2 a = unpack_bf16(v.x), b = unpack_bf16(v.y), c = unpack_bf16(v.z), d = unpack_bf16(v.w);
      acc[0] += wt * a.x; acc[1] += wt * a.y; acc[2] += wt * b.x; acc[3] += wt * b.y;
      acc[4] += wt * c.x; acc[5] += wt * c.y; acc[6] += wt * d.x; acc[7] += wt * d.y;
    }
    uint4 o;
    o.x = pack_bf16(acc[0], acc[1]); o.y = pack_bf16(acc[2], acc[3]);
    o.z = pack_bf16(acc[4], acc[5]); o.w = pack_bf16(acc[6], acc[7]);
    *reinterpret_cast<uint4*>(out + static_cast<size_t>(t) * H + i) = o;
  }
}

}  // namespace b200

using namespace b200;

GLLM_EXPORT int gllm_moe_topk_softmax(const void* logits, int64_t ld, void* w_out, void* id_out, int T, int E, int K,
                                      int renorm, void* stream) {
  if (T <= 0) return 0;
  // K > E would return padding ids >= E (they index expert_map next)
  if (E < 1 || E > 512 || K < 1 || K > 32 || K > E) {
    fprintf(stderr, "[gllm_b200] topk_softmax: unsupported E=%d K=%d (1 <= K <= min(E, 32), E <= 512)\n", E, K);
    return 1;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int blocks = (T * 32 + 255) / 256;
  auto L = reinterpret_cast<const __nv_bfloat16*>(logits);
  auto W = reinterpret_cast<float*>(w_out);
  auto I = reinterpret_cast<int32_t*>(id_out);
  const int vpt = (E + 31) / 32;
  if (vpt <= 1) topk_softmax_kernel<1><<<blocks, 256, 0, st>>>(L, ld, W, I, T, E, K, renorm);
  else if (vpt <= 2) topk_softmax_kernel<2><<<blocks, 256, 0, st>>>(L, ld, W, I, T, E, K, renorm);
  else if (vpt <= 4) topk_softmax_kernel<4><<<blocks, 256, 0, st>>>(L, ld, W, I, T, E, K, renorm);
  else if (vpt <= 8) topk_softmax_kernel<8><<<blocks, 256, 0, st>>>(L, ld, W, I, T, E, K, renorm);
  else topk_softmax_kernel<16><<<blocks, 256, 0, st>>>(L, ld, W, I, T, E, K, renorm);
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

GLLM_EXPORT int gllm_moe_grouped_topk(const void* logits, int64_t ld, const void* bias, void* w_out, void* id_out,
                                      int T, int E, int K, int n_group, int topk_group, int renorm, int sigmoid,
                                      float scaling, void* stream) {
  if (T <= 0) return 0;
  const int vpt = (E + 31) / 32;
  // one warp per token: E <= 512; group scores live one per lane: n_group <= 32; the K winners must come from the
  // experts of the topk_group best groups, else the kernel would return padding ids >= E
  if (E < 1 || E > 512 || K < 1 || K > 32 || K > E || n_group < 1 || n_group > 32 || E % n_group != 0 ||
      topk_group < 1 || K > min(topk_group, n_group) * (E / n_group)) {
    fprintf(stderr, "[gllm_b200] grouped_topk: unsupported E=%d K=%d groups=%d topk_group=%d\n", E, K, n_group,
            topk_group);
    return 1;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int blocks = (T * 32 + 255) / 256;
  auto L = reinterpret_cast<const __nv_bfloat16*>(logits);
  auto B = reinterpret_cast<const float*>(bias);
  auto W = reinterpret_cast<float*>(w_out);
  auto I = reinterpret_cast<int32_t*>(id_out);
#define GT(V) grouped_topk_kernel<V><<<blocks, 256, 0, st>>>(L, ld, B, W, I, T, E, K, n_group, topk_group, renorm, sigmoid, scaling)
  if (vpt <= 1) GT(1);
  else if (vpt <= 2) GT(2);
  else if (vpt <= 4) GT(4);
  else if (vpt <= 8) GT(8);
  else GT(16);
#undef GT
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

// meta: int32[2 + 3*E_local + 1] scratch (zeroed here); tile_expert: int32[max_tiles]; slot_pos: int32[n_slots];
// xs: bf16 [max_tiles*128, H] (caller zero-fills padding rows once; stale finite rows are harmless).
GLLM_EXPORT int gllm_moe_align_gather(const void* ids, const void* expert_map, int T, int top_k, int E_local,
                                      void* meta, void* tile_expert, int max_tiles, void* slot_pos, const void* x,
                                      int64_t ldx, void* xs, int H, const void* n_valid, void* stream) {
  const int n_slots = T * top_k;
  if (n_slots <= 0) return 0;
  // moe_offsets_kernel keeps the offsets in a fixed shared array; the gather copies rows in 16-byte pieces
  if (E_local < 1 || E_local > 1024 || H % 8 != 0 || ldx % 8 != 0 || reinterpret_cast<uintptr_t>(x) % 16 != 0 ||
      reinterpret_cast<uintptr_t>(xs) % 16 != 0) {
    fprintf(stderr, "[gllm_b200] moe_align_gather: unsupported E_local=%d H=%d ldx=%lld or misaligned x / xs\n",
            E_local, H, static_cast<long long>(ldx));
    return 1;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CUDA_CHECK_RET(cudaMemsetAsync(meta, 0, sizeof(int32_t) * (2 + 3 * E_local + 1), st));
  moe_count_kernel<<<(n_slots + 255) / 256, 256, 0, st>>>(reinterpret_cast<const int32_t*>(ids),
                                                           reinterpret_cast<const int32_t*>(expert_map), n_slots,
                                                           E_local, reinterpret_cast<int32_t*>(meta),
                                                           reinterpret_cast<const int32_t*>(n_valid));
  moe_offsets_kernel<<<1, 256, 0, st>>>(reinterpret_cast<int32_t*>(meta), reinterpret_cast<int32_t*>(tile_expert),
                                        E_local, max_tiles);
  moe_scatter_gather_kernel<<<(n_slots * 32 + 255) / 256, 256, 0, st>>>(
      reinterpret_cast<const int32_t*>(ids), reinterpret_cast<const int32_t*>(expert_map), n_slots, top_k, E_local,
      reinterpret_cast<int32_t*>(meta), reinterpret_cast<int32_t*>(slot_pos),
      reinterpret_cast<const __nv_bfloat16*>(x), ldx, reinterpret_cast<__nv_bfloat16*>(xs), H,
      reinterpret_cast<const int32_t*>(n_valid));
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

GLLM_EXPORT int gllm_moe_combine(const void* y, const void* slot_pos, const void* w, void* out, int T, int top_k,
                                 int H, void* stream) {
  if (T <= 0) return 0;
  moe_combine_kernel<<<T, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(y), reinterpret_cast<const int32_t*>(slot_pos),
      reinterpret_cast<const float*>(w), reinterpret_cast<__nv_bfloat16*>(out), top_k, H);
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}
