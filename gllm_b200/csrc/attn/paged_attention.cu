// Paged flash attention for sm_90a (prefill with chunked-prefill/prefix offsets, and
// split-KV decode), replacing the reference's `flash_attn_varlen_func` call on the paged cache
// (gllm/layers/attention.py:49-61; FA2 sm_80 binary, SURVEY §2.3 K1).
//
// Data movement is Hopper-native: every KV page is fetched by one TMA tensor copy
// (cp.async.bulk.tensor.3d, 128-byte swizzle) into an mbarrier-synchronised multi-stage ring
// filled by a dedicated producer warp; math warps consume the swizzled tiles with ldmatrix and
// run the online-softmax recurrence on tensor cores (m16n8k16, fp32 accumulate).
//
//  * decode  : grid (Hkv, seqs, splits). The G = Hq/Hkv query heads that share a KV head are
//              packed into the 16 MMA rows so each KV byte is read once per group; the four
//              math warps split every 64-token tile (flash-decoding inside the CTA) and merge
//              their (m, l, O) at the end. The KV range of each split is derived from the
//              device-side seq_lens, so CUDA-graph replays adapt to the real context length.
//  * prefill : grid (q tiles, seqs, Hkv * G/GP). 64 rows = (64/GP tokens) x (GP heads); the four
//              math warps split the rows; causal mask uses ctx_len = seq_len - q_len.
//
// KV cache layout: [num_pages, Hkv, D/64, page_size, 64] (see rope_kv.cu).
#include "attn_common.cuh"

namespace b200 {

struct AttnParams {
  const __nv_bfloat16* q;  // [tokens, Hq, D] with token stride q_ts (elements)
  int64_t q_ts;
  __nv_bfloat16* out;      // [tokens, Hq, D] contiguous
  float* part_o;           // decode split workspace [seqs, Hq, splits, D] (fp32)
  float* part_lse;         // [seqs, Hq, splits]
  const int32_t* block_table;  // [seqs, max_blocks]
  const int32_t* seq_lens;     // [seqs] KV length including the new tokens
  const int32_t* q_start;      // [seqs + 1] cumulative query offsets (prefill); null => token == seq (decode)
  int max_blocks, Hq, Hkv, G, GP, page_size, num_splits;
  int seq_offset;  // first sequence index handled by this launch
  float scale_log2;
  // decode with num_splits > 1: arrival counter per (sequence, head group); the LAST split CTA to finish merges
  // the partial results itself (no separate merge launch). Zero at rest, re-armed by the merging CTA.
  uint32_t* split_cnt;
};

template <int D>
struct AttnSmem {
  static constexpr int kTileBytes = kTileN * D * 2;        // one K (or V) tile
  static constexpr int kStageBytes = 2 * kTileBytes;       // K + V
  static constexpr int kStages = (D <= 64) ? 4 : (D <= 128 ? 3 : 2);
  static constexpr int kBytes = kStages * kStageBytes + 1024 + 128;
};

// ---------------------------------------------------------------------------------------------
// producer: stream the KV tiles [tile_begin, tile_end) of one sequence / kv head
// ---------------------------------------------------------------------------------------------
template <int D>
__device__ __forceinline__ void kv_producer(const CUtensorMap* tk, const CUtensorMap* tv, uint8_t* smem,
                                            uint64_t* full_bar, uint64_t* empty_bar, const int32_t* bt, int kvh,
                                            int Hkv, int page_size, int seq_len, int tile_begin, int tile_end) {
  using SM = AttnSmem<D>;
  const int pages_per_tile = kTileN / page_size;
  const int page_bytes = page_size * D * 2;
  const int last_page = (seq_len - 1) / page_size;
  uint32_t it = 0;
  for (int tile = tile_begin; tile < tile_end; ++tile, ++it) {
    const int s = it % SM::kStages;
    const uint32_t ph = (it / SM::kStages) & 1;
    mbar_wait(&empty_bar[s], ph ^ 1);
    uint8_t* sk = smem + s * SM::kStageBytes;
    uint8_t* sv = sk + SM::kTileBytes;
    mbar_expect_tx(&full_bar[s], SM::kStageBytes);
    for (int j = 0; j < pages_per_tile; ++j) {
      int pi = tile * pages_per_tile + j;
      if (pi > last_page) pi = last_page;  // keep smem finite for masked columns
      const int page = bt[pi];
      const int slab = (page * Hkv + kvh) * (D / 64);
      tma_load_3d(sk + j * page_bytes, tk, &full_bar[s], 0, 0, slab);
      tma_load_3d(sv + j * page_bytes, tv, &full_bar[s], 0, 0, slab);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// decode kernel
// ---------------------------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(kAttnThreads)
attn_decode_kernel(const __grid_constant__ CUtensorMap tmap_k, const __grid_constant__ CUtensorMap tmap_v,
                   const AttnParams p) {
  using SM = AttnSmem<D>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + SM::kStages * SM::kStageBytes);
  uint64_t* empty_bar = full_bar + SM::kStages;

  griddep_launch();
  griddep_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int groups_per_kv = p.G / p.GP;
  const int kvh = blockIdx.x / groups_per_kv;
  const int hbase = kvh * p.G + (blockIdx.x % groups_per_kv) * p.GP;
  const int seq = blockIdx.y + p.seq_offset;
  const int split = blockIdx.z;
  const int seq_len = p.seq_lens[seq];
  const int n_tiles = (seq_len + kTileN - 1) / kTileN;
  const int tps = (n_tiles + p.num_splits - 1) / p.num_splits;
  const int tile_begin = min(split * tps, n_tiles);
  const int tile_end = min(tile_begin + tps, n_tiles);
  const int page_bytes = p.page_size * D * 2;

  if (threadIdx.x == 0) {
    for (int i = 0; i < SM::kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kMathWarps);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kMathWarps) {
    if (lane == 0 && tile_end > tile_begin) {
      kv_producer<D>(&tmap_k, &tmap_v, smem, full_bar, empty_bar, p.block_table + (size_t)seq * p.max_blocks, kvh,
                     p.Hkv, p.page_size, seq_len, tile_begin, tile_end);
    }
    return;
  }

  // ---------------- math warps ----------------
  const int g = lane >> 2, t = lane & 3;
  // Q fragments: rows = heads hbase + r (r < GP), token = seq (one query token per sequence)
  uint32_t qf[D / 16][4];
  {
    const __nv_bfloat16* qb = p.q + (size_t)seq * p.q_ts;
#pragma unroll
    for (int ks = 0; ks < D / 16; ++ks) {
      const int c = ks * 16 + 2 * t;
      qf[ks][0] = (g < p.GP) ? *reinterpret_cast<const uint32_t*>(qb + (size_t)(hbase + g) * D + c) : 0u;
      qf[ks][1] = (g + 8 < p.GP) ? *reinterpret_cast<const uint32_t*>(qb + (size_t)(hbase + g + 8) * D + c) : 0u;
      qf[ks][2] = (g < p.GP) ? *reinterpret_cast<const uint32_t*>(qb + (size_t)(hbase + g) * D + c + 8) : 0u;
      qf[ks][3] = (g + 8 < p.GP) ? *reinterpret_cast<const uint32_t*>(qb + (size_t)(hbase + g + 8) * D + c + 8) : 0u;
    }
  }
  float o[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_run[2] = {0.f, 0.f};

  uint32_t it = 0;
  for (int tile = tile_begin; tile < tile_end; ++tile, ++it) {
    const int s = it % SM::kStages;
    const uint32_t ph = (it / SM::kStages) & 1;
    mbar_wait(&full_bar[s], ph);
    const uint32_t sk = smem_u32(smem + s * SM::kStageBytes);
    const uint32_t sv = sk + SM::kTileBytes;
    const int tok0 = warp * 16;  // this warp's 16 tokens inside the tile

    // S = Q K^T  (16 rows x 16 tokens)
    float sc[2][4];
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < D / 16; ks += 2) {
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
        uint32_t b0, b1, b2, b3;
        const int tok = tok0 + nt * 8 + (lane & 7);
        const int c8 = ks * 2 + (lane >> 3);
        ldsm_x4(sk + tile_off(tok, c8, p.page_size, page_bytes), b0, b1, b2, b3);
        mma_bf16_16816(sc[nt], qf[ks], b0, b1);
        mma_bf16_16816(sc[nt], qf[ks + 1], b2, b3);
      }
    }
    // mask + online softmax (rows g and g+8)
    const int abs0 = tile * kTileN + tok0 + 2 * t;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int col = abs0 + nt * 8 + (e & 1);
        float v = sc[nt][e] * p.scale_log2;
        if (col >= seq_len) v = -INFINITY;
        sc[nt][e] = v;
        mx[e >> 1] = fmaxf(mx[e >> 1], v);
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    }
    float alpha[2], m_use[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float m_new = fmaxf(m_run[r], mx[r]);
      m_use[r] = (m_new == -INFINITY) ? 0.f : m_new;
      alpha[r] = exp2f(m_run[r] - m_use[r]);
      m_run[r] = m_new;
      l_run[r] *= alpha[r];
    }
    uint32_t pa[4];
    {
      float pv[2][4];
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          pv[nt][e] = exp2f(sc[nt][e] - m_use[e >> 1]);
          l_run[e >> 1] += pv[nt][e];
        }
      pa[0] = pack_bf16(pv[0][0], pv[0][1]);
      pa[1] = pack_bf16(pv[0][2], pv[0][3]);
      pa[2] = pack_bf16(pv[1][0], pv[1][1]);
      pa[3] = pack_bf16(pv[1][2], pv[1][3]);
    }
#pragma unroll
    for (int nd = 0; nd < D / 8; ++nd) {
      o[nd][0] *= alpha[0]; o[nd][1] *= alpha[0];
      o[nd][2] *= alpha[1]; o[nd][3] *= alpha[1];
    }
    // O += P V   (k = this warp's 16 tokens)
#pragma unroll
    for (int nd = 0; nd < D / 8; nd += 2) {
      uint32_t b0, b1, b2, b3;
      const int tok = tok0 + ((lane >> 3) & 1) * 8 + (lane & 7);
      const int c8 = nd + (lane >> 4);
      ldsm_x4_t(sv + tile_off(tok, c8, p.page_size, page_bytes), b0, b1, b2, b3);
      mma_bf16_16816(o[nd], pa, b0, b1);
      mma_bf16_16816(o[nd + 1], pa, b2, b3);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[s]);
  }

  // ---------------- merge the four warps ----------------
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
  asm volatile("bar.sync 1, 128;" ::: "memory");  // every warp is done with the KV ring
  float* red_o = reinterpret_cast<float*>(smem);                 // [4][16][D]
  float* red_m = red_o + kMathWarps * 16 * D;                    // [4][16]
  float* red_l = red_m + kMathWarps * 16;                        // [4][16]
#pragma unroll
  for (int nd = 0; nd < D / 8; ++nd) {
    const int c = nd * 8 + 2 * t;
    *reinterpret_cast<float2*>(red_o + (warp * 16 + g) * D + c) = make_float2(o[nd][0], o[nd][1]);
    *reinterpret_cast<float2*>(red_o + (warp * 16 + g + 8) * D + c) = make_float2(o[nd][2], o[nd][3]);
  }
  if (t == 0) {
    red_m[warp * 16 + g] = m_run[0]; red_m[warp * 16 + g + 8] = m_run[1];
    red_l[warp * 16 + g] = l_run[0]; red_l[warp * 16 + g + 8] = l_run[1];
  }
  asm volatile("bar.sync 1, 128;" ::: "memory");
  // 128 threads: thread -> (row = tid / 8, 16 columns chunk loop)
  const int tid = threadIdx.x;
  const int row = tid >> 3;  // 0..15
  if (row < p.GP) {
    float mw[kMathWarps], m_all = -INFINITY;
#pragma unroll
    for (int w = 0; w < kMathWarps; ++w) { mw[w] = red_m[w * 16 + row]; m_all = fmaxf(m_all, mw[w]); }
    float wgt[kMathWarps], l_all = 0.f;
#pragma unroll
    for (int w = 0; w < kMathWarps; ++w) {
      wgt[w] = (mw[w] == -INFINITY) ? 0.f : exp2f(mw[w] - m_all);
      l_all += wgt[w] * red_l[w * 16 + row];
    }
    const float inv = l_all > 0.f ? 1.f / l_all : 0.f;
    const int head = hbase + row;
    for (int c = (tid & 7) * 4; c < D; c += 32) {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int w = 0; w < kMathWarps; ++w) {
        const float4 v = *reinterpret_cast<const float4*>(red_o + (w * 16 + row) * D + c);
        acc.x += wgt[w] * v.x; acc.y += wgt[w] * v.y; acc.z += wgt[w] * v.z; acc.w += wgt[w] * v.w;
      }
      acc.x *= inv; acc.y *= inv; acc.z *= inv; acc.w *= inv;
      if (p.num_splits == 1) {
        uint2 ov = make_uint2(pack_bf16(acc.x, acc.y), pack_bf16(acc.z, acc.w));
        *reinterpret_cast<uint2*>(p.out + ((size_t)seq * p.Hq + head) * D + c) = ov;
      } else {
        *reinterpret_cast<float4*>(p.part_o + (((size_t)seq * p.Hq + head) * p.num_splits + split) * D + c) = acc;
      }
    }
    if (p.num_splits > 1 && (tid & 7) == 0) {
      // log2-domain LSE of this split
      p.part_lse[((size_t)seq * p.Hq + head) * p.num_splits + split] =
          (l_all > 0.f) ? (m_all + log2f(l_all)) : -INFINITY;
    }
  }
  if (p.num_splits > 1 && p.split_cnt != nullptr) {
    // ---------------- last-arriver merge of the KV splits ----------------
    __shared__ uint32_t s_last;
    __threadfence();
    asm volatile("bar.sync 1, 128;" ::: "memory");
    if (tid == 0) {
      uint32_t* cnt = p.split_cnt + (size_t)seq * gridDim.x + blockIdx.x;
      const uint32_t old = atomicAdd(cnt, 1u);
      s_last = (old == (uint32_t)p.num_splits - 1u) ? 1u : 0u;
      if (s_last) *cnt = 0u;
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    if (s_last && row < p.GP) {
      __threadfence();
      const int head = hbase + row;
      const size_t sh = (size_t)seq * p.Hq + head;
      float m = -INFINITY;
      for (int sp = 0; sp < p.num_splits; ++sp) m = fmaxf(m, __ldcg(p.part_lse + sh * p.num_splits + sp));
      float den = 0.f;
      for (int sp = 0; sp < p.num_splits; ++sp) {
        const float l = __ldcg(p.part_lse + sh * p.num_splits + sp);
        den += (l == -INFINITY) ? 0.f : exp2f(l - m);
      }
      const float inv = den > 0.f ? 1.f / den : 0.f;
      for (int c = (tid & 7) * 4; c < D; c += 32) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int sp = 0; sp < p.num_splits; ++sp) {
          const float l = __ldcg(p.part_lse + sh * p.num_splits + sp);
          const float w = (l == -INFINITY) ? 0.f : exp2f(l - m) * inv;
          const float4 v = __ldcg(reinterpret_cast<const float4*>(p.part_o + (sh * p.num_splits + sp) * D + c));
          acc.x += w * v.x; acc.y += w * v.y; acc.z += w * v.z; acc.w += w * v.w;
        }
        *reinterpret_cast<uint2*>(p.out + sh * D + c) = make_uint2(pack_bf16(acc.x, acc.y), pack_bf16(acc.z, acc.w));
      }
    }
  }
}

// out[seq, head, :] = sum_s softmax_s(lse) * part_o[seq, head, s, :]
__global__ void attn_merge_kernel(const float* __restrict__ part_o, const float* __restrict__ part_lse,
                                  __nv_bfloat16* __restrict__ out, int num_splits, int D) {
  griddep_launch();
  griddep_wait();
  const size_t sh = blockIdx.x;  // seq * Hq + head
  float m = -INFINITY;
  for (int s = 0; s < num_splits; ++s) m = fmaxf(m, part_lse[sh * num_splits + s]);
  float den = 0.f;
  for (int s = 0; s < num_splits; ++s) {
    const float l = part_lse[sh * num_splits + s];
    den += (l == -INFINITY) ? 0.f : exp2f(l - m);
  }
  const float inv = den > 0.f ? 1.f / den : 0.f;
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    float acc = 0.f;
    for (int s = 0; s < num_splits; ++s) {
      const float l = part_lse[sh * num_splits + s];
      const float w = (l == -INFINITY) ? 0.f : exp2f(l - m);
      acc += w * part_o[(sh * num_splits + s) * D + c];
    }
    out[sh * D + c] = __float2bfloat16(acc * inv);
  }
}

// ---------------------------------------------------------------------------------------------
// prefill kernel: 64 rows = (64 / GP) tokens x GP heads, warps split rows
// ---------------------------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(kAttnThreads)
attn_prefill_kernel(const __grid_constant__ CUtensorMap tmap_k, const __grid_constant__ CUtensorMap tmap_v,
                    const AttnParams p) {
  using SM = AttnSmem<D>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + SM::kStages * SM::kStageBytes);
  uint64_t* empty_bar = full_bar + SM::kStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int seq = blockIdx.y + p.seq_offset;
  const int groups_per_kv = p.G / p.GP;
  const int kvh = blockIdx.z / groups_per_kv;
  const int hbase = kvh * p.G + (blockIdx.z % groups_per_kv) * p.GP;
  const int q_begin = p.q_start[seq], q_len = p.q_start[seq + 1] - q_begin;
  const int toks_per_tile = 64 / p.GP;
  // process the heaviest (last) query tiles first
  const int n_qtiles = (q_len + toks_per_tile - 1) / toks_per_tile;
  if ((int)blockIdx.x >= n_qtiles) return;
  const int qt = n_qtiles - 1 - blockIdx.x;
  const int tok_base = qt * toks_per_tile;
  const int seq_len = p.seq_lens[seq];
  const int ctx_len = seq_len - q_len;
  const int last_tok = min(tok_base + toks_per_tile, q_len) - 1;
  const int kv_end = ctx_len + last_tok + 1;  // causal horizon of this tile
  const int n_tiles = (kv_end + kTileN - 1) / kTileN;
  const int page_bytes = p.page_size * D * 2;

  if (threadIdx.x == 0) {
    for (int i = 0; i < SM::kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kMathWarps);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kMathWarps) {
    if (lane == 0) {
      kv_producer<D>(&tmap_k, &tmap_v, smem, full_bar, empty_bar, p.block_table + (size_t)seq * p.max_blocks, kvh,
                     p.Hkv, p.page_size, seq_len, 0, n_tiles);
    }
    return;
  }

  const int g = lane >> 2, t = lane & 3;
  // this thread's two rows
  int r_tok[2], r_head[2];
  bool r_ok[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = warp * 16 + g + r * 8;
    r_tok[r] = tok_base + row / p.GP;
    r_head[r] = hbase + row % p.GP;
    r_ok[r] = r_tok[r] < q_len;
  }
  uint32_t qf[D / 16][4];
#pragma unroll
  for (int ks = 0; ks < D / 16; ++ks) {
    const int c = ks * 16 + 2 * t;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const __nv_bfloat16* qp = p.q + (size_t)(q_begin + r_tok[r]) * p.q_ts + (size_t)r_head[r] * D + c;
      qf[ks][r] = r_ok[r] ? *reinterpret_cast<const uint32_t*>(qp) : 0u;
      qf[ks][r + 2] = r_ok[r] ? *reinterpret_cast<const uint32_t*>(qp + 8) : 0u;
    }
  }
  float o[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_run[2] = {0.f, 0.f};
  const int lim[2] = {ctx_len + r_tok[0], ctx_len + r_tok[1]};  // last visible key per row

  for (int tile = 0; tile < n_tiles; ++tile) {
    const int s = tile % SM::kStages;
    const uint32_t ph = (tile / SM::kStages) & 1;
    mbar_wait(&full_bar[s], ph);
    const uint32_t sk = smem_u32(smem + s * SM::kStageBytes);
    const uint32_t sv = sk + SM::kTileBytes;

    float sc[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < D / 16; ks += 2) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        uint32_t b0, b1, b2, b3;
        const int tok = nt * 8 + (lane & 7);
        const int c8 = ks * 2 + (lane >> 3);
        ldsm_x4(sk + tile_off(tok, c8, p.page_size, page_bytes), b0, b1, b2, b3);
        mma_bf16_16816(sc[nt], qf[ks], b0, b1);
        mma_bf16_16816(sc[nt], qf[ks + 1], b2, b3);
      }
    }
    const int abs0 = tile * kTileN + 2 * t;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int col = abs0 + nt * 8 + (e & 1);
        float v = sc[nt][e] * p.scale_log2;
        if (col > lim[e >> 1]) v = -INFINITY;
        sc[nt][e] = v;
        mx[e >> 1] = fmaxf(mx[e >> 1], v);
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    }
    float alpha[2], m_use[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float m_new = fmaxf(m_run[r], mx[r]);
      m_use[r] = (m_new == -INFINITY) ? 0.f : m_new;
      alpha[r] = exp2f(m_run[r] - m_use[r]);
      m_run[r] = m_new;
      l_run[r] *= alpha[r];
    }
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        sc[nt][e] = exp2f(sc[nt][e] - m_use[e >> 1]);
        l_run[e >> 1] += sc[nt][e];
      }
#pragma unroll
    for (int nd = 0; nd < D / 8; ++nd) {
      o[nd][0] *= alpha[0]; o[nd][1] *= alpha[0];
      o[nd][2] *= alpha[1]; o[nd][3] *= alpha[1];
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {  // 16-token k-steps
      uint32_t pa[4];
      pa[0] = pack_bf16(sc[2 * kk][0], sc[2 * kk][1]);
      pa[1] = pack_bf16(sc[2 * kk][2], sc[2 * kk][3]);
      pa[2] = pack_bf16(sc[2 * kk + 1][0], sc[2 * kk + 1][1]);
      pa[3] = pack_bf16(sc[2 * kk + 1][2], sc[2 * kk + 1][3]);
#pragma unroll
      for (int nd = 0; nd < D / 8; nd += 2) {
        uint32_t b0, b1, b2, b3;
        const int tok = kk * 16 + ((lane >> 3) & 1) * 8 + (lane & 7);
        const int c8 = nd + (lane >> 4);
        ldsm_x4_t(sv + tile_off(tok, c8, p.page_size, page_bytes), b0, b1, b2, b3);
        mma_bf16_16816(o[nd], pa, b0, b1);
        mma_bf16_16816(o[nd + 1], pa, b2, b3);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[s]);
  }

#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (!r_ok[r]) continue;
    const float inv = l_run[r] > 0.f ? 1.f / l_run[r] : 0.f;
    __nv_bfloat16* op = p.out + ((size_t)(q_begin + r_tok[r]) * p.Hq + r_head[r]) * D + 2 * t;
#pragma unroll
    for (int nd = 0; nd < D / 8; ++nd) {
      *reinterpret_cast<uint32_t*>(op + nd * 8) = pack_bf16(o[nd][2 * r] * inv, o[nd][2 * r + 1] * inv);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
// shared with mla_attention.cu
int launch_attn_merge(const float* part_o, const float* part_lse, __nv_bfloat16* out, int rows, int num_splits, int D,
                      cudaStream_t st) {
  CUDA_CHECK_RET(launch_pdl(attn_merge_kernel, dim3(rows), dim3(D < 128 ? D : 128), 0, st, part_o, part_lse, out,
                            num_splits, D));
  return 0;
}

static int largest_divisor_leq(int G, int cap, int must_divide) {
  for (int d = (G < cap ? G : cap); d >= 1; --d) {
    if (G % d == 0 && (must_divide == 0 || must_divide % d == 0)) return d;
  }
  return 1;
}

template <int D>
static int launch_decode(const CUtensorMap& tk, const CUtensorMap& tv, const AttnParams& p, int num_seqs,
                         cudaStream_t st) {
  using SM = AttnSmem<D>;
  static PerDeviceOnce configured;
  if (configured.need()) {
    CUDA_CHECK_RET(cudaFuncSetAttribute(attn_decode_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM::kBytes));
    configured.done();
  }
  dim3 grid(p.Hkv * (p.G / p.GP), num_seqs, p.num_splits);
  CUDA_CHECK_RET(launch_pdl(attn_decode_kernel<D>, grid, dim3(kAttnThreads), SM::kBytes, st, tk, tv, p));
  return 0;
}

template <int D>
static int launch_prefill(const CUtensorMap& tk, const CUtensorMap& tv, const AttnParams& p, int num_seqs,
                          int max_q_len, cudaStream_t st) {
  using SM = AttnSmem<D>;
  static PerDeviceOnce configured;
  if (configured.need()) {
    CUDA_CHECK_RET(cudaFuncSetAttribute(attn_prefill_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM::kBytes));
    configured.done();
  }
  const int toks_per_tile = 64 / p.GP;
  dim3 grid((max_q_len + toks_per_tile - 1) / toks_per_tile, num_seqs, p.Hkv * (p.G / p.GP));
  attn_prefill_kernel<D><<<grid, kAttnThreads, SM::kBytes, st>>>(tk, tv, p);
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

}  // namespace b200

using namespace b200;

// Decode: one query token per sequence; q row i belongs to sequence seq_offset + i... (q is indexed
// by the absolute sequence index, as are block_table / seq_lens).
GLLM_EXPORT int gllm_attn_decode(const void* q, int64_t q_ts, void* out, const void* k_cache, const void* v_cache,
                                 int64_t num_pages, const void* block_table, const void* seq_lens, void* part_o,
                                 void* part_lse, int num_seqs, int seq_offset, int max_blocks, int Hq, int Hkv,
                                 int D, int page_size, int num_splits, float scale, void* split_cnt, void* stream) {
  if (num_seqs <= 0) return 0;
  if (page_size < 8 || kTileN % page_size != 0 || Hq % Hkv != 0) {
    fprintf(stderr, "[gllm_b200] attn_decode: unsupported page_size=%d / heads\n", page_size);
    return 1;
  }
  CUtensorMap tk, tv;
  if (get_kv_tmap(k_cache, num_pages, Hkv, D, page_size, &tk)) return 1;
  if (get_kv_tmap(v_cache, num_pages, Hkv, D, page_size, &tv)) return 1;
  AttnParams p;
  p.q = reinterpret_cast<const __nv_bfloat16*>(q); p.q_ts = q_ts;
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.part_o = reinterpret_cast<float*>(part_o);
  p.part_lse = reinterpret_cast<float*>(part_lse);
  p.block_table = reinterpret_cast<const int32_t*>(block_table);
  p.seq_lens = reinterpret_cast<const int32_t*>(seq_lens);
  p.q_start = nullptr;
  p.max_blocks = max_blocks; p.Hq = Hq; p.Hkv = Hkv; p.G = Hq / Hkv;
  p.GP = largest_divisor_leq(p.G, 16, 0);
  p.page_size = page_size; p.num_splits = num_splits < 1 ? 1 : num_splits;
  p.seq_offset = seq_offset;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.split_cnt = reinterpret_cast<uint32_t*>(split_cnt);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int rc;
  switch (D) {
    case 64: rc = launch_decode<64>(tk, tv, p, num_seqs, st); break;
    case 128: rc = launch_decode<128>(tk, tv, p, num_seqs, st); break;
    case 256: rc = launch_decode<256>(tk, tv, p, num_seqs, st); break;
    default:
      fprintf(stderr, "[gllm_b200] attn_decode: unsupported head_dim %d\n", D);
      return 1;
  }
  if (rc) return rc;
  if (p.num_splits > 1 && p.split_cnt == nullptr) {
    // merge covers sequences [seq_offset, seq_offset + num_seqs)
    const size_t off = (size_t)seq_offset * Hq;
    CUDA_CHECK_RET(launch_pdl(attn_merge_kernel, dim3(num_seqs * Hq), dim3(D < 128 ? D : 128), 0, st,
                              p.part_o + off * p.num_splits * D, p.part_lse + off * p.num_splits,
                              p.out + off * D, p.num_splits, D));
  }
  return 0;
}

// Prefill / mixed: sequences [seq_offset, seq_offset + num_seqs) with query ranges q_start[seq]..q_start[seq+1]
GLLM_EXPORT int gllm_attn_prefill(const void* q, int64_t q_ts, void* out, const void* k_cache, const void* v_cache,
                                  int64_t num_pages, const void* block_table, const void* seq_lens,
                                  const void* q_start, int num_seqs, int seq_offset, int max_q_len, int max_blocks,
                                  int Hq, int Hkv, int D, int page_size, float scale, void* stream) {
  if (num_seqs <= 0 || max_q_len <= 0) return 0;
  if (page_size < 8 || kTileN % page_size != 0 || Hq % Hkv != 0) {
    fprintf(stderr, "[gllm_b200] attn_prefill: unsupported page_size=%d / heads\n", page_size);
    return 1;
  }
  CUtensorMap tk, tv;
  if (get_kv_tmap(k_cache, num_pages, Hkv, D, page_size, &tk)) return 1;
  if (get_kv_tmap(v_cache, num_pages, Hkv, D, page_size, &tv)) return 1;
  AttnParams p;
  p.q = reinterpret_cast<const __nv_bfloat16*>(q); p.q_ts = q_ts;
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.part_o = nullptr; p.part_lse = nullptr;
  p.block_table = reinterpret_cast<const int32_t*>(block_table);
  p.seq_lens = reinterpret_cast<const int32_t*>(seq_lens);
  p.q_start = reinterpret_cast<const int32_t*>(q_start);
  p.max_blocks = max_blocks; p.Hq = Hq; p.Hkv = Hkv; p.G = Hq / Hkv;
  p.GP = largest_divisor_leq(p.G, 64, 64);
  p.page_size = page_size; p.num_splits = 1; p.seq_offset = seq_offset;
  p.scale_log2 = scale * 1.4426950408889634f;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (D) {
    case 64: return launch_prefill<64>(tk, tv, p, num_seqs, max_q_len, st);
    case 128: return launch_prefill<128>(tk, tv, p, num_seqs, max_q_len, st);
    case 256: return launch_prefill<256>(tk, tv, p, num_seqs, max_q_len, st);
    default:
      fprintf(stderr, "[gllm_b200] attn_prefill: unsupported head_dim %d\n", D);
      return 1;
  }
}
