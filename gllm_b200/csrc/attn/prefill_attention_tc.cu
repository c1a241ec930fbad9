// wgmma paged flash attention for prefill (chunked-prefill and prefix offsets included): the tensor-core
// successor of the mma.sync prefill kernel in paged_attention.cu (same arguments, same paged KV cache;
// reference call site: gllm/layers/attention.py:49-61, flash_attn_varlen_func on the paged cache).
// GLLM_ATTN_TC=0 (ops/sm100.py) selects the mma.sync kernel instead.
//
// One CTA = 128 query rows (128/GP tokens x GP heads that share one KV head, GQA-packed like the mma.sync kernel)
// x the causal prefix of one sequence, walked in tiles of KV keys:
//
//   warpgroup 0 (1 thread)  TMA producer : page boxes [page_size][64] of K and V -> smem tiles [D/64][KV][64] (SW128)
//   warpgroups 1-2          64 query rows each:
//                             S = Q K^T   wgmma, A = Q smem K-major, B = K tile K-major, S in registers
//                             softmax     row max / exp2 / row sum in registers (a row lives in 4 lanes of a quad)
//                             O += P V    wgmma, A = P from registers (the S fragment converted to bf16 in place),
//                                         B = V tile **MN-major**, O in registers
//
// The V operand: the cache stores V as [key][d] (d contiguous), i.e. the contraction dimension (keys) runs along
// ROWS of the tile. That is the MN-major canonical layout of the wgmma shared-memory descriptor
//     SW128, MN-major, in 16-byte units: ((8, n), (8, k)) : ((1, LBO), (8, SBO))
// -> 64 d-values (128 B) contiguous, next 64 d-values LBO bytes away (= one [KV][64] slab), 8 keys are 8
// consecutive 128-byte rows, the next 8 keys SBO = 1024 B away; a K = 16 step advances the start address by 2048 B.
#include "attn_common.cuh"

namespace b200 {

static constexpr int kTcRows = 128;                      // query rows per CTA (2 x wgmma M)
static constexpr int kTcThreads = 384;

struct TcAttnParams {
  const __nv_bfloat16* q;
  int64_t q_ts;
  __nv_bfloat16* out;
  const int32_t* block_table;
  const int32_t* seq_lens;
  const int32_t* q_start;
  int max_blocks, Hq, Hkv, G, GP, page_size, seq_offset;
  float scale_log2;
};

template <int D, int KV>
struct TcSmem {
  static constexpr int kQBytes = kTcRows * D * 2;
  static constexpr int kTileBytes = KV * D * 2;            // one K (or V) tile
  static constexpr int kStageBytes = 2 * kTileBytes;
  // as many KV stages as fit next to Q (227 KB per CTA), at most 4
  static constexpr int kFit = (232448 - 2048 - kQBytes) / kStageBytes;
  static constexpr int kStages = kFit > 4 ? 4 : kFit;
  static constexpr int kBarOff = kQBytes + kStages * kStageBytes;
  static constexpr int kBytes = kBarOff + 256 + 1024;
  static_assert(kStages >= 2, "needs two KV stages");
};

// byte offset of (row, 16-byte chunk c) in a K-major SW128 operand tile stored as [c / 8][128 rows][128 B]
__device__ __forceinline__ uint32_t a_tile_off(int row, int c) {
  return (c >> 3) * (kTcRows * 128) + row * 128 + (((c & 7) ^ (row & 7)) << 4);
}

template <int D, int KV>
__global__ void __launch_bounds__(kTcThreads, 1)
attn_prefill_tc_kernel(const __grid_constant__ CUtensorMap tmap_k, const __grid_constant__ CUtensorMap tmap_v,
                       const TcAttnParams p) {
  using SM = TcSmem<D, KV>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sq = smem;
  uint8_t* skv = smem + SM::kQBytes;                   // KV ring
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + SM::kBarOff);
  uint64_t* kv_full = bars;                            // [kStages]  TMA -> MMA warpgroups
  uint64_t* kv_empty = kv_full + SM::kStages;          // [kStages]  8 consumer warps -> producer

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int seq = blockIdx.y + p.seq_offset;
  const int groups_per_kv = p.G / p.GP;
  const int kvh = blockIdx.z / groups_per_kv;
  const int hbase = kvh * p.G + (blockIdx.z % groups_per_kv) * p.GP;
  const int q_begin = p.q_start[seq], q_len = p.q_start[seq + 1] - q_begin;
  const int toks_per_tile = kTcRows / p.GP;
  const int n_qtiles = (q_len + toks_per_tile - 1) / toks_per_tile;
  if (static_cast<int>(blockIdx.x) >= n_qtiles) return;
  const int qt = n_qtiles - 1 - blockIdx.x;            // heaviest (last) query tiles first
  const int tok_base = qt * toks_per_tile;
  const int seq_len = p.seq_lens[seq];
  const int ctx_len = seq_len - q_len;
  const int last_tok = min(tok_base + toks_per_tile, q_len) - 1;
  const int kv_end = ctx_len + last_tok + 1;           // causal horizon of this tile
  const int n_tiles = (kv_end + KV - 1) / KV;

  if (threadIdx.x == 0) {
    for (int i = 0; i < SM::kStages; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ------------------------------------------------------------------ TMA producer
    regs_dealloc<40>();
    if (warp == 0 && lane == 0) {
      const int32_t* bt = p.block_table + static_cast<size_t>(seq) * p.max_blocks;
      const int pages_per_tile = KV / p.page_size;
      const int page_rows_bytes = p.page_size * 128;
      const int last_page = (seq_len - 1) / p.page_size;
      for (int tile = 0; tile < n_tiles; ++tile) {
        const int s = tile % SM::kStages;
        const uint32_t ph = (tile / SM::kStages) & 1;
        mbar_wait(&kv_empty[s], ph ^ 1);
        uint8_t* sk = skv + s * SM::kStageBytes;
        uint8_t* sv = sk + SM::kTileBytes;
        mbar_expect_tx(&kv_full[s], SM::kStageBytes);
        for (int j = 0; j < pages_per_tile; ++j) {
          int pi = tile * pages_per_tile + j;
          if (pi > last_page) pi = last_page;          // masked columns: keep the data finite
          const int slab0 = (bt[pi] * p.Hkv + kvh) * (D / 64);
#pragma unroll
          for (int sl = 0; sl < D / 64; ++sl) {
            const int off = sl * (KV * 128) + j * page_rows_bytes;
            tma_load_3d(sk + off, &tmap_k, &kv_full[s], 0, 0, slab0 + sl);
            tma_load_3d(sv + off, &tmap_v, &kv_full[s], 0, 0, slab0 + sl);
          }
        }
      }
    }
    return;
  }
  // -------------------------------------------------------------------- MMA + softmax warpgroups
  regs_alloc<232>();
  const int ct = threadIdx.x - 128;                    // 0..255
  const int g = ct >> 7;
  const int wq = (ct >> 5) & 3;
  {  // stage Q as the K-major SW128 A operand: thread ct copies row ct / 2, half (ct & 1) of the head dim
    const int row = ct >> 1;
    const int tok = tok_base + row / p.GP;
    const int head = hbase + row % p.GP;
    const bool ok = tok < q_len;
    const uint4* qp = reinterpret_cast<const uint4*>(p.q + static_cast<size_t>(q_begin + (ok ? tok : 0)) * p.q_ts +
                                                     static_cast<size_t>(head) * D);
#pragma unroll
    for (int c0 = 0; c0 < D / 16; ++c0) {
      const int c = (ct & 1) * (D / 16) + c0;
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (ok) v = ld_nc_v4(qp + c);
      *reinterpret_cast<uint4*>(sq + a_tile_off(row, c)) = v;
    }
    fence_proxy_async_smem();                          // Q visible to the tensor core (async proxy)
    asm volatile("bar.sync 1, 256;" ::: "memory");
  }
  // fragment rows of this thread: r[h] = 64 g + 16 wq + lane / 4 + 8 h; columns 8 j + 2 (lane % 4) + {0, 1}
  int tok[2], head[2], lim[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = 64 * g + 16 * wq + (lane >> 2) + 8 * h;
    tok[h] = tok_base + row / p.GP;
    head[h] = hbase + row % p.GP;
    lim[h] = ctx_len + tok[h];                         // last visible key of this row
  }
  const int cq = 2 * (lane & 3);
  const uint32_t q_addr = smem_u32(sq) + g * (64 * 128);
  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  for (int tile = 0; tile < n_tiles; ++tile) {
    const int s = tile % SM::kStages;
    mbar_wait(&kv_full[s], (tile / SM::kStages) & 1);
    const uint32_t k_addr = smem_u32(skv + s * SM::kStageBytes);
    const uint32_t v_addr = k_addr + SM::kTileBytes;
    float sc[KV / 2];
    wgmma_fence();
#pragma unroll
    for (int kd = 0; kd < D / 64; ++kd) {
      const uint64_t da = make_sw128_kmajor_desc(q_addr + kd * (kTcRows * 128));
      const uint64_t db = make_sw128_kmajor_desc(k_addr + kd * (KV * 128));
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_bf16_ss<KV>(sc, da + kk * 2, db + kk * 2, (kd | kk) != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(sc);

    const int key0 = tile * KV;
    const bool need_mask = key0 + KV - 1 > ctx_len + tok_base;   // CTA-uniform: a diagonal tile
    if (need_mask) {
#pragma unroll
      for (int j = 0; j < KV / 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (key0 + 8 * j + cq + (e & 1) > lim[e >> 1]) sc[4 * j + e] = -INFINITY;
    }
    float alpha[2], m_use[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < KV / 8; ++j) mx = fmaxf(mx, fmaxf(sc[4 * j + 2 * h], sc[4 * j + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[h], mx * p.scale_log2);
      m_use[h] = (m_new == -INFINITY) ? 0.f : m_new;
      alpha[h] = exp2f(m_run[h] - m_use[h]);
      m_run[h] = m_new;
    }
    // P = exp2(S * scale - m) as bf16 A fragments (k16 chunk t: keys 16 t .. 16 t + 15), per-thread row sums
    uint32_t pa[KV / 16][4];
    float sum[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < KV / 8; ++j) {
      float x[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        x[e] = exp2f(fmaf(sc[4 * j + e], p.scale_log2, -m_use[e >> 1]));
        sum[e >> 1] += x[e];
      }
      pa[j >> 1][(j & 1) * 2] = pack_bf16(x[0], x[1]);
      pa[j >> 1][(j & 1) * 2 + 1] = pack_bf16(x[2], x[3]);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) l_run[h] = l_run[h] * alpha[h] + sum[h];
#pragma unroll
    for (int j = 0; j < D / 8; ++j) {
      o[4 * j] *= alpha[0]; o[4 * j + 1] *= alpha[0];
      o[4 * j + 2] *= alpha[1]; o[4 * j + 3] *= alpha[1];
    }
    wgmma_fence();
#pragma unroll
    for (int t = 0; t < KV / 16; ++t) {
      const uint64_t dv = make_sw128_desc(v_addr + t * 2048, (KV * 128) >> 4, 1024 >> 4);
      wgmma_bf16_rs_tb<D>(o, pa[t], dv, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
    if (lane == 0) mbar_arrive(&kv_empty[s]);          // K and V of this stage consumed
  }
  // ---- epilogue: O / l -> bf16 -> global
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = l > 0.f ? 1.f / l : 0.f;
    if (tok[h] >= q_len) continue;
    __nv_bfloat16* op = p.out + (static_cast<size_t>(q_begin + tok[h]) * p.Hq + head[h]) * D;
#pragma unroll
    for (int j = 0; j < D / 8; ++j)
      *reinterpret_cast<uint32_t*>(op + 8 * j + cq) = pack_bf16(o[4 * j + 2 * h] * inv, o[4 * j + 2 * h + 1] * inv);
  }
}

// tensor map over the paged cache with ONE 64-wide slab per box ([page_size][64]), so that a KV tile can be
// assembled slab-major ([D/64][KV][64]) — the layout both wgmma operand forms need
static int get_kv_slab_tmap(const void* base, int64_t num_pages, int Hkv, int D, int page_size, CUtensorMap* out) {
  static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> cache;
  static std::mutex mu;
  TmapKey key{base, num_pages, Hkv, D, page_size};
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find(key);
  if (it != cache.end()) {
    *out = it->second;
    return 0;
  }
  CUtensorMap m;
  cuuint64_t dims[3] = {64, (cuuint64_t)page_size, (cuuint64_t)(num_pages * Hkv * (D / 64))};
  cuuint64_t strides[2] = {128, (cuuint64_t)page_size * 128};
  cuuint32_t box[3] = {64, (cuuint32_t)page_size, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = get_encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box,
                               estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "[gllm_b200] KV slab tensor-map encode failed (%d)\n", (int)r);
    return 1;
  }
  cache.emplace(key, m);
  *out = m;
  return 0;
}

template <int D, int KV>
static int launch_prefill_tc(const CUtensorMap& tk, const CUtensorMap& tv, const TcAttnParams& p, int num_seqs,
                             int max_q_len, cudaStream_t st) {
  using SM = TcSmem<D, KV>;
  static PerDeviceOnce configured;
  if (configured.need()) {
    CUDA_CHECK_RET(cudaFuncSetAttribute(attn_prefill_tc_kernel<D, KV>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        SM::kBytes));
    configured.done();
  }
  const int toks_per_tile = kTcRows / p.GP;
  dim3 grid((max_q_len + toks_per_tile - 1) / toks_per_tile, num_seqs, p.Hkv * (p.G / p.GP));
  attn_prefill_tc_kernel<D, KV><<<grid, kTcThreads, SM::kBytes, st>>>(tk, tv, p);
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

}  // namespace b200

using namespace b200;

// Same contract as gllm_attn_prefill (paged_attention.cu). Returns 2 when the shape is outside this kernel's
// envelope (head_dim 64 / 128, page_size dividing the KV tile) — the caller then uses the mma.sync kernel.
// kv_tile: 64 or 128 keys per pipeline stage.
GLLM_EXPORT int gllm_attn_prefill_tc(const void* q, int64_t q_ts, void* out, const void* k_cache, const void* v_cache,
                                     int64_t num_pages, const void* block_table, const void* seq_lens,
                                     const void* q_start, int num_seqs, int seq_offset, int max_q_len,
                                     int max_blocks, int Hq, int Hkv, int D, int page_size, float scale, int kv_tile,
                                     void* stream) {
  if (num_seqs <= 0 || max_q_len <= 0) return 0;
  // a page larger than the requested KV tile: stream it as one 128-key tile (the mma.sync kernel, whose tile is 64
  // keys, cannot take such pages)
  if (page_size == 128 && kv_tile == 64) kv_tile = 128;
  if ((D != 64 && D != 128) || (kv_tile != 64 && kv_tile != 128) || page_size < 8 || kv_tile % page_size != 0 ||
      Hq % Hkv != 0)
    return 2;
  CUtensorMap tk, tv;
  if (get_kv_slab_tmap(k_cache, num_pages, Hkv, D, page_size, &tk)) return 1;
  if (get_kv_slab_tmap(v_cache, num_pages, Hkv, D, page_size, &tv)) return 1;
  TcAttnParams p;
  p.q = reinterpret_cast<const __nv_bfloat16*>(q); p.q_ts = q_ts;
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.block_table = reinterpret_cast<const int32_t*>(block_table);
  p.seq_lens = reinterpret_cast<const int32_t*>(seq_lens);
  p.q_start = reinterpret_cast<const int32_t*>(q_start);
  p.max_blocks = max_blocks; p.Hq = Hq; p.Hkv = Hkv; p.G = Hq / Hkv;
  p.GP = 1;
  for (int d = (p.G < kTcRows ? p.G : kTcRows); d >= 1; --d)
    if (p.G % d == 0 && kTcRows % d == 0) { p.GP = d; break; }
  p.page_size = page_size; p.seq_offset = seq_offset;
  p.scale_log2 = scale * 1.4426950408889634f;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (D == 128) {
    return kv_tile == 128 ? launch_prefill_tc<128, 128>(tk, tv, p, num_seqs, max_q_len, st)
                          : launch_prefill_tc<128, 64>(tk, tv, p, num_seqs, max_q_len, st);
  }
  return kv_tile == 128 ? launch_prefill_tc<64, 128>(tk, tv, p, num_seqs, max_q_len, st)
                        : launch_prefill_tc<64, 64>(tk, tv, p, num_seqs, max_q_len, st);
}
