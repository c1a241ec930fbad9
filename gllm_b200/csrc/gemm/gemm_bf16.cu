// Persistent, warp-specialised bf16 GEMM for sm_90a:
//
//     C[M, N] = A[M, K] · W[N, K]^T  (+ bias)           (nn.Linear layout, both K-major)
//
//   * operands staged by TMA (128-byte swizzle) through an mbarrier ring filled by one producer warp,
//   * two consumer warpgroups, each multiplying 64 rows of the 128 x BN tile with wgmma.mma_async
//     (m64nBNk16, both operands from shared memory, fp32 accumulators in registers),
//   * the consumers apply the fused epilogue (bias, SiLU-gate for the merged gate/up projection),
//   * optional fused collectives over NVLink peer memory (SURVEY §2.4 X1/X2):
//       - all-gather ⊕ GEMM: the TMA producer gates each M tile on per-row-block
//         "ready" flags that peer ranks set after pushing their activation shard,
//       - GEMM ⊕ reduce-scatter: the epilogue stores each partial tile straight into the
//         owner rank's staging buffer (P2P st.global) and bumps a system-scope counter.
//
// Replaces the reference's cuBLAS F.linear call sites (gllm/layers/linear.py:130,247,339)
// and its GEMM -> NCCL all_reduce sequence (gllm/layers/linear.py:247-250).
#include "../common/host_utils.h"
#include "../common/ptx.cuh"
#include <string.h>

namespace b200 {

static constexpr int kBlockM = 128;
static constexpr int kBlockK = 64;  // 64 bf16 = 128 B = one swizzle atom row
static constexpr int kMmaK = 16;
static constexpr int kNumThreads = 384;  // warpgroup 0: TMA producer, warpgroups 1-2: MMA + epilogue
static constexpr int kConsumers = 256;
static constexpr int kMaxPeers = 8;

enum Epilogue : int { kEpiStore = 0, kEpiSiluMul = 1 };

struct GemmParams {
  int M, N, K;
  __nv_bfloat16* C;
  int ldc;
  const __nv_bfloat16* bias;
  // all-gather gating (null => disabled)
  const uint32_t* a_ready;      // arrival counters, one per 128-row block of A (written by peers)
  const uint32_t* a_expected;   // device-resident expected counts (CUDA-graph safe), comm/tp_fused.cu
  int m_rot;                    // first M tile to visit (this rank's shard)
  // reduce-scatter push (rs_world == 0 => disabled)
  int rs_world, rs_rank, rows_per_rank;
  uint32_t rs_inc;
  __nv_bfloat16* peer_out[kMaxPeers];
  uint32_t* peer_cnt[kMaxPeers];
  // rs_bcast: every row goes to EVERY rank's staging slot (one-shot all-reduce for decode-sized T: each rank
  // then reduces all rows itself, comm/tp_fused.cu bcast mode) instead of only to the row's owner
  int rs_bcast;
  // grouped (MoE) mode: M tile t multiplies the weight slab of expert tile_expert[t]
  const int32_t* tile_expert;
  const int32_t* num_m_tiles_ptr;  // device scalar: number of live M tiles
  int n_per_expert;
  // per-row destination table (EP combine push): row r of C is stored at row_dest[r] (any rank's memory
  // mapped over NVLink); 0 = padding row, not stored. comm/ep_a2a.cu builds the table.
  const int64_t* row_dest;
  // batched mode (batch > 0): `batch` independent [rows_per_batch, K] x [N, K]^T products over strided operands —
  // A is a 3-D tensor map (k, row, batch), batch b uses the weight slab b ([batch, N, K] contiguous) and writes
  // C + row * ldc + b * c_batch_stride. MLA weight absorption (q_nope·W_UK, out_lat·W_UV per head) runs on it
  // instead of a cuBLAS bmm (SURVEY §2.3 K13; reference: gllm/layers/attention.py:463-484).
  int batch, rows_per_batch;
  int64_t c_batch_stride;
  // split-K (decode-sized M): unit = (tile, k-slice); partials go through an fp32 workspace in a
  // thread-private layout, the last-arriving CTA of a tile sums them in slice order and runs the epilogue
  int split_k;
  float* ws;
  uint32_t* tile_cnt;
};

template <int BN>
struct GemmCfg {
  static constexpr int kABytes = kBlockM * kBlockK * 2;
  static constexpr int kBBytes = BN * kBlockK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  // epilogue staging: 8 warps x 16 rows x 64 output columns (bf16) + 8 x 16 destination row pointers
  static constexpr int kEpiBytes = 8 * 16 * 128 + 8 * 16 * 8;
  static constexpr int kSmemBudget = 224 * 1024 - kEpiBytes;
  static constexpr int kStagesRaw = kSmemBudget / kStageBytes;
  static constexpr int kStages = kStagesRaw > 8 ? 8 : kStagesRaw;
  // barriers: full[S], empty[S]
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align*/ + 256 + kEpiBytes;
};

template <int BN, int EPI>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const GemmParams p) {
  using Cfg = GemmCfg<BN>;
  constexpr int S = Cfg::kStages;
  constexpr int NACC = BN / 2;  // fp32 accumulators per consumer thread (64 x BN per warpgroup)

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S * Cfg::kStageBytes);
  uint64_t* empty_bar = full_bar + S;
  uint8_t* epi_smem = smem + S * Cfg::kStageBytes + 256;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // Programmatic dependent launch: dependents may start their prologue now; we ourselves may already be running
  // while the previous kernel drains. Grouped (MoE) mode reads device-side tile metadata right away, so it
  // waits here; the dense path first puts weight tiles in flight (producer warp below) and waits afterwards.
  griddep_launch();
  const bool grouped = p.tile_expert != nullptr || p.num_m_tiles_ptr != nullptr || p.batch > 0;
  if (grouped) griddep_wait();

  const int tpb = p.batch > 0 ? (p.rows_per_batch + kBlockM - 1) / kBlockM : 0;   // M tiles per batch entry
  const int num_m = p.batch > 0 ? p.batch * tpb
                    : p.num_m_tiles_ptr != nullptr ? min(*p.num_m_tiles_ptr, (p.M + kBlockM - 1) / kBlockM)
                                                   : (p.M + kBlockM - 1) / kBlockM;
  const int num_n = (p.N + BN - 1) / BN;
  const int num_tiles = num_m * num_n;
  const int num_kb = (p.K + kBlockK - 1) / kBlockK;
  const int split = p.split_k > 1 ? p.split_k : 1;
  const int kpb = (num_kb + split - 1) / split;  // k-blocks per unit (host guarantees no empty slice)
  const int num_units = num_tiles * split;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int i = 0; i < S; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kConsumers / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== TMA producer (one thread) =====================
    regs_dealloc<40>();
    if (warp == 0 && lane == 0) {
      uint32_t it = 0;
      // weights (B) do not depend on the previous kernel: put the first stages' B tiles in flight, then wait
      uint32_t pre = 0;
      if (!grouped) {
        if (static_cast<int>(blockIdx.x) < num_units) {
          const int tile = blockIdx.x / split;
          const int kb0 = (blockIdx.x - tile * split) * kpb;
          const int kb1 = min(num_kb, kb0 + kpb);
          const int n0 = (tile / num_m) * BN;
          pre = static_cast<uint32_t>(min(S, kb1 - kb0));
          for (uint32_t i = 0; i < pre; ++i) {
            uint8_t* sb = smem + i * Cfg::kStageBytes + Cfg::kABytes;
            mbar_expect_tx(&full_bar[i], Cfg::kStageBytes);
            tma_load_2d(sb, &tmap_b, &full_bar[i], (kb0 + static_cast<int>(i)) * kBlockK, n0, kEvictNormal);
          }
        }
        griddep_wait();
      }
      for (int unit = blockIdx.x; unit < num_units; unit += gridDim.x) {
        const int tile = unit / split;
        const int kb0 = (unit - tile * split) * kpb;
        const int kb1 = min(num_kb, kb0 + kpb);
        // M tiles are visited starting from this rank's own row shard (m_rot), so an all-gather ⊕ GEMM
        // works on local rows while the peers' rows are still arriving over NVLink
        const int mt = ((tile % num_m) + p.m_rot) % num_m;
        const int m0 = mt * kBlockM;
        const int n0 = (tile / num_m) * BN;
        const int bidx = p.batch > 0 ? mt / tpb : 0;
        const int b_row_off = p.batch > 0 ? bidx * p.n_per_expert
                              : p.tile_expert != nullptr ? p.tile_expert[mt] * p.n_per_expert : 0;
        if (p.a_ready != nullptr) {
          // all-gather ⊕ GEMM: the 128-row block `mt` of A is complete once its arrival counter reached
          // the device-resident expected value (advanced by rs_reduce_norm, comm/tp_fused.cu)
          const uint32_t want = *reinterpret_cast<const volatile uint32_t*>(p.a_expected + mt);
          SpinGuard guard;
          while (static_cast<int32_t>(ld_acquire_sys(p.a_ready + mt) - want) < 0) guard.poll();
          asm volatile("fence.proxy.async;" ::: "memory");
        }
        for (int kb = kb0; kb < kb1; ++kb, ++it) {
          const int s = it % S;
          const uint32_t ph = (it / S) & 1;
          uint8_t* sa = smem + s * Cfg::kStageBytes;
          uint8_t* sb = sa + Cfg::kABytes;
          if (it < pre) {  // B tile of this stage is already in flight (issued before griddep_wait)
            tma_load_2d(sa, &tmap_a, &full_bar[s], kb * kBlockK, m0, kEvictNormal);
            continue;
          }
          mbar_wait(&empty_bar[s], ph ^ 1);
          mbar_expect_tx(&full_bar[s], Cfg::kStageBytes);
          if (p.batch > 0) tma_load_3d(sa, &tmap_a, &full_bar[s], kb * kBlockK, (mt - bidx * tpb) * kBlockM, bidx);
          else tma_load_2d(sa, &tmap_a, &full_bar[s], kb * kBlockK, m0, kEvictNormal);
          tma_load_2d(sb, &tmap_b, &full_bar[s], kb * kBlockK, n0 + b_row_off, kEvictNormal);
        }
      }
    }
  } else {
    // ===================== MMA + epilogue warpgroups =====================
    regs_alloc<232>();
    if (!grouped) griddep_wait();
    const int ct = threadIdx.x - 128;   // consumer thread 0..255
    const int g = ct >> 7;              // warpgroup: rows [64 g, 64 g + 64) of the tile
    const int wq = (ct >> 5) & 3;       // warp inside the warpgroup: 16 rows each
    const int cw = ct >> 5;             // consumer warp 0..7
    // accumulator fragment: acc[4 j + {0,1}] = (row r0, cols 8 j + 2 (lane % 4) + {0,1}), acc[4 j + {2,3}] = row r0 + 8
    const int cq = 2 * (lane & 3);
    uint32_t it = 0;
    for (int unit = blockIdx.x; unit < num_units; unit += gridDim.x) {
      const int tile = unit / split;
      const int kb0 = (unit - tile * split) * kpb;
      const int kb1 = min(num_kb, kb0 + kpb);
      const int m0 = (((tile % num_m) + p.m_rot) % num_m) * kBlockM;
      const int n0 = (tile / num_m) * BN;

      float acc[NACC];
#pragma unroll
      for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
      // one wgmma group in flight: stage kb is released once the group of kb + 1 has been issued and kb's retired
      int prev_s = -1;
      for (int kb = kb0; kb < kb1; ++kb, ++it) {
        const int s = it % S;
        mbar_wait(&full_bar[s], (it / S) & 1);
        const uint32_t a_addr = smem_u32(smem + s * Cfg::kStageBytes) + g * (64 * 128);
        const uint32_t b_addr = smem_u32(smem + s * Cfg::kStageBytes + Cfg::kABytes);
        const uint64_t da = make_sw128_kmajor_desc(a_addr);
        const uint64_t db = make_sw128_kmajor_desc(b_addr);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / kMmaK; ++k) {
          // advance 32 B (16 bf16) along K inside the swizzle atom: +2 in 16-byte units
          wgmma_bf16_ss<BN>(acc, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), (kb > kb0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev_s >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_s]);
        prev_s = s;
      }
      wgmma_wait<0>();
      reg_fence(acc);
      if (prev_s >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_s]);

      int64_t c_off = 0;
      if (p.batch > 0) c_off = static_cast<int64_t>((m0 / kBlockM) / tpb) * p.c_batch_stride;
      const int out_N = (EPI == kEpiSiluMul) ? p.N / 2 : p.N;
      const int out_n0 = (EPI == kEpiSiluMul) ? n0 / 2 : n0;
      constexpr int OUT_W = (EPI == kEpiSiluMul) ? BN / 2 : BN;   // output columns of this tile

      if (split > 1) {
        // thread-private workspace layout: [unit][j][consumer thread] float4 — the reader of a value is the thread
        // that wrote it, so every access is a fully coalesced 512-byte warp transaction
        auto ws_ptr = [&](int u, int j) {
          return reinterpret_cast<float4*>(p.ws) + ((static_cast<size_t>(u) * (BN / 8) + j) * kConsumers + ct);
        };
#pragma unroll
        for (int j = 0; j < BN / 8; ++j)
          *ws_ptr(unit, j) = make_float4(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]);
        // every k-slice CTA of this tile reduces and stores its own 1/split column share (reduce-scatter
        // through L2): wait until all partners have published their partials. The partners are co-resident
        // (persistent grid, one CTA per SM, grid % split == 0 keeps a tile's slices in the same round).
        __threadfence();
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (ct == 0) {
          atomicAdd(p.tile_cnt + 2 * tile, 1u);
          SpinGuard guard;
          while (ld_acquire_gpu(p.tile_cnt + 2 * tile) < static_cast<uint32_t>(split)) guard.poll();
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        const int ks = unit - tile * split;
        const int share = OUT_W / split;
        const int c_lo = ks * share, c_hi = c_lo + share;
        // accumulators of this unit's column share: the slice-ordered sum of the partials
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int oc = (EPI == kEpiSiluMul && j * 8 >= BN / 2) ? j * 8 - BN / 2 : j * 8;
          if (oc < c_lo || oc >= c_hi) continue;
          float4 a4 = make_float4(0.f, 0.f, 0.f, 0.f);
          for (int sidx = 0; sidx < split; ++sidx) {
            const float4 x = __ldcg(ws_ptr(tile * split + sidx, j));
            a4.x += x.x; a4.y += x.y; a4.z += x.z; a4.w += x.w;
          }
          acc[4 * j] = a4.x; acc[4 * j + 1] = a4.y; acc[4 * j + 2] = a4.z; acc[4 * j + 3] = a4.w;
        }
      }
      const int ks = unit - tile * split;
      const int share = OUT_W / split;
      const int c_lo = ks * share, c_hi = c_lo + share;

      // destination row pointers (local C, or the owner rank's staging buffer for RS) of this warp's 16 rows
      unsigned long long* rowptr = reinterpret_cast<unsigned long long*>(epi_smem + 8 * 16 * 128) + cw * 16;
      if (lane < 16) {
        const int h = lane >> 3;
        const int rl = lane & 7;
        // row of (lane / 4 == rl) is owned by lanes 4 rl .. 4 rl + 3; recompute it here for lane < 16
        int row = m0 + 64 * g + 16 * wq + rl + 8 * h;
        bool ok = row < p.M;
        if (p.batch > 0) {
          const int mt = m0 / kBlockM, bidx = mt / tpb;
          row = (mt - bidx * tpb) * kBlockM + 64 * g + 16 * wq + rl + 8 * h;
          ok = row < p.rows_per_batch;
        }
        __nv_bfloat16* crow = nullptr;
        if (ok && p.row_dest != nullptr) {
          crow = reinterpret_cast<__nv_bfloat16*>(p.row_dest[row]);
          ok = crow != nullptr;
        } else if (ok) {
          if (p.rs_world > 0) {
            const int owner = p.rs_bcast ? 0 : row / p.rows_per_rank;
            const int r_local = row - owner * p.rows_per_rank;
            crow = p.peer_out[owner] + (static_cast<size_t>(p.rs_rank) * p.rows_per_rank + r_local) * p.ldc;
          } else {
            crow = p.C + static_cast<size_t>(row) * p.ldc + c_off;
          }
        }
        rowptr[rl + 8 * h] = ok ? reinterpret_cast<unsigned long long>(crow) : 0ull;
      }

      // Output tiles go through a per-warp swizzled smem transpose so that every global (or peer / NVLink)
      // store instruction writes full row segments instead of scattered 4-byte pieces.
      constexpr int W = OUT_W < 64 ? OUT_W : 64;                  // columns per staged chunk
      constexpr int LPR = W / 8;                                  // lanes (16 B each) per staged row
      constexpr int RPI = 32 / LPR;                               // rows per store instruction
      uint8_t* stg = epi_smem + cw * 2048;
      auto stage_put = [&](int jc, int h, float f0, float f1) {   // 2 output columns of row (lane / 4 + 8 h)
        const int r = (lane >> 2) + 8 * h;
        *reinterpret_cast<uint32_t*>(stg + r * (W * 2) + ((jc ^ (r & (LPR - 1) & 7)) * 16) + cq * 2) =
            pack_bf16(f0, f1);
      };
      auto stage_flush = [&](int col0, int col_lo, int col_hi) {  // col0: first output column of the staged chunk
        __syncwarp();
#pragma unroll
        for (int i2 = 0; i2 < 16 / RPI; ++i2) {
          const int r = i2 * RPI + lane / LPR;
          const int ch = lane % LPR;
          const uint4 o = *reinterpret_cast<const uint4*>(stg + r * (W * 2) + ((ch ^ (r & (LPR - 1) & 7)) * 16));
          __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(rowptr[r]);
          const int col = col0 + ch * 8;
          if (dst != nullptr && col < out_N && col >= col_lo && col < col_hi) {
            if (p.rs_bcast) {
              const ptrdiff_t delta = (dst - p.peer_out[0]) + col;
              for (int pr = 0; pr < p.rs_world; ++pr) st_v4(p.peer_out[pr] + delta, o);
            } else {
              st_v4(dst + col, o);
            }
          }
        }
        __syncwarp();
      };

      __syncwarp();
#pragma unroll
      for (int cc = 0; cc < OUT_W; cc += W) {
        if (cc + W <= c_lo || cc >= c_hi) continue;
#pragma unroll
        for (int jj = 0; jj < W / 8; ++jj) {
          const int j = cc / 8 + jj;             // output column group
          const int col = out_n0 + 8 * j + cq;
          if constexpr (EPI == kEpiStore) {
            float b0 = 0.f, b1 = 0.f;
            if (p.bias != nullptr && col < out_N) {
              const float2 bv = unpack_bf16(*reinterpret_cast<const uint32_t*>(p.bias + col));
              b0 = bv.x; b1 = bv.y;
            }
            stage_put(jj, 0, acc[4 * j] + b0, acc[4 * j + 1] + b1);
            stage_put(jj, 1, acc[4 * j + 2] + b0, acc[4 * j + 3] + b1);
          } else {
            // SiLU-gate: tile columns [0, BN/2) hold gate, [BN/2, BN) hold up for the same
            // BN/2 output features (weights are interleaved per tile at load time).
            const int ju = j + BN / 16;
            float o[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float gv = acc[4 * j + e];
              o[e] = gv / (1.0f + __expf(-gv)) * acc[4 * ju + e];
            }
            stage_put(jj, 0, o[0], o[1]);
            stage_put(jj, 1, o[2], o[3]);
          }
        }
        stage_flush(out_n0 + cc, out_n0 + c_lo, out_n0 + c_hi);
      }

      if (split > 1) {
        // depart: the last slice to finish reading re-arms both counters for the next launch
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (ct == 0) {
          const uint32_t t = atomicAdd(p.tile_cnt + 2 * tile + 1, 1u);
          if (t == static_cast<uint32_t>(split - 1)) {
            p.tile_cnt[2 * tile] = 0u;
            p.tile_cnt[2 * tile + 1] = 0u;
          }
        }
      }

      if (p.rs_world > 0) {
        // GEMM ⊕ reduce-scatter: all eight consumer warps have stored their rows; publish the
        // tile to every owner rank whose rows it covers.
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (ct == 0) {
          __threadfence_system();
          const int m1 = min(m0 + kBlockM, p.M);
          const int o0 = p.rs_bcast ? 0 : m0 / p.rows_per_rank;
          const int o1 = p.rs_bcast ? p.rs_world - 1 : (m1 - 1) / p.rows_per_rank;
          for (int o = o0; o <= o1; ++o) {
            red_add_relaxed_sys(p.peer_cnt[o] + p.rs_rank, p.rs_inc);
          }
        }
      }
    }
  }
}

template <int BN, int EPI>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p,
                       cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  static PerDeviceOnce configured;
  auto kern = gemm_bf16_kernel<BN, EPI>;
  if (configured.need()) {
    CUDA_CHECK_RET(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        Cfg::kSmemBytes));
    configured.done();
  }
  const int num_m = (p.M + kBlockM - 1) / kBlockM;
  const int num_n = (p.N + BN - 1) / BN;
  const int split = p.split_k > 1 ? p.split_k : 1;
  const int tiles = num_m * num_n * split;
  const int sms = (num_sms() / split) * split;  // split-K slices of a tile must run in the same round
  const int grid = tiles < sms ? tiles : sms;
  CUDA_CHECK_RET(launch_pdl(kern, dim3(grid), dim3(kNumThreads), Cfg::kSmemBytes, stream, ta, tb, p));
  return 0;
}

static int pick_bn(int M, int N, int epi, int forced) {
  if (forced > 0) return forced;
  const int sms = num_sms();
  const int num_m = (M + kBlockM - 1) / kBlockM;
  int best = 128;
  double best_cost = 1e30;
  const int cands[4] = {256, 128, 64, 32};
  for (int i = 0; i < 4; ++i) {
    const int bn = cands[i];
    if (epi == kEpiSiluMul && bn < 64) continue;
    const int tiles = num_m * ((N + bn - 1) / bn);
    const int waves = (tiles + sms - 1) / sms;
    // per-tile cost model: MMA time ∝ bn, plus a fixed per-tile overhead (A traffic, epilogue)
    const double cost = waves * (bn + 48.0);
    if (cost < best_cost) {
      best_cost = cost;
      best = bn;
    }
  }
  return best;
}

// Decode-sized M: few output tiles, so tile shape and a K split are chosen together. Cost model in SM clocks
// (an estimate, not a measurement): a 64-deep k-block costs ~650 clk for BN=256 and ~420 clk for BN<=128 (SMEM
// fill bound: 16 KB of A per k-block regardless of BN), a split-K round adds ~2000 + 24*BN.
static void pick_split(int M, int N, int K, int epi, int forced_bn, int64_t ws_bytes, int max_tiles, int* bn_out,
                       int* split_out) {
  const int sms = num_sms();
  const int num_m = (M + kBlockM - 1) / kBlockM;
  const int num_kb = (K + kBlockK - 1) / kBlockK;
  double best = 1e30;
  const int cands[4] = {256, 128, 64, 32};
  for (int i = 0; i < 4; ++i) {
    const int bn = cands[i];
    if (forced_bn > 0 && bn != forced_bn) continue;
    if (epi == kEpiSiluMul && bn < 64) continue;
    const int tiles = num_m * ((N + bn - 1) / bn);
    const double t_kb = bn >= 256 ? 650.0 : 420.0;
    for (int split = 1; split <= 8; split *= 2) {
      const int kpb = (num_kb + split - 1) / split;
      const int out_w = epi == kEpiSiluMul ? bn / 2 : bn;
      if (split > 1) {
        if (kpb < 4 || (split - 1) * kpb >= num_kb) continue;            // no empty / tiny slices
        if (out_w / split < (epi == kEpiSiluMul ? 16 : 32)) continue;     // column share granularity
        if (static_cast<int64_t>(tiles) * split * kBlockM * bn * 4 > ws_bytes || tiles > max_tiles) continue;
      }
      const int units = tiles * split;
      const int grid = (sms / split) * split;
      const int waves = (units + grid - 1) / grid;
      double unit_clk = kpb * t_kb + 700.0;
      if (split > 1) unit_clk += 24.0 * bn + 2000.0;                      // partial write + rendezvous + share sum
      const double cost = waves * unit_clk;
      if (cost < best) { best = cost; *bn_out = bn; *split_out = split; }
    }
  }
}

}  // namespace b200

using namespace b200;

// C-ABI entry point. All pointers are device pointers; `stream` is a cudaStream_t.
// a_rows: number of valid rows addressable in A (>= M).  epi: 0 store, 1 SiLU-gate.
// comm: optional pointer to a host-side GemmComm block (may be null).
struct GemmComm {
  const uint32_t* a_ready;
  const uint32_t* a_expected;
  int m_rot;
  int rs_world, rs_rank, rows_per_rank;
  uint32_t rs_inc;
  void* peer_out[kMaxPeers];
  uint32_t* peer_cnt[kMaxPeers];
  int rs_bcast;
};

static int g_max_split_m = -1, g_force_split = -1;

// (tile width, split-K factor) for a plain / all-gather-gated / reduce-scatter GEMM. Deterministic in its
// arguments: the consumer of a GEMM ⊕ reduce-scatter calls it again (gllm_gemm_bf16_tiles_covering) to know
// how many unit arrivals to expect.
static void choose_cfg(int M, int N, int K, int epi, int force_bn, int64_t ws_bytes, int max_tiles, int* bn_out,
                       int* split_out) {
  int bn = pick_bn(M, N, epi, force_bn);
  int split = 1;
  if (g_max_split_m < 0) {
    const char* e = getenv("GLLM_GEMM_SPLITK_MAX_M");
    g_max_split_m = e ? atoi(e) : 512;
  }
  if (g_force_split < 0) {
    const char* e = getenv("GLLM_GEMM_FORCE_SPLITK");  // tuning aid: only legal (bn, split) pairs
    g_force_split = e ? atoi(e) : 0;
  }
  if (ws_bytes > 0 && M <= g_max_split_m) pick_split(M, N, K, epi, force_bn, ws_bytes, max_tiles, &bn, &split);
  if (g_force_split > 0 && ws_bytes > 0) {
    split = g_force_split;
    const int num_kb = (K + kBlockK - 1) / kBlockK;
    const int kpb = (num_kb + split - 1) / split;
    const int out_w = epi == kEpiSiluMul ? bn / 2 : bn;
    const int tiles = ((M + kBlockM - 1) / kBlockM) * ((N + bn - 1) / bn);
    if ((split - 1) * kpb >= num_kb || out_w / split < (epi == kEpiSiluMul ? 16 : 32) || (split & (split - 1)) ||
        static_cast<int64_t>(tiles) * split * kBlockM * bn * 4 > ws_bytes || tiles > max_tiles)
      split = 1;
  }
  *bn_out = bn;
  *split_out = split;
}

// tuning aid (benchmarks/gemm_tune.py): force a split factor / the M ceiling of the split-K path at run time
GLLM_EXPORT int gllm_gemm_tune(int force_split, int max_split_m) {
  g_force_split = force_split;
  g_max_split_m = max_split_m;
  return 0;
}

GLLM_EXPORT int gllm_gemm_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, void* C,
                               int64_t ldc, int M, int N, int K, const void* bias, int epi,
                               int force_bn, const GemmComm* comm, void* ws, int64_t ws_bytes, void* tile_cnt,
                               int max_tiles, void* stream) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if ((K % 8) != 0 || (N % 8) != 0 || (lda % 8) != 0 || (ldw % 8) != 0 || (ldc % 8) != 0) {
    fprintf(stderr, "[gllm_b200] gemm_bf16: K, N and leading dims must be multiples of 8\n");
    return 1;
  }
  int bn = 128, split = 1;
  choose_cfg(M, N, K, epi, force_bn, ws != nullptr && tile_cnt != nullptr ? ws_bytes : 0, max_tiles, &bn, &split);
  CUtensorMap ta, tb;
  if (make_tmap_2d(&ta, A, M, K, lda * 2, kBlockM, kBlockK, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16)) return 1;
  if (make_tmap_2d(&tb, W, N, K, ldw * 2, bn, kBlockK, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16)) return 1;
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.split_k = split;
  p.ws = reinterpret_cast<float*>(ws);
  p.tile_cnt = reinterpret_cast<uint32_t*>(tile_cnt);
  p.M = M; p.N = N; p.K = K;
  p.C = reinterpret_cast<__nv_bfloat16*>(C);
  p.ldc = static_cast<int>(ldc);
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  if (comm != nullptr) {
    p.a_ready = comm->a_ready;
    p.a_expected = comm->a_expected;
    p.m_rot = comm->m_rot;
    p.rs_world = comm->rs_world;
    p.rs_rank = comm->rs_rank;
    p.rows_per_rank = comm->rows_per_rank;
    p.rs_bcast = comm->rs_bcast;
    p.rs_inc = comm->rs_inc;
    for (int i = 0; i < kMaxPeers; ++i) {
      p.peer_out[i] = reinterpret_cast<__nv_bfloat16*>(comm->peer_out[i]);
      p.peer_cnt[i] = comm->peer_cnt[i];
    }
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
#define DISPATCH(BN_)                                                          \
  case BN_:                                                                    \
    return epi == kEpiSiluMul ? launch_gemm<BN_, kEpiSiluMul>(ta, tb, p, st)   \
                              : launch_gemm<BN_, kEpiStore>(ta, tb, p, st);
  switch (bn) {
    DISPATCH(256)
    DISPATCH(128)
    DISPATCH(64)
    case 32:
      return launch_gemm<32, kEpiStore>(ta, tb, p, st);
    default:
      fprintf(stderr, "[gllm_b200] gemm_bf16: unsupported BN %d\n", bn);
      return 1;
  }
#undef DISPATCH
}

// Number of (m_tile, n_tile) pairs whose rows intersect [row0, row1) — used by the consumer
// of a fused GEMM ⊕ reduce-scatter to know how many tile arrivals to expect per source rank.
GLLM_EXPORT int gllm_gemm_bf16_tiles_covering(int M, int N, int K, int epi, int force_bn, int row0, int row1,
                                              int64_t ws_bytes, int max_tiles) {
  if (row1 > M) row1 = M;
  if (row1 <= row0) return 0;
  int bn = 128, split = 1;
  choose_cfg(M, N, K, epi, force_bn, ws_bytes, max_tiles, &bn, &split);
  const int t0 = row0 / kBlockM;
  const int t1 = (row1 - 1) / kBlockM;
  return (t1 - t0 + 1) * ((N + bn - 1) / bn) * split;  // every k-slice unit publishes its column share
}

// Batched GEMM over strided operands: for b in [0, B): C[:, b, :] = A[:, b, :] · W[b]^T with A [T, B, K] (row stride
// lda_t, batch stride lda_b, elements), W [B, N, K] contiguous, C [T, B, N] (row stride ldc_t, batch stride ldc_b).
GLLM_EXPORT int gllm_gemm_bf16_batched(const void* A, int64_t lda_t, int64_t lda_b, const void* W, void* C,
                                       int64_t ldc_t, int64_t ldc_b, int T, int B, int N, int K, void* stream) {
  if (T <= 0 || B <= 0) return 0;
  if ((K % 8) != 0 || (N % 8) != 0 || (lda_t % 8) != 0 || (lda_b % 8) != 0 || (ldc_t % 8) != 0 || (ldc_b % 8) != 0) {
    fprintf(stderr, "[gllm_b200] gemm_bf16_batched: K, N and strides must be multiples of 8\n");
    return 1;
  }
  const int bn = 128;
  CUtensorMap ta, tb;
  if (make_tmap_3d(&ta, A, K, T, B, lda_t * 2, lda_b * 2, kBlockK, kBlockM, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16)) return 1;
  if (make_tmap_2d(&tb, W, static_cast<uint64_t>(B) * N, K, static_cast<uint64_t>(K) * 2, bn, kBlockK,
                   CU_TENSOR_MAP_DATA_TYPE_BFLOAT16)) return 1;
  GemmParams p;
  memset(&p, 0, sizeof(p));
  const int tpb = (T + kBlockM - 1) / kBlockM;
  p.M = B * tpb * kBlockM; p.N = N; p.K = K;
  p.C = reinterpret_cast<__nv_bfloat16*>(C);
  p.ldc = static_cast<int>(ldc_t);
  p.batch = B;
  p.rows_per_batch = T;
  p.c_batch_stride = ldc_b;
  p.n_per_expert = N;
  return launch_gemm<128, kEpiStore>(ta, tb, p, reinterpret_cast<cudaStream_t>(stream));
}

// Grouped (MoE) GEMM: rows of A are expert-sorted and padded to 128-row tiles; tile t uses the weight
// slab W[tile_expert[t]] ([E, N, K] contiguous). The live tile count is read on the device.
// epi: 0 store, 1 SiLU-gate (slab rows interleaved per 64 like the dense gate/up weight).
GLLM_EXPORT int gllm_moe_grouped_gemm(const void* A, int64_t lda, const void* W, void* C, int64_t ldc,
                                      int max_tiles, int N, int K, int E, const void* tile_expert,
                                      const void* num_tiles_ptr, int epi, const void* row_dest, void* stream) {
  if (max_tiles <= 0) return 0;
  if ((K % 8) != 0 || (N % 8) != 0 || (lda % 8) != 0 || (ldc % 8) != 0) return 1;
  const int bn = 128;  // 64|64 gate/up interleave for the SiLU epilogue; good balance for expert tiles
  CUtensorMap ta, tb;
  const int M = max_tiles * kBlockM;
  if (make_tmap_2d(&ta, A, M, K, lda * 2, kBlockM, kBlockK, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16)) return 1;
  if (make_tmap_2d(&tb, W, static_cast<uint64_t>(E) * N, K, static_cast<uint64_t>(K) * 2, bn, kBlockK,
                   CU_TENSOR_MAP_DATA_TYPE_BFLOAT16)) return 1;
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = M; p.N = N; p.K = K;
  p.C = reinterpret_cast<__nv_bfloat16*>(C);
  p.ldc = static_cast<int>(ldc);
  p.tile_expert = reinterpret_cast<const int32_t*>(tile_expert);
  p.num_m_tiles_ptr = reinterpret_cast<const int32_t*>(num_tiles_ptr);
  p.n_per_expert = N;
  p.row_dest = reinterpret_cast<const int64_t*>(row_dest);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return epi == kEpiSiluMul ? launch_gemm<128, kEpiSiluMul>(ta, tb, p, st) : launch_gemm<128, kEpiStore>(ta, tb, p, st);
}
