// Small-M (decode) bf16 GEMM for sm_90a: swap-AB + split-K weight-streaming kernel.
//
//     C[M, N] = A[M, K] · W[N, K]^T        with M <= 256 (a decode micro-batch)
//
// For M << 128 a 128 x BN tile spends the SM's L2->SMEM fill bandwidth on the 128-row activation tile that
// every CTA re-reads, not on weights. Here the operands are swapped: the *weights* fill the 128-row MMA M
// slot (every byte fetched is a weight byte that must come from HBM anyway) and the tokens sit in the MMA
// N slot (N = BT = M rounded up to 16, 32, 64, 128 or 256), so one k-block stage is 16 KB of weights +
// BT x 128 B of activations. N/128 weight tiles are too few to fill 132 SMs for the attention projections,
// so K is split S ways; partial tiles go to an fp32 workspace (L2 resident) and the last CTA to arrive for
// a tile reduces them in a fixed order (deterministic), applies bias / SiLU-gate and stores bf16.
//
// Same warp specialisation as gemm_bf16.cu: warpgroup 0 TMA producer, warpgroups 1-2 wgmma (64 weight rows
// each, accumulators in registers) and epilogue.
#include <string.h>

#include "../common/host_utils.h"
#include "../common/ptx.cuh"

namespace b200 {

static constexpr int kWTile = 128;  // weight rows per tile (MMA M)
static constexpr int kBK = 64;
static constexpr int kSmThreads = 384;
static constexpr int kSmConsumers = 256;

struct SmallMParams {
  int M, N, K, BT;  // BT: token tile (multiple of 16, >= M)
  int S;            // split-K factor
  int kb_per_split;
  __nv_bfloat16* C;
  int ldc;
  const __nv_bfloat16* bias;
  float* ws;              // [num_n_tiles * S][BT][128] fp32 partials
  uint32_t* counters;     // [num_n_tiles], zero on entry, self-resetting
  int silu;               // 1: weight rows interleaved per 128: tile 2g = gate, tile 2g+1 = up
  int stages;
};

template <int BT>
__global__ void __launch_bounds__(kSmThreads, 1)
gemm_smallm_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x,
                   const SmallMParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int S = p.stages;
  constexpr int w_bytes = kWTile * kBK * 2;
  constexpr int x_bytes = BT * kBK * 2;
  constexpr int stage_bytes = w_bytes + x_bytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S * stage_bytes);
  uint64_t* empty_bar = full_bar + S;
  uint32_t* flag_smem = reinterpret_cast<uint32_t*>(empty_bar + S);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_n = (p.N + kWTile - 1) / kWTile;
  const int num_units = num_n * p.S;
  const int num_kb = (p.K + kBK - 1) / kBK;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_w);
    tma_prefetch_desc(&tmap_x);
    for (int i = 0; i < S; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kSmConsumers / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();

  griddep_launch();
  if (warp < 4) {
    regs_dealloc<40>();
    if (warp == 0 && lane == 0) {
      uint32_t it = 0;
      // PDL: weight tiles of the first stages go in flight before waiting for the previous kernel
      uint32_t pre = 0;
      if (static_cast<int>(blockIdx.x) < num_units) {
        const int nt = blockIdx.x / p.S, sp = blockIdx.x % p.S;
        const int kb0 = sp * p.kb_per_split;
        const int kb1 = min(kb0 + p.kb_per_split, num_kb);
        pre = static_cast<uint32_t>(min(S, kb1 - kb0));
        for (uint32_t i = 0; i < pre; ++i) {
          mbar_expect_tx(&full_bar[i], stage_bytes);
          tma_load_2d(smem + i * stage_bytes, &tmap_w, &full_bar[i], (kb0 + static_cast<int>(i)) * kBK, nt * kWTile,
                      kEvictFirst);
        }
      }
      griddep_wait();
      for (int u = blockIdx.x; u < num_units; u += gridDim.x) {
        const int nt = u / p.S, sp = u % p.S;
        const int kb0 = sp * p.kb_per_split;
        const int kb1 = min(kb0 + p.kb_per_split, num_kb);
        for (int kb = kb0; kb < kb1; ++kb, ++it) {
          const int s = it % S;
          const uint32_t ph = (it / S) & 1;
          uint8_t* sw = smem + s * stage_bytes;
          uint8_t* sx = sw + w_bytes;
          if (it < pre) {
            tma_load_2d(sx, &tmap_x, &full_bar[s], kb * kBK, 0, kEvictLast);
            continue;
          }
          mbar_wait(&empty_bar[s], ph ^ 1);
          mbar_expect_tx(&full_bar[s], stage_bytes);
          tma_load_2d(sw, &tmap_w, &full_bar[s], kb * kBK, nt * kWTile, kEvictFirst);
          tma_load_2d(sx, &tmap_x, &full_bar[s], kb * kBK, 0, kEvictLast);
        }
      }
    }
  } else {
    // ===================== MMA + epilogue =====================
    regs_alloc<232>();
    griddep_wait();
    const int ct = threadIdx.x - 128;      // 0..255
    const int g = ct >> 7;                 // warpgroup: weight rows [64 g, 64 g + 64) of the tile
    const int wq = (ct >> 5) & 3;
    // accumulator fragment: acc[4 j + {0,1}] = (weight row e0, tokens 8 j + 2 (lane % 4) + {0,1}); +{2,3}: e0 + 8
    const int e0 = 64 * g + 16 * wq + (lane >> 2);
    const int mq = 2 * (lane & 3);
    const bool direct = (p.S == 1 && !p.silu);
    uint32_t it = 0;
    for (int u = blockIdx.x; u < num_units; u += gridDim.x) {
      const int nt = u / p.S, sp = u % p.S;
      const int kb0 = sp * p.kb_per_split;
      const int kb1 = min(kb0 + p.kb_per_split, num_kb);
      float acc[BT / 2];
#pragma unroll
      for (int i = 0; i < BT / 2; ++i) acc[i] = 0.f;
      int prev_s = -1;
      for (int kb = kb0; kb < kb1; ++kb, ++it) {
        const int s = it % S;
        mbar_wait(&full_bar[s], (it / S) & 1);
        const uint32_t w_addr = smem_u32(smem + s * stage_bytes);
        const uint64_t dw = make_sw128_kmajor_desc(w_addr + g * (64 * 128));
        const uint64_t dx = make_sw128_kmajor_desc(w_addr + w_bytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBK / 16; ++k)
          wgmma_bf16_ss<BT>(acc, dw + (uint64_t)(k * 2), dx + (uint64_t)(k * 2), (kb > kb0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev_s >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_s]);
        prev_s = s;
      }
      wgmma_wait<0>();
      reg_fence(acc);
      if (prev_s >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_s]);

      if (direct) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int n = nt * kWTile + e0 + 8 * h;
          if (n >= p.N) continue;
          const float b = p.bias != nullptr ? __bfloat162float(p.bias[n]) : 0.f;
#pragma unroll
          for (int j = 0; j < BT / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int m = 8 * j + mq + e;
              if (m < p.M) p.C[static_cast<size_t>(m) * p.ldc + n] = __float2bfloat16(acc[4 * j + 2 * h + e] + b);
            }
          }
        }
        continue;
      }
      // partial tile in the workspace is token-major: ws[unit][m][128]
      float* __restrict__ wsu = p.ws + static_cast<size_t>(u) * BT * kWTile + e0;
#pragma unroll
      for (int j = 0; j < BT / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int m = 8 * j + mq + e;
          if (m < p.M) {
            wsu[static_cast<size_t>(m) * kWTile] = acc[4 * j + e];
            wsu[static_cast<size_t>(m) * kWTile + 8] = acc[4 * j + 2 + e];
          }
        }
      }

      // publish the partial tile; the last split to arrive reduces (fixed order => deterministic)
      __threadfence();
      asm volatile("bar.sync 1, 256;" ::: "memory");
      // SiLU-gate: weight rows are interleaved per 128 (tile 2g = gate, tile 2g+1 = up of the same 128
      // features), so a *pair* of tiles (2 S units) completes one output group.
      const int grp = p.silu ? (nt >> 1) : nt;
      const uint32_t need = static_cast<uint32_t>(p.silu ? 2 * p.S : p.S);
      if (ct == 0) {
        const uint32_t old = atomicAdd(p.counters + grp, 1u);
        *flag_smem = (old == need - 1u) ? 1u : 0u;
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      const uint32_t last = *flag_smem;
      asm volatile("bar.sync 1, 256;" ::: "memory");   // flag read by all before the next unit rewrites it
      if (last) {
        __threadfence();
        const float* __restrict__ base =
            p.ws + static_cast<size_t>(p.silu ? 2 * grp : nt) * p.S * BT * kWTile;
        const size_t unit_stride = static_cast<size_t>(BT) * kWTile;
        const int n4 = ct & 31;   // float4 column group
        const int mr = ct >> 5;   // 0..7
        constexpr int U = 2;      // rows in flight per thread
        constexpr int RS = 8;     // rows per pass of the 256 threads
        if (!p.silu) {
          const int ncol = nt * kWTile + n4 * 4;
          float bb[4] = {0.f, 0.f, 0.f, 0.f};
          if (p.bias != nullptr) {
#pragma unroll
            for (int j = 0; j < 4; ++j) if (ncol + j < p.N) bb[j] = __bfloat162float(p.bias[ncol + j]);
          }
          for (int m0 = 0; m0 < p.M; m0 += RS * U) {
            float4 a[U];
#pragma unroll
            for (int uu = 0; uu < U; ++uu) {
              const int m = m0 + uu * RS + mr;
              a[uu] = make_float4(bb[0], bb[1], bb[2], bb[3]);
              if (m < p.M) {
                for (int s2 = 0; s2 < p.S; ++s2) {
                  const float4 t = __ldcg(reinterpret_cast<const float4*>(
                      base + s2 * unit_stride + static_cast<size_t>(m) * kWTile + n4 * 4));
                  a[uu].x += t.x; a[uu].y += t.y; a[uu].z += t.z; a[uu].w += t.w;
                }
              }
            }
#pragma unroll
            for (int uu = 0; uu < U; ++uu) {
              const int m = m0 + uu * RS + mr;
              if (m < p.M) {
                __nv_bfloat16* dst = p.C + static_cast<size_t>(m) * p.ldc + ncol;
                if (ncol + 3 < p.N) {
                  *reinterpret_cast<uint2*>(dst) = make_uint2(pack_bf16(a[uu].x, a[uu].y), pack_bf16(a[uu].z, a[uu].w));
                } else {
                  const float v[4] = {a[uu].x, a[uu].y, a[uu].z, a[uu].w};
                  for (int j = 0; j < 4; ++j) if (ncol + j < p.N) dst[j] = __float2bfloat16(v[j]);
                }
              }
            }
          }
        } else {
          // gate partials live in the units of tile 2g, up partials in the units of tile 2g+1
          const int f = grp * kWTile + n4 * 4;
          const float* __restrict__ base_up = base + static_cast<size_t>(p.S) * unit_stride;
          for (int m0 = 0; m0 < p.M; m0 += RS * U) {
            float4 gg[U], up[U];
#pragma unroll
            for (int uu = 0; uu < U; ++uu) {
              const int m = m0 + uu * RS + mr;
              gg[uu] = make_float4(0.f, 0.f, 0.f, 0.f);
              up[uu] = gg[uu];
              if (m < p.M) {
                for (int s2 = 0; s2 < p.S; ++s2) {
                  const size_t off = s2 * unit_stride + static_cast<size_t>(m) * kWTile + n4 * 4;
                  const float4 tg = __ldcg(reinterpret_cast<const float4*>(base + off));
                  const float4 tu = __ldcg(reinterpret_cast<const float4*>(base_up + off));
                  gg[uu].x += tg.x; gg[uu].y += tg.y; gg[uu].z += tg.z; gg[uu].w += tg.w;
                  up[uu].x += tu.x; up[uu].y += tu.y; up[uu].z += tu.z; up[uu].w += tu.w;
                }
              }
            }
#pragma unroll
            for (int uu = 0; uu < U; ++uu) {
              const int m = m0 + uu * RS + mr;
              if (m < p.M && f + 3 < p.N / 2) {
                const float o0 = gg[uu].x / (1.f + __expf(-gg[uu].x)) * up[uu].x;
                const float o1 = gg[uu].y / (1.f + __expf(-gg[uu].y)) * up[uu].y;
                const float o2 = gg[uu].z / (1.f + __expf(-gg[uu].z)) * up[uu].z;
                const float o3 = gg[uu].w / (1.f + __expf(-gg[uu].w)) * up[uu].w;
                *reinterpret_cast<uint2*>(p.C + static_cast<size_t>(m) * p.ldc + f) =
                    make_uint2(pack_bf16(o0, o1), pack_bf16(o2, o3));
              }
            }
          }
        }
        if (ct == 0) p.counters[grp] = 0u;  // ready for the next launch
      }
    }
  }
}

template <int BT>
static int launch_smallm(const CUtensorMap& tw, const CUtensorMap& tx, const SmallMParams& p, int grid, int smem_bytes,
                         cudaStream_t st) {
  static PerDeviceOnce configured;
  if (configured.need()) {
    CUDA_CHECK_RET(cudaFuncSetAttribute(gemm_smallm_kernel<BT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    configured.done();
  }
  CUDA_CHECK_RET(launch_pdl(gemm_smallm_kernel<BT>, dim3(grid), dim3(kSmThreads), smem_bytes, st, tw, tx, p));
  return 0;
}

}  // namespace b200

using namespace b200;

// ws: fp32 workspace of at least gllm_gemm_smallm_ws_floats() elements; counters: >= ceil(N/128)
// uint32 zeros. silu: weight rows interleaved per 128 (gate|up), output has N/2 columns.
GLLM_EXPORT int gllm_gemm_smallm(const void* A, int64_t lda, const void* W, int64_t ldw, void* C, int64_t ldc,
                                 int M, int N, int K, const void* bias, int silu, int force_split, void* ws,
                                 int64_t ws_floats, void* counters, void* stream) {
  if (M <= 0 || N <= 0) return 0;
  // N and ldc as in gllm_gemm_bf16: the split-K reduction stores 4 bf16 (8 bytes) at C + m * ldc + 4 j
  if (M > 256 || (K % 8) != 0 || (N % 8) != 0 || (lda % 8) != 0 || (ldw % 8) != 0 || (ldc % 8) != 0) {
    fprintf(stderr, "[gllm_b200] gemm_smallm: unsupported shape M=%d N=%d K=%d (N, K and leading dims must be "
            "multiples of 8)\n", M, N, K);
    return 1;
  }
  SmallMParams p;
  memset(&p, 0, sizeof(p));
  p.M = M; p.N = N; p.K = K;
  p.BT = M <= 16 ? 16 : M <= 32 ? 32 : M <= 64 ? 64 : M <= 128 ? 128 : 256;  // wgmma N of the token tile
  const int num_n = (N + kWTile - 1) / kWTile;
  const int num_kb = (K + kBK - 1) / kBK;
  const int sms = num_sms();
  // split-K: minimise waves * (k-blocks per unit + fixed per-unit overhead)
  int best_s = 1;
  double best_cost = 1e30;
  for (int s = 1; s <= 16 && s <= num_kb; ++s) {
    const int kbs = (num_kb + s - 1) / s;
    if ((s - 1) * kbs >= num_kb) continue;  // empty split
    const int units = num_n * s;
    if ((s > 1 || silu) && static_cast<int64_t>(units) * kWTile * p.BT > ws_floats) continue;
    const int waves = (units + sms - 1) / sms;
    // unit of cost = one k-block of this shape (fill-bound: (16 KB + BT*128 B) / 64 B/clk)
    const double kb_cyc = 256.0 + 2.0 * p.BT;
    const double ovh = 2.0 + 30.0 * p.BT / kb_cyc;                // prologue + accumulator drain/store per unit
    const double red = (s > 1) ? 4.0 * M * s / kb_cyc : 0.0;      // last-arriver reduction
    const double cost = waves * (kbs + ovh) + red;
    if (cost < best_cost - 1e-9) { best_cost = cost; best_s = s; }
  }
  if (force_split > 0) {
    best_s = force_split;
    while (best_s > 1 && ((best_s - 1) * ((num_kb + best_s - 1) / best_s) >= num_kb ||
                          static_cast<int64_t>(num_n) * best_s * kWTile * p.BT > ws_floats)) --best_s;
  }
  p.S = best_s;
  p.kb_per_split = (num_kb + p.S - 1) / p.S;
  if (static_cast<int64_t>(num_n) * p.S * kWTile * p.BT > ws_floats && !(p.S == 1 && !silu)) {
    fprintf(stderr, "[gllm_b200] gemm_smallm: workspace too small\n");
    return 1;
  }
  p.C = reinterpret_cast<__nv_bfloat16*>(C);
  p.ldc = static_cast<int>(ldc);
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  p.ws = reinterpret_cast<float*>(ws);
  p.counters = reinterpret_cast<uint32_t*>(counters);
  p.silu = silu;
  const int stage_bytes = kWTile * kBK * 2 + p.BT * kBK * 2;
  int stages = (216 * 1024) / stage_bytes;
  if (stages > 12) stages = 12;
  p.stages = stages;
  const int smem_bytes = stages * stage_bytes + 1024 + 512;
  CUtensorMap tw, tx;
  if (make_tmap_2d(&tw, W, N, K, ldw * 2, kWTile, kBK, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16)) return 1;
  if (make_tmap_2d(&tx, A, M, K, lda * 2, p.BT, kBK, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16)) return 1;
  const int units = num_n * p.S;
  const int grid = units < sms ? units : sms;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (p.BT) {
    case 16: return launch_smallm<16>(tw, tx, p, grid, smem_bytes, st);
    case 32: return launch_smallm<32>(tw, tx, p, grid, smem_bytes, st);
    case 64: return launch_smallm<64>(tw, tx, p, grid, smem_bytes, st);
    case 128: return launch_smallm<128>(tw, tx, p, grid, smem_bytes, st);
    default: return launch_smallm<256>(tw, tx, p, grid, smem_bytes, st);
  }
}
