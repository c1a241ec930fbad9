// W4A16 GEMM for sm_90a: int4 weights with 16-bit group scales and uint8 zero points, bf16 activations.
//
//     C[M, N] = A[M, K] · W[N, K]^T,     W[n, k] = bf16( fp32(s[k/g, n]) · (q[n, k] − z[k/g, n]) )
//
// Swap-AB like gemm_bf16_smallm.cu: the weights fill the MMA M slot (two consumer warpgroups x 64 rows = a 128-row
// tile) and the tokens sit in the MMA N slot in tiles of BT = 16 .. 256. A producer warp streams, through an mbarrier
// ring, per 128-wide k-block: the packed codes of the weight tile (8 KB), the scale and zero rows of the groups the
// k-block touches, and the activation tile (two 128-byte-swizzled boxes, K-major). The consumers dequantise straight
// into the wgmma A fragment in registers and issue `wgmma` with A from registers and B from shared memory.
//
// Device layout (built by ops.ref.w4a16_pack; the same bytes on the CPU and the GPU):
//   packed  int32 [Np, Kp/8], Np = N rounded up to 16, Kp = K rounded up to 128. Rows = N, K-major: block (16 rows,
//           128 k) is 1 KB, holding 256 words in the order [k-half h][lane l][k-step j] (j < 4): the word is the 8
//           codes of lane l's m64k16 A fragment for k-step 4h + j, nibble e = element e of the fragment (a[e/2],
//           low half first). One 16-byte shared load gives a lane its fragments of four k-steps, conflict free.
//   scales  fp16 or bf16 [G, N], G = ceil(K/g) (transposed checkpoint scales: one TMA row per group)
//   zeros   uint8 [G, Np] (zero points, already +1 for GPTQ v1)
// g is 32, 64, 128 or at least K (one group).
//
// Numerics: 2^23 + q is built by OR-ing the code into the mantissa of 2^23, and (2^23 + q) − (2^23 + z) is exact, as
// is its product with the fp32 scale (a 16-bit scale has at most 11 significant bits, |q − z| <= 16); the product is
// rounded to bf16 once. So the GEMM multiplies exactly the dequantised W of ops.ref.w4a16_dequant.
//
// For small M, K is split S ways as in the bf16 small-M kernel: partial tiles go to the fp32 workspace and the last
// CTA to arrive for a (token tile, weight tile) reduces them in a fixed order, so every call returns the same bits.
// Larger M sweeps token tiles of 256, re-streaming (from L2) and re-dequantising the weight tile per token tile.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <string.h>

#include "../common/host_utils.h"
#include "../common/ptx.cuh"
#include "../common/wgmma.cuh"

namespace b200 {

static constexpr int kW4Tile = 128;     // weight rows per tile (2 warpgroups x 64)
static constexpr int kW4BK = 128;       // k per stage
static constexpr int kW4Threads = 384;  // warpgroup 0: producer, 1-2: consumers
static constexpr int kW4Consumers = 256;
static constexpr int kW4WBytes = kW4Tile * kW4BK / 2;   // 8 KB of codes
static constexpr int kW4SBytes = 4 * kW4Tile * 2;       // up to 4 group rows of scales
static constexpr int kW4ZBytes = 1024;                  // up to 4 group rows of zeros (512 B), 1 KB aligned

struct W4Params {
  int M, N, K, BT;
  int S, kb_per_split;
  int num_m;        // token tiles
  int group;        // g (>= K: one group)
  int gps;          // group rows loaded per stage: max(1, 128 / g)
  int gsh;          // k-step -> group row in the stage: j >> gsh
  int scale_bf16;   // scales are bf16 (else fp16)
  __nv_bfloat16* C;
  int ldc;
  const __nv_bfloat16* bias;
  float* ws;            // [units][BT][128] fp32 partials
  uint32_t* counters;   // [num_n * num_m], zero on entry, self-resetting
  int stages;
};

__device__ __forceinline__ float w4_scale(const uint16_t* s, int i, int bf16) {
  const uint16_t v = s[i];
  return bf16 ? __uint_as_float(static_cast<uint32_t>(v) << 16) : __half2float(__ushort_as_half(v));
}

// one word of 8 codes -> the bf16 A fragment of one k-step: a[p] = (elements 2p, 2p + 1), rows r0 (p even) / r0 + 8
__device__ __forceinline__ void w4_dequant(uint32_t (&a)[4], uint32_t w, float zf0, float zf1, float s0, float s1) {
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const float zf = (p & 1) ? zf1 : zf0;
    const float s = (p & 1) ? s1 : s0;
    const float lo = __uint_as_float(0x4B000000u | ((w >> (8 * p)) & 0xFu)) - zf;
    const float hi = __uint_as_float(0x4B000000u | ((w >> (8 * p + 4)) & 0xFu)) - zf;
    a[p] = pack_bf16(__fmul_rn(lo, s), __fmul_rn(hi, s));
  }
}

template <int BT>
__global__ void __launch_bounds__(kW4Threads, 1)
gemm_w4a16_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x,
                  const __grid_constant__ CUtensorMap tmap_s, const __grid_constant__ CUtensorMap tmap_z,
                  const W4Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int NS = p.stages;
  constexpr int x_bytes = BT * kW4BK * 2;
  constexpr int stage_bytes = kW4WBytes + x_bytes + kW4SBytes + kW4ZBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + NS * stage_bytes);
  uint64_t* empty_bar = full_bar + NS;
  uint32_t* flag_smem = reinterpret_cast<uint32_t*>(empty_bar + NS);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_n = (p.N + kW4Tile - 1) / kW4Tile;
  const int num_units = num_n * p.num_m * p.S;
  const int num_kb = (p.K + kW4BK - 1) / kW4BK;
  const uint32_t tx_bytes = kW4WBytes + x_bytes + p.gps * (kW4Tile * 2 + kW4Tile);

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_w);
    tma_prefetch_desc(&tmap_x);
    tma_prefetch_desc(&tmap_s);
    tma_prefetch_desc(&tmap_z);
    for (int i = 0; i < NS; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kW4Consumers / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();

  griddep_launch();
  if (warp < 4) {
    regs_dealloc<40>();
    if (warp == 0 && lane == 0) {
      // weights, scales and zeros of the first stages go in flight before waiting for the previous kernel
      auto load_w = [&](int s, int kb, int nt) {
        uint8_t* st = smem + s * stage_bytes;
        const int grow = static_cast<int>((static_cast<int64_t>(kb) * kW4BK) / p.group);
        tma_load_2d(st, &tmap_w, &full_bar[s], kb * (kW4BK / 2), nt * kW4Tile, kEvictFirst);
        tma_load_2d(st + kW4WBytes + x_bytes, &tmap_s, &full_bar[s], nt * kW4Tile, grow, kEvictFirst);
        tma_load_2d(st + kW4WBytes + x_bytes + kW4SBytes, &tmap_z, &full_bar[s], nt * kW4Tile, grow, kEvictFirst);
      };
      uint32_t it = 0, pre = 0;
      if (static_cast<int>(blockIdx.x) < num_units) {
        const int grp = blockIdx.x / p.S, sp = blockIdx.x % p.S;
        const int kb0 = sp * p.kb_per_split;
        const int kb1 = min(kb0 + p.kb_per_split, num_kb);
        pre = static_cast<uint32_t>(max(0, min(NS, kb1 - kb0)));
        for (uint32_t i = 0; i < pre; ++i) {
          mbar_expect_tx(&full_bar[i], tx_bytes);
          load_w(static_cast<int>(i), kb0 + static_cast<int>(i), grp / p.num_m);
        }
      }
      griddep_wait();
      for (int u = blockIdx.x; u < num_units; u += gridDim.x) {
        const int grp = u / p.S, sp = u % p.S;
        const int nt = grp / p.num_m, mt = grp % p.num_m;
        const int kb0 = sp * p.kb_per_split;
        const int kb1 = min(kb0 + p.kb_per_split, num_kb);
        for (int kb = kb0; kb < kb1; ++kb, ++it) {
          const int s = it % NS;
          if (it >= pre) {
            mbar_wait(&empty_bar[s], ((it / NS) & 1) ^ 1);
            mbar_expect_tx(&full_bar[s], tx_bytes);
            load_w(s, kb, nt);
          }
          uint8_t* sx = smem + s * stage_bytes + kW4WBytes;
          tma_load_2d(sx, &tmap_x, &full_bar[s], kb * kW4BK, mt * BT, kEvictLast);
          tma_load_2d(sx + x_bytes / 2, &tmap_x, &full_bar[s], kb * kW4BK + 64, mt * BT, kEvictLast);
        }
      }
    }
  } else {
    // ===================== dequant + MMA + epilogue =====================
    regs_alloc<232>();
    griddep_wait();
    const int ct = threadIdx.x - 128;      // 0..255
    const int g = ct >> 7;                 // warpgroup: weight rows [64 g, 64 g + 64) of the tile
    const int wq = (ct >> 5) & 3;
    // A fragment rows of this lane: r0 and r0 + 8; accumulator rows the same
    const int r0 = 64 * g + 16 * wq + (lane >> 2);
    const int mq = 2 * (lane & 3);
    const bool direct = (p.S == 1);
    uint32_t it = 0;
    for (int u = blockIdx.x; u < num_units; u += gridDim.x) {
      const int grp = u / p.S, sp = u % p.S;
      const int nt = grp / p.num_m, mt = grp % p.num_m;
      const int kb0 = sp * p.kb_per_split;
      const int kb1 = min(kb0 + p.kb_per_split, num_kb);
      float acc[BT / 2];
#pragma unroll
      for (int i = 0; i < BT / 2; ++i) acc[i] = 0.f;
      for (int kb = kb0; kb < kb1; ++kb, ++it) {
        const int s = it % NS;
        mbar_wait(&full_bar[s], (it / NS) & 1);
        const uint8_t* st = smem + s * stage_bytes;
        const uint4 wa = *reinterpret_cast<const uint4*>(st + (4 * g + wq) * 1024 + lane * 16);
        const uint4 wb = *reinterpret_cast<const uint4*>(st + (4 * g + wq) * 1024 + 512 + lane * 16);
        const uint16_t* ss = reinterpret_cast<const uint16_t*>(st + kW4WBytes + x_bytes);
        const uint8_t* sz = st + kW4WBytes + x_bytes + kW4SBytes;
        const uint32_t words[8] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w};
        uint32_t a[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int gr = j >> p.gsh;
          const float s0 = w4_scale(ss, gr * kW4Tile + r0, p.scale_bf16);
          const float s1 = w4_scale(ss, gr * kW4Tile + r0 + 8, p.scale_bf16);
          const float zf0 = __uint_as_float(0x4B000000u | sz[gr * kW4Tile + r0]);
          const float zf1 = __uint_as_float(0x4B000000u | sz[gr * kW4Tile + r0 + 8]);
          w4_dequant(a[j], words[j], zf0, zf1, s0, s1);
        }
        const uint64_t dx = make_sw128_kmajor_desc(smem_u32(st + kW4WBytes));
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < 8; ++j)
          wgmma_bf16_rs<BT>(acc, a[j], dx + static_cast<uint64_t>((j >> 2) * (x_bytes / 2 / 16) + (j & 3) * 2), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence(acc);
        if (lane == 0) mbar_arrive(&empty_bar[s]);
      }
      const int m_base = mt * BT;
      const int mv = min(BT, p.M - m_base);   // valid token rows of this tile

      if (direct) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int n = nt * kW4Tile + r0 + 8 * h;
          if (n >= p.N) continue;
          const float b = p.bias != nullptr ? __bfloat162float(p.bias[n]) : 0.f;
#pragma unroll
          for (int j = 0; j < BT / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int m = 8 * j + mq + e;
              if (m < mv)
                p.C[static_cast<size_t>(m_base + m) * p.ldc + n] = __float2bfloat16(acc[4 * j + 2 * h + e] + b);
            }
          }
        }
        continue;
      }
      // partial tile in the workspace is token-major: ws[unit][m][128]
      float* __restrict__ wsu = p.ws + static_cast<size_t>(u) * BT * kW4Tile + r0;
#pragma unroll
      for (int j = 0; j < BT / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int m = 8 * j + mq + e;
          if (m < mv) {
            wsu[static_cast<size_t>(m) * kW4Tile] = acc[4 * j + e];
            wsu[static_cast<size_t>(m) * kW4Tile + 8] = acc[4 * j + 2 + e];
          }
        }
      }
      // publish the partial tile; the last split to arrive reduces (fixed order => deterministic)
      __threadfence();
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (ct == 0) {
        const uint32_t old = atomicAdd(p.counters + grp, 1u);
        *flag_smem = (old == static_cast<uint32_t>(p.S) - 1u) ? 1u : 0u;
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      const uint32_t last = *flag_smem;
      asm volatile("bar.sync 1, 256;" ::: "memory");   // flag read by all before the next unit rewrites it
      if (last) {
        __threadfence();
        const float* __restrict__ base = p.ws + static_cast<size_t>(grp) * p.S * BT * kW4Tile;
        const size_t unit_stride = static_cast<size_t>(BT) * kW4Tile;
        const int n4 = ct & 31;   // float4 column group
        const int mr = ct >> 5;   // 0..7
        const int ncol = nt * kW4Tile + n4 * 4;
        float bb[4] = {0.f, 0.f, 0.f, 0.f};
        if (p.bias != nullptr) {
#pragma unroll
          for (int j = 0; j < 4; ++j) if (ncol + j < p.N) bb[j] = __bfloat162float(p.bias[ncol + j]);
        }
        for (int m = mr; m < mv; m += 8) {
          float4 a = make_float4(bb[0], bb[1], bb[2], bb[3]);
          for (int s2 = 0; s2 < p.S; ++s2) {
            const float4 t = __ldcg(reinterpret_cast<const float4*>(base + s2 * unit_stride +
                                                                    static_cast<size_t>(m) * kW4Tile + n4 * 4));
            a.x += t.x; a.y += t.y; a.z += t.z; a.w += t.w;
          }
          __nv_bfloat16* dst = p.C + static_cast<size_t>(m_base + m) * p.ldc + ncol;
          if (ncol + 3 < p.N) {
            *reinterpret_cast<uint2*>(dst) = make_uint2(pack_bf16(a.x, a.y), pack_bf16(a.z, a.w));
          } else {
            const float v[4] = {a.x, a.y, a.z, a.w};
            for (int j = 0; j < 4; ++j) if (ncol + j < p.N) dst[j] = __float2bfloat16(v[j]);
          }
        }
        if (ct == 0) p.counters[grp] = 0u;  // ready for the next launch
      }
    }
  }
}

template <int BT>
static int launch_w4a16(const CUtensorMap& tw, const CUtensorMap& tx, const CUtensorMap& ts, const CUtensorMap& tz,
                        const W4Params& p, int grid, int smem_bytes, cudaStream_t st) {
  static PerDeviceOnce configured;
  if (configured.need()) {
    CUDA_CHECK_RET(cudaFuncSetAttribute(gemm_w4a16_kernel<BT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        227 * 1024));
    configured.done();
  }
  CUDA_CHECK_RET(launch_pdl(gemm_w4a16_kernel<BT>, dim3(grid), dim3(kW4Threads), smem_bytes, st, tw, tx, ts, tz, p));
  return 0;
}

}  // namespace b200

using namespace b200;

// A bf16 [M, K] (row pitch lda elements); Wq / scales / zeros in the device layout above (N a multiple of 8, K of
// 32); C bf16 [M, N] (row pitch ldc); bias bf16 [N] or null. ws: fp32 split-K workspace of ws_floats elements;
// counters: uint32 zeros, at least ceil(N/128) * ceil(M/256). force_split > 0 forces the split-K factor.
GLLM_EXPORT int gllm_gemm_w4a16(const void* A, int64_t lda, const void* Wq, const void* scales, const void* zeros,
                                int scale_bf16, int group, void* C, int64_t ldc, int M, int N, int K,
                                const void* bias, int force_split, void* ws, int64_t ws_floats, void* counters,
                                int64_t num_counters, void* stream) {
  if (M <= 0 || N <= 0) return 0;
  if ((K % 32) != 0 || (N % 8) != 0 || (lda % 8) != 0 || (ldc % 8) != 0 ||
      !(group == 32 || group == 64 || group == 128 || group >= K)) {
    fprintf(stderr, "[gllm_b200] gemm_w4a16: unsupported shape M=%d N=%d K=%d g=%d (N and leading dims must be "
            "multiples of 8, K of 32, g 32/64/128 or >= K)\n", M, N, K, group);
    return 1;
  }
  W4Params p;
  memset(&p, 0, sizeof(p));
  p.M = M; p.N = N; p.K = K;
  p.BT = M <= 16 ? 16 : M <= 32 ? 32 : M <= 64 ? 64 : M <= 128 ? 128 : 256;
  p.num_m = (M + p.BT - 1) / p.BT;
  p.group = group;
  p.gps = group < kW4BK ? kW4BK / group : 1;
  p.gsh = group == 32 ? 1 : group == 64 ? 2 : 3;
  p.scale_bf16 = scale_bf16;
  const int num_n = (N + kW4Tile - 1) / kW4Tile;
  const int num_kb = (K + kW4BK - 1) / kW4BK;
  const int tiles = num_n * p.num_m;
  const int sms = num_sms();
  // split-K: minimise waves * (k-blocks per unit + fixed per-unit overhead), as gllm_gemm_smallm. The choice depends
  // on M only through the token tile, so a CUDA-graph bucket and the eager batch it pads compute each row alike.
  int best_s = 1;
  double best_cost = 1e30;
  for (int s = 1; s <= 16 && s <= num_kb; ++s) {
    const int kbs = (num_kb + s - 1) / s;
    if ((s - 1) * kbs >= num_kb) continue;  // empty split
    const int units = tiles * s;
    if (s > 1 && (static_cast<int64_t>(units) * kW4Tile * p.BT > ws_floats || tiles > num_counters)) continue;
    const int waves = (units + sms - 1) / sms;
    const double kb_cyc = 128.0 + 4.0 * p.BT;                    // (8 KB + BT * 256 B) / 64 B/clk
    const double ovh = 2.0 + 30.0 * p.BT / kb_cyc;
    const double red = (s > 1) ? 4.0 * p.BT * s / kb_cyc : 0.0;
    const double cost = waves * (kbs + ovh) + red;
    if (cost < best_cost - 1e-9) { best_cost = cost; best_s = s; }
  }
  if (force_split > 0) {
    best_s = force_split;
    while (best_s > 1 && ((best_s - 1) * ((num_kb + best_s - 1) / best_s) >= num_kb ||
                          static_cast<int64_t>(tiles) * best_s * kW4Tile * p.BT > ws_floats ||
                          tiles > num_counters)) --best_s;
  }
  p.S = best_s;
  p.kb_per_split = (num_kb + p.S - 1) / p.S;
  p.C = reinterpret_cast<__nv_bfloat16*>(C);
  p.ldc = static_cast<int>(ldc);
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  p.ws = reinterpret_cast<float*>(ws);
  p.counters = reinterpret_cast<uint32_t*>(counters);
  const int stage_bytes = kW4WBytes + p.BT * kW4BK * 2 + kW4SBytes + kW4ZBytes;
  int stages = (227 * 1024 - 2048) / stage_bytes;
  if (stages > 12) stages = 12;
  p.stages = stages;
  const int smem_bytes = stages * stage_bytes + 1024 + 512;
  const int np = (N + 15) / 16 * 16, kp = (K + kW4BK - 1) / kW4BK * kW4BK;
  const int G = (K + group - 1) / group;
  CUtensorMap tw, tx, ts, tz;
  if (make_tmap_2d(&tw, Wq, np, kp / 2, kp / 2, kW4Tile, kW4BK / 2, CU_TENSOR_MAP_DATA_TYPE_UINT8, false)) return 1;
  if (make_tmap_2d(&tx, A, M, K, lda * 2, p.BT, 64, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16)) return 1;
  if (make_tmap_2d(&ts, scales, G, N, static_cast<uint64_t>(N) * 2, p.gps, kW4Tile, CU_TENSOR_MAP_DATA_TYPE_UINT16,
                   false)) return 1;
  if (make_tmap_2d(&tz, zeros, G, np, np, p.gps, kW4Tile, CU_TENSOR_MAP_DATA_TYPE_UINT8, false)) return 1;
  const int units = tiles * p.S;
  const int grid = units < sms ? units : sms;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (p.BT) {
    case 16: return launch_w4a16<16>(tw, tx, ts, tz, p, grid, smem_bytes, st);
    case 32: return launch_w4a16<32>(tw, tx, ts, tz, p, grid, smem_bytes, st);
    case 64: return launch_w4a16<64>(tw, tx, ts, tz, p, grid, smem_bytes, st);
    case 128: return launch_w4a16<128>(tw, tx, ts, tz, p, grid, smem_bytes, st);
    default: return launch_w4a16<256>(tw, tx, ts, tz, p, grid, smem_bytes, st);
  }
}
