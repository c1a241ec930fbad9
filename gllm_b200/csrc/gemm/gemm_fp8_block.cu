// Block-scaled FP8 (e4m3) GEMM for sm_90a, DeepSeek-V3 / Qwen3-FP8 checkpoint semantics
// (reference: gllm/layers/quantization/fp8.py:54-250 — Triton w8a8_block_fp8_matmul):
//
//   C[M,N] = sum_kb  (A8[M, kb] · W8[N, kb]^T) * a_s[M, kb] * w_s[N/128, kb]      (+ bias) -> bf16
//   A8: activations quantised per token per 128-wide K group (dynamic, amax/448), a_s fp32 [K/128, M]
//       (stored K-block-major so a warp's 32 rows read 32 consecutive floats)
//   W8: weights e4m3 [N, K] with fp32 scales per 128x128 block, w_s [N/128, K/128]
//
// The checkpoint scales are arbitrary fp32 values, so each 128-deep K block is multiplied by
// `wgmma.mma_async ... e4m3.e4m3` into its own register accumulator (4 MMAs of K=32, the first one
// overwriting) and then promoted: acc += partial * a_s[row] * w_s[tile] in fp32 registers. Two consumer
// warpgroups own 64 rows each of the 128 x 128 tile. Same TMA (SWIZZLE_128B, 128 fp8 = one 128-byte row) /
// mbarrier ring as gemm_bf16.cu.
//
// The same kernel, instantiated with kW8A8 = true, is the large-M W8A8 GEMM of per-channel / per-tensor FP8
// checkpoints: a_s fp32 [M] (one scale per token), w_s fp32 [N] (one per output channel). Each 128-deep K block is
// promoted unscaled (acc += partial, since wgmma's e4m3 accumulator keeps fewer bits than fp32) and the epilogue
// applies y = bf16(acc * a_s[m] * w_s[n] + bias[n]). K only needs to be a multiple of 16 (the TMA row pitch): the
// last K block is zero-filled by TMA.
//
// Also here: the dynamic per-token-group activation quantiser (reference fp8.py:354-552) and the per-token one of
// the W8A8 path.
#include <cuda_fp8.h>
#include <string.h>

#include "../common/host_utils.h"
#include "../common/ptx.cuh"

namespace b200 {

static constexpr int kFBM = 128, kFBN = 128, kFBK = 128;  // K block = 128 fp8 = 128 B
static constexpr int kFStages = 6;
static constexpr int kFThreads = 384;  // warpgroup 0: TMA producer, warpgroups 1-2: MMA + epilogue

struct Fp8Params {
  int M, N, K;
  __nv_bfloat16* C;
  int ldc;
  const float* a_s;  // [K/128, M]  (W8A8: [M])
  int lda_s;         // = M (row pitch of a_s)
  const float* w_s;  // [N/128, K/128]  (grouped: [E][N/64][K/128], one scale row per 64 weight rows; W8A8: [N])
  const __nv_bfloat16* bias;
  // grouped (MoE) mode: M tile t multiplies the e4m3 slab of expert tile_expert[t]; the weight scales are
  // stored per 64-row half tile so a [64 gate | 64 up] interleaved tile can carry two different block scales
  const int32_t* tile_expert;
  const int32_t* num_m_tiles_ptr;
  int n_per_expert;      // rows of one expert slab
  int64_t ws_stride_e;   // floats per expert in w_s
  int silu;              // 1: out[:, j] = silu(acc[j]) * acc[64 + j]  (64 output columns per tile)
};

template <bool kW8A8>
__global__ void __launch_bounds__(kFThreads, 1)
gemm_fp8_block_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                      const Fp8Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int kABytes = kFBM * kFBK, kBBytes = kFBN * kFBK, kStageBytes = kABytes + kBBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kFStages * kStageBytes);
  uint64_t* empty_bar = full_bar + kFStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool grouped = p.tile_expert != nullptr;
  const int num_m = p.num_m_tiles_ptr != nullptr ? min(*p.num_m_tiles_ptr, (p.M + kFBM - 1) / kFBM)
                                                 : (p.M + kFBM - 1) / kFBM;
  const int num_n = (p.N + kFBN - 1) / kFBN;
  const int num_tiles = num_m * num_n;
  const int num_kb = kW8A8 ? (p.K + kFBK - 1) / kFBK : p.K / kFBK;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int i = 0; i < kFStages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 8); }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp < 4) {
    regs_dealloc<40>();
    if (warp == 0 && lane == 0) {
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m0 = (tile % num_m) * kFBM, n0 = (tile / num_m) * kFBN;
        const int b_row_off = grouped ? p.tile_expert[tile % num_m] * p.n_per_expert : 0;
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const int s = it % kFStages;
          mbar_wait(&empty_bar[s], ((it / kFStages) & 1) ^ 1);
          uint8_t* sa = smem + s * kStageBytes;
          mbar_expect_tx(&full_bar[s], kStageBytes);
          tma_load_2d(sa, &tmap_a, &full_bar[s], kb * kFBK, m0, kEvictNormal);
          tma_load_2d(sa + kABytes, &tmap_b, &full_bar[s], kb * kFBK, n0 + b_row_off, kEvictNormal);
        }
      }
    }
  } else {
    regs_alloc<232>();
    const int ct = threadIdx.x - 128;
    const int g = ct >> 7, wq = (ct >> 5) & 3;
    const int r_in = 64 * g + 16 * wq + (lane >> 2);   // rows r_in and r_in + 8 of the tile
    const int cq = 2 * (lane & 3);                     // columns 8 j + cq + {0, 1}
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m0 = (tile % num_m) * kFBM, n0 = (tile / num_m) * kFBN;
      const int row0 = m0 + r_in, row1 = row0 + 8;
      float acc[kFBN / 2], part[kFBN / 2];
#pragma unroll
      for (int i = 0; i < kFBN / 2; ++i) acc[i] = 0.f;
      for (int kb = 0; kb < num_kb; ++kb, ++it) {
        const int s = it % kFStages;
        mbar_wait(&full_bar[s], (it / kFStages) & 1);
        const uint32_t a_addr = smem_u32(smem + s * kStageBytes);
        const uint64_t da = make_sw128_kmajor_desc(a_addr + g * (64 * 128));
        const uint64_t db = make_sw128_kmajor_desc(a_addr + kABytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kFBK / 32; ++k)  // K = 32 for 8-bit operands: +32 B per step
          wgmma_e4m3_ss<kFBN>(part, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), k > 0 ? 1u : 0u);
        wgmma_commit();
        if constexpr (kW8A8) {
          wgmma_wait<0>();
          reg_fence(part);
          if (lane == 0) mbar_arrive(&empty_bar[s]);
#pragma unroll
          for (int i = 0; i < kFBN / 2; ++i) acc[i] += part[i];
          continue;
        }
        // scales of this K block load while the tensor core runs
        const float sa0 = row0 < p.M ? p.a_s[static_cast<size_t>(kb) * p.lda_s + row0] : 0.f;
        const float sa1 = row1 < p.M ? p.a_s[static_cast<size_t>(kb) * p.lda_s + row1] : 0.f;
        float sw, sw_hi;
        if (grouped) {
          const float* ws = p.w_s + static_cast<size_t>(p.tile_expert[tile % num_m]) * p.ws_stride_e +
                            static_cast<size_t>(n0 / 64) * num_kb + kb;
          sw = ws[0];
          sw_hi = ws[num_kb];
        } else {
          sw = sw_hi = p.w_s[static_cast<size_t>(n0 / kFBN) * num_kb + kb];
        }
        wgmma_wait<0>();
        reg_fence(part);
        if (lane == 0) mbar_arrive(&empty_bar[s]);
#pragma unroll
        for (int j = 0; j < kFBN / 8; ++j) {
          const float w = j < 8 ? sw : sw_hi;   // columns < 64 / >= 64
          acc[4 * j] = fmaf(part[4 * j], sa0 * w, acc[4 * j]);
          acc[4 * j + 1] = fmaf(part[4 * j + 1], sa0 * w, acc[4 * j + 1]);
          acc[4 * j + 2] = fmaf(part[4 * j + 2], sa1 * w, acc[4 * j + 2]);
          acc[4 * j + 3] = fmaf(part[4 * j + 3], sa1 * w, acc[4 * j + 3]);
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = h ? row1 : row0;
        if (row >= p.M) continue;
        __nv_bfloat16* crow = p.C + static_cast<size_t>(row) * p.ldc;
        if constexpr (kW8A8) {
          const float sx = p.a_s[row];
#pragma unroll
          for (int j = 0; j < kFBN / 8; ++j) {
            const int col = n0 + 8 * j + cq;
            if (col < p.N) {
              const float2 sw = *reinterpret_cast<const float2*>(p.w_s + col);
              float f0 = __fmul_rn(__fmul_rn(acc[4 * j + 2 * h], sx), sw.x);
              float f1 = __fmul_rn(__fmul_rn(acc[4 * j + 2 * h + 1], sx), sw.y);
              if (p.bias != nullptr) {
                const float2 bv = unpack_bf16(*reinterpret_cast<const uint32_t*>(p.bias + col));
                f0 = __fadd_rn(f0, bv.x); f1 = __fadd_rn(f1, bv.y);
              }
              *reinterpret_cast<uint32_t*>(crow + col) = pack_bf16(f0, f1);
            }
          }
        } else if (p.silu) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int col = n0 / 2 + 8 * j + cq;
            if (col < p.N / 2) {
              float f[2];
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const float gv = acc[4 * j + 2 * h + e];
                f[e] = gv / (1.0f + __expf(-gv)) * acc[4 * (j + 8) + 2 * h + e];
              }
              *reinterpret_cast<uint32_t*>(crow + col) = pack_bf16(f[0], f[1]);
            }
          }
        } else {
#pragma unroll
          for (int j = 0; j < kFBN / 8; ++j) {
            const int col = n0 + 8 * j + cq;
            if (col < p.N) {
              float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
              if (p.bias != nullptr) {
                const float2 bv = unpack_bf16(*reinterpret_cast<const uint32_t*>(p.bias + col));
                f0 += bv.x; f1 += bv.y;
              }
              *reinterpret_cast<uint32_t*>(crow + col) = pack_bf16(f0, f1);
            }
          }
        }
      }
    }
  }
}

// dynamic per-token-group (128) quantisation: x bf16 [M,K] -> q e4m3 [M,K], scales fp32 [K/128, M]
__global__ void fp8_quant_group_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, __nv_fp8_e4m3* __restrict__ q,
                                       float* __restrict__ scales, int M, int K) {
  // one warp per (row, group): 32 lanes x 4 elements = 128
  const int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int groups = K / 128;
  if (wid >= M * groups) return;
  const int row = wid / groups, g = wid % groups;
  const __nv_bfloat16* src = x + static_cast<size_t>(row) * ldx + g * 128 + lane * 4;
  const uint2 raw = *reinterpret_cast<const uint2*>(src);
  const float2 a = unpack_bf16(raw.x), b = unpack_bf16(raw.y);
  float amax = fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(b.x), fabsf(b.y)));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  amax = fmaxf(amax, 1e-10f);
  const float scale = amax / 448.f;
  const float inv = 1.f / scale;
  __nv_fp8_e4m3 o4[4] = {__nv_fp8_e4m3(a.x * inv), __nv_fp8_e4m3(a.y * inv), __nv_fp8_e4m3(b.x * inv),
                         __nv_fp8_e4m3(b.y * inv)};
  *reinterpret_cast<uint32_t*>(q + static_cast<size_t>(row) * K + g * 128 + lane * 4) = *reinterpret_cast<uint32_t*>(o4);
  if (lane == 0) scales[static_cast<size_t>(g) * M + row] = scale;
}

// Per-token quantisation of the W8A8 path: x bf16 [M, K] (row stride ldx) -> q e4m3 [M, K] contiguous, s fp32 [M].
// One CTA per row. Dynamic (static_scale == nullptr): s = max(amax |x|, 1e-10) / 448 and q = e4m3_rn(x * (1 / s)),
// the reciprocal taken first. Static: s = *static_scale and q = e4m3_rn(clamp(x / s, +-448)). Every division is
// correctly rounded (the library builds with fast math), so ops.ref.fp8_quant_token gives the same bits.
static constexpr int kQThreads = 256;

__device__ __forceinline__ __nv_fp8_e4m3 to_e4m3(float v) {
  __nv_fp8_e4m3 r;
  r.__x = __nv_cvt_float_to_fp8(v, __NV_SATFINITE, __NV_E4M3);
  return r;
}

template <bool kVec>   // kVec: K, ldx and x 16-byte aligned: 8 elements per load
__global__ void __launch_bounds__(kQThreads)
fp8_quant_token_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, __nv_fp8_e4m3* __restrict__ q,
                       float* __restrict__ scales, const float* __restrict__ static_scale, int K) {
  __shared__ float red[kQThreads / 32];
  const int row = blockIdx.x;
  const __nv_bfloat16* src = x + static_cast<size_t>(row) * ldx;
  __nv_fp8_e4m3* dst = q + static_cast<size_t>(row) * K;
  float s;
  if (static_scale != nullptr) {
    s = *static_scale;
  } else {
    float amax = 0.f;
    if constexpr (kVec) {
      for (int k = threadIdx.x * 8; k < K; k += kQThreads * 8) {
        const uint4 raw = *reinterpret_cast<const uint4*>(src + k);
        const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = unpack_bf16(w[i]);
          amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));
        }
      }
    } else {
      for (int k = threadIdx.x; k < K; k += kQThreads) amax = fmaxf(amax, fabsf(__bfloat162float(src[k])));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = amax;
    __syncthreads();
    amax = red[0];
#pragma unroll
    for (int i = 1; i < kQThreads / 32; ++i) amax = fmaxf(amax, red[i]);
    s = __fdiv_rn(fmaxf(amax, 1e-10f), 448.f);
  }
  const bool dyn = static_scale == nullptr;
  const float inv = __frcp_rn(s);
  auto quant = [&](float v) {
    return to_e4m3(dyn ? __fmul_rn(v, inv) : fminf(fmaxf(__fdiv_rn(v, s), -448.f), 448.f));
  };
  if constexpr (kVec) {
    for (int k = threadIdx.x * 8; k < K; k += kQThreads * 8) {
      const uint4 raw = *reinterpret_cast<const uint4*>(src + k);
      const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
      __nv_fp8_e4m3 o[8];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = unpack_bf16(w[i]);
        o[2 * i] = quant(f.x);
        o[2 * i + 1] = quant(f.y);
      }
      *reinterpret_cast<uint2*>(dst + k) = *reinterpret_cast<const uint2*>(o);
    }
  } else {
    for (int k = threadIdx.x; k < K; k += kQThreads) dst[k] = quant(__bfloat162float(src[k]));
  }
  if (threadIdx.x == 0) scales[row] = s;
}

}  // namespace b200

using namespace b200;

GLLM_EXPORT int gllm_fp8_quant_group(const void* x, int64_t ldx, void* q, void* scales, int M, int K, void* stream) {
  if (M <= 0) return 0;
  if (K % 128 != 0) return 1;
  const int warps = M * (K / 128);
  fp8_quant_group_kernel<<<(warps * 32 + 255) / 256, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), ldx, reinterpret_cast<__nv_fp8_e4m3*>(q),
      reinterpret_cast<float*>(scales), M, K);
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

// A8 [M,K] e4m3 contiguous, a_s [K/128, M]; W8 [N,K] e4m3 contiguous, w_s [ceil(N/128), K/128]
GLLM_EXPORT int gllm_gemm_fp8_block(const void* A8, const void* a_s, const void* W8, const void* w_s, void* C,
                                    int64_t ldc, int M, int N, int K, const void* bias, void* stream) {
  if (M <= 0 || N <= 0) return 0;
  if (K % 128 != 0 || N % 8 != 0) {
    fprintf(stderr, "[gllm_b200] gemm_fp8_block: K %% 128 and N %% 8 required\n");
    return 1;
  }
  CUtensorMap ta, tb;
  if (make_tmap_2d(&ta, A8, M, K, K, kFBM, kFBK, CU_TENSOR_MAP_DATA_TYPE_UINT8)) return 1;
  if (make_tmap_2d(&tb, W8, N, K, K, kFBN, kFBK, CU_TENSOR_MAP_DATA_TYPE_UINT8)) return 1;
  Fp8Params p;
  p.M = M; p.N = N; p.K = K;
  p.C = reinterpret_cast<__nv_bfloat16*>(C);
  p.ldc = static_cast<int>(ldc);
  p.a_s = reinterpret_cast<const float*>(a_s);
  p.lda_s = M;
  p.w_s = reinterpret_cast<const float*>(w_s);
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  p.tile_expert = nullptr; p.num_m_tiles_ptr = nullptr; p.n_per_expert = 0; p.ws_stride_e = 0; p.silu = 0;
  constexpr int smem_bytes = kFStages * (kFBM * kFBK + kFBN * kFBK) + 1024 + 256;
  static PerDeviceOnce configured;
  if (configured.need()) {
    CUDA_CHECK_RET(cudaFuncSetAttribute(gemm_fp8_block_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    configured.done();
  }
  const int tiles = ((M + kFBM - 1) / kFBM) * ((N + kFBN - 1) / kFBN);
  const int grid = tiles < num_sms() ? tiles : num_sms();
  gemm_fp8_block_kernel<false><<<grid, kFThreads, smem_bytes, reinterpret_cast<cudaStream_t>(stream)>>>(ta, tb, p);
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

// Grouped (MoE) block-scaled fp8 GEMM: A8 [max_tiles*128, K] e4m3 (expert-sorted, 128-row tiles), a_s
// [K/128, max_tiles*128]; W8 [E, N, K] e4m3, w_s [E, N/64, K/128] (one scale row per 64 weight rows);
// epi 1 = SiLU gate on [64 gate | 64 up] interleaved tiles -> C [rows, N/2].
GLLM_EXPORT int gllm_moe_grouped_gemm_fp8(const void* A8, const void* a_s, const void* W8, const void* w_s, void* C,
                                          int64_t ldc, int max_tiles, int N, int K, int E, const void* tile_expert,
                                          const void* num_tiles_ptr, int epi, void* stream) {
  if (max_tiles <= 0) return 0;
  if (K % 128 != 0 || N % 128 != 0) {
    fprintf(stderr, "[gllm_b200] moe_grouped_gemm_fp8: K %% 128 and N %% 128 required\n");
    return 1;
  }
  const int M = max_tiles * kFBM;
  CUtensorMap ta, tb;
  if (make_tmap_2d(&ta, A8, M, K, K, kFBM, kFBK, CU_TENSOR_MAP_DATA_TYPE_UINT8)) return 1;
  if (make_tmap_2d(&tb, W8, static_cast<uint64_t>(E) * N, K, K, kFBN, kFBK, CU_TENSOR_MAP_DATA_TYPE_UINT8)) return 1;
  Fp8Params p;
  p.M = M; p.N = N; p.K = K;
  p.C = reinterpret_cast<__nv_bfloat16*>(C);
  p.ldc = static_cast<int>(ldc);
  p.a_s = reinterpret_cast<const float*>(a_s);
  p.lda_s = M;
  p.w_s = reinterpret_cast<const float*>(w_s);
  p.bias = nullptr;
  p.tile_expert = reinterpret_cast<const int32_t*>(tile_expert);
  p.num_m_tiles_ptr = reinterpret_cast<const int32_t*>(num_tiles_ptr);
  p.n_per_expert = N;
  p.ws_stride_e = static_cast<int64_t>(N / 64) * (K / 128);
  p.silu = epi == 1 ? 1 : 0;
  constexpr int smem_bytes = kFStages * (kFBM * kFBK + kFBN * kFBK) + 1024 + 256;
  CUDA_CHECK_RET(cudaFuncSetAttribute(gemm_fp8_block_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
  const int tiles = max_tiles * (N / kFBN);
  const int grid = tiles < num_sms() ? tiles : num_sms();
  gemm_fp8_block_kernel<false><<<grid, kFThreads, smem_bytes, reinterpret_cast<cudaStream_t>(stream)>>>(ta, tb, p);
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

// x bf16 [M, K] (row stride ldx) -> q e4m3 [M, K] contiguous, s fp32 [M]; static_scale: fp32 scalar or null (dynamic)
GLLM_EXPORT int gllm_fp8_quant_token(const void* x, int64_t ldx, void* q, void* scales, const void* static_scale, int M,
                                     int K, void* stream) {
  if (M <= 0) return 0;
  const bool vec = K % 8 == 0 && ldx % 8 == 0 && reinterpret_cast<uintptr_t>(x) % 16 == 0;
  auto kern = vec ? fp8_quant_token_kernel<true> : fp8_quant_token_kernel<false>;
  kern<<<M, kQThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), ldx, reinterpret_cast<__nv_fp8_e4m3*>(q),
      reinterpret_cast<float*>(scales), reinterpret_cast<const float*>(static_scale), K);
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

// Large-M W8A8 GEMM: A8 [M, K] e4m3 contiguous with per-token scales a_s fp32 [M]; W8 [N, K] e4m3 contiguous with
// per-channel scales w_s fp32 [N]. C[m, n] = bf16(acc * a_s[m] * w_s[n] + bias[n]).
GLLM_EXPORT int gllm_gemm_fp8_w8a8(const void* A8, const void* a_s, const void* W8, const void* w_s, void* C,
                                   int64_t ldc, int M, int N, int K, const void* bias, void* stream) {
  if (M <= 0 || N <= 0) return 0;
  if (K % 16 != 0 || N % 8 != 0 || ldc % 2 != 0) {
    fprintf(stderr, "[gllm_b200] gemm_fp8_w8a8: K %% 16, N %% 8 and even ldc required (M=%d N=%d K=%d)\n", M, N, K);
    return 1;
  }
  CUtensorMap ta, tb;
  if (make_tmap_2d(&ta, A8, M, K, K, kFBM, kFBK, CU_TENSOR_MAP_DATA_TYPE_UINT8)) return 1;
  if (make_tmap_2d(&tb, W8, N, K, K, kFBN, kFBK, CU_TENSOR_MAP_DATA_TYPE_UINT8)) return 1;
  Fp8Params p;
  memset(&p, 0, sizeof(p));
  p.M = M; p.N = N; p.K = K;
  p.C = reinterpret_cast<__nv_bfloat16*>(C);
  p.ldc = static_cast<int>(ldc);
  p.a_s = reinterpret_cast<const float*>(a_s);
  p.lda_s = M;
  p.w_s = reinterpret_cast<const float*>(w_s);
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  constexpr int smem_bytes = kFStages * (kFBM * kFBK + kFBN * kFBK) + 1024 + 256;
  static PerDeviceOnce configured;
  if (configured.need()) {
    CUDA_CHECK_RET(cudaFuncSetAttribute(gemm_fp8_block_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        smem_bytes));
    configured.done();
  }
  const int tiles = ((M + kFBM - 1) / kFBM) * ((N + kFBN - 1) / kFBN);
  const int grid = tiles < num_sms() ? tiles : num_sms();
  gemm_fp8_block_kernel<true><<<grid, kFThreads, smem_bytes, reinterpret_cast<cudaStream_t>(stream)>>>(ta, tb, p);
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}
