// RMSNorm (+ fused residual add) and SiLU-gate for sm_90a.
//
// Memory-bound row kernels: 16-byte vector loads/stores, the row stays in registers between
// the reduction and the scale pass, one CTA per token row. They replace the reference's
// vLLM `_C.rms_norm` / `_C.fused_add_rms_norm` / `_C.silu_and_mul` binaries
// (gllm/layers/layernorm.py:28-43, gllm/layers/activation.py:12).
#include "../common/host_utils.h"
#include "../common/ptx.cuh"

namespace b200 {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_sum(v);
  if (lane == 0) red[warp] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  float t = (lane < nw) ? red[lane] : 0.f;
  t = warp_sum(t);
  return t;
}

// NV = 16-byte vectors per thread.
template <int NV, bool kAdd>
__global__ void rmsnorm_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* residual,
                               const __nv_bfloat16* __restrict__ w, __nv_bfloat16* out,
                               __nv_bfloat16* residual_out, int H, int64_t ldx, float eps) {
  __shared__ float red[32];
  griddep_launch();  // let the next kernel (usually a GEMM) start its prologue + weight prefetch now
  griddep_wait();    // ... while this one waits for its own producer to finish
  const int row = blockIdx.x;
  const int nvec = H >> 3;
  const __nv_bfloat16* xr = x + static_cast<size_t>(row) * ldx;
  float v[NV][8];
  float ss = 0.f;
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const int i = threadIdx.x + j * blockDim.x;
    if (i < nvec) {
      uint4 a = *reinterpret_cast<const uint4*>(xr + i * 8);
      float2 f0 = unpack_bf16(a.x), f1 = unpack_bf16(a.y), f2 = unpack_bf16(a.z), f3 = unpack_bf16(a.w);
      v[j][0] = f0.x; v[j][1] = f0.y; v[j][2] = f1.x; v[j][3] = f1.y;
      v[j][4] = f2.x; v[j][5] = f2.y; v[j][6] = f3.x; v[j][7] = f3.y;
      if constexpr (kAdd) {
        uint4 r = *reinterpret_cast<const uint4*>(residual + static_cast<size_t>(row) * H + i * 8);
        float2 r0 = unpack_bf16(r.x), r1 = unpack_bf16(r.y), r2 = unpack_bf16(r.z), r3 = unpack_bf16(r.w);
        v[j][0] += r0.x; v[j][1] += r0.y; v[j][2] += r1.x; v[j][3] += r1.y;
        v[j][4] += r2.x; v[j][5] += r2.y; v[j][6] += r3.x; v[j][7] += r3.y;
        uint4 o;
        o.x = pack_bf16(v[j][0], v[j][1]); o.y = pack_bf16(v[j][2], v[j][3]);
        o.z = pack_bf16(v[j][4], v[j][5]); o.w = pack_bf16(v[j][6], v[j][7]);
        *reinterpret_cast<uint4*>(residual_out + static_cast<size_t>(row) * H + i * 8) = o;
        // the normalised value is computed from the bf16-rounded sum (matches the reference,
        // which re-reads the residual it just stored)
        float2 q0 = unpack_bf16(o.x), q1 = unpack_bf16(o.y), q2 = unpack_bf16(o.z), q3 = unpack_bf16(o.w);
        v[j][0] = q0.x; v[j][1] = q0.y; v[j][2] = q1.x; v[j][3] = q1.y;
        v[j][4] = q2.x; v[j][5] = q2.y; v[j][6] = q3.x; v[j][7] = q3.y;
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) ss += v[j][e] * v[j][e];
    }
  }
  ss = block_sum(ss, red);
  const float inv = rsqrtf(ss / static_cast<float>(H) + eps);
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const int i = threadIdx.x + j * blockDim.x;
    if (i < nvec) {
      uint4 wv = *reinterpret_cast<const uint4*>(w + i * 8);
      float2 w0 = unpack_bf16(wv.x), w1 = unpack_bf16(wv.y), w2 = unpack_bf16(wv.z), w3 = unpack_bf16(wv.w);
      uint4 o;
      o.x = pack_bf16(v[j][0] * inv * w0.x, v[j][1] * inv * w0.y);
      o.y = pack_bf16(v[j][2] * inv * w1.x, v[j][3] * inv * w1.y);
      o.z = pack_bf16(v[j][4] * inv * w2.x, v[j][5] * inv * w2.y);
      o.w = pack_bf16(v[j][6] * inv * w3.x, v[j][7] * inv * w3.y);
      *reinterpret_cast<uint4*>(out + static_cast<size_t>(row) * H + i * 8) = o;
    }
  }
}

__global__ void silu_and_mul_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ out,
                                    int I, int64_t ldx) {
  const int row = blockIdx.y;
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (i >= I) return;
  const __nv_bfloat16* xr = x + static_cast<size_t>(row) * ldx;
  uint4 g = ld_nc_v4(xr + i);
  uint4 u = ld_nc_v4(xr + I + i);
  uint32_t gg[4] = {g.x, g.y, g.z, g.w}, uu[4] = {u.x, u.y, u.z, u.w}, oo[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    float2 a = unpack_bf16(gg[e]), b = unpack_bf16(uu[e]);
    oo[e] = pack_bf16(a.x / (1.f + __expf(-a.x)) * b.x, a.y / (1.f + __expf(-a.y)) * b.y);
  }
  *reinterpret_cast<uint4*>(out + static_cast<size_t>(row) * I + i) = make_uint4(oo[0], oo[1], oo[2], oo[3]);
}

// out[t, :] = table[ids[t] - vocab_start, :] if the id is in [vocab_start, vocab_end) else 0
__global__ void embedding_kernel(const int32_t* __restrict__ ids, const __nv_bfloat16* __restrict__ table,
                                 __nv_bfloat16* __restrict__ out, int H, int vocab_start, int vocab_end) {
  const int t = blockIdx.x;
  const int id = ids[t];
  const bool ok = id >= vocab_start && id < vocab_end;
  const __nv_bfloat16* src = table + static_cast<size_t>(ok ? id - vocab_start : 0) * H;
  for (int i = threadIdx.x * 8; i < H; i += blockDim.x * 8) {
    uint4 v = ok ? *reinterpret_cast<const uint4*>(src + i) : make_uint4(0, 0, 0, 0);
    *reinterpret_cast<uint4*>(out + static_cast<size_t>(t) * H + i) = v;
  }
}

// out[i, :] = src[idx[i], :]
__global__ void gather_rows_kernel(const __nv_bfloat16* __restrict__ src, const int32_t* __restrict__ idx,
                                   __nv_bfloat16* __restrict__ out, int H) {
  const int t = blockIdx.x;
  const __nv_bfloat16* s = src + static_cast<size_t>(idx[t]) * H;
  for (int i = threadIdx.x * 8; i < H; i += blockDim.x * 8) {
    *reinterpret_cast<uint4*>(out + static_cast<size_t>(t) * H + i) = *reinterpret_cast<const uint4*>(s + i);
  }
}

}  // namespace b200

using namespace b200;

// residual == nullptr: out = rmsnorm(x) * w
// residual != nullptr: residual_out = x + residual ; out = rmsnorm(residual_out) * w
GLLM_EXPORT int gllm_rmsnorm(const void* x, const void* residual, const void* w, void* out,
                             void* residual_out, int T, int H, int64_t ldx, float eps, void* stream) {
  if (T <= 0) return 0;
  if (H % 8 != 0) {
    fprintf(stderr, "[gllm_b200] rmsnorm: H must be a multiple of 8\n");
    return 1;
  }
  const int nvec = H / 8;
  int threads = ((nvec + 31) / 32) * 32;
  int nv = 1;
  while (threads > 1024) {
    nv *= 2;
    threads = (((nvec + nv - 1) / nv + 31) / 32) * 32;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  auto X = reinterpret_cast<const __nv_bfloat16*>(x);
  auto R = reinterpret_cast<const __nv_bfloat16*>(residual);
  auto W = reinterpret_cast<const __nv_bfloat16*>(w);
  auto O = reinterpret_cast<__nv_bfloat16*>(out);
  auto RO = reinterpret_cast<__nv_bfloat16*>(residual_out);
#define LAUNCH(NV_)                                                                              \
  if (R != nullptr)                                                                              \
    CUDA_CHECK_RET(launch_pdl(rmsnorm_kernel<NV_, true>, dim3(T), dim3(threads), 0, st, X, R, W, O, RO, H, ldx, eps)); \
  else                                                                                           \
    CUDA_CHECK_RET(launch_pdl(rmsnorm_kernel<NV_, false>, dim3(T), dim3(threads), 0, st, X, R, W, O, RO, H, ldx, eps));
  if (nv == 1) { LAUNCH(1) }
  else if (nv == 2) { LAUNCH(2) }
  else if (nv == 4) { LAUNCH(4) }
  else {
    fprintf(stderr, "[gllm_b200] rmsnorm: H=%d too large\n", H);
    return 1;
  }
#undef LAUNCH
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

GLLM_EXPORT int gllm_silu_and_mul(const void* x, void* out, int T, int I, int64_t ldx, void* stream) {
  if (T <= 0) return 0;
  if (I % 8 != 0) return 1;
  dim3 grid((I / 8 + 255) / 256, T);
  silu_and_mul_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<__nv_bfloat16*>(out), I, ldx);
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

GLLM_EXPORT int gllm_embedding(const void* ids, const void* table, void* out, int T, int H,
                               int vocab_start, int vocab_end, void* stream) {
  if (T <= 0) return 0;
  embedding_kernel<<<T, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const int32_t*>(ids), reinterpret_cast<const __nv_bfloat16*>(table),
      reinterpret_cast<__nv_bfloat16*>(out), H, vocab_start, vocab_end);
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

GLLM_EXPORT int gllm_gather_rows(const void* src, const void* idx, void* out, int n, int H, void* stream) {
  if (n <= 0) return 0;
  gather_rows_kernel<<<n, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(src), reinterpret_cast<const int32_t*>(idx),
      reinterpret_cast<__nv_bfloat16*>(out), H);
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}
