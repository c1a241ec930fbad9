// Multi-LoRA kernels for sm_90a: the per-row adapter delta of a linear layer, y += (x · Aᵀ) · Bᵀ, where every
// token row may use a different adapter (or none).
//
// Rows are grouped per adapter by a per-batch CSR that the host builds once per step and every layer reuses:
//   slots[S]      adapter slot of group g (index into the stacked [L, ...] weights)
//   row_off[S+1]  rows[row_off[g] .. row_off[g+1]) are the token rows of group g
//   rows[T]       every token row once: the adapter groups first, then the rows without an adapter
// A CTA works on one (group, tile) pair, so an adapter's A and B tiles are read once per launch and per row tile of
// that adapter, never once per row. Rows without an adapter do no work in shrink / expand-add.
//
//   lora_shrink          U[T, M] = x[T, K] · A_slot(row)[M, K]ᵀ     M = m·r for the m modules that share x.
//                        mma.sync m16n8k16 (bf16 in, fp32 accumulate) over 64-row x 64-column tiles of a group's
//                        rows, split over K so a decode-sized launch still spreads A's bytes over the SMs. Each K
//                        slice stores its partial sums; a second kernel adds them in slice order, so U is the same
//                        bits on every run, eager or CUDA graph (without a split, the tile writes U directly).
//   lora_expand_add      y[T, N] += U_m · B_m,slotᵀ in place. Column n belongs to module m = (n >= n1) + (n >= n2)
//                        and reads U[:, m·r : (m+1)·r]. fp32 accumulation, one bf16 rounding of y.
//   lora_expand_silu_mul gate/up pre-activations [T, 2I] in the 128-row interleaved layout of the fused SiLU-gate
//                        GEMM (ops.ref.interleave_gate_up) -> out[T, I] = SiLU(gate + dg) · (up + du); the rows
//                        without an adapter (the last group, which also covers CUDA-graph padding rows) get
//                        SiLU(gate) · up.
#include "../common/host_utils.h"
#include "../common/ptx.cuh"

namespace b200 {
namespace lora {

constexpr int kMaxRank = 64;

// ---------------------------------------------------------------------------------------------------------------
// shrink
// ---------------------------------------------------------------------------------------------------------------
constexpr int SBM = 64, SBN = 64, SBK = 32, SPAD = 8;   // padded smem rows (80 B): conflict-free fragment loads

__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// grid (m_tiles * k_splits, row tiles, groups), 128 threads: warp w owns rows [16w, 16w + 16) of the tile.
// K slice ks stores its partial sums into out + ks * T * M (row-major [T, M]).
__global__ void __launch_bounds__(128) shrink_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx,
                                                     const __nv_bfloat16* __restrict__ A, float* __restrict__ out,
                                                     int T, int K, int M, int k_chunk, int m_tiles,
                                                     const int32_t* __restrict__ slots,
                                                     const int32_t* __restrict__ row_off,
                                                     const int32_t* __restrict__ rows) {
  __shared__ __align__(16) __nv_bfloat16 xs[SBM][SBK + SPAD];
  __shared__ __align__(16) __nv_bfloat16 as[SBN][SBK + SPAD];
  __shared__ int32_t rid[SBM];
  const int g = blockIdx.z;
  const int r0 = row_off[g] + blockIdx.y * SBM, r1 = row_off[g + 1];
  if (r0 >= r1) return;
  const int nrows = min(SBM, r1 - r0);
  const int mt = blockIdx.x % m_tiles, ks = blockIdx.x / m_tiles;
  const int n0 = mt * SBN;
  const int k0 = ks * k_chunk, k1 = min(K, k0 + k_chunk);
  if (k0 >= k1) return;
  const __nv_bfloat16* Aslot = A + static_cast<size_t>(slots[g]) * M * K;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, gq = lane >> 2, tq = lane & 3;
  if (tid < SBM) rid[tid] = tid < nrows ? rows[r0 + tid] : -1;
  __syncthreads();
  float acc[SBN / 8][4];
#pragma unroll
  for (int j = 0; j < SBN / 8; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
  for (int kb = k0; kb < k1; kb += SBK) {
    // 64 rows x 4 chunks of 8 bf16, for each operand: two chunks per thread
#pragma unroll
    for (int it = 0; it < 2; ++it) {
      const int q = tid + it * 128, row = q >> 2, c = (q & 3) * 8, k = kb + c;
      uint4 vx = make_uint4(0, 0, 0, 0), va = make_uint4(0, 0, 0, 0);
      const int rr = rid[row];
      if (rr >= 0 && k < k1) vx = *reinterpret_cast<const uint4*>(x + static_cast<size_t>(rr) * ldx + k);
      if (n0 + row < M && k < k1) va = ld_nc_v4(Aslot + static_cast<size_t>(n0 + row) * K + k);
      *reinterpret_cast<uint4*>(&xs[row][c]) = vx;
      *reinterpret_cast<uint4*>(&as[row][c]) = va;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < SBK; kk += 16) {
      uint32_t a[4];
      const int ar = warp * 16 + gq;
      a[0] = *reinterpret_cast<const uint32_t*>(&xs[ar][kk + 2 * tq]);
      a[1] = *reinterpret_cast<const uint32_t*>(&xs[ar + 8][kk + 2 * tq]);
      a[2] = *reinterpret_cast<const uint32_t*>(&xs[ar][kk + 2 * tq + 8]);
      a[3] = *reinterpret_cast<const uint32_t*>(&xs[ar + 8][kk + 2 * tq + 8]);
#pragma unroll
      for (int j = 0; j < SBN / 8; ++j) {
        const uint32_t b0 = *reinterpret_cast<const uint32_t*>(&as[8 * j + gq][kk + 2 * tq]);
        const uint32_t b1 = *reinterpret_cast<const uint32_t*>(&as[8 * j + gq][kk + 2 * tq + 8]);
        mma16816(acc[j], a, b0, b1);
      }
    }
    __syncthreads();
  }
  const int ra = rid[warp * 16 + gq], rb = rid[warp * 16 + gq + 8];
  float* P = out + static_cast<size_t>(ks) * T * M;
#pragma unroll
  for (int j = 0; j < SBN / 8; ++j) {
    const int col = n0 + 8 * j + 2 * tq;
    if (ra >= 0) {
      if (col < M) P[static_cast<size_t>(ra) * M + col] = acc[j][0];
      if (col + 1 < M) P[static_cast<size_t>(ra) * M + col + 1] = acc[j][1];
    }
    if (rb >= 0) {
      if (col < M) P[static_cast<size_t>(rb) * M + col] = acc[j][2];
      if (col + 1 < M) P[static_cast<size_t>(rb) * M + col + 1] = acc[j][3];
    }
  }
}

// U[row, c] = sum over K slices s = 0, 1, ... of P[s, row, c] for the adapter rows (rows[0 .. row_off[S])), 0 for
// every other row. rows[0 .. T) lists each of the T rows once.
__global__ void __launch_bounds__(256) shrink_reduce_kernel(const float* __restrict__ P, float* __restrict__ U, int T,
                                                            int M, int k_splits, int S,
                                                            const int32_t* __restrict__ row_off,
                                                            const int32_t* __restrict__ rows) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= T * M) return;
  const int i = idx / M, c = idx - i * M;
  const int row = rows[i];
  float v = 0.f;
  if (i < row_off[S]) {
    for (int s = 0; s < k_splits; ++s) v += P[(static_cast<size_t>(s) * T + row) * M + c];
  }
  U[static_cast<size_t>(row) * M + c] = v;
}

// ---------------------------------------------------------------------------------------------------------------
// expand
// ---------------------------------------------------------------------------------------------------------------
constexpr int EBN = 128, EROWS = 64, ECHUNK = 16;

// B rows [n0, n0 + EBN) of one adapter ([N, r] row-major, contiguous) -> dst[k * EBN + c] (fp32 or bf16)
template <typename TS>
__device__ __forceinline__ void load_b_tile(TS* dst, const __nv_bfloat16* B, int n0, int N, int r) {
  const int cpr = r >> 3;  // 16-byte chunks per B row
  for (int q = threadIdx.x; q < EBN * cpr; q += blockDim.x) {
    const int c = q / cpr, k0 = (q - c * cpr) * 8;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (n0 + c < N) v = ld_nc_v4(B + static_cast<size_t>(n0 + c) * r + k0);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = unpack_bf16(w[e]);
      dst[(k0 + 2 * e) * EBN + c] = static_cast<TS>(f.x);
      dst[(k0 + 2 * e + 1) * EBN + c] = static_cast<TS>(f.y);
    }
  }
}

// rows [i0, i0 + n) of a group -> us[i][0 .. width) from U (fp32, row stride ldu); rid[i] = token row
__device__ __forceinline__ void load_u_rows(float* us, int32_t* rid, const float* U, int64_t ldu, int width,
                                            const int32_t* rows, int i0, int n) {
  if (threadIdx.x < ECHUNK) rid[threadIdx.x] = threadIdx.x < n ? rows[i0 + threadIdx.x] : -1;
  __syncthreads();
  for (int q = threadIdx.x; q < ECHUNK * width; q += blockDim.x) {
    const int i = q / width, j = q - i * width;
    us[q] = i < n ? U[static_cast<size_t>(rid[i]) * ldu + j] : 0.f;
  }
  __syncthreads();
}

// grid (ceil(N / EBN), row tiles, groups), 256 threads: column c = tid % EBN, rows of parity tid / EBN.
__global__ void __launch_bounds__(256) expand_add_kernel(const float* __restrict__ U, int64_t ldu,
                                                         const __nv_bfloat16* __restrict__ B,
                                                         __nv_bfloat16* y, int64_t ldy, int N, int r, int n1, int n2,
                                                         int width, const int32_t* __restrict__ slots,
                                                         const int32_t* __restrict__ row_off,
                                                         const int32_t* __restrict__ rows) {
  __shared__ float bs[kMaxRank * EBN];
  __shared__ float us[ECHUNK * 3 * kMaxRank];
  __shared__ int32_t rid[ECHUNK];
  const int g = blockIdx.z;
  const int r0 = row_off[g] + blockIdx.y * EROWS, r1 = min(row_off[g + 1], r0 + EROWS);
  if (r0 >= r1) return;
  const int n0 = blockIdx.x * EBN;
  load_b_tile(bs, B + static_cast<size_t>(slots[g]) * N * r, n0, N, r);
  const int c = threadIdx.x % EBN, par = threadIdx.x / EBN;
  const int n = n0 + c;
  const int ub = ((n >= n1) + (n >= n2)) * r;
  for (int i0 = r0; i0 < r1; i0 += ECHUNK) {
    const int cnt = min(ECHUNK, r1 - i0);
    __syncthreads();   // previous chunk's readers are done with us / rid
    load_u_rows(us, rid, U, ldu, width, rows, i0, cnt);
    if (n < N) {
      for (int i = par; i < cnt; i += 2) {
        const float* u = us + i * width + ub;
        float acc = 0.f;
        for (int k = 0; k < r; ++k) acc = fmaf(u[k], bs[k * EBN + c], acc);
        __nv_bfloat16* p = y + static_cast<size_t>(rid[i]) * ldy + n;
        *p = __float2bfloat16_rn(__bfloat162float(*p) + acc);
      }
    }
  }
}

__device__ __forceinline__ float silu(float v) { return v / (1.f + __expf(-v)); }

// grid (I / 128, row tiles, groups + 1), 256 threads. Group S (the last) holds the rows without an adapter:
// rows[row_off[S] .. T_pad).
__global__ void __launch_bounds__(256) expand_silu_mul_kernel(const __nv_bfloat16* __restrict__ pre, int64_t ldp,
                                                              const float* __restrict__ U, int64_t ldu,
                                                              const __nv_bfloat16* __restrict__ B,
                                                              __nv_bfloat16* __restrict__ out, int64_t ldo, int I,
                                                              int r, int S, int T_pad,
                                                              const int32_t* __restrict__ slots,
                                                              const int32_t* __restrict__ row_off,
                                                              const int32_t* __restrict__ rows) {
  __shared__ __nv_bfloat16 bg[kMaxRank * EBN], bu[kMaxRank * EBN];
  __shared__ float us[ECHUNK * 2 * kMaxRank];
  __shared__ int32_t rid[ECHUNK];
  const int g = blockIdx.z;
  const bool base = g == S;
  const int gend = base ? T_pad : row_off[g + 1];
  const int r0 = row_off[g] + blockIdx.y * EROWS, r1 = min(gend, r0 + EROWS);
  if (r0 >= r1) return;
  const int blk = blockIdx.x;
  const int c = threadIdx.x % EBN, par = threadIdx.x / EBN;
  const int gcol = blk * 2 * EBN + c, ucol = gcol + EBN, j = blk * EBN + c;
  if (!base) {
    const __nv_bfloat16* Bs = B + static_cast<size_t>(slots[g]) * 2 * I * r;
    load_b_tile(bg, Bs, blk * 2 * EBN, 2 * I, r);
    load_b_tile(bu, Bs, blk * 2 * EBN + EBN, 2 * I, r);
  }
  for (int i0 = r0; i0 < r1; i0 += ECHUNK) {
    const int cnt = min(ECHUNK, r1 - i0);
    __syncthreads();
    if (base) {
      if (threadIdx.x < ECHUNK) rid[threadIdx.x] = threadIdx.x < cnt ? rows[i0 + threadIdx.x] : -1;
      __syncthreads();
    } else {
      load_u_rows(us, rid, U, ldu, 2 * r, rows, i0, cnt);
    }
    for (int i = par; i < cnt; i += 2) {
      const int row = rid[i];
      float gv = __bfloat162float(pre[static_cast<size_t>(row) * ldp + gcol]);
      float uv = __bfloat162float(pre[static_cast<size_t>(row) * ldp + ucol]);
      if (!base) {
        const float* u = us + i * 2 * r;
        float dg = 0.f, du = 0.f;
        for (int k = 0; k < r; ++k) {
          dg = fmaf(u[k], __bfloat162float(bg[k * EBN + c]), dg);
          du = fmaf(u[r + k], __bfloat162float(bu[k * EBN + c]), du);
        }
        gv += dg;
        uv += du;
      }
      out[static_cast<size_t>(row) * ldo + j] = __float2bfloat16_rn(silu(gv) * uv);
    }
  }
}

}  // namespace lora
}  // namespace b200

using namespace b200::lora;

static bool lora_rank_ok(int r) { return r >= 8 && r <= kMaxRank && r % 8 == 0; }

// U [T, M] fp32 (rows without an adapter get 0). k_splits: K slices per tile (>= 1); with more than one, `ws` holds
// k_splits * T * M floats of partial sums and a second, fixed-order kernel reduces them. rows[0 .. T) must list
// every row once (InputData's CSR; CUDA-graph padding rows included).
GLLM_EXPORT int gllm_lora_shrink(const void* x, int64_t ldx, const void* A, void* U, void* ws, int T, int K, int M,
                                 const void* slots, const void* row_off, const void* rows, int S, int k_splits,
                                 void* stream) {
  if (T <= 0) return 0;
  if (K % 8 != 0 || ldx % 8 != 0 || M <= 0 || M > 3 * kMaxRank || k_splits < 1 || (k_splits > 1 && ws == nullptr))
    return 2;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int k_chunk = (K + k_splits - 1) / k_splits;
  k_chunk = (k_chunk + SBK - 1) / SBK * SBK;
  k_splits = (K + k_chunk - 1) / k_chunk;      // every slice non-empty: each writes all of its tile's partials
  if (S <= 0 || k_splits == 1) CUDA_CHECK_RET(cudaMemsetAsync(U, 0, static_cast<size_t>(T) * M * sizeof(float), st));
  if (S <= 0) return 0;
  const int m_tiles = (M + SBN - 1) / SBN;
  dim3 grid(m_tiles * k_splits, (T + SBM - 1) / SBM, S);
  float* out = reinterpret_cast<float*>(k_splits == 1 ? U : ws);
  shrink_kernel<<<grid, 128, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(x), ldx,
                                      reinterpret_cast<const __nv_bfloat16*>(A), out, T, K, M, k_chunk, m_tiles,
                                      reinterpret_cast<const int32_t*>(slots),
                                      reinterpret_cast<const int32_t*>(row_off), reinterpret_cast<const int32_t*>(rows));
  CUDA_CHECK_RET(cudaGetLastError());
  if (k_splits > 1) {
    shrink_reduce_kernel<<<(T * M + 255) / 256, 256, 0, st>>>(out, reinterpret_cast<float*>(U), T, M, k_splits, S,
                                                              reinterpret_cast<const int32_t*>(row_off),
                                                              reinterpret_cast<const int32_t*>(rows));
    CUDA_CHECK_RET(cudaGetLastError());
  }
  return 0;
}

// y [T, N] bf16 (row stride ldy) += U[:, m*r : (m+1)*r] · B_slot[n, :]; module m of column n: (n >= n1) + (n >= n2).
// U holds `width` = (modules) * r used columns with row stride ldu.
GLLM_EXPORT int gllm_lora_expand_add(const void* U, int64_t ldu, const void* B, void* y, int64_t ldy, int T, int N,
                                     int r, int n1, int n2, int width, const void* slots, const void* row_off,
                                     const void* rows, int S, void* stream) {
  if (T <= 0 || S <= 0) return 0;
  if (!lora_rank_ok(r) || width > 3 * kMaxRank || width > ldu) return 2;
  dim3 grid((N + EBN - 1) / EBN, (T + EROWS - 1) / EROWS, S);
  expand_add_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float*>(U), ldu, reinterpret_cast<const __nv_bfloat16*>(B),
      reinterpret_cast<__nv_bfloat16*>(y), ldy, N, r, n1, n2, width, reinterpret_cast<const int32_t*>(slots),
      reinterpret_cast<const int32_t*>(row_off), reinterpret_cast<const int32_t*>(rows));
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

// out [T_pad, I] = SiLU(gate + dg) * (up + du) from the interleaved pre-activations pre [T_pad, 2I]; U [T, 2r] holds
// the gate then the up shrink results; B [L, 2I, r] is interleaved like the weight. I % 128 == 0.
GLLM_EXPORT int gllm_lora_expand_silu_mul(const void* pre, int64_t ldp, const void* U, int64_t ldu, const void* B,
                                          void* out, int64_t ldo, int T_pad, int I, int r, const void* slots,
                                          const void* row_off, const void* rows, int S, void* stream) {
  if (T_pad <= 0) return 0;
  if (!lora_rank_ok(r) || I % EBN != 0 || 2 * r > ldu) return 2;
  dim3 grid(I / EBN, (T_pad + EROWS - 1) / EROWS, S + 1);
  expand_silu_mul_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(pre), ldp, reinterpret_cast<const float*>(U), ldu,
      reinterpret_cast<const __nv_bfloat16*>(B), reinterpret_cast<__nv_bfloat16*>(out), ldo, I, r, S, T_pad,
      reinterpret_cast<const int32_t*>(slots), reinterpret_cast<const int32_t*>(row_off),
      reinterpret_cast<const int32_t*>(rows));
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}
