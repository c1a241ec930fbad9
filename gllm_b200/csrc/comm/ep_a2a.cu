// Expert-parallel all-to-all over NVLink peer memory (SURVEY §2.4 X3).
//
// Activations are token-sharded (the fused TP layout, comm/tp_fused.cu). Per MoE block:
//
//   dispatch   every (token, top-k choice) of this rank's shard claims a row in the EXPERT OWNER's receive
//              pool with one remote atomic and stores the token row + (local expert, source) there (P2P st)
//   experts    the owner runs align -> grouped wgmma GEMM1 (SiLU gate) -> grouped GEMM2 over the pool;
//              GEMM2's epilogue stores every output row straight into the TOKEN OWNER's combine buffer
//              through a per-row destination table (gemm_bf16.cu `row_dest`) — the return all-to-all is the
//              GEMM epilogue, there is no separate send
//   combine    the token owner waits for the peers' "returned" flags and sums the k weighted rows
//
// Synchronisation is device-resident and monotonic (call counter + per-source flags), so the block replays
// inside CUDA graphs. Pools are double-buffered by call parity: a peer can only be one MoE call ahead.
// The reference's EP is the degenerate form (replicated tokens, local-expert masking, all-reduce of partial
// sums: gllm/layers/moe/fused_moe_triton/layer.py:326-369); this is the dispatch/combine form.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../common/host_utils.h"
#include "../common/ptx.cuh"

namespace b200 {

static constexpr int kMaxEp = 8;
// ctrl words (uint32) in every rank's symmetric control block
static constexpr int kCtrlPool = 0;     // rows claimed in this rank's receive pool
static constexpr int kCtrlDispatch = 8; // [src] call index of the last finished dispatch from rank src
static constexpr int kCtrlReturn = 16;  // [src] call index of the last finished return from rank src

struct EpState {      // local (non-symmetric) device state
  uint32_t calls;     // MoE calls issued so far (monotonic)
  uint32_t ticket;    // last-CTA election
};

struct EpPeers {
  __nv_bfloat16* recv_x[kMaxEp];
  int32_t* recv_e[kMaxEp];
  int32_t* recv_src[kMaxEp];
  uint32_t* ctrl[kMaxEp];
  __nv_bfloat16* comb[kMaxEp];
};

__device__ __forceinline__ uint32_t pack_src(int rank, int kidx, int row) {
  return (static_cast<uint32_t>(rank) << 26) | (static_cast<uint32_t>(kidx) << 20) | static_cast<uint32_t>(row);
}

// one warp per (token, choice) slot of the local shard
__global__ void ep_dispatch_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, const int32_t* __restrict__ ids,
                                   int n_slots, int top_k, int H, int experts_per_rank, int ep, int rank,
                                   const EpPeers peers, EpState* st) {
  const int slot = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (slot < n_slots) {
    const int e = ids[slot];
    int owner = e / experts_per_rank;
    if (owner >= ep) owner = ep - 1;  // remainder experts live on the last rank
    const int le = e - owner * experts_per_rank;
    uint32_t r = 0;
    if (lane == 0) r = atomicAdd_system(peers.ctrl[owner] + kCtrlPool, 1u);
    r = __shfl_sync(0xffffffffu, r, 0);
    const int tok = slot / top_k;
    const __nv_bfloat16* src = x + static_cast<size_t>(tok) * ldx;
    __nv_bfloat16* dst = peers.recv_x[owner] + static_cast<size_t>(r) * H;
    for (int i = lane * 8; i < H; i += 256) st_v4(dst + i, *reinterpret_cast<const uint4*>(src + i));
    if (lane == 0) {
      peers.recv_e[owner][r] = le;
      peers.recv_src[owner][r] = static_cast<int32_t>(pack_src(rank, slot - tok * top_k, tok));
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();  // cumulative over the CTA's peer stores (ordered before by the barrier)
    const uint32_t t = atomicAdd(&st->ticket, 1u);
    if (t == gridDim.x - 1) {
      st->ticket = 0;
      const uint32_t call = st->calls + 1;
      st->calls = call;
      __threadfence_system();
      for (int p = 0; p < ep; ++p) st_relaxed_sys(peers.ctrl[p] + kCtrlDispatch + rank, call);
    }
  }
}

__global__ void ep_wait_kernel(const uint32_t* flags, const EpState* st, int ep) {
  if (threadIdx.x < ep) {
    const uint32_t call = *reinterpret_cast<const volatile uint32_t*>(&st->calls);
    SpinGuard guard;
    while (static_cast<int32_t>(ld_acquire_sys(flags + threadIdx.x) - call) < 0) guard.poll();
  }
}

// sorted-row -> destination address in the token owner's combine buffer
__global__ void ep_row_dest_kernel(const int32_t* __restrict__ slot_pos, const int32_t* __restrict__ recv_src,
                                   const uint32_t* __restrict__ n_valid, int r_max, int top_k, int H,
                                   const EpPeers peers, int64_t* __restrict__ row_dest) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= r_max || i >= static_cast<int>(*n_valid)) return;
  const int pos = slot_pos[i];
  if (pos < 0) return;
  const uint32_t s = static_cast<uint32_t>(recv_src[i]);
  const int src_rank = s >> 26, kidx = (s >> 20) & 63, row = s & 0xfffff;
  row_dest[pos] = reinterpret_cast<int64_t>(peers.comb[src_rank] + (static_cast<size_t>(row) * top_k + kidx) * H);
}

__global__ void ep_signal_kernel(const EpPeers peers, int ep, int rank, const EpState* st) {
  if (threadIdx.x == 0) {
    __threadfence_system();
    const uint32_t call = st->calls;
    for (int p = 0; p < ep; ++p) st_relaxed_sys(peers.ctrl[p] + kCtrlReturn + rank, call);
  }
}

// out[t] = sum_j w[t, j] * comb[t, j]; also recycles this rank's receive pool for the call after next
__global__ void ep_combine_kernel(const __nv_bfloat16* __restrict__ comb, const float* __restrict__ w,
                                  __nv_bfloat16* __restrict__ out, uint32_t* ctrl, const EpState* st, int ep,
                                  int n_rows, int top_k, int H) {
  if (threadIdx.x < ep) {
    const uint32_t call = *reinterpret_cast<const volatile uint32_t*>(&st->calls);
    SpinGuard guard;
    while (static_cast<int32_t>(ld_acquire_sys(ctrl + kCtrlReturn + threadIdx.x) - call) < 0) guard.poll();
  }
  __syncthreads();
  if (blockIdx.x == 0 && threadIdx.x == 0) ctrl[kCtrlPool] = 0;
  const int t = blockIdx.x;
  if (t >= n_rows) return;
  for (int i = threadIdx.x * 8; i < H; i += blockDim.x * 8) {
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int j = 0; j < top_k; ++j) {
      const float wt = w[t * top_k + j];
      const uint4 v = __ldcg(reinterpret_cast<const uint4*>(comb + (static_cast<size_t>(t) * top_k + j) * H + i));
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

struct EpArgs {
  void* recv_x[kMaxEp];
  void* recv_e[kMaxEp];
  void* recv_src[kMaxEp];
  void* ctrl[kMaxEp];
  void* comb[kMaxEp];
  void* state;
  int ep, rank, experts_per_rank, top_k, H, r_max;
};

static EpPeers to_peers(const EpArgs* a) {
  EpPeers p;
  for (int i = 0; i < kMaxEp; ++i) {
    p.recv_x[i] = reinterpret_cast<__nv_bfloat16*>(a->recv_x[i]);
    p.recv_e[i] = reinterpret_cast<int32_t*>(a->recv_e[i]);
    p.recv_src[i] = reinterpret_cast<int32_t*>(a->recv_src[i]);
    p.ctrl[i] = reinterpret_cast<uint32_t*>(a->ctrl[i]);
    p.comb[i] = reinterpret_cast<__nv_bfloat16*>(a->comb[i]);
  }
  return p;
}

GLLM_EXPORT int gllm_ep_state_bytes() { return static_cast<int>(sizeof(EpState)); }

// dispatch this rank's shard (x [n_rows, H], ids [n_rows, top_k]) and wait until every rank has dispatched
GLLM_EXPORT int gllm_ep_dispatch(const EpArgs* a, const void* x, int64_t ldx, const void* ids, int n_rows,
                                 void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int n_slots = n_rows * a->top_k;
  const int blocks = n_slots > 0 ? (n_slots * 32 + 255) / 256 : 1;
  ep_dispatch_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(x), ldx,
                                             reinterpret_cast<const int32_t*>(ids), n_slots, a->top_k, a->H,
                                             a->experts_per_rank, a->ep, a->rank, to_peers(a),
                                             reinterpret_cast<EpState*>(a->state));
  ep_wait_kernel<<<1, 32, 0, st>>>(reinterpret_cast<const uint32_t*>(a->ctrl[a->rank]) + kCtrlDispatch,
                                   reinterpret_cast<const EpState*>(a->state), a->ep);
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

GLLM_EXPORT int gllm_ep_row_dest(const EpArgs* a, const void* slot_pos, void* row_dest, int rows, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CUDA_CHECK_RET(cudaMemsetAsync(row_dest, 0, sizeof(int64_t) * rows, st));
  ep_row_dest_kernel<<<(a->r_max + 255) / 256, 256, 0, st>>>(
      reinterpret_cast<const int32_t*>(slot_pos), reinterpret_cast<const int32_t*>(a->recv_src[a->rank]),
      reinterpret_cast<const uint32_t*>(a->ctrl[a->rank]) + kCtrlPool, a->r_max, a->top_k, a->H, to_peers(a),
      reinterpret_cast<int64_t*>(row_dest));
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

// after GEMM2 pushed its rows: publish "returned", wait for the peers, sum the k choices of every local token
GLLM_EXPORT int gllm_ep_combine(const EpArgs* a, const void* topk_w, void* out, int n_rows, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ep_signal_kernel<<<1, 32, 0, st>>>(to_peers(a), a->ep, a->rank, reinterpret_cast<const EpState*>(a->state));
  ep_combine_kernel<<<n_rows > 0 ? n_rows : 1, 256, 0, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(a->comb[a->rank]), reinterpret_cast<const float*>(topk_w),
      reinterpret_cast<__nv_bfloat16*>(out), reinterpret_cast<uint32_t*>(a->ctrl[a->rank]),
      reinterpret_cast<const EpState*>(a->state), a->ep, n_rows, a->top_k, a->H);
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}
