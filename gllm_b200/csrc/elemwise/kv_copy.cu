// Paged KV-cache page copy for sm_90a (parallel sampling: the partial last prompt page of a request that fans
// out into several choices is copied once per extra choice).
//
// One launch copies a list of (src, dst) page pairs across every layer tensor of this rank. Each tensor is laid
// out page-major (`[pages, ...]`, see memory_manager.KVCache), so a page is one contiguous run of `page_bytes`
// bytes at `base + page * page_bytes`. The layer base pointers come from a device array, so the launch count does
// not grow with the number of layers. Memory-bound: 16-byte vector loads and stores, four in flight per thread.
#include "../common/host_utils.h"

namespace b200 {

constexpr int kCopyThreads = 256;
constexpr int kCopyUnroll = 4;
constexpr int kCopyChunk = kCopyThreads * kCopyUnroll;   // 16-byte vectors per block and chunk (16 KiB)

// grid.x = tensor * n_pairs + pair, grid.y = chunk of the page
__global__ void __launch_bounds__(kCopyThreads) kv_copy_pages_kernel(const uint64_t* __restrict__ bases,
                                                                      const int32_t* __restrict__ pairs, int n_pairs,
                                                                      int64_t page_vecs) {
  const int tensor = blockIdx.x / n_pairs;
  const int pair = blockIdx.x - tensor * n_pairs;
  uint4* base = reinterpret_cast<uint4*>(bases[tensor]);
  const uint4* src = base + static_cast<int64_t>(pairs[2 * pair]) * page_vecs;
  uint4* dst = base + static_cast<int64_t>(pairs[2 * pair + 1]) * page_vecs;
  const int64_t i0 = static_cast<int64_t>(blockIdx.y) * kCopyChunk + threadIdx.x;
  uint4 v[kCopyUnroll];
#pragma unroll
  for (int u = 0; u < kCopyUnroll; ++u) {
    const int64_t i = i0 + u * kCopyThreads;
    if (i < page_vecs) v[u] = __ldcs(src + i);     // streamed once: do not keep it in L2
  }
#pragma unroll
  for (int u = 0; u < kCopyUnroll; ++u) {
    const int64_t i = i0 + u * kCopyThreads;
    if (i < page_vecs) dst[i] = v[u];
  }
}

}  // namespace b200

using namespace b200;

// bases: device uint64 [num_tensors] layer base pointers (16-byte aligned); pairs: device int32 [n_pairs, 2]
// (src page, dst page). The caller has checked the pairs (distinct dst pages, no dst is a src, no dummy page, all
// below the page count); this entry point checks the shapes it can see.
GLLM_EXPORT int gllm_kv_copy_pages(const void* bases, int num_tensors, int64_t page_bytes, const void* pairs,
                                   int n_pairs, void* stream) {
  if (n_pairs <= 0 || num_tensors <= 0) return 0;
  if (page_bytes <= 0 || page_bytes % 16 != 0) {
    fprintf(stderr, "[gllm_b200] kv_copy_pages: page_bytes=%lld must be a positive multiple of 16\n",
            (long long)page_bytes);
    return 1;
  }
  const int64_t blocks_x = static_cast<int64_t>(num_tensors) * n_pairs;
  const int64_t page_vecs = page_bytes / 16;
  const int64_t chunks = (page_vecs + kCopyChunk - 1) / kCopyChunk;
  if (blocks_x > 0x7fffffffLL || chunks > 65535) {
    fprintf(stderr, "[gllm_b200] kv_copy_pages: %d tensors x %d pairs of %lld bytes is too large for one launch\n",
            num_tensors, n_pairs, (long long)page_bytes);
    return 1;
  }
  kv_copy_pages_kernel<<<dim3(static_cast<unsigned>(blocks_x), static_cast<unsigned>(chunks)), kCopyThreads, 0,
                         reinterpret_cast<cudaStream_t>(stream)>>>(reinterpret_cast<const uint64_t*>(bases),
                                                                  reinterpret_cast<const int32_t*>(pairs), n_pairs,
                                                                  page_vecs);
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}
