// Fused sampling for sm_90a: repetition penalty -> temperature -> top-k -> top-p -> draw.
//
// The reference does this with ~15 PyTorch ops including a full-vocabulary sort
// (gllm/layers/sampler.py:8-54). Here one CTA per sequence makes a handful of passes over its
// logits row (L2-resident) and never sorts:
//   pass A : transformed logit t(x) = penalty(x) / temperature, row max m, Z = sum exp(t - m)
//   top-k  : 4-pass MSB radix select on the order-preserving integer key of t  -> threshold key
//   top-p  : 4-pass radix select on probability mass among the top-k survivors -> threshold key
//   draw   : exponential race  argmax_i  exp(t_i - m) / E_i ,  E_i ~ Exp(1)   (== Gumbel-max,
//            the same distribution the reference draws with `probs / Exp(1)` then argmax)
// Greedy rows (top_k == 1) take a single argmax pass. A vocab-parallel variant returns the
// per-rank (max, index) pair so TP ranks only exchange B x 2 scalars (SURVEY §2.4 X4).
//
// Per-request sampling parameters (OpenAI `frequency_penalty` / `presence_penalty` / `logit_bias` / `seed`):
//   bias row : a row with one adds bias[slot, token] to the penalised logit before the temperature,
//              x2 = penalty(x) - f * c_j - p * [c_j > 0] + logit_bias_j. The row is persistent per-slot state kept
//              by bias_rebuild_kernel (slot (re)assignment) and bias_account_kernel (after every sampled token).
//   seed     : a seeded row keys its exponential race by (seed, position of the token being produced, token id)
//              instead of (engine seed + step counter, batch row, token id), so its draw depends on the logits alone.
#include "../common/host_utils.h"
#include "../common/ptx.cuh"

namespace b200 {

static constexpr int kSampleThreads = 1024;

__device__ __forceinline__ uint32_t f2key(float f) {
  // order-preserving map float -> uint32 (larger float => larger key)
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ uint32_t hash_u32(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
  return x;
}

__device__ __forceinline__ float rand_exp(uint64_t seed, uint32_t row, uint32_t idx) {
  uint32_t h = hash_u32(static_cast<uint32_t>(seed) ^ hash_u32(row * 0x9E3779B9u + 0x85ebca6bu) ^
                        hash_u32(idx + static_cast<uint32_t>(seed >> 32) * 0xc2b2ae35u));
  h = hash_u32(h ^ 0x27d4eb2fu);
  const float u = (static_cast<float>(h >> 8) + 0.5f) * (1.0f / 16777216.0f);  // (0,1)
  return -__logf(u);
}

template <typename T>
__device__ __forceinline__ float load_logit(const T* p, int i);
template <>
__device__ __forceinline__ float load_logit<__nv_bfloat16>(const __nv_bfloat16* p, int i) {
  return __bfloat162float(p[i]);
}
template <>
__device__ __forceinline__ float load_logit<float>(const float* p, int i) { return p[i]; }

// seen: optional [B, ceil(V/32)] bitmask of tokens that already appeared (prompt + output)
// bias_row: optional full-vocabulary additive row (frequency / presence penalties and logit_bias), indexed by token id
__device__ __forceinline__ float transform(float x, int i, const uint32_t* seen_row, float penalty,
                                           const float* bias_row, float inv_temp) {
  if (seen_row != nullptr && penalty != 1.0f) {
    if ((seen_row[i >> 5] >> (i & 31)) & 1u) x = x > 0.f ? x / penalty : x * penalty;
  }
  if (bias_row != nullptr) x += bias_row[i];
  return x * inv_temp;
}

// Per-row RNG key of the exponential race: (engine seed + step, batch row) by default; (request seed, position of the
// token being produced) for a seeded row (seed_pos >= 0).
__device__ __forceinline__ void race_key(const int64_t* seeds, const int32_t* seed_pos, int row, uint64_t seed,
                                         uint32_t step, uint64_t& key, uint32_t& krow) {
  key = seed + step;
  krow = static_cast<uint32_t>(row);
  if (seeds != nullptr && seed_pos != nullptr) {
    const int pos = seed_pos[row];
    if (pos >= 0) {
      key = static_cast<uint64_t>(seeds[row]);
      krow = static_cast<uint32_t>(pos);
    }
  }
}

__device__ __forceinline__ const float* bias_row_of(const float* bias, int64_t bias_ld, const int32_t* bias_slot,
                                                    int row) {
  if (bias == nullptr || bias_slot == nullptr) return nullptr;
  const int s = bias_slot[row];
  return s >= 0 ? bias + static_cast<size_t>(s) * bias_ld : nullptr;
}

struct BlockScratch {
  float fred[32];
  int ired[32];
  unsigned int hist_cnt[256];
  float hist_mass[256];
  uint32_t sel_prefix;
  int sel_k_left;
  float sel_mass_left;
  float bcast_f[2];
  int bcast_i;
};

__device__ __forceinline__ float block_max(float v, BlockScratch& s) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if (lane == 0) s.fred[warp] = v;
  __syncthreads();
  float t = lane < (blockDim.x >> 5) ? s.fred[lane] : -INFINITY;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t = fmaxf(t, __shfl_xor_sync(0xffffffffu, t, o));
  return t;
}
__device__ __forceinline__ float block_sumf(float v, BlockScratch& s) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if (lane == 0) s.fred[warp] = v;
  __syncthreads();
  float t = lane < (blockDim.x >> 5) ? s.fred[lane] : 0.f;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  return t;
}
// argmax with smallest-index tie break
__device__ __forceinline__ void block_argmax(float& v, int& idx, BlockScratch& s) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
    if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; }
  }
  __syncthreads();
  if (lane == 0) { s.fred[warp] = v; s.ired[warp] = idx; }
  __syncthreads();
  float tv = lane < (blockDim.x >> 5) ? s.fred[lane] : -INFINITY;
  int ti = lane < (blockDim.x >> 5) ? s.ired[lane] : 0x7fffffff;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, tv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, ti, o);
    if (ov > tv || (ov == tv && oi < ti)) { tv = ov; ti = oi; }
  }
  v = tv; idx = ti;
}

// Row accessors: the select-and-draw core below works on "element i of this row" through one of these.
//   GlobalRow : a logits row in global memory (penalty / temperature applied on the fly)
//   CandRow   : vocab-parallel candidate list gathered from all TP ranks (already transformed), see
//               vp_candidates_kernel / vp_final_kernel
template <typename T>
struct GlobalRow {
  const T* lr;
  const uint32_t* seen_row;
  const float* bias_row;
  float pen, inv_temp;
  int vocab_offset;
  __device__ __forceinline__ float val(int i) const {
    return transform(load_logit<T>(lr, i), i + vocab_offset, seen_row, pen, bias_row, inv_temp);
  }
  __device__ __forceinline__ int token(int i) const { return i + vocab_offset; }
};

struct CandRow {
  const float* base;   // gathered buffer [tp][B][W]
  int C, W, row;
  size_t rank_stride;  // B * W
  __device__ __forceinline__ const float* at(int i) const {
    const int r = i / C;
    return base + r * rank_stride + static_cast<size_t>(row) * W + (i - r * C);
  }
  __device__ __forceinline__ float val(int i) const { return *at(i); }
  __device__ __forceinline__ int token(int i) const { return __float_as_int(at(i)[C]); }
};

// MSB radix select of the `k`-th largest key among elements with key >= floor_key (phase 0: by count) or of the
// key where the cumulative probability mass (descending) reaches `mass_target` (phase 1). Leaves the selected key in
// S.sel_prefix and the remaining count / mass inside that key's bucket in S.sel_k_left / S.sel_mass_left.
template <class Row>
__device__ __forceinline__ void radix_select(const Row& R, int V, int phase, uint32_t floor_key, int k,
                                             float mass_target, float m, BlockScratch& S) {
  if (threadIdx.x == 0) {
    S.sel_prefix = 0u;
    S.sel_k_left = k;
    S.sel_mass_left = mass_target;
  }
  __syncthreads();
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    const uint32_t prefix = S.sel_prefix;
    const uint32_t pmask = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
    for (int b = threadIdx.x; b < 256; b += blockDim.x) { S.hist_cnt[b] = 0u; S.hist_mass[b] = 0.f; }
    __syncthreads();
    for (int i = threadIdx.x; i < V; i += blockDim.x) {
      const float x = R.val(i);
      const uint32_t key = f2key(x);
      if (key >= floor_key && (key & pmask) == prefix) {
        const uint32_t b = (key >> shift) & 0xffu;
        if (phase == 0) atomicAdd(&S.hist_cnt[b], 1u);
        else atomicAdd(&S.hist_mass[b], __expf(x - m));
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      // walk bins from the largest key downwards
      int b = 255;
      if (phase == 0) {
        int left = S.sel_k_left;
        for (; b > 0; --b) {
          const int c = static_cast<int>(S.hist_cnt[b]);
          if (c >= left) break;
          left -= c;
        }
        S.sel_k_left = left;
      } else {
        float left = S.sel_mass_left;
        for (; b > 0; --b) {
          const float c = S.hist_mass[b];
          if (c >= left) break;
          left -= c;
        }
        S.sel_mass_left = left;
      }
      S.sel_prefix = prefix | (static_cast<uint32_t>(b) << shift);
    }
    __syncthreads();
  }
}

// top-k -> top-p -> exponential race over the elements of one row. `m` = row max of the transformed values,
// `mass_all` = sum exp(val - m) over the WHOLE distribution (for a candidate row that includes the mass of the
// vocabulary entries that are not candidates). Returns (score, token) of the winner in thread 0.
template <class Row>
__device__ __forceinline__ void select_and_draw(const Row& R, int V, int k, float tp, float m, float mass_all,
                                                uint64_t seed, uint32_t row, BlockScratch& S, float& best_out,
                                                int& tok_out) {
  uint32_t thr_key = 0u;  // everything survives
  float mass_total = mass_all;
  for (int phase = 0; phase < 2; ++phase) {
    // phase 0: top-k by count; phase 1: top-p by mass (within survivors of phase 0)
    if (phase == 0 && k >= V) continue;
    if (phase == 1 && tp >= 1.0f) continue;
    const uint32_t floor_key = thr_key;
    radix_select(R, V, phase, floor_key, k, tp * mass_total, m, S);
    thr_key = S.sel_prefix > floor_key ? S.sel_prefix : floor_key;
    if (phase == 0) {
      // mass of the top-k survivors (denominator for top-p)
      float z = 0.f;
      for (int i = threadIdx.x; i < V; i += blockDim.x) {
        const float x = R.val(i);
        if (f2key(x) >= thr_key) z += __expf(x - m);
      }
      mass_total = block_sumf(z, S);
    }
    __syncthreads();
  }
  // ---- draw: exponential race among survivors (== Gumbel-max; the RNG is keyed by the TOKEN id, so a row draws
  // the same token whether it is sampled from the full vocabulary or from gathered vocab-parallel candidates) ----
  float best = -INFINITY;
  int besti = 0x7fffffff;
  for (int i = threadIdx.x; i < V; i += blockDim.x) {
    const float x = R.val(i);
    if (f2key(x) >= thr_key && x > -INFINITY) {
      const int tok = R.token(i);
      const float e = rand_exp(seed, row, static_cast<uint32_t>(tok));
      const float score = (x - m) - __logf(e);  // log(p_i / E_i)
      if (score > best || (score == best && tok < besti)) { best = score; besti = tok; }
    }
  }
  block_argmax(best, besti, S);
  best_out = best;
  tok_out = besti;
}

template <typename T>
__global__ void __launch_bounds__(kSampleThreads)
sample_kernel(const T* __restrict__ logits, int64_t ld, int V, const float* __restrict__ temperature,
              const int32_t* __restrict__ top_k, const float* __restrict__ top_p,
              const float* __restrict__ rep_penalty, const uint32_t* __restrict__ seen, int seen_words,
              const int32_t* __restrict__ slot_idx, uint64_t seed, const int64_t* __restrict__ step_ptr, int32_t* __restrict__ out_tokens,
              float* __restrict__ out_max, int vocab_offset, const float* __restrict__ bias, int64_t bias_ld,
              const int32_t* __restrict__ bias_slot, const int64_t* __restrict__ seeds,
              const int32_t* __restrict__ seed_pos) {
  __shared__ BlockScratch S;
  const int row = blockIdx.x;
  const uint32_t* seen_row =
      seen != nullptr ? seen + static_cast<size_t>(slot_idx != nullptr ? slot_idx[row] : row) * seen_words : nullptr;
  const float temp = temperature != nullptr ? temperature[row] : 1.0f;
  GlobalRow<T> R;
  R.lr = logits + static_cast<size_t>(row) * ld;
  R.seen_row = seen_row;
  R.bias_row = bias_row_of(bias, bias_ld, bias_slot, row);
  R.inv_temp = (temp <= 1e-5f) ? 1.0f : 1.0f / temp;
  R.pen = rep_penalty != nullptr ? rep_penalty[row] : 1.0f;
  R.vocab_offset = vocab_offset;
  int k = top_k != nullptr ? top_k[row] : 1;
  if (k <= 0 || k > V) k = V;
  const float tp = top_p != nullptr ? top_p[row] : 1.0f;

  // ---- pass A: max / argmax ----
  float vmax = -INFINITY;
  int imax = 0x7fffffff;
  for (int i = threadIdx.x; i < V; i += blockDim.x) {
    const float x = R.val(i);
    if (x > vmax) { vmax = x; imax = i; }
  }
  block_argmax(vmax, imax, S);
  if (k == 1) {
    if (threadIdx.x == 0) {
      out_tokens[row] = imax + vocab_offset;
      if (out_max != nullptr) out_max[row] = vmax;
    }
    return;
  }
  const float m = vmax;
  float z = 0.f;
  for (int i = threadIdx.x; i < V; i += blockDim.x) z += __expf(R.val(i) - m);
  const float mass_all = block_sumf(z, S);
  const uint32_t step = step_ptr != nullptr ? static_cast<uint32_t>(*step_ptr) : 0u;
  uint64_t key;
  uint32_t krow;
  race_key(seeds, seed_pos, row, seed, step, key, krow);
  float best;
  int tok;
  select_and_draw(R, V, k, tp, m, mass_all, key, krow, S, best, tok);
  if (threadIdx.x == 0) {
    out_tokens[row] = tok;
    if (out_max != nullptr) out_max[row] = best;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Vocab-parallel sampling (SURVEY §2.4 X4): the [B, V] logits are never gathered. Every TP rank reduces its own
// vocab shard to a fixed-size record per row — its C best candidates after penalty and temperature (value + token
// id), the shard's softmax statistics (max, sum exp) and, for rows that sample from the whole vocabulary, the
// shard's exponential-race winner — the ranks all-gather these records (B x (2C+4) floats per rank instead of
// B x V/tp logits) and vp_final_kernel finishes top-k / top-p / draw on the tp x C candidates with the exact global
// normalisation. Exact whenever the surviving set has at most C tokens (always true for top_k <= C; for top-p-only
// rows whenever the nucleus fits — the global top-C tokens are always among the candidates); beyond that the nucleus
// is truncated to the candidates. Rows with neither top-k nor top-p are exact: Gumbel-max needs no normalisation.
// Replaces the reference's logits all-gather + full-vocab sort (gllm/layers/vocab_parallel_embedding.py:423-435,
// gllm/layers/sampler.py:8-54).
// ------------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kSampleThreads)
vp_candidates_kernel(const T* __restrict__ logits, int64_t ld, int V, int V_full, int C,
                     const float* __restrict__ temperature, const int32_t* __restrict__ top_k,
                     const float* __restrict__ top_p, const float* __restrict__ rep_penalty,
                     const uint32_t* __restrict__ seen, int seen_words, const int32_t* __restrict__ slot_idx,
                     uint64_t seed, const int64_t* __restrict__ step_ptr, float* __restrict__ out, int vocab_offset,
                     const float* __restrict__ bias, int64_t bias_ld, const int32_t* __restrict__ bias_slot,
                     const int64_t* __restrict__ seeds, const int32_t* __restrict__ seed_pos) {
  __shared__ BlockScratch S;
  __shared__ int s_cnt, s_eq;
  const int row = blockIdx.x;
  const int W = 2 * C + 4;
  float* o = out + static_cast<size_t>(row) * W;
  const uint32_t* seen_row =
      seen != nullptr ? seen + static_cast<size_t>(slot_idx != nullptr ? slot_idx[row] : row) * seen_words : nullptr;
  const float temp = temperature != nullptr ? temperature[row] : 1.0f;
  GlobalRow<T> R;
  R.lr = logits + static_cast<size_t>(row) * ld;
  R.seen_row = seen_row;
  R.bias_row = bias_row_of(bias, bias_ld, bias_slot, row);
  R.inv_temp = (temp <= 1e-5f) ? 1.0f : 1.0f / temp;
  R.pen = rep_penalty != nullptr ? rep_penalty[row] : 1.0f;
  R.vocab_offset = vocab_offset;
  int k = top_k != nullptr ? top_k[row] : 1;
  if (k <= 0 || k > V_full) k = V_full;
  const float tp = top_p != nullptr ? top_p[row] : 1.0f;
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    o[i] = -INFINITY;
    o[C + i] = __int_as_float(0);
  }
  if (threadIdx.x == 0) { s_cnt = 0; s_eq = 0; }
  if (V <= 0) {   // a shard made of padding only
    if (threadIdx.x == 0) { o[2 * C] = -INFINITY; o[2 * C + 1] = 0.f; o[2 * C + 2] = -INFINITY; o[2 * C + 3] = __int_as_float(0); }
    return;
  }
  float vmax = -INFINITY;
  int imax = 0x7fffffff;
  for (int i = threadIdx.x; i < V; i += blockDim.x) {
    const float x = R.val(i);
    if (x > vmax) { vmax = x; imax = i; }
  }
  block_argmax(vmax, imax, S);
  const float m = vmax;
  float z = 0.f;
  for (int i = threadIdx.x; i < V; i += blockDim.x) z += __expf(R.val(i) - m);
  z = block_sumf(z, S);
  float race = -INFINITY;
  int race_tok = 0;
  if (k >= V_full && tp >= 1.0f) {
    // unfiltered row: the exponential race needs no normalisation, run it on the shard (scores are relative to the
    // shard max m: the final kernel shifts them to the global max)
    const uint32_t step = step_ptr != nullptr ? static_cast<uint32_t>(*step_ptr) : 0u;
    uint64_t key;
    uint32_t krow;
    race_key(seeds, seed_pos, row, seed, step, key, krow);
    float best = -INFINITY;
    int besti = 0x7fffffff;
    for (int i = threadIdx.x; i < V; i += blockDim.x) {
      const float x = R.val(i);
      const float e = rand_exp(key, krow, static_cast<uint32_t>(i + vocab_offset));
      const float score = (x - m) - __logf(e);
      if (score > best || (score == best && i + vocab_offset < besti)) { best = score; besti = i + vocab_offset; }
    }
    block_argmax(best, besti, S);
    race = best;
    race_tok = besti;
  }
  if (threadIdx.x == 0) {
    o[2 * C] = m;
    o[2 * C + 1] = z;
    o[2 * C + 2] = race;
    o[2 * C + 3] = __int_as_float(race_tok);
  }
  int ck = k < C ? k : C;
  if (ck > V) ck = V;
  if (ck == 1) {
    if (threadIdx.x == 0) { o[0] = vmax; o[C] = __int_as_float(imax + vocab_offset); }
    return;
  }
  // the ck largest values of the shard: radix-select the ck-th largest key, then compact
  radix_select(R, V, 0, 0u, ck, 0.f, m, S);
  const uint32_t thr = S.sel_prefix;
  const int eq_take = S.sel_k_left;     // how many elements with key == thr belong to the ck largest
  __syncthreads();
  for (int i = threadIdx.x; i < V; i += blockDim.x) {
    const float x = R.val(i);
    const uint32_t key = f2key(x);
    bool take = key > thr;
    if (key == thr) take = atomicAdd(&s_eq, 1) < eq_take;
    if (take) {
      const int pos = atomicAdd(&s_cnt, 1);
      if (pos < C) { o[pos] = x; o[C + pos] = __int_as_float(i + vocab_offset); }
    }
  }
}

__global__ void __launch_bounds__(256)
vp_final_kernel(const float* __restrict__ gathered, int tp, int B, int C, int V_full,
                const int32_t* __restrict__ top_k, const float* __restrict__ top_p, uint64_t seed,
                const int64_t* __restrict__ step_ptr, int32_t* __restrict__ out_tokens,
                const int64_t* __restrict__ seeds, const int32_t* __restrict__ seed_pos) {
  __shared__ BlockScratch S;
  const int row = blockIdx.x;
  const int W = 2 * C + 4;
  CandRow R;
  R.base = gathered;
  R.C = C;
  R.W = W;
  R.row = row;
  R.rank_stride = static_cast<size_t>(B) * W;
  const int n = tp * C;
  int k = top_k != nullptr ? top_k[row] : 1;
  if (k <= 0 || k > V_full) k = V_full;
  const float tpv = top_p != nullptr ? top_p[row] : 1.0f;
  // global softmax statistics from the per-rank (max, sum exp) pairs
  float gm = -INFINITY;
  for (int r = 0; r < tp; ++r) gm = fmaxf(gm, gathered[r * R.rank_stride + static_cast<size_t>(row) * W + 2 * C]);
  float gz = 0.f;
  for (int r = 0; r < tp; ++r) {
    const float* st = gathered + r * R.rank_stride + static_cast<size_t>(row) * W + 2 * C;
    if (st[1] > 0.f) gz += st[1] * __expf(st[0] - gm);
  }
  if (k >= V_full && tpv >= 1.0f) {
    // unfiltered: best shard-race winner after shifting every shard's scores to the global max
    if (threadIdx.x == 0) {
      float best = -INFINITY;
      int tok = 0;
      for (int r = 0; r < tp; ++r) {
        const float* st = gathered + r * R.rank_stride + static_cast<size_t>(row) * W + 2 * C;
        const float sc = st[2] + (st[0] - gm);
        const int t = __float_as_int(st[3]);
        if (sc > best || (sc == best && t < tok)) { best = sc; tok = t; }
      }
      out_tokens[row] = tok;
    }
    return;
  }
  if (k > n) k = n;   // top_k beyond the candidate capacity: truncated to the candidates (see header comment)
  const uint32_t step = step_ptr != nullptr ? static_cast<uint32_t>(*step_ptr) : 0u;
  float best;
  int tok;
  if (k == 1) {
    float v = -INFINITY;
    int t = 0x7fffffff;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const float x = R.val(i);
      const int ti = R.token(i);
      if (x > v || (x == v && ti < t)) { v = x; t = ti; }
    }
    block_argmax(v, t, S);
    tok = t;
  } else {
    uint64_t key;
    uint32_t krow;
    race_key(seeds, seed_pos, row, seed, step, key, krow);
    select_and_draw(R, n, k, tpv, gm, gz, key, krow, S, best, tok);
  }
  if (threadIdx.x == 0) out_tokens[row] = tok;
}

// ------------------------------------------------------------------------------------------------------------------
// Token log-probabilities of the raw model distribution: log_softmax of the fp32 logits over the real vocabulary,
// taken before repetition penalty, temperature, top-k and top-p. Vocab-parallel like the sampler above: the [E, V]
// logits are never gathered. Every TP rank reduces its shard of each requesting row to a record of W = 2N + 3 floats
//   [0, N)   the shard's N largest raw logits, unordered (-inf where the shard has fewer than N real columns)
//   [N, 2N)  their token ids bit-cast to float (kLpNoToken where the shard has fewer than N real columns)
//   2N       shard max m        2N + 1   sum exp(x - m) over the shard
//   2N + 2   raw logit of the row's sampled token if this shard holds it, -inf otherwise
// the ranks all-gather the records (tp = 1 on one GPU) and logprobs_final_kernel forms the global log-sum-exp and
// merges the tp x N candidates to the global top N, ordered by logit, ties to the lower token id (block_argmax's rule).
// ------------------------------------------------------------------------------------------------------------------
static constexpr int kMaxLogprobs = 20;
static constexpr int kLpNoToken = 0x7fffffff;

// One CTA per requesting row. Passes over the row (L2-resident after the LM head): 2 when N == 0 (max, sum exp),
// 7 when N > 0 (max, sum exp, the 4 radix-select passes for the N-th largest key, one compaction pass).
template <typename T>
__global__ void __launch_bounds__(kSampleThreads)
logprobs_shard_kernel(const T* __restrict__ logits, int64_t ld, int V, int N, const int32_t* __restrict__ rows,
                      const int32_t* __restrict__ tokens, float* __restrict__ out, int vocab_offset) {
  __shared__ BlockScratch S;
  __shared__ int s_cnt, s_eq;
  const int row = rows != nullptr ? rows[blockIdx.x] : static_cast<int>(blockIdx.x);
  float* o = out + static_cast<size_t>(blockIdx.x) * (2 * N + 3);
  GlobalRow<T> R;   // penalty 1, temperature 1: the raw logits
  R.lr = logits + static_cast<size_t>(row) * ld;
  R.seen_row = nullptr;
  R.bias_row = nullptr;
  R.pen = 1.0f;
  R.inv_temp = 1.0f;
  R.vocab_offset = vocab_offset;
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    o[i] = -INFINITY;
    o[N + i] = __int_as_float(kLpNoToken);
  }
  if (threadIdx.x == 0) {
    s_cnt = 0;
    s_eq = 0;
    const int local = tokens[row] - vocab_offset;
    o[2 * N + 2] = (local >= 0 && local < V) ? R.val(local) : -INFINITY;
  }
  if (V <= 0) {   // a shard made of padding only
    if (threadIdx.x == 0) { o[2 * N] = -INFINITY; o[2 * N + 1] = 0.f; }
    return;
  }
  float vmax = -INFINITY;
  for (int i = threadIdx.x; i < V; i += blockDim.x) vmax = fmaxf(vmax, R.val(i));
  const float m = block_max(vmax, S);
  float z = 0.f;
  if (m > -INFINITY)
    for (int i = threadIdx.x; i < V; i += blockDim.x) z += __expf(R.val(i) - m);
  z = block_sumf(z, S);
  if (threadIdx.x == 0) { o[2 * N] = m; o[2 * N + 1] = z; }
  const int k = N < V ? N : V;
  if (k <= 0) return;
  // the k largest logits of the shard: radix-select the k-th largest key, then compact
  radix_select(R, V, 0, 0u, k, 0.f, m, S);
  const uint32_t thr = S.sel_prefix;
  const int eq_take = S.sel_k_left;                                // elements with key == thr among the k largest
  const int eq_all = static_cast<int>(S.hist_cnt[thr & 0xffu]);    // elements with key == thr (last radix pass)
  __syncthreads();
  if (eq_take >= eq_all) {
    // no tie is cut at the k-th place: every key >= thr is taken, in any order
    for (int i = threadIdx.x; i < V; i += blockDim.x) {
      const float x = R.val(i);
      if (f2key(x) >= thr) {
        const int pos = atomicAdd(&s_cnt, 1);
        o[pos] = x;
        o[N + pos] = __int_as_float(i + vocab_offset);
      }
    }
    return;
  }
  // a tie is cut at the k-th place: the lowest token ids win, so the equal keys are ranked in index order, one
  // blockDim-wide chunk at a time (ballot + per-warp prefix counts)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (int base = 0; base < V; base += blockDim.x) {
    const int i = base + threadIdx.x;
    const float x = i < V ? R.val(i) : -INFINITY;
    const uint32_t key = i < V ? f2key(x) : 0u;
    if (i < V && key > thr) {
      const int pos = atomicAdd(&s_cnt, 1);
      o[pos] = x;
      o[N + pos] = __int_as_float(i + vocab_offset);
    }
    const bool eq = i < V && key == thr;
    const unsigned bal = __ballot_sync(0xffffffffu, eq);
    if (lane == 0) S.ired[warp] = __popc(bal);
    __syncthreads();
    int before = s_eq + __popc(bal & ((1u << lane) - 1u));
    for (int w = 0; w < warp; ++w) before += S.ired[w];
    if (eq && before < eq_take) {
      const int pos = atomicAdd(&s_cnt, 1);
      o[pos] = x;
      o[N + pos] = __int_as_float(i + vocab_offset);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int tot = 0;
      for (int w = 0; w < nwarps; ++w) tot += S.ired[w];
      s_eq += tot;
    }
    __syncthreads();
  }
}

// One CTA per requesting row; `gathered` [tp, E, 2N+3] = every rank's shard records. Writes [E, 1 + 2N] fp32:
// the sampled token's log-prob, then N x (token id bit-cast to float, log-prob) ordered by logit, ties to the lower
// token id. Slots beyond the real vocabulary hold token id -1 and log-prob -inf.
__global__ void __launch_bounds__(256)
logprobs_final_kernel(const float* __restrict__ gathered, int tp, int E, int N, float* __restrict__ out) {
  extern __shared__ float cand[];   // [tp * N] logits, then [tp * N] token ids
  const int row = blockIdx.x;
  const int W = 2 * N + 3;
  const size_t rank_stride = static_cast<size_t>(E) * W;
  const float* rec = gathered + static_cast<size_t>(row) * W;
  float gm = -INFINITY, chosen = -INFINITY;
  for (int r = 0; r < tp; ++r) {
    gm = fmaxf(gm, rec[r * rank_stride + 2 * N]);
    chosen = fmaxf(chosen, rec[r * rank_stride + 2 * N + 2]);   // -inf on every rank but the token's owner
  }
  float gz = 0.f;
  for (int r = 0; r < tp; ++r) {
    const float* st = rec + r * rank_stride + 2 * N;
    if (st[1] > 0.f) gz += st[1] * __expf(st[0] - gm);
  }
  const float lse = gm + __logf(gz);
  float* o = out + static_cast<size_t>(row) * (1 + 2 * N);
  if (threadIdx.x == 0) o[0] = chosen - lse;
  const int n = tp * N;
  int* cand_tok = reinterpret_cast<int*>(cand + n);
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int r = i / N, c = i - r * N;
    cand[i] = rec[r * rank_stride + c];
    cand_tok[i] = __float_as_int(rec[r * rank_stride + N + c]);
  }
  __syncthreads();
  // rank of candidate i = number of candidates ahead of it in (logit desc, token asc, slot asc) order: a permutation
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float v = cand[i];
    const int t = cand_tok[i];
    int rank = 0;
    for (int j = 0; j < n; ++j) {
      const float vj = cand[j];
      const int tj = cand_tok[j];
      rank += (vj > v) || (vj == v && (tj < t || (tj == t && j < i)));
    }
    if (rank < N) {
      const bool real = t != kLpNoToken;
      o[1 + 2 * rank] = __int_as_float(real ? t : -1);
      o[2 + 2 * rank] = real ? v - lse : -INFINITY;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Prompt log-probabilities (scoring): Q rows of LM-head logits, each with its own target token (the next prompt
// token). Q is a whole prompt, far more rows than the sampled ones, and a tile of them does not stay in L2 for
// the 2 - 7 passes of logprobs_shard_kernel. For N <= 1 (perplexity, and the is-greedy check of evaluation
// harnesses) one pass over the row suffices: an online max / sum-exp with rescaling, a running argmax (ties to the
// lower token id, as block_argmax) and the target's raw logit. The record is logprobs_shard_kernel's [2N+3] layout,
// so the all-gather and logprobs_final_kernel are shared. Rows with N > 1 take logprobs_shard_kernel.
// ------------------------------------------------------------------------------------------------------------------
static constexpr int kPromptLpThreads = 512;

// (m, s) of a set of logits: s = sum exp(x - m). Merging with m = -inf (an empty or all -inf set) adds nothing.
__device__ __forceinline__ void lse_merge(float& m, float& s, float m2, float s2) {
  if (m2 == -INFINITY) return;
  if (m == -INFINITY) { m = m2; s = s2; return; }
  if (m2 > m) { s = s * __expf(m - m2) + s2; m = m2; }
  else s += s2 * __expf(m2 - m);
}

__device__ __forceinline__ void plp_take(float x, int i, float& m, float& s, float& bv, int& bi) {
  if (x > bv || (x == bv && i < bi)) { bv = x; bi = i; }
  if (x > m) { s = (m == -INFINITY ? 0.f : s * __expf(m - x)) + 1.f; m = x; }
  else if (x > -INFINITY) s += __expf(x - m);
}

// One CTA per row. logits [Q, ld]: row q is scored against targets[q]; V real columns; out [Q, 2N+3], N in {0, 1}.
template <typename T>
__global__ void __launch_bounds__(kPromptLpThreads)
prompt_logprobs_shard_kernel(const T* __restrict__ logits, int64_t ld, int V, int N,
                             const int32_t* __restrict__ targets, float* __restrict__ out, int vocab_offset) {
  __shared__ BlockScratch S;
  __shared__ float s_m[32], s_s[32];
  const int row = blockIdx.x;
  const T* lr = logits + static_cast<size_t>(row) * ld;
  float* o = out + static_cast<size_t>(row) * (2 * N + 3);
  if (threadIdx.x == 0) {
    const int local = targets[row] - vocab_offset;
    o[2 * N + 2] = (local >= 0 && local < V) ? load_logit<T>(lr, local) : -INFINITY;
  }
  if (V <= 0) {   // a shard made of padding only
    if (threadIdx.x == 0) {
      o[2 * N] = -INFINITY;
      o[2 * N + 1] = 0.f;
      if (N) { o[0] = -INFINITY; o[1] = __int_as_float(kLpNoToken); }
    }
    return;
  }
  float m = -INFINITY, s = 0.f, bv = -INFINITY;
  int bi = kLpNoToken;
  constexpr int kVec = 16 / sizeof(T);
  int head = 0;   // columns [0, head) go through 16-byte loads, the rest one by one
  if ((reinterpret_cast<uintptr_t>(lr) & 15u) == 0) head = V / kVec * kVec;
  const uint4* lv = reinterpret_cast<const uint4*>(lr);
  for (int v = threadIdx.x; v < head / kVec; v += blockDim.x) {
    const uint4 raw = __ldg(lv + v);
    const T* e = reinterpret_cast<const T*>(&raw);
    float x[kVec];
    float vm = -INFINITY;
#pragma unroll
    for (int j = 0; j < kVec; ++j) {
      x[j] = load_logit<T>(e, j);
      vm = fmaxf(vm, x[j]);
    }
    const int base = v * kVec;
#pragma unroll
    for (int j = 0; j < kVec; ++j)
      if (x[j] > bv) { bv = x[j]; bi = base + j; }   // ascending ids within the thread: strict > keeps the lowest
    if (bi == kLpNoToken && vm == -INFINITY) bi = base;   // an all -inf prefix: the lowest id still wins
    if (vm > -INFINITY) {
      if (vm > m) { s = (m == -INFINITY ? 0.f : s * __expf(m - vm)); m = vm; }
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < kVec; ++j) acc += __expf(x[j] - m);
      s += acc;
    }
  }
  for (int i = head + threadIdx.x; i < V; i += blockDim.x) plp_take(load_logit<T>(lr, i), i, m, s, bv, bi);
  // block merge of (m, s)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, off);
    const float s2 = __shfl_xor_sync(0xffffffffu, s, off);
    lse_merge(m, s, m2, s2);
  }
  if (lane == 0) { s_m[warp] = m; s_s[warp] = s; }
  block_argmax(bv, bi, S);   // (its __syncthreads also publish s_m / s_s)
  if (threadIdx.x == 0) {
    float gm = -INFINITY, gs = 0.f;
    for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) lse_merge(gm, gs, s_m[w], s_s[w]);
    o[2 * N] = gm;
    o[2 * N + 1] = gs;
    if (N) {
      o[0] = bv;
      o[1] = __int_as_float(bi == kLpNoToken ? kLpNoToken : bi + vocab_offset);
    }
  }
}

// set bit `token` of row `row` in the seen-token bitmask: one thread per (row, token) pair
__global__ void mark_seen_kernel(uint32_t* seen, int seen_words, const int32_t* rows, const int32_t* tokens, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int tok = tokens[i];
  if (tok < 0) return;
  atomicOr(&seen[static_cast<size_t>(rows[i]) * seen_words + (tok >> 5)], 1u << (tok & 31));
}

// ------------------------------------------------------------------------------------------------------------------
// Bias rows of the frequency / presence penalties and logit_bias. Per slot: an fp32 row bias[slot, V] holding
// -f * c_j - p * [c_j > 0] + logit_bias_j and a bitmask out_seen[slot, ceil(V/32)] of the tokens generated so far
// (c_j > 0), so the presence term is charged once. Every sampling rank keeps full-vocabulary rows.
//
// Ordering invariant: both kernels run on the compute stream, after the forward and the sampler of their step. A
// lookahead step still in flight when its sequence finishes (a zombie row) therefore completes its accounting on the
// slot before any later batch can rebuild and reuse that slot: the rebuild is enqueued behind it on the same stream.
// ------------------------------------------------------------------------------------------------------------------

// One thread per emitting row: charge the token just sampled. Rows without a bias row (bias_slot < 0) do nothing.
// A slot appears at most once per step (one sequence per slot, one token per sequence), so nothing races.
__global__ void bias_account_kernel(float* __restrict__ bias, int64_t bias_ld, uint32_t* __restrict__ out_seen,
                                    int seen_words, const int32_t* __restrict__ bias_slot,
                                    const int32_t* __restrict__ tokens, const float* __restrict__ freq,
                                    const float* __restrict__ pres, int E) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= E) return;
  const int slot = bias_slot[r];
  const int tok = tokens[r];
  if (slot < 0 || tok < 0) return;
  uint32_t* w = out_seen + static_cast<size_t>(slot) * seen_words + (tok >> 5);
  const uint32_t bit = 1u << (tok & 31);
  const bool first = (atomicOr(w, bit) & bit) == 0u;
  float* b = bias + static_cast<size_t>(slot) * bias_ld + tok;
  *b = *b - (first ? freq[r] + pres[r] : freq[r]);
}

// One CTA per (re)assigned slot: clear the row, scatter the request's logit_bias, then replay the counts of the output
// tokens known so far in output order — the same fp32 operations bias_account_kernel performs token by token, so a
// recomputed sequence gets back bit for bit the row it had. Thread t replays the tokens of the bitmask words w with
// w % blockDim == t, in order, so every element (and every out_seen word) has exactly one writer.
__global__ void __launch_bounds__(1024)
bias_rebuild_kernel(float* __restrict__ bias, int64_t bias_ld, uint32_t* __restrict__ out_seen, int seen_words,
                    int V, const int32_t* __restrict__ slots, const float* __restrict__ pen,
                    const int32_t* __restrict__ lb_off, const int32_t* __restrict__ lb_ids,
                    const float* __restrict__ lb_vals, const int32_t* __restrict__ out_off,
                    const int32_t* __restrict__ out_toks) {
  const int r = blockIdx.x;
  const int slot = slots[r];
  float* row = bias + static_cast<size_t>(slot) * bias_ld;
  uint32_t* seen = out_seen + static_cast<size_t>(slot) * seen_words;
  for (int i = threadIdx.x; i < V; i += blockDim.x) row[i] = 0.f;
  for (int i = threadIdx.x; i < seen_words; i += blockDim.x) seen[i] = 0u;
  __syncthreads();
  for (int i = lb_off[r] + threadIdx.x; i < lb_off[r + 1]; i += blockDim.x) {
    const int tok = lb_ids[i];
    if (tok >= 0 && tok < V) row[tok] = lb_vals[i];   // (ids are validated on the host; never write past the row)
  }
  __syncthreads();
  const float f = pen[2 * r], p = pen[2 * r + 1];
  for (int i = out_off[r]; i < out_off[r + 1]; ++i) {
    const int tok = out_toks[i];
    if (tok < 0 || tok >= V || (tok >> 5) % static_cast<int>(blockDim.x) != static_cast<int>(threadIdx.x)) continue;
    const uint32_t bit = 1u << (tok & 31);
    const bool first = (seen[tok >> 5] & bit) == 0u;
    seen[tok >> 5] |= bit;
    row[tok] = row[tok] - (first ? f + p : f);
  }
}

}  // namespace b200

using namespace b200;

// dtype: 0 = bf16 logits, 1 = fp32 logits. All per-row parameter arrays may be null (defaults:
// temperature 1, top_k 1 (greedy), top_p 1, penalty 1). out_max (optional) receives the winning
// score/logit per row — used by the vocab-parallel reduction. step_ptr: optional device int64
// mixed into the RNG stream so CUDA-graph replays draw fresh numbers.
GLLM_EXPORT int gllm_sample(const void* logits, int dtype, int64_t ld, void* out_tokens, int B, int V,
                            const void* temperature, const void* top_k, const void* top_p,
                            const void* rep_penalty, const void* seen, int seen_words,
                            const void* slot_idx, uint64_t seed,
                            const void* step_ptr, void* out_max, int vocab_offset, const void* bias, int64_t bias_ld,
                            const void* bias_slot, const void* seeds, const void* seed_pos, void* stream) {
  if (B <= 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == 0) {
    sample_kernel<__nv_bfloat16><<<B, kSampleThreads, 0, st>>>(
        reinterpret_cast<const __nv_bfloat16*>(logits), ld, V, reinterpret_cast<const float*>(temperature),
        reinterpret_cast<const int32_t*>(top_k), reinterpret_cast<const float*>(top_p),
        reinterpret_cast<const float*>(rep_penalty), reinterpret_cast<const uint32_t*>(seen), seen_words,
        reinterpret_cast<const int32_t*>(slot_idx), seed,
        reinterpret_cast<const int64_t*>(step_ptr), reinterpret_cast<int32_t*>(out_tokens),
        reinterpret_cast<float*>(out_max), vocab_offset, reinterpret_cast<const float*>(bias), bias_ld,
        reinterpret_cast<const int32_t*>(bias_slot), reinterpret_cast<const int64_t*>(seeds),
        reinterpret_cast<const int32_t*>(seed_pos));
  } else {
    sample_kernel<float><<<B, kSampleThreads, 0, st>>>(
        reinterpret_cast<const float*>(logits), ld, V, reinterpret_cast<const float*>(temperature),
        reinterpret_cast<const int32_t*>(top_k), reinterpret_cast<const float*>(top_p),
        reinterpret_cast<const float*>(rep_penalty), reinterpret_cast<const uint32_t*>(seen), seen_words,
        reinterpret_cast<const int32_t*>(slot_idx), seed,
        reinterpret_cast<const int64_t*>(step_ptr), reinterpret_cast<int32_t*>(out_tokens),
        reinterpret_cast<float*>(out_max), vocab_offset, reinterpret_cast<const float*>(bias), bias_ld,
        reinterpret_cast<const int32_t*>(bias_slot), reinterpret_cast<const int64_t*>(seeds),
        reinterpret_cast<const int32_t*>(seed_pos));
  }
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

// Vocab-parallel sampling, stage 1: this rank's record per row, `out` [B, 2C+4] fp32 (see vp_candidates_kernel).
GLLM_EXPORT int gllm_vp_candidates(const void* logits, int dtype, int64_t ld, void* out, int B, int V, int V_full,
                                   int C, const void* temperature, const void* top_k, const void* top_p,
                                   const void* rep_penalty, const void* seen, int seen_words, const void* slot_idx,
                                   uint64_t seed, const void* step_ptr, int vocab_offset, const void* bias,
                                   int64_t bias_ld, const void* bias_slot, const void* seeds, const void* seed_pos,
                                   void* stream) {
  if (B <= 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
#define VP_CAND(T_)                                                                                                \
  vp_candidates_kernel<T_><<<B, kSampleThreads, 0, st>>>(                                                          \
      reinterpret_cast<const T_*>(logits), ld, V, V_full, C, reinterpret_cast<const float*>(temperature),          \
      reinterpret_cast<const int32_t*>(top_k), reinterpret_cast<const float*>(top_p),                              \
      reinterpret_cast<const float*>(rep_penalty), reinterpret_cast<const uint32_t*>(seen), seen_words,            \
      reinterpret_cast<const int32_t*>(slot_idx), seed, reinterpret_cast<const int64_t*>(step_ptr),                \
      reinterpret_cast<float*>(out), vocab_offset, reinterpret_cast<const float*>(bias), bias_ld,              \
      reinterpret_cast<const int32_t*>(bias_slot), reinterpret_cast<const int64_t*>(seeds),                        \
      reinterpret_cast<const int32_t*>(seed_pos))
  if (dtype == 0) VP_CAND(__nv_bfloat16); else VP_CAND(float);
#undef VP_CAND
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

// Vocab-parallel sampling, stage 2: `gathered` [tp, B, 2C+4] = every rank's stage-1 records.
GLLM_EXPORT int gllm_vp_final(const void* gathered, int tp, int B, int C, int V_full, const void* top_k,
                              const void* top_p, uint64_t seed, const void* step_ptr, void* out_tokens,
                              const void* seeds, const void* seed_pos, void* stream) {
  if (B <= 0) return 0;
  vp_final_kernel<<<B, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float*>(gathered), tp, B, C, V_full, reinterpret_cast<const int32_t*>(top_k),
      reinterpret_cast<const float*>(top_p), seed, reinterpret_cast<const int64_t*>(step_ptr),
      reinterpret_cast<int32_t*>(out_tokens), reinterpret_cast<const int64_t*>(seeds),
      reinterpret_cast<const int32_t*>(seed_pos));
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

// Log-probabilities, stage 1: `out` [E, 2N+3] fp32, one record per requesting row (see logprobs_shard_kernel).
// rows: int32 [E] logits row of each requesting row (null: row i); tokens: int32 sampled token per logits row;
// V: real vocabulary columns of this shard; vocab_offset: token id of its column 0.
GLLM_EXPORT int gllm_logprobs_shard(const void* logits, int dtype, int64_t ld, int E, int V, int N, const void* rows,
                                    const void* tokens, void* out, int vocab_offset, void* stream) {
  if (N < 0 || N > kMaxLogprobs) return 2;
  if (E <= 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
#define LP_SHARD(T_)                                                                                               \
  logprobs_shard_kernel<T_><<<E, kSampleThreads, 0, st>>>(                                                         \
      reinterpret_cast<const T_*>(logits), ld, V, N, reinterpret_cast<const int32_t*>(rows),                       \
      reinterpret_cast<const int32_t*>(tokens), reinterpret_cast<float*>(out), vocab_offset)
  if (dtype == 0) LP_SHARD(__nv_bfloat16); else LP_SHARD(float);
#undef LP_SHARD
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

// Prompt log-probabilities, stage 1: `out` [Q, 2N+3] fp32 for N in {0, 1} (see prompt_logprobs_shard_kernel).
// logits [Q, ld]: row q is scored against targets[q]; V: real vocabulary columns of this shard; vocab_offset: token id
// of its column 0.
GLLM_EXPORT int gllm_prompt_logprobs_shard(const void* logits, int dtype, int64_t ld, int Q, int V, int N,
                                           const void* targets, void* out, int vocab_offset, void* stream) {
  if (N < 0 || N > 1) return 2;
  if (Q <= 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
#define PLP_SHARD(T_)                                                                                              \
  prompt_logprobs_shard_kernel<T_><<<Q, kPromptLpThreads, 0, st>>>(                                                \
      reinterpret_cast<const T_*>(logits), ld, V, N, reinterpret_cast<const int32_t*>(targets),                    \
      reinterpret_cast<float*>(out), vocab_offset)
  if (dtype == 0) PLP_SHARD(__nv_bfloat16); else PLP_SHARD(float);
#undef PLP_SHARD
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

// Log-probabilities, stage 2: `gathered` [tp, E, 2N+3] = every rank's stage-1 records -> `out` [E, 1 + 2N] fp32.
GLLM_EXPORT int gllm_logprobs_final(const void* gathered, int tp, int E, int N, void* out, void* stream) {
  if (N < 0 || N > kMaxLogprobs || tp <= 0) return 2;
  if (E <= 0) return 0;
  const size_t smem = static_cast<size_t>(2) * tp * N * sizeof(float);
  logprobs_final_kernel<<<E, 256, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float*>(gathered), tp, E, N, reinterpret_cast<float*>(out));
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

GLLM_EXPORT int gllm_mark_seen(void* seen, int seen_words, const void* rows, const void* tokens, int n,
                               void* stream) {
  if (n <= 0) return 0;
  mark_seen_kernel<<<(n + 255) / 256, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<uint32_t*>(seen), seen_words, reinterpret_cast<const int32_t*>(rows),
      reinterpret_cast<const int32_t*>(tokens), n);
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

// Bias rows: charge the sampled token of every emitting row that has one (see bias_account_kernel).
GLLM_EXPORT int gllm_bias_account(void* bias, int64_t bias_ld, void* out_seen, int seen_words, const void* bias_slot,
                                  const void* tokens, const void* freq, const void* pres, int E, void* stream) {
  if (E <= 0) return 0;
  bias_account_kernel<<<(E + 127) / 128, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<float*>(bias), bias_ld, reinterpret_cast<uint32_t*>(out_seen), seen_words,
      reinterpret_cast<const int32_t*>(bias_slot), reinterpret_cast<const int32_t*>(tokens),
      reinterpret_cast<const float*>(freq), reinterpret_cast<const float*>(pres), E);
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}

// Bias rows: rebuild R (re)assigned slots (see bias_rebuild_kernel). pen: fp32 [R, 2] (frequency, presence);
// lb_off / out_off: int32 [R + 1] offsets into lb_ids / lb_vals and out_toks.
GLLM_EXPORT int gllm_bias_rebuild(void* bias, int64_t bias_ld, void* out_seen, int seen_words, int V, int R,
                                  const void* slots, const void* pen, const void* lb_off, const void* lb_ids,
                                  const void* lb_vals, const void* out_off, const void* out_toks, void* stream) {
  if (R <= 0) return 0;
  bias_rebuild_kernel<<<R, 1024, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<float*>(bias), bias_ld, reinterpret_cast<uint32_t*>(out_seen), seen_words, V,
      reinterpret_cast<const int32_t*>(slots), reinterpret_cast<const float*>(pen),
      reinterpret_cast<const int32_t*>(lb_off), reinterpret_cast<const int32_t*>(lb_ids),
      reinterpret_cast<const float*>(lb_vals), reinterpret_cast<const int32_t*>(out_off),
      reinterpret_cast<const int32_t*>(out_toks));
  CUDA_CHECK_RET(cudaGetLastError());
  return 0;
}
