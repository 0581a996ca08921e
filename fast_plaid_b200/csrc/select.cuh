// The canonical ranking order and the block-wide selection steps that use it (device only).
//
// Every stage that keeps "the best few" -- the probe, K3b, the shard threshold, K6 and the merge -- uses one rule:
// larger value first, then smaller id (DESIGN §2, "Ties").  It is one 64-bit key,
//   (order-preserving value key << 32) | (0xffffffff - id),
// so that a larger key ranks first; key 0 is an empty slot.  Ids are truncated to 32 bits.
//
// The block-wide steps assume 1024-thread blocks and are called by every thread of the block, except
// warp_find_bucket (warp 0 only).
#pragma once
#include "common.cuh"

constexpr int SEL_THREADS = 1024;
constexpr int SEL_BINS = 2048;  // linear value buckets of the bucket searches

// ---- keys ----
__device__ __forceinline__ uint64_t rank_key(uint32_t value_key, uint32_t id) {
  return (uint64_t(value_key) << 32) | uint64_t(0xffffffffu - id);
}
__device__ __forceinline__ uint64_t rank_key_f32(float v, uint32_t id) { return rank_key(f32_key(v), id); }
__device__ __forceinline__ uint64_t rank_key_f16(uint16_t h, uint32_t id) { return rank_key(f16_key(h), id); }
__device__ __forceinline__ uint32_t rank_key_id(uint64_t key) { return 0xffffffffu - uint32_t(key); }
__device__ __forceinline__ uint32_t rank_key_vkey(uint64_t key) { return uint32_t(key >> 32); }  // the value key
__device__ __forceinline__ float rank_key_f32_value(uint64_t key) { return f32_unkey(rank_key_vkey(key)); }

// ---- block-wide steps ----

// Bitonic sort of keys[0, P) into descending order, P a power of two; pay[0, P), when given, is permuted along with
// the keys (a payload of any trivially copyable type: the merge carries 16-bit record indices to save shared
// memory).  Ends with __syncthreads().
template <typename Pay = uint32_t>
__device__ __forceinline__ void block_sort_desc(uint64_t* keys, int P, Pay* pay = nullptr) {
  const int tid = threadIdx.x;
  for (int k = 2; k <= P; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < P; i += SEL_THREADS) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const bool up = (i & k) == 0;
          const uint64_t x = keys[i], y = keys[ixj];
          if ((x < y) == up) {
            keys[i] = y;
            keys[ixj] = x;
            if (pay) {
              const Pay px = pay[i];
              pay[i] = pay[ixj];
              pay[ixj] = px;
            }
          }
        }
      }
      __syncthreads();
    }
  }
}

// Min and max over the threads' partial mn / mx (fminf / fmaxf, so NaNs are skipped); every thread gets them.
// s_red: 64 floats of shared memory.  Contains one __syncthreads().
__device__ __forceinline__ void block_min_max(float& mn, float& mx, float* s_red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, off));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
  }
  if (lane == 0) {
    s_red[warp] = mn;
    s_red[32 + warp] = mx;
  }
  __syncthreads();
  mn = s_red[lane];
  mx = s_red[32 + lane];
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, off));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
  }
}

// The SEL_BINS linear value buckets from lo, `scale` buckets per unit value (scale = (SEL_BINS - 1) / range): a
// larger v never falls into a lower bucket, so every value of a higher bucket is strictly larger.
//
// NaN is outside this order: value_bucket puts it in bucket 0, while rank_key_f32 ranks a (positive) NaN above
// +inf.  So a selection that mixes the bucket search with the key order (K3b's fast and radix paths) would rank a
// NaN differently by path.  No NaN reaches one: every score is a sum of maxima (__hmax2 in K3 / K5, K7's maxima)
// that drop NaN operands.  (Those maxima start from the padding sentinel -10000, so centroid scores below it are
// clipped to it, which the reference does only when the batch is padded: the selection tests keep their injected
// tables above it.)
__device__ __forceinline__ int value_bucket(float v, float lo, float scale) {
  return min(SEL_BINS - 1, max(0, __float2int_rz((v - lo) * scale)));
}

// Warp 0: the bucket t with count(bucket > t) < need <= count(bucket >= t) of a histogram of nbins (a multiple of
// 32) buckets in ascending order.  The one lane that finds it returns true with *t and *rest = need - count(bucket >
// t), the entries still to take from bucket t; when the histogram holds fewer than need entries, no lane does.
__device__ __forceinline__ bool warp_find_bucket(const int* hist, int nbins, int need, int* t, int* rest) {
  const int lane = threadIdx.x & 31;
  const int per = nbins / 32;  // buckets per lane, lane 31 owns the top ones
  int mine = 0;
  for (int k = 0; k < per; ++k) mine += hist[lane * per + k];
  int above = 0;  // entries of the lanes above this one
  for (int l = 31; l >= 0; --l) {
    const int c = __shfl_sync(0xffffffffu, mine, l);
    if (l > lane) above += c;
  }
  if (above >= need || above + mine < need) return false;
  int cum = above, d = lane * per + per - 1;
  for (; d > lane * per; --d) {
    const int h = hist[d];
    if (cum + h >= need) break;
    cum += h;
  }
  *t = d;
  *rest = need - cum;
  return true;
}
