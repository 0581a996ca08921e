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
constexpr int SEL_BCAP = 2048;  // capacity of block_select_keys's threshold bucket on the fast path
constexpr int SEL_FV = 8;       // independent loads in flight per thread in block_select_keys's value passes
constexpr int SEL_VPT = 4;      // ... and in its radix passes

// Digits of the 64-bit key for the radix passes, most significant first: 11+11+10 bits cover the value key, the rest
// only matters when values tie at the threshold.
static __constant__ int SEL_DIGIT_LO[6] = {53, 42, 32, 21, 10, 0};
static __constant__ int SEL_DIGIT_W[6] = {11, 11, 10, 11, 11, 10};

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

// Exclusive prefix of the threads' counts c over the block; *total gets the sum.  warp_sums: 32 ints of shared memory.
// Contains two __syncthreads().
__device__ __forceinline__ int block_exclusive_scan(int c, int* warp_sums, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = c;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, off);
    if (lane >= off) incl += v;
  }
  if (lane == 31) warp_sums[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    const int ws = warp_sums[lane];
    int wincl = ws;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, wincl, off);
      if (lane >= off) wincl += v;
    }
    warp_sums[lane] = wincl - ws;
    if (lane == 31) *total = wincl;
  }
  __syncthreads();
  return warp_sums[warp] + incl - c;
}

// The `need` (>= 1) largest keys among entries [0, n) of a key source, sorted descending into keys[0, Rp2) (Rp2 a
// power of two >= need, the slots past them 0); returns their number, min(need, present entries).  The source gives
// load(i), one independent load per entry (SEL_FV or SEL_VPT of them in flight per thread), and from what it loaded
// present(x) (an absent entry is never selected), value(x) and key(x, i): the keys of present entries are distinct,
// and the high half of each is the value key of its fp32 value.  empty() stands in for the loads past n: it is absent,
// or its value is NaN.  A dense source has every entry present, so the first pass does not count them (the count
// would hold every load's predicate until its value arrives).  I is the type of the entry index.
//
// When more than `need` entries are present, SEL_BINS linear value buckets over the values' [min, max] isolate the
// bucket of the need-th, and only that bucket is ordered by the whole key.  value_bucket is monotone, so every entry
// of a higher bucket is strictly larger: the selection is exact.  (The radix passes below start from the top bits of
// the key, where a row's values share sign, exponent and the leading mantissa bits: a handful of hot bins, so every
// entry pays a ballot + match_any + contended shared atomic, three passes long.)  When the range is degenerate or that
// bucket holds more than SEL_BCAP entries, radix passes over the 64-bit key find the need-th key T, and every key >= T
// is taken.
template <typename Src, typename I>
__device__ __forceinline__ int block_select_keys(const Src& src, I n, int need, uint64_t* keys, int Rp2) {
  using X = decltype(src.load(I(0)));
  __shared__ int hist[SEL_BINS];
  __shared__ uint64_t bkeys[SEL_BCAP];  // fast path: keys of the threshold bucket
  __shared__ float s_red[64];
  __shared__ uint64_t s_prefix, s_mask;
  __shared__ int s_need, s_hd, s_cnt, s_cnt2, s_fast, s_present;
  const int tid = threadIdx.x, lane = tid & 31;
  float mn = INFINITY, mx = -INFINITY;
  int present = 0;
  for (I i0 = tid; i0 < n; i0 += SEL_THREADS * SEL_FV) {
    X x[SEL_FV];
#pragma unroll
    for (int u = 0; u < SEL_FV; ++u) x[u] = (i0 + u * SEL_THREADS < n) ? src.load(i0 + u * SEL_THREADS) : Src::empty();
#pragma unroll
    for (int u = 0; u < SEL_FV; ++u) {
      const bool in = src.present(x[u]);
      const float v = in ? src.value(x[u]) : NAN;  // fminf / fmaxf skip NaN
      mn = fminf(mn, v);
      mx = fmaxf(mx, v);
      if constexpr (!Src::dense) present += in;
    }
  }
  for (int i = tid; i < SEL_BINS; i += SEL_THREADS) hist[i] = 0;
  if (tid == 0) {
    s_cnt = 0;
    s_cnt2 = 0;
    s_fast = 0;
    s_present = Src::dense ? int(n) : 0;
  }
  block_min_max(mn, mx, s_red);
  if constexpr (!Src::dense) {
    if (present) atomicAdd(&s_present, present);
    __syncthreads();
  }
  if (s_present <= need) {  // every present entry is selected
    for (I i = tid; i < n; i += SEL_THREADS) {
      const X x = src.load(i);
      if (src.present(x)) keys[atomicAdd(&s_cnt, 1)] = src.key(x, i);
    }
    __syncthreads();
  } else {
    const float range = mx - mn;
    // finite, non-degenerate range (NaN / inf values or all-equal values take the radix path)
    const bool usable = range > 0.f && range < 3.0e38f;
    const float scale = usable ? float(SEL_BINS - 1) / range : 0.f;
    if (usable) {
      for (I i0 = tid; i0 < n; i0 += SEL_THREADS * SEL_FV) {
        X x[SEL_FV];
#pragma unroll
        for (int u = 0; u < SEL_FV; ++u) x[u] = (i0 + u * SEL_THREADS < n) ? src.load(i0 + u * SEL_THREADS) : X{};
#pragma unroll
        for (int u = 0; u < SEL_FV; ++u)
          if (i0 + u * SEL_THREADS < n && src.present(x[u]))
            atomicAdd(&hist[value_bucket(src.value(x[u]), mn, scale)], 1);
      }
      __syncthreads();
      int hd, rest;
      if (tid < 32 && warp_find_bucket(hist, SEL_BINS, need, &hd, &rest)) {
        s_need = rest;
        s_hd = hd;
        s_fast = hist[hd] <= SEL_BCAP ? 1 : 0;
      }
      __syncthreads();
      if (s_fast) {
        const int t = s_hd;
        for (I i0 = tid; i0 < n; i0 += SEL_THREADS * SEL_FV) {
          X x[SEL_FV];
#pragma unroll
          for (int u = 0; u < SEL_FV; ++u) x[u] = (i0 + u * SEL_THREADS < n) ? src.load(i0 + u * SEL_THREADS) : X{};
#pragma unroll
          for (int u = 0; u < SEL_FV; ++u) {
            const I i = i0 + u * SEL_THREADS;
            if (i < n && src.present(x[u])) {
              const int bk = value_bucket(src.value(x[u]), mn, scale);
              if (bk > t) {
                keys[atomicAdd(&s_cnt, 1)] = src.key(x[u], i);  // fewer than need of these
              } else if (bk == t) {
                bkeys[atomicAdd(&s_cnt2, 1)] = src.key(x[u], i);  // at most SEL_BCAP of these
              }
            }
          }
        }
        __syncthreads();
        const int c2 = s_cnt2, need2 = s_need;
        for (int i = c2 + tid; i < SEL_BCAP; i += SEL_THREADS) bkeys[i] = 0ull;
        __syncthreads();
        block_sort_desc(bkeys, SEL_BCAP);
        const int c1 = s_cnt;
        for (int i = tid; i < need2; i += SEL_THREADS) keys[c1 + i] = bkeys[i];
        __syncthreads();
        if (tid == 0) s_cnt = c1 + need2;  // == need
        __syncthreads();
      }
    }
    if (!s_fast) {  // radix passes over the 64-bit key: the threshold key T, then every key >= T
      if (tid == 0) {
        s_need = need;
        s_prefix = 0;
        s_mask = 0;
      }
      const I stride = SEL_THREADS * SEL_VPT;
      const I n_up = (n + stride - 1) / stride * stride;  // whole warps iterate together
      for (int pass = 0; pass < 6; ++pass) {
        const int lo = SEL_DIGIT_LO[pass], width = SEL_DIGIT_W[pass];
        const uint64_t dmask = (1ull << width) - 1ull;
        for (int i = tid; i < SEL_BINS; i += SEL_THREADS) hist[i] = 0;
        __syncthreads();
        const uint64_t prefix = s_prefix, mask = s_mask;
        for (I i0 = tid; i0 < n_up; i0 += stride) {
          X x[SEL_VPT];
#pragma unroll
          for (int u = 0; u < SEL_VPT; ++u) x[u] = (i0 + u * SEL_THREADS < n) ? src.load(i0 + u * SEL_THREADS) : X{};
#pragma unroll
          for (int u = 0; u < SEL_VPT; ++u) {
            const I i = i0 + u * SEL_THREADS;
            const bool valid = i < n && src.present(x[u]);
            const uint64_t key = valid ? src.key(x[u], i) : 0ull;
            const bool in = valid && ((key & mask) == prefix);
            const unsigned act = __ballot_sync(0xffffffffu, in);
            if (in) {
              const int bin = int((key >> lo) & dmask);
              const unsigned peers = __match_any_sync(act, bin);
              if (lane == __ffs(peers) - 1) atomicAdd(&hist[bin], __popc(peers));
            }
          }
        }
        __syncthreads();
        int d, rest;
        if (tid < 32 && warp_find_bucket(hist, 1 << width, s_need, &d, &rest)) {
          s_need = rest;
          s_hd = hist[d];
          s_prefix = prefix | (uint64_t(d) << lo);
          s_mask = mask | (dmask << lo);
        }
        __syncthreads();
        if (s_hd == s_need) break;  // the whole bucket is selected
      }
      const uint64_t T = s_prefix;  // unprocessed low bits are zero
      for (I i0 = tid; i0 < n_up; i0 += stride) {
        X x[SEL_VPT];
#pragma unroll
        for (int u = 0; u < SEL_VPT; ++u) x[u] = (i0 + u * SEL_THREADS < n) ? src.load(i0 + u * SEL_THREADS) : X{};
#pragma unroll
        for (int u = 0; u < SEL_VPT; ++u) {
          const I i = i0 + u * SEL_THREADS;
          if (i < n && src.present(x[u])) {
            const uint64_t key = src.key(x[u], i);
            if (key >= T) {
              const int pos = atomicAdd(&s_cnt, 1);
              if (pos < Rp2) keys[pos] = key;
            }
          }
        }
      }
    }
  }
  __syncthreads();
  const int cnt = min(s_cnt, Rp2);
  for (int i = cnt + tid; i < Rp2; i += SEL_THREADS) keys[i] = 0ull;
  __syncthreads();
  block_sort_desc(keys, Rp2);
  return cnt;
}

// Row `row` of a ranking (ids and scores [.., top_k], counts [..]): the first min(n, top_k) of the sorted keys[0, n),
// as document doc_id_base + id and score, then -1 / -inf up to top_k; the count is min(n, top_k).
__device__ __forceinline__ void block_write_ranking(const uint64_t* keys, int n, int top_k, int64_t doc_id_base,
                                                    int64_t* out_ids, float* out_scores, int32_t* out_counts,
                                                    int64_t row) {
  const int cnt = min(n, top_k);
  for (int i = threadIdx.x; i < top_k; i += SEL_THREADS) {
    int64_t id = -1;
    float sc = -INFINITY;
    if (i < cnt) {
      id = doc_id_base + int64_t(rank_key_id(keys[i]));
      sc = rank_key_f32_value(keys[i]);
    }
    out_ids[row * top_k + i] = id;
    out_scores[row * top_k + i] = sc;
  }
  if (threadIdx.x == 0) out_counts[row] = cnt;
}

// The group rule over the canonically sorted keys[0, P) (0 for an empty slot): entry i, of group group_of(i), is kept
// when fewer than m entries of its group come before it.  Sorted descending, the (group, position) keys
// rank_key(group, i) put a group's entries side by side with its best position first, so entry j of them is kept when
// the entry m places before it is of another group.  The kept entries' key_of(i) go to gkeys[0, count) in rank order;
// returns count.  gkeys [P] is also the scratch of the (group, position) keys, and may be keys itself when group_of
// and key_of do not read keys; kept: P bytes of shared memory.
template <typename GroupOf, typename KeyOf>
__device__ __forceinline__ int block_group_rule(const uint64_t* keys, int P, int m, GroupOf group_of, KeyOf key_of,
                                                uint64_t* gkeys, unsigned char* kept) {
  __shared__ int warp_sums[32];
  __shared__ int s_total;
  const int tid = threadIdx.x;
  for (int i = tid; i < P; i += SEL_THREADS) {
    gkeys[i] = keys[i] ? rank_key(uint32_t(group_of(i)), uint32_t(i)) : 0ull;
    kept[i] = 0;
  }
  __syncthreads();
  block_sort_desc(gkeys, P);
  for (int j = tid; j < P; j += SEL_THREADS) {
    const uint64_t g = gkeys[j];
    if (g && (j < m || rank_key_vkey(gkeys[j - m]) != rank_key_vkey(g))) kept[rank_key_id(g)] = 1;
  }
  __syncthreads();
  // ordered compaction of the kept positions: thread t owns positions [t * per, (t + 1) * per)
  const int per = P > SEL_THREADS ? P / SEL_THREADS : 1;
  const int i0 = tid * per;
  int c = 0;
  for (int u = 0; u < per; ++u) c += (i0 + u < P && kept[i0 + u]) ? 1 : 0;
  int pos = block_exclusive_scan(c, warp_sums, &s_total);
  for (int u = 0; u < per; ++u)
    if (i0 + u < P && kept[i0 + u]) gkeys[pos++] = key_of(i0 + u);
  __syncthreads();
  return s_total;
}

// Record j in [0, n_shards * R) of query b in a shard merge's gathered records [n_shards, B, R]
__device__ __forceinline__ const fpb_record& merge_record(const fpb_record* all, int B, int R, int b, int j) {
  return all[(int64_t(j / R) * B + b) * R + j % R];
}

// The shard merge's global pruning rule (search.rs:605-619 on the whole index) over query b's `total` records: their
// (approx, doc id) keys sorted descending into keys[0, P) (P a power of two >= total; a padding record, doc_id < 0, is
// an empty key), each slot's record index carried into pay[0, P).  Returns the number of slots kept,
// min(valid records, n_keep).
__device__ __forceinline__ int block_merge_prune(const fpb_record* all, int B, int R, int b, int total, int P,
                                                 int n_keep, uint64_t* keys, uint16_t* pay) {
  __shared__ int s_valid;
  if (threadIdx.x == 0) s_valid = 0;
  __syncthreads();
  int local_valid = 0;
  for (int i = threadIdx.x; i < P; i += SEL_THREADS) {
    uint64_t k = 0;
    if (i < total) {
      const fpb_record rec = merge_record(all, B, R, b, i);
      if (rec.doc_id >= 0) {
        k = rank_key_f32(rec.approx, uint32_t(rec.doc_id));
        ++local_valid;
      }
    }
    keys[i] = k;
    pay[i] = uint16_t(i);
  }
  if (local_valid) atomicAdd(&s_valid, local_valid);
  __syncthreads();
  block_sort_desc(keys, P, pay);
  return min(s_valid, n_keep);
}
