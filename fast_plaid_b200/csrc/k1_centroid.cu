// K1  : centroid scores  S[b][k][q] = fp16( sum_d C[k][d] * q_b[q][d] )     (search.rs:491)
// K1b : per query token, the n_ivf_probe best centroids                      (search.rs:520-528)
//
// v1 data path: legacy tensor-core MMA (mma.sync m16n8k16, fp16 in / fp32 accumulate), one
// rounding to fp16 at the end exactly like ATen's half matmul.  Every CTA keeps a tile of 128
// centroid rows resident (fragments in registers) and streams all query tokens of the batch
// past it, so the centroid table is read from HBM once per batch instead of once per query
// as the reference does.  The epilogue writes S in the [b][k][q] layout the approximate stage
// gathers from (one contiguous Qp*2-byte row per centroid and query) and, per 128-row tile,
// the column maxima that let K1b find the top-n cells by touching ~n tiles instead of all K.
#include "kernels.h"
#include "select.cuh"

namespace {

constexpr int K1_THREADS = 256;
constexpr int K1_ROWS = 128;

template <int D, int QC>
struct K1Smem {
  static constexpr int LDS = D + 8;   // +16 B pad: conflict-free ldmatrix
  static constexpr int STG = QC + 8;
  static constexpr int bytes = (K1_ROWS * LDS + QC * LDS + 8 * 16 * STG + 8 * QC) * 2;
};

template <int D, int QC>
__global__ void __launch_bounds__(K1_THREADS)
k1_centroid_scores_kernel(const __half* __restrict__ C, int K, const __half* __restrict__ Qpad,
                          int B, int Qp, __half* __restrict__ S, __half* __restrict__ tmax,
                          int n_tiles, int b_per_cta) {
  constexpr int LDS = K1Smem<D, QC>::LDS;
  constexpr int STG = K1Smem<D, QC>::STG;
  constexpr int NT = QC / 8;
  constexpr int KS = D / 16;
  static_assert(NT % 2 == 0, "QC must be a multiple of 16");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __half* Cs = reinterpret_cast<__half*>(smem_raw);
  __half* Qs = Cs + K1_ROWS * LDS;
  __half* stage = Qs + QC * LDS;
  __half* cmax = stage + 8 * 16 * STG;

  const int tile = blockIdx.x;
  const int row0 = tile * K1_ROWS;
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;

  for (int i = tid; i < K1_ROWS * (D / 8); i += K1_THREADS) {
    const int r = i / (D / 8), c8 = i % (D / 8);
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (row0 + r < K) v = *reinterpret_cast<const uint4*>(C + int64_t(row0 + r) * D + c8 * 8);
    *reinterpret_cast<uint4*>(Cs + r * LDS + c8 * 8) = v;
  }
  __syncthreads();

  uint32_t a[KS][4];
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) {
    const uint32_t addr = smem_u32(Cs + (warp * 16 + (lane & 15)) * LDS + ks * 16 + (lane >> 4) * 8);
    ldmatrix_x4(a[ks][0], a[ks][1], a[ks][2], a[ks][3], addr);
  }

  const int g = lane >> 2, t = lane & 3;
  const bool valid0 = (row0 + warp * 16 + g) < K;
  const bool valid1 = (row0 + warp * 16 + g + 8) < K;
  const __half2 ninf2 = __half2half2(__ushort_as_half(0xFC00));
  __half* st = stage + warp * 16 * STG;

  const int b_begin = blockIdx.y * b_per_cta;
  const int b_end = min(B, b_begin + b_per_cta);
  for (int b = b_begin; b < b_end; ++b) {
    for (int qc0 = 0; qc0 < Qp; qc0 += QC) {
      __syncthreads();  // previous round done with Qs / cmax
      for (int i = tid; i < QC * (D / 8); i += K1_THREADS) {
        const int n = i / (D / 8), c8 = i % (D / 8);
        *reinterpret_cast<uint4*>(Qs + n * LDS + c8 * 8) =
            *reinterpret_cast<const uint4*>(Qpad + (int64_t(b) * Qp + qc0 + n) * D + c8 * 8);
      }
      __syncthreads();

      float acc[NT][4];
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
        for (int nt = 0; nt < NT; nt += 2) {
          const int mat = lane >> 3;
          const int n = (nt + (mat >> 1)) * 8 + (lane & 7);
          const int k = ks * 16 + (mat & 1) * 8;
          uint32_t b0, b1, b2, b3;
          ldmatrix_x4(b0, b1, b2, b3, smem_u32(Qs + n * LDS + k));
          mma_16816(acc[nt], a[ks], b0, b1);
          mma_16816(acc[nt + 1], a[ks], b2, b3);
        }
      }

#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const uint32_t p0 = pack_half2_rn(acc[nt][0], acc[nt][1]);
        const uint32_t p1 = pack_half2_rn(acc[nt][2], acc[nt][3]);
        *reinterpret_cast<uint32_t*>(st + g * STG + nt * 8 + 2 * t) = p0;
        *reinterpret_cast<uint32_t*>(st + (g + 8) * STG + nt * 8 + 2 * t) = p1;
        __half2 m = __hmax2(valid0 ? u32_as_half2(p0) : ninf2, valid1 ? u32_as_half2(p1) : ninf2);
        m = __hmax2(m, u32_as_half2(__shfl_xor_sync(0xffffffffu, half2_as_u32(m), 4)));
        m = __hmax2(m, u32_as_half2(__shfl_xor_sync(0xffffffffu, half2_as_u32(m), 8)));
        m = __hmax2(m, u32_as_half2(__shfl_xor_sync(0xffffffffu, half2_as_u32(m), 16)));
        if (g == 0) *reinterpret_cast<uint32_t*>(cmax + warp * QC + nt * 8 + 2 * t) = half2_as_u32(m);
      }
      __syncwarp();
      // the warp's 16 x QC block: rows are contiguous in S when QC == Qp
      for (int i = lane; i < 16 * (QC / 8); i += 32) {
        const int r = i / (QC / 8), c8 = i % (QC / 8);
        const int row = row0 + warp * 16 + r;
        if (row < K)
          *reinterpret_cast<uint4*>(S + (int64_t(b) * K + row) * Qp + qc0 + c8 * 8) =
              *reinterpret_cast<const uint4*>(st + r * STG + c8 * 8);
      }
      __syncthreads();
      if (tid < QC) {
        __half m = cmax[tid];
#pragma unroll
        for (int w = 1; w < 8; ++w) m = __hmax(m, cmax[w * QC + tid]);
        tmax[(int64_t(b) * Qp + qc0 + tid) * n_tiles + tile] = m;
      }
    }
  }
}

// ---- warp-held sorted top-n list (lane i holds the i-th best key; 0 = empty) -----------
__device__ __forceinline__ uint64_t shfl64(uint64_t v, int src) {
  uint32_t lo = __shfl_sync(0xffffffffu, uint32_t(v), src);
  uint32_t hi = __shfl_sync(0xffffffffu, uint32_t(v >> 32), src);
  return (uint64_t(hi) << 32) | lo;
}
__device__ __forceinline__ uint64_t shfl_up64(uint64_t v) {
  uint32_t lo = __shfl_up_sync(0xffffffffu, uint32_t(v), 1);
  uint32_t hi = __shfl_up_sync(0xffffffffu, uint32_t(v >> 32), 1);
  return (uint64_t(hi) << 32) | lo;
}
__device__ __forceinline__ void topn_insert(uint64_t& mine, int n, uint64_t x, int lane) {
  const unsigned gt = __ballot_sync(0xffffffffu, mine > x);
  const int pos = __popc(gt);
  const uint64_t up = shfl_up64(mine);
  if (pos < n) {
    if (lane == pos) mine = x;
    else if (lane > pos) mine = up;
    if (lane >= n) mine = 0;
  }
}
// Offer the keys held by the lanes (one each); keys equal to 0 are ignored.
__device__ __forceinline__ void topn_offer(uint64_t& mine, int n, uint64_t key, int lane) {
  uint64_t thr = shfl64(mine, n - 1);
  unsigned bits = __ballot_sync(0xffffffffu, key > thr);
  while (bits) {
    const int src = __ffs(bits) - 1;
    bits &= bits - 1;
    const uint64_t x = shfl64(key, src);
    if (x > thr) {  // uniform: x and thr are warp-uniform
      topn_insert(mine, n, x, lane);
      thr = shfl64(mine, n - 1);
    }
  }
}

// One warp per (query, query token).  Canonical tie rule: larger score first, then smaller
// centroid id (the reference's topk(sorted=false) leaves ties implementation-defined).
__global__ void __launch_bounds__(256)
k1b_probe_kernel(const __half* __restrict__ S, const __half* __restrict__ tmax, int K, int B, int Q,
                 int Qp, int n_tiles, int n_probe, int32_t* __restrict__ cells) {
  const int lane = threadIdx.x & 31;
  const int wg = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (wg >= B * Q) return;
  const int b = wg / Q, q = wg % Q;
  const uint16_t* tm = reinterpret_cast<const uint16_t*>(tmax) + (int64_t(b) * Qp + q) * n_tiles;

  // pass 1: n-th largest tile maximum -> tau (any top-n element lives in a tile whose max >= tau)
  uint64_t mine = 0;
  for (int base = 0; base < n_tiles; base += 32) {
    const int tix = base + lane;
    uint64_t key = 0;
    if (tix < n_tiles) key = rank_key_f16(tm[tix], uint32_t(tix));
    topn_offer(mine, n_probe, key, lane);
  }
  const uint32_t tau = rank_key_vkey(shfl64(mine, n_probe - 1));  // 0 when fewer than n tiles

  // pass 2: exact top-n over the rows of the qualifying tiles
  mine = 0;
  const uint16_t* Sb = reinterpret_cast<const uint16_t*>(S) + int64_t(b) * K * Qp + q;
  for (int base = 0; base < n_tiles; base += 32) {
    const int tix = base + lane;
    bool qual = false;
    if (tix < n_tiles) qual = f16_key(tm[tix]) >= tau;
    unsigned tb = __ballot_sync(0xffffffffu, qual);
    while (tb) {
      const int tl = __ffs(tb) - 1;
      tb &= tb - 1;
      const int r0 = (base + tl) * K1_ROWS;
#pragma unroll
      for (int j = 0; j < K1_ROWS / 32; ++j) {
        const int row = r0 + j * 32 + lane;
        uint64_t key = 0;
        if (row < K) {
          const uint32_t k16 = f16_key(Sb[int64_t(row) * Qp]);
          if (k16 >= tau) key = rank_key(k16, uint32_t(row));
        }
        topn_offer(mine, n_probe, key, lane);
      }
    }
  }
  if (lane < n_probe) {
    int32_t c = -1;
    if (mine != 0) c = int32_t(rank_key_id(mine));
    cells[(int64_t(b) * Q + q) * n_probe + lane] = c;
  }
}

// Subset variant (search.rs:494-517): the top-n is taken over the centroids that occur in the
// subset's documents only (clist, ascending), n = min(n_ivf_probe, #such centroids).
__global__ void __launch_bounds__(256)
k1b_probe_subset_kernel(const __half* __restrict__ S, int K, int B, int Q, int Qp, int n_probe,
                        const int32_t* __restrict__ clist, const int32_t* __restrict__ n_clist,
                        int32_t* __restrict__ cells) {
  const int lane = threadIdx.x & 31;
  const int wg = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (wg >= B * Q) return;
  const int b = wg / Q, q = wg % Q;
  const int nc = n_clist[b];
  const int n = min(n_probe, nc);
  const int32_t* cl = clist + int64_t(b) * K;
  const uint16_t* Sb = reinterpret_cast<const uint16_t*>(S) + int64_t(b) * K * Qp + q;
  uint64_t mine = 0;
  if (n > 0) {
    for (int base = 0; base < nc; base += 32) {
      const int i = base + lane;
      uint64_t key = 0;
      if (i < nc) {
        const int c = cl[i];
        key = rank_key_f16(Sb[int64_t(c) * Qp], uint32_t(c));
      }
      topn_offer(mine, n, key, lane);
    }
  }
  if (lane < n_probe) {
    int32_t c = -1;
    if (lane < n && mine != 0) c = int32_t(rank_key_id(mine));
    cells[(int64_t(b) * Q + q) * n_probe + lane] = c;
  }
}

// ---- wide probe (FPB_WARP_PROBE < n <= FPB_MAX_PROBE): one 1024-thread CTA per (query, query token) -------------
// The n best keys are found by an exact threshold on the 16-bit value key (two levels of 256-bucket histograms and
// warp_find_bucket), then every key above the threshold and the first keys at it in id order are gathered and
// block_sort_desc puts them in rank order.  Items are visited in warp groups of 32 consecutive ones, so that a source
// can skip a whole group by a bound on its keys (the rows of one tile by the tile maximum).
struct WideSmem {
  uint64_t keys[FPB_MAX_PROBE];
  int hist[256];
  int wsum[32];
  int sel[2];  // threshold bucket (-1: fewer keys than needed) and the entries still to take from it
  int n_out;
};

// The tile maxima of one S column
struct TileItems {
  const uint16_t* tm;
  int n_tiles;
  __device__ int count() const { return n_tiles; }
  __device__ bool live(int, uint32_t) const { return true; }
  __device__ uint32_t key(int i) const { return f16_key(tm[i]); }
};
// The rows of one S column; the 32-row group starting at g lies in tile g / K1_ROWS
struct RowItems {
  const uint16_t* col;
  const uint16_t* tm;
  int K, Qp;
  __device__ int count() const { return K; }
  __device__ bool live(int g, uint32_t floor) const { return f16_key(tm[g / K1_ROWS]) >= floor; }
  __device__ uint32_t key(int i) const { return f16_key(col[int64_t(i) * Qp]); }
  __device__ uint32_t id(int i) const { return uint32_t(i); }
};
// The rows of one S column named by an ascending centroid list
struct ListItems {
  const uint16_t* col;
  const int32_t* cl;
  int nc, Qp;
  __device__ int count() const { return nc; }
  __device__ bool live(int, uint32_t) const { return true; }
  __device__ uint32_t key(int i) const { return f16_key(col[int64_t(cl[i]) * Qp]); }
  __device__ uint32_t id(int i) const { return uint32_t(cl[i]); }
};

// f(key, i) for every item i whose key is >= floor
template <class Items, class F>
__device__ __forceinline__ void wide_for_each(const Items& it, uint32_t floor, F f) {
  const int n = it.count(), lane = threadIdx.x & 31;
  for (int g = (threadIdx.x >> 5) * 32; g < n; g += SEL_THREADS) {
    if (!it.live(g, floor)) continue;  // warp-uniform
    const int i = g + lane;
    if (i < n) {
      const uint32_t k = it.key(i);
      if (k >= floor) f(k, i);
    }
  }
}

// The threshold T of the `need` (>= 1) best keys >= floor: count(key > T) < need <= count(key >= T), with
// *rest = need - count(key > T) and *ties = count(key == T).  False, in every thread, when fewer than `need` keys
// are >= floor.
template <class Items>
__device__ bool wide_threshold(const Items& it, uint32_t floor, int need, WideSmem& s, uint32_t* T, int* rest,
                               int* ties) {
  const int tid = threadIdx.x;
  int hi = 0;
  for (int level = 0; level < 2; ++level) {
    for (int i = tid; i < 256; i += SEL_THREADS) s.hist[i] = 0;
    if (tid == 0) s.sel[0] = -1;
    __syncthreads();
    if (level == 0) {
      wide_for_each(it, floor, [&](uint32_t k, int) { atomicAdd(&s.hist[k >> 8], 1); });
    } else {
      wide_for_each(it, max(floor, uint32_t(hi) << 8), [&](uint32_t k, int) {
        if (int(k >> 8) == hi) atomicAdd(&s.hist[k & 255], 1);
      });
    }
    __syncthreads();
    if (tid < 32) {
      int t, r;
      if (warp_find_bucket(s.hist, 256, need, &t, &r)) {
        s.sel[0] = t;
        s.sel[1] = r;
      }
    }
    __syncthreads();
    const int t = s.sel[0], r = s.sel[1];
    if (t < 0) return false;
    if (level == 0) {
      hi = t;
      need = r;
    } else {
      *T = (uint32_t(hi) << 8) | uint32_t(t);
      *rest = r;
      *ties = s.hist[t];
    }
    __syncthreads();  // everyone has read hist and sel
  }
  return true;
}

// s.keys[0, s.n_out) = the keys above T and the first `rest` items at T in item order (all of them when there are
// `ties` == rest), as 64-bit rank keys.  Items must be in ascending id order.
template <class Items>
__device__ void wide_gather(const Items& it, uint32_t T, int rest, int ties, WideSmem& s) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s.n_out = 0;
  __syncthreads();
  auto push = [&](uint32_t k, int i) { s.keys[atomicAdd(&s.n_out, 1)] = rank_key(k, it.id(i)); };
  if (ties == rest) {
    wide_for_each(it, T, push);
    __syncthreads();
    return;
  }
  wide_for_each(it, T + 1, push);
  // the ties in item order: 1024-item chunks and a block-wide count of the ties before each item
  const int n = it.count();
  int base = 0;
  for (int c0 = 0; c0 < n && base < rest; c0 += SEL_THREADS) {
    const int i = c0 + tid;
    bool tie = false;
    if (i < n && it.live(i & ~31, T)) tie = it.key(i) == T;
    const unsigned bal = __ballot_sync(0xffffffffu, tie);
    __syncthreads();  // the previous chunk is done with wsum
    if (lane == 0) s.wsum[warp] = __popc(bal);
    __syncthreads();
    int before = base + __popc(bal & ((1u << lane) - 1u)), total = 0;
    for (int w = 0; w < 32; ++w) {
      const int c = s.wsum[w];
      if (w < warp) before += c;
      total += c;
    }
    if (tie && before < rest) s.keys[atomicAdd(&s.n_out, 1)] = rank_key(T, it.id(i));
    base += total;
  }
  __syncthreads();
}

// The `need` best items in s.keys[0, s.n_out) (every item >= floor when fewer), in no particular order
template <class Items>
__device__ void wide_select(const Items& it, uint32_t floor, int need, WideSmem& s) {
  uint32_t T;
  int rest, ties;
  if (need <= 0) {
    if (threadIdx.x == 0) s.n_out = 0;
    __syncthreads();
  } else if (wide_threshold(it, floor, need, s, &T, &rest, &ties)) {
    wide_gather(it, T, rest, ties, s);
  } else {
    wide_gather(it, floor, 0, 0, s);
  }
}

// out[0, n_probe) = the ids of s.keys[0, s.n_out) in rank order, then -1
__device__ void wide_write_cells(WideSmem& s, int n_probe, int32_t* out) {
  const int m = s.n_out;
  int P = 1;
  while (P < m) P <<= 1;
  for (int i = m + threadIdx.x; i < P; i += SEL_THREADS) s.keys[i] = 0;
  __syncthreads();
  block_sort_desc(s.keys, P);
  for (int i = threadIdx.x; i < n_probe; i += SEL_THREADS) out[i] = i < m ? int32_t(rank_key_id(s.keys[i])) : -1;
}

// grid B*Q.  The tile pruning of k1b_probe_kernel: tau = the n-th best tile maximum bounds the n-th best score from
// below, so only the rows of tiles whose maximum is >= tau are read (all of them when there are fewer than n tiles).
__global__ void __launch_bounds__(SEL_THREADS)
k1b_probe_wide_kernel(const __half* __restrict__ S, const __half* __restrict__ tmax, int K, int Q, int Qp,
                      int n_tiles, int n_probe, int32_t* __restrict__ cells) {
  __shared__ WideSmem s;
  const int b = blockIdx.x / Q, q = blockIdx.x % Q;
  const uint16_t* tm = reinterpret_cast<const uint16_t*>(tmax) + (int64_t(b) * Qp + q) * n_tiles;
  const uint16_t* col = reinterpret_cast<const uint16_t*>(S) + int64_t(b) * K * Qp + q;
  uint32_t tau = 0, T;
  int rest, ties;
  if (wide_threshold(TileItems{tm, n_tiles}, 0u, n_probe, s, &T, &rest, &ties)) tau = T;
  wide_select(RowItems{col, tm, K, Qp}, tau, n_probe, s);
  wide_write_cells(s, n_probe, cells + int64_t(blockIdx.x) * n_probe);
}

// grid B*Q.  The subset probe of k1b_probe_subset_kernel: n = min(n_probe, #centroids of the subset's documents).
__global__ void __launch_bounds__(SEL_THREADS)
k1b_probe_subset_wide_kernel(const __half* __restrict__ S, int K, int Q, int Qp, int n_probe,
                             const int32_t* __restrict__ clist, const int32_t* __restrict__ n_clist,
                             int32_t* __restrict__ cells) {
  __shared__ WideSmem s;
  const int b = blockIdx.x / Q, q = blockIdx.x % Q;
  const int nc = n_clist[b];
  const uint16_t* col = reinterpret_cast<const uint16_t*>(S) + int64_t(b) * K * Qp + q;
  wide_select(ListItems{col, clist + int64_t(b) * K, nc, Qp}, 0u, min(n_probe, nc), s);
  wide_write_cells(s, n_probe, cells + int64_t(blockIdx.x) * n_probe);
}

__global__ void pad_queries_kernel(const __half* __restrict__ q, __half* __restrict__ out, int B, int Q,
                                   int Qp, int D) {
  const int64_t n8 = int64_t(B) * Qp * (D / 8);
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n8; i += int64_t(gridDim.x) * blockDim.x) {
    const int c8 = int(i % (D / 8));
    const int64_t row = i / (D / 8);
    const int qq = int(row % Qp);
    const int64_t b = row / Qp;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (qq < Q) v = *reinterpret_cast<const uint4*>(q + (b * Q + qq) * D + c8 * 8);
    *reinterpret_cast<uint4*>(out + row * D + c8 * 8) = v;
  }
}

template <int D, int QC>
int launch_k1_t(const fpb_index* ix, const Ws& ws, cudaStream_t st) {
  const fpb_layout& L = *ws.L;
  auto kern = k1_centroid_scores_kernel<D, QC>;
  constexpr int smem = K1Smem<D, QC>::bytes;
  // opt in on every launch: the attribute is per device and the call costs about a microsecond
  FPB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  // split the batch over gridDim.y only when the centroid tiles alone cannot fill the chip
  int ysplit = 1;
  const int want = 2 * ix->sm_count;
  if (L.n_tiles < want) ysplit = min(L.B, (want + L.n_tiles - 1) / L.n_tiles);
  const int b_per_cta = (L.B + ysplit - 1) / ysplit;
  ysplit = (L.B + b_per_cta - 1) / b_per_cta;
  dim3 grid(L.n_tiles, ysplit);
  kern<<<grid, K1_THREADS, smem, st>>>(ix->centroids, int(ix->K), ws.queries(), L.B, L.Qp, ws.S(),
                                       ws.tmax(), L.n_tiles, b_per_cta);
  FPB_LAUNCH_CHECK("k1_centroid_scores");
  return FPB_OK;
}

template <int D>
int launch_k1_d(const fpb_index* ix, const Ws& ws, cudaStream_t st) {
  const int Qp = ws.L->Qp;
  if (Qp == 16) return launch_k1_t<D, 16>(ix, ws, st);
  if (Qp == 32) return launch_k1_t<D, 32>(ix, ws, st);
  return launch_k1_t<D, 64>(ix, ws, st);  // Qp in {64,128,256}: 64-column chunks
}

// The K1 variant of a launch, the whole rule: the wgmma kernel (k1_centroid_v2.cu) at dim 128 and Qp <= 128 when
// the centroid table has a TMA descriptor, unless FPB_K1=v1 pins the mma.sync kernel; the mma.sync kernel with
// QC = min(Qp, 64) otherwise.
enum class K1Kernel { wgmma, mma };
K1Kernel k1_kernel(const fpb_index* ix, const fpb_layout& L) {
  const bool wgmma = !fpb_env_is("FPB_K1", "v1") && ix->dim == 128 && L.Qp <= 128 && ix->has_tmap;
  return wgmma ? K1Kernel::wgmma : K1Kernel::mma;
}

}  // namespace

int launch_pad_queries(const fpb_index* ix, const Ws& ws, const __half* d_queries, cudaStream_t st) {
  const fpb_layout& L = *ws.L;
  const int64_t n8 = int64_t(L.B) * L.Qp * (ix->dim / 8);
  const int blocks = int(((n8 + 255) / 256) < 4096 ? ((n8 + 255) / 256) : 4096);
  pad_queries_kernel<<<blocks, 256, 0, st>>>(d_queries, ws.queries(), L.B, L.Q, L.Qp, ix->dim);
  FPB_LAUNCH_CHECK("pad_queries");
  return FPB_OK;
}

int launch_centroid_scores(const fpb_index* ix, const Ws& ws, cudaStream_t st) {
  if (k1_kernel(ix, *ws.L) == K1Kernel::wgmma) return launch_centroid_scores_v2(ix, ws, st);
  return fpb_with_codec(ix->dim, ix->nbits, "centroid scoring", [&](auto c) { return launch_k1_d<c.D>(ix, ws, st); });
}

int launch_probe(const fpb_index* ix, const Ws& ws, bool subset, cudaStream_t st) {
  const fpb_layout& L = *ws.L;
  if (L.n_probe > FPB_WARP_PROBE) {
    if (subset) {
      k1b_probe_subset_wide_kernel<<<L.B * L.Q, SEL_THREADS, 0, st>>>(ws.S(), int(ix->K), L.Q, L.Qp, L.n_probe,
                                                                      ws.clist(), ws.n_clist(), ws.cells());
      FPB_LAUNCH_CHECK("k1b_probe_subset_wide");
      return FPB_OK;
    }
    k1b_probe_wide_kernel<<<L.B * L.Q, SEL_THREADS, 0, st>>>(ws.S(), ws.tmax(), int(ix->K), L.Q, L.Qp, L.n_tiles,
                                                             L.n_probe, ws.cells());
    FPB_LAUNCH_CHECK("k1b_probe_wide");
    return FPB_OK;
  }
  const int warps = L.B * L.Q;
  const int blocks = (warps + 7) / 8;
  if (subset) {
    k1b_probe_subset_kernel<<<blocks, 256, 0, st>>>(ws.S(), int(ix->K), L.B, L.Q, L.Qp, L.n_probe, ws.clist(),
                                                    ws.n_clist(), ws.cells());
    FPB_LAUNCH_CHECK("k1b_probe_subset");
    return FPB_OK;
  }
  k1b_probe_kernel<<<blocks, 256, 0, st>>>(ws.S(), ws.tmax(), int(ix->K), L.B, L.Q, L.Qp, L.n_tiles,
                                           L.n_probe, ws.cells());
  FPB_LAUNCH_CHECK("k1b_probe");
  return FPB_OK;
}
