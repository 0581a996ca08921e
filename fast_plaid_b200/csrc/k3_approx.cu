// K3  : approximate (centroid-only) document scores                       (search.rs:554-592)
//         approx[d] = sum_{q<Q}^{fp32}  max_{t<len(d)}  S[b][code[d,t]][q]     (fp16 max)
//
// The reference gathers S rows into a [tokens, Q] tensor, pads it to [2000, maxlen, Q], masks, maxes and
// sums, 128 times per query with two host syncs each.  A one-pass GPU formulation (one warp walks one
// candidate, every token gathers its Qp*2-byte S row) is bound by the L1 data pipe: one wavefront per
// gathered row, 4.87 G rows per batch on cfg-3.  Going faster needs FEWER ROWS, exactly:
//
//   1. tau[b,q]   = the level a candidate holds on average LAMBDA tokens at or above, estimated from sampled
//                   candidates (K1's tile maxima only floor the histogram).  Any value is correct; it only moves
//                   work between the two passes
//   2. hi[b,c]    = exists q: S[b,c,q] >= tau[b,q]          (a K-bit map per query, in shared memory)
//   3. bound pass : walk every candidate, test one bit per token, gather ONLY the rows of high centroids
//                   (19.4 % of the tokens on cfg-3 at LAMBDA = 2, DESIGN §4).  With m_q = max over the gathered rows:
//                     m_q >= tau_q  =>  m_q is the true column maximum (every skipped row is < tau_q <= m_q)
//                     otherwise     =>  m_q <= true maximum < tau_q
//                   so   lb = sum_q m_q  <=  approx  <=  sum_q max(m_q, tau_q) = ub,  with lb == ub == approx
//                   bit for bit when every column is resolved (fp32 addition is monotone in each operand and
//                   both sums use the summation order of the exact kernel).
//   4. threshold  : T = a value such that at least n_full_scores/4 candidates have lb >= T.
//   5. exact pass : the unresolved candidates with ub >= T are re-scored with all their rows.
//   A candidate left with an upper bound has approx <= ub < T <= the scores of >= n_full_scores/4 others:
//   it cannot enter the pruned list whatever the tie rule, and K3b (which only orders by value) never
//   selects it.  The pruned list and everything after it are bit-identical to scoring every candidate.
#include <math.h>

#include <cooperative_groups.h>

#include "kernels.h"
#include "select.cuh"

namespace {

constexpr int64_t K3_TWO_PASS_MIN_TOKENS = 200000000;  // B * index tokens below which one pass is used by default
constexpr int K3_THREADS = 256;
constexpr int K3A_DOCS_PER_CHUNK = 128;  // bound pass: documents per chunk
// exact pass: documents per chunk, at most (the one-pass mode's granule), and the most queries' refine lists the
// resident CTAs' chunks may span (k3_prefix_kernel).  Smaller chunks only where the lists are short: on clustered
// corpora, whose long lists gather few distinct rows, chunks below 64 only add queue overhead.
constexpr int K3_EXACT_MAX_DOCS = 64;
constexpr int K3_EXACT_QUERIES_IN_FLIGHT = 4;
// bound pass: per-warp ring of high codes waiting for their gather (a power of two >= one group + one batch)
constexpr int K3_WQ_FOR(int W, int FLUSH) { int n = 64; while (n < 32 * W + FLUSH) n <<= 1; return n; }

// chunk prefix of the dynamic work queue: work[b] = first chunk of query b, work[B] = total, work[B+1] = counter,
// work[B+2] = documents per chunk.  per_chunk > 0 fixes the granule (the bound pass, the one-pass mode).  per_chunk = 0
// sizes it for the exact pass's refine lists (`ctas` CTAs resident): the chunks are taken in query order, so the resident CTAs cover about
// K3_EXACT_QUERIES_IN_FLIGHT queries' documents and what they gather of S stays in L2.  It is a multiple of the warps
// per CTA, from one document per warp up to K3_EXACT_MAX_DOCS.  pin (such a multiple, 0 = none) overrides it.
__global__ void k3_prefix_kernel(const int32_t* __restrict__ n_items, int B, int per_chunk, int ctas, int pin,
                                 int32_t* __restrict__ work) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    if (per_chunk <= 0) {
      constexpr int WARPS = K3_THREADS / 32;
      int64_t total = 0;
      for (int b = 0; b < B; ++b) total += n_items[b];
      const int64_t g = K3_EXACT_QUERIES_IN_FLIGHT * total / (int64_t(B) * ctas) / WARPS * WARPS;
      per_chunk = pin > 0 ? pin : int(g < WARPS ? WARPS : (g > K3_EXACT_MAX_DOCS ? K3_EXACT_MAX_DOCS : g));
    }
    int acc = 0;
    for (int b = 0; b < B; ++b) {
      work[b] = acc;
      acc += (n_items[b] + per_chunk - 1) / per_chunk;
    }
    work[B] = acc;
    work[B + 1] = 0;
    work[B + 2] = per_chunk;
  }
}

// next (query, chunk) of the queue; s_b = -1 when it is empty.  Called by every thread of the CTA.
__device__ __forceinline__ void k3_next_chunk(int32_t* work, int B, int* s_b, int* s_c) {
  __syncthreads();
  if (threadIdx.x == 0) {
    const int c = atomicAdd(&work[B + 1], 1);
    if (c >= work[B]) {
      *s_b = -1;
    } else {
      int lo = 0, hi = B - 1;  // largest b with work[b] <= c
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (work[mid] <= c) lo = mid; else hi = mid - 1;
      }
      *s_b = lo;
      *s_c = c - work[lo];
    }
  }
  __syncthreads();
}

// One lane's running column maxima: the 8 columns col0 = 8 * (lane % LPR) .. col0 + 7 of its S rows, as four half2.
struct K3Cols {
  __half2 h[4];

  // every column at the padding sentinel, below any score.  The kernels make one before their loops and copy it: the
  // conversion is an asm statement that the compiler does not hoist.
  static __device__ __forceinline__ K3Cols empty() {
    const __half2 s = __float2half2_rn(FPB_PAD_SENTINEL);
    return K3Cols{{s, s, s, s}};
  }
  // the columns as the lane's 16 bytes of an S row
  __device__ __forceinline__ uint4 row() const {
    return make_uint4(half2_as_u32(h[0]), half2_as_u32(h[1]), half2_as_u32(h[2]), half2_as_u32(h[3]));
  }
  // fold in the lane's 16 bytes of one S row (or of tau)
  __device__ __forceinline__ void fold(uint4 v) {
    h[0] = __hmax2(h[0], u32_as_half2(v.x));
    h[1] = __hmax2(h[1], u32_as_half2(v.y));
    h[2] = __hmax2(h[2], u32_as_half2(v.z));
    h[3] = __hmax2(h[3], u32_as_half2(v.w));
  }
  // fold in the maxima that lane ^ off holds in src
  __device__ __forceinline__ void fold_xor(const K3Cols& src, int off) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
      h[i] = __hmax2(h[i], u32_as_half2(__shfl_xor_sync(0xffffffffu, half2_as_u32(src.h[i]), off)));
  }
  // maxima across the lane groups: xor offsets FROM, 2 * FROM, .. below TO
  template <int FROM, int TO = 32>
  __device__ __forceinline__ void reduce() {
#pragma unroll
    for (int off = FROM; off < TO; off <<= 1) fold_xor(*this, off);
  }
  // The fp32 sum over the real query tokens (sum_dim_intlist(.., Kind::Float), search.rs:401), after reduce<LPR>():
  // the lane's 8 columns in order, then across the LPR lanes of a row.  This order of the additions is the contract
  // between the bound pass and the exact pass: lb, ub and the exact score are all summed here, which is what makes
  // lb == ub == approx bit for bit when every column is resolved.  FULLQ (Q == Qp: every column is a real query
  // token) makes the same additions in the same order.
  template <int LPR, bool FULLQ = false>
  __device__ __forceinline__ float sum(int col0, int Q) const {
    float s = 0.f;
    float2 f[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) f[i] = __half22float2(h[i]);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (FULLQ || col0 + 2 * i < Q) s += f[i].x;
      if (FULLQ || col0 + 2 * i + 1 < Q) s += f[i].y;
    }
#pragma unroll
    for (int off = 1; off < LPR; off <<= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    return s;
  }
};

// ---------------------------------------------------------------------------------------
// The walk layout (fpb_index::walk_codes, built once at index load by k3_walk_layout_kernel).  Every K3 walker
// visits a document as whole 32-token windows of its own: aligned 128-byte code loads and no masks, and a slot
// whose code is >= K (padding) gathers nothing.  In the bound pass each lane of a window tests the bitmap word
// code >> 5 in shared memory, whose bank is (code >> 5) & 31, fixed by the code and not by the query.  The 32
// tests of a window cost as many shared-memory wavefronts as the most crowded bank holds distinct words: ~3.5 for
// 32 random codes.  So each document's tokens are stable-sorted by bank and dealt round-robin over its
// ceil(len/32) windows -- a bank with c tokens gets at most ceil(c / windows) slots of any window -- and a window's
// empty slots take padding codes (fpb_walk_pad_code) in banks its real codes leave free.
// ---------------------------------------------------------------------------------------
constexpr int K3_WALK_THREADS = 256;

__global__ void __launch_bounds__(K3_WALK_THREADS)
k3_walk_layout_kernel(const int64_t* __restrict__ doc_offsets, const int32_t* __restrict__ codes,
                      const int64_t* __restrict__ walk_win, int64_t N, int hb_words, int32_t* __restrict__ walk_codes) {
  __shared__ int s_cnt[K3_WALK_THREADS / 32][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned lt_mask;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(lt_mask));
  int* cnt = s_cnt[warp];
  for (int64_t d = int64_t(blockIdx.x) * (K3_WALK_THREADS / 32) + warp; d < N;
       d += int64_t(gridDim.x) * (K3_WALK_THREADS / 32)) {
    const int64_t o0 = doc_offsets[d];
    const int len = int(doc_offsets[d + 1] - o0);
    const int nw = (len + 31) >> 5;
    int32_t* out = walk_codes + walk_win[d] * 32;
    // tokens per bank, then each bank's first position in the stable order by bank
    cnt[lane] = 0;
    __syncwarp();
    for (int t0 = 0; t0 < len; t0 += 32) {
      const bool act = t0 + lane < len;
      const unsigned am = __ballot_sync(0xffffffffu, act);
      if (act) {
        const int bank = (__ldg(codes + o0 + t0 + lane) >> 5) & 31;
        const unsigned peers = __match_any_sync(am, bank);
        if ((peers & lt_mask) == 0u) cnt[bank] += __popc(peers);
      }
      __syncwarp();
    }
    {
      const int c = cnt[lane];
      int incl = c;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, off);
        if (lane >= off) incl += v;
      }
      __syncwarp();
      cnt[lane] = incl - c;
      __syncwarp();
    }
    // sorted position i goes to slot i / nw of window i % nw
    for (int t0 = 0; t0 < len; t0 += 32) {
      const bool act = t0 + lane < len;
      const unsigned am = __ballot_sync(0xffffffffu, act);
      int code = 0, bank = 0, i = 0;
      unsigned peers = 0u;
      if (act) {
        code = __ldg(codes + o0 + t0 + lane);
        bank = (code >> 5) & 31;
        peers = __match_any_sync(am, bank);
        i = cnt[bank] + __popc(peers & lt_mask);
      }
      __syncwarp();
      if (act && (peers & lt_mask) == 0u) cnt[bank] += __popc(peers);
      __syncwarp();
      if (act) out[(i % nw) * 32 + i / nw] = code;
    }
    __syncwarp();  // the stores above are read back below
    // window w holds the positions i < len with i % nw == w; each empty slot takes the next bank no real code of
    // the window uses (a window of r real codes uses at most r banks, so 32 - r are free)
    for (int w = 0; w < nw; ++w) {
      const int r = (len - w + nw - 1) / nw;
      const unsigned used = __reduce_or_sync(0xffffffffu, lane < r ? 1u << ((out[w * 32 + lane] >> 5) & 31) : 0u);
      if (lane >= r) out[w * 32 + lane] = fpb_walk_pad_code(hb_words, int(__fns(~used, 0, lane - r + 1)));
    }
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------
// Exact pass / one-pass scoring.  One warp walks one candidate; each S row (Qp fp16 = LPR x 16 B) is fetched
// by LPR adjacent lanes, so a warp-wide load touches 32/LPR distinct rows, and the running maxima stay in
// registers.  `list` (the bound pass's refine list) selects the candidates; NULL = all of them.
// How the codes reach the lanes depends on Qp.  Up to Qp = 32 the LPR lanes of a group load "their" LPR
// consecutive codes themselves with one vector load (the lanes of a group read the same 4*LPR bytes: a broadcast;
// the windows of the walk layout are 128-byte aligned, so the vector loads are too), which keeps __shfl_sync -- it
// runs through the same L1 data pipe as the gathers -- out of the loop.  Above that each lane loads one code of a
// window and the codes are shuffled to the groups.
// ---------------------------------------------------------------------------------------
constexpr int K3_EXACT_UNROLL = 2;  // windows whose code loads are in flight at once
constexpr int K3_EXACT_MINB = 6;    // resident CTAs per SM

// the slot of a window that holds the first code a lane loads: its group's first (vector loads) or its own
template <int LPR>
__device__ __forceinline__ int first_code(int lane) {
  if constexpr (LPR <= 4) return lane / LPR * LPR;
  else return lane;
}
template <int LPR>
__device__ __forceinline__ void load_codes(int (&c)[LPR], const int32_t* p) {
  if constexpr (LPR == 2) {
    const int2 v = __ldg(reinterpret_cast<const int2*>(p));
    c[0] = v.x; c[1] = v.y;
  } else {
#pragma unroll
    for (int i = 0; i < LPR / 4; ++i) {
      const int4 v = __ldg(reinterpret_cast<const int4*>(p) + i);
      c[4 * i + 0] = v.x; c[4 * i + 1] = v.y; c[4 * i + 2] = v.z; c[4 * i + 3] = v.w;
    }
  }
}

// LIST: the refine-list walk, documents per chunk from work[B+2]; otherwise the one-pass mode over every candidate in
// chunks of K3_EXACT_MAX_DOCS (a compile-time constant, as the one-pass walk has always been built)
template <int LPR, bool LIST>
__global__ void __launch_bounds__(K3_THREADS, K3_EXACT_MINB)
k3_exact_kernel(const __half* __restrict__ S, int64_t K, int Q, const int64_t* __restrict__ doc_offsets,
                const int32_t* __restrict__ walk_codes, const int64_t* __restrict__ walk_win,
                const int32_t* __restrict__ cand, int cand_cap, const int32_t* __restrict__ n_cand,
                const int32_t* __restrict__ list, const int32_t* __restrict__ n_list,
                int32_t* __restrict__ work, int B, float* __restrict__ approx,
                unsigned long long* __restrict__ stats) {
  constexpr int QP = LPR * 8;
  constexpr int TPI = 32 / LPR;
  constexpr int UNROLL = K3_EXACT_UNROLL;
  __shared__ int s_b, s_c;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int sub = lane % LPR, grp = lane / LPR;
  const int Ki = int(K);
  const K3Cols empty = K3Cols::empty();
  unsigned long long rows = 0;
  const int per_chunk = LIST ? work[B + 2] : K3_EXACT_MAX_DOCS;

  for (;;) {
    k3_next_chunk(work, B, &s_b, &s_c);
    const int b = s_b;
    if (b < 0) break;
    const int n = LIST ? n_list[b] : n_cand[b];
    const uint4* Sb = reinterpret_cast<const uint4*>(S + int64_t(b) * K * QP) + sub;
    const int32_t* cb = cand + int64_t(b) * cand_cap;
    const int32_t* lb = LIST ? list + int64_t(b) * cand_cap : nullptr;
    float* ab = approx + int64_t(b) * cand_cap;

    for (int i = 0; i < per_chunk / (K3_THREADS / 32); ++i) {
      const int j = s_c * per_chunk + i * (K3_THREADS / 32) + warp;
      if (j >= n) break;
      const int idx = LIST ? lb[j] : j;
      const int d = cb[idx];
      const int64_t o0 = doc_offsets[d];
      const int len = int(doc_offsets[d + 1] - o0);
      rows += unsigned(len);
      const int nw = (len + 31) >> 5;
      const int32_t* cw = walk_codes + walk_win[d] * 32 + first_code<LPR>(lane);
      K3Cols m = empty;
      for (int w0 = 0; w0 < nw; w0 += UNROLL) {
        if constexpr (LPR <= 4) {  // vector loads of the group's codes
          int c[UNROLL][LPR];
#pragma unroll
          for (int u = 0; u < UNROLL; ++u) {
            if (w0 + u < nw) {
              load_codes<LPR>(c[u], cw + (w0 + u) * 32);
            } else {
#pragma unroll
              for (int jj = 0; jj < LPR; ++jj) c[u][jj] = Ki;
            }
          }
#pragma unroll
          for (int u = 0; u < UNROLL; ++u) {
#pragma unroll
            for (int jj = 0; jj < LPR; ++jj) {
              if (c[u][jj] < Ki) m.fold(__ldg(Sb + int64_t(c[u][jj]) * LPR));
            }
          }
        } else {  // one code per lane, shuffled to the groups
          int code[UNROLL];
#pragma unroll
          for (int u = 0; u < UNROLL; ++u) code[u] = (w0 + u < nw) ? __ldg(cw + (w0 + u) * 32) : Ki;
#pragma unroll
          for (int u = 0; u < UNROLL; ++u) {
#pragma unroll
            for (int jj = 0; jj < LPR; ++jj) {
              const int c = __shfl_sync(0xffffffffu, code[u], jj * TPI + grp);
              if (c < Ki) m.fold(__ldg(Sb + int64_t(c) * LPR));
            }
          }
        }
      }
      m.reduce<LPR>();
      const float s = m.sum<LPR>(sub * 8, Q);
      if (lane == 0) ab[idx] = s;
    }
  }
  if (stats && lane == 0 && rows) atomicAdd(stats + 2, rows);
}

// ---------------------------------------------------------------------------------------
// Two-pass scheme, step 1: tau[b,q].  Any value is correct; what it should be is decided by the candidates, not by
// the centroid table: with tau_q at the level that a candidate document holds on average LAMBDA tokens at or above
// it, a column stays unresolved with probability ~exp(-LAMBDA) and a row is gathered with probability
// ~Q*LAMBDA/len, whatever the score distribution (uniform codes, clustered topics, short documents).  So tau_q is
// estimated from a sample: up to K3_TAU_DOCS candidates per query (evenly spaced), every token's S row, and per
// column the (LAMBDA * #sampled docs)-th largest value, found with a two-level 256-bin radix select on the 16-bit
// order-preserving keys.  One CTA per query; columns are handled 32 at a time.
// ---------------------------------------------------------------------------------------
constexpr int K3_TAU_DOCS = 64;
constexpr int K3_TAU_THREADS = 1024;

// The level-1 histogram costs one shared-memory atomic per sampled value; almost all of them fall far below the
// answer.  The smallest of the column's tile maxima (K1 writes one per 128 centroids) sits near the 94th percentile
// of the column, well below any useful tau, so values under it are not counted; if that ever leaves fewer than the
// wanted rank (tau would be below the floor), the level is redone without a floor.
template <int LPR>
__global__ void __launch_bounds__(K3_TAU_THREADS)
k3_tau_kernel(const __half* __restrict__ S, int64_t K, int Q, const int64_t* __restrict__ doc_offsets,
              const int32_t* __restrict__ walk_codes, const int64_t* __restrict__ walk_win,
              const int32_t* __restrict__ cand, int cand_cap,
              const int32_t* __restrict__ n_cand, const __half* __restrict__ tmax, int n_tiles, float lambda,
              __half* __restrict__ tau) {
  constexpr int QP = LPR * 8, TPI = 32 / LPR;
  constexpr int SUBS = LPR < 4 ? LPR : 4;  // lane subs (8 columns each) handled per round
  __shared__ int hist[32][256];
  __shared__ int s_bin[32], s_rem[32];
  __shared__ uint32_t s_floor[32];
  __shared__ int s_redo;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int sub = lane % LPR, grp = lane / LPR;
  const int Ki = int(K);
  uint16_t* out = reinterpret_cast<uint16_t*>(tau) + int64_t(b) * QP;
  const int n = n_cand[b];
  const int ns = min(n, K3_TAU_DOCS);
  const int32_t* cb = cand + int64_t(b) * cand_cap;
  const uint4* Sb = reinterpret_cast<const uint4*>(S + int64_t(b) * K * QP);
  const int want = max(1, __float2int_rn(lambda * float(ns)));  // rank (from the top) of the selected value

  for (int g0 = 0; g0 < LPR; g0 += SUBS) {
    const bool mine = sub >= g0 && sub < g0 + SUBS;
    const int qrow = (sub - g0) * 8;  // first of this lane's 8 histogram rows
    __syncthreads();  // the previous round's last reads of s_redo / s_floor / s_bin are done
    // floor of the round's columns: the smallest tile maximum (one warp per column)
    for (int col = warp; col < SUBS * 8; col += K3_TAU_THREADS / 32) {
      const int q = g0 * 8 + col;
      uint32_t mn = 0xffffu;
      if (q < Q) {
        const uint16_t* tm = reinterpret_cast<const uint16_t*>(tmax) + (int64_t(b) * QP + q) * n_tiles;
        for (int i = lane; i < n_tiles; i += 32) mn = min(mn, f16_key(tm[i]));
      }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, off));
      if (lane == 0) s_floor[col] = mn;
    }
    if (tid == 0) s_redo = 0;
    __syncthreads();
    for (int level = 0; level < 2; ++level) {
      for (int i = tid; i < 32 * 256; i += K3_TAU_THREADS) (&hist[0][0])[i] = 0;
      __syncthreads();
      uint32_t fl[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) fl[e] = (mine && !s_redo) ? s_floor[qrow + e] : 0u;
      for (int j = warp; j < ns; j += K3_TAU_THREADS / 32) {
        const int d = cb[int64_t(j) * n / ns];
        const int nw = int((doc_offsets[d + 1] - doc_offsets[d] + 31) >> 5);
        const int32_t* cw = walk_codes + walk_win[d] * 32 + lane;
        for (int w = 0; w < nw; ++w) {
          const int code = __ldg(cw + w * 32);
          // all LPR row gathers of the window go out before the first histogram update (the kernel is a chain of
          // dependent latencies otherwise)
          constexpr int JB = LPR < 8 ? LPR : 8;  // gathers in flight per lane
#pragma unroll 1
          for (int j0 = 0; j0 < LPR; j0 += JB) {
          uint4 vv[JB];
          int cc[JB];
#pragma unroll
          for (int jj = 0; jj < JB; ++jj) {
            cc[jj] = __shfl_sync(0xffffffffu, code, (j0 + jj) * TPI + grp);
            vv[jj] = make_uint4(0u, 0u, 0u, 0u);
            if (cc[jj] < Ki && mine) vv[jj] = __ldg(Sb + int64_t(cc[jj]) * LPR + sub);
          }
#pragma unroll
          for (int jj = 0; jj < JB; ++jj) {
            const int c = cc[jj];
            if (c < Ki && mine) {
              const uint4 v = vv[jj];
              const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
              for (int e = 0; e < 8; ++e) {
                const uint32_t key = f16_key(uint16_t(w[e >> 1] >> ((e & 1) * 16)));
                if (level == 0) {
                  if (key >= fl[e]) atomicAdd(&hist[qrow + e][key >> 8], 1);
                } else if (int(key >> 8) == s_bin[qrow + e]) {
                  atomicAdd(&hist[qrow + e][key & 255u], 1);
                }
              }
            }
          }
          }
        }
      }
      __syncthreads();
      if (tid < 32) {  // one thread per column of the round: walk the bins from the top
        const int need = level == 0 ? want : s_rem[tid];
        int cum = 0, bin = 255;
        for (; bin > 0; --bin) {
          if (cum + hist[tid][bin] >= need) break;
          cum += hist[tid][bin];
        }
        if (level == 0) {
          s_bin[tid] = bin;
          s_rem[tid] = need - cum;
          // fewer counted values than the wanted rank although a floor was applied: count everything once more
          if (bin == 0 && cum + hist[tid][0] < need && !s_redo && tid < SUBS * 8 && g0 * 8 + tid < Q &&
              s_floor[tid] != 0u)
            atomicExch(&s_redo, 2);
        } else {
          const int q = g0 * 8 + tid;
          if (q < QP) {
            uint32_t key = (uint32_t(s_bin[tid]) << 8) | uint32_t(bin);
            // fewer sampled values than `want` (tiny documents): everything is "high" -> every column resolves
            if (s_bin[tid] == 0 && bin == 0) key = f16_key(0xFC00u);  // -inf
            uint16_t h = uint16_t((key & 0x8000u) ? (key & 0x7fffu) : (~key & 0xffffu));  // inverse of f16_key
            if (q >= Q) h = 0x7C00u;  // padded column: +inf, never "high", excluded from every sum
            if (q < QP && tid < SUBS * 8) out[q] = h;
          }
        }
      }
      __syncthreads();
      if (level == 0 && s_redo == 2) {  // CTA-uniform: the floor hid too much, redo level 0 without it
        __syncthreads();
        if (tid == 0) s_redo = 1;
        __syncthreads();
        level = -1;
      }
    }
  }
}

// step 2: hi[b,c] = exists q: S[b,c,q] >= tau[b,q].  One warp per 32 consecutive centroids = one bitmap word;
// LPR lanes per row, so every warp-wide load is 512 contiguous bytes of S.
template <int LPR>
__global__ void __launch_bounds__(256)
k3_hibits_kernel(const __half* __restrict__ S, int64_t K, const __half* __restrict__ tau,
                 uint32_t* __restrict__ hibits, int hb_words) {
  constexpr int QP = LPR * 8, TPI = 32 / LPR;
  const int b = blockIdx.y, lane = threadIdx.x & 31;
  const int64_t word = int64_t(blockIdx.x) * 8 + (threadIdx.x >> 5);
  const int64_t c0 = word * 32;
  if (c0 >= K) return;  // warp-uniform
  const int sub = lane % LPR, grp = lane / LPR;
  const uint4 t = *reinterpret_cast<const uint4*>(tau + int64_t(b) * QP + sub * 8);
  const uint4* Sb = reinterpret_cast<const uint4*>(S + int64_t(b) * K * QP);
  constexpr uint32_t GMASK = (LPR == 32) ? 0xffffffffu : ((1u << (LPR & 31)) - 1u);
  bool mine = false;
#pragma unroll
  for (int j = 0; j < LPR; ++j) {
    const int64_t c = c0 + j * TPI + grp;
    bool h = false;
    if (c < K) {
      const uint4 v = ldg_nc_na(Sb + c * LPR + sub);
      const unsigned any = __hge2_mask(u32_as_half2(v.x), u32_as_half2(t.x)) |
                           __hge2_mask(u32_as_half2(v.y), u32_as_half2(t.y)) |
                           __hge2_mask(u32_as_half2(v.z), u32_as_half2(t.z)) |
                           __hge2_mask(u32_as_half2(v.w), u32_as_half2(t.w));
      h = any != 0u;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, h);
    // centroid c0 + l (l = this lane) was handled in iteration l / TPI by lane group l % TPI
    if (lane / TPI == j) mine = ((bal >> ((lane % TPI) * LPR)) & GMASK) != 0u;
  }
  const unsigned w = __ballot_sync(0xffffffffu, mine);
  if (lane == 0) hibits[int64_t(b) * hb_words + word] = w;
}

// step 3: the bound pass.  Shared memory: the query's K-bit map, one ring of high codes per warp, and the offsets /
// lengths of the chunk's documents (staged by the first K3A_DOCS_PER_CHUNK threads so that the dependent
// candidate -> offset loads are paid once per chunk, not once per document).  A warp walks its documents as a stream
// of W-window groups and always has the NEXT group's code loads in flight while it tests, queues and gathers the
// current one.  A straightforward version of this kernel is ISSUE-bound (about 90 warp instructions per 32-token
// window, a third of them branches and generic-address arithmetic around the shared-memory accesses), so the
// per-window path is written branch-free with explicit 32-bit
// shared addresses: predicated code load, one LDS of the bitmap word, a wrap-around funnel shift for the bit, ballot,
// predicated STS into the ring.  The 32 words after the bitmap are zero: the walk layout's padding codes test them,
// and so do the windows of a group past the end of the document (all lanes one word: a broadcast).
__device__ __forceinline__ uint32_t k3_lds(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
// One window's queue step in a single block so that the bit is tested ONCE: p = bit c of the bitmap word, ballot,
// rank of this lane among the set lanes, predicated store of the code into the ring.  The ring is aligned to its
// size, so "position modulo the ring, plus its base" is one logic op.  Returns the ballot; tail_bytes is the
// warp-uniform fill pointer in bytes.
__device__ __forceinline__ unsigned k3_push(uint32_t word, uint32_t code, uint32_t ring_base, uint32_t ring_mask_bytes,
                                            uint32_t tail_bytes, uint32_t lt_mask) {
  unsigned mask;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      ".reg .b32 t, r;\n"
      "shf.r.wrap.b32 t, %1, 0, %2;\n"   // word >> (code & 31)
      "and.b32 t, t, 1;\n"
      "setp.ne.u32 p, t, 0;\n"
      "vote.sync.ballot.b32 %0, p, 0xffffffff;\n"
      "and.b32 r, %0, %6;\n"
      "popc.b32 r, r;\n"
      "shl.b32 r, r, 2;\n"
      "add.u32 r, r, %5;\n"
      "and.b32 r, r, %4;\n"
      "or.b32 r, r, %3;\n"
      "@p st.shared.u32 [r], %2;\n"
      "}"
      : "=r"(mask)
      : "r"(word), "r"(code), "r"(ring_base), "r"(ring_mask_bytes), "r"(tail_bytes), "r"(lt_mask)
      : "memory");
  return mask;
}

constexpr int K3_BOUND_U = 4;     // gathers in flight per lane and batch
constexpr int K3_BOUND_MINB = 4;  // resident CTAs per SM (64 registers)

// One batch of gathers from the warp's ring: entry head + k * TPI + grp (k < K3_BOUND_U) is lane group grp's k-th
// row, all loads go out before the first fold.  A full batch takes FLUSH = K3_BOUND_U * TPI entries; the drain
// (DRAIN) at the end of a document takes the rem < FLUSH that are left and folds `empty` in place of the rest.
template <int LPR, int WQ, bool DRAIN>
__device__ __forceinline__ void k3_gather(K3Cols& m, const K3Cols& empty, const uint4* Sb, uint32_t sb_wq,
                                          uint32_t head, uint32_t rem, int grp) {
  constexpr int TPI = 32 / LPR;
  uint4 v[K3_BOUND_U];
#pragma unroll
  for (int k = 0; k < K3_BOUND_U; ++k) {
    const uint32_t jj = k * TPI + grp;
    if (DRAIN) v[k] = empty.row();
    if (!DRAIN || jj < rem) {
      const uint32_t code = k3_lds(sb_wq + (((head + jj) & (WQ - 1)) << 2));
      v[k] = __ldg(Sb + int64_t(code) * LPR);
    }
  }
#pragma unroll
  for (int k = 0; k < K3_BOUND_U; ++k) m.fold(v[k]);
}

// End of a document in the bound pass: the maxima across the lane groups (xor offsets LPR .. below TO; a paired
// epilogue has folded offset 16 already), then lower bound = the maxima over the gathered rows, upper bound = the
// unresolved columns raised to tau, stored at [at] by `writer`.  Both are K3Cols::sum, the exact pass's order, and fp32
// addition is monotone, so lb <= approx <= ub; when no column was raised the two are the same additions of the same
// values, and whenever lb == ub the score is pinned between them: "resolved" needs no flag, it IS lb == ub.
template <int LPR, bool FULLQ, int TO>
__device__ __forceinline__ void k3_store_bounds(K3Cols m, uint4 tq, int col0, int Q, bool writer, float* ub,
                                                float* lb, int at) {
  m.reduce<LPR, TO>();
  const float l = m.sum<LPR, FULLQ>(col0, Q);
  m.fold(tq);  // every column raised to tau
  const float u = m.sum<LPR, FULLQ>(col0, Q);
  if (writer) {
    ub[at] = u;
    lb[at] = l;
  }
}

template <int LPR, int W, bool FULLQ>
__global__ void __launch_bounds__(K3_THREADS, K3_BOUND_MINB)
k3_bound_kernel(const __half* __restrict__ S, int64_t K, int Q, const int64_t* __restrict__ doc_offsets,
                const int32_t* __restrict__ walk_codes, const int64_t* __restrict__ walk_win,
                const int32_t* __restrict__ cand, int cand_cap,
                const int32_t* __restrict__ n_cand, int32_t* __restrict__ work, int B,
                const __half* __restrict__ tau, const uint32_t* __restrict__ hibits, int hb_words,
                float* __restrict__ ub_out, float* __restrict__ lb_out, unsigned long long* __restrict__ stats) {
  constexpr int QP = LPR * 8;
  constexpr int TPI = 32 / LPR;   // rows per warp-wide gather
  constexpr int FLUSH = K3_BOUND_U * TPI;  // rows per batch of gathers (<= 64)
  constexpr int DPW = K3A_DOCS_PER_CHUNK / (K3_THREADS / 32);  // documents per warp and chunk
  constexpr int WQ = K3_WQ_FOR(W, FLUSH);  // ring entries per warp: one group of pushes on top of an unflushed rest
  static_assert(FLUSH + 32 * W <= WQ, "ring too small");
  extern __shared__ __align__(16) uint32_t k3_smem[];  // [hb_words + 32] bitmap + 32 zero words | [warps][WQ] rings
  __shared__ int s_b, s_c;
  __shared__ int64_t s_w0[K3A_DOCS_PER_CHUNK];
  __shared__ int s_len[K3A_DOCS_PER_CHUNK];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int sub = lane % LPR, grp = lane / LPR;
  const uint32_t sb_bm = smem_u32(k3_smem);
  // rings: aligned to their size (WQ * 4 bytes) so that k3_push can OR the base in
  const uint32_t sb_wq = ((sb_bm + uint32_t(hb_words + 32) * 4u + (WQ * 4u - 1u)) & ~(WQ * 4u - 1u)) + uint32_t(warp) * (WQ * 4u);
  const int INV = hb_words * 32;  // a code whose bit lives in a zero word
  unsigned lt_mask;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(lt_mask));
  const K3Cols empty = K3Cols::empty();
  unsigned rows = 0, toks = 0;  // per warp over the CTA's life: far below 2^32
  int cur_b = -1;
  if (tid < 32) k3_smem[hb_words + tid] = 0u;  // never overwritten: the bitmap copy below covers hb_words words

  for (;;) {
    k3_next_chunk(work, B, &s_b, &s_c);
    const int b = s_b;
    if (b < 0) break;
    const int n = n_cand[b];
    const int32_t* cb = cand + int64_t(b) * cand_cap;
    if (tid < K3A_DOCS_PER_CHUNK) {  // stage the chunk's document extents
      const int idx = s_c * K3A_DOCS_PER_CHUNK + tid;
      int64_t w0 = 0;
      int len = -1;  // -1: no such document
      if (idx < n) {
        const int d = cb[idx];
        w0 = walk_win[d];
        len = int(doc_offsets[d + 1] - doc_offsets[d]);
      }
      s_w0[tid] = w0;
      s_len[tid] = len;
    }
    if (b != cur_b) {  // CTA-uniform; every warp is past the previous chunk (barrier in k3_next_chunk)
      const uint4* src = reinterpret_cast<const uint4*>(hibits + int64_t(b) * hb_words);
      for (int i = tid; i < hb_words / 4; i += K3_THREADS) reinterpret_cast<uint4*>(k3_smem)[i] = src[i];
      cur_b = b;
    }
    __syncthreads();
    const uint4* Sb = reinterpret_cast<const uint4*>(S + int64_t(b) * K * QP) + sub;
    const uint4* tqp = reinterpret_cast<const uint4*>(tau + int64_t(b) * QP + sub * 8);
    float* ub_chunk = ub_out + int64_t(b) * cand_cap + int64_t(s_c) * K3A_DOCS_PER_CHUNK;
    float* lb_chunk = lb_out + int64_t(b) * cand_cap + int64_t(s_c) * K3A_DOCS_PER_CHUNK;

    // ---- the warp's documents are slots warp*DPW .. warp*DPW + DPW - 1 of the chunk, walked group by group ----
    int slot = warp * DPW;
    const int slot_end = slot + DPW;
    int len = s_len[slot];
    if (len < 0) continue;  // warp-uniform: this warp has no document in the (last, partial) chunk
    // left = windows of the document not yet walked (including the current group's), one 128-byte line each
    int left = (len + 31) >> 5;
    const int32_t* cw = walk_codes + s_w0[slot] * 32 + lane;
    int c[W];
#pragma unroll
    for (int u = 0; u < W; ++u) {
      c[u] = INV;
      if (u < left) c[u] = __ldg(cw + 32 * u);
    }
    uint32_t head = 0, tail = 0;
    K3Cols m = empty;
    // Up to Qp = 64 (LPR <= 8) the end-of-document work (maxima across the lane groups, two column sums) is done for
    // two documents at once -- the first of a pair is parked in `a`, then the lower half of the warp finishes one
    // document and the upper half the other: half the shuffles, conversions and additions per document
    K3Cols a = empty;
    int slot_a = -1;

    for (;;) {
      // ---- the next group: same document or the next slot; its code loads go out now ----
      const bool last_of_doc = left <= W;
      int nlen = len, nleft = left - W;
      const int32_t* ncw = cw + 32 * W;
      if (last_of_doc) {
        nlen = (slot + 1 < slot_end) ? s_len[slot + 1] : -1;
        nleft = 0;
        if (nlen >= 0) {
          nleft = (nlen + 31) >> 5;
          ncw = walk_codes + s_w0[slot + 1] * 32 + lane;
        }
      }
      int nx[W];
#pragma unroll
      for (int u = 0; u < W; ++u) {
        nx[u] = INV;
        if (u < nleft) nx[u] = __ldg(ncw + 32 * u);
      }
      // ---- current group: bit of every token (W independent shared loads), queue the high codes ----
      uint32_t wbit[W];
#pragma unroll
      for (int u = 0; u < W; ++u) wbit[u] = k3_lds(sb_bm + ((uint32_t(c[u]) >> 5) << 2));
#pragma unroll
      for (int u = 0; u < W; ++u) {
        const unsigned mask = k3_push(wbit[u], uint32_t(c[u]), sb_wq, WQ * 4u - 1u, tail << 2, lt_mask);
        tail += __popc(mask);
      }
      __syncwarp();
      // ---- gather in full batches ----
      while (tail - head >= FLUSH) {
        k3_gather<LPR, WQ, false>(m, empty, Sb, sb_wq, head, 0u, grp);
        head += FLUSH;
      }
      if (last_of_doc) {
        k3_gather<LPR, WQ, true>(m, empty, Sb, sb_wq, head, tail - head, grp);  // drain: fewer than FLUSH codes left
        rows += tail;
        toks += unsigned(len);
        const uint4 tq = __ldg(tqp);
        const int col0 = sub * 8;
        if (LPR <= 8 && slot_a < 0 && nlen >= 0) {
          a = m;  // park: the next document completes the pair
          slot_a = slot;
        } else if (LPR <= 8 && slot_a >= 0) {
          const bool up = lane >= 16;  // lower half: the parked document, upper half: this one
          K3Cols x, y;
#pragma unroll
          for (int i = 0; i < 4; ++i) {  // select values: a select of m's and a's addresses puts them in local memory
            const uint32_t mi = half2_as_u32(m.h[i]), ai = half2_as_u32(a.h[i]);
            x.h[i] = u32_as_half2(up ? mi : ai);
            y.h[i] = u32_as_half2(up ? ai : mi);
          }
          x.fold_xor(y, 16);
          k3_store_bounds<LPR, FULLQ, 16>(x, tq, col0, Q, (lane & 15) == 0, ub_chunk, lb_chunk, up ? slot : slot_a);
          slot_a = -1;
        } else {
          k3_store_bounds<LPR, FULLQ, 32>(m, tq, col0, Q, lane == 0, ub_chunk, lb_chunk, slot);
        }
        if (nlen < 0) break;  // no further document for this warp in the chunk
        head = tail = 0;
        m = empty;
        ++slot;
      }
      __syncwarp();  // the ring slots read above may be overwritten by the next group's pushes
#pragma unroll
      for (int u = 0; u < W; ++u) c[u] = nx[u];
      len = nlen;
      left = nleft;
      cw = ncw;
    }
  }
  if (stats && lane == 0) {
    if (rows) atomicAdd(stats + 0, (unsigned long long)rows);
    if (toks) atomicAdd(stats + 1, (unsigned long long)toks);
  }
}

// step 4: per query the pruning threshold T (at least n_dec candidates have lb >= T; found with two levels of
// 2048 value buckets, so outliers only cost resolution) and the list of unresolved candidates with ub >= T.
// One cluster of K3_REFINE_CTAS CTAs per query (one CTA per query would leave half of the GPU idle), each over its
// own slice of the candidates.  The minimum and maximum, the two histograms and the smallest selected value are
// merged through distributed shared memory: integer counts, minima and maxima do not depend on how the candidates are
// split, so every CTA finds the buckets and the T that one CTA over all of them would.  The list is compacted through
// a counter in the first CTA's shared memory: the set is the same, only its order depends on the schedule.
constexpr int K3_REFINE_CTAS = 4;

__global__ void __cluster_dims__(K3_REFINE_CTAS, 1, 1) __launch_bounds__(1024, 2)
k3_refine_list_kernel(const float* __restrict__ ub, const float* __restrict__ lb, int cand_cap,
                      const int32_t* __restrict__ n_cand, int n_dec, int refine_all, int32_t* __restrict__ list,
                      int32_t* __restrict__ n_list, float* __restrict__ thresh) {
  namespace cg = cooperative_groups;
  const cg::cluster_group cluster = cg::this_cluster();
  __shared__ int hist[SEL_BINS];  // this CTA's counts
  __shared__ int hsum[SEL_BINS];  // the cluster's
  __shared__ float s_red[64];
  __shared__ float s_part[3];     // this CTA's minimum, maximum and smallest selected value
  __shared__ int s_t, s_need, s_cnt;
  const int rank = int(cluster.block_rank());
  const int b = blockIdx.x / K3_REFINE_CTAS, tid = threadIdx.x, lane = tid & 31;
  const int n = n_cand[b];
  const int per = (n + K3_REFINE_CTAS - 1) / K3_REFINE_CTAS;
  const int lo = min(n, rank * per), hi = min(n, lo + per);  // this CTA's slice
  const float* ubb = ub + int64_t(b) * cand_cap;
  const float* lbb = lb + int64_t(b) * cand_cap;
  int32_t* out = list + int64_t(b) * cand_cap;
  constexpr int FV = 8;
  if (tid == 0) s_cnt = 0;
  // hsum = the sum of the cluster's hist; afterwards every CTA may clear its hist again
  auto merge_hist = [&]() {
    cluster.sync();
    for (int i = tid; i < SEL_BINS; i += 1024) {
      int c = 0;
#pragma unroll
      for (int r = 0; r < K3_REFINE_CTAS; ++r) c += cluster.map_shared_rank(hist, r)[i];
      hsum[i] = c;
    }
    cluster.sync();
  };
  // the minimum (or maximum) of s_part[k] over the cluster, folded into v
  auto merge_part = [&](int k, float v, bool is_max) {
#pragma unroll
    for (int r = 0; r < K3_REFINE_CTAS; ++r) {
      const float x = cluster.map_shared_rank(s_part, r)[k];
      v = is_max ? fmaxf(v, x) : fminf(v, x);
    }
    return v;
  };
  float T = -INFINITY;
  if (!refine_all && n > n_dec) {  // n <= n_dec: nothing is pruned (search.rs:605 / :615), every score is needed
    float mn = INFINITY, mx = -INFINITY;
    for (int i0 = lo + tid; i0 < hi; i0 += 1024 * FV) {
      float v[FV];
#pragma unroll
      for (int u = 0; u < FV; ++u) v[u] = (i0 + u * 1024 < hi) ? lbb[i0 + u * 1024] : NAN;  // fmin/fmax skip NaN
#pragma unroll
      for (int u = 0; u < FV; ++u) {
        mn = fminf(mn, v[u]);
        mx = fmaxf(mx, v[u]);
      }
    }
    block_min_max(mn, mx, s_red);
    if (tid == 0) {
      s_part[0] = mn;
      s_part[1] = mx;
    }
    cluster.sync();
    mn = merge_part(0, mn, false);
    mx = merge_part(1, mx, true);
    const float range = mx - mn;
    if (range > 0.f && range < 3.0e38f) {
      // level 1: 2048 buckets over [mn, mx]
      const float scale1 = float(SEL_BINS - 1) / range;
      for (int i = tid; i < SEL_BINS; i += 1024) hist[i] = 0;
      __syncthreads();
      for (int i0 = lo + tid; i0 < hi; i0 += 1024 * FV) {
        float v[FV];
#pragma unroll
        for (int u = 0; u < FV; ++u) v[u] = (i0 + u * 1024 < hi) ? lbb[i0 + u * 1024] : 0.f;
#pragma unroll
        for (int u = 0; u < FV; ++u)
          if (i0 + u * 1024 < hi && v[u] == v[u]) atomicAdd(&hist[value_bucket(v[u], mn, scale1)], 1);
      }
      if (tid == 0) s_t = -1;
      merge_hist();
      if (tid < 32) warp_find_bucket(hsum, SEL_BINS, n_dec, &s_t, &s_need);
      __syncthreads();
      const int t1 = s_t, need1 = s_need;
      __syncthreads();
      if (t1 >= 0) {  // (t1 < 0 only if NaNs leave fewer than n_dec comparable values: T stays -inf)
        // level 2: 2048 buckets inside bucket t1
        const float lo1 = mn + float(t1) / scale1;
        const float scale2 = float(SEL_BINS - 1) * scale1;
        for (int i = tid; i < SEL_BINS; i += 1024) hist[i] = 0;
        __syncthreads();
        for (int i0 = lo + tid; i0 < hi; i0 += 1024 * FV) {
          float v[FV];
#pragma unroll
          for (int u = 0; u < FV; ++u) v[u] = (i0 + u * 1024 < hi) ? lbb[i0 + u * 1024] : 0.f;
#pragma unroll
          for (int u = 0; u < FV; ++u)
            if (i0 + u * 1024 < hi && v[u] == v[u] && value_bucket(v[u], mn, scale1) == t1)
              atomicAdd(&hist[value_bucket(v[u], lo1, scale2)], 1);
        }
        if (tid == 0) s_t = -1;
        merge_hist();
        if (tid < 32) warp_find_bucket(hsum, SEL_BINS, need1, &s_t, &s_need);
        __syncthreads();
        const int t2 = s_t;
        // T = the smallest value of the selected upper set {b1 > t1} u {b1 == t1, b2 >= t2}: it holds >= n_dec values
        float tmin = INFINITY;
        if (t2 >= 0) {
          for (int i0 = lo + tid; i0 < hi; i0 += 1024 * FV) {
            float v[FV];
#pragma unroll
            for (int u = 0; u < FV; ++u) v[u] = (i0 + u * 1024 < hi) ? lbb[i0 + u * 1024] : NAN;
#pragma unroll
            for (int u = 0; u < FV; ++u) {
              if (v[u] == v[u]) {
                const int b1 = value_bucket(v[u], mn, scale1);
                if (b1 > t1 || (b1 == t1 && value_bucket(v[u], lo1, scale2) >= t2)) tmin = fminf(tmin, v[u]);
              }
            }
          }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) tmin = fminf(tmin, __shfl_xor_sync(0xffffffffu, tmin, off));
        __syncthreads();
        if (lane == 0) s_red[tid >> 5] = tmin;
        __syncthreads();
        tmin = s_red[lane];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) tmin = fminf(tmin, __shfl_xor_sync(0xffffffffu, tmin, off));
        if (tid == 0) s_part[2] = tmin;
        cluster.sync();
        tmin = merge_part(2, tmin, false);
        if (t2 >= 0 && tmin < INFINITY) T = tmin;
      }
    } else if (range == 0.f) {
      T = mn;  // every lower bound is the same value: all n > n_dec candidates have lb >= mn
    }
  }
  cluster.sync();  // the first CTA's counter is zero
  int* cnt = cluster.map_shared_rank(&s_cnt, 0);
  const int hi_up = lo + (hi - lo + 1023) / 1024 * 1024;
  for (int i = lo + tid; i < hi_up; i += 1024) {
    bool take = false;
    if (i < hi) {
      const float u = ubb[i], l = lbb[i];
      take = (l < u) && (u >= T);
    }
    const unsigned m = __ballot_sync(0xffffffffu, take);
    int base = 0;
    if (lane == 0 && m) base = atomicAdd(cnt, __popc(m));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (take) out[base + __popc(m & ((1u << lane) - 1u))] = i;
  }
  cluster.sync();  // every CTA's count is in
  if (rank == 0 && tid == 0) {
    n_list[b] = s_cnt;
    thresh[b] = T;
  }
}

// exact scoring of `list` (NULL: every candidate) into approx: the work queue over the list lengths (n_cand and
// K3_EXACT_MAX_DOCS documents per chunk without a list), then the kernel.  FPB_K3_EXACT_DOCS_PER_CHUNK (kernels.h: a
// multiple of the 8 warps of a CTA, up to K3_EXACT_MAX_DOCS) pins the documents per chunk of the refine-list walk;
// the scores do not depend on it, and the tests use it.
template <int LPR>
int launch_k3_exact(const fpb_index* ix, const Ws& ws, const int32_t* list, const int32_t* n_list, int32_t* work,
                    cudaStream_t st) {
  const fpb_layout& L = *ws.L;
  static int per_sm = 0;  // resident CTAs per SM: fixed by the kernel's resources, asked once per instantiation
  if (per_sm == 0) {
    int n = 0;
    FPB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k3_exact_kernel<LPR, true>, K3_THREADS, 0));
    per_sm = n < 1 ? 1 : n;
  }
  const int pin = fpb_env_int("FPB_K3_EXACT_DOCS_PER_CHUNK", 1, K3_EXACT_MAX_DOCS);
  const int pinned = pin % (K3_THREADS / 32) == 0 ? pin : 0;
  // the one-pass mode (no list) keeps K3_EXACT_MAX_DOCS: its candidate lists are long, and the sizing rule is
  // measured on the refine lists only
  k3_prefix_kernel<<<1, 32, 0, st>>>(list ? n_list : ws.n_cand(), L.B, list ? 0 : K3_EXACT_MAX_DOCS,
                                     ix->sm_count * per_sm, pinned, work);
  FPB_LAUNCH_CHECK("k3_prefix");
  auto kern = list ? k3_exact_kernel<LPR, true> : k3_exact_kernel<LPR, false>;
  kern<<<ix->sm_count * 8, K3_THREADS, 0, st>>>(ws.S(), ix->K, L.Q, ix->doc_offsets, ix->walk_codes, ix->walk_win,
                                                ws.cand(), L.cand_cap, ws.n_cand(), list, n_list, work, L.B,
                                                ws.approx(), ws.stats());
  FPB_LAUNCH_CHECK("k3_exact");
  return FPB_OK;
}

// LAMBDA of k3_tau_kernel: the expected number of tokens per candidate and column at or above tau.  A document is
// resolved when all of its Q columns are, so the useful level grows with log Q: LAMBDA = ln(Q) - 1.45 (2.0 at
// Q = 32, 2.7 at Q = 64).  FPB_K3_LAMBDA (kernels.h) overrides it (tuning only: every value gives the same results);
// one process can sweep it (tools/profile_approx.py).
float k3_tau_lambda(int Q) {
  const float pinned = fpb_env_float("FPB_K3_LAMBDA");
  const float x = pinned > 0.f ? pinned : logf(float(Q < 2 ? 2 : Q)) - 1.45f;
  return x < 0.5f ? 0.5f : (x > 64.f ? 64.f : x);
}

// The bound pass with W windows per group (all their code loads in flight at once, the next group's prefetched),
// K3_BOUND_U gathers per lane and batch, up to K3_BOUND_MINB CTAs per SM.
template <int LPR, int W>
int launch_k3_bound(const fpb_index* ix, const Ws& ws, cudaStream_t st) {
  const fpb_layout& L = *ws.L;
  auto kern = L.Q == L.Qp ? k3_bound_kernel<LPR, W, true> : k3_bound_kernel<LPR, W, false>;
  const int wq = K3_WQ_FOR(W, K3_BOUND_U * (32 / LPR));
  // bitmap + 32 zero words, then the rings (+ alignment slack)
  const size_t smem = size_t(L.hb_words + 32) * 4 + size_t(K3_THREADS / 32 + 1) * wq * 4;
  FPB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  // resident CTAs per SM: limited by the bitmap (228 KB of shared memory per SM, 1 KB reserved per CTA; the
  // static shared memory is ~1.6 KB)
  int per_sm = int((227 * 1024) / (smem + 1024 + 2048));
  per_sm = per_sm < 1 ? 1 : (per_sm > K3_BOUND_MINB ? K3_BOUND_MINB : per_sm);
  kern<<<ix->sm_count * per_sm, K3_THREADS, smem, st>>>(ws.S(), ix->K, L.Q, ix->doc_offsets, ix->walk_codes,
                                                        ix->walk_win, ws.cand(), L.cand_cap, ws.n_cand(), ws.work(),
                                                        L.B, ws.tau(), ws.hibits(), L.hb_words, ws.approx(), ws.lb(),
                                                        ws.stats());
  FPB_LAUNCH_CHECK("k3_bound");
  return FPB_OK;
}

template <int LPR>
int launch_k3_t(const fpb_index* ix, const Ws& ws, int flags, cudaStream_t st) {
  const fpb_layout& L = *ws.L;
  // one-pass scoring: asked for, or the K-bit map of a query does not fit next to a second CTA's, or (nothing asked
  // for) the job is too small to repay the fixed cost of the two passes -- results are identical in every case
  const bool forced = (flags & (FPB_FLAG_APPROX_TWO_PASS | FPB_FLAG_APPROX_EXACT_ALL)) != 0;
  const bool small_job = int64_t(L.B) * ix->E < K3_TWO_PASS_MIN_TOKENS;
  if ((flags & FPB_FLAG_APPROX_DIRECT) || size_t(L.hb_words) * 4 > 96 * 1024 || (!forced && small_job)) {
    FPB_CUDA_CHECK(cudaMemsetAsync(ws.n_refine(), 0, size_t(L.B) * 4, st));  // nothing was re-scored
    return launch_k3_exact<LPR>(ix, ws, nullptr, nullptr, ws.work(), st);
  }
  k3_tau_kernel<LPR><<<L.B, K3_TAU_THREADS, 0, st>>>(ws.S(), ix->K, L.Q, ix->doc_offsets, ix->walk_codes,
                                                     ix->walk_win, ws.cand(), L.cand_cap, ws.n_cand(), ws.tmax(),
                                                     L.n_tiles, k3_tau_lambda(L.Q), ws.tau());
  FPB_LAUNCH_CHECK("k3_tau");
  {
    dim3 grid(unsigned((ix->K + 255) / 256), unsigned(L.B));
    k3_hibits_kernel<LPR><<<grid, 256, 0, st>>>(ws.S(), ix->K, ws.tau(), ws.hibits(), L.hb_words);
    FPB_LAUNCH_CHECK("k3_hibits");
  }
  k3_prefix_kernel<<<1, 32, 0, st>>>(ws.n_cand(), L.B, K3A_DOCS_PER_CHUNK, 0, 0, ws.work());
  FPB_LAUNCH_CHECK("k3_prefix");
  {
    // windows per group: the index's choice (fpb_index::walk_group), FPB_K3_GROUP (kernels.h) overrides it (tuning
    // only: every value gives the same results)
    const int pin = fpb_env_int("FPB_K3_GROUP", 4, 6);
    const int g = pin ? pin : ix->walk_group;
    const int rc = g == 4 ? launch_k3_bound<LPR, 4>(ix, ws, st)
                 : g == 5 ? launch_k3_bound<LPR, 5>(ix, ws, st) : launch_k3_bound<LPR, 6>(ix, ws, st);
    if (rc != FPB_OK) return rc;
  }
  k3_refine_list_kernel<<<L.B * K3_REFINE_CTAS, 1024, 0, st>>>(ws.approx(), ws.lb(), L.cand_cap, ws.n_cand(), L.R,
                                              (flags & FPB_FLAG_APPROX_EXACT_ALL) ? 1 : 0, ws.refine(), ws.n_refine(),
                                              ws.thresh());
  FPB_LAUNCH_CHECK("k3_refine_list");
  return launch_k3_exact<LPR>(ix, ws, ws.refine(), ws.n_refine(), ws.work2(), st);
}

}  // namespace

int launch_approx(const fpb_index* ix, const Ws& ws, int flags, cudaStream_t st) {
  const fpb_layout& L = *ws.L;
  switch (L.Qp / 8) {
    case 2: return launch_k3_t<2>(ix, ws, flags, st);
    case 4: return launch_k3_t<4>(ix, ws, flags, st);
    case 8: return launch_k3_t<8>(ix, ws, flags, st);
    case 16: return launch_k3_t<16>(ix, ws, flags, st);
    case 32: return launch_k3_t<32>(ix, ws, flags, st);
    default:
      fpb_set_error("approx scoring: unsupported padded query length %d", L.Qp);
      return FPB_ERR_UNSUPPORTED;
  }
}

int launch_walk_layout(const fpb_index* ix, cudaStream_t st) {
  if (ix->N == 0) return FPB_OK;
  const int64_t warps = K3_WALK_THREADS / 32;
  const int64_t need = (ix->N + warps - 1) / warps;
  const int blocks = int(need < int64_t(ix->sm_count) * 16 ? need : int64_t(ix->sm_count) * 16);
  k3_walk_layout_kernel<<<blocks, K3_WALK_THREADS, 0, st>>>(ix->doc_offsets, ix->doc_codes, ix->walk_win, ix->N,
                                                            fpb_hb_words(ix->K), ix->walk_codes);
  FPB_LAUNCH_CHECK("k3_walk_layout");
  return FPB_OK;
}
