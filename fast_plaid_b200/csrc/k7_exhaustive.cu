// K7 : exhaustive exact MaxSim -- every local document against every query of a batch (fpb_exhaustive_scores).
//
//   scores[b, d] = RN_fp32( sum_{q<Q} fp16( max_t e_hat[d, t] . q[b, q] ) )
//
// K5's formula and rounding points up to the last one: the fp16 maxima are the same, their sum is exact and rounded
// once to fp32 where K5 keeps an fp32 running sum (see the last point below).
//
// The approximate pipeline exact-scores n_full_scores/4 documents per query; here every document meets every
// query, a GEMM-shaped problem of 2 * dim * E * B * Q FLOP, and the cost to avoid is decoding a token more than
// once.  Each CTA takes chunks of consecutive documents, decodes 256 of their tokens at a time into a resident
// shared-memory tile (the B operand) and streams every query row of the batch past it (the A operand):
//
//   * query rows: query b owns rows [b*Qs, b*Qs + Q) of a dense row array (Qs = Q rounded up to 16, so the 16
//     rows of an MMA warp belong to one query); rows q >= Q are zero and are left out of the sum;
//   * 256 threads = two warpgroups.  Both decode the tile with the generic path of the shared decoder
//     (decode.cuh: Decoder, then ehat_chunk per 16-byte SWIZZLE_128B chunk; at nbits 1 two lanes of 8 packed bytes
//     per token, as at nbits 2) in v5's 8-token passes: pass p of a
//     document is its tokens 8p..8p+7, a partial pass repeats the last token (a duplicate cannot change a
//     maximum), passes of consecutive documents follow each other, and a document is split only where it
//     crosses a tile boundary.  Then the 128-row A stages are cp.async-loaded one stage ahead, and
//     warpgroup c multiplies its 64 rows against the tile with wgmma.m64n128k16 (two 128-token blocks issued
//     back to back; the epilogue starts once both have completed);
//   * the per-document maxima come straight out of the accumulator registers (column group j = one pass, as in
//     v5).  A document whose passes cross a tile boundary keeps its running row maxima in a per-CTA carry array
//     (global memory, L2-resident) until its last tile;
//   * the sum over q: every fp16 maximum is an integer multiple of 2^-24 below 2^16 in magnitude, so the fp32
//     sum is computed as the exact 64-bit integer sum of m * 2^24 (a warp adds its 16 rows, then one integer
//     atomicAdd per warp and document) and rounded once to fp32 by k7_finalize.  Integer addition is
//     associative: the result does not depend on the order of the atomics, on the grid or on how a batch is
//     split into calls.  Where the fp32 running sum of K5 / the reference is exact (every partial sum fits 24
//     significant bits, the usual case) the two are bit-identical; elsewhere they can differ in the last bit.
//
// The list walk (LIST = true, fpb_search_exhaustive_subset) is the same kernel over per-list document lists instead
// of the range [0, N): a chunk is (list l, positions i0 .. i0+nd) of l's sorted-unique list, the query rows are
// grouped by list (list l's rows [row0[l], row1[l]) start on a 64-row boundary, so one warpgroup's rows belong to one
// list), only the A stages that hold rows of l are streamed, a warpgroup without rows of l runs no MMA, and a row
// counts only when its query searches l.  Decoder, MMA sequence and fixed-point sum are those of the full scan, so
// every score is bit-identical to the full scan's score of the same document.
#include "decode.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace {

constexpr int K7_THREADS = 256;          // two warpgroups: both decode, both run MMAs
constexpr int K7_TILE = 256;             // decoded token rows resident per tile
constexpr int K7_PASSES = K7_TILE / 8;   // 32 passes of 8 tokens
constexpr int K7_RB = 128;               // query rows per A stage (64 per warpgroup)
constexpr int K7_MAX_DOCS = 32;          // documents per chunk (one warp scans their pass counts)
static_assert(K7_TILE == 2 * 128, "the MMA loop keeps two 128-column accumulator blocks");

template <int D>
struct K7Smem {
  static constexpr int b_kblock = K7_TILE * 128;  // B: tile rows x 128 B per 64-element K block
  static constexpr int a_kblock = K7_RB * 128;
  static constexpr int a_stage = (D / 64) * a_kblock;
  static constexpr int b_off = 0;
  static constexpr int a_off = b_off + (D / 64) * b_kblock;
  static constexpr int lut_off = a_off + 2 * a_stage;
  static constexpr int do0_off = lut_off + 512 * 4;           // int64 first token row of every chunk document
  static constexpr int trow_off = do0_off + K7_MAX_DOCS * 8;  // int64 first token row of every tile pass
  static constexpr int dlen_off = trow_off + K7_PASSES * 8;   // int tokens of every chunk document
  static constexpr int dnp_off = dlen_off + K7_MAX_DOCS * 4;  // int passes of every chunk document
  static constexpr int dpfx_off = dnp_off + K7_MAX_DOCS * 4;  // int passes of the chunk before the document
  static constexpr int tnv_off = dpfx_off + K7_MAX_DOCS * 4;  // int valid tokens of every tile pass
  static constexpr int tdoc_off = tnv_off + K7_PASSES * 4;    // int document (chunk slot) of every tile pass
  static constexpr int tseg_off = tdoc_off + K7_PASSES * 4;    // int first tile pass of every segment (+ end)
  static constexpr int tsegd_off = tseg_off + (K7_PASSES + 4) * 4;  // int document of every segment
  static constexpr int misc_off = tsegd_off + K7_PASSES * 4;
  static constexpr int bytes = misc_off + 64 + 1024;          // + slack for the 1024-byte alignment
};
static_assert(K7Smem<128>::bytes <= 227 * 1024, "K7 shared memory");

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// fp16(m) * 2^24 as an integer: exact for every fp16 value (the smallest subnormal is 2^-24, |m| <= 65504)
__device__ __forceinline__ long long k7_fixed(float m) {
  return __float2ll_rn(__half2float(__float2half_rn(m)) * 16777216.0f);
}

// The work of a launch.  K7_ALL is the product; the other two are timing variants that time one part of the loop
// alone (tools/bench_exhaustive.py, FPB_K7=mma|decode).  Their scores are meaningless.
enum K7Part { K7_ALL = 0, K7_MMA_ONLY = 1, K7_DECODE_ONLY = 2 };

// The lists of a list walk (read only when LIST): the kernel's N is then the list capacity `cap`, the row stride of
// `ids` and of `acc`
struct K7Lists {
  const int32_t* ids;        // [n_lists, cap] sorted-unique local document ids of every list
  const int32_t* count;      // [n_lists] their numbers
  const int32_t* chunk_pfx;  // [n_lists + 1] first chunk of every list (a list without queries has none)
  ExListTable t;             // query-row ranges of the lists, query and first token of every 16-row group
  int n_lists;
};

template <int D, int NBITS, int PART, bool LIST = false>
__global__ void __launch_bounds__(K7_THREADS, 1)
k7_exhaustive_kernel(const __half* __restrict__ C, const int64_t* __restrict__ doc_offsets,
                     const int32_t* __restrict__ codes, const uint8_t* __restrict__ residuals,
                     const __half* __restrict__ norms, WPerm wp, const __half* __restrict__ rows, int B, int Q,
                     int Qs, int n_rows, int64_t N, int docs_per_chunk, unsigned long long* __restrict__ acc,
                     float* __restrict__ carry_all, int* __restrict__ counter, K7Lists lst) {
  using S = K7Smem<D>;
  constexpr int PD = D * NBITS / 8;
  using Dec = Decoder<NBITS>;
  constexpr int LPT = PD / Dec::LANE_BYTES;  // lanes per token, LANE_BYTES packed bytes each
  constexpr int EPL = D / LPT;           // elements per lane
  constexpr int NH2 = EPL / 2;
  constexpr int TPR = K7_THREADS / LPT;  // tokens per decode round
  constexpr int ROUNDS = K7_TILE / TPR;
  constexpr int KS = D / 16;             // MMA k steps
  constexpr int CPR = D / 8;             // 16-byte chunks per row
  extern __shared__ unsigned char smem_dyn[];
  const uint32_t dyn_addr = smem_u32(smem_dyn);
  unsigned char* base = smem_dyn + ((1024u - (dyn_addr & 1023u)) & 1023u);  // SWIZZLE_128B atoms are 1024 B
  unsigned char* smB = base + S::b_off;
  unsigned char* smA = base + S::a_off;
  uint32_t* lut = reinterpret_cast<uint32_t*>(base + S::lut_off);
  int64_t* doc_o0 = reinterpret_cast<int64_t*>(base + S::do0_off);
  int64_t* t_row = reinterpret_cast<int64_t*>(base + S::trow_off);
  int* doc_len = reinterpret_cast<int*>(base + S::dlen_off);
  int* doc_np = reinterpret_cast<int*>(base + S::dnp_off);
  int* doc_pfx = reinterpret_cast<int*>(base + S::dpfx_off);
  int* t_nv = reinterpret_cast<int*>(base + S::tnv_off);
  int* t_doc = reinterpret_cast<int*>(base + S::tdoc_off);
  int* t_seg = reinterpret_cast<int*>(base + S::tseg_off);
  int* t_segdoc = reinterpret_cast<int*>(base + S::tsegd_off);
  int* misc = reinterpret_cast<int*>(base + S::misc_off);  // [0] chunk, [1] passes of the chunk, [2] tile segments

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int c = warp >> 2, w = warp & 3, quad = lane & 3;
  float* carry = carry_all + int64_t(blockIdx.x) * n_rows;
  Dec::build(lut, wp, tid, K7_THREADS);
  const int64_t n_chunks = LIST ? int64_t(lst.chunk_pfx[lst.n_lists]) : (N + docs_per_chunk - 1) / docs_per_chunk;
  const int n_rb = n_rows / K7_RB;

  // A stage: 128 query rows, K-major SWIZZLE_128B, one cp.async group per stage
  auto load_a = [&](int rb, int stage) {
    const __half* src = rows + int64_t(rb) * K7_RB * D;
    unsigned char* dst = smA + stage * S::a_stage;
    for (int i = tid; i < K7_RB * CPR; i += K7_THREADS) {
      const int r = i / CPR, cc = i % CPR;
      cp_async16(smem_u32(dst + sw128_off(r, cc, S::a_kblock)), src + int64_t(r) * D + cc * 8);
    }
    cp_async_commit();
  };

  for (;;) {
    __syncthreads();  // every role is done with the previous chunk's tables
    if (tid == 0) misc[0] = atomicAdd(counter, 1);
    if constexpr (LIST) {
      if (tid == 0 && misc[0] < n_chunks) {  // the chunk's list: the last l with chunk_pfx[l] <= chunk
        int lo = 0, hi = lst.n_lists - 1;
        while (lo < hi) {
          const int mid = (lo + hi + 1) >> 1;
          if (lst.chunk_pfx[mid] <= misc[0]) lo = mid;
          else hi = mid - 1;
        }
        misc[4] = lo;
      }
    }
    __syncthreads();
    const int64_t chunk = misc[0];
    if (chunk >= n_chunks) break;
    // full scan: documents d0 .. d0+nd-1.  List walk: positions d0 .. d0+nd-1 of list l, whose queries own the
    // query rows [row0, row1)
    int64_t d0;
    int nd, row0 = 0, row1 = 0;
    const int32_t* list = nullptr;
    if constexpr (LIST) {
      const int l = misc[4];
      d0 = (chunk - lst.chunk_pfx[l]) * docs_per_chunk;
      nd = min(docs_per_chunk, lst.count[l] - int(d0));
      list = lst.ids + int64_t(l) * N;
      row0 = lst.t.row0[l];
      row1 = lst.t.row1[l];
    } else {
      d0 = chunk * docs_per_chunk;
      nd = int(min(int64_t(docs_per_chunk), N - d0));
    }

    // ---- chunk metadata (warp 0): documents and their pass prefix ----
    if (warp == 0) {
      int np = 0, len = 0;
      int64_t o0 = 0;
      if (lane < nd) {
        const int64_t d = LIST ? int64_t(list[d0 + lane]) : d0 + lane;
        o0 = doc_offsets[d];
        len = int(doc_offsets[d + 1] - o0);
        np = (len + 7) >> 3;
      }
      int incl = np;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, off);
        if (lane >= off) incl += t;
      }
      if (lane < nd) {
        doc_o0[lane] = o0;
        doc_len[lane] = len;
        doc_np[lane] = np;
        doc_pfx[lane] = incl - np;
      }
      if (lane == 31) misc[1] = incl;
    }
    __syncthreads();
    const int n_pass = misc[1];

    for (int p0 = 0; p0 < n_pass; p0 += K7_PASSES) {
      const int tp = min(K7_PASSES, n_pass - p0);
      // ---- tile table: pass -> (first row, valid tokens, document) ----
      if (tid < tp) {
        const int g = p0 + tid;
        int i = 0;
        while (doc_pfx[i] + doc_np[i] <= g) ++i;  // documents without tokens own no pass and are skipped
        const int k = g - doc_pfx[i];
        t_row[tid] = doc_o0[i] + 8 * k;
        t_nv[tid] = min(8, doc_len[i] - 8 * k);
        t_doc[tid] = i;
      }
      if (warp == 0) {  // segments: maximal runs of tile passes of one document (the table above is warp 0's)
        __syncwarp();
        const bool start = lane < tp && (lane == 0 || t_doc[lane] != t_doc[lane - 1]);
        const unsigned starts = __ballot_sync(0xffffffffu, start);
        if (start) {
          const int sg = __popc(starts & ((1u << lane) - 1u));
          t_seg[sg] = lane;
          t_segdoc[sg] = t_doc[lane];
        }
        if (lane == 0) {
          misc[2] = __popc(starts);
          t_seg[__popc(starts)] = tp;
        }
      }
      // the A stages to stream: every one, or those that hold rows of the chunk's list
      const int rb_first = LIST ? row0 / K7_RB : 0;
      const int rb_end = LIST ? (row1 + K7_RB - 1) / K7_RB : n_rb;
      load_a(rb_first, rb_first & 1);  // in flight during the decode
      __syncthreads();

      // ---- decode the tile once: row r = tile pass r/8, token r%8 ----
      {
        const int sub = tid % LPT;
        const int nrow = tp * 8;
        int64_t tok[ROUNDS];
        int code[ROUNDS];
        typename Dec::Raw rv[ROUNDS];
#pragma unroll
        for (int u = 0; u < ROUNDS; ++u) {  // every load of the tile in flight before the first decode
          const int r = u * TPR + tid / LPT;
          tok[u] = 0;
          code[u] = 0;
          rv[u] = typename Dec::Raw{};
          if (r < nrow) {
            const int p = r >> 3;
            tok[u] = t_row[p] + min(r & 7, t_nv[p] - 1);
            code[u] = __ldg(codes + tok[u]);
            rv[u] = Dec::load(residuals + tok[u] * PD, sub);
          }
        }
#pragma unroll
        for (int u = 0; u < ROUNDS; ++u) {
          const int r = u * TPR + tid / LPT;
          if (r < nrow) {
            __half2 e[NH2];
            Dec::decode(lut, rv[u], reinterpret_cast<const uint4*>(C + int64_t(code[u]) * D + sub * EPL), e);
            const float nf = __half2float(norms[tok[u]]);
            const float rc = __frcp_rn(nf);
#pragma unroll
            for (int i = 0; i < EPL / 8; ++i)
              *reinterpret_cast<uint4*>(smB + sw128_off(r, sub * (EPL / 8) + i, S::b_kblock)) = ehat_chunk(e, i, nf, rc);
          }
        }
      }

      // ---- stream every query row past the tile ----
      const bool two_blocks = tp > 16;
      for (int rb = rb_first; rb < (PART == K7_DECODE_ONLY ? 0 : rb_end); ++rb) {
        if (rb + 1 < rb_end) {
          load_a(rb + 1, (rb + 1) & 1);
          cp_async_wait<1>();
        } else {
          cp_async_wait<0>();
        }
        fence_proxy_async();  // this thread's cp.async rows and decoded rows -> visible to wgmma
        __syncthreads();

        const uint32_t a_addr = smem_u32(smA + (rb & 1) * S::a_stage) + c * 8 * 1024;  // warpgroup c: rows 64c..
        const uint32_t b_addr = smem_u32(smB);
        // list walk: a warpgroup whose 64 rows hold no query of the chunk's list runs no MMA (warpgroup-uniform)
        const int wg_row = rb * K7_RB + c * 64;
        const bool mma = !LIST || (wg_row >= row0 && wg_row < row1);
        float acc0[64], acc1[64];
        if (mma) {
          wgmma_fence();
#pragma unroll
          for (int ks = 0; ks < KS; ++ks) {
            const uint32_t ka = (ks >> 2) * S::a_kblock + (ks & 3) * 32;
            const uint32_t kb = (ks >> 2) * S::b_kblock + (ks & 3) * 32;
            wgmma_m64n128k16(acc0, gmma_desc(a_addr + ka), gmma_desc(b_addr + kb), ks > 0 ? 1u : 0u);
          }
          wgmma_commit();
          if (two_blocks) {
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) {
              const uint32_t ka = (ks >> 2) * S::a_kblock + (ks & 3) * 32;
              const uint32_t kb = (ks >> 2) * S::b_kblock + (ks & 3) * 32;
              wgmma_m64n128k16(acc1, gmma_desc(a_addr + ka), gmma_desc(b_addr + 16 * 1024 + kb), ks > 0 ? 1u : 0u);
            }
            wgmma_commit();
          }
        }

        // thread (w, lane) holds rows wrow + lane/4 (+8) of the warp's 16 rows, all of query b.  List walk: the
        // table gives the query of the 16-row group (-1: padding) and the token of its first row, and a row is live
        // only when its query searches the chunk's list
        const int wrow = rb * K7_RB + c * 64 + 16 * w;
        const int r0 = wrow + (lane >> 2);
        const int gq = LIST ? lst.t.grp_query[wrow >> 4] : 0, gt = LIST ? lst.t.grp_tok[wrow >> 4] : 0;
        const int b = LIST ? max(gq, 0) : wrow / Qs, q0 = (LIST ? gt : wrow % Qs) + (lane >> 2);
        // warp-uniform: some row of this warp is a real query token
        const bool live = LIST ? gq >= 0 && gt < Q && wrow >= row0 && wrow < row1 : b < B && wrow % Qs < Q;
        int di = 0;
        float m0 = -INFINITY, m1 = -INFINITY;
        auto flush = [&]() {
          m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1));
          m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
          m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1));
          m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
          if (!live) return;
          const int pfx = doc_pfx[di], np = doc_np[di];
          if (pfx < p0 && quad == 0) {  // the document began in an earlier tile
            m0 = fmaxf(m0, __ldcg(carry + r0));
            m1 = fmaxf(m1, __ldcg(carry + r0 + 8));
          }
          if (pfx + np > p0 + K7_PASSES) {  // ... or goes on in the next one: keep the running maxima
            if (quad == 0) {
              __stcg(carry + r0, m0);
              __stcg(carry + r0 + 8, m1);
            }
            return;
          }
          long long v = 0;
          if (quad == 0) v = (q0 < Q ? k7_fixed(m0) : 0ll) + (q0 + 8 < Q ? k7_fixed(m1) : 0ll);
          v += __shfl_xor_sync(0xffffffffu, v, 4);
          v += __shfl_xor_sync(0xffffffffu, v, 8);
          v += __shfl_xor_sync(0xffffffffu, v, 16);
          if (lane == 0) atomicAdd(acc + int64_t(b) * N + d0 + di, static_cast<unsigned long long>(v));
        };
        // both blocks complete before the epilogue: reading acc0 while acc1 is in flight makes ptxas serialise
        // every wgmma of the kernel (C7514)
        wgmma_wait0();
        if (PART != K7_MMA_ONLY) {
          // per-pass maxima of rows r0, r0 + 8 (accumulator column group j = pass j of the block), then one masked
          // maximum and one flush per segment: the same code whatever the documents, no branch per pass
          float pm0[K7_PASSES], pm1[K7_PASSES];
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            pm0[j] = fmaxf(acc0[4 * j], acc0[4 * j + 1]);
            pm1[j] = fmaxf(acc0[4 * j + 2], acc0[4 * j + 3]);
          }
          if (two_blocks) {
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              pm0[16 + j] = fmaxf(acc1[4 * j], acc1[4 * j + 1]);
              pm1[16 + j] = fmaxf(acc1[4 * j + 2], acc1[4 * j + 3]);
            }
          } else {
#pragma unroll
            for (int j = 16; j < K7_PASSES; ++j) pm0[j] = pm1[j] = -INFINITY;
          }
          if (!mma) {  // a warpgroup that ran no MMA has no maxima
#pragma unroll
            for (int j = 0; j < K7_PASSES; ++j) pm0[j] = pm1[j] = -INFINITY;
          }
          const int n_seg = misc[2];
          for (int sg = 0; sg < n_seg; ++sg) {
            const int j0 = t_seg[sg], j1 = t_seg[sg + 1];
            di = t_segdoc[sg];
            m0 = m1 = -INFINITY;
#pragma unroll
            for (int j = 0; j < K7_PASSES; ++j) {
              const bool in = j >= j0 && j < j1;
              m0 = fmaxf(m0, in ? pm0[j] : -INFINITY);
              m1 = fmaxf(m1, in ? pm1[j] : -INFINITY);
            }
            flush();
          }
        } else {
          // timing variant: keep every accumulator live so that no MMA is dropped as dead code
          float x = -INFINITY;
#pragma unroll
          for (int j = 0; j < 64; ++j) x = fmaxf(x, two_blocks ? fmaxf(acc0[j], acc1[j]) : acc0[j]);
          if (x == 1234.5f) misc[3] = 1;
        }
        __syncthreads();  // both warpgroups are done with this A stage (and, after the last one, with the tile)
      }
    }
  }
}

// query b, token q -> row b*Qs + q of the dense row array; every other row is zero.  With grp_query (list walk):
// row r belongs to query grp_query[r/16] (-1: padding), token grp_tok[r/16] + r%16
__global__ void k7_pack_rows_kernel(const __half* __restrict__ q, int B, int Q, int Qs, int D, int64_t n_chunks16,
                                    const int32_t* __restrict__ grp_query, const int32_t* __restrict__ grp_tok,
                                    __half* __restrict__ rows) {
  const int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
  if (i >= n_chunks16) return;
  const int cpr = D / 8;
  const int64_t r = i / cpr;
  const int cc = int(i % cpr);
  int64_t b = r / Qs;
  int qq = int(r % Qs);
  if (grp_query) {
    b = grp_query[r >> 4];
    qq = grp_tok[r >> 4] + int(r & 15);
  }
  uint4 v = make_uint4(0u, 0u, 0u, 0u);
  if (b >= 0 && b < B && qq < Q) v = *reinterpret_cast<const uint4*>(q + (b * Q + qq) * D + cc * 8);
  reinterpret_cast<uint4*>(rows)[i] = v;
}

// exact fixed-point sum -> fp32 score; a document without tokens scores Q times the padding sentinel
__device__ __forceinline__ float k7_score(unsigned long long sum, bool empty, int Q) {
  return empty ? float(Q) * FPB_PAD_SENTINEL : __ll2float_rn(static_cast<long long>(sum)) * (1.0f / 16777216.0f);
}

// BIAS: the score of document d is biased by bias[d] (fpb_index_with_bias); the <false> instances ignore `bias`
template <bool BIAS>
__global__ void k7_finalize_kernel(const unsigned long long* __restrict__ acc, const int64_t* __restrict__ doc_offsets,
                                   int64_t N, int64_t total, int Q, float* __restrict__ scores,
                                   const float* __restrict__ bias) {
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t d = i % N;
    scores[i] = fpb_biased<BIAS>(k7_score(acc[i], doc_offsets[d + 1] == doc_offsets[d], Q), bias, d);
  }
}

// list walk: row b of the [B, cap] arrays k3b_select reads -- the scores of query b's list, its local document ids
// (the candidates, ascending) and their number.  Positions past the end of the list are not written.
template <bool BIAS>
__global__ void k7_list_finalize_kernel(const unsigned long long* __restrict__ acc,
                                        const int64_t* __restrict__ doc_offsets, const int32_t* __restrict__ ids,
                                        const int32_t* __restrict__ count, const int32_t* __restrict__ qlist,
                                        int64_t cap, int64_t total, int Q, float* __restrict__ scores,
                                        int32_t* __restrict__ cand, int32_t* __restrict__ n_cand,
                                        const float* __restrict__ bias) {
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t b = i / cap, p = i % cap;
    const int l = qlist[b], n = count[l];
    if (p == 0) n_cand[b] = n;
    if (p < n) {
      const int32_t d = ids[l * cap + p];
      cand[i] = d;
      scores[i] = fpb_biased<BIAS>(k7_score(acc[i], doc_offsets[d + 1] == doc_offsets[d], Q), bias, d);
    }
  }
}

// list walk, one CTA: pfx[l] = chunks of the lists before l (ceil(count / dpc) for a list that some query searches,
// none otherwise), pfx[n_lists] = all of them
__global__ void __launch_bounds__(1024)
k7_list_chunks_kernel(const int32_t* __restrict__ count, ExListTable t, int n_lists, int dpc, int32_t* __restrict__ pfx) {
  __shared__ int warp_sums[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int per = (n_lists + 1023) / 1024, l0 = min(n_lists, tid * per), l1 = min(n_lists, l0 + per);
  auto chunks = [&](int l) { return t.row1[l] > t.row0[l] ? (count[l] + dpc - 1) / dpc : 0; };
  int sum = 0;
  for (int l = l0; l < l1; ++l) sum += chunks(l);
  int incl = sum;
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
    warp_sums[lane] = wincl - ws;  // exclusive
  }
  __syncthreads();
  int run = warp_sums[warp] + incl - sum;
  for (int l = l0; l < l1; ++l) {
    pfx[l] = run;
    run += chunks(l);
  }
  if (tid == 1023) pfx[n_lists] = run;
}

// documents per chunk: as many as one warp scans, fewer (down to 4, as in v5) when that leaves too few chunks of
// `n_docs` documents to balance the SMs.  FPB_K7_DOCS_PER_CHUNK (kernels.h) pins it: the result does not depend on
// it, and the tests use it to run the multi-document chunk walk on small indexes.
int k7_docs_per_chunk(const fpb_index* ix, int64_t n_docs) {
  if (const int pin = fpb_env_int("FPB_K7_DOCS_PER_CHUNK", 1, K7_MAX_DOCS)) return pin;
  int dpc = K7_MAX_DOCS;
  while (dpc > 4 && (n_docs + dpc - 1) / dpc < int64_t(ix->sm_count) * 8) dpc >>= 1;
  return dpc;
}

// The K7 variant of a full scan, the whole rule: the timing variant FPB_K7=mma|decode asks for at dim 128 / nbits 4,
// the product (K7_ALL) otherwise.
K7Part k7_part(const fpb_index* ix) {
  if (ix->dim != 128 || ix->nbits != 4) return K7_ALL;
  if (fpb_env_is("FPB_K7", "mma")) return K7_MMA_ONLY;
  if (fpb_env_is("FPB_K7", "decode")) return K7_DECODE_ONLY;
  return K7_ALL;
}

template <int D, int NBITS, int PART, bool LIST = false>
int launch_k7_t(const fpb_index* ix, const ExLayout& X, char* ws, int dpc, cudaStream_t st,
                const K7Lists& lst = K7Lists{}) {
  auto kern = k7_exhaustive_kernel<D, NBITS, PART, LIST>;
  constexpr int smem = K7Smem<D>::bytes;
  // opt in on every launch: the attribute is per device and the call costs about a microsecond
  FPB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  // list walk: at most one partial chunk per list on top of the expected total length
  const int64_t chunks = LIST ? (X.list_docs + dpc - 1) / dpc + X.n_lists : (ix->N + dpc - 1) / dpc;
  const int blocks = int(chunks < X.grid ? chunks : X.grid);
  kern<<<blocks, K7_THREADS, smem, st>>>(ix->centroids, ix->doc_offsets, ix->doc_codes, ix->doc_residuals,
                                         ix->token_norms, ix->w_perm, reinterpret_cast<const __half*>(ws + X.off_rows), X.B,
                                         X.Q, X.Qs, X.n_rows, LIST ? X.cap : ix->N, dpc,
                                         reinterpret_cast<unsigned long long*>(ws + X.off_acc),
                                         reinterpret_cast<float*>(ws + X.off_carry),
                                         reinterpret_cast<int*>(ws + X.off_counter), lst);
  FPB_LAUNCH_CHECK("k7_exhaustive");
  return FPB_OK;
}

int finalize_blocks(const fpb_index* ix, int64_t total) {
  const int64_t want = (total + 255) / 256;
  return int(want < int64_t(ix->sm_count) * 16 ? want : int64_t(ix->sm_count) * 16);
}

}  // namespace

int launch_exhaustive_scores(const fpb_index* ix, const ExLayout& X, char* ws, const __half* d_queries,
                             float* d_scores, cudaStream_t st) {
  if (ix->N == 0) return FPB_OK;
  const int64_t n16 = int64_t(X.n_rows) * (ix->dim / 8);
  k7_pack_rows_kernel<<<int((n16 + 255) / 256), 256, 0, st>>>(d_queries, X.B, X.Q, X.Qs, ix->dim, n16, nullptr,
                                                               nullptr, reinterpret_cast<__half*>(ws + X.off_rows));
  FPB_LAUNCH_CHECK("k7_pack_rows");
  FPB_CUDA_CHECK(cudaMemsetAsync(ws + X.off_acc, 0, size_t(X.B) * ix->N * 8, st));
  FPB_CUDA_CHECK(cudaMemsetAsync(ws + X.off_counter, 0, sizeof(int), st));
  const K7Part part = k7_part(ix);
  const int dpc = k7_docs_per_chunk(ix, ix->N);
  FPB_TRY(fpb_with_codec(ix->dim, ix->nbits, "exhaustive search", [&](auto c) {
    if constexpr (c.D == 128 && c.NBITS == 4) {  // the timing variants exist at this codec only
      if (part == K7_MMA_ONLY) return launch_k7_t<128, 4, K7_MMA_ONLY>(ix, X, ws, dpc, st);
      if (part == K7_DECODE_ONLY) return launch_k7_t<128, 4, K7_DECODE_ONLY>(ix, X, ws, dpc, st);
    }
    return launch_k7_t<c.D, c.NBITS, K7_ALL>(ix, X, ws, dpc, st);
  }));
  const int64_t total = int64_t(X.B) * ix->N;
  (ix->doc_bias ? k7_finalize_kernel<true> : k7_finalize_kernel<false>)<<<finalize_blocks(ix, total), 256, 0, st>>>(
      reinterpret_cast<const unsigned long long*>(ws + X.off_acc), ix->doc_offsets, ix->N, total, X.Q, d_scores,
      ix->doc_bias);
  FPB_LAUNCH_CHECK("k7_finalize");
  return FPB_OK;
}

int launch_exhaustive_list_scores(const fpb_index* ix, const ExLayout& X, char* ws, const __half* d_queries,
                                  const ExLists& lists, cudaStream_t st) {
  const ExListTable t = ExListTable::at(reinterpret_cast<int32_t*>(ws + X.off_table), X.n_lists, X.B, X.n_rows);
  int32_t* ids = reinterpret_cast<int32_t*>(ws + X.off_lists);
  int32_t* count = reinterpret_cast<int32_t*>(ws + X.off_lcount);
  int32_t* chunk_pfx = reinterpret_cast<int32_t*>(ws + X.off_chunks);
  // 1. every list sorted and deduplicated: a document bitmap per list, compacted in id order
  uint32_t* bitmap = reinterpret_cast<uint32_t*>(ws + X.off_bitmap);
  if (lists.d_filters) {
    FPB_TRY(launch_filter_lists(ix, lists.d_filters, lists.n_bits, X.n_lists, bitmap, X.words, ids, int(X.cap), count,
                                st));
  } else {
    FPB_TRY(launch_doc_bitmap(ix, lists.d_list_ids, lists.d_list_offsets, lists.max_list_len, X.n_lists, bitmap,
                              X.words, st));
    FPB_TRY(launch_compact(bitmap, nullptr, X.words, ids, int(X.cap), count, X.n_lists, st));
  }
  const int dpc = k7_docs_per_chunk(ix, X.list_docs);
  k7_list_chunks_kernel<<<1, 1024, 0, st>>>(count, t, X.n_lists, dpc, chunk_pfx);
  FPB_LAUNCH_CHECK("k7_list_chunks");
  // 2. the query rows, grouped by list
  const int64_t n16 = int64_t(X.n_rows) * (ix->dim / 8);
  k7_pack_rows_kernel<<<int((n16 + 255) / 256), 256, 0, st>>>(d_queries, X.B, X.Q, X.Qs, ix->dim, n16, t.grp_query,
                                                               t.grp_tok, reinterpret_cast<__half*>(ws + X.off_rows));
  FPB_LAUNCH_CHECK("k7_pack_rows");
  FPB_CUDA_CHECK(cudaMemsetAsync(ws + X.off_acc, 0, size_t(X.B) * X.cap * 8, st));
  FPB_CUDA_CHECK(cudaMemsetAsync(ws + X.off_counter, 0, sizeof(int), st));
  // 3. K7 over the lists
  const K7Lists lst{ids, count, chunk_pfx, t, X.n_lists};
  FPB_TRY(fpb_with_codec(ix->dim, ix->nbits, "exhaustive search",
                         [&](auto c) { return launch_k7_t<c.D, c.NBITS, K7_ALL, true>(ix, X, ws, dpc, st, lst); }));
  // 4. the [B, cap] scores, candidates and counts of the selection
  const int64_t total = int64_t(X.B) * X.cap;
  (ix->doc_bias ? k7_list_finalize_kernel<true> : k7_list_finalize_kernel<false>)<<<finalize_blocks(ix, total), 256, 0,
                                                                                      st>>>(
      reinterpret_cast<const unsigned long long*>(ws + X.off_acc), ix->doc_offsets, ids, count, t.qlist, X.cap, total,
      X.Q, reinterpret_cast<float*>(ws + X.off_scores), reinterpret_cast<int32_t*>(ws + X.off_cand),
      reinterpret_cast<int32_t*>(ws + X.off_n_cand), ix->doc_bias);
  FPB_LAUNCH_CHECK("k7_list_finalize");
  return FPB_OK;
}
