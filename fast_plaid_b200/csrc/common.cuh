// Shared definitions for the sm_90a PLAID search kernels.
#pragma once

#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <mutex>

#include "../../include/fastplaid_b200.h"

struct WPerm {
  uint16_t v[16];
};

// The walk layout's two growable buffers (fpb_buffer_*), shared by an index and every index appended to it
// (fpb_index_append): a handle covers the first N + 1 entries of win and the windows they name, and the last
// fpb_index_destroy frees them.  n_docs is the number of documents laid out so far: only a handle over all of them
// may append, so that two appends never write the same windows.
struct fpb_walk {
  std::atomic<int> refs;
  std::mutex mu;  // held by an append
  fpb_buffer* codes;
  fpb_buffer* win;
  int64_t n_docs;
};

// Immutable index handle (replaces LoadedIndex, rust/search/load.rs:50-56).  Holds only
// borrowed device pointers plus the small derived codec table.
struct fpb_index {
  int device;
  int nbits;
  int dim;
  int pd;  // packed residual bytes per token = dim*nbits/8
  int sm_count;
  int64_t K;        // centroids
  int64_t N;        // local documents
  int64_t E;        // local tokens
  int64_t n_ivf;
  int64_t max_doc_len;
  int64_t doc_id_base;
  const __half* centroids;
  const int64_t* doc_offsets;
  const int32_t* doc_codes;
  const uint8_t* doc_residuals;
  // derived at load time: fp16 norm of every decompressed token, n_t = fp16(sqrt(sum_fp32 e^2)) (search.rs:86-93).
  // It is a property of the token, not of the (query, document) pair: the MaxSim kernels read it (2 B/token)
  // instead of re-deriving it for every pair.  Caller-owned buffer filled by fpb_index_create.
  const __half* token_norms;
  // derived at load time, shared through `walk` (refcounted): the approximate stage's copy of the codes (k3_approx.cu).  Document
  // d owns the 32-token windows walk_win[d] .. walk_win[d+1] - 1 (ceil(len/32) of them) of walk_codes; its codes
  // are dealt over them so that the bitmap words they test in shared memory spread over the 32 banks, and empty
  // slots hold padding codes >= K (fpb_walk_pad_code).  A max over a document's tokens does not depend on their
  // order, so every approximate score is unchanged.
  int32_t* walk_codes;  // [32 * walk_win[N]]
  int64_t* walk_win;    // [N + 1]
  fpb_walk* walk;       // the buffers behind walk_codes / walk_win
  // windows per group of the bound pass (4, 5 or 6), chosen at load: the group count of a document is rounded up to
  // whole groups, and the windows past its end still cost their bit tests, so the width that wastes the fewest
  // window slots over the index is taken (every 300-token document is 10 windows: 5; 1024 tokens: 4)
  int walk_group;
  // window slots of the whole index at groups of 4, 5 and 6 windows, from which walk_group is chosen: sums over the
  // documents, so an append adds its documents' slots
  int64_t walk_slots[3];
  const int64_t* ivf_offsets;  // nullptr => compress_only
  const int32_t* ivf_pids;
  // w_perm[i] = bucket_weights[bitrev_nbits(i)]  (closed form of the two LUTs of
  // residual_codec.rs:83-140): element j of a byte is w_perm[(byte >> (8-nbits*(j+1))) & mask]
  // (fp16 bit patterns, passed by value to every decoding kernel)
  WPerm w_perm;
  // TMA descriptor of the centroid table: 2-D [K, dim] fp16, box 64 x 128, SWIZZLE_128B
  // (cuTensorMapEncodeTiled through cudaGetDriverEntryPoint; has_tmap = 0 if unavailable)
  alignas(64) unsigned char tmap_centroids[128];
  int has_tmap;
  // grouped results (fpb_index_with_groups, groups.cu): the group of every local document, [N] in [0, n_groups),
  // borrowed like the other arrays; NULL / 0 on a handle without groups
  const int32_t* doc_group;
  int64_t n_groups;
  // documents kept per group (fpb_index_with_groups_max), in [1, FPB_MAX_PER_GROUP] on a handle with groups
  int max_per_group;
  // a shard-grouped handle (fpb_index_with_shard_groups) also carries the group of every document of the WHOLE
  // document-sharded index, [n_total_docs] by global id, for the merge across ranks; NULL / 0 otherwise
  const int32_t* global_group;
  int64_t n_total_docs;
  // biased scores (fpb_index_with_bias): an fp32 bias per local document, [N] by local id, borrowed like doc_group.
  // Every exact score is finished as __fadd_rn(score, doc_bias[d]) where it is stored (K5, K7's finalize), so that
  // everything that selects on it sees the biased score; NULL on a handle without a bias
  const float* doc_bias;
};

// The exact score of document d as every selection sees it: with a bias (BIAS, the template flag of the kernels that
// finish exact scores), one fp32 addition rounded to nearest, never contracted into a neighbouring multiply
template <bool BIAS>
__device__ __forceinline__ float fpb_biased(float s, const float* __restrict__ bias, int64_t d) {
  if constexpr (BIAS) return __fadd_rn(s, bias[d]);
  return s;
}

void fpb_set_error(const char* fmt, ...);

#define FPB_CUDA_CHECK(expr)                                                              \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      fpb_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return FPB_ERR_CUDA;                                                                \
    }                                                                                     \
  } while (0)

#define FPB_LAUNCH_CHECK(name)                                                            \
  do {                                                                                    \
    cudaError_t _e = cudaGetLastError();                                                  \
    if (_e != cudaSuccess) {                                                              \
      fpb_set_error("launch of %s failed: %s", name, cudaGetErrorString(_e));            \
      return FPB_ERR_CUDA;                                                                \
    }                                                                                     \
  } while (0)

// evaluate an FPB_* status expression; return its status from the caller unless it is FPB_OK
#define FPB_TRY(expr)              \
  do {                             \
    const int _rc = (expr);        \
    if (_rc != FPB_OK) return _rc; \
  } while (0)

static inline int64_t fpb_align256(int64_t x) { return (x + 255) & ~int64_t(255); }
// Words of a query's K-bit map of high centroids (two-pass approximate stage): a multiple of 4, so that the map is
// uint4-copyable.  The bound pass keeps 32 zero words after it in shared memory, one per bank.
static inline int fpb_hb_words(int64_t K) { return int(((K + 31) / 32 + 3) / 4 * 4); }
// The padding code of the walk layout whose bitmap word (hb_words + l' with (hb_words + l') % 32 == bank) is a zero
// word in `bank`: it never tests high, never adds a bank conflict to a window whose real codes leave `bank` free,
// and is >= K, so the walkers skip its gather.
__host__ __device__ inline int32_t fpb_walk_pad_code(int hb_words, int bank) {
  return int32_t(hb_words + ((bank - hb_words) & 31)) * 32;
}
static inline int fpb_next_pow2(int x) {
  int p = 1;
  while (p < x) p <<= 1;
  return p;
}

// ---------------------------------------------------------------------------------------
// Device helpers
// ---------------------------------------------------------------------------------------

// Monotone map float -> uint32 (larger float => larger key); -0.0 is folded onto +0.0 so
// that the canonical tie rule ("equal value => smaller id first") sees them as equal.
__device__ __forceinline__ uint32_t f32_key(float f) {
  uint32_t u = __float_as_uint(f);
  if ((u << 1) == 0u) u = 0u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float f32_unkey(uint32_t k) {
  uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  return __uint_as_float(u);
}
__device__ __forceinline__ uint32_t f16_key(uint16_t h) {
  uint32_t u = h;
  if ((u & 0x7fffu) == 0u) u = 0u;
  return (u & 0x8000u) ? (~u & 0xffffu) : (u | 0x8000u);
}

__device__ __forceinline__ uint4 ldg_nc_na(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void ldmatrix_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3,
                                            uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}

// D(16x8,f32) += A(16x16,f16,row) * B(16x8,f16,col)
__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0,
                                          uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint32_t pack_half2_rn(float lo, float hi) {
  __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ __half2 u32_as_half2(uint32_t u) { return *reinterpret_cast<__half2*>(&u); }
__device__ __forceinline__ uint32_t half2_as_u32(__half2 h) { return *reinterpret_cast<uint32_t*>(&h); }

// The padding sentinel of colbert_score_reduce: masked_fill(-9999.0) on an fp16 tensor
// stores -10000.0 (search.rs:395; fp16 spacing is 8 in [8192, 16384)).
#define FPB_PAD_SENTINEL (-10000.0f)
