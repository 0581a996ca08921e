// Search filters.  A filter's one device form is a packed bitmap over GLOBAL document ids: row f of a
// [n_filters, ceil(n_bits / 32)] uint32 array, bit i of word w standing for document 32 w + i.  Id lists and boolean
// masks are turned into it on the device (fpb_filter_from_ids / fpb_filter_from_mask), and a search takes the
// bitmaps plus a host map from query to filter.  The filter stage then builds, once per DISTINCT filter, exactly the
// per-query structures the list path's subset_mark_kernel builds once per query (the document bitmap `sbitmap` over
// the index's local range and the bitmap `cbitmap` of the centroids those documents touch), and copies them to the
// other queries of the filter.  Everything after it (k2_compact into clist, the subset probe, K2, K3, K5, K6; K7's
// list walk in the exhaustive search) runs unchanged on the same bytes.
#include <algorithm>
#include <vector>

#include "entry.h"

namespace {

int64_t filter_words(int64_t n_bits) { return (n_bits + 31) / 32; }

// ids [n_ids]: element i belongs to row f when row_offsets[f] <= i < row_offsets[f + 1]; ids outside [0, n_bits)
// and elements outside every row are ignored
__global__ void __launch_bounds__(256)
filter_ids_kernel(const int64_t* __restrict__ ids, int64_t n_ids, const int64_t* __restrict__ row_offsets,
                  int n_filters, int64_t n_bits, int64_t words, uint32_t* __restrict__ bitmap) {
  const int64_t first = row_offsets[0], last = row_offsets[n_filters];
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n_ids; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t id = ids[i];
    if (id < 0 || id >= n_bits || i < first || i >= last) continue;
    int lo = 0, hi = n_filters - 1;  // the last row starting at or before i
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (row_offsets[mid] <= i) lo = mid; else hi = mid - 1;
    }
    atomicOr(bitmap + int64_t(lo) * words + (id >> 5), 1u << (id & 31));
  }
}

// mask [n_filters, n_bits] (nonzero byte = set) -> bitmap [n_filters, words]: one warp per output word, one ballot
__global__ void __launch_bounds__(256)
filter_mask_kernel(const uint8_t* __restrict__ mask, int n_filters, int64_t n_bits, int64_t words,
                   uint32_t* __restrict__ bitmap) {
  const int lane = threadIdx.x & 31;
  const int64_t total = int64_t(n_filters) * words;
  const int64_t stride = (int64_t(gridDim.x) * blockDim.x) >> 5;
  for (int64_t w = (blockIdx.x * int64_t(blockDim.x) + threadIdx.x) >> 5; w < total; w += stride) {
    const int64_t f = w / words, bit = (w - f * words) * 32 + lane;
    const uint32_t v = __ballot_sync(0xffffffffu, bit < n_bits && mask[f * n_bits + bit] != 0);
    if (lane == 0) bitmap[w] = v;
  }
}

// Row b of `out` ([rows, out_words]) = bits [base, base + n) of filter row qf[b] (row b when qf is NULL), bits past n
// cleared.  With `src`, only the rows with src[b] == b (the first query of each filter) are written.
__global__ void __launch_bounds__(256)
filter_expand_kernel(const uint32_t* __restrict__ filters, int64_t fwords, int64_t base, int64_t n,
                     const int32_t* __restrict__ src, const int32_t* __restrict__ qf, uint32_t* __restrict__ out,
                     int out_words) {
  const int b = blockIdx.y;
  if (src && src[b] != b) return;
  const uint32_t* row = filters + int64_t(qf ? qf[b] : b) * fwords;
  uint32_t* o = out + int64_t(b) * out_words;
  const int64_t w0 = base >> 5;
  const int sh = int(base & 31);
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < out_words; j += gridDim.x * blockDim.x) {
    const int64_t g = w0 + j;
    const uint32_t lo = g < fwords ? row[g] : 0u;
    const uint32_t hi = g + 1 < fwords ? row[g + 1] : 0u;
    uint32_t v = __funnelshift_r(lo, hi, sh);
    const int64_t left = n - int64_t(j) * 32;  // bits of word j inside the range
    if (left <= 0) v = 0u;
    else if (left < 32) v &= (1u << left) - 1u;
    o[j] = v;
  }
}

// Row b of cbitmap |= the centroids of every local document set in row b of sbitmap, for the rows with src[b] == b.
// One warp per document-bitmap word.  SHARED: accumulated in a [cwords] shared-memory bitmap that the CTA ORs into
// the row once; otherwise straight into the row with global atomics (K too large for shared memory).
template <bool SHARED>
__global__ void __launch_bounds__(256)
filter_centroids_kernel(const uint32_t* __restrict__ sbitmap, int words, const int64_t* __restrict__ doc_offsets,
                        const int32_t* __restrict__ codes, const int32_t* __restrict__ src,
                        uint32_t* __restrict__ cbitmap, int cwords) {
  extern __shared__ uint32_t s_cb[];
  const int b = blockIdx.y;
  if (src[b] != b) return;  // uniform over the CTA
  uint32_t* cb = cbitmap + int64_t(b) * cwords;
  if constexpr (SHARED) {
    for (int i = threadIdx.x; i < cwords; i += blockDim.x) s_cb[i] = 0u;
    __syncthreads();
  }
  uint32_t* acc = SHARED ? s_cb : cb;
  const uint32_t* sb = sbitmap + int64_t(b) * words;
  const int lane = threadIdx.x & 31, warps = blockDim.x >> 5;
  for (int64_t j = int64_t(blockIdx.x) * warps + (threadIdx.x >> 5); j < words; j += int64_t(gridDim.x) * warps) {
    uint32_t m = sb[j];
    while (m) {
      const int64_t d = j * 32 + (__ffs(m) - 1);
      m &= m - 1;
      const int64_t o1 = doc_offsets[d + 1];
      for (int64_t t = doc_offsets[d] + lane; t < o1; t += 32) {
        const int c = __ldg(codes + t);
        atomicOr(acc + (c >> 5), 1u << (c & 31));
      }
    }
  }
  if constexpr (SHARED) {
    __syncthreads();
    for (int i = threadIdx.x; i < cwords; i += blockDim.x) {
      const uint32_t v = s_cb[i];
      if (v) atomicOr(cb + i, v);
    }
  }
}

// row b of rows ([B, words]) = row src[b], for every b with src[b] != b
__global__ void __launch_bounds__(256)
filter_broadcast_kernel(const int32_t* __restrict__ src, uint32_t* __restrict__ rows, int words) {
  const int b = blockIdx.y, s = src[b];
  if (s == b) return;
  const uint32_t* from = rows + int64_t(s) * words;
  uint32_t* to = rows + int64_t(b) * words;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < words; j += gridDim.x * blockDim.x) to[j] = from[j];
}

int blocks_for(int64_t items, int per_block, int cap) {
  const int64_t need = (items + per_block - 1) / per_block;
  return int(need < 1 ? 1 : (need < cap ? need : cap));
}

int max_optin_smem(int device) {
  int v = 0;
  if (cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, device) != cudaSuccess) return 0;
  return v;
}

}  // namespace

bool fpb_filter_centroids_in_shared(const fpb_index* ix, int cwords) {
  return int64_t(cwords) * 4 <= max_optin_smem(ix->device);
}

int launch_filter(const fpb_index* ix, const Ws& ws, const uint32_t* d_filters, int n_filters, int64_t n_bits,
                  const int32_t* h_query_filter, cudaStream_t st) {
  const fpb_layout& L = *ws.L;
  if (L.off_sbitmap == L.off_cbitmap) {
    fpb_set_error("filtered search needs a workspace laid out with FPB_FLAG_SUBSET");
    return FPB_ERR_INVALID;
  }
  const int B = L.B;
  FPB_CUDA_CHECK(cudaMemsetAsync(ws.cbitmap(), 0, size_t(B) * L.cbitmap_words * 4, st));
  if (ix->N == 0) {
    FPB_CUDA_CHECK(cudaMemsetAsync(ws.sbitmap(), 0, size_t(B) * L.bitmap_words * 4, st));
    return FPB_OK;
  }
  // src[b]: the first query of b's filter; qf[b]: b's filter.  Staged in K2's bitmap region (>= 2 words per query
  // when N >= 1), which K2 clears before it uses it.
  std::vector<int32_t> table(size_t(2) * B);
  std::vector<int32_t> first(size_t(n_filters), -1);
  bool shared = false;
  for (int b = 0; b < B; ++b) {
    int32_t& f0 = first[h_query_filter[b]];
    if (f0 < 0) f0 = b;
    else shared = true;
    table[b] = f0;
    table[B + b] = h_query_filter[b];
  }
  int32_t* d_src = reinterpret_cast<int32_t*>(ws.bitmap());
  int32_t* d_qf = d_src + B;
  // pageable source: staged before the call returns, so the host table may go out of scope
  FPB_CUDA_CHECK(cudaMemcpyAsync(d_src, table.data(), table.size() * 4, cudaMemcpyHostToDevice, st));
  const int cap = ix->sm_count * 4;
  filter_expand_kernel<<<dim3(blocks_for(L.bitmap_words, 256, cap), B), 256, 0, st>>>(
      d_filters, filter_words(n_bits), ix->doc_id_base, ix->N, d_src, d_qf, ws.sbitmap(), L.bitmap_words);
  FPB_LAUNCH_CHECK("filter_expand");
  const int n_rows = int(first.size()) - int(std::count(first.begin(), first.end(), -1));
  const int per_row = blocks_for(L.bitmap_words, 8 * 4, std::max(1, ix->sm_count * 2 / n_rows));
  const int cwords = L.cbitmap_words;
  if (fpb_filter_centroids_in_shared(ix, cwords)) {
    const int smem = cwords * 4;
    FPB_CUDA_CHECK(cudaFuncSetAttribute(filter_centroids_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        smem));
    filter_centroids_kernel<true><<<dim3(per_row, B), 256, smem, st>>>(ws.sbitmap(), L.bitmap_words, ix->doc_offsets,
                                                                     ix->doc_codes, d_src, ws.cbitmap(), cwords);
  } else {
    filter_centroids_kernel<false><<<dim3(per_row, B), 256, 0, st>>>(ws.sbitmap(), L.bitmap_words, ix->doc_offsets,
                                                                    ix->doc_codes, d_src, ws.cbitmap(), cwords);
  }
  FPB_LAUNCH_CHECK("filter_centroids");
  if (shared) {
    filter_broadcast_kernel<<<dim3(blocks_for(L.bitmap_words, 256, cap), B), 256, 0, st>>>(d_src, ws.sbitmap(),
                                                                                          L.bitmap_words);
    FPB_LAUNCH_CHECK("filter_broadcast");
    filter_broadcast_kernel<<<dim3(blocks_for(cwords, 256, cap), B), 256, 0, st>>>(d_src, ws.cbitmap(), cwords);
    FPB_LAUNCH_CHECK("filter_broadcast");
  }
  return FPB_OK;
}

int launch_filter_lists(const fpb_index* ix, const uint32_t* d_filters, int64_t n_bits, int n_lists,
                        uint32_t* bitmap, int words, int32_t* ids, int cap, int32_t* count, cudaStream_t st) {
  if (words > 0) {
    filter_expand_kernel<<<dim3(blocks_for(words, 256, ix->sm_count * 4), n_lists), 256, 0, st>>>(
        d_filters, filter_words(n_bits), ix->doc_id_base, ix->N, nullptr, nullptr, bitmap, words);
    FPB_LAUNCH_CHECK("filter_expand");
  }
  return launch_compact(bitmap, nullptr, words, ids, cap, count, n_lists, st);
}

int check_filter_args(const char* who, const uint32_t* d_filters, int n_filters, int64_t n_bits,
                      const int32_t* h_query_filter, int B) {
  if (!d_filters || !h_query_filter) {
    fpb_set_error("%s: NULL filter bitmap or query-filter map", who);
    return FPB_ERR_INVALID;
  }
  if (n_filters < 1 || n_bits < 0) {
    fpb_set_error("%s: n_filters=%d must be >= 1 and n_bits=%lld >= 0", who, n_filters, (long long)n_bits);
    return FPB_ERR_INVALID;
  }
  if (n_filters > 65535) {  // one grid row per filter
    fpb_set_error("%s: n_filters=%d exceeds the supported maximum of 65535", who, n_filters);
    return FPB_ERR_UNSUPPORTED;
  }
  for (int b = 0; b < B; ++b) {
    if (h_query_filter[b] < 0 || h_query_filter[b] >= n_filters) {
      fpb_set_error("%s: h_query_filter[%d]=%d is not in [0, n_filters=%d)", who, b, h_query_filter[b], n_filters);
      return FPB_ERR_INVALID;
    }
  }
  return FPB_OK;
}

extern "C" int fpb_filter_from_ids(int device, const int64_t* d_ids, int64_t n_ids, int n_filters,
                                   const int64_t* d_row_offsets, int64_t n_bits, uint32_t* d_bitmap, void* stream) {
  if ((n_ids > 0 && !d_ids) || !d_row_offsets || !d_bitmap) {
    fpb_set_error("fpb_filter_from_ids: NULL ids, row offsets or bitmap");
    return FPB_ERR_INVALID;
  }
  if (n_filters < 1 || n_bits < 0 || n_ids < 0) {
    fpb_set_error("fpb_filter_from_ids: n_filters=%d must be >= 1, n_bits=%lld and n_ids=%lld >= 0", n_filters,
                  (long long)n_bits, (long long)n_ids);
    return FPB_ERR_INVALID;
  }
  const int64_t words = filter_words(n_bits);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  FPB_CUDA_CHECK(cudaSetDevice(device));
  if (words == 0) return FPB_OK;
  FPB_CUDA_CHECK(cudaMemsetAsync(d_bitmap, 0, size_t(n_filters) * words * 4, st));
  if (n_ids == 0) return FPB_OK;
  int sms = 0;
  FPB_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  filter_ids_kernel<<<blocks_for(n_ids, 256, sms * 16), 256, 0, st>>>(d_ids, n_ids, d_row_offsets, n_filters, n_bits,
                                                                      words, d_bitmap);
  FPB_LAUNCH_CHECK("filter_ids");
  return FPB_OK;
}

extern "C" int fpb_filter_from_mask(int device, const uint8_t* d_mask, int n_filters, int64_t n_bits,
                                    uint32_t* d_bitmap, void* stream) {
  if (!d_mask || !d_bitmap) {
    fpb_set_error("fpb_filter_from_mask: NULL mask or bitmap");
    return FPB_ERR_INVALID;
  }
  if (n_filters < 1 || n_bits < 0) {
    fpb_set_error("fpb_filter_from_mask: n_filters=%d must be >= 1 and n_bits=%lld >= 0", n_filters,
                  (long long)n_bits);
    return FPB_ERR_INVALID;
  }
  const int64_t words = filter_words(n_bits);
  FPB_CUDA_CHECK(cudaSetDevice(device));
  if (words == 0) return FPB_OK;
  int sms = 0;
  FPB_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  filter_mask_kernel<<<blocks_for(int64_t(n_filters) * words, 8, sms * 16), 256, 0,
                       static_cast<cudaStream_t>(stream)>>>(d_mask, n_filters, n_bits, words, d_bitmap);
  FPB_LAUNCH_CHECK("filter_mask");
  return FPB_OK;
}
