// Shrinking an index: fpb_docs_compact (the kept documents' offsets and rows, in order, in new arrays) and
// fpb_ivf_delete (the inverted file of the kept documents, renumbered).  Both find how many dropped documents lie
// below a document d in O(1): a bitmap of the dropped documents and a rank table, rank[w] = dropped documents in
// bitmap words < w, give rank[d / 32] + popc(the word's bits below d).
#include <string.h>

#include "kernels.h"

namespace {

constexpr int DEL_THREADS = 256;

// The dropped documents' bits (bitmap zeroed by the caller), and, when dlen is not NULL, each one's token count.
// An id outside [0, n_docs) or not above the one before it sets *bad and is left out.
__global__ void __launch_bounds__(DEL_THREADS)
drop_mark_kernel(const int32_t* __restrict__ drop, int64_t n_drop, int64_t n_docs, const int64_t* __restrict__ offsets,
                 uint32_t* __restrict__ bitmap, int64_t* __restrict__ dlen, int* __restrict__ bad) {
  for (int64_t i = int64_t(blockIdx.x) * DEL_THREADS + threadIdx.x; i < n_drop; i += int64_t(gridDim.x) * DEL_THREADS) {
    const int64_t id = drop[i];
    const bool ok = id >= 0 && id < n_docs && (i == 0 || drop[i - 1] < id);
    if (!ok) *bad = 1;
    else atomicOr(bitmap + (id >> 5), 1u << (id & 31));
    if (dlen) dlen[i] = ok ? offsets[id + 1] - offsets[id] : 0;
  }
}

__global__ void __launch_bounds__(DEL_THREADS)
word_count_kernel(const uint32_t* __restrict__ bitmap, int64_t words, int64_t* __restrict__ count) {
  for (int64_t w = int64_t(blockIdx.x) * DEL_THREADS + threadIdx.x; w < words; w += int64_t(gridDim.x) * DEL_THREADS)
    count[w] = __popc(bitmap[w]);
}

__device__ __forceinline__ bool is_dropped(const uint32_t* bitmap, int64_t d) { return (bitmap[d >> 5] >> (d & 31)) & 1u; }

__device__ __forceinline__ int64_t dropped_below(const uint32_t* bitmap, const int64_t* rank, int64_t d) {
  return rank[d >> 5] + __popc(bitmap[d >> 5] & ((1u << (d & 31)) - 1u));
}

// Kept document d (and d = n_docs, the end) -> out[d - dropped below d] = offsets[d] - tokens of the dropped below d.
__global__ void __launch_bounds__(DEL_THREADS)
compact_offsets_kernel(const int64_t* __restrict__ offsets, int64_t n_docs, const uint32_t* __restrict__ bitmap,
                       const int64_t* __restrict__ rank, const int64_t* __restrict__ dprefix, int64_t* __restrict__ out) {
  for (int64_t d = int64_t(blockIdx.x) * DEL_THREADS + threadIdx.x; d <= n_docs; d += int64_t(gridDim.x) * DEL_THREADS) {
    if (d < n_docs && is_dropped(bitmap, d)) continue;
    const int64_t below = dropped_below(bitmap, rank, d);
    out[d - below] = offsets[d] - dprefix[below];
  }
}

// One warp per kept document: its codes, residual rows (16-byte vectors, pd / 16 per row) and, when norms is not NULL,
// token norms, from its old place to out_offsets[its rank among the kept].
__global__ void __launch_bounds__(DEL_THREADS)
compact_rows_kernel(const int64_t* __restrict__ offsets, int64_t n_docs, const uint32_t* __restrict__ bitmap,
                    const int64_t* __restrict__ rank, const int64_t* __restrict__ out_offsets, int vec_per_row,
                    const int32_t* __restrict__ codes, const uint4* __restrict__ res, const __half* __restrict__ norms,
                    int32_t* __restrict__ out_codes, uint4* __restrict__ out_res, __half* __restrict__ out_norms) {
  const int lane = threadIdx.x & 31;
  for (int64_t d = (int64_t(blockIdx.x) * DEL_THREADS + threadIdx.x) / 32; d < n_docs;
       d += int64_t(gridDim.x) * (DEL_THREADS / 32)) {
    if (is_dropped(bitmap, d)) continue;
    const int64_t src = offsets[d], len = offsets[d + 1] - src;
    const int64_t dst = out_offsets[d - dropped_below(bitmap, rank, d)];
    const uint4* s = res + src * vec_per_row;
    uint4* o = out_res + dst * vec_per_row;
    const int64_t nv = len * vec_per_row;
    int64_t i = lane;
    for (; i + 96 < nv; i += 128) {  // four 16-byte loads in flight per lane
      const uint4 a = s[i], b = s[i + 32], c = s[i + 64], e = s[i + 96];
      o[i] = a;
      o[i + 32] = b;
      o[i + 64] = c;
      o[i + 96] = e;
    }
    for (; i < nv; i += 32) o[i] = s[i];
    for (int64_t t = lane; t < len; t += 32) {
      out_codes[dst + t] = codes[src + t];
      if (norms) out_norms[dst + t] = norms[src + t];
    }
  }
}

// One warp per cell: its postings whose document is kept, counted into count[c] (count != NULL) or written, in order
// and renumbered, from out_pids[out_offsets[c]].  A posting outside [0, n_docs) sets *bad.
__global__ void __launch_bounds__(DEL_THREADS)
ivf_keep_kernel(const int64_t* __restrict__ ivf_offsets, const int32_t* __restrict__ pids, int64_t n_cells,
                int64_t n_docs, const uint32_t* __restrict__ bitmap, const int64_t* __restrict__ rank,
                int64_t* __restrict__ count, const int64_t* __restrict__ out_offsets, int32_t* __restrict__ out_pids,
                int* __restrict__ bad) {
  const int lane = threadIdx.x & 31;
  const uint32_t lt = (1u << lane) - 1u;
  for (int64_t c = (int64_t(blockIdx.x) * DEL_THREADS + threadIdx.x) / 32; c < n_cells;
       c += int64_t(gridDim.x) * (DEL_THREADS / 32)) {
    const int64_t o1 = ivf_offsets[c + 1];
    int64_t at = count ? 0 : out_offsets[c];
    for (int64_t i0 = ivf_offsets[c]; i0 < o1; i0 += 32) {
      const int64_t i = i0 + lane;
      bool keep = false;
      int64_t p = 0;
      if (i < o1) {
        p = pids[i];
        if (p < 0 || p >= n_docs) *bad = 1;
        else keep = !is_dropped(bitmap, p);
      }
      const uint32_t m = __ballot_sync(0xffffffffu, keep);
      if (!count && keep) out_pids[at + __popc(m & lt)] = int32_t(p - dropped_below(bitmap, rank, p));
      at += __popc(m);
    }
    if (count && lane == 0) count[c] = at;
  }
}

// Device scratch of the rank table over n_docs documents: words = n_docs / 32 + 1 (the word of d = n_docs exists, and
// has no bit set), so that the end of the index ranks like a kept document.
struct DropRank {
  int64_t words;
  uint32_t* bitmap;  // [words]
  int64_t* wcount;   // [words]
  int64_t* rank;     // [words + 1]
  int* bad;
  static int64_t words_for(int64_t n_docs) { return (n_docs >> 5) + 1; }
  static int64_t bytes(int64_t n_docs) {
    const int64_t w = words_for(n_docs);
    return fpb_align256(w * 4) + fpb_align256(w * 8) + fpb_align256((w + 1) * 8) + 256;
  }
  static DropRank at(char* p, int64_t n_docs) {
    const int64_t w = words_for(n_docs);
    DropRank r;
    r.words = w;
    r.bitmap = reinterpret_cast<uint32_t*>(p);
    r.wcount = reinterpret_cast<int64_t*>(p + fpb_align256(w * 4));
    r.rank = reinterpret_cast<int64_t*>(p + fpb_align256(w * 4) + fpb_align256(w * 8));
    r.bad = reinterpret_cast<int*>(p + fpb_align256(w * 4) + fpb_align256(w * 8) + fpb_align256((w + 1) * 8));
    return r;
  }
};

// The bitmap and rank table of the dropped ids (and, when dlen is not NULL, their token counts), after checking that
// the ids are sorted, unique and in [0, n_docs).  Synchronises `st` once.
int build_drop_rank(const char* who, const DropRank& r, const int32_t* d_drop, int64_t n_drop, int64_t n_docs,
                    const int64_t* d_offsets, int64_t* dlen, int sm_count, cudaStream_t st) {
  FPB_CUDA_CHECK(cudaMemsetAsync(r.bitmap, 0, r.words * 4, st));
  FPB_CUDA_CHECK(cudaMemsetAsync(r.bad, 0, sizeof(int), st));
  if (n_drop > 0) {
    drop_mark_kernel<<<fpb_grid_for(n_drop, DEL_THREADS, sm_count), DEL_THREADS, 0, st>>>(d_drop, n_drop, n_docs,
                                                                                          d_offsets, r.bitmap, dlen,
                                                                                          r.bad);
    FPB_LAUNCH_CHECK("drop_mark");
  }
  int flag = 0;
  FPB_CUDA_CHECK(cudaMemcpyAsync(&flag, r.bad, sizeof(int), cudaMemcpyDeviceToHost, st));
  FPB_CUDA_CHECK(cudaStreamSynchronize(st));
  if (flag) {
    fpb_set_error("%s: the dropped ids must be sorted, unique and in [0, %lld)", who, (long long)n_docs);
    return FPB_ERR_INVALID;
  }
  word_count_kernel<<<fpb_grid_for(r.words, DEL_THREADS, sm_count), DEL_THREADS, 0, st>>>(r.bitmap, r.words, r.wcount);
  FPB_LAUNCH_CHECK("word_count");
  return launch_offsets_scan(nullptr, r.wcount, r.words, r.rank, nullptr, st);
}

int sm_count_of(int device, int* sm_count) {
  FPB_CUDA_CHECK(cudaSetDevice(device));
  FPB_CUDA_CHECK(cudaDeviceGetAttribute(sm_count, cudaDevAttrMultiProcessorCount, device));
  return FPB_OK;
}

}  // namespace

extern "C" int fpb_docs_compact(int device, int64_t n_docs, const int64_t* d_doc_offsets, const int32_t* d_doc_codes,
                                const uint8_t* d_doc_residuals, const void* d_token_norms, int pd,
                                const int32_t* d_drop, int64_t n_drop, int64_t* d_out_offsets, int32_t* d_out_codes,
                                uint8_t* d_out_residuals, void* d_out_norms, int64_t out_capacity,
                                int64_t* h_n_tokens, void* stream) {
  if (n_docs < 0 || n_drop < 0 || n_drop > n_docs || out_capacity < 0 || !d_doc_offsets || !d_out_offsets ||
      !h_n_tokens || (n_drop > 0 && !d_drop)) {
    fpb_set_error("fpb_docs_compact: bad sizes or NULL pointers");
    return FPB_ERR_INVALID;
  }
  if (d_out_codes && (!d_doc_codes || !d_doc_residuals || !d_out_residuals || !d_token_norms != !d_out_norms)) {
    fpb_set_error("fpb_docs_compact: NULL row arrays (codes and residuals, in and out; norms in both or in neither)");
    return FPB_ERR_INVALID;
  }
  if ((reinterpret_cast<uintptr_t>(d_doc_residuals) | reinterpret_cast<uintptr_t>(d_out_residuals)) & 15) {
    fpb_set_error("fpb_docs_compact: the residual arrays must be 16-byte aligned");
    return FPB_ERR_INVALID;
  }
  if (pd != 16 && pd != 32 && pd != 64) {
    fpb_set_error("fpb_docs_compact: %d bytes per residual row; supported: 16, 32 and 64", pd);
    return FPB_ERR_UNSUPPORTED;
  }
  if (n_docs >= (int64_t(1) << 31)) {
    fpb_set_error("fpb_docs_compact: n_docs must fit in int32");
    return FPB_ERR_UNSUPPORTED;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int sm_count = 0;
  FPB_TRY(sm_count_of(device, &sm_count));
  const int64_t rank_bytes = DropRank::bytes(n_docs), drop_bytes = fpb_align256(n_drop * 8 + 8);
  char* scratch = nullptr;
  FPB_CUDA_CHECK(cudaMalloc(&scratch, rank_bytes + 2 * drop_bytes));
  const DropRank r = DropRank::at(scratch, n_docs);
  int64_t* dlen = reinterpret_cast<int64_t*>(scratch + rank_bytes);               // [n_drop] tokens of each dropped
  int64_t* dprefix = reinterpret_cast<int64_t*>(scratch + rank_bytes + drop_bytes);  // [n_drop + 1] their prefix
  auto run = [&]() -> int {
    FPB_TRY(build_drop_rank("fpb_docs_compact", r, d_drop, n_drop, n_docs, d_doc_offsets, dlen, sm_count, st));
    FPB_TRY(launch_offsets_scan(nullptr, dlen, n_drop, dprefix, nullptr, st));
    compact_offsets_kernel<<<fpb_grid_for(n_docs + 1, DEL_THREADS, sm_count), DEL_THREADS, 0, st>>>(
        d_doc_offsets, n_docs, r.bitmap, r.rank, dprefix, d_out_offsets);
    FPB_LAUNCH_CHECK("compact_offsets");
    int64_t total = 0;
    FPB_CUDA_CHECK(cudaMemcpyAsync(&total, d_out_offsets + (n_docs - n_drop), sizeof(int64_t), cudaMemcpyDeviceToHost,
                                   st));
    FPB_CUDA_CHECK(cudaStreamSynchronize(st));
    *h_n_tokens = total;
    if (!d_out_codes) return FPB_OK;  // the offsets and the size alone
    if (total > out_capacity) {
      fpb_set_error("fpb_docs_compact: %lld tokens do not fit in %lld", (long long)total, (long long)out_capacity);
      return FPB_ERR_INVALID;
    }
    if (n_docs - n_drop > 0) {
      compact_rows_kernel<<<fpb_grid_for((n_docs - n_drop) * 32, DEL_THREADS, sm_count), DEL_THREADS, 0, st>>>(
          d_doc_offsets, n_docs, r.bitmap, r.rank, d_out_offsets, pd / 16, d_doc_codes,
          reinterpret_cast<const uint4*>(d_doc_residuals), static_cast<const __half*>(d_token_norms), d_out_codes,
          reinterpret_cast<uint4*>(d_out_residuals), static_cast<__half*>(d_out_norms));
      FPB_LAUNCH_CHECK("compact_rows");
    }
    FPB_CUDA_CHECK(cudaStreamSynchronize(st));
    return FPB_OK;
  };
  const int rc = run();
  cudaStreamSynchronize(st);
  cudaFree(scratch);
  return rc;
}

extern "C" int fpb_ivf_delete(int device, int64_t n_cells, const int64_t* d_ivf_offsets, const int32_t* d_ivf_pids,
                              int64_t n_docs, const int32_t* d_drop, int64_t n_drop, int64_t* d_out_offsets,
                              int32_t* d_out_pids, int64_t out_capacity, int64_t* h_n_ivf, void* stream) {
  if (n_cells <= 0 || n_docs < 0 || n_drop < 0 || n_drop > n_docs || out_capacity < 0 || !d_ivf_offsets ||
      !d_out_offsets || !h_n_ivf || (n_drop > 0 && !d_drop)) {
    fpb_set_error("fpb_ivf_delete: bad sizes or NULL pointers");
    return FPB_ERR_INVALID;
  }
  if (n_docs >= (int64_t(1) << 31)) {
    fpb_set_error("fpb_ivf_delete: document ids must fit in int32");
    return FPB_ERR_UNSUPPORTED;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int sm_count = 0;
  FPB_TRY(sm_count_of(device, &sm_count));
  int64_t n_old = 0;
  FPB_CUDA_CHECK(cudaMemcpyAsync(&n_old, d_ivf_offsets + n_cells, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  FPB_CUDA_CHECK(cudaStreamSynchronize(st));
  if (n_old > 0 && !d_ivf_pids) {
    fpb_set_error("fpb_ivf_delete: d_ivf_pids is NULL");
    return FPB_ERR_INVALID;
  }
  const int64_t rank_bytes = DropRank::bytes(n_docs);
  char* scratch = nullptr;
  FPB_CUDA_CHECK(cudaMalloc(&scratch, rank_bytes + fpb_align256(n_cells * 8)));
  const DropRank r = DropRank::at(scratch, n_docs);
  int64_t* count = reinterpret_cast<int64_t*>(scratch + rank_bytes);
  const int cell_grid = fpb_grid_for(n_cells * 32, DEL_THREADS, sm_count);
  auto run = [&]() -> int {
    FPB_TRY(build_drop_rank("fpb_ivf_delete", r, d_drop, n_drop, n_docs, nullptr, nullptr, sm_count, st));
    // pass 1 counts each cell's kept postings, the scan places the lists, pass 2 writes them
    ivf_keep_kernel<<<cell_grid, DEL_THREADS, 0, st>>>(d_ivf_offsets, d_ivf_pids, n_cells, n_docs, r.bitmap, r.rank,
                                                       count, nullptr, nullptr, r.bad);
    FPB_LAUNCH_CHECK("ivf_keep");
    FPB_TRY(launch_offsets_scan(nullptr, count, n_cells, d_out_offsets, nullptr, st));
    int64_t total = 0;
    int flag = 0;
    FPB_CUDA_CHECK(cudaMemcpyAsync(&total, d_out_offsets + n_cells, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    FPB_CUDA_CHECK(cudaMemcpyAsync(&flag, r.bad, sizeof(int), cudaMemcpyDeviceToHost, st));
    FPB_CUDA_CHECK(cudaStreamSynchronize(st));
    if (flag) {
      fpb_set_error("fpb_ivf_delete: a posting lies outside [0, %lld)", (long long)n_docs);
      return FPB_ERR_INVALID;
    }
    *h_n_ivf = total;
    if (!d_out_pids) return FPB_OK;  // the offsets and the size alone
    if (total > out_capacity) {
      fpb_set_error("fpb_ivf_delete: %lld postings do not fit in %lld", (long long)total, (long long)out_capacity);
      return FPB_ERR_INVALID;
    }
    ivf_keep_kernel<<<cell_grid, DEL_THREADS, 0, st>>>(d_ivf_offsets, d_ivf_pids, n_cells, n_docs, r.bitmap, r.rank,
                                                       nullptr, d_out_offsets, d_out_pids, r.bad);
    FPB_LAUNCH_CHECK("ivf_keep");
    FPB_CUDA_CHECK(cudaStreamSynchronize(st));
    return FPB_OK;
  };
  const int rc = run();
  cudaStreamSynchronize(st);
  cudaFree(scratch);
  return rc;
}
