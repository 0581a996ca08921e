// Growing an index in place: fpb_index_append (a handle over the grown arrays, the derived tables extended for the
// new documents only) and fpb_ivf_append (the inverted file merged with the new documents' postings).
#include <string.h>

#include "kernels.h"

namespace {

constexpr int IVF_THREADS = 256;
// bytes of the per-slab document bitmap of fpb_ivf_append: [words, n_cells] u32, one bit per (cell, new document)
constexpr int64_t IVF_BITMAP_BYTES = int64_t(64) << 20;

// One warp per new document of the slab [d0, d0 + 32 * words): the bit of (code, document) of each of its tokens.
// Setting a bit twice is a no-op, so a document's repeated codes give one posting.
__global__ void __launch_bounds__(IVF_THREADS)
ivf_mark_kernel(const int64_t* __restrict__ offsets, const int32_t* __restrict__ codes, int64_t d0, int64_t d1,
                int64_t n_cells, uint32_t* __restrict__ bitmap, int* __restrict__ bad) {
  const int lane = threadIdx.x & 31;
  for (int64_t d = d0 + (int64_t(blockIdx.x) * IVF_THREADS + threadIdx.x) / 32; d < d1;
       d += int64_t(gridDim.x) * (IVF_THREADS / 32)) {
    const int64_t dl = d - d0;
    const uint32_t bit = 1u << (dl & 31);
    uint32_t* row = bitmap + (dl >> 5) * n_cells;
    for (int64_t t = offsets[d] + lane; t < offsets[d + 1]; t += 32) {
      const int32_t c = codes[t];
      if (c < 0 || c >= n_cells) {
        *bad = 1;
        continue;
      }
      atomicOr(row + c, bit);
    }
  }
}

// One thread per cell: add the slab's documents in the cell to count[c] (count != NULL), or write their ids in
// ascending order at cursor[c] and advance it.
__global__ void __launch_bounds__(IVF_THREADS)
ivf_slab_kernel(const uint32_t* __restrict__ bitmap, int words, int64_t n_cells, int64_t id0,
                int64_t* __restrict__ count, int64_t* __restrict__ cursor, int32_t* __restrict__ pids) {
  for (int64_t c = int64_t(blockIdx.x) * IVF_THREADS + threadIdx.x; c < n_cells; c += int64_t(gridDim.x) * IVF_THREADS) {
    if (count) {
      int64_t n = 0;
      for (int w = 0; w < words; ++w) n += __popc(bitmap[w * n_cells + c]);
      count[c] += n;
      continue;
    }
    int64_t at = cursor[c];
    for (int w = 0; w < words; ++w) {
      uint32_t m = bitmap[w * n_cells + c];
      while (m) {
        const int b = __ffs(m) - 1;
        m &= m - 1;
        pids[at++] = int32_t(id0 + 32 * int64_t(w) + b);
      }
    }
    cursor[c] = at;
  }
}

// The old lists in their shifted places: posting i of cell c moves by out[c] - old[c].
__global__ void __launch_bounds__(IVF_THREADS)
ivf_shift_kernel(const int64_t* __restrict__ old_offsets, const int32_t* __restrict__ old_pids, int64_t n_cells,
                 int64_t n_old, const int64_t* __restrict__ out_offsets, int32_t* __restrict__ out_pids) {
  for (int64_t i = int64_t(blockIdx.x) * IVF_THREADS + threadIdx.x; i < n_old; i += int64_t(gridDim.x) * IVF_THREADS) {
    int64_t lo = 0, hi = n_cells;  // the last cell c with old_offsets[c] <= i
    while (hi - lo > 1) {
      const int64_t mid = (lo + hi) >> 1;
      if (old_offsets[mid] <= i) lo = mid;
      else hi = mid;
    }
    out_pids[i + out_offsets[lo] - old_offsets[lo]] = old_pids[i];
  }
}

}  // namespace

extern "C" int fpb_ivf_append(int device, int64_t n_cells, const int64_t* d_ivf_offsets, const int32_t* d_ivf_pids,
                              int64_t n_old_docs, int64_t n_new_docs, const int64_t* d_new_offsets,
                              const int32_t* d_new_codes, int64_t* d_out_offsets, int32_t* d_out_pids,
                              int64_t out_capacity, int64_t* h_n_ivf, void* stream) {
  if (n_cells <= 0 || n_old_docs < 0 || n_new_docs < 0 || out_capacity < 0 || !d_ivf_offsets || !d_out_offsets ||
      !h_n_ivf || (n_new_docs > 0 && (!d_new_offsets || !d_new_codes))) {
    fpb_set_error("fpb_ivf_append: bad sizes or NULL pointers");
    return FPB_ERR_INVALID;
  }
  if (n_old_docs + n_new_docs >= (int64_t(1) << 31)) {
    fpb_set_error("fpb_ivf_append: document ids must fit in int32");
    return FPB_ERR_UNSUPPORTED;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  FPB_CUDA_CHECK(cudaSetDevice(device));
  int sm_count = 0;
  FPB_CUDA_CHECK(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, device));
  int64_t n_old = 0;
  FPB_CUDA_CHECK(cudaMemcpyAsync(&n_old, d_ivf_offsets + n_cells, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  FPB_CUDA_CHECK(cudaStreamSynchronize(st));
  if (n_old > 0 && !d_ivf_pids) {
    fpb_set_error("fpb_ivf_append: d_ivf_pids is NULL");
    return FPB_ERR_INVALID;
  }
  // slabs of 32 * words new documents, so that the bitmap stays within IVF_BITMAP_BYTES
  const int64_t words_all = (n_new_docs + 31) / 32;
  int64_t words64 = IVF_BITMAP_BYTES / 4 / n_cells;
  words64 = words64 < 1 ? 1 : (words64 > words_all ? words_all : words64);
  const int words = int(words64 < 1 ? 1 : words64);
  const int64_t slab = 32 * int64_t(words);
  char* scratch = nullptr;
  const int64_t bitmap_bytes = fpb_align256(int64_t(words) * n_cells * 4);
  const int64_t vec_bytes = fpb_align256(n_cells * 8);
  FPB_CUDA_CHECK(cudaMalloc(&scratch, bitmap_bytes + 2 * vec_bytes + 256));
  uint32_t* bitmap = reinterpret_cast<uint32_t*>(scratch);
  int64_t* count = reinterpret_cast<int64_t*>(scratch + bitmap_bytes);
  int64_t* cursor = reinterpret_cast<int64_t*>(scratch + bitmap_bytes + vec_bytes);
  int* bad = reinterpret_cast<int*>(scratch + bitmap_bytes + 2 * vec_bytes);
  const int cell_grid = fpb_grid_for(n_cells, IVF_THREADS, sm_count);
  auto run = [&]() -> int {
    FPB_CUDA_CHECK(cudaMemsetAsync(count, 0, n_cells * 8, st));
    FPB_CUDA_CHECK(cudaMemsetAsync(bad, 0, sizeof(int), st));
    // pass 1 counts each cell's new postings, pass 2 writes them; both rebuild every slab's bitmap
    for (int pass = 0; pass < 2; ++pass) {
      if (pass == 1) {
        // the new offsets, and cursor[c] = where the new ids of cell c go, after its shifted old list
        FPB_TRY(launch_offsets_scan(d_ivf_offsets, count, n_cells, d_out_offsets, cursor, st));
        int64_t total = 0;
        int flag = 0;
        FPB_CUDA_CHECK(cudaMemcpyAsync(&total, d_out_offsets + n_cells, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
        FPB_CUDA_CHECK(cudaMemcpyAsync(&flag, bad, sizeof(int), cudaMemcpyDeviceToHost, st));
        FPB_CUDA_CHECK(cudaStreamSynchronize(st));
        if (flag) {
          fpb_set_error("fpb_ivf_append: a new code lies outside [0, %lld)", (long long)n_cells);
          return FPB_ERR_INVALID;
        }
        *h_n_ivf = total;
        if (!d_out_pids) return FPB_OK;  // the offsets and the size alone
        if (total > out_capacity) {
          fpb_set_error("fpb_ivf_append: %lld postings do not fit in %lld", (long long)total, (long long)out_capacity);
          return FPB_ERR_INVALID;
        }
        if (n_old > 0) {
          ivf_shift_kernel<<<fpb_grid_for(n_old, IVF_THREADS, sm_count), IVF_THREADS, 0, st>>>(
              d_ivf_offsets, d_ivf_pids, n_cells, n_old, d_out_offsets, d_out_pids);
          FPB_LAUNCH_CHECK("ivf_shift");
        }
      }
      for (int64_t d0 = 0; d0 < n_new_docs; d0 += slab) {
        const int64_t d1 = d0 + slab < n_new_docs ? d0 + slab : n_new_docs;
        FPB_CUDA_CHECK(cudaMemsetAsync(bitmap, 0, int64_t(words) * n_cells * 4, st));
        ivf_mark_kernel<<<fpb_grid_for((d1 - d0) * 32, IVF_THREADS, sm_count), IVF_THREADS, 0, st>>>(
            d_new_offsets, d_new_codes, d0, d1, n_cells, bitmap, bad);
        FPB_LAUNCH_CHECK("ivf_mark");
        ivf_slab_kernel<<<cell_grid, IVF_THREADS, 0, st>>>(bitmap, words, n_cells, n_old_docs + d0,
                                                           pass == 0 ? count : nullptr, cursor, d_out_pids);
        FPB_LAUNCH_CHECK("ivf_slab");
      }
    }
    FPB_CUDA_CHECK(cudaStreamSynchronize(st));
    return FPB_OK;
  };
  const int rc = run();
  cudaStreamSynchronize(st);
  cudaFree(scratch);
  return rc;
}

extern "C" int fpb_index_append(fpb_index** out, const fpb_index* ix, int64_t n_docs, int64_t n_tokens,
                                const int64_t* d_doc_offsets, const int32_t* d_doc_codes,
                                const uint8_t* d_doc_residuals, void* d_token_norms, const int64_t* d_ivf_offsets,
                                const int32_t* d_ivf_pids, int64_t n_ivf, int64_t max_doc_len) {
  if (!out) {
    fpb_set_error("fpb_index_append: out is NULL");
    return FPB_ERR_INVALID;
  }
  *out = nullptr;
  if (!ix || !d_doc_offsets || !d_doc_codes || !d_doc_residuals || !d_token_norms) {
    fpb_set_error("fpb_index_append: NULL index or array pointer");
    return FPB_ERR_INVALID;
  }
  if (n_docs < ix->N || n_tokens < ix->E || n_ivf < 0 || max_doc_len < ix->max_doc_len) {
    fpb_set_error("fpb_index_append: an index of %lld documents and %lld tokens cannot shrink to %lld and %lld",
                  (long long)ix->N, (long long)ix->E, (long long)n_docs, (long long)n_tokens);
    return FPB_ERR_INVALID;
  }
  if (n_docs >= (int64_t(1) << 31)) {
    fpb_set_error("fpb_index_append: n_docs must fit in int32 per shard");
    return FPB_ERR_UNSUPPORTED;
  }
  if ((ix->ivf_offsets == nullptr) != (d_ivf_offsets == nullptr) || (d_ivf_offsets && !d_ivf_pids)) {
    fpb_set_error("fpb_index_append: the grown index must have an inverted file exactly when the old one has");
    return FPB_ERR_INVALID;
  }
  fpb_walk* w = ix->walk;
  std::lock_guard<std::mutex> lock(w->mu);
  if (w->n_docs != ix->N) {
    fpb_set_error("fpb_index_append: the index of %lld documents has already been appended to (%lld laid out)",
                  (long long)ix->N, (long long)w->n_docs);
    return FPB_ERR_INVALID;
  }
  FPB_CUDA_CHECK(cudaSetDevice(ix->device));
  int64_t ends[2];
  FPB_CUDA_CHECK(cudaMemcpy(&ends[0], d_doc_offsets + ix->N, sizeof(int64_t), cudaMemcpyDeviceToHost));
  FPB_CUDA_CHECK(cudaMemcpy(&ends[1], d_doc_offsets + n_docs, sizeof(int64_t), cudaMemcpyDeviceToHost));
  if (ends[0] != ix->E || ends[1] != n_tokens) {
    fpb_set_error("fpb_index_append: offsets[%lld] = %lld and offsets[%lld] = %lld, expected %lld and %lld",
                  (long long)ix->N, (long long)ends[0], (long long)n_docs, (long long)ends[1], (long long)ix->E,
                  (long long)n_tokens);
    return FPB_ERR_INVALID;
  }
  fpb_index* nx = new fpb_index(*ix);
  nx->N = n_docs;
  nx->E = n_tokens;
  nx->n_ivf = n_ivf;
  nx->max_doc_len = max_doc_len;
  nx->doc_offsets = d_doc_offsets;
  nx->doc_codes = d_doc_codes;
  nx->doc_residuals = d_doc_residuals;
  nx->token_norms = static_cast<const __half*>(d_token_norms);
  nx->ivf_offsets = d_ivf_offsets;
  nx->ivf_pids = d_ivf_pids;
  nx->doc_group = nullptr;  // a group map covers the old documents only
  nx->n_groups = 0;
  nx->max_per_group = 0;
  nx->global_group = nullptr;
  nx->n_total_docs = 0;
  nx->doc_bias = nullptr;  // so does a bias
  int rc = launch_token_norms(nx, static_cast<__half*>(d_token_norms), ix->E, nullptr);
  if (rc == FPB_OK) rc = fpb_extend_walk_layout(nx, ix->N);  // synchronises the device
  if (rc != FPB_OK) {
    delete nx;  // the old handle's windows are untouched: a failed append can be retried
    return rc;
  }
  w->n_docs = n_docs;
  ++w->refs;
  *out = nx;
  return FPB_OK;
}
