// K2 : candidate documents = sorted-unique union of the IVF lists of the probed cells
//      (search.rs:531-541: unique cells -> ivf lookup -> sort -> unique_consecutive).
//
// The reference concatenates the lists, radix-sorts ~300k int64 ids and compacts, per query.
// Here every probed list is OR-ed into a per-query bitmap over the local doc ids and the
// bitmap is compacted in index order, which yields the sorted-unique id list directly.
#include "kernels.h"

namespace {

// grid (Q*n_probe, B): one CTA per probe slot.  A slot whose cell already appears in an
// earlier slot of the same query is skipped (unique_dim of search.rs:531-532).
__global__ void __launch_bounds__(128)
k2_mark_kernel(const int32_t* __restrict__ cells, int slots, const int64_t* __restrict__ ivf_offsets,
               const int32_t* __restrict__ ivf_pids, uint32_t* __restrict__ bitmap, int bitmap_words) {
  const int b = blockIdx.y, s = blockIdx.x;
  const int32_t* cq = cells + int64_t(b) * slots;
  const int32_t c = cq[s];
  if (c < 0) return;
  int dup = 0;
  for (int i = threadIdx.x; i < s; i += blockDim.x) dup |= (cq[i] == c);
  if (__syncthreads_or(dup)) return;
  const int64_t o0 = ivf_offsets[c], o1 = ivf_offsets[c + 1];
  uint32_t* bm = bitmap + int64_t(b) * bitmap_words;
  for (int64_t i = o0 + threadIdx.x; i < o1; i += blockDim.x) {
    const int32_t pid = __ldg(ivf_pids + i);
    atomicOr(bm + (pid >> 5), 1u << (pid & 31));
  }
}

// A wide probe (n_probe > FPB_WARP_PROBE): grid (ceil(slots / 8), B), one warp per probe slot.  The slot that sets
// its cell's bit in the query's centroid bitmap walks the cell's IVF list; every other slot of that cell stops there.
__global__ void __launch_bounds__(256)
k2_mark_wide_kernel(const int32_t* __restrict__ cells, int slots, const int64_t* __restrict__ ivf_offsets,
                    const int32_t* __restrict__ ivf_pids, uint32_t* __restrict__ cell_bitmap, int cell_words,
                    uint32_t* __restrict__ bitmap, int bitmap_words) {
  const int b = blockIdx.y, lane = threadIdx.x & 31;
  const int s = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (s >= slots) return;
  const int32_t c = cells[int64_t(b) * slots + s];
  if (c < 0) return;
  int first = 0;
  if (lane == 0) {
    const uint32_t bit = 1u << (c & 31);
    first = (atomicOr(cell_bitmap + int64_t(b) * cell_words + (c >> 5), bit) & bit) == 0;
  }
  if (!__shfl_sync(0xffffffffu, first, 0)) return;
  const int64_t o0 = ivf_offsets[c], o1 = ivf_offsets[c + 1];
  uint32_t* bm = bitmap + int64_t(b) * bitmap_words;
  for (int64_t i = o0 + lane; i < o1; i += 32) {
    const int32_t pid = __ldg(ivf_pids + i);
    atomicOr(bm + (pid >> 5), 1u << (pid & 31));
  }
}

// one CTA per query: ordered compaction of the bitmap into cand[b][0..n_cand[b])
__global__ void __launch_bounds__(1024)
k2_compact_kernel(const uint32_t* __restrict__ bitmap, const uint32_t* __restrict__ mask, int bitmap_words,
                  int32_t* __restrict__ cand, int cand_cap, int32_t* __restrict__ n_cand) {
  __shared__ int warp_sums[32];
  __shared__ int s_base;
  const int b = blockIdx.x;
  const uint32_t* bm = bitmap + int64_t(b) * bitmap_words;
  const uint32_t* mk = mask ? mask + int64_t(b) * bitmap_words : nullptr;  // subset intersection (search.rs:544-547)
  int32_t* out = cand + int64_t(b) * cand_cap;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_base = 0;
  __syncthreads();
  for (int w0 = 0; w0 < bitmap_words; w0 += 4096) {
    const int wi = w0 + tid * 4;  // 4 consecutive words per thread keeps the output ordered
    uint32_t w[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      w[u] = (wi + u < bitmap_words) ? bm[wi + u] : 0u;
      if (mk && wi + u < bitmap_words) w[u] &= mk[wi + u];
    }
    const int c = __popc(w[0]) + __popc(w[1]) + __popc(w[2]) + __popc(w[3]);
    int incl = c;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, off);
      if (lane >= off) incl += v;
    }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int ws = warp_sums[lane];
      int wincl = ws;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, wincl, off);
        if (lane >= off) wincl += v;
      }
      warp_sums[lane] = wincl - ws;  // exclusive
    }
    __syncthreads();
    const int base = s_base;
    int pos = base + warp_sums[warp] + incl - c;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      uint32_t x = w[u];
      while (x) {
        const int bit = __ffs(x) - 1;
        x &= x - 1;
        out[pos++] = (wi + u) * 32 + bit;
      }
    }
    __syncthreads();
    if (tid == 1023) s_base = base + warp_sums[31] + incl;  // total of this round
    __syncthreads();
  }
  if (tid == 0) n_cand[b] = s_base;
}

// The subset's documents as a bitmap and the centroids occurring in them as a second bitmap
// (search.rs:496-503: lookup of the subset's codes + unique).  One warp per subset document.  cbitmap == NULL: the
// document bitmap alone.
__global__ void __launch_bounds__(256)
subset_mark_kernel(const int32_t* __restrict__ ids, const int64_t* __restrict__ offsets,
                   const int64_t* __restrict__ doc_offsets, const int32_t* __restrict__ codes, int64_t n_docs,
                   int64_t doc_id_base, uint32_t* __restrict__ sbitmap, int bitmap_words,
                   uint32_t* __restrict__ cbitmap, int cbitmap_words) {
  const int b = blockIdx.y;
  const int lane = threadIdx.x & 31;
  const int64_t i = offsets[b] + int64_t(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= offsets[b + 1]) return;
  const int64_t d = int64_t(ids[i]) - doc_id_base;
  if (d < 0 || d >= n_docs) return;  // not in this shard / invalid id: ignored
  if (lane == 0) atomicOr(sbitmap + int64_t(b) * bitmap_words + (d >> 5), 1u << (d & 31));
  if (!cbitmap) return;
  uint32_t* cb = cbitmap + int64_t(b) * cbitmap_words;
  const int64_t o0 = doc_offsets[d], o1 = doc_offsets[d + 1];
  for (int64_t t = o0 + lane; t < o1; t += 32) {
    const int c = __ldg(codes + t);
    atomicOr(cb + (c >> 5), 1u << (c & 31));
  }
}

}  // namespace

int launch_compact(const uint32_t* bitmap, const uint32_t* mask, int words, int32_t* out, int cap, int32_t* n_out,
                   int B, cudaStream_t st) {
  k2_compact_kernel<<<B, 1024, 0, st>>>(bitmap, mask, words, out, cap, n_out);
  FPB_LAUNCH_CHECK("k2_compact");
  return FPB_OK;
}

// marks the per-query document bitmap and the bitmap of centroids those documents touch (no compaction)
int launch_subset_mark(const fpb_index* ix, const Ws& ws, const int32_t* d_ids, const int64_t* d_offsets,
                       int64_t max_len, cudaStream_t st) {
  const fpb_layout& L = *ws.L;
  if (L.off_sbitmap == L.off_cbitmap) {
    fpb_set_error("subset search needs a workspace laid out with FPB_FLAG_SUBSET");
    return FPB_ERR_INVALID;
  }
  FPB_CUDA_CHECK(cudaMemsetAsync(ws.cbitmap(), 0, size_t(L.B) * L.cbitmap_words * 4, st));
  FPB_CUDA_CHECK(cudaMemsetAsync(ws.sbitmap(), 0, size_t(L.B) * L.bitmap_words * 4, st));
  if (max_len > 0) {
    dim3 grid(unsigned((max_len + 7) / 8), L.B);
    subset_mark_kernel<<<grid, 256, 0, st>>>(d_ids, d_offsets, ix->doc_offsets, ix->doc_codes, ix->N,
                                             ix->doc_id_base, ws.sbitmap(), L.bitmap_words, ws.cbitmap(),
                                             L.cbitmap_words);
    FPB_LAUNCH_CHECK("subset_mark");
  }
  return FPB_OK;
}

int launch_doc_bitmap(const fpb_index* ix, const int32_t* d_ids, const int64_t* d_offsets, int64_t max_len,
                      int n_lists, uint32_t* bitmap, int words, cudaStream_t st) {
  FPB_CUDA_CHECK(cudaMemsetAsync(bitmap, 0, size_t(n_lists) * words * 4, st));
  if (max_len > 0) {
    dim3 grid(unsigned((max_len + 7) / 8), n_lists);
    subset_mark_kernel<<<grid, 256, 0, st>>>(d_ids, d_offsets, ix->doc_offsets, ix->doc_codes, ix->N,
                                             ix->doc_id_base, bitmap, words, nullptr, 0);
    FPB_LAUNCH_CHECK("subset_mark");
  }
  return FPB_OK;
}

int launch_subset_compact(const fpb_index* ix, const Ws& ws, cudaStream_t st) {
  const fpb_layout& L = *ws.L;
  return launch_compact(ws.cbitmap(), nullptr, L.cbitmap_words, ws.clist(), int(ix->K), ws.n_clist(), L.B, st);
}

namespace {
// cbitmap[i] = OR over shards of all[s][i]   (document-sharded subset search: the centroids the
// subset documents touch are the union over the shards that hold them)
__global__ void or_bitmaps_kernel(const uint32_t* __restrict__ all, int n_shards, int64_t words,
                                  uint32_t* __restrict__ out) {
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < words; i += int64_t(gridDim.x) * blockDim.x) {
    uint32_t v = 0;
    for (int s = 0; s < n_shards; ++s) v |= all[int64_t(s) * words + i];
    out[i] = v;
  }
}
}  // namespace

int launch_subset_merge(const fpb_index* ix, const Ws& ws, const uint32_t* d_all, int n_shards, cudaStream_t st) {
  const fpb_layout& L = *ws.L;
  const int64_t words = int64_t(L.B) * L.cbitmap_words;
  const int blocks = int((words + 255) / 256 < 1184 ? (words + 255) / 256 : 1184);
  or_bitmaps_kernel<<<blocks, 256, 0, st>>>(d_all, n_shards, words, ws.cbitmap());
  FPB_LAUNCH_CHECK("or_bitmaps");
  return launch_subset_compact(ix, ws, st);
}

int launch_candidates(const fpb_index* ix, const Ws& ws, bool subset, cudaStream_t st) {
  const fpb_layout& L = *ws.L;
  FPB_CUDA_CHECK(cudaMemsetAsync(ws.bitmap(), 0, size_t(L.B) * L.bitmap_words * 4, st));
  const int slots = L.Q * L.n_probe;
  if (L.n_probe > FPB_WARP_PROBE) {
    FPB_CUDA_CHECK(cudaMemsetAsync(ws.probe_bitmap(), 0, fpb_probe_bitmap_bytes(L), st));
    dim3 grid((slots + 7) / 8, L.B);
    k2_mark_wide_kernel<<<grid, 256, 0, st>>>(ws.cells(), slots, ix->ivf_offsets, ix->ivf_pids, ws.probe_bitmap(),
                                              L.cbitmap_words, ws.bitmap(), L.bitmap_words);
    FPB_LAUNCH_CHECK("k2_mark_wide");
  } else {
    dim3 grid(slots, L.B);
    k2_mark_kernel<<<grid, 128, 0, st>>>(ws.cells(), slots, ix->ivf_offsets, ix->ivf_pids, ws.bitmap(),
                                         L.bitmap_words);
    FPB_LAUNCH_CHECK("k2_mark");
  }
  return launch_compact(ws.bitmap(), subset ? ws.sbitmap() : nullptr, L.bitmap_words, ws.cand(), L.cand_cap,
                        ws.n_cand(), L.B, st);
}

int launch_subset(const fpb_index* ix, const Ws& ws, const int32_t* d_ids, const int64_t* d_offsets,
                  int64_t max_len, cudaStream_t st) {
  const int rc = launch_subset_mark(ix, ws, d_ids, d_offsets, max_len, st);
  return rc != FPB_OK ? rc : launch_subset_compact(ix, ws, st);
}
