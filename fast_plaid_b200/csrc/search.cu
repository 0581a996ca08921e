// Whole-batch search pipeline behind the C ABI (replaces pysearch -> search_many -> search,
// rust/lib.rs:195-223, rust/search/search.rs:219-288, :471-696).  One stream, no host
// synchronisation between the stages: every intermediate size is bounded up front
// (<= Q*n_ivf_probe cells, <= N candidates, <= n_full_scores/4 re-ranked documents).
#include "kernels.h"

namespace {

int prepare(const fpb_index* ix, int B, int Q, const fpb_params* p, void* d_ws, size_t ws_bytes,
            fpb_layout* L, bool need_ivf) {
  if (!ix || !p || !d_ws) {
    fpb_set_error("search: NULL index, params or workspace");
    return FPB_ERR_INVALID;
  }
  if (need_ivf && !ix->ivf_offsets) {
    // same text as rust/search/search.rs:227-232
    fpb_set_error(
        "This index was built with compress_only=True and does not support search. "
        "Rebuild with compress_only=False to enable search.");
    return FPB_ERR_NO_IVF;
  }
  const int rc = fpb_workspace_layout(ix, B, Q, p, L);
  if (rc != FPB_OK) return rc;
  if (size_t(L->total_bytes) > ws_bytes) {
    fpb_set_error("workspace too small: need %lld bytes, have %zu", (long long)L->total_bytes, ws_bytes);
    return FPB_ERR_WORKSPACE;
  }
  if ((reinterpret_cast<uintptr_t>(d_ws) & 255u) != 0) {
    fpb_set_error("workspace must be 256-byte aligned");
    return FPB_ERR_INVALID;
  }
  FPB_CUDA_CHECK(cudaSetDevice(ix->device));
  return FPB_OK;
}

int run_until_maxsim(const fpb_index* ix, const Ws& ws, const __half* d_queries, cudaStream_t st,
                     const int32_t* d_subset_ids = nullptr, const int64_t* d_subset_offsets = nullptr,
                     int64_t max_subset_len = 0) {
  const bool subset = d_subset_ids != nullptr || d_subset_offsets != nullptr;
  FPB_TRY(launch_pad_queries(ix, ws, d_queries, st));
  FPB_TRY(launch_centroid_scores(ix, ws, st));
  if (subset) FPB_TRY(launch_subset(ix, ws, d_subset_ids, d_subset_offsets, max_subset_len, st));
  FPB_TRY(launch_probe(ix, ws, subset, st));
  FPB_TRY(launch_candidates(ix, ws, subset, st));
  FPB_TRY(launch_approx(ix, ws, ws.L->flags, st));
  FPB_TRY(launch_select(ws, st));
  FPB_TRY(launch_maxsim(ix, ws, st));
  return FPB_OK;
}

}  // namespace

extern "C" int fpb_search_batch(const fpb_index* ix, const void* d_queries, int B, int Q,
                                const fpb_params* p, void* d_ws, size_t ws_bytes, int64_t* d_out_ids,
                                float* d_out_scores, int32_t* d_out_counts, void* stream) {
  fpb_layout L;
  FPB_TRY(prepare(ix, B, Q, p, d_ws, ws_bytes, &L, true));
  if (!d_queries || !d_out_ids || !d_out_scores || !d_out_counts) {
    fpb_set_error("fpb_search_batch: NULL query or output pointer");
    return FPB_ERR_INVALID;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Ws ws{&L, static_cast<char*>(d_ws)};
  FPB_TRY(run_until_maxsim(ix, ws, static_cast<const __half*>(d_queries), st));
  FPB_TRY(launch_rank(ix, ws, p->top_k, d_out_ids, d_out_scores, d_out_counts, st));
  return FPB_OK;
}

extern "C" int fpb_search_batch_subset(const fpb_index* ix, const void* d_queries, int B, int Q,
                                       const fpb_params* p, const int32_t* d_subset_ids,
                                       const int64_t* d_subset_offsets, int64_t max_subset_len, void* d_ws,
                                       size_t ws_bytes, int64_t* d_out_ids, float* d_out_scores,
                                       int32_t* d_out_counts, void* stream) {
  fpb_layout L;
  FPB_TRY(prepare(ix, B, Q, p, d_ws, ws_bytes, &L, true));
  if (!d_queries || !d_out_ids || !d_out_scores || !d_out_counts || !d_subset_offsets) {
    fpb_set_error("fpb_search_batch_subset: NULL query, subset-offset or output pointer");
    return FPB_ERR_INVALID;
  }
  if (!(p->flags & FPB_FLAG_SUBSET)) {
    fpb_set_error("fpb_search_batch_subset: params->flags must contain FPB_FLAG_SUBSET");
    return FPB_ERR_INVALID;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Ws ws{&L, static_cast<char*>(d_ws)};
  FPB_TRY(run_until_maxsim(ix, ws, static_cast<const __half*>(d_queries), st, d_subset_ids, d_subset_offsets,
                           max_subset_len));
  FPB_TRY(launch_rank(ix, ws, p->top_k, d_out_ids, d_out_scores, d_out_counts, st));
  return FPB_OK;
}

extern "C" int fpb_search_batch_host(const fpb_index* ix, const void* h_queries, int B, int Q,
                                     const fpb_params* p, void* d_ws, size_t ws_bytes, void* d_queries_staging,
                                     int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts,
                                     int64_t* h_out_ids, float* h_out_scores, int32_t* h_out_counts,
                                     void* stream) {
  if (!ix || !p || !h_queries || !d_queries_staging || !h_out_ids || !h_out_scores || !h_out_counts) {
    fpb_set_error("fpb_search_batch_host: NULL pointer");
    return FPB_ERR_INVALID;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  FPB_CUDA_CHECK(cudaSetDevice(ix->device));
  FPB_CUDA_CHECK(cudaMemcpyAsync(d_queries_staging, h_queries, size_t(B) * Q * ix->dim * 2,
                                 cudaMemcpyHostToDevice, st));
  FPB_TRY(fpb_search_batch(ix, d_queries_staging, B, Q, p, d_ws, ws_bytes, d_out_ids, d_out_scores,
                           d_out_counts, stream));
  const size_t n = size_t(B) * p->top_k;
  FPB_CUDA_CHECK(cudaMemcpyAsync(h_out_ids, d_out_ids, n * 8, cudaMemcpyDeviceToHost, st));
  FPB_CUDA_CHECK(cudaMemcpyAsync(h_out_scores, d_out_scores, n * 4, cudaMemcpyDeviceToHost, st));
  FPB_CUDA_CHECK(cudaMemcpyAsync(h_out_counts, d_out_counts, size_t(B) * 4, cudaMemcpyDeviceToHost, st));
  FPB_CUDA_CHECK(cudaStreamSynchronize(st));
  return FPB_OK;
}

extern "C" int fpb_search_shard(const fpb_index* ix, const void* d_queries, int B, int Q,
                                const fpb_params* p, void* d_ws, size_t ws_bytes, fpb_record* d_records,
                                void* stream) {
  fpb_layout L;
  FPB_TRY(prepare(ix, B, Q, p, d_ws, ws_bytes, &L, true));
  if (!d_queries || !d_records) {
    fpb_set_error("fpb_search_shard: NULL query or record pointer");
    return FPB_ERR_INVALID;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Ws ws{&L, static_cast<char*>(d_ws)};
  FPB_TRY(run_until_maxsim(ix, ws, static_cast<const __half*>(d_queries), st));
  FPB_TRY(launch_emit_records(ix, ws, d_records, st));
  return FPB_OK;
}

extern "C" int fpb_shard_approx_keys(const fpb_index* ix, const void* d_queries, int B, int Q,
                                     const fpb_params* p, void* d_ws, size_t ws_bytes, uint64_t* d_keys,
                                     void* stream) {
  fpb_layout L;
  FPB_TRY(prepare(ix, B, Q, p, d_ws, ws_bytes, &L, true));
  if (!d_queries || !d_keys) {
    fpb_set_error("fpb_shard_approx_keys: NULL query or key pointer");
    return FPB_ERR_INVALID;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Ws ws{&L, static_cast<char*>(d_ws)};
  FPB_TRY(launch_pad_queries(ix, ws, static_cast<const __half*>(d_queries), st));
  FPB_TRY(launch_centroid_scores(ix, ws, st));
  FPB_TRY(launch_probe(ix, ws, false, st));
  FPB_TRY(launch_candidates(ix, ws, false, st));
  FPB_TRY(launch_approx(ix, ws, ws.L->flags, st));
  FPB_TRY(launch_select(ws, st));
  return launch_emit_keys(ix, ws, d_keys, st);
}

extern "C" int fpb_shard_subset_begin(const fpb_index* ix, const void* d_queries, int B, int Q, const fpb_params* p,
                                      const int32_t* d_subset_ids, const int64_t* d_subset_offsets,
                                      int64_t max_subset_len, void* d_ws, size_t ws_bytes,
                                      uint32_t* d_cbitmap_out, void* stream) {
  fpb_layout L;
  FPB_TRY(prepare(ix, B, Q, p, d_ws, ws_bytes, &L, true));
  if (!d_queries || !d_subset_offsets || !d_cbitmap_out || !(p->flags & FPB_FLAG_SUBSET)) {
    fpb_set_error("fpb_shard_subset_begin: NULL pointer or FPB_FLAG_SUBSET not set");
    return FPB_ERR_INVALID;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Ws ws{&L, static_cast<char*>(d_ws)};
  FPB_TRY(launch_pad_queries(ix, ws, static_cast<const __half*>(d_queries), st));
  FPB_TRY(launch_centroid_scores(ix, ws, st));
  FPB_TRY(launch_subset_mark(ix, ws, d_subset_ids, d_subset_offsets, max_subset_len, st));
  FPB_CUDA_CHECK(cudaMemcpyAsync(d_cbitmap_out, ws.cbitmap(), size_t(L.B) * L.cbitmap_words * 4,
                                 cudaMemcpyDeviceToDevice, st));
  return FPB_OK;
}

extern "C" int fpb_shard_subset_keys(const fpb_index* ix, int B, int Q, const fpb_params* p, void* d_ws,
                                     size_t ws_bytes, const uint32_t* d_all_cbitmaps, int n_shards,
                                     uint64_t* d_keys, void* stream) {
  fpb_layout L;
  FPB_TRY(prepare(ix, B, Q, p, d_ws, ws_bytes, &L, true));
  if (!d_all_cbitmaps || !d_keys || n_shards < 1 || !(p->flags & FPB_FLAG_SUBSET)) {
    fpb_set_error("fpb_shard_subset_keys: bad arguments or FPB_FLAG_SUBSET not set");
    return FPB_ERR_INVALID;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Ws ws{&L, static_cast<char*>(d_ws)};
  FPB_TRY(launch_subset_merge(ix, ws, d_all_cbitmaps, n_shards, st));
  FPB_TRY(launch_probe(ix, ws, true, st));
  FPB_TRY(launch_candidates(ix, ws, true, st));
  FPB_TRY(launch_approx(ix, ws, ws.L->flags, st));
  FPB_TRY(launch_select(ws, st));
  return launch_emit_keys(ix, ws, d_keys, st);
}

extern "C" int fpb_shard_apply_threshold(const fpb_index* ix, const uint64_t* d_all_keys, int n_shards,
                                         int shard_rank, int B, int Q, const fpb_params* p, void* d_ws,
                                         size_t ws_bytes, void* stream) {
  fpb_layout L;
  FPB_TRY(prepare(ix, B, Q, p, d_ws, ws_bytes, &L, false));
  if (!d_all_keys || n_shards < 1 || shard_rank < 0 || shard_rank >= n_shards) {
    fpb_set_error("fpb_shard_apply_threshold: bad arguments");
    return FPB_ERR_INVALID;
  }
  Ws ws{&L, static_cast<char*>(d_ws)};
  return launch_apply_threshold(ws, d_all_keys, n_shards, shard_rank, static_cast<cudaStream_t>(stream));
}

extern "C" int fpb_shard_exact_records(const fpb_index* ix, int B, int Q, const fpb_params* p, void* d_ws,
                                       size_t ws_bytes, fpb_record* d_records, void* stream) {
  fpb_layout L;
  FPB_TRY(prepare(ix, B, Q, p, d_ws, ws_bytes, &L, false));
  if (!d_records) {
    fpb_set_error("fpb_shard_exact_records: NULL record pointer");
    return FPB_ERR_INVALID;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Ws ws{&L, static_cast<char*>(d_ws)};
  FPB_TRY(launch_maxsim(ix, ws, st));
  return launch_emit_records(ix, ws, d_records, st);
}

// ---- stage-level entry points ----------------------------------------------------------
#define FPB_STAGE_PROLOGUE(need_ivf)                                   \
  fpb_layout L;                                                        \
  FPB_TRY(prepare(ix, B, Q, p, d_ws, ws_bytes, &L, need_ivf));         \
  cudaStream_t st = static_cast<cudaStream_t>(stream);                 \
  Ws ws{&L, static_cast<char*>(d_ws)};

extern "C" int fpb_stage_centroid_scores(const fpb_index* ix, const void* d_queries, int B, int Q,
                                         const fpb_params* p, void* d_ws, size_t ws_bytes, void* stream) {
  FPB_STAGE_PROLOGUE(false)
  if (!d_queries) {
    fpb_set_error("fpb_stage_centroid_scores: NULL queries");
    return FPB_ERR_INVALID;
  }
  FPB_TRY(launch_pad_queries(ix, ws, static_cast<const __half*>(d_queries), st));
  return launch_centroid_scores(ix, ws, st);
}
extern "C" int fpb_stage_subset(const fpb_index* ix, const int32_t* d_subset_ids, const int64_t* d_subset_offsets,
                                int64_t max_subset_len, int B, int Q, const fpb_params* p, void* d_ws,
                                size_t ws_bytes, void* stream) {
  FPB_STAGE_PROLOGUE(false)
  if (!d_subset_offsets || !(p->flags & FPB_FLAG_SUBSET)) {
    fpb_set_error("fpb_stage_subset: NULL offsets or FPB_FLAG_SUBSET not set");
    return FPB_ERR_INVALID;
  }
  return launch_subset(ix, ws, d_subset_ids, d_subset_offsets, max_subset_len, st);
}
extern "C" int fpb_stage_probe(const fpb_index* ix, int B, int Q, const fpb_params* p, void* d_ws,
                               size_t ws_bytes, void* stream) {
  FPB_STAGE_PROLOGUE(false)
  return launch_probe(ix, ws, (p->flags & FPB_FLAG_SUBSET) != 0, st);
}
extern "C" int fpb_stage_candidates(const fpb_index* ix, int B, int Q, const fpb_params* p, void* d_ws,
                                    size_t ws_bytes, void* stream) {
  FPB_STAGE_PROLOGUE(true)
  return launch_candidates(ix, ws, (p->flags & FPB_FLAG_SUBSET) != 0, st);
}
extern "C" int fpb_stage_approx(const fpb_index* ix, int B, int Q, const fpb_params* p, void* d_ws,
                                size_t ws_bytes, void* stream) {
  FPB_STAGE_PROLOGUE(false)
  return launch_approx(ix, ws, p->flags, st);
}
extern "C" int fpb_stage_select(const fpb_index* ix, int B, int Q, const fpb_params* p, void* d_ws,
                                size_t ws_bytes, void* stream) {
  FPB_STAGE_PROLOGUE(false)
  return launch_select(ws, st);
}
extern "C" int fpb_stage_maxsim(const fpb_index* ix, int B, int Q, const fpb_params* p, void* d_ws,
                                size_t ws_bytes, void* stream) {
  FPB_STAGE_PROLOGUE(false)
  return launch_maxsim(ix, ws, st);
}
extern "C" int fpb_stage_rank(const fpb_index* ix, int B, int Q, const fpb_params* p, void* d_ws,
                              size_t ws_bytes, int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts,
                              void* stream) {
  FPB_STAGE_PROLOGUE(false)
  if (!d_out_ids || !d_out_scores || !d_out_counts) {
    fpb_set_error("fpb_stage_rank: NULL output pointer");
    return FPB_ERR_INVALID;
  }
  return launch_rank(ix, ws, p->top_k, d_out_ids, d_out_scores, d_out_counts, st);
}
extern "C" int fpb_stage_records(const fpb_index* ix, int B, int Q, const fpb_params* p, void* d_ws,
                                 size_t ws_bytes, fpb_record* d_records, void* stream) {
  FPB_STAGE_PROLOGUE(false)
  if (!d_records) {
    fpb_set_error("fpb_stage_records: NULL record pointer");
    return FPB_ERR_INVALID;
  }
  return launch_emit_records(ix, ws, d_records, st);
}
extern "C" int fpb_stage_keys(const fpb_index* ix, int B, int Q, const fpb_params* p, void* d_ws, size_t ws_bytes,
                              uint64_t* d_keys, void* stream) {
  FPB_STAGE_PROLOGUE(false)
  if (!d_keys) {
    fpb_set_error("fpb_stage_keys: NULL key pointer");
    return FPB_ERR_INVALID;
  }
  return launch_emit_keys(ix, ws, d_keys, st);
}
