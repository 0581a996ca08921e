// Whole-batch search pipeline behind the C ABI (replaces pysearch -> search_many -> search,
// rust/lib.rs:195-223, rust/search/search.rs:219-288, :471-696).  One stream, no host
// synchronisation between the stages: every intermediate size is bounded up front
// (<= Q*n_ivf_probe cells, <= N candidates, <= n_full_scores/4 re-ranked documents).
#include "entry.h"

namespace {

int run_until_maxsim(const fpb_index* ix, const Call& c, const void* d_queries,
                     const int32_t* d_subset_ids = nullptr, const int64_t* d_subset_offsets = nullptr,
                     int64_t max_subset_len = 0) {
  const bool subset = d_subset_ids != nullptr || d_subset_offsets != nullptr;
  FPB_TRY(run_centroid_scores(ix, c.ws, d_queries, c.st));
  if (subset) FPB_TRY(launch_subset(ix, c.ws, d_subset_ids, d_subset_offsets, max_subset_len, c.st));
  FPB_TRY(run_probe_to_select(ix, c.ws, subset, c.st));
  return launch_maxsim(ix, c.ws, c.st);
}

// fpb_search_batch and fpb_search_batch_subset (without a subset when both subset arrays are NULL)
int search_batch(const fpb_index* ix, const void* d_queries, int B, int Q, const fpb_params* p,
                 const int32_t* d_subset_ids, const int64_t* d_subset_offsets, int64_t max_subset_len, void* d_ws,
                 size_t ws_bytes, int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts, void* stream) {
  Call c;
  FPB_TRY(c.begin(ix, B, Q, p, d_ws, ws_bytes, true, stream));
  FPB_TRY(run_until_maxsim(ix, c, d_queries, d_subset_ids, d_subset_offsets, max_subset_len));
  return launch_rank(ix, c.ws, p->top_k, d_out_ids, d_out_scores, d_out_counts, c.st);
}

}  // namespace

extern "C" int fpb_search_batch(const fpb_index* ix, const void* d_queries, int B, int Q,
                                const fpb_params* p, void* d_ws, size_t ws_bytes, int64_t* d_out_ids,
                                float* d_out_scores, int32_t* d_out_counts, void* stream) {
  if (!d_queries || !d_out_ids || !d_out_scores || !d_out_counts) {
    fpb_set_error("fpb_search_batch: NULL query or output pointer");
    return FPB_ERR_INVALID;
  }
  return search_batch(ix, d_queries, B, Q, p, nullptr, nullptr, 0, d_ws, ws_bytes, d_out_ids, d_out_scores,
                      d_out_counts, stream);
}

extern "C" int fpb_search_batch_subset(const fpb_index* ix, const void* d_queries, int B, int Q,
                                       const fpb_params* p, const int32_t* d_subset_ids,
                                       const int64_t* d_subset_offsets, int64_t max_subset_len, void* d_ws,
                                       size_t ws_bytes, int64_t* d_out_ids, float* d_out_scores,
                                       int32_t* d_out_counts, void* stream) {
  if (!d_queries || !d_out_ids || !d_out_scores || !d_out_counts || !d_subset_offsets) {
    fpb_set_error("fpb_search_batch_subset: NULL query, subset-offset or output pointer");
    return FPB_ERR_INVALID;
  }
  if (p && !(p->flags & FPB_FLAG_SUBSET)) {
    fpb_set_error("fpb_search_batch_subset: params->flags must contain FPB_FLAG_SUBSET");
    return FPB_ERR_INVALID;
  }
  return search_batch(ix, d_queries, B, Q, p, d_subset_ids, d_subset_offsets, max_subset_len, d_ws, ws_bytes,
                      d_out_ids, d_out_scores, d_out_counts, stream);
}

extern "C" int fpb_search_batch_host(const fpb_index* ix, const void* h_queries, int B, int Q,
                                     const fpb_params* p, void* d_ws, size_t ws_bytes, void* d_queries_staging,
                                     int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts,
                                     int64_t* h_out_ids, float* h_out_scores, int32_t* h_out_counts,
                                     void* stream) {
  return search_via_host("fpb_search_batch_host", ix, h_queries, B, Q, p, d_queries_staging, d_out_ids, d_out_scores,
                         d_out_counts, h_out_ids, h_out_scores, h_out_counts, stream, [&] {
                           return fpb_search_batch(ix, d_queries_staging, B, Q, p, d_ws, ws_bytes, d_out_ids,
                                                   d_out_scores, d_out_counts, stream);
                         });
}

extern "C" int fpb_search_shard(const fpb_index* ix, const void* d_queries, int B, int Q,
                                const fpb_params* p, void* d_ws, size_t ws_bytes, fpb_record* d_records,
                                void* stream) {
  if (!d_queries || !d_records) {
    fpb_set_error("fpb_search_shard: NULL query or record pointer");
    return FPB_ERR_INVALID;
  }
  Call c;
  FPB_TRY(c.begin(ix, B, Q, p, d_ws, ws_bytes, true, stream));
  FPB_TRY(run_until_maxsim(ix, c, d_queries));
  return launch_emit_records(ix, c.ws, d_records, c.st);
}

extern "C" int fpb_shard_approx_keys(const fpb_index* ix, const void* d_queries, int B, int Q,
                                     const fpb_params* p, void* d_ws, size_t ws_bytes, uint64_t* d_keys,
                                     void* stream) {
  if (!d_queries || !d_keys) {
    fpb_set_error("fpb_shard_approx_keys: NULL query or key pointer");
    return FPB_ERR_INVALID;
  }
  Call c;
  FPB_TRY(c.begin(ix, B, Q, p, d_ws, ws_bytes, true, stream));
  FPB_TRY(run_centroid_scores(ix, c.ws, d_queries, c.st));
  FPB_TRY(run_probe_to_select(ix, c.ws, false, c.st));
  return launch_emit_keys(ix, c.ws, d_keys, c.st);
}

extern "C" int fpb_shard_subset_begin(const fpb_index* ix, const void* d_queries, int B, int Q, const fpb_params* p,
                                      const int32_t* d_subset_ids, const int64_t* d_subset_offsets,
                                      int64_t max_subset_len, void* d_ws, size_t ws_bytes,
                                      uint32_t* d_cbitmap_out, void* stream) {
  if (!d_queries || !d_subset_offsets || !d_cbitmap_out || (p && !(p->flags & FPB_FLAG_SUBSET))) {
    fpb_set_error("fpb_shard_subset_begin: NULL pointer or FPB_FLAG_SUBSET not set");
    return FPB_ERR_INVALID;
  }
  Call c;
  FPB_TRY(c.begin(ix, B, Q, p, d_ws, ws_bytes, true, stream));
  FPB_TRY(run_centroid_scores(ix, c.ws, d_queries, c.st));
  FPB_TRY(launch_subset_mark(ix, c.ws, d_subset_ids, d_subset_offsets, max_subset_len, c.st));
  FPB_CUDA_CHECK(cudaMemcpyAsync(d_cbitmap_out, c.ws.cbitmap(), size_t(c.L.B) * c.L.cbitmap_words * 4,
                                 cudaMemcpyDeviceToDevice, c.st));
  return FPB_OK;
}

extern "C" int fpb_shard_subset_keys(const fpb_index* ix, int B, int Q, const fpb_params* p, void* d_ws,
                                     size_t ws_bytes, const uint32_t* d_all_cbitmaps, int n_shards,
                                     uint64_t* d_keys, void* stream) {
  if (!d_all_cbitmaps || !d_keys || n_shards < 1 || (p && !(p->flags & FPB_FLAG_SUBSET))) {
    fpb_set_error("fpb_shard_subset_keys: bad arguments or FPB_FLAG_SUBSET not set");
    return FPB_ERR_INVALID;
  }
  Call c;
  FPB_TRY(c.begin(ix, B, Q, p, d_ws, ws_bytes, true, stream));
  FPB_TRY(launch_subset_merge(ix, c.ws, d_all_cbitmaps, n_shards, c.st));
  FPB_TRY(run_probe_to_select(ix, c.ws, true, c.st));
  return launch_emit_keys(ix, c.ws, d_keys, c.st);
}

extern "C" int fpb_shard_apply_threshold(const fpb_index* ix, const uint64_t* d_all_keys, int n_shards,
                                         int shard_rank, int B, int Q, const fpb_params* p, void* d_ws,
                                         size_t ws_bytes, void* stream) {
  if (!d_all_keys || n_shards < 1 || shard_rank < 0 || shard_rank >= n_shards) {
    fpb_set_error("fpb_shard_apply_threshold: bad arguments");
    return FPB_ERR_INVALID;
  }
  Call c;
  FPB_TRY(c.begin(ix, B, Q, p, d_ws, ws_bytes, false, stream));
  return launch_apply_threshold(c.ws, d_all_keys, n_shards, shard_rank, c.st);
}

extern "C" int fpb_shard_exact_records(const fpb_index* ix, int B, int Q, const fpb_params* p, void* d_ws,
                                       size_t ws_bytes, fpb_record* d_records, void* stream) {
  if (!d_records) {
    fpb_set_error("fpb_shard_exact_records: NULL record pointer");
    return FPB_ERR_INVALID;
  }
  Call c;
  FPB_TRY(c.begin(ix, B, Q, p, d_ws, ws_bytes, false, stream));
  FPB_TRY(launch_maxsim(ix, c.ws, c.st));
  return launch_emit_records(ix, c.ws, d_records, c.st);
}

// ---- stage-level entry points ----------------------------------------------------------
extern "C" int fpb_stage_centroid_scores(const fpb_index* ix, const void* d_queries, int B, int Q,
                                         const fpb_params* p, void* d_ws, size_t ws_bytes, void* stream) {
  if (!d_queries) {
    fpb_set_error("fpb_stage_centroid_scores: NULL queries");
    return FPB_ERR_INVALID;
  }
  Call c;
  FPB_TRY(c.begin(ix, B, Q, p, d_ws, ws_bytes, false, stream));
  return run_centroid_scores(ix, c.ws, d_queries, c.st);
}
extern "C" int fpb_stage_subset(const fpb_index* ix, const int32_t* d_subset_ids, const int64_t* d_subset_offsets,
                                int64_t max_subset_len, int B, int Q, const fpb_params* p, void* d_ws,
                                size_t ws_bytes, void* stream) {
  if (!d_subset_offsets || (p && !(p->flags & FPB_FLAG_SUBSET))) {
    fpb_set_error("fpb_stage_subset: NULL offsets or FPB_FLAG_SUBSET not set");
    return FPB_ERR_INVALID;
  }
  Call c;
  FPB_TRY(c.begin(ix, B, Q, p, d_ws, ws_bytes, false, stream));
  return launch_subset(ix, c.ws, d_subset_ids, d_subset_offsets, max_subset_len, c.st);
}
extern "C" int fpb_stage_probe(const fpb_index* ix, int B, int Q, const fpb_params* p, void* d_ws,
                               size_t ws_bytes, void* stream) {
  Call c;
  FPB_TRY(c.begin(ix, B, Q, p, d_ws, ws_bytes, false, stream));
  return launch_probe(ix, c.ws, (p->flags & FPB_FLAG_SUBSET) != 0, c.st);
}
extern "C" int fpb_stage_candidates(const fpb_index* ix, int B, int Q, const fpb_params* p, void* d_ws,
                                    size_t ws_bytes, void* stream) {
  Call c;
  FPB_TRY(c.begin(ix, B, Q, p, d_ws, ws_bytes, true, stream));
  return launch_candidates(ix, c.ws, (p->flags & FPB_FLAG_SUBSET) != 0, c.st);
}
extern "C" int fpb_stage_approx(const fpb_index* ix, int B, int Q, const fpb_params* p, void* d_ws,
                                size_t ws_bytes, void* stream) {
  Call c;
  FPB_TRY(c.begin(ix, B, Q, p, d_ws, ws_bytes, false, stream));
  return launch_approx(ix, c.ws, p->flags, c.st);
}
extern "C" int fpb_stage_select(const fpb_index* ix, int B, int Q, const fpb_params* p, void* d_ws,
                                size_t ws_bytes, void* stream) {
  Call c;
  FPB_TRY(c.begin(ix, B, Q, p, d_ws, ws_bytes, false, stream));
  return launch_select(c.ws, c.st);
}
extern "C" int fpb_stage_maxsim(const fpb_index* ix, int B, int Q, const fpb_params* p, void* d_ws,
                                size_t ws_bytes, void* stream) {
  Call c;
  FPB_TRY(c.begin(ix, B, Q, p, d_ws, ws_bytes, false, stream));
  return launch_maxsim(ix, c.ws, c.st);
}
extern "C" int fpb_stage_rank(const fpb_index* ix, int B, int Q, const fpb_params* p, void* d_ws,
                              size_t ws_bytes, int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts,
                              void* stream) {
  if (!d_out_ids || !d_out_scores || !d_out_counts) {
    fpb_set_error("fpb_stage_rank: NULL output pointer");
    return FPB_ERR_INVALID;
  }
  Call c;
  FPB_TRY(c.begin(ix, B, Q, p, d_ws, ws_bytes, false, stream));
  return launch_rank(ix, c.ws, p->top_k, d_out_ids, d_out_scores, d_out_counts, c.st);
}
extern "C" int fpb_stage_records(const fpb_index* ix, int B, int Q, const fpb_params* p, void* d_ws,
                                 size_t ws_bytes, fpb_record* d_records, void* stream) {
  if (!d_records) {
    fpb_set_error("fpb_stage_records: NULL record pointer");
    return FPB_ERR_INVALID;
  }
  Call c;
  FPB_TRY(c.begin(ix, B, Q, p, d_ws, ws_bytes, false, stream));
  return launch_emit_records(ix, c.ws, d_records, c.st);
}
extern "C" int fpb_stage_keys(const fpb_index* ix, int B, int Q, const fpb_params* p, void* d_ws, size_t ws_bytes,
                              uint64_t* d_keys, void* stream) {
  if (!d_keys) {
    fpb_set_error("fpb_stage_keys: NULL key pointer");
    return FPB_ERR_INVALID;
  }
  Call c;
  FPB_TRY(c.begin(ix, B, Q, p, d_ws, ws_bytes, false, stream));
  return launch_emit_keys(ix, c.ws, d_keys, c.st);
}
