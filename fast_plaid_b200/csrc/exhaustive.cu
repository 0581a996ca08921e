// Exhaustive exact search behind the C ABI: K7 scores every document of the index against every query, then
// the approximate pipeline's own selection (k3b_select, with every document a candidate) and ranking (k6_rank)
// turn the [B, N] score array into the top_k.  Works on every index, including compress_only ones (no IVF is read).
#include <algorithm>
#include <vector>

#include "kernels.h"

int check_exhaustive_shapes(int B, int Q, int top_k) {
  if (B <= 0 || Q <= 0 || top_k < 0) {
    fpb_set_error("exhaustive search: B=%d Q=%d top_k=%d must be positive", B, Q, top_k);
    return FPB_ERR_INVALID;
  }
  if (Q > 256) {
    fpb_set_error("queries with more than 256 tokens are not supported (Q=%d)", Q);
    return FPB_ERR_UNSUPPORTED;
  }
  if (top_k > FPB_EX_MAX_TOP_K) {
    fpb_set_error("exhaustive search: top_k=%d exceeds the supported maximum of %d", top_k, FPB_EX_MAX_TOP_K);
    return FPB_ERR_UNSUPPORTED;
  }
  return FPB_OK;
}

namespace {

// n_lists = 0: the full scan.  n_lists > 0: a list walk over lists of at most max_list_len ids.
int exhaustive_layout(const fpb_index* ix, int B, int Q, int top_k, ExLayout* X, int n_lists = 0,
                      int64_t max_list_len = 0) {
  // the shape limits first: they do not depend on the index
  FPB_TRY(check_exhaustive_shapes(B, Q, top_k));
  if (!ix) {
    fpb_set_error("exhaustive search: NULL index");
    return FPB_ERR_INVALID;
  }
  const bool lists = n_lists > 0;
  const int64_t N = ix->N;
  const int64_t cap = lists ? std::max<int64_t>(1, std::min(N, max_list_len)) : (N > 0 ? N : 1);
  if (lists && int64_t(std::min(B, n_lists)) * cap > INT32_MAX) {  // the chunk counter is 32-bit
    fpb_set_error("exhaustive subset search: %d lists of up to %lld documents in one call; split the batch",
                  std::min(B, n_lists), (long long)cap);
    return FPB_ERR_UNSUPPORTED;
  }
  *X = ExLayout{};
  X->B = B;
  X->Q = Q;
  X->Qs = (Q + 15) / 16 * 16;
  X->n_rows = int((int64_t(B) * X->Qs + (lists ? 48 * int64_t(n_lists) : 0) + 127) / 128 * 128);
  X->top_k = top_k;
  X->grid = ix->sm_count;
  int64_t off = 0;
  auto take = [&](int64_t bytes) {
    const int64_t o = off;
    off += fpb_align256(bytes);
    return o;
  };
  X->off_rows = take(int64_t(X->n_rows) * ix->dim * 2);
  X->off_acc = take(int64_t(B) * (lists ? cap : N) * 8);
  X->off_carry = take(int64_t(X->grid) * X->n_rows * 4);
  X->off_counter = take(4);
  const bool sel = top_k > 0;
  X->off_scores = take(sel ? int64_t(B) * cap * 4 : 0);
  X->off_n_rerank = take(sel ? int64_t(B) * 4 : 0);
  X->off_rerank = take(sel ? int64_t(B) * top_k * 4 : 0);
  X->off_rerank_approx = take(sel ? int64_t(B) * top_k * 4 : 0);
  if (lists) {
    X->n_lists = n_lists;
    X->words = int((N + 31) / 32);
    X->cap = cap;
    X->off_bitmap = take(int64_t(n_lists) * X->words * 4);
    X->off_lists = take(int64_t(n_lists) * cap * 4);
    X->off_lcount = take(int64_t(n_lists) * 4);
    X->off_chunks = take((int64_t(n_lists) + 1) * 4);
    X->off_table = take(ExListTable::ints(n_lists, B, X->n_rows) * 4);
    X->off_cand = take(int64_t(B) * cap * 4);
    X->off_n_cand = take(int64_t(B) * 4);
  }
  if (sel && ix->doc_group) {
    const int64_t cols = lists ? cap : N;  // accumulator entries per query
    const int64_t keys = int64_t(ix->max_per_group) * ix->n_groups;  // m rounds of n_groups keys per query
    X->off_gkeys = keys <= cols ? X->off_acc : take(int64_t(B) * keys * 8);
  }
  if (sel && ix->global_group) X->off_sel_ids = take(int64_t(B) * top_k * 8);
  X->total_bytes = off;
  return FPB_OK;
}

// the list arguments that do not need h_query_list (n_lists >= 1: a list walk is never the full scan)
int check_lists(int n_lists, int64_t max_list_len) {
  if (n_lists < 1 || max_list_len < 0) {
    fpb_set_error("exhaustive subset search: n_lists=%d must be >= 1 and max_list_len=%lld >= 0", n_lists,
                  (long long)max_list_len);
    return FPB_ERR_INVALID;
  }
  if (n_lists > 65535) {  // one grid row of the marking kernel per list
    fpb_set_error("exhaustive subset search: n_lists=%d exceeds the supported maximum of 65535", n_lists);
    return FPB_ERR_UNSUPPORTED;
  }
  return FPB_OK;
}

int check_workspace(const ExLayout& X, void* d_ws, size_t ws_bytes) {
  if (!d_ws) {
    fpb_set_error("exhaustive search: NULL workspace");
    return FPB_ERR_INVALID;
  }
  if (size_t(X.total_bytes) > ws_bytes) {
    fpb_set_error("workspace too small: need %lld bytes, have %zu", (long long)X.total_bytes, ws_bytes);
    return FPB_ERR_WORKSPACE;
  }
  if ((reinterpret_cast<uintptr_t>(d_ws) & 255u) != 0) {
    fpb_set_error("workspace must be 256-byte aligned");
    return FPB_ERR_INVALID;
  }
  return FPB_OK;
}

}  // namespace

extern "C" int fpb_exhaustive_workspace_bytes(const fpb_index* ix, int B, int Q, int top_k, size_t* out) {
  if (!out) {
    fpb_set_error("fpb_exhaustive_workspace_bytes: NULL output pointer");
    return FPB_ERR_INVALID;
  }
  ExLayout X;  // top_k = 0: the workspace of fpb_exhaustive_scores alone
  FPB_TRY(exhaustive_layout(ix, B, Q, top_k, &X));
  *out = size_t(X.total_bytes);
  return FPB_OK;
}

extern "C" int fpb_exhaustive_scores(const fpb_index* ix, const void* d_queries, int B, int Q, void* d_ws,
                                     size_t ws_bytes, float* d_scores, void* stream) {
  FPB_TRY(fpb_refuse_shard_groups("fpb_exhaustive_scores", ix));
  ExLayout X;
  FPB_TRY(exhaustive_layout(ix, B, Q, 0, &X));
  FPB_TRY(check_workspace(X, d_ws, ws_bytes));
  if (!d_queries || !d_scores) {
    fpb_set_error("fpb_exhaustive_scores: NULL query or score pointer");
    return FPB_ERR_INVALID;
  }
  if ((reinterpret_cast<uintptr_t>(d_queries) & 15u) != 0) {
    fpb_set_error("fpb_exhaustive_scores: queries must be 16-byte aligned");
    return FPB_ERR_INVALID;
  }
  FPB_CUDA_CHECK(cudaSetDevice(ix->device));
  return launch_exhaustive_scores(ix, X, static_cast<char*>(d_ws), static_cast<const __half*>(d_queries), d_scores,
                                  static_cast<cudaStream_t>(stream));
}

namespace {

// The selected lists of a full scan, in the workspace: per query the n_sel[b] best local documents (ids, scores)
// by (score desc, id asc), rows of stride top_k.  On a handle with groups nothing is selected: all_scores holds the
// [B, N] scores and gkeys the group keys' room (and, on a shard-grouped handle, out_ids the room of global ids).
struct ExSelected {
  int32_t* n_sel;
  int32_t* ids;
  float* scores;
  float* all_scores;
  uint64_t* gkeys;
  int64_t* out_ids;
};

// The grouped ranking of exact search: m rounds of the group maximum over the [B, cols] scores (the m best keys of
// every group), then the top_k largest of these m * n_groups keys
int rank_groups(const fpb_index* ix, const float* scores, const int32_t* cand, const int32_t* n, int64_t cols, int B,
                int top_k, uint64_t* gkeys, int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts,
                cudaStream_t st) {
  FPB_TRY(launch_group_max(scores, cand, n, cols, B, ix->doc_group, ix->n_groups, ix->max_per_group, gkeys,
                           ix->sm_count, st));
  return launch_group_select(gkeys, int64_t(ix->max_per_group) * ix->n_groups, B, top_k, ix->doc_id_base, d_out_ids,
                             d_out_scores, d_out_counts, st);
}

// The checks and the whole computation of a full-scan search up to its selected lists: K7 scores every document,
// k3b_select keeps the top_k of each query with every document a candidate.
int exhaustive_select(const char* who, const fpb_index* ix, const void* d_queries, int B, int Q, int top_k,
                      void* d_ws, size_t ws_bytes, bool outputs_ok, cudaStream_t st, ExSelected* out) {
  if (top_k < 1) {
    fpb_set_error("%s: top_k=%d must be >= 1", who, top_k);
    return FPB_ERR_INVALID;
  }
  ExLayout X;
  FPB_TRY(exhaustive_layout(ix, B, Q, top_k, &X));
  FPB_TRY(check_workspace(X, d_ws, ws_bytes));
  if (!d_queries || !outputs_ok) {
    fpb_set_error("%s: NULL query or output pointer", who);
    return FPB_ERR_INVALID;
  }
  if ((reinterpret_cast<uintptr_t>(d_queries) & 15u) != 0) {
    fpb_set_error("%s: queries must be 16-byte aligned", who);
    return FPB_ERR_INVALID;
  }
  FPB_CUDA_CHECK(cudaSetDevice(ix->device));
  char* base = static_cast<char*>(d_ws);
  float* scores = reinterpret_cast<float*>(base + X.off_scores);
  out->n_sel = reinterpret_cast<int32_t*>(base + X.off_n_rerank);
  out->ids = reinterpret_cast<int32_t*>(base + X.off_rerank);
  out->scores = reinterpret_cast<float*>(base + X.off_rerank_approx);
  out->all_scores = scores;
  out->gkeys = reinterpret_cast<uint64_t*>(base + X.off_gkeys);
  out->out_ids = reinterpret_cast<int64_t*>(base + X.off_sel_ids);
  FPB_TRY(launch_exhaustive_scores(ix, X, base, static_cast<const __half*>(d_queries), scores, st));
  if (ix->doc_group) return FPB_OK;
  // every document is a candidate, and its "approximate" score is its exact one: the selected list holds the exact
  // scores that k6_rank orders
  return launch_select(scores, nullptr, nullptr, int(ix->N), B, top_k, out->ids, out->scores, out->n_sel, st);
}

}  // namespace

extern "C" int fpb_search_exhaustive(const fpb_index* ix, const void* d_queries, int B, int Q, int top_k, void* d_ws,
                                     size_t ws_bytes, int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts,
                                     void* stream) {
  FPB_TRY(fpb_refuse_shard_groups("fpb_search_exhaustive", ix));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ExSelected sel;
  FPB_TRY(exhaustive_select("fpb_search_exhaustive", ix, d_queries, B, Q, top_k, d_ws, ws_bytes,
                            d_out_ids && d_out_scores && d_out_counts, st, &sel));
  if (ix->doc_group)
    return rank_groups(ix, sel.all_scores, nullptr, nullptr, ix->N, B, top_k, sel.gkeys, d_out_ids, d_out_scores,
                       d_out_counts, st);
  return launch_rank(sel.scores, sel.ids, sel.n_sel, top_k, B, top_k, ix->doc_id_base, d_out_ids, d_out_scores,
                     d_out_counts, st);
}

extern "C" int fpb_stage_group_rank(const fpb_index* ix, const float* d_scores, const int32_t* d_cand,
                                    const int32_t* d_n, int64_t cols, int B, int top_k, void* d_gkeys,
                                    size_t gkeys_bytes, int64_t* d_out_ids, float* d_out_scores,
                                    int32_t* d_out_counts, void* stream) {
  const char* who = "fpb_stage_group_rank";
  if (!ix || !ix->doc_group) {
    fpb_set_error("%s: needs an index handle with groups (fpb_index_with_groups_max)", who);
    return FPB_ERR_INVALID;
  }
  FPB_TRY(fpb_refuse_shard_groups(who, ix));
  if (!d_scores || !d_gkeys || !d_out_ids || !d_out_scores || !d_out_counts) {
    fpb_set_error("%s: NULL score, key or output pointer", who);
    return FPB_ERR_INVALID;
  }
  if (B < 1 || cols < 1) {
    fpb_set_error("%s: B=%d and cols=%lld must be >= 1", who, B, (long long)cols);
    return FPB_ERR_INVALID;
  }
  if (top_k < 1 || top_k > FPB_EX_MAX_TOP_K) {
    fpb_set_error("%s: top_k=%d must be in [1, %d]", who, top_k, FPB_EX_MAX_TOP_K);
    return FPB_ERR_INVALID;
  }
  const uint64_t row_keys = uint64_t(ix->max_per_group) * uint64_t(ix->n_groups);  // < 2^37: no overflow below
  if (gkeys_bytes / 8 / uint64_t(B) < row_keys) {
    fpb_set_error("%s: key scratch too small: need %d * %llu * 8 bytes, have %zu", who, B,
                  (unsigned long long)row_keys, gkeys_bytes);
    return FPB_ERR_WORKSPACE;
  }
  FPB_CUDA_CHECK(cudaSetDevice(ix->device));
  return rank_groups(ix, d_scores, d_cand, d_n, cols, B, top_k, static_cast<uint64_t*>(d_gkeys), d_out_ids,
                     d_out_scores, d_out_counts, static_cast<cudaStream_t>(stream));
}

extern "C" int fpb_shard_exhaustive_records(const fpb_index* ix, const void* d_queries, int B, int Q, int top_k,
                                            void* d_ws, size_t ws_bytes, fpb_record* d_records, void* stream) {
  FPB_TRY(fpb_refuse_unsharded_groups("fpb_shard_exhaustive_records", ix));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ExSelected sel;
  FPB_TRY(exhaustive_select("fpb_shard_exhaustive_records", ix, d_queries, B, Q, top_k, d_ws, ws_bytes,
                            d_records != nullptr, st, &sel));
  if (ix->doc_group) {
    // this shard's top_k under the rule (its local group map), then one record per result: a tail (-inf, -1) is
    // a padding record
    FPB_TRY(rank_groups(ix, sel.all_scores, nullptr, nullptr, ix->N, B, top_k, sel.gkeys, sel.out_ids, sel.scores,
                        sel.n_sel, st));
    return launch_results_to_records(sel.out_ids, sel.scores, B, top_k, d_records, st);
  }
  // approx = exact = the score: the merge's "R best by approx" is then the global top_k, ordered by the same score
  return launch_emit_records(sel.scores, sel.scores, sel.ids, sel.n_sel, B, top_k, ix->doc_id_base, d_records, st);
}

extern "C" int fpb_exhaustive_subset_workspace_bytes(const fpb_index* ix, int B, int Q, int top_k, int n_lists,
                                                     int64_t max_list_len, size_t* out) {
  if (!out) {
    fpb_set_error("fpb_exhaustive_subset_workspace_bytes: NULL output pointer");
    return FPB_ERR_INVALID;
  }
  if (top_k < 1) {
    fpb_set_error("fpb_exhaustive_subset_workspace_bytes: top_k=%d must be >= 1", top_k);
    return FPB_ERR_INVALID;
  }
  FPB_TRY(check_exhaustive_shapes(B, Q, top_k));
  FPB_TRY(check_lists(n_lists, max_list_len));
  ExLayout X;
  FPB_TRY(exhaustive_layout(ix, B, Q, top_k, &X, n_lists, max_list_len));
  *out = size_t(X.total_bytes);
  return FPB_OK;
}

namespace {

// The list walk of fpb_search_exhaustive_subset and fpb_search_exhaustive_filter once their shapes and lists are
// checked: the index and workspace checks, then the pointers (lists_ok: the list pointers are usable), the host
// table, K7 over the lists, selection and ranking.
int exhaustive_list_search(const char* who, const fpb_index* ix, const void* d_queries, int B, int Q, int top_k,
                           const ExLists& lists, bool lists_ok, int n_lists, int64_t max_list_len,
                           const int32_t* h_query_list,
                           void* d_ws, size_t ws_bytes, int64_t* d_out_ids, float* d_out_scores,
                           int32_t* d_out_counts, void* stream) {
  FPB_TRY(fpb_refuse_shard_groups(who, ix));
  ExLayout X;
  FPB_TRY(exhaustive_layout(ix, B, Q, top_k, &X, n_lists, max_list_len));
  FPB_TRY(check_workspace(X, d_ws, ws_bytes));
  if (!d_queries || !lists_ok || !d_out_ids || !d_out_scores || !d_out_counts) {
    fpb_set_error("%s: NULL query, list or output pointer", who);
    return FPB_ERR_INVALID;
  }
  if ((reinterpret_cast<uintptr_t>(d_queries) & 15u) != 0) {
    fpb_set_error("%s: queries must be 16-byte aligned", who);
    return FPB_ERR_INVALID;
  }

  // the table of the list walk: list l's queries own consecutive rows from a 64-row boundary, in query order
  std::vector<int32_t> table(size_t(ExListTable::ints(n_lists, B, X.n_rows)));
  const ExListTable t = ExListTable::at(table.data(), n_lists, B, X.n_rows);
  std::fill(t.grp_query, t.grp_query + X.n_rows / 16, -1);
  std::vector<int32_t> n_queries(size_t(n_lists), 0);
  for (int b = 0; b < B; ++b) ++n_queries[h_query_list[b]];
  int row = 0, active = 0;
  for (int l = 0; l < n_lists; ++l) {
    t.row0[l] = row;
    t.row1[l] = row + n_queries[l] * X.Qs;
    if (n_queries[l] > 0) {
      row = (t.row1[l] + 63) / 64 * 64;
      ++active;
    }
  }
  std::vector<int32_t> next(t.row0, t.row0 + n_lists);
  for (int b = 0; b < B; ++b) {
    const int l = h_query_list[b];
    t.qlist[b] = l;
    for (int r = next[l]; r < next[l] + X.Qs; r += 16) {
      t.grp_query[r / 16] = b;
      t.grp_tok[r / 16] = r - next[l];
    }
    next[l] += X.Qs;
  }
  X.list_docs = int64_t(active) * X.cap;

  FPB_CUDA_CHECK(cudaSetDevice(ix->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  char* base = static_cast<char*>(d_ws);
  // pageable source: staged before the call returns, so the host table may go out of scope
  FPB_CUDA_CHECK(cudaMemcpyAsync(base + X.off_table, table.data(), table.size() * 4, cudaMemcpyHostToDevice, st));
  FPB_TRY(launch_exhaustive_list_scores(ix, X, base, static_cast<const __half*>(d_queries), lists, st));
  float* scores = reinterpret_cast<float*>(base + X.off_scores);
  int32_t* cand = reinterpret_cast<int32_t*>(base + X.off_cand);
  int32_t* n_cand = reinterpret_cast<int32_t*>(base + X.off_n_cand);
  if (ix->doc_group)
    return rank_groups(ix, scores, cand, n_cand, X.cap, B, top_k, reinterpret_cast<uint64_t*>(base + X.off_gkeys),
                       d_out_ids, d_out_scores, d_out_counts, st);
  int32_t* n_sel = reinterpret_cast<int32_t*>(base + X.off_n_rerank);
  int32_t* sel_ids = reinterpret_cast<int32_t*>(base + X.off_rerank);
  float* sel_scores = reinterpret_cast<float*>(base + X.off_rerank_approx);
  // the candidates of a query are its list's documents in id order, so k3b_select's tie rule (candidate index asc)
  // is the id order, and the selected scores are the exact ones that k6_rank orders
  FPB_TRY(launch_select(scores, cand, n_cand, int(X.cap), B, top_k, sel_ids, sel_scores, n_sel, st));
  FPB_TRY(launch_rank(sel_scores, sel_ids, n_sel, top_k, B, top_k, ix->doc_id_base, d_out_ids, d_out_scores,
                      d_out_counts, st));
  return FPB_OK;
}

}  // namespace

extern "C" int fpb_search_exhaustive_subset(const fpb_index* ix, const void* d_queries, int B, int Q, int top_k,
                                            const int32_t* d_list_ids, const int64_t* d_list_offsets, int n_lists,
                                            int64_t max_list_len, const int32_t* h_query_list, void* d_ws,
                                            size_t ws_bytes, int64_t* d_out_ids, float* d_out_scores,
                                            int32_t* d_out_counts, void* stream) {
  // shapes, then the lists, then the index
  if (top_k < 1) {
    fpb_set_error("fpb_search_exhaustive_subset: top_k=%d must be >= 1", top_k);
    return FPB_ERR_INVALID;
  }
  FPB_TRY(check_exhaustive_shapes(B, Q, top_k));
  FPB_TRY(check_lists(n_lists, max_list_len));
  if (!h_query_list) {
    fpb_set_error("fpb_search_exhaustive_subset: NULL h_query_list");
    return FPB_ERR_INVALID;
  }
  for (int b = 0; b < B; ++b) {
    if (h_query_list[b] < 0 || h_query_list[b] >= n_lists) {
      fpb_set_error("fpb_search_exhaustive_subset: h_query_list[%d]=%d is not in [0, n_lists=%d)", b,
                    h_query_list[b], n_lists);
      return FPB_ERR_INVALID;
    }
  }
  const ExLists lists{d_list_ids, d_list_offsets, max_list_len, nullptr, 0};
  return exhaustive_list_search("fpb_search_exhaustive_subset", ix, d_queries, B, Q, top_k, lists,
                                d_list_offsets && (max_list_len == 0 || d_list_ids), n_lists, max_list_len,
                                h_query_list, d_ws, ws_bytes, d_out_ids, d_out_scores, d_out_counts, stream);
}

extern "C" int fpb_exhaustive_filter_workspace_bytes(const fpb_index* ix, int B, int Q, int top_k, int n_filters,
                                                     int64_t max_count, size_t* out) {
  if (!out) {
    fpb_set_error("fpb_exhaustive_filter_workspace_bytes: NULL output pointer");
    return FPB_ERR_INVALID;
  }
  if (top_k < 1) {
    fpb_set_error("fpb_exhaustive_filter_workspace_bytes: top_k=%d must be >= 1", top_k);
    return FPB_ERR_INVALID;
  }
  FPB_TRY(check_exhaustive_shapes(B, Q, top_k));
  FPB_TRY(check_lists(n_filters, max_count));
  ExLayout X;
  FPB_TRY(exhaustive_layout(ix, B, Q, top_k, &X, n_filters, max_count));
  *out = size_t(X.total_bytes);
  return FPB_OK;
}

extern "C" int fpb_search_exhaustive_filter(const fpb_index* ix, const void* d_queries, int B, int Q, int top_k,
                                            const uint32_t* d_filters, int n_filters, int64_t n_bits,
                                            int64_t max_count, const int32_t* h_query_filter, void* d_ws,
                                            size_t ws_bytes, int64_t* d_out_ids, float* d_out_scores,
                                            int32_t* d_out_counts, void* stream) {
  const char* who = "fpb_search_exhaustive_filter";
  if (top_k < 1) {
    fpb_set_error("%s: top_k=%d must be >= 1", who, top_k);
    return FPB_ERR_INVALID;
  }
  FPB_TRY(check_exhaustive_shapes(B, Q, top_k));
  FPB_TRY(check_filter_args(who, d_filters, n_filters, n_bits, h_query_filter, B));
  if (max_count < 0) {
    fpb_set_error("%s: max_count=%lld must be >= 0", who, (long long)max_count);
    return FPB_ERR_INVALID;
  }
  const ExLists lists{nullptr, nullptr, 0, d_filters, n_bits};
  return exhaustive_list_search(who, ix, d_queries, B, Q, top_k, lists, true, n_filters, max_count, h_query_filter,
                                d_ws, ws_bytes, d_out_ids, d_out_scores, d_out_counts, stream);
}
