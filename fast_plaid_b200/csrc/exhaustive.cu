// Exhaustive exact search behind the C ABI: K7 scores every document of the index against every query, then
// the approximate pipeline's own selection (k3b_select, with every document a candidate) and ranking (k6_rank)
// turn the [B, N] score array into the top_k.  Works on every index, including compress_only ones (no IVF is read).
#include <algorithm>
#include <vector>

#include "kernels.h"

namespace {

constexpr int EX_MAX_TOP_K = 4096;  // the k6_rank bound (one shared-memory bitonic sort per query)

int check_shapes(int B, int Q, int top_k) {
  if (B <= 0 || Q <= 0 || top_k < 0) {
    fpb_set_error("exhaustive search: B=%d Q=%d top_k=%d must be positive", B, Q, top_k);
    return FPB_ERR_INVALID;
  }
  if (Q > 256) {
    fpb_set_error("queries with more than 256 tokens are not supported (Q=%d)", Q);
    return FPB_ERR_UNSUPPORTED;
  }
  if (top_k > EX_MAX_TOP_K) {
    fpb_set_error("exhaustive search: top_k=%d exceeds the supported maximum of %d", top_k, EX_MAX_TOP_K);
    return FPB_ERR_UNSUPPORTED;
  }
  return FPB_OK;
}

// n_lists = 0: the full scan.  n_lists > 0: a list walk over lists of at most max_list_len ids.
int exhaustive_layout(const fpb_index* ix, int B, int Q, int top_k, ExLayout* X, int n_lists = 0,
                      int64_t max_list_len = 0) {
  // the shape limits first: they do not depend on the index
  FPB_TRY(check_shapes(B, Q, top_k));
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

extern "C" int fpb_search_exhaustive(const fpb_index* ix, const void* d_queries, int B, int Q, int top_k, void* d_ws,
                                     size_t ws_bytes, int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts,
                                     void* stream) {
  if (top_k < 1) {
    fpb_set_error("fpb_search_exhaustive: top_k=%d must be >= 1", top_k);
    return FPB_ERR_INVALID;
  }
  ExLayout X;
  FPB_TRY(exhaustive_layout(ix, B, Q, top_k, &X));
  FPB_TRY(check_workspace(X, d_ws, ws_bytes));
  if (!d_queries || !d_out_ids || !d_out_scores || !d_out_counts) {
    fpb_set_error("fpb_search_exhaustive: NULL query or output pointer");
    return FPB_ERR_INVALID;
  }
  if ((reinterpret_cast<uintptr_t>(d_queries) & 15u) != 0) {
    fpb_set_error("fpb_search_exhaustive: queries must be 16-byte aligned");
    return FPB_ERR_INVALID;
  }
  FPB_CUDA_CHECK(cudaSetDevice(ix->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  char* base = static_cast<char*>(d_ws);
  float* scores = reinterpret_cast<float*>(base + X.off_scores);
  int32_t* n_sel = reinterpret_cast<int32_t*>(base + X.off_n_rerank);
  int32_t* sel_ids = reinterpret_cast<int32_t*>(base + X.off_rerank);
  float* sel_scores = reinterpret_cast<float*>(base + X.off_rerank_approx);
  FPB_TRY(launch_exhaustive_scores(ix, X, base, static_cast<const __half*>(d_queries), scores, st));
  // every document is a candidate, and its "approximate" score is its exact one: the selected list holds the exact
  // scores that k6_rank orders
  FPB_TRY(launch_select(scores, nullptr, nullptr, int(ix->N), B, top_k, sel_ids, sel_scores, n_sel, st));
  FPB_TRY(launch_rank(sel_scores, sel_ids, n_sel, top_k, B, top_k, ix->doc_id_base, d_out_ids, d_out_scores,
                      d_out_counts, st));
  return FPB_OK;
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
  FPB_TRY(check_shapes(B, Q, top_k));
  FPB_TRY(check_lists(n_lists, max_list_len));
  ExLayout X;
  FPB_TRY(exhaustive_layout(ix, B, Q, top_k, &X, n_lists, max_list_len));
  *out = size_t(X.total_bytes);
  return FPB_OK;
}

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
  FPB_TRY(check_shapes(B, Q, top_k));
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
  ExLayout X;
  FPB_TRY(exhaustive_layout(ix, B, Q, top_k, &X, n_lists, max_list_len));
  FPB_TRY(check_workspace(X, d_ws, ws_bytes));
  if (!d_queries || !d_list_offsets || (max_list_len > 0 && !d_list_ids) || !d_out_ids || !d_out_scores ||
      !d_out_counts) {
    fpb_set_error("fpb_search_exhaustive_subset: NULL query, list or output pointer");
    return FPB_ERR_INVALID;
  }
  if ((reinterpret_cast<uintptr_t>(d_queries) & 15u) != 0) {
    fpb_set_error("fpb_search_exhaustive_subset: queries must be 16-byte aligned");
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
  FPB_TRY(launch_exhaustive_list_scores(ix, X, base, static_cast<const __half*>(d_queries), d_list_ids,
                                        d_list_offsets, max_list_len, st));
  float* scores = reinterpret_cast<float*>(base + X.off_scores);
  int32_t* cand = reinterpret_cast<int32_t*>(base + X.off_cand);
  int32_t* n_cand = reinterpret_cast<int32_t*>(base + X.off_n_cand);
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
