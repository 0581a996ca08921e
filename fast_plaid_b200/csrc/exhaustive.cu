// Exhaustive exact search behind the C ABI: K7 scores every document of the index against every query, then
// the approximate pipeline's own selection (k3b_select, with every document a candidate) and ranking (k6_rank)
// turn the [B, N] score array into the top_k.  Works on every index, including compress_only ones (no IVF is read).
#include "kernels.h"

namespace {

constexpr int EX_MAX_TOP_K = 4096;  // the k6_rank bound (one shared-memory bitonic sort per query)

int exhaustive_layout(const fpb_index* ix, int B, int Q, int top_k, ExLayout* X) {
  // the shape limits first: they do not depend on the index
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
  if (!ix) {
    fpb_set_error("exhaustive search: NULL index");
    return FPB_ERR_INVALID;
  }
  X->B = B;
  X->Q = Q;
  X->Qs = (Q + 15) / 16 * 16;
  X->n_rows = int((int64_t(B) * X->Qs + 127) / 128 * 128);
  X->top_k = top_k;
  X->grid = ix->sm_count;
  const int64_t N = ix->N, cap = N > 0 ? N : 1;
  int64_t off = 0;
  auto take = [&](int64_t bytes) {
    const int64_t o = off;
    off += fpb_align256(bytes);
    return o;
  };
  X->off_rows = take(int64_t(X->n_rows) * ix->dim * 2);
  X->off_acc = take(int64_t(B) * N * 8);
  X->off_carry = take(int64_t(X->grid) * X->n_rows * 4);
  X->off_counter = take(4);
  const bool sel = top_k > 0;
  X->off_scores = take(sel ? int64_t(B) * cap * 4 : 0);
  X->off_n_rerank = take(sel ? int64_t(B) * 4 : 0);
  X->off_rerank = take(sel ? int64_t(B) * top_k * 4 : 0);
  X->off_rerank_approx = take(sel ? int64_t(B) * top_k * 4 : 0);
  X->total_bytes = off;
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
