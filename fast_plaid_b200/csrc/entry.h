// What the search entry points of the C ABI (search.cu, comm.cu) share: the checks of their index, parameters and
// workspace, the prologue built from them, and the stage sequences more than one entry point runs.
#pragma once
#include "kernels.h"

// Each check sets the error message when it fails.
inline int fpb_require_ivf(const fpb_index* ix) {
  if (ix->ivf_offsets) return FPB_OK;
  // same text as rust/search/search.rs:227-232
  fpb_set_error(
      "This index was built with compress_only=True and does not support search. "
      "Rebuild with compress_only=False to enable search.");
  return FPB_ERR_NO_IVF;
}
inline int fpb_require_bytes(const char* what, int64_t need, size_t have) {
  if (size_t(need) <= have) return FPB_OK;
  fpb_set_error("%s too small: need %lld bytes, have %zu", what, (long long)need, have);
  return FPB_ERR_WORKSPACE;
}
inline int fpb_require_aligned(const char* what, const void* p) {
  if ((reinterpret_cast<uintptr_t>(p) & 255u) == 0) return FPB_OK;
  fpb_set_error("%s must be 256-byte aligned", what);
  return FPB_ERR_INVALID;
}

// One call's workspace, laid out for its B x Q queries, and the stream its stages run on.
struct Call {
  fpb_layout L;
  Ws ws{&L, nullptr};
  cudaStream_t st = nullptr;

  Call() = default;
  Call(const Call&) = delete;  // ws points into this object
  Call& operator=(const Call&) = delete;

  // The prologue: checks the index, the parameters and the workspace (need_ivf: the call reads the inverted file,
  // which a compress_only index lacks), lays the workspace out and selects the index's device.
  int begin(const fpb_index* ix, int B, int Q, const fpb_params* p, void* d_ws, size_t ws_bytes, bool need_ivf,
            void* stream) {
    if (!ix || !p || !d_ws) {
      fpb_set_error("search: NULL index, params or workspace");
      return FPB_ERR_INVALID;
    }
    if (need_ivf) FPB_TRY(fpb_require_ivf(ix));
    FPB_TRY(fpb_workspace_layout(ix, B, Q, p, &L));
    FPB_TRY(fpb_require_bytes("workspace", L.total_bytes, ws_bytes));
    FPB_TRY(fpb_require_aligned("workspace", d_ws));
    FPB_CUDA_CHECK(cudaSetDevice(ix->device));
    ws.base = static_cast<char*>(d_ws);
    st = static_cast<cudaStream_t>(stream);
    return FPB_OK;
  }
};

// Pad the queries into the workspace, then K1.
inline int run_centroid_scores(const fpb_index* ix, const Ws& ws, const void* d_queries, cudaStream_t st) {
  FPB_TRY(launch_pad_queries(ix, ws, static_cast<const __half*>(d_queries), st));
  return launch_centroid_scores(ix, ws, st);
}

// Probe, candidates, approximate scores, and the R best of them (K1b, K2, K3, K3b).
inline int run_probe_to_select(const fpb_index* ix, const Ws& ws, bool subset, cudaStream_t st) {
  FPB_TRY(launch_probe(ix, ws, subset, st));
  FPB_TRY(launch_candidates(ix, ws, subset, st));
  FPB_TRY(launch_approx(ix, ws, ws.L->flags, st));
  return launch_select(ws, st);
}

// The host-buffer form of a device search: copies the B x Q queries into d_queries, runs `search` on them, copies
// its results back and waits for the stream.
template <class Search>
int search_via_host(const char* name, const fpb_index* ix, const void* h_queries, int B, int Q, const fpb_params* p,
                    void* d_queries, const int64_t* d_out_ids, const float* d_out_scores, const int32_t* d_out_counts,
                    int64_t* h_out_ids, float* h_out_scores, int32_t* h_out_counts, void* stream, Search search) {
  if (!ix || !p || !h_queries || !d_queries || !h_out_ids || !h_out_scores || !h_out_counts) {
    fpb_set_error("%s: NULL pointer", name);
    return FPB_ERR_INVALID;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  FPB_CUDA_CHECK(cudaSetDevice(ix->device));
  FPB_CUDA_CHECK(cudaMemcpyAsync(d_queries, h_queries, size_t(B) * Q * ix->dim * 2, cudaMemcpyHostToDevice, st));
  FPB_TRY(search());
  const size_t n = size_t(B) * p->top_k;
  FPB_CUDA_CHECK(cudaMemcpyAsync(h_out_ids, d_out_ids, n * 8, cudaMemcpyDeviceToHost, st));
  FPB_CUDA_CHECK(cudaMemcpyAsync(h_out_scores, d_out_scores, n * 4, cudaMemcpyDeviceToHost, st));
  FPB_CUDA_CHECK(cudaMemcpyAsync(h_out_counts, d_out_counts, size_t(B) * 4, cudaMemcpyDeviceToHost, st));
  FPB_CUDA_CHECK(cudaStreamSynchronize(st));
  return FPB_OK;
}
