// Internal launchers (one per pipeline stage).  All are asynchronous on `stream`.
#pragma once
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

// ---- Residual codecs: the (dim, nbits) pairs an index may have ----------------------------------------------------
template <int D_, int NBITS_>
struct Codec {
  static constexpr int D = D_, NBITS = NBITS_;
};
// The one list of them, nbits 2 and 4 at dim 64 and 128, nbits 1 at dim 128: f(Codec<D, NBITS>{}) for each in turn
// until one returns true.
template <class F>
constexpr bool fpb_any_codec(F&& f) {
  return f(Codec<128, 4>{}) || f(Codec<128, 2>{}) || f(Codec<64, 4>{}) || f(Codec<64, 2>{}) || f(Codec<128, 1>{});
}
constexpr bool fpb_codec_supported(int dim, int nbits) {
  return fpb_any_codec([=](auto c) { return c.D == dim && c.NBITS == nbits; });
}
// sets the error "<who>: unsupported embedding dim=.. with nbits=..", naming the supported pairs
inline int fpb_codec_error(const char* who, int dim, int nbits) {
  fpb_set_error("%s: unsupported embedding dim=%d with nbits=%d: this build supports nbits 2 and 4 at dim 64 and 128, "
                "nbits 1 at dim 128", who, dim, nbits);
  return FPB_ERR_UNSUPPORTED;
}
// f(Codec<dim, nbits>{}), an FPB_* status, or the codec error.  f is instantiated at every supported pair: a launch
// that exists at some pairs only selects them with `if constexpr`.
template <class F>
int fpb_with_codec(int dim, int nbits, const char* who, F&& f) {
  int rc = FPB_OK;
  const bool found = fpb_any_codec([&](auto c) {
    if (c.D != dim || c.NBITS != nbits) return false;
    rc = f(c);
    return true;
  });
  return found ? rc : fpb_codec_error(who, dim, nbits);
}

// ---- Tuning pins: environment variables that pin a choice the engine otherwise makes, for A/B timing and tests ----
// Each is read at every launch, so one process can switch.  A value not listed is ignored, as if the variable were
// unset.  Apart from FPB_K7, none changes a result.
//   FPB_K1=v1                      K1 on the mma.sync kernel, not wgmma
//   FPB_K5=v1                      the generic K5, not v4 or v5
//   FPB_K5_DOCS_PER_CHUNK=1..32    v5's documents per chunk, still capped by its pass table
//   FPB_K7=mma|decode              K7's timing variants at dim 128 / nbits 4 (their scores are meaningless)
//   FPB_K7_DOCS_PER_CHUNK=1..32    K7's documents per chunk
//   FPB_K3_EXACT_DOCS_PER_CHUNK=n  the exact pass's documents per chunk of a refine list, n = 8, 16, .., 64
//   FPB_K3_LAMBDA=x                x > 0, clamped to [0.5, 64]: the bound pass's tau level (k3_tau_lambda)
//   FPB_K3_GROUP=4|5|6             the bound pass's windows per group, instead of fpb_index::walk_group
inline const char* fpb_env(const char* name) {  // NULL when unset or empty
  const char* e = getenv(name);
  return e && *e ? e : nullptr;
}
inline bool fpb_env_is(const char* name, const char* value) {
  const char* e = fpb_env(name);
  return e && strcmp(e, value) == 0;
}
// the integer value of `name`; 0 when it is unset, not an integer or outside [lo, hi]
inline int fpb_env_int(const char* name, int lo, int hi) {
  const char* e = fpb_env(name);
  if (!e) return 0;
  char* end;
  const long v = strtol(e, &end, 10);
  return *end == '\0' && v >= lo && v <= hi ? int(v) : 0;
}
// the float value of `name`; 0 when it is unset or not a number
inline float fpb_env_float(const char* name) {
  const char* e = fpb_env(name);
  if (!e) return 0.f;
  char* end;
  const float v = strtof(e, &end);
  return *end == '\0' ? v : 0.f;
}

// ---- The probe: n_ivf_probe in [1, FPB_MAX_PROBE] cells per query token ------------------------------------------
// Up to FPB_WARP_PROBE cells, K1b keeps a warp-held list and K2 drops a repeated cell by scanning the query's earlier
// probe slots.  Above it, K1b selects block-wide and K2 drops repeats with a per-query bitmap over the centroids
// ([B, cbitmap_words] u32), stored in the cells' region after the [B, Q, n_probe] cells.
constexpr int FPB_WARP_PROBE = 32;
constexpr int FPB_MAX_PROBE = 4096;
inline int64_t fpb_cells_bytes(const fpb_layout& L) { return int64_t(L.B) * L.Q * L.n_probe * 4; }
inline int64_t fpb_probe_bitmap_bytes(const fpb_layout& L) {
  return L.n_probe > FPB_WARP_PROBE ? int64_t(L.B) * L.cbitmap_words * 4 : 0;
}

struct Ws {
  const fpb_layout* L;
  char* base;
  __half* queries() const { return reinterpret_cast<__half*>(base + L->off_queries); }
  __half* S() const { return reinterpret_cast<__half*>(base + L->off_S); }
  __half* tmax() const { return reinterpret_cast<__half*>(base + L->off_tmax); }
  int32_t* cells() const { return reinterpret_cast<int32_t*>(base + L->off_cells); }
  uint32_t* probe_bitmap() const {  // n_probe > FPB_WARP_PROBE only
    return reinterpret_cast<uint32_t*>(base + L->off_cells + fpb_align256(fpb_cells_bytes(*L)));
  }
  uint32_t* bitmap() const { return reinterpret_cast<uint32_t*>(base + L->off_bitmap); }
  int32_t* n_cand() const { return reinterpret_cast<int32_t*>(base + L->off_n_cand); }
  int32_t* cand() const { return reinterpret_cast<int32_t*>(base + L->off_cand); }
  float* approx() const { return reinterpret_cast<float*>(base + L->off_approx); }
  int32_t* work() const { return reinterpret_cast<int32_t*>(base + L->off_work); }
  int32_t* n_rerank() const { return reinterpret_cast<int32_t*>(base + L->off_n_rerank); }
  int32_t* rerank() const { return reinterpret_cast<int32_t*>(base + L->off_rerank); }
  float* rerank_approx() const { return reinterpret_cast<float*>(base + L->off_rerank_approx); }
  float* exact() const { return reinterpret_cast<float*>(base + L->off_exact); }
  uint32_t* cbitmap() const { return reinterpret_cast<uint32_t*>(base + L->off_cbitmap); }
  int32_t* clist() const { return reinterpret_cast<int32_t*>(base + L->off_clist); }
  int32_t* n_clist() const { return reinterpret_cast<int32_t*>(base + L->off_n_clist); }
  uint32_t* sbitmap() const { return reinterpret_cast<uint32_t*>(base + L->off_sbitmap); }
  __half* tau() const { return reinterpret_cast<__half*>(base + L->off_tau); }
  uint32_t* hibits() const { return reinterpret_cast<uint32_t*>(base + L->off_hibits); }
  float* lb() const { return reinterpret_cast<float*>(base + L->off_lb); }
  int32_t* refine() const { return reinterpret_cast<int32_t*>(base + L->off_refine); }
  int32_t* n_refine() const { return reinterpret_cast<int32_t*>(base + L->off_n_refine); }
  float* thresh() const { return reinterpret_cast<float*>(base + L->off_thresh); }
  int32_t* work2() const { return reinterpret_cast<int32_t*>(base + L->off_work2); }
  unsigned long long* stats() const { return reinterpret_cast<unsigned long long*>(base + L->off_stats); }
};

int launch_pad_queries(const fpb_index* ix, const Ws& ws, const __half* d_queries, cudaStream_t st);
int launch_centroid_scores(const fpb_index* ix, const Ws& ws, cudaStream_t st);   // K1 (dispatch)
int launch_centroid_scores_v2(const fpb_index* ix, const Ws& ws, cudaStream_t st);  // K1 on wgmma
int launch_probe(const fpb_index* ix, const Ws& ws, bool subset, cudaStream_t st);       // K1b
int launch_candidates(const fpb_index* ix, const Ws& ws, bool subset, cudaStream_t st);  // K2
int launch_subset_mark(const fpb_index* ix, const Ws& ws, const int32_t* d_ids, const int64_t* d_offsets,
                       int64_t max_len, cudaStream_t st);
int launch_subset_compact(const fpb_index* ix, const Ws& ws, cudaStream_t st);
int launch_subset_merge(const fpb_index* ix, const Ws& ws, const uint32_t* d_all, int n_shards, cudaStream_t st);
int launch_subset(const fpb_index* ix, const Ws& ws, const int32_t* d_ids, const int64_t* d_offsets,
                  int64_t max_len, cudaStream_t st);                                      // subset structures
int launch_compact(const uint32_t* bitmap, const uint32_t* mask, int words, int32_t* out, int cap, int32_t* n_out,
                   int B, cudaStream_t st);
int launch_approx(const fpb_index* ix, const Ws& ws, int flags, cudaStream_t st); // K3 (flags: FPB_FLAG_APPROX_*)
int launch_walk_layout(const fpb_index* ix, cudaStream_t st);                     // K3's walk_codes (index load)
// K3b: per query b the R best of the n_cand[b] scores in row b of `scores` (row stride `stride`) by (score desc,
// candidate index asc); their ids (cand[b, i], or i itself when cand is NULL: then every one of the `stride` entries
// of a row is a candidate and n_cand is not read), their scores and their count go to rerank, rerank_scores [B, R]
// and n_rerank.
int launch_select(const float* scores, const int32_t* cand, const int32_t* n_cand, int stride, int B, int R,
                  int32_t* rerank, float* rerank_scores, int32_t* n_rerank, cudaStream_t st);
int launch_maxsim(const fpb_index* ix, const Ws& ws, cudaStream_t st);            // K5 (dispatch)
int launch_token_norms(const fpb_index* ix, __half* d_out, cudaStream_t st);      // per-token fp16 norms (index load)
int launch_maxsim_v4(const fpb_index* ix, const Ws& ws, cudaStream_t st);  // K5 v4 (register operands)
int launch_maxsim_v5(const fpb_index* ix, const Ws& ws, cudaStream_t st);  // K5 v5 (wgmma, 16 decode warps)
// 8-token passes per v5 chunk: a document of more passes than this goes to the generic kernel
constexpr int V5_MAX_PASS = 2048;
// K6: per query b the top_k of the n[b] (score, id) pairs in row b of scores / ids (row stride R) in the canonical
// order, ids offset by doc_id_base
int launch_rank(const float* scores, const int32_t* ids, const int32_t* n, int R, int B, int top_k,
                int64_t doc_id_base, int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts, cudaStream_t st);
// The shard threshold and the shard merge sort all n_shards*R records of a query in shared memory: at most
// FPB_MERGE_MAX_RECORDS of them.  check_merge_records sets the error (prefixed by `who`) and returns
// FPB_ERR_UNSUPPORTED above that, FPB_OK otherwise.
constexpr int FPB_MERGE_MAX_RECORDS = 16384;
int check_merge_records(const char* who, int n_shards, int R);
int launch_emit_keys(const fpb_index* ix, const Ws& ws, uint64_t* d_keys, cudaStream_t st);
int launch_apply_threshold(const Ws& ws, const uint64_t* d_all_keys, int n_shards, int rank, cudaStream_t st,
                           int b_stride = 0);
int launch_merge(const fpb_record* d_all_records, int n_shards, int b_stride, int n_queries, int R, int top_k,
                 int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts, cudaStream_t stream);
int launch_emit_records(const fpb_index* ix, const Ws& ws, fpb_record* d_records, cudaStream_t st);

// K3b and K6 of the search: select by the candidates' approximate scores, rank by the exact ones
inline int launch_select(const Ws& ws, cudaStream_t st) {
  return launch_select(ws.approx(), ws.cand(), ws.n_cand(), ws.L->cand_cap, ws.L->B, ws.L->R, ws.rerank(),
                       ws.rerank_approx(), ws.n_rerank(), st);
}
inline int launch_rank(const fpb_index* ix, const Ws& ws, int top_k, int64_t* d_out_ids, float* d_out_scores,
                       int32_t* d_out_counts, cudaStream_t st) {
  return launch_rank(ws.exact(), ws.rerank(), ws.n_rerank(), ws.L->R, ws.L->B, top_k, ix->doc_id_base, d_out_ids,
                     d_out_scores, d_out_counts, st);
}

// the document bitmap alone of subset_mark_kernel, [n_lists, words]: list l owns d_ids[d_offsets[l] ..
// d_offsets[l+1]) (global ids; ids outside the index are ignored)
int launch_doc_bitmap(const fpb_index* ix, const int32_t* d_ids, const int64_t* d_offsets, int64_t max_len,
                      int n_lists, uint32_t* bitmap, int words, cudaStream_t st);

// Workspace of the exhaustive search (exhaustive.cu).  The selection part (top_k > 0) holds the [B, N] scores that
// k3b_select reads (every document a candidate) and the [B, top_k] list it writes for k6_rank.  A list walk
// (n_lists > 0, fpb_search_exhaustive_subset) has [B, cap] scores instead, with their candidates, and the lists.
struct ExLayout {
  int B, Q, Qs, n_rows, top_k, grid;  // Qs = Q rounded up to 16; n_rows = B*Qs rounded up to 128; grid = K7 CTAs
  int64_t off_rows;     // f16 [n_rows, dim] dense query rows
  int64_t off_acc;      // u64 [B, N] fixed-point score sums ([B, cap] in a list walk)
  int64_t off_carry;    // f32 [grid, n_rows] running maxima of documents that cross a tile boundary
  int64_t off_counter;  // i32 chunk counter
  int64_t off_scores, off_n_rerank, off_rerank, off_rerank_approx;  // selection (top_k > 0)
  // list walk only (zero bytes otherwise).  n_rows = B*Qs + 48*n_lists rounded up to 128: every list's rows start on
  // a 64-row boundary.  list_docs = cap x the number of lists some query searches (set per call).
  int n_lists, words;       // lists; uint32 words of a document bitmap
  int64_t cap, list_docs;   // positions per list = min(N, max_list_len) (at least 1)
  int64_t off_bitmap;       // u32 [n_lists, words] documents of every list
  int64_t off_lists;        // i32 [n_lists, cap] sorted-unique local ids of every list
  int64_t off_lcount;       // i32 [n_lists] their numbers
  int64_t off_chunks;       // i32 [n_lists + 1] chunk prefix of the lists
  int64_t off_table;        // i32 ExListTable, built on the host
  int64_t off_cand;         // i32 [B, cap] query b's candidates (its list's ids)
  int64_t off_n_cand;       // i32 [B] their numbers
  int64_t total_bytes;
};

// The host-built table of a list walk (int32, in the workspace at off_table)
struct ExListTable {
  int32_t* row0;       // [n_lists] first query row of every list (64-row aligned)
  int32_t* row1;       // [n_lists] end of its rows (= row0 for a list no query searches)
  int32_t* qlist;      // [B] the list every query searches
  int32_t* grp_query;  // [n_rows / 16] query of every 16-row group of the row array, -1 for padding
  int32_t* grp_tok;    // [n_rows / 16] token of the group's first row
  static int64_t ints(int n_lists, int B, int n_rows) { return 2 * int64_t(n_lists) + B + 2 * int64_t(n_rows / 16); }
  static ExListTable at(int32_t* t, int n_lists, int B, int n_rows) {
    int32_t* q = t + 2 * int64_t(n_lists);
    return {t, t + n_lists, q, q + B, q + B + n_rows / 16};
  }
};

int launch_exhaustive_scores(const fpb_index* ix, const ExLayout& X, char* ws, const __half* d_queries,
                             float* d_scores, cudaStream_t st);  // K7 + finalize
// list walk: canonical lists, K7 over them, and the [B, cap] scores / candidates / counts of the layout
int launch_exhaustive_list_scores(const fpb_index* ix, const ExLayout& X, char* ws, const __half* d_queries,
                                  const int32_t* d_list_ids, const int64_t* d_list_offsets, int64_t max_list_len,
                                  cudaStream_t st);
