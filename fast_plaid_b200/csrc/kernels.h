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
// One block scans count [n] (i64): out[0] = 0, out[c + 1] = old[c + 1] + count[0..c], and, when cursor is not NULL,
// cursor[c] = out[c + 1] - count[c].  old == NULL reads as zeros.  The inverted file's new offsets (append, delete)
// and the delete's rank tables (scan.cu).
int launch_offsets_scan(const int64_t* old_offsets, const int64_t* count, int64_t n, int64_t* out, int64_t* cursor,
                        cudaStream_t st);
// blocks of a grid-stride loop over `items` items at `per_block` per block: at most 16 per SM, at least 1
inline int fpb_grid_for(int64_t items, int per_block, int sm_count) {
  const int64_t need = (items + per_block - 1) / per_block;
  const int64_t cap = int64_t(sm_count) * 16;
  return int(need < 1 ? 1 : (need < cap ? need : cap));
}
int launch_walk_layout(const fpb_index* ix, int64_t d0, cudaStream_t st);  // K3's walk_codes of documents [d0, N)
// the walk layout of documents [d0, N) in ix->walk's buffers, and walk_group (index.cu)
int fpb_extend_walk_layout(fpb_index* ix, int64_t d0);
// K3b: per query b the R best of the n_cand[b] scores in row b of `scores` (row stride `stride`) by (score desc,
// candidate index asc); their ids (cand[b, i], or i itself when cand is NULL: then every one of the `stride` entries
// of a row is a candidate and n_cand is not read), their scores and their count go to rerank, rerank_scores [B, R]
// and n_rerank.
int launch_select(const float* scores, const int32_t* cand, const int32_t* n_cand, int stride, int B, int R,
                  int32_t* rerank, float* rerank_scores, int32_t* n_rerank, cudaStream_t st);
int launch_maxsim(const fpb_index* ix, const Ws& ws, cudaStream_t st);            // K5 (dispatch)
// per-token fp16 norms of tokens [t0, E) into d_out[t0, E) (index load and append)
int launch_token_norms(const fpb_index* ix, __half* d_out, int64_t t0, cudaStream_t st);
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
// per query b the records of the n_sel[b] selected documents in row b of exact / approx / ids (row stride R):
// (approx, exact, doc_id_base + id), then padding records (-inf, -inf, -1) up to R
int launch_emit_records(const float* exact, const float* approx, const int32_t* ids, const int32_t* n_sel, int B,
                        int R, int64_t doc_id_base, fpb_record* d_records, cudaStream_t st);

// ---- Grouped results (groups.cu), on a handle of fpb_index_with_groups ----
// K6 by group: launch_rank's arguments, then at most max_per_group documents per group (its best ones), in the
// canonical order
int launch_rank_grouped(const float* scores, const int32_t* ids, const int32_t* n, int R, int B, int top_k,
                        int64_t doc_id_base, const int32_t* doc_group, int64_t n_groups, int max_per_group,
                        int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts, cudaStream_t st);
// gkeys [B, m * n_groups] (cleared here), m = max_per_group: round r (at offset r * n_groups of a row) holds per
// (query, group) the largest rank_key_f32(score, local id) below round r - 1's key, over row b of scores (stride
// cols), n[b] entries (n NULL: cols), entry p being document cand[b, p] (cand NULL: p).  Round 0 is the group's best.
int launch_group_max(const float* scores, const int32_t* cand, const int32_t* n, int64_t cols, int B,
                     const int32_t* doc_group, int64_t n_groups, int max_per_group, uint64_t* gkeys, int sm_count,
                     cudaStream_t st);
// per query the top_k largest non-empty keys of its gkeys row (n_groups keys), written as K6 writes its ranking
int launch_group_select(const uint64_t* gkeys, int64_t n_groups, int B, int top_k, int64_t doc_id_base,
                        int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts, cudaStream_t st);
// The grouped shard merge: launch_merge's records and query layout, the n_keep best by approx kept, ordered by exact,
// then at most max_per_group documents per group, the group of global id d being global_group[d] (a record whose id
// is outside [0, n_total_docs) or whose group is negative is skipped).  Checks every argument before any CUDA call.
int launch_merge_grouped(const fpb_record* d_all_records, int n_shards, int b_stride, int n_queries, int R, int n_keep,
                         int top_k, const int32_t* global_group, int64_t n_total_docs, int max_per_group,
                         int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts, cudaStream_t stream);
// records [B, top_k] of K6-style results: (score, score, id) for every entry, so a tail (-inf, -1) is a padding record
int launch_results_to_records(const int64_t* ids, const float* scores, int B, int top_k, fpb_record* d_records,
                              cudaStream_t st);
// The entry points that do not rank for a caller (sharded steps, records, keys) refuse a handle with groups, before
// any CUDA call
inline int fpb_refuse_groups(const char* who, const fpb_index* ix) {
  if (!ix || !ix->doc_group) return FPB_OK;
  fpb_set_error("%s: an index handle with groups (fpb_index_with_groups) is not supported here", who);
  return FPB_ERR_UNSUPPORTED;
}
// The sharded entry points that merge across ranks take a shard-grouped handle (fpb_index_with_shard_groups) and refuse
// the other handles with groups, which carry no map of the whole index
inline int fpb_refuse_unsharded_groups(const char* who, const fpb_index* ix) {
  return ix && ix->global_group ? FPB_OK : fpb_refuse_groups(who, ix);
}
// Every other entry point refuses a shard-grouped handle, before any CUDA call
inline int fpb_refuse_shard_groups(const char* who, const fpb_index* ix) {
  if (!ix || !ix->global_group) return FPB_OK;
  fpb_set_error("%s: a shard-grouped index handle (fpb_index_with_shard_groups) is accepted by the sharded search "
                "entry points only", who);
  return FPB_ERR_UNSUPPORTED;
}

// K3b and K6 of the search: select by the candidates' approximate scores, rank by the exact ones (by group when the
// handle carries groups)
inline int launch_select(const Ws& ws, cudaStream_t st) {
  return launch_select(ws.approx(), ws.cand(), ws.n_cand(), ws.L->cand_cap, ws.L->B, ws.L->R, ws.rerank(),
                       ws.rerank_approx(), ws.n_rerank(), st);
}
inline int launch_rank(const fpb_index* ix, const Ws& ws, int top_k, int64_t* d_out_ids, float* d_out_scores,
                       int32_t* d_out_counts, cudaStream_t st) {
  if (ix->doc_group)
    return launch_rank_grouped(ws.exact(), ws.rerank(), ws.n_rerank(), ws.L->R, ws.L->B, top_k, ix->doc_id_base,
                               ix->doc_group, ix->n_groups, ix->max_per_group, d_out_ids, d_out_scores,
                               d_out_counts, st);
  return launch_rank(ws.exact(), ws.rerank(), ws.n_rerank(), ws.L->R, ws.L->B, top_k, ix->doc_id_base, d_out_ids,
                     d_out_scores, d_out_counts, st);
}
// the records of the search's re-ranked list, for the shard merge
inline int launch_emit_records(const fpb_index* ix, const Ws& ws, fpb_record* d_records, cudaStream_t st) {
  return launch_emit_records(ws.exact(), ws.rerank_approx(), ws.rerank(), ws.n_rerank(), ws.L->B, ws.L->R,
                             ix->doc_id_base, d_records, st);
}

// the document bitmap alone of subset_mark_kernel, [n_lists, words]: list l owns d_ids[d_offsets[l] ..
// d_offsets[l+1]) (global ids; ids outside the index are ignored)
int launch_doc_bitmap(const fpb_index* ix, const int32_t* d_ids, const int64_t* d_offsets, int64_t max_len,
                      int n_lists, uint32_t* bitmap, int words, cudaStream_t st);

// ---- Filters (filter.cu): packed bitmaps over GLOBAL document ids, [n_filters, ceil(n_bits / 32)] uint32 ----------
// The arguments every filtered entry point checks before any CUDA call: non-NULL bitmaps and map, 1 <= n_filters <=
// 65535, n_bits >= 0, h_query_filter[b] in [0, n_filters) for b < B.  Sets the error (prefixed by `who`).
int check_filter_args(const char* who, const uint32_t* d_filters, int n_filters, int64_t n_bits,
                      const int32_t* h_query_filter, int B);
// The filter stage of a search: the sbitmap / cbitmap rows of the workspace (FPB_FLAG_SUBSET) that subset_mark_kernel
// builds from id lists, built once per distinct filter and copied to the other queries of the filter (no compaction)
int launch_filter(const fpb_index* ix, const Ws& ws, const uint32_t* d_filters, int n_filters, int64_t n_bits,
                  const int32_t* h_query_filter, cudaStream_t st);
// whether the filter stage accumulates a row's centroid bitmap (cwords words) in shared memory
bool fpb_filter_centroids_in_shared(const fpb_index* ix, int cwords);
// The exhaustive search's lists from filter rows: list l is the index's range of filter l, as a document bitmap
// [n_lists, words] and then its sorted local ids ids [n_lists, cap] and their numbers count [n_lists].  A list of more
// than cap documents keeps its first cap.
int launch_filter_lists(const fpb_index* ix, const uint32_t* d_filters, int64_t n_bits, int n_lists,
                        uint32_t* bitmap, int words, int32_t* ids, int cap, int32_t* count, cudaStream_t st);

// The shape limits of the exhaustive search: B >= 1, 1 <= Q <= 256, 0 <= top_k <= FPB_EX_MAX_TOP_K (top_k = 0: the
// scores alone).  Sets the error and returns FPB_ERR_INVALID / FPB_ERR_UNSUPPORTED outside them.
constexpr int FPB_EX_MAX_TOP_K = 4096;  // the k6_rank bound (one shared-memory bitonic sort per query)
int check_exhaustive_shapes(int B, int Q, int top_k);

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
  // a handle with groups (top_k > 0): u64 [B, max_per_group * n_groups] group keys, in the accumulator region (free
  // once K7 is finalized) when they fit there, after everything else otherwise
  int64_t off_gkeys;
  // a shard-grouped handle (top_k > 0): i64 [B, top_k] the ids of the shard's grouped top_k, before they become records
  int64_t off_sel_ids;
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
// The documents of a list walk's lists: id lists (d_list_ids / d_list_offsets / max_list_len, launch_doc_bitmap), or
// filter rows when d_filters is not NULL (launch_filter_lists)
struct ExLists {
  const int32_t* d_list_ids;
  const int64_t* d_list_offsets;
  int64_t max_list_len;
  const uint32_t* d_filters;
  int64_t n_bits;
};
// list walk: canonical lists, K7 over them, and the [B, cap] scores / candidates / counts of the layout
int launch_exhaustive_list_scores(const fpb_index* ix, const ExLayout& X, char* ws, const __half* d_queries,
                                  const ExLists& lists, cudaStream_t st);
