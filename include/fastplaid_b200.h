/*
 * fastplaid_b200.h -- C ABI of the H100-native PLAID search engine.
 *
 * This is the drop-in boundary for the search hot path of lightonai/fast-plaid
 * (v1.4.6 @ 87f96f6).  In the reference that path sits behind the PyO3 module
 * `fast_plaid.fast_plaid_rust` (rust/lib.rs:366-383).  Each entry point below names the
 * reference interface it replaces.  Conventions:
 *
 *   - plain C types only; every pointer named `d_*` is a DEVICE pointer on the index's
 *     GPU, every pointer named `h_*` is a HOST pointer, `stream` is a cudaStream_t
 *     passed as void* (NULL = legacy default stream);
 *   - every function returns 0 on success or a negative code; the message is available
 *     from fpb_last_error() (thread-local).  No exception crosses the boundary.  The
 *     reference's PyValueError / PyRuntimeError (rust/utils/errors.rs:5-7) are raised by
 *     the Python host from these codes;
 *   - every entry point that takes a `stream` runs all its device work on it, and is
 *     asynchronous w.r.t. the host unless its name ends in `_host` (those synchronise the
 *     stream before returning) or its comment says "Synchronous on `stream`" (the index
 *     maintenance calls that read a size back).  The small host tables a call builds
 *     (the query map of a filtered or list-subset search) are copied from pageable memory
 *     before the call returns, without waiting for the stream;
 *   - an fpb_index is immutable after creation and may be searched concurrently from
 *     several host threads on different streams with different workspaces, like the
 *     reference's `LoadedIndex` (`unsafe impl Send/Sync`, rust/search/load.rs:58-59).
 *     It does NOT own the big arrays: the caller (PyTorch) keeps them alive.
 */
#ifndef FASTPLAID_B200_H_
#define FASTPLAID_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FPB_OK 0
#define FPB_ERR_INVALID (-1)  /* bad argument -> Python ValueError  (errors.rs:5-7)   */
#define FPB_ERR_CUDA (-2)     /* CUDA runtime failure -> RuntimeError                  */
#define FPB_ERR_UNSUPPORTED (-3)
#define FPB_ERR_WORKSPACE (-4) /* workspace too small                                  */
#define FPB_ERR_NO_IVF (-5)   /* compress_only index: search refused (search.rs:227-232) */

typedef struct fpb_index fpb_index;
struct fpb_record;

/* Thread-local message of the last failing call in this thread. */
const char* fpb_last_error(void);
/* ABI version (bumped on any signature change). */
int fpb_abi_version(void);

/*
 * fpb_index_create  -- replaces `construct_index` (rust/search/load.rs:122-186) and
 * `ResidualCodec::load` (rust/utils/residual_codec.rs:72-152).
 *
 *   d_centroids       f16 [n_centroids, dim], row-major            (load.rs:145)
 *   d_bucket_weights  f16 [1 << nbits]                              (load.rs:150)
 *   d_doc_offsets     i64 [n_docs + 1], exclusive cumsum of doclens (tensor.rs:221-224)
 *   d_doc_codes       i32 [n_tokens]   (narrowed from the on-disk int64 by the loader)
 *   d_doc_residuals   u8  [n_tokens, dim*nbits/8]
 *   d_token_norms     f16 [n_tokens]  OUTPUT, caller-owned like the other arrays: filled here with the fp16 norm of
 *                     every decompressed token (the `norm(...)` of decompress_residuals, search.rs:86-93), which the
 *                     MaxSim / reconstruct kernels then read instead of recomputing it per (query, document) pair
 *   d_ivf_offsets     i64 [n_centroids + 1]  or NULL for a compress_only index
 *   d_ivf_pids        i32 [n_ivf]            (LOCAL doc ids, ascending within a list)
 *   doc_id_base       global id of local doc 0 (document sharding; 0 on one GPU)
 *
 * The two 256-entry LUTs of the reference collapse into one (1<<nbits)-entry permuted
 * weight table w_perm[i] = bucket_weights[bitrev_nbits(i)] built here on the host.
 *
 * Supported (dim, nbits): nbits 2 and 4 at dim 64 and 128, nbits 1 at dim 128 (16-byte residual rows).  Anything
 * else, dim 64 with nbits 1 included, returns FPB_ERR_UNSUPPORTED before any CUDA call, with a message naming dim
 * and nbits.
 *
 * The handle also allocates one derived device array, in growable buffers it shares with the handles appended to
 * it (fpb_index_append) and that the last fpb_index_destroy frees: the approximate stage's copy of the codes, each
 * document's tokens reordered into whole 32-token windows (4 bytes per token rounded up to a multiple of 32 per
 * document, plus 8 bytes per document).
 */
int fpb_index_create(fpb_index** out, int device, int nbits, int dim, int64_t n_centroids,
                     const void* d_centroids, const void* d_bucket_weights, int64_t n_docs,
                     const int64_t* d_doc_offsets, const int32_t* d_doc_codes,
                     const uint8_t* d_doc_residuals, void* d_token_norms, const int64_t* d_ivf_offsets,
                     const int32_t* d_ivf_pids, int64_t n_ivf, int64_t max_doc_len,
                     int64_t doc_id_base);
void fpb_index_destroy(fpb_index* index);
/* The walk layout of an index (tests and tools): *n_windows = number of 32-code windows; when non-NULL, d_codes
 * (i32 [32 * n_windows]) and d_win (i64 [n_docs + 1], first window of each document) receive device copies.
 * Synchronous. */
int fpb_index_walk_layout(const fpb_index* index, int64_t* n_windows, int32_t* d_codes, int64_t* d_win);
/* Windows per group of the approximate stage's bound pass (4, 5 or 6), chosen from the walk layout; -1 on NULL. */
int fpb_index_walk_group(const fpb_index* index);

/*
 * Growable device buffers: address space reserved once on `device` (max_bytes, or the device's memory when 0),
 * backed by physical memory mapped in 2 MB granules as it is committed (the driver's virtual memory management).
 * fpb_buffer_ptr never changes, so an index's arrays can grow in place while a handle over their first bytes stays
 * valid.  fpb_buffer_commit(b, bytes) maps up to at least `bytes` from the start (a no-op when already mapped) and
 * leaves the mapped contents as they are; it is synchronous.  fpb_buffer_destroy unmaps and frees everything: no
 * work may still read the buffer, and no handle may still use it.
 */
typedef struct fpb_buffer fpb_buffer;
int fpb_buffer_reserve(fpb_buffer** out, int device, size_t max_bytes);
int fpb_buffer_commit(fpb_buffer* buffer, size_t bytes);
void* fpb_buffer_ptr(const fpb_buffer* buffer);
size_t fpb_buffer_mapped_bytes(const fpb_buffer* buffer);
void fpb_buffer_destroy(fpb_buffer* buffer);

/*
 * fpb_index_append -- a new handle over `index` grown to n_docs >= N documents and n_tokens >= E tokens.  The
 * caller has appended the new documents' data: d_doc_offsets (i64 [n_docs + 1]) starts with the old handle's N + 1
 * offsets, and d_doc_codes / d_doc_residuals hold the old handle's E tokens followed by the new ones.  The arrays may
 * be the old handle's own buffers grown in place (fpb_buffer_*) or copies.  d_token_norms holds the old handle's
 * E norms; the norms of tokens [E, n_tokens) are computed here.  The walk layout is extended for the new documents
 * only, in the old handle's shared buffers, and walk_group is re-chosen: both equal what fpb_index_create builds for
 * the grown index.  d_ivf_offsets / d_ivf_pids / n_ivf are the grown index's inverted file (fpb_ivf_append), NULL /
 * 0 for a compress_only index exactly when the old one has none; max_doc_len is the grown index's.
 *
 * The old handle stays valid and unchanged, so searches on it may continue.  Only a handle over all the documents
 * laid out so far may append (appending twice to the same handle is refused).  Bad sizes, NULL pointers and an IVF
 * that differs in kind from the old handle's are refused before any CUDA call; an offsets array whose entry N is not
 * E, or whose entry n_docs is not n_tokens, is refused before any kernel.  Synchronous.
 */
int fpb_index_append(fpb_index** out, const fpb_index* index, int64_t n_docs, int64_t n_tokens,
                     const int64_t* d_doc_offsets, const int32_t* d_doc_codes, const uint8_t* d_doc_residuals,
                     void* d_token_norms, const int64_t* d_ivf_offsets, const int32_t* d_ivf_pids, int64_t n_ivf,
                     int64_t max_doc_len);

/*
 * fpb_index_with_groups -- grouped results: a new handle over every array of `index` (shared, like
 * fpb_index_append's handles share the walk layout) that also carries d_doc_group (i32 [n_docs], borrowed: the caller
 * keeps it alive until the handle's last search has run), the group of every local document, dense in [0, n_groups).
 * Each query then gets at most one document per group: the group's best under the canonical order (score desc, then
 * id asc), these ranked in that order, d_out_counts[b] = min(top_k, groups present), tails id -1 / score -inf, and
 * every score the ungrouped search's, bit for bit.  A document whose group is outside [0, n_groups) is skipped.
 *   - fpb_search_batch, _subset, _filter, _host and fpb_stage_rank group the re-ranked list (the n_full_scores / 4
 *     documents of the approximate stage): the ungrouped search with top_k = n_full_scores / 4, each group's first
 *     document kept, cut to top_k.  So fewer than top_k documents can come back; a larger n_full_scores gives more.
 *   - fpb_search_exhaustive, _subset and _filter are exact: the exhaustive ranking (of the query's list) with each
 *     group's first document kept.  top_k <= 4096 counts groups.  Their *_workspace_bytes include the group keys'
 *     scratch, [B, n_groups] u64 beyond what the accumulator region holds.
 *   - The sharded entry points and those that emit records or keys return FPB_ERR_UNSUPPORTED.
 * NULL pointers and n_groups outside [1, INT32_MAX] are refused before any CUDA call.  Destroy the handle with
 * fpb_index_destroy; `index` stays valid.  fpb_index_append on it returns a handle without groups.
 *
 * fpb_index_with_groups_max -- the same handle carrying max_per_group = m in [1, FPB_MAX_PER_GROUP]: each query keeps
 * up to m documents per group.  The ranking is the canonical one (restricted to the query's subset) with a document
 * kept when fewer than m documents of its group were kept before it; top_k counts documents, scores stay the
 * ungrouped ones bit for bit.  m = 1 is fpb_index_with_groups; m >= the largest group gives the ungrouped ranking.
 *   - The search entry points apply the rule to the re-ranked list, as above.
 *   - The exhaustive entry points stay exact: m rounds of the group maximum, round r bounded by round r - 1's key.
 *     Their *_workspace_bytes report the larger scratch, [B, m * n_groups] u64 beyond what the accumulator region
 *     holds.
 * m outside [1, FPB_MAX_PER_GROUP] is refused with the other arguments, before any CUDA call.
 */
int fpb_index_with_groups(fpb_index** out, const fpb_index* index, const int32_t* d_doc_group, int64_t n_groups);
#define FPB_MAX_PER_GROUP 64
int fpb_index_with_groups_max(fpb_index** out, const fpb_index* index, const int32_t* d_doc_group, int64_t n_groups,
                              int max_per_group);

/*
 * fpb_index_with_bias -- biased scores: a new handle over every array of `index` (shared, like fpb_index_with_groups'
 * handles) that also carries d_doc_bias (f32 [n_docs], borrowed: the caller keeps it alive until the handle's last
 * search has run), a finite bias per local document.  Every exact score the handle produces is then
 * s'_d = s_d + d_doc_bias[d], one fp32 addition rounded to nearest, and everything that ranks or selects on exact scores
 * sees s'_d:
 *   - fpb_exhaustive_scores returns the biased table, and fpb_search_exhaustive, _subset and _filter rank every
 *     (listed) document by s'_d, exactly, with or without groups;
 *   - fpb_search_batch, _subset, _filter, _host and fpb_stage_maxsim bias the n_full_scores / 4 documents they re-rank:
 *     the candidate stage is unchanged, so the result is the unbiased search with top_k = n_full_scores / 4, biased,
 *     re-sorted by (score desc, id asc), grouped if the handle has groups, cut to top_k;
 *   - the sharded entry points and their records carry s'_d (each rank passes its slice of the whole index's bias).
 * The derived handles compose in either order: fpb_index_with_groups(_max) and fpb_index_with_shard_groups on a biased
 * handle keep the bias, and fpb_index_with_bias on a grouped handle keeps its groups.  A bias of +-inf or NaN is not
 * checked here (the caller refuses it: a NaN would break the selections' order); a finite sum that overflows is
 * +-inf, which ranks like any other value.  NULL pointers and n_docs != the index's document count are refused before
 * any CUDA call.  Destroy the handle with fpb_index_destroy; `index` stays valid.  fpb_index_append on it returns a
 * handle without a bias.
 */
int fpb_index_with_bias(fpb_index** out, const fpb_index* index, const float* d_doc_bias, int64_t n_docs);

/*
 * fpb_ivf_append -- the inverted file of an index of n_old_docs documents grown by n_new_docs documents (ids
 * n_old_docs ..): for every one of the n_cells cells, its old list (d_ivf_offsets i64 [n_cells + 1] into d_ivf_pids)
 * followed by the ascending ids of the new documents with a token in that cell.  The new documents' codes are
 * d_new_codes (i32, d_new_offsets i64 [n_new_docs + 1] from 0).  Writes d_out_offsets (i64 [n_cells + 1]), sets
 * *h_n_ivf to the number of postings and, unless d_out_pids is NULL (a call that sizes the output), writes them to
 * d_out_pids (i32, room for out_capacity ids).  A code outside [0, n_cells) is refused.  Equal to building the
 * inverted file of the whole index from scratch.  Synchronous on `stream`.
 */
int fpb_ivf_append(int device, int64_t n_cells, const int64_t* d_ivf_offsets, const int32_t* d_ivf_pids,
                   int64_t n_old_docs, int64_t n_new_docs, const int64_t* d_new_offsets, const int32_t* d_new_codes,
                   int64_t* d_out_offsets, int32_t* d_out_pids, int64_t out_capacity, int64_t* h_n_ivf,
                   void* stream);

/*
 * Deleting documents -- replaces `delete_from_index`'s filtering and renumbering (rust/index/delete.rs:26-145) on the
 * device.  Both entry points take the dropped ids as d_drop (i32 [n_drop], sorted, unique, in [0, n_docs); ids out of
 * order or out of range are refused before any row is written).  Kept documents keep their order; a kept document's
 * new id is its old id minus the number of dropped ids below it.  The inputs are only read, so a handle over them
 * stays valid.  Bad sizes and NULL pointers are refused before any CUDA call.  Synchronous on `stream`.
 *
 * fpb_docs_compact -- the kept documents of an index of n_docs documents (d_doc_offsets i64 [n_docs + 1]): writes
 * their offsets to d_out_offsets (i64 [n_docs - n_drop + 1], from 0) and sets *h_n_tokens to their token count.
 * Unless d_out_codes is NULL (a call that sizes the output), also copies their codes (i32), residual rows (u8, pd =
 * 16, 32 or 64 bytes each, 16-byte aligned arrays) and, when both norm pointers are non-NULL, token norms (f16) into
 * the out arrays (room for out_capacity tokens).  fpb_index_create on the compacted arrays computes the norms itself.
 *
 * fpb_ivf_delete -- the inverted file of the kept documents from the old one (d_ivf_offsets i64 [n_cells + 1] into
 * d_ivf_pids): every cell's postings of kept documents, renumbered, in their order.  Writes d_out_offsets (i64
 * [n_cells + 1]), sets *h_n_ivf to the number of postings and, unless d_out_pids is NULL (a call that sizes the
 * output), writes them to d_out_pids (i32, room for out_capacity ids).  Equal to building the inverted file of the
 * kept documents from scratch.
 */
int fpb_docs_compact(int device, int64_t n_docs, const int64_t* d_doc_offsets, const int32_t* d_doc_codes,
                     const uint8_t* d_doc_residuals, const void* d_token_norms, int pd, const int32_t* d_drop,
                     int64_t n_drop, int64_t* d_out_offsets, int32_t* d_out_codes, uint8_t* d_out_residuals,
                     void* d_out_norms, int64_t out_capacity, int64_t* h_n_tokens, void* stream);
int fpb_ivf_delete(int device, int64_t n_cells, const int64_t* d_ivf_offsets, const int32_t* d_ivf_pids,
                   int64_t n_docs, const int32_t* d_drop, int64_t n_drop, int64_t* d_out_offsets, int32_t* d_out_pids,
                   int64_t out_capacity, int64_t* h_n_ivf, void* stream);

/* Search parameters -- mirrors `SearchParameters` (rust/search/search.rs:171-200).
 * `batch_size` (document batch of the approximate stage) only bounds memory in the
 * reference and does not change values (search.rs:558-586); it is accepted and ignored. */
typedef struct fpb_params {
  int32_t n_ivf_probe;   /* search.rs:185, default 8; 1..4096 (n >= K probes every centroid) */
  int32_t n_full_scores; /* search.rs:179, default 4096 */
  int32_t top_k;         /* search.rs:182               */
  int32_t batch_size;    /* search.rs:176, ignored      */
  int32_t flags;         /* FPB_FLAG_*                  */
} fpb_params;

/* The workspace carries the per-query subset structures (search.rs:494-517, :544-547). */
#define FPB_FLAG_SUBSET 1
/* Approximate stage (search.rs:554-592).  By default it is computed in two exact passes: a bound pass
 * that gathers only the score rows of "high" centroids and yields, per candidate, an upper and a lower
 * bound of its approximate score (equal when the candidate is resolved), then an exact pass over the
 * unresolved candidates whose upper bound reaches the n_full_scores/4-th best lower bound.  Every
 * candidate that can enter the pruned list carries its exact score; the others keep an upper bound that
 * is strictly below the pruning threshold, so the pruned list, its scores and everything after it are
 * bit-identical to scoring every candidate.
 *   FPB_FLAG_APPROX_EXACT_ALL : also refine the candidates below the threshold (off_approx then holds
 *                               the exact score of EVERY candidate; parity tests)
 *   FPB_FLAG_APPROX_DIRECT    : one-pass scoring of every candidate (the A/B alternative)
 *   FPB_FLAG_APPROX_TWO_PASS  : two passes whatever the size of the job
 * With none of them the library picks: the two passes carry ~0.5 ms of fixed cost (threshold sample, bitmap,
 * refine list), so a call whose batch x index is too small to repay it (B * n_tokens < 2e8) is scored in one pass. */
#define FPB_FLAG_APPROX_EXACT_ALL 2
#define FPB_FLAG_APPROX_DIRECT 4
#define FPB_FLAG_APPROX_TWO_PASS 8

/* Byte offsets of every intermediate inside the workspace, so the parity tests can read
 * each stage (S, probed cells, candidates, approx scores, rerank list, exact scores)
 * exactly as the oracle dumps them.  All offsets are multiples of 256. */
typedef struct fpb_layout {
  int64_t total_bytes;
  int32_t B, Q, Qp, n_tiles, R, n_probe, cand_cap, bitmap_words;
  int32_t cbitmap_words, reserved0;
  int64_t off_queries;   /* f16 [B, Qp, D]  zero-padded queries                       */
  int64_t off_S;         /* f16 [B, K, Qp]  centroid scores          (search.rs:491)  */
  int64_t off_tmax;      /* f16 [B, Qp, n_tiles] per-128-centroid-tile column maxima  */
  int64_t off_cells;     /* i32 [B, Q, n_probe]  probed cells        (search.rs:520-528) */
  int64_t off_bitmap;    /* u32 [B, bitmap_words]                                     */
  int64_t off_n_cand;    /* i32 [B]                                                   */
  int64_t off_cand;      /* i32 [B, cand_cap] sorted unique doc ids  (search.rs:535-541) */
  int64_t off_approx;    /* f32 [B, cand_cap]                        (search.rs:554-592) */
  int64_t off_work;      /* i32 [B + 8] chunk prefix + counters                       */
  int64_t off_n_rerank;  /* i32 [B]                                                   */
  int64_t off_rerank;    /* i32 [B, R] doc ids, (approx desc, id asc) (search.rs:602-619) */
  int64_t off_rerank_approx; /* f32 [B, R]                                            */
  int64_t off_exact;     /* f32 [B, R]                               (search.rs:651-656) */
  /* only with FPB_FLAG_SUBSET (otherwise zero-sized): */
  int64_t off_cbitmap;   /* u32 [B, cbitmap_words] centroids present in the subset docs (search.rs:496-503) */
  int64_t off_clist;     /* i32 [B, K] the same as a sorted list                      */
  int64_t off_n_clist;   /* i32 [B]                                                   */
  int64_t off_sbitmap;   /* u32 [B, bitmap_words] the subset's documents              */
  /* two-pass approximate stage: */
  int64_t off_tau;       /* f16 [B, Qp]  per query token the "high" score threshold (+inf on padded columns) */
  int64_t off_hibits;    /* u32 [B, hb_words] centroid c is high: exists q with S[b,c,q] >= tau[b,q] */
  int64_t off_lb;        /* f32 [B, cand_cap] lower bound of the approximate score (== off_approx entry when resolved) */
  int64_t off_refine;    /* i32 [B, cand_cap] candidate indices re-scored exactly by the second pass */
  int64_t off_n_refine;  /* i32 [B]                                                   */
  int64_t off_thresh;    /* f32 [B] pruning threshold used by the second pass (-inf: refine all) */
  int64_t off_work2;     /* i32 [B + 8] chunk prefix + counter of the second pass     */
  int64_t off_stats;     /* u64 [8] counters: [0] rows gathered by the bound pass, [1] tokens walked by it,
                            [2] rows gathered by the exact pass (accumulated until the caller clears them) */
  int32_t hb_words, flags; /* flags = params->flags the layout was made for */
} fpb_layout;

/* Workspace sizing for a batch of B queries of Q tokens. */
int fpb_workspace_layout(const fpb_index* index, int B, int Q, const fpb_params* params,
                         fpb_layout* out);

/*
 * fpb_search_batch -- replaces `pysearch` -> `search_many` -> `search`
 * (rust/lib.rs:195-223, rust/search/search.rs:219-288, :471-696) for a whole batch.
 *
 *   d_queries     f16 [B, Q, dim]  (already cast to fp16, fast_plaid.py:241)
 *   d_out_ids     i64 [B, top_k]   global doc ids, rank order
 *   d_out_scores  f32 [B, top_k]
 *   d_out_counts  i32 [B]          min(top_k, #reranked)  (search.rs:666)
 * Unused tail entries are id -1 / score -inf.
 */
int fpb_search_batch(const fpb_index* index, const void* d_queries, int B, int Q,
                     const fpb_params* params, void* d_workspace, size_t workspace_bytes,
                     int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts,
                     void* stream);

/* Search restricted, per query, to a subset of documents (`subset=` of FastPlaid.search,
 * search.rs:494-517 + :544-547): probing is limited to the centroids that occur in the subset's
 * documents and the candidate set is intersected with the subset.
 *   d_subset_ids      i32 [total]  GLOBAL doc ids, query b owns [offsets[b], offsets[b+1])
 *   d_subset_offsets  i64 [B+1]
 *   max_subset_len    the largest per-query subset length (grid sizing)
 * params->flags must contain FPB_FLAG_SUBSET (it sizes the workspace). */
int fpb_search_batch_subset(const fpb_index* index, const void* d_queries, int B, int Q,
                            const fpb_params* params, const int32_t* d_subset_ids,
                            const int64_t* d_subset_offsets, int64_t max_subset_len, void* d_workspace,
                            size_t workspace_bytes, int64_t* d_out_ids, float* d_out_scores,
                            int32_t* d_out_counts, void* stream);

/* ---- Filters: one device form for every `subset=` form ----
 * A filter is a packed bitmap over GLOBAL document ids: row f of d_bitmap [n_filters, ceil(n_bits / 32)] uint32,
 * bit (id & 31) of word (id >> 5) set when document `id` is in filter f.  Ids >= n_bits are never set.
 *   fpb_filter_from_ids   d_ids i64 [n_ids], row f owning [d_row_offsets[f], d_row_offsets[f+1]) (device i64
 *                         [n_filters + 1]); any order, duplicates count once, ids outside [0, n_bits) and elements
 *                         outside every row are ignored.  The bitmap is cleared first.
 *   fpb_filter_from_mask  d_mask [n_filters, n_bits] bytes (bool / uint8, nonzero = set), one ballot per word.
 * Both refuse NULL pointers, n_filters < 1 and n_bits < 0 before any CUDA call; n_bits = 0 writes nothing. */
int fpb_filter_from_ids(int device, const int64_t* d_ids, int64_t n_ids, int n_filters, const int64_t* d_row_offsets,
                        int64_t n_bits, uint32_t* d_bitmap, void* stream);
int fpb_filter_from_mask(int device, const uint8_t* d_mask, int n_filters, int64_t n_bits, uint32_t* d_bitmap,
                         void* stream);

/* fpb_search_batch_subset with query b restricted to filter h_query_filter[b] (HOST i32 [B], each in
 * [0, n_filters); read during the call only) of d_filters [n_filters, ceil(n_bits / 32)].  The document bitmap and
 * the centroid bitmap of the subset stage are built once per distinct filter and copied to the other queries of
 * that filter; everything after them is the subset search's.  For the same documents the result is the bytes of
 * fpb_search_batch_subset.  params->flags must contain FPB_FLAG_SUBSET; the workspace is fpb_workspace_layout's.
 * NULL pointers, n_filters outside [1, 65535], n_bits < 0, a map entry out of range and a missing FPB_FLAG_SUBSET are
 * refused before any CUDA call. */
int fpb_search_batch_filter(const fpb_index* index, const void* d_queries, int B, int Q, const fpb_params* params,
                            const uint32_t* d_filters, int n_filters, int64_t n_bits, const int32_t* h_query_filter,
                            void* d_workspace, size_t workspace_bytes, int64_t* d_out_ids, float* d_out_scores,
                            int32_t* d_out_counts, void* stream);

/* Same call with HOST buffers: H2D of the queries, the search, D2H of the results and a
 * stream synchronise all happen inside.  d_out_* are device scratch of the same shapes. */
int fpb_search_batch_host(const fpb_index* index, const void* h_queries, int B, int Q,
                          const fpb_params* params, void* d_workspace, size_t workspace_bytes,
                          void* d_queries_staging, int64_t* d_out_ids, float* d_out_scores,
                          int32_t* d_out_counts, int64_t* h_out_ids, float* h_out_scores,
                          int32_t* h_out_counts, void* stream);

/* ---- stage-level entry points (parity tests, roofline bench).  Each runs one stage of
 * search.rs on the workspace laid out by fpb_workspace_layout. ---- */
int fpb_stage_centroid_scores(const fpb_index*, const void* d_queries, int B, int Q,
                              const fpb_params*, void* d_workspace, size_t, void* stream); /* search.rs:491 */
int fpb_stage_subset(const fpb_index*, const int32_t* d_subset_ids, const int64_t* d_subset_offsets,
                     int64_t max_subset_len, int B, int Q, const fpb_params*, void* d_workspace, size_t,
                     void* stream); /* search.rs:496-503: run between centroid_scores and probe */
int fpb_stage_filter(const fpb_index*, const uint32_t* d_filters, int n_filters, int64_t n_bits,
                     const int32_t* h_query_filter, int B, int Q, const fpb_params*, void* d_workspace, size_t,
                     void* stream); /* the filter form of fpb_stage_subset (fpb_search_batch_filter) */
int fpb_stage_probe(const fpb_index*, int B, int Q, const fpb_params*, void* d_workspace,
                    size_t, void* stream); /* search.rs:520-532 */
int fpb_stage_candidates(const fpb_index*, int B, int Q, const fpb_params*, void* d_workspace,
                         size_t, void* stream); /* search.rs:535-541 */
int fpb_stage_approx(const fpb_index*, int B, int Q, const fpb_params*, void* d_workspace,
                     size_t, void* stream); /* search.rs:554-592 */
int fpb_stage_select(const fpb_index*, int B, int Q, const fpb_params*, void* d_workspace,
                     size_t, void* stream); /* search.rs:602-619 */
int fpb_stage_maxsim(const fpb_index*, int B, int Q, const fpb_params*, void* d_workspace,
                     size_t, void* stream); /* search.rs:626-656 (+ decompress :53-107) */
int fpb_stage_rank(const fpb_index*, int B, int Q, const fpb_params*, void* d_workspace,
                   size_t, int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts,
                   void* stream); /* search.rs:659-666 */

int fpb_stage_keys(const fpb_index*, int B, int Q, const fpb_params*, void* d_workspace, size_t,
                   uint64_t* d_keys, void* stream); /* sharded two-step mode: emit [B, R] approx keys */
int fpb_stage_records(const fpb_index*, int B, int Q, const fpb_params*, void* d_workspace, size_t,
                      struct fpb_record* d_records, void* stream); /* sharded mode: emit [B, R] records */
/* The exact grouped ranking of fpb_search_exhaustive over caller-given scores (tests): row b of d_scores [B, cols]
 * holds d_n[b] scores (d_n NULL: cols); entry p scores local document d_cand[b * cols + p] (d_cand NULL: p), which
 * must lie in [0, N).  d_gkeys: at least B * max_per_group * n_groups * 8 bytes of scratch.  A handle without groups
 * or a shard-grouped one, NULL pointers, B or cols below 1, top_k outside [1, 4096] and too little scratch are
 * refused before any CUDA call. */
int fpb_stage_group_rank(const fpb_index* grouped, const float* d_scores, const int32_t* d_cand, const int32_t* d_n,
                         int64_t cols, int B, int top_k, void* d_gkeys, size_t gkeys_bytes, int64_t* d_out_ids,
                         float* d_out_scores, int32_t* d_out_counts, void* stream);

/* ---- document-sharded search (new; the reference replicates the index and splits the
 * query list, fast_plaid.py:893-928).  Each rank runs fpb_search_shard on its shard and
 * emits R fixed-size records per query; the host all-gathers them (NCCL) and every rank
 * runs fpb_merge_shards, which re-applies the reference's GLOBAL pruning rule
 * (top n_full_scores/4 by approximate score, search.rs:605-619) before the final sort.
 * The merge sorts a query's n_shards*R records in shared memory: n_shards*R <= 16384 (e.g. 4 shards at
 * n_full_scores = 16384, 8 at 8192), FPB_ERR_UNSUPPORTED above.  fpb_shard_apply_threshold has the same limit. */
struct fpb_record {
  float approx;   /* -inf for padding */
  float exact;
  int64_t doc_id; /* global id, -1 for padding */
};
typedef struct fpb_record fpb_record;

int fpb_search_shard(const fpb_index* index, const void* d_queries, int B, int Q,
                     const fpb_params* params, void* d_workspace, size_t workspace_bytes,
                     fpb_record* d_records /* [B, R] */, void* stream);
int fpb_merge_shards(const fpb_record* d_all_records /* [n_shards, B, R] */, int n_shards,
                     int B, int R, int top_k, int64_t* d_out_ids, float* d_out_scores,
                     int32_t* d_out_counts, void* stream);

/* Two-step variant (exact-scores only the documents that survive the GLOBAL pruning, so the
 * MaxSim work divides by the number of shards):
 *   1. fpb_shard_approx_keys : stages up to the local pruning; emits [B, R] 64-bit keys
 *                              (approx score, then smaller global id first; 0 = padding)
 *   2. all-gather of the keys; fpb_shard_apply_threshold finds, per query, the R-th best key of
 *      the whole index and shrinks this shard's re-rank list to the entries at or above it
 *   3. fpb_shard_exact_records : MaxSim on the shrunk lists, emits [B, R] fpb_record
 *   4. all-gather of the records; fpb_merge_shards ranks them. */
int fpb_shard_approx_keys(const fpb_index* index, const void* d_queries, int B, int Q,
                          const fpb_params* params, void* d_workspace, size_t workspace_bytes,
                          uint64_t* d_keys /* [B, R] */, void* stream);
/* Step 1 with a `subset` (search.rs:493-515, :544-551).  The reference restricts probing to the centroids
 * that the subset documents touch; with the documents sharded that set is the UNION over the shards:
 *   1a. fpb_shard_subset_begin : centroid scores + this shard's document bitmap and centroid bitmap;
 *                                copies the centroid bitmap ([B, layout.cbitmap_words] uint32) out
 *   1b. all-gather of the bitmaps; fpb_shard_subset_keys ORs them, probes, and continues like
 *       fpb_shard_approx_keys.  Subset ids are GLOBAL document ids (ids outside this shard are ignored).
 * params->flags must contain FPB_FLAG_SUBSET in both calls and in the later steps' layout. */
int fpb_shard_subset_begin(const fpb_index* index, const void* d_queries, int B, int Q,
                           const fpb_params* params, const int32_t* d_subset_ids,
                           const int64_t* d_subset_offsets, int64_t max_subset_len, void* d_workspace,
                           size_t workspace_bytes, uint32_t* d_cbitmap_out, void* stream);
/* 1a with filters (fpb_search_batch_filter's arguments): each shard expands only its own range
 * [doc_id_base, doc_id_base + n_docs) of the global bitmaps.  Then 1b and the later steps as above. */
int fpb_shard_filter_begin(const fpb_index* index, const void* d_queries, int B, int Q, const fpb_params* params,
                           const uint32_t* d_filters, int n_filters, int64_t n_bits, const int32_t* h_query_filter,
                           void* d_workspace, size_t workspace_bytes, uint32_t* d_cbitmap_out, void* stream);
int fpb_shard_subset_keys(const fpb_index* index, int B, int Q, const fpb_params* params, void* d_workspace,
                          size_t workspace_bytes, const uint32_t* d_all_cbitmaps /* [n_shards, B, words] */,
                          int n_shards, uint64_t* d_keys /* [B, R] */, void* stream);
int fpb_shard_apply_threshold(const fpb_index* index, const uint64_t* d_all_keys /* [n_shards, B, R] */,
                              int n_shards, int shard_rank, int B, int Q, const fpb_params* params,
                              void* d_workspace, size_t workspace_bytes, void* stream);
int fpb_shard_exact_records(const fpb_index* index, int B, int Q, const fpb_params* params,
                            void* d_workspace, size_t workspace_bytes, fpb_record* d_records, void* stream);

/* ---- the same exchange below the C ABI (SURVEY.md 8e: fpb_comm_init / fpb_search_batch_sharded) ----
 * An fpb_comm wraps one NCCL communicator (libnccl.so.2 is resolved at run time; without it these calls
 * return FPB_ERR_UNSUPPORTED and everything else keeps working).  Rank 0 makes the id with
 * fpb_comm_unique_id, the host distributes the FPB_COMM_ID_BYTES bytes by whatever means it has, every
 * rank calls fpb_comm_create (collective).
 *
 * fpb_search_batch_sharded searches the WHOLE batch on a grid of  n_query_groups x (nranks/n_query_groups)
 * document shards: rank r holds document shard r % n_shards (contiguous range, `doc_id_base` of its index)
 * and searches the queries of group r / n_shards (B split into n_query_groups contiguous slices).  Both
 * ncclAllGather calls (approximate-score keys, then the records of the globally surviving documents) are
 * issued on `stream` from inside the call; every rank returns the result of every query.
 *   d_queries  f16 [B, Q, dim]  the same batch on every rank
 *   d_ws       workspace of fpb_workspace_layout(index, ceil(B / n_query_groups), Q, params)
 *   d_scratch  fpb_sharded_scratch_bytes(ceil(B / n_query_groups), n_full_scores / 4, nranks) bytes
 * The merge limit of fpb_merge_shards applies with n_shards = nranks / n_query_groups; a search above it
 * returns FPB_ERR_UNSUPPORTED on every rank before the first all-gather. */
#define FPB_COMM_ID_BYTES 128
typedef struct fpb_comm fpb_comm;
int fpb_comm_unique_id(void* out_id /* FPB_COMM_ID_BYTES */);
int fpb_comm_create(fpb_comm** out, int nranks, int rank, const void* unique_id, int device);
void fpb_comm_destroy(fpb_comm* comm);
int fpb_comm_nccl_version(void); /* 0 when NCCL is not loadable */
int64_t fpb_sharded_scratch_bytes(int b_local, int R, int nranks);
int fpb_search_batch_sharded(const fpb_index* index, fpb_comm* comm, int n_query_groups, const void* d_queries,
                             int B, int Q, const fpb_params* params, void* d_workspace, size_t workspace_bytes,
                             void* d_scratch, size_t scratch_bytes, int64_t* d_out_ids, float* d_out_scores,
                             int32_t* d_out_counts, void* stream);
/* The same with HOST buffers (H2D of the queries, D2H of the results, stream synchronise inside). */
int fpb_search_batch_sharded_host(const fpb_index* index, fpb_comm* comm, int n_query_groups, const void* h_queries,
                                  int B, int Q, const fpb_params* params, void* d_workspace, size_t workspace_bytes,
                                  void* d_scratch, size_t scratch_bytes, void* d_queries_staging, int64_t* d_out_ids,
                                  float* d_out_scores, int32_t* d_out_counts, int64_t* h_out_ids, float* h_out_scores,
                                  int32_t* h_out_counts, void* stream);

/* ---- exhaustive exact search (new; the reference has no such mode) ----
 * Scores EVERY local document against every query with the exact MaxSim formula of the re-rank stage
 * (search.rs:626-656: same decoder, same fp16 rounding of each token score, an empty document scores
 * Q * -10000), then ranks them.  No IVF is read, so a compress_only index can be searched this way.
 * One rounding point differs: the sum over the Q query tokens is the EXACT sum of the fp16 maxima, rounded once
 * to fp32, where the re-rank stage keeps an fp32 running sum.  The two agree whenever that running sum is exact
 * (the usual case); otherwise a document's score from fpb_search_batch and from these calls can differ in the
 * last bit.  The exact sum is what makes the result independent of the order of the work.
 *   fpb_exhaustive_workspace_bytes : workspace of fpb_search_exhaustive for B queries of Q <= 256 tokens and
 *                                    1 <= top_k <= 4096 (FPB_ERR_UNSUPPORTED above), or with top_k = 0 of
 *                                    fpb_exhaustive_scores alone; 256-byte aligned
 *   fpb_exhaustive_scores  d_queries f16 [B, Q, dim] (16-byte aligned), d_scores f32 [B, n_docs] (local ids)
 *   fpb_search_exhaustive  outputs as fpb_search_batch: global ids in rank order (score desc, then id asc),
 *                          d_out_counts[b] = min(top_k, n_docs), unused tail entries id -1 / score -inf
 * Every (dim, nbits) that fpb_index_create accepts is searched, nbits 1 at dim 128 included.
 * Deterministic: the same inputs give the same bytes, whatever B and however a batch is split into calls. */
int fpb_exhaustive_workspace_bytes(const fpb_index* index, int B, int Q, int top_k, size_t* out);
int fpb_exhaustive_scores(const fpb_index* index, const void* d_queries, int B, int Q, void* d_workspace,
                          size_t workspace_bytes, float* d_scores, void* stream);
int fpb_search_exhaustive(const fpb_index* index, const void* d_queries, int B, int Q, int top_k, void* d_workspace,
                          size_t workspace_bytes, int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts,
                          void* stream);

/* Exhaustive exact search over document lists: query b is scored against the documents of list h_query_list[b]
 * only (filtered exact search, exact re-ranking of a candidate list).  Queries that share a list share one decode
 * of each of its documents.
 *   d_list_ids      i32 [total]  GLOBAL doc ids, list l owns [d_list_offsets[l], d_list_offsets[l+1]); any order,
 *                                duplicates count once, ids outside [doc_id_base, doc_id_base + n_docs) are ignored
 *                                (the convention of fpb_search_batch_subset)
 *   d_list_offsets  i64 [n_lists + 1]
 *   max_list_len    at least the length of every list (it sizes the workspace: min(n_docs, max_list_len) positions
 *                   per list; like max_subset_len)
 *   h_query_list    HOST i32 [B], the list of every query, each in [0, n_lists); read during the call only
 * Outputs as fpb_search_exhaustive, over the SET of valid documents of the query's list: global ids in rank order
 * (score desc, then id asc), d_out_counts[b] = min(top_k, set size) (0 for an empty list), tails id -1 / score -inf.
 * Every score is bit-identical to fpb_exhaustive_scores' score of the same document: the same decoder, MMA sequence
 * and exact sum.  The result does not depend on how queries are grouped into lists or on how a batch is split.
 * Limits as fpb_exhaustive_workspace_bytes (1 <= top_k <= 4096, Q <= 256); 1 <= n_lists <= 65535.  The arguments
 * are checked in the order shapes, lists, index.  fpb_exhaustive_subset_workspace_bytes: the workspace (256-byte
 * aligned) of a call with these shapes and lists. */
int fpb_exhaustive_subset_workspace_bytes(const fpb_index* index, int B, int Q, int top_k, int n_lists,
                                          int64_t max_list_len, size_t* out);
int fpb_search_exhaustive_subset(const fpb_index* index, const void* d_queries, int B, int Q, int top_k,
                                 const int32_t* d_list_ids, const int64_t* d_list_offsets, int n_lists,
                                 int64_t max_list_len, const int32_t* h_query_list, void* d_workspace,
                                 size_t workspace_bytes, int64_t* d_out_ids, float* d_out_scores,
                                 int32_t* d_out_counts, void* stream);

/* fpb_search_exhaustive_subset with filters (fpb_search_batch_filter's d_filters / n_filters / n_bits /
 * h_query_filter): list l is this index's range of filter l, so every query of a filter shares one decode of its
 * documents.  max_count bounds the set documents of every filter inside [doc_id_base, doc_id_base + n_docs): it
 * sizes the workspace like max_list_len.  A filter with more documents in the range than max_count is cut to its
 * first max_count of them (in id order), so its queries are ranked among those only: pass the exact maximum (or
 * more) for the full result.
 * Results and limits are those of fpb_search_exhaustive_subset (n_filters <= 65535).
 * fpb_exhaustive_filter_workspace_bytes: the workspace of a call with these shapes and filters. */
int fpb_exhaustive_filter_workspace_bytes(const fpb_index* index, int B, int Q, int top_k, int n_filters,
                                          int64_t max_count, size_t* out);
int fpb_search_exhaustive_filter(const fpb_index* index, const void* d_queries, int B, int Q, int top_k,
                                 const uint32_t* d_filters, int n_filters, int64_t n_bits, int64_t max_count,
                                 const int32_t* h_query_filter, void* d_workspace, size_t workspace_bytes,
                                 int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts, void* stream);

/* Exhaustive search on a document-sharded index: the result of fpb_search_exhaustive on one GPU holding the whole
 * index, byte for byte (global ids in rank order, counts = min(top_k, total documents), tails id -1 / score -inf).
 * K7's scores do not depend on how the documents are split, so only the top-k lists have to be combined.
 *   fpb_shard_exhaustive_records : the step-wise form.  Runs fpb_search_exhaustive's scan and selection on this
 *       shard and writes, per query, one fpb_record per selected document (approx = exact = its score, global id
 *       doc_id_base + local id), then padding records (-inf, -inf, -1) up to top_k.  d_records [B, top_k];
 *       workspace of fpb_exhaustive_workspace_bytes(index, B, Q, top_k).  The shards' records, all-gathered to
 *       [n_shards, B, top_k], go to fpb_merge_shards(..., n_shards, B, R = top_k, top_k, ...): with approx equal
 *       to exact, its "keep the R best by approx, order them by exact" is the global top_k.
 *   fpb_search_exhaustive_sharded : the whole exchange in one call on `stream`, on the grid of
 *       fpb_search_batch_sharded (rank r holds document shard r % n_shards and searches the queries of group
 *       r / n_shards); one ncclAllGather of [ceil(B / n_query_groups), top_k] records, then every rank merges every
 *       query.  Collective: every rank passes the same batch and gets every query's result.
 *         d_ws       fpb_exhaustive_workspace_bytes(index, ceil(B / n_query_groups), Q, top_k) bytes
 *         d_scratch  fpb_sharded_scratch_bytes(ceil(B / n_query_groups), top_k, nranks) bytes
 * Limits: those of fpb_search_exhaustive (1 <= top_k <= 4096, Q <= 256) and the merge limit of fpb_merge_shards,
 * n_shards * top_k <= 16384 with n_shards = nranks / n_query_groups.  fpb_search_exhaustive_sharded refuses a call
 * outside them, NULL arguments and a query-group count that does not divide the ranks on every rank before the
 * all-gather, with the shapes checked first. */
int fpb_shard_exhaustive_records(const fpb_index* index, const void* d_queries, int B, int Q, int top_k,
                                 void* d_workspace, size_t workspace_bytes, fpb_record* d_records /* [B, top_k] */,
                                 void* stream);
int fpb_search_exhaustive_sharded(const fpb_index* index, fpb_comm* comm, int n_query_groups, const void* d_queries,
                                  int B, int Q, int top_k, void* d_workspace, size_t workspace_bytes, void* d_scratch,
                                  size_t scratch_bytes, int64_t* d_out_ids, float* d_out_scores,
                                  int32_t* d_out_counts, void* stream);

/* Grouped results on a document-sharded index: the bytes that fpb_index_with_groups_max gives on one GPU holding the
 * whole index, at every shard count and query-group grid.
 *   fpb_index_with_shard_groups -- a shard-grouped handle over `index` (one shard, documents [doc_id_base,
 *       doc_id_base + n_docs) of an index of n_total_docs): d_doc_group (i32 [n_docs]) is the group of each local
 *       document, dense in [0, n_groups); d_global_group (i32 [n_total_docs]) is the group of every document of the
 *       WHOLE index by global id, the same map on every rank (its ids need not match d_doc_group's: only which
 *       documents share a group matters).  Both are borrowed, like fpb_index_with_groups' array.  Accepted by:
 *         - fpb_search_batch_sharded and _host: the local stages run ungrouped and the final merge applies the rule
 *           to the n_full_scores / 4 documents it keeps, as fpb_search_batch does on one GPU;
 *         - fpb_shard_exhaustive_records: this shard's top_k under the rule (exact, by the local map), one record per
 *           result (approx = exact = score), then padding records (-inf, -inf, -1);
 *         - fpb_search_exhaustive_sharded: those records, one all-gather, then the grouped merge of all of them.
 *       fpb_exhaustive_workspace_bytes on it adds the group keys (as on a grouped handle) and B * top_k i64.  Every
 *       other entry point returns FPB_ERR_UNSUPPORTED on it; the step-wise approximate steps (fpb_shard_*) take the
 *       plain handle and group only in fpb_merge_shards_grouped.  Handles of fpb_index_with_groups(_max) stay refused
 *       by the sharded entry points: they carry no map of the whole index.
 *   fpb_merge_shards_grouped -- the step-wise merge: fpb_merge_shards' records [n_shards, B, R], of which the n_keep
 *       best by approx are kept (n_keep = R for the approximate search, n_shards * R for the exhaustive records, whose
 *       approx is their exact score), ordered by exact, then at most max_per_group documents per group kept by
 *       d_global_group, the first top_k of them written as fpb_merge_shards writes its ranking.  A record whose id is
 *       outside [0, n_total_docs) or whose group is negative is skipped.  Its shared memory is 11 bytes per record
 *       slot (180 KB at the merge limit); it needs no scratch.
 * Exact search stays exact: each shard sends the first top_k documents it keeps under the rule, and every document
 * the rule keeps on the whole index is among its shard's first top_k (DESIGN §7).  Both calls refuse NULL pointers,
 * n_groups or n_total_docs outside [1, INT32_MAX], max_per_group outside [1, FPB_MAX_PER_GROUP] and n_keep outside
 * [1, n_shards * R] with FPB_ERR_INVALID before any CUDA call, and the merge limit of fpb_merge_shards with
 * FPB_ERR_UNSUPPORTED (the sharded entry points on every rank before the first all-gather).  fpb_index_with_shard_groups
 * also refuses an n_total_docs below the end of the shard's range. */
int fpb_index_with_shard_groups(fpb_index** out, const fpb_index* index, const int32_t* d_doc_group, int64_t n_groups,
                                int max_per_group, const int32_t* d_global_group, int64_t n_total_docs);
int fpb_merge_shards_grouped(const fpb_record* d_all_records /* [n_shards, B, R] */, int n_shards, int B, int R,
                             int n_keep, int top_k, const int32_t* d_global_group, int64_t n_total_docs,
                             int max_per_group, int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts,
                             void* stream);

/* ---- by-products of the MaxSim kernel ("next" rows of SURVEY.md 8f-3) ---- */
/* reconstruct_embeddings (rust/utils/embeddings.rs:12-69): decompressed, normalised
 * fp16 rows of the given local docs, concatenated.  d_out: f16 [sum(len), dim]. */
int fpb_reconstruct(const fpb_index* index, const int32_t* d_doc_ids, int n, const int64_t* d_out_offsets,
                    void* d_out, void* stream);
/* token matrices of search_many_with_token_scores (search.rs:668-686):
 * d_out f16 [n, max_len, Q] row t = doc token, col = query token, for n (query, doc) pairs. */
int fpb_token_scores(const fpb_index* index, const void* d_queries, int Q, const int32_t* d_query_of,
                     const int32_t* d_doc_ids, int n, int64_t max_len, void* d_out, void* stream);

/* ---- index build: the encode step of create_index (rust/index/create.rs:404-428) ----
 * codes[t] = argmax_k fp16(<x_t, c_k>) (compress_into_codes, create.rs:148-170; ties -> smallest k),
 * residuals[t] = packed bucket indices of fp16(x_t - c[codes[t]]) against `cutoffs`
 * (bucketize right=false + LSB-first bits + big-endian packbits, create.rs:413-427, :176-184).
 *   d_tokens f16 [n_tokens, dim], d_centroids f16 [n_centroids, dim], d_cutoffs f32 [(1<<nbits)-1]
 *   d_codes i32 [n_tokens], d_residuals u8 [n_tokens, dim*nbits/8]
 * fpb_encode takes dim 128 with nbits 1, 2 or 4 and refuses anything else with FPB_ERR_UNSUPPORTED before any
 * CUDA call. */
/* Host utility: round-to-nearest-even fp32 -> fp16 cast of a query batch (the cast search_on_device does
 * on the host, fast_plaid.py:241), single-threaded with F16C.  The _portable variant is the same
 * conversion in plain C, exported so the tests can compare the two. */
int fpb_cast_f32_to_f16_host(const float* h_src, void* h_dst, size_t n);
int fpb_cast_f32_to_f16_host_portable(const float* h_src, void* h_dst, size_t n);

int fpb_encode(int device, int nbits, int dim, int64_t n_centroids, const void* d_centroids,
               const void* d_tokens, int64_t n_tokens, const float* d_cutoffs, int32_t* d_codes,
               uint8_t* d_residuals, void* stream);

/* ---- index build: Lloyd iterations of the centroid k-means (python/fast_plaid/search/kmeans.py:60-223) ----
 * fpb_kmeans_assign : assign[i] = argmax_k (<x_i, c_k> + bias[k]) in fp32 on the tensor cores; with
 *                     bias[k] = -|c_k|^2 / 2 that is the nearest centroid by squared distance (kmeans.py:153-160);
 *                     ties -> smallest k.   d_points f16 [n, 128], d_centroids f16 [K, 128], d_bias f32 [K]
 * fpb_kmeans_update : centroid k <- mean of its points, as a deterministic segmented sum: d_order i64 [n] = point
 *                     indices sorted by assignment, d_seg_offsets i64 [K+1]; empty segments are left untouched
 *                     (the caller re-seeds them, kmeans.py:196-205); d_shift f32 [K] (optional) receives
 *                     |new - old| per centroid for the convergence test */
int fpb_kmeans_assign(int device, int dim, int64_t n_centroids, const void* d_centroids, const float* d_bias,
                      const void* d_points, int64_t n_points, int32_t* d_assign, void* stream);
int fpb_kmeans_update(int device, int dim, int64_t n_centroids, const void* d_points, const int64_t* d_order,
                      const int64_t* d_seg_offsets, void* d_centroids, float* d_shift, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FASTPLAID_B200_H_ */
