// Grouped results (DESIGN §7): each query returns at most m documents per group, the group's m best under the
// canonical order (score desc, then id asc), and these in the canonical order.  A handle made by
// fpb_index_with_groups(_max) carries the group of every local document, dense ids in [0, n_groups), and m.
//   - The re-ranked list of a search (<= 4096 documents per query): K6's canonical sort, then the first m entries of
//     each group, kept in rank order (k6_rank_grouped_kernel).
//   - Exact search: the maximum canonical key of every (query, group) pair over the exact scores (group_max_kernel),
//     then the top_k largest of those keys per query (group_select_kernel).  The maximum key is the group's
//     canonical best document, and a maximum does not depend on the order of the atomics.  At m > 1, m rounds of
//     the maximum (group_round_max_kernel), round r bounded by round r - 1's key, give the m best keys of every
//     group, and the selection runs over all m * n_groups of them.
//   - A document-sharded index (fpb_index_with_shard_groups, DESIGN §7): each shard's exact search selects its own
//     top_k under the rule, and the merge across ranks (k6_merge_grouped_kernel) applies the rule again to the union
//     with the group map of the whole index; the approximate search merges ungrouped records the same way.
// A group id outside [0, n_groups) is skipped: the host remap never makes one, but the C ABI is public.
#include "kernels.h"
#include "select.cuh"

namespace {

__device__ __forceinline__ bool group_ok(int32_t g, int64_t n_groups) { return g >= 0 && int64_t(g) < n_groups; }

// Grouped K6, one CTA per query: row b of exact / rerank (stride R) holds the scores and local ids of n_rerank[b]
// documents, of which the first m of each group in the canonical order are kept (ONE: the instance for m = 1, which
// ignores m).  Shared memory: the canonical keys [Rp2], then gkeys [Rp2], the group rule's (group, rank position)
// keys and then the kept keys in rank order.
template <bool ONE>
__global__ void __launch_bounds__(1024)
k6_rank_grouped_kernel(const float* __restrict__ exact, const int32_t* __restrict__ rerank,
                       const int32_t* __restrict__ n_rerank, int R, int Rp2, int top_k, int64_t doc_id_base,
                       const int32_t* __restrict__ doc_group, int64_t n_groups, int64_t* __restrict__ out_ids,
                       float* __restrict__ out_scores, int32_t* __restrict__ out_counts, int m) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint64_t* keys = reinterpret_cast<uint64_t*>(smem_raw);
  uint64_t* gkeys = keys + Rp2;
  __shared__ unsigned char kept[FPB_EX_MAX_TOP_K];  // kept[i]: rank position i is among its group's m best
  const int b = blockIdx.x;
  const int n = n_rerank[b];
  // the canonical order of the re-ranked documents (a document of no valid group is left out)
  for (int i = threadIdx.x; i < Rp2; i += 1024) {
    uint64_t k = 0;
    if (i < n) {
      const int32_t d = rerank[int64_t(b) * R + i];
      if (group_ok(doc_group[d], n_groups)) k = rank_key_f32(exact[int64_t(b) * R + i], uint32_t(d));
    }
    keys[i] = k;
  }
  __syncthreads();
  block_sort_desc(keys, Rp2);
  const int cnt = block_group_rule(
      keys, Rp2, ONE ? 1 : m, [&](int i) { return doc_group[rank_key_id(keys[i])]; }, [&](int i) { return keys[i]; },
      gkeys, kept);
  block_write_ranking(gkeys, cnt, top_k, doc_id_base, out_ids, out_scores, out_counts, b);
}

// The group maximum of exact search.  Row b of `scores` (stride cols) holds n[b] scores (n == NULL: all cols), entry p
// scoring local document cand[b * cols + p] (cand == NULL: p).  gkeys (rows of stride row_stride, zeroed) receives
// at b * row_stride + g, per (query, group), the largest rank_key_f32(score, document); with a `bound` (same layout),
// the largest below bound[b * row_stride + g], so a group whose bound is 0 is skipped.  A thread reduces GM_PER
// consecutive entries run by run (one atomic per run of one group), and the warp combines the lanes whose last runs
// share a group, so one group or long runs of one group cost one atomic per warp and pass.
constexpr int GM_PER = 8;
__device__ __forceinline__ void group_max(const float* __restrict__ scores, const int32_t* __restrict__ cand,
                                          const int32_t* __restrict__ n, int64_t cols, int B,
                                          const int32_t* __restrict__ doc_group, int64_t n_groups, int64_t row_stride,
                                          const unsigned long long* __restrict__ bound,
                                          unsigned long long* __restrict__ gkeys) {
  const int lane = threadIdx.x & 31;
  const int64_t runs = (cols + GM_PER - 1) / GM_PER, total = int64_t(B) * runs;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;  // a multiple of 32: whole warps iterate together
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i - lane < total; i += stride) {
    int64_t b = 0, p0 = 0, len = 0;
    if (i < total) {
      b = i / runs;
      p0 = (i % runs) * GM_PER;
      len = n ? n[b] : cols;
    }
    uint64_t best = 0, lim = 0;
    int64_t g_cur = -1, g_lim = -1;
#pragma unroll
    for (int u = 0; u < GM_PER; ++u) {
      const int64_t p = p0 + u;
      if (p < len) {
        const int32_t d = cand ? cand[b * cols + p] : int32_t(p);
        const int32_t g = doc_group[d];
        if (group_ok(g, n_groups)) {
          const uint64_t k = rank_key_f32(scores[b * cols + p], uint32_t(d));
          if (bound) {  // one load per run: the bound is the (query, group)'s
            if (g != g_lim) {
              g_lim = g;
              lim = bound[b * row_stride + g];
            }
            if (k >= lim) continue;
          }
          if (g != g_cur) {
            if (best) atomicMax(&gkeys[b * row_stride + g_cur], (unsigned long long)best);
            g_cur = g;
            best = k;
          } else if (k > best) {
            best = k;
          }
        }
      }
    }
    const unsigned long long slot = best ? (unsigned long long)(b * row_stride + g_cur) : ~0ull;
    const unsigned peers = __match_any_sync(0xffffffffu, slot);
    const uint32_t hi = __reduce_max_sync(peers, uint32_t(best >> 32));
    const uint32_t lo = __reduce_max_sync(peers, uint32_t(best >> 32) == hi ? uint32_t(best) : 0u);
    if (best && lane == __ffs(peers) - 1) atomicMax(&gkeys[slot], (unsigned long long)((uint64_t(hi) << 32) | lo));
  }
}

// gkeys [B, n_groups]: each group's best
__global__ void __launch_bounds__(256)
group_max_kernel(const float* __restrict__ scores, const int32_t* __restrict__ cand, const int32_t* __restrict__ n,
                 int64_t cols, int B, const int32_t* __restrict__ doc_group, int64_t n_groups,
                 unsigned long long* __restrict__ gkeys) {
  group_max(scores, cand, n, cols, B, doc_group, n_groups, n_groups, nullptr, gkeys);
}

// One round of the m best keys per group: rows of stride m * n_groups, bound NULL in the first round, else the
// previous round's keys
__global__ void __launch_bounds__(256)
group_round_max_kernel(const float* __restrict__ scores, const int32_t* __restrict__ cand,
                       const int32_t* __restrict__ n, int64_t cols, int B, const int32_t* __restrict__ doc_group,
                       int64_t n_groups, int64_t row_stride, const unsigned long long* __restrict__ bound,
                       unsigned long long* __restrict__ gkeys) {
  group_max(scores, cand, n, cols, B, doc_group, n_groups, row_stride, bound, gkeys);
}

// group_select's entries: the keys of a gkeys row, 0 for an empty one
struct RowKeys {
  static constexpr bool dense = false;
  const unsigned long long* row;
  __device__ static uint64_t empty() { return 0; }
  __device__ uint64_t load(int64_t i) const { return row[i]; }
  __device__ bool present(uint64_t k) const { return k != 0; }
  __device__ float value(uint64_t k) const { return rank_key_f32_value(k); }
  __device__ uint64_t key(uint64_t k, int64_t) const { return k; }
};

// One CTA per query: the top_k largest non-empty keys of row b of gkeys [B, n_groups], in descending order, written
// as K6 writes its ranking.  The keys are distinct (each names its own document), so the top_k are the keys at or
// above the top_k-th.
__global__ void __launch_bounds__(1024)
group_select_kernel(const unsigned long long* __restrict__ gkeys, int64_t n_groups, int top_k, int Rp2,
                    int64_t doc_id_base, int64_t* __restrict__ out_ids, float* __restrict__ out_scores,
                    int32_t* __restrict__ out_counts) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint64_t* keys = reinterpret_cast<uint64_t*>(smem_raw);  // [Rp2]
  const int b = blockIdx.x;
  const int cnt = block_select_keys(RowKeys{gkeys + int64_t(b) * n_groups}, n_groups, top_k, keys, Rp2);
  block_write_ranking(keys, cnt, top_k, doc_id_base, out_ids, out_scores, out_counts, b);
}

// The grouped shard merge, one CTA per query, over the gathered records in k6_merge_kernel's layout
// ([query group][n_shards, B, R]).  It is k6_merge_kernel followed by grouped K6's rule:
//   1. keep the n_keep best records by (approx desc, id asc) -- skipped when n_keep covers every record;
//   2. order them by (exact desc, id asc);
//   3. keep sorted position i when fewer than m documents of its group come before it (global_group by global id);
//   4. write the first top_k kept ones.
// Shared memory, 11 bytes per record slot (180 KB at the merge limit): keys [P] (the approximate keys, then the exact
// keys of the Kp2 = next_pow2(min(n_keep, total)) first slots, then the (group, position) keys, then the kept keys),
// pay [P] (the record index of each slot, carried through both sorts) and kept [P].  The kept keys are rebuilt from
// the records.
__global__ void __launch_bounds__(1024)
k6_merge_grouped_kernel(const fpb_record* __restrict__ all_groups, int n_shards, int B, int R, int P, int Kp2,
                        int n_keep, int top_k, const int32_t* __restrict__ global_group, int64_t n_total_docs, int m,
                        int64_t* __restrict__ out_ids, float* __restrict__ out_scores,
                        int32_t* __restrict__ out_counts) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint64_t* keys = reinterpret_cast<uint64_t*>(smem_raw);  // [P]
  uint16_t* pay = reinterpret_cast<uint16_t*>(keys + P);    // [P] record index (P <= 2^14)
  unsigned char* kept = reinterpret_cast<unsigned char*>(pay + P);  // [P]
  const int b = blockIdx.x % B;
  const fpb_record* all = all_groups + int64_t(blockIdx.x / B) * n_shards * B * R;
  const int total = n_shards * R;
  auto record = [&](int j) -> const fpb_record& { return merge_record(all, B, R, b, j); };
  // 1. the global pruning rule, as k6_merge_kernel applies it
  const bool prune = n_keep < total;
  const int cand = prune ? block_merge_prune(all, B, R, b, total, P, n_keep, keys, pay) : total;  // slots [0, cand)
  // 2. the canonical order of the candidates; a padding record, or one of no valid group, is left out
  for (int i = threadIdx.x; i < Kp2; i += 1024) {
    uint64_t k = 0;
    if (i < cand) {
      const int j = prune ? int(pay[i]) : i;
      const fpb_record rec = record(j);
      if (rec.doc_id >= 0 && rec.doc_id < n_total_docs && global_group[rec.doc_id] >= 0)
        k = rank_key_f32(rec.exact, uint32_t(rec.doc_id));
      pay[i] = uint16_t(j);
    }
    keys[i] = k;
  }
  __syncthreads();
  block_sort_desc(keys, Kp2, pay);
  // 3. the group rule, its (group, position) keys in place of the exact keys, which are read back from the records
  const int cnt = block_group_rule(
      keys, Kp2, m, [&](int i) { return global_group[record(pay[i]).doc_id]; },
      [&](int i) {
        const fpb_record rec = record(pay[i]);
        return rank_key_f32(rec.exact, uint32_t(rec.doc_id));  // the value K6 writes (-0 as +0)
      },
      keys, kept);
  block_write_ranking(keys, cnt, top_k, 0, out_ids, out_scores, out_counts, blockIdx.x);
}

__global__ void results_to_records_kernel(const int64_t* __restrict__ ids, const float* __restrict__ scores, int64_t n,
                                          fpb_record* __restrict__ rec) {
  const int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  fpb_record o;
  o.approx = scores[i];
  o.exact = scores[i];
  o.doc_id = ids[i];
  rec[i] = o;
}

}  // namespace

int launch_rank_grouped(const float* scores, const int32_t* ids, const int32_t* n, int R, int B, int top_k,
                        int64_t doc_id_base, const int32_t* doc_group, int64_t n_groups, int max_per_group,
                        int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts, cudaStream_t st) {
  const int Rp2 = fpb_next_pow2(R);
  const size_t smem = size_t(Rp2) * 16;  // 64 KB at R = 4096: opt in
  const bool one = max_per_group <= 1;
  const auto kernel = one ? k6_rank_grouped_kernel<true> : k6_rank_grouped_kernel<false>;
  FPB_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  kernel<<<B, 1024, smem, st>>>(scores, ids, n, R, Rp2, top_k, doc_id_base, doc_group, n_groups, d_out_ids,
                                d_out_scores, d_out_counts, max_per_group);
  FPB_LAUNCH_CHECK("k6_rank_grouped");
  return FPB_OK;
}

int launch_group_max(const float* scores, const int32_t* cand, const int32_t* n, int64_t cols, int B,
                     const int32_t* doc_group, int64_t n_groups, int max_per_group, uint64_t* gkeys, int sm_count,
                     cudaStream_t st) {
  const int m = max_per_group > 1 ? max_per_group : 1;
  FPB_CUDA_CHECK(cudaMemsetAsync(gkeys, 0, size_t(B) * m * n_groups * 8, st));
  const int64_t total = int64_t(B) * ((cols + GM_PER - 1) / GM_PER);
  const int grid = fpb_grid_for(total, 256, sm_count);
  auto* keys = reinterpret_cast<unsigned long long*>(gkeys);
  if (m == 1) {
    group_max_kernel<<<grid, 256, 0, st>>>(scores, cand, n, cols, B, doc_group, n_groups, keys);
    FPB_LAUNCH_CHECK("group_max");
    return FPB_OK;
  }
  // round r: each group's best key below its round r - 1 key, so after m rounds a row holds the m best keys of
  // every group (fewer, the rest 0, for a group of fewer documents)
  const int64_t stride = int64_t(m) * n_groups;
  for (int r = 0; r < m; ++r) {
    group_round_max_kernel<<<grid, 256, 0, st>>>(scores, cand, n, cols, B, doc_group, n_groups, stride,
                                                 r ? keys + (r - 1) * n_groups : nullptr, keys + r * n_groups);
    FPB_LAUNCH_CHECK("group_round_max");
  }
  return FPB_OK;
}

int launch_group_select(const uint64_t* gkeys, int64_t n_groups, int B, int top_k, int64_t doc_id_base,
                        int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts, cudaStream_t st) {
  const int Rp2 = fpb_next_pow2(top_k);
  // dynamic keys[] (32 KB at top_k = 4096) on top of 25 KB of static shared memory: opt in
  FPB_CUDA_CHECK(cudaFuncSetAttribute(group_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Rp2 * 8));
  group_select_kernel<<<B, 1024, size_t(Rp2) * 8, st>>>(reinterpret_cast<const unsigned long long*>(gkeys), n_groups,
                                                       top_k, Rp2, doc_id_base, d_out_ids, d_out_scores,
                                                       d_out_counts);
  FPB_LAUNCH_CHECK("group_select");
  return FPB_OK;
}

int launch_merge_grouped(const fpb_record* d_all_records, int n_shards, int b_stride, int n_queries, int R, int n_keep,
                         int top_k, const int32_t* global_group, int64_t n_total_docs, int max_per_group,
                         int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts, cudaStream_t stream) {
  const char* who = "fpb_merge_shards_grouped";
  if (!d_all_records || !global_group || !d_out_ids || !d_out_scores || !d_out_counts) {
    fpb_set_error("%s: NULL record, group or output pointer", who);
    return FPB_ERR_INVALID;
  }
  if (n_shards < 1 || b_stride < 1 || R < 1 || top_k < 1 || n_queries < 0) {
    fpb_set_error("%s: n_shards=%d B=%d R=%d top_k=%d must be >= 1", who, n_shards, b_stride, R, top_k);
    return FPB_ERR_INVALID;
  }
  if (n_total_docs < 1 || n_total_docs > INT32_MAX) {
    fpb_set_error("%s: n_total_docs=%lld must be in [1, %d]", who, (long long)n_total_docs, INT32_MAX);
    return FPB_ERR_INVALID;
  }
  if (max_per_group < 1 || max_per_group > FPB_MAX_PER_GROUP) {
    fpb_set_error("%s: max_per_group=%d must be in [1, %d]", who, max_per_group, FPB_MAX_PER_GROUP);
    return FPB_ERR_INVALID;
  }
  if (n_keep < 1 || int64_t(n_keep) > int64_t(n_shards) * R) {
    fpb_set_error("%s: n_keep=%d must be in [1, n_shards*R = %lld]", who, n_keep, (long long)(int64_t(n_shards) * R));
    return FPB_ERR_INVALID;
  }
  FPB_TRY(check_merge_records(who, n_shards, R));
  if (n_queries == 0) return FPB_OK;
  const int total = n_shards * R;
  const int P = fpb_next_pow2(total);
  const int Kp2 = fpb_next_pow2(n_keep < total ? n_keep : total);
  const size_t smem = size_t(P) * (8 + 2 + 1);  // keys, pay, kept: 180 224 B at the limit
  // opt in on every launch: the attribute is per device and the call costs about a microsecond
  FPB_CUDA_CHECK(cudaFuncSetAttribute(k6_merge_grouped_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  k6_merge_grouped_kernel<<<n_queries, 1024, smem, stream>>>(d_all_records, n_shards, b_stride, R, P, Kp2, n_keep,
                                                            top_k, global_group, n_total_docs, max_per_group,
                                                            d_out_ids, d_out_scores, d_out_counts);
  FPB_LAUNCH_CHECK("k6_merge_grouped");
  return FPB_OK;
}

int launch_results_to_records(const int64_t* ids, const float* scores, int B, int top_k, fpb_record* d_records,
                              cudaStream_t st) {
  const int64_t n = int64_t(B) * top_k;
  results_to_records_kernel<<<int((n + 255) / 256), 256, 0, st>>>(ids, scores, n, d_records);
  FPB_LAUNCH_CHECK("results_to_records");
  return FPB_OK;
}

extern "C" int fpb_merge_shards_grouped(const fpb_record* d_all_records, int n_shards, int B, int R, int n_keep,
                                        int top_k, const int32_t* d_global_group, int64_t n_total_docs,
                                        int max_per_group, int64_t* d_out_ids, float* d_out_scores,
                                        int32_t* d_out_counts, void* stream) {
  return launch_merge_grouped(d_all_records, n_shards, B, B, R, n_keep, top_k, d_global_group, n_total_docs,
                              max_per_group, d_out_ids, d_out_scores, d_out_counts, static_cast<cudaStream_t>(stream));
}

namespace {

int index_with_groups(const char* who, fpb_index** out, const fpb_index* ix, const int32_t* d_doc_group,
                      int64_t n_groups, int max_per_group) {
  if (!out) {
    fpb_set_error("%s: out is NULL", who);
    return FPB_ERR_INVALID;
  }
  *out = nullptr;
  if (!ix || !d_doc_group) {
    fpb_set_error("%s: NULL index or group array", who);
    return FPB_ERR_INVALID;
  }
  if (n_groups < 1 || n_groups > INT32_MAX) {
    fpb_set_error("%s: n_groups=%lld must be in [1, %d]", who, (long long)n_groups, INT32_MAX);
    return FPB_ERR_INVALID;
  }
  if (max_per_group < 1 || max_per_group > FPB_MAX_PER_GROUP) {
    fpb_set_error("%s: max_per_group=%d must be in [1, %d]", who, max_per_group, FPB_MAX_PER_GROUP);
    return FPB_ERR_INVALID;
  }
  fpb_index* gx = new fpb_index(*ix);
  gx->doc_group = d_doc_group;
  gx->n_groups = n_groups;
  gx->max_per_group = max_per_group;
  gx->global_group = nullptr;  // fpb_index_with_shard_groups sets them
  gx->n_total_docs = 0;
  if (gx->walk) ++gx->walk->refs;
  *out = gx;
  return FPB_OK;
}

}  // namespace

extern "C" int fpb_index_with_groups(fpb_index** out, const fpb_index* ix, const int32_t* d_doc_group,
                                     int64_t n_groups) {
  return index_with_groups("fpb_index_with_groups", out, ix, d_doc_group, n_groups, 1);
}

extern "C" int fpb_index_with_groups_max(fpb_index** out, const fpb_index* ix, const int32_t* d_doc_group,
                                         int64_t n_groups, int max_per_group) {
  return index_with_groups("fpb_index_with_groups_max", out, ix, d_doc_group, n_groups, max_per_group);
}

extern "C" int fpb_index_with_shard_groups(fpb_index** out, const fpb_index* ix, const int32_t* d_doc_group,
                                           int64_t n_groups, int max_per_group, const int32_t* d_global_group,
                                           int64_t n_total_docs) {
  const char* who = "fpb_index_with_shard_groups";
  if (out) *out = nullptr;
  if (out && ix && !d_global_group) {
    fpb_set_error("%s: NULL global group array", who);
    return FPB_ERR_INVALID;
  }
  if (out && ix && (n_total_docs < 1 || n_total_docs > INT32_MAX || ix->doc_id_base + ix->N > n_total_docs)) {
    fpb_set_error("%s: n_total_docs=%lld must be in [1, %d] and cover the shard's documents [%lld, %lld)", who,
                  (long long)n_total_docs, INT32_MAX, (long long)ix->doc_id_base, (long long)(ix->doc_id_base + ix->N));
    return FPB_ERR_INVALID;
  }
  FPB_TRY(index_with_groups(who, out, ix, d_doc_group, n_groups, max_per_group));
  (*out)->global_group = d_global_group;
  (*out)->n_total_docs = n_total_docs;
  return FPB_OK;
}
