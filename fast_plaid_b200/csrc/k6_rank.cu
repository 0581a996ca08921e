// Everything that orders documents by the canonical key (select.cuh): K3b, the pruning to the n_full_scores/4 best
// candidates (search.rs:602-619); K6, the final ranking (search.rs:659-666); and the document-sharded merge and
// threshold (new, SURVEY.md 8e).
//
// Canonical order: larger score first, then smaller doc id.  (The reference's non-stable sort(descending) leaves
// equal scores in an implementation-defined order.)
#include "kernels.h"
#include "select.cuh"

namespace {

// ---------------------------------------------------------------------------------------
// K3b: top-n_dec by (score desc, candidate index asc) -- candidate index order is doc id
// order, so this is the canonical rule "larger score, then smaller doc id".  Equivalent to
// the reference's topk(n_full) followed by topk(n_full/4) up to tie order.
// ---------------------------------------------------------------------------------------

// K3b's entries: candidate i of a row and its score
struct CandidateScores {
  static constexpr bool dense = true;
  const float* scores;
  __device__ static float empty() { return NAN; }
  __device__ float load(int i) const { return scores[i]; }
  __device__ bool present(float) const { return true; }
  __device__ float value(float v) const { return v; }
  __device__ uint64_t key(float v, int i) const { return rank_key_f32(v, uint32_t(i)); }
};

// Row b of `approx` (stride cand_cap) holds the scores of n_cand[b] candidates, candidate i being document
// cand[b, i].  cand == NULL: all cand_cap entries of the row are candidates, candidate i being document i.  Two CTAs
// per SM: 32 registers, which the selection fits without spilling.
__global__ void __launch_bounds__(1024, 2)
k3b_select_kernel(const float* __restrict__ approx, const int32_t* __restrict__ cand, int cand_cap,
                  const int32_t* __restrict__ n_cand, int n_dec, int Rp2, int32_t* __restrict__ rerank,
                  float* __restrict__ rerank_approx, int32_t* __restrict__ n_rerank) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint64_t* keys = reinterpret_cast<uint64_t*>(smem_raw);
  const int b = blockIdx.x, tid = threadIdx.x;
  const int n = cand ? n_cand[b] : cand_cap;
  const float* ab = approx + int64_t(b) * cand_cap;
  const int32_t* cb = cand ? cand + int64_t(b) * cand_cap : nullptr;
  int32_t* rr = rerank + int64_t(b) * n_dec;
  float* ra = rerank_approx + int64_t(b) * n_dec;
  if (n <= n_dec) {  // search.rs:605 / :615 conditions false: nothing is pruned
    for (int i = tid; i < n; i += 1024) {
      rr[i] = cb ? cb[i] : i;
      ra[i] = ab[i];
    }
    if (tid == 0) n_rerank[b] = n;
    return;
  }
  block_select_keys(CandidateScores{ab}, n, n_dec, keys, Rp2);
  for (int r = tid; r < n_dec; r += 1024) {
    const uint32_t idx = rank_key_id(keys[r]);
    rr[r] = cb ? cb[idx] : int32_t(idx);
    ra[r] = ab[idx];
  }
  if (tid == 0) n_rerank[b] = n_dec;
}

// K6, one CTA per query: row b of exact / rerank (stride R) holds the scores and ids of n_rerank[b] documents
__global__ void __launch_bounds__(1024)
k6_rank_kernel(const float* __restrict__ exact, const int32_t* __restrict__ rerank,
               const int32_t* __restrict__ n_rerank, int R, int Rp2, int top_k, int64_t doc_id_base,
               int64_t* __restrict__ out_ids, float* __restrict__ out_scores, int32_t* __restrict__ out_counts) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint64_t* keys = reinterpret_cast<uint64_t*>(smem_raw);
  const int b = blockIdx.x, tid = threadIdx.x;
  const int n = n_rerank[b];
  for (int i = tid; i < Rp2; i += 1024) {
    uint64_t k = 0;
    if (i < n) k = rank_key_f32(exact[int64_t(b) * R + i], uint32_t(rerank[int64_t(b) * R + i]));
    keys[i] = k;
  }
  __syncthreads();
  block_sort_desc(keys, Rp2);
  block_write_ranking(keys, n, top_k, doc_id_base, out_ids, out_scores, out_counts, b);
}

__global__ void emit_records_kernel(const float* __restrict__ exact, const float* __restrict__ rerank_approx,
                                    const int32_t* __restrict__ rerank, const int32_t* __restrict__ n_rerank,
                                    int B, int R, int64_t doc_id_base, fpb_record* __restrict__ rec) {
  const int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
  if (i >= int64_t(B) * R) return;
  const int b = int(i / R), r = int(i % R);
  fpb_record o;
  if (r < n_rerank[b]) {
    o.approx = rerank_approx[i];
    o.exact = exact[i];
    o.doc_id = doc_id_base + rerank[i];
  } else {
    o.approx = -INFINITY;
    o.exact = -INFINITY;
    o.doc_id = -1;
  }
  rec[i] = o;
}

// one CTA per query: re-apply the global pruning rule over the gathered records, then rank.
//   keep the R best by (approx desc, doc id asc)   -- search.rs:605-619 on the whole index
//   order them by  (exact desc, doc id asc)        -- search.rs:659
__global__ void __launch_bounds__(1024)
k6_merge_kernel(const fpb_record* __restrict__ all_groups, int n_shards, int B, int R, int P, int Rp2, int top_k,
                int64_t* __restrict__ out_ids, float* __restrict__ out_scores, int32_t* __restrict__ out_counts) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint64_t* keys = reinterpret_cast<uint64_t*>(smem_raw);  // [P]
  uint64_t* keys2 = keys + P;                               // [Rp2]
  uint16_t* pay = reinterpret_cast<uint16_t*>(keys2 + Rp2);  // [P] record index carried through the sort (P <= 2^14)
  // query blockIdx.x of the whole batch = query `b` of query group blockIdx.x / B, whose records are the
  // [n_shards, B, R] block of that group (one group: the block index is the query)
  const int b = blockIdx.x % B;
  const fpb_record* all = all_groups + int64_t(blockIdx.x / B) * n_shards * B * R;
  const int keep = block_merge_prune(all, B, R, b, n_shards * R, P, R, keys, pay);
  for (int i = threadIdx.x; i < Rp2; i += 1024) {
    uint64_t k2 = 0;
    if (i < keep) {
      const fpb_record rec = merge_record(all, B, R, b, pay[i]);
      k2 = rank_key_f32(rec.exact, uint32_t(rec.doc_id));
    }
    keys2[i] = k2;
  }
  __syncthreads();
  block_sort_desc(keys2, Rp2);
  block_write_ranking(keys2, keep, top_k, 0, out_ids, out_scores, out_counts, blockIdx.x);
}

// two-step sharded search, step 1: 64-bit keys of the local pruned list
__global__ void emit_keys_kernel(const float* __restrict__ rerank_approx, const int32_t* __restrict__ rerank,
                                 const int32_t* __restrict__ n_rerank, int B, int R, int64_t doc_id_base,
                                 uint64_t* __restrict__ keys) {
  const int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
  if (i >= int64_t(B) * R) return;
  const int b = int(i / R), r = int(i % R);
  uint64_t k = 0;
  if (r < n_rerank[b]) k = rank_key_f32(rerank_approx[i], uint32_t(doc_id_base + rerank[i]));
  keys[i] = k;
}

// step 2: global R-th best key per query; the local list keeps (in order) the entries at or above
// it.  One CTA per query.
__global__ void __launch_bounds__(1024)
apply_threshold_kernel(const uint64_t* __restrict__ all, int n_shards, int rank, int B, int R, int P,
                       int32_t* __restrict__ n_rerank, int32_t* __restrict__ rerank,
                       float* __restrict__ rerank_approx) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint64_t* keys = reinterpret_cast<uint64_t*>(smem_raw);
  __shared__ int warp_sums[32];
  __shared__ int s_base;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int total = n_shards * R;
  for (int i = tid; i < P; i += 1024) {
    uint64_t k = 0;
    if (i < total) k = all[(int64_t(i / R) * B + b) * R + (i % R)];
    keys[i] = k;
  }
  __syncthreads();
  block_sort_desc(keys, P);
  const uint64_t T = keys[R - 1];  // 0 when the whole index has fewer than R candidates
  // ordered compaction of the local list (it is in id order when nothing was pruned locally):
  // thread t owns entries [t*PER, (t+1)*PER), one block-wide exclusive scan gives the positions
  const uint64_t* mine = all + (int64_t(rank) * B + b) * R;
  int32_t* rr = rerank + int64_t(b) * R;
  float* ra = rerank_approx + int64_t(b) * R;
  int32_t* tmp_id = reinterpret_cast<int32_t*>(keys);   // reuse the sort buffer (P*8 >= R*8 bytes)
  float* tmp_ap = reinterpret_cast<float*>(tmp_id + R);
  const int n_old = n_rerank[b];
  constexpr int PER = 4;  // R <= 4096
  int32_t id[PER];
  float ap[PER];
  bool keep[PER];
  int c = 0;
#pragma unroll
  for (int u = 0; u < PER; ++u) {
    const int i = tid * PER + u;
    keep[u] = false;
    if (i < n_old && i < R) {
      const uint64_t k = mine[i];
      keep[u] = (k != 0) && (k >= T);
      id[u] = rr[i];
      ap[u] = ra[i];
    }
    c += keep[u] ? 1 : 0;
  }
  // the scan's first barrier also orders every read of T / keys[] before tmp_* overwrites the buffer
  int pos = block_exclusive_scan(c, warp_sums, &s_base);
#pragma unroll
  for (int u = 0; u < PER; ++u) {
    if (keep[u]) {
      tmp_id[pos] = id[u];
      tmp_ap[pos] = ap[u];
      ++pos;
    }
  }
  __syncthreads();
  const int n_new = s_base;
  for (int i = tid; i < n_new; i += 1024) {
    rr[i] = tmp_id[i];
    ra[i] = tmp_ap[i];
  }
  if (tid == 0) n_rerank[b] = n_new;
}

}  // namespace

// The merge sorts a query's n_shards*R records in shared memory: (P + Rp2)*8 + P*2 bytes with P = next_pow2 of
// their number, 196 608 B at the limit, under the 200 KB the merge and the threshold opt in to.
int check_merge_records(const char* who, int n_shards, int R) {
  if (int64_t(n_shards) * R > FPB_MERGE_MAX_RECORDS) {
    fpb_set_error("%s: n_shards*R = %d*%d records per query exceed the %d the shard merge sorts in shared memory", who,
                  n_shards, R, FPB_MERGE_MAX_RECORDS);
    return FPB_ERR_UNSUPPORTED;
  }
  return FPB_OK;
}

int launch_emit_keys(const fpb_index* ix, const Ws& ws, uint64_t* d_keys, cudaStream_t st) {
  const fpb_layout& L = *ws.L;
  const int64_t n = int64_t(L.B) * L.R;
  emit_keys_kernel<<<int((n + 255) / 256), 256, 0, st>>>(ws.rerank_approx(), ws.rerank(), ws.n_rerank(), L.B, L.R,
                                                        ix->doc_id_base, d_keys);
  FPB_LAUNCH_CHECK("emit_keys");
  return FPB_OK;
}

int launch_apply_threshold(const Ws& ws, const uint64_t* d_all_keys, int n_shards, int rank, cudaStream_t st,
                           int b_stride) {
  const fpb_layout& L = *ws.L;
  if (b_stride <= 0) b_stride = L.B;  // queries per shard in the gathered key array
  FPB_TRY(check_merge_records("apply_threshold", n_shards, L.R));
  const int P = fpb_next_pow2(n_shards * L.R);
  const size_t smem = size_t(P) * 8;
  // opt in on every launch: the attribute is per device and the call costs about a microsecond
  FPB_CUDA_CHECK(cudaFuncSetAttribute(apply_threshold_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  apply_threshold_kernel<<<L.B, 1024, smem, st>>>(d_all_keys, n_shards, rank, b_stride, L.R, P, ws.n_rerank(),
                                                  ws.rerank(), ws.rerank_approx());
  FPB_LAUNCH_CHECK("apply_threshold");
  return FPB_OK;
}

int launch_select(const float* scores, const int32_t* cand, const int32_t* n_cand, int stride, int B, int R,
                  int32_t* rerank, float* rerank_scores, int32_t* n_rerank, cudaStream_t st) {
  const int Rp2 = fpb_next_pow2(R);
  // dynamic keys[] (8 B x Rp2, 32 KB at the maximum R = 4096) on top of 25 KB of static shared memory: opt in
  // (per device: cudaFuncSetAttribute applies to the current device only, and the call is cheap)
  FPB_CUDA_CHECK(cudaFuncSetAttribute(k3b_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Rp2 * 8));
  k3b_select_kernel<<<B, 1024, size_t(Rp2) * 8, st>>>(scores, cand, stride, n_cand, R, Rp2, rerank, rerank_scores,
                                                     n_rerank);
  FPB_LAUNCH_CHECK("k3b_select");
  return FPB_OK;
}

int launch_rank(const float* scores, const int32_t* ids, const int32_t* n, int R, int B, int top_k,
                int64_t doc_id_base, int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts,
                cudaStream_t st) {
  const int Rp2 = fpb_next_pow2(R);
  k6_rank_kernel<<<B, 1024, size_t(Rp2) * 8, st>>>(scores, ids, n, R, Rp2, top_k, doc_id_base, d_out_ids,
                                                  d_out_scores, d_out_counts);
  FPB_LAUNCH_CHECK("k6_rank");
  return FPB_OK;
}

int launch_emit_records(const float* exact, const float* approx, const int32_t* ids, const int32_t* n_sel, int B,
                        int R, int64_t doc_id_base, fpb_record* d_records, cudaStream_t st) {
  const int64_t n = int64_t(B) * R;
  emit_records_kernel<<<int((n + 255) / 256), 256, 0, st>>>(exact, approx, ids, n_sel, B, R, doc_id_base, d_records);
  FPB_LAUNCH_CHECK("emit_records");
  return FPB_OK;
}

extern "C" int fpb_merge_shards(const fpb_record* d_all_records, int n_shards, int B, int R, int top_k,
                                int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts, void* stream) {
  return launch_merge(d_all_records, n_shards, B, B, R, top_k, d_out_ids, d_out_scores, d_out_counts,
                      static_cast<cudaStream_t>(stream));
}

// merge of `n_queries` queries of gathered records laid out [n_groups][n_shards, b_stride, R]: query q is query
// q % b_stride of group q / b_stride (n_queries <= b_stride: one group)
int launch_merge(const fpb_record* d_all_records, int n_shards, int b_stride, int n_queries, int R, int top_k,
                 int64_t* d_out_ids, float* d_out_scores, int32_t* d_out_counts, cudaStream_t stream) {
  const int B = b_stride;
  if (!d_all_records || n_shards < 1 || B < 1 || R < 1 || top_k < 1 || n_queries < 0) {
    fpb_set_error("fpb_merge_shards: bad arguments");
    return FPB_ERR_INVALID;
  }
  FPB_TRY(check_merge_records("fpb_merge_shards", n_shards, R));
  if (n_queries == 0) return FPB_OK;
  const int P = fpb_next_pow2(n_shards * R);
  const int Rp2 = fpb_next_pow2(R);
  const size_t smem = size_t(P + Rp2) * 8 + size_t(P) * sizeof(uint16_t);
  // opt in on every launch: the attribute is per device and the call costs about a microsecond
  FPB_CUDA_CHECK(cudaFuncSetAttribute(k6_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  k6_merge_kernel<<<n_queries, 1024, smem, stream>>>(d_all_records, n_shards, B, R, P, Rp2, top_k, d_out_ids,
                                                    d_out_scores, d_out_counts);
  FPB_LAUNCH_CHECK("k6_merge");
  return FPB_OK;
}
