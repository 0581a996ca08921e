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

// Digits of the 64-bit key, most significant first: 11+11+10 bits cover the score, the rest
// only matters when scores tie at the threshold.
__constant__ int K3B_LO[6] = {53, 42, 32, 21, 10, 0};
__constant__ int K3B_W[6] = {11, 11, 10, 11, 11, 10};
constexpr int K3B_VPT = 4;  // independent loads in flight per thread
constexpr int K3B_BCAP = 2048;  // capacity of the threshold bucket on the fast path

// Row b of `approx` (stride cand_cap) holds the scores of n_cand[b] candidates, candidate i being document
// cand[b, i].  cand == NULL: all cand_cap entries of the row are candidates, candidate i being document i.
__global__ void __launch_bounds__(1024)
k3b_select_kernel(const float* __restrict__ approx, const int32_t* __restrict__ cand, int cand_cap,
                  const int32_t* __restrict__ n_cand, int n_dec, int Rp2, int32_t* __restrict__ rerank,
                  float* __restrict__ rerank_approx, int32_t* __restrict__ n_rerank) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint64_t* keys = reinterpret_cast<uint64_t*>(smem_raw);
  __shared__ int hist[SEL_BINS];
  __shared__ int s_need, s_hd, s_cnt;
  __shared__ uint64_t s_prefix, s_mask;
  __shared__ uint64_t bkeys[K3B_BCAP];  // fast path: keys of the threshold bucket
  __shared__ float s_red[64];
  __shared__ int s_cnt2, s_fast;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
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
  // ---- fast path: 2048 buckets over the VALUE range [min, max] of this query's scores ----
  // The radix passes below start from the top bits of the float key, where the scores of one query share
  // sign, exponent and the leading mantissa bits: a handful of hot bins, so every element pays a ballot +
  // match_any + contended shared atomic, three passes long (0.49 ms on cfg-3).  A linear bucketisation of the
  // actual value range spreads the scores, one histogram pass isolates the threshold bucket, and only that
  // bucket (typically n / 2048 elements) is ordered by the exact 64-bit key.  value_bucket() is monotone, so
  // every element of a higher bucket is strictly larger: the selection is exactly the same.
  {
    constexpr int FV = 8;  // independent loads in flight per thread
    float mn = INFINITY, mx = -INFINITY;
    for (int i0 = tid; i0 < n; i0 += 1024 * FV) {
      float v[FV];
#pragma unroll
      for (int u = 0; u < FV; ++u) v[u] = (i0 + u * 1024 < n) ? ab[i0 + u * 1024] : NAN;  // fmin/fmax skip NaN
#pragma unroll
      for (int u = 0; u < FV; ++u) {
        mn = fminf(mn, v[u]);
        mx = fmaxf(mx, v[u]);
      }
    }
    for (int i = tid; i < SEL_BINS; i += 1024) hist[i] = 0;
    if (tid == 0) {
      s_cnt = 0;
      s_cnt2 = 0;
      s_fast = 0;
    }
    block_min_max(mn, mx, s_red);
    const float range = mx - mn;
    // finite, non-degenerate range (NaN / inf scores or all-equal scores take the radix path)
    const bool usable = range > 0.f && range < 3.0e38f;
    const float scale = usable ? float(SEL_BINS - 1) / range : 0.f;
    if (usable) {
      for (int i0 = tid; i0 < n; i0 += 1024 * FV) {
        float v[FV];
#pragma unroll
        for (int u = 0; u < FV; ++u) v[u] = (i0 + u * 1024 < n) ? ab[i0 + u * 1024] : 0.f;
#pragma unroll
        for (int u = 0; u < FV; ++u)
          if (i0 + u * 1024 < n) atomicAdd(&hist[value_bucket(v[u], mn, scale)], 1);
      }
      __syncthreads();
      int hd, rest;
      if (tid < 32 && warp_find_bucket(hist, SEL_BINS, n_dec, &hd, &rest)) {
        s_need = rest;
        s_hd = hd;
        s_fast = hist[hd] <= K3B_BCAP ? 1 : 0;
      }
      __syncthreads();
      if (s_fast) {
        const int t = s_hd;
        for (int i0 = tid; i0 < n; i0 += 1024 * FV) {
          float v[FV];
#pragma unroll
          for (int u = 0; u < FV; ++u) v[u] = (i0 + u * 1024 < n) ? ab[i0 + u * 1024] : 0.f;
#pragma unroll
          for (int u = 0; u < FV; ++u) {
            const int i = i0 + u * 1024;
            if (i < n) {
              const int bk = value_bucket(v[u], mn, scale);
              if (bk > t) {
                keys[atomicAdd(&s_cnt, 1)] = rank_key_f32(v[u], uint32_t(i));    // fewer than n_dec of these
              } else if (bk == t) {
                bkeys[atomicAdd(&s_cnt2, 1)] = rank_key_f32(v[u], uint32_t(i));  // at most K3B_BCAP of these
              }
            }
          }
        }
        __syncthreads();
        const int c2 = s_cnt2, need2 = s_need;
        for (int i = c2 + tid; i < K3B_BCAP; i += 1024) bkeys[i] = 0ull;
        __syncthreads();
        block_sort_desc(bkeys, K3B_BCAP);
        const int c1 = s_cnt;
        for (int i = tid; i < need2; i += 1024) keys[c1 + i] = bkeys[i];
        __syncthreads();
        if (tid == 0) s_cnt = c1 + need2;  // == n_dec
        __syncthreads();
      }
    }
  }
  if (!s_fast) {  // ---- radix passes over the 64-bit key: the threshold key T, then every key >= T ----
    if (tid == 0) {
      s_need = n_dec;
      s_prefix = 0;
      s_mask = 0;
    }
    const int stride = 1024 * K3B_VPT;
    const int n_up = (n + stride - 1) / stride * stride;
    for (int pass = 0; pass < 6; ++pass) {
      const int lo = K3B_LO[pass], width = K3B_W[pass];
      const uint64_t dmask = (1ull << width) - 1ull;
      for (int i = tid; i < SEL_BINS; i += 1024) hist[i] = 0;
      __syncthreads();
      const uint64_t prefix = s_prefix, mask = s_mask;
      for (int i0 = tid; i0 < n_up; i0 += stride) {
        float v[K3B_VPT];
#pragma unroll
        for (int u = 0; u < K3B_VPT; ++u) {
          const int i = i0 + u * 1024;
          v[u] = (i < n) ? ab[i] : 0.f;
        }
#pragma unroll
        for (int u = 0; u < K3B_VPT; ++u) {
          const int i = i0 + u * 1024;
          const bool valid = i < n;
          const uint64_t key = valid ? rank_key_f32(v[u], uint32_t(i)) : 0ull;
          const bool in = valid && ((key & mask) == prefix);
          const unsigned act = __ballot_sync(0xffffffffu, in);
          if (in) {
            const int bin = int((key >> lo) & dmask);
            const unsigned peers = __match_any_sync(act, bin);
            if (lane == __ffs(peers) - 1) atomicAdd(&hist[bin], __popc(peers));
          }
        }
      }
      __syncthreads();
      int d, rest;
      if (tid < 32 && warp_find_bucket(hist, 1 << width, s_need, &d, &rest)) {
        s_need = rest;
        s_hd = hist[d];
        s_prefix = prefix | (uint64_t(d) << lo);
        s_mask = mask | (dmask << lo);
      }
      __syncthreads();
      if (s_hd == s_need) break;  // the whole bucket is selected
    }
    const uint64_t T = s_prefix;  // unprocessed low bits are zero
    if (tid == 0) s_cnt = 0;
    __syncthreads();
    for (int i0 = tid; i0 < n_up; i0 += stride) {
      float v[K3B_VPT];
#pragma unroll
      for (int u = 0; u < K3B_VPT; ++u) {
        const int i = i0 + u * 1024;
        v[u] = (i < n) ? ab[i] : 0.f;
      }
#pragma unroll
      for (int u = 0; u < K3B_VPT; ++u) {
        const int i = i0 + u * 1024;
        if (i < n) {
          const uint64_t key = rank_key_f32(v[u], uint32_t(i));
          if (key >= T) {
            const int pos = atomicAdd(&s_cnt, 1);
            if (pos < Rp2) keys[pos] = key;
          }
        }
      }
    }
  }
  __syncthreads();
  const int cnt = min(s_cnt, Rp2);
  for (int i = cnt + tid; i < Rp2; i += 1024) keys[i] = 0ull;
  __syncthreads();
  block_sort_desc(keys, Rp2);
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
  const int cnt = min(top_k, n);
  for (int i = tid; i < top_k; i += 1024) {
    int64_t id = -1;
    float sc = -INFINITY;
    if (i < cnt) {
      id = doc_id_base + int64_t(rank_key_id(keys[i]));
      sc = rank_key_f32_value(keys[i]);
    }
    out_ids[int64_t(b) * top_k + i] = id;
    out_scores[int64_t(b) * top_k + i] = sc;
  }
  if (tid == 0) out_counts[b] = cnt;
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
  __shared__ int s_valid;
  // query blockIdx.x of the whole batch = query `b` of query group blockIdx.x / B, whose records are the
  // [n_shards, B, R] block of that group (one group: the block index is the query)
  const int b = blockIdx.x % B, tid = threadIdx.x;
  const fpb_record* all = all_groups + int64_t(blockIdx.x / B) * n_shards * B * R;
  out_ids += int64_t(blockIdx.x - b) * top_k;
  out_scores += int64_t(blockIdx.x - b) * top_k;
  out_counts += blockIdx.x - b;
  const int total = n_shards * R;
  if (tid == 0) s_valid = 0;
  __syncthreads();
  int local_valid = 0;
  for (int i = tid; i < P; i += 1024) {
    uint64_t k = 0;
    if (i < total) {
      const int s = i / R, r = i % R;
      const fpb_record rec = all[(int64_t(s) * B + b) * R + r];
      if (rec.doc_id >= 0) {
        k = rank_key_f32(rec.approx, uint32_t(rec.doc_id));
        ++local_valid;
      }
    }
    keys[i] = k;
    pay[i] = uint16_t(i);
  }
  if (local_valid) atomicAdd(&s_valid, local_valid);
  __syncthreads();
  block_sort_desc(keys, P, pay);
  const int keep = min(s_valid, R);
  for (int i = tid; i < Rp2; i += 1024) {
    uint64_t k2 = 0;
    if (i < keep) {
      const int j = int(pay[i]);
      const int s = j / R, r = j % R;
      const fpb_record rec = all[(int64_t(s) * B + b) * R + r];
      k2 = rank_key_f32(rec.exact, uint32_t(rec.doc_id));
    }
    keys2[i] = k2;
  }
  __syncthreads();
  block_sort_desc(keys2, Rp2);
  const int cnt = min(top_k, keep);
  for (int i = tid; i < top_k; i += 1024) {
    int64_t id = -1;
    float sc = -INFINITY;
    if (i < cnt) {
      id = int64_t(rank_key_id(keys2[i]));
      sc = rank_key_f32_value(keys2[i]);
    }
    out_ids[int64_t(b) * top_k + i] = id;
    out_scores[int64_t(b) * top_k + i] = sc;
  }
  if (tid == 0) out_counts[b] = cnt;
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
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
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
  int incl = c;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, off);
    if (lane >= off) incl += v;
  }
  if (lane == 31) warp_sums[warp] = incl;
  __syncthreads();  // also: everybody has read T / keys[] before tmp_* overwrites the buffer
  if (warp == 0) {
    const int ws = warp_sums[lane];
    int wincl = ws;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, wincl, off);
      if (lane >= off) wincl += v;
    }
    warp_sums[lane] = wincl - ws;
    if (lane == 31) s_base = wincl;
  }
  __syncthreads();
  int pos = warp_sums[warp] + incl - c;
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
