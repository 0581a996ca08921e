// Document-sharded search below the C ABI (SURVEY.md 8e; replaces the reference's one-thread-per-GPU
// dispatch over a replicated index, python/fast_plaid/search/fast_plaid.py:893-928).
//
// The ranks of one communicator form a grid of  query groups x document shards:  rank r is document
// shard  r % n_doc_shards  of query group  r / n_doc_shards.  A query group searches its contiguous slice
// of the batch; its document shards each hold a contiguous range of the documents (centroids replicated).
// The path has one real exchange, because the reference prunes GLOBALLY to the n_full_scores/4 best
// approximate scores before exact scoring (search.rs:605-619):
//     local stages up to the pruned list  ->  ncclAllGather of [B_local, R] 64-bit keys
//     -> global threshold, the local list shrinks to the survivors  ->  MaxSim on them
//     -> ncclAllGather of [B_local, R] (approx, exact, id) records  ->  every rank merges every query.
// Both collectives run on the caller's stream, issued from here: one call per batch, no host round trip.
// With one query group this is plain document sharding; with several, K1 / the probe run on B / n_groups
// queries per GPU instead of being replicated on all of them.
//
// NCCL is resolved at run time (dlopen of libnccl.so.2 -- inside a PyTorch process that is the copy torch
// already loaded), so the library has no link-time dependency on it and single-GPU use needs no NCCL.
#include <dlfcn.h>
#include <nccl.h>
#include <string.h>

#include <mutex>

#include "entry.h"

namespace {

struct NcclApi {
  decltype(&ncclGetUniqueId) GetUniqueId = nullptr;
  decltype(&ncclCommInitRank) CommInitRank = nullptr;
  decltype(&ncclCommDestroy) CommDestroy = nullptr;
  decltype(&ncclAllGather) AllGather = nullptr;
  decltype(&ncclGetErrorString) GetErrorString = nullptr;
  decltype(&ncclGetVersion) GetVersion = nullptr;
  bool ok = false;
};

NcclApi& nccl() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return;
    api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(dlsym(h, "ncclGetUniqueId"));
    api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(dlsym(h, "ncclCommInitRank"));
    api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(dlsym(h, "ncclCommDestroy"));
    api.AllGather = reinterpret_cast<decltype(api.AllGather)>(dlsym(h, "ncclAllGather"));
    api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(dlsym(h, "ncclGetErrorString"));
    api.GetVersion = reinterpret_cast<decltype(api.GetVersion)>(dlsym(h, "ncclGetVersion"));
    api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllGather && api.GetErrorString;
  });
  return api;
}

#define FPB_NCCL_CHECK(expr)                                                                   \
  do {                                                                                         \
    ncclResult_t _r = (expr);                                                                  \
    if (_r != ncclSuccess) {                                                                   \
      fpb_set_error("%s failed: %s (%s:%d)", #expr, nccl().GetErrorString(_r), __FILE__, __LINE__); \
      return FPB_ERR_CUDA;                                                                     \
    }                                                                                          \
  } while (0)

}  // namespace

struct fpb_comm {
  ncclComm_t comm;
  int nranks, rank, device;
};

static_assert(sizeof(ncclUniqueId) == FPB_COMM_ID_BYTES, "FPB_COMM_ID_BYTES must be sizeof(ncclUniqueId)");

extern "C" int fpb_comm_unique_id(void* out_id) {
  if (!out_id) {
    fpb_set_error("fpb_comm_unique_id: NULL output");
    return FPB_ERR_INVALID;
  }
  if (!nccl().ok) {
    const char* why = dlerror();
    fpb_set_error("NCCL (libnccl.so.2) could not be loaded: %s", why ? why : "symbols missing");
    return FPB_ERR_UNSUPPORTED;
  }
  ncclUniqueId id;
  FPB_NCCL_CHECK(nccl().GetUniqueId(&id));
  memcpy(out_id, &id, sizeof(id));
  return FPB_OK;
}

extern "C" int fpb_comm_create(fpb_comm** out, int nranks, int rank, const void* unique_id, int device) {
  if (!out || !unique_id || nranks < 1 || rank < 0 || rank >= nranks) {
    fpb_set_error("fpb_comm_create: bad arguments (nranks=%d rank=%d)", nranks, rank);
    return FPB_ERR_INVALID;
  }
  *out = nullptr;
  if (!nccl().ok) {
    fpb_set_error("NCCL (libnccl.so.2) could not be loaded");
    return FPB_ERR_UNSUPPORTED;
  }
  FPB_CUDA_CHECK(cudaSetDevice(device));
  ncclUniqueId id;
  memcpy(&id, unique_id, sizeof(id));
  ncclComm_t c;
  FPB_NCCL_CHECK(nccl().CommInitRank(&c, nranks, id, rank));
  fpb_comm* h = new fpb_comm();
  h->comm = c;
  h->nranks = nranks;
  h->rank = rank;
  h->device = device;
  *out = h;
  return FPB_OK;
}

extern "C" void fpb_comm_destroy(fpb_comm* comm) {
  if (!comm) return;
  if (nccl().ok && comm->comm) {
    cudaSetDevice(comm->device);
    nccl().CommDestroy(comm->comm);
  }
  delete comm;
}

extern "C" int fpb_comm_nccl_version(void) {
  int v = 0;
  if (nccl().ok && nccl().GetVersion) nccl().GetVersion(&v);
  return v;
}

extern "C" int64_t fpb_sharded_scratch_bytes(int b_local, int R, int nranks) {
  if (b_local < 1 || R < 1 || nranks < 1) return 0;
  const int64_t per_rank = int64_t(b_local) * R;
  // keys (local + gathered) and records (local + gathered), each block 256-byte aligned
  return fpb_align256(per_rank * 8) + fpb_align256(per_rank * 8 * nranks) + fpb_align256(per_rank * 16) +
         fpb_align256(per_rank * 16 * nranks);
}

extern "C" int fpb_search_batch_sharded(const fpb_index* ix, fpb_comm* comm, int n_query_groups, const void* d_queries,
                                        int B, int Q, const fpb_params* p, void* d_ws, size_t ws_bytes, void* d_scratch,
                                        size_t scratch_bytes, int64_t* d_out_ids, float* d_out_scores,
                                        int32_t* d_out_counts, void* stream) {
  if (!ix || !comm || !p || !d_queries || !d_ws || !d_scratch || !d_out_ids || !d_out_scores || !d_out_counts) {
    fpb_set_error("fpb_search_batch_sharded: NULL argument");
    return FPB_ERR_INVALID;
  }
  if (n_query_groups < 1 || comm->nranks % n_query_groups != 0 || B < 1) {
    fpb_set_error("fpb_search_batch_sharded: %d query groups do not divide %d ranks (B=%d)", n_query_groups,
                  comm->nranks, B);
    return FPB_ERR_INVALID;
  }
  if (p->flags & FPB_FLAG_SUBSET) {
    fpb_set_error("fpb_search_batch_sharded: subset search goes through the fpb_shard_subset_* steps");
    return FPB_ERR_UNSUPPORTED;
  }
  FPB_TRY(fpb_require_ivf(ix));
  const int n_shards = comm->nranks / n_query_groups;  // document shards per query group
  const int group = comm->rank / n_shards, shard = comm->rank % n_shards;
  const int b_local = (B + n_query_groups - 1) / n_query_groups;   // slots per rank in the gathered arrays
  const int q0 = group * b_local;
  const int nb = B - q0 < 0 ? 0 : (B - q0 < b_local ? B - q0 : b_local);  // queries of this group
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  FPB_CUDA_CHECK(cudaSetDevice(ix->device));

  fpb_layout L;
  memset(&L, 0, sizeof(L));
  int R = p->n_full_scores / 4;
  if (R < 1) R = 1;
  if (nb > 0) {
    FPB_TRY(fpb_workspace_layout(ix, nb, Q, p, &L));
    FPB_TRY(fpb_require_bytes("workspace", L.total_bytes, ws_bytes));
    R = L.R;
  }
  // refused here, before the first collective: every rank has the same parameters, so every rank returns here
  FPB_TRY(check_merge_records("fpb_search_batch_sharded", n_shards, R));
  FPB_TRY(fpb_require_bytes("scratch", fpb_sharded_scratch_bytes(b_local, R, comm->nranks), scratch_bytes));
  FPB_TRY(fpb_require_aligned("workspace", d_ws));
  FPB_TRY(fpb_require_aligned("scratch", d_scratch));
  const int64_t per_rank = int64_t(b_local) * R;
  char* sc = static_cast<char*>(d_scratch);
  uint64_t* keys = reinterpret_cast<uint64_t*>(sc);
  sc += fpb_align256(per_rank * 8);
  uint64_t* all_keys = reinterpret_cast<uint64_t*>(sc);
  sc += fpb_align256(per_rank * 8 * comm->nranks);
  fpb_record* recs = reinterpret_cast<fpb_record*>(sc);
  sc += fpb_align256(per_rank * 16);
  fpb_record* all_recs = reinterpret_cast<fpb_record*>(sc);

  Ws ws{&L, static_cast<char*>(d_ws)};
  // slots of this group that hold no query (ragged last group): keys 0 / record id -1 are the padding values
  if (nb < b_local) {
    FPB_CUDA_CHECK(cudaMemsetAsync(keys, 0, size_t(per_rank) * 8, st));
    FPB_CUDA_CHECK(cudaMemsetAsync(recs, 0xFF, size_t(per_rank) * 16, st));
  }
  // ---- step 1: local stages up to the pruned list, keys of it ----
  if (nb > 0) {
    FPB_TRY(run_centroid_scores(ix, ws, static_cast<const __half*>(d_queries) + int64_t(q0) * Q * ix->dim, st));
    FPB_TRY(run_probe_to_select(ix, ws, false, st));
    FPB_TRY(launch_emit_keys(ix, ws, keys, st));
  }
  FPB_NCCL_CHECK(nccl().AllGather(keys, all_keys, size_t(per_rank) * 8, ncclUint8, comm->comm, st));
  // ---- step 2: global threshold over this group's shards, exact scores of the survivors, records ----
  if (nb > 0) {
    FPB_TRY(launch_apply_threshold(ws, all_keys + int64_t(group) * n_shards * per_rank, n_shards, shard, st, b_local));
    FPB_TRY(launch_maxsim(ix, ws, st));
    FPB_TRY(launch_emit_records(ix, ws, recs, st));
  }
  FPB_NCCL_CHECK(nccl().AllGather(recs, all_recs, size_t(per_rank) * 16, ncclUint8, comm->comm, st));
  // ---- every rank ranks every query in ONE launch: query q belongs to group q / b_local, whose records are the
  //      [n_shards, b_local, R] block of that group in the gathered array (launch_merge with n_queries > b_stride) ----
  FPB_TRY(launch_merge(all_recs, n_shards, b_local, B, R, p->top_k, d_out_ids, d_out_scores, d_out_counts, st));
  return FPB_OK;
}

extern "C" int fpb_search_batch_sharded_host(const fpb_index* ix, fpb_comm* comm, int n_query_groups,
                                             const void* h_queries, int B, int Q, const fpb_params* p, void* d_ws,
                                             size_t ws_bytes, void* d_scratch, size_t scratch_bytes,
                                             void* d_queries_staging, int64_t* d_out_ids, float* d_out_scores,
                                             int32_t* d_out_counts, int64_t* h_out_ids, float* h_out_scores,
                                             int32_t* h_out_counts, void* stream) {
  return search_via_host("fpb_search_batch_sharded_host", ix, h_queries, B, Q, p, d_queries_staging, d_out_ids,
                         d_out_scores, d_out_counts, h_out_ids, h_out_scores, h_out_counts, stream, [&] {
                           return fpb_search_batch_sharded(ix, comm, n_query_groups, d_queries_staging, B, Q, p, d_ws,
                                                           ws_bytes, d_scratch, scratch_bytes, d_out_ids,
                                                           d_out_scores, d_out_counts, stream);
                         });
}
