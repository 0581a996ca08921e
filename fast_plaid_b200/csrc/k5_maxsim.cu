// K5 : fused residual decompression + exact MaxSim           (search.rs:626-656, :53-107)
//
//   e_hat  = the decoded, normalised token (decode.cuh: decompress_slice; n from the token_norm table)
//   ts     = fp16( sum_fp32 e_hat[t] . q[j] )                          tensor-core MMA, fp32 acc
//   score  = sum_{j<Q}^{fp32} max_{t<len} ts[t][j]
//
// The reference materialises the decompressed rows ([tokens,128] fp16 plus several
// temporaries), pads them to [R, maxlen, 128], runs a batched HGEMM and three more passes.
// Here the decompressed rows exist only as a 64-token shared-memory tile that is fed
// straight to the MMA; per token the kernel reads the packed residual (pd bytes), the code
// (4 B) and the centroid row (L2-resident table).
//
// v1 data path: mma.sync m16n8k16 (legacy tensor path) with a CTA of 4 warps per document.
#include "decode.cuh"
#include "kernels.h"

namespace {

constexpr int K5_THREADS = 128;
constexpr int K5_TILE = 64;

template <int D, int QP>
struct K5Smem {
  static constexpr int LDS = D + 8;
  static constexpr int bytes = (K5_TILE * LDS + QP * LDS) * 2 + 4 * QP * 2 + 256 * 8;
};

template <int D, int NBITS, int QP>
__global__ void __launch_bounds__(K5_THREADS)
k5_maxsim_kernel(const __half* __restrict__ C, const int64_t* __restrict__ doc_offsets,
                 const int32_t* __restrict__ codes, const uint8_t* __restrict__ residuals,
                 const __half* __restrict__ norms, WPerm wp,
                 const __half* __restrict__ Qpad, int Q, int B, int R, const int32_t* __restrict__ n_rerank,
                 const int32_t* __restrict__ rerank, float* __restrict__ exact) {
  constexpr int LDS = K5Smem<D, QP>::LDS;
  constexpr int LPT = lanes_per_token<D, NBITS>();
  constexpr int KS = D / 16;
  constexpr int QC = QP < 64 ? QP : 64;
  constexpr int NT = QC / 8;
  constexpr int NTQ = QP / 8;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __half* As = reinterpret_cast<__half*>(smem_raw);
  __half* Qs = As + K5_TILE * LDS;
  __half* wmax = Qs + QP * LDS;                                  // [4][QP]
  uint32_t* lut = reinterpret_cast<uint32_t*>(wmax + 4 * QP);    // 256 x 8 B reserved

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  Decoder<NBITS>::build(lut, wp, tid, K5_THREADS);
  const __half2 sentinel = __float2half2_rn(FPB_PAD_SENTINEL);
  int cur_b = -1;

  for (int w = blockIdx.x; w < B * R; w += gridDim.x) {
    const int b = w / R, r = w % R;
    if (r >= n_rerank[b]) continue;
    __syncthreads();  // previous document finished with As / Qs / wmax (also covers the LUT build)
    if (b != cur_b) {
      for (int i = tid; i < QP * (D / 8); i += K5_THREADS) {
        const int n = i / (D / 8), c8 = i % (D / 8);
        *reinterpret_cast<uint4*>(Qs + n * LDS + c8 * 8) =
            *reinterpret_cast<const uint4*>(Qpad + (int64_t(b) * QP + n) * D + c8 * 8);
      }
      cur_b = b;
    }
    const int d = rerank[int64_t(b) * R + r];
    const int64_t o0 = doc_offsets[d];
    const int len = int(doc_offsets[d + 1] - o0);

    __half2 mx[NTQ];
#pragma unroll
    for (int i = 0; i < NTQ; ++i) mx[i] = sentinel;

    for (int tile0 = 0; tile0 < len; tile0 += K5_TILE) {
      // ---- decompress up to 64 tokens into As (tokens past the end repeat the last one) ----
      for (int tok = tid / LPT; tok < K5_TILE; tok += K5_THREADS / LPT) {
        const int tt = min(tile0 + tok, len - 1);
        const int code = __ldg(codes + o0 + tt);
        decompress_slice<D, NBITS, LPT>(lut, residuals, C, norms, o0 + tt, code, tid % LPT, As + tok * LDS);
      }
      __syncthreads();
      // ---- ts = A(64 x D) . Q^T, 16 rows per warp ----
      uint32_t a[KS][4];
#pragma unroll
      for (int ks = 0; ks < KS; ++ks)
        ldmatrix_x4(a[ks][0], a[ks][1], a[ks][2], a[ks][3],
                    smem_u32(As + (warp * 16 + (lane & 15)) * LDS + ks * 16 + (lane >> 4) * 8));
      const bool v0 = (tile0 + warp * 16 + g) < len;
      const bool v1 = (tile0 + warp * 16 + g + 8) < len;
#pragma unroll
      for (int qc = 0; qc < QP / QC; ++qc) {
        float acc[NT][4];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
          for (int nt = 0; nt < NT; nt += 2) {
            const int mat = lane >> 3;
            const int n = qc * QC + (nt + (mat >> 1)) * 8 + (lane & 7);
            const int k = ks * 16 + (mat & 1) * 8;
            uint32_t b0, b1, b2, b3;
            ldmatrix_x4(b0, b1, b2, b3, smem_u32(Qs + n * LDS + k));
            mma_16816(acc[nt], a[ks], b0, b1);
            mma_16816(acc[nt + 1], a[ks], b2, b3);
          }
        }
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
          const __half2 h0 = v0 ? __floats2half2_rn(acc[nt][0], acc[nt][1]) : sentinel;
          const __half2 h1 = v1 ? __floats2half2_rn(acc[nt][2], acc[nt][3]) : sentinel;
          mx[qc * NT + nt] = __hmax2(mx[qc * NT + nt], __hmax2(h0, h1));
        }
      }
      __syncthreads();  // As is rewritten by the next tile
    }
    // ---- column maxima over the warp's rows, then over the 4 warps; fp32 sum over q < Q ----
#pragma unroll
    for (int i = 0; i < NTQ; ++i) {
      __half2 m = mx[i];
      m = __hmax2(m, u32_as_half2(__shfl_xor_sync(0xffffffffu, half2_as_u32(m), 4)));
      m = __hmax2(m, u32_as_half2(__shfl_xor_sync(0xffffffffu, half2_as_u32(m), 8)));
      m = __hmax2(m, u32_as_half2(__shfl_xor_sync(0xffffffffu, half2_as_u32(m), 16)));
      if (g == 0) *reinterpret_cast<uint32_t*>(wmax + warp * QP + i * 8 + 2 * t) = half2_as_u32(m);
    }
    __syncthreads();
    if (warp == 0) {
      float s = 0.f;
      for (int q = lane; q < Q; q += 32) {
        __half m = __hmax(__hmax(wmax[q], wmax[QP + q]), __hmax(wmax[2 * QP + q], wmax[3 * QP + q]));
        s += __half2float(m);
      }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
      if (lane == 0) exact[int64_t(b) * R + r] = s;
    }
  }
}

// reconstruct_embeddings (rust/utils/embeddings.rs:12-69): same decompression, rows to HBM.
template <int D, int NBITS>
__global__ void __launch_bounds__(K5_THREADS)
k5_reconstruct_kernel(const __half* __restrict__ C, const int64_t* __restrict__ doc_offsets,
                      const int32_t* __restrict__ codes, const uint8_t* __restrict__ residuals,
                      const __half* __restrict__ norms, WPerm wp,
                      const int32_t* __restrict__ doc_ids, int n, const int64_t* __restrict__ out_offsets,
                      __half* __restrict__ out) {
  constexpr int LPT = lanes_per_token<D, NBITS>();
  __shared__ uint32_t lut[512];
  Decoder<NBITS>::build(lut, wp, threadIdx.x, K5_THREADS);
  __syncthreads();
  for (int i = blockIdx.x; i < n; i += gridDim.x) {
    const int d = doc_ids[i];
    const int64_t o0 = doc_offsets[d];
    const int len = int(doc_offsets[d + 1] - o0);
    const int64_t oo = out_offsets[i];
    const int len_up = (len + (K5_THREADS / LPT) - 1) / (K5_THREADS / LPT) * (K5_THREADS / LPT);
    for (int tok = threadIdx.x / LPT; tok < len_up; tok += K5_THREADS / LPT) {
      const int tt = min(tok, len - 1);  // whole LPT groups stay convergent for the shuffles
      if (len > 0) {
        const int code = __ldg(codes + o0 + tt);
        // duplicate writes of the last row by the padding groups store identical bytes
        decompress_slice<D, NBITS, LPT>(lut, residuals, C, norms, o0 + tt, code, threadIdx.x % LPT, out + (oo + tt) * D);
      }
    }
  }
}

// token matrices (search.rs:668-686): ts[pair][t][q] for explicit (query, doc) pairs.
template <int D, int NBITS>
__global__ void __launch_bounds__(K5_THREADS)
k5_token_scores_kernel(const __half* __restrict__ C, const int64_t* __restrict__ doc_offsets,
                       const int32_t* __restrict__ codes, const uint8_t* __restrict__ residuals,
                       const __half* __restrict__ norms, WPerm wp,
                       const __half* __restrict__ queries, int Q, const int32_t* __restrict__ query_of,
                       const int32_t* __restrict__ doc_ids, int n, int64_t max_len, __half* __restrict__ out) {
  // Simple CUDA-core formulation (this is an off-metric by-product): one token per LPT lanes,
  // the dot products are accumulated in fp32 in index order and rounded once to fp16.
  constexpr int LPT = lanes_per_token<D, NBITS>();
  constexpr int EPL = D / LPT;
  __shared__ uint32_t lut[512];
  __shared__ __align__(16) __half row[K5_THREADS / LPT][D + 8];
  Decoder<NBITS>::build(lut, wp, threadIdx.x, K5_THREADS);
  __syncthreads();
  const int grp = threadIdx.x / LPT, sub = threadIdx.x % LPT;
  for (int i = blockIdx.x; i < n; i += gridDim.x) {
    const int d = doc_ids[i];
    const __half* qb = queries + int64_t(query_of[i]) * Q * D;
    const int64_t o0 = doc_offsets[d];
    const int len = int(doc_offsets[d + 1] - o0);
    if (len <= 0) continue;
    const int step = K5_THREADS / LPT;
    const int len_up = (len + step - 1) / step * step;
    for (int tok = grp; tok < len_up; tok += step) {
      const int tt = min(tok, len - 1);
      const int code = __ldg(codes + o0 + tt);
      decompress_slice<D, NBITS, LPT>(lut, residuals, C, norms, o0 + tt, code, sub, &row[grp][0]);
      __syncwarp();
      if (tok < len) {
        for (int q = sub; q < Q; q += LPT) {
          float acc = 0.f;
          for (int k = 0; k < D; ++k) acc = __fmaf_rn(__half2float(row[grp][k]), __half2float(qb[int64_t(q) * D + k]), acc);
          out[(int64_t(i) * max_len + tok) * Q + q] = __float2half_rn(acc);
        }
      }
      __syncwarp();
    }
    (void)EPL;
  }
}

// The per-token norm table (fpb_index_create): one token per LPT lanes.
template <int D, int NBITS>
__global__ void __launch_bounds__(K5_THREADS)
k5_token_norms_kernel(const __half* __restrict__ C, const int32_t* __restrict__ codes,
                      const uint8_t* __restrict__ residuals, WPerm wp, int64_t n_tokens, __half* __restrict__ out) {
  constexpr int LPT = lanes_per_token<D, NBITS>();
  __shared__ uint32_t lut[512];
  Decoder<NBITS>::build(lut, wp, threadIdx.x, K5_THREADS);
  __syncthreads();
  const int sub = threadIdx.x % LPT;
  const int64_t per_cta = K5_THREADS / LPT;
  const int64_t n_up = (n_tokens + per_cta - 1) / per_cta * per_cta;  // whole LPT groups stay convergent for the shuffles
  for (int64_t t = int64_t(blockIdx.x) * per_cta + threadIdx.x / LPT; t < n_up; t += int64_t(gridDim.x) * per_cta) {
    const int64_t tt = t < n_tokens ? t : n_tokens - 1;
    const __half nrm = token_norm<D, NBITS, LPT>(lut, residuals, C, tt, __ldg(codes + tt), sub);
    if (sub == 0 && t < n_tokens) out[t] = nrm;
  }
}

template <int D, int NBITS, int QP>
int launch_k5_t(const fpb_index* ix, const Ws& ws, cudaStream_t st) {
  const fpb_layout& L = *ws.L;
  auto kern = k5_maxsim_kernel<D, NBITS, QP>;
  constexpr int smem = K5Smem<D, QP>::bytes;
  // opt in on every launch: the attribute is per device and the call costs about a microsecond
  FPB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const int64_t items = int64_t(L.B) * L.R;
  const int blocks = int(items < int64_t(ix->sm_count) * 8 ? items : int64_t(ix->sm_count) * 8);
  kern<<<blocks, K5_THREADS, smem, st>>>(ix->centroids, ix->doc_offsets, ix->doc_codes, ix->doc_residuals, ix->token_norms,
                                         ix->w_perm, ws.queries(), L.Q, L.B, L.R, ws.n_rerank(), ws.rerank(), ws.exact());
  FPB_LAUNCH_CHECK("k5_maxsim");
  return FPB_OK;
}

template <int D, int NBITS>
int launch_k5_q(const fpb_index* ix, const Ws& ws, cudaStream_t st) {
  switch (ws.L->Qp) {
    case 16: return launch_k5_t<D, NBITS, 16>(ix, ws, st);
    case 32: return launch_k5_t<D, NBITS, 32>(ix, ws, st);
    case 64: return launch_k5_t<D, NBITS, 64>(ix, ws, st);
    case 128: return launch_k5_t<D, NBITS, 128>(ix, ws, st);
    case 256: return launch_k5_t<D, NBITS, 256>(ix, ws, st);
    default:
      fpb_set_error("maxsim: unsupported padded query length %d", ws.L->Qp);
      return FPB_ERR_UNSUPPORTED;
  }
}

// The K5 variant of a launch, the whole rule.  v4 and v5 decode dim 128 / nbits 4 only: v4 (register-resident
// operands, mma.sync) takes Qp <= 32, v5 (wgmma) 32 < Qp <= 128 when a document's 8-token passes fit its pass table.
// Everything else (other codecs, Qp = 256, an index whose longest document is empty or longer than the pass table)
// takes the generic kernel, as does FPB_K5=v1 (the A/B alternative).
enum class K5Kernel { generic, v4, v5 };
K5Kernel k5_kernel(const fpb_index* ix, const fpb_layout& L) {
  if (fpb_env_is("FPB_K5", "v1") || ix->dim != 128 || ix->nbits != 4) return K5Kernel::generic;
  if (L.Qp <= 32) return K5Kernel::v4;
  const int64_t passes_per_doc = (ix->max_doc_len + 7) / 8;
  if (L.Qp <= 128 && passes_per_doc >= 1 && passes_per_doc <= V5_MAX_PASS) return K5Kernel::v5;
  return K5Kernel::generic;
}

}  // namespace

int launch_token_norms(const fpb_index* ix, __half* d_out, cudaStream_t st) {
  const int blocks = ix->sm_count * 8;
  return fpb_with_codec(ix->dim, ix->nbits, "token norms", [&](auto c) {
    k5_token_norms_kernel<c.D, c.NBITS><<<blocks, K5_THREADS, 0, st>>>(ix->centroids, ix->doc_codes,
                                                                       ix->doc_residuals, ix->w_perm, ix->E, d_out);
    FPB_LAUNCH_CHECK("k5_token_norms");
    return FPB_OK;
  });
}

int launch_maxsim(const fpb_index* ix, const Ws& ws, cudaStream_t st) {
  switch (k5_kernel(ix, *ws.L)) {
    case K5Kernel::v4: return launch_maxsim_v4(ix, ws, st);
    case K5Kernel::v5: return launch_maxsim_v5(ix, ws, st);
    case K5Kernel::generic: break;
  }
  return fpb_with_codec(ix->dim, ix->nbits, "maxsim", [&](auto c) { return launch_k5_q<c.D, c.NBITS>(ix, ws, st); });
}

extern "C" int fpb_reconstruct(const fpb_index* ix, const int32_t* d_doc_ids, int n,
                               const int64_t* d_out_offsets, void* d_out, void* stream) {
  if (!ix || n < 0) {
    fpb_set_error("fpb_reconstruct: bad arguments");
    return FPB_ERR_INVALID;
  }
  if (n == 0) return FPB_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int blocks = min(n, ix->sm_count * 8);
  return fpb_with_codec(ix->dim, ix->nbits, "fpb_reconstruct", [&](auto c) {
    k5_reconstruct_kernel<c.D, c.NBITS><<<blocks, K5_THREADS, 0, st>>>(
        ix->centroids, ix->doc_offsets, ix->doc_codes, ix->doc_residuals, ix->token_norms, ix->w_perm, d_doc_ids, n,
        d_out_offsets, static_cast<__half*>(d_out));
    FPB_LAUNCH_CHECK("k5_reconstruct");
    return FPB_OK;
  });
}

extern "C" int fpb_token_scores(const fpb_index* ix, const void* d_queries, int Q, const int32_t* d_query_of,
                                const int32_t* d_doc_ids, int n, int64_t max_len, void* d_out, void* stream) {
  if (!ix || n < 0 || Q <= 0) {
    fpb_set_error("fpb_token_scores: bad arguments");
    return FPB_ERR_INVALID;
  }
  if (n == 0) return FPB_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int blocks = min(n, ix->sm_count * 8);
  return fpb_with_codec(ix->dim, ix->nbits, "fpb_token_scores", [&](auto c) {
    k5_token_scores_kernel<c.D, c.NBITS><<<blocks, K5_THREADS, 0, st>>>(
        ix->centroids, ix->doc_offsets, ix->doc_codes, ix->doc_residuals, ix->token_norms, ix->w_perm,
        static_cast<const __half*>(d_queries), Q, d_query_of, d_doc_ids, n, max_len, static_cast<__half*>(d_out));
    FPB_LAUNCH_CHECK("k5_token_scores");
    return FPB_OK;
  });
}
