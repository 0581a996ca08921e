// Index-build encode kernels (SURVEY.md 8(f-1); replaces the per-batch closure of create_index,
// rust/index/create.rs:404-428):
//   * assign : code[t] = argmax_k fp16(<x_t, c_k>)  (compress_into_codes, create.rs:148-170) on
//              the warpgroup MMA -- the K1 v2 pipeline (TMA-fed centroid tiles, register
//              accumulators) with an argmax epilogue instead of the S store; ties -> smallest
//              centroid id, which is what ATen's CPU argmax returns
//   * pack   : residual = fp16(x - c[code]); bucket = #cutoffs < residual (bucketize right=false,
//              create.rs:413-414); each index written LSB-first into nbits bits, bits packed
//              big-endian per byte (create.rs:416-427, packbits :176-184)
#include <cuda.h>
#include <string.h>

#include "kernels.h"
#include "wgmma.cuh"

namespace {

constexpr int EN_THREADS = 288;
constexpr int EN_PRODUCER_WARP = 8;
constexpr int EN_STAGES = 3;
constexpr int EN_KBLOCK = 128 * 128;
constexpr int EN_TILE = 2 * EN_KBLOCK;

struct EnSmem {
  static constexpr int a_off = 0;
  static constexpr int b_off = EN_TILE;
  static constexpr int bar_off = b_off + EN_STAGES * EN_TILE;
  static constexpr int bytes = bar_off + 256 + 1024;
};

// KMEANS = false: code = argmax_k fp16(<x, c_k>)                      (index-build encode)
// KMEANS = true : code = argmax_k (<x, c_k> + bias[k]) in fp32, bias[k] = -|c_k|^2 / 2, i.e. the nearest centroid
//                 by squared distance (the assignment step of Lloyd's algorithm, kmeans.py:153-160)
// 288 threads: warpgroups 0-1 each own 64 token rows of the 128-token tile (wgmma.m64n128k16 on the shared
// centroid stage, accumulators in registers, running argmax per row), warp 8 streams the centroid tiles by TMA.
template <bool KMEANS>
__global__ void __launch_bounds__(EN_THREADS, 1)
encode_assign_kernel(const __grid_constant__ CUtensorMap tmap_c, int K, const __half* __restrict__ X, int64_t n,
                     int32_t* __restrict__ codes, int n_ctiles, const float* __restrict__ bias) {
  extern __shared__ unsigned char smem_dyn[];
  const uint32_t dyn_addr = smem_u32(smem_dyn);
  unsigned char* base = smem_dyn + ((1024u - (dyn_addr & 1023u)) & 1023u);
  unsigned char* smA = base + EnSmem::a_off;
  unsigned char* smB = base + EnSmem::b_off;
  uint64_t* bars = reinterpret_cast<uint64_t*>(base + EnSmem::bar_off);
  const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + EN_STAGES);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  if (tid == 0) {
    for (int s = 0; s < EN_STAGES; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, 8);  // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int64_t n_ttiles = (n + 127) / 128;
  uint32_t it = 0;  // centroid tiles streamed so far by this CTA (pipeline state persists across token tiles)
  for (int64_t tt = blockIdx.x; tt < n_ttiles; tt += gridDim.x) {
    __syncthreads();  // every role is done with the previous token tile (A tile can be replaced)
    for (int i = tid; i < 128 * 16; i += EN_THREADS) {
      const int r = i >> 4, c = i & 15;
      const int64_t tok = tt * 128 + r;
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (tok < n) v = __ldg(reinterpret_cast<const uint4*>(X + tok * 128) + c);
      *reinterpret_cast<uint4*>(smA + sw128_off(r, c, EN_KBLOCK)) = v;
    }
    fence_proxy_async();
    __syncthreads();

    if (warp == EN_PRODUCER_WARP) {
      if (lane == 0) {
        for (int i = 0; i < n_ctiles; ++i) {
          const uint32_t g = it + i;
          const int stage = g % EN_STAGES;
          mbar_wait(bar_empty + 8 * stage, ((g / EN_STAGES) & 1) ^ 1);
          const uint32_t dst = smem_u32(smB + stage * EN_TILE);
          const uint32_t bar = bar_full + 8 * stage;
          mbar_arrive_expect_tx(bar, uint32_t(EN_TILE));
#pragma unroll
          for (int kb = 0; kb < 2; ++kb) tma_load_2d(dst + kb * EN_KBLOCK, &tmap_c, kb * 64, i * 128, bar);
        }
      }
      __syncwarp();
    } else {
      const int wg = warp >> 2, w = warp & 3, quad = lane & 3;
      const uint32_t a_addr = smem_u32(smA) + wg * 8 * 1024;  // token rows 64 wg .. 64 wg + 63
      float best[2] = {-INFINITY, -INFINITY};
      int best_k[2] = {0, 0};
      for (int i = 0; i < n_ctiles; ++i) {
        const uint32_t g = it + i;
        const int stage = g % EN_STAGES;
        const int k0 = i * 128;
        const int rows_valid = min(128, K - k0);
        float acc[64];
        mbar_wait(bar_full + 8 * stage, (g / EN_STAGES) & 1);
        const uint32_t b_addr = smem_u32(smB + stage * EN_TILE);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
          const uint32_t off = (ks >> 2) * EN_KBLOCK + (ks & 3) * 32;
          wgmma_m64n128k16(acc, gmma_desc(a_addr + off), gmma_desc(b_addr + off), ks > 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait0();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + 8 * stage);
        // columns visited in increasing centroid order per thread: the first maximum wins
#pragma unroll
        for (int j = 0; j < 16; ++j) {
#pragma unroll
          for (int x = 0; x < 2; ++x) {
            const int c = 8 * j + 2 * quad + x;
            const float bc = KMEANS && c < rows_valid ? __ldg(bias + k0 + c) : 0.f;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              // encode: the reference compares fp16 scores (half matmul output)
              const float a = acc[4 * j + 2 * h + x];
              const float v = KMEANS ? a + bc : __half2float(__float2half_rn(a));
              if (c < rows_valid && v > best[h]) {
                best[h] = v;
                best_k[h] = k0 + c;
              }
            }
          }
        }
      }
      // merge the four lanes of a row: larger score, ties -> smaller centroid id (ATen's CPU argmax)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int off = 1; off <= 2; off <<= 1) {
          const float ob = __shfl_xor_sync(0xffffffffu, best[h], off);
          const int ok = __shfl_xor_sync(0xffffffffu, best_k[h], off);
          if (ob > best[h] || (ob == best[h] && ok < best_k[h])) {
            best[h] = ob;
            best_k[h] = ok;
          }
        }
        const int64_t tok = tt * 128 + 64 * wg + 16 * w + (lane >> 2) + 8 * h;
        if (quad == 0 && tok < n) codes[tok] = best_k[h];
      }
    }
    it += uint32_t(n_ctiles);
  }
}

// residual = fp16(x - c[code]) -> bucket index -> packed bits.  One thread per output byte.
template <int NBITS>
__global__ void encode_pack_kernel(const __half* __restrict__ X, const __half* __restrict__ C,
                                   const int32_t* __restrict__ codes, const float* __restrict__ cutoffs, int64_t n,
                                   int dim, uint8_t* __restrict__ out) {
  constexpr int PER = 8 / NBITS;       // elements per byte
  constexpr int NCUT = (1 << NBITS) - 1;
  __shared__ float cut[NCUT];
  if (threadIdx.x < NCUT) cut[threadIdx.x] = cutoffs[threadIdx.x];
  __syncthreads();
  const int pd = dim / PER;
  const int64_t total = n * pd;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t t = i / pd;
    const int j = int(i % pd);
    const __half* x = X + t * dim + j * PER;
    const __half* c = C + int64_t(codes[t]) * dim + j * PER;
    uint32_t byte = 0;
#pragma unroll
    for (int e = 0; e < PER; ++e) {
      const float r = __half2float(__hsub(x[e], c[e]));  // one fp16 subtraction, like the reference
      int b = 0;
#pragma unroll
      for (int k = 0; k < NCUT; ++k) b += (cut[k] < r) ? 1 : 0;  // bucketize(right=false)
      uint32_t rev = 0;  // LSB-first bit order inside the element's field
#pragma unroll
      for (int k = 0; k < NBITS; ++k) rev |= ((uint32_t(b) >> k) & 1u) << (NBITS - 1 - k);
      byte |= rev << (8 - NBITS * (e + 1));
    }
    out[i] = uint8_t(byte);
  }
}

typedef CUresult (*en_encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                       const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                       CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

}  // namespace

// tensor map of the centroid table + launch of the assign kernel (shared by fpb_encode and fpb_kmeans_assign)
static int launch_assign(int device, int64_t n_centroids, const void* d_centroids, const void* d_tokens,
                         int64_t n_tokens, int32_t* d_codes, const float* d_bias, cudaStream_t st, const char* who) {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn ||
      qres != cudaDriverEntryPointSuccess) {
    fpb_set_error("%s: cuTensorMapEncodeTiled is not available from this driver", who);
    return FPB_ERR_CUDA;
  }
  CUtensorMap tm;
  const cuuint64_t gdim[2] = {128, cuuint64_t(n_centroids)};
  const cuuint64_t gstride[1] = {256};
  const cuuint32_t box[2] = {64, 128};
  const cuuint32_t estr[2] = {1, 1};
  if (reinterpret_cast<en_encode_tiled_fn>(fn)(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(d_centroids),
                                               gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) {
    fpb_set_error("%s: cuTensorMapEncodeTiled failed", who);
    return FPB_ERR_CUDA;
  }
  cudaDeviceProp prop;
  FPB_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
  const int64_t n_ttiles = (n_tokens + 127) / 128;
  const int blocks = int(n_ttiles < prop.multiProcessorCount ? n_ttiles : prop.multiProcessorCount);
  const int n_ctiles = int((n_centroids + 127) / 128);
  // opt in on every launch: the attribute is per device and the call costs about a microsecond
  if (d_bias) {
    FPB_CUDA_CHECK(cudaFuncSetAttribute(encode_assign_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, EnSmem::bytes));
    encode_assign_kernel<true><<<blocks, EN_THREADS, EnSmem::bytes, st>>>(tm, int(n_centroids),
                                                                         static_cast<const __half*>(d_tokens), n_tokens,
                                                                         d_codes, n_ctiles, d_bias);
  } else {
    FPB_CUDA_CHECK(cudaFuncSetAttribute(encode_assign_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, EnSmem::bytes));
    encode_assign_kernel<false><<<blocks, EN_THREADS, EnSmem::bytes, st>>>(tm, int(n_centroids),
                                                                          static_cast<const __half*>(d_tokens), n_tokens,
                                                                          d_codes, n_ctiles, nullptr);
  }
  FPB_LAUNCH_CHECK("encode_assign");
  return FPB_OK;
}

// Centroid update of Lloyd's algorithm as a deterministic segmented mean: `order` lists the point indices sorted by
// assigned centroid, `seg_offsets[k] .. seg_offsets[k+1]` is centroid k's segment.  One warp per centroid, each lane
// sums four dimensions in fp32 in segment order; empty segments leave the output row untouched and count 0.
__global__ void __launch_bounds__(256)
segment_mean_kernel(const __half* __restrict__ X, const int64_t* __restrict__ order,
                    const int64_t* __restrict__ seg_offsets, int64_t K, __half* __restrict__ out,
                    float* __restrict__ shift) {
  const int lane = threadIdx.x & 31;
  const int64_t k = int64_t(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (k >= K) return;
  const int64_t s0 = seg_offsets[k], s1 = seg_offsets[k + 1];
  if (s1 <= s0) return;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  for (int64_t i = s0; i < s1; ++i) {
    const uint2 v = __ldg(reinterpret_cast<const uint2*>(X + order[i] * 128) + lane);
    const float2 f0 = __half22float2(u32_as_half2(v.x)), f1 = __half22float2(u32_as_half2(v.y));
    a0 += f0.x; a1 += f0.y; a2 += f1.x; a3 += f1.y;
  }
  const float inv = 1.0f / float(s1 - s0);
  const __half2 h0 = __floats2half2_rn(a0 * inv, a1 * inv), h1 = __floats2half2_rn(a2 * inv, a3 * inv);
  uint2* dst = reinterpret_cast<uint2*>(out + k * 128) + lane;
  if (shift) {  // |new - old| of this centroid, for the convergence test (kmeans.py:213-218)
    const uint2 old = *dst;
    const float2 o0 = __half22float2(u32_as_half2(old.x)), o1 = __half22float2(u32_as_half2(old.y));
    const float2 n0 = __half22float2(h0), n1 = __half22float2(h1);
    float d = (n0.x - o0.x) * (n0.x - o0.x) + (n0.y - o0.y) * (n0.y - o0.y) + (n1.x - o1.x) * (n1.x - o1.x) +
              (n1.y - o1.y) * (n1.y - o1.y);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) d += __shfl_xor_sync(0xffffffffu, d, off);
    if (lane == 0) shift[k] = sqrtf(d);
  }
  *dst = make_uint2(half2_as_u32(h0), half2_as_u32(h1));
}

extern "C" int fpb_kmeans_assign(int device, int dim, int64_t n_centroids, const void* d_centroids,
                                 const float* d_bias, const void* d_points, int64_t n_points, int32_t* d_assign,
                                 void* stream) {
  if (dim != 128) {
    fpb_set_error("fpb_kmeans_assign: this build handles dim=128 (got %d)", dim);
    return FPB_ERR_UNSUPPORTED;
  }
  if (!d_centroids || !d_bias || !d_points || !d_assign || n_centroids < 1 || n_points < 0) {
    fpb_set_error("fpb_kmeans_assign: bad arguments");
    return FPB_ERR_INVALID;
  }
  if (n_points == 0) return FPB_OK;
  FPB_CUDA_CHECK(cudaSetDevice(device));
  return launch_assign(device, n_centroids, d_centroids, d_points, n_points, d_assign, d_bias,
                       static_cast<cudaStream_t>(stream), "fpb_kmeans_assign");
}

extern "C" int fpb_kmeans_update(int device, int dim, int64_t n_centroids, const void* d_points,
                                 const int64_t* d_order, const int64_t* d_seg_offsets, void* d_centroids,
                                 float* d_shift, void* stream) {
  if (dim != 128) {
    fpb_set_error("fpb_kmeans_update: this build handles dim=128 (got %d)", dim);
    return FPB_ERR_UNSUPPORTED;
  }
  if (!d_points || !d_order || !d_seg_offsets || !d_centroids || n_centroids < 1) {
    fpb_set_error("fpb_kmeans_update: bad arguments");
    return FPB_ERR_INVALID;
  }
  FPB_CUDA_CHECK(cudaSetDevice(device));
  segment_mean_kernel<<<unsigned((n_centroids + 7) / 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __half*>(d_points), d_order, d_seg_offsets, n_centroids, static_cast<__half*>(d_centroids),
      d_shift);
  FPB_LAUNCH_CHECK("segment_mean");
  return FPB_OK;
}

extern "C" int fpb_encode(int device, int nbits, int dim, int64_t n_centroids, const void* d_centroids,
                          const void* d_tokens, int64_t n_tokens, const float* d_cutoffs, int32_t* d_codes,
                          uint8_t* d_residuals, void* stream) {
  if (dim != 128 || !fpb_codec_supported(dim, nbits)) {
    fpb_set_error("fpb_encode: this build encodes dim=128 with nbits 2 or 4, and dim=128 with nbits 1 (got dim=%d nbits=%d)",
                  dim, nbits);
    return FPB_ERR_UNSUPPORTED;
  }
  if (!d_centroids || !d_tokens || !d_cutoffs || !d_codes || !d_residuals || n_centroids < 1 || n_tokens < 0) {
    fpb_set_error("fpb_encode: bad arguments");
    return FPB_ERR_INVALID;
  }
  if (n_tokens == 0) return FPB_OK;
  FPB_CUDA_CHECK(cudaSetDevice(device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  {
    const int rc = launch_assign(device, n_centroids, d_centroids, d_tokens, n_tokens, d_codes, nullptr, st, "fpb_encode");
    if (rc != FPB_OK) return rc;
  }
  const int pd = dim * nbits / 8;
  const int64_t total = n_tokens * pd;
  const int pblocks = int(((total + 255) / 256) < 65535 * 16 ? ((total + 255) / 256) : 65535 * 16);
  return fpb_with_codec(dim, nbits, "fpb_encode", [&](auto c) {
    encode_pack_kernel<c.NBITS><<<pblocks, 256, 0, st>>>(static_cast<const __half*>(d_tokens),
                                                         static_cast<const __half*>(d_centroids), d_codes, d_cutoffs,
                                                         n_tokens, dim, d_residuals);
    FPB_LAUNCH_CHECK("encode_pack");
    return FPB_OK;
  });
}
