// K1 v2 : centroid scores S = fp16(C . q^T) on the Hopper warpgroup MMA (search.rs:491), dim = 128, Qp <= 128.
//
// GEMM view: D[token][centroid] = sum_k Qtok[token][k] * C[centroid][k] with M = 128 query tokens
// (A operand, resident for the CTA's lifetime), N = 128 centroids per tile (B operand, streamed
// through a 3-stage shared-memory ring in the K-major SWIZZLE_128B layout), K = 128.  Two consumer
// warpgroups each own 64 token rows: per tile they issue 8 wgmma.m64n128k16 on the same B stage and
// keep the fp32 accumulators in registers.  One accumulator row = one query token, so the
// per-128-centroid-tile maximum K1b needs is a per-row max over the columns (4 lanes share a row),
// and the fp16 tile is transposed through shared memory into [centroid][q] blocks that are
// contiguous in S[b][k][q] and leave with one bulk-async copy each
// (cp.async.bulk.global.shared::cta) -- the write of S never touches the LSU.
//
// The centroid tiles arrive by TMA (cp.async.bulk.tensor.2d with a SWIZZLE_128B tensor map): one
// elected thread of the producer warp arms the stage's mbarrier with the byte count and issues two
// 64-column boxes; rows past K are zero-filled by the TMA unit.
//
// 288 threads: warpgroups 0-1 MMA + epilogue, warp 8 TMA producer.
#include <cuda.h>
#include <string.h>

#include "kernels.h"
#include "wgmma.cuh"

namespace {

constexpr int G1_THREADS = 288;
constexpr int G1_PRODUCER_WARP = 8;
constexpr int G1_STAGES = 3;
constexpr int G1_KBLOCK = 128 * 128;      // bytes: 128 rows x 128 B
constexpr int G1_TILE = 2 * G1_KBLOCK;    // 32 KB operand tile (K = 128)
constexpr int G1_STAGING = 128 * 128 * 2;  // 32 KB fp16 output tile

struct G1Smem {
  static constexpr int a_off = 0;
  static constexpr int b_off = G1_TILE;
  static constexpr int st_off = b_off + G1_STAGES * G1_TILE;
  static constexpr int bar_off = st_off + 2 * G1_STAGING;
  static constexpr int bytes = bar_off + 256 + 1024;  // + slack for the 1024-byte alignment
};
static_assert(G1Smem::bytes <= 227 * 1024, "K1 v2 shared memory");

__global__ void __launch_bounds__(G1_THREADS, 1)
k1_centroid_v2_kernel(const __grid_constant__ CUtensorMap tmap_c, int K, const __half* __restrict__ Qpad, int B, int Qp,
                      __half* __restrict__ S, __half* __restrict__ tmax, int n_ctiles, int tiles_per_split) {
  extern __shared__ unsigned char smem_dyn[];
  const uint32_t dyn_addr = smem_u32(smem_dyn);
  unsigned char* base = smem_dyn + ((1024u - (dyn_addr & 1023u)) & 1023u);  // SWIZZLE_128B atoms are 1024 B
  unsigned char* smA = base + G1Smem::a_off;
  unsigned char* smB = base + G1Smem::b_off;
  unsigned char* smS = base + G1Smem::st_off;
  uint64_t* bars = reinterpret_cast<uint64_t*>(base + G1Smem::bar_off);
  const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + G1_STAGES);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tt = blockIdx.x;                      // token tile
  const int ct_begin = blockIdx.y * tiles_per_split;
  const int ct_end = min(n_ctiles, ct_begin + tiles_per_split);
  const int n_tokens = B * Qp;

  // ---- setup: A tile (128 query tokens), barriers ----
  for (int i = tid; i < 128 * 16; i += G1_THREADS) {
    const int r = i >> 4, c = i & 15;
    const int tok = tt * 128 + r;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (tok < n_tokens) v = *reinterpret_cast<const uint4*>(Qpad + int64_t(tok) * 128 + c * 8);
    *reinterpret_cast<uint4*>(smA + sw128_off(r, c, G1_KBLOCK)) = v;
  }
  fence_proxy_async();
  if (tid == 0) {
    for (int s = 0; s < G1_STAGES; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, 8);  // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  const int n_my = ct_end - ct_begin;

  if (warp == G1_PRODUCER_WARP) {
    // =========================== TMA producer: centroid tiles -> swizzled smem ===========================
    if (lane == 0) {
      for (int i = 0; i < n_my; ++i) {
        const int stage = i % G1_STAGES;
        mbar_wait(bar_empty + 8 * stage, ((i / G1_STAGES) & 1) ^ 1);
        const int k0 = (ct_begin + i) * 128;
        const uint32_t dst = smem_u32(smB + stage * G1_TILE);
        const uint32_t bar = bar_full + 8 * stage;
        mbar_arrive_expect_tx(bar, uint32_t(G1_TILE));
#pragma unroll
        for (int kb = 0; kb < 2; ++kb) tma_load_2d(dst + kb * G1_KBLOCK, &tmap_c, kb * 64, k0, bar);
      }
    }
    __syncwarp();
  } else {
    // =========================== MMA + epilogue (warpgroups 0, 1) ===========================
    const int wg = warp >> 2, w = warp & 3;
    const int quad = lane & 3;
    const uint32_t a_addr = smem_u32(smA) + wg * 8 * 1024;  // token rows 64 wg .. 64 wg + 63
    const int n_blk = 128 / Qp;                            // query blocks inside the token tile
    const uint32_t blk_bytes = uint32_t(128 * Qp * 2);
    int trow[2], tok[2];
    uint32_t my[2];  // byte offset of the row's (centroid 0, q) entry in a staging buffer
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      trow[h] = 64 * wg + 16 * w + (lane >> 2) + 8 * h;  // token row inside the tile == accumulator row
      tok[h] = tt * 128 + trow[h];
      my[h] = (trow[h] / Qp) * blk_bytes + (trow[h] % Qp) * 2;
    }
    for (int i = 0; i < n_my; ++i) {
      const int stage = i % G1_STAGES, sb = i & 1;
      const int ct = ct_begin + i;
      const int k0 = ct * 128;
      const int rows_valid = min(128, K - k0);
      float acc[64];
      mbar_wait(bar_full + 8 * stage, (i / G1_STAGES) & 1);
      const uint32_t b_addr = smem_u32(smB + stage * G1_TILE);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
        const uint32_t off = (ks >> 2) * G1_KBLOCK + (ks & 3) * 32;
        wgmma_m64n128k16(acc, gmma_desc(a_addr + off), gmma_desc(b_addr + off), ks > 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait0();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty + 8 * stage);  // stage reusable: this warp's MMAs have read it

      // the bulk stores issued from this staging buffer two tiles ago must have finished reading it
      if (tid < n_blk) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
      asm volatile("bar.sync 1, 256;" ::: "memory");
      unsigned char* stg = smS + sb * G1_STAGING;
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int j = 0; j < 16; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int h = e >> 1, c = 8 * j + 2 * quad + (e & 1);
          const float f = acc[4 * j + e];
          if (c < rows_valid) mx[h] = fmaxf(mx[h], f);
          *reinterpret_cast<__half*>(stg + my[h] + c * (Qp * 2)) = __float2half_rn(f);
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
        if (quad == 0 && tok[h] < n_tokens)
          tmax[int64_t(tok[h]) * n_ctiles + ct] = __float2half_rn(mx[h]);  // tok = b * Qp + q
      }
      fence_proxy_async();
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (tid < n_blk) {
        const int bb = (tt * 128) / Qp + tid;    // query of block `tid`
        if (bb < B) {
          const __half* dst = S + (int64_t(bb) * K + k0) * Qp;
          const uint32_t bytes = uint32_t(rows_valid * Qp * 2);
          asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst),
                       "r"(smem_u32(stg + tid * blk_bytes)), "r"(bytes)
                       : "memory");
        }
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      }
    }
    if (tid < n_blk) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  }
}

}  // namespace

// dim 128, Qp <= 128 and a TMA descriptor: k1_centroid.cu's rule launches v2 only there
int launch_centroid_scores_v2(const fpb_index* ix, const Ws& ws, cudaStream_t st) {
  const fpb_layout& L = *ws.L;
  // opt in on every launch: the attribute is per device and the call costs about a microsecond
  FPB_CUDA_CHECK(cudaFuncSetAttribute(k1_centroid_v2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, G1Smem::bytes));
  const int n_ttiles = (L.B * L.Qp + 127) / 128;
  const int n_ctiles = L.n_tiles;
  int splits = ix->sm_count / n_ttiles;
  if (splits < 1) splits = 1;
  if (splits > n_ctiles) splits = n_ctiles;
  const int per = (n_ctiles + splits - 1) / splits;
  splits = (n_ctiles + per - 1) / per;
  dim3 grid(n_ttiles, splits);
  CUtensorMap tm;
  memcpy(&tm, ix->tmap_centroids, sizeof(tm));
  k1_centroid_v2_kernel<<<grid, G1_THREADS, G1Smem::bytes, st>>>(tm, int(ix->K), ws.queries(), L.B, L.Qp,
                                                                ws.S(), ws.tmax(), n_ctiles, per);
  FPB_LAUNCH_CHECK("k1_centroid_v2");
  return FPB_OK;
}
