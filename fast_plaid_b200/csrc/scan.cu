// The offsets scan shared by the inverted-file merge (append.cu) and the compactions of a delete (delete.cu).
#include "kernels.h"

namespace {

// One block: out[c + 1] = old[c + 1] + (count of entries <= c), out[0] = 0, and cursor[c] = out[c + 1] - count[c].
// old == NULL reads as zeros (a plain inclusive scan into out[1..]); cursor may be NULL.
__global__ void __launch_bounds__(1024)
offsets_scan_kernel(const int64_t* __restrict__ old_offsets, const int64_t* __restrict__ count, int64_t n,
                    int64_t* __restrict__ out, int64_t* __restrict__ cursor) {
  __shared__ int64_t s_warp[32];
  __shared__ int64_t s_carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    s_carry = 0;
    out[0] = 0;
  }
  __syncthreads();
  for (int64_t c0 = 0; c0 < n; c0 += 1024) {
    const int64_t c = c0 + threadIdx.x;
    const int64_t v = c < n ? count[c] : 0;
    int64_t incl = v;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int64_t u = __shfl_up_sync(0xffffffffu, incl, off);
      if (lane >= off) incl += u;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int64_t w = s_warp[lane];
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int64_t u = __shfl_up_sync(0xffffffffu, w, off);
        if (lane >= off) w += u;
      }
      s_warp[lane] = w;
    }
    __syncthreads();
    const int64_t before = s_carry + (warp > 0 ? s_warp[warp - 1] : 0) + incl - v;  // entries < c
    if (c < n) {
      const int64_t base = old_offsets ? old_offsets[c + 1] : 0;
      out[c + 1] = base + before + v;
      if (cursor) cursor[c] = base + before;
    }
    __syncthreads();
    if (threadIdx.x == 0) s_carry += s_warp[31];
    __syncthreads();
  }
}

}  // namespace

int launch_offsets_scan(const int64_t* old_offsets, const int64_t* count, int64_t n, int64_t* out, int64_t* cursor,
                        cudaStream_t st) {
  offsets_scan_kernel<<<1, 1024, 0, st>>>(old_offsets, count, n, out, cursor);
  FPB_LAUNCH_CHECK("offsets_scan");
  return FPB_OK;
}
