// Block-level exclusive scan shared by the count -> scan -> ordered-write kernels (csrc/mesh.cu, csrc/poisson.cu).
#pragma once
#include <cuda_runtime.h>

namespace s3r {

// Exclusive block scan of one value per thread (blockDim.x == NT, a multiple of 32); *total gets the block's sum.
template <int NT>
__device__ long long block_exclusive_scan(long long v, long long* total) {
  __shared__ long long warp_sums[NT / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long x = v;
  for (int o = 1; o < 32; o <<= 1) {
    const long long y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[warp] = x;
  __syncthreads();
  if (warp == 0) {
    long long s = lane < NT / 32 ? warp_sums[lane] : 0;
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    if (lane < NT / 32) warp_sums[lane] = s;   // inclusive over warps
  }
  __syncthreads();
  const long long before = warp ? warp_sums[warp - 1] : 0;
  *total = warp_sums[NT / 32 - 1];
  __syncthreads();   // warp_sums may be reused by the next call
  return before + x - v;
}

}  // namespace s3r
