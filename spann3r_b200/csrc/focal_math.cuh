// Scalar pieces of the 'median' focal estimate (dust3r/post_process.py:26-36): the per-pixel focal votes and the
// order-preserving integer key of a float, `__host__ __device__` so that tests/native/focal_host_check.cpp can pin the
// arithmetic on the CPU (bit-exact against the real reference function) -- the library only calls it from kernels.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define S3R_FHD __host__ __device__ __forceinline__
#else
#define S3R_FHD inline
#endif

namespace s3r {
namespace focal {

// vote j of one image: j < hw -> fx vote (u * z) / x of pixel j, else fy vote (v * z) / y of pixel j - hw, with
// (u, v) = (column - ppx, row - ppy); fp32, IEEE multiply then divide exactly like the reference's tensor expression.
S3R_FHD float vote(const float* pts, long long j, long long hw, int W, float ppx, float ppy) {
  const bool second = j >= hw;
  const long long i = second ? j - hw : j;
  const float z = pts[3 * i + 2];
  if (!second) {
    const float u = (float)(i % W) - ppx;
    const float m = u * z;
    return m / pts[3 * i];
  }
  const float v = (float)(i / W) - ppy;
  const float m = v * z;
  return m / pts[3 * i + 1];
}

S3R_FHD uint32_t float_bits(float f) {
#if defined(__CUDA_ARCH__)
  return __float_as_uint(f);
#else
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
#endif
}
S3R_FHD float bits_float(uint32_t u) {
#if defined(__CUDA_ARCH__)
  return __uint_as_float(u);
#else
  float f;
  memcpy(&f, &u, 4);
  return f;
#endif
}
// ascending float order == ascending unsigned key order (-inf lowest, +inf highest); -0.0 sorts just below +0.0, which
// is immaterial for a value-level median
S3R_FHD uint32_t order_key(float f) {
  const uint32_t u = float_bits(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
S3R_FHD float key_value(uint32_t k) { return bits_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// one digit of an 8-bit radix select: the bin of the 256-bin histogram that holds the element of rank k (0-based,
// ascending); k becomes that element's rank inside the bin.  Ranks beyond the total land in bin 255.
S3R_FHD int radix_pick(const int* hist, long long& k) {
  int bin = 0;
  while (bin < 255 && k >= hist[bin]) k -= hist[bin++];
  return bin;
}

}  // namespace focal
}  // namespace s3r
