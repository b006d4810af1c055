// Pillow's 8-bit separable Lanczos passes (src/libImaging/Resample.c: ImagingResampleHorizontal_8bpc / Vertical_8bpc),
// one output element at a time.  Shared by the single-frame kernels of preprocess.cu and the batched sequence kernels of
// views.cu, so that a view of a batch gets exactly the single-frame kernel's bits.
#pragma once
#include <cstdint>

namespace s3r {

constexpr int kPrec = 32 - 8 - 2;   // PRECISION_BITS of Resample.c

__device__ __forceinline__ int clip8(int v) {   // clip8(): (in >> PRECISION_BITS) clamped to [0, 255]
  v >>= kPrec;
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

// Horizontal pass of one block = one source row x 128 output columns starting at x0 (blockDim.x == 128).  The source
// span those columns need is staged in `span` (shared memory) with coalesced byte loads, then thread t computes output
// column x0 + t (3 channels).  srow: the row's first byte; bounds[x] = (first source column, tap count), kk[x][ksize]
// fixed-point taps; drow: the output row [out_cols, 3].
__device__ __forceinline__ void resample_h_u8_block(const uint8_t* __restrict__ srow, int out_cols, int x0,
                                                    const int* __restrict__ bounds, const int* __restrict__ kk, int ksize,
                                                    uint8_t* span, uint8_t* __restrict__ drow) {
  const int xl = min(x0 + 127, out_cols - 1);
  const int s0 = bounds[2 * x0];                                  // first source column of the block's span
  const int s1 = bounds[2 * xl] + bounds[2 * xl + 1];             // one past the last
  const uint8_t* sp = srow + 3LL * s0;
  const int nbytes = 3 * (s1 - s0);
  for (int i = threadIdx.x; i < nbytes; i += 128) span[i] = sp[i];
  __syncthreads();
  const int x = x0 + threadIdx.x;
  if (x >= out_cols) return;
  const int b0 = bounds[2 * x] - s0, n = bounds[2 * x + 1];
  const int* k = kk + (long long)x * ksize;
  int a0 = 1 << (kPrec - 1), a1 = a0, a2 = a0;
  for (int i = 0; i < n; ++i) {
    const int c = __ldg(k + i);
    const uint8_t* p = span + 3 * (b0 + i);
    a0 += p[0] * c;
    a1 += p[1] * c;
    a2 += p[2] * c;
  }
  uint8_t* o = drow + 3LL * x;
  o[0] = (uint8_t)clip8(a0);
  o[1] = (uint8_t)clip8(a1);
  o[2] = (uint8_t)clip8(a2);
}

// Vertical pass of one byte column j (= x * 3 + c) of output row y of the uint8 intermediate tmp [*, cols, 3]: the
// uint8 value of the resized image.
__device__ __forceinline__ int resample_v_u8_value(const uint8_t* __restrict__ tmp, int cols, int j, int y,
                                                   const int* __restrict__ bounds, const int* __restrict__ kk, int ksize) {
  const int y0 = bounds[2 * y], n = bounds[2 * y + 1];
  const int* k = kk + (long long)y * ksize;
  const uint8_t* p = tmp + (long long)y0 * cols * 3 + j;
  int a = 1 << (kPrec - 1);
  for (int i = 0; i < n; ++i) a += (int)p[(long long)i * cols * 3] * __ldg(k + i);
  return clip8(a);
}

// ImgNorm (ToTensor + Normalize((0.5,) * 3, (0.5,) * 3)) of one uint8 value: ((v / 255) - 0.5) / 0.5 in fp32, the
// operation order of torchvision's ToTensor / Normalize.
__device__ __forceinline__ float img_norm_u8(int v) {
  const float f = (float)v / 255.0f;
  return (f - 0.5f) / 0.5f;
}

// Vertical pass + ImgNorm of one byte column j of output row y.
__device__ __forceinline__ float resample_v_u8_norm_value(const uint8_t* __restrict__ tmp, int cols, int j, int y,
                                                          const int* __restrict__ bounds, const int* __restrict__ kk,
                                                          int ksize) {
  return img_norm_u8(resample_v_u8_value(tmp, cols, j, y, bounds, kk, ksize));
}

}  // namespace s3r
