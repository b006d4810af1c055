// Input adapter on the GPU (SURVEY.md section 8f rank 3): the reference's per-frame preprocessing between the decoded
// RGB image and the network input -- centre crop, PIL Lanczos down-scale, centred crop, ToTensor + Normalize(0.5, 0.5)
// (spann3r/datasets/demo.py:57-86 -> dust3r/datasets/base/base_stereo_view_dataset.py:143-194 ->
// dust3r/datasets/utils/cropping.py:55-124 -> dust3r/utils/image.py:23).  The down-scale is Pillow's 8-bit separable
// resampler (src/libImaging/Resample.c: ImagingResampleHorizontal_8bpc / Vertical_8bpc): integer arithmetic, 22-bit
// fixed-point coefficients, uint8 intermediate -- reproduced BIT-EXACTLY here; the coefficient tables come from the host
// (spann3r_b200/preprocess.py, Pillow's precompute_coeffs).  Both crops are folded into the passes: only the rows /
// columns that survive the final crop are ever computed.
//
// HBM-bound byte work: one read of the crop of the source image, one small uint8 intermediate, one fp32 write.
#include "../../include/spann3r_b200.h"
#include "gemm.cuh"

#include "common.cuh"
#include "resample_u8.cuh"

namespace s3r {

// Horizontal pass.  Block = one source row x 128 output columns (resample_u8.cuh).
// src: RGB rows of `row_stride` bytes, first needed row / column already applied by the caller through the pointer and
// the bounds; bounds[x] = (first source column, tap count), kk[x][ksize] fixed-point taps.
__global__ void __launch_bounds__(128) resample_h_u8_kernel(const uint8_t* __restrict__ src, long long row_stride,
                                                            int out_cols, const int* __restrict__ bounds,
                                                            const int* __restrict__ kk, int ksize,
                                                            uint8_t* __restrict__ dst) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ uint8_t span[];
  const int row = blockIdx.y;
  resample_h_u8_block(src + (long long)row * row_stride, out_cols, blockIdx.x * 128, bounds, kk, ksize, span,
                      dst + (long long)row * out_cols * 3);
}

// Vertical pass + ToTensor + Normalize: thread = one byte column of the intermediate (x * 3 + c, coalesced across the
// warp), block row = one output row.  dst [3, out_rows, cols] fp32.
__global__ void __launch_bounds__(256) resample_v_u8_norm_kernel(const uint8_t* __restrict__ tmp, int cols,
                                                                 int out_rows, const int* __restrict__ bounds,
                                                                 const int* __restrict__ kk, int ksize,
                                                                 float* __restrict__ dst) {
  pdl_launch_dependents();
  pdl_wait();
  const int j = blockIdx.x * 256 + threadIdx.x;   // byte column
  if (j >= cols * 3) return;
  const int x = j / 3, c = j - 3 * x;
  const int y = blockIdx.y;
  dst[((long long)c * out_rows + y) * cols + x] = resample_v_u8_norm_value(tmp, cols, j, y, bounds, kk, ksize);
}

}  // namespace s3r

using namespace s3r;

extern "C" {

int s3r_resample_h_u8(const uint8_t* src, int64_t row_stride, int rows, int out_cols, const int32_t* bounds,
                      const int32_t* kk, int ksize, int max_span, uint8_t* dst, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (rows <= 0 || out_cols <= 0) return 0;
  const size_t smem = (size_t)3 * max_span;
  if (smem > 160 * 1024) {
    set_error("resample_h: source span of %d pixels per 128 output columns is too large", max_span);
    return -1;
  }
  static PerDeviceOnce once;
  if (smem > 48 * 1024 && !once.cur()) {
    cudaFuncSetAttribute(resample_h_u8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
    once.cur() = true;
  }
  launch_pdl(resample_h_u8_kernel, dim3((out_cols + 127) / 128, rows), dim3(128), smem, st, src, row_stride, out_cols, bounds,
             kk, ksize, dst);
  return cudaGetLastError() == cudaSuccess ? 0 : -6;
}

int s3r_resample_v_u8_norm(const uint8_t* tmp, int cols, int out_rows, const int32_t* bounds, const int32_t* kk,
                           int ksize, float* dst, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (out_rows <= 0 || cols <= 0) return 0;
  launch_pdl(resample_v_u8_norm_kernel, dim3((cols * 3 + 255) / 256, out_rows), dim3(256), 0, st, tmp, cols, out_rows,
             bounds, kk, ksize, dst);
  return cudaGetLastError() == cudaSuccess ? 0 : -6;
}

}  // extern "C"
