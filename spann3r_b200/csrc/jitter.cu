// Training views on the GPU (spann3r_b200/train_views.py): torchvision's ColorJitter on the PIL image the reference's
// training datasets hand it (dust3r/datasets/utils/transforms.py: Compose([ColorJitter(0.5, 0.5, 0.5, 0.1), ImgNorm])),
// bit for bit, for a whole batch of views per launch:
//   * views_resample_v_u8_kernel: the vertical Lanczos pass of views.cu, stopping at the uint8 image ColorJitter sees;
//   * views_color_jitter_kernel: one CTA per view applies the drawn ops in the drawn order (jitter_math.cuh), then
//     ImgNorm, and writes the view's img, transposed for portrait views.
// Contrast blends toward the mean L of the image the ops before it leave, so a view with contrast takes two passes over
// its pixels: the exact integer sum of L (a fixed-order block reduction), then every op.  The second pass recomputes
// the ops before contrast instead of storing the intermediate image; the source stays in shared memory when it fits.
#include "../../include/spann3r_b200.h"

#include "common.cuh"
#include "jitter_math.cuh"
#include "kernels.cuh"
#include "resample_u8.cuh"

namespace s3r {

constexpr int kJitThreads = 512;
constexpr size_t kJitSmemMax = 200 * 1024;   // a 224 x 224 view (147 KiB) stays on chip, a 512 x 384 one (576 KiB) not

// grid (256-byte-column blocks, output rows, views): views_resample_v_norm_kernel's body without ImgNorm.
__global__ void __launch_bounds__(256) views_resample_v_u8_kernel(const s3r_view_image_desc* __restrict__ descs,
                                                                  const s3r_view_jitter_desc* __restrict__ jit) {
  pdl_launch_dependents();
  pdl_wait();
  const s3r_view_image_desc& d = descs[blockIdx.z];
  const int cols = d.cols, out_rows = d.out_rows;
  const int j = blockIdx.x * 256 + threadIdx.x;   // byte column
  const int y = blockIdx.y;
  if (j >= cols * 3 || y >= out_rows) return;
  jit[blockIdx.z].u8[(long long)y * cols * 3 + j] = (uint8_t)resample_v_u8_value(d.tmp, cols, j, y, d.bv, d.kv, d.ksv);
}

// grid (views); block kJitThreads.  stage: copy the view's u8 image to shared memory first (dynamic smem >= 3 * pixels).
__global__ void __launch_bounds__(kJitThreads) views_color_jitter_kernel(const s3r_view_jitter_desc* __restrict__ jit,
                                                                         int stage) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __align__(16) uint8_t staged[];
  __shared__ long long warp_sum[kJitThreads / 32];
  __shared__ int mean_s;
  const s3r_view_jitter_desc& d = jit[blockIdx.x];
  const int rows = d.rows, cols = d.cols, transpose = d.transpose;
  const long long n = (long long)rows * cols;
  jitter::Params p;
#pragma unroll
  for (int k = 0; k < 4; ++k) p.order[k] = d.order[k];
  p.skip = d.skip;
  p.factor[0] = d.brightness;
  p.factor[1] = d.contrast;
  p.factor[2] = d.saturation;
  p.hue_shift = d.hue_shift;
  const int kc = jitter::contrast_pos(p);
  const uint8_t* src = d.u8;
  if (kc < 4 && stage) {   // two passes read the image: keep it on chip
    const long long nb = 3 * n;
    long long done = 0;
    if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) {
      const long long n16 = nb / 16;
      for (long long i = threadIdx.x; i < n16; i += kJitThreads)
        reinterpret_cast<uint4*>(staged)[i] = __ldg(reinterpret_cast<const uint4*>(src) + i);
      done = n16 * 16;
    }
    for (long long i = done + threadIdx.x; i < nb; i += kJitThreads) staged[i] = src[i];
    __syncthreads();
    src = staged;
  }
  int mean = 0;
  if (kc < 4) {
    long long s = 0;
    for (long long i = threadIdx.x; i < n; i += kJitThreads) {
      int r = src[3 * i], g = src[3 * i + 1], b = src[3 * i + 2];
      jitter::apply_ops(p, 0, kc, 0, r, g, b);
      s += jitter::luma(r, g, b);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      long long t = 0;
      for (int w = 0; w < kJitThreads / 32; ++w) t += warp_sum[w];
      mean_s = jitter::contrast_mean(t, n);
    }
    __syncthreads();
    mean = mean_s;
  }
  for (long long i = threadIdx.x; i < n; i += kJitThreads) {
    int c[3] = {src[3 * i], src[3 * i + 1], src[3 * i + 2]};
    jitter::apply_ops(p, 0, 4, mean, c[0], c[1], c[2]);
    long long o = i;
    if (transpose) {
      const long long y = i / cols, x = i - y * cols;
      o = x * rows + y;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) d.img[k * n + o] = img_norm_u8(c[k]);
  }
}

}  // namespace s3r

using namespace s3r;

extern "C" {

int s3r_views_resample_v_u8(const s3r_view_image_desc* descs, const s3r_view_jitter_desc* jit, int n, int max_out_rows,
                            int max_cols, void* stream) {
  if (n <= 0 || max_out_rows <= 0 || max_cols <= 0) return 0;
  if (descs == nullptr || jit == nullptr || n > 65535 || max_out_rows > 65535) {
    set_error("s3r_views_resample_v_u8: bad arguments (n=%d, max_out_rows=%d)", n, max_out_rows);
    return -2;
  }
  launch_pdl(views_resample_v_u8_kernel, dim3((max_cols * 3 + 255) / 256, max_out_rows, n), dim3(256), 0,
             reinterpret_cast<cudaStream_t>(stream), descs, jit);
  return cudaGetLastError() == cudaSuccess ? 0 : -6;
}

int s3r_views_color_jitter(const s3r_view_jitter_desc* jit, int n, int64_t max_pixels, void* stream) {
  if (n <= 0 || max_pixels <= 0) return 0;
  if (jit == nullptr || n > 0x7fffffff) {
    set_error("s3r_views_color_jitter: bad arguments (n=%d, max_pixels=%lld)", n, (long long)max_pixels);
    return -2;
  }
  const size_t smem = (size_t)3 * (size_t)max_pixels;
  const int stage = smem <= kJitSmemMax;
  static PerDeviceOnce once;
  if (stage && smem > 48 * 1024 && !once.cur()) {
    cudaFuncSetAttribute(views_color_jitter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kJitSmemMax);
    once.cur() = true;
  }
  launch_pdl(views_color_jitter_kernel, dim3(n), dim3(kJitThreads), stage ? smem : 0,
             reinterpret_cast<cudaStream_t>(stream), jit, stage);
  return cudaGetLastError() == cudaSuccess ? 0 : -6;
}

}  // extern "C"
