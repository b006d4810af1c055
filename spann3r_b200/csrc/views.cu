// Dataset views on the GPU (spann3r_b200/views.py): what BaseStereoViewDataset.__getitem__ does to every view after the
// dataset has decoded it (dust3r/datasets/base/base_stereo_view_dataset.py:63-194, dust3r/datasets/utils/cropping.py,
// dust3r/utils/geometry.py:165-217), for a whole sequence per launch:
//   * depth: crop on the principal point, cv2 INTER_NEAREST rescale, centred crop, unprojection to world points and the
//     validity mask, fused in one kernel (views_depth_kernel; the crops and the nearest rescale are two host index
//     tables per view, the arithmetic is views_math.cuh);
//   * image: the input adapter's Pillow-exact Lanczos passes (resample_u8.cuh) with the view index in the grid.
// transpose_to_landscape is folded into the output indexing.  The host plans every view; the per-view descriptors are
// read from device memory (include/spann3r_b200.h).
#include "../../include/spann3r_b200.h"

#include "common.cuh"
#include "kernels.cuh"
#include "resample_u8.cuh"
#include "views_math.cuh"

namespace s3r {

// grid (pixel blocks, views); thread = one output pixel of one view.
__global__ void __launch_bounds__(256) views_depth_kernel(const s3r_view_depth_desc* __restrict__ descs) {
  pdl_launch_dependents();
  pdl_wait();
  const s3r_view_depth_desc& d = descs[blockIdx.y];
  const int w = d.w, h = d.h;
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= (long long)w * h) return;
  const int y = (int)(i / w), x = (int)(i - (long long)y * w);
  const float z = d.depth[(long long)__ldg(d.row_src + y) * d.depth_stride + __ldg(d.col_src + x)];
  if (!isfinite(z)) *d.nonfinite = 1;
  views::ViewCam c;
#pragma unroll
  for (int k = 0; k < 4; ++k) c.intr[k] = d.intr[k];
#pragma unroll
  for (int k = 0; k < 12; ++k) c.pose[k] = d.pose[k];
  float xc[3], xw[3];
  views::unproject(c, x, y, z, xc);
  views::to_world(c, xc, xw);
  const long long o = d.transpose ? (long long)x * h + y : i;
  d.depthmap[o] = z;
  d.pts3d[3 * o] = xw[0];
  d.pts3d[3 * o + 1] = xw[1];
  d.pts3d[3 * o + 2] = xw[2];
  d.valid[o] = views::valid_point(z, xw) ? 1 : 0;
}

// grid (128-column blocks, source rows, views): resample_h_u8_kernel of every view.
__global__ void __launch_bounds__(128) views_resample_h_kernel(const s3r_view_image_desc* __restrict__ descs) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ uint8_t span[];
  const s3r_view_image_desc& d = descs[blockIdx.z];
  const int row = blockIdx.y, x0 = blockIdx.x * 128;
  if (row >= d.rows || x0 >= d.cols) return;     // the whole block leaves: this view is smaller than the grid
  resample_h_u8_block(d.src + (long long)row * d.row_stride, d.cols, x0, d.bh, d.kh, d.ksh, span,
                      d.tmp + (long long)row * d.cols * 3);
}

// grid (256-byte-column blocks, output rows, views): resample_v_u8_norm_kernel of every view, transposed on request.
__global__ void __launch_bounds__(256) views_resample_v_norm_kernel(const s3r_view_image_desc* __restrict__ descs) {
  pdl_launch_dependents();
  pdl_wait();
  const s3r_view_image_desc& d = descs[blockIdx.z];
  const int cols = d.cols, out_rows = d.out_rows;
  const int j = blockIdx.x * 256 + threadIdx.x;   // byte column
  const int y = blockIdx.y;
  if (j >= cols * 3 || y >= out_rows) return;
  const int x = j / 3, c = j - 3 * x;
  const float v = resample_v_u8_norm_value(d.tmp, cols, j, y, d.bv, d.kv, d.ksv);
  const long long o = d.transpose ? ((long long)c * cols + x) * out_rows + y : ((long long)c * out_rows + y) * cols + x;
  d.img[o] = v;
}

}  // namespace s3r

using namespace s3r;

extern "C" {

int s3r_views_abi_sizeof(int which) {
  switch (which) {
    case 0: return (int)sizeof(s3r_view_depth_desc);
    case 1: return (int)sizeof(s3r_view_image_desc);
    case 2: return (int)sizeof(s3r_view_jitter_desc);
  }
  return -1;
}

int s3r_views_depth(const s3r_view_depth_desc* descs, int n, int64_t max_pixels, void* stream) {
  if (n <= 0 || max_pixels <= 0) return 0;
  if (descs == nullptr || n > 65535 || (max_pixels + 255) / 256 > 0x7fffffff) {
    set_error("s3r_views_depth: bad arguments (n=%d, max_pixels=%lld)", n, (long long)max_pixels);
    return -2;
  }
  launch_pdl(views_depth_kernel, dim3((unsigned)((max_pixels + 255) / 256), n), dim3(256), 0,
             reinterpret_cast<cudaStream_t>(stream), descs);
  return cudaGetLastError() == cudaSuccess ? 0 : -6;
}

int s3r_views_resample_h(const s3r_view_image_desc* descs, int n, int max_rows, int max_cols, int max_span,
                         void* stream) {
  if (n <= 0 || max_rows <= 0 || max_cols <= 0) return 0;
  if (descs == nullptr || n > 65535 || max_rows > 65535 || max_span <= 0) {
    set_error("s3r_views_resample_h: bad arguments (n=%d, max_rows=%d, max_span=%d)", n, max_rows, max_span);
    return -2;
  }
  const size_t smem = (size_t)3 * max_span;
  if (smem > 160 * 1024) {
    set_error("s3r_views_resample_h: source span of %d pixels per 128 output columns is too large", max_span);
    return -1;
  }
  static PerDeviceOnce once;
  if (smem > 48 * 1024 && !once.cur()) {
    cudaFuncSetAttribute(views_resample_h_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
    once.cur() = true;
  }
  launch_pdl(views_resample_h_kernel, dim3((max_cols + 127) / 128, max_rows, n), dim3(128), smem,
             reinterpret_cast<cudaStream_t>(stream), descs);
  return cudaGetLastError() == cudaSuccess ? 0 : -6;
}

int s3r_views_resample_v_norm(const s3r_view_image_desc* descs, int n, int max_out_rows, int max_cols, void* stream) {
  if (n <= 0 || max_out_rows <= 0 || max_cols <= 0) return 0;
  if (descs == nullptr || n > 65535 || max_out_rows > 65535) {
    set_error("s3r_views_resample_v_norm: bad arguments (n=%d, max_out_rows=%d)", n, max_out_rows);
    return -2;
  }
  launch_pdl(views_resample_v_norm_kernel, dim3((max_cols * 3 + 255) / 256, max_out_rows, n), dim3(256), 0,
             reinterpret_cast<cudaStream_t>(stream), descs);
  return cudaGetLastError() == cudaSuccess ? 0 : -6;
}

}  // extern "C"
