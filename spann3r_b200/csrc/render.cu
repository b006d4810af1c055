// Headless point rendering on the GPU: what the reference's spann3r/tools/vis.py:render_frames draws through an Open3D
// window (point_size 1, black background), as a deterministic z-buffered point rasteriser.
//
//   render_splat_kernel    one thread per input point: project (render_math.cuh), then a 64-bit atomicMin of
//                          (fp32 depth bits << 32 | global point index) into the pixel's key.  The minimum over keys does
//                          not depend on the order the atomics land in, so the frame does not depend on scheduling:
//                          the nearest fp32 depth wins and equal depths go to the smaller index (GL_LESS draw order).
//   render_resolve_kernel  one thread per output pixel: empty key -> black, else the winning point's fp32 colour as
//                          uint8 RGB.
//
// The key buffer (w * h uint64) is the only state.  Static mode keeps it across frames and splats only the new frame's
// points, so frame i equals a from-scratch render of frames 0..i at O(H W) work per frame; dynamic mode clears it first.
#include "../../include/spann3r_b200.h"
#include "gemm.cuh"

#include <math.h>

#include "render_math.cuh"

namespace s3r {

using namespace render;

namespace {

constexpr int kRenderThreads = 256;

__global__ void __launch_bounds__(kRenderThreads)
    render_splat_kernel(const float* __restrict__ pts, const uint8_t* __restrict__ mask, long long n,
                        unsigned long long id0, const Camera cam, double z_near, int w, int h,
                        unsigned long long* __restrict__ keys) {
  const long long i = blockIdx.x * (long long)kRenderThreads + threadIdx.x;
  if (i >= n || (mask && !mask[i])) return;
  uint64_t key;
  const long long pix = project_point(cam, z_near, w, h, pts[3 * i], pts[3 * i + 1], pts[3 * i + 2],
                                      (uint32_t)(id0 + (unsigned long long)i), &key);
  if (pix >= 0) atomicMin(keys + pix, (unsigned long long)key);
}

__global__ void __launch_bounds__(kRenderThreads)
    render_resolve_kernel(const unsigned long long* __restrict__ keys, const float* __restrict__ colors, long long npix,
                          uint8_t* __restrict__ out) {
  const long long i = blockIdx.x * (long long)kRenderThreads + threadIdx.x;
  if (i >= npix) return;
  const unsigned long long k = keys[i];
  uint8_t rgb[3] = {0, 0, 0};
  if (k != kEmptyKey) {
    const float* c = colors + 3 * (k & 0xffffffffULL);
    for (int a = 0; a < 3; ++a) rgb[a] = color_u8(c[a]);
  }
  for (int a = 0; a < 3; ++a) out[3 * i + a] = rgb[a];
}

bool size_ok(int w, int h) { return w >= 1 && h >= 1 && (long long)w * h < (1LL << 31); }

bool keys_ok(const void* keys) { return keys && (uintptr_t)keys % 8 == 0; }

int launched(const char* what) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: launch failed: %s", what, cudaGetErrorString(e));
    return -6;
  }
  return 0;
}

}  // namespace

}  // namespace s3r

using namespace s3r;

extern "C" {

size_t s3r_render_workspace_bytes(int w, int h) {
  return size_ok(w, h) ? sizeof(unsigned long long) * (size_t)w * h : 0;
}

int s3r_render_clear(void* keys, int w, int h, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!keys_ok(keys) || !size_ok(w, h)) {
    set_error("render_clear: bad arguments (w=%d h=%d; need w, h >= 1, w * h < 2^31 and an 8-byte aligned key buffer)",
              w, h);
    return -1;
  }
  if (cudaMemsetAsync(keys, 0xff, s3r_render_workspace_bytes(w, h), st) != cudaSuccess) return launched("render_clear");
  return 0;
}

int s3r_render_splat(const float* pts, const uint8_t* mask, int64_t n, int64_t id0, const double* camera, double z_near,
                     int w, int h, void* keys, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!pts || !camera || !keys_ok(keys) || !size_ok(w, h) || n < 0 || id0 < 0 || id0 + n >= (1LL << 32)) {
    set_error("render_splat: bad arguments (n=%lld id0=%lld w=%d h=%d; need id0 + n < 2^32, w, h >= 1, w * h < 2^31 and "
              "non-null pointers)", n, id0, w, h);
    return -1;
  }
  if (!(z_near >= 0.0) || !isfinite(z_near)) {
    set_error("render_splat: z_near=%g must be finite and >= 0", z_near);
    return -1;
  }
  for (int i = 0; i < 16; ++i) {
    if (!isfinite(camera[i])) {
      set_error("render_splat: camera[%d]=%g is not finite", i, camera[i]);
      return -1;
    }
  }
  Camera cam;
  for (int i = 0; i < 12; ++i) cam.rt[i] = camera[i];
  cam.fx = camera[12]; cam.fy = camera[13]; cam.cx = camera[14]; cam.cy = camera[15];
  if (n == 0) return 0;
  const long long blocks = (n + kRenderThreads - 1) / kRenderThreads;
  render_splat_kernel<<<(unsigned)blocks, kRenderThreads, 0, st>>>(pts, mask, n, (unsigned long long)id0, cam, z_near, w,
                                                                   h, (unsigned long long*)keys);
  return launched("render_splat");
}

int s3r_render_resolve(const void* keys, const float* colors, int w, int h, uint8_t* out, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!keys_ok(keys) || !colors || !out || !size_ok(w, h)) {
    set_error("render_resolve: bad arguments (w=%d h=%d; need w, h >= 1, w * h < 2^31, an 8-byte aligned key buffer and "
              "non-null pointers)", w, h);
    return -1;
  }
  const long long npix = (long long)w * h;
  render_resolve_kernel<<<(unsigned)((npix + kRenderThreads - 1) / kRenderThreads), kRenderThreads, 0, st>>>(
      (const unsigned long long*)keys, colors, npix, out);
  return launched("render_resolve");
}

}  // extern "C"
