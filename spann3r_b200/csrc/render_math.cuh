// Scalar math of the point rasteriser (csrc/render.cu): the camera projection of one point to a pixel and a 64-bit depth
// key, and the fp32 colour -> uint8 conversion.  `__host__ __device__` with no CUDA dependencies, so
// tests/native/render_host_check.cpp compiles THIS header with g++ and tests/test_vis.py checks it bit for bit against
// a numpy restatement on the CPU.
//
// Pinhole model with pixel centres at integer coordinates (OpenCV / Open3D intrinsics): a world point p maps to the
// camera point q = R p + t, then to u = fx (qx / qz) + cx, v = fy (qy / qz) + cy, and lands on the pixel whose centre is
// nearest: col = floor(u + 0.5), row = floor(v + 0.5).  Every step is one rounded fp64 operation in a fixed order, so
// the pixel a point lands on does not depend on the compiler.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "pointcloud_math.cuh"   // S3R_HD, mul_rn / add_rn, apply_rt

namespace s3r {
namespace render {

using pcl::add_rn;
using pcl::mul_rn;

// [R | t] (3x4 row-major, world -> camera) and the intrinsics; s3r_render_splat's `camera` array in this order.
struct Camera {
  double rt[12];
  double fx, fy, cx, cy;
};

// An empty z-buffer entry.  No point's key reaches it: the depth bits of a positive float are at most 0x7f800000.
constexpr uint64_t kEmptyKey = ~0ULL;

#if defined(__CUDA_ARCH__)
S3R_HD double div_rn(double a, double b) { return __ddiv_rn(a, b); }
S3R_HD float to_f32_rn(double a) { return __double2float_rn(a); }
S3R_HD uint32_t f32_bits(float f) { return (uint32_t)__float_as_uint(f); }
#else
S3R_HD double div_rn(double a, double b) { return a / b; }
S3R_HD float to_f32_rn(double a) { return (float)a; }
S3R_HD uint32_t f32_bits(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
}
#endif

// Projects the fp32 point (x, y, z) with global index `id`.  Returns the pixel index row * w + col and sets *key to
// (bits(fp32(qz)) << 32) | id, or returns -1 when the point is dropped: q not finite, qz <= z_near, or the pixel outside
// [0, w) x [0, h) (checked in fp64, so no out-of-range value is ever converted to an integer).  The smallest key of a
// pixel is its nearest point at fp32 depth resolution, ties going to the smaller id.
S3R_HD long long project_point(const Camera& c, double z_near, int w, int h, float x, float y, float z, uint32_t id,
                               uint64_t* key) {
  const double p[3] = {(double)x, (double)y, (double)z};
  double q[3];
  pcl::apply_rt(c.rt, p, q);
  if (!(isfinite(q[0]) && isfinite(q[1]) && isfinite(q[2])) || !(q[2] > z_near)) return -1;
  const double u = add_rn(mul_rn(c.fx, div_rn(q[0], q[2])), c.cx);
  const double v = add_rn(mul_rn(c.fy, div_rn(q[1], q[2])), c.cy);
  const double col = floor(add_rn(u, 0.5)), row = floor(add_rn(v, 0.5));
  if (!(col >= 0.0 && col < (double)w && row >= 0.0 && row < (double)h)) return -1;   // NaN fails too
  *key = ((uint64_t)f32_bits(to_f32_rn(q[2])) << 32) | (uint64_t)id;
  return (long long)row * w + (long long)col;
}

// floor(min(1, max(0, c)) * 255 + 0.5) in fp64: exact for an fp32 c (c * 255 needs 32 significant bits), so it is
// round-half-up of the exact product.  NaN -> 0 (fmax / fmin ignore a NaN operand, as std::max(0., c) does).
S3R_HD uint8_t color_u8(float c) {
  const double s = fmin(1.0, fmax(0.0, (double)c));
  return (uint8_t)floor(add_rn(mul_rn(s, 255.0), 0.5));
}

}  // namespace render
}  // namespace s3r
