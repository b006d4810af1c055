// Scalar math of the dataset view builder (csrc/views.cu): one depth pixel -> camera point -> world point, and the
// validity rule.  `__host__ __device__` with no CUDA dependencies, so tests/native/views_host_check.cpp compiles THIS
// header with g++ and tests/test_views.py checks it bit for bit against a numpy restatement on the CPU.
//
// The arithmetic is numpy's, as dust3r/utils/geometry.py:165-217 runs it on float32 inputs:
//   x = fp32(((fp64(u) - fp64(cu)) * fp64(z)) / fp64(fu))      int64 meshgrid - float32 scalar promotes to float64
//   y = fp32(((fp64(v) - fp64(cv)) * fp64(z)) / fp64(fv)),  z as is
//   X_world[i] = ((0 + R[i][0] x) + R[i][1] y) + R[i][2] z + t[i]   in fp32, each product and sum rounded on its own
// The last line is np.einsum("ik,vuk->vui") (a zero-initialised output accumulated over k, no FMA) followed by the
// broadcast add of t.  Every operation is an explicitly rounded intrinsic on the device, so nothing is contracted.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define S3R_VHD __host__ __device__ __forceinline__
#else
#define S3R_VHD inline
#endif

namespace s3r {
namespace views {

#if defined(__CUDA_ARCH__)
// NaN results follow the x86 SSE / AVX rules numpy's loops run under, so that a NaN in pts3d (a view without pose,
// inf * 0 from an overflowing depth) has the reference's bits and not the GPU's canonical 0x7fffffff: a NaN operand
// is returned quieted (the first one when both are), an invalid operation returns the default NaN 0xffc00000.
S3R_VHD float quiet_f(float a) { return __uint_as_float(__float_as_uint(a) | 0x00400000u); }
S3R_VHD double quiet_d(double a) {
  return __longlong_as_double(__double_as_longlong(a) | 0x0008000000000000LL);
}
S3R_VHD float fmul_rn(float a, float b) {
  if (isnan(a)) return quiet_f(a);
  if (isnan(b)) return quiet_f(b);
  const float r = __fmul_rn(a, b);
  return isnan(r) ? __uint_as_float(0xffc00000u) : r;
}
S3R_VHD float fadd_rn(float a, float b) {
  if (isnan(a)) return quiet_f(a);
  if (isnan(b)) return quiet_f(b);
  const float r = __fadd_rn(a, b);
  return isnan(r) ? __uint_as_float(0xffc00000u) : r;
}
#define S3R_VIEWS_D_OP(name, intrinsic)                                             \
  S3R_VHD double name(double a, double b) {                                         \
    if (isnan(a)) return quiet_d(a);                                                \
    if (isnan(b)) return quiet_d(b);                                                \
    const double r = intrinsic(a, b);                                               \
    return isnan(r) ? __longlong_as_double((long long)0xfff8000000000000ULL) : r;   \
  }
S3R_VIEWS_D_OP(dsub_rn, __dsub_rn)
S3R_VIEWS_D_OP(dmul_rn, __dmul_rn)
S3R_VIEWS_D_OP(ddiv_rn, __ddiv_rn)
#undef S3R_VIEWS_D_OP
// cvtsd2ss keeps the sign and the top 23 payload bits of a NaN
S3R_VHD float to_f32_rn(double a) {
  if (isnan(a)) {
    const unsigned long long u = (unsigned long long)__double_as_longlong(a);
    return __uint_as_float((unsigned)(u >> 32 & 0x80000000u) | 0x7fc00000u | (unsigned)(u >> 29 & 0x003fffffu));
  }
  return __double2float_rn(a);
}
#else
S3R_VHD float fmul_rn(float a, float b) { return a * b; }
S3R_VHD float fadd_rn(float a, float b) { return a + b; }
S3R_VHD double dsub_rn(double a, double b) { return a - b; }
S3R_VHD double dmul_rn(double a, double b) { return a * b; }
S3R_VHD double ddiv_rn(double a, double b) { return a / b; }
S3R_VHD float to_f32_rn(double a) { return (float)a; }
#endif

// intr = (fu, fv, cu, cv) of the final fp32 intrinsics; pose = [R | t] of the camera-to-world pose, 3x4 row-major fp32.
struct ViewCam {
  float intr[4];
  float pose[12];
};

// Camera point of pixel (u, v) (column, row of the cropped view, before any transpose) at depth z.
S3R_VHD void unproject(const ViewCam& c, int u, int v, float z, float* xc) {
  xc[0] = to_f32_rn(ddiv_rn(dmul_rn(dsub_rn((double)u, (double)c.intr[2]), (double)z), (double)c.intr[0]));
  xc[1] = to_f32_rn(ddiv_rn(dmul_rn(dsub_rn((double)v, (double)c.intr[3]), (double)z), (double)c.intr[1]));
  xc[2] = z;
}

// World point R xc + t.
S3R_VHD void to_world(const ViewCam& c, const float* xc, float* xw) {
  for (int i = 0; i < 3; ++i) {
    const float* r = c.pose + 4 * i;
    float acc = 0.0f;
    acc = fadd_rn(acc, fmul_rn(r[0], xc[0]));
    acc = fadd_rn(acc, fmul_rn(r[1], xc[1]));
    acc = fadd_rn(acc, fmul_rn(r[2], xc[2]));
    xw[i] = fadd_rn(acc, r[3]);
  }
}

// valid_mask = (depth > 0) & isfinite(pts3d).all(-1)   (base_stereo_view_dataset.py:100-103)
S3R_VHD bool valid_point(float z, const float* xw) {
  return z > 0.0f && isfinite(xw[0]) && isfinite(xw[1]) && isfinite(xw[2]);
}

}  // namespace views
}  // namespace s3r
