// Per-pixel arithmetic of Spann3R's training / test criteria (spann3r/loss.py:129-369 over dust3r/losses.py:52-59),
// `__host__ __device__` so that the same lines can be compiled for the CPU and pinned against numpy; the library only
// calls them from the kernels of loss.cu.  Every fp32 step is rounded separately (no fused multiply-add), in the order
// the reference's tensor expressions round them, so that the medians are selected among the same values.
#pragma once
#include "focal_math.cuh"

#if defined(__CUDA_ARCH__)
#define S3R_LMUL(a, b) __fmul_rn(a, b)
#define S3R_LADD(a, b) __fadd_rn(a, b)
#define S3R_LSUB(a, b) __fsub_rn(a, b)
#else
#define S3R_LMUL(a, b) ((float)((float)(a) * (float)(b)))
#define S3R_LADD(a, b) ((float)((float)(a) + (float)(b)))
#define S3R_LSUB(a, b) ((float)((float)(a) - (float)(b)))
#endif

namespace s3r {
namespace lossm {

// |v| = sqrt((x x + y y) + z z), each step rounded
S3R_FHD float norm3(float x, float y, float z) {
  return sqrtf(S3R_LADD(S3R_LADD(S3R_LMUL(x, x), S3R_LMUL(y, y)), S3R_LMUL(z, z)));
}

// The alignment of one point set of one batch element: v = (p / factor), then v.z -= shift, then v *= mul.
// factor = 1, shift = 0, mul = 1 leave a coordinate bit-identical, so the same formula serves every criterion.
struct Align {
  float factor, shift, mul;
};
S3R_FHD void align(const float* p, const Align& a, float* v) {
  v[0] = S3R_LMUL(p[0] / a.factor, a.mul);
  v[1] = S3R_LMUL(p[1] / a.factor, a.mul);
  v[2] = S3R_LMUL(S3R_LSUB(p[2] / a.factor, a.shift), a.mul);
}

// Value a median stage selects over (kind 0: z after normalisation; 1..3: coordinate kind-1 after normalisation and
// shift; 4: |v - centre| of the normalised, shifted point).
S3R_FHD float stage_value(const float* p, float factor, float shift, const float* centre, int kind) {
  const float x = p[0] / factor, y = p[1] / factor, z = p[2] / factor;
  if (kind == 0) return z;
  const float zs = S3R_LSUB(z, shift);
  if (kind == 1) return x;
  if (kind == 2) return y;
  if (kind == 3) return zs;
  return norm3(S3R_LSUB(x, centre[0]), S3R_LSUB(y, centre[1]), S3R_LSUB(zs, centre[2]));
}

// L21 distance d = |pr - gt| and the difference u = pr - gt
S3R_FHD float l21(const float* pr, const float* gt, float* u) {
  u[0] = S3R_LSUB(pr[0], gt[0]);
  u[1] = S3R_LSUB(pr[1], gt[1]);
  u[2] = S3R_LSUB(pr[2], gt[2]);
  return norm3(u[0], u[1], u[2]);
}

// ConfLoss_t's per-pixel term d c - alpha log c (spann3r/loss.py:283)
S3R_FHD float conf_term(float d, float c, float alpha) { return S3R_LSUB(S3R_LMUL(d, c), S3R_LMUL(alpha, logf(c))); }

// Gradient of a pixel's prediction p: g_d = dLoss/dd (fp64), the point's u and d after alignment, scale = mul / factor
// (the alignment's Jacobian; shift and mul are constants), plus the norm-factor term coef * g'(|p|) p / |p| where
// coef = dLoss/dfactor / (pooled valid count) and g' = 1 ('avg_dis') or 1 / (1 + |p|) ('avg_log1p').  The L21 and the
// norm gradients are 0 at a zero vector (torch's norm backward).
S3R_FHD void pred_grad(const float* p, const float* u, float d, double g_d, double scale, double coef, int log1p_mode,
                       float* g) {
  double gx = 0.0, gy = 0.0, gz = 0.0;
  if (d > 0.f) {
    const double s = g_d * scale / (double)d;
    gx = s * u[0];
    gy = s * u[1];
    gz = s * u[2];
  }
  if (coef != 0.0) {
    const float n = norm3(p[0], p[1], p[2]);
    if (n > 0.f) {
      const double s = coef / (double)n / (log1p_mode ? 1.0 + (double)n : 1.0);
      gx += s * p[0];
      gy += s * p[1];
      gz += s * p[2];
    }
  }
  g[0] = (float)gx;
  g[1] = (float)gy;
  g[2] = (float)gz;
}

}  // namespace lossm
}  // namespace s3r
