// Scalar geometry of the GPU PnP-RANSAC (csrc/pnp.cu): P3P minimal solver, reprojection, Gauss-Newton normal
// equations, 6x6 solve, SO(3) exp / log.  Everything is `__host__ __device__` double precision with no CUDA
// dependencies, so tests/native/pnp_host_check.cpp can compile THIS header with g++ and pin the arithmetic on the
// CPU (a test of the product's device math, not a product path -- the library itself only ever calls it from
// kernels).
//
// What it replaces: `cv2.solvePnPRansac(pts3d, pixel grid, K, 0)` as demo.py:170-180 calls it per frame (OpenCV is an
// unpinned third-party dependency of the reference; 4.13.0 in this image): RANSAC over minimal pose hypotheses scored
// by reprojection error (default threshold 8 px), then a non-linear least-squares refinement of the best model on its
// inliers.  Published algorithms restated here: Grunert's P3P (depth ratios u = s2/s1, v = s3/s1 from the law of
// cosines; Haralick et al. 1994, eq. for u linear in v, quartic in v), absolute orientation of two triangles by
// orthonormal frames, Gauss-Newton on the reprojection error with a left-multiplicative SO(3) update.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define S3R_HD __host__ __device__ __forceinline__
#else
#define S3R_HD inline
#endif

namespace s3r {
namespace pnp {

struct Pose {   // x_cam = R x_world + t, R row-major
  double R[9];
  double t[3];
};
struct Cam {
  double fx, fy, cx, cy;
};

S3R_HD double dot3(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
S3R_HD void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}
S3R_HD double normalize3(double* a) {
  const double n = sqrt(dot3(a, a));
  if (n > 0) {
    a[0] /= n; a[1] /= n; a[2] /= n;
  }
  return n;
}
S3R_HD void transform(const Pose& T, const double* X, double* Xc) {
  Xc[0] = T.R[0] * X[0] + T.R[1] * X[1] + T.R[2] * X[2] + T.t[0];
  Xc[1] = T.R[3] * X[0] + T.R[4] * X[1] + T.R[5] * X[2] + T.t[1];
  Xc[2] = T.R[6] * X[0] + T.R[7] * X[1] + T.R[8] * X[2] + T.t[2];
}

// Squared reprojection error of world point X against pixel (u, v); +inf behind the camera / non-finite.
S3R_HD double reproj_err2(const Pose& T, const Cam& k, const double* X, double u, double v) {
  double Xc[3];
  transform(T, X, Xc);
  if (!(Xc[2] > 1e-12)) return 1e300;
  const double du = k.fx * Xc[0] / Xc[2] + k.cx - u, dv = k.fy * Xc[1] / Xc[2] + k.cy - v;
  const double e = du * du + dv * dv;
  return e == e ? e : 1e300;
}

// ---- quartic roots: Durand-Kerner on the monic polynomial, complex arithmetic spelled out --------------------
// c[0..4] = coefficients of c0 + c1 x + ... + c4 x^4, c4 != 0.  Writes the real roots (|imag| small), returns how many.
S3R_HD int quartic_real_roots(const double* c, double* roots) {
  double a[4];   // monic: x^4 + a3 x^3 + a2 x^2 + a1 x + a0
  for (int i = 0; i < 4; ++i) a[i] = c[i] / c[4];
  // scale x = s y so that the roots are O(1): s = max_k |a_{4-k}|^(1/k)
  double s = 0;
  for (int k = 1; k <= 4; ++k) {
    const double m = pow(fabs(a[4 - k]), 1.0 / k);
    if (m > s) s = m;
  }
  if (!(s > 0) || !(s < 1e150)) {
    if (s == 0) {   // x^4 = 0
      roots[0] = 0;
      return 1;
    }
    return 0;
  }
  double b[4];   // y^4 + b3 y^3 + ... : b_{4-k} = a_{4-k} / s^k
  {
    double sk = s;
    for (int k = 1; k <= 4; ++k) {
      b[4 - k] = a[4 - k] / sk;
      sk *= s;
    }
  }
  double zr[4], zi[4];
  {   // starting points on a circle of radius ~ root bound / 2, irrational phase
    const double r0 = 1.3;
    for (int k = 0; k < 4; ++k) {
      const double ang = 0.4 + 1.5707963267948966 * k;
      zr[k] = r0 * cos(ang);
      zi[k] = r0 * sin(ang);
    }
  }
  for (int it = 0; it < 200; ++it) {
    double delta = 0;
    for (int k = 0; k < 4; ++k) {
      // p(z) by Horner
      double pr = 1, pi = 0;
      for (int j = 3; j >= 0; --j) {
        const double tr = pr * zr[k] - pi * zi[k] + b[j], ti = pr * zi[k] + pi * zr[k];
        pr = tr;
        pi = ti;
      }
      // q = prod_{j != k} (z_k - z_j)
      double qr = 1, qi = 0;
      for (int j = 0; j < 4; ++j) {
        if (j == k) continue;
        const double dr = zr[k] - zr[j], di = zi[k] - zi[j];
        const double tr = qr * dr - qi * di, ti = qr * di + qi * dr;
        qr = tr;
        qi = ti;
      }
      const double den = qr * qr + qi * qi;
      if (den < 1e-300) continue;
      const double wr = (pr * qr + pi * qi) / den, wi = (pi * qr - pr * qi) / den;
      zr[k] -= wr;
      zi[k] -= wi;
      const double d = fabs(wr) + fabs(wi);
      if (d > delta) delta = d;
    }
    if (delta < 1e-15) break;
  }
  int n = 0;
  for (int k = 0; k < 4; ++k) {
    if (fabs(zi[k]) > 1e-6 * (1.0 + fabs(zr[k]))) continue;
    double y = zr[k];
    for (int it = 0; it < 3; ++it) {   // Newton polish on the real axis
      const double p = (((y + b[3]) * y + b[2]) * y + b[1]) * y + b[0];
      const double dp = ((4 * y + 3 * b[3]) * y + 2 * b[2]) * y + b[1];
      if (fabs(dp) < 1e-300) break;
      y -= p / dp;
    }
    roots[n++] = y * s;
  }
  return n;
}

// ---- P3P (Grunert) --------------------------------------------------------------------------------------------
// P[i] world points, f[i] UNIT bearing vectors in the camera frame.  Returns the number of poses written (<= 4).
S3R_HD int p3p(const double P[3][3], const double f[3][3], Pose* out) {
  double d12[3], d13[3], d23[3];
  for (int i = 0; i < 3; ++i) {
    d12[i] = P[1][i] - P[0][i];
    d13[i] = P[2][i] - P[0][i];
    d23[i] = P[2][i] - P[1][i];
  }
  const double a2 = dot3(d23, d23), b2 = dot3(d13, d13), c2 = dot3(d12, d12);
  if (!(a2 > 1e-20 && b2 > 1e-20 && c2 > 1e-20)) return 0;
  const double ca = dot3(f[1], f[2]), cb = dot3(f[0], f[2]), cg = dot3(f[0], f[1]);
  const double q = (a2 - c2) / b2, r = c2 / b2;
  // u = s2/s1 = num(v) / den(v), v = s3/s1:  num = (q-1) v^2 - 2 q cb v + (1+q),  den = 2 (cg - ca v)
  const double nu[3] = {1 + q, -2 * q * cb, q - 1};
  const double de[2] = {2 * cg, -2 * ca};
  // quartic: num^2 + den^2 - 2 cg num den - r (1 - 2 cb v + v^2) den^2 = 0
  double p[5] = {0, 0, 0, 0, 0};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) p[i + j] += nu[i] * nu[j];
  double dd[3] = {0, 0, 0};
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 2; ++j) dd[i + j] += de[i] * de[j];
  for (int i = 0; i < 3; ++i) p[i] += dd[i];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 2; ++j) p[i + j] -= 2 * cg * nu[i] * de[j];
  const double w[3] = {1, -2 * cb, 1};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) p[i + j] -= r * w[i] * dd[j];
  double pm = 0;
  for (int i = 0; i < 5; ++i) pm = fmax(pm, fabs(p[i]));
  if (!(pm > 0) || fabs(p[4]) < 1e-12 * pm) return 0;
  double roots[4];
  const int nr = quartic_real_roots(p, roots);
  // orthonormal frame of the world triangle
  double e1[3] = {d12[0], d12[1], d12[2]}, e2[3], e3[3];
  if (normalize3(e1) < 1e-12) return 0;
  cross3(e1, d13, e3);
  if (normalize3(e3) < 1e-12) return 0;   // collinear sample
  cross3(e3, e1, e2);
  int n = 0;
  for (int k = 0; k < nr; ++k) {
    const double v = roots[k];
    if (!(v > 1e-9)) continue;
    const double den = de[0] + de[1] * v;
    if (fabs(den) < 1e-12) continue;
    const double u = ((nu[2] * v + nu[1]) * v + nu[0]) / den;
    if (!(u > 1e-9)) continue;
    const double g = 1 + u * u - 2 * u * cg;
    if (!(g > 1e-14)) continue;
    const double s1 = sqrt(c2 / g), s2 = u * s1, s3 = v * s1;
    double Y[3][3];
    for (int i = 0; i < 3; ++i) {
      Y[0][i] = s1 * f[0][i];
      Y[1][i] = s2 * f[1][i];
      Y[2][i] = s3 * f[2][i];
    }
    double y12[3], y13[3], g1[3], g2[3], g3[3];
    for (int i = 0; i < 3; ++i) {
      y12[i] = Y[1][i] - Y[0][i];
      y13[i] = Y[2][i] - Y[0][i];
      g1[i] = y12[i];
    }
    if (normalize3(g1) < 1e-12) continue;
    cross3(g1, y13, g3);
    if (normalize3(g3) < 1e-12) continue;
    cross3(g3, g1, g2);
    Pose& T = out[n];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) T.R[3 * i + j] = g1[i] * e1[j] + g2[i] * e2[j] + g3[i] * e3[j];
    for (int i = 0; i < 3; ++i) T.t[i] = Y[0][i] - (T.R[3 * i] * P[0][0] + T.R[3 * i + 1] * P[0][1] + T.R[3 * i + 2] * P[0][2]);
    bool ok = true;
    for (int i = 0; i < 9; ++i) ok = ok && (T.R[i] == T.R[i]);
    for (int i = 0; i < 3; ++i) ok = ok && (T.t[i] == T.t[i]) && fabs(T.t[i]) < 1e100;
    if (ok) ++n;
  }
  return n;
}

// ---- Gauss-Newton on the reprojection error ---------------------------------------------------------------------
// acc[0..20] upper triangle of H = sum J^T J (row-major: (0,0) (0,1) .. (0,5) (1,1) ..), acc[21..26] g = sum J^T r,
// acc[27] = sum |r|^2, acc[28] = number of points used.  delta = (omega, dt): x_cam' = exp(omega) x_cam + dt.
constexpr int kAcc = 29;
S3R_HD void gn_accumulate(const Pose& T, const Cam& k, const double* X, double u, double v, double* acc) {
  double Xc[3];
  transform(T, X, Xc);
  if (!(Xc[2] > 1e-12)) return;
  const double iz = 1.0 / Xc[2], x = Xc[0] * iz, y = Xc[1] * iz;
  const double ru = k.fx * x + k.cx - u, rv = k.fy * y + k.cy - v;
  if (!(ru == ru && rv == rv)) return;
  const double Ju[6] = {-k.fx * x * y, k.fx * (1 + x * x), -k.fx * y, k.fx * iz, 0, -k.fx * x * iz};
  const double Jv[6] = {-k.fy * (1 + y * y), k.fy * x * y, k.fy * x, 0, k.fy * iz, -k.fy * y * iz};
  int o = 0;
  for (int i = 0; i < 6; ++i)
    for (int j = i; j < 6; ++j) acc[o++] += Ju[i] * Ju[j] + Jv[i] * Jv[j];
  for (int i = 0; i < 6; ++i) acc[21 + i] += Ju[i] * ru + Jv[i] * rv;
  acc[27] += ru * ru + rv * rv;
  acc[28] += 1.0;
}

S3R_HD void so3_exp(const double* w, double* R) {
  const double th2 = dot3(w, w), th = sqrt(th2);
  double A, B;   // R = I + A [w]x + B [w]x^2
  if (th < 1e-8) {
    A = 1 - th2 / 6;
    B = 0.5 - th2 / 24;
  } else {
    A = sin(th) / th;
    B = (1 - cos(th)) / th2;
  }
  const double wx = w[0], wy = w[1], wz = w[2];
  R[0] = 1 - B * (wy * wy + wz * wz); R[1] = -A * wz + B * wx * wy;      R[2] = A * wy + B * wx * wz;
  R[3] = A * wz + B * wx * wy;        R[4] = 1 - B * (wx * wx + wz * wz); R[5] = -A * wx + B * wy * wz;
  R[6] = -A * wy + B * wx * wz;       R[7] = A * wx + B * wy * wz;       R[8] = 1 - B * (wx * wx + wy * wy);
}

// Rodrigues vector of a rotation matrix (the `rvec` cv2 returns), through the unit quaternion: Shepperd's method takes
// the largest of |qw|, |qx|, |qy|, |qz| from the diagonal and the rest from the off-diagonal sums / differences, and
// th = 2 atan2(|q_xyz|, qw).  Accurate to rounding at every angle; acos of the trace with the skew part divided by
// sin(th) loses digits as th approaches pi (1e-11 at pi - 0.006).
S3R_HD void so3_log(const double* R, double* w) {
  const double tr = R[0] + R[4] + R[8];
  double q[4];   // (qw, qx, qy, qz) times 4 * (the largest component)
  if (tr >= R[0] && tr >= R[4] && tr >= R[8]) {
    const double s = 1 + tr;
    q[0] = s; q[1] = R[7] - R[5]; q[2] = R[2] - R[6]; q[3] = R[3] - R[1];
  } else if (R[0] >= R[4] && R[0] >= R[8]) {
    const double s = 1 + R[0] - R[4] - R[8];
    q[0] = R[7] - R[5]; q[1] = s; q[2] = R[1] + R[3]; q[3] = R[2] + R[6];
  } else if (R[4] >= R[8]) {
    const double s = 1 + R[4] - R[0] - R[8];
    q[0] = R[2] - R[6]; q[1] = R[1] + R[3]; q[2] = s; q[3] = R[5] + R[7];
  } else {
    const double s = 1 + R[8] - R[0] - R[4];
    q[0] = R[3] - R[1]; q[1] = R[2] + R[6]; q[2] = R[5] + R[7]; q[3] = s;
  }
  if (q[0] < 0) {   // the quaternion with qw >= 0: th in [0, pi]
    for (int i = 0; i < 4; ++i) q[i] = -q[i];
  }
  const double n = sqrt(q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  // th / |q_xyz| with the common scale divided out; 2 / qw is its limit (to 1e-16 relative) at th < ~1e-8
  const double k = n > 1e-8 * q[0] ? 2 * atan2(n, q[0]) / n : 2 / q[0];
  w[0] = k * q[1]; w[1] = k * q[2]; w[2] = k * q[3];
}

// One damped Gauss-Newton step from the accumulated sums: solve (H + lambda diag(H)) delta = -g by Cholesky, apply
// R <- exp(omega) R, t <- exp(omega) t + dt.  Returns false (pose untouched) when H is not positive definite.
S3R_HD bool gn_step(const double* acc, double lambda, Pose& T) {
  double H[36], g[6];
  int o = 0;
  for (int i = 0; i < 6; ++i)
    for (int j = i; j < 6; ++j) {
      H[6 * i + j] = acc[o];
      H[6 * j + i] = acc[o];
      ++o;
    }
  for (int i = 0; i < 6; ++i) {
    g[i] = -acc[21 + i];
    H[7 * i] *= (1 + lambda);
  }
  double L[36];
  for (int i = 0; i < 36; ++i) L[i] = 0;
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j <= i; ++j) {
      double s = H[6 * i + j];
      for (int k = 0; k < j; ++k) s -= L[6 * i + k] * L[6 * j + k];
      if (i == j) {
        if (!(s > 1e-300)) return false;
        L[6 * i + i] = sqrt(s);
      } else {
        L[6 * i + j] = s / L[6 * j + j];
      }
    }
  double yv[6], d[6];
  for (int i = 0; i < 6; ++i) {
    double s = g[i];
    for (int k = 0; k < i; ++k) s -= L[6 * i + k] * yv[k];
    yv[i] = s / L[6 * i + i];
  }
  for (int i = 5; i >= 0; --i) {
    double s = yv[i];
    for (int k = i + 1; k < 6; ++k) s -= L[6 * k + i] * d[k];
    d[i] = s / L[6 * i + i];
  }
  for (int i = 0; i < 6; ++i)
    if (!(d[i] == d[i])) return false;
  double E[9], Rn[9], tn[3];
  so3_exp(d, E);
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) Rn[3 * i + j] = E[3 * i] * T.R[j] + E[3 * i + 1] * T.R[3 + j] + E[3 * i + 2] * T.R[6 + j];
    tn[i] = E[3 * i] * T.t[0] + E[3 * i + 1] * T.t[1] + E[3 * i + 2] * T.t[2] + d[3 + i];
  }
  for (int i = 0; i < 9; ++i) T.R[i] = Rn[i];
  for (int i = 0; i < 3; ++i) T.t[i] = tn[i];
  return true;
}

// Counter-based sample index: SplitMix64 of (seed, hypothesis, slot, attempt) reduced to [0, n).
S3R_HD unsigned long long mix64(unsigned long long z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
S3R_HD long long sample_index(unsigned long long seed, int hyp, int slot, int attempt, long long n) {
  const unsigned long long h = mix64(mix64(seed ^ (0x51ED27ull * (unsigned long long)(hyp + 1))) + 977ull * slot + 7919ull * attempt);
  return (long long)(h % (unsigned long long)n);
}


// World point i and its pixel: img == nullptr means the dense pixel grid of demo.py:166-168 (u = i % width,
// v = i / width).  False for non-finite points.
S3R_HD bool load_point(const float* pts, const float* img, long long i, int width, double* X, double& u, double& v) {
  const float x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
  X[0] = x; X[1] = y; X[2] = z;
  if (img) {
    u = img[2 * i];
    v = img[2 * i + 1];
  } else {
    u = (double)(i % width);
    v = (double)(i / width);
  }
  const double s = X[0] + X[1] + X[2] + u + v;
  return s == s && fabs(s) < 1e30;
}

// Minimal sample `hyp` (three distinct finite points chosen by the counter-based hash) -> up to 4 poses.
S3R_HD int sample_hypotheses(unsigned long long seed, int hyp, const float* pts, const float* img, long long n, int width,
                             const Cam& k, Pose* out) {
  double P[3][3], f[3][3];
  long long idx[3] = {-1, -1, -1};
  for (int s = 0; s < 3; ++s) {
    bool got = false;
    for (int att = 0; att < 16 && !got; ++att) {
      const long long i = sample_index(seed, hyp, s, att, n);
      if (i == idx[0] || i == idx[1]) continue;
      double u, v;
      if (!load_point(pts, img, i, width, P[s], u, v)) continue;
      f[s][0] = (u - k.cx) / k.fx;
      f[s][1] = (v - k.cy) / k.fy;
      f[s][2] = 1.0;
      normalize3(f[s]);
      idx[s] = i;
      got = true;
    }
    if (!got) return 0;
  }
  return p3p(P, f, out);
}

}  // namespace pnp
}  // namespace s3r
