// Scalar geometry of the point-cloud evaluation (csrc/pointcloud.cu): rounding-pinned squared distances, the box lower
// bound the spatial index prunes with, 63-bit Morton keys, a 3x3 symmetric eigen solver (normals), a 3x3 SVD and the
// Umeyama / Kabsch rigid fit (ICP).  Everything is `__host__ __device__` double precision with no CUDA dependencies, so
// tests/native/recon_host_check.cpp compiles THIS header with g++ and checks it against numpy on the CPU.
//
// Published algorithms restated here: cyclic Jacobi rotations for the symmetric eigenproblem and one-sided (Hestenes)
// Jacobi for the SVD (Golub & Van Loan, 4th ed., 8.5 and 8.6.3); Umeyama's least-squares similarity (IEEE PAMI 13(4),
// 1991) without the scale, reflection fixed by the sign of det -- what Open3D's TransformationEstimationPointToPoint
// documents it computes.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define S3R_HD __host__ __device__ __forceinline__
#else
#define S3R_HD inline
#endif

namespace s3r {
namespace pcl {

// Round-to-nearest multiply / add that nvcc may not contract into an FMA.  The squared distance must be formed as
// ((dx*dx + dy*dy) + dz*dz) with every step rounded, as scipy's cKDTree does, so the two agree to the last bit and the
// box lower bound below stays a true lower bound of it.
#if defined(__CUDA_ARCH__)
S3R_HD double mul_rn(double a, double b) { return __dmul_rn(a, b); }
S3R_HD double add_rn(double a, double b) { return __dadd_rn(a, b); }
S3R_HD double sub_rn(double a, double b) { return __dsub_rn(a, b); }
#else
S3R_HD double mul_rn(double a, double b) { return a * b; }
S3R_HD double add_rn(double a, double b) { return a + b; }
S3R_HD double sub_rn(double a, double b) { return a - b; }
#endif

S3R_HD double dist2(const double* q, const double* p) {
  const double dx = sub_rn(q[0], p[0]), dy = sub_rn(q[1], p[1]), dz = sub_rn(q[2], p[2]);
  return add_rn(add_rn(mul_rn(dx, dx), mul_rn(dy, dy)), mul_rn(dz, dz));
}

// Squared distance from q to the box [lo, hi], rounded like dist2: for every point p inside the box each |q - p| per axis
// rounds to at least the gap, so box_lb2 <= dist2(q, p) holds in floating point, not only in exact arithmetic.  An empty
// box (lo = +inf, hi = -inf) gives +inf.
S3R_HD double box_lb2(const double* q, const double* lo, const double* hi) {
  double g[3];
  for (int a = 0; a < 3; ++a) {
    const double below = sub_rn(lo[a], q[a]), above = sub_rn(q[a], hi[a]);
    g[a] = below > 0 ? below : (above > 0 ? above : 0.0);
  }
  return add_rn(add_rn(mul_rn(g[0], g[0]), mul_rn(g[1], g[1])), mul_rn(g[2], g[2]));
}

// x' = R x + t for a 3x4 row-major [R | t], each row summed as ((r0 x + r1 y) + r2 z) + t.
S3R_HD void apply_rt(const double* T, const double* x, double* y) {
  for (int r = 0; r < 3; ++r)
    y[r] = add_rn(add_rn(add_rn(mul_rn(T[4 * r], x[0]), mul_rn(T[4 * r + 1], x[1])), mul_rn(T[4 * r + 2], x[2])), T[4 * r + 3]);
}

// 21 bits of one coordinate inside [lo, lo + ext], spread to every third bit.
S3R_HD uint64_t spread21(uint64_t v) {
  v &= 0x1fffffULL;
  v = (v | (v << 32)) & 0x1f00000000ffffULL;
  v = (v | (v << 16)) & 0x1f0000ff0000ffULL;
  v = (v | (v << 8)) & 0x100f00f00f00f00fULL;
  v = (v | (v << 4)) & 0x10c30c30c30c30c3ULL;
  v = (v | (v << 2)) & 0x1249249249249249ULL;
  return v;
}
S3R_HD uint64_t quantize21(double x, double lo, double inv_ext) {
  double f = (x - lo) * inv_ext * 2097151.0;
  f = f < 0 ? 0 : (f > 2097151.0 ? 2097151.0 : f);
  return (uint64_t)f;
}
// 63-bit Morton key (x in the lowest bit of each triple).  Only the ORDER depends on it; exactness does not.
S3R_HD uint64_t morton63(const double* p, const double* lo, const double* inv_ext) {
  return spread21(quantize21(p[0], lo[0], inv_ext[0])) | (spread21(quantize21(p[1], lo[1], inv_ext[1])) << 1) |
         (spread21(quantize21(p[2], lo[2], inv_ext[2])) << 2);
}

// ---------------------------------------------------------------------------------------------------------------------
// Symmetric 3x3 eigenproblem by cyclic Jacobi: A (row-major, symmetric) -> eigenvalues w[3], eigenvectors as the
// COLUMNS of V (row-major), unsorted.
// ---------------------------------------------------------------------------------------------------------------------
S3R_HD void sym3_eigen(const double* A_in, double* w, double* V) {
  double A[9];
  for (int i = 0; i < 9; ++i) {
    A[i] = A_in[i];
    V[i] = (i % 4 == 0) ? 1.0 : 0.0;
  }
  for (int sweep = 0; sweep < 32; ++sweep) {
    const double off = fabs(A[1]) + fabs(A[2]) + fabs(A[5]);
    const double diag = fabs(A[0]) + fabs(A[4]) + fabs(A[8]);
    if (off == 0.0 || off <= 1e-300 || off < 1e-18 * diag) break;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        const double apq = A[3 * p + q];
        if (apq == 0.0) continue;
        const double app = A[3 * p + p], aqq = A[3 * q + q];
        const double theta = (aqq - app) / (2.0 * apq);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 3; ++k) {   // A <- A J (columns p, q)
          const double akp = A[3 * k + p], akq = A[3 * k + q];
          A[3 * k + p] = c * akp - s * akq;
          A[3 * k + q] = s * akp + c * akq;
        }
        for (int k = 0; k < 3; ++k) {   // A <- J^T A (rows p, q)
          const double apk = A[3 * p + k], aqk = A[3 * q + k];
          A[3 * p + k] = c * apk - s * aqk;
          A[3 * q + k] = s * apk + c * aqk;
        }
        A[3 * p + q] = A[3 * q + p] = 0.0;
        for (int k = 0; k < 3; ++k) {   // V <- V J
          const double vkp = V[3 * k + p], vkq = V[3 * k + q];
          V[3 * k + p] = c * vkp - s * vkq;
          V[3 * k + q] = s * vkp + c * vkq;
        }
      }
  }
  w[0] = A[0]; w[1] = A[4]; w[2] = A[8];
}

// Unit eigenvector of the smallest eigenvalue of the symmetric C (ties: the lowest column of the solver); (0, 0, 1)
// when C is zero.  The sign is whatever the solver produced.
S3R_HD void smallest_eigvec(const double* C, double* n) {
  double m = 0;
  for (int i = 0; i < 9; ++i) m = fabs(C[i]) > m ? fabs(C[i]) : m;
  if (!(m > 0)) {
    n[0] = 0; n[1] = 0; n[2] = 1;
    return;
  }
  double A[9], w[3], V[9];
  for (int i = 0; i < 9; ++i) A[i] = C[i] / m;   // scale-free: DTU clouds are in millimetres
  sym3_eigen(A, w, V);
  int j = 0;
  if (w[1] < w[j]) j = 1;
  if (w[2] < w[j]) j = 2;
  double x = V[j], y = V[3 + j], z = V[6 + j];
  const double r = sqrt(x * x + y * y + z * z);
  n[0] = x / r; n[1] = y / r; n[2] = z / r;
}

// Covariance (mean-centred, divided by k) of k points, then its smallest eigenvector -- the normal of a k-NN set.
// pt(i, a): coordinate a of neighbour i.  Fewer than 3 points -> (0, 0, 1).
template <class P>
S3R_HD void knn_normal(const P& pt, int k, double* n) {
  if (k < 3) {
    n[0] = 0; n[1] = 0; n[2] = 1;
    return;
  }
  double mu[3] = {0, 0, 0};
  for (int i = 0; i < k; ++i)
    for (int a = 0; a < 3; ++a) mu[a] += pt(i, a);
  for (int a = 0; a < 3; ++a) mu[a] /= k;
  double C[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int i = 0; i < k; ++i) {
    const double d[3] = {pt(i, 0) - mu[0], pt(i, 1) - mu[1], pt(i, 2) - mu[2]};
    for (int a = 0; a < 3; ++a)
      for (int b = a; b < 3; ++b) C[3 * a + b] += d[a] * d[b];
  }
  for (int a = 0; a < 3; ++a)
    for (int b = a; b < 3; ++b) C[3 * b + a] = C[3 * a + b] = C[3 * a + b] / k;
  smallest_eigvec(C, n);
}

// ---------------------------------------------------------------------------------------------------------------------
// 3x3 SVD by one-sided Jacobi: M = U diag(s) V^T, s descending, det(U) = +1 (the third left vector is u0 x u1; a rank
// deficient M gets an arbitrary orthonormal completion).  Row-major; U and V hold the vectors as columns.
// ---------------------------------------------------------------------------------------------------------------------
S3R_HD void svd3(const double* M, double* U, double* s, double* V) {
  double B[9];
  for (int i = 0; i < 9; ++i) {
    B[i] = M[i];
    V[i] = (i % 4 == 0) ? 1.0 : 0.0;
  }
  for (int sweep = 0; sweep < 40; ++sweep) {
    bool rotated = false;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        double alpha = 0, beta = 0, gamma = 0;
        for (int k = 0; k < 3; ++k) {
          alpha += B[3 * k + p] * B[3 * k + p];
          beta += B[3 * k + q] * B[3 * k + q];
          gamma += B[3 * k + p] * B[3 * k + q];
        }
        if (gamma == 0.0 || fabs(gamma) <= 1e-17 * sqrt(alpha * beta)) continue;
        rotated = true;
        const double zeta = (beta - alpha) / (2.0 * gamma);
        const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / sqrt(1.0 + t * t), sn = c * t;
        for (int k = 0; k < 3; ++k) {
          const double bp = B[3 * k + p], bq = B[3 * k + q];
          B[3 * k + p] = c * bp - sn * bq;
          B[3 * k + q] = sn * bp + c * bq;
          const double vp = V[3 * k + p], vq = V[3 * k + q];
          V[3 * k + p] = c * vp - sn * vq;
          V[3 * k + q] = sn * vp + c * vq;
        }
      }
    if (!rotated) break;
  }
  double nrm[3];
  for (int j = 0; j < 3; ++j) nrm[j] = sqrt(B[j] * B[j] + B[3 + j] * B[3 + j] + B[6 + j] * B[6 + j]);
  int ord[3] = {0, 1, 2};   // descending, stable
  for (int i = 0; i < 3; ++i)
    for (int j = i + 1; j < 3; ++j)
      if (nrm[ord[j]] > nrm[ord[i]]) {
        const int tmp = ord[i]; ord[i] = ord[j]; ord[j] = tmp;
      }
  double Vs[9];
  for (int j = 0; j < 3; ++j) {
    s[j] = nrm[ord[j]];
    for (int k = 0; k < 3; ++k) Vs[3 * k + j] = V[3 * k + ord[j]];
  }
  for (int i = 0; i < 9; ++i) V[i] = Vs[i];
  double u[3][3];
  const double tiny = 1e-300;
  for (int j = 0; j < 2; ++j) {
    const bool ok = s[j] > tiny && s[j] > 1e-15 * s[0];
    for (int k = 0; k < 3; ++k) u[j][k] = ok ? B[3 * k + ord[j]] / s[j] : 0.0;
    if (!ok) {
      if (j == 0) {
        u[0][0] = 1; u[0][1] = 0; u[0][2] = 0;
      } else {   // any unit vector orthogonal to u0: cross with the axis u0 is least aligned with
        const int a = fabs(u[0][0]) <= fabs(u[0][1]) ? (fabs(u[0][0]) <= fabs(u[0][2]) ? 0 : 2) : (fabs(u[0][1]) <= fabs(u[0][2]) ? 1 : 2);
        double e[3] = {0, 0, 0};
        e[a] = 1;
        u[1][0] = u[0][1] * e[2] - u[0][2] * e[1];
        u[1][1] = u[0][2] * e[0] - u[0][0] * e[2];
        u[1][2] = u[0][0] * e[1] - u[0][1] * e[0];
        const double r = sqrt(u[1][0] * u[1][0] + u[1][1] * u[1][1] + u[1][2] * u[1][2]);
        for (int k = 0; k < 3; ++k) u[1][k] /= r;
      }
    }
  }
  // re-orthogonalise u1 against u0 (one Gram-Schmidt step), then u2 = u0 x u1
  double d = u[0][0] * u[1][0] + u[0][1] * u[1][1] + u[0][2] * u[1][2];
  for (int k = 0; k < 3; ++k) u[1][k] -= d * u[0][k];
  d = sqrt(u[1][0] * u[1][0] + u[1][1] * u[1][1] + u[1][2] * u[1][2]);
  for (int k = 0; k < 3; ++k) u[1][k] /= d;
  u[2][0] = u[0][1] * u[1][2] - u[0][2] * u[1][1];
  u[2][1] = u[0][2] * u[1][0] - u[0][0] * u[1][2];
  u[2][2] = u[0][0] * u[1][1] - u[0][1] * u[1][0];
  for (int j = 0; j < 3; ++j)
    for (int k = 0; k < 3; ++k) U[3 * k + j] = u[j][k];
}

S3R_HD double det3(const double* A) {
  return A[0] * (A[4] * A[8] - A[5] * A[7]) - A[1] * (A[3] * A[8] - A[5] * A[6]) + A[2] * (A[3] * A[7] - A[4] * A[6]);
}

// Rigid least-squares fit dst ~ R src + t from the correspondence sums, taken relative to a fixed shift c (both clouds
// shifted by the same c, so t comes back in the original frame):
//   acc[0] = count, acc[1] = sum d^2 (unused here), acc[2..4] = sum (src - c), acc[5..7] = sum (dst - c),
//   acc[8..16] = sum (src - c)_a (dst - c)_b at 8 + 3a + b.
// Out: 3x4 row-major [R | t].  count == 0 -> identity.  Sigma = cov(dst, src) = U S V^T, R = U diag(1, 1, det(U V^T)) V^T.
S3R_HD void umeyama_rt(const double* acc, const double* c, double* T) {
  for (int i = 0; i < 12; ++i) T[i] = (i % 5 == 0) ? 1.0 : 0.0;
  const double n = acc[0];
  if (!(n > 0)) return;
  double ms[3], md[3];
  for (int a = 0; a < 3; ++a) {
    ms[a] = acc[2 + a] / n;
    md[a] = acc[5 + a] / n;
  }
  double S[9];   // S[a][b] = cov(dst_a, src_b)
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) S[3 * a + b] = acc[8 + 3 * b + a] / n - md[a] * ms[b];
  double U[9], s[3], V[9];
  svd3(S, U, s, V);
  const double d = det3(V) < 0 ? -1.0 : 1.0;   // det(U) = +1 by construction
  double R[9];
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) R[3 * a + b] = U[3 * a] * V[3 * b] + U[3 * a + 1] * V[3 * b + 1] + d * U[3 * a + 2] * V[3 * b + 2];
  for (int a = 0; a < 3; ++a) {
    const double Rms = R[3 * a] * ms[0] + R[3 * a + 1] * ms[1] + R[3 * a + 2] * ms[2];
    const double Rc = R[3 * a] * c[0] + R[3 * a + 1] * c[1] + R[3 * a + 2] * c[2];
    T[4 * a] = R[3 * a]; T[4 * a + 1] = R[3 * a + 1]; T[4 * a + 2] = R[3 * a + 2];
    T[4 * a + 3] = (md[a] - Rms) + (c[a] - Rc);
  }
}

// T <- U T for 3x4 rigid transforms.
S3R_HD void compose_rt(const double* U, double* T) {
  double O[12];
  for (int a = 0; a < 3; ++a) {
    for (int b = 0; b < 4; ++b)
      O[4 * a + b] = U[4 * a] * T[b] + U[4 * a + 1] * T[4 + b] + U[4 * a + 2] * T[8 + b] + (b == 3 ? U[4 * a + 3] : 0.0);
  }
  for (int i = 0; i < 12; ++i) T[i] = O[i];
}

}  // namespace pcl
}  // namespace s3r
