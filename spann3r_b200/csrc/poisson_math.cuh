// Scalar math of the screened Poisson reconstruction (csrc/poisson.cu): the grid geometry, trilinear hat weights, the
// element tables of the dense-grid discretisation, marching tetrahedra on the Kuhn split, and numpy's 'linear'
// quantile lerp.  `__host__ __device__` with no CUDA dependencies, so tests/native/poisson_host_check.cpp compiles THIS
// header with g++ and tests/test_poisson.py checks it bit for bit against a numpy restatement on the CPU.
//
// The discrete problem (restated in numpy / scipy by the tests):
//   * Cube of side L = scale * (largest bounding-box extent) centred on the box; R = 2^depth cells per side, h = L / R,
//     (R + 1)^3 nodes with trilinear hats phi_i.  Node (x, y, z) has linear index (z (R + 1) + y) (R + 1) + x, cell
//     (x, y, z) has (z R + y) R + x.  A sample lies in cell clamp(floor((p - origin) / h), 0, R - 1) per axis.
//   * a = (occupied cells) h^2 / N per sample; unit normals (a zero normal stays zero); v_j = (a / h^3) sum phi_j(s) n_s.
//   * (K + beta S) chi = b with K_ij = int grad phi_i . grad phi_j, S_ij = sum_s phi_i(s) phi_j(s), beta = kAlpha a,
//     b_i = int grad phi_i . V with V = sum_j v_j phi_j; natural (Neumann) boundary: every integral runs over the cube.
//     On one cell with unit-cube corners p, q (bit 0 = x, 1 = y, 2 = z):
//       int grad phi_p . grad phi_q = h * stiffness(popcount(p ^ q))
//       int d_d phi_p phi_q         = h^2 * (p_d ? +1 : -1) * divergence(#axes e != d with p_e != q_e)
//   * Iso value: the mean of chi interpolated at the samples.  Surface: marching tetrahedra on the Kuhn split.
//   Every rounded step below is one fp64 operation in a fixed order (mul_rn / add_rn / sub_rn / div_rn).
#pragma once
#include <math.h>
#include <stdint.h>

#include "pointcloud_math.cuh"   // S3R_HD, mul_rn / add_rn / sub_rn
#include "render_math.cuh"       // div_rn, to_f32_rn

namespace s3r {
namespace poisson {

using pcl::add_rn;
using pcl::mul_rn;
using pcl::sub_rn;
using render::div_rn;
using render::to_f32_rn;

constexpr double kAlpha = 4.0;   // screening weight of Kazhdan & Hoppe 2013's experiments: beta = kAlpha * a
constexpr int kMinDepth = 1, kMaxDepth = 10;

S3R_HD double stiffness(int differing_axes) {
  return differing_axes == 0 ? 1.0 / 3.0 : differing_axes == 1 ? 0.0 : -1.0 / 12.0;
}
// Row sum of |stiffness| over one cell's 8 corners: 1/3 + 3 * 0 + 3 / 12 + 1 / 12 (the l1-Jacobi diagonal, / h)
constexpr double kStiffnessL1 = 2.0 / 3.0;
S3R_HD double divergence(int differing_other_axes) {
  return differing_other_axes == 0 ? 1.0 / 18.0 : differing_other_axes == 1 ? 1.0 / 36.0 : 1.0 / 72.0;
}
S3R_HD int popcount3(int m) { return (m & 1) + ((m >> 1) & 1) + ((m >> 2) & 1); }

// Geometry of the cube from the bounding box: origin (its lower corner), side L and spacing h at `depth`.
S3R_HD void grid_geometry(const double* lo, const double* hi, double scale, int depth, double* origin, double* L,
                          double* h) {
  double m = 0.0;
  for (int d = 0; d < 3; ++d) {
    const double e = sub_rn(hi[d], lo[d]);
    m = e > m ? e : m;
  }
  *L = mul_rn(scale, m);
  for (int d = 0; d < 3; ++d) origin[d] = sub_rn(mul_rn(add_rn(lo[d], hi[d]), 0.5), mul_rn(*L, 0.5));
  *h = div_rn(*L, (double)(1 << depth));
}

// Grid coordinate of one axis: (p - origin) / h.
S3R_HD double grid_coord(double p, double origin, double h) { return div_rn(sub_rn(p, origin), h); }

S3R_HD int cell_of(double g, int R) {
  const double f = floor(g);
  return f < 0.0 ? 0 : f > (double)(R - 1) ? R - 1 : (int)f;
}

// Hat weight of corner q (bit 0 = x, 1 = y, 2 = z) at local coordinates f: ((wx wy) wz), w = f or 1 - f.
S3R_HD double corner_weight(const double* f, int q) {
  const double wx = (q & 1) ? f[0] : sub_rn(1.0, f[0]);
  const double wy = (q & 2) ? f[1] : sub_rn(1.0, f[1]);
  const double wz = (q & 4) ? f[2] : sub_rn(1.0, f[2]);
  return mul_rn(mul_rn(wx, wy), wz);
}

// n / |n|, |n| = sqrt((nx nx + ny ny) + nz nz); a zero normal stays zero.
S3R_HD void unit_normal(const double* n, double* u) {
  const double nn = sqrt(add_rn(add_rn(mul_rn(n[0], n[0]), mul_rn(n[1], n[1])), mul_rn(n[2], n[2])));
  for (int d = 0; d < 3; ++d) u[d] = nn > 0.0 ? div_rn(n[d], nn) : 0.0;
}

S3R_HD double node_coord(double origin, double h, int i) { return add_rn(origin, mul_rn(h, (double)i)); }

// ---------------------------------------------------------------------------------------------------------------------
// Marching tetrahedra.  Cell corners are masks (bit 0 = +x, 1 = +y, 2 = +z).  Kuhn tetrahedron t has corners 0, e_a,
// e_a + e_b, 7 for the t-th permutation (a, b, c) of the axes in lexicographic order; its orientation is the
// permutation's sign.  A node is "outside" when chi > iso.  Tet-local edge k joins local vertices kTetEdge[k]; the edge
// from corner u to corner w (u a subset of w) is owned by node (cell + u) in direction w ^ u.
// kCaseTris[code]: triangle count, then tet-local edges of up to two triangles, for a positively oriented tetrahedron
// and code = sum outside(v_k) << k; the geometric normal points towards the outside vertices.  A negatively oriented
// tetrahedron swaps each triangle's last two edges.
// ---------------------------------------------------------------------------------------------------------------------
S3R_HD int tet_corner(int t, int k) {
  // axes as masks, permutations (0 1 2) (0 2 1) (1 0 2) (1 2 0) (2 0 1) (2 1 0)
  const int a = t < 2 ? 1 : t < 4 ? 2 : 4;
  const int b = (t == 0 || t == 5) ? 2 : (t == 1 || t == 3) ? 4 : 1;
  return k == 0 ? 0 : k == 1 ? a : k == 2 ? (a | b) : 7;
}
S3R_HD bool tet_positive(int t) { return t == 0 || t == 3 || t == 4; }
S3R_HD int tet_edge_vertex(int e, int end) {
  // (0 1) (0 2) (0 3) (1 2) (1 3) (2 3)
  const int a = e < 3 ? 0 : e < 5 ? 1 : 2;
  const int b = e == 0 ? 1 : (e == 1 || e == 3) ? 2 : 3;
  return end ? b : a;
}
S3R_HD int case_triangles(int code, int* edges) {
  static const signed char kCaseTris[16][7] = {
      {0, 0, 0, 0, 0, 0, 0}, {1, 0, 2, 1, 0, 0, 0}, {1, 0, 3, 4, 0, 0, 0}, {2, 1, 3, 4, 1, 4, 2},
      {1, 1, 5, 3, 0, 0, 0}, {2, 0, 5, 3, 0, 2, 5}, {2, 0, 1, 5, 0, 5, 4}, {1, 2, 5, 4, 0, 0, 0},
      {1, 2, 4, 5, 0, 0, 0}, {2, 0, 4, 5, 0, 5, 1}, {2, 0, 5, 2, 0, 3, 5}, {1, 1, 3, 5, 0, 0, 0},
      {2, 1, 2, 4, 1, 4, 3}, {1, 0, 4, 3, 0, 0, 0}, {1, 0, 1, 2, 0, 0, 0}, {0, 0, 0, 0, 0, 0, 0}};
  const int n = kCaseTris[code][0];
  for (int i = 0; i < 3 * n; ++i) edges[i] = kCaseTris[code][1 + i];
  return n;
}

// One coordinate of the vertex on the edge from node value va at xa to vb at xb (exactly one of va, vb > iso):
// t = (iso - va) / (vb - va), x = xa + t (xb - xa), rounded once to fp32.
S3R_HD float edge_point(double xa, double xb, double va, double vb, double iso) {
  const double t = div_rn(sub_rn(iso, va), sub_rn(vb, va));
  return to_f32_rn(add_rn(xa, mul_rn(t, sub_rn(xb, xa))));
}

// ---------------------------------------------------------------------------------------------------------------------
// numpy's default ('linear') quantile of n values: virtual index (n - 1) q; the order statistics floor and floor + 1
// (both n - 1 at or past the end, where numpy's gamma is taken against index -1); lerp(a, b, g) = a + (b - a) g, or
// b - (b - a) (1 - g) when g >= 0.5.
// ---------------------------------------------------------------------------------------------------------------------
S3R_HD void quantile_ranks(long long n, double q, long long* lo, long long* hi, double* gamma) {
  const double vi = mul_rn((double)(n - 1), q);
  if (vi >= (double)(n - 1)) {
    *lo = *hi = n - 1;
    *gamma = sub_rn(vi, -1.0);
    return;
  }
  const double f = floor(vi);
  *lo = (long long)f;
  *hi = *lo + 1;
  *gamma = sub_rn(vi, f);
}

S3R_HD double quantile_lerp(double a, double b, double g) {
  const double d = sub_rn(b, a);
  return g >= 0.5 ? sub_rn(b, mul_rn(d, sub_rn(1.0, g))) : add_rn(a, mul_rn(d, g));
}

}  // namespace poisson
}  // namespace s3r
