// TEST HARNESS (not a product path): compiles the product's device math header, spann3r_b200/csrc/poisson_math.cuh,
// with g++ so tests/test_poisson.py can check the grid geometry, hat weights, marching-tetrahedra tables, edge points and
// numpy's quantile lerp bit for bit against oracle/poisson_oracle.py without a GPU.
#include "../../spann3r_b200/csrc/poisson_math.cuh"

using namespace s3r::poisson;

extern "C" void ph_geometry(const double* lo, const double* hi, double scale, int depth, double* out5) {
  grid_geometry(lo, hi, scale, depth, out5, out5 + 3, out5 + 4);
}

// n points [n, 3] -> cells [n, 3], local coordinates [n, 3], corner weights [n, 8]
extern "C" void ph_locate(const double* p, long long n, const double* origin, double h, int R, long long* cells,
                          double* f, double* w) {
  for (long long i = 0; i < n; ++i) {
    for (int d = 0; d < 3; ++d) {
      const double g = grid_coord(p[3 * i + d], origin[d], h);
      cells[3 * i + d] = cell_of(g, R);
      f[3 * i + d] = sub_rn(g, (double)cells[3 * i + d]);
    }
    for (int q = 0; q < 8; ++q) w[8 * i + q] = corner_weight(f + 3 * i, q);
  }
}

extern "C" void ph_unit_normals(const double* n, long long count, double* u) {
  for (long long i = 0; i < count; ++i) unit_normal(n + 3 * i, u + 3 * i);
}

// tetrahedron t -> its 4 corner masks; returns 1 when positively oriented
extern "C" int ph_tet(int t, int* corners) {
  for (int k = 0; k < 4; ++k) corners[k] = tet_corner(t, k);
  return tet_positive(t) ? 1 : 0;
}

extern "C" int ph_case(int code, int* edges) { return case_triangles(code, edges); }

extern "C" void ph_edge_vertices(int* out12) {
  for (int e = 0; e < 6; ++e) {
    out12[2 * e] = tet_edge_vertex(e, 0);
    out12[2 * e + 1] = tet_edge_vertex(e, 1);
  }
}

extern "C" void ph_edge_points(const double* xa, const double* xb, const double* va, const double* vb, double iso,
                               long long n, float* out) {
  for (long long i = 0; i < n; ++i) out[i] = edge_point(xa[i], xb[i], va[i], vb[i], iso);
}

extern "C" double ph_quantile(const double* sorted, long long n, double q) {
  long long lo, hi;
  double g;
  quantile_ranks(n, q, &lo, &hi, &g);
  return quantile_lerp(sorted[lo], sorted[hi], g);
}
