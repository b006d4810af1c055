// TEST HARNESS (not a product path): compiles the product's device math header, spann3r_b200/csrc/pointcloud_math.cuh,
// with g++ so tests/test_recon_eval.py can check the Umeyama / Kabsch fit, the 3x3 eigen solver, the k-NN normal and
// the box lower bound of the spatial index against numpy without a GPU.
#include "../../spann3r_b200/csrc/pointcloud_math.cuh"

using namespace s3r::pcl;

// dst ~ R src + t from n pairs; the sums are taken relative to the shift c, as csrc/pointcloud.cu accumulates them.
extern "C" void rc_umeyama(const double* src, const double* dst, int n, const double* c, double* T12) {
  double acc[17] = {0};
  for (int i = 0; i < n; ++i) {
    double ps[3], qs[3];
    for (int a = 0; a < 3; ++a) {
      ps[a] = src[3 * i + a] - c[a];
      qs[a] = dst[3 * i + a] - c[a];
    }
    acc[0] += 1;
    for (int a = 0; a < 3; ++a) {
      acc[2 + a] += ps[a];
      acc[5 + a] += qs[a];
      for (int b = 0; b < 3; ++b) acc[8 + 3 * a + b] += ps[a] * qs[b];
    }
  }
  umeyama_rt(acc, c, T12);
}

extern "C" void rc_smallest_eigvec(const double* C9, double* n3) { smallest_eigvec(C9, n3); }

struct Flat {
  const double* p;
  double operator()(int i, int a) const { return p[3 * i + a]; }
};
extern "C" void rc_knn_normal(const double* pts, int k, double* n3) { knn_normal(Flat{pts}, k, n3); }

extern "C" double rc_dist2(const double* q, const double* p) { return dist2(q, p); }
extern "C" double rc_box_lb2(const double* q, const double* lo, const double* hi) { return box_lb2(q, lo, hi); }
