// TEST HARNESS (not a product path): compiles the product's device math header, spann3r_b200/csrc/render_math.cuh,
// with g++ so tests/test_vis.py can check the point projection, the depth key and the colour rounding bit for bit
// against oracle/render_oracle.py without a GPU.
#include "../../spann3r_b200/csrc/render_math.cuh"

using namespace s3r::render;

// n fp32 points [n, 3] with global indices id0 + i -> pix[i] (row * w + col, -1 = dropped), key[i] (kEmptyKey = dropped).
extern "C" void rh_project(const float* pts, long long n, const double* camera, double z_near, int w, int h,
                           long long id0, long long* pix, unsigned long long* key) {
  Camera c;
  for (int i = 0; i < 12; ++i) c.rt[i] = camera[i];
  c.fx = camera[12]; c.fy = camera[13]; c.cx = camera[14]; c.cy = camera[15];
  for (long long i = 0; i < n; ++i) {
    uint64_t k = kEmptyKey;
    pix[i] = project_point(c, z_near, w, h, pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], (uint32_t)(id0 + i), &k);
    key[i] = pix[i] >= 0 ? k : kEmptyKey;
  }
}

extern "C" void rh_color_u8(const float* c, long long n, unsigned char* out) {
  for (long long i = 0; i < n; ++i) out[i] = color_u8(c[i]);
}
