// TEST HARNESS (not a product path): compiles the product's device math header, spann3r_b200/csrc/views_math.cuh,
// with g++ so tests/test_views.py can check the unprojection, the world transform and the validity rule bit for bit
// against oracle/views_oracle.py without a GPU.
#include "../../spann3r_b200/csrc/views_math.cuh"

using namespace s3r::views;

// depth [h, w] fp32, intr (fu, fv, cu, cv), pose 3x4 row-major -> cam [h, w, 3], world [h, w, 3], valid [h, w] (0 / 1)
extern "C" void vh_points(const float* depth, int h, int w, const float* intr, const float* pose, float* cam, float* world,
                          unsigned char* valid) {
  ViewCam c;
  for (int i = 0; i < 4; ++i) c.intr[i] = intr[i];
  for (int i = 0; i < 12; ++i) c.pose[i] = pose[i];
  for (int y = 0; y < h; ++y) {
    for (int x = 0; x < w; ++x) {
      const long long i = (long long)y * w + x;
      unproject(c, x, y, depth[i], cam + 3 * i);
      to_world(c, cam + 3 * i, world + 3 * i);
      valid[i] = valid_point(depth[i], world + 3 * i) ? 1 : 0;
    }
  }
}
