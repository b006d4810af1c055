// TEST HARNESS (not a product path): compiles the product's device math header, spann3r_b200/csrc/mesh_math.cuh, with
// g++ so tests/test_mesh.py can check app.py's grid faces and the triangle rasteriser's coverage, depth and keys bit for
// bit against oracle/mesh_oracle.py without a GPU.
#include "../../spann3r_b200/csrc/mesh_math.cuh"

using namespace s3r::mesh;

static Camera camera_of(const double* camera) {
  Camera c;
  for (int i = 0; i < 12; ++i) c.rt[i] = camera[i];
  c.fx = camera[12]; c.fy = camera[13]; c.cx = camera[14]; c.cy = camera[15];
  return c;
}

// candidate faces g0 .. g0 + n - 1 of a T x H x W grid -> faces [n, 3], colour pixel [n]
extern "C" void mh_grid_faces(long long g0, long long n, int H, int W, long long* faces, long long* color) {
  for (long long i = 0; i < n; ++i) {
    const GridFace f = grid_face(g0 + i, H, W);
    for (int a = 0; a < 3; ++a) faces[3 * i + a] = f.v[a];
    color[i] = f.color;
  }
}

// The whole draw, serially: keys [h * w] <- min(keys, key of every covered centre of every face); cover[h * w] counts
// the covered centres (before the depth test), so a caller can check that a tessellation covers each centre once.
extern "C" void mh_raster(const float* verts, long long n_verts, const int* faces, long long n_faces, long long id0,
                          const double* camera, double z_near, double z_far, int w, int h, unsigned long long* keys,
                          int* cover) {
  const Camera c = camera_of(camera);
  for (long long f = 0; f < n_faces; ++f) {
    const int* ix = faces + 3 * f;
    if (ix[0] < 0 || ix[1] < 0 || ix[2] < 0 || ix[0] >= n_verts || ix[1] >= n_verts || ix[2] >= n_verts) continue;
    Tri t;
    if (!setup_tri(c, z_near, w, h, verts + 3LL * ix[0], verts + 3LL * ix[1], verts + 3LL * ix[2], &t)) continue;
    for (int r = t.r0; r <= t.r1; ++r)
      for (int col = t.c0; col <= t.c1; ++col) {
        // coverage alone: the key with an infinite far plane is empty only when the centre is not covered or the
        // depth is not finite
        const uint64_t k = tri_key(t, col, r, z_far, (uint32_t)(id0 + f));
        const uint64_t any = tri_key(t, col, r, INFINITY, (uint32_t)(id0 + f));
        const long long p = (long long)r * w + col;
        if (any != kEmptyKey && cover) ++cover[p];
        if (k < keys[p]) keys[p] = k;
      }
  }
}
