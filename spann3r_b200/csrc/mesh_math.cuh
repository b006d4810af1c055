// Scalar math of the triangle mesh kernels (csrc/mesh.cu): app.py's pixel-grid faces, and the projection, coverage and
// depth of the z-buffered triangle rasteriser.  `__host__ __device__` with no CUDA dependencies, so
// tests/native/mesh_host_check.cpp compiles THIS header with g++ and tests/test_mesh.py checks it bit for bit against
// a numpy restatement on the CPU.
//
// Rasteriser conventions (those of render_math.cuh): pinhole camera, [R | t] world -> camera, pixel centres at integer
// (u, v) = (col, row), row 0 at the top.  Every step is one rounded fp64 operation in a fixed order.
//   * A vertex projects to (u, v, qz) exactly as project_point projects a point; a triangle is skipped when a vertex is
//     not finite or has qz <= z_near (no near-plane clipping).
//   * Edge function of the directed edge a -> b at p: E(a, b, p) = (px - ax) (by - ay) - (py - ay) (bx - ax).  It is
//     always evaluated from the lexicographically smaller (x, y) end and negated when the edge runs the other way, so
//     E(b, a, p) == -E(a, b, p) exactly: two triangles that share an edge see the same value with opposite signs.
//   * Signed area: E of the three vertices sorted by (x, y), negated for an odd permutation, so it is exactly invariant
//     under rotation of the vertex order and exactly negated by reversal.  Area > 0 (counter-clockwise on the image,
//     GL's default front face) is drawn; area <= 0 (back face, degenerate) or a non-finite area is skipped.
//   * A centre p is covered when every edge has E > 0, or E == 0 and the edge is a top or left edge (top-left rule in
//     image coordinates): dy > 0, or dy == 0 and dx < 0, with (dx, dy) = b - a.  Reversing an edge flips both tests, so
//     a centre on a shared edge goes to exactly one of the two triangles.
//   * Depth is perspective-correct: b_i = E_i / area, 1 / z = (b0 / z0 + b1 / z1) + b2 / z2, depth = fp32(1 / (1 / z)).
//     A depth that is not finite, or > z_far, is dropped.  The key is (bits(depth) << 32) | face id, as for points.
#pragma once
#include <math.h>
#include <stdint.h>

#include "render_math.cuh"   // Camera, kEmptyKey, mul_rn / add_rn / div_rn, to_f32_rn, f32_bits

namespace s3r {
namespace mesh {

using pcl::add_rn;
using pcl::mul_rn;
using pcl::sub_rn;
using render::Camera;
using render::div_rn;
using render::f32_bits;
using render::kEmptyKey;
using render::to_f32_rn;

// ---------------------------------------------------------------------------------------------------------------------
// app.py's pts3d_to_trimesh + cat_meshes: candidate face g of a T x H x W grid, in app.py's order.  With Q = (H-1)(W-1)
// quads per frame, g = (t * 4 + block) * Q + quad, quads row-major.  Corners (frame-local) i1 = top-left, i2 = top-right,
// i3 = bottom-left, i4 = bottom-right; blocks [i1,i2,i3], [i3,i2,i1], [i2,i3,i4], [i4,i3,i2].  Blocks 0-1 take the
// colour of the quad's top-left pixel, blocks 2-3 that of its bottom-right pixel.  Indices are offset by t H W.
// ---------------------------------------------------------------------------------------------------------------------
struct GridFace {
  long long v[3];   // global vertex indices
  long long color;  // global pixel index of the face colour
};

S3R_HD GridFace grid_face(long long g, int H, int W) {
  const long long Q = (long long)(H - 1) * (W - 1);
  const long long q = g % Q, tb = g / Q;
  const long long t = tb / 4, block = tb % 4;
  const long long base = t * H * W;
  const long long i1 = base + (q / (W - 1)) * W + q % (W - 1);
  const long long i2 = i1 + 1, i3 = i1 + W, i4 = i3 + 1;
  GridFace f;
  switch (block) {
    case 0: f.v[0] = i1; f.v[1] = i2; f.v[2] = i3; break;
    case 1: f.v[0] = i3; f.v[1] = i2; f.v[2] = i1; break;
    case 2: f.v[0] = i2; f.v[1] = i3; f.v[2] = i4; break;
    default: f.v[0] = i4; f.v[1] = i3; f.v[2] = i2; break;
  }
  f.color = block < 2 ? i1 : i4;
  return f;
}

// ---------------------------------------------------------------------------------------------------------------------
// Triangle rasteriser
// ---------------------------------------------------------------------------------------------------------------------
struct Vert {
  double x, y, z;   // pixel coordinates (u, v) and camera depth qz
};

// project_point's operation order; false when q is not finite, qz <= z_near or u, v are not finite.
S3R_HD bool project_vertex(const Camera& c, double z_near, float x, float y, float z, Vert* o) {
  const double p[3] = {(double)x, (double)y, (double)z};
  double q[3];
  pcl::apply_rt(c.rt, p, q);
  if (!(isfinite(q[0]) && isfinite(q[1]) && isfinite(q[2])) || !(q[2] > z_near)) return false;
  o->x = add_rn(mul_rn(c.fx, div_rn(q[0], q[2])), c.cx);
  o->y = add_rn(mul_rn(c.fy, div_rn(q[1], q[2])), c.cy);
  o->z = q[2];
  return isfinite(o->x) && isfinite(o->y);
}

S3R_HD bool vert_less(const Vert& a, const Vert& b) { return a.x < b.x || (a.x == b.x && a.y < b.y); }

S3R_HD double edge_raw(const Vert& a, const Vert& b, double px, double py) {
  return sub_rn(mul_rn(sub_rn(px, a.x), sub_rn(b.y, a.y)), mul_rn(sub_rn(py, a.y), sub_rn(b.x, a.x)));
}

// E(a, b, p), exactly antisymmetric in (a, b).
S3R_HD double edge_fn(const Vert& a, const Vert& b, double px, double py) {
  return vert_less(b, a) ? -edge_raw(b, a, px, py) : edge_raw(a, b, px, py);
}

// Signed area (twice it): E of the sorted vertices, sign of the sorting permutation.
S3R_HD double tri_area(const Vert& v0, const Vert& v1, const Vert& v2) {
  Vert a = v0, b = v1, c = v2, t;
  bool odd = false;
  if (vert_less(b, a)) { t = a; a = b; b = t; odd = !odd; }
  if (vert_less(c, b)) { t = b; b = c; c = t; odd = !odd; }
  if (vert_less(b, a)) { t = a; a = b; b = t; odd = !odd; }
  const double s = edge_raw(a, b, c.x, c.y);
  return odd ? -s : s;
}

S3R_HD bool top_left(const Vert& a, const Vert& b) {
  const double dx = sub_rn(b.x, a.x), dy = sub_rn(b.y, a.y);
  return dy > 0.0 || (dy == 0.0 && dx < 0.0);
}

// A triangle ready to be scanned: its vertices, area, which edges own their zero line, and its pixel bounding box
// (inclusive, clipped to the image; empty when c0 > c1 or r0 > r1).
struct Tri {
  Vert v[3];
  double area;
  bool tl[3];   // edge i is v[i+1] -> v[i+2]
  int c0, c1, r0, r1;
};

// false when the triangle draws nothing: a vertex dropped by project_vertex, area <= 0 or not finite, or a bounding box
// that misses every pixel centre.  The bounding box is clipped in fp64 before any conversion to int.
S3R_HD bool setup_tri(const Camera& c, double z_near, int w, int h, const float* p0, const float* p1, const float* p2,
                      Tri* t) {
  if (!project_vertex(c, z_near, p0[0], p0[1], p0[2], &t->v[0]) ||
      !project_vertex(c, z_near, p1[0], p1[1], p1[2], &t->v[1]) ||
      !project_vertex(c, z_near, p2[0], p2[1], p2[2], &t->v[2]))
    return false;
  t->area = tri_area(t->v[0], t->v[1], t->v[2]);
  if (!(t->area > 0.0) || !isfinite(t->area)) return false;
  t->tl[0] = top_left(t->v[1], t->v[2]);
  t->tl[1] = top_left(t->v[2], t->v[0]);
  t->tl[2] = top_left(t->v[0], t->v[1]);
  const double xmin = fmin(fmin(t->v[0].x, t->v[1].x), t->v[2].x), xmax = fmax(fmax(t->v[0].x, t->v[1].x), t->v[2].x);
  const double ymin = fmin(fmin(t->v[0].y, t->v[1].y), t->v[2].y), ymax = fmax(fmax(t->v[0].y, t->v[1].y), t->v[2].y);
  const double c0 = fmax(ceil(xmin), 0.0), c1 = fmin(floor(xmax), (double)(w - 1));
  const double r0 = fmax(ceil(ymin), 0.0), r1 = fmin(floor(ymax), (double)(h - 1));
  if (!(c0 <= c1 && r0 <= r1)) return false;
  t->c0 = (int)c0; t->c1 = (int)c1; t->r0 = (int)r0; t->r1 = (int)r1;
  return true;
}

// The key of the triangle at pixel centre (col, row), or kEmptyKey when the centre is not covered or the depth is
// dropped (not finite or > z_far).
S3R_HD uint64_t tri_key(const Tri& t, int col, int row, double z_far, uint32_t id) {
  const double px = (double)col, py = (double)row;
  const double e0 = edge_fn(t.v[1], t.v[2], px, py);
  if (!(e0 > 0.0 || (e0 == 0.0 && t.tl[0]))) return kEmptyKey;
  const double e1 = edge_fn(t.v[2], t.v[0], px, py);
  if (!(e1 > 0.0 || (e1 == 0.0 && t.tl[1]))) return kEmptyKey;
  const double e2 = edge_fn(t.v[0], t.v[1], px, py);
  if (!(e2 > 0.0 || (e2 == 0.0 && t.tl[2]))) return kEmptyKey;
  const double iz = add_rn(add_rn(div_rn(div_rn(e0, t.area), t.v[0].z), div_rn(div_rn(e1, t.area), t.v[1].z)),
                           div_rn(div_rn(e2, t.area), t.v[2].z));
  const float depth = to_f32_rn(div_rn(1.0, iz));
  if (!isfinite(depth) || (double)depth > z_far) return kEmptyKey;
  return ((uint64_t)f32_bits(depth) << 32) | (uint64_t)id;
}

}  // namespace mesh
}  // namespace s3r
