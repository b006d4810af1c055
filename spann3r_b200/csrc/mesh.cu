// Triangle meshes on the GPU: app.py's pixel-grid mesh (pts3d_to_trimesh + cat_meshes) and a z-buffered triangle
// rasteriser for spann3r/tools/render_dtu.py's depth maps and for drawing that mesh.
//
//   mesh_grid_count_kernel  one CTA per tile of kGridTile candidate faces (app.py's order, mesh_math.cuh grid_face):
//                           the number of faces whose three corners are valid.
//   mesh_grid_scan_kernel   one CTA: exclusive scan of the tile counts, the total after the last tile.
//   mesh_grid_write_kernel  one CTA per tile again: a block scan of the per-thread counts places every kept face at its
//                           tile's offset, so the face list keeps app.py's order and no atomic decides it.
//   raster_kernel           one thread per triangle (projection, area, bounding box in mesh_math.cuh), then a 64-bit
//                           atomicMin of (fp32 depth bits << 32 | face id) per covered pixel centre into the point
//                           rasteriser's key buffer.  A triangle whose bounding box holds more than kRasterBigBox
//                           pixels is not scanned by its thread: it goes to the CTA's second pass, in which all of the
//                           CTA's threads stride over that one triangle's box.  The minimum does not depend on the order
//                           the atomics land in, so the result depends neither on scheduling nor on the pass.
//   raster_resolve_kernel   one thread per pixel: fp32 depth (0 where empty) and int32 face id (-1 where empty).
#include "kernels.cuh"

#include <math.h>

#include "mesh_math.cuh"

#ifndef S3R_RASTER_BIG_BBOX
#define S3R_RASTER_BIG_BBOX 256
#endif

namespace s3r {

using namespace mesh;

namespace {

constexpr int kGridThreads = 256, kGridPerThread = 8, kGridTile = kGridThreads * kGridPerThread;
constexpr int kScanThreads = 1024;
constexpr int kRasterThreads = 256;
constexpr long long kRasterBigBox = S3R_RASTER_BIG_BBOX;   // pixels; chosen with tools/bench_mesh.py (DESIGN.md §6)

// Exclusive block scan of one value per thread (blockDim.x == NT, a multiple of 32); *total gets the block's sum.
template <int NT>
__device__ long long block_exclusive_scan(long long v, long long* total) {
  __shared__ long long warp_sums[NT / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long x = v;
  for (int o = 1; o < 32; o <<= 1) {
    const long long y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[warp] = x;
  __syncthreads();
  if (warp == 0) {
    long long s = lane < NT / 32 ? warp_sums[lane] : 0;
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    if (lane < NT / 32) warp_sums[lane] = s;   // inclusive over warps
  }
  __syncthreads();
  const long long before = warp ? warp_sums[warp - 1] : 0;
  *total = warp_sums[NT / 32 - 1];
  __syncthreads();   // warp_sums may be reused by the next call
  return before + x - v;
}

__device__ __forceinline__ bool face_valid(const uint8_t* __restrict__ valid, const GridFace& f) {
  return valid[f.v[0]] && valid[f.v[1]] && valid[f.v[2]];
}

__global__ void __launch_bounds__(kGridThreads)
    mesh_grid_count_kernel(const uint8_t* __restrict__ valid, int H, int W, long long n_cand,
                           long long* __restrict__ counts) {
  const long long g0 = blockIdx.x * (long long)kGridTile + threadIdx.x * (long long)kGridPerThread;
  long long n = 0;
  for (int j = 0; j < kGridPerThread; ++j)
    if (g0 + j < n_cand) n += face_valid(valid, grid_face(g0 + j, H, W));
  long long total;
  block_exclusive_scan<kGridThreads>(n, &total);
  if (threadIdx.x == 0) counts[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kScanThreads) mesh_grid_scan_kernel(long long* __restrict__ counts, long long n_tiles) {
  long long carry = 0;
  for (long long base = 0; base < n_tiles; base += kScanThreads) {
    const long long i = base + threadIdx.x;
    const long long v = i < n_tiles ? counts[i] : 0;
    long long total;
    const long long ex = block_exclusive_scan<kScanThreads>(v, &total);
    if (i < n_tiles) counts[i] = carry + ex;
    carry += total;
  }
  if (threadIdx.x == 0) counts[n_tiles] = carry;
}

__global__ void __launch_bounds__(kGridThreads)
    mesh_grid_write_kernel(const uint8_t* __restrict__ valid, const float* __restrict__ images, int H, int W,
                           long long n_cand, const long long* __restrict__ offsets, int* __restrict__ faces,
                           float* __restrict__ colors) {
  const long long g0 = blockIdx.x * (long long)kGridTile + threadIdx.x * (long long)kGridPerThread;
  unsigned keep = 0;
  long long n = 0;
  for (int j = 0; j < kGridPerThread; ++j)
    if (g0 + j < n_cand && face_valid(valid, grid_face(g0 + j, H, W))) {
      keep |= 1u << j;
      ++n;
    }
  long long total;
  long long o = offsets[blockIdx.x] + block_exclusive_scan<kGridThreads>(n, &total);
  for (int j = 0; j < kGridPerThread; ++j) {
    if (!(keep >> j & 1u)) continue;
    const GridFace f = grid_face(g0 + j, H, W);
    for (int a = 0; a < 3; ++a) {
      faces[3 * o + a] = (int)f.v[a];
      colors[3 * o + a] = images[3 * f.color + a];
    }
    ++o;
  }
}

__device__ __forceinline__ bool load_tri(const float* __restrict__ verts, long long n_verts,
                                         const int* __restrict__ faces, long long f, const Camera& cam, double z_near,
                                         int w, int h, Tri* t) {
  const int a = faces[3 * f], b = faces[3 * f + 1], c = faces[3 * f + 2];
  if (a < 0 || b < 0 || c < 0 || a >= n_verts || b >= n_verts || c >= n_verts) return false;
  return setup_tri(cam, z_near, w, h, verts + 3LL * a, verts + 3LL * b, verts + 3LL * c, t);
}

__global__ void __launch_bounds__(kRasterThreads)
    raster_kernel(const float* __restrict__ verts, long long n_verts, const int* __restrict__ faces, long long n_faces,
                  unsigned id0, const Camera cam, double z_near, double z_far, int w, int h,
                  unsigned long long* __restrict__ keys) {
  __shared__ int big[kRasterThreads];
  __shared__ int n_big;
  if (threadIdx.x == 0) n_big = 0;
  __syncthreads();
  const long long f = blockIdx.x * (long long)kRasterThreads + threadIdx.x;
  Tri t;
  if (f < n_faces && load_tri(verts, n_verts, faces, f, cam, z_near, w, h, &t)) {
    const long long box = (long long)(t.c1 - t.c0 + 1) * (t.r1 - t.r0 + 1);
    if (box > kRasterBigBox) {
      big[atomicAdd(&n_big, 1)] = threadIdx.x;   // the order of this list does not reach the result
    } else {
      const unsigned id = id0 + (unsigned)f;
      for (int r = t.r0; r <= t.r1; ++r)
        for (int c = t.c0; c <= t.c1; ++c) {
          const uint64_t k = tri_key(t, c, r, z_far, id);
          if (k != kEmptyKey) atomicMin(keys + (long long)r * w + c, (unsigned long long)k);
        }
    }
  }
  __syncthreads();
  // second pass: the CTA's large triangles one at a time, every thread on a share of the box
  for (int j = 0; j < n_big; ++j) {
    const long long g = blockIdx.x * (long long)kRasterThreads + big[j];
    Tri s;
    load_tri(verts, n_verts, faces, g, cam, z_near, w, h, &s);   // the same setup its own thread made
    const int bw = s.c1 - s.c0 + 1;
    const long long box = (long long)bw * (s.r1 - s.r0 + 1);
    const unsigned id = id0 + (unsigned)g;
    for (long long k = threadIdx.x; k < box; k += kRasterThreads) {
      const int r = s.r0 + (int)(k / bw), c = s.c0 + (int)(k % bw);
      const uint64_t key = tri_key(s, c, r, z_far, id);
      if (key != kEmptyKey) atomicMin(keys + (long long)r * w + c, (unsigned long long)key);
    }
  }
}

__global__ void __launch_bounds__(kRasterThreads)
    raster_resolve_kernel(const unsigned long long* __restrict__ keys, long long npix, float* __restrict__ depth,
                          int* __restrict__ face) {
  const long long i = blockIdx.x * (long long)kRasterThreads + threadIdx.x;
  if (i >= npix) return;
  const unsigned long long k = keys[i];
  depth[i] = k == kEmptyKey ? 0.0f : __uint_as_float((unsigned)(k >> 32));
  face[i] = k == kEmptyKey ? -1 : (int)(k & 0xffffffffULL);
}

bool grid_ok(int T, int H, int W) {
  return T >= 1 && H >= 1 && W >= 1 && (long long)T * H * W < (1LL << 31);
}

long long grid_tiles(int T, int H, int W) {
  const long long n_cand = 4LL * T * (H - 1) * (W - 1);
  return (n_cand + kGridTile - 1) / kGridTile;
}

bool raster_size_ok(int w, int h) { return w >= 1 && h >= 1 && (long long)w * h < (1LL << 31); }

int launched(const char* what) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: launch failed: %s", what, cudaGetErrorString(e));
    return -6;
  }
  return 0;
}

}  // namespace

size_t mesh_grid_workspace_bytes(int T, int H, int W) {
  return grid_ok(T, H, W) ? sizeof(long long) * (size_t)(grid_tiles(T, H, W) + 1) : 0;
}

int launch_mesh_grid_count(const uint8_t* valid, int T, int H, int W, void* workspace, size_t workspace_bytes,
                           long long* n_faces, cudaStream_t st) {
  if (!grid_ok(T, H, W) || !valid || !workspace || (uintptr_t)workspace % 8 || !n_faces ||
      workspace_bytes < mesh_grid_workspace_bytes(T, H, W)) {
    set_error("mesh_grid_count: bad arguments (T=%d H=%d W=%d workspace_bytes=%zu; need T, H, W >= 1, T * H * W < 2^31, "
              "an 8-byte aligned workspace of mesh_grid_workspace_bytes and non-null pointers)", T, H, W, workspace_bytes);
    return -1;
  }
  const long long n_cand = 4LL * T * (H - 1) * (W - 1), n_tiles = grid_tiles(T, H, W);
  long long* counts = (long long*)workspace;
  if (n_tiles > 0) {
    mesh_grid_count_kernel<<<(unsigned)n_tiles, kGridThreads, 0, st>>>(valid, H, W, n_cand, counts);
    if (int e = launched("mesh_grid_count")) return e;
  }
  mesh_grid_scan_kernel<<<1, kScanThreads, 0, st>>>(counts, n_tiles);
  if (int e = launched("mesh_grid_scan")) return e;
  if (cudaMemcpyAsync(n_faces, counts + n_tiles, sizeof(long long), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
      cudaStreamSynchronize(st) != cudaSuccess)
    return launched("mesh_grid_count (face count read)");
  return 0;
}

int launch_mesh_grid_faces(const uint8_t* valid, const float* images, int T, int H, int W, const void* workspace,
                           size_t workspace_bytes, int* faces, float* colors, cudaStream_t st) {
  if (!grid_ok(T, H, W) || !valid || !images || !workspace || (uintptr_t)workspace % 8 ||
      workspace_bytes < mesh_grid_workspace_bytes(T, H, W)) {
    set_error("mesh_grid_faces: bad arguments (T=%d H=%d W=%d workspace_bytes=%zu; need T, H, W >= 1, T * H * W < 2^31, "
              "the workspace mesh_grid_count filled and non-null pointers)", T, H, W, workspace_bytes);
    return -1;
  }
  const long long n_cand = 4LL * T * (H - 1) * (W - 1), n_tiles = grid_tiles(T, H, W);
  if (n_tiles == 0) return 0;
  if (!faces || !colors) {
    set_error("mesh_grid_faces: faces and colors must be non-null");
    return -1;
  }
  mesh_grid_write_kernel<<<(unsigned)n_tiles, kGridThreads, 0, st>>>(valid, images, H, W, n_cand,
                                                                      (const long long*)workspace, faces, colors);
  return launched("mesh_grid_faces");
}

int launch_raster_triangles(const float* verts, long long n_verts, const int* faces, long long n_faces, long long id0,
                            const double* camera, double z_near, double z_far, int w, int h, void* keys,
                            cudaStream_t st) {
  if (!verts || !faces || !camera || !keys || (uintptr_t)keys % 8 || !raster_size_ok(w, h) || n_verts < 0 ||
      n_verts >= (1LL << 31) || n_faces < 0 || id0 < 0 || id0 + n_faces >= (1LL << 31)) {
    set_error("raster_triangles: bad arguments (n_verts=%lld n_faces=%lld id0=%lld w=%d h=%d; need n_verts < 2^31, "
              "id0 + n_faces < 2^31, w, h >= 1, w * h < 2^31, an 8-byte aligned key buffer and non-null pointers)",
              n_verts, n_faces, id0, w, h);
    return -1;
  }
  if (!(z_near >= 0.0) || !isfinite(z_near) || !(z_far > z_near)) {
    set_error("raster_triangles: z_near=%g must be finite and >= 0, and z_far=%g > z_near (inf allowed)", z_near, z_far);
    return -1;
  }
  for (int i = 0; i < 16; ++i) {
    if (!isfinite(camera[i])) {
      set_error("raster_triangles: camera[%d]=%g is not finite", i, camera[i]);
      return -1;
    }
  }
  Camera cam;
  for (int i = 0; i < 12; ++i) cam.rt[i] = camera[i];
  cam.fx = camera[12]; cam.fy = camera[13]; cam.cx = camera[14]; cam.cy = camera[15];
  if (n_faces == 0) return 0;
  raster_kernel<<<(unsigned)((n_faces + kRasterThreads - 1) / kRasterThreads), kRasterThreads, 0, st>>>(
      verts, n_verts, faces, n_faces, (unsigned)id0, cam, z_near, z_far, w, h, (unsigned long long*)keys);
  return launched("raster_triangles");
}

int launch_raster_resolve(const void* keys, int w, int h, float* depth, int* face, cudaStream_t st) {
  if (!keys || (uintptr_t)keys % 8 || !depth || !face || !raster_size_ok(w, h)) {
    set_error("raster_resolve: bad arguments (w=%d h=%d; need w, h >= 1, w * h < 2^31, an 8-byte aligned key buffer and "
              "non-null pointers)", w, h);
    return -1;
  }
  const long long npix = (long long)w * h;
  raster_resolve_kernel<<<(unsigned)((npix + kRasterThreads - 1) / kRasterThreads), kRasterThreads, 0, st>>>(
      (const unsigned long long*)keys, npix, depth, face);
  return launched("raster_resolve");
}

}  // namespace s3r
