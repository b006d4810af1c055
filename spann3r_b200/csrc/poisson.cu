// Screened Poisson surface reconstruction on a dense grid (the discrete problem: csrc/poisson_math.cuh), for
// spann3r/tools/render_dtu.py's get_mesh_from_ply without Open3D.  No floating-point atomics anywhere: every sum runs
// in a fixed order, so two calls on the same input give bitwise-identical results.
//
//   setup    poisson_box_{partial,final}   bounding box (fixed-order min / max) and the cube's geometry
//            poisson_keys_kernel           finest-cell key of every sample
//            pcl_radix_sort (pointcloud.cu) stable sort of (key, sample index)
//            poisson_gather_kernel         fp64 positions and unit normals in sorted order
//            poisson_ranges_kernel         [lo, hi) sample range of every cell (dense), occupied-cell count
//            poisson_weights_kernel        a, beta, a / h^3
//            poisson_blocks_kernel         8 x 8 screening block of every occupied cell, stored at the slot of its
//                                          first sorted sample; one thread per (cell, row)
//            poisson_splat_kernel          v at every node: a gather over its <= 8 cells' sample ranges
//            poisson_rhs_kernel            b at every node from v, through the element divergence tables
//            poisson_density_kernel        sample counts at the nodes of the depth max(depth - 2, 1) grid
//   solve    conjugate gradients on (K + beta S) chi = b, preconditioned by one geometric-multigrid V-cycle:
//            poisson_apply_kernel          A x, an l1-Jacobi sweep or a residual at one level, node-centric over the
//                                          node's cells (K from the element table; S from the blocks on the finest
//                                          level only: the coarse levels carry the stiffness alone)
//            poisson_restrict_kernel / poisson_prolong_kernel   trilinear transfer between nested grids
//            poisson_dot_{partial,final}   fixed-order dot products; the host reads each one
//            poisson_iso_{partial,final}   mean of chi at the samples
//   extract  marching tetrahedra, count -> scan -> emit: per-node crossing counts and per-cell triangle counts,
//            poisson_scan_* (tile sums, one-CTA scan of the tiles, per-tile block scan), one device -> host read of
//            both totals, then poisson_vertex_kernel / poisson_face_kernel write at their offsets;
//            poisson_vertex_density_kernel interpolates the density grid at every vertex.
//   trim     pcl_quantile: two exact order statistics (pointcloud.cu's radix select) and numpy's lerp;
//            mesh_compact_*: remove masked vertices and the faces that use them, renumbering in order.
#include "../../include/spann3r_b200.h"
#include "kernels.cuh"

#include <math.h>
#include <string.h>

#include "poisson_math.cuh"
#include "scan.cuh"

namespace s3r {

using namespace poisson;

namespace {

constexpr int kThreads = 256;
constexpr int kBoxBlocks = 264;
constexpr int kDotBlocks = 528;        // fixed, so every sum has the same order on any GPU
constexpr int kScanPer = 4, kScanTile = kThreads * kScanPer;
constexpr int kPreSweeps = 2;          // l1-Jacobi sweeps before and after each coarse-grid correction
constexpr int kCoarsestSweeps = 8;     // on the coarsest level (depth 1: 3^3 nodes); even, the result lands in e1

struct Meta {
  double lo[3], hi[3], origin[3];
  double L, h, a, beta, coef;
  unsigned long long occupied;
  double dot;                          // the last fixed-order dot product
  double iso;
  long long sizes[2];                  // vertex and face counts of the extraction
};

inline size_t align256(size_t x) { return (x + 255) / 256 * 256; }

long long nodes_of(int depth) { return (long long)((1 << depth) + 1) * ((1 << depth) + 1) * ((1 << depth) + 1); }
long long cells_of(int depth) { return (long long)(1 << depth) * (1 << depth) * (1 << depth); }
int density_depth(int depth) { return depth - 2 > 1 ? depth - 2 : 1; }

struct Layout {
  Meta* meta;
  uint64_t* keys[2];
  int* vals[2];
  unsigned* hist;
  double *spts, *snrm;                 // [n, 3] in sorted order
  int *cell_lo, *cell_hi;              // [R^3]
  double* blocks;                      // [n, 64]: a cell's block at its first sorted sample
  double *b, *x, *r, *p, *q, *z, *t;   // [(R + 1)^3]
  double* lvl[kMaxDepth][3];           // levels 1 .. depth - 1: right-hand side, two iterates
  double* dens;                        // [(Rd + 1)^3]
  double* part;                        // [kDotBlocks * 6]
  long long* tiles;                    // scan tile sums
  size_t bytes;
  size_t offset[8];
};

long long tiles_of(long long n) { return (n + kScanTile - 1) / kScanTile; }

Layout carve(void* base, long long n, int depth) {
  Layout w;
  const long long NN = nodes_of(depth), NC = cells_of(depth), NNd = nodes_of(density_depth(depth));
  const uintptr_t p0 = (uintptr_t)base;
  size_t o = 0;
  auto take = [&](size_t bytes) {
    const uintptr_t at = p0 + o;
    o += align256(bytes);
    return at;
  };
  w.meta = (Meta*)take(sizeof(Meta));
  for (int i = 0; i < 2; ++i) {
    w.keys[i] = (uint64_t*)take(sizeof(uint64_t) * n);
    w.vals[i] = (int*)take(sizeof(int) * n);
  }
  w.hist = (unsigned*)take(sizeof(unsigned) * pcl_sort_hist_words(n));
  w.spts = (double*)take(sizeof(double) * 3 * n);
  w.snrm = (double*)take(sizeof(double) * 3 * n);
  w.cell_lo = (int*)take(sizeof(int) * NC);
  w.cell_hi = (int*)take(sizeof(int) * NC);
  w.blocks = (double*)take(sizeof(double) * 64 * n);
  double** fine[7] = {&w.b, &w.x, &w.r, &w.p, &w.q, &w.z, &w.t};
  for (double** f : fine) *f = (double*)take(sizeof(double) * NN);
  for (int l = 1; l < depth; ++l)
    for (int k = 0; k < 3; ++k) w.lvl[l][k] = (double*)take(sizeof(double) * nodes_of(l));
  w.dens = (double*)take(sizeof(double) * NNd);
  w.part = (double*)take(sizeof(double) * kDotBlocks * 6);
  w.tiles = (long long*)take(sizeof(long long) * (tiles_of(NN > NC ? NN : NC) + 2));
  w.bytes = o;
  const uintptr_t named[8] = {(uintptr_t)w.vals[0], (uintptr_t)w.b, (uintptr_t)w.x, (uintptr_t)w.blocks,
                              (uintptr_t)w.cell_lo, (uintptr_t)w.cell_hi, (uintptr_t)w.dens, (uintptr_t)w.meta};
  for (int i = 0; i < 8; ++i) w.offset[i] = named[i] - p0;
  return w;
}

// the sorted sample order: the radix sort passes that cover a key of 3 depth bits leave it in buffer (passes & 1)
int sort_passes(int depth) { return (3 * depth + 7) / 8; }

__device__ __forceinline__ void load3(const void* p, int f64, long long i, double* x) {
  if (f64) {
    const double* q = (const double*)p + 3 * i;
    x[0] = q[0]; x[1] = q[1]; x[2] = q[2];
  } else {
    const float* q = (const float*)p + 3 * i;
    x[0] = q[0]; x[1] = q[1]; x[2] = q[2];
  }
}

__device__ __forceinline__ void locate(const double* p, const Meta* m, double h, int R, int* c, double* f) {
  for (int d = 0; d < 3; ++d) {
    const double g = grid_coord(p[d], m->origin[d], h);
    c[d] = cell_of(g, R);
    f[d] = sub_rn(g, (double)c[d]);
  }
}

__device__ __forceinline__ void node_xyz(long long i, int n1, int* v) {
  v[0] = (int)(i % n1);
  v[1] = (int)(i / n1 % n1);
  v[2] = (int)(i / ((long long)n1 * n1));
}

__device__ __forceinline__ long long nidx(int x, int y, int z, int n1) { return ((long long)z * n1 + y) * n1 + x; }

// ---------------------------------------------------------------------------------------------------------------------
// setup
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) poisson_box_partial(const void* __restrict__ pts, int f64, long long n,
                                                                double* __restrict__ part) {
  __shared__ double s[6][kThreads];
  double m[6] = {INFINITY, INFINITY, INFINITY, -INFINITY, -INFINITY, -INFINITY};
  for (long long i = blockIdx.x * (long long)kThreads + threadIdx.x; i < n; i += (long long)kThreads * kBoxBlocks) {
    double x[3];
    load3(pts, f64, i, x);
    for (int a = 0; a < 3; ++a) {
      m[a] = fmin(m[a], x[a]);
      m[3 + a] = fmax(m[3 + a], x[a]);
    }
  }
  for (int a = 0; a < 6; ++a) s[a][threadIdx.x] = m[a];
  __syncthreads();
  for (int o = kThreads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o)
      for (int a = 0; a < 6; ++a)
        s[a][threadIdx.x] = a < 3 ? fmin(s[a][threadIdx.x], s[a][threadIdx.x + o]) : fmax(s[a][threadIdx.x], s[a][threadIdx.x + o]);
    __syncthreads();
  }
  if (threadIdx.x < 6) part[blockIdx.x * 6 + threadIdx.x] = s[threadIdx.x][0];
}

__global__ void __launch_bounds__(32) poisson_box_final(const double* __restrict__ part, double scale, int depth,
                                                        Meta* __restrict__ m) {
  if (threadIdx.x != 0) return;
  for (int a = 0; a < 3; ++a) {
    double lo = INFINITY, hi = -INFINITY;
    for (int b = 0; b < kBoxBlocks; ++b) {
      lo = fmin(lo, part[b * 6 + a]);
      hi = fmax(hi, part[b * 6 + 3 + a]);
    }
    m->lo[a] = lo;
    m->hi[a] = hi;
  }
  grid_geometry(m->lo, m->hi, scale, depth, m->origin, &m->L, &m->h);
  m->occupied = 0;
}

__global__ void __launch_bounds__(kThreads) poisson_keys_kernel(const void* __restrict__ pts, int f64, long long n,
                                                                const Meta* __restrict__ m, int R,
                                                                uint64_t* __restrict__ keys, int* __restrict__ vals) {
  const long long i = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (i >= n) return;
  double x[3], f[3];
  int c[3];
  load3(pts, f64, i, x);
  locate(x, m, m->h, R, c, f);
  keys[i] = ((uint64_t)c[2] * R + c[1]) * R + c[0];
  vals[i] = (int)i;
}

__global__ void __launch_bounds__(kThreads) poisson_gather_kernel(const void* __restrict__ pts,
                                                                  const void* __restrict__ nrm, int f64, long long n,
                                                                  const int* __restrict__ order,
                                                                  double* __restrict__ spts, double* __restrict__ snrm) {
  const long long i = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (i >= n) return;
  const int o = order[i];
  double x[3], v[3], u[3];
  load3(pts, f64, o, x);
  load3(nrm, f64, o, v);
  unit_normal(v, u);
  for (int a = 0; a < 3; ++a) {
    spts[3 * i + a] = x[a];
    snrm[3 * i + a] = u[a];
  }
}

__global__ void __launch_bounds__(kThreads) poisson_ranges_kernel(const uint64_t* __restrict__ keys, long long n,
                                                                  int* __restrict__ lo, int* __restrict__ hi,
                                                                  Meta* __restrict__ m) {
  const long long i = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (i >= n) return;
  const uint64_t k = keys[i];
  if (i == 0 || keys[i - 1] != k) {
    lo[k] = (int)i;
    atomicAdd(&m->occupied, 1ULL);   // an integer count: the total does not depend on the order
  }
  if (i == n - 1 || keys[i + 1] != k) hi[k] = (int)(i + 1);
}

__global__ void __launch_bounds__(32) poisson_weights_kernel(long long n, Meta* __restrict__ m) {
  if (threadIdx.x != 0) return;
  const double h = m->h;
  m->a = div_rn(mul_rn((double)m->occupied, mul_rn(h, h)), (double)n);
  m->beta = mul_rn(kAlpha, m->a);
  m->coef = div_rn(m->a, mul_rn(mul_rn(h, h), h));
}

__global__ void __launch_bounds__(kThreads) poisson_blocks_kernel(const uint64_t* __restrict__ keys, long long n,
                                                                  const int* __restrict__ lo, const int* __restrict__ hi,
                                                                  const double* __restrict__ spts,
                                                                  const Meta* __restrict__ m, int R,
                                                                  double* __restrict__ blocks) {
  const long long g = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (g >= 8 * n) return;
  const long long i = g >> 3;
  const int row = (int)(g & 7);
  const uint64_t k = keys[i];
  if (lo[k] != i) return;
  double acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int j = lo[k]; j < hi[k]; ++j) {
    int c[3];
    double f[3];
    locate(spts + 3LL * j, m, m->h, R, c, f);
    const double wp = corner_weight(f, row);
    for (int q = 0; q < 8; ++q) acc[q] += wp * corner_weight(f, q);
  }
  for (int q = 0; q < 8; ++q) blocks[64 * i + 8 * row + q] = acc[q];
}

// v at every node: the samples of its <= 8 cells, cells in (z, y, x) order, samples in sorted order
__global__ void __launch_bounds__(kThreads) poisson_splat_kernel(const int* __restrict__ lo, const int* __restrict__ hi,
                                                                 const double* __restrict__ spts,
                                                                 const double* __restrict__ snrm,
                                                                 const Meta* __restrict__ m, int R,
                                                                 double* __restrict__ v0, double* __restrict__ v1,
                                                                 double* __restrict__ v2) {
  const int n1 = R + 1;
  const long long i = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (i >= (long long)n1 * n1 * n1) return;
  int v[3];
  node_xyz(i, n1, v);
  double acc[3] = {0, 0, 0};
  for (int cz = v[2] - 1; cz <= v[2]; ++cz)
    for (int cy = v[1] - 1; cy <= v[1]; ++cy)
      for (int cx = v[0] - 1; cx <= v[0]; ++cx) {
        if (cx < 0 || cy < 0 || cz < 0 || cx >= R || cy >= R || cz >= R) continue;
        const long long cell = ((long long)cz * R + cy) * R + cx;
        const int p = (v[0] - cx) | (v[1] - cy) << 1 | (v[2] - cz) << 2;
        for (int j = lo[cell]; j < hi[cell]; ++j) {
          int c[3];
          double f[3];
          locate(spts + 3LL * j, m, m->h, R, c, f);
          const double w = corner_weight(f, p);
          for (int a = 0; a < 3; ++a) acc[a] += w * snrm[3LL * j + a];
        }
      }
  v0[i] = m->coef * acc[0];
  v1[i] = m->coef * acc[1];
  v2[i] = m->coef * acc[2];
}

__global__ void __launch_bounds__(kThreads) poisson_rhs_kernel(const double* __restrict__ v0,
                                                               const double* __restrict__ v1,
                                                               const double* __restrict__ v2,
                                                               const Meta* __restrict__ m, int R,
                                                               double* __restrict__ b) {
  const int n1 = R + 1;
  const long long i = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (i >= (long long)n1 * n1 * n1) return;
  int v[3];
  node_xyz(i, n1, v);
  const double* vd[3] = {v0, v1, v2};
  double acc = 0;
  for (int cz = v[2] - 1; cz <= v[2]; ++cz)
    for (int cy = v[1] - 1; cy <= v[1]; ++cy)
      for (int cx = v[0] - 1; cx <= v[0]; ++cx) {
        if (cx < 0 || cy < 0 || cz < 0 || cx >= R || cy >= R || cz >= R) continue;
        const int p = (v[0] - cx) | (v[1] - cy) << 1 | (v[2] - cz) << 2;
        for (int q = 0; q < 8; ++q) {
          const long long j = nidx(cx + (q & 1), cy + (q >> 1 & 1), cz + (q >> 2), n1);
          for (int d = 0; d < 3; ++d) {
            const int other = (p ^ q) & ~(1 << d);
            const double c = divergence(popcount3(other));
            acc += ((p >> d) & 1 ? c : -c) * vd[d][j];
          }
        }
      }
  b[i] = mul_rn(m->h, m->h) * acc;
}

// sample counts at the nodes of the depth-dd grid: its cells gather the samples of the finer cells they contain
__global__ void __launch_bounds__(kThreads) poisson_density_kernel(const int* __restrict__ lo, const int* __restrict__ hi,
                                                                   const double* __restrict__ spts,
                                                                   const Meta* __restrict__ m, int R, int dd,
                                                                   double* __restrict__ dens) {
  const int Rd = 1 << dd, n1 = Rd + 1, ratio = R / Rd;
  const long long i = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (i >= (long long)n1 * n1 * n1) return;
  const double hd = div_rn(m->L, (double)Rd);
  int v[3];
  node_xyz(i, n1, v);
  double acc = 0;
  for (int cz = v[2] - 1; cz <= v[2]; ++cz)
    for (int cy = v[1] - 1; cy <= v[1]; ++cy)
      for (int cx = v[0] - 1; cx <= v[0]; ++cx) {
        if (cx < 0 || cy < 0 || cz < 0 || cx >= Rd || cy >= Rd || cz >= Rd) continue;
        const int p = (v[0] - cx) | (v[1] - cy) << 1 | (v[2] - cz) << 2;
        const int C[3] = {cx, cy, cz};
        for (int fz = cz * ratio; fz < (cz + 1) * ratio; ++fz)
          for (int fy = cy * ratio; fy < (cy + 1) * ratio; ++fy)
            for (int fx = cx * ratio; fx < (cx + 1) * ratio; ++fx) {
              const long long cell = ((long long)fz * R + fy) * R + fx;
              for (int j = lo[cell]; j < hi[cell]; ++j) {
                double f[3];
                for (int d = 0; d < 3; ++d) f[d] = sub_rn(grid_coord(spts[3LL * j + d], m->origin[d], hd), (double)C[d]);
                acc += corner_weight(f, p);
              }
            }
      }
  dens[i] = div_rn(acc, mul_rn(mul_rn(hd, hd), hd));
}

// ---------------------------------------------------------------------------------------------------------------------
// solve
// ---------------------------------------------------------------------------------------------------------------------
enum { kApply = 0, kSweep = 1, kResidual = 2 };

// kApply: out = A x.  kSweep: out = x + (r - A x) / D, D the l1 row sum of A (x == nullptr: out = r / D).
// kResidual: out = r - A x.  A = h K (+ beta S on the finest level, kFine).
template <bool kFine, int kMode>
__global__ void __launch_bounds__(kThreads) poisson_apply_kernel(const double* __restrict__ x,
                                                                 const double* __restrict__ r, double* __restrict__ out,
                                                                 int R, double h, double beta,
                                                                 const int* __restrict__ lo, const int* __restrict__ hi,
                                                                 const double* __restrict__ blocks) {
  const int n1 = R + 1;
  const long long i = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (i >= (long long)n1 * n1 * n1) return;
  int v[3];
  node_xyz(i, n1, v);
  double kx = 0, sx = 0, sl1 = 0;
  int cells = 0;
  for (int cz = v[2] - 1; cz <= v[2]; ++cz)
    for (int cy = v[1] - 1; cy <= v[1]; ++cy)
      for (int cx = v[0] - 1; cx <= v[0]; ++cx) {
        if (cx < 0 || cy < 0 || cz < 0 || cx >= R || cy >= R || cz >= R) continue;
        ++cells;
        const int p = (v[0] - cx) | (v[1] - cy) << 1 | (v[2] - cz) << 2;
        const double* blk = nullptr;
        if (kFine) {
          const long long cell = ((long long)cz * R + cy) * R + cx;
          const int s = lo[cell];
          if (hi[cell] > s) blk = blocks + 64LL * s + 8 * p;
        }
        if (blk && kMode == kSweep)
          for (int q = 0; q < 8; ++q) sl1 += blk[q];
        if (x)
          for (int q = 0; q < 8; ++q) {
            const double xq = x[nidx(cx + (q & 1), cy + (q >> 1 & 1), cz + (q >> 2), n1)];
            kx += stiffness(popcount3(p ^ q)) * xq;
            if (blk) sx += blk[q] * xq;
          }
      }
  const double ax = h * kx + beta * sx;
  if (kMode == kApply) {
    out[i] = ax;
  } else if (kMode == kResidual) {
    out[i] = r[i] - ax;
  } else {
    const double D = h * (kStiffnessL1 * cells) + beta * sl1;
    out[i] = (x ? x[i] : 0.0) + (r[i] - ax) / D;
  }
}

// coarse node I gathers the fine residual at the 27 fine nodes around 2 I, weights prod_d (1 or 1/2)
__global__ void __launch_bounds__(kThreads) poisson_restrict_kernel(const double* __restrict__ fine, int Rf,
                                                                    double* __restrict__ coarse) {
  const int nc = Rf / 2 + 1, nf = Rf + 1;
  const long long i = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (i >= (long long)nc * nc * nc) return;
  int v[3];
  node_xyz(i, nc, v);
  double acc = 0;
  for (int dz = -1; dz <= 1; ++dz)
    for (int dy = -1; dy <= 1; ++dy)
      for (int dx = -1; dx <= 1; ++dx) {
        const int x = 2 * v[0] + dx, y = 2 * v[1] + dy, z = 2 * v[2] + dz;
        if (x < 0 || y < 0 || z < 0 || x >= nf || y >= nf || z >= nf) continue;
        const double w = (dx ? 0.5 : 1.0) * (dy ? 0.5 : 1.0) * (dz ? 0.5 : 1.0);
        acc += w * fine[nidx(x, y, z, nf)];
      }
  coarse[i] = acc;
}

// fine node j += trilinear interpolation of the coarse correction
__global__ void __launch_bounds__(kThreads) poisson_prolong_kernel(const double* __restrict__ coarse, int Rf,
                                                                   double* __restrict__ fine) {
  const int nc = Rf / 2 + 1, nf = Rf + 1;
  const long long i = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (i >= (long long)nf * nf * nf) return;
  int v[3];
  node_xyz(i, nf, v);
  double acc = 0;
  for (int kz = 0; kz <= (v[2] & 1); ++kz)
    for (int ky = 0; ky <= (v[1] & 1); ++ky)
      for (int kx = 0; kx <= (v[0] & 1); ++kx) {
        const double w = ((v[0] & 1) ? 0.5 : 1.0) * ((v[1] & 1) ? 0.5 : 1.0) * ((v[2] & 1) ? 0.5 : 1.0);
        acc += w * coarse[nidx(v[0] / 2 + kx, v[1] / 2 + ky, v[2] / 2 + kz, nc)];
      }
  fine[i] += acc;
}

__device__ __forceinline__ void block_sum_to(double s, double* out) {
  __shared__ double sh[kThreads];
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int o = kThreads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = sh[0];
}

__global__ void __launch_bounds__(kThreads) poisson_dot_partial(const double* __restrict__ a,
                                                                const double* __restrict__ b, long long n,
                                                                double* __restrict__ part) {
  double s = 0;
  for (long long i = blockIdx.x * (long long)kThreads + threadIdx.x; i < n; i += (long long)kThreads * kDotBlocks)
    s += a[i] * b[i];
  block_sum_to(s, part + blockIdx.x);
}

__global__ void __launch_bounds__(kThreads) poisson_dot_final(const double* __restrict__ part, double* __restrict__ out) {
  double s = 0;
  for (int b = threadIdx.x; b < kDotBlocks; b += kThreads) s += part[b];
  block_sum_to(s, out);
}

__global__ void __launch_bounds__(kThreads) poisson_cg_update(double* __restrict__ x, double* __restrict__ r,
                                                              const double* __restrict__ p,
                                                              const double* __restrict__ q, double alpha, long long n) {
  const long long i = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (i >= n) return;
  x[i] += alpha * p[i];
  r[i] -= alpha * q[i];
}

__global__ void __launch_bounds__(kThreads) poisson_cg_direction(double* __restrict__ p, const double* __restrict__ z,
                                                                 double beta, long long n) {
  const long long i = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (i >= n) return;
  p[i] = z[i] + beta * p[i];
}

__global__ void __launch_bounds__(kThreads) poisson_iso_partial(const double* __restrict__ spts, long long n,
                                                                const double* __restrict__ x,
                                                                const Meta* __restrict__ m, int R,
                                                                double* __restrict__ part) {
  double s = 0;
  for (long long i = blockIdx.x * (long long)kThreads + threadIdx.x; i < n; i += (long long)kThreads * kDotBlocks) {
    int c[3];
    double f[3];
    locate(spts + 3 * i, m, m->h, R, c, f);
    double chi = 0;
    for (int q = 0; q < 8; ++q)
      chi += corner_weight(f, q) * x[nidx(c[0] + (q & 1), c[1] + (q >> 1 & 1), c[2] + (q >> 2), R + 1)];
    s += chi;
  }
  block_sum_to(s, part + blockIdx.x);
}

__global__ void __launch_bounds__(kThreads) poisson_iso_final(const double* __restrict__ part, long long n,
                                                              Meta* __restrict__ m) {
  __shared__ double total;
  double s = 0;
  for (int b = threadIdx.x; b < kDotBlocks; b += kThreads) s += part[b];
  block_sum_to(s, &total);
  __syncthreads();
  if (threadIdx.x == 0) m->iso = total / (double)n;
}

// ---------------------------------------------------------------------------------------------------------------------
// extraction
// ---------------------------------------------------------------------------------------------------------------------
// bit d - 1: the edge from node v to v + (d & 1, d >> 1 & 1, d >> 2) crosses the iso value
__device__ __forceinline__ int edge_mask(const double* __restrict__ x, const int* v, int n1, double iso) {
  const bool o = x[nidx(v[0], v[1], v[2], n1)] > iso;
  int mask = 0;
  for (int d = 1; d < 8; ++d) {
    const int a = v[0] + (d & 1), b = v[1] + (d >> 1 & 1), c = v[2] + (d >> 2);
    if (a >= n1 || b >= n1 || c >= n1) continue;
    if ((x[nidx(a, b, c, n1)] > iso) != o) mask |= 1 << (d - 1);
  }
  return mask;
}

__device__ __forceinline__ int cell_code(const double* __restrict__ x, int cx, int cy, int cz, int n1, double iso) {
  int code = 0;
  for (int q = 0; q < 8; ++q) code |= (x[nidx(cx + (q & 1), cy + (q >> 1 & 1), cz + (q >> 2), n1)] > iso) << q;
  return code;
}

__device__ __forceinline__ int tet_code(int corners, int t) {
  int code = 0;
  for (int k = 0; k < 4; ++k) code |= ((corners >> tet_corner(t, k)) & 1) << k;
  return code;
}

__global__ void __launch_bounds__(kThreads) poisson_node_count_kernel(const double* __restrict__ x,
                                                                      const Meta* __restrict__ m, int R,
                                                                      int* __restrict__ cnt) {
  const int n1 = R + 1;
  const long long i = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (i >= (long long)n1 * n1 * n1) return;
  int v[3];
  node_xyz(i, n1, v);
  cnt[i] = __popc(edge_mask(x, v, n1, m->iso));
}

__global__ void __launch_bounds__(kThreads) poisson_cell_count_kernel(const double* __restrict__ x,
                                                                      const Meta* __restrict__ m, int R,
                                                                      int* __restrict__ cnt) {
  const long long i = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (i >= (long long)R * R * R) return;
  int v[3];
  node_xyz(i, R, v);
  const int code = cell_code(x, v[0], v[1], v[2], R + 1, m->iso);
  int n = 0;
  if (code != 0 && code != 255)
    for (int t = 0; t < 6; ++t) {
      int e[6];
      n += case_triangles(tet_code(code, t), e);
    }
  cnt[i] = n;
}

// tile sums of int counts, kScanPer per thread
__global__ void __launch_bounds__(kThreads) poisson_scan_tiles(const int* __restrict__ cnt, long long n,
                                                               long long* __restrict__ tiles) {
  const long long i0 = blockIdx.x * (long long)kScanTile + threadIdx.x * (long long)kScanPer;
  long long s = 0;
  for (int j = 0; j < kScanPer; ++j)
    if (i0 + j < n) s += cnt[i0 + j];
  long long total;
  block_exclusive_scan<kThreads>(s, &total);
  if (threadIdx.x == 0) tiles[blockIdx.x] = total;
}

// exclusive scan of the tile sums in place (one CTA); tiles[n_tiles] <- the total
__global__ void __launch_bounds__(1024) poisson_scan_top(long long* __restrict__ tiles, long long n_tiles) {
  long long carry = 0;
  for (long long base = 0; base < n_tiles; base += 1024) {
    const long long i = base + threadIdx.x;
    const long long v = i < n_tiles ? tiles[i] : 0;
    long long total;
    const long long ex = block_exclusive_scan<1024>(v, &total);
    if (i < n_tiles) tiles[i] = carry + ex;
    carry += total;
  }
  if (threadIdx.x == 0) tiles[n_tiles] = carry;
}

__global__ void __launch_bounds__(kThreads) poisson_scan_write(const int* __restrict__ cnt, long long n,
                                                               const long long* __restrict__ tiles,
                                                               long long* __restrict__ off) {
  const long long i0 = blockIdx.x * (long long)kScanTile + threadIdx.x * (long long)kScanPer;
  long long s = 0;
  for (int j = 0; j < kScanPer; ++j)
    if (i0 + j < n) s += cnt[i0 + j];
  long long total;
  long long o = tiles[blockIdx.x] + block_exclusive_scan<kThreads>(s, &total);
  for (int j = 0; j < kScanPer; ++j)
    if (i0 + j < n) {
      off[i0 + j] = o;
      o += cnt[i0 + j];
    }
}

// exclusive offsets of n int counts into off, the total into tiles[tiles_of(n)]
void scan_counts(const int* cnt, long long n, long long* tiles, long long* off, cudaStream_t st) {
  const long long nt = tiles_of(n);
  poisson_scan_tiles<<<(unsigned)nt, kThreads, 0, st>>>(cnt, n, tiles);
  poisson_scan_top<<<1, 1024, 0, st>>>(tiles, nt);
  poisson_scan_write<<<(unsigned)nt, kThreads, 0, st>>>(cnt, n, tiles, off);
}

__global__ void __launch_bounds__(kThreads) poisson_vertex_kernel(const double* __restrict__ x,
                                                                  const Meta* __restrict__ m, int R,
                                                                  const long long* __restrict__ node_off,
                                                                  float* __restrict__ verts) {
  const int n1 = R + 1;
  const long long i = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (i >= (long long)n1 * n1 * n1) return;
  int v[3];
  node_xyz(i, n1, v);
  const double iso = m->iso;
  const int mask = edge_mask(x, v, n1, iso);
  if (!mask) return;
  long long o = node_off[i];
  const double va = x[i];
  for (int d = 1; d < 8; ++d) {
    if (!(mask >> (d - 1) & 1)) continue;
    const int w[3] = {v[0] + (d & 1), v[1] + (d >> 1 & 1), v[2] + (d >> 2)};
    const double vb = x[nidx(w[0], w[1], w[2], n1)];
    for (int a = 0; a < 3; ++a)
      verts[3 * o + a] = edge_point(node_coord(m->origin[a], m->h, v[a]), node_coord(m->origin[a], m->h, w[a]), va, vb,
                                    iso);
    ++o;
  }
}

__global__ void __launch_bounds__(kThreads) poisson_face_kernel(const double* __restrict__ x,
                                                                const Meta* __restrict__ m, int R,
                                                                const long long* __restrict__ node_off,
                                                                const long long* __restrict__ cell_off,
                                                                long long* __restrict__ faces) {
  const int n1 = R + 1;
  const long long i = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (i >= (long long)R * R * R) return;
  int v[3];
  node_xyz(i, R, v);
  const double iso = m->iso;
  const int code = cell_code(x, v[0], v[1], v[2], n1, iso);
  if (code == 0 || code == 255) return;
  // edge masks of the corners that own tetrahedron edges (all but corner 7)
  int masks[7];
  for (int u = 0; u < 7; ++u) {
    const int c[3] = {v[0] + (u & 1), v[1] + (u >> 1 & 1), v[2] + (u >> 2)};
    masks[u] = edge_mask(x, c, n1, iso);
  }
  long long o = cell_off[i];
  for (int t = 0; t < 6; ++t) {
    int e[6];
    const int nt = case_triangles(tet_code(code, t), e);
    for (int k = 0; k < nt; ++k) {
      int tri[3] = {e[3 * k], e[3 * k + 1], e[3 * k + 2]};
      if (!tet_positive(t)) {
        const int s = tri[1];
        tri[1] = tri[2];
        tri[2] = s;
      }
      for (int a = 0; a < 3; ++a) {
        const int u = tet_corner(t, tet_edge_vertex(tri[a], 0)), w = tet_corner(t, tet_edge_vertex(tri[a], 1));
        const int d = w ^ u;
        const long long owner = nidx(v[0] + (u & 1), v[1] + (u >> 1 & 1), v[2] + (u >> 2), n1);
        faces[3 * o + a] = node_off[owner] + __popc(masks[u] & ((1 << (d - 1)) - 1));
      }
      ++o;
    }
  }
}

__global__ void __launch_bounds__(kThreads) poisson_vertex_density_kernel(const float* __restrict__ verts, long long nv,
                                                                          const double* __restrict__ dgrid,
                                                                          const Meta* __restrict__ m, int dd,
                                                                          double* __restrict__ out) {
  const long long i = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (i >= nv) return;
  const int Rd = 1 << dd;
  const double hd = div_rn(m->L, (double)Rd);
  const double p[3] = {verts[3 * i], verts[3 * i + 1], verts[3 * i + 2]};
  int c[3];
  double f[3];
  locate(p, m, hd, Rd, c, f);
  double s = 0;
  for (int q = 0; q < 8; ++q)
    s = add_rn(s, mul_rn(corner_weight(f, q), dgrid[nidx(c[0] + (q & 1), c[1] + (q >> 1 & 1), c[2] + (q >> 2), Rd + 1)]));
  out[i] = s;
}

__global__ void __launch_bounds__(32) poisson_quantile_kernel(const double* __restrict__ picked, double gamma,
                                                              double* __restrict__ out) {
  if (threadIdx.x == 0) *out = quantile_lerp(picked[0], picked[1], gamma);
}

// ---------------------------------------------------------------------------------------------------------------------
// remove_vertices_by_mask
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) compact_vertex_flags(const uint8_t* __restrict__ mask, long long n,
                                                                 int* __restrict__ keep) {
  const long long i = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (i < n) keep[i] = mask[i] ? 0 : 1;
}

__global__ void __launch_bounds__(kThreads) compact_face_flags(const long long* __restrict__ faces, long long nf,
                                                               const int* __restrict__ vkeep, int* __restrict__ keep) {
  const long long i = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (i < nf) keep[i] = vkeep[faces[3 * i]] & vkeep[faces[3 * i + 1]] & vkeep[faces[3 * i + 2]];
}

__global__ void __launch_bounds__(kThreads) compact_vertices(const float* __restrict__ v, long long n,
                                                             const int* __restrict__ keep,
                                                             const long long* __restrict__ off, float* __restrict__ out) {
  const long long i = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (i >= n || !keep[i]) return;
  for (int a = 0; a < 3; ++a) out[3 * off[i] + a] = v[3 * i + a];
}

__global__ void __launch_bounds__(kThreads) compact_faces(const long long* __restrict__ f, long long nf,
                                                          const int* __restrict__ keep,
                                                          const long long* __restrict__ off,
                                                          const long long* __restrict__ voff,
                                                          long long* __restrict__ out) {
  const long long i = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (i >= nf || !keep[i]) return;
  for (int a = 0; a < 3; ++a) out[3 * off[i] + a] = voff[f[3 * i + a]];
}

struct CompactLayout {
  int *vkeep, *fkeep;
  long long *voff, *foff, *vtiles, *ftiles;
  size_t bytes;
};

CompactLayout carve_compact(void* base, long long nv, long long nf) {
  CompactLayout w;
  const uintptr_t p0 = (uintptr_t)base;
  size_t o = 0;
  auto take = [&](size_t bytes) {
    const uintptr_t at = p0 + o;
    o += align256(bytes);
    return at;
  };
  w.vkeep = (int*)take(sizeof(int) * nv);
  w.fkeep = (int*)take(sizeof(int) * nf);
  w.voff = (long long*)take(sizeof(long long) * nv);
  w.foff = (long long*)take(sizeof(long long) * nf);
  w.vtiles = (long long*)take(sizeof(long long) * (tiles_of(nv) + 1));
  w.ftiles = (long long*)take(sizeof(long long) * (tiles_of(nf) + 1));
  w.bytes = o;
  return w;
}

// ---------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------
bool args_ok(long long n, int depth) { return n >= 4 && n < (1LL << 31) && depth >= kMinDepth && depth <= kMaxDepth; }

unsigned grid_for(long long n) { return (unsigned)((n + kThreads - 1) / kThreads); }

int launched(const char* what) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: launch failed: %s", what, cudaGetErrorString(e));
    return -6;
  }
  return 0;
}

int check_ws(const char* what, long long n, int depth, const void* ws, size_t ws_bytes) {
  if (!args_ok(n, depth) || !ws || (uintptr_t)ws % 256 || ws_bytes < s3r_poisson_workspace_bytes(n, depth)) {
    set_error("%s: bad arguments (n=%lld depth=%d workspace_bytes=%zu; need 4 <= n < 2^31, 1 <= depth <= 10 and a "
              "256-byte aligned workspace of s3r_poisson_workspace_bytes(n, depth) bytes)", what, n, depth, ws_bytes);
    return -1;
  }
  return 0;
}

int read_meta(const Layout& w, Meta* host, cudaStream_t st, const char* what) {
  if (cudaMemcpyAsync(host, w.meta, sizeof(Meta), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
      cudaStreamSynchronize(st) != cudaSuccess)
    return launched(what);
  return 0;
}

struct Solver {
  Layout w;
  int depth;
  double L, h, beta;
  cudaStream_t st;

  double level_h(int l) const { return L / (double)(1 << l); }

  template <int kMode>
  void apply(int l, const double* x, const double* r, double* out) const {
    const int R = 1 << l;
    const unsigned g = grid_for(nodes_of(l));
    if (l == depth)
      poisson_apply_kernel<true, kMode><<<g, kThreads, 0, st>>>(x, r, out, R, h, beta, w.cell_lo, w.cell_hi, w.blocks);
    else
      poisson_apply_kernel<false, kMode><<<g, kThreads, 0, st>>>(x, r, out, R, level_h(l), 0.0, nullptr, nullptr,
                                                                  nullptr);
  }

  // One V-cycle from a zero guess at level l on right-hand side r; returns the buffer holding the correction.
  const double* vcycle(int l, const double* r) const {
    const bool fine = l == depth;
    double* e0 = fine ? w.z : w.lvl[l][1];
    double* e1 = fine ? w.t : w.lvl[l][2];
    double* res = fine ? w.q : w.lvl[l][1];
    const bool coarsest = l == 1;
    const int sweeps = coarsest ? kCoarsestSweeps : kPreSweeps;
    apply<kSweep>(l, nullptr, r, e0);
    for (int k = 1; k < sweeps; ++k) {
      if (k & 1) apply<kSweep>(l, e0, r, e1);
      else apply<kSweep>(l, e1, r, e0);
    }
    if (coarsest) return e1;
    apply<kResidual>(l, e1, r, res);
    poisson_restrict_kernel<<<grid_for(nodes_of(l - 1)), kThreads, 0, st>>>(res, 1 << l, w.lvl[l - 1][0]);
    const double* ec = vcycle(l - 1, w.lvl[l - 1][0]);
    poisson_prolong_kernel<<<grid_for(nodes_of(l)), kThreads, 0, st>>>(ec, 1 << l, e1);
    for (int k = 0; k < kPreSweeps; ++k) {
      if (k & 1) apply<kSweep>(l, e0, r, e1);
      else apply<kSweep>(l, e1, r, e0);
    }
    return e1;
  }

  double dot(const double* a, const double* b, long long n) const {
    poisson_dot_partial<<<kDotBlocks, kThreads, 0, st>>>(a, b, n, w.part);
    poisson_dot_final<<<1, kThreads, 0, st>>>(w.part, &w.meta->dot);
    double h_out = NAN;
    if (cudaMemcpyAsync(&h_out, &w.meta->dot, sizeof(double), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess)
      return NAN;
    return h_out;
  }
};

}  // namespace

// After the solve, r / p / q / z are free: node counts in q, node offsets in r, cell counts in z, cell offsets in p.
}  // namespace s3r

using namespace s3r;

extern "C" {

size_t s3r_poisson_workspace_bytes(int64_t n, int depth) {
  return args_ok(n, depth) ? carve(nullptr, n, depth).bytes : 0;
}

size_t s3r_poisson_offset(int64_t n, int depth, int which) {
  if (!args_ok(n, depth) || which < 0 || which > 7) return (size_t)-1;
  const Layout w = carve(nullptr, n, depth);
  // 0: sorted sample order: the sort's final value buffer
  if (which == 0) return (uintptr_t)w.vals[sort_passes(depth) & 1];
  return w.offset[which];
}

int s3r_poisson_setup(const void* pts, const void* nrm, int f64, int64_t n, int depth, double scale, void* ws,
                      size_t ws_bytes, double* info, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int e = check_ws("poisson_setup", n, depth, ws, ws_bytes)) return e;
  if (!pts || !nrm || !info || !(scale >= 1.0) || !isfinite(scale)) {
    set_error("poisson_setup: points, normals and info must be non-null and scale finite and >= 1 (got %g)", scale);
    return -1;
  }
  const Layout w = carve(ws, n, depth);
  const int R = 1 << depth, passes = sort_passes(depth), dd = density_depth(depth);
  const long long NN = nodes_of(depth), NC = cells_of(depth);
  poisson_box_partial<<<kBoxBlocks, kThreads, 0, st>>>(pts, f64, n, w.part);
  poisson_box_final<<<1, 32, 0, st>>>(w.part, scale, depth, w.meta);
  Meta m;
  if (int e = read_meta(w, &m, st, "poisson_setup (bounding box)")) return e;
  if (!(m.L > 0.0) || !isfinite(m.L) || !isfinite(m.h) || !(m.h > 0.0)) {
    set_error("poisson_setup: the bounding box has zero extent or is not finite (L=%g)", m.L);
    return -2;
  }
  poisson_keys_kernel<<<grid_for(n), kThreads, 0, st>>>(pts, f64, n, w.meta, R, w.keys[0], w.vals[0]);
  if (int e = launch_pcl_radix_sort(w.keys, w.vals, n, passes, w.hist, st)) return e;
  const uint64_t* keys = w.keys[passes & 1];
  const int* order = w.vals[passes & 1];
  poisson_gather_kernel<<<grid_for(n), kThreads, 0, st>>>(pts, nrm, f64, n, order, w.spts, w.snrm);
  cudaMemsetAsync(w.cell_lo, 0, sizeof(int) * NC, st);
  cudaMemsetAsync(w.cell_hi, 0, sizeof(int) * NC, st);
  poisson_ranges_kernel<<<grid_for(n), kThreads, 0, st>>>(keys, n, w.cell_lo, w.cell_hi, w.meta);
  poisson_weights_kernel<<<1, 32, 0, st>>>(n, w.meta);
  poisson_blocks_kernel<<<grid_for(8 * n), kThreads, 0, st>>>(keys, n, w.cell_lo, w.cell_hi, w.spts, w.meta, R, w.blocks);
  // v lives in the solver's q, z, t until b is built
  poisson_splat_kernel<<<grid_for(NN), kThreads, 0, st>>>(w.cell_lo, w.cell_hi, w.spts, w.snrm, w.meta, R, w.q, w.z, w.t);
  poisson_rhs_kernel<<<grid_for(NN), kThreads, 0, st>>>(w.q, w.z, w.t, w.meta, R, w.b);
  poisson_density_kernel<<<grid_for(nodes_of(dd)), kThreads, 0, st>>>(w.cell_lo, w.cell_hi, w.spts, w.meta, R, dd, w.dens);
  if (int e = read_meta(w, &m, st, "poisson_setup")) return e;
  info[0] = m.origin[0]; info[1] = m.origin[1]; info[2] = m.origin[2];
  info[3] = m.L; info[4] = m.h; info[5] = m.a; info[6] = m.beta; info[7] = (double)m.occupied;
  return 0;
}

int s3r_poisson_solve(int64_t n, int depth, double tol, int max_iter, void* ws, size_t ws_bytes, double* info,
                      void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int e = check_ws("poisson_solve", n, depth, ws, ws_bytes)) return e;
  if (!info || !(tol > 0.0) || max_iter < 1) {
    set_error("poisson_solve: info must be non-null, tol > 0 and max_iter >= 1 (got tol=%g max_iter=%d)", tol, max_iter);
    return -1;
  }
  Solver s;
  s.w = carve(ws, n, depth);
  s.depth = depth;
  s.st = st;
  Meta m;
  if (int e = read_meta(s.w, &m, st, "poisson_solve")) return e;
  s.L = m.L;
  s.h = m.h;
  s.beta = m.beta;
  const long long NN = nodes_of(depth);
  const unsigned g = grid_for(NN);
  const Layout& w = s.w;
  cudaMemsetAsync(w.x, 0, sizeof(double) * NN, st);
  cudaMemcpyAsync(w.r, w.b, sizeof(double) * NN, cudaMemcpyDeviceToDevice, st);
  const double bb = s.dot(w.b, w.b, NN);
  if (!isfinite(bb)) return launched("poisson_solve (|b|)");
  int it = 0;
  double rel = 0.0;
  if (bb > 0.0) {
    const double* zp = s.vcycle(depth, w.r);
    double rz = s.dot(w.r, zp, NN);
    cudaMemcpyAsync(w.p, zp, sizeof(double) * NN, cudaMemcpyDeviceToDevice, st);
    rel = 1.0;
    while (true) {
      if (it == max_iter) {
        set_error("poisson_solve: no convergence to a relative residual of %g within %d iterations (reached %g)", tol,
                  max_iter, rel);
        info[0] = it; info[1] = rel; info[2] = NAN;
        return -7;
      }
      ++it;
      s.apply<kApply>(depth, w.p, nullptr, w.q);
      const double pq = s.dot(w.p, w.q, NN);
      const double alpha = rz / pq;
      poisson_cg_update<<<g, kThreads, 0, st>>>(w.x, w.r, w.p, w.q, alpha, NN);
      rel = sqrt(s.dot(w.r, w.r, NN) / bb);
      if (!isfinite(rel)) return launched("poisson_solve (residual)");
      if (rel <= tol) {
        // confirm on the true residual b - A x before stopping
        s.apply<kResidual>(depth, w.x, w.b, w.r);
        rel = sqrt(s.dot(w.r, w.r, NN) / bb);
        if (rel <= tol) break;
      }
      zp = s.vcycle(depth, w.r);
      const double rz_new = s.dot(w.r, zp, NN);
      poisson_cg_direction<<<g, kThreads, 0, st>>>(w.p, zp, rz_new / rz, NN);
      rz = rz_new;
    }
  }
  poisson_iso_partial<<<kDotBlocks, kThreads, 0, st>>>(w.spts, n, w.x, w.meta, 1 << depth, w.part);
  poisson_iso_final<<<1, kThreads, 0, st>>>(w.part, n, w.meta);
  if (int e = read_meta(w, &m, st, "poisson_solve (iso value)")) return e;
  info[0] = it;
  info[1] = rel;
  info[2] = m.iso;
  return 0;
}

int s3r_poisson_extract_count(int64_t n, int depth, void* ws, size_t ws_bytes, int64_t* sizes, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int e = check_ws("poisson_extract_count", n, depth, ws, ws_bytes)) return e;
  if (!sizes) {
    set_error("poisson_extract_count: sizes must be non-null");
    return -1;
  }
  const Layout w = carve(ws, n, depth);
  const int R = 1 << depth;
  const long long NN = nodes_of(depth), NC = cells_of(depth);
  int* ncnt = (int*)w.q;
  int* ccnt = (int*)w.z;
  poisson_node_count_kernel<<<grid_for(NN), kThreads, 0, st>>>(w.x, w.meta, R, ncnt);
  scan_counts(ncnt, NN, w.tiles, (long long*)w.r, st);
  cudaMemcpyAsync(&w.meta->sizes[0], w.tiles + tiles_of(NN), sizeof(long long), cudaMemcpyDeviceToDevice, st);
  poisson_cell_count_kernel<<<grid_for(NC), kThreads, 0, st>>>(w.x, w.meta, R, ccnt);
  scan_counts(ccnt, NC, w.tiles, (long long*)w.p, st);
  cudaMemcpyAsync(&w.meta->sizes[1], w.tiles + tiles_of(NC), sizeof(long long), cudaMemcpyDeviceToDevice, st);
  if (cudaMemcpyAsync(sizes, w.meta->sizes, 2 * sizeof(long long), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
      cudaStreamSynchronize(st) != cudaSuccess)
    return launched("poisson_extract_count (sizes read)");
  return launched("poisson_extract_count");
}

int s3r_poisson_extract(int64_t n, int depth, void* ws, size_t ws_bytes, float* verts, int64_t* faces_, double* dens,
                        void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  long long* faces = reinterpret_cast<long long*>(faces_);
  if (int e = check_ws("poisson_extract", n, depth, ws, ws_bytes)) return e;
  Meta m;
  const Layout w = carve(ws, n, depth);
  if (int e = read_meta(w, &m, st, "poisson_extract")) return e;
  const long long nv = m.sizes[0], nf = m.sizes[1];
  if ((nv && (!verts || !dens)) || (nf && !faces)) {
    set_error("poisson_extract: vertices, densities (%lld) and faces (%lld) must be non-null", nv, nf);
    return -1;
  }
  const int R = 1 << depth;
  if (nv) {
    poisson_vertex_kernel<<<grid_for(nodes_of(depth)), kThreads, 0, st>>>(w.x, w.meta, R, (const long long*)w.r, verts);
    poisson_vertex_density_kernel<<<grid_for(nv), kThreads, 0, st>>>(verts, nv, w.dens, w.meta, density_depth(depth),
                                                                      dens);
  }
  if (nf)
    poisson_face_kernel<<<grid_for(cells_of(depth)), kThreads, 0, st>>>(w.x, w.meta, R, (const long long*)w.r,
                                                                        (const long long*)w.p, faces);
  return launched("poisson_extract");
}

int s3r_pcl_quantile(const double* x, int64_t n, double q, void* workspace, double* out, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!x || !workspace || !out || n < 1 || n >= (1LL << 31) || !(q >= 0.0 && q <= 1.0)) {
    set_error("pcl_quantile: bad arguments (n=%lld q=%g; need 1 <= n < 2^31, 0 <= q <= 1, non-null pointers)", n, q);
    return -1;
  }
  long long lo, hi;
  double gamma;
  quantile_ranks(n, q, &lo, &hi, &gamma);
  const double* picked = nullptr;
  if (int e = launch_pcl_select_ranks(x, n, lo, hi, workspace, &picked, st)) return e;
  poisson_quantile_kernel<<<1, 32, 0, st>>>(picked, gamma, out);
  return launched("pcl_quantile");
}

size_t s3r_mesh_compact_workspace_bytes(int64_t nv, int64_t nf) {
  return nv >= 1 && nv < (1LL << 31) && nf >= 0 && nf < (1LL << 31) ? carve_compact(nullptr, nv, nf).bytes : 0;
}

int s3r_mesh_compact_count(const uint8_t* mask, const int64_t* faces_, int64_t nv, int64_t nf, void* ws,
                           size_t ws_bytes, int64_t* sizes, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long* faces = reinterpret_cast<const long long*>(faces_);
  if (!mask || !ws || !sizes || (nf && !faces) || (uintptr_t)ws % 256 || s3r_mesh_compact_workspace_bytes(nv, nf) == 0 ||
      ws_bytes < s3r_mesh_compact_workspace_bytes(nv, nf)) {
    set_error("mesh_compact_count: bad arguments (n_verts=%lld n_faces=%lld workspace_bytes=%zu; need 1 <= n_verts, "
              "n_faces < 2^31, a 256-byte aligned workspace of s3r_mesh_compact_workspace_bytes and non-null pointers)",
              nv, nf, ws_bytes);
    return -1;
  }
  const CompactLayout w = carve_compact(ws, nv, nf);
  compact_vertex_flags<<<grid_for(nv), kThreads, 0, st>>>(mask, nv, w.vkeep);
  scan_counts(w.vkeep, nv, w.vtiles, w.voff, st);
  long long h[2] = {0, 0};
  if (nf) {
    compact_face_flags<<<grid_for(nf), kThreads, 0, st>>>(faces, nf, w.vkeep, w.fkeep);
    scan_counts(w.fkeep, nf, w.ftiles, w.foff, st);
    cudaMemcpyAsync(&h[1], w.ftiles + tiles_of(nf), sizeof(long long), cudaMemcpyDeviceToHost, st);
  }
  if (cudaMemcpyAsync(&h[0], w.vtiles + tiles_of(nv), sizeof(long long), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
      cudaStreamSynchronize(st) != cudaSuccess)
    return launched("mesh_compact_count (sizes read)");
  sizes[0] = h[0];
  sizes[1] = h[1];
  return launched("mesh_compact_count");
}

int s3r_mesh_compact(const float* verts, const int64_t* faces_, int64_t nv, int64_t nf, const void* ws,
                     size_t ws_bytes, float* out_verts, int64_t* out_faces_, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long* faces = reinterpret_cast<const long long*>(faces_);
  long long* out_faces = reinterpret_cast<long long*>(out_faces_);
  if (!verts || !ws || !out_verts || (nf && (!faces || !out_faces)) || (uintptr_t)ws % 256 ||
      s3r_mesh_compact_workspace_bytes(nv, nf) == 0 || ws_bytes < s3r_mesh_compact_workspace_bytes(nv, nf)) {
    set_error("mesh_compact: bad arguments (n_verts=%lld n_faces=%lld workspace_bytes=%zu; need the workspace "
              "s3r_mesh_compact_count filled and non-null pointers)", nv, nf, ws_bytes);
    return -1;
  }
  const CompactLayout w = carve_compact(const_cast<void*>(ws), nv, nf);
  compact_vertices<<<grid_for(nv), kThreads, 0, st>>>(verts, nv, w.vkeep, w.voff, out_verts);
  if (nf) compact_faces<<<grid_for(nf), kThreads, 0, st>>>(faces, nf, w.fkeep, w.foff, w.voff, out_faces);
  return launched("mesh_compact");
}

}  // extern "C"
