// Reconstruction metrics on the GPU: what the reference's eval.py:189-218 runs on host copies of every reconstruction --
// Open3D point-to-point ICP, 30-NN PCA normals, and spann3r/tools/eval_recon.py's accuracy / completion (scipy cKDTree
// nearest-neighbour queries, mean, median, |n . n|).
//
//   Spatial index over one cloud (exact for any distribution; far outliers only cost speed):
//     1. pcl_box_partial / pcl_box_final      bounding box, fixed-order reduction
//     2. pcl_keys_kernel                      63-bit Morton key of every point (21 bits per axis)
//     3. pcl_sort_{hist,scan,scatter} x 8     stable LSD radix sort of (key, original index), 8-bit digits
//     4. pcl_gather_kernel                    fp64 points in sorted order
//     5. pcl_leaf_kernel + pcl_level_kernel   buckets of 32 consecutive sorted points with their real AABB, and an
//                                             implicit complete binary tree of AABBs over them (node i: children 2i,
//                                             2i+1; leaf b = node L + b), built bottom-up
//   Queries (one per thread, stack traversal, near child first; a box is pruned only when its fp64 lower bound is
//   STRICTLY greater than the best squared distance so far, so ties are always visited and break to the smallest
//   original index):
//     pcl_nn_kernel       1-NN with an optional rigid transform of the query and a distance bound
//     pcl_normals_kernel  k-NN (k <= 32) of every indexed point, covariance, smallest eigenvector
//   ICP: pcl_icp_corr_kernel / pcl_icp_update_kernel x (max_iteration + 1) -- fixed launch count, a device-side done flag,
//   per-pass sums in a fixed block order relative to the target's box centre, the Umeyama update on one thread.
//   Statistics of an fp64 vector: fixed-order mean, exact median by a 64-bit radix select (8 x 8-bit passes on the bit
//   pattern, which orders like the value for non-negative doubles once -0.0 is keyed as +0.0), count below a threshold.
#include "kernels.cuh"

#include <climits>
#include <math.h>

#include "pointcloud_math.cuh"

namespace s3r {

using namespace pcl;

namespace {

constexpr int kBucket = 32;
constexpr int kBoxBlocks = 264;
constexpr int kSortTile = 4096;      // elements per block of one radix pass (16 sub-tiles of 256)
constexpr int kStack = 32;           // traversal stack: tree depth is at most 26 for n < 2^31
constexpr int kIcpBlocks = 1056;     // fixed, so the per-pass sums do not depend on the GPU
constexpr int kIcpThreads = 128;
constexpr int kAccN = 17;            // ICP sums: count, sum d^2, sum src (3), sum dst (3), sum src dst^T (9)
constexpr int kStatBlocks = 264;
constexpr int kIcpHeader = 19;       // out: T 4x4, fitness, rmse, passes; then per-pass counts, per-pass rmse
constexpr unsigned long long kNegZero = 0x8000000000000000ULL;   // bit pattern of -0.0

inline size_t align256(size_t x) { return (x + 255) / 256 * 256; }

struct Index {
  double* meta;         // lo[3], hi[3], centre[3], inv_ext[3]
  double* pts;          // [n, 3] in Morton order
  int* orig;            // [n] original index of each sorted point
  double* box;          // [2L, 6] lo xyz, hi xyz (node 0 unused)
  uint64_t* keys[2];
  int* vals[2];
  unsigned* hist;       // [256, nblk]
  double* part;         // [kBoxBlocks, 6]
  long long n;
  int L, nblk;
  size_t bytes;
};

Index carve_index(void* base, long long n) {
  Index x;
  x.n = n;
  const long long nb = (n + kBucket - 1) / kBucket;
  x.L = 1;
  while (x.L < nb) x.L <<= 1;
  x.nblk = (int)((n + kSortTile - 1) / kSortTile);
  size_t o = 0;
  const uintptr_t p = (uintptr_t)base;
  x.meta = (double*)(p + o); o += align256(sizeof(double) * 12);
  x.pts = (double*)(p + o); o += align256(sizeof(double) * 3 * n);
  x.orig = (int*)(p + o); o += align256(sizeof(int) * n);
  x.box = (double*)(p + o); o += align256(sizeof(double) * 6 * 2 * (size_t)x.L);
  for (int i = 0; i < 2; ++i) {
    x.keys[i] = (uint64_t*)(p + o); o += align256(sizeof(uint64_t) * n);
    x.vals[i] = (int*)(p + o); o += align256(sizeof(int) * n);
  }
  x.hist = (unsigned*)(p + o); o += align256(sizeof(unsigned) * 256 * (size_t)x.nblk);
  x.part = (double*)(p + o); o += align256(sizeof(double) * 6 * kBoxBlocks);
  x.bytes = o;
  return x;
}

__device__ __forceinline__ void load_point(const void* pts, int f64, long long i, const double* T, double* out) {
  double x[3];
  if (f64) {
    const double* p = (const double*)pts + 3 * i;
    x[0] = p[0]; x[1] = p[1]; x[2] = p[2];
  } else {
    const float* p = (const float*)pts + 3 * i;
    x[0] = p[0]; x[1] = p[1]; x[2] = p[2];
  }
  if (T) {
    apply_rt(T, x, out);
  } else {
    out[0] = x[0]; out[1] = x[1]; out[2] = x[2];
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// index build
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) pcl_box_partial(const void* __restrict__ pts, int f64, long long n,
                                                       const double* __restrict__ T, double* __restrict__ part) {
  __shared__ double s[6][256];
  double m[6] = {INFINITY, INFINITY, INFINITY, -INFINITY, -INFINITY, -INFINITY};
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += 256LL * kBoxBlocks) {
    double x[3];
    load_point(pts, f64, i, T, x);
    for (int a = 0; a < 3; ++a) {
      m[a] = fmin(m[a], x[a]);
      m[3 + a] = fmax(m[3 + a], x[a]);
    }
  }
  for (int a = 0; a < 6; ++a) s[a][threadIdx.x] = m[a];
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o)
      for (int a = 0; a < 6; ++a)
        s[a][threadIdx.x] = a < 3 ? fmin(s[a][threadIdx.x], s[a][threadIdx.x + o]) : fmax(s[a][threadIdx.x], s[a][threadIdx.x + o]);
    __syncthreads();
  }
  if (threadIdx.x < 6) part[blockIdx.x * 6 + threadIdx.x] = s[threadIdx.x][0];
}

__global__ void __launch_bounds__(32) pcl_box_final(const double* __restrict__ part, double* __restrict__ meta) {
  if (threadIdx.x >= 3) return;
  const int a = threadIdx.x;
  double lo = INFINITY, hi = -INFINITY;
  for (int b = 0; b < kBoxBlocks; ++b) {
    lo = fmin(lo, part[b * 6 + a]);
    hi = fmax(hi, part[b * 6 + 3 + a]);
  }
  meta[a] = lo;
  meta[3 + a] = hi;
  meta[6 + a] = 0.5 * (lo + hi);
  meta[9 + a] = hi > lo ? 1.0 / (hi - lo) : 0.0;
}

__global__ void __launch_bounds__(256) pcl_keys_kernel(const void* __restrict__ pts, int f64, long long n,
                                                       const double* __restrict__ T, const double* __restrict__ meta,
                                                       uint64_t* __restrict__ keys, int* __restrict__ vals) {
  const long long i = blockIdx.x * 256LL + threadIdx.x;
  if (i >= n) return;
  double x[3];
  load_point(pts, f64, i, T, x);
  keys[i] = morton63(x, meta, meta + 9);
  vals[i] = (int)i;
}

__global__ void __launch_bounds__(256) pcl_sort_hist(const uint64_t* __restrict__ keys, long long n, int shift, int nblk,
                                                     unsigned* __restrict__ hist) {
  __shared__ unsigned h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const long long t0 = (long long)blockIdx.x * kSortTile;
  const long long t1 = t0 + kSortTile < n ? t0 + kSortTile : n;
  for (long long i = t0 + threadIdx.x; i < t1; i += 256) atomicAdd(&h[(keys[i] >> shift) & 255], 1u);
  __syncthreads();
  hist[(long long)threadIdx.x * nblk + blockIdx.x] = h[threadIdx.x];
}

// exclusive scan of the digit-major histogram [256, nblk] in place (one block)
__global__ void __launch_bounds__(1024) pcl_sort_scan(unsigned* __restrict__ hist, long long total) {
  __shared__ unsigned s[1024];
  const long long chunk = (total + 1023) / 1024;
  const long long c0 = threadIdx.x * chunk, c1 = c0 + chunk < total ? c0 + chunk : total;
  unsigned sum = 0;
  for (long long i = c0; i < c1; ++i) sum += hist[i];
  s[threadIdx.x] = sum;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {
    const unsigned v = threadIdx.x >= o ? s[threadIdx.x - o] : 0u;
    __syncthreads();
    s[threadIdx.x] += v;
    __syncthreads();
  }
  unsigned run = s[threadIdx.x] - sum;
  for (long long i = c0; i < c1; ++i) {
    const unsigned v = hist[i];
    hist[i] = run;
    run += v;
  }
}

// stable scatter: sub-tiles of 256 in order, warps in order inside a sub-tile, lanes in order inside a warp
__global__ void __launch_bounds__(256) pcl_sort_scatter(const uint64_t* __restrict__ kin, const int* __restrict__ vin,
                                                        long long n, int shift, int nblk, const unsigned* __restrict__ hist,
                                                        uint64_t* __restrict__ kout, int* __restrict__ vout) {
  __shared__ unsigned base[256];
  __shared__ unsigned wcnt[8][256];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  base[tid] = hist[(long long)tid * nblk + blockIdx.x];
  const long long t0 = (long long)blockIdx.x * kSortTile;
  const long long t1 = t0 + kSortTile < n ? t0 + kSortTile : n;
  for (long long s0 = t0; s0 < t1; s0 += 256) {
    for (int w = 0; w < 8; ++w) wcnt[w][tid] = 0;
    __syncthreads();
    const long long i = s0 + tid;
    const bool valid = i < t1;
    uint64_t key = 0;
    int val = 0;
    unsigned digit = 256;
    if (valid) {
      key = kin[i];
      val = vin[i];
      digit = (unsigned)(key >> shift) & 255u;
    }
    const unsigned peers = __match_any_sync(0xffffffffu, digit);
    const unsigned rank = __popc(peers & ((1u << lane) - 1u));
    if (valid && rank == 0) wcnt[warp][digit] = __popc(peers);
    __syncthreads();
    {
      unsigned run = base[tid];
      for (int w = 0; w < 8; ++w) {
        const unsigned c = wcnt[w][tid];
        wcnt[w][tid] = run;
        run += c;
      }
      base[tid] = run;
    }
    __syncthreads();
    if (valid) {
      const unsigned pos = wcnt[warp][digit] + rank;
      kout[pos] = key;
      vout[pos] = val;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256) pcl_gather_kernel(const void* __restrict__ pts, int f64, long long n,
                                                         const double* __restrict__ T, const int* __restrict__ vals,
                                                         double* __restrict__ out, int* __restrict__ orig) {
  const long long i = blockIdx.x * 256LL + threadIdx.x;
  if (i >= n) return;
  const int o = vals[i];
  double x[3];
  load_point(pts, f64, o, T, x);
  out[3 * i] = x[0]; out[3 * i + 1] = x[1]; out[3 * i + 2] = x[2];
  orig[i] = o;
}

__global__ void __launch_bounds__(256) pcl_leaf_kernel(const double* __restrict__ pts, long long n, int L,
                                                       double* __restrict__ box) {
  const long long b = blockIdx.x * 256LL + threadIdx.x;
  if (b >= L) return;
  double m[6] = {INFINITY, INFINITY, INFINITY, -INFINITY, -INFINITY, -INFINITY};
  const long long j0 = b * kBucket, j1 = j0 + kBucket < n ? j0 + kBucket : n;
  for (long long j = j0; j < j1; ++j)
    for (int a = 0; a < 3; ++a) {
      m[a] = fmin(m[a], pts[3 * j + a]);
      m[3 + a] = fmax(m[3 + a], pts[3 * j + a]);
    }
  for (int a = 0; a < 6; ++a) box[6 * (L + b) + a] = m[a];
}

__global__ void __launch_bounds__(256) pcl_level_kernel(int first, int count, double* __restrict__ box) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= count) return;
  const int node = first + i;
  const double* c0 = box + 6 * (2 * node);
  const double* c1 = c0 + 6;
  for (int a = 0; a < 3; ++a) {
    box[6 * node + a] = fmin(c0[a], c1[a]);
    box[6 * node + 3 + a] = fmax(c0[3 + a], c1[3 + a]);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// queries
// ---------------------------------------------------------------------------------------------------------------------
struct IndexView {
  const double* pts;
  const int* orig;
  const double* box;
  long long n;
  int L;
};

IndexView view_of(const Index& x) { return IndexView{x.pts, x.orig, x.box, x.n, x.L}; }

// 1-NN: on entry best2 = the squared distance bound (inclusive) and best = INT_MAX; on exit best is the original index of
// the nearest point (smallest index on ties) or still INT_MAX, pos its sorted position.
__device__ __forceinline__ void nn_search(const IndexView& ix, const double* q, double& best2, int& best, long long& pos) {
  int st_node[kStack];
  double st_lb[kStack];
  int sp = 0, node = 1;
  while (true) {
    if (node >= ix.L) {
      const long long j0 = (long long)(node - ix.L) * kBucket;
      const long long j1 = j0 + kBucket < ix.n ? j0 + kBucket : ix.n;
      for (long long j = j0; j < j1; ++j) {
        const double d2 = dist2(q, ix.pts + 3 * j);
        if (d2 <= best2) {
          const int o = ix.orig[j];
          if (d2 < best2 || o < best) {
            best2 = d2;
            best = o;
            pos = j;
          }
        }
      }
    } else {
      int c0 = 2 * node, c1 = c0 + 1;
      double l0 = box_lb2(q, ix.box + 6 * c0, ix.box + 6 * c0 + 3);
      double l1 = box_lb2(q, ix.box + 6 * c1, ix.box + 6 * c1 + 3);
      if (l1 < l0) {
        const int tn = c0; c0 = c1; c1 = tn;
        const double tl = l0; l0 = l1; l1 = tl;
      }
      if (l0 <= best2) {
        if (l1 <= best2) {
          st_node[sp] = c1;
          st_lb[sp] = l1;
          ++sp;
        }
        node = c0;
        continue;
      }
    }
    bool more = false;
    while (sp > 0) {
      --sp;
      if (st_lb[sp] <= best2) {
        node = st_node[sp];
        more = true;
        break;
      }
    }
    if (!more) break;
  }
}

__global__ void __launch_bounds__(128) pcl_nn_kernel(IndexView ix, const void* __restrict__ q, int f64, long long nq,
                                                     const double* __restrict__ T, double max_d2, double* __restrict__ dist,
                                                     long long* __restrict__ idx) {
  const long long i = blockIdx.x * 128LL + threadIdx.x;
  if (i >= nq) return;
  double x[3];
  load_point(q, f64, i, T, x);
  double best2 = max_d2;
  int best = INT_MAX;
  long long pos = -1;
  nn_search(ix, x, best2, best, pos);
  const bool hit = best != INT_MAX;
  dist[i] = hit ? sqrt(best2) : INFINITY;
  idx[i] = hit ? (long long)best : -1LL;
}

struct SortedPts {
  const double* pts;
  const int* cand;
  __host__ __device__ double operator()(int i, int a) const { return pts[3LL * cand[i] + a]; }
};

// k nearest neighbours (the point itself included) of every indexed point, in sorted order for locality; the normal is
// written at the point's original index.
__global__ void __launch_bounds__(128) pcl_normals_kernel(IndexView ix, int k, double* __restrict__ normals) {
  const long long i = blockIdx.x * 128LL + threadIdx.x;
  if (i >= ix.n) return;
  const double q[3] = {ix.pts[3 * i], ix.pts[3 * i + 1], ix.pts[3 * i + 2]};
  double cd[32];
  int cj[32];      // sorted positions of the candidates, ordered by (d2, original index)
  int cnt = 0;
  int st_node[kStack];
  double st_lb[kStack];
  int sp = 0, node = 1;
  while (true) {
    const double worst = cnt == k ? cd[k - 1] : INFINITY;
    if (node >= ix.L) {
      const long long j0 = (long long)(node - ix.L) * kBucket;
      const long long j1 = j0 + kBucket < ix.n ? j0 + kBucket : ix.n;
      for (long long j = j0; j < j1; ++j) {
        const double d2 = dist2(q, ix.pts + 3 * j);
        const double w = cnt == k ? cd[k - 1] : INFINITY;
        if (d2 > w) continue;
        const int o = ix.orig[j];
        if (cnt == k && d2 == w && o > ix.orig[cj[k - 1]]) continue;
        int p = cnt < k ? cnt++ : k - 1;
        while (p > 0 && (cd[p - 1] > d2 || (cd[p - 1] == d2 && ix.orig[cj[p - 1]] > o))) {
          cd[p] = cd[p - 1];
          cj[p] = cj[p - 1];
          --p;
        }
        cd[p] = d2;
        cj[p] = (int)j;
      }
    } else {
      int c0 = 2 * node, c1 = c0 + 1;
      double l0 = box_lb2(q, ix.box + 6 * c0, ix.box + 6 * c0 + 3);
      double l1 = box_lb2(q, ix.box + 6 * c1, ix.box + 6 * c1 + 3);
      if (l1 < l0) {
        const int tn = c0; c0 = c1; c1 = tn;
        const double tl = l0; l0 = l1; l1 = tl;
      }
      if (l0 <= worst) {
        if (l1 <= worst) {
          st_node[sp] = c1;
          st_lb[sp] = l1;
          ++sp;
        }
        node = c0;
        continue;
      }
    }
    bool more = false;
    const double w = cnt == k ? cd[k - 1] : INFINITY;
    while (sp > 0) {
      --sp;
      if (st_lb[sp] <= w) {
        node = st_node[sp];
        more = true;
        break;
      }
    }
    if (!more) break;
  }
  double nrm[3];
  knn_normal(SortedPts{ix.pts, cj}, cnt, nrm);
  double* o = normals + 3LL * ix.orig[i];
  o[0] = nrm[0]; o[1] = nrm[1]; o[2] = nrm[2];
}

// ---------------------------------------------------------------------------------------------------------------------
// ICP
// ---------------------------------------------------------------------------------------------------------------------
struct IcpState {
  double T[12];
  double prev_fitness, prev_rmse;
  int pass, done;
};

__global__ void __launch_bounds__(32) pcl_icp_init(const double* __restrict__ init, int max_iteration, IcpState* st,
                                                   double* __restrict__ out) {
  if (threadIdx.x != 0) return;
  for (int i = 0; i < 12; ++i) st->T[i] = init ? init[i] : ((i % 5 == 0) ? 1.0 : 0.0);
  st->prev_fitness = st->prev_rmse = 0;
  st->pass = 0;
  st->done = 0;
  for (int i = 0; i < kIcpHeader + 2 * (max_iteration + 1); ++i) out[i] = 0;
}

__global__ void __launch_bounds__(kIcpThreads) pcl_icp_corr_kernel(IndexView ix, const double* __restrict__ meta,
                                                                   const void* __restrict__ src, int f64, long long ns,
                                                                   double max_d2, const IcpState* __restrict__ st,
                                                                   double* __restrict__ part) {
  if (st->done) return;
  __shared__ double s_w[kIcpThreads / 32][kAccN];
  double T[12];
  for (int i = 0; i < 12; ++i) T[i] = st->T[i];
  const double c[3] = {meta[6], meta[7], meta[8]};
  double acc[kAccN];
#pragma unroll
  for (int j = 0; j < kAccN; ++j) acc[j] = 0;
  for (long long i = blockIdx.x * (long long)kIcpThreads + threadIdx.x; i < ns; i += (long long)kIcpThreads * kIcpBlocks) {
    double x[3];
    load_point(src, f64, i, T, x);
    double best2 = max_d2;
    int best = INT_MAX;
    long long pos = -1;
    nn_search(ix, x, best2, best, pos);
    if (best == INT_MAX) continue;
    const double ps[3] = {x[0] - c[0], x[1] - c[1], x[2] - c[2]};
    const double qs[3] = {ix.pts[3 * pos] - c[0], ix.pts[3 * pos + 1] - c[1], ix.pts[3 * pos + 2] - c[2]};
    acc[0] += 1.0;
    acc[1] += best2;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      acc[2 + a] += ps[a];
      acc[5 + a] += qs[a];
#pragma unroll
      for (int b = 0; b < 3; ++b) acc[8 + 3 * a + b] += ps[a] * qs[b];
    }
  }
  const int tid = threadIdx.x;
#pragma unroll
  for (int j = 0; j < kAccN; ++j) {
    double v = acc[j];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if ((tid & 31) == 0) s_w[tid >> 5][j] = v;
  }
  __syncthreads();
  if (tid < kAccN) {
    double s = 0;
    for (int w = 0; w < kIcpThreads / 32; ++w) s += s_w[w][tid];
    part[(long long)blockIdx.x * kAccN + tid] = s;
  }
}

__global__ void __launch_bounds__(32) pcl_icp_update_kernel(const double* __restrict__ part, const double* __restrict__ meta,
                                                            long long ns, int max_iteration, double rel_fitness,
                                                            double rel_rmse, IcpState* st, double* __restrict__ out) {
  if (st->done) return;
  __shared__ double acc[kAccN];
  const int tid = threadIdx.x;
  if (tid < kAccN) {
    double s = 0;
    for (int b = 0; b < kIcpBlocks; ++b) s += part[(long long)b * kAccN + tid];
    acc[tid] = s;
  }
  __syncthreads();
  if (tid != 0) return;
  const int j = st->pass;
  const double cnt = acc[0];
  const double fitness = cnt / (double)ns;
  const double rmse = cnt > 0 ? sqrt(acc[1] / cnt) : 0.0;
  for (int r = 0; r < 3; ++r)
    for (int cc = 0; cc < 4; ++cc) out[4 * r + cc] = st->T[4 * r + cc];
  out[12] = out[13] = out[14] = 0;
  out[15] = 1;
  out[16] = fitness;
  out[17] = rmse;
  out[18] = j + 1;
  out[kIcpHeader + j] = cnt;
  out[kIcpHeader + max_iteration + 1 + j] = rmse;
  if ((j >= 1 && fabs(st->prev_fitness - fitness) < rel_fitness && fabs(st->prev_rmse - rmse) < rel_rmse) ||
      j == max_iteration) {
    st->done = 1;
    return;
  }
  double U[12];
  umeyama_rt(acc, meta + 6, U);
  compose_rt(U, st->T);
  st->prev_fitness = fitness;
  st->prev_rmse = rmse;
  st->pass = j + 1;
}

// ---------------------------------------------------------------------------------------------------------------------
// statistics of an fp64 vector
// ---------------------------------------------------------------------------------------------------------------------
struct SelectState {
  unsigned hist[256];
  unsigned long long prefix, k;
};
struct StatsWs {
  double sum[kStatBlocks];
  unsigned long long below[kStatBlocks];
  SelectState sel[2];   // ranks (n - 1) / 2 and n / 2: np.median's two middle order statistics
};

__global__ void __launch_bounds__(256) pcl_stats_partial(const double* __restrict__ x, long long n, double thr,
                                                         StatsWs* ws) {
  __shared__ double s[256];
  __shared__ unsigned long long c[256];
  double sum = 0;
  unsigned long long cnt = 0;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += 256LL * kStatBlocks) {
    const double v = x[i];
    sum += v;
    cnt += v < thr ? 1 : 0;
  }
  s[threadIdx.x] = sum;
  c[threadIdx.x] = cnt;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      s[threadIdx.x] += s[threadIdx.x + o];
      c[threadIdx.x] += c[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    ws->sum[blockIdx.x] = s[0];
    ws->below[blockIdx.x] = c[0];
  }
}

__global__ void __launch_bounds__(256) pcl_select_hist(const double* __restrict__ x, long long n, int pass, StatsWs* ws) {
  __shared__ unsigned h[256];
  SelectState& S = ws->sel[blockIdx.y];
  h[threadIdx.x] = 0;
  __syncthreads();
  const int shift = 56 - 8 * pass;
  const unsigned long long prefix = S.prefix;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += 256LL * kStatBlocks) {
    unsigned long long key = (unsigned long long)__double_as_longlong(x[i]);
    if (key == kNegZero) key = 0;   // -0.0 == +0.0; its sign bit alone would sort it above +inf
    if (pass > 0 && (key >> (shift + 8)) != prefix) continue;
    atomicAdd(&h[(key >> shift) & 255], 1u);
  }
  __syncthreads();
  if (h[threadIdx.x]) atomicAdd(&S.hist[threadIdx.x], h[threadIdx.x]);
}

__global__ void __launch_bounds__(32) pcl_select_pick(long long n, int pass, StatsWs* ws) {
  if (threadIdx.x >= 2) return;
  SelectState& S = ws->sel[threadIdx.x];
  unsigned long long k = pass == 0 ? (unsigned long long)(threadIdx.x == 0 ? (n - 1) / 2 : n / 2) : S.k;
  int bin = 0;
  while (bin < 255 && k >= S.hist[bin]) k -= S.hist[bin++];
  S.prefix = (S.prefix << 8) | (unsigned long long)bin;
  S.k = k;
  for (int i = 0; i < 256; ++i) S.hist[i] = 0;
}

__global__ void __launch_bounds__(32) pcl_stats_final(long long n, const StatsWs* ws, double* __restrict__ out) {
  if (threadIdx.x != 0) return;
  double s = 0;
  unsigned long long c = 0;
  for (int b = 0; b < kStatBlocks; ++b) {
    s += ws->sum[b];
    c += ws->below[b];
  }
  const double lo = __longlong_as_double((long long)ws->sel[0].prefix);
  const double hi = __longlong_as_double((long long)ws->sel[1].prefix);
  out[0] = s / (double)n;
  out[1] = (n & 1) ? lo : (lo + hi) / 2.0;
  out[2] = (double)c;
}

__global__ void __launch_bounds__(256) pcl_abs_dot_kernel(const double* __restrict__ a, const double* __restrict__ b,
                                                          const long long* __restrict__ idx, long long n,
                                                          double* __restrict__ out) {
  const long long i = blockIdx.x * 256LL + threadIdx.x;
  if (i >= n) return;
  const long long j = idx[i];
  const double* p = a + 3 * i;
  const double* q = b + 3 * j;
  out[i] = fabs(add_rn(add_rn(mul_rn(p[0], q[0]), mul_rn(p[1], q[1])), mul_rn(p[2], q[2])));
}

bool n_ok(long long n) { return n >= 1 && n < (1LL << 31); }

// The largest squared distance whose sqrt is <= max_dist: the bound is inclusive on the DISTANCE, as the caller sees it
// (sqrt rounds, so max_dist * max_dist alone can drop a point at exactly max_dist).
double bound2(double max_dist) {
  if (isinf(max_dist)) return INFINITY;
  double m2 = max_dist * max_dist;
  while (sqrt(nextafter(m2, INFINITY)) <= max_dist) m2 = nextafter(m2, INFINITY);
  while (m2 > 0 && sqrt(m2) > max_dist) m2 = nextafter(m2, 0.0);
  return m2;
}

int launched(const char* what) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: launch failed: %s", what, cudaGetErrorString(e));
    return -6;
  }
  return 0;
}

}  // namespace

size_t pcl_index_bytes(long long n) { return n_ok(n) ? carve_index(nullptr, n).bytes : 0; }

int launch_pcl_index_build(const void* pts, int f64, long long n, const double* T, void* index, cudaStream_t st) {
  if (!pts || !index || !n_ok(n)) {
    set_error("pcl_index_build: bad arguments (n=%lld; need 1 <= n < 2^31 and non-null pointers)", n);
    return -1;
  }
  if ((uintptr_t)index % 16 != 0) {
    set_error("pcl_index_build: index workspace must be 16-byte aligned");
    return -1;
  }
  Index x = carve_index(index, n);
  pcl_box_partial<<<kBoxBlocks, 256, 0, st>>>(pts, f64, n, T, x.part);
  pcl_box_final<<<1, 32, 0, st>>>(x.part, x.meta);
  const int g = (int)((n + 255) / 256);
  pcl_keys_kernel<<<g, 256, 0, st>>>(pts, f64, n, T, x.meta, x.keys[0], x.vals[0]);
  for (int pass = 0; pass < 8; ++pass) {
    const int a = pass & 1;
    pcl_sort_hist<<<x.nblk, 256, 0, st>>>(x.keys[a], n, 8 * pass, x.nblk, x.hist);
    pcl_sort_scan<<<1, 1024, 0, st>>>(x.hist, 256LL * x.nblk);
    pcl_sort_scatter<<<x.nblk, 256, 0, st>>>(x.keys[a], x.vals[a], n, 8 * pass, x.nblk, x.hist, x.keys[a ^ 1],
                                             x.vals[a ^ 1]);
  }
  pcl_gather_kernel<<<g, 256, 0, st>>>(pts, f64, n, T, x.vals[0], x.pts, x.orig);
  pcl_leaf_kernel<<<(x.L + 255) / 256, 256, 0, st>>>(x.pts, n, x.L, x.box);
  for (int first = x.L / 2; first >= 1; first /= 2)
    pcl_level_kernel<<<(first + 255) / 256, 256, 0, st>>>(first, first, x.box);
  return launched("pcl_index_build");
}

int launch_pcl_nearest(const void* index, long long n, const void* q, int f64, long long nq, const double* T,
                       double max_dist, double* dist, long long* idx, cudaStream_t st) {
  if (!index || !q || !dist || !idx || !n_ok(n) || !n_ok(nq) || !(max_dist >= 0)) {
    set_error("pcl_nearest: bad arguments (n=%lld nq=%lld max_dist=%g)", n, nq, max_dist);
    return -1;
  }
  const Index x = carve_index(const_cast<void*>(index), n);
  const double max_d2 = bound2(max_dist);
  pcl_nn_kernel<<<(int)((nq + 127) / 128), 128, 0, st>>>(view_of(x), q, f64, nq, T, max_d2, dist, idx);
  return launched("pcl_nearest");
}

int launch_pcl_normals(const void* index, long long n, int k, double* normals, cudaStream_t st) {
  if (!index || !normals || !n_ok(n) || k < 1 || k > 32) {
    set_error("pcl_normals: bad arguments (n=%lld k=%d; need 1 <= k <= 32)", n, k);
    return -1;
  }
  const Index x = carve_index(const_cast<void*>(index), n);
  const int ke = (long long)k < n ? k : (int)n;
  pcl_normals_kernel<<<(int)((n + 127) / 128), 128, 0, st>>>(view_of(x), ke, normals);
  return launched("pcl_normals");
}

size_t pcl_icp_workspace_bytes() { return align256(sizeof(IcpState)) + align256(sizeof(double) * kIcpBlocks * kAccN); }

int launch_pcl_icp(const void* src, int f64, long long ns, const void* target_index, long long nt, double max_corr,
                   const double* init, int max_iteration, double rel_fitness, double rel_rmse, void* workspace,
                   double* out, cudaStream_t st) {
  if (!src || !target_index || !workspace || !out || !n_ok(ns) || !n_ok(nt) || !(max_corr >= 0) || max_iteration < 0 ||
      max_iteration > 10000 || !(rel_fitness >= 0) || !(rel_rmse >= 0)) {
    set_error("pcl_icp: bad arguments (ns=%lld nt=%lld max_corr=%g max_iteration=%d)", ns, nt, max_corr, max_iteration);
    return -1;
  }
  if ((uintptr_t)workspace % 16 != 0) {
    set_error("pcl_icp: workspace must be 16-byte aligned");
    return -1;
  }
  const Index x = carve_index(const_cast<void*>(target_index), nt);
  IcpState* state = (IcpState*)workspace;
  double* part = (double*)((uintptr_t)workspace + align256(sizeof(IcpState)));
  const double max_d2 = bound2(max_corr);
  pcl_icp_init<<<1, 32, 0, st>>>(init, max_iteration, state, out);
  for (int j = 0; j <= max_iteration; ++j) {
    pcl_icp_corr_kernel<<<kIcpBlocks, kIcpThreads, 0, st>>>(view_of(x), x.meta, src, f64, ns, max_d2, state, part);
    pcl_icp_update_kernel<<<1, 32, 0, st>>>(part, x.meta, ns, max_iteration, rel_fitness, rel_rmse, state, out);
  }
  return launched("pcl_icp");
}

size_t pcl_stats_workspace_bytes() { return align256(sizeof(StatsWs)); }

int launch_pcl_stats(const double* v, long long n, double threshold, void* workspace, double* out, cudaStream_t st) {
  if (!v || !workspace || !out || !n_ok(n)) {
    set_error("pcl_stats: bad arguments (n=%lld)", n);
    return -1;
  }
  StatsWs* ws = (StatsWs*)workspace;
  cudaMemsetAsync(ws->sel, 0, sizeof(ws->sel), st);
  pcl_stats_partial<<<kStatBlocks, 256, 0, st>>>(v, n, threshold, ws);
  for (int pass = 0; pass < 8; ++pass) {
    pcl_select_hist<<<dim3(kStatBlocks, 2), 256, 0, st>>>(v, n, pass, ws);
    pcl_select_pick<<<1, 32, 0, st>>>(n, pass, ws);
  }
  pcl_stats_final<<<1, 32, 0, st>>>(n, ws, out);
  return launched("pcl_stats");
}

int launch_pcl_abs_dot(const double* a, const double* b, const long long* idx, long long n, double* out, cudaStream_t st) {
  if (!a || !b || !idx || !out || !n_ok(n)) {
    set_error("pcl_abs_dot: bad arguments (n=%lld)", n);
    return -1;
  }
  pcl_abs_dot_kernel<<<(int)((n + 255) / 256), 256, 0, st>>>(a, b, idx, n, out);
  return launched("pcl_abs_dot");
}

}  // namespace s3r
