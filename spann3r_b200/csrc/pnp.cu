// Post-path geometry on the GPU (SURVEY.md section 8f rank 4, second step): the per-frame camera pose that demo.py:166-180
// obtains with `cv2.solvePnPRansac(pts3d.reshape(-1, 3), pixel grid, K, 0)` on a CPU copy of every pointmap
// (~0.3 s per 512x384 frame with OpenCV 4.13 on the host -- 60x the network's time per frame).  Batched over frames,
// everything stays on the device:
//
//   1. pnp_hyp_kernel     one thread per minimal sample (3 points picked by a counter-based hash): Grunert P3P,
//                         up to 4 poses each                                                        (pnp_math.cuh)
//   2. pnp_score_kernel   inlier count (reprojection error < threshold, default 8 px) of EVERY hypothesis over EVERY
//                         point: a block = 256 hypotheses x one slab of points staged through shared memory, integer
//                         atomics (deterministic)
//   3. pnp_select_kernel  best hypothesis (ties -> lowest index)
//   4. pnp_mask_kernel    its inlier mask (what cv2 returns as `inliers`)
//   5. pnp_gn_partial_kernel / pnp_gn_update_kernel x (iters + 1): damped Gauss-Newton (Levenberg-Marquardt
//                         accept / reject on the device, no host round trip) on the inliers' reprojection error --
//                         the same least-squares problem cv2's final SOLVEPNP_ITERATIVE refinement solves; 148
//                         fixed-order partial sums of the 6x6 normal equations in fp64, then one thread solves.
//
// HBM-bound point work (12 B per point per pass, the 2.4 MB pointmap stays in L2); the result is the least-squares
// optimum on the inlier set, so it agrees with cv2 to ~1e-14 on clean data and to the few-inlier difference of two
// RANSAC runs (~1e-4) otherwise -- tests/test_pnp.py.
#include "../../include/spann3r_b200.h"
#include "gemm.cuh"

#include "common.cuh"
#include "pnp_math.cuh"

namespace s3r {

using namespace pnp;

constexpr int kPnpBlocks = 148;

struct PnpState {
  Pose good;
  double good_acc[kAcc];
  double good_cost, lambda;
  int have_good, valid;
  long long best_count;
};

static inline size_t align256(size_t x) { return (x + 255) / 256 * 256; }

struct PnpWorkspace {
  Pose* hyps;        // [B, Hn]
  int* valid;        // [B, Hn]
  int* counts;       // [B, Hn]
  Pose* pose;        // [B] current iterate
  PnpState* state;   // [B]
  double* partial;   // [B, kPnpBlocks, kAcc]
  size_t bytes;
};

static PnpWorkspace carve(void* base, int B, int Hn) {
  PnpWorkspace w;
  size_t o = 0;
  const uintptr_t p = (uintptr_t)base;
  w.hyps = (Pose*)(p + o); o += align256(sizeof(Pose) * (size_t)B * Hn);
  w.valid = (int*)(p + o); o += align256(sizeof(int) * (size_t)B * Hn);
  w.counts = (int*)(p + o); o += align256(sizeof(int) * (size_t)B * Hn);
  w.pose = (Pose*)(p + o); o += align256(sizeof(Pose) * (size_t)B);
  w.state = (PnpState*)(p + o); o += align256(sizeof(PnpState) * (size_t)B);
  w.partial = (double*)(p + o); o += align256(sizeof(double) * (size_t)B * kPnpBlocks * kAcc);
  w.bytes = o;
  return w;
}

__global__ void __launch_bounds__(64) pnp_hyp_kernel(const float* __restrict__ pts, const float* __restrict__ img,
                                                     long long n, int width, Cam k, unsigned long long seed,
                                                     int n_samples, Pose* __restrict__ hyps, int* __restrict__ valid) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (m >= n_samples) return;
  const int Hn = 4 * n_samples;
  Pose h[4];
  const int c = sample_hypotheses(seed, m, pts + (long long)b * n * 3, img ? img + (long long)b * n * 2 : nullptr, n, width,
                                  k, h);
  for (int j = 0; j < 4; ++j) {
    const long long o = (long long)b * Hn + 4 * m + j;
    valid[o] = j < c ? 1 : 0;
    if (j < c) hyps[o] = h[j];
  }
}

__global__ void __launch_bounds__(256) pnp_score_kernel(const float* __restrict__ pts, const float* __restrict__ img,
                                                        long long n, int width, Cam k, double thr2,
                                                        const Pose* __restrict__ hyps, const int* __restrict__ valid,
                                                        int Hn, int* __restrict__ counts) {
  __shared__ double sX[256][5];
  const int tid = threadIdx.x, b = blockIdx.z;
  const int h = blockIdx.y * 256 + tid;
  const bool act = h < Hn && valid[(long long)b * Hn + h] != 0;
  Pose T;
  if (act) T = hyps[(long long)b * Hn + h];
  const float* p = pts + (long long)b * n * 3;
  const float* im = img ? img + (long long)b * n * 2 : nullptr;
  const long long per = (n + gridDim.x - 1) / gridDim.x;
  const long long i0 = blockIdx.x * per, i1 = (i0 + per < n) ? i0 + per : n;
  int count = 0;
  for (long long base = i0; base < i1; base += 256) {
    const long long i = base + tid;
    double X[3] = {0, 0, 0}, u = 0, v = 0;
    const bool ok = i < i1 && load_point(p, im, i, width, X, u, v);
    sX[tid][0] = X[0]; sX[tid][1] = X[1]; sX[tid][2] = X[2];
    sX[tid][3] = u;
    sX[tid][4] = ok ? v : nan("");
    __syncthreads();
    const int m = (int)((i1 - base < 256) ? i1 - base : 256);
    if (act) {
      for (int j = 0; j < m; ++j) {
        const double vv = sX[j][4];
        if (vv == vv && reproj_err2(T, k, &sX[j][0], sX[j][3], vv) < thr2) ++count;
      }
    }
    __syncthreads();
  }
  if (act && count) atomicAdd(&counts[(long long)b * Hn + h], count);
}

__global__ void __launch_bounds__(256) pnp_select_kernel(const Pose* __restrict__ hyps, const int* __restrict__ valid,
                                                         const int* __restrict__ counts, int Hn, Pose* __restrict__ pose,
                                                         PnpState* __restrict__ state) {
  __shared__ int s_cnt[256], s_idx[256];
  const int b = blockIdx.x, tid = threadIdx.x;
  int bc = -1, bi = 0x7fffffff;
  for (int h = tid; h < Hn; h += 256) {
    if (!valid[(long long)b * Hn + h]) continue;
    const int c = counts[(long long)b * Hn + h];
    if (c > bc || (c == bc && h < bi)) {
      bc = c;
      bi = h;
    }
  }
  s_cnt[tid] = bc;
  s_idx[tid] = bi;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (tid < o) {
      const int c2 = s_cnt[tid + o], i2 = s_idx[tid + o];
      if (c2 > s_cnt[tid] || (c2 == s_cnt[tid] && i2 < s_idx[tid])) {
        s_cnt[tid] = c2;
        s_idx[tid] = i2;
      }
    }
    __syncthreads();
  }
  if (tid == 0) {
    PnpState& st = state[b];
    st.valid = s_cnt[0] >= 4 ? 1 : 0;
    st.best_count = s_cnt[0] > 0 ? s_cnt[0] : 0;
    st.have_good = 0;
    st.good_cost = 0;
    st.lambda = 1e-4;
    Pose T;
    for (int i = 0; i < 9; ++i) T.R[i] = (i % 4 == 0) ? 1.0 : 0.0;
    T.t[0] = T.t[1] = T.t[2] = 0;
    if (st.valid) T = hyps[(long long)b * Hn + s_idx[0]];
    pose[b] = T;
    st.good = T;
  }
}

__global__ void __launch_bounds__(256) pnp_mask_kernel(const float* __restrict__ pts, const float* __restrict__ img,
                                                       long long n, int width, Cam k, double thr2,
                                                       const Pose* __restrict__ pose, const PnpState* __restrict__ state,
                                                       unsigned char* __restrict__ mask) {
  const int b = blockIdx.y;
  const Pose T = pose[b];
  const bool valid = state[b].valid != 0;
  const float* p = pts + (long long)b * n * 3;
  const float* im = img ? img + (long long)b * n * 2 : nullptr;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += 256LL * gridDim.x) {
    double X[3], u, v;
    const bool in = valid && load_point(p, im, i, width, X, u, v) && reproj_err2(T, k, X, u, v) < thr2;
    mask[(long long)b * n + i] = in ? 1 : 0;
  }
}

__global__ void __launch_bounds__(256) pnp_gn_partial_kernel(const float* __restrict__ pts, const float* __restrict__ img,
                                                             long long n, int width, Cam k,
                                                             const unsigned char* __restrict__ mask,
                                                             const Pose* __restrict__ pose, double* __restrict__ partial) {
  __shared__ double s_w[8][kAcc];
  const int b = blockIdx.y, tid = threadIdx.x;
  const Pose T = pose[b];
  const float* p = pts + (long long)b * n * 3;
  const float* im = img ? img + (long long)b * n * 2 : nullptr;
  const unsigned char* mk = mask + (long long)b * n;
  double acc[kAcc];
#pragma unroll
  for (int j = 0; j < kAcc; ++j) acc[j] = 0;
  for (long long i = blockIdx.x * 256LL + tid; i < n; i += 256LL * kPnpBlocks) {
    if (!mk[i]) continue;
    double X[3], u, v;
    if (!load_point(p, im, i, width, X, u, v)) continue;
    gn_accumulate(T, k, X, u, v, acc);
  }
#pragma unroll
  for (int j = 0; j < kAcc; ++j) {
    double x = acc[j];
    for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
    if ((tid & 31) == 0) s_w[tid >> 5][j] = x;
  }
  __syncthreads();
  if (tid < kAcc) {
    double s = 0;
    for (int w = 0; w < 8; ++w) s += s_w[w][tid];
    partial[((long long)b * kPnpBlocks + blockIdx.x) * kAcc + tid] = s;
  }
}

// out [b, 18]: R (9, row-major), t (3), rvec (3), inliers of the RANSAC model, RMS reprojection error of the
// refined pose on them (px), success (1 / 0)
__global__ void __launch_bounds__(32) pnp_gn_update_kernel(const double* __restrict__ partial, Pose* __restrict__ pose,
                                                           PnpState* __restrict__ state, int final_pass,
                                                           double* __restrict__ out) {
  __shared__ double acc[kAcc];
  const int b = blockIdx.x, tid = threadIdx.x;
  if (tid < kAcc) {
    double s = 0;
    for (int blk = 0; blk < kPnpBlocks; ++blk) s += partial[((long long)b * kPnpBlocks + blk) * kAcc + tid];
    acc[tid] = s;
  }
  __syncthreads();
  if (tid != 0) return;
  PnpState& st = state[b];
  if (st.valid) {
    if (!st.have_good || acc[27] <= st.good_cost) {   // accept the iterate the sums were taken at
      st.good = pose[b];
      for (int j = 0; j < kAcc; ++j) st.good_acc[j] = acc[j];
      st.good_cost = acc[27];
      st.have_good = 1;
      st.lambda = st.lambda * 0.1 > 1e-9 ? st.lambda * 0.1 : 1e-9;
    } else {                                          // reject: back to the last good iterate, more damping
      st.lambda = st.lambda * 10 < 1e6 ? st.lambda * 10 : 1e6;
    }
    Pose T = st.good;
    if (!final_pass) gn_step(st.good_acc, st.lambda, T);
    pose[b] = T;
  }
  if (final_pass) {
    double* o = out + (long long)b * 18;
    const Pose& G = st.good;
    for (int i = 0; i < 9; ++i) o[i] = G.R[i];
    for (int i = 0; i < 3; ++i) o[9 + i] = G.t[i];
    so3_log(G.R, o + 12);
    o[15] = st.valid ? (double)st.best_count : 0.0;   // the inlier count of the mask returned (empty on failure)
    o[16] = (st.valid && st.good_acc[28] > 0) ? sqrt(st.good_cost / st.good_acc[28]) : 0.0;
    o[17] = st.valid ? 1.0 : 0.0;
  }
}

}  // namespace s3r

using namespace s3r;

extern "C" {

size_t s3r_pnp_workspace_bytes(int B, int n_samples) {
  if (B <= 0 || n_samples <= 0) return 0;
  return carve(nullptr, B, 4 * n_samples).bytes;
}

int s3r_pnp_ransac(const float* pts3d, const float* img_pts, int B, int64_t n, int width, double fx, double fy, double cx,
                   double cy, float reproj_err, int n_samples, int refine_iters, uint64_t seed, void* workspace,
                   double* out, uint8_t* inlier_mask, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!pts3d || !workspace || !out || !inlier_mask || B <= 0 || n < 4 || n_samples <= 0 || n_samples > 4096 ||
      refine_iters < 0 || refine_iters > 100 || !(reproj_err > 0) || !(fx > 0) || !(fy > 0) || (!img_pts && width <= 0)) {
    set_error("pnp_ransac: bad arguments (b=%d n=%lld width=%d samples=%d iters=%d)", B, n, width, n_samples, refine_iters);
    return -1;
  }
  const int Hn = 4 * n_samples;
  if ((uintptr_t)workspace % 16 != 0) {
    set_error("pnp_ransac: workspace must be 16-byte aligned");
    return -1;
  }
  PnpWorkspace w = carve(workspace, B, Hn);
  const Cam k{fx, fy, cx, cy};
  const double thr2 = (double)reproj_err * (double)reproj_err;
  cudaMemsetAsync(w.counts, 0, sizeof(int) * (size_t)B * Hn, st);
  pnp_hyp_kernel<<<dim3((n_samples + 63) / 64, B), 64, 0, st>>>(pts3d, img_pts, n, width, k, seed, n_samples, w.hyps, w.valid);
  const int slabs = (int)((n + 2047) / 2048 < 74 ? (n + 2047) / 2048 : 74);
  pnp_score_kernel<<<dim3(slabs, (Hn + 255) / 256, B), 256, 0, st>>>(pts3d, img_pts, n, width, k, thr2, w.hyps, w.valid, Hn,
                                                                      w.counts);
  pnp_select_kernel<<<B, 256, 0, st>>>(w.hyps, w.valid, w.counts, Hn, w.pose, w.state);
  pnp_mask_kernel<<<dim3(kPnpBlocks, B), 256, 0, st>>>(pts3d, img_pts, n, width, k, thr2, w.pose, w.state, inlier_mask);
  for (int it = 0; it <= refine_iters; ++it) {
    pnp_gn_partial_kernel<<<dim3(kPnpBlocks, B), 256, 0, st>>>(pts3d, img_pts, n, width, k, inlier_mask, w.pose, w.partial);
    pnp_gn_update_kernel<<<B, 32, 0, st>>>(w.partial, w.pose, w.state, it == refine_iters ? 1 : 0, out);
  }
  if (cudaGetLastError() != cudaSuccess) {
    set_error("pnp_ransac: launch failed");
    return -6;
  }
  return 0;
}

}  // extern "C"
