// Post-path geometry on the GPU (SURVEY.md section 8f rank 4, first step): focal length of the first camera from its
// pointmap, the reference's `estimate_focal_knowing_depth(..., focal_mode='weiszfeld')`
// (dust3r/post_process.py:12-60, called by demo.py:148-150 on a CPU copy of preds[0]['pts3d']).
//
//   a = (x/z, y/z) with non-finite values -> 0,  p = (i - ppx, j - ppy)
//   f0 = sum(a.p) / sum(a.a);   10 x:  w = 1 / max(|p - f a|, 1e-8),  f = sum(w a.p) / sum(w a.a)
//
// NaN propagates as in the reference's torch ops: a frame with no usable x / z (every z = 0, every point NaN) gives
// f0 = 0 / 0 and returns NaN, through the weight floor and the final clip alike.
// (the reference's means cancel in the ratio).  Each iteration is two fixed-shape launches -- 148 x 256-thread partial
// sums per image in a fixed order, then one block per image -- so the result is deterministic; the pointmap
// (2.4 MB at 512 x 384) stays in L2 across the 11 passes and never crosses PCIe.
#include "../../include/spann3r_b200.h"
#include "gemm.cuh"

#include "common.cuh"
#include "focal_math.cuh"

namespace s3r {

constexpr int kFocalBlocks = 148;

__global__ void __launch_bounds__(256) focal_partial_kernel(const float* __restrict__ pts, int H, int W, float ppx,
                                                            float ppy, const float* __restrict__ focal, int first,
                                                            float* __restrict__ part) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float r0[256], r1[256];
  const int b = blockIdx.y;
  const long long n = (long long)H * W;
  const float* p = pts + (long long)b * n * 3;
  const float f = first ? 0.f : focal[b];
  float s_px = 0.f, s_xx = 0.f;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += 256LL * kFocalBlocks) {
    const float x = p[3 * i], y = p[3 * i + 1], z = p[3 * i + 2];
    float ax = x / z, ay = y / z;
    if (!isfinite(ax)) ax = 0.f;     // nan_to_num(posinf=0, neginf=0): nan -> 0 as well
    if (!isfinite(ay)) ay = 0.f;
    const float u = (float)(i % W) - ppx, v = (float)(i / W) - ppy;
    const float d_px = ax * u + ay * v, d_xx = ax * ax + ay * ay;
    float w = 1.f;
    if (!first) {
      const float du = u - f * ax, dv = v - f * ay;
      const float dis = sqrtf(du * du + dv * dv);
      w = 1.0f / (dis < 1e-8f ? 1e-8f : dis);   // dis.clip(min=1e-8): a NaN distance stays NaN (fmaxf would drop it)
    }
    s_px += w * d_px;
    s_xx += w * d_xx;
  }
  r0[threadIdx.x] = s_px;
  r1[threadIdx.x] = s_xx;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      r0[threadIdx.x] += r0[threadIdx.x + o];
      r1[threadIdx.x] += r1[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    part[((long long)b * kFocalBlocks + blockIdx.x) * 2] = r0[0];
    part[((long long)b * kFocalBlocks + blockIdx.x) * 2 + 1] = r1[0];
  }
}

__global__ void __launch_bounds__(256) focal_final_kernel(const float* __restrict__ part, float lo, float hi, int last,
                                                          float* __restrict__ focal) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float r0[256], r1[256];
  const int b = blockIdx.x;
  r0[threadIdx.x] = threadIdx.x < kFocalBlocks ? part[((long long)b * kFocalBlocks + threadIdx.x) * 2] : 0.f;
  r1[threadIdx.x] = threadIdx.x < kFocalBlocks ? part[((long long)b * kFocalBlocks + threadIdx.x) * 2 + 1] : 0.f;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      r0[threadIdx.x] += r0[threadIdx.x + o];
      r1[threadIdx.x] += r1[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    float f = r0[0] / r1[0];
    if (last) {   // focal.clip(min_focal * base, max_focal * base): a NaN focal (no usable x / z) stays NaN
      f = f < lo ? lo : f;
      f = f > hi ? hi : f;
    }
    focal[b] = f;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// focal_mode='median' (dust3r/post_process.py:26-36): nanmedian over the 2*H*W votes (u z / x, v z / y) of an image.
// The median is an ELEMENT of the vote set, so it is selected, not averaged: 4 passes of an 8-bit radix select on the
// order-preserving integer key of the fp32 votes (recomputed on the fly, never materialised); integer histogram
// atomics only -> bit-exact and deterministic.  Per pass: focal_median_hist_kernel (148 blocks per image, shared-memory
// histogram of the keys that match the prefix found so far) + focal_median_pick_kernel (one block per image: the bin
// that holds rank k, the lower median as torch.nanmedian defines it).
// scratch (int32): per image 256 histogram bins + {prefix, k_lo, k_hi, state}.
// ------------------------------------------------------------------------------------------------------------------
constexpr int kMedianBlocks = 148;
constexpr int kMedianScratch = 256 + 4;

__global__ void __launch_bounds__(256) focal_median_hist_kernel(const float* __restrict__ pts, int H, int W, float ppx,
                                                                float ppy, int pass, int* __restrict__ scratch) {
  __shared__ int hist[256];
  const int b = blockIdx.y;
  int* sc = scratch + (long long)b * kMedianScratch;
  hist[threadIdx.x] = 0;
  __syncthreads();
  const long long hw = (long long)H * W, n2 = 2 * hw;
  const float* p = pts + (long long)b * hw * 3;
  const int shift = 24 - 8 * pass;
  const uint32_t prefix = (uint32_t)sc[256];
  if (sc[259] >= 0) {   // state < 0: no finite-or-infinite vote at all (every vote NaN) -> result NaN, nothing to count
    for (long long j = blockIdx.x * 256LL + threadIdx.x; j < n2; j += 256LL * kMedianBlocks) {
      const float f = focal::vote(p, j, hw, W, ppx, ppy);
      if (f != f) continue;
      const uint32_t key = focal::order_key(f);
      if (pass > 0 && (key >> (shift + 8)) != prefix) continue;
      atomicAdd(&hist[(key >> shift) & 255], 1);
    }
  }
  __syncthreads();
  if (hist[threadIdx.x]) atomicAdd(&sc[threadIdx.x], hist[threadIdx.x]);
}

__global__ void __launch_bounds__(32) focal_median_pick_kernel(int* __restrict__ scratch, int pass, float lo, float hi,
                                                               float* __restrict__ focal) {
  if (threadIdx.x != 0) return;
  const int b = blockIdx.x;
  int* sc = scratch + (long long)b * kMedianScratch;
  if (sc[259] >= 0) {
    long long k = ((long long)(uint32_t)sc[258] << 32) | (uint32_t)sc[257];
    if (pass == 0) {
      long long n = 0;
      for (int i = 0; i < 256; ++i) n += sc[i];
      if (n == 0) sc[259] = -1;
      k = (n - 1) / 2;
    }
    if (sc[259] >= 0) {
      const int bin = focal::radix_pick(sc, k);
      sc[256] = (int)((((uint32_t)sc[256]) << 8) | (uint32_t)bin);
      sc[257] = (int)(uint32_t)(k & 0xffffffffll);
      sc[258] = (int)(uint32_t)(k >> 32);
    }
  }
  for (int i = 0; i < 256; ++i) sc[i] = 0;
  if (pass == 3) {
    float f = sc[259] >= 0 ? focal::key_value((uint32_t)sc[256]) : nanf("");
    f = fminf(fmaxf(f, lo), hi);   // focal.clip(min, max): NaN stays NaN (fmaxf / fminf return the non-NaN operand, so
    if (sc[259] < 0) f = nanf("");  // restore it explicitly)
    focal[b] = f;
  }
}

}  // namespace s3r

using namespace s3r;

extern "C" {

int s3r_focal_weiszfeld(const float* pts3d, int B, int H, int W, float ppx, float ppy, int iters, float lo, float hi,
                        float* scratch, float* focal, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (B <= 0 || H <= 0 || W <= 0 || iters < 0) {
    set_error("focal_weiszfeld: bad arguments");
    return -1;
  }
  for (int it = 0; it <= iters; ++it) {
    launch_pdl(focal_partial_kernel, dim3(kFocalBlocks, B), dim3(256), 0, st, pts3d, H, W, ppx, ppy, (const float*)focal,
               it == 0 ? 1 : 0, scratch);
    launch_pdl(focal_final_kernel, dim3(B), dim3(256), 0, st, (const float*)scratch, lo, hi, it == iters ? 1 : 0, focal);
  }
  return cudaGetLastError() == cudaSuccess ? 0 : -6;
}

int s3r_focal_median(const float* pts3d, int B, int H, int W, float ppx, float ppy, float lo, float hi, int32_t* scratch,
                     float* focal, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!pts3d || !scratch || !focal || B <= 0 || H <= 0 || W <= 0) {
    set_error("focal_median: bad arguments");
    return -1;
  }
  cudaMemsetAsync(scratch, 0, sizeof(int) * (size_t)B * kMedianScratch, st);
  for (int pass = 0; pass < 4; ++pass) {
    focal_median_hist_kernel<<<dim3(kMedianBlocks, B), 256, 0, st>>>(pts3d, H, W, ppx, ppy, pass, scratch);
    focal_median_pick_kernel<<<B, 32, 0, st>>>(scratch, pass, lo, hi, focal);
  }
  return cudaGetLastError() == cudaSuccess ? 0 : -6;
}

}  // extern "C"
