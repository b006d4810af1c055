// Host interfaces that one .cu file defines and another calls: the launchers and launch plans the engine (engine.cu)
// and the Poisson reconstruction (poisson.cu) share with the files that hold their kernels.  The public entry points are
// declared in include/spann3r_b200.h and defined beside their kernels.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "gemm.cuh"
#include <cuda.h>

namespace s3r {

int launch_split(const float* x, long long ldx, __nv_bfloat16* hi, __nv_bfloat16* lo, long long ldp, int col0,
                 long long rows, int C, int relu, cudaStream_t st);
// fp32 rows -> planes + per-32-column (sum, sum of squares) in the GEMM producer's stats_out layout (+ optional fp32 copy)
int launch_split_stats(const float* x, long long ldx, long long rows, int C, float* out, long long ldo, __nv_bfloat16* hi,
                       __nv_bfloat16* lo, long long ldp, float2* stats, cudaStream_t st);
int launch_layernorm(const float* x, long long ldx, const float* w, const float* b, long long wb_group_stride,
                     long long rows_per_group, float eps, long long rows, int C, float* out, long long ldo,
                     __nv_bfloat16* hi, __nv_bfloat16* lo, long long ldp, int col0, long long swap_rows,
                     cudaStream_t st);
int launch_im2col_patch16(const float* img, long long sb, long long sc, long long sy, long long sx, int B, int gh,
                          int gw, __nv_bfloat16* hi, __nv_bfloat16* lo, cudaStream_t st);
int launch_im2col_3x3s2(const __nv_bfloat16* ihi, const __nv_bfloat16* ilo, int NB, int H, int W, int C, int Ho, int Wo,
                        __nv_bfloat16* ohi, __nv_bfloat16* olo, cudaStream_t st);
// (Ho, Wo) = output size, <= (2H, 2W) (cropped), 0 = exactly 2x
int launch_upsample2x(const float* x, int NB, int H, int W, int C, float* out, __nv_bfloat16* hi, __nv_bfloat16* lo,
                      cudaStream_t st, int Ho = 0, int Wo = 0);

struct AttnArgs {
  alignas(64) CUtensorMap tmQ;   // (64, nq, BH)  box (32,128,1)
  alignas(64) CUtensorMap tmK;   // (64, nk, BH)  box (32,128,1)
  alignas(64) CUtensorMap tmV;   // (nk, 64, BH)  box (32, 64,1), row stride nk_pad
  int nq, nk, heads;
  __nv_bfloat16* o_hi;
  __nv_bfloat16* o_lo;
  float* o_f32;
  long long ldo;
};
// One launch of the fused attention core (attention.cu): the arguments of s3r_attention (include/spann3r_b200.h)
struct AttnDesc {
  const float *q, *k, *vt;
  int bh, heads, nq, nk, nk_pad;
  __nv_bfloat16 *o_hi, *o_lo;
  float* o_f32;
  long long ldo;
};
struct AttnPlan {
  AttnArgs args;
  dim3 grid;
  double flops;
};
// Checks every rule of s3r_attention before any CUDA call, then encodes the three tensor maps and fills the arguments,
// outputs included; nq, nk or bh <= 0 leaves an empty plan.  Returns 0 or a negative error, last_error() naming the field.
int attn_plan(const AttnDesc& d, AttnPlan* plan);
// Launches the plan as it is (an empty one: nothing), without validation or tensor-map encoding.
int attn_launch(const AttnPlan& plan, cudaStream_t st);

// spatial memory (memory.cu)
// longest bank the softmax takes: one fp32 score row in shared memory, up to 200 KB of it
constexpr int MEM_SOFTMAX_MAX_LEN = 200 * 1024 / 4;
// One int per batch item ("slot") of a memory stage, passed by value as a launch parameter: n == 1 holds one value for
// every slot (any batch size), otherwise v[b] is slot b's (b < MEM_MAX_SLOTS == S3R_MAX_SLOTS).
constexpr int MEM_MAX_SLOTS = 64;
struct SlotInts {
  int n;
  int v[MEM_MAX_SLOTS];
  __host__ __device__ int operator[](int b) const { return v[n == 1 ? 0 : b]; }
};
inline SlotInts slot_uniform(int x) { SlotInts s{}; s.n = 1; s.v[0] = x; return s; }
// rows = slots * nq; row r belongs to slot r / nq and has lens[r / nq] scores; Mpad (multiple of 8) >= every length
int launch_mem_softmax(const float* S, long long ldS, long long rows, int nq, const SlotInts& lens, int Mmax, int Mpad,
                       float scale, float thresh, __nv_bfloat16* phi, __nv_bfloat16* plo, long long ldP, cudaStream_t st,
                       float drop_p = 0.f, unsigned long long seed = 0);
// part: scratch of B * ceil(nq/32) rows of ld_part floats (ld_part >= Mmax rounded up to 8); slot b adds columns < lens[b]
int launch_mem_colsum(const __nv_bfloat16* phi, const __nv_bfloat16* plo, long long ldP, int B, int nq, const SlotInts& lens,
                      int Mmax, float* mem_attn, long long ld_attn, float* part, long long ld_part, cudaStream_t st);
// slot b (on[b] != 0) is written at columns col0[b] + t
int launch_split_transpose(const float* x, int B, int T, int C, __nv_bfloat16* ohi, __nv_bfloat16* olo, long long ldo,
                           long long out_batch_stride, const SlotInts& col0, const SlotInts& on, cudaStream_t st);
// slot b compares with wm[b] frames of P tokens starting at token start[b] of its k rows; out[b * ldo + t], t < ldo,
// is -inf for t >= wm[b]
int launch_check_sim(const float* feat, const float* k, long long k_batch_stride, int B, const SlotInts& start,
                     const SlotInts& wm, int P, int C, float* scratch, float* out, int ldo, cudaStream_t st);

// radix select and sort (pointcloud.cu), also run by the Poisson reconstruction (poisson.cu)
// order statistics of ranks r0, r1 of non-negative fp64 values, exact; *picked <- device pointer to the two values
// inside the workspace (s3r_pcl_stats_workspace_bytes())
int launch_pcl_select_ranks(const double* v, long long n, long long r0, long long r1, void* workspace,
                            const double** picked, cudaStream_t st);
// stable LSD radix sort of (key, value) over `passes` 8-bit digits, ping-ponging keys[0] <-> keys[1] (the result is in
// keys[passes & 1]); hist: pcl_sort_hist_words(n) unsigned words
long long pcl_sort_hist_words(long long n);
int launch_pcl_radix_sort(uint64_t* const keys[2], int* const vals[2], long long n, int passes, unsigned* hist,
                          cudaStream_t st);

}  // namespace s3r
