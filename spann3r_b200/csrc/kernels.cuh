// Launchers of the non-GEMM kernels (definitions in elementwise.cu, attention.cu, memory.cu).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "gemm.cuh"
#include <cuda.h>

namespace s3r {

int launch_split(const float* x, long long ldx, __nv_bfloat16* hi, __nv_bfloat16* lo, long long ldp, int col0,
                 long long rows, int C, int relu, cudaStream_t st);
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
int launch_rope2d(float* tokens, const long long* pos, long long BN, int H, int D, long long stride_tok,
                  long long stride_head, float base, float fwd, cudaStream_t st);

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
struct AttnPlan {
  AttnArgs args;
  dim3 grid;
  double flops;
};
int attn_plan_init(AttnPlan* plan, const float* q, const float* k, const float* vt, int BH, int heads, int nq, int nk,
                   int nk_pad);
int attn_launch(const AttnPlan& plan, __nv_bfloat16* o_hi, __nv_bfloat16* o_lo, float* o_f32, long long ldo,
                cudaStream_t st);

// spatial memory (memory.cu)
int launch_mem_softmax(const float* S, long long ldS, long long rows, int M, int Mpad, float scale, float thresh,
                       __nv_bfloat16* phi, __nv_bfloat16* plo, long long ldP, cudaStream_t st, float drop_p = 0.f,
                       unsigned long long seed = 0);
// training-mode dropout of the memory read: out[i] = keep-scale (0 or 1 / (1 - p)) of flat element i under `seed`
int launch_dropout_mask(float* out, long long n, unsigned long long seed, float p, cudaStream_t st);
// part: scratch of B * ceil(nq/32) rows of ld_part floats (ld_part >= M rounded up to 8)
int launch_mem_colsum(const __nv_bfloat16* phi, const __nv_bfloat16* plo, long long ldP, int B, int nq, int M,
                      float* mem_attn, long long ld_attn, float* part, long long ld_part, cudaStream_t st);
int launch_split_transpose(const float* x, int B, int T, int C, __nv_bfloat16* ohi, __nv_bfloat16* olo, long long ldo,
                           long long out_batch_stride, int col0, cudaStream_t st);
int launch_check_sim(const float* feat, const float* wm, long long wm_batch_stride, int B, int T, int P, int C,
                     float* scratch, float* out, cudaStream_t st);

// input adapter (preprocess.cu): Pillow's 8-bit Lanczos resample passes, crops folded in
int launch_resample_h_u8(const uint8_t* src, long long row_stride, int rows, int out_cols, const int* bounds,
                         const int* kk, int ksize, int max_span, uint8_t* dst, cudaStream_t st);
int launch_resample_v_u8_norm(const uint8_t* tmp, int cols, int out_rows, const int* bounds, const int* kk, int ksize,
                              float* dst, cudaStream_t st);

// post-path geometry (geometry.cu): scratch = B * 148 * 2 floats
int launch_focal_weiszfeld(const float* pts3d, int B, int H, int W, float ppx, float ppy, int iters, float lo, float hi,
                           float* scratch, float* focal, cudaStream_t st);

// post-path geometry (pnp.cu): batched P3P-RANSAC + Gauss-Newton camera pose from a pointmap (cv2.solvePnPRansac of demo.py)
size_t pnp_workspace_bytes(int B, int n_samples);
int launch_pnp_ransac(const float* pts3d, const float* img_pts, int B, long long n, int width, double fx, double fy,
                      double cx, double cy, float reproj_err, int n_samples, int refine_iters, unsigned long long seed,
                      void* workspace, double* out, unsigned char* inlier_mask, cudaStream_t st);

// focal_mode='median' of the same reference function: exact radix select; scratch = B * 260 int32
int launch_focal_median(const float* pts3d, int B, int H, int W, float ppx, float ppy, float lo, float hi, int* scratch,
                        float* focal, cudaStream_t st);

int launch_conf_score(const float* conf, long long n, float* scratch256, float* out, cudaStream_t st);

// fused attention (attention.cu): O = softmax(Q K^T) V per (batch*head), tf32 wgmma, split-bf16 output
int launch_attention(const float* q, const float* k, const float* vt, int BH, int heads, int nq, int nk, int nk_pad,
                     __nv_bfloat16* o_hi, __nv_bfloat16* o_lo, float* o_f32, long long ldo, cudaStream_t st);

}  // namespace s3r
