// Launchers of the non-GEMM kernels (definitions in elementwise.cu, attention.cu, memory.cu).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "gemm.cuh"
#include <cuda.h>

struct s3r_loss_desc;   // include/spann3r_b200.h
struct s3r_attn_train_desc;

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
// training-mode dropout of the memory read: out[i] = keep-scale (0 or 1 / (1 - p)) of flat element i under `seed`
int launch_dropout_mask(float* out, long long n, unsigned long long seed, float p, cudaStream_t st);
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
int launch_conf_score_batched(const float* conf, int batch, long long hw, float* scratch, float* out, cudaStream_t st);

// reconstruction metrics (pointcloud.cu): spatial index, 1-NN, k-NN normals, point-to-point ICP, vector statistics
size_t pcl_index_bytes(long long n);
int launch_pcl_index_build(const void* pts, int f64, long long n, const double* T, void* index, cudaStream_t st);
int launch_pcl_nearest(const void* index, long long n, const void* q, int f64, long long nq, const double* T,
                       double max_dist, double* dist, long long* idx, cudaStream_t st);
int launch_pcl_normals(const void* index, long long n, int k, double* normals, cudaStream_t st);
size_t pcl_icp_workspace_bytes();
int launch_pcl_icp(const void* src, int f64, long long ns, const void* target_index, long long nt, double max_corr,
                   const double* init, int max_iteration, double rel_fitness, double rel_rmse, void* workspace,
                   double* out, cudaStream_t st);
size_t pcl_stats_workspace_bytes();
int launch_pcl_stats(const double* v, long long n, double threshold, void* workspace, double* out, cudaStream_t st);
int launch_pcl_abs_dot(const double* a, const double* b, const long long* idx, long long n, double* out, cudaStream_t st);

// headless point rendering (render.cu): z-buffer of w * h uint64 keys, clear / splat one frame / resolve to RGB
size_t render_workspace_bytes(int w, int h);
int launch_render_clear(void* keys, int w, int h, cudaStream_t st);
int launch_render_splat(const float* pts, const uint8_t* mask, long long n, long long id0, const double* camera,
                        double z_near, int w, int h, void* keys, cudaStream_t st);
int launch_render_resolve(const void* keys, const float* colors, int w, int h, uint8_t* out, cudaStream_t st);

// triangle meshes (mesh.cu): app.py's pixel-grid faces (count + scan, then ordered writes) and the triangle rasteriser
// into the render key buffer, with its depth / face resolve
size_t mesh_grid_workspace_bytes(int T, int H, int W);
int launch_mesh_grid_count(const uint8_t* valid, int T, int H, int W, void* workspace, size_t workspace_bytes,
                           long long* n_faces, cudaStream_t st);
int launch_mesh_grid_faces(const uint8_t* valid, const float* images, int T, int H, int W, const void* workspace,
                           size_t workspace_bytes, int* faces, float* colors, cudaStream_t st);
int launch_raster_triangles(const float* verts, long long n_verts, const int* faces, long long n_faces, long long id0,
                            const double* camera, double z_near, double z_far, int w, int h, void* keys,
                            cudaStream_t st);
int launch_raster_resolve(const void* keys, int w, int h, float* depth, int* face, cudaStream_t st);

// conv backward (conv_wgrad.cu): weight gradient over pixels (split-bf16 wgmma, split contraction + fixed-order reduce)
// and the col2im of the 3x3 stride-2 conv; both validate their arguments before any CUDA call
size_t conv_wgrad_workspace_bytes(int NB, int H, int W, int N, int Kc, int taps);
int launch_conv_wgrad(const __nv_bfloat16* dy_hi, const __nv_bfloat16* dy_lo, long long ldy, const __nv_bfloat16* x_hi,
                      const __nv_bfloat16* x_lo, long long ldx, int NB, int H, int W, int N, int Kc, int taps,
                      void* workspace, size_t workspace_bytes, float* dw, cudaStream_t st);
int launch_col2im_3x3s2(const float* cols, int NB, int H, int W, int C, int Ho, int Wo, float* out, cudaStream_t st);

// training / test criteria (loss.cu): validate the descriptor before any CUDA call
size_t loss_workspace_bytes(const s3r_loss_desc* d);
int launch_loss_forward(const s3r_loss_desc* d, void* ws, size_t ws_bytes, float* gt_out, float* pred_out,
                        uint8_t* valid_out, double* results, cudaStream_t st);
int launch_loss_backward(const s3r_loss_desc* d, const void* ws, size_t ws_bytes, const float* upstream,
                         float* grad_pred, float* grad_conf, cudaStream_t st);

// attention of the training backward (attention_train.cu): split-bf16 flash forward / backward; validate before any
// CUDA call
size_t attn_train_workspace_bytes(const s3r_attn_train_desc* d);
int launch_attn_train_forward(const s3r_attn_train_desc* d, float* o, float* lse, cudaStream_t st);
int launch_attn_train_backward(const s3r_attn_train_desc* d, const float* o, const float* lse, const float* d_o,
                               void* workspace, size_t workspace_bytes, float* dq, float* dk, float* dv, cudaStream_t st);

}  // namespace s3r
