/* spann3r_b200 -- C ABI of the H100-native (sm_90a) Spann3R forward path (libspann3r_b200.so).
 *
 * The reference (HengyiWang/spann3r) is Python over PyTorch; its only native boundary is the
 * pybind module `curope` (croco/models/curope/curope.cpp:49-69).  This header is the boundary a
 * maintainer binds instead: flat extern "C" entry points, device pointers + sizes, an explicit
 * cudaStream_t (as void*), int status returns (0 = ok, < 0 = error, text via s3r_last_error()).
 * No torch types, no exceptions, no host synchronisation inside any call, nothing allocated that
 * the caller must free except the opaque engine handle.
 *
 * Number format.  Every weight GEMM / convolution on the path consumes fp32 values carried as two
 * bf16 planes (hi = bf16(x), lo = bf16(x - hi)) and issues three wgmma tensor-core MMAs per product
 * (DESIGN.md section 3).  "planes" below always means such a (hi, lo) pair of identical layout.
 * Opt-in bf16 precision (s3r_gemm_desc.precision = 1, s3r_engine_create_ex): a GEMM multiplies the hi planes only,
 * one MMA per product; producers still write both planes.
 *
 * Each entry point cites the reference code it replaces (paths relative to the reference root).
 */
#ifndef SPANN3R_B200_H_
#define SPANN3R_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define S3R_VERSION 100

/* epilogue modes of s3r_gemm */
enum { S3R_EPI_PLAIN = 0, S3R_EPI_PIXSHUF = 1, S3R_EPI_QKV = 2, S3R_EPI_HEADTAIL = 3 };
enum { S3R_ACT_NONE = 0, S3R_ACT_GELU = 1, S3R_ACT_RELU = 2 };

int s3r_version(void);
/* sizeof(s3r_gemm_desc / s3r_model_w / s3r_bank / s3r_loss_desc / s3r_attn_train_desc) as compiled: bindings check their
 * mirrors against these */
int s3r_abi_sizeof(int which /* 0 gemm_desc, 1 model_w, 2 bank, 3 loss_desc, 4 attn_train_desc */);
/* last error text of the calling thread ("" if none) */
const char* s3r_last_error(void);
/* 1 if a CUDA device of compute capability 9.0 (H100, sm_90a) is visible, else 0 (never falls back to CPU) */
int s3r_device_ok(void);

/* ---- op level ------------------------------------------------------------------------------ */

/* fp32 [rows, c] (row stride ldx) -> planes [rows, ldp] at column col0, optional ReLU first.
 * c, ldx, ldp and col0 are multiples of 4 (16-byte loads, 8-byte stores).
 * Replaces nothing in the reference; it is the format conversion at the head of a GEMM chain. */
int s3r_split(const float* x, int64_t ldx, void* hi, void* lo, int64_t ldp, int col0, int64_t rows, int c, int relu,
              void* stream);

/* nn.LayerNorm over the last dim (c = 768 or 1024), fp32 and/or planes out.
 * croco/models/blocks.py:116-130,176-191 (norm1/2/3/norm_y, eps 1e-6), dust3r/model.py:151,203
 * (enc_norm, dec_norm), spann3r/model.py:245-247 (norm_q/k/v, eps 1e-5).
 * Groups: row r uses weight set (r / rows_per_group) at w + set*wb_group_stride (0 = one set).
 * swap_rows > 0: two groups of swap_rows rows (rows == 2 * swap_rows, rows_per_group == swap_rows); output rows
 * and weight sets are exchanged between the groups (the twin decoders' norm_y, dust3r/model.py:197-199).
 * ldx, wb_group_stride, ldo (with out), ldp and col0 (with planes) are multiples of 4. */
int s3r_layernorm(const float* x, int64_t ldx, const float* w, const float* b, int64_t wb_group_stride,
                  int64_t rows_per_group, float eps, int64_t rows, int c, float* out, int64_t ldo, void* hi, void* lo,
                  int64_t ldp, int col0, int64_t swap_rows, void* stream);

/* In-place 2-D RoPE, drop-in for curope.rope_2d(tokens[B,N,H,D], pos[B,N,2] int64, base, fwd)
 * (croco/models/curope/curope.cpp:49-65, kernels.cu:18-81); fp32 tokens, D contiguous, strides in
 * elements.  Unlike the reference kernel it runs on the given stream, not the legacy stream 0. */
int s3r_rope2d_inplace(float* tokens, const int64_t* pos, int64_t bn, int h, int d, int64_t stride_tok,
                       int64_t stride_head, float base, float fwd, void* stream);

/* Patch im2col for Conv2d(3, E, k=16, s=16): img with element strides (sb, sc, sy, sx) ->
 * planes [b*gh*gw, 768], k = c*256 + i*16 + j.  dust3r/patch_embed.py:19-29. */
int s3r_im2col_patch16(const float* img, int64_t sb, int64_t sc, int64_t sy, int64_t sx, int b, int gh, int gw,
                       void* hi, void* lo, void* stream);
/* im2col for Conv2d(C, C, 3, stride 2, pad 1): planes [nb,h,w,c] -> planes [nb*ho*wo, 9*c], c a multiple of 8.
 * croco/models/dpt_block.py:396-408 (act_4_postprocess). */
int s3r_im2col_3x3s2(const void* ihi, const void* ilo, int nb, int h, int w, int c, int ho, int wo, void* ohi,
                     void* olo, void* stream);
/* Bilinear x2, align_corners=True, channels-last fp32 [nb,h,w,c] -> fp32 and/or planes [nb,2h,2w,c].
 * croco/models/dpt_block.py:214-215, 246-253. */
int s3r_upsample2x(const float* x, int nb, int h, int w, int c, float* out, void* hi, void* lo, void* stream);

/* ---- convolution backward (training): the weight gradient of the DPT-head convolutions ---------------------------
 * dW[n, tap, c] = sum over b, y, x of dY[b, y, x, n] * X[b, y + dy(tap), x + dx(tap), c]  (fp32, split-bf16 x3 products)
 *   dy planes [nb, h, w, n] (row stride ldy elements), x planes [nb, h, w, kc] (row stride ldx), device pointers,
 *   16-byte aligned; n, kc, ldy, ldx multiples of 8.  taps = 1 (no shift: 1x1 convs, and ConvTranspose / patch /
 *   stride-2 wgrads over re-laid-out operands) or 9 (3x3 stride 1 pad 1, tap = 3 (dy + 1) + (dx + 1); reads outside the
 *   image are zero).  dw fp32 [n, taps, kc] = the packed-weight layout, i.e. the gradient of a Conv2d weight [n, kc, 3, 3]
 *   permuted (0, 2, 3, 1).  workspace: s3r_conv_wgrad_workspace_bytes(...) bytes (0 = unsupported shape) of caller-owned
 *   device memory for the per-CTA partials, summed in a fixed order: two calls on the same inputs give bitwise-identical dw.
 *   Backward of croco/models/dpt_block.py (every Conv2d / ConvTranspose2d), dust3r/patch_embed.py:19-29 and
 *   spann3r/model.py:310 (pos_patch_embed). */
size_t s3r_conv_wgrad_workspace_bytes(int nb, int h, int w, int n, int kc, int taps);
int s3r_conv_wgrad(const void* dy_hi, const void* dy_lo, int64_t ldy, const void* x_hi, const void* x_lo, int64_t ldx,
                   int nb, int h, int w, int n, int kc, int taps, void* workspace, size_t workspace_bytes, float* dw,
                   void* stream);
/* Adjoint of s3r_im2col_3x3s2 in fp32: cols [nb*ho*wo, 9*c] (k = tap*c + channel) -> out [nb, h, w, c], each input pixel
 * the sum of the (at most 4) taps that read it, in tap order (deterministic).  c a multiple of 8, ho = (h+1)/2,
 * wo = (w+1)/2.  The input gradient of the stride-2 conv of croco/models/dpt_block.py:396-408 (act_4_postprocess). */
int s3r_col2im_3x3s2(const float* cols, int nb, int h, int w, int c, int ho, int wo, float* out, void* stream);

/* The tensor-core workhorse: D = A * B^T with fused epilogue (see EPI modes).
 *   A planes [groups*nb, h, w, kc] (a linear layer is h = 1, w = rows), B planes [groups*n, taps, kc],
 *   taps = 1 (linear / 1x1 conv / ConvTranspose with kernel == stride) or 9 (3x3, stride 1, pad 1).
 * Replaces nn.Linear / Conv2d / ConvTranspose2d calls of croco/models/blocks.py:73-79,94-112,149-169,
 * dust3r/model.py:189-190, spann3r/model.py:250-261,310 and croco/models/dpt_block.py (all convs).
 * n is a multiple of 32 (the epilogue stores whole 32-column chunks), except in an S3R_EPI_PLAIN launch whose only
 * output is out_f32, without residuals, with ldo >= n rounded up to 32 (the memory read's scores): there columns n ..
 * of the last chunk are written too, with unspecified values.  ldr1, ldr2, ldo, ldp and plane_col0 are
 * non-negative multiples of 4 below 2^31 (16-byte residual / fp32 accesses, 8-byte plane stores); res1 may be
 * out_f32 with ldr1 == ldo (in-place residual, as the engine's proj / cproj / fc2 launches).  Every rule is
 * checked before the driver is touched: a rejected descriptor returns -1 and names the field in s3r_last_error().
 * force_bn: 0 = the planner's tile width, or 64, 96 or 128; S3R_EPI_HEADTAIL always runs 128 wide. */
typedef struct s3r_gemm_desc {
  const void* a_hi; const void* a_lo;
  const void* b_hi; const void* b_lo;
  int groups, nb, h, w, kc, taps, n;
  int epi, act, plane_relu, force_bn;
  const float* bias;                       /* [groups*n] (PIXSHUF: [groups*ps_cout]) or NULL */
  const float* res1; int64_t ldr1;         /* optional residual adds, indexed like out_f32 */
  const float* res2; int64_t ldr2;
  float* out_f32; int64_t ldo;             /* optional fp32 output [groups*rows, ldo] */
  void* out_hi; void* out_lo; int64_t ldp; int plane_col0;   /* optional planes output */
  /* S3R_EPI_PIXSHUF: ConvTranspose2d(kernel == stride == ps_s), n = ps_s*ps_s*ps_cout, col = (i, j, co) */
  int ps_s, ps_cout;
  /* S3R_EPI_QKV: columns are q_c-wide roles starting at q_role_base (0 q, 1 k, 2 v); q,k get 2-D RoPE
   * from q_pos ([groups*rows, 2] int32 (y, x)) and the (cos, sin) table q_cs [maxpos, 16, 2]; q is scaled by
   * q_scale; outputs q_out/k_out [groups*q_nb, heads, q_ntok, 64], vt_out [groups*q_nb, heads, 64, q_ntok_pad],
   * all rounded to tf32.  n is a multiple of q_c with q_role_base + n/q_c <= 5, and the output of every role the
   * columns reach is non-NULL; q_ntok <= q_ntok_pad, a multiple of 4 (columns q_ntok.. of V^T are left untouched);
   * q_rope needs q_pos and q_cs.  Under a_swap the positions of a row follow its A operand: columns >= swap_col0 of
   * group g are rotated by the positions of group groups-1-g (the other stream's tokens, as the cross-attention k).
   * croco/models/blocks.py:97-104,154-160 + models/pos_embed.py:112-159. */
  int q_c, q_role_base, q_ntok, q_ntok_pad, q_rope, q_nb;
  const int32_t* q_pos; const float* q_cs;
  float* q_out; float* k_out; float* vt_out; float q_scale;
  /* S3R_EPI_HEADTAIL (n == 128): ReLU -> Conv2d(128, 4, 1) (ht_w [groups,4,128], ht_b [groups,4]) ->
   * postprocess: pts3d = xyz/|xyz| * expm1(|xyz|), conf = 1 + exp(x3).
   * croco/models/dpt_block.py:318-324, dust3r/heads/postprocess.py:10-58. */
  const float* ht_w; const float* ht_b; float* ht_pts; float* ht_conf;
  /* Folded LayerNorm (croco/models/blocks.py:127-130,186-191: every Linear that follows a LayerNorm).  Consumer:
   * A = planes of the RAW residual stream x, B = planes of W diag(gamma), bias = b + W beta, ln_cs [groups*n] = row
   * sums of the B planes (hi + lo), ln_stats [A rows, ln_np] float2 (sum, sum of squares) per 32-column chunk of x
   * (ln_np = kc/32, even and <= 32: kc % 64 == 0, kc <= 1024, taps == 1); the epilogue applies
   * rstd_r * (acc - mean_r * ln_cs[col]) + bias = LN(x) W^T + b.  The variance is E[x^2] - mean^2 in fp32 from these
   * one-pass sums, and the GEMM runs on the raw x, so the error grows with |mean_r| / std_r: rows up to 3 are held to
   * the GEMM's 3e-5 relative error (tests/test_epilogue_gpu.py); every folded LayerNorm input of the model stays
   * below 0.11 (both synthetic checkpoints).
   * a_swap = 1: group g reads A rows / statistics of group groups-1-g (norm_y of the twin decoders,
   * dust3r/model.py:197-199).  Producer (EPI_PLAIN, n % 32 == 0): stats_out [rows, n/32] float2 receives the chunk
   * sums of the rows it writes.  All NULL / 0 = plain GEMM. */
  const float* ln_stats; int ln_np; float ln_eps; const float* ln_cs; int a_swap;
  float* stats_out;
  /* diagnostics: %globaltimer stamps of CTA 0 in slots 0..6 of a 16 x uint64 buffer (entry, prologue done, dependency
   * wait done, first operands landed, accumulator ready, epilogue done, exit; tools/trace_gemm.py); NULL = off. */
  uint64_t* trace;
  /* merged projections: a_swap applies to output columns >= swap_col0 only (0 = all; a multiple of 256), and EPI_QKV
   * roles 3 / 4 (columns 3*q_c .. 5*q_c) are a second K / V^T pair written to k2_out / vt2_out -- the decoder's
   * self-attention qkv and cross-attention k, v projections (croco/models/blocks.py:186-189) as ONE launch */
  int swap_col0; float* k2_out; float* vt2_out;
  /* 0: split bf16, three MMAs per product (hi*lo + lo*hi + hi*hi), fp32-grade.  1: bf16, one MMA (hi*hi) with fp32
   * accumulation; a_lo and b_lo are not read and may be NULL, and a folded LayerNorm's ln_cs must then be the row sums of
   * the hi plane alone (s3r_lin.cs_hi); S3R_EPI_HEADTAIL is split only.  Any other value is rejected. */
  int precision;
  /* operand layout: lda / ldb are the row strides (elements) of an A pixel / a B row, non-negative multiples of 8
   * (0 = dense: kc resp. taps*kc); b_group_rows (>= 0, 0 = n) is the number of B rows between consecutive groups.
   * b_static = 1: B is never written by the work this launch depends on (packed weights), so the kernel may stage its
   * first B tiles before the programmatic-dependent-launch wait; 0 = B is loaded after the wait. */
  int64_t lda, ldb, b_group_rows;
  int b_static;
} s3r_gemm_desc;
int s3r_gemm(const s3r_gemm_desc* d, void* stream);
/* tile width the planner would pick (64/96/128), for tests */
int s3r_gemm_tile_n(const s3r_gemm_desc* d);
/* the planner's rule alone, without a descriptor or a device: the tile width for m_tiles 128-row tiles x n columns on
 * sms SMs, never straddling column col_align (a_swap's swap_col0; 0 = none); force_bn as in s3r_gemm_desc.  -1 = rejected. */
int s3r_gemm_plan_bn(int64_t m_tiles, int n, int sms, int col_align, int force_bn);

/* Fused multi-head attention core, head dim 64: O = softmax(Q K^T) V per (batch*head) on tf32 wgmma.
 *   q [bh, nq, 64], k [bh, nk, 64] (already RoPE'd / scaled by the QKV epilogue), vt [bh, 64, nk_pad];
 *   output [b*nq, heads*64] as planes (o_hi and o_lo both, or neither) and/or fp32, row stride ldo: even and
 *   >= heads*64; bh a multiple of heads and <= 65535; nk_pad >= nk, a multiple of 4: columns nk .. nk_pad-1 of vt are
 *   never read.  q, k, vt 16-byte aligned, o_f32 8-byte, o_hi / o_lo 4-byte.  Every rule is checked before any CUDA
 *   call (-1, last error naming the field); then nq, nk or bh <= 0 returns 0 and launches nothing.
 * croco/models/blocks.py:106-110 (self), :162-166 (cross). */
int s3r_attention(const float* q, const float* k, const float* vt, int bh, int heads, int nq, int nk, int nk_pad,
                  void* o_hi, void* o_lo, float* o_f32, int64_t ldo, void* stream);

/* Offline-mode view score: out[0] = mean((conf-1)/conf) over n values (spann3r/model.py:346-352, 372-381);
 * scratch256 = 256 floats of device scratch.  Deterministic. */
int s3r_conf_score(const float* conf, int64_t n, float* scratch256, float* out, void* stream);
/* The same score for every image of the engine's confidence output conf [2, batch, H, W] (hw = H * W):
 * out[i] = s3r_conf_score of image i (i = head * batch + b), bitwise, in one launch pair.
 * scratch = 2 * batch * 256 floats of device scratch.  1 <= batch <= 32767, hw >= 1, non-null pointers. */
int s3r_conf_score_batched(const float* conf, int batch, int64_t hw, float* scratch, float* out, void* stream);

/* ---- input adapter (SURVEY.md section 8f rank 3): the reference's CPU preprocessing in front of the path -----------
 * spann3r/datasets/demo.py:57-86 -> dust3r/datasets/base/base_stereo_view_dataset.py:143-194 (centre crop, Lanczos
 * down-scale, centred crop) -> dust3r/utils/image.py:23 (ToTensor + Normalize).  The down-scale is Pillow's 8-bit
 * separable resampler (Resample.c), reproduced bit-exactly; the host supplies Pillow's coefficient tables:
 * bounds [n, 2] int32 (first source index, tap count) and kk [n, ksize] int32 (22-bit fixed point), already shifted so
 * that index 0 is the first row / column passed in.
 * s3r_resample_h_u8: src = RGB uint8 rows (row_stride bytes apart), `rows` rows -> dst [rows, out_cols, 3] uint8;
 *   max_span = largest number of source pixels any block of 128 consecutive output columns touches.
 * s3r_resample_v_u8_norm: tmp [*, cols, 3] uint8 -> dst [3, out_rows, cols] fp32 = ((v / 255) - 0.5) / 0.5. */
int s3r_resample_h_u8(const uint8_t* src, int64_t row_stride, int rows, int out_cols, const int32_t* bounds,
                      const int32_t* kk, int ksize, int max_span, uint8_t* dst, void* stream);
int s3r_resample_v_u8_norm(const uint8_t* tmp, int cols, int out_rows, const int32_t* bounds, const int32_t* kk, int ksize,
                           float* dst, void* stream);

/* ---- post-path geometry (SURVEY.md section 8f rank 4, first step) ---------------------------------------------------
 * dust3r/post_process.py:12-60 estimate_focal_knowing_depth(pts3d, pp, focal_mode='weiszfeld') as demo.py:148-150 calls
 * it: pts3d [b, h, w, 3] fp32 (device), principal point (ppx, ppy), `iters` re-weighting rounds (the reference: 10),
 * result clipped to [lo, hi] -> focal [b] (device).  scratch: b * 148 * 2 floats.  Deterministic. */
int s3r_focal_weiszfeld(const float* pts3d, int b, int h, int w, float ppx, float ppy, int iters, float lo, float hi,
                        float* scratch, float* focal, void* stream);

/* The same function with focal_mode='median' (its default; dust3r/post_process.py:26-36): nanmedian of the 2*h*w per-pixel
 * votes (u z / x, v z / y), i.e. an element of the vote set -- selected exactly by a 4 x 8-bit radix select on the fp32
 * votes' ordered keys, so the result is bit-identical to the reference's.  scratch: b * 260 int32.  All-NaN votes -> NaN. */
int s3r_focal_median(const float* pts3d, int b, int h, int w, float ppx, float ppy, float lo, float hi, int32_t* scratch,
                     float* focal, void* stream);

/* ---- post-path geometry, second step: camera pose from a pointmap ----------------------------------------------------
 * Replaces `cv2.solvePnPRansac(pts.reshape(-1,3), pixel grid, intrinsic, zeros(4))` of demo.py:166-180 (one CPU call per
 * frame on a host copy of the pointmap), batched over b frames and entirely on the device: P3P hypotheses from
 * n_samples minimal samples (cv2's iterationsCount; counter-based hash of `seed`), inlier counts at `reproj_err` px
 * (cv2's default 8.0) over all n points, then `refine_iters` damped Gauss-Newton rounds on the best model's inliers
 * (cv2's final SOLVEPNP_ITERATIVE refinement solves the same least-squares problem).
 *   pts3d [b, n, 3] fp32; img_pts [b, n, 2] fp32 or NULL = the dense pixel grid (u = i % width, v = i / width);
 *   out [b, 18] fp64: R (9, row-major, x_cam = R x + t), t (3), rvec (3, Rodrigues), inlier count of the RANSAC model,
 *   RMS reprojection error after refinement (px), success (1/0);  inlier_mask [b, n] uint8 (cv2's `inliers`, as a mask);
 *   workspace: s3r_pnp_workspace_bytes(b, n_samples) bytes, 16-byte aligned.  Deterministic for a given seed. */
size_t s3r_pnp_workspace_bytes(int b, int n_samples);
int s3r_pnp_ransac(const float* pts3d, const float* img_pts, int b, int64_t n, int width, double fx, double fy, double cx,
                   double cy, float reproj_err, int n_samples, int refine_iters, uint64_t seed, void* workspace,
                   double* out, uint8_t* inlier_mask, void* stream);

/* ---- reconstruction metrics: eval.py:189-218 on the device ------------------------------------------------------------
 * Open3D point-to-point ICP, 30-NN normals and spann3r/tools/eval_recon.py accuracy / completion (scipy cKDTree queries).
 * Points are [n, 3] fp32 (is_f64 = 0) or fp64 (is_f64 = 1); all arithmetic is fp64.  1 <= n < 2^31 everywhere.
 * transform: optional 3x4 row-major fp64 [R | t] on the device, applied to every input point (NULL = identity).
 *
 * Spatial index over one cloud: s3r_pcl_index_bytes(n) bytes of caller-owned device memory, 16-byte aligned (0 = n out of
 * range).  Every call that takes an index takes the n it was built with.  The index holds the (transformed) points. */
size_t s3r_pcl_index_bytes(int64_t n);
int s3r_pcl_index_build(const void* pts, int is_f64, int64_t n, const double* transform, void* index, void* stream);
/* Exact 1-NN of nq queries (optionally transformed): dist [nq] fp64 (sqrt of ((dx dx + dy dy) + dz dz), each step
 * rounded), idx [nq] int64 original index; ties -> the smallest index; nothing within max_dist (inclusive; +inf = no
 * bound) -> idx -1, dist +inf. */
int s3r_pcl_nearest(const void* index, int64_t n, const void* queries, int is_f64, int64_t nq, const double* transform,
                    double max_dist, double* dist, int64_t* idx, void* stream);
/* Normal of every indexed point: unit eigenvector of the smallest eigenvalue of the mean-centred covariance of its
 * k nearest points (itself included; 1 <= k <= 32; ties -> smaller index), sign as the solver produces it, in original
 * order -> normals [n, 3] fp64.  Fewer than 3 points or a zero covariance -> (0, 0, 1). */
int s3r_pcl_normals(const void* index, int64_t n, int k, double* normals, void* stream);
/* Point-to-point ICP of ns source points onto an indexed target, with the semantics of Open3D's registration_icp +
 * TransformationEstimationPointToPoint: pass j pairs each source point (under the current T) with its nearest target point
 * within max_correspondence_distance; stop after pass j if j >= 1 and |d fitness| < relative_fitness and |d rmse| <
 * relative_rmse, or j == max_iteration; else T <- Umeyama(correspondences) T.  No host synchronisation: 2 *
 * (max_iteration + 1) launches, later ones return at once after convergence.  init: 3x4 fp64 (device) or NULL.
 * workspace: s3r_pcl_icp_workspace_bytes() bytes, 16-byte aligned.  out (fp64, 19 + 2 * (max_iteration + 1)):
 * T of the last pass (4x4 row-major), its fitness, its inlier rmse, the number of passes, then per pass the
 * correspondence count and the inlier rmse (max_iteration + 1 slots each; unused slots 0). */
size_t s3r_pcl_icp_workspace_bytes(void);
int s3r_pcl_icp(const void* source, int is_f64, int64_t ns, const void* target_index, int64_t nt,
                double max_correspondence_distance, const double* init, int max_iteration, double relative_fitness,
                double relative_rmse, void* workspace, double* out, void* stream);
/* x [n] fp64, non-negative -> out[0] mean (fixed-order sum), out[1] exact median (np.median: the mean of the two middle
 * order statistics for even n; a -0.0 in the middle comes back as +0.0), out[2] count of x < threshold.  workspace: s3r_pcl_stats_workspace_bytes() bytes. */
size_t s3r_pcl_stats_workspace_bytes(void);
int s3r_pcl_stats(const double* x, int64_t n, double threshold, void* workspace, double* out, void* stream);
/* out[i] = |a[i] . b[idx[i]]| for a [n, 3], b [*, 3] fp64, idx [n] int64 (eval_recon.py's normal consistency). */
int s3r_pcl_abs_dot(const double* a, const double* b, const int64_t* idx, int64_t n, double* out, void* stream);

/* ---- headless point rendering: spann3r/tools/vis.py:render_frames (an Open3D window, point_size 1) ---------------------
 * A z-buffer of width * height uint64 keys in caller-owned device memory, 8-byte aligned:
 * s3r_render_workspace_bytes(width, height) bytes (0 = size out of range; width, height >= 1, width * height < 2^31).
 * s3r_render_clear empties it.  s3r_render_splat projects n fp32 points [n, 3] with global indices id0 .. id0 + n - 1
 * (id0 + n < 2^32), skipping those whose uint8 mask entry is 0 (mask NULL = keep all):
 *   camera (HOST, 16 doubles): [R | t] 3x4 row-major (world -> camera), fx, fy, cx, cy, all finite;
 *   q = R p + t in fp64 as ((R0 x + R1 y) + R2 z) + t, kept if finite and q.z > z_near (finite, >= 0);
 *   u = fx (qx / qz) + cx, v = fy (qy / qz) + cy; pixel (floor(u + 0.5), floor(v + 0.5)) if inside the image;
 *   key = bits(fp32(qz)) << 32 | index, atomicMin into the pixel: the nearest fp32 depth wins, ties -> smaller index.
 * s3r_render_resolve writes rgb [height, width, 3] uint8: black where empty, else floor(min(1, max(0, c)) * 255 + 0.5)
 * of colors[index] (fp32 [*, 3], indexed by the global point index).  Deterministic: the result does not depend on the
 * order of splat calls between two clears. */
size_t s3r_render_workspace_bytes(int width, int height);
int s3r_render_clear(void* keys, int width, int height, void* stream);
int s3r_render_splat(const float* pts, const uint8_t* mask, int64_t n, int64_t id0, const double* camera, double z_near,
                     int width, int height, void* keys, void* stream);
int s3r_render_resolve(const void* keys, const float* colors, int width, int height, uint8_t* rgb, void* stream);

/* ---- triangle meshes: app.py's pts3d_to_trimesh + cat_meshes, and a z-buffered triangle rasteriser ---------------------
 * Pixel-grid mesh of T frames of H x W pixels (T * H * W < 2^31), valid [T, H, W] uint8, images [T, H, W, 3] fp32.
 * Candidate faces in app.py's order: per frame the blocks [i1,i2,i3], [i3,i2,i1], [i2,i3,i4], [i4,i3,i2] (i1..i4 the
 * quad's top-left, top-right, bottom-left, bottom-right pixel), quads row-major inside a block, indices offset by t H W.
 * A face is kept when its three corners are valid; kept faces keep their order.  Colour: blocks 0-1 the quad's top-left
 * pixel, blocks 2-3 its bottom-right pixel.
 *   s3r_mesh_grid_workspace_bytes(T, H, W): device workspace bytes (0 = size out of range), 8-byte aligned.
 *   s3r_mesh_grid_count: per-tile counts and their scan into the workspace; *n_faces (HOST) <- the number of kept
 *     faces.  Synchronises `stream` (one device -> host read).
 *   s3r_mesh_grid_faces: with that workspace, faces [n_faces, 3] int32 and colors [n_faces, 3] fp32.
 * s3r_raster_triangles draws n_faces triangles faces [n_faces, 3] int32 (indices into verts [n_verts, 3] fp32; faces
 * with an index out of range are skipped) with face ids id0 .. id0 + n_faces - 1 (id0 + n_faces < 2^31) into the key
 * buffer of s3r_render_workspace_bytes / s3r_render_clear:
 *   camera (HOST, 16 doubles) as for s3r_render_splat; pixel centres at integer (u, v), row 0 at the top;
 *   a triangle is skipped when a vertex is not finite or has camera depth <= z_near (finite, >= 0), when it is a back
 *   face (clockwise on the image) or degenerate; a centre is covered by fp64 edge functions with a top-left rule, so a
 *   centre on an edge shared by two triangles goes to exactly one of them;
 *   depth = fp32(1 / ((b0 / z0 + b1 / z1) + b2 / z2)) with fp64 barycentrics b; depths > z_far (> z_near; inf allowed)
 *   are dropped; key = bits(depth) << 32 | face id, atomicMin: nearest depth wins, ties -> smaller face id.
 * s3r_raster_resolve writes depth [height, width] fp32 (0 where empty) and face [height, width] int32 (-1 where empty).
 * Deterministic: the result depends neither on scheduling nor on the order faces are submitted in. */
size_t s3r_mesh_grid_workspace_bytes(int T, int H, int W);
int s3r_mesh_grid_count(const uint8_t* valid, int T, int H, int W, void* workspace, size_t workspace_bytes,
                        int64_t* n_faces, void* stream);
int s3r_mesh_grid_faces(const uint8_t* valid, const float* images, int T, int H, int W, const void* workspace,
                        size_t workspace_bytes, int32_t* faces, float* colors, void* stream);
int s3r_raster_triangles(const float* verts, int64_t n_verts, const int32_t* faces, int64_t n_faces, int64_t id0,
                         const double* camera, double z_near, double z_far, int width, int height, void* keys,
                         void* stream);
int s3r_raster_resolve(const void* keys, int width, int height, float* depth, int32_t* face, void* stream);

/* ---- training / test criteria: spann3r/loss.py:129-369 (Regr3D_t, its ShiftInv / ScaleInv / ScaleShiftInv variants,
 * ConfLoss_t) with L21 (dust3r/losses.py:52-59), forward and backward --------------------------------------------------
 * F >= 2 views of B sequences of H x W pixels.  Pred slot k < F-1 is preds_all[k][0] (frame k: 'pts3d' for k = 0, else
 * 'pts3d_in_other_view'), slot F-1+i is preds_all[i][1]['pts3d_in_other_view'] (frame i+1); every map is a contiguous
 * fp32 [B, H, W, 3] (conf [B, H, W]) device tensor.  gt_pts / valid / pred / conf are HOST arrays of device pointers
 * (F, F, 2(F-1), 2(F-1) entries); the library copies them into the workspace.
 *   norm_mode 0 (False), 1 'avg_dis', 2 'avg_log1p'; gt_scale, fix_first as Regr3D_t; shift_inv / scale_inv select the
 *   variant (both = Regr3D_t_ScaleShiftInv); conf_loss = ConfLoss_t(alpha) over the criterion (needs conf), else the
 *   per-term means are summed ('mean' reduction); conf may be NULL without conf_loss (details conf_left/right then 0);
 *   has_dist_clip: valid &= |pts3d| <= dist_clip (untransformed points). */
typedef struct s3r_loss_desc {
  int frames, batch, height, width;
  int norm_mode, gt_scale, fix_first, shift_inv, scale_inv, conf_loss, has_dist_clip;
  float alpha, dist_clip;
  const float* pose0;                /* device [B, 4, 4] camera_pose of view 0 (cam-to-world) */
  const float* const* gt_pts;        /* [F] -> [B, H, W, 3] pts3d (world) */
  const uint8_t* const* valid;       /* [F] -> [B, H, W] bool valid_mask */
  const float* const* pred;          /* [2(F-1)] -> [B, H, W, 3] */
  const float* const* conf;          /* [2(F-1)] -> [B, H, W], or NULL */
} s3r_loss_desc;
/* results (fp64, device): S3R_LOSS_RES_HEADER values, then S3R_LOSS_RES_PER_B per batch element.
 * Header: loss, factor_loss, pts3d_1, pts3d_2, loss_left, loss_right, conf_left, conf_right, conf_loss_1, conf_loss2,
 * conf_mean, then the batch means of gt_shift_z, pred_shift_z, gt_scale, pred_scale (clipped), the count k of
 * pr_factor > gt_factor (-1: no factor_loss), the number of terms without a valid pixel; zeros up to the header size.
 * Per b: gt_factor (1 without), pr_factor (1 without), gt_shift_z, pred_shift_z, gt_scale, pred_scale (clipped). */
#define S3R_LOSS_RES_HEADER 20
#define S3R_LOSS_RES_PER_B 6
/* bytes of caller-owned device workspace (256-byte aligned) for one forward + its backward; 0 = invalid descriptor */
size_t s3r_loss_workspace_bytes(const s3r_loss_desc* d);
/* One criterion evaluation.  Optional outputs (NULL = not written): gt_out [F, B, H, W, 3] and pred_out [2(F-1), B, H,
 * W, 3], the aligned maps get_all_pts3d_t returns; valid_out [F, B, H, W] uint8 masks.  No host synchronisation; sums
 * in fp64 in a fixed order (bitwise reproducible); medians exact (torch.nanmedian's lower median). */
int s3r_loss_forward(const s3r_loss_desc* d, void* workspace, size_t workspace_bytes, float* gt_out, float* pred_out,
                     uint8_t* valid_out, double* results, void* stream);
/* Gradients of upstream[0] * loss + upstream[1] * factor_loss (upstream: device fp32 [2]) with respect to every pred slot
 * -> grad_pred [2(F-1), B, H, W, 3] and, with conf_loss, every conf slot -> grad_conf [2(F-1), B, H, W] (else unused).
 * The workspace is the forward's, unchanged since, with the same descriptor. */
int s3r_loss_backward(const s3r_loss_desc* d, const void* workspace, size_t workspace_bytes, const float* upstream,
                      float* grad_pred, float* grad_conf, void* stream);

/* ---- attention of the training backward: O = softmax(scale Q K^T) V and its gradients (croco/models/blocks.py:106-110,
 * 162-166 under training), split-bf16 (~fp32-accurate) with no materialised scores: the forward keeps O and one
 * log-sum-exp per row, the backward rebuilds the probabilities from it.  No float atomics: bitwise reproducible.
 *   q [batch, heads, nq, dh], k / v [batch, heads, nk, dh]: device fp32, element strides of (batch, head, token) below,
 *   non-negative multiples of 4, dh contiguous; dh 48 or 64; nq, nk >= 1 (may differ); batch * heads <= 65535. */
typedef struct s3r_attn_train_desc {
  int batch, heads, nq, nk, dh;
  float scale;                       /* softmax scale, dh^-0.5 for the model's attentions */
  const float* q;
  const float* k;
  const float* v;
  int64_t q_stride[3], k_stride[3], v_stride[3];
} s3r_attn_train_desc;
/* bytes of caller-owned device workspace s3r_attn_train_backward needs (a multiple of 256); 0 = invalid descriptor */
size_t s3r_attn_train_workspace_bytes(const s3r_attn_train_desc* d);
/* o: fp32 [batch, nq, heads * dh] (head h in columns [h dh, h dh + dh)); lse: fp32 [batch * heads, nq], the natural log
 * of each row's sum of exp(scale q.k) */
int s3r_attn_train_forward(const s3r_attn_train_desc* d, float* o, float* lse, void* stream);
/* d_o: the gradient of o, same layout; o, lse: the forward's outputs -> dq [batch, heads, nq, dh], dk / dv [batch,
 * heads, nk, dh], contiguous fp32 */
int s3r_attn_train_backward(const s3r_attn_train_desc* d, const float* o, const float* lse, const float* d_o,
                            void* workspace, size_t workspace_bytes, float* dq, float* dk, float* dv, void* stream);

/* ---- model level: the per-frame forward path -------------------------------------------------
 * Packed weights.  The host (spann3r_b200/weights.py) converts the reference state dict ONCE into
 * split-bf16 planes laid out [groups*N, taps*Kc] (K contiguous) plus fp32 biases / LayerNorm params,
 * and hands the engine a table of device pointers; the engine never sees parameter names.
 * "Grouped" entries stack two weight sets that run as one launch: the twin decoders
 * (dust3r.dec_blocks / dec_blocks2, dust3r/model.py:194-200), the two key heads (attn_head_1/2)
 * and the two DPT heads (downstream_head1/2). */
typedef struct s3r_planes { const void* hi; const void* lo; } s3r_planes;
typedef struct s3r_ln { const float* w; const float* b; } s3r_ln;      /* grouped: [G, C] contiguous */
/* b may be NULL.  cs != NULL marks a LayerNorm-folded linear: w = planes of W diag(gamma), b = b + W beta,
 * cs [G*N] = row sums of the planes (see s3r_gemm_desc.ln_cs); the preceding s3r_ln is then unused by the engine.
 * cs_hi [G*N] = row sums of the hi plane alone: what a bf16-precision GEMM's tensor core sees (required with cs by
 * engines of precision 1). */
typedef struct s3r_lin { s3r_planes w; const float* b; const float* cs; const float* cs_hi; } s3r_lin;

typedef struct s3r_block_w {       /* croco/models/blocks.py:114-130 */
  s3r_ln norm1; s3r_lin qkv; s3r_lin proj; s3r_ln norm2; s3r_lin fc1; s3r_lin fc2;
} s3r_block_w;
typedef struct s3r_decblock_w {    /* croco/models/blocks.py:171-191, two streams as 2 groups */
  /* qkv: per group [attn.qkv (norm1 folded); cross_attn.projk; cross_attn.projv (norm_y folded)], N = 5 * 768 */
  s3r_ln norm1; s3r_lin qkv; s3r_lin proj; s3r_ln norm_y; s3r_ln norm2; s3r_lin q; s3r_lin cproj;
  s3r_ln norm3; s3r_lin fc1; s3r_lin fc2;
} s3r_decblock_w;
typedef struct s3r_rcu_w { s3r_lin conv1; s3r_lin conv2; } s3r_rcu_w;                 /* dpt_block.py:121-142 */
typedef struct s3r_fusion_w { s3r_rcu_w rcu1; s3r_rcu_w rcu2; s3r_lin out_conv; } s3r_fusion_w; /* :189-218 */
typedef struct s3r_dpt_w {         /* dust3r/heads/dpt_head.py:34-65; both heads as 2 groups */
  s3r_lin act1_conv, act1_up, act2_conv, act2_up, act3_conv, act4_conv, act4_down;
  s3r_lin layer_rn[4];
  s3r_fusion_w refine[4];          /* refine[i] = scratch.refinenet{i+1} */
  s3r_lin head0, head2;
  const float* head4_w;            /* [2, 4, 128] */
  const float* head4_b;            /* [2, 4] */
} s3r_dpt_w;
typedef struct s3r_model_w {
  s3r_lin patch_embed; s3r_block_w enc[24]; s3r_ln enc_norm;
  s3r_lin decoder_embed; s3r_decblock_w dec[12]; s3r_ln dec_norm;
  s3r_lin key_fc1, key_fc2;
  s3r_dpt_w dpt;
  s3r_lin pos_patch_embed; s3r_block_w val[6]; s3r_ln value_norm; s3r_lin value_out;
  s3r_ln norm_q, norm_k, norm_v;
  const float* rope_cs;            /* [rope_maxpos, 16, 2] (cos, sin), models/pos_embed.py:120-129 */
  int rope_maxpos;
  /* Width of the value encoder (spann3r/model.py:225).  0 or 1024: the default encoder (pos_patch_embed on the pointmap,
   * 16 heads of 64).  768: Spann3R(use_feat=True), fed with head 1's last decoder tokens, 16 heads of 48; pos_patch_embed
   * is unused.  Its blocks are packed with every 48-wide head in a 64-wide slot, zeros in the padding: head h, half
   * s (y / x), in-half index i < 24 -> column 64 h + 32 s + (i < 12 ? i : 16 + (i - 12)) of q, k and v, so
   *   qkv  = planes [3 * 1024, 768] (zero rows, zero bias and cs there; norm1 folded as usual),
   *   proj = planes [768, 1024] (zero columns); fc1, fc2, value_norm, value_out are ordinary 768-wide layers.
   * A padding column of q / k / v is exactly 0, adds exactly 0 to Q K^T and to the output, so the result is the
   * 48-wide attention's. */
  int value_dim;
  /* value_dim == 768: the (cos, sin) table of the value blocks' RoPE, [rope_maxpos, 16, 2]; entry j < 12 has angle
   * pos * 100^(-j/12) (models/pos_embed.py:120-129 with D = 24), entries 12..15 are (1, 0) and rotate the zero pairs */
  const float* rope_cs_v;
} s3r_model_w;

/* The spatial-memory bank of one batch of sequences (spann3r/model.py:11-95), caller-owned buffers.
 * Keys / values are kept pre-normalised (LN_k / LN_v applied at write time) as planes for the read
 * GEMMs, plus the raw fp32 rows (similarity gate, return_memory). */
typedef struct s3r_bank {
  void* kn_hi; void* kn_lo;        /* [B, cap, 1024] */
  void* vnt_hi; void* vnt_lo;      /* [B, 1024, cap]  (transposed) */
  float* k_raw; float* v_raw;      /* [B, cap, 1024] */
  float* attn; float* count;       /* [B, cap] */
  int cap;                         /* multiple of 8 */
  int len;                         /* tokens currently stored */
} s3r_bank;

typedef struct s3r_engine s3r_engine;
/* One engine per (device, batch of sequences, image size).  Allocates its own activation workspace
 * (freed by destroy); `max_images` bounds the images one encode call may batch (>= 2*batch). */
s3r_engine* s3r_engine_create(const s3r_model_w* w, int batch, int height, int width, int max_images);
/* The same with a GEMM precision (s3r_gemm_desc.precision): 0 is s3r_engine_create.  1 runs every GEMM of encode, decode,
 * keyheads and value on one bf16 product; heads, the memory read / append / similarity gate and the attention cores keep
 * their arithmetic.  Other values: NULL, with the reason in s3r_last_error(). */
s3r_engine* s3r_engine_create_ex(const s3r_model_w* w, int batch, int height, int width, int max_images, int precision);
void s3r_engine_destroy(s3r_engine* e);
/* dust3r/model.py:131-154 _encode_image: img [nimg,3,H,W] fp32 -> feat [nimg, N, 1024] fp32 */
int s3r_engine_encode(s3r_engine* e, const float* img, int nimg, float* feat, void* stream);
/* dust3r/model.py:186-205 _decoder on (f1, f2) [B,N,1024]; hooks stay inside the engine for
 * keyheads()/heads(); dec_all (nullable) receives all 12 layer outputs [12, 2, B*N, 768] (last one normed). */
int s3r_engine_decode(s3r_engine* e, const float* f1, const float* f2, float* dec_all, void* stream);
/* spann3r/model.py:299-303 encode_feat_key for both heads: cat(feat_i, dec_i[-1]) -> [B,N,1024] */
int s3r_engine_keyheads(s3r_engine* e, const float* feat1, const float* feat2, float* k1, float* k2, void* stream);
/* dust3r/model.py:207-211 + heads/dpt_head.py + postprocess.py: pts [2,B,H,W,3], conf [2,B,H,W] */
int s3r_engine_heads(s3r_engine* e, float* pts, float* conf, void* stream);
/* spann3r/model.py:305-320 encode_cur_value, plus the `cur_v + feat_k1` of :519-521: out [B,N,1024].
 * pts3d = head 1's pointmap exactly as s3r_engine_heads wrote it ([B,H,W,3]).  flags:
 *   S3R_VALUE_PTS_TRANSPOSED  portrait frame (H > W): the reference's landscape wrapper (dust3r/utils/misc.py:66-94,
 *                             landscape_only=True at spann3r/model.py:222) gives the value encoder the map with
 *                             axes 1, 2 swapped; read it that way (patch grid W/16 x H/16), no copy
 *   S3R_VALUE_ROPE            Spann3R(mem_pos_enc=True): RoPE inside the value encoder's blocks (spann3r/model.py:231)
 *   S3R_VALUE_DEC_TOKENS      Spann3R(use_feat=True), required by and only valid on a value_dim == 768 engine
 *                             (spann3r/model.py:312-314): the first pointer is dec1[-1] = dec_norm of head 1's last
 *                             decoder layer, [B, N, 768] fp32, or NULL for the engine's own copy from its last
 *                             s3r_engine_decode.  Positions are the frame's own patch grid (no transposition: together
 *                             with S3R_VALUE_PTS_TRANSPOSED it is an error).
 * Flag / width errors are reported before any CUDA call. */
#define S3R_VALUE_PTS_TRANSPOSED 1
#define S3R_VALUE_ROPE 2
#define S3R_VALUE_DEC_TOKENS 4
int s3r_engine_value(s3r_engine* e, const float* pts3d, const float* feat_k1, int flags, float* out, void* stream);
/* spann3r/model.py:145-183 memory_read (eval: thresh = 5e-4; 0 disables): out = attn.V + feat; bank.attn += colsum */
int s3r_engine_memory_read(s3r_engine* e, const s3r_bank* bank, const float* feat, float thresh, float* out,
                           void* stream);
/* training mode of the same read (spann3r/model.py:474 `attn_thresh=0`, :167-168 `mem_dropout`): nn.Dropout(drop_p) on the
 * softmax output, before the (normally disabled) threshold.  The keep decision of element (b, row, column) is Philox4x32-10
 * of (seed, (b * N + row) * len + column): reproducible, regenerated for the backward pass / tests by s3r_dropout_mask */
int s3r_engine_memory_read_train(s3r_engine* e, const s3r_bank* bank, const float* feat, float thresh, float drop_p,
                                 uint64_t seed, float* out, void* stream);
/* out[i] = 0 or 1/(1-p): the keep-scale the training-mode read applies to flat element i = (b * N + row) * len + column */
int s3r_dropout_mask(float* out, int64_t n, uint64_t seed, float p, void* stream);
/* spann3r/model.py:80-95 add_mem: append N tokens at bank.len (caller then sets len += N) */
int s3r_engine_memory_append(s3r_engine* e, const s3r_bank* bank, const float* feat_k, const float* feat_v,
                             void* stream);
/* spann3r/model.py:97-118 check_sim: out[b, t] = mean cosine vs each of the last wm frames (device array [B, wm]) */
int s3r_engine_check_sim(s3r_engine* e, const s3r_bank* bank, const float* feat_k, int wm, float* out, void* stream);
/* Per-slot memory stages: independent sequences in one batch.  Slot b is batch item b of the engine and owns its region
 * of the bank buffers; its length is lens[b] (host array of e's batch size; bank->len is not read).  The engine's batch
 * must be at most S3R_MAX_SLOTS.  Every argument is validated before anything is launched.
 * Tail contract: in every slot, the K_n rows and V_n^T columns in [lens[b], max(lens)) must hold finite values (the
 * probabilities there are zero, and 0 * NaN is NaN on the tensor core); a zero-initialised bank whose resets and prunes
 * zero what they leave behind satisfies it. */
#define S3R_MAX_SLOTS 64
/* memory_read with per-slot lengths (eval mode: no dropout).  A slot of length 0 reads nothing: out[b] = feat[b] exactly.
 * bank.attn of slot b gains the column sums of its columns < lens[b] only.  0 <= lens[b] <= cap. */
int s3r_engine_memory_read_slots(s3r_engine* e, const s3r_bank* bank, const int* lens, const float* feat, float thresh,
                                 float* out, void* stream);
/* add_mem per slot: slot b with append[b] != 0 takes its N tokens at offset lens[b] (lens[b] + N <= cap; the caller then
 * adds N to its length); a slot with append[b] == 0 is left untouched. */
int s3r_engine_memory_append_slots(s3r_engine* e, const s3r_bank* bank, const int* lens, const int* append,
                                   const float* feat_k, const float* feat_v, void* stream);
/* check_sim per slot: out[b, t] (device array [B, 8]) = mean cosine vs frame t of the last wm[b] frames ending at lens[b]
 * (0 <= wm[b] <= 8, wm[b] * N <= lens[b]); entries t >= wm[b] are -inf, so a row's max is the slot's gate value. */
int s3r_engine_check_sim_slots(s3r_engine* e, const s3r_bank* bank, const int* lens, const int* wm, const float* feat_k,
                               float* out, void* stream);
/* algorithmic FLOPs (2*M*N*K of every tensor-core launch) issued since the last call; resets the counter */
double s3r_engine_take_flops(s3r_engine* e);
/* Per-launch CUDA-event timing of the tensor-core kernels (bench.py roofline leg): switch on, run, read.
 * profile_read synchronises the device; out = {gemm_ms, gemm_flops, gemm_launches, attn_ms, attn_flops, attn_launches} */
void s3r_engine_profile(s3r_engine* e, int on);
/* per-launch list (in launch order) of the recorded tensor-core launches: duration [ms], algorithmic FLOPs, kind
 * (0 split GEMM / conv, 1 attention, 2 one-product bf16 GEMM); returns the count (call before profile_read, which consumes
 * the records).  profile_read counts kinds 0 and 2 as GEMMs. */
int s3r_engine_profile_list(s3r_engine* e, double* ms, double* flops, int* kind, int cap);
int s3r_engine_profile_read(s3r_engine* e, double* out);
/* number of kernel launches since the last call; resets the counter */
long long s3r_engine_take_launches(s3r_engine* e);

/* ---- dataset views (spann3r_b200/views.py): the tail of BaseStereoViewDataset.__getitem__ on the device -----------
 * dust3r/datasets/base/base_stereo_view_dataset.py:63-194 (crop on the principal point, Lanczos image / nearest depth
 * rescale, centred crop, ImgNorm, depthmap_to_absolute_camera_coordinates, valid_mask, transpose_to_landscape) for a
 * sequence of views, one launch per pass.  The host plans every view (crops, index and coefficient tables, final
 * intrinsics); the descriptor arrays below live in DEVICE memory, one entry per view.
 *
 * s3r_views_depth: out pixel (x, y) of the w x h cropped view reads depth[row_src[y] * depth_stride + col_src[x]]
 * (crop 1, cv2 INTER_NEAREST resize and crop 2 folded into the two index tables) and writes depthmap, pts3d (world,
 * fp32, [.., 3]) and valid (uint8 0 / 1) at y * w + x, or at x * h + y when `transpose` is set (a portrait view stored
 * landscape).  intr = (fu, fv, cu, cv), pose = 3x4 row-major [R | t] (NaN for a view without pose).  A non-finite depth
 * value read sets *nonfinite = 1 (the reference asserts on it).  max_pixels >= every w * h, 1 <= n <= 65535.
 *
 * s3r_views_resample_h / s3r_views_resample_v_norm: s3r_resample_h_u8 / s3r_resample_v_u8_norm of every view in one
 * launch each, bit for bit; img [3, out_rows, cols] fp32, or [3, cols, out_rows] when `transpose` is set.
 * max_rows / max_out_rows / max_cols bound every view's rows / out_rows / cols, max_span every view's span (see
 * s3r_resample_h_u8). */
typedef struct s3r_view_depth_desc {
  const float* depth;
  const int32_t* col_src;
  const int32_t* row_src;
  float* depthmap;
  float* pts3d;
  uint8_t* valid;
  int32_t* nonfinite;
  int64_t depth_stride;
  int32_t w, h, transpose;
  float intr[4];
  float pose[12];
} s3r_view_depth_desc;

typedef struct s3r_view_image_desc {
  const uint8_t* src;
  const int32_t* bh;
  const int32_t* kh;
  const int32_t* bv;
  const int32_t* kv;
  uint8_t* tmp;
  float* img;
  int64_t row_stride;
  int32_t rows, cols, out_rows, ksh, ksv, transpose;
} s3r_view_image_desc;

/* sizeof the view descriptors (which = 0: depth, 1: image, 2: s3r_view_jitter_desc below), for the bindings to check
 * their mirrors */
int s3r_views_abi_sizeof(int which);
int s3r_views_depth(const s3r_view_depth_desc* descs, int n, int64_t max_pixels, void* stream);
int s3r_views_resample_h(const s3r_view_image_desc* descs, int n, int max_rows, int max_cols, int max_span, void* stream);
int s3r_views_resample_v_norm(const s3r_view_image_desc* descs, int n, int max_out_rows, int max_cols, void* stream);

/* ---- training views: torchvision's ColorJitter (PIL path) before ImgNorm, bit for bit (spann3r_b200/train_views.py) --
 * s3r_views_resample_v_u8: the vertical pass of s3r_views_resample_v_norm without ImgNorm: view v's uint8 image
 * [out_rows, cols, 3] (before any transpose) goes to jit[v].u8.  descs / jit: device arrays of n entries each.
 *
 * s3r_views_color_jitter: one CTA per view.  Applies the view's ops in `order` (0 brightness, 1 contrast, 2 saturation,
 * 3 hue; bit k of `skip` set: op k's factor was None and it is not applied) to u8 [rows, cols, 3], with Pillow's rules
 * (csrc/jitter_math.cuh): brightness / contrast / saturation are Image.blend toward black / the image's mean L / each
 * pixel's L with the fp32 factor, hue adds `hue_shift` (= (int32) trunc(hue_factor * 255)) to the uint8 HSV hue mod 256.
 * Then ImgNorm, writing img [3, rows, cols] fp32, or [3, cols, rows] when `transpose` is set.  The contrast mean is an
 * exact integer reduction.  max_pixels >= every rows * cols.  u8 is only read. */
typedef struct s3r_view_jitter_desc {
  uint8_t* u8;
  float* img;
  int32_t rows, cols, transpose;
  int32_t order[4];
  int32_t skip;
  float brightness, contrast, saturation;
  int32_t hue_shift;
} s3r_view_jitter_desc;

int s3r_views_resample_v_u8(const s3r_view_image_desc* descs, const s3r_view_jitter_desc* jit, int n, int max_out_rows,
                            int max_cols, void* stream);
int s3r_views_color_jitter(const s3r_view_jitter_desc* jit, int n, int64_t max_pixels, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SPANN3R_B200_H_ */
