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
/* sizeof(s3r_gemm_desc / s3r_model_w / s3r_bank) as compiled: bindings check their mirrors against these */
int s3r_abi_sizeof(int which /* 0 gemm_desc, 1 model_w, 2 bank */);
/* last error text of the calling thread ("" if none) */
const char* s3r_last_error(void);
/* 1 if a CUDA device of compute capability 9.0 (H100, sm_90a) is visible, else 0 (never falls back to CPU) */
int s3r_device_ok(void);

/* ---- op level ------------------------------------------------------------------------------ */

/* fp32 [rows, c] (row stride ldx) -> planes [rows, ldp] at column col0, optional ReLU first.
 * Replaces nothing in the reference; it is the format conversion at the head of a GEMM chain. */
int s3r_split(const float* x, int64_t ldx, void* hi, void* lo, int64_t ldp, int col0, int64_t rows, int c, int relu,
              void* stream);

/* nn.LayerNorm over the last dim (c = 768 or 1024), fp32 and/or planes out.
 * croco/models/blocks.py:116-130,176-191 (norm1/2/3/norm_y, eps 1e-6), dust3r/model.py:151,203
 * (enc_norm, dec_norm), spann3r/model.py:245-247 (norm_q/k/v, eps 1e-5).
 * Groups: row r uses weight set (r / rows_per_group) at w + set*wb_group_stride (0 = one set).
 * swap_rows > 0: two groups of swap_rows rows; output rows and weight sets are exchanged between
 * the groups (the twin decoders' norm_y, dust3r/model.py:197-199). */
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
/* im2col for Conv2d(C, C, 3, stride 2, pad 1): planes [nb,h,w,c] -> planes [nb*ho*wo, 9*c].
 * croco/models/dpt_block.py:396-408 (act_4_postprocess). */
int s3r_im2col_3x3s2(const void* ihi, const void* ilo, int nb, int h, int w, int c, int ho, int wo, void* ohi,
                     void* olo, void* stream);
/* Bilinear x2, align_corners=True, channels-last fp32 [nb,h,w,c] -> fp32 and/or planes [nb,2h,2w,c].
 * croco/models/dpt_block.py:214-215, 246-253. */
int s3r_upsample2x(const float* x, int nb, int h, int w, int c, float* out, void* hi, void* lo, void* stream);

/* The tensor-core workhorse: D = A * B^T with fused epilogue (see EPI modes).
 *   A planes [groups*nb, h, w, kc] (a linear layer is h = 1, w = rows), B planes [groups*n, taps, kc],
 *   taps = 1 (linear / 1x1 conv / ConvTranspose with kernel == stride) or 9 (3x3, stride 1, pad 1).
 * Replaces nn.Linear / Conv2d / ConvTranspose2d calls of croco/models/blocks.py:73-79,94-112,149-169,
 * dust3r/model.py:189-190, spann3r/model.py:250-261,310 and croco/models/dpt_block.py (all convs). */
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
   * all rounded to tf32.  croco/models/blocks.py:97-104,154-160 + models/pos_embed.py:112-159. */
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
   * (ln_np = kc/32); the epilogue applies rstd_r * (acc - mean_r * ln_cs[col]) + bias = LN(x) W^T + b.
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
} s3r_gemm_desc;
int s3r_gemm(const s3r_gemm_desc* d, void* stream);
/* tile width the planner would pick (64/128), for tests */
int s3r_gemm_tile_n(const s3r_gemm_desc* d);

/* Fused multi-head attention core, head dim 64: O = softmax(Q K^T) V per (batch*head) on tf32 wgmma.
 *   q [bh, nq, 64], k [bh, nk, 64] (already RoPE'd / scaled by the QKV epilogue), vt [bh, 64, nk_pad];
 *   output [b*nq, heads*64] as planes and/or fp32 (row stride ldo).
 * croco/models/blocks.py:106-110 (self), :162-166 (cross). */
int s3r_attention(const float* q, const float* k, const float* vt, int bh, int heads, int nq, int nk, int nk_pad,
                  void* o_hi, void* o_lo, float* o_f32, int64_t ldo, void* stream);

/* Offline-mode view score: out[0] = mean((conf-1)/conf) over n values (spann3r/model.py:346-352, 372-381);
 * scratch256 = 256 floats of device scratch.  Deterministic. */
int s3r_conf_score(const float* conf, int64_t n, float* scratch256, float* out, void* stream);

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
 * cs [G*N] = row sums of the planes (see s3r_gemm_desc.ln_cs); the preceding s3r_ln is then unused by the engine. */
typedef struct s3r_lin { s3r_planes w; const float* b; const float* cs; } s3r_lin;

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
 *   S3R_VALUE_ROPE            Spann3R(mem_pos_enc=True): RoPE inside the value encoder's blocks (spann3r/model.py:231) */
#define S3R_VALUE_PTS_TRANSPOSED 1
#define S3R_VALUE_ROPE 2
int s3r_engine_value(s3r_engine* e, const float* pts3d, const float* feat_k1, int flags, float* out, void* stream);
/* spann3r/model.py:145-183 memory_read (eval: thresh = 5e-4; 0 disables): out = attn.V + feat; bank.attn += colsum */
int s3r_engine_memory_read(s3r_engine* e, const s3r_bank* bank, const float* feat, float thresh, float* out,
                           void* stream);
/* training mode of the same read (spann3r/model.py:474 `attn_thresh=0`, :167-168 `mem_dropout`): nn.Dropout(drop_p) on the
 * softmax output, before the (normally disabled) threshold.  The keep decision of element (b, row, column) is Philox4x32-10
 * of (seed, (b * N + row) * len + column): reproducible, regenerated for the backward pass / tests by s3r_dropout_mask */
int s3r_engine_memory_read_train(s3r_engine* e, const s3r_bank* bank, const float* feat, float thresh, float drop_p,
                                 uint64_t seed, float* out, void* stream);
/* Tuning knobs of the GEMM planner, read when an engine builds its plans (first pass of a stage): "prefetch_b" (weight
 * tiles staged before the programmatic-dependent-launch wait; default 1).  The call exists so that two engines of one
 * process can be planned differently and timed alternately. */
int s3r_set_option(const char* name, int value);
/* out[i] = 0 or 1/(1-p): the keep-scale the training-mode read applies to flat element i = (b * N + row) * len + column */
int s3r_dropout_mask(float* out, int64_t n, uint64_t seed, float p, void* stream);
/* spann3r/model.py:80-95 add_mem: append N tokens at bank.len (caller then sets len += N) */
int s3r_engine_memory_append(s3r_engine* e, const s3r_bank* bank, const float* feat_k, const float* feat_v,
                             void* stream);
/* spann3r/model.py:97-118 check_sim: out[b, t] = mean cosine vs each of the last wm frames (device array [B, wm]) */
int s3r_engine_check_sim(s3r_engine* e, const s3r_bank* bank, const float* feat_k, int wm, float* out, void* stream);
/* algorithmic FLOPs (2*M*N*K of every tensor-core launch) issued since the last call; resets the counter */
double s3r_engine_take_flops(s3r_engine* e);
/* Per-launch CUDA-event timing of the tensor-core kernels (bench.py roofline leg): switch on, run, read.
 * profile_read synchronises the device; out = {gemm_ms, gemm_flops, gemm_launches, attn_ms, attn_flops, attn_launches} */
void s3r_engine_profile(s3r_engine* e, int on);
/* per-launch list (in launch order) of the recorded tensor-core launches: duration [ms], algorithmic FLOPs, kind
 * (0 GEMM / conv, 1 attention); returns the count (call before profile_read, which consumes the records) */
int s3r_engine_profile_list(s3r_engine* e, double* ms, double* flops, int* kind, int cap);
int s3r_engine_profile_read(s3r_engine* e, double* out);
/* number of kernel launches since the last call; resets the counter */
long long s3r_engine_take_launches(s3r_engine* e);

#ifdef __cplusplus
}
#endif
#endif /* SPANN3R_B200_H_ */
