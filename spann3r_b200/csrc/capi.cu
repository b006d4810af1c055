// extern "C" boundary of libspann3r_b200.so (declared in include/spann3r_b200.h) -- op level.
#include "../../include/spann3r_b200.h"

#include <cstring>

#include "gemm.cuh"
#include "kernels.cuh"

using namespace s3r;

static inline cudaStream_t S(void* s) { return reinterpret_cast<cudaStream_t>(s); }
static inline __nv_bfloat16* B(void* p) { return reinterpret_cast<__nv_bfloat16*>(p); }
static inline const __nv_bfloat16* B(const void* p) { return reinterpret_cast<const __nv_bfloat16*>(p); }

extern "C" {

int s3r_version(void) { return S3R_VERSION; }
int s3r_abi_sizeof(int which) {
  switch (which) {
    case 0: return (int)sizeof(s3r_gemm_desc);
    case 1: return (int)sizeof(s3r_model_w);
    case 2: return (int)sizeof(s3r_bank);
    case 3: return (int)sizeof(s3r_loss_desc);
    case 4: return (int)sizeof(s3r_attn_train_desc);
  }
  return -1;
}
const char* s3r_last_error(void) { return s3r::last_error(); }

int s3r_device_ok(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) {
    cudaGetLastError();
    return 0;
  }
  int dev = 0, major = 0, minor = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  return (major == 9 && minor == 0) ? 1 : 0;
}

int s3r_split(const float* x, int64_t ldx, void* hi, void* lo, int64_t ldp, int col0, int64_t rows, int c, int relu,
              void* stream) {
  return launch_split(x, ldx, B(hi), B(lo), ldp, col0, rows, c, relu, S(stream));
}

int s3r_layernorm(const float* x, int64_t ldx, const float* w, const float* b, int64_t wb_group_stride,
                  int64_t rows_per_group, float eps, int64_t rows, int c, float* out, int64_t ldo, void* hi, void* lo,
                  int64_t ldp, int col0, int64_t swap_rows, void* stream) {
  return launch_layernorm(x, ldx, w, b, wb_group_stride, rows_per_group, eps, rows, c, out, ldo, B(hi), B(lo), ldp,
                          col0, swap_rows, S(stream));
}

int s3r_rope2d_inplace(float* tokens, const int64_t* pos, int64_t bn, int h, int d, int64_t stride_tok,
                       int64_t stride_head, float base, float fwd, void* stream) {
  return launch_rope2d(tokens, reinterpret_cast<const long long*>(pos), bn, h, d, stride_tok, stride_head, base, fwd,
                       S(stream));
}

int s3r_im2col_patch16(const float* img, int64_t sb, int64_t sc, int64_t sy, int64_t sx, int b, int gh, int gw,
                       void* hi, void* lo, void* stream) {
  return launch_im2col_patch16(img, sb, sc, sy, sx, b, gh, gw, B(hi), B(lo), S(stream));
}

int s3r_im2col_3x3s2(const void* ihi, const void* ilo, int nb, int h, int w, int c, int ho, int wo, void* ohi,
                     void* olo, void* stream) {
  return launch_im2col_3x3s2(B(ihi), B(ilo), nb, h, w, c, ho, wo, B(ohi), B(olo), S(stream));
}

int s3r_upsample2x(const float* x, int nb, int h, int w, int c, float* out, void* hi, void* lo, void* stream) {
  return launch_upsample2x(x, nb, h, w, c, out, B(hi), B(lo), S(stream));
}

size_t s3r_conv_wgrad_workspace_bytes(int nb, int h, int w, int n, int kc, int taps) {
  return conv_wgrad_workspace_bytes(nb, h, w, n, kc, taps);
}
int s3r_conv_wgrad(const void* dy_hi, const void* dy_lo, int64_t ldy, const void* x_hi, const void* x_lo, int64_t ldx,
                   int nb, int h, int w, int n, int kc, int taps, void* workspace, size_t workspace_bytes, float* dw,
                   void* stream) {
  return launch_conv_wgrad(B(dy_hi), B(dy_lo), ldy, B(x_hi), B(x_lo), ldx, nb, h, w, n, kc, taps, workspace,
                           workspace_bytes, dw, S(stream));
}
int s3r_col2im_3x3s2(const float* cols, int nb, int h, int w, int c, int ho, int wo, float* out, void* stream) {
  return launch_col2im_3x3s2(cols, nb, h, w, c, ho, wo, out, S(stream));
}

// Row strides and column offsets of the epilogue's fp32 (float4) and planes (uint2) accesses: multiples of 4 elements
// that fit the kernel's int fields.
static bool bad_ld(int64_t ld) { return ld < 0 || ld > INT32_MAX || ld % 4 != 0; }

// Every descriptor rule the epilogue relies on, checked before anything touches the driver.
static int check_desc(const s3r_gemm_desc* d) {
  if (d->precision != GEMM_SPLIT && d->precision != GEMM_BF16) {
    set_error("s3r_gemm: precision=%d must be 0 (split bf16) or 1 (one bf16 product)", d->precision);
    return -1;
  }
  if (d->precision == GEMM_BF16 && d->epi == S3R_EPI_HEADTAIL) {
    set_error("s3r_gemm: precision=1 does not support EPI_HEADTAIL (the DPT head tail is split-only)");
    return -1;
  }
  if (d->n <= 0 || d->n % 32 != 0) {
    set_error("s3r_gemm: n=%d must be a positive multiple of 32 (the epilogue stores whole 32-column chunks)", d->n);
    return -1;
  }
  if (d->epi == S3R_EPI_HEADTAIL && d->n != 128) {
    set_error("s3r_gemm: EPI_HEADTAIL needs n == 128");
    return -1;
  }
  if (d->epi == S3R_EPI_PIXSHUF && (d->ps_s <= 0 || d->ps_cout % 32 != 0 || d->n != d->ps_s * d->ps_s * d->ps_cout)) {
    set_error("s3r_gemm: EPI_PIXSHUF needs n == s*s*cout and cout %% 32 == 0");
    return -1;
  }
  const struct { const char* name; bool used; int64_t v; } lds[5] = {
      {"ldr1", d->res1 != nullptr, d->ldr1}, {"ldr2", d->res2 != nullptr, d->ldr2}, {"ldo", d->out_f32 != nullptr, d->ldo},
      {"ldp", d->out_hi != nullptr, d->ldp}, {"plane_col0", d->out_hi != nullptr, d->plane_col0}};
  for (const auto& l : lds)
    if (l.used && bad_ld(l.v)) {
      set_error("s3r_gemm: %s=%lld must be a non-negative multiple of 4 below 2^31 (vector accesses)", l.name,
                (long long)l.v);
      return -1;
    }
  if (d->epi == S3R_EPI_QKV) {
    if (d->q_c <= 0 || d->q_c % 64 != 0 || d->h != 1 || d->q_ntok <= 0 || d->w != d->q_nb * d->q_ntok) {
      set_error("s3r_gemm: EPI_QKV needs q_c %% 64 == 0, h == 1, w == q_nb*q_ntok");
      return -1;
    }
    if (d->n % d->q_c != 0) {
      set_error("s3r_gemm: EPI_QKV n=%d must be a multiple of q_c=%d", d->n, d->q_c);
      return -1;
    }
    if (d->q_role_base < 0 || d->q_role_base + d->n / d->q_c > 5) {
      set_error("s3r_gemm: EPI_QKV q_role_base=%d + n/q_c=%d must stay within the 5 roles", d->q_role_base,
                d->n / d->q_c);
      return -1;
    }
    if (d->q_ntok_pad < d->q_ntok || d->q_ntok_pad % 4 != 0) {
      set_error("s3r_gemm: EPI_QKV q_ntok_pad=%d must be >= q_ntok=%d and a multiple of 4", d->q_ntok_pad, d->q_ntok);
      return -1;
    }
    static const char* const kRoleOut[5] = {"q_out", "k_out", "vt_out", "k2_out", "vt2_out"};
    for (int role = d->q_role_base; role < d->q_role_base + d->n / d->q_c; ++role) {
      const void* p = role == 0 ? (const void*)d->q_out : role == 1 ? (const void*)d->k_out : role == 2 ? (const void*)d->vt_out
                    : role == 3 ? (const void*)d->k2_out : (const void*)d->vt2_out;
      if (!p) {
        set_error("s3r_gemm: EPI_QKV role %d is written but %s is NULL", role, kRoleOut[role]);
        return -1;
      }
    }
    if (d->q_rope && (!d->q_pos || !d->q_cs)) {
      set_error("s3r_gemm: EPI_QKV with q_rope needs %s", d->q_pos ? "q_cs" : "q_pos");
      return -1;
    }
  }
  if (d->ln_stats) {
    if (d->ln_cs == nullptr || d->ln_np * 32 != d->kc || d->taps != 1 || d->epi == S3R_EPI_PIXSHUF) {
      set_error("s3r_gemm: folded LayerNorm needs ln_cs, ln_np == kc/32, taps == 1 and a non-PIXSHUF epilogue");
      return -1;
    }
    if (d->ln_np < 2 || d->ln_np > 32 || d->ln_np % 2 != 0) {
      set_error("s3r_gemm: folded LayerNorm needs an even ln_np in [2, 32] (kc %% 64 == 0, kc <= 1024), got ln_np=%d",
                d->ln_np);
      return -1;
    }
  }
  if (d->swap_col0 % 256 != 0) {
    set_error("s3r_gemm: swap_col0 must be a multiple of 256");
    return -1;
  }
  if (d->stats_out && d->epi != S3R_EPI_PLAIN) {
    set_error("s3r_gemm: stats_out needs EPI_PLAIN");
    return -1;
  }
  return 0;
}

static int fill_plan(const s3r_gemm_desc* d, GemmPlan* plan) {
  int r = check_desc(d);
  if (r) return r;
  const int force_bn = d->epi == S3R_EPI_HEADTAIL ? (d->force_bn == 128 ? 128 : 1128) : d->force_bn;
  r = gemm_plan_init(plan, B(d->a_hi), B(d->a_lo), B(d->b_hi), B(d->b_lo), d->groups, d->nb, d->h, d->w, d->kc,
                     d->taps, d->n, force_bn, 0, 0, 0, d->precision, d->a_swap ? d->swap_col0 : 0);
  if (r) return r;
  GemmArgs& a = plan->args;
  a.epi = d->epi; a.act = d->act; a.plane_relu = d->plane_relu;
  a.bias = d->bias;
  a.res1 = d->res1; a.ldr1 = (int)d->ldr1;
  a.res2 = d->res2; a.ldr2 = (int)d->ldr2;
  a.out_f32 = d->out_f32; a.ldo = (int)d->ldo;
  a.out_hi = B(d->out_hi); a.out_lo = B(d->out_lo); a.ldp = (int)d->ldp; a.plane_col0 = d->plane_col0;
  if (d->epi == S3R_EPI_PIXSHUF) {
    a.ps_s = d->ps_s; a.ps_cout = d->ps_cout;
    a.out_group_rows = (long long)d->nb * d->h * d->ps_s * d->w * d->ps_s;
  }
  if (d->epi == S3R_EPI_QKV) {
    a.q_C = d->q_c; a.q_role_base = d->q_role_base; a.q_ntok = d->q_ntok; a.q_ntok_pad = d->q_ntok_pad;
    a.q_rope = d->q_rope; a.q_nb = d->q_nb; a.q_pos = d->q_pos;
    a.q_cs = reinterpret_cast<const float2*>(d->q_cs);
    a.q_out = d->q_out; a.k_out = d->k_out; a.vt_out = d->vt_out; a.q_scale = d->q_scale;
    a.k2_out = d->k2_out; a.vt2_out = d->vt2_out;
  }
  if (d->epi == S3R_EPI_HEADTAIL) {
    a.ht_w = d->ht_w; a.ht_b = d->ht_b; a.ht_pts = d->ht_pts; a.ht_conf = d->ht_conf;
  }
  if (d->ln_stats) {
    a.ln_stats = reinterpret_cast<const float2*>(d->ln_stats); a.ln_np = d->ln_np; a.ln_eps = d->ln_eps; a.ln_cs = d->ln_cs;
  }
  a.a_swap = d->a_swap ? 1 : 0;
  a.swap_col0 = d->swap_col0;
  a.stats_out = reinterpret_cast<float2*>(d->stats_out);
  a.trace = reinterpret_cast<unsigned long long*>(d->trace);
  return 0;
}

int s3r_gemm(const s3r_gemm_desc* d, void* stream) {
  GemmPlan plan;
  int r = fill_plan(d, &plan);
  if (r) return r;
  return gemm_launch(plan, S(stream));
}

int s3r_gemm_tile_n(const s3r_gemm_desc* d) {
  GemmPlan plan;
  int r = fill_plan(d, &plan);
  if (r) return r;
  return plan.bn;
}

int s3r_gemm_plan_bn(int64_t m_tiles, int n, int sms, int col_align, int force_bn) {
  if (m_tiles < 1 || n < 1 || sms < 1 || col_align < 0) {
    set_error("s3r_gemm_plan_bn: m_tiles=%lld n=%d sms=%d col_align=%d (positive; col_align >= 0)", (long long)m_tiles,
              n, sms, col_align);
    return -1;
  }
  return gemm_choose_bn(m_tiles, n, sms, col_align, force_bn);
}

int s3r_resample_h_u8(const uint8_t* src, int64_t row_stride, int rows, int out_cols, const int32_t* bounds,
                      const int32_t* kk, int ksize, int max_span, uint8_t* dst, void* stream) {
  return launch_resample_h_u8(src, row_stride, rows, out_cols, bounds, kk, ksize, max_span, dst, S(stream));
}
int s3r_resample_v_u8_norm(const uint8_t* tmp, int cols, int out_rows, const int32_t* bounds, const int32_t* kk, int ksize,
                           float* dst, void* stream) {
  return launch_resample_v_u8_norm(tmp, cols, out_rows, bounds, kk, ksize, dst, S(stream));
}

int s3r_focal_weiszfeld(const float* pts3d, int b, int h, int w, float ppx, float ppy, int iters, float lo, float hi,
                        float* scratch, float* focal, void* stream) {
  return launch_focal_weiszfeld(pts3d, b, h, w, ppx, ppy, iters, lo, hi, scratch, focal, S(stream));
}

int s3r_focal_median(const float* pts3d, int b, int h, int w, float ppx, float ppy, float lo, float hi, int32_t* scratch,
                     float* focal, void* stream) {
  return launch_focal_median(pts3d, b, h, w, ppx, ppy, lo, hi, scratch, focal, S(stream));
}

size_t s3r_pnp_workspace_bytes(int b, int n_samples) {
  if (b <= 0 || n_samples <= 0) return 0;
  return pnp_workspace_bytes(b, n_samples);
}
int s3r_pnp_ransac(const float* pts3d, const float* img_pts, int b, int64_t n, int width, double fx, double fy, double cx,
                   double cy, float reproj_err, int n_samples, int refine_iters, uint64_t seed, void* workspace,
                   double* out, uint8_t* inlier_mask, void* stream) {
  return launch_pnp_ransac(pts3d, img_pts, b, n, width, fx, fy, cx, cy, reproj_err, n_samples, refine_iters, seed,
                           workspace, out, inlier_mask, S(stream));
}

size_t s3r_pcl_index_bytes(int64_t n) { return pcl_index_bytes(n); }
int s3r_pcl_index_build(const void* pts, int is_f64, int64_t n, const double* transform, void* index, void* stream) {
  return launch_pcl_index_build(pts, is_f64, n, transform, index, S(stream));
}
int s3r_pcl_nearest(const void* index, int64_t n, const void* queries, int is_f64, int64_t nq, const double* transform,
                    double max_dist, double* dist, int64_t* idx, void* stream) {
  return launch_pcl_nearest(index, n, queries, is_f64, nq, transform, max_dist, dist, reinterpret_cast<long long*>(idx),
                            S(stream));
}
int s3r_pcl_normals(const void* index, int64_t n, int k, double* normals, void* stream) {
  return launch_pcl_normals(index, n, k, normals, S(stream));
}
size_t s3r_pcl_icp_workspace_bytes(void) { return pcl_icp_workspace_bytes(); }
int s3r_pcl_icp(const void* source, int is_f64, int64_t ns, const void* target_index, int64_t nt,
                double max_correspondence_distance, const double* init, int max_iteration, double relative_fitness,
                double relative_rmse, void* workspace, double* out, void* stream) {
  return launch_pcl_icp(source, is_f64, ns, target_index, nt, max_correspondence_distance, init, max_iteration,
                        relative_fitness, relative_rmse, workspace, out, S(stream));
}
size_t s3r_pcl_stats_workspace_bytes(void) { return pcl_stats_workspace_bytes(); }
int s3r_pcl_stats(const double* x, int64_t n, double threshold, void* workspace, double* out, void* stream) {
  return launch_pcl_stats(x, n, threshold, workspace, out, S(stream));
}
int s3r_pcl_abs_dot(const double* a, const double* b, const int64_t* idx, int64_t n, double* out, void* stream) {
  return launch_pcl_abs_dot(a, b, reinterpret_cast<const long long*>(idx), n, out, S(stream));
}

size_t s3r_render_workspace_bytes(int width, int height) { return render_workspace_bytes(width, height); }
int s3r_render_clear(void* keys, int width, int height, void* stream) {
  return launch_render_clear(keys, width, height, S(stream));
}
int s3r_render_splat(const float* pts, const uint8_t* mask, int64_t n, int64_t id0, const double* camera, double z_near,
                     int width, int height, void* keys, void* stream) {
  return launch_render_splat(pts, mask, n, id0, camera, z_near, width, height, keys, S(stream));
}
int s3r_render_resolve(const void* keys, const float* colors, int width, int height, uint8_t* rgb, void* stream) {
  return launch_render_resolve(keys, colors, width, height, rgb, S(stream));
}

size_t s3r_loss_workspace_bytes(const s3r_loss_desc* d) { return loss_workspace_bytes(d); }
int s3r_loss_forward(const s3r_loss_desc* d, void* workspace, size_t workspace_bytes, float* gt_out, float* pred_out,
                     uint8_t* valid_out, double* results, void* stream) {
  return launch_loss_forward(d, workspace, workspace_bytes, gt_out, pred_out, valid_out, results, S(stream));
}
int s3r_loss_backward(const s3r_loss_desc* d, const void* workspace, size_t workspace_bytes, const float* upstream,
                      float* grad_pred, float* grad_conf, void* stream) {
  return launch_loss_backward(d, workspace, workspace_bytes, upstream, grad_pred, grad_conf, S(stream));
}

size_t s3r_attn_train_workspace_bytes(const s3r_attn_train_desc* d) { return attn_train_workspace_bytes(d); }
int s3r_attn_train_forward(const s3r_attn_train_desc* d, float* o, float* lse, void* stream) {
  return launch_attn_train_forward(d, o, lse, S(stream));
}
int s3r_attn_train_backward(const s3r_attn_train_desc* d, const float* o, const float* lse, const float* d_o,
                            void* workspace, size_t workspace_bytes, float* dq, float* dk, float* dv, void* stream) {
  return launch_attn_train_backward(d, o, lse, d_o, workspace, workspace_bytes, dq, dk, dv, S(stream));
}

int s3r_conf_score(const float* conf, int64_t n, float* scratch256, float* out, void* stream) {
  return launch_conf_score(conf, n, scratch256, out, S(stream));
}
int s3r_conf_score_batched(const float* conf, int batch, int64_t hw, float* scratch, float* out, void* stream) {
  return launch_conf_score_batched(conf, batch, hw, scratch, out, S(stream));
}

int s3r_set_option(const char* name, int value) {
  s3r::Options& o = s3r::options();
  if (!name) { set_error("s3r_set_option: null name"); return -1; }
  if (!strcmp(name, "prefetch_b")) o.prefetch_b = value;
  else { set_error("s3r_set_option: unknown option '%s' (prefetch_b)", name); return -1; }
  return 0;
}

int s3r_dropout_mask(float* out, int64_t n, uint64_t seed, float p, void* stream) {
  if (!out && n > 0) {
    set_error("s3r_dropout_mask: null output");
    return -1;
  }
  return launch_dropout_mask(out, n, seed, p, S(stream));
}

int s3r_attention(const float* q, const float* k, const float* vt, int bh, int heads, int nq, int nk, int nk_pad,
                  void* o_hi, void* o_lo, float* o_f32, int64_t ldo, void* stream) {
  return launch_attention(q, k, vt, bh, heads, nq, nk, nk_pad, B(o_hi), B(o_lo), o_f32, ldo, S(stream));
}

}  // extern "C"
