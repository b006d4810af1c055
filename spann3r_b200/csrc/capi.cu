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

static int fill_plan(const s3r_gemm_desc* d, GemmPlan* plan) {
  if (d->epi == S3R_EPI_HEADTAIL && d->n != 128) {
    set_error("s3r_gemm: EPI_HEADTAIL needs n == 128");
    return -1;
  }
  const int force_bn = d->epi == S3R_EPI_HEADTAIL ? (d->force_bn == 128 ? 128 : 1128) : d->force_bn;
  int r = gemm_plan_init(plan, B(d->a_hi), B(d->a_lo), B(d->b_hi), B(d->b_lo), d->groups, d->nb, d->h, d->w, d->kc,
                         d->taps, d->n, force_bn);
  if (r) return r;
  GemmArgs& a = plan->args;
  a.epi = d->epi; a.act = d->act; a.plane_relu = d->plane_relu;
  a.bias = d->bias;
  a.res1 = d->res1; a.ldr1 = (int)d->ldr1;
  a.res2 = d->res2; a.ldr2 = (int)d->ldr2;
  a.out_f32 = d->out_f32; a.ldo = (int)d->ldo;
  a.out_hi = B(d->out_hi); a.out_lo = B(d->out_lo); a.ldp = (int)d->ldp; a.plane_col0 = d->plane_col0;
  if (d->epi == S3R_EPI_PIXSHUF) {
    if (d->ps_s <= 0 || d->ps_cout % 32 != 0 || d->n != d->ps_s * d->ps_s * d->ps_cout) {
      set_error("s3r_gemm: EPI_PIXSHUF needs n == s*s*cout and cout %% 32 == 0");
      return -1;
    }
    a.ps_s = d->ps_s; a.ps_cout = d->ps_cout;
    a.out_group_rows = (long long)d->nb * d->h * d->ps_s * d->w * d->ps_s;
  }
  if (d->epi == S3R_EPI_QKV) {
    if (d->q_c % 64 != 0 || d->h != 1 || d->q_ntok <= 0 || d->w != d->q_nb * d->q_ntok) {
      set_error("s3r_gemm: EPI_QKV needs q_c %% 64 == 0, h == 1, w == q_nb*q_ntok");
      return -1;
    }
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
    if (d->ln_cs == nullptr || d->ln_np * 32 != d->kc || d->taps != 1 || d->epi == S3R_EPI_PIXSHUF) {
      set_error("s3r_gemm: folded LayerNorm needs ln_cs, ln_np == kc/32, taps == 1 and a non-PIXSHUF epilogue");
      return -1;
    }
    a.ln_stats = reinterpret_cast<const float2*>(d->ln_stats); a.ln_np = d->ln_np; a.ln_eps = d->ln_eps; a.ln_cs = d->ln_cs;
  }
  a.a_swap = d->a_swap ? 1 : 0;
  if (d->swap_col0 % 256 != 0) {
    set_error("s3r_gemm: swap_col0 must be a multiple of 256");
    return -1;
  }
  a.swap_col0 = d->swap_col0;
  if (d->stats_out) {
    if (d->epi != S3R_EPI_PLAIN || d->n % 32 != 0) {
      set_error("s3r_gemm: stats_out needs EPI_PLAIN and n %% 32 == 0");
      return -1;
    }
    a.stats_out = reinterpret_cast<float2*>(d->stats_out);
  }
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

int s3r_conf_score(const float* conf, int64_t n, float* scratch256, float* out, void* stream) {
  return launch_conf_score(conf, n, scratch256, out, S(stream));
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
