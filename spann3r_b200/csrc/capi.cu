// extern "C" boundary of libspann3r_b200.so (declared in include/spann3r_b200.h) -- op level.
#include "../../include/spann3r_b200.h"

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

int s3r_gemm(const s3r_gemm_desc* d, void* stream) {
  GemmPlan plan;
  if (int r = gemm_plan(*d, &plan)) return r;
  return gemm_launch(plan, S(stream));
}

int s3r_gemm_tile_n(const s3r_gemm_desc* d) {
  GemmPlan plan;
  if (int r = gemm_plan(*d, &plan)) return r;
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

size_t s3r_mesh_grid_workspace_bytes(int T, int H, int W) { return mesh_grid_workspace_bytes(T, H, W); }
int s3r_mesh_grid_count(const uint8_t* valid, int T, int H, int W, void* workspace, size_t workspace_bytes,
                        int64_t* n_faces, void* stream) {
  return launch_mesh_grid_count(valid, T, H, W, workspace, workspace_bytes, reinterpret_cast<long long*>(n_faces),
                                S(stream));
}
int s3r_mesh_grid_faces(const uint8_t* valid, const float* images, int T, int H, int W, const void* workspace,
                        size_t workspace_bytes, int32_t* faces, float* colors, void* stream) {
  return launch_mesh_grid_faces(valid, images, T, H, W, workspace, workspace_bytes, faces, colors, S(stream));
}
int s3r_raster_triangles(const float* verts, int64_t n_verts, const int32_t* faces, int64_t n_faces, int64_t id0,
                         const double* camera, double z_near, double z_far, int width, int height, void* keys,
                         void* stream) {
  return launch_raster_triangles(verts, n_verts, faces, n_faces, id0, camera, z_near, z_far, width, height, keys,
                                 S(stream));
}
int s3r_raster_resolve(const void* keys, int width, int height, float* depth, int32_t* face, void* stream) {
  return launch_raster_resolve(keys, width, height, depth, face, S(stream));
}

size_t s3r_poisson_workspace_bytes(int64_t n, int depth) { return poisson_workspace_bytes(n, depth); }
size_t s3r_poisson_offset(int64_t n, int depth, int which) { return poisson_offset(n, depth, which); }
int s3r_poisson_setup(const void* points, const void* normals, int is_f64, int64_t n, int depth, double scale,
                      void* workspace, size_t workspace_bytes, double* info, void* stream) {
  return launch_poisson_setup(points, normals, is_f64, n, depth, scale, workspace, workspace_bytes, info, S(stream));
}
int s3r_poisson_solve(int64_t n, int depth, double tol, int max_iter, void* workspace, size_t workspace_bytes,
                      double* info, void* stream) {
  return launch_poisson_solve(n, depth, tol, max_iter, workspace, workspace_bytes, info, S(stream));
}
int s3r_poisson_extract_count(int64_t n, int depth, void* workspace, size_t workspace_bytes, int64_t* sizes,
                              void* stream) {
  return launch_poisson_extract_count(n, depth, workspace, workspace_bytes, reinterpret_cast<long long*>(sizes),
                                      S(stream));
}
int s3r_poisson_extract(int64_t n, int depth, void* workspace, size_t workspace_bytes, float* vertices, int64_t* faces,
                        double* densities, void* stream) {
  return launch_poisson_extract(n, depth, workspace, workspace_bytes, vertices, reinterpret_cast<long long*>(faces),
                                densities, S(stream));
}
int s3r_pcl_quantile(const double* x, int64_t n, double q, void* workspace, double* out, void* stream) {
  return launch_pcl_quantile(x, n, q, workspace, out, S(stream));
}
size_t s3r_mesh_compact_workspace_bytes(int64_t n_verts, int64_t n_faces) {
  return mesh_compact_workspace_bytes(n_verts, n_faces);
}
int s3r_mesh_compact_count(const uint8_t* mask, const int64_t* faces, int64_t n_verts, int64_t n_faces, void* workspace,
                           size_t workspace_bytes, int64_t* sizes, void* stream) {
  return launch_mesh_compact_count(mask, reinterpret_cast<const long long*>(faces), n_verts, n_faces, workspace,
                                   workspace_bytes, reinterpret_cast<long long*>(sizes), S(stream));
}
int s3r_mesh_compact(const float* vertices, const int64_t* faces, int64_t n_verts, int64_t n_faces,
                     const void* workspace, size_t workspace_bytes, float* out_vertices, int64_t* out_faces,
                     void* stream) {
  return launch_mesh_compact(vertices, reinterpret_cast<const long long*>(faces), n_verts, n_faces, workspace,
                             workspace_bytes, out_vertices, reinterpret_cast<long long*>(out_faces), S(stream));
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

int s3r_dropout_mask(float* out, int64_t n, uint64_t seed, float p, void* stream) {
  if (!out && n > 0) {
    set_error("s3r_dropout_mask: null output");
    return -1;
  }
  return launch_dropout_mask(out, n, seed, p, S(stream));
}

int s3r_attention(const float* q, const float* k, const float* vt, int bh, int heads, int nq, int nk, int nk_pad,
                  void* o_hi, void* o_lo, float* o_f32, int64_t ldo, void* stream) {
  const AttnDesc d = {q, k, vt, bh, heads, nq, nk, nk_pad, B(o_hi), B(o_lo), o_f32, ldo};
  AttnPlan plan;
  if (int r = attn_plan(d, &plan)) return r;
  return attn_launch(plan, S(stream));
}

}  // extern "C"
