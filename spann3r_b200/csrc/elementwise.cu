// Bandwidth-bound helper kernels of the Spann3R forward path (sm_90a): LayerNorm with split-bf16
// re-encode, fp32 -> split-bf16, patch im2col, stride-2 im2col, bilinear x2 upsample (align_corners),
// and the curope-compatible in-place RoPE shim.  All are plain coalesced / 128-bit vectorised
// CUDA-core kernels: the data they touch (<= a few MB per call, except the DPT upsamples) lives in
// the 126 MB L2 between the tensor-core kernels that produce and consume it.
#include "kernels.cuh"

#include "common.cuh"

namespace s3r {

// ------------------------------------------------------------------------------------------------
// fp32 [rows, C] (row stride ldx) -> bf16 hi/lo planes [rows, ldp] at column col0; optional ReLU
// ------------------------------------------------------------------------------------------------
__global__ void split_kernel(const float* __restrict__ x, long long ldx, __nv_bfloat16* __restrict__ hi,
                             __nv_bfloat16* __restrict__ lo, long long ldp, int col0, long long rows, int C,
                             int relu) {
  pdl_launch_dependents();
  pdl_wait();
  const int c4 = C >> 2;
  const long long total = rows * c4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / c4;
    const int c = (int)(i - r * c4) << 2;
    float4 v = *reinterpret_cast<const float4*>(x + r * ldx + c);
    if (relu) {
      v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
    }
    __nv_bfloat16 h0, l0, h1, l1, h2, l2, h3, l3;
    split_bf16(v.x, h0, l0); split_bf16(v.y, h1, l1); split_bf16(v.z, h2, l2); split_bf16(v.w, h3, l3);
    const long long o = r * ldp + col0 + c;
    *reinterpret_cast<uint2*>(hi + o) = make_uint2(pack_bf16(h0, h1), pack_bf16(h2, h3));
    *reinterpret_cast<uint2*>(lo + o) = make_uint2(pack_bf16(l0, l1), pack_bf16(l2, l3));
  }
}

int launch_split(const float* x, long long ldx, __nv_bfloat16* hi, __nv_bfloat16* lo, long long ldp, int col0,
                 long long rows, int C, int relu, cudaStream_t st) {
  if (C % 4) { set_error("split: C %% 4 != 0"); return -1; }
  const long long total = rows * (C / 4);
  if (total == 0) return 0;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  launch_pdl(split_kernel, dim3(blocks), dim3(256), 0, st, x, ldx, hi, lo, ldp, col0, rows, C, relu);
  return cudaGetLastError() == cudaSuccess ? 0 : -6;
}

// ------------------------------------------------------------------------------------------------
// LayerNorm over the last dim (nn.LayerNorm, eps 1e-6 in the ViT blocks croco.py:34, 1e-5 for
// norm_q/k/v spann3r/model.py:245-247).  One warp per row, the row lives in registers, two-pass
// mean / variance in fp32.  Emits fp32 and/or split-bf16 planes.  `swap_rows` > 0 writes row r of
// group g into group (1-g) (groups of `swap_rows` rows): the twin decoders cross-attend to each
// other's stream (dust3r/model.py:197-199), and this puts norm_y(y_other) where the grouped K/V
// projection GEMM expects it.
// ------------------------------------------------------------------------------------------------
template <int NV>  // float4 per lane: C = NV * 128
__global__ void layernorm_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ w,
                                 const float* __restrict__ b, long long wb_group_stride, long long rows_per_group,
                                 float eps, long long rows, float* __restrict__ out, long long ldo,
                                 __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, long long ldp,
                                 int col0, long long swap_rows) {
  pdl_launch_dependents();
  pdl_wait();
  constexpr int C = NV * 128;
  const long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float4* xp = reinterpret_cast<const float4*>(x + row * ldx);
  float4 v[NV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    v[i] = xp[i * 32 + lane];
    s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s * (1.0f / C);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float a = v[i].x - mean, bb = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    q += (a * a + bb * bb) + (c * c + d * d);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q * (1.0f / C) + eps);
  long long grp = rows_per_group > 0 ? row / rows_per_group : 0;
  if (swap_rows > 0) grp = 1 - grp;  // norm_y of block g is applied to the OTHER stream's tokens
  const float4* wp = reinterpret_cast<const float4*>(w + grp * wb_group_stride);
  const float4* bp = reinterpret_cast<const float4*>(b + grp * wb_group_stride);
  long long orow = row;
  if (swap_rows > 0) orow = (row < swap_rows) ? row + swap_rows : row - swap_rows;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float4 ww = __ldg(wp + i * 32 + lane), bb = __ldg(bp + i * 32 + lane);
    float4 y;
    y.x = (v[i].x - mean) * rstd * ww.x + bb.x;
    y.y = (v[i].y - mean) * rstd * ww.y + bb.y;
    y.z = (v[i].z - mean) * rstd * ww.z + bb.z;
    y.w = (v[i].w - mean) * rstd * ww.w + bb.w;
    const int c = (i * 32 + lane) * 4;
    if (out) *reinterpret_cast<float4*>(out + orow * ldo + c) = y;
    if (hi) {
      __nv_bfloat16 h0, l0, h1, l1, h2, l2, h3, l3;
      split_bf16(y.x, h0, l0); split_bf16(y.y, h1, l1); split_bf16(y.z, h2, l2); split_bf16(y.w, h3, l3);
      const long long o = orow * ldp + col0 + c;
      *reinterpret_cast<uint2*>(hi + o) = make_uint2(pack_bf16(h0, h1), pack_bf16(h2, h3));
      *reinterpret_cast<uint2*>(lo + o) = make_uint2(pack_bf16(l0, l1), pack_bf16(l2, l3));
    }
  }
}

int launch_layernorm(const float* x, long long ldx, const float* w, const float* b, long long wb_group_stride,
                     long long rows_per_group, float eps, long long rows, int C, float* out, long long ldo,
                     __nv_bfloat16* hi, __nv_bfloat16* lo, long long ldp, int col0, long long swap_rows,
                     cudaStream_t st) {
  if (rows == 0) return 0;
  const int wpb = 8;
  dim3 grid((unsigned)((rows + wpb - 1) / wpb)), block(wpb * 32);
#define LN_CASE(NV)                                                                                            \
  case NV * 128:                                                                                               \
    launch_pdl(layernorm_kernel<NV>, dim3(grid), dim3(block), 0, st, x, ldx, w, b, wb_group_stride, rows_per_group, eps, rows, out, \
                                                 ldo, hi, lo, ldp, col0, swap_rows);                           \
    break;
  switch (C) {
    LN_CASE(6)
    LN_CASE(8)
    default:
      set_error("layernorm: unsupported C=%d (768 or 1024)", C);
      return -1;
  }
#undef LN_CASE
  return cudaGetLastError() == cudaSuccess ? 0 : -6;
}

// ------------------------------------------------------------------------------------------------
// Patch im2col for Conv2d(3, E, k=16, s=16) (dust3r/patch_embed.py:19-29, blocks.py:212-225):
// token (b, py, px), k = c*256 + i*16 + j  <-  img[b, c, py*16+i, px*16+j], generic element strides so the
// same kernel reads NCHW images and the NHWC pts3d map of pos_patch_embed (spann3r/model.py:317).
// ------------------------------------------------------------------------------------------------
__global__ void im2col_patch16_kernel(const float* __restrict__ img, long long sb, long long sc, long long sy,
                                      long long sx, int B, int gh, int gw, __nv_bfloat16* __restrict__ hi,
                                      __nv_bfloat16* __restrict__ lo) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = (long long)B * gh * gw * 48;  // (token, c, i): 16 consecutive j each
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int ci = (int)(idx % 48);
    const long long tok = idx / 48;
    const int c = ci >> 4, i = ci & 15;
    const int px = (int)(tok % gw);
    const int py = (int)((tok / gw) % gh);
    const int b = (int)(tok / ((long long)gw * gh));
    const float* src = img + b * sb + c * sc + (long long)(py * 16 + i) * sy + (long long)(px * 16) * sx;
    uint32_t ph[8], pl[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      __nv_bfloat16 h0, l0, h1, l1;
      split_bf16(src[(2 * j) * sx], h0, l0);
      split_bf16(src[(2 * j + 1) * sx], h1, l1);
      ph[j] = pack_bf16(h0, h1);
      pl[j] = pack_bf16(l0, l1);
    }
    const long long o = tok * 768 + c * 256 + i * 16;
    uint4* hp = reinterpret_cast<uint4*>(hi + o);
    uint4* lp = reinterpret_cast<uint4*>(lo + o);
    hp[0] = make_uint4(ph[0], ph[1], ph[2], ph[3]);
    hp[1] = make_uint4(ph[4], ph[5], ph[6], ph[7]);
    lp[0] = make_uint4(pl[0], pl[1], pl[2], pl[3]);
    lp[1] = make_uint4(pl[4], pl[5], pl[6], pl[7]);
  }
}

int launch_im2col_patch16(const float* img, long long sb, long long sc, long long sy, long long sx, int B, int gh,
                          int gw, __nv_bfloat16* hi, __nv_bfloat16* lo, cudaStream_t st) {
  const long long total = (long long)B * gh * gw * 48;
  if (total == 0) return 0;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  launch_pdl(im2col_patch16_kernel, dim3(blocks), dim3(256), 0, st, img, sb, sc, sy, sx, B, gh, gw, hi, lo);
  return cudaGetLastError() == cudaSuccess ? 0 : -6;
}

// ------------------------------------------------------------------------------------------------
// im2col for the one strided conv on the path: Conv2d(768,768,k=3,s=2,p=1) of act_postprocess[3]
// (dpt_block.py:396-408).  planes [NB,H,W,C] -> planes [NB*Ho*Wo, 9*C], k = tap*C + c.
// ------------------------------------------------------------------------------------------------
__global__ void im2col_3x3s2_kernel(const __nv_bfloat16* __restrict__ ihi, const __nv_bfloat16* __restrict__ ilo,
                                    int NB, int H, int W, int C, int Ho, int Wo, __nv_bfloat16* __restrict__ ohi,
                                    __nv_bfloat16* __restrict__ olo) {
  pdl_launch_dependents();
  pdl_wait();
  const int c8 = C >> 3;
  const long long total = (long long)NB * Ho * Wo * 9 * c8;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int cc = (int)(idx % c8);
    long long t = idx / c8;
    const int tap = (int)(t % 9);
    t /= 9;
    const int wo = (int)(t % Wo);
    const int ho = (int)((t / Wo) % Ho);
    const int nb = (int)(t / ((long long)Wo * Ho));
    const int h = ho * 2 + tap / 3 - 1, w = wo * 2 + tap % 3 - 1;
    uint4 vh = make_uint4(0, 0, 0, 0), vl = vh;
    if (h >= 0 && h < H && w >= 0 && w < W) {
      const long long src = (((long long)nb * H + h) * W + w) * C + cc * 8;
      vh = *reinterpret_cast<const uint4*>(ihi + src);
      vl = *reinterpret_cast<const uint4*>(ilo + src);
    }
    const long long dst = t * (9LL * C) + (long long)tap * C + cc * 8;
    *reinterpret_cast<uint4*>(ohi + dst) = vh;
    *reinterpret_cast<uint4*>(olo + dst) = vl;
  }
}

int launch_im2col_3x3s2(const __nv_bfloat16* ihi, const __nv_bfloat16* ilo, int NB, int H, int W, int C, int Ho, int Wo,
                        __nv_bfloat16* ohi, __nv_bfloat16* olo, cudaStream_t st) {
  const long long total = (long long)NB * Ho * Wo * 9 * (C / 8);
  if (total == 0) return 0;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  launch_pdl(im2col_3x3s2_kernel, dim3(blocks), dim3(256), 0, st, ihi, ilo, NB, H, W, C, Ho, Wo, ohi, olo);
  return cudaGetLastError() == cudaSuccess ? 0 : -6;
}

// ------------------------------------------------------------------------------------------------
// Bilinear x2 upsample, align_corners=True (F.interpolate in dpt_block.py:214-215, Interpolate :246-253),
// channels-last fp32 [NB,H,W,C] -> fp32 and/or split-bf16 planes [NB,2H,2W,C].  Index/weight arithmetic
// follows ATen's upsample_bilinear2d (scale = (in-1)/(out-1); src = scale*dst; lambda1 = src - floor).
// ------------------------------------------------------------------------------------------------
// Grid: x = 256-thread slabs of one output row's (pixel, 4-channel group) items, y = output row, z = image: the row
// quantities (h0, vertical weights) are per block, the per-item index math is one 32-bit divide (a shift when C/8 is a power
// of two: C = 128 / 256 on this path).  Round 1's flat 64-bit index (five 64-bit div / mod per item) ran at 0.20 of the
// HBM peak.  The 4 source float4 of neighbouring items overlap and come from L1 / L2.
__global__ void __launch_bounds__(256) upsample2x_kernel(const float* __restrict__ x, int H, int W, int C, float* __restrict__ out,
                                                         __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, int Ho,
                                                         int Wo, int c8_shift) {
  pdl_launch_dependents();
  pdl_wait();
  // (Ho, Wo) <= (2H, 2W): the output may be cropped (dust3r/heads/dpt_head.py:56 crops refinenet4's output to the next
  // level's size when the patch grid is odd); the interpolation grid is always that of the full 2H x 2W image.
  // One item = one output pixel x 8 channels: eight 16-byte loads in flight per thread, 16-byte plane stores.
  const int c8 = C >> 3;
  const unsigned item = blockIdx.x * 256u + threadIdx.x;
  if (item >= (unsigned)(Wo * c8)) return;
  const int wo = c8_shift >= 0 ? (int)(item >> c8_shift) : (int)(item / (unsigned)c8);
  const int c = (int)(item - (unsigned)wo * (unsigned)c8) << 3;
  const int ho = blockIdx.y, nb = blockIdx.z;
  const float sh = (2 * H > 1) ? (float)(H - 1) / (float)(2 * H - 1) : 0.f;
  const float sw = (2 * W > 1) ? (float)(W - 1) / (float)(2 * W - 1) : 0.f;
  const float hr = sh * ho, wr = sw * wo;
  const int h0 = (int)hr, w0 = (int)wr;
  const int hp = (h0 < H - 1) ? 1 : 0, wp = (w0 < W - 1) ? 1 : 0;
  const float h1l = hr - h0, h0l = 1.f - h1l, w1l = wr - w0, w0l = 1.f - w1l;
  const float* base = x + (((long long)nb * H + h0) * W + w0) * C + c;
  float4 v[4][2];
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    v[0][k] = *reinterpret_cast<const float4*>(base + 4 * k);
    v[1][k] = *reinterpret_cast<const float4*>(base + (long long)wp * C + 4 * k);
    v[2][k] = *reinterpret_cast<const float4*>(base + (long long)hp * W * C + 4 * k);
    v[3][k] = *reinterpret_cast<const float4*>(base + (long long)hp * W * C + (long long)wp * C + 4 * k);
  }
  float4 y[2];
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    y[k].x = h0l * (w0l * v[0][k].x + w1l * v[1][k].x) + h1l * (w0l * v[2][k].x + w1l * v[3][k].x);
    y[k].y = h0l * (w0l * v[0][k].y + w1l * v[1][k].y) + h1l * (w0l * v[2][k].y + w1l * v[3][k].y);
    y[k].z = h0l * (w0l * v[0][k].z + w1l * v[1][k].z) + h1l * (w0l * v[2][k].z + w1l * v[3][k].z);
    y[k].w = h0l * (w0l * v[0][k].w + w1l * v[1][k].w) + h1l * (w0l * v[2][k].w + w1l * v[3][k].w);
  }
  const long long o = (((long long)nb * Ho + ho) * Wo + wo) * C + c;
  if (out) {
    *reinterpret_cast<float4*>(out + o) = y[0];
    *reinterpret_cast<float4*>(out + o + 4) = y[1];
  }
  if (hi) {
    uint32_t h[4], l[4];
    split2_bf16(y[0].x, y[0].y, h[0], l[0]);
    split2_bf16(y[0].z, y[0].w, h[1], l[1]);
    split2_bf16(y[1].x, y[1].y, h[2], l[2]);
    split2_bf16(y[1].z, y[1].w, h[3], l[3]);
    *reinterpret_cast<uint4*>(hi + o) = make_uint4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<uint4*>(lo + o) = make_uint4(l[0], l[1], l[2], l[3]);
  }
}

int launch_upsample2x(const float* x, int NB, int H, int W, int C, float* out, __nv_bfloat16* hi, __nv_bfloat16* lo,
                      cudaStream_t st, int Ho, int Wo) {
  if (C % 8) { set_error("upsample2x: C %% 8 != 0"); return -1; }
  if (Ho <= 0) Ho = 2 * H;
  if (Wo <= 0) Wo = 2 * W;
  if (Ho > 2 * H || Wo > 2 * W) { set_error("upsample2x: output %dx%d larger than 2x input", Ho, Wo); return -1; }
  if (NB <= 0 || Ho == 0 || Wo == 0) return 0;
  if (Ho > 65535 || NB > 65535) { set_error("upsample2x: %d rows x %d images exceed the grid limits", Ho, NB); return -1; }
  const int c8 = C / 8;
  int shift = -1;
  if ((c8 & (c8 - 1)) == 0) { shift = 0; while ((1 << shift) < c8) ++shift; }
  const dim3 grid((unsigned)((Wo * c8 + 255) / 256), (unsigned)Ho, (unsigned)NB);
  launch_pdl(upsample2x_kernel, grid, dim3(256), 0, st, x, H, W, C, out, hi, lo, Ho, Wo, shift);
  return cudaGetLastError() == cudaSuccess ? 0 : -6;
}

// ------------------------------------------------------------------------------------------------
// curope-compatible shim: in-place 2-D RoPE on tokens[B,N,H,D] (fp32), pos[B,N,2] int64.
// Same contract as rope_2d (croco/models/curope/curope.cpp:49-65, kernels.cu:18-81): first D/2
// channels rotate with pos[...,0] (y), last D/2 with pos[...,1] (x); pairs (d, d+D/4);
// inv_freq = fwd / base^(q/(D/4)).  One thread per (token, head, half, q).  The fused path never
// calls this (RoPE is applied in the QKV-projection epilogue); it exists for drop-in use at the
// curope boundary and as a unit-parity target.
// ------------------------------------------------------------------------------------------------
__global__ void rope2d_kernel(float* __restrict__ tokens, const long long* __restrict__ pos, long long BN, int H, int D,
                              long long stride_tok, long long stride_head, float base, float fwd) {
  pdl_launch_dependents();
  pdl_wait();
  const int Q = D >> 2;
  const long long total = BN * H * 2 * Q;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int q = (int)(idx % Q);
    long long t = idx / Q;
    const int half = (int)(t & 1);
    t >>= 1;
    const int h = (int)(t % H);
    const long long tok = t / H;
    const float p = (float)pos[tok * 2 + half];
    const float inv_freq = fwd / powf(base, (float)q / (float)Q);
    float s, c;
    sincosf(p * inv_freq, &s, &c);
    float* ptr = tokens + tok * stride_tok + h * stride_head + half * (D >> 1) + q;
    const float u = ptr[0], v = ptr[Q];
    ptr[0] = u * c - v * s;
    ptr[Q] = v * c + u * s;
  }
}

int launch_rope2d(float* tokens, const long long* pos, long long BN, int H, int D, long long stride_tok,
                  long long stride_head, float base, float fwd, cudaStream_t st) {
  if (D % 4) { set_error("rope2d: D %% 4 != 0"); return -1; }
  const long long total = BN * H * (D / 2);
  if (total == 0) return 0;
  long long blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  launch_pdl(rope2d_kernel, dim3((int)blocks), dim3(256), 0, st, tokens, pos, BN, H, D, stride_tok, stride_head, base, fwd);
  return cudaGetLastError() == cudaSuccess ? 0 : -6;
}

}  // namespace s3r
