// Scalar math of torchvision's ColorJitter on PIL images (csrc/jitter.cu): the four Pillow operations it chains, one
// pixel at a time.  `__host__ __device__` with no CUDA dependencies, so tests/native/jitter_host_check.cpp compiles THIS
// header with g++ (-ffp-contract=off) and tests/test_train_views.py checks it exhaustively against Pillow itself.
//
// The rules, each restated from Pillow's documented behaviour and pinned by those tests:
//   L(r, g, b)          = (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16                 ITU-R 601-2 luma, 16-bit fixed
//   blend(a, b, alpha)  = t = a + alpha * (b - a) in fp32 (alpha as torchvision drew it, an fp32 value);
//                         0 <= alpha <= 1: trunc(t); otherwise t clamped to [0, 255] and truncated     (Image.blend)
//   brightness          = blend(0, x, f)
//   contrast            = blend(m, x, f), m = int(sum(L) / count + 0.5) over the current image      (ImageStat mean)
//   saturation          = blend(L(pixel), x, f) per channel
//   hue                 = RGB -> HSV (colorsys' formulas in Pillow's fp32 / fp64 mix), h += shift mod 256, HSV -> RGB
// Every fp32 / fp64 operation is an explicitly rounded intrinsic on the device, so nothing is contracted into an FMA.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define S3R_JHD __host__ __device__ __forceinline__
#else
#define S3R_JHD inline
#endif

namespace s3r {
namespace jitter {

enum Op { kBrightness = 0, kContrast = 1, kSaturation = 2, kHue = 3 };

#if defined(__CUDA_ARCH__)
S3R_JHD float fadd(float a, float b) { return __fadd_rn(a, b); }
S3R_JHD float fsub(float a, float b) { return __fsub_rn(a, b); }
S3R_JHD float fmul(float a, float b) { return __fmul_rn(a, b); }
S3R_JHD float fdiv(float a, float b) { return __fdiv_rn(a, b); }
S3R_JHD double dadd(double a, double b) { return __dadd_rn(a, b); }
S3R_JHD double dsub(double a, double b) { return __dsub_rn(a, b); }
S3R_JHD double dmul(double a, double b) { return __dmul_rn(a, b); }
S3R_JHD double ddiv(double a, double b) { return __ddiv_rn(a, b); }
#else
S3R_JHD float fadd(float a, float b) { return a + b; }
S3R_JHD float fsub(float a, float b) { return a - b; }
S3R_JHD float fmul(float a, float b) { return a * b; }
S3R_JHD float fdiv(float a, float b) { return a / b; }
S3R_JHD double dadd(double a, double b) { return a + b; }
S3R_JHD double dsub(double a, double b) { return a - b; }
S3R_JHD double dmul(double a, double b) { return a * b; }
S3R_JHD double ddiv(double a, double b) { return a / b; }
#endif

S3R_JHD int clamp8(int v) { return v <= 0 ? 0 : (v < 256 ? v : 255); }

S3R_JHD int luma(int r, int g, int b) { return (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16; }

// Image.blend of one channel: in1 the degenerate value, in2 the image's.
S3R_JHD int blend(int in1, int in2, float alpha) {
  const float t = fadd((float)in1, fmul(alpha, (float)(in2 - in1)));
  if (alpha >= 0.0f && alpha <= 1.0f) return (int)t;        // t stays within [min(in1, in2), max(in1, in2)]
  if (t <= 0.0f) return 0;
  if (t >= 255.0f) return 255;
  return (int)t;
}

// ImageStat's mean of the L image, rounded as ImageEnhance.Contrast rounds it.
S3R_JHD int contrast_mean(long long sum_l, long long count) {
  return (int)dadd(ddiv((double)sum_l, (double)count), 0.5);
}

S3R_JHD void rgb_to_hsv(int r, int g, int b, int& h, int& s, int& v) {
  const int mx = r > g ? (r > b ? r : b) : (g > b ? g : b);
  const int mn = r < g ? (r < b ? r : b) : (g < b ? g : b);
  v = mx;
  if (mx == mn) {
    h = s = 0;
    return;
  }
  const float cr = (float)(mx - mn);
  const float sf = fdiv(cr, (float)mx);
  const float rc = fdiv((float)(mx - r), cr), gc = fdiv((float)(mx - g), cr), bc = fdiv((float)(mx - b), cr);
  float hf;
  if (r == mx) hf = fsub(bc, gc);
  else if (g == mx) hf = (float)dsub(dadd(2.0, (double)rc), (double)bc);
  else hf = (float)dsub(dadd(4.0, (double)gc), (double)rc);
  hf = (float)fmod(dadd(ddiv((double)hf, 6.0), 1.0), 1.0);
  h = clamp8((int)dmul((double)hf, 255.0));
  s = clamp8((int)dmul((double)sf, 255.0));
}

S3R_JHD void hsv_to_rgb(int h, int s, int v, int& r, int& g, int& b) {
  if (s == 0) {
    r = g = b = v;
    return;
  }
  const double h6 = ddiv(dmul((double)h, 6.0), 255.0);
  const int i = (int)floor(h6);                               // 0..6
  const float f = (float)dsub(h6, (double)i);
  const float fs = (float)ddiv((double)s, 255.0);
  const double dv = (double)v;
  const int p = clamp8((int)round(dmul(dv, dsub(1.0, (double)fs))));
  const int q = clamp8((int)round(dmul(dv, dsub(1.0, (double)fmul(fs, f)))));
  const int t = clamp8((int)round(dmul(dv, dsub(1.0, dmul((double)fs, dsub(1.0, (double)f))))));
  switch (i % 6) {
    case 0: r = v, g = t, b = p; break;
    case 1: r = q, g = v, b = p; break;
    case 2: r = p, g = v, b = t; break;
    case 3: r = p, g = q, b = v; break;
    case 4: r = t, g = p, b = v; break;
    default: r = v, g = p, b = q; break;
  }
}

// hue_shift: (int32) trunc(hue_factor * 255), added to the uint8 hue mod 256.
S3R_JHD void shift_hue(int& r, int& g, int& b, int hue_shift) {
  int h, s, v;
  rgb_to_hsv(r, g, b, h, s, v);
  hsv_to_rgb((h + hue_shift) & 255, s, v, r, g, b);
}

// One view's drawn parameters.  order: a permutation of the four ops; skip bit k: op k's factor is None.
struct Params {
  int order[4];
  int skip;
  float factor[3];     // brightness, contrast, saturation
  int hue_shift;
};

// Position of contrast in the order, or 4 when it does not run: the ops before it form the image it takes the mean of.
S3R_JHD int contrast_pos(const Params& p) {
  int pos = 4;
  for (int k = 3; k >= 0; --k)
    if (p.order[k] == kContrast) pos = k;
  return (p.skip & (1 << kContrast)) ? 4 : pos;
}

// Ops order[k0..k1) on one pixel, skipping the None ones; contrast blends toward `mean`.  The loop runs over all four
// slots so that `order` is only indexed by constants (registers, not a local-memory array, on the device).
S3R_JHD void apply_ops(const Params& p, int k0, int k1, int mean, int& r, int& g, int& b) {
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (int k = 0; k < 4; ++k) {
    const int op = p.order[k];
    if (k < k0 || k >= k1 || (p.skip & (1 << op))) continue;
    switch (op) {
      case kBrightness:
        r = blend(0, r, p.factor[0]), g = blend(0, g, p.factor[0]), b = blend(0, b, p.factor[0]);
        break;
      case kContrast:
        r = blend(mean, r, p.factor[1]), g = blend(mean, g, p.factor[1]), b = blend(mean, b, p.factor[1]);
        break;
      case kSaturation: {
        const int l = luma(r, g, b);
        r = blend(l, r, p.factor[2]), g = blend(l, g, p.factor[2]), b = blend(l, b, p.factor[2]);
        break;
      }
      default:
        shift_hue(r, g, b, p.hue_shift);
        break;
    }
  }
}

}  // namespace jitter
}  // namespace s3r
