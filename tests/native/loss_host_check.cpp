// TEST HARNESS (not a product path): the per-pixel arithmetic of the criteria (spann3r_b200/csrc/loss_math.cuh) and the
// order-preserving keys of focal_math.cuh, compiled for the CPU and exposed over arrays, plus the exact lower median of
// one stage value kind run sequentially with the same 4 x 8-bit radix select the median kernels of csrc/loss.cu perform.
#include <vector>

#include "../../spann3r_b200/csrc/loss_math.cuh"

using namespace s3r;

extern "C" {

void loss_norm3(const float* v, long long n, float* out) {
  for (long long i = 0; i < n; ++i) out[i] = lossm::norm3(v[3 * i], v[3 * i + 1], v[3 * i + 2]);
}

void loss_align(const float* p, long long n, float factor, float shift, float mul, float* out) {
  const lossm::Align a{factor, shift, mul};
  for (long long i = 0; i < n; ++i) lossm::align(p + 3 * i, a, out + 3 * i);
}

void loss_stage_value(const float* p, long long n, float factor, float shift, const float* centre, int kind, float* out) {
  for (long long i = 0; i < n; ++i) out[i] = lossm::stage_value(p + 3 * i, factor, shift, centre, kind);
}

void loss_l21(const float* pr, const float* gt, long long n, float* u, float* d) {
  for (long long i = 0; i < n; ++i) d[i] = lossm::l21(pr + 3 * i, gt + 3 * i, u + 3 * i);
}

void loss_conf_term(const float* d, const float* c, long long n, float alpha, float* out) {
  for (long long i = 0; i < n; ++i) out[i] = lossm::conf_term(d[i], c[i], alpha);
}

void loss_pred_grad(const float* p, const float* u, const float* d, long long n, double g_d, double scale, double coef,
                    int log1p_mode, float* g) {
  for (long long i = 0; i < n; ++i) lossm::pred_grad(p + 3 * i, u + 3 * i, d[i], g_d, scale, coef, log1p_mode, g + 3 * i);
}

void loss_order_key(const float* v, long long n, uint32_t* out) {
  for (long long i = 0; i < n; ++i) out[i] = focal::order_key(v[i]);
}

void loss_key_value(const uint32_t* k, long long n, float* out) {
  for (long long i = 0; i < n; ++i) out[i] = focal::key_value(k[i]);
}

// lower median (torch.nanmedian) of stage_value(kind) over the valid points p[n, 3]; NaN when no value is left
float loss_median(const float* p, const uint8_t* valid, long long n, float factor, float shift, const float* centre,
                  int kind) {
  uint32_t prefix = 0;
  long long k = 0;
  for (int pass = 0; pass < 4; ++pass) {
    const int shift_bits = 24 - 8 * pass;
    int hist[256] = {0};
    for (long long i = 0; i < n; ++i) {
      if (!valid[i]) continue;
      const float v = lossm::stage_value(p + 3 * i, factor, shift, centre, kind);
      if (v != v) continue;
      const uint32_t key = focal::order_key(v);
      if (pass > 0 && (key >> (shift_bits + 8)) != prefix) continue;
      ++hist[(key >> shift_bits) & 255];
    }
    if (pass == 0) {
      long long total = 0;
      for (int b = 0; b < 256; ++b) total += hist[b];
      if (total == 0) return nanf("");
      k = (total - 1) / 2;
    }
    prefix = (prefix << 8) | (uint32_t)focal::radix_pick(hist, k);
  }
  return focal::key_value(prefix);
}

}  // extern "C"
