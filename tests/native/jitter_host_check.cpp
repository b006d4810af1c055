// TEST HARNESS (not a product path): compiles the product's device math header, spann3r_b200/csrc/jitter_math.cuh,
// with g++ so tests/test_train_views.py can check every ColorJitter rule against Pillow / torchvision without a GPU,
// and run one view through the same two-pass order the kernel of csrc/jitter.cu runs.
#include "../../spann3r_b200/csrc/jitter_math.cuh"

using namespace s3r::jitter;

extern "C" {

// rgb [n, 3] -> hsv [n, 3]
void jh_rgb_to_hsv(const unsigned char* rgb, long long n, unsigned char* hsv) {
  for (long long i = 0; i < n; ++i) {
    int h, s, v;
    rgb_to_hsv(rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2], h, s, v);
    hsv[3 * i] = (unsigned char)h, hsv[3 * i + 1] = (unsigned char)s, hsv[3 * i + 2] = (unsigned char)v;
  }
}

// hsv [n, 3] -> rgb [n, 3]
void jh_hsv_to_rgb(const unsigned char* hsv, long long n, unsigned char* rgb) {
  for (long long i = 0; i < n; ++i) {
    int r, g, b;
    hsv_to_rgb(hsv[3 * i], hsv[3 * i + 1], hsv[3 * i + 2], r, g, b);
    rgb[3 * i] = (unsigned char)r, rgb[3 * i + 1] = (unsigned char)g, rgb[3 * i + 2] = (unsigned char)b;
  }
}

// rgb [n, 3] -> rgb [n, 3] with the hue shifted
void jh_shift_hue(const unsigned char* rgb, long long n, int hue_shift, unsigned char* out) {
  for (long long i = 0; i < n; ++i) {
    int r = rgb[3 * i], g = rgb[3 * i + 1], b = rgb[3 * i + 2];
    shift_hue(r, g, b, hue_shift);
    out[3 * i] = (unsigned char)r, out[3 * i + 1] = (unsigned char)g, out[3 * i + 2] = (unsigned char)b;
  }
}

void jh_luma(const unsigned char* rgb, long long n, unsigned char* out) {
  for (long long i = 0; i < n; ++i) out[i] = (unsigned char)luma(rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2]);
}

void jh_blend(const unsigned char* in1, const unsigned char* in2, long long n, float alpha, unsigned char* out) {
  for (long long i = 0; i < n; ++i) out[i] = (unsigned char)blend(in1[i], in2[i], alpha);
}

int jh_contrast_mean(long long sum_l, long long count) { return contrast_mean(sum_l, count); }

// One view: rgb [h, w, 3] -> jitter (order, skip, factors b / c / s, hue shift) -> ImgNorm -> img [3, h, w] fp32, in the
// kernel's two passes (the mean of L over the image the ops before contrast leave, then every op in order).
void jh_view(const unsigned char* rgb, int h, int w, const int* order, int skip, const float* factors, int hue_shift,
             float* img) {
  Params p;
  for (int k = 0; k < 4; ++k) p.order[k] = order[k];
  p.skip = skip;
  for (int k = 0; k < 3; ++k) p.factor[k] = factors[k];
  p.hue_shift = hue_shift;
  const long long n = (long long)h * w;
  const int kc = contrast_pos(p);
  int mean = 0;
  if (kc < 4) {
    long long sum = 0;
    for (long long i = 0; i < n; ++i) {
      int r = rgb[3 * i], g = rgb[3 * i + 1], b = rgb[3 * i + 2];
      apply_ops(p, 0, kc, 0, r, g, b);
      sum += luma(r, g, b);
    }
    mean = contrast_mean(sum, n);
  }
  for (long long i = 0; i < n; ++i) {
    int c[3] = {rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2]};
    apply_ops(p, 0, 4, mean, c[0], c[1], c[2]);
    for (int k = 0; k < 3; ++k) img[k * n + i] = ((float)c[k] / 255.0f - 0.5f) / 0.5f;
  }
}

}  // extern "C"
