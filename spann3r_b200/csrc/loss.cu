// Spann3R's training and test criteria on the GPU: Regr3D_t and its shift / scale invariant variants, and ConfLoss_t
// over them (spann3r/loss.py:129-369), forward and backward.
//
// One call covers F views of B sequences.  Pred slot k < F-1 is the left prediction L[k] of pair k (frame k), slot
// F-1+i the right prediction R[i] of pair i (frame i+1).  Every frame f has one "primary" slot, L[f] or R[F-2] for the
// last frame: the primary slots are the pred list `pr_l + [pr_r[-1]]` that the norm factor and the medians read.
// A device table of the per-view pointers lives in the workspace, so every kernel walks all frames from one launch and
// the number of launches does not depend on F:
//   loss_prep_kernel           gt = inv(pose0) pts3d (fp64 inverse, fp64 product), validity (valid_mask, dist_clip on
//                              the untransformed norm), per-block fp64 sums: valid count, sum g(|gt|), sum g(|pred|)
//   loss_prep_reduce_kernel    fixed-order sums -> pooled counts, gt_factor / pr_factor per batch element
//   loss_median_hist/pick      exact lower median (torch.nanmedian) of one value kind over all valid pixels of all
//                              frames of a batch element: 4 x 8-bit radix passes on order-preserving keys, integer
//                              histograms only (3 stages for the scale-shift invariant criterion: z, centre, norm)
//   loss_forward_kernel        alignment, L21, conf term; per-block fp64 partials; optional aligned maps
//   loss_forward_reduce_kernel fixed-order sums -> loss, factor_loss, details, monitoring, backward coefficients
//   loss_backward_kernel       dLoss/dpred for every slot and dLoss/dconf from the two upstream scalars
// No float atomics anywhere: results are bitwise reproducible.
#include "../../include/spann3r_b200.h"
#include "common.cuh"
#include "gemm.cuh"
#include "loss_math.cuh"

#include <vector>

namespace s3r {

namespace {

constexpr int kThreads = 256;
constexpr int kPixPerBlock = 2048;
constexpr int kPrepVals = 3;     // count, sum g(|gt|), sum g(|pred|)
constexpr int kLossVals = 5;     // sum d, sum conf term, sum conf (valid), sum conf (all), sum w(c) u.p / d
constexpr int kHist = 260;       // 256 bins + prefix, k_lo, k_hi, state
constexpr int kPerB = 16;        // state doubles per batch element (see StateB)
constexpr double kFactorMin = 1e-8;

// per batch element state (doubles): factors, medians (gt: 3..7, pred: 8..12 = kind 0 z, 1..3 centre, 4 scale),
// backward coefficients of the norm factor
enum StateB { SB_FG = 0, SB_FP = 1, SB_FP_RAW = 2, SB_GMED = 3, SB_PMED = 8, SB_K1 = 13, SB_K2 = 14 };

struct Cfg {
  int F, B, S, nblk;
  long long P;
  int norm_mode, fix_first, gt_scale, shift_inv, scale_inv, conf_loss, has_conf, has_clip;
  float alpha, dist_clip;
};

struct Ws {
  const float** gt_in;      // [F]
  const uint8_t** valid_in; // [F]
  const float** pred;       // [S]
  const float** conf;       // [S]
  float* gt;                // [F, B, P, 3] transformed gt
  uint8_t* valid;           // [F, B, P]
  double* prep;             // [F, B, nblk, kPrepVals]
  double* state;            // [F] pooled counts, [1] pooled norm count, [B * kPerB], [S] term weights
  int* hist;                // [6 B, kHist]
  double* part;             // [S, B, nblk, kLossVals]
};

inline size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

struct Layout {
  size_t table, gt, valid, prep, state, hist, part, total;
};

Layout layout(int F, int B, long long P, int nblk) {
  const int S = 2 * (F - 1);
  Layout L;
  size_t o = 0;
  L.table = o; o = align_up(o + sizeof(void*) * (size_t)(2 * F + 2 * S));
  L.gt = o;    o = align_up(o + sizeof(float) * 3 * (size_t)F * B * P);
  L.valid = o; o = align_up(o + (size_t)F * B * P);
  L.prep = o;  o = align_up(o + sizeof(double) * (size_t)F * B * nblk * kPrepVals);
  L.state = o; o = align_up(o + sizeof(double) * (size_t)(F + 1 + B * kPerB + S));
  L.hist = o;  o = align_up(o + sizeof(int) * (size_t)6 * B * kHist);
  L.part = o;  o = align_up(o + sizeof(double) * (size_t)S * B * nblk * kLossVals);
  L.total = o;
  return L;
}

__device__ __forceinline__ int slot_frame(int k, int F) { return k < F - 1 ? k : k - (F - 1) + 1; }
__device__ __forceinline__ int primary_slot(int f, int F) { return f < F - 1 ? f : 2 * F - 3; }

// sum of K doubles over the block (256 threads), fixed order; result valid in thread 0
template <int K>
__device__ __forceinline__ void block_sum(double* v) {
  __shared__ double red[kThreads / 32][K];
#pragma unroll
  for (int i = 0; i < K; ++i)
    for (int o = 16; o > 0; o >>= 1) v[i] += __shfl_down_sync(0xffffffffu, v[i], o);
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int i = 0; i < K; ++i) red[w][i] = v[i];
  __syncthreads();
  if (threadIdx.x == 0)
#pragma unroll
    for (int i = 0; i < K; ++i) {
      double s = 0.0;
      for (int j = 0; j < kThreads / 32; ++j) s += red[j][i];
      v[i] = s;
    }
}

__device__ __forceinline__ void alignments(const Cfg& c, const double* sb, lossm::Align& ag, lossm::Align& ap) {
  ag.factor = (float)sb[SB_FG];
  ap.factor = (float)sb[SB_FP];
  ag.shift = c.shift_inv ? (float)sb[SB_GMED] : 0.f;
  ap.shift = c.shift_inv ? (float)sb[SB_PMED] : 0.f;
  ag.mul = 1.f;
  ap.mul = 1.f;
  if (c.scale_inv) {
    const float gs = (float)sb[SB_GMED + 4];
    float ps = (float)sb[SB_PMED + 4];
    if (ps == ps) ps = fminf(fmaxf(ps, 1e-3f), 1e3f);   // pred_scale.clip(1e-3, 1e3); NaN stays NaN
    if (c.gt_scale) {
      ap.mul = gs / ps;
    } else {
      ap.mul = ps / gs;
      ag.mul = gs / ps;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) loss_prep_kernel(Cfg c, Ws w, const float* __restrict__ pose0) {
  const int blk = blockIdx.x, f = blockIdx.y, b = blockIdx.z;
  __shared__ double T[12];
  if (threadIdx.x == 0) {
    // inverse of the 4x4 camera_pose[0][b] in fp64 (Gauss-Jordan, partial pivoting); rows 0..2 kept
    double a[4][8];
    for (int i = 0; i < 4; ++i)
      for (int j = 0; j < 4; ++j) {
        a[i][j] = (double)pose0[(long long)b * 16 + i * 4 + j];
        a[i][4 + j] = i == j ? 1.0 : 0.0;
      }
    for (int col = 0; col < 4; ++col) {
      int piv = col;
      for (int r = col + 1; r < 4; ++r)
        if (fabs(a[r][col]) > fabs(a[piv][col])) piv = r;
      if (piv != col)
        for (int j = 0; j < 8; ++j) {
          const double t = a[col][j];
          a[col][j] = a[piv][j];
          a[piv][j] = t;
        }
      const double inv = 1.0 / a[col][col];
      for (int j = 0; j < 8; ++j) a[col][j] *= inv;
      for (int r = 0; r < 4; ++r)
        if (r != col) {
          const double m = a[r][col];
          for (int j = 0; j < 8; ++j) a[r][j] -= m * a[col][j];
        }
    }
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 4; ++j) T[i * 4 + j] = a[i][4 + j];
  }
  __syncthreads();
  const long long img = (long long)f * c.B + b;
  const float* src = w.gt_in[f] + (long long)b * c.P * 3;
  const uint8_t* vin = w.valid_in[f] + (long long)b * c.P;
  const float* pr = w.pred[primary_slot(f, c.F)] + (long long)b * c.P * 3;
  float* dst = w.gt + img * c.P * 3;
  uint8_t* vout = w.valid + img * c.P;
  const bool lg = c.norm_mode == 2;
  double acc[kPrepVals] = {0.0, 0.0, 0.0};
  const long long p1 = min(c.P, (long long)(blk + 1) * kPixPerBlock);
  for (long long p = (long long)blk * kPixPerBlock + threadIdx.x; p < p1; p += kThreads) {
    const float x = src[3 * p], y = src[3 * p + 1], z = src[3 * p + 2];
    float g[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) g[i] = (float)(T[i * 4] * x + T[i * 4 + 1] * y + T[i * 4 + 2] * z + T[i * 4 + 3]);
    dst[3 * p] = g[0];
    dst[3 * p + 1] = g[1];
    dst[3 * p + 2] = g[2];
    bool v = vin[p] != 0;
    if (c.has_clip) v = v && lossm::norm3(x, y, z) <= c.dist_clip;
    vout[p] = v ? 1 : 0;
    if (v) {
      const float ng = lossm::norm3(g[0], g[1], g[2]);
      const float np = lossm::norm3(pr[3 * p], pr[3 * p + 1], pr[3 * p + 2]);
      acc[0] += 1.0;
      acc[1] += (double)(lg ? log1pf(ng) : ng);
      acc[2] += (double)(lg ? log1pf(np) : np);
    }
  }
  block_sum<kPrepVals>(acc);
  if (threadIdx.x == 0) {
    double* o = w.prep + (img * c.nblk + blk) * kPrepVals;
    for (int i = 0; i < kPrepVals; ++i) o[i] = acc[i];
  }
}

__global__ void __launch_bounds__(kThreads) loss_prep_reduce_kernel(Cfg c, Ws w) {
  const int pairs = c.F * c.B;
  for (int q = threadIdx.x; q < pairs; q += kThreads) {     // one thread per (frame, b): its blocks in order
    double* o = w.prep + (long long)q * c.nblk * kPrepVals;
    double s[kPrepVals] = {0.0, 0.0, 0.0};
    for (int k = 0; k < c.nblk; ++k)
      for (int i = 0; i < kPrepVals; ++i) s[i] += o[k * kPrepVals + i];
    for (int i = 0; i < kPrepVals; ++i) o[i] = s[i];
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  double* st = w.state;
  const int nf = c.fix_first ? 1 : c.F;      // frames of the norm factor
  double ntot = 0.0;
  for (int f = 0; f < c.F; ++f) {
    double n = 0.0;
    for (int b = 0; b < c.B; ++b) n += w.prep[((long long)f * c.B + b) * c.nblk * kPrepVals];
    st[f] = n;
    if (f < nf) ntot += n;
  }
  st[c.F] = ntot;
  const bool norm = c.norm_mode != 0;
  for (int b = 0; b < c.B; ++b) {
    double sg = 0.0, sp = 0.0;
    for (int f = 0; f < nf; ++f) {
      const double* o = w.prep + ((long long)f * c.B + b) * c.nblk * kPrepVals;
      sg += o[1];
      sp += o[2];
    }
    // norm_factor = sum / (pooled count + 1e-8), clipped at 1e-8, held in fp32 as the reference holds it; a NaN
    // factor (a NaN point among the valid ones) stays NaN, as torch's clip keeps it, where fmax would give 1e-8
    const double fg = sg / (ntot + 1e-8), fp = sp / (ntot + 1e-8);
    double* sb = st + c.F + 1 + b * kPerB;
    for (int i = 0; i < kPerB; ++i) sb[i] = 0.0;
    sb[SB_FG] = (norm && !c.gt_scale) ? (double)(float)(fg == fg ? fmax(fg, kFactorMin) : fg) : 1.0;
    sb[SB_FP] = norm ? (double)(float)(fp == fp ? fmax(fp, kFactorMin) : fp) : 1.0;
    sb[SB_FP_RAW] = fp;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// median stages: stage 0 = z (jobs 2B), 1 = centre x, y, z (jobs 6B), 2 = norm about the centre (jobs 2B)
__device__ __forceinline__ void job_of(int stage, int j, int B, int& set, int& b, int& kind) {
  if (stage == 1) {
    set = j / (3 * B);
    kind = 1 + (j / B) % 3;
  } else {
    set = j / B;
    kind = stage == 0 ? 0 : 4;
  }
  b = j % B;
}

__global__ void __launch_bounds__(kThreads) loss_median_hist_kernel(Cfg c, Ws w, int stage, int pass) {
  __shared__ int hist[256];
  const int blk = blockIdx.x, f = blockIdx.y, j = blockIdx.z;
  int set, b, kind;
  job_of(stage, j, c.B, set, b, kind);
  int* sc = w.hist + (long long)j * kHist;
  hist[threadIdx.x] = 0;
  __syncthreads();
  if (sc[259] >= 0) {
    const double* sb = w.state + c.F + 1 + b * kPerB;
    const int mo = set == 0 ? SB_GMED : SB_PMED;
    const float factor = (float)sb[set == 0 ? SB_FG : SB_FP];
    const float shift = c.shift_inv ? (float)sb[mo] : 0.f;
    const float centre[3] = {(float)sb[mo + 1], (float)sb[mo + 2], (float)sb[mo + 3]};
    const long long img = (long long)f * c.B + b;
    const float* pts = set == 0 ? w.gt + img * c.P * 3 : w.pred[primary_slot(f, c.F)] + (long long)b * c.P * 3;
    const uint8_t* v = w.valid + img * c.P;
    const int shift_bits = 24 - 8 * pass;
    const uint32_t prefix = (uint32_t)sc[256];
    const long long p1 = min(c.P, (long long)(blk + 1) * kPixPerBlock);
    for (long long p = (long long)blk * kPixPerBlock + threadIdx.x; p < p1; p += kThreads) {
      if (!v[p]) continue;
      const float val = lossm::stage_value(pts + 3 * p, factor, shift, centre, kind);
      if (val != val) continue;
      const uint32_t key = focal::order_key(val);
      if (pass > 0 && (key >> (shift_bits + 8)) != prefix) continue;
      atomicAdd(&hist[(key >> shift_bits) & 255], 1);
    }
  }
  __syncthreads();
  if (hist[threadIdx.x]) atomicAdd(&sc[threadIdx.x], hist[threadIdx.x]);
}

__global__ void loss_median_pick_kernel(Cfg c, Ws w, int stage, int pass, int jobs) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= jobs) return;
  int set, b, kind;
  job_of(stage, j, c.B, set, b, kind);
  int* sc = w.hist + (long long)j * kHist;
  if (sc[259] >= 0) {
    long long k = ((long long)(uint32_t)sc[258] << 32) | (uint32_t)sc[257];
    if (pass == 0) {
      long long n = 0;
      for (int i = 0; i < 256; ++i) n += sc[i];
      if (n == 0) sc[259] = -1;
      k = (n - 1) / 2;            // the lower median, as torch.nanmedian
    }
    if (sc[259] >= 0) {
      const int bin = focal::radix_pick(sc, k);
      sc[256] = (int)((((uint32_t)sc[256]) << 8) | (uint32_t)bin);
      sc[257] = (int)(uint32_t)(k & 0xffffffffll);
      sc[258] = (int)(uint32_t)(k >> 32);
    }
  }
  for (int i = 0; i < 256; ++i) sc[i] = 0;
  if (pass == 3) {
    const float m = sc[259] >= 0 ? focal::key_value((uint32_t)sc[256]) : nanf("");
    w.state[c.F + 1 + b * kPerB + (set == 0 ? SB_GMED : SB_PMED) + kind] = (double)m;
    sc[256] = sc[257] = sc[258] = sc[259] = 0;   // ready for the next stage
  }
}

// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) loss_forward_kernel(Cfg c, Ws w, float* __restrict__ gt_out,
                                                                float* __restrict__ pred_out) {
  const int blk = blockIdx.x, k = blockIdx.y, b = blockIdx.z;
  const int f = slot_frame(k, c.F);
  const double* sb = w.state + c.F + 1 + b * kPerB;
  lossm::Align ag, ap;
  alignments(c, sb, ag, ap);
  const long long img = (long long)f * c.B + b;
  const float* x = w.pred[k] + (long long)b * c.P * 3;
  const float* cf = c.has_conf ? w.conf[k] + (long long)b * c.P : nullptr;
  const float* gt = w.gt + img * c.P * 3;
  const uint8_t* v = w.valid + img * c.P;
  float* po = pred_out ? pred_out + ((long long)k * c.B + b) * c.P * 3 : nullptr;
  float* go = (gt_out && primary_slot(f, c.F) == k) ? gt_out + img * c.P * 3 : nullptr;
  double acc[kLossVals] = {0.0, 0.0, 0.0, 0.0, 0.0};
  const long long p1 = min(c.P, (long long)(blk + 1) * kPixPerBlock);
  for (long long p = (long long)blk * kPixPerBlock + threadIdx.x; p < p1; p += kThreads) {
    float pr[3], g[3], u[3];
    lossm::align(x + 3 * p, ap, pr);
    const float cv = cf ? cf[p] : 1.f;
    if (cf) acc[3] += (double)cv;
    if (po) {
      po[3 * p] = pr[0];
      po[3 * p + 1] = pr[1];
      po[3 * p + 2] = pr[2];
    }
    if (!go && !v[p]) continue;
    lossm::align(gt + 3 * p, ag, g);
    if (go) {
      go[3 * p] = g[0];
      go[3 * p + 1] = g[1];
      go[3 * p + 2] = g[2];
    }
    if (!v[p]) continue;
    const float d = lossm::l21(pr, g, u);
    acc[0] += (double)d;
    if (cf) {
      acc[1] += (double)lossm::conf_term(d, cv, c.alpha);
      acc[2] += (double)cv;
    }
    if (d > 0.f) {
      const float* xp = x + 3 * p;
      const double ux = (double)u[0] * xp[0] + (double)u[1] * xp[1] + (double)u[2] * xp[2];
      acc[4] += (c.conf_loss ? (double)cv : 1.0) * ux / (double)d;
    }
  }
  block_sum<kLossVals>(acc);
  if (threadIdx.x == 0) {
    double* o = w.part + (((long long)k * c.B + b) * c.nblk + blk) * kLossVals;
    for (int i = 0; i < kLossVals; ++i) o[i] = acc[i];
  }
}

__global__ void __launch_bounds__(kThreads) loss_forward_reduce_kernel(Cfg c, Ws w, double* __restrict__ res) {
  const int pairs = c.S * c.B;
  for (int q = threadIdx.x; q < pairs; q += kThreads) {
    double* o = w.part + (long long)q * c.nblk * kLossVals;
    double s[kLossVals] = {0.0, 0.0, 0.0, 0.0, 0.0};
    for (int k = 0; k < c.nblk; ++k)
      for (int i = 0; i < kLossVals; ++i) s[i] += o[k * kLossVals + i];
    for (int i = 0; i < kLossVals; ++i) o[i] = s[i];
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  const int F = c.F, S = c.S, B = c.B;
  double* st = w.state;
  double* wk = st + F + 1 + B * kPerB;
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  double loss = 0.0, conf_mean = 0.0, left = 0.0, right = 0.0, cleft = 0.0, cright = 0.0, empty = 0.0;
  double m[2] = {0.0, 0.0}, cl[2] = {0.0, 0.0};
  for (int k = 0; k < S; ++k) {
    double sd = 0.0, scl = 0.0, scv = 0.0, sca = 0.0;
    for (int b = 0; b < B; ++b) {
      const double* o = w.part + ((long long)k * B + b) * c.nblk * kLossVals;
      sd += o[0];
      scl += o[1];
      scv += o[2];
      sca += o[3];
    }
    const double n = st[slot_frame(k, F)];
    if (n == 0.0) empty += 1.0;
    // per-term mean: 'mean' reduction gives 0 for an empty term, 'none' + numpy mean gives NaN
    const double mk = n > 0.0 ? sd / n : (c.conf_loss ? nan : 0.0);
    const double clk = n > 0.0 ? scl / n : nan;
    if (c.conf_loss) {
      wk[k] = n > 0.0 ? 2.0 / (S * n) : 0.0;
      loss += 2.0 * clk;
      conf_mean += n > 0.0 ? scv / n : nan;
    } else {
      wk[k] = n > 0.0 ? 1.0 / n : 0.0;
      loss += mk;
    }
    if (k < 2) {
      m[k] = mk;
      cl[k] = 2.0 * clk;
    }
    const double call = sca / ((double)B * (double)c.P);
    if (k >= 1 && k <= F - 2) {            // L[1..F-2]
      left += mk;
      cleft += call;
    }
    if (k >= F - 1 && k <= 2 * F - 4) {    // R[0..F-3]
      right += mk;
      cright += call;
    }
  }
  if (c.conf_loss) {
    loss /= S;
    conf_mean /= S;
  }
  // factor_loss: pr_factor[pr_factor > gt_factor] (elementwise over b) broadcast against gt_factor [B,1,1,1]
  const bool factors = c.norm_mode != 0 && !c.gt_scale;
  double fl = 0.0, kcount = factors ? 0.0 : -1.0;
  if (factors) {
    for (int j = 0; j < B; ++j) {
      const double* sj = st + F + 1 + j * kPerB;
      if ((float)sj[SB_FP] > (float)sj[SB_FG]) kcount += 1.0;
    }
    for (int j = 0; j < B; ++j) {
      double* sj = st + F + 1 + j * kPerB;
      const bool sel = (float)sj[SB_FP] > (float)sj[SB_FG];
      double g = 0.0;
      for (int b = 0; b < B && sel; ++b) {
        const double dlt = sj[SB_FP] - st[F + 1 + b * kPerB + SB_FG];
        fl += fabs(dlt);
        g += dlt > 0.0 ? 1.0 : (dlt < 0.0 ? -1.0 : 0.0);
      }
      sj[SB_K2] = kcount > 0.0 ? g / (B * kcount) : 0.0;
    }
    if (kcount > 0.0) fl /= B * kcount;
  }
  double mon[4] = {0.0, 0.0, 0.0, 0.0};
  for (int b = 0; b < B; ++b) {
    double* sb = st + F + 1 + b * kPerB;
    lossm::Align ag, ap;
    alignments(c, sb, ag, ap);
    // dLoss/dpr_factor through the points: -(mul / factor^2) sum_k w_k sum w(c) u.p / d
    double a = 0.0;
    for (int k = 0; k < S; ++k) a += wk[k] * w.part[((long long)k * B + b) * c.nblk * kLossVals + 4];
    const double fpv = sb[SB_FP];
    sb[SB_K1] = c.norm_mode != 0 ? -((double)ap.mul / (fpv * fpv)) * a : 0.0;
    if (!(c.norm_mode != 0 && sb[SB_FP_RAW] >= kFactorMin)) sb[SB_K1] = sb[SB_K2] = 0.0;   // clip active: no gradient
    float ps = (float)sb[SB_PMED + 4];
    if (ps == ps) ps = fminf(fmaxf(ps, 1e-3f), 1e3f);
    mon[0] += sb[SB_GMED];
    mon[1] += sb[SB_PMED];
    mon[2] += sb[SB_GMED + 4];
    mon[3] += (double)ps;
    double* r = res + S3R_LOSS_RES_HEADER + b * S3R_LOSS_RES_PER_B;
    r[0] = sb[SB_FG];
    r[1] = sb[SB_FP];
    r[2] = sb[SB_GMED];
    r[3] = sb[SB_PMED];
    r[4] = sb[SB_GMED + 4];
    r[5] = (double)ps;
  }
  res[0] = loss;
  res[1] = fl;
  res[2] = m[0];
  res[3] = m[1];
  res[4] = left;
  res[5] = right;
  res[6] = cleft;
  res[7] = cright;
  res[8] = cl[0];
  res[9] = cl[1];
  res[10] = conf_mean;
  for (int i = 0; i < 4; ++i) res[11 + i] = mon[i] / B;
  res[15] = kcount;
  res[16] = empty;
  for (int i = 17; i < S3R_LOSS_RES_HEADER; ++i) res[i] = 0.0;
}

__global__ void __launch_bounds__(kThreads) loss_backward_kernel(Cfg c, Ws w, const float* __restrict__ upstream,
                                                                 float* __restrict__ grad_pred,
                                                                 float* __restrict__ grad_conf) {
  const int blk = blockIdx.x, k = blockIdx.y, b = blockIdx.z;
  const int f = slot_frame(k, c.F);
  const double* sb = w.state + c.F + 1 + b * kPerB;
  const double wk = w.state[c.F + 1 + c.B * kPerB + k];
  const double gl = (double)upstream[0], gf = (double)upstream[1];
  lossm::Align ag, ap;
  alignments(c, sb, ag, ap);
  const bool in_norm = primary_slot(f, c.F) == k && (!c.fix_first || f == 0);
  const double coef = in_norm ? (gl * sb[SB_K1] + gf * sb[SB_K2]) / (w.state[c.F] + 1e-8) : 0.0;
  const double scale = (double)ap.mul / (double)ap.factor;
  const long long img = (long long)f * c.B + b;
  const float* x = w.pred[k] + (long long)b * c.P * 3;
  const float* cf = c.has_conf ? w.conf[k] + (long long)b * c.P : nullptr;
  const float* gt = w.gt + img * c.P * 3;
  const uint8_t* v = w.valid + img * c.P;
  float* gp = grad_pred + ((long long)k * c.B + b) * c.P * 3;
  float* gc = grad_conf ? grad_conf + ((long long)k * c.B + b) * c.P : nullptr;
  const long long p1 = min(c.P, (long long)(blk + 1) * kPixPerBlock);
  for (long long p = (long long)blk * kPixPerBlock + threadIdx.x; p < p1; p += kThreads) {
    float gr[3] = {0.f, 0.f, 0.f};
    float gcv = 0.f;
    if (v[p]) {
      float pr[3], g[3], u[3];
      lossm::align(x + 3 * p, ap, pr);
      lossm::align(gt + 3 * p, ag, g);
      const float d = lossm::l21(pr, g, u);
      const float cv = cf ? cf[p] : 1.f;
      const double g_d = gl * wk * (c.conf_loss ? (double)cv : 1.0);
      lossm::pred_grad(x + 3 * p, u, d, g_d, scale, coef, c.norm_mode == 2, gr);
      if (c.conf_loss) gcv = (float)(gl * wk * ((double)d - (double)c.alpha / (double)cv));
    }
    gp[3 * p] = gr[0];
    gp[3 * p + 1] = gr[1];
    gp[3 * p + 2] = gr[2];
    if (gc) gc[p] = gcv;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
int check_desc(const s3r_loss_desc* d, const char* who, Cfg& c) {
  if (!d) {
    set_error("%s: null descriptor", who);
    return -1;
  }
  if (d->frames < 2 || d->batch < 1 || d->height < 1 || d->width < 1) {
    set_error("%s: needs frames >= 2, batch >= 1 and a non-empty image (got F=%d B=%d H=%d W=%d)", who, d->frames,
              d->batch, d->height, d->width);
    return -1;
  }
  if (d->norm_mode < 0 || d->norm_mode > 2 || d->alpha < 0.f || (d->conf_loss && !d->conf)) {
    set_error("%s: norm_mode must be 0, 1 or 2, alpha >= 0, and conf_loss needs conf pointers", who);
    return -1;
  }
  const int F = d->frames, S = 2 * (F - 1);
  if (!d->pose0 || !d->gt_pts || !d->valid || !d->pred) {
    set_error("%s: null pose0 / gt_pts / valid / pred", who);
    return -1;
  }
  for (int f = 0; f < F; ++f)
    if (!d->gt_pts[f] || !d->valid[f]) {
      set_error("%s: null gt_pts / valid pointer of frame %d", who, f);
      return -1;
    }
  for (int k = 0; k < S; ++k)
    if (!d->pred[k] || (d->conf && !d->conf[k])) {
      set_error("%s: null pred / conf pointer of slot %d", who, k);
      return -1;
    }
  c.F = F;
  c.B = d->batch;
  c.S = S;
  c.P = (long long)d->height * d->width;
  c.nblk = (int)((c.P + kPixPerBlock - 1) / kPixPerBlock);
  if (c.nblk > 65535 || (long long)S * d->batch > 65535 || (long long)6 * d->batch > 65535) {
    set_error("%s: image or batch too large", who);
    return -1;
  }
  c.norm_mode = d->norm_mode;
  c.fix_first = d->fix_first ? 1 : 0;
  c.gt_scale = d->gt_scale ? 1 : 0;
  c.shift_inv = d->shift_inv ? 1 : 0;
  c.scale_inv = d->scale_inv ? 1 : 0;
  c.conf_loss = d->conf_loss ? 1 : 0;
  c.has_conf = d->conf ? 1 : 0;
  c.has_clip = d->has_dist_clip ? 1 : 0;
  c.alpha = d->alpha;
  c.dist_clip = d->dist_clip;
  return 0;
}

Ws bind(const Cfg& c, void* ws) {
  const Layout L = layout(c.F, c.B, c.P, c.nblk);
  char* p = static_cast<char*>(ws);
  Ws w;
  w.gt = reinterpret_cast<float*>(p + L.gt);
  w.valid = reinterpret_cast<uint8_t*>(p + L.valid);
  w.prep = reinterpret_cast<double*>(p + L.prep);
  w.state = reinterpret_cast<double*>(p + L.state);
  w.hist = reinterpret_cast<int*>(p + L.hist);
  w.part = reinterpret_cast<double*>(p + L.part);
  const float** tab = reinterpret_cast<const float**>(p + L.table);
  w.gt_in = tab;
  w.valid_in = reinterpret_cast<const uint8_t**>(tab + c.F);
  w.pred = tab + 2 * c.F;
  w.conf = tab + 2 * c.F + c.S;
  return w;
}

}  // namespace

}  // namespace s3r

using namespace s3r;

extern "C" {

size_t s3r_loss_workspace_bytes(const s3r_loss_desc* d) {
  Cfg c;
  if (check_desc(d, "loss_workspace_bytes", c)) return 0;
  return layout(c.F, c.B, c.P, c.nblk).total;
}

int s3r_loss_forward(const s3r_loss_desc* d, void* ws, size_t ws_bytes, float* gt_out, float* pred_out,
                     uint8_t* valid_out, double* results, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Cfg c;
  if (check_desc(d, "loss_forward", c)) return -1;
  const Layout L = layout(c.F, c.B, c.P, c.nblk);
  if (!ws || ws_bytes < L.total || !results) {
    set_error("loss_forward: workspace of %zu bytes (needs %zu) or null results", ws_bytes, L.total);
    return -1;
  }
  // the per-view pointer table: gt, valid, pred, conf
  const int n = 2 * c.F + 2 * c.S;
  std::vector<const void*> host(n);
  for (int f = 0; f < c.F; ++f) {
    host[f] = d->gt_pts[f];
    host[c.F + f] = d->valid[f];
  }
  for (int k = 0; k < c.S; ++k) {
    host[2 * c.F + k] = d->pred[k];
    host[2 * c.F + c.S + k] = d->conf ? d->conf[k] : nullptr;
  }
  Ws w = bind(c, ws);
  // pageable source: the copy is staged before the call returns, so the vector may go out of scope
  cudaMemcpyAsync(static_cast<char*>(ws) + L.table, host.data(), sizeof(void*) * n, cudaMemcpyHostToDevice, st);
  cudaMemsetAsync(w.hist, 0, sizeof(int) * (size_t)6 * c.B * kHist, st);
  loss_prep_kernel<<<dim3(c.nblk, c.F, c.B), kThreads, 0, st>>>(c, w, d->pose0);
  loss_prep_reduce_kernel<<<1, kThreads, 0, st>>>(c, w);
  const int stages[3] = {c.shift_inv ? 1 : 0, c.scale_inv ? 1 : 0, c.scale_inv ? 1 : 0};
  for (int s = 0; s < 3; ++s) {
    if (!stages[s]) continue;
    const int jobs = (s == 1 ? 6 : 2) * c.B;
    for (int pass = 0; pass < 4; ++pass) {
      loss_median_hist_kernel<<<dim3(c.nblk, c.F, jobs), kThreads, 0, st>>>(c, w, s, pass);
      loss_median_pick_kernel<<<(jobs + 63) / 64, 64, 0, st>>>(c, w, s, pass, jobs);
    }
  }
  loss_forward_kernel<<<dim3(c.nblk, c.S, c.B), kThreads, 0, st>>>(c, w, gt_out, pred_out);
  loss_forward_reduce_kernel<<<1, kThreads, 0, st>>>(c, w, results);
  if (valid_out) cudaMemcpyAsync(valid_out, w.valid, (size_t)c.F * c.B * c.P, cudaMemcpyDeviceToDevice, st);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("loss_forward: %s", cudaGetErrorString(e));
    return -6;
  }
  return 0;
}

int s3r_loss_backward(const s3r_loss_desc* d, const void* ws, size_t ws_bytes, const float* upstream,
                      float* grad_pred, float* grad_conf, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Cfg c;
  if (check_desc(d, "loss_backward", c)) return -1;
  const Layout L = layout(c.F, c.B, c.P, c.nblk);
  if (!ws || ws_bytes < L.total || !upstream || !grad_pred || (c.conf_loss && !grad_conf)) {
    set_error("loss_backward: workspace of %zu bytes (needs %zu), null upstream / grad_pred, or conf_loss without grad_conf",
              ws_bytes, L.total);
    return -1;
  }
  Ws w = bind(c, const_cast<void*>(ws));
  loss_backward_kernel<<<dim3(c.nblk, c.S, c.B), kThreads, 0, st>>>(c, w, upstream, grad_pred,
                                                                   c.conf_loss ? grad_conf : nullptr);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("loss_backward: %s", cudaGetErrorString(e));
    return -6;
  }
  return 0;
}

}  // extern "C"
