// Backward of the DPT-head convolutions on sm_90a: the conv weight gradient (wgrad) as a split-bf16 wgmma GEMM that
// contracts over pixels, and the col2im of the one stride-2 conv.
//
//   dW[n, tap, c] = sum_{b, y, x} dY[b, y, x, n] * X[b, y + dy(tap), x + dx(tap), c]          (fp32 result)
//
// dY [NB, H, W, N] and X [NB, H, W, Kc] are the engine's split-bf16 planes, NHWC.  taps = 1 (no shift: 1x1 convs, and the
// ConvTranspose / patch / stride-2 wgrads over re-laid-out operands) or 9 (3x3, stride 1, pad 1: tap = 3 (dy + 1) + dx + 1).
// dW [N, taps, Kc] is the engine's packed-weight layout, i.e. PyTorch's weight.permute(0, 2, 3, 1).
//
// No transposed copies: both operands are read straight from the NHWC planes by TMA, 64 channels x (bw x bh = 64) pixels
// per box -- the 4-D box geometry of gemm_plan, with the tap offset on X's pixel coordinates and the zero fill of
// out-of-bounds pixels as the conv's zero padding.  A box lands in shared memory as 64 rows (pixels, the contraction) of
// 128 bytes (channels), SWIZZLE_128B: exactly wgmma's MN-major 128-byte-swizzle canonical layout, so the MMAs read it with
// the transpose bits set.  The contraction is split over CTAs (the conv's output is at most a few hundred 128 x 128 tiles,
// the pixel count up to ~200 k); every (tile, split) pair writes its fp32 partial to a caller-owned workspace, and a second
// pass sums the partials in split order.  No atomics: the result is bitwise reproducible for a given shape.
//
// Structure per CTA (one output tile of 128 dY channels x 128 X channels for one tap, one pixel range):
//   warp 0        TMA producer: per k-block of 64 pixels up to 8 boxes (dY hi / lo, X hi / lo; two 64-channel boxes each)
//                 into a 3-deep ring of 64 KB stages.
//   warpgroups 1, 2  consumers: warpgroup g owns dY channels [64 g, 64 g + 64) of the tile and issues per 16-pixel step
//                 3 wgmma (hi*lo, lo*hi, hi*hi) per 64-channel X box into 64 x 64 fp32 register accumulators.
#include <cstring>

#include "../../include/spann3r_b200.h"
#include "common.cuh"
#include "gemm.cuh"
#include "wgmma.cuh"

namespace s3r {

namespace {
constexpr int kCh = 64;                    // channels per TMA box: one 128-byte swizzle span
constexpr int kPix = 64;                   // pixels per k-block: one TMA box of bw x bh
constexpr int kTile = 2 * kCh;             // 128 dY channels x 128 X channels per CTA
constexpr int kBox = kPix * kCh * 2;       // 8 KB
constexpr int kStageBytes = 8 * kBox;      // dY hi, dY lo, X hi, X lo: two boxes each
constexpr int kStages = 3;
constexpr int kSmem = kStages * kStageBytes + 1024 /*align slack*/ + 64 /*barriers*/;
constexpr int kThreads = 384;              // producer warpgroup + two consumer warpgroups
constexpr int kSlots = 132;                // CTAs per wave: one per SM of an H100 SXM (the split depends on the shape only)
constexpr int kMaxSplits = 256;
constexpr int kChunk = 4;                  // k-blocks (256 pixels) per tensor-core accumulation chain, see consume()
}  // namespace

struct WgradArgs {
  alignas(64) CUtensorMap tmY_hi;
  alignas(64) CUtensorMap tmY_lo;
  alignas(64) CUtensorMap tmX_hi;
  alignas(64) CUtensorMap tmX_lo;
  int N, Kc, taps;
  int bw, bh, tiles_w, tiles_h;
  int n_tiles, c_tiles, tiles;   // tiles = taps * n_tiles * c_tiles
  long long pblocks;             // NB * tiles_h * tiles_w k-blocks of 64 pixels
  int splits;
  float* part;                   // [splits, N, taps, Kc]
};

struct WgradPlan {
  int bw, bh, tiles_w, tiles_h, n_tiles, c_tiles, tiles, splits;
  long long pblocks;
};

static int next_pow2_int(int x) {
  int p = 1;
  while (p < x) p <<= 1;
  return p;
}

// Geometry and split count from the shape alone (no device query), so the summation order -- and with it every bit of
// dW -- is the same on every run and every device.  Split s covers k-blocks [s P / S, (s + 1) P / S).  S minimises
// waves(tiles * S) * (P / S + c0): the makespan of a static schedule of one-CTA-per-SM work items, c0 = 8 k-blocks the
// cost of a CTA's prologue, pipeline fill and partial store.
static void wgrad_plan(int NB, int H, int W, int N, int Kc, int taps, WgradPlan* p) {
  p->bw = W >= kPix ? kPix : next_pow2_int(W);
  p->bh = kPix / p->bw;
  p->tiles_w = (W + p->bw - 1) / p->bw;
  p->tiles_h = (H + p->bh - 1) / p->bh;
  p->n_tiles = (N + kTile - 1) / kTile;
  p->c_tiles = (Kc + kTile - 1) / kTile;
  p->tiles = taps * p->n_tiles * p->c_tiles;
  p->pblocks = (long long)NB * p->tiles_h * p->tiles_w;
  const long long smax = p->pblocks < kMaxSplits ? p->pblocks : kMaxSplits;
  double best = 1e300;
  int bs = 1;
  for (long long s = 1; s <= smax; ++s) {
    const double waves = (double)((p->tiles * s + kSlots - 1) / kSlots);
    const double cost = waves * ((double)((p->pblocks + s - 1) / s) + 8.0);
    if (cost < best * (1.0 - 1e-9)) {
      best = cost;
      bs = (int)s;
    }
  }
  p->splits = bs;
}

static bool valid_shape(int NB, int H, int W, int N, int Kc, int taps) {
  return NB >= 1 && H >= 1 && W >= 1 && N >= 8 && N % 8 == 0 && Kc >= 8 && Kc % 8 == 0 && (taps == 1 || taps == 9) &&
         (long long)NB * H * W < (1LL << 31);
}

// wgmma shared-memory descriptor of an MN-major operand stored as TMA SWIZZLE_128B wrote it: 128-byte rows along the
// contraction (one pixel each, 64 channels), 8-row swizzle atoms 1024 bytes apart.  Every operand here is a single
// 64-channel span, so both byte offsets (the stride between 8-row groups along K, and between 64-element spans along MN,
// which a one-span operand never takes) are set to the 1024-byte atom stride.
__device__ __forceinline__ uint64_t wgmma_desc_sw128_mnmajor(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)(1024 >> 4) << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

__device__ __forceinline__ void mma3(float (&acc)[32], uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo,
                                     int scale_d) {
  wgmma_bf16_n64_mn(acc, a_hi, b_lo, scale_d);
  wgmma_bf16_n64_mn(acc, a_lo, b_hi, 1);
  wgmma_bf16_n64_mn(acc, a_hi, b_hi, 1);
}

// one warp's rows r, r + 8 of a 64 x 64 accumulator (fragment layout: wgmma.cuh) at X channels [c0, c0 + 64)
__device__ __forceinline__ void store_frag(const float (&acc)[32], float* base, const WgradArgs& a, int r, int tap, int c0,
                                           int lane) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = c0 + 8 * i + 2 * (lane & 3);
    if (c >= a.Kc) continue;   // Kc % 8 == 0: c + 1 < Kc too
    if (r < a.N)
      *reinterpret_cast<float2*>(base + ((long long)r * a.taps + tap) * a.Kc + c) = make_float2(acc[4 * i], acc[4 * i + 1]);
    if (r + 8 < a.N)
      *reinterpret_cast<float2*>(base + ((long long)(r + 8) * a.taps + tap) * a.Kc + c) =
          make_float2(acc[4 * i + 2], acc[4 * i + 3]);
  }
}

// Consumer warpgroup `wg` of a tile with XV (1 or 2) 64-channel X boxes: the MMA loop over its k-blocks, then the store of
// its 64 dY channels x 64 XV X channels to this split's partial [N, taps, Kc].
// Two-level sum: the tensor core accumulates kChunk k-blocks (256 pixels) from zero, then the chunk is added to an fp32
// register total with round-to-nearest FADDs.  One chain over the whole pixel range of a split (up to ~15 k pixels) lost
// ~5e-5 relative on the 200 k-pixel head.2 wgrad; chunked, the error is that of the shorter chains.
template <int XV>
__device__ __forceinline__ void consume(const WgradArgs& a, uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                        long long kb0, long long kb1, int wg, int split, int tap, int n0, int c0) {
  const int lane = threadIdx.x & 31;
  const int wq = ((threadIdx.x >> 5) - 4) & 3;
  float acc0[32], acc1[32], tot0[32], tot1[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) acc0[j] = acc1[j] = tot0[j] = tot1[j] = 0.f;
  const uint32_t smem_u = __shfl_sync(0xffffffffu, smem_u32(smem), 0);
  int stage = 0;
  uint32_t phase = 0;
  for (long long kc = kb0; kc < kb1; kc += kChunk) {
    const int nk = (kb1 - kc < kChunk) ? (int)(kb1 - kc) : kChunk;
    int prev = -1;
    for (int i = 0; i < nk; ++i) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t s = smem_u + stage * kStageBytes;
      const uint64_t ya_hi = wgmma_desc_sw128_mnmajor(s + wg * kBox);
      const uint64_t ya_lo = wgmma_desc_sw128_mnmajor(s + (2 + wg) * kBox);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kPix / 16; ++kk) {
        const uint64_t ko = (uint64_t)((kk * 16 * 128) >> 4);   // 16 pixels = two 1024-byte swizzle atoms
        const int sd = (i == 0 && kk == 0) ? 0 : 1;              // a chunk starts from zero
        mma3(acc0, ya_hi + ko, ya_lo + ko, wgmma_desc_sw128_mnmajor(s + 4 * kBox) + ko,
             wgmma_desc_sw128_mnmajor(s + 6 * kBox) + ko, sd);
        if constexpr (XV == 2)
          mma3(acc1, ya_hi + ko, ya_lo + ko, wgmma_desc_sw128_mnmajor(s + 5 * kBox) + ko,
               wgmma_desc_sw128_mnmajor(s + 7 * kBox) + ko, sd);
      }
      wgmma_commit();
      wgmma_wait<1>();   // the previous k-block's MMAs have retired: its stage goes back to the producer
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      prev = stage;
      if (++stage == kStages) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[prev]);
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      tot0[j] += acc0[j];
      if constexpr (XV == 2) tot1[j] += acc1[j];
    }
  }

  const int r = n0 + wg * kCh + wq * 16 + (lane >> 2);
  float* base = a.part + (long long)split * a.N * a.taps * a.Kc;
  store_frag(tot0, base, a, r, tap, c0, lane);
  if constexpr (XV == 2) store_frag(tot1, base, a, r, tap, c0 + kCh, lane);
}

__global__ void __launch_bounds__(kThreads, 1) conv_wgrad_kernel(const __grid_constant__ WgradArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes);
  uint64_t* empty_bar = full_bar + kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tile = blockIdx.x % a.tiles;     // CTAs of one split run side by side and share their pixel rows in L2
  const int split = blockIdx.x / a.tiles;
  const int per_tap = a.n_tiles * a.c_tiles;
  const int tap = tile / per_tap;
  const int nt = (tile - tap * per_tap) / a.c_tiles;
  const int ct = tile - tap * per_tap - nt * a.c_tiles;
  const int n0 = nt * kTile, c0 = ct * kTile;
  const int yv = (n0 + kCh < a.N) ? 2 : 1;   // 64-channel boxes of the tile that hold any channel
  const int xv = (c0 + kCh < a.Kc) ? 2 : 1;
  const long long kb0 = split * a.pblocks / a.splits;
  const long long kb1 = (split + 1) * a.pblocks / a.splits;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&a.tmY_hi);
    tma_prefetch_desc(&a.tmY_lo);
    tma_prefetch_desc(&a.tmX_hi);
    tma_prefetch_desc(&a.tmX_lo);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 4 * yv);   // one arrival per warp of the active consumer warpgroups
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();   // operands come from the previous kernels; the partials may still be read by the previous reduce

  if (warp < 4) {
    // ------------------------------------------------------------------ TMA producer (warp 0; registers handed to the consumers)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp != 0) return;
    const int dy = a.taps == 9 ? tap / 3 - 1 : 0;
    const int dx = a.taps == 9 ? tap % 3 - 1 : 0;
    const uint32_t bytes = (uint32_t)(2 * (yv + xv) * kBox);
    int stage = 0;
    uint32_t phase = 0;
    for (long long kb = kb0; kb < kb1; ++kb) {
      const int tw = (int)(kb % a.tiles_w);
      const long long t = kb / a.tiles_w;
      const int th = (int)(t % a.tiles_h);
      const int img = (int)(t / a.tiles_h);
      const int w0 = tw * a.bw, h0 = th * a.bh;
      mbar_wait(&empty_bar[stage], phase ^ 1);
      if (lane == 0) {
        uint8_t* s = smem + stage * kStageBytes;
        uint64_t* fb = &full_bar[stage];
        mbar_arrive_expect_tx(fb, bytes);
        for (int j = 0; j < yv; ++j) {
          tma_load_4d(s + j * kBox, &a.tmY_hi, fb, n0 + j * kCh, w0, h0, img);
          tma_load_4d(s + (2 + j) * kBox, &a.tmY_lo, fb, n0 + j * kCh, w0, h0, img);
        }
        for (int j = 0; j < xv; ++j) {
          tma_load_4d(s + (4 + j) * kBox, &a.tmX_hi, fb, c0 + j * kCh, w0 + dx, h0 + dy, img);
          tma_load_4d(s + (6 + j) * kBox, &a.tmX_lo, fb, c0 + j * kCh, w0 + dx, h0 + dy, img);
        }
      }
      __syncwarp();
      if (++stage == kStages) {
        stage = 0;
        phase ^= 1;
      }
    }
  } else {
    // ------------------------------------------------------------------ consumers
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int wg = (warp - 4) >> 2;
    if (wg >= yv) return;   // no dY channel in this half of the tile
    if (xv == 2) consume<2>(a, smem, full_bar, empty_bar, kb0, kb1, wg, split, tap, n0, c0);
    else consume<1>(a, smem, full_bar, empty_bar, kb0, kb1, wg, split, tap, n0, c0);
  }
}

// dW[i] = sum over splits s = 0, 1, ... of part[s][i], in that order
__global__ void wgrad_reduce_kernel(const float4* __restrict__ part, long long n4, int splits, float4* __restrict__ dw) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 s = part[i];
    for (int k = 1; k < splits; ++k) {
      const float4 v = part[k * n4 + i];
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    dw[i] = s;
  }
}

static int encode_nhwc(CUtensorMap* m, const void* base, int NB, int H, int W, int C, long long ld, int bw, int bh) {
  const uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)NB};
  const uint64_t str[3] = {(uint64_t)ld * 2, (uint64_t)ld * W * 2, (uint64_t)ld * W * H * 2};
  const uint32_t box[4] = {(uint32_t)kCh, (uint32_t)bw, (uint32_t)bh, 1};
  return encode_tmap(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, base, dims, str, box);
}

static bool misaligned(const void* p) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) & 15) != 0; }

// ------------------------------------------------------------------------------------------------
// col2im of Conv2d(C, C, 3, stride 2, pad 1): the adjoint of im2col_3x3s2 (elementwise.cu).
//   cols fp32 [NB*Ho*Wo, 9*C] (k = tap*C + c)  ->  out fp32 [NB, H, W, C]
// Gather form: each input pixel sums the (at most 4) output pixel / tap pairs that read it, taps in ascending order, so the
// result is deterministic without atomics.
// ------------------------------------------------------------------------------------------------
__global__ void col2im_3x3s2_kernel(const float* __restrict__ cols, int NB, int H, int W, int C, int Ho, int Wo,
                                    float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int c4 = C >> 2;
  const long long total = (long long)NB * H * W * c4;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int cc = (int)(idx % c4);
    const long long t = idx / c4;
    const int x = (int)(t % W);
    const int y = (int)((t / W) % H);
    const int nb = (int)(t / ((long long)W * H));
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int ty = y + 1 - ky;                 // = 2 * oy
      if (ty < 0 || (ty & 1) || (ty >> 1) >= Ho) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int tx = x + 1 - kx;
        if (tx < 0 || (tx & 1) || (tx >> 1) >= Wo) continue;
        const long long row = ((long long)nb * Ho + (ty >> 1)) * Wo + (tx >> 1);
        const float4 v = *reinterpret_cast<const float4*>(cols + row * 9 * C + (ky * 3 + kx) * C + cc * 4);
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
      }
    }
    *reinterpret_cast<float4*>(out + t * C + cc * 4) = s;
  }
}

}  // namespace s3r

using namespace s3r;

extern "C" {

size_t s3r_conv_wgrad_workspace_bytes(int NB, int H, int W, int N, int Kc, int taps) {
  if (!valid_shape(NB, H, W, N, Kc, taps)) return 0;
  WgradPlan p;
  wgrad_plan(NB, H, W, N, Kc, taps, &p);
  return (size_t)p.splits * N * taps * Kc * sizeof(float);
}

int s3r_conv_wgrad(const void* dy_hi, const void* dy_lo, int64_t ldy, const void* x_hi, const void* x_lo, int64_t ldx,
                   int NB, int H, int W, int N, int Kc, int taps, void* workspace, size_t workspace_bytes, float* dw,
                   void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!valid_shape(NB, H, W, N, Kc, taps)) {
    set_error("s3r_conv_wgrad: unsupported shape nb=%d h=%d w=%d n=%d kc=%d taps=%d (n, kc multiples of 8, taps in {1,9}, "
              "nb*h*w < 2^31)", NB, H, W, N, Kc, taps);
    return -1;
  }
  if (ldy < N || ldy % 8 != 0 || ldx < Kc || ldx % 8 != 0) {
    set_error("s3r_conv_wgrad: row strides ldy=%lld (n=%d) / ldx=%lld (kc=%d) must cover the row and be multiples of 8",
              ldy, N, ldx, Kc);
    return -1;
  }
  if (misaligned(dy_hi) || misaligned(dy_lo) || misaligned(x_hi) || misaligned(x_lo) || misaligned(dw) ||
      misaligned(workspace)) {
    set_error("s3r_conv_wgrad: null or not 16-byte aligned pointer");
    return -1;
  }
  const size_t need = s3r_conv_wgrad_workspace_bytes(NB, H, W, N, Kc, taps);
  if (workspace_bytes < need) {
    set_error("s3r_conv_wgrad: workspace of %zu bytes, %zu needed (s3r_conv_wgrad_workspace_bytes)", workspace_bytes, need);
    return -1;
  }
  WgradPlan p;
  wgrad_plan(NB, H, W, N, Kc, taps, &p);
  WgradArgs a;
  memset(&a, 0, sizeof(a));
  int r;
  if ((r = encode_nhwc(&a.tmY_hi, dy_hi, NB, H, W, N, ldy, p.bw, p.bh))) return r;
  if ((r = encode_nhwc(&a.tmY_lo, dy_lo, NB, H, W, N, ldy, p.bw, p.bh))) return r;
  if ((r = encode_nhwc(&a.tmX_hi, x_hi, NB, H, W, Kc, ldx, p.bw, p.bh))) return r;
  if ((r = encode_nhwc(&a.tmX_lo, x_lo, NB, H, W, Kc, ldx, p.bw, p.bh))) return r;
  a.N = N; a.Kc = Kc; a.taps = taps;
  a.bw = p.bw; a.bh = p.bh; a.tiles_w = p.tiles_w; a.tiles_h = p.tiles_h;
  a.n_tiles = p.n_tiles; a.c_tiles = p.c_tiles; a.tiles = p.tiles;
  a.pblocks = p.pblocks; a.splits = p.splits;
  a.part = reinterpret_cast<float*>(workspace);

  static PerDeviceOnce once;
  bool& attr_set = once.cur();
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(conv_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
    if (e != cudaSuccess) {
      set_error("s3r_conv_wgrad: cudaFuncSetAttribute(smem=%d): %s", kSmem, cudaGetErrorString(e));
      return -5;
    }
    attr_set = true;
  }
  cudaError_t e = launch_pdl(conv_wgrad_kernel, dim3((unsigned)(p.tiles * p.splits)), dim3(kThreads), kSmem, st, a);
  if (e != cudaSuccess) {
    set_error("s3r_conv_wgrad: launch failed: %s", cudaGetErrorString(e));
    return -6;
  }
  const long long n4 = (long long)N * taps * Kc / 4;
  long long blocks = (n4 + 255) / 256;
  if (blocks > 132 * 8) blocks = 132 * 8;
  e = launch_pdl(wgrad_reduce_kernel, dim3((unsigned)blocks), dim3(256), 0, st,
                 reinterpret_cast<const float4*>(workspace), n4, p.splits, reinterpret_cast<float4*>(dw));
  if (e != cudaSuccess) {
    set_error("s3r_conv_wgrad: reduce launch failed: %s", cudaGetErrorString(e));
    return -6;
  }
  return 0;
}

int s3r_col2im_3x3s2(const float* cols, int NB, int H, int W, int C, int Ho, int Wo, float* out, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (NB < 1 || H < 1 || W < 1 || C < 8 || C % 8 != 0 || Ho != (H + 1) / 2 || Wo != (W + 1) / 2 ||
      (long long)NB * H * W * C >= (1LL << 40)) {
    set_error("s3r_col2im_3x3s2: unsupported shape nb=%d h=%d w=%d c=%d ho=%d wo=%d (c a multiple of 8, ho = (h+1)/2, "
              "wo = (w+1)/2)", NB, H, W, C, Ho, Wo);
    return -1;
  }
  if (misaligned(cols) || misaligned(out)) {
    set_error("s3r_col2im_3x3s2: null or not 16-byte aligned pointer");
    return -1;
  }
  const long long total = (long long)NB * H * W * (C / 4);
  long long blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  cudaError_t e = launch_pdl(col2im_3x3s2_kernel, dim3((unsigned)blocks), dim3(256), 0, st, cols, NB, H, W, C, Ho, Wo, out);
  if (e != cudaSuccess) {
    set_error("s3r_col2im_3x3s2: launch failed: %s", cudaGetErrorString(e));
    return -6;
  }
  return 0;
}

}  // extern "C"
