// Split-bf16 ("bf16x3") GEMM / implicit-GEMM 3x3 convolution on Hopper wgmma tensor cores, sm_90a.
//
//   D[pixel, n] = sum_{tap, k} A[pixel shifted by tap, k] * Wt[n, tap, k]      (fp32 result)
//
// Replaces, on the Spann3R forward path, every nn.Linear (croco/models/blocks.py:73-79,94-112,
// 149-169; dust3r/model.py:189-190; spann3r/model.py:250-261,310), the patch-embedding conv
// (dust3r/patch_embed.py:19-29, after an im2col kernel), and every Conv2d / ConvTranspose2d of the
// DPT head (croco/models/dpt_block.py:33-75,121-142,189-218,318-324,356-410).
//
// Structure: persistent, warp-specialised, one CTA per SM, 128 x BN output tiles.
//   warpgroup 0   TMA producer (one warp; registers handed to the consumers with setmaxnreg): per k-block four
//                 SWIZZLE_64B boxes (A_hi, A_lo: 128 pixels x 32 ch; B_hi, B_lo: BN x 32) into a STAGES-deep smem
//                 ring (5 / 6 / 7 stages at BN = 128 / 96 / 64); a 3x3 conv is 9 taps whose A box is the same 4-D tensor
//                 map at (w+dx, h+dy) -- out-of-bounds pixels are zero-filled by TMA, which is exactly the conv's zero
//                 padding.
//   warpgroups 1, 2  consumers: each owns 64 rows of the tile and issues per k-block 2 K-steps x 3 wgmma (hi*lo,
//                 lo*hi, hi*hi) into a 64 x BN fp32 register accumulator, one k-block in flight.  The epilogue is run
//                 by the same 8 warps: the accumulator goes through shared memory 2 x 32 columns at a time into the
//                 thread = tile row layout of gemm_epilogue.cuh (fused bias / GELU / ReLU / residual adds / split-bf16
//                 re-encode / RoPE + head split / ConvTranspose pixel shuffle / DPT head tail + postprocess).  The
//                 producer keeps filling the ring for the next tile meanwhile.
#include "gemm.cuh"

#include "../../include/spann3r_b200.h"

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "common.cuh"
#include "gemm_epilogue.cuh"
#include "wgmma.cuh"

namespace s3r {

static constexpr int BM = 128;
// 32-channel k-blocks: one 64-byte swizzle span per row.  A stage is then 32 KB at BN = 128, so the ring is 5 deep;
// the consumers hold 2 stages (the k-block being issued and the one retiring), which leaves 3 k-blocks of loads in
// flight to cover the TMA / L2 latency (64-channel k-blocks fit only 2 stages at BN = 128: at most 1 in flight).
static constexpr int BK = 32;
static constexpr CUtensorMapSwizzle kSwizzle = CU_TENSOR_MAP_SWIZZLE_64B;   // BK * 2 bytes per row
static constexpr int kEpiWarps = 8;     // the two consumer warpgroups
static constexpr int kNumThreads = 128 + 32 * kEpiWarps;
static constexpr int kSmemMax = 227 * 1024;
static constexpr int kAccLD = 36;       // accumulator staging row stride (floats): 16-byte rows, conflict-free row reads
static constexpr int kAccBytes = 2 * BM * kAccLD * 4;   // two 32-column chunks (one per column half) of all 128 rows

// NP = tensor-core products per k16 step: 3 (split bf16: hi*lo, lo*hi, hi*hi) or 1 (hi*hi only, the bf16 precision).
// A stage holds the planes the products read: A_hi [A_lo] B_hi [B_lo].
template <int BN, int NP>
struct GemmCfg {
  static constexpr int PLANES = NP == 3 ? 2 : 1;
  static constexpr int A_TILE = BM * BK * 2;  // bytes, one plane
  static constexpr int B_TILE = BN * BK * 2;
  static constexpr int B_OFF = PLANES * A_TILE;   // first B plane in a stage
  static constexpr int STAGE = PLANES * (A_TILE + B_TILE);
  static constexpr int COLV = 2 * 2 * BN * 4;  // per tile parity: staged bias + LN-fold column sums of the tile
  static constexpr int HT = 4 * 2 * 32 * 16;   // EPI_HEADTAIL hand-over slots (per lane quadrant, two tile parities)
  static constexpr int FIXED = 1024 /*align slack*/ + 256 /*barriers*/ + kAccBytes + COLV + HT;
  static constexpr int STAGES = (kSmemMax - FIXED) / STAGE;
  static constexpr int SMEM = STAGES * STAGE + FIXED;
  static_assert(NP == 3 || NP == 1, "split (3 products) or bf16 (1 product)");
  // split: 32 / 28 / 24 KB stages at BN = 128 / 96 / 64; one product: 16 / 14 / 12 KB, the same 32-channel k-blocks
  // (DESIGN.md §4)
  static_assert(STAGES == (NP == 3 ? (BN == 128 ? 5 : BN == 96 ? 6 : 7) : (BN == 128 ? 11 : BN == 96 ? 13 : 15)),
                "ring depth (DESIGN.md §4)");
  static_assert(2 * STAGES * 8 <= 256, "full + empty barriers fit their 256-byte slot");
  static_assert(Stg<32>::WARP_BYTES == 32 * kAccLD * 4, "a warp's staging tile is its own rows of the accumulator chunk");
};

template <int BN>
__device__ __forceinline__ void wgmma_bf16(float (&d)[BN / 2], uint64_t da, uint64_t db, int scale_d) {
  if constexpr (BN == 64) wgmma_bf16_n64(d, da, db, scale_d);
  else if constexpr (BN == 96) wgmma_bf16_n96(d, da, db, scale_d);
  else wgmma_bf16_n128(d, da, db, scale_d);
}

template <int BN, int EPI, int NP>
__global__ void __launch_bounds__(kNumThreads, 1) gemm_bf16x3_kernel(const __grid_constant__ GemmArgs args) {
  using Cfg = GemmCfg<BN, NP>;
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment by pointer arithmetic on the __shared__ array (an integer round trip would lose the address
  // space and turn every access through `smem` into a generic LD / ST)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::STAGES * Cfg::STAGE);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + Cfg::STAGES;
  float* sacc = reinterpret_cast<float*>(smem + Cfg::STAGES * Cfg::STAGE + 256);   // [2][BM][kAccLD]
  float* colv = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(sacc) + kAccBytes);   // [2 parities][bias | colsum][BN]
  float4* hts = reinterpret_cast<float4*>(reinterpret_cast<uint8_t*>(colv) + Cfg::COLV);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // CTA 0's timeline: the pointer is read from the parameters at each stamp, not held in registers through the kernel
  const bool trace = blockIdx.x == 0 && args.trace != nullptr;
  if (trace && threadIdx.x == 0) args.trace[0] = globaltimer_ns();

  const int n_tiles = (args.N + BN - 1) / BN;
  const int m_tiles = args.tiles_w * args.tiles_h * args.NB;
  const int tiles_per_group = n_tiles * m_tiles;
  const int total_tiles = tiles_per_group * args.groups;
  const int num_kb = args.taps * args.kpt;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&args.tmA_hi);
    tma_prefetch_desc(&args.tmB_hi);
    if constexpr (NP == 3) {
      tma_prefetch_desc(&args.tmA_lo);
      tma_prefetch_desc(&args.tmB_lo);
    }
    for (int i = 0; i < Cfg::STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kEpiWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  if (trace && threadIdx.x == 0) args.trace[1] = globaltimer_ns();
  // Weights do not depend on the previous kernel: the producer stages the B tiles of the first ring pass of this CTA's first
  // tile BEFORE the dependency wait (their HBM / L2 latency overlaps the previous kernel's tail); the A tiles of those
  // stages follow after the wait, on the same full barrier (expect_tx covers the whole stage).
  int pre_b = 0;
  if (warp == 0 && args.b_static && (int)blockIdx.x < total_tiles) {
    const int tile = blockIdx.x;
    const int g = tile / tiles_per_group;
    const int nt = (tile - g * tiles_per_group) % n_tiles;
    const int brow = g * args.b_group_rows + nt * BN;
    pre_b = num_kb < Cfg::STAGES ? num_kb : Cfg::STAGES;
    if (lane == 0) {
      for (int kb = 0; kb < pre_b; ++kb) {
        const int tap = kb / args.kpt, kc = (kb - tap * args.kpt) * BK;
        uint8_t* s = smem + kb * Cfg::STAGE;
        mbar_arrive_expect_tx(&full_bar[kb], Cfg::STAGE);
        tma_load_3d(s + Cfg::B_OFF, &args.tmB_hi, &full_bar[kb], kc, tap, brow);
        if constexpr (NP == 3) tma_load_3d(s + Cfg::B_OFF + Cfg::B_TILE, &args.tmB_lo, &full_bar[kb], kc, tap, brow);
      }
    }
    __syncwarp();
  }
  pdl_wait();  // everything above overlapped the previous kernel's tail; activations are touched only below
  if (trace && threadIdx.x == 0) args.trace[2] = globaltimer_ns();

  if (warp < 4) {
    // ------------------------------------------------------------------ TMA producer (warp 0; warps 1..3 idle)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0) {
      // whole warp in uniform control flow, one elected lane issues; tap / channel coordinates advance incrementally
      const uint32_t smem_u = __shfl_sync(0xffffffffu, smem_u32(smem), 0);
      const uint32_t full_u = __shfl_sync(0xffffffffu, smem_u32(full_bar), 0);
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int g = tile / tiles_per_group;
        const int rem = tile - g * tiles_per_group;
        const int mt = rem / n_tiles;
        const int nt = rem - mt * n_tiles;
        const int tw = mt % args.tiles_w;
        const int th = (mt / args.tiles_w) % args.tiles_h;
        const int nb = mt / (args.tiles_w * args.tiles_h);
        const int w0 = tw * args.bw, h0 = th * args.bh;
        const int img = ((args.a_swap && nt * BN >= args.swap_col0) ? (args.groups - 1 - g) : g) * args.NB + nb;
        const int brow = g * args.b_group_rows + nt * BN;
        int tap = 0, kc = 0, dx = (args.taps == 9) ? -1 : 0, dy = dx;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          const bool b_done = (tile == (int)blockIdx.x) && (kb < pre_b);   // B (and the expect_tx) went out before the wait
          if (elect_one()) {
            const uint32_t s = smem_u + stage * Cfg::STAGE;
            const uint32_t fb = full_u + stage * 8;
            if (!b_done) mbar_arrive_expect_tx_u(fb, Cfg::STAGE);
            tma_load_4d_u(s, &args.tmA_hi, fb, kc, w0 + dx, h0 + dy, img);
            if constexpr (NP == 3) tma_load_4d_u(s + Cfg::A_TILE, &args.tmA_lo, fb, kc, w0 + dx, h0 + dy, img);
            if (!b_done) {
              tma_load_3d_u(s + Cfg::B_OFF, &args.tmB_hi, fb, kc, tap, brow);
              if constexpr (NP == 3) tma_load_3d_u(s + Cfg::B_OFF + Cfg::B_TILE, &args.tmB_lo, fb, kc, tap, brow);
            }
          }
          __syncwarp();
          kc += BK;
          if (kc >= args.kpt * BK) {   // next tap: (dy, dx) walk the 3x3 window row by row
            kc = 0;
            ++tap;
            if (++dx > 1) {
              dx = -1;
              ++dy;
            }
          }
          if (++stage == Cfg::STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ consumers: MMA, then epilogue
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int cw = warp - 4;            // consumer warp 0..7
    const int wg = cw >> 2;             // MMA: warpgroup wg owns tile rows [64 wg, 64 wg + 64)
    const int wq = cw & 3;              //      and this warp rows 16 wq + (lane / 4) (+8) of them
    const int quad = cw & 3;            // epilogue: thread = tile row quad * 32 + lane ...
    const int half = cw >> 2;           // ... of column half `half`
    // The tile's NCH 32-column chunks go to the two column halves, CH rounds of one chunk per half: half h takes chunks
    // [h CH, h CH + CH).  At BN = 96 that is chunks 0, 1 for half 0 and chunk 2 for half 1, which sits out the second
    // round (and still joins every barrier).
    constexpr int NCH = BN / 32;
    constexpr int CH = (NCH + 1) / 2;
    const uint32_t smem_u = __shfl_sync(0xffffffffu, smem_u32(smem), 0);
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++it) {
      const int g = tile / tiles_per_group;
      const int rem = tile - g * tiles_per_group;
      const int mt = rem / n_tiles;
      const int nt = rem - mt * n_tiles;
      const int tw = mt % args.tiles_w;
      const int th = (mt / args.tiles_w) % args.tiles_h;
      const int nb = mt / (args.tiles_w * args.tiles_h);

      // everything that does not need the accumulator is requested before the main loop: the tile's bias / colsum
      // columns (-> smem), the rows' LayerNorm statistics, RoPE positions and output addresses, and the residual values
      // of the first chunk
      float* sb = colv + (it & 1) * 2 * BN;
      float* scs = sb + BN;
      epi_stage_cols<EPI, BN>(args, sb, scs, g, nt, (int)threadIdx.x - 128, 32 * kEpiWarps);
      const TileGeom tg = make_geom(args, g, nb, th, tw, nt * BN);
      EpiRow er;
      EpiTRows tr;
      epi_tile_pre<EPI, 32>(args, tg, quad, lane, er, tr);
      float4 res[8];
      const int cfirst = nt * BN + half * CH * 32;
      if (cfirst < args.N) epi_prefetch_res<EPI, 32>(args, tr, res, cfirst, lane);
      // staged columns visible to all consumer warps; every warp is also done with the previous tile's staging buffer
      asm volatile("bar.sync 1, %0;" ::"n"(32 * kEpiWarps) : "memory");

      float acc[BN / 2];
#pragma unroll
      for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        if (trace && kb == 0 && it == 0 && threadIdx.x == 128) args.trace[3] = globaltimer_ns();
        const uint32_t sa = smem_u + stage * Cfg::STAGE;
        const uint64_t da_hi = wgmma_desc_sw64_kmajor(sa + wg * (64 * BK * 2));
        const uint64_t db_hi = wgmma_desc_sw64_kmajor(sa + Cfg::B_OFF);
        wgmma_fence();
        if constexpr (NP == 3) {
          const uint64_t da_lo = wgmma_desc_sw64_kmajor(sa + Cfg::A_TILE + wg * (64 * BK * 2));
          const uint64_t db_lo = wgmma_desc_sw64_kmajor(sa + Cfg::B_OFF + Cfg::B_TILE);
#pragma unroll
          for (int kk = 0; kk < BK / 16; ++kk) {
            const uint64_t ko = (uint64_t)(kk * 32 >> 4);  // 16 bf16 = 32 bytes along K inside the swizzle span
            wgmma_bf16<BN>(acc, da_hi + ko, db_lo + ko, 1);
            wgmma_bf16<BN>(acc, da_lo + ko, db_hi + ko, 1);
            wgmma_bf16<BN>(acc, da_hi + ko, db_hi + ko, 1);
          }
        } else {
#pragma unroll
          for (int kk = 0; kk < BK / 16; ++kk) {
            const uint64_t ko = (uint64_t)(kk * 32 >> 4);
            wgmma_bf16<BN>(acc, da_hi + ko, db_hi + ko, 1);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();   // the previous k-block's MMAs have retired: its stage goes back to the producer
        if (prev >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        prev = stage;
        if (++stage == Cfg::STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      if (trace && it == 0 && threadIdx.x == 128) args.trace[4] = globaltimer_ns();

      float ht_acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int cc = 0; cc < CH; ++cc) {
        if (cc > 0) asm volatile("bar.sync 1, %0;" ::"n"(32 * kEpiWarps) : "memory");   // previous chunk consumed
        // accumulator fragment -> staging rows: round cc's chunk of each column half
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (h * CH + cc >= NCH) continue;
          float* dst = sacc + h * (BM * kAccLD);
#pragma unroll
          for (int ii = 0; ii < 4; ++ii) {
            const int i = (h * CH + cc) * 4 + ii;                 // 8-column block of the accumulator
            const int r = wg * 64 + wq * 16 + (lane >> 2);
            const int c = ii * 8 + 2 * (lane & 3);
            *reinterpret_cast<float2*>(dst + r * kAccLD + c) = make_float2(acc[4 * i], acc[4 * i + 1]);
            *reinterpret_cast<float2*>(dst + (r + 8) * kAccLD + c) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
          }
        }
        asm volatile("bar.sync 1, %0;" ::"n"(32 * kEpiWarps) : "memory");
        float* myrows = sacc + half * (BM * kAccLD) + quad * 32 * kAccLD;   // also this warp's staging tile below
        float v[32];
        {
          const float4* src = reinterpret_cast<const float4*>(myrows + lane * kAccLD);
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            const float4 t = src[q];
            v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
          }
        }
        __syncwarp();
        const int c = half * CH + cc;
        const int col0 = nt * BN + c * 32;
        if (col0 < args.N && (NCH % 2 == 0 || c < NCH)) {   // warp-uniform
          const int res_next = (cc + 1 < CH && (NCH % 2 == 0 || c + 1 < NCH) && col0 + 32 < args.N) ? col0 + 32 : -1;
          epi_chunk<EPI, 32>(args, v, sb + c * 32, scs + c * 32, myrows, tg, er, tr, res, col0, res_next, lane, ht_acc);
        }
      }

      if constexpr (EPI == EPI_HEADTAIL) {
        // the row's 4 dot products are split over the two column halves: half 1 hands its partial sums to half 0
        // (two alternating slots), 64-thread named barrier per lane quadrant
        float4* slot = hts + (quad * 2 + (it & 1)) * 32;
        if (half == 1) slot[lane] = make_float4(ht_acc[0], ht_acc[1], ht_acc[2], ht_acc[3]);
        asm volatile("bar.sync %0, 64;" ::"r"(2 + quad) : "memory");
        if (half == 0) {
          const float4 p = slot[lane];
          ht_acc[0] += p.x; ht_acc[1] += p.y; ht_acc[2] += p.z; ht_acc[3] += p.w;
          epi_headtail_finish(args, tg, er, ht_acc);
        }
      }
    }
    if (trace && threadIdx.x == 128) args.trace[5] = globaltimer_ns();   // epilogue of this CTA's last tile done
  }
  if (trace && threadIdx.x == 128) args.trace[6] = globaltimer_ns();     // exit (the producer warpgroup has no work left)
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
const char* last_error() { return g_err; }
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess)
      return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

// dims/box innermost-first; strides_bytes has rank-1 entries (dims 1..rank-1).
int encode_tmap(CUtensorMap* out, CUtensorMapDataType dt, int rank, const void* base, const uint64_t* dims,
                const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swizzle) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return -3;
  }
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  cuuint64_t d[5], s[4];
  cuuint32_t b[5];
  for (int i = 0; i < rank; ++i) {
    d[i] = dims[i];
    b[i] = box[i];
  }
  for (int i = 0; i + 1 < rank; ++i) s[i] = strides_bytes[i];
  CUresult r = enc(out, dt, (cuuint32_t)rank, const_cast<void*>(base), d, s, b, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed: %d (rank %d dims %llu %llu %llu %llu box %u %u %u %u base %p)", (int)r,
              rank, (unsigned long long)d[0], (unsigned long long)(rank > 1 ? d[1] : 0),
              (unsigned long long)(rank > 2 ? d[2] : 0), (unsigned long long)(rank > 3 ? d[3] : 0), b[0],
              rank > 1 ? b[1] : 0, rank > 2 ? b[2] : 0, rank > 3 ? b[3] : 0, base);
    return -4;
  }
  return 0;
}

static int next_pow2(int x) {
  int p = 1;
  while (p < x) p <<= 1;
  return p;
}

static int g_num_sms[64] = {};   // per device ordinal
int num_sms() {
  int dev = 0;
  cudaGetDevice(&dev);
  int& n = g_num_sms[dev & 63];
  if (!n) {
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

// Tile shape: 128 x 64, 128 x 96 or 128 x 128, the cheapest under makespan = waves x (bytes staged per k-block), with
// waves = ceil(tiles / SMs) for the persistent static schedule and 24 / 28 / 32 KB staged per k-block at BN = 64 / 96 / 128
// (split planes; the one-product ring halves every figure, which keeps the ranking).  Ties go to the wider tile.  A
// 64-row warpgroup holds a 64 x BN fp32 accumulator in registers next to the epilogue's working set, so 128 is the widest
// tile.  col_align (0 = none) is a column no tile may straddle: a_swap's swap_col0, since the producer and the epilogue
// pick the swapped A group once per tile; a width that does not divide it is never chosen, and rejected when forced.
int gemm_choose_bn(long long m_tiles, int N, int sms, int col_align, int force_bn) {
  auto fits = [&](int bn) { return col_align == 0 || col_align % bn == 0; };
  auto cost = [&](int bn, double kb) {
    const long long tiles = m_tiles * ((N + bn - 1) / bn);
    return (double)((tiles + sms - 1) / sms) * kb;
  };
  if (force_bn != 0) {
    if (force_bn != 64 && force_bn != 96 && force_bn != 128) {
      set_error("gemm planner: force_bn %d (64, 96, 128 or 0)", force_bn);
      return -1;
    }
    if (!fits(force_bn)) {
      set_error("gemm planner: force_bn %d: the tile would straddle swap_col0 = %d", force_bn, col_align);
      return -1;
    }
    return force_bn;
  }
  if (col_align % 64 != 0) {
    set_error("gemm planner: swap_col0 = %d is not a multiple of 64 (no tile width fits it)", col_align);
    return -1;
  }
  int bn = 64;
  double best = cost(64, 24.0);
  if (fits(96) && cost(96, 28.0) <= best) {
    bn = 96;
    best = cost(96, 28.0);
  }
  if (N > 64 && fits(128) && cost(128, 32.0) <= best) bn = 128;
  return bn;
}

// Row strides and column offsets of the epilogue's fp32 (float4) and planes (uint2) accesses: multiples of 4 elements
// that fit the kernel's int fields.
static bool bad_ld(int64_t ld) { return ld < 0 || ld > INT32_MAX || ld % 4 != 0; }

// Every descriptor rule the producer and the epilogue rely on, checked before anything touches the driver.
static int check_desc(const s3r_gemm_desc& d) {
  if (d.precision != GEMM_SPLIT && d.precision != GEMM_BF16) {
    set_error("s3r_gemm: precision=%d must be 0 (split bf16) or 1 (one bf16 product)", d.precision);
    return -1;
  }
  if (d.precision == GEMM_BF16 && d.epi == S3R_EPI_HEADTAIL) {
    set_error("s3r_gemm: precision=1 does not support EPI_HEADTAIL (the DPT head tail is split-only)");
    return -1;
  }
  if (d.taps != 1 && d.taps != 9) {
    set_error("s3r_gemm: taps=%d must be 1 or 9", d.taps);
    return -1;
  }
  if (d.taps == 9 && d.kc % 8 != 0) {
    set_error("s3r_gemm: kc=%d of a 3x3 conv must be a multiple of 8 (16-byte tap stride)", d.kc);
    return -1;
  }
  // TMA row strides: multiples of 16 bytes
  const struct { const char* name; int64_t v; } strides[2] = {{"lda", d.lda ? d.lda : d.kc},
                                                              {"ldb", d.ldb ? d.ldb : (int64_t)d.kc * d.taps}};
  for (const auto& s : strides)
    if (s.v < 0 || s.v % 8 != 0) {
      set_error("s3r_gemm: %s=%lld must be a non-negative multiple of 8 (0 = dense)", s.name, (long long)s.v);
      return -1;
    }
  if (d.b_group_rows < 0 || d.b_group_rows > INT32_MAX) {
    set_error("s3r_gemm: b_group_rows=%lld must be in [0, 2^31) (0 = n)", (long long)d.b_group_rows);
    return -1;
  }
  // the epilogue stores whole 32-column chunks; past n that is only harmless in a bare fp32 output wide enough for them
  const bool chunk_tail_ok = d.epi == S3R_EPI_PLAIN && !d.out_hi && !d.stats_out && !d.res1 && !d.res2 && d.out_f32 &&
                             d.ldo >= (d.n + 31) / 32 * 32;
  if (d.n <= 0 || (d.n % 32 != 0 && !chunk_tail_ok)) {
    set_error("s3r_gemm: n=%d must be a positive multiple of 32 (the epilogue stores whole 32-column chunks; only a bare "
              "out_f32 with ldo >= n rounded up to 32 may take the tail)", d.n);
    return -1;
  }
  if (d.epi == S3R_EPI_HEADTAIL && d.n != 128) {
    set_error("s3r_gemm: EPI_HEADTAIL needs n == 128");
    return -1;
  }
  if (d.epi == S3R_EPI_PIXSHUF && (d.ps_s <= 0 || d.ps_cout % 32 != 0 || d.n != d.ps_s * d.ps_s * d.ps_cout)) {
    set_error("s3r_gemm: EPI_PIXSHUF needs n == s*s*cout and cout %% 32 == 0");
    return -1;
  }
  const struct { const char* name; bool used; int64_t v; } lds[5] = {
      {"ldr1", d.res1 != nullptr, d.ldr1}, {"ldr2", d.res2 != nullptr, d.ldr2}, {"ldo", d.out_f32 != nullptr, d.ldo},
      {"ldp", d.out_hi != nullptr, d.ldp}, {"plane_col0", d.out_hi != nullptr, d.plane_col0}};
  for (const auto& l : lds)
    if (l.used && bad_ld(l.v)) {
      set_error("s3r_gemm: %s=%lld must be a non-negative multiple of 4 below 2^31 (vector accesses)", l.name,
                (long long)l.v);
      return -1;
    }
  if (d.epi == S3R_EPI_QKV) {
    if (d.q_c <= 0 || d.q_c % 64 != 0 || d.h != 1 || d.q_ntok <= 0 || d.w != d.q_nb * d.q_ntok) {
      set_error("s3r_gemm: EPI_QKV needs q_c %% 64 == 0, h == 1, w == q_nb*q_ntok");
      return -1;
    }
    if (d.n % d.q_c != 0) {
      set_error("s3r_gemm: EPI_QKV n=%d must be a multiple of q_c=%d", d.n, d.q_c);
      return -1;
    }
    if (d.q_role_base < 0 || d.q_role_base + d.n / d.q_c > 5) {
      set_error("s3r_gemm: EPI_QKV q_role_base=%d + n/q_c=%d must stay within the 5 roles", d.q_role_base,
                d.n / d.q_c);
      return -1;
    }
    if (d.q_ntok_pad < d.q_ntok || d.q_ntok_pad % 4 != 0) {
      set_error("s3r_gemm: EPI_QKV q_ntok_pad=%d must be >= q_ntok=%d and a multiple of 4", d.q_ntok_pad, d.q_ntok);
      return -1;
    }
    static const char* const kRoleOut[5] = {"q_out", "k_out", "vt_out", "k2_out", "vt2_out"};
    const float* const role_out[5] = {d.q_out, d.k_out, d.vt_out, d.k2_out, d.vt2_out};
    for (int role = d.q_role_base; role < d.q_role_base + d.n / d.q_c; ++role)
      if (!role_out[role]) {
        set_error("s3r_gemm: EPI_QKV role %d is written but %s is NULL", role, kRoleOut[role]);
        return -1;
      }
    if (d.q_rope && (!d.q_pos || !d.q_cs)) {
      set_error("s3r_gemm: EPI_QKV with q_rope needs %s", d.q_pos ? "q_cs" : "q_pos");
      return -1;
    }
  }
  if (d.ln_stats) {
    if (d.ln_cs == nullptr || d.ln_np * 32 != d.kc || d.taps != 1 || d.epi == S3R_EPI_PIXSHUF) {
      set_error("s3r_gemm: folded LayerNorm needs ln_cs, ln_np == kc/32, taps == 1 and a non-PIXSHUF epilogue");
      return -1;
    }
    if (d.ln_np < 2 || d.ln_np > 32 || d.ln_np % 2 != 0) {
      set_error("s3r_gemm: folded LayerNorm needs an even ln_np in [2, 32] (kc %% 64 == 0, kc <= 1024), got ln_np=%d",
                d.ln_np);
      return -1;
    }
  }
  if (d.swap_col0 % 256 != 0) {
    set_error("s3r_gemm: swap_col0 must be a multiple of 256");
    return -1;
  }
  if (d.stats_out && d.epi != S3R_EPI_PLAIN) {
    set_error("s3r_gemm: stats_out needs EPI_PLAIN");
    return -1;
  }
  return 0;
}

void gemm_set_epilogue(const s3r_gemm_desc& d, GemmArgs& a) {
  a.epi = d.epi; a.act = d.act; a.plane_relu = d.plane_relu;
  a.bias = d.bias;
  a.res1 = d.res1; a.ldr1 = (int)d.ldr1;
  a.res2 = d.res2; a.ldr2 = (int)d.ldr2;
  a.out_f32 = d.out_f32; a.ldo = (int)d.ldo;
  a.out_hi = (__nv_bfloat16*)d.out_hi; a.out_lo = (__nv_bfloat16*)d.out_lo; a.ldp = (int)d.ldp;
  a.plane_col0 = d.plane_col0;
  if (d.epi == S3R_EPI_PIXSHUF) {
    a.ps_s = d.ps_s; a.ps_cout = d.ps_cout;
    a.out_group_rows = (long long)d.nb * d.h * d.ps_s * d.w * d.ps_s;
  }
  if (d.epi == S3R_EPI_QKV) {
    a.q_C = d.q_c; a.q_role_base = d.q_role_base; a.q_ntok = d.q_ntok; a.q_ntok_pad = d.q_ntok_pad;
    a.q_rope = d.q_rope; a.q_nb = d.q_nb; a.q_pos = d.q_pos;
    a.q_cs = reinterpret_cast<const float2*>(d.q_cs);
    a.q_out = d.q_out; a.k_out = d.k_out; a.vt_out = d.vt_out; a.q_scale = d.q_scale;
    a.k2_out = d.k2_out; a.vt2_out = d.vt2_out;
  }
  if (d.epi == S3R_EPI_HEADTAIL) {
    a.ht_w = d.ht_w; a.ht_b = d.ht_b; a.ht_pts = d.ht_pts; a.ht_conf = d.ht_conf;
  }
  if (d.ln_stats) {
    a.ln_stats = reinterpret_cast<const float2*>(d.ln_stats); a.ln_np = d.ln_np; a.ln_eps = d.ln_eps; a.ln_cs = d.ln_cs;
  }
  a.a_swap = d.a_swap ? 1 : 0;
  a.swap_col0 = d.swap_col0;
  a.stats_out = reinterpret_cast<float2*>(d.stats_out);
  a.trace = reinterpret_cast<unsigned long long*>(d.trace);
  a.b_static = d.b_static ? 1 : 0;
}

int gemm_plan(const s3r_gemm_desc& d, GemmPlan* plan) {
  memset(plan, 0, sizeof(*plan));
  if (int r = check_desc(d)) return r;
  const int groups = d.groups, NB = d.nb, H = d.h, W = d.w, Kc = d.kc, taps = d.taps, N = d.n;
  const long long lda = d.lda ? d.lda : Kc, ldb = d.ldb ? d.ldb : (long long)Kc * taps;
  const long long b_group_rows = d.b_group_rows ? d.b_group_rows : N;
  plan->precision = d.precision;
  GemmArgs& a = plan->args;
  a.b_group_rows = (int)b_group_rows;
  a.W = W; a.H = H; a.NB = NB; a.N = N; a.Kc = Kc; a.taps = taps;
  a.kpt = (Kc + BK - 1) / BK;
  a.bw = W >= 128 ? 128 : next_pow2(W);
  a.bh = 128 / a.bw;
  a.tiles_w = (W + a.bw - 1) / a.bw;
  a.tiles_h = (H + a.bh - 1) / a.bh;
  a.out_group_rows = (long long)NB * H * W;
  const long long m_tiles = (long long)a.tiles_w * a.tiles_h * NB * groups;
  // the DPT head tail's hand-over pairs the two column halves of a 128-wide tile (launch_epi)
  const int bn = gemm_choose_bn(m_tiles, N, num_sms(), d.a_swap ? d.swap_col0 : 0,
                                d.epi == S3R_EPI_HEADTAIL ? 128 : d.force_bn);
  if (bn < 0) return -1;
  plan->bn = bn;

  const uint64_t esz = 2;
  {
    uint64_t dims[4] = {(uint64_t)Kc, (uint64_t)W, (uint64_t)H, (uint64_t)NB * groups};
    uint64_t str[3] = {(uint64_t)lda * esz, (uint64_t)lda * W * esz, (uint64_t)lda * W * H * esz};
    uint32_t box[4] = {(uint32_t)BK, (uint32_t)a.bw, (uint32_t)a.bh, 1};
    int r;
    if ((r = encode_tmap(&a.tmA_hi, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, d.a_hi, dims, str, box, kSwizzle))) return r;
    if (d.precision == GEMM_SPLIT &&
        (r = encode_tmap(&a.tmA_lo, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, d.a_lo, dims, str, box, kSwizzle)))
      return r;
  }
  {
    uint64_t dims[3] = {(uint64_t)Kc, (uint64_t)taps, (uint64_t)(b_group_rows * (groups - 1) + N)};
    // with a single tap the tap stride is never used, but must still be a multiple of 16 bytes
    uint64_t str[2] = {(uint64_t)(taps == 1 ? ldb : Kc) * esz, (uint64_t)ldb * esz};
    uint32_t box[3] = {(uint32_t)BK, 1, (uint32_t)bn};
    int r;
    if ((r = encode_tmap(&a.tmB_hi, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, d.b_hi, dims, str, box, kSwizzle))) return r;
    if (d.precision == GEMM_SPLIT &&
        (r = encode_tmap(&a.tmB_lo, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, d.b_lo, dims, str, box, kSwizzle)))
      return r;
  }
  const long long n_tiles = (N + bn - 1) / bn;
  const long long total = m_tiles * n_tiles;
  a.groups = groups;
  plan->grid = dim3((unsigned)((total < num_sms()) ? total : num_sms()), 1, 1);  // persistent: <= 1 CTA per SM
  plan->flops = 2.0 * (double)NB * H * W * groups * (double)N * (double)Kc * taps;
  gemm_set_epilogue(d, a);
  return 0;
}

template <int BN, int EPI, int NP>
static int launch_bn(const GemmPlan& plan, cudaStream_t stream) {
  using Cfg = GemmCfg<BN, NP>;
  static PerDeviceOnce once;
  bool& attr_set = once.cur();
  if (!attr_set) {
    cudaError_t e =
        cudaFuncSetAttribute(gemm_bf16x3_kernel<BN, EPI, NP>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM);
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(smem=%d): %s", Cfg::SMEM, cudaGetErrorString(e));
      return -5;
    }
    attr_set = true;
  }
  cudaError_t e = launch_pdl(gemm_bf16x3_kernel<BN, EPI, NP>, plan.grid, dim3(kNumThreads), Cfg::SMEM, stream, plan.args);
  if (e != cudaSuccess) {
    set_error("gemm launch failed: %s", cudaGetErrorString(e));
    return -6;
  }
  return 0;
}

template <int BN, int NP>
static int launch_epi(const GemmPlan& plan, cudaStream_t stream) {
  switch (plan.args.epi) {
    case EPI_PLAIN: return launch_bn<BN, EPI_PLAIN, NP>(plan, stream);
    case EPI_PIXSHUF: return launch_bn<BN, EPI_PIXSHUF, NP>(plan, stream);
    case EPI_QKV: return launch_bn<BN, EPI_QKV, NP>(plan, stream);
    case EPI_HEADTAIL:
      // the DPT head tail runs in heads(), which is always split; not instantiated at one product (it would spill), nor
      // at BN = 96 (its hand-over pairs the two column halves; the planner pins it to 128)
      if constexpr (NP == 3 && BN != 96) return launch_bn<BN, EPI_HEADTAIL, NP>(plan, stream);
      break;
  }
  set_error("gemm_launch: bad epilogue mode %d", plan.args.epi);
  return -1;
}

template <int NP>
static int launch_np(const GemmPlan& plan, cudaStream_t stream) {
  switch (plan.bn) {
    case 64: return launch_epi<64, NP>(plan, stream);
    case 96: return launch_epi<96, NP>(plan, stream);
    case 128: return launch_epi<128, NP>(plan, stream);
  }
  set_error("gemm_launch: bad bn %d", plan.bn);
  return -1;
}

int gemm_launch(const GemmPlan& plan, cudaStream_t stream) {
  switch (plan.precision) {
    case GEMM_SPLIT: return launch_np<3>(plan, stream);
    case GEMM_BF16: return launch_np<1>(plan, stream);
  }
  set_error("gemm_launch: bad precision %d", plan.precision);
  return -1;
}

}  // namespace s3r

using namespace s3r;

extern "C" {

int s3r_gemm(const s3r_gemm_desc* d, void* stream) {
  GemmPlan plan;
  if (int r = gemm_plan(*d, &plan)) return r;
  return gemm_launch(plan, static_cast<cudaStream_t>(stream));
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

}  // extern "C"
