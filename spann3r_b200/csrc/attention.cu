// Fused multi-head attention core for head dim 64 on Hopper wgmma (tf32), sm_90a.
//
//   O[b, q, h*64:(h+1)*64] = softmax_k( Q[b,h,q,:] . K[b,h,k,:] ) V[b,h,k,:]
//
// Replaces the materialised `q @ k.T -> softmax -> @ v` of croco/models/blocks.py:106-110 (self
// attention of Block / DecoderBlock) and :162-166 (CrossAttention).  Q and K arrive already rotated
// (2-D RoPE), Q pre-scaled by 64^-0.5, V transposed, all rounded to tf32 by the QKV-projection GEMM
// epilogue (gemm.cu, EPI_QKV), so RoPE never exists as a separate op or tensor.
//
// One CTA per (128-query tile, batch*head), 384 threads: warpgroup 0 = TMA producer (Q once, K / V^T per 128-key
// block into a 3-stage ring), warpgroups 1 and 2 each own 64 query rows for ALL KV blocks: S = Q K^T into registers
// (wgmma, A and B from shared memory), exact online softmax in registers, O += P V with P as the register A operand.
// Output: split-bf16 planes (A operand of the following projection GEMM) and/or fp32.
#include "common.cuh"
#include "kernels.cuh"
#include "wgmma.cuh"

#include <cstdlib>
#include <cstring>

namespace s3r {

namespace attn {
constexpr int BQ = 128;   // queries per CTA
constexpr int BKV = 128;  // keys per block
constexpr int D = 64;
constexpr int Q_BYTES = BQ * D * 4;       // 32 KB (2 swizzle atoms of [128 x 32 f32])
constexpr int K_BYTES = BKV * D * 4;      // 32 KB
constexpr int V_BYTES = D * BKV * 4;      // 32 KB (4 atoms of [64 x 32 f32])
constexpr int KV_STAGES = 3;
constexpr int SMEM = Q_BYTES + KV_STAGES * (K_BYTES + V_BYTES) + 1024 + 256;
constexpr int kThreads = 384;             // warpgroup 0: warp 0 TMA (1..3 idle); warpgroups 1, 2: MMA + softmax
constexpr int kConsumerWarps = 8;
}  // namespace attn

__global__ void __launch_bounds__(attn::kThreads, 1) attention_kernel(const __grid_constant__ AttnArgs args) {
  using namespace attn;
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment by pointer arithmetic on the __shared__ array (an integer round trip would lose the address
  // space and turn every access through `smem` into a generic LD / ST)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sQ = smem;
  uint8_t* sKV = sQ + Q_BYTES;                      // stage s: K at s*(K+V), V after K
  uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + KV_STAGES * (K_BYTES + V_BYTES));
  uint64_t* q_full = bars;                          // 1
  uint64_t* kv_full = bars + 1;                     // KV_STAGES
  uint64_t* kv_empty = bars + 1 + KV_STAGES;        // KV_STAGES

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * BQ;
  const int bh = blockIdx.y;
  const int nblk = (args.nk + BKV - 1) / BKV;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&args.tmQ);
    tma_prefetch_desc(&args.tmK);
    tma_prefetch_desc(&args.tmV);
    mbar_init(q_full, 1);
    for (int i = 0; i < KV_STAGES; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], kConsumerWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  if (warp < 4) {
    // register re-balancing: the TMA warpgroup needs few registers, each consumer thread holds S, P and O fragments
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0 && lane == 0) {
      mbar_arrive_expect_tx(q_full, Q_BYTES);
      tma_load_3d(sQ, &args.tmQ, q_full, 0, q0, bh);
      tma_load_3d(sQ + Q_BYTES / 2, &args.tmQ, q_full, 32, q0, bh);
      for (int j = 0; j < nblk; ++j) {
        const int st = j % KV_STAGES;
        const uint32_t ph = (j / KV_STAGES) & 1;
        mbar_wait(&kv_empty[st], ph ^ 1);
        uint8_t* k = sKV + st * (K_BYTES + V_BYTES);
        uint8_t* v = k + K_BYTES;
        mbar_arrive_expect_tx(&kv_full[st], K_BYTES + V_BYTES);
        tma_load_3d(k, &args.tmK, &kv_full[st], 0, j * BKV, bh);
        tma_load_3d(k + K_BYTES / 2, &args.tmK, &kv_full[st], 32, j * BKV, bh);
#pragma unroll
        for (int a = 0; a < 4; ++a) tma_load_3d(v + a * (V_BYTES / 4), &args.tmV, &kv_full[st], j * BKV + a * 32, 0, bh);
      }
    }
    return;
  }

  // ------------------------------------------------------------------ consumers
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int wg = (warp - 4) >> 2;        // rows [64 wg, 64 wg + 64) of the query tile
  const int wq = warp & 3;               // this warp: rows 16 wq + g and 16 wq + g + 8 of them
  const int g = lane >> 2, t4 = lane & 3;
  const uint32_t aQ = __shfl_sync(0xffffffffu, smem_u32(sQ), 0) + wg * (64 * 128);
  const uint32_t aKV = __shfl_sync(0xffffffffu, smem_u32(sKV), 0);
  constexpr float kLog2e = 1.4426950408889634f;

  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // rows g and g + 8: running max, partial row sums
  // P fragment sources: key 8kk + t4 of a row is column 2 (t4 / 2) + (t4 & 1) of lane 4g + t4 / 2, key 8kk + t4 + 4 the
  // same column of lane 4g + 2 + t4 / 2
  const int src_lo = (lane & ~3) | (t4 >> 1), src_hi = src_lo + 2;
  const bool odd = (t4 & 1) != 0;

  mbar_wait(q_full, 0);
  for (int j = 0; j < nblk; ++j) {
    const int st = j % KV_STAGES;
    mbar_wait(&kv_full[st], (j / KV_STAGES) & 1);
    const uint32_t aK = aKV + st * (K_BYTES + V_BYTES);
    const uint32_t aV = aK + K_BYTES;

    // S = Q K^T: 64 x 128 per warpgroup, 8 K-steps of 8 (two 32-wide swizzle atoms of the head dim)
    float s[64];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      const uint32_t part = (kk >> 2) * (Q_BYTES / 2), ko = (kk & 3) * 2;
      wgmma_tf32_n128_ss(s, wgmma_desc_sw128_kmajor(aQ + part) + ko, wgmma_desc_sw128_kmajor(aK + part) + ko, kk > 0);
    }
    wgmma_commit();
    wgmma_wait<0>();

    const int kbase = j * BKV;
    if (kbase + BKV > args.nk) {   // ragged last block: keys beyond nk do not exist
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int c = kbase + 8 * i + 2 * t4;
        if (c >= args.nk) { s[4 * i] = -INFINITY; s[4 * i + 2] = -INFINITY; }
        if (c + 1 >= args.nk) { s[4 * i + 1] = -INFINITY; s[4 * i + 3] = -INFINITY; }
      }
    }
    float b0 = -INFINITY, b1 = -INFINITY;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      b0 = fmaxf(b0, fmaxf(s[4 * i], s[4 * i + 1]));
      b1 = fmaxf(b1, fmaxf(s[4 * i + 2], s[4 * i + 3]));
    }
#pragma unroll
    for (int x = 1; x < 4; x <<= 1) {
      b0 = fmaxf(b0, __shfl_xor_sync(0xffffffffu, b0, x));
      b1 = fmaxf(b1, __shfl_xor_sync(0xffffffffu, b1, x));
    }
    const float n0 = fmaxf(m0, b0), n1 = fmaxf(m1, b1);
    const float al0 = (j == 0) ? 0.f : exp2f((m0 - n0) * kLog2e);
    const float al1 = (j == 0) ? 0.f : exp2f((m1 - n1) * kLog2e);
    m0 = n0;
    m1 = n1;
    const float nr0 = -n0 * kLog2e, nr1 = -n1 * kLog2e;
    float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      const bool r1 = (i & 2) != 0;
      const float e = exp2f(fmaf(s[i], kLog2e, r1 ? nr1 : nr0));            // exp(s - max); exp(-inf) = 0
      const uint32_t rb = (__float_as_uint(e) + 0x1000u) & 0xffffe000u;     // round to tf32 (the MMA truncates)
      s[i] = __uint_as_float(rb);
      if (r1) ps1 += s[i]; else ps0 += s[i];
    }
    l0 = l0 * al0 + ps0;
    l1 = l1 * al1 + ps1;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      o[4 * i] *= al0; o[4 * i + 1] *= al0;
      o[4 * i + 2] *= al1; o[4 * i + 3] *= al1;
    }

    // P (accumulator layout) -> tf32 A fragments: a0 (g, k), a1 (g+8, k), a2 (g, k+4), a3 (g+8, k+4), k = t4
    uint32_t pa[16][4];
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      const float x0 = __shfl_sync(0xffffffffu, s[4 * kk], src_lo), x1 = __shfl_sync(0xffffffffu, s[4 * kk + 1], src_lo);
      const float y0 = __shfl_sync(0xffffffffu, s[4 * kk + 2], src_lo), y1 = __shfl_sync(0xffffffffu, s[4 * kk + 3], src_lo);
      const float z0 = __shfl_sync(0xffffffffu, s[4 * kk], src_hi), z1 = __shfl_sync(0xffffffffu, s[4 * kk + 1], src_hi);
      const float w0 = __shfl_sync(0xffffffffu, s[4 * kk + 2], src_hi), w1 = __shfl_sync(0xffffffffu, s[4 * kk + 3], src_hi);
      pa[kk][0] = __float_as_uint(odd ? x1 : x0);
      pa[kk][1] = __float_as_uint(odd ? y1 : y0);
      pa[kk][2] = __float_as_uint(odd ? z1 : z0);
      pa[kk][3] = __float_as_uint(odd ? w1 : w0);
    }
    // O += P V: 16 K-steps of 8 keys; V^T is stored as four 32-key swizzle atoms of [64 x 32 f32]
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk)
      wgmma_tf32_n64_rs(o, pa[kk], wgmma_desc_sw128_kmajor(aV + (kk >> 2) * (V_BYTES / 4)) + (kk & 3) * 2, 1);
    wgmma_commit();
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[st]);   // this warp's reads of the stage have retired
  }

#pragma unroll
  for (int x = 1; x < 4; x <<= 1) {
    l0 += __shfl_xor_sync(0xffffffffu, l0, x);
    l1 += __shfl_xor_sync(0xffffffffu, l1, x);
  }
  const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
  const int b = bh / args.heads, h = bh - b * args.heads;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int q = q0 + wg * 64 + wq * 16 + g + 8 * r;
    if (q >= args.nq) continue;
    const float inv = r ? inv1 : inv0;
    const long long row = ((long long)b * args.nq + q) * args.ldo + h * D;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float x = o[4 * i + 2 * r] * inv, y = o[4 * i + 2 * r + 1] * inv;
      const long long off = row + 8 * i + 2 * t4;
      if (args.o_f32) *reinterpret_cast<float2*>(args.o_f32 + off) = make_float2(x, y);
      if (args.o_hi) {
        uint32_t hh, ll;
        split2_bf16(x, y, hh, ll);
        *reinterpret_cast<uint32_t*>(args.o_hi + off) = hh;
        *reinterpret_cast<uint32_t*>(args.o_lo + off) = ll;
      }
    }
  }
}

int attn_plan_init(AttnPlan* plan, const float* q, const float* k, const float* vt, int BH, int heads, int nq, int nk,
                   int nk_pad) {
  using namespace attn;
  memset(plan, 0, sizeof(*plan));
  if (nk_pad % 4 != 0 || nk_pad < nk) {
    set_error("attention: nk_pad=%d must be >= nk=%d and a multiple of 4", nk_pad, nk);
    return -1;
  }
  AttnArgs& a = plan->args;
  {
    uint64_t dims[3] = {64, (uint64_t)nq, (uint64_t)BH};
    uint64_t str[2] = {64 * 4, (uint64_t)nq * 64 * 4};
    uint32_t box[3] = {32, (uint32_t)BQ, 1};
    int r = encode_tmap(&a.tmQ, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, q, dims, str, box);
    if (r) return r;
  }
  {
    uint64_t dims[3] = {64, (uint64_t)nk, (uint64_t)BH};
    uint64_t str[2] = {64 * 4, (uint64_t)nk * 64 * 4};
    uint32_t box[3] = {32, (uint32_t)BKV, 1};
    int r = encode_tmap(&a.tmK, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, k, dims, str, box);
    if (r) return r;
  }
  {
    uint64_t dims[3] = {(uint64_t)nk, 64, (uint64_t)BH};
    uint64_t str[2] = {(uint64_t)nk_pad * 4, (uint64_t)nk_pad * 64 * 4};
    uint32_t box[3] = {32, 64, 1};
    int r = encode_tmap(&a.tmV, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, vt, dims, str, box);
    if (r) return r;
  }
  a.nq = nq; a.nk = nk; a.heads = heads;
  plan->grid = dim3((nq + BQ - 1) / BQ, BH);
  plan->flops = 4.0 * BH * (double)nq * nk * 64;
  return 0;
}

static int attn_launch_args(const AttnPlan& plan, const AttnArgs& a, cudaStream_t st) {
  using namespace attn;
  static PerDeviceOnce once;
  bool& attr_set = once.cur();
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) {
      set_error("attention: cudaFuncSetAttribute(smem=%d): %s", SMEM, cudaGetErrorString(e));
      return -5;
    }
    attr_set = true;
  }
  cudaError_t e = launch_pdl(attention_kernel, plan.grid, dim3(kThreads), SMEM, st, a);
  if (e != cudaSuccess) {
    set_error("attention launch failed: %s", cudaGetErrorString(e));
    return -6;
  }
  return 0;
}

int attn_launch(const AttnPlan& plan, __nv_bfloat16* o_hi, __nv_bfloat16* o_lo, float* o_f32, long long ldo,
                cudaStream_t st) {
  AttnArgs a = plan.args;
  a.o_hi = o_hi; a.o_lo = o_lo; a.o_f32 = o_f32; a.ldo = ldo;
  return attn_launch_args(plan, a, st);
}

int launch_attention(const float* q, const float* k, const float* vt, int BH, int heads, int nq, int nk, int nk_pad,
                     __nv_bfloat16* o_hi, __nv_bfloat16* o_lo, float* o_f32, long long ldo, cudaStream_t st) {
  if (nq <= 0 || nk <= 0 || BH <= 0) return 0;
  AttnPlan plan;
  int r = attn_plan_init(&plan, q, k, vt, BH, heads, nq, nk, nk_pad);
  if (r) return r;
  return attn_launch(plan, o_hi, o_lo, o_f32, ldo, st);
}

}  // namespace s3r
