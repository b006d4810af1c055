// Attention of the training backward on sm_90a: a flash forward that keeps O and one log-sum-exp per row, and a backward
// that rebuilds the probabilities from that log-sum-exp -- no [images * heads, nq, nk] score or probability tensor exists
// at any point, so the memory is O(N) instead of O(N^2).
//
//   S = scale Q K^T,  P = softmax(S) = exp(S - LSE),  O = P V
//   D = rowsum(dO o O),  dS = P o (dO V^T - D),  dQ = scale dS K,  dK = scale dS^T Q,  dV = P^T dO
//
// Arithmetic: every product (Q K^T and P V forward; Q K^T, dO V^T, P^T dO, dS^T Q and dS K backward) is split-bf16 on the
// tensor cores: x = hi + lo with hi = bf16(x), lo = bf16(x - hi), and a . b = hi.hi + hi.lo + lo.hi accumulated in fp32
// (DESIGN §3), so the result is fp32-grade whatever torch.backends.cuda.matmul.allow_tf32 says.  The softmax, its
// running max / sum, D and dS are fp32.
//
// Layout: q, k, v are fp32 [batch, heads, n, dh] with arbitrary element strides (multiples of 4) and dh contiguous, as
// the recompute's views of the qkv Linear produce them; O and dO are [batch, nq, heads * dh] (what the attention's proj
// reads), LSE is [batch * heads, nq], dQ / dK / dV are contiguous [batch, heads, n, dh].  Each CTA stages 64-row tiles
// into shared memory, splitting fp32 into hi / lo planes on the way, with the head dim zero-padded to 64 (dh = 48: the
// padding columns contribute exact zeros) and rows past nq / nk zero-filled and masked out of the softmax, so nq and nk
// may be any value >= 1.
//
// Kernels (4 warps each; a warp owns 16 rows of the CTA's 64-row tile and issues mma.sync m16n8k16 bf16):
//   attn_train_fwd_kernel   one CTA per (64 queries, batch * head), loop over key tiles: online softmax, O and LSE.
//   attn_train_rowdot_kernel  D = rowsum(dO o O), one warp per row, fixed butterfly order.
//   attn_train_dkdv_kernel  one CTA per (64 keys, batch * head), loop over query tiles: dK, dV in registers.
//   attn_train_dq_kernel    one CTA per (64 queries, batch * head), loop over key tiles: dQ in registers.
// dQ has its own pass (and so its own Q K^T and dO V^T) instead of float atomics: every output element is written once,
// by one thread, after a fixed-order loop, so two calls give bitwise-identical results.
//
// The fp32 accumulator of an m16n8 tile holds, per thread, rows (g, g + 8) x columns (2t, 2t + 1) (g = lane / 4,
// t = lane % 4); two neighbouring n8 tiles are exactly the m16k16 A fragment of the next product, so P and dS feed it
// as hi / lo registers without any shuffle.
#include <cmath>
#include <cstdint>
#include <cstring>

#include "../../include/spann3r_b200.h"
#include "common.cuh"
#include "gemm.cuh"

namespace s3r {
namespace {

constexpr int kT = 64;              // rows of a query / key tile
constexpr int kPitch = 72;          // bf16 row pitch of a shared tile: 144 B, conflict-free 32-bit fragment loads
constexpr int kTile = kT * kPitch;  // bf16 elements of one shared plane
constexpr int kThreads = 128;
constexpr int kDkdvSmem = 12 * kTile * 2 + 2 * kT * 4;
constexpr int kDqSmem = 10 * kTile * 2;

struct Src {
  const float* p;
  long long sb, sh, sn;             // element strides of batch, head, token
};

struct Params {
  Src q, k, v, o, dout;
  int heads, nq, nk, dh;
  long long rows;                   // batch * heads * nq
  float scale;
  float* o_out;
  float* lse;
  float* dvec;
  float* dq;
  float* dk;
  float* dv;
};

__device__ __forceinline__ uint32_t pack_split(float a, float b, uint32_t& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  const float2 hf = __bfloat1622float2(h);
  const __nv_bfloat162 l = __floats2bfloat162_rn(a - hf.x, b - hf.y);
  lo = *reinterpret_cast<const uint32_t*>(&l);
  return *reinterpret_cast<const uint32_t*>(&h);
}

__device__ __forceinline__ void mma(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// c += a . b in split-bf16: the two small cross terms first, then hi . hi
__device__ __forceinline__ void mma3(float (&c)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4], const uint32_t (&bh)[2],
                                     const uint32_t (&bl)[2]) {
  mma(c, al, bh[0], bh[1]);
  mma(c, ah, bl[0], bl[1]);
  mma(c, ah, bh[0], bh[1]);
}

__device__ __forceinline__ uint32_t ld32(const __nv_bfloat16* s, int row, int col) {
  return *reinterpret_cast<const uint32_t*>(s + row * kPitch + col);
}

// A fragment (16 x 16) at rows r0.., contraction columns k0.. of a row-major [rows][k] plane
__device__ __forceinline__ void frag_a(uint32_t (&a)[4], const __nv_bfloat16* s, int r0, int k0, int g, int t) {
  a[0] = ld32(s, r0 + g, k0 + 2 * t);
  a[1] = ld32(s, r0 + g + 8, k0 + 2 * t);
  a[2] = ld32(s, r0 + g, k0 + 2 * t + 8);
  a[3] = ld32(s, r0 + g + 8, k0 + 2 * t + 8);
}

// B fragment (16 x 8) at output columns n0.., contraction k0.. of a plane stored [n][k]
__device__ __forceinline__ void frag_b(uint32_t (&bh)[2], uint32_t (&bl)[2], const __nv_bfloat16* hi, const __nv_bfloat16* lo,
                                       int n0, int k0, int g, int t) {
  bh[0] = ld32(hi, n0 + g, k0 + 2 * t);
  bh[1] = ld32(hi, n0 + g, k0 + 2 * t + 8);
  bl[0] = ld32(lo, n0 + g, k0 + 2 * t);
  bl[1] = ld32(lo, n0 + g, k0 + 2 * t + 8);
}

// A fragments (hi, lo) of contraction block kk from a 16 x 64 fp32 accumulator c[8][4]
__device__ __forceinline__ void frag_acc(uint32_t (&ah)[4], uint32_t (&al)[4], const float (&c)[8][4], int kk) {
  ah[0] = pack_split(c[2 * kk][0], c[2 * kk][1], al[0]);
  ah[1] = pack_split(c[2 * kk][2], c[2 * kk][3], al[1]);
  ah[2] = pack_split(c[2 * kk + 1][0], c[2 * kk + 1][1], al[2]);
  ah[3] = pack_split(c[2 * kk + 1][2], c[2 * kk + 1][3], al[3]);
}

__device__ __forceinline__ void zero(float (&c)[8][4]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) c[j][0] = c[j][1] = c[j][2] = c[j][3] = 0.f;
}

// Rows [r0, r0 + 64) x columns [0, 64) of slice (b, h) of `s` into split planes: row-major [row][col] into (hi, lo) and /
// or transposed [col][row] into (thi, tlo).  Rows >= n and columns >= dh are zero.
__device__ __forceinline__ void load_tile(const Src& s, int b, int h, int r0, int n, int dh, __nv_bfloat16* hi,
                                          __nv_bfloat16* lo, __nv_bfloat16* thi, __nv_bfloat16* tlo) {
  const float* base = s.p + (long long)b * s.sb + (long long)h * s.sh;
  for (int i = threadIdx.x; i < kT * 16; i += kThreads) {
    const int r = i >> 4, c = (i & 15) * 4;
    float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r0 + r < n && c < dh) x = __ldg(reinterpret_cast<const float4*>(base + (long long)(r0 + r) * s.sn + c));
    uint32_t l01, l23;
    const uint32_t h01 = pack_split(x.x, x.y, l01), h23 = pack_split(x.z, x.w, l23);
    if (hi) {
      *reinterpret_cast<uint2*>(hi + r * kPitch + c) = make_uint2(h01, h23);
      *reinterpret_cast<uint2*>(lo + r * kPitch + c) = make_uint2(l01, l23);
    }
    if (thi) {
      const uint32_t hv[2] = {h01, h23}, lv[2] = {l01, l23};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const unsigned short hb = (unsigned short)(hv[e >> 1] >> (16 * (e & 1)));
        const unsigned short lb = (unsigned short)(lv[e >> 1] >> (16 * (e & 1)));
        reinterpret_cast<unsigned short*>(thi)[(c + e) * kPitch + r] = hb;
        reinterpret_cast<unsigned short*>(tlo)[(c + e) * kPitch + r] = lb;
      }
    }
  }
}

__global__ void __launch_bounds__(kThreads) attn_train_fwd_kernel(const Params p) {
  __shared__ __align__(16) __nv_bfloat16 sm[4 * kTile];
  __nv_bfloat16 *sKh = sm, *sKl = sm + kTile, *sVh = sm + 2 * kTile, *sVl = sm + 3 * kTile;   // K [key][d], V^T [d][key]
  const int bh = blockIdx.y, b = bh / p.heads, h = bh % p.heads;
  const int q0 = blockIdx.x * kT;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int r0 = warp * 16;

  uint32_t qh[4][4], ql[4][4];
  load_tile(p.q, b, h, q0, p.nq, p.dh, sKh, sKl, nullptr, nullptr);
  __syncthreads();
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    frag_a(qh[kk], sKh, r0, 16 * kk, g, t);
    frag_a(ql[kk], sKl, r0, 16 * kk, g, t);
  }

  float o[8][4];
  zero(o);
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // rows g, g + 8 (l: this thread's columns only)
  for (int j0 = 0; j0 < p.nk; j0 += kT) {
    __syncthreads();
    load_tile(p.k, b, h, j0, p.nk, p.dh, sKh, sKl, nullptr, nullptr);
    load_tile(p.v, b, h, j0, p.nk, p.dh, nullptr, nullptr, sVh, sVl);
    __syncthreads();
    float s[8][4];
    zero(s);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        uint32_t bh_[2], bl_[2];
        frag_b(bh_, bl_, sKh, sKl, 8 * j, 16 * kk, g, t);
        mma3(s[j], qh[kk], ql[kk], bh_, bl_);
      }
    }
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int col = j0 + 8 * j + 2 * t + (e & 1);
        s[j][e] = col < p.nk ? s[j][e] * p.scale : -INFINITY;
      }
      mx0 = fmaxf(mx0, fmaxf(s[j][0], s[j][1]));
      mx1 = fmaxf(mx1, fmaxf(s[j][2], s[j][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float n0 = fmaxf(m0, mx0), n1 = fmaxf(m1, mx1);     // finite: key j0 < nk is in every tile
    const float c0 = expf(m0 - n0), c1 = expf(m1 - n1);
    m0 = n0;
    m1 = n1;
    float ls0 = 0.f, ls1 = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s[j][0] = expf(s[j][0] - n0);
      s[j][1] = expf(s[j][1] - n0);
      s[j][2] = expf(s[j][2] - n1);
      s[j][3] = expf(s[j][3] - n1);
      ls0 += s[j][0] + s[j][1];
      ls1 += s[j][2] + s[j][3];
      o[j][0] *= c0;
      o[j][1] *= c0;
      o[j][2] *= c1;
      o[j][3] *= c1;
    }
    l0 = l0 * c0 + ls0;
    l1 = l1 * c1 + ls1;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t ah[4], al[4];
      frag_acc(ah, al, s, kk);
#pragma unroll
      for (int jd = 0; jd < 8; ++jd) {
        uint32_t bh_[2], bl_[2];
        frag_b(bh_, bl_, sVh, sVl, 8 * jd, 16 * kk, g, t);
        mma3(o[jd], ah, al, bh_, bl_);
      }
    }
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.f / l0, i1 = 1.f / l1;
  const int row0 = q0 + r0 + g, row1 = row0 + 8;
  const long long ld = (long long)p.heads * p.dh;
  float* ob = p.o_out + (long long)b * p.nq * ld + (long long)h * p.dh;
#pragma unroll
  for (int jd = 0; jd < 8; ++jd) {
    const int col = 8 * jd + 2 * t;
    if (col < p.dh) {
      if (row0 < p.nq) *reinterpret_cast<float2*>(ob + row0 * ld + col) = make_float2(o[jd][0] * i0, o[jd][1] * i0);
      if (row1 < p.nq) *reinterpret_cast<float2*>(ob + row1 * ld + col) = make_float2(o[jd][2] * i1, o[jd][3] * i1);
    }
  }
  if (t == 0) {
    if (row0 < p.nq) p.lse[(long long)bh * p.nq + row0] = m0 + logf(l0);
    if (row1 < p.nq) p.lse[(long long)bh * p.nq + row1] = m1 + logf(l1);
  }
}

// D[bh, i] = sum_d dO[b, i, h dh + d] O[b, i, h dh + d]: one warp per row, lanes d and d + 32, butterfly sum
__global__ void __launch_bounds__(256) attn_train_rowdot_kernel(const Params p) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= p.rows) return;
  const long long bh = row / p.nq, i = row % p.nq;
  const long long b = bh / p.heads, h = bh % p.heads;
  const long long off = b * p.o.sb + i * p.o.sn + h * p.o.sh;
  float acc = 0.f;
  if (lane < p.dh) acc = p.dout.p[off + lane] * p.o.p[off + lane];
  if (lane + 32 < p.dh) acc += p.dout.p[off + lane + 32] * p.o.p[off + lane + 32];
#pragma unroll
  for (int w = 16; w >= 1; w >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, w);
  if (lane == 0) p.dvec[row] = acc;
}

__global__ void __launch_bounds__(kThreads) attn_train_dkdv_kernel(const Params p) {
  extern __shared__ __align__(16) __nv_bfloat16 dsm[];
  __nv_bfloat16 *sKh = dsm, *sKl = dsm + kTile, *sVh = dsm + 2 * kTile, *sVl = dsm + 3 * kTile;
  __nv_bfloat16 *sQh = dsm + 4 * kTile, *sQl = dsm + 5 * kTile, *sQth = dsm + 6 * kTile, *sQtl = dsm + 7 * kTile;
  __nv_bfloat16 *sGh = dsm + 8 * kTile, *sGl = dsm + 9 * kTile, *sGth = dsm + 10 * kTile, *sGtl = dsm + 11 * kTile;
  float* sLse = reinterpret_cast<float*>(dsm + 12 * kTile);
  float* sD = sLse + kT;
  const int bh = blockIdx.y, b = bh / p.heads, h = bh % p.heads;
  const int k0 = blockIdx.x * kT;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int r0 = warp * 16;   // this warp's keys within the tile

  load_tile(p.k, b, h, k0, p.nk, p.dh, sKh, sKl, nullptr, nullptr);
  load_tile(p.v, b, h, k0, p.nk, p.dh, sVh, sVl, nullptr, nullptr);
  float dk[8][4], dv[8][4];
  zero(dk);
  zero(dv);
  for (int i0 = 0; i0 < p.nq; i0 += kT) {
    __syncthreads();
    load_tile(p.q, b, h, i0, p.nq, p.dh, sQh, sQl, sQth, sQtl);
    load_tile(p.dout, b, h, i0, p.nq, p.dh, sGh, sGl, sGth, sGtl);
    if (threadIdx.x < kT) {
      const int i = i0 + threadIdx.x;
      sLse[threadIdx.x] = i < p.nq ? p.lse[(long long)bh * p.nq + i] : INFINITY;   // exp(s - inf) = 0: no such query
      sD[threadIdx.x] = i < p.nq ? p.dvec[(long long)bh * p.nq + i] : 0.f;
    }
    __syncthreads();
    float st[8][4];   // S^T: this warp's 16 keys x the tile's 64 queries, then P^T, then dS^T
    zero(st);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t ah[4], al[4];
      frag_a(ah, sKh, r0, 16 * kk, g, t);
      frag_a(al, sKl, r0, 16 * kk, g, t);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        uint32_t bh_[2], bl_[2];
        frag_b(bh_, bl_, sQh, sQl, 8 * j, 16 * kk, g, t);
        mma3(st[j], ah, al, bh_, bl_);
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) st[j][e] = expf(st[j][e] * p.scale - sLse[8 * j + 2 * t + (e & 1)]);
    }
    // dV += P^T dO
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t ah[4], al[4];
      frag_acc(ah, al, st, kk);
#pragma unroll
      for (int jd = 0; jd < 8; ++jd) {
        uint32_t bh_[2], bl_[2];
        frag_b(bh_, bl_, sGth, sGtl, 8 * jd, 16 * kk, g, t);
        mma3(dv[jd], ah, al, bh_, bl_);
      }
    }
    // dP^T = V dO^T, dS^T = P^T o (dP^T - D)
    float dp[8][4];
    zero(dp);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t ah[4], al[4];
      frag_a(ah, sVh, r0, 16 * kk, g, t);
      frag_a(al, sVl, r0, 16 * kk, g, t);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        uint32_t bh_[2], bl_[2];
        frag_b(bh_, bl_, sGh, sGl, 8 * j, 16 * kk, g, t);
        mma3(dp[j], ah, al, bh_, bl_);
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) st[j][e] *= dp[j][e] - sD[8 * j + 2 * t + (e & 1)];
    }
    // dK += dS^T Q (scaled at the end)
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t ah[4], al[4];
      frag_acc(ah, al, st, kk);
#pragma unroll
      for (int jd = 0; jd < 8; ++jd) {
        uint32_t bh_[2], bl_[2];
        frag_b(bh_, bl_, sQth, sQtl, 8 * jd, 16 * kk, g, t);
        mma3(dk[jd], ah, al, bh_, bl_);
      }
    }
  }
  const int row0 = k0 + r0 + g, row1 = row0 + 8;
  const long long base = (long long)bh * p.nk * p.dh;
#pragma unroll
  for (int jd = 0; jd < 8; ++jd) {
    const int col = 8 * jd + 2 * t;
    if (col < p.dh) {
      if (row0 < p.nk) {
        *reinterpret_cast<float2*>(p.dk + base + (long long)row0 * p.dh + col) = make_float2(dk[jd][0] * p.scale, dk[jd][1] * p.scale);
        *reinterpret_cast<float2*>(p.dv + base + (long long)row0 * p.dh + col) = make_float2(dv[jd][0], dv[jd][1]);
      }
      if (row1 < p.nk) {
        *reinterpret_cast<float2*>(p.dk + base + (long long)row1 * p.dh + col) = make_float2(dk[jd][2] * p.scale, dk[jd][3] * p.scale);
        *reinterpret_cast<float2*>(p.dv + base + (long long)row1 * p.dh + col) = make_float2(dv[jd][2], dv[jd][3]);
      }
    }
  }
}

__global__ void __launch_bounds__(kThreads) attn_train_dq_kernel(const Params p) {
  extern __shared__ __align__(16) __nv_bfloat16 dsm[];
  __nv_bfloat16 *sQh = dsm, *sQl = dsm + kTile, *sGh = dsm + 2 * kTile, *sGl = dsm + 3 * kTile;
  __nv_bfloat16 *sKh = dsm + 4 * kTile, *sKl = dsm + 5 * kTile, *sKth = dsm + 6 * kTile, *sKtl = dsm + 7 * kTile;
  __nv_bfloat16 *sVh = dsm + 8 * kTile, *sVl = dsm + 9 * kTile;
  const int bh = blockIdx.y, b = bh / p.heads, h = bh % p.heads;
  const int q0 = blockIdx.x * kT;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int r0 = warp * 16;
  const int row0 = q0 + r0 + g, row1 = row0 + 8;
  const float lse0 = row0 < p.nq ? p.lse[(long long)bh * p.nq + row0] : 0.f;
  const float lse1 = row1 < p.nq ? p.lse[(long long)bh * p.nq + row1] : 0.f;
  const float d0 = row0 < p.nq ? p.dvec[(long long)bh * p.nq + row0] : 0.f;
  const float d1 = row1 < p.nq ? p.dvec[(long long)bh * p.nq + row1] : 0.f;

  load_tile(p.q, b, h, q0, p.nq, p.dh, sQh, sQl, nullptr, nullptr);
  load_tile(p.dout, b, h, q0, p.nq, p.dh, sGh, sGl, nullptr, nullptr);
  float dq[8][4];
  zero(dq);
  for (int j0 = 0; j0 < p.nk; j0 += kT) {
    __syncthreads();
    load_tile(p.k, b, h, j0, p.nk, p.dh, sKh, sKl, sKth, sKtl);
    load_tile(p.v, b, h, j0, p.nk, p.dh, sVh, sVl, nullptr, nullptr);
    __syncthreads();
    float s[8][4], dp[8][4];   // S, then P, then dS
    zero(s);
    zero(dp);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t ah[4], al[4], gh[4], gl[4];
      frag_a(ah, sQh, r0, 16 * kk, g, t);
      frag_a(al, sQl, r0, 16 * kk, g, t);
      frag_a(gh, sGh, r0, 16 * kk, g, t);
      frag_a(gl, sGl, r0, 16 * kk, g, t);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        uint32_t bh_[2], bl_[2];
        frag_b(bh_, bl_, sKh, sKl, 8 * j, 16 * kk, g, t);
        mma3(s[j], ah, al, bh_, bl_);
        frag_b(bh_, bl_, sVh, sVl, 8 * j, 16 * kk, g, t);
        mma3(dp[j], gh, gl, bh_, bl_);
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int col = j0 + 8 * j + 2 * t + (e & 1);
        const float pr = col < p.nk ? expf(s[j][e] * p.scale - (e < 2 ? lse0 : lse1)) : 0.f;
        s[j][e] = pr * (dp[j][e] - (e < 2 ? d0 : d1));
      }
    }
    // dQ += dS K (scaled at the end)
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t ah[4], al[4];
      frag_acc(ah, al, s, kk);
#pragma unroll
      for (int jd = 0; jd < 8; ++jd) {
        uint32_t bh_[2], bl_[2];
        frag_b(bh_, bl_, sKth, sKtl, 8 * jd, 16 * kk, g, t);
        mma3(dq[jd], ah, al, bh_, bl_);
      }
    }
  }
  const long long base = (long long)bh * p.nq * p.dh;
#pragma unroll
  for (int jd = 0; jd < 8; ++jd) {
    const int col = 8 * jd + 2 * t;
    if (col < p.dh) {
      if (row0 < p.nq)
        *reinterpret_cast<float2*>(p.dq + base + (long long)row0 * p.dh + col) = make_float2(dq[jd][0] * p.scale, dq[jd][1] * p.scale);
      if (row1 < p.nq)
        *reinterpret_cast<float2*>(p.dq + base + (long long)row1 * p.dh + col) = make_float2(dq[jd][2] * p.scale, dq[jd][3] * p.scale);
    }
  }
}

bool misaligned(const void* p) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) & 15) != 0; }

bool bad_strides(const int64_t (&s)[3]) {
  for (int i = 0; i < 3; ++i)
    if (s[i] < 0 || s[i] % 4 != 0) return true;
  return false;
}

int check_desc(const s3r_attn_train_desc* d, const char* who) {
  if (!d) {
    set_error("%s: null descriptor", who);
    return -1;
  }
  if (d->batch < 1 || d->heads < 1 || d->nq < 1 || d->nk < 1) {
    set_error("%s: sizes must be >= 1 (batch=%d heads=%d nq=%d nk=%d)", who, d->batch, d->heads, d->nq, d->nk);
    return -1;
  }
  if (d->dh != 48 && d->dh != 64) {
    set_error("%s: dh=%d, must be 48 or 64", who, d->dh);
    return -1;
  }
  if ((long long)d->batch * d->heads > 65535) {
    set_error("%s: batch*heads=%lld, at most 65535", who, (long long)d->batch * d->heads);
    return -1;
  }
  if (!(d->scale > 0.f) || !std::isfinite(d->scale)) {
    set_error("%s: scale must be positive and finite", who);
    return -1;
  }
  if (misaligned(d->q) || misaligned(d->k) || misaligned(d->v)) {
    set_error("%s: null or not 16-byte aligned pointer (q, k, v)", who);
    return -1;
  }
  if (bad_strides(d->q_stride) || bad_strides(d->k_stride) || bad_strides(d->v_stride)) {
    set_error("%s: q / k / v strides must be non-negative multiples of 4 elements", who);
    return -1;
  }
  return 0;
}

Params make_params(const s3r_attn_train_desc* d) {
  Params p;
  memset(&p, 0, sizeof(p));
  p.q = {d->q, d->q_stride[0], d->q_stride[1], d->q_stride[2]};
  p.k = {d->k, d->k_stride[0], d->k_stride[1], d->k_stride[2]};
  p.v = {d->v, d->v_stride[0], d->v_stride[1], d->v_stride[2]};
  p.heads = d->heads;
  p.nq = d->nq;
  p.nk = d->nk;
  p.dh = d->dh;
  p.rows = (long long)d->batch * d->heads * d->nq;
  p.scale = d->scale;
  return p;
}

// [batch, nq, heads * dh] as a Src
Src token_major(const float* x, const s3r_attn_train_desc* d) {
  const long long ld = (long long)d->heads * d->dh;
  return {x, (long long)d->nq * ld, d->dh, ld};
}

}  // namespace

}  // namespace s3r

using namespace s3r;

extern "C" {

size_t s3r_attn_train_workspace_bytes(const s3r_attn_train_desc* d) {
  if (check_desc(d, "s3r_attn_train_workspace_bytes")) return 0;
  const size_t rows = (size_t)d->batch * d->heads * d->nq;
  return (rows * sizeof(float) + 255) / 256 * 256;
}

int s3r_attn_train_forward(const s3r_attn_train_desc* d, float* o, float* lse, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int r = check_desc(d, "s3r_attn_train_forward")) return r;
  if (misaligned(o) || misaligned(lse)) {
    set_error("s3r_attn_train_forward: null or not 16-byte aligned pointer (o, lse)");
    return -1;
  }
  Params p = make_params(d);
  p.o_out = o;
  p.lse = lse;
  const dim3 grid((unsigned)((d->nq + kT - 1) / kT), (unsigned)(d->batch * d->heads));
  attn_train_fwd_kernel<<<grid, kThreads, 0, st>>>(p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("s3r_attn_train_forward: launch failed: %s", cudaGetErrorString(e));
    return -6;
  }
  return 0;
}

int s3r_attn_train_backward(const s3r_attn_train_desc* d, const float* o, const float* lse, const float* d_o,
                            void* workspace, size_t workspace_bytes, float* dq, float* dk, float* dv, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int r = check_desc(d, "s3r_attn_train_backward")) return r;
  if (misaligned(o) || misaligned(lse) || misaligned(d_o) || misaligned(dq) || misaligned(dk) || misaligned(dv) ||
      misaligned(workspace)) {
    set_error("s3r_attn_train_backward: null or not 16-byte aligned pointer (o, lse, d_o, workspace, dq, dk, dv)");
    return -1;
  }
  const size_t need = s3r_attn_train_workspace_bytes(d);
  if (workspace_bytes < need) {
    set_error("s3r_attn_train_backward: workspace of %zu bytes, %zu needed (s3r_attn_train_workspace_bytes)",
              workspace_bytes, need);
    return -1;
  }
  Params p = make_params(d);
  p.o = token_major(o, d);
  p.dout = token_major(d_o, d);
  p.lse = const_cast<float*>(lse);
  p.dvec = reinterpret_cast<float*>(workspace);
  p.dq = dq;
  p.dk = dk;
  p.dv = dv;

  static PerDeviceOnce once;
  bool& attr_set = once.cur();
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(attn_train_dkdv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kDkdvSmem);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(attn_train_dq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kDqSmem);
    if (e != cudaSuccess) {
      set_error("s3r_attn_train_backward: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      return -5;
    }
    attr_set = true;
  }
  const unsigned bh = (unsigned)(d->batch * d->heads);
  attn_train_rowdot_kernel<<<(unsigned)((p.rows + 7) / 8), 256, 0, st>>>(p);
  attn_train_dkdv_kernel<<<dim3((unsigned)((d->nk + kT - 1) / kT), bh), kThreads, kDkdvSmem, st>>>(p);
  attn_train_dq_kernel<<<dim3((unsigned)((d->nq + kT - 1) / kT), bh), kThreads, kDqSmem, st>>>(p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("s3r_attn_train_backward: launch failed: %s", cudaGetErrorString(e));
    return -6;
  }
  return 0;
}

}  // extern "C"
