// Spatial-memory kernels (spann3r/model.py:97-118,145-183): the softmax / threshold / renormalise
// stage between the two tensor-core GEMMs of the bank read, the attention column sums, the transposed
// split-bf16 write of bank values, and the working-memory similarity gate.
//
// Bank layout in HBM (DESIGN.md §2): keys and values are stored PRE-NORMALISED (LN_k / LN_v applied once at
// write time; LayerNorm is per token, so this equals normalising the whole bank on every read as the
// reference does) as split-bf16 planes: K_n [B, Mcap, 1024] (GEMM B operand of S = Q K^T) and V_n^T
// [B, 1024, Mcap] (K-major B operand of O = P V).  Both are streamed by TMA in 128-byte rows.
#include "../../include/spann3r_b200.h"
#include "common.cuh"
#include "kernels.cuh"

namespace s3r {

// ------------------------------------------------------------------------------------------------
// One CTA per query row.  S row (raw dot products) -> softmax(S*scale) -> zero entries < thresh ->
// renormalise (spann3r/model.py:157-172) -> split-bf16 planes P[row, 0:Mpad] (zero padded).
// A row whose every weight is below the threshold divides 0/0 exactly like the reference (NaN).
// ------------------------------------------------------------------------------------------------
// Training mode (spann3r/model.py:167-168, nn.Dropout(p) on the softmax output): element (r, i) is kept with probability
// 1 - p and scaled by 1 / (1 - p).  The keep decision is a pure function of (seed, r * M + i) -- Philox4x32-10, four
// consecutive elements per counter -- so the backward pass and the tests can regenerate the exact mask
// (`dropout_mask_kernel`, s3r_dropout_mask).
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, ctr.x), lo0 = 0xD2511F53u * ctr.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, ctr.z), lo1 = 0xCD9E8D57u * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += 0x9E3779B9u;
    key.y += 0xBB67AE85u;
  }
  return ctr;
}
// keep-scale of element `idx` (0 or 1 / (1 - p)): u = 24 random bits / 2^24 in [0, 1), kept when u >= p
__device__ __forceinline__ float dropout_scale(unsigned long long seed, unsigned long long idx, float p, float keep_scale) {
  const unsigned long long c = idx >> 2;
  const uint4 r = philox4x32_10(make_uint4((uint32_t)c, (uint32_t)(c >> 32), 0u, 0u),
                                make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  const uint32_t w = (idx & 3) == 0 ? r.x : (idx & 3) == 1 ? r.y : (idx & 3) == 2 ? r.z : r.w;
  const float u = (float)(w >> 8) * (1.0f / 16777216.0f);
  return u >= p ? keep_scale : 0.f;
}

// keep-scale 1 / (1 - p) is evaluated on the host in double and rounded once, as torch.nn.functional.dropout does
__global__ void dropout_mask_kernel(float* __restrict__ out, long long n, unsigned long long seed, float p, float ks) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = dropout_scale(seed, (unsigned long long)i, p, ks);
}

// Row r belongs to slot r / nq and reads that slot's length M = lens[r / nq] (its bank); a slot of length 0 gets an
// all-zero row, so that P V adds nothing to its queries.
__global__ void __launch_bounds__(256) mem_softmax_kernel(const float* __restrict__ S, long long ldS, int nq,
                                                          const SlotInts lens, int Mpad, float scale, float thresh,
                                                          __nv_bfloat16* __restrict__ phi, __nv_bfloat16* __restrict__ plo,
                                                          long long ldP, float drop_p, float keep_scale,
                                                          unsigned long long seed) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float row[];
  __shared__ float red[8];
  const long long r = blockIdx.x;
  const int M = lens[(int)(r / nq)];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (M == 0) {
    for (int i = tid; i < (Mpad >> 2); i += 256) {
      *reinterpret_cast<uint2*>(phi + r * ldP + 4 * i) = make_uint2(0u, 0u);
      *reinterpret_cast<uint2*>(plo + r * ldP + 4 * i) = make_uint2(0u, 0u);
    }
    return;
  }
  const float* s = S + r * ldS;
  auto block_reduce = [&](float v, bool is_max) -> float {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float t = __shfl_xor_sync(0xffffffffu, v, o);
      v = is_max ? fmaxf(v, t) : v + t;
    }
    __syncthreads();
    if (lane == 0) red[wid] = v;
    __syncthreads();
    float x = red[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) x = is_max ? fmaxf(x, red[i]) : x + red[i];
    return x;
  };
  // Three passes over the row held in shared memory, 128-bit everywhere (the S row and both plane rows are 16-byte aligned:
  // ldS / ldP are multiples of 32); the M % 4 tail, if any, is scalar.
  const int M4 = M >> 2;
  float4* row4 = reinterpret_cast<float4*>(row);
  const float4* s4 = reinterpret_cast<const float4*>(s);
  float mx = -INFINITY;
  for (int i = tid; i < M4; i += 256) {
    float4 v = s4[i];
    v.x *= scale; v.y *= scale; v.z *= scale; v.w *= scale;
    row4[i] = v;
    mx = fmaxf(fmaxf(mx, fmaxf(v.x, v.y)), fmaxf(v.z, v.w));
  }
  for (int i = 4 * M4 + tid; i < M; i += 256) {
    const float v = s[i] * scale;
    row[i] = v;
    mx = fmaxf(mx, v);
  }
  mx = block_reduce(mx, true);
  float sum = 0.f;
  for (int i = tid; i < M4; i += 256) {
    float4 v = row4[i];
    v.x = expf(v.x - mx); v.y = expf(v.y - mx); v.z = expf(v.z - mx); v.w = expf(v.w - mx);
    row4[i] = v;
    sum += (v.x + v.y) + (v.z + v.w);
  }
  for (int i = 4 * M4 + tid; i < M; i += 256) {
    const float e = expf(row[i] - mx);
    row[i] = e;
    sum += e;
  }
  sum = block_reduce(sum, false);
  const float inv = 1.0f / sum;
  const unsigned long long row_base = (unsigned long long)r * (unsigned long long)M;
  auto weight = [&](float e, int i) -> float {
    float a = e * inv;
    // dropout BEFORE the threshold, as in the reference (training runs with attn_thresh = 0)
    if (drop_p > 0.f) a *= dropout_scale(seed, row_base + i, drop_p, keep_scale);
    if (thresh > 0.f && a < thresh) a = 0.f;
    return a;
  };
  float sum2 = 0.f;
  for (int i = tid; i < M4; i += 256) {
    float4 v = row4[i];
    v.x = weight(v.x, 4 * i); v.y = weight(v.y, 4 * i + 1); v.z = weight(v.z, 4 * i + 2); v.w = weight(v.w, 4 * i + 3);
    row4[i] = v;
    sum2 += (v.x + v.y) + (v.z + v.w);
  }
  for (int i = 4 * M4 + tid; i < M; i += 256) {
    const float a = weight(row[i], i);
    row[i] = a;
    sum2 += a;
  }
  float inv2 = 1.0f;
  if (thresh > 0.f) {
    sum2 = block_reduce(sum2, false);
    inv2 = 1.0f / sum2;  // 0/0 -> NaN when the whole row was cut, as in the reference
  } else {
    __syncthreads();     // the plane pass below reads other threads' entries
  }
  __nv_bfloat16* ph = phi + r * ldP;
  __nv_bfloat16* pl = plo + r * ldP;
  const int P4 = Mpad >> 2;   // Mpad is a multiple of 8
  for (int i = tid; i < P4; i += 256) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (i < M4) {
      v = row4[i];
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (4 * i + j < M) (&v.x)[j] = row[4 * i + j];
    }
    if (thresh > 0.f) { v.x *= inv2; v.y *= inv2; v.z *= inv2; v.w *= inv2; }
    uint32_t h01, l01, h23, l23;
    split2_bf16(v.x, v.y, h01, l01);
    split2_bf16(v.z, v.w, h23, l23);
    *reinterpret_cast<uint2*>(ph + 4 * i) = make_uint2(h01, h23);
    *reinterpret_cast<uint2*>(pl + 4 * i) = make_uint2(l01, l23);
  }
}

int launch_mem_softmax(const float* S, long long ldS, long long rows, int nq, const SlotInts& lens, int Mmax, int Mpad,
                       float scale, float thresh, __nv_bfloat16* phi, __nv_bfloat16* plo, long long ldP, cudaStream_t st,
                       float drop_p, unsigned long long seed) {
  if (rows == 0 || Mmax == 0) return 0;
  const size_t smem = (size_t)Mmax * sizeof(float);
  if (Mmax > MEM_SOFTMAX_MAX_LEN) {
    set_error("mem_softmax: bank of %d tokens exceeds the %d-token row buffer", Mmax, MEM_SOFTMAX_MAX_LEN);
    return -1;
  }
  // Opt in to the large row buffer on first use, whatever this call's size: the kernel's static shared memory counts
  // against the same 48 KB default, so a row of exactly 48 KB (12288 tokens) already needs it.
  static PerDeviceOnce once;
  if (!once.cur()) {
    cudaFuncSetAttribute(mem_softmax_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MEM_SOFTMAX_MAX_LEN * 4);
    once.cur() = true;
  }
  launch_pdl(mem_softmax_kernel, dim3((unsigned)rows), dim3(256), smem, st, S, ldS, nq, lens, Mpad, scale, thresh, phi, plo,
             ldP, drop_p, (float)(1.0 / (1.0 - (double)drop_p)), seed);
  const cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) {
    set_error("mem_softmax: launch of %d rows x %d tokens failed: %s", (int)rows, Mmax, cudaGetErrorString(err));
    return -6;
  }
  return 0;
}

// ------------------------------------------------------------------------------------------------
// mem_attn[b, m] += sum over the N query rows of attn[b, :, m]   (spann3r/model.py:180-181).
// Two fixed-shape passes, fixed summation order (deterministic: the prune ranking depends on it).
//   pass 1: block = 32 column-octets (256 columns, 16-byte loads of both planes) x 8 row lanes over a chunk of
//           CS_ROWS rows -> partial[b, chunk, m]     (grid = columns/256 x chunks x B: hundreds of CTAs in flight)
//   pass 2: mem_attn[b, m] += partial[b, 0, m] + partial[b, 1, m] + ...   in chunk order
// ------------------------------------------------------------------------------------------------
constexpr int CS_ROWS = 32;
__global__ void __launch_bounds__(256) mem_colsum_partial_kernel(const __nv_bfloat16* __restrict__ phi,
                                                                 const __nv_bfloat16* __restrict__ plo, long long ldP,
                                                                 int nq, int Mpad, float* __restrict__ part,
                                                                 long long ld_part) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[8][256];
  const int oct = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int m0 = blockIdx.x * 256 + oct * 8;
  const int chunk = blockIdx.y, b = blockIdx.z;
  const int r0 = chunk * CS_ROWS, r1 = min(nq, r0 + CS_ROWS);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (m0 < Mpad) {
    for (int r = r0 + rl; r < r1; r += 8) {
      const long long o = ((long long)b * nq + r) * ldP + m0;
      const uint4 h = *reinterpret_cast<const uint4*>(phi + o);
      const uint4 l = *reinterpret_cast<const uint4*>(plo + o);
      const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        acc[2 * j] += __uint_as_float(hw[j] << 16) + __uint_as_float(lw[j] << 16);
        acc[2 * j + 1] += __uint_as_float(hw[j] & 0xffff0000u) + __uint_as_float(lw[j] & 0xffff0000u);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[rl][oct * 8 + j] = acc[j];
  __syncthreads();
  const int m = blockIdx.x * 256 + threadIdx.x;
  if (m < Mpad) {
    float s = red[0][threadIdx.x];
#pragma unroll
    for (int i = 1; i < 8; ++i) s += red[i][threadIdx.x];
    part[((long long)b * gridDim.y + chunk) * ld_part + m] = s;
  }
}
__global__ void __launch_bounds__(256) mem_colsum_final_kernel(const float* __restrict__ part, long long ld_part,
                                                               int chunks, const SlotInts lens, float* __restrict__ mem_attn,
                                                               long long ld_attn) {
  pdl_launch_dependents();
  pdl_wait();
  const int m = blockIdx.x * 256 + threadIdx.x, b = blockIdx.y;
  if (m >= lens[b]) return;
  const float* p = part + (long long)b * chunks * ld_part + m;
  float s = 0.f;
  for (int c = 0; c < chunks; ++c) s += p[c * ld_part];
  mem_attn[b * ld_attn + m] += s;
}

// P planes are zero beyond each slot's length up to Mpad (mem_softmax_kernel) and ldP, Mpad are multiples of 8 (16-byte
// loads).
int launch_mem_colsum(const __nv_bfloat16* phi, const __nv_bfloat16* plo, long long ldP, int B, int nq, const SlotInts& lens,
                      int Mmax, float* mem_attn, long long ld_attn, float* part, long long ld_part, cudaStream_t st) {
  if (Mmax == 0) return 0;
  const int Mpad = (Mmax + 7) / 8 * 8;
  const int chunks = (nq + CS_ROWS - 1) / CS_ROWS;
  if (ldP % 8 != 0 || ld_part < Mpad) {
    set_error("mem_colsum: ldP=%lld must be a multiple of 8 and ld_part=%lld >= %d", ldP, ld_part, Mpad);
    return -1;
  }
  launch_pdl(mem_colsum_partial_kernel, dim3((Mpad + 255) / 256, chunks, B), dim3(256), 0, st, phi, plo, ldP, nq, Mpad,
             part, ld_part);
  launch_pdl(mem_colsum_final_kernel, dim3((Mmax + 255) / 256, B), dim3(256), 0, st, (const float*)part, ld_part, chunks, lens,
             mem_attn, ld_attn);
  return cudaGetLastError() == cudaSuccess ? 0 : -6;
}
int mem_colsum_chunks(int nq) { return (nq + CS_ROWS - 1) / CS_ROWS; }

// ------------------------------------------------------------------------------------------------
// fp32 x[b, t, c] (t < T, c < C)  ->  split-bf16 planes out[b, c, col0[b] + t] (row stride ldo) for the slots b with
// on[b] != 0: the transposed write that appends normalised values to the V_n^T bank.  32x32 smem tile transpose.
// ------------------------------------------------------------------------------------------------
__global__ void split_transpose_kernel(const float* __restrict__ x, int T, int C, __nv_bfloat16* __restrict__ ohi,
                                       __nv_bfloat16* __restrict__ olo, long long ldo, long long out_batch_stride,
                                       const SlotInts col0s, const SlotInts on) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  if (!on[b]) return;
  const int col0 = col0s[b];
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const float* xb = x + (long long)b * T * C;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int t = t0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (t < T && c < C) ? xb[(long long)t * C + c] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, t = t0 + threadIdx.x;
    if (c < C && t < T) {
      __nv_bfloat16 h, l;
      split_bf16(tile[threadIdx.x][i], h, l);
      const long long o = (long long)b * out_batch_stride + (long long)c * ldo + col0 + t;
      ohi[o] = h;
      olo[o] = l;
    }
  }
}

int launch_split_transpose(const float* x, int B, int T, int C, __nv_bfloat16* ohi, __nv_bfloat16* olo, long long ldo,
                           long long out_batch_stride, const SlotInts& col0, const SlotInts& on, cudaStream_t st) {
  if (B * T * C == 0) return 0;
  dim3 grid((T + 31) / 32, (C + 31) / 32, B), block(32, 8);
  launch_pdl(split_transpose_kernel, dim3(grid), dim3(block), 0, st, x, T, C, ohi, olo, ldo, out_batch_stride, col0, on);
  return cudaGetLastError() == cudaSuccess ? 0 : -6;
}

// ------------------------------------------------------------------------------------------------
// Similarity gate (spann3r/model.py:97-118): out[b, t] = mean_p cos(feat_k[b,p,:], wm[b,t,p,:]) for the
// last `wm` frames of the raw key bank.  One warp per (b, t, p); per-(b,t) sums are reduced in a fixed
// order by a second tiny kernel so the > 0.95 decision is reproducible.  Each slot b has its own window: wm[b] frames
// from token start[b] of its rows; T = max wm[b], and warps / outputs past a slot's wm[b] are idle / -inf.
// ------------------------------------------------------------------------------------------------
__global__ void cos_rows_kernel(const float* __restrict__ feat, const float* __restrict__ kraw, long long k_batch_stride,
                                int B, int T, const SlotInts start, const SlotInts wm, int P, int C,
                                float* __restrict__ cosv) {
  pdl_launch_dependents();
  pdl_wait();
  const long long w = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long total = (long long)B * T * P;
  if (w >= total) return;
  const int lane = threadIdx.x & 31;
  const int p = (int)(w % P);
  const int t = (int)((w / P) % T);
  const int b = (int)(w / ((long long)P * T));
  if (t >= wm[b]) return;
  const float4* a = reinterpret_cast<const float4*>(feat + ((long long)b * P + p) * C);
  const float4* k = reinterpret_cast<const float4*>(kraw + (long long)b * k_batch_stride +
                                                    ((long long)start[b] + (long long)t * P + p) * C);
  float dot = 0.f, na = 0.f, nk = 0.f;
  for (int i = lane; i < C / 4; i += 32) {
    const float4 x = a[i], y = k[i];
    dot += x.x * y.x + x.y * y.y + x.z * y.z + x.w * y.w;
    na += x.x * x.x + x.y * x.y + x.z * x.z + x.w * x.w;
    nk += y.x * y.x + y.y * y.y + y.z * y.z + y.w * y.w;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    dot += __shfl_xor_sync(0xffffffffu, dot, o);
    na += __shfl_xor_sync(0xffffffffu, na, o);
    nk += __shfl_xor_sync(0xffffffffu, nk, o);
  }
  if (lane == 0) cosv[w] = dot / (fmaxf(sqrtf(na), 1e-12f) * fmaxf(sqrtf(nk), 1e-12f));  // F.normalize eps
}

// one block per output (b, t < ldo); cosv holds T frames per slot
__global__ void mean_rows_kernel(const float* __restrict__ cosv, int T, const SlotInts wm, int P, float* __restrict__ out,
                                 int ldo) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[256];
  const int b = blockIdx.x / ldo, t = blockIdx.x % ldo;
  if (t >= wm[b]) {
    if (threadIdx.x == 0) out[blockIdx.x] = -INFINITY;
    return;
  }
  const float* c = cosv + ((long long)b * T + t) * P;
  float s = 0.f;
  for (int i = threadIdx.x; i < P; i += 256) s += c[i];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[blockIdx.x] = red[0] / (float)P;
}

int launch_check_sim(const float* feat, const float* k, long long k_batch_stride, int B, const SlotInts& start,
                     const SlotInts& wm, int P, int C, float* scratch, float* out, int ldo, cudaStream_t st) {
  if (B * ldo * P == 0) return 0;
  if (C % 4) { set_error("check_sim: C %% 4 != 0"); return -1; }
  int T = 0;
  for (int b = 0; b < (wm.n == 1 ? 1 : B); ++b) T = wm[b] > T ? wm[b] : T;
  const long long total = (long long)B * T * P;
  if (total > 0)
    launch_pdl(cos_rows_kernel, dim3((unsigned)((total + 7) / 8)), dim3(256), 0, st, feat, k, k_batch_stride, B, T, start,
               wm, P, C, scratch);
  launch_pdl(mean_rows_kernel, dim3(B * ldo), dim3(256), 0, st, (const float*)scratch, T, wm, P, out, ldo);
  return cudaGetLastError() == cudaSuccess ? 0 : -6;
}

// ------------------------------------------------------------------------------------------------
// Confidence score of the offline mode (spann3r/model.py:346-352, 372-381): mean over all pixels of
// (conf - 1) / conf.  Two fixed-shape passes (256 partial sums, then one block): deterministic.
// The batched score runs the same two kernels with one grid row (partials) / one block (final) per image: image y
// reads conf + y * n and owns part[y * 256 .. + 256), so each image's value is bitwise the single-image one.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) conf_partial_kernel(const float* __restrict__ conf, long long n, float* __restrict__ part) {
  pdl_launch_dependents();
  pdl_wait();
  conf += blockIdx.y * n;
  part += blockIdx.y * 256LL;
  __shared__ float red[256];
  float s = 0.f;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += 256LL * gridDim.x) {
    const float c = conf[i];
    s += (c - 1.0f) / c;
  }
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[blockIdx.x] = red[0];
}
__global__ void __launch_bounds__(256) conf_final_kernel(const float* __restrict__ part, int nparts, long long n, float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  part += blockIdx.x * 256LL;
  __shared__ float red[256];
  red[threadIdx.x] = threadIdx.x < nparts ? part[threadIdx.x] : 0.f;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[blockIdx.x] = red[0] / (float)n;
}

}  // namespace s3r

using namespace s3r;

extern "C" {

int s3r_dropout_mask(float* out, int64_t n, uint64_t seed, float p, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!out && n > 0) {
    set_error("s3r_dropout_mask: null output");
    return -1;
  }
  if (n <= 0) return 0;
  if (!(p >= 0.f && p < 1.f)) {
    set_error("dropout_mask: p=%g outside [0, 1)", (double)p);
    return -1;
  }
  const long long blocks = (n + 255) / 256;
  dropout_mask_kernel<<<(unsigned)(blocks < 2048 ? blocks : 2048), 256, 0, st>>>(out, n, seed, p,
                                                                                  (float)(1.0 / (1.0 - (double)p)));
  return cudaGetLastError() == cudaSuccess ? 0 : -6;
}

int s3r_conf_score(const float* conf, int64_t n, float* scratch256, float* out, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (n <= 0) { set_error("conf_score: empty input"); return -1; }
  launch_pdl(conf_partial_kernel, dim3(256), dim3(256), 0, st, conf, n, scratch256);
  launch_pdl(conf_final_kernel, dim3(1), dim3(256), 0, st, (const float*)scratch256, 256, n, out);
  return cudaGetLastError() == cudaSuccess ? 0 : -6;
}

int s3r_conf_score_batched(const float* conf, int batch, int64_t hw, float* scratch, float* out, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (batch < 1 || batch > 32767) { set_error("conf_score_batched: batch %d outside [1, 32767]", batch); return -1; }
  if (hw < 1) { set_error("conf_score_batched: H*W = %lld must be >= 1", hw); return -1; }
  if (!conf || !scratch || !out) { set_error("conf_score_batched: null pointer"); return -1; }
  const unsigned images = 2u * (unsigned)batch;
  launch_pdl(conf_partial_kernel, dim3(256, images), dim3(256), 0, st, conf, hw, scratch);
  launch_pdl(conf_final_kernel, dim3(images), dim3(256), 0, st, (const float*)scratch, 256, hw, out);
  return cudaGetLastError() == cudaSuccess ? 0 : -6;
}

}  // extern "C"
