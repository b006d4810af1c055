// Fused epilogue of the split-bf16 GEMM engine (gemm.cu).
//
// Two domains.  Every thread holds one accumulator ROW (32 consecutive columns per chunk): everything that
// is per column or per row -- folded LayerNorm, bias, activation, RoPE -- is done there.  Global memory is then touched
// in a TRANSPOSED domain: the warp stages its 32 x 32 chunk in shared memory and re-reads it so that 8 consecutive
// lanes cover one row's 128 bytes; residual loads, fp32 / split-bf16 stores, LayerNorm statistics and the q / k
// head-split stores are issued from there.  With thread = row every 16-byte access of a warp hits 32 different cache
// lines (32 L1 wavefronts per instruction); transposed, an instruction covers 4 whole rows (4 wavefronts).
#pragma once
#include "common.cuh"
#include "gemm.cuh"

namespace s3r {

// Staging tile of one warp: 32 rows x SW columns (SW = 32, or 16 where shared memory is short: two passes per chunk),
// row stride SW + 4 floats (16-byte aligned rows, conflict-free for the 128-bit row writes and the transposed reads).
// Transposed mapping: LPR = SW / 4 lanes per row, 32 / LPR rows per instruction, NIT = LPR instructions per pass.
template <int SW>
struct Stg {
  static constexpr int LD = SW + 4;
  static constexpr int WARP_BYTES = 32 * LD * 4;
  static constexpr int LPR = SW / 4;          // lanes per row
  static constexpr int RPI = 32 / LPR;        // rows per instruction
  static constexpr int NIT = 32 / RPI;        // instructions per pass (= LPR)
  static constexpr int NPASS = 32 / SW;       // passes per 32-column chunk
};

__device__ __forceinline__ float4 ld_f4(const float* p) { return *reinterpret_cast<const float4*>(p); }

__device__ __forceinline__ void apply_act(float (&v)[32], int act) {
  if (act == ACT_GELU) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float4 t = gelu_erf4(make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]));
      v[4 * q] = t.x;
      v[4 * q + 1] = t.y;
      v[4 * q + 2] = t.z;
      v[4 * q + 3] = t.w;
    }
  } else if (act == ACT_RELU) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.0f);
  }
}

// Per-tile column vectors staged in shared memory by the epilogue warps BEFORE they wait for the accumulator (the
// loads overlap the main loop): sb[j] = bias of tile column j (0 when there is none), scs[j] = column sum of the
// LayerNorm-folded weights (ln_cs, see GemmArgs).  Call with every epilogue thread, then barrier among them.
template <int EPI, int BN>
__device__ __forceinline__ void epi_stage_cols(const GemmArgs& args, float* sb, float* scs, int g, int nt, int tid_e,
                                               int nthr_e) {
  for (int j = tid_e; j < BN; j += nthr_e) {
    const int col = nt * BN + j;
    float b = 0.f, c = 0.f;
    if (col < args.N) {
      if (args.bias != nullptr)
        b = __ldg(args.bias + ((EPI == EPI_PIXSHUF) ? (long long)g * args.ps_cout + (col % args.ps_cout)
                                                    : (long long)g * args.N + col));
      if (args.ln_cs != nullptr) c = __ldg(args.ln_cs + (long long)g * args.N + col);
    }
    sb[j] = b;
    scs[j] = c;
  }
}

// Tile geometry: accumulator row r (0..127) of pixel tile (nb, th, tw) -> pixel (h, w); bw is a power of two.
struct TileGeom {
  int g, ga, nb, h0, w0, lbw, bwm;   // ga: group whose rows this tile reads as A (a_swap)
};
__device__ __forceinline__ TileGeom make_geom(const GemmArgs& args, int g, int nb, int th, int tw, int col_first) {
  TileGeom t;
  t.g = g; t.nb = nb; t.h0 = th * args.bh; t.w0 = tw * args.bw;
  t.ga = (args.a_swap && col_first >= args.swap_col0) ? (args.groups - 1 - g) : g;
  t.lbw = 31 - __clz(args.bw);
  t.bwm = args.bw - 1;
  return t;
}
__device__ __forceinline__ bool row_pixel(const GemmArgs& args, const TileGeom& t, int r, int& h, int& w, long long& pix) {
  h = t.h0 + (r >> t.lbw);
  w = t.w0 + (r & t.bwm);
  pix = ((long long)t.nb * args.H + h) * args.W + w;   // row inside the group
  return (h < args.H) && (w < args.W);
}

// Row-domain state of one thread for one tile.
struct EpiRow {
  float rstd = 1.f, rm = 0.f;   // folded LayerNorm: rstd, rstd * mean of the A row
  int py = 0, px = 0;           // RoPE position of the row (EPI_QKV)
  bool valid = false;
  long long pix = 0, grow = 0;  // row inside the group / global output row (EPI_PLAIN)
  int h = 0, w = 0;
};
// Transposed-domain state: lane serves rows rr = it * RPI + lane / LPR, it < NIT (NIT <= 8), four columns each.
struct EpiTRows {
  long long key[8];   // PLAIN: global output row; QKV: (gb * heads * ntok + t) * 64; PIXSHUF: global output row of the
                      // pixel's sub-pixel (0, 0); -1 = no pixel
};

// Everything that does not need the accumulator; called before the accumulator wait so that its global loads overlap
// the main loop.  LayerNorm statistics: (sum, sum of squares) per 32-column chunk of the A row, ln_np <= 32 chunks,
// read cooperatively -- 16 lanes take one row's chunk pairs as float4 (one coalesced 256-byte read per row instead
// of 16 strided 16-byte reads per thread), two rows per iteration, fixed reduction order.
template <int EPI, int SW>
__device__ __forceinline__ void epi_tile_pre(const GemmArgs& args, const TileGeom& tg, int quad, int lane, EpiRow& er,
                                             EpiTRows& tr) {
  using S = Stg<SW>;
  const int r = quad * 32 + lane;
  er.valid = row_pixel(args, tg, r, er.h, er.w, er.pix);
  er.grow = (long long)tg.g * args.out_group_rows + er.pix;
  if (args.ln_stats != nullptr) {
    const int ga = tg.ga;
    const int np2 = args.ln_np >> 1;
    const int sub = lane & 15, half = lane >> 4;
    float s1 = 0.f, s2 = 0.f;
    float4 t[16];   // all 16 loads are in flight before the first reduction (one L2 round trip, not sixteen)
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int rr = quad * 32 + 2 * i + half;
      int h2, w2;
      long long pix2;
      const bool v2 = row_pixel(args, tg, rr, h2, w2, pix2);
      t[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (v2 && sub < np2)
        t[i] = ld_f4(reinterpret_cast<const float*>(args.ln_stats + ((long long)ga * args.out_group_rows + pix2) * args.ln_np) + 4 * sub);
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      float a = t[i].x + t[i].z, b = t[i].y + t[i].w;
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
      }
      const float a0 = __shfl_sync(0xffffffffu, a, 0), a1 = __shfl_sync(0xffffffffu, a, 16);
      const float b0 = __shfl_sync(0xffffffffu, b, 0), b1 = __shfl_sync(0xffffffffu, b, 16);
      if (lane == 2 * i) { s1 = a0; s2 = b0; }
      if (lane == 2 * i + 1) { s1 = a1; s2 = b1; }
    }
    const float inv_c = 1.0f / (float)(args.ln_np * 32);
    const float mean = s1 * inv_c;
    const float var = fmaxf(s2 * inv_c - mean * mean, 0.f);
    er.rstd = rsqrtf(var + args.ln_eps);
    er.rm = er.rstd * mean;
  }
  if constexpr (EPI == EPI_QKV) {
    if (args.q_rope && er.valid) {   // positions of the token whose row is the A operand (group ga under a_swap)
      const long long prow = (long long)tg.ga * args.out_group_rows + er.pix;
      er.py = args.q_pos[prow * 2];
      er.px = args.q_pos[prow * 2 + 1];
    }
  }
  if constexpr (EPI != EPI_HEADTAIL) {
#pragma unroll
    for (int it = 0; it < S::NIT; ++it) {
      const int rr = quad * 32 + it * S::RPI + lane / S::LPR;
      int h2, w2;
      long long pix2;
      const bool v2 = row_pixel(args, tg, rr, h2, w2, pix2);
      long long key = -1;
      if (v2) {
        if constexpr (EPI == EPI_PLAIN) {
          key = (long long)tg.g * args.out_group_rows + pix2;
        } else if constexpr (EPI == EPI_QKV) {
          const int bidx = (int)(pix2 / args.q_ntok);
          const int t = (int)(pix2 - (long long)bidx * args.q_ntok);
          const long long gb = (long long)tg.g * args.q_nb + bidx;
          key = (gb * (args.q_C >> 6) * args.q_ntok + t) * 64;
        } else {   // the output row of sub-pixel (0, 0); epi_chunk adds the chunk's (i, j) offset
          const int s = args.ps_s;
          key = (long long)tg.g * args.out_group_rows + ((long long)tg.nb * (args.H * s) + h2 * s) * (args.W * s) + w2 * s;
        }
      }
      tr.key[it] = key;
    }
  }
}

// Residual values of a tile's first 32-column chunk in the transposed layout (EPI_PLAIN; epi_chunk requests each
// following chunk's values as it consumes the current ones).
template <int EPI, int SW>
__device__ __forceinline__ void epi_prefetch_res(const GemmArgs& args, const EpiTRows& tr, float4 (&rp)[8], int col0,
                                                 int lane) {
  using S = Stg<SW>;
  if constexpr (EPI == EPI_PLAIN) {
    if (args.res1 != nullptr) {
      const int cq = (lane % S::LPR) * 4;
#pragma unroll
      for (int p = 0; p < S::NPASS; ++p)
#pragma unroll
        for (int it = 0; it < S::NIT; ++it)
          if (tr.key[it] >= 0)
            rp[p * S::NIT + it] = ld_f4(args.res1 + tr.key[it] * args.ldr1 + col0 + p * SW + cq);
    }
  }
}

// One 32-column chunk.  v: this thread's accumulator row; sb / scs: the chunk's staged bias / colsum values; stg: the
// warp's staging tile; rp: prefetched residual (transposed layout), refilled slot by slot with the residual of the
// chunk at column res_next (EPI_PLAIN; -1 = none), so one buffer serves every chunk with the next one's loads in flight;
// ht_acc: running dot products of EPI_HEADTAIL.
template <int EPI, int SW>
__device__ __forceinline__ void epi_chunk(const GemmArgs& args, float (&v)[32], const float* sb, const float* scs,
                                          float* stg, const TileGeom& tg, const EpiRow& er, const EpiTRows& tr,
                                          float4 (&rp)[8], int col0, int res_next, int lane, float (&ht_acc)[4]) {
  // ---------------------------------------------------------------- row domain
  if (args.ln_stats != nullptr) {
    const float4* c4 = reinterpret_cast<const float4*>(scs);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float4 c = c4[q];
      v[4 * q + 0] = fmaf(er.rstd, v[4 * q + 0], -er.rm * c.x);
      v[4 * q + 1] = fmaf(er.rstd, v[4 * q + 1], -er.rm * c.y);
      v[4 * q + 2] = fmaf(er.rstd, v[4 * q + 2], -er.rm * c.z);
      v[4 * q + 3] = fmaf(er.rstd, v[4 * q + 3], -er.rm * c.w);
    }
  }
  {
    const float4* b4 = reinterpret_cast<const float4*>(sb);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float4 b = b4[q];
      v[4 * q + 0] += b.x;
      v[4 * q + 1] += b.y;
      v[4 * q + 2] += b.z;
      v[4 * q + 3] += b.w;
    }
  }
  if (args.act != ACT_NONE) apply_act(v, args.act);

  if constexpr (EPI == EPI_HEADTAIL) {   // dpt_block.py:318-324 (ReLU, 1x1 conv) + heads/postprocess.py:10-58
    const float* wt = args.ht_w + (long long)tg.g * 4 * 128 + col0;
#pragma unroll
    for (int o = 0; o < 4; ++o) {
      const float4* wp = reinterpret_cast<const float4*>(wt + o * 128);
      float acc = ht_acc[o];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float4 t = __ldg(wp + q);
        acc = fmaf(v[4 * q + 0], t.x, acc);
        acc = fmaf(v[4 * q + 1], t.y, acc);
        acc = fmaf(v[4 * q + 2], t.z, acc);
        acc = fmaf(v[4 * q + 3], t.w, acc);
      }
      ht_acc[o] = acc;
    }
    return;
  }

  int role = 0, head = 0, d0 = 0;
  if constexpr (EPI == EPI_QKV) {
    // croco/models/blocks.py:97-104 (self) / :154-160 (cross) + RoPE2D (pos_embed.py:112-159,
    // curope/kernels.cu:18-81): head dim 64 = [y half | x half], each half = 16 (u, v) pairs
    // (j, j+16) rotated by pos * 100^(-j/16).
    role = args.q_role_base + col0 / args.q_C;  // 0 q, 1 k, 2 v, 3 second k, 4 second v
    const int cc = col0 % args.q_C;
    head = cc >> 6;
    d0 = cc & 63;  // 0 or 32
    const bool is_v = (role == 2 || role == 4);
    if (!is_v && args.q_rope) {
      const int p = (d0 >> 5) ? er.px : er.py;
      const float2* cs = args.q_cs + p * 16;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float2 t2 = __ldg(cs + j);
        const float u = v[j], x = v[j + 16];
        v[j] = u * t2.x - x * t2.y;
        v[j + 16] = x * t2.x + u * t2.y;
      }
    }
    if (role == 0) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] *= args.q_scale;
    }
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = to_tf32(v[j]);
    if (is_v) {   // V^T: for a fixed column the warp's 32 rows are 32 consecutive tokens -> already coalesced
      if (er.valid) {
        const int heads = args.q_C >> 6;
        const int bidx = (int)(er.pix / args.q_ntok);
        const int t = (int)(er.pix - (long long)bidx * args.q_ntok);
        const long long gb = (long long)tg.g * args.q_nb + bidx;
        float* op = (role == 2 ? args.vt_out : args.vt2_out) + ((gb * heads + head) * 64 + d0) * (long long)args.q_ntok_pad + t;
#pragma unroll
        for (int j = 0; j < 32; ++j) op[(long long)j * args.q_ntok_pad] = v[j];
      }
      return;
    }
  }

  // ---------------------------------------------------------------- stage, then transposed domain
  using S = Stg<SW>;
  const int cq = (lane % S::LPR) * 4;
  const int lr = lane / S::LPR;
  int ocol0 = col0;
  int ps_i = 0, ps_j = 0;
  if constexpr (EPI == EPI_PIXSHUF) {
    const int ij = col0 / args.ps_cout;
    ocol0 = col0 - ij * args.ps_cout;
    ps_i = ij / args.ps_s;
    ps_j = ij - ps_i * args.ps_s;
  }
  float st1[S::NIT], st2[S::NIT];   // LayerNorm statistics of the chunk, accumulated over the passes
#pragma unroll
  for (int it = 0; it < S::NIT; ++it) st1[it] = st2[it] = 0.f;
#pragma unroll
  for (int p = 0; p < S::NPASS; ++p) {
    {
      float4* sp = reinterpret_cast<float4*>(stg + lane * S::LD);
#pragma unroll
      for (int q = 0; q < SW / 4; ++q) {
        const int j = p * SW + 4 * q;
        sp[q] = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
      }
    }
    __syncwarp();
    const int ocol = ocol0 + p * SW + cq;
#pragma unroll
    for (int it = 0; it < S::NIT; ++it) {
      const long long key = tr.key[it];
      float4 x = *reinterpret_cast<const float4*>(stg + (it * S::RPI + lr) * S::LD + cq);
      if constexpr (EPI == EPI_QKV) {
        if (key >= 0) {
          float* op = (role == 0 ? args.q_out : role == 1 ? args.k_out : args.k2_out) + key +
                      (long long)head * args.q_ntok * 64 + d0 + p * SW + cq;
          *reinterpret_cast<float4*>(op) = x;
        }
      } else {
        long long orow = key;
        if constexpr (EPI == EPI_PIXSHUF) {
          if (key >= 0) orow = key + (long long)ps_i * (args.W * args.ps_s) + ps_j;
        }
        const bool ok = key >= 0;
        if (ok) {
          if (args.res1 != nullptr) {
            float4 t;
            if constexpr (EPI == EPI_PLAIN) {
              t = rp[p * S::NIT + it];
              if (res_next >= 0) rp[p * S::NIT + it] = ld_f4(args.res1 + orow * args.ldr1 + res_next + p * SW + cq);
            } else {
              t = ld_f4(args.res1 + orow * args.ldr1 + ocol);
            }
            x.x += t.x; x.y += t.y; x.z += t.z; x.w += t.w;
          }
          if (args.res2 != nullptr) {
            const float4 t = ld_f4(args.res2 + orow * args.ldr2 + ocol);
            x.x += t.x; x.y += t.y; x.z += t.z; x.w += t.w;
          }
        }
        if constexpr (EPI == EPI_PLAIN) {
          if (args.stats_out != nullptr) {   // (sum, sum of squares) of the row over this chunk: LayerNorm statistics
            st1[it] += (x.x + x.y) + (x.z + x.w);   // of the residual stream for the NEXT GEMM's folded LayerNorm
            st2[it] += fmaf(x.x, x.x, fmaf(x.y, x.y, fmaf(x.z, x.z, x.w * x.w)));
            if (p == S::NPASS - 1) {
              float s1 = st1[it], s2 = st2[it];
#pragma unroll
              for (int o = 1; o < S::LPR; o <<= 1) {
                s1 += __shfl_xor_sync(0xffffffffu, s1, o);
                s2 += __shfl_xor_sync(0xffffffffu, s2, o);
              }
              if (ok && (lane % S::LPR) == 0)
                args.stats_out[orow * (long long)(args.N >> 5) + (col0 >> 5)] = make_float2(s1, s2);
            }
          }
        }
        if (ok) {
          if (args.out_f32 != nullptr) *reinterpret_cast<float4*>(args.out_f32 + orow * args.ldo + ocol) = x;
          if (args.out_hi != nullptr) {
            if (args.plane_relu) {
              x.x = fmaxf(x.x, 0.f); x.y = fmaxf(x.y, 0.f); x.z = fmaxf(x.z, 0.f); x.w = fmaxf(x.w, 0.f);
            }
            uint32_t h0, l0, h1, l1;
            split2_bf16(x.x, x.y, h0, l0);
            split2_bf16(x.z, x.w, h1, l1);
            const long long po = orow * args.ldp + args.plane_col0 + ocol;
            *reinterpret_cast<uint2*>(args.out_hi + po) = make_uint2(h0, h1);
            *reinterpret_cast<uint2*>(args.out_lo + po) = make_uint2(l0, l1);
          }
        }
      }
    }
    __syncwarp();   // the staging tile is rewritten by the next pass / chunk
  }
}

// EPI_HEADTAIL: after the last chunk, the row's 4 dot products -> pts3d / conf (heads/postprocess.py:10-58)
__device__ __forceinline__ void epi_headtail_finish(const GemmArgs& args, const TileGeom& tg, const EpiRow& er,
                                                    const float (&ht_acc)[4]) {
  if (!er.valid) return;
  const float* b4 = args.ht_b + tg.g * 4;
  const float x = ht_acc[0] + b4[0], y = ht_acc[1] + b4[1], z = ht_acc[2] + b4[2], cf = ht_acc[3] + b4[3];
  const float d = sqrtf(x * x + y * y + z * z);
  const float sc = expm1f(d) / fmaxf(d, 1e-8f);
  float* pp = args.ht_pts + er.grow * 3;
  pp[0] = x * sc;
  pp[1] = y * sc;
  pp[2] = z * sc;
  args.ht_conf[er.grow] = 1.0f + expf(cf);
}

}  // namespace s3r
