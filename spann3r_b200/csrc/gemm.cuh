// Host-visible description of one launch of the split-bf16 wgmma GEMM / implicit-GEMM conv engine.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace s3r {

enum EpiMode : int {
  EPI_PLAIN = 0,      // out[row, col]
  EPI_PIXSHUF = 1,    // ConvTranspose2d with kernel == stride: col=(i,j,co) scatters to pixel (h*s+i, w*s+j)
  EPI_QKV = 2,        // q/k/v head split (+ 2-D RoPE on q,k; q pre-scaled; v stored transposed), tf32-rounded
  EPI_HEADTAIL = 3,   // DPT head tail: ReLU -> 1x1 conv (128->4) -> postprocess (pts3d, conf)
};
enum Act : int { ACT_NONE = 0, ACT_GELU = 1, ACT_RELU = 2 };

// A operand: activations as two bf16 planes laid out [G*NB, H, W, C] (C contiguous).  A plain
// linear layer is the degenerate image H=1, W=rows.  B operand: weights as two bf16 planes laid
// out [G*N, taps, Kc] (Kc contiguous).  Groups (G) share every shape and differ only in data.
struct GemmArgs {
  alignas(64) CUtensorMap tmA_hi;
  alignas(64) CUtensorMap tmA_lo;
  alignas(64) CUtensorMap tmB_hi;
  alignas(64) CUtensorMap tmB_lo;
  // geometry
  int groups;
  int W, H, NB;        // pixel space of one group
  int bw, bh;          // tile box, bw*bh == 128
  int tiles_w, tiles_h;
  int N;               // output columns per group
  int Kc, taps, kpt;   // channels per tap, 1 or 9 taps, k-blocks (of 64) per tap
  int b_group_rows;    // B rows between groups
  // epilogue
  int epi, act, plane_relu;
  const float* bias;   // [G*N] (EPI_PIXSHUF: [G*Cout]) or null
  const float* res1; int ldr1;
  const float* res2; int ldr2;
  float* out_f32; int ldo;            // row stride in elements
  __nv_bfloat16* out_hi; __nv_bfloat16* out_lo; int ldp; int plane_col0;
  long long out_group_rows;           // rows of `out`/`res`/planes per group
  // Folded LayerNorm (consumer side): A holds the planes of the RAW residual stream x, the weights carry gamma
  // (W' = W diag(gamma), bias' = b + W beta), and the epilogue applies rstd_r * (acc - mean_r * ln_cs[col]) + bias'.
  // ln_stats [A rows, ln_np] = (sum, sum of squares) per 32-column chunk of x, written by the producer's epilogue.
  const float2* ln_stats; int ln_np; float ln_eps;
  const float* ln_cs;                 // [G*N] column sums of W' (as the tensor core sees it: hi + lo planes)
  int b_static;                       // 1: B is a packed WEIGHT (never written on this stream): the producer may stage its first
                                      // B tiles before griddepcontrol.wait, while the previous kernel still runs
  int a_swap;                         // 1: group g reads the A rows (and statistics) of group G-1-g (norm_y of the twin decoders)
  int swap_col0;                      // ... for output columns >= swap_col0 only (0 = all); must be a multiple of the tile width
  // Producer side (EPI_PLAIN): write (sum, sum of squares) of every output row chunk, [rows, N/32]
  float2* stats_out;
  // optional timeline of CTA 0 (tools/trace_gemm.py): %globaltimer stamps [0..6] = entry, prologue done, dependency wait
  // done, first operands landed, first accumulator ready, last epilogue done, exit; null = off
  unsigned long long* trace;
  // EPI_PIXSHUF
  int ps_s, ps_cout;
  // EPI_QKV
  int q_C, q_role_base, q_ntok, q_ntok_pad, q_rope, q_nb;   // q_nb: batch items per group
  const int* q_pos;        // [G*rows, 2] (y, x) per A row
  const float2* q_cs;      // [maxpos, 16] (cos, sin)
  float* q_out; float* k_out; float* vt_out;
  float* k2_out; float* vt2_out;       // roles 3 / 4: a second K / V^T pair (the cross-attention K/V of the merged decoder launch)
  float q_scale;
  // EPI_HEADTAIL
  const float* ht_w;       // [G, 4, 128]
  const float* ht_b;       // [G, 4]
  float* ht_pts;           // [G*rows, 3]
  float* ht_conf;          // [G*rows]
};

struct GemmPlan {
  GemmArgs args;
  dim3 grid;
  int bn;          // 64 / 128
  int b_static;    // engine: B is a packed weight and the prefetch option was on when the plan was built
  double flops;    // algorithmic 2*M*N*K (all groups), for roofline accounting
};

// Encodes the four tensor maps and picks the tile shape.  Returns 0 or a negative error.
// lda / ldb: row strides (elements) of A pixels / B rows (0 = dense: Kc resp. taps*Kc);
// b_group_rows: rows between consecutive groups of B (0 = N).
// force_bn: 0 = planner's choice; 64 / 128 = that tile width; 256, 1128, 2064, 2128, 2256 = the nearest width the kernel has
// (128, 128, 64, 128, 128).
int gemm_plan_init(GemmPlan* plan,
                   const __nv_bfloat16* a_hi, const __nv_bfloat16* a_lo,   // [G*NB, H, W, Kc]
                   const __nv_bfloat16* b_hi, const __nv_bfloat16* b_lo,   // [G*N, taps, Kc]
                   int groups, int NB, int H, int W, int Kc, int taps, int N, int force_bn = 0,
                   long long lda = 0, long long ldb = 0, long long b_group_rows = 0);
int gemm_launch(const GemmPlan& plan, cudaStream_t stream);

// Tuning knobs of the tile planner / producers (s3r_set_option): read when a plan is BUILT, so two engines of one
// process can be planned under different settings and timed alternately (tools/ab_inproc.py).
struct Options {
  int prefetch_b = 1;   // stage the first weight tiles before griddepcontrol.wait
};
Options& options();
int num_sms();

int encode_tmap(CUtensorMap* out, CUtensorMapDataType dt, int rank, const void* base, const uint64_t* dims,
                const uint64_t* strides_bytes, const uint32_t* box);
const char* last_error();
void set_error(const char* fmt, ...);

}  // namespace s3r
