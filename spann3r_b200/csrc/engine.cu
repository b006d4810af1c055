// Model-level runtime of libspann3r_b200.so: sequences the sm_90a kernels of one frame step of
// Spann3R.forward (spann3r/model.py:473-539) -- encoder, twin decoder, key heads, DPT heads, value
// encoder, spatial-memory read / append -- over an engine-owned activation workspace, with every
// tensor-map / tile plan built once per shape and replayed (no per-call descriptor encoding, no host
// synchronisation, no allocation after create()).  The two decoder streams, the two key heads and
// the two DPT heads run as 2-group launches of the same kernels.
#include "../../include/spann3r_b200.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <tuple>
#include <utility>
#include <vector>

#include "gemm.cuh"
#include "kernels.cuh"

using namespace s3r;

namespace {

struct Planes {
  __nv_bfloat16* hi = nullptr;
  __nv_bfloat16* lo = nullptr;
};
inline Planes WP(const s3r_planes& p) {
  Planes r;
  r.hi = (__nv_bfloat16*)p.hi;
  r.lo = (__nv_bfloat16*)p.lo;
  return r;
}

struct Geom {
  int groups = 1, NB = 1, H = 1, W = 1, Kc = 0, taps = 1, N = 0, force_bn = 0;
  int b_static = 1;   // B = packed weights (everything except the two memory-read GEMMs, whose B is the bank)
  long long lda = 0, ldb = 0, b_group_rows = 0;
};

struct Epi {
  int epi = EPI_PLAIN, act = ACT_NONE, plane_relu = 0;
  const float* bias = nullptr;
  const float* res1 = nullptr; int ldr1 = 0;
  const float* res2 = nullptr; int ldr2 = 0;
  float* out = nullptr; int ldo = 0;
  Planes op; int ldp = 0, col0 = 0;
  int ps_s = 0, ps_cout = 0;
  int q_C = 0, q_role_base = 0, q_ntok = 0, q_ntok_pad = 0, q_rope = 0, q_nb = 0;
  const int* q_pos = nullptr; const float2* q_cs = nullptr;
  float *q_out = nullptr, *k_out = nullptr, *vt_out = nullptr; float q_scale = 1.f;
  float *k2_out = nullptr, *vt2_out = nullptr; int swap_col0 = 0;
  const float *ht_w = nullptr, *ht_b = nullptr; float *ht_pts = nullptr, *ht_conf = nullptr;
  // folded LayerNorm: consumer side (statistics of the A rows + column sums of the gamma-folded weights) ...
  const float2* ln_stats = nullptr; int ln_np = 0; float ln_eps = 0.f; const float* ln_cs = nullptr; int a_swap = 0;
  float2* stats_out = nullptr;   // ... and producer side (chunk sums of the rows this GEMM writes)
};

// Plans are created on the first pass through a stage and replayed afterwards (same call order).
struct PlanCache {
  std::vector<GemmPlan> gemms;
  std::vector<AttnPlan> attns;
  size_t gc = 0, ac = 0;
  bool building = true;
  void begin() {
    gc = ac = 0;
    if (building) {   // a previous first pass failed half way (e.g. a plan_init error): start the plan list over
      gemms.clear();
      attns.clear();
    }
  }
  void end() { building = false; }
};

}  // namespace

struct s3r_engine {
  s3r_model_w w;
  int B, H, W, gh, gw, N, Npad, max_images;
  int device = 0;   // ordinal the workspace lives on; every stage call must be made with this device current
  std::vector<void*> allocs;
  double flops = 0;
  long long launches = 0;
  int status = 0;
  // optional per-launch timing of the tensor-core kernels (bench.py roofline leg)
  bool profiling = false;
  struct Timed { cudaEvent_t a, b; double flops; int kind; };   // kind 0 = GEMM/conv, 1 = attention
  std::vector<Timed> timed;
  std::vector<cudaEvent_t> ev_pool;
  cudaEvent_t get_event() {
    if (!ev_pool.empty()) { cudaEvent_t e = ev_pool.back(); ev_pool.pop_back(); return e; }
    cudaEvent_t e; cudaEventCreate(&e); return e;
  }

  // lookup tables
  int* pos = nullptr;  // [max_rows, 2] (y, x)
  int* pos_t = nullptr;  // [B*N, 2]: positions of the landscape-transposed grid (gw x gh), value encoder of portrait frames
  // encoder / value-encoder workspace (rows up to max_images*N, dim 1024)
  float* X = nullptr; Planes P, P2, Pim, AO, Hb; float *Qb = nullptr, *Kb = nullptr, *Vtb = nullptr;
  float2 *St1 = nullptr, *St2 = nullptr;   // LayerNorm chunk statistics of the residual stream (block input / after attention)
  // decoder workspace (2 groups x R rows, dim 768)
  float2 *Sa = nullptr, *Sb = nullptr, *Sc = nullptr;
  float* Xd = nullptr; Planes Pa, Pb, Pc, AOd, Hd, E0, Hk6, Hk9, Hk12, KH, KHh; float *Qd = nullptr, *Kd = nullptr, *Vtd = nullptr;
  float *Kd2 = nullptr, *Vtd2 = nullptr;   // cross-attention K / V^T (written by the merged qkv launch, read after self attention)
  float* D12 = nullptr; float* KO = nullptr;
  // DPT workspace
  Planes T1, T2, T4, T4c, A1, A2, A3, A4;       // act_postprocess stages
  float* Lf[4] = {nullptr, nullptr, nullptr, nullptr}; Planes Lr[4];  // layer_rn outputs (fp32 + relu planes)
  Planes Ra, Rb; float* Rf = nullptr; Planes Rfr; float* Rlow = nullptr; float* Rpath = nullptr; Planes P1;
  float* H0 = nullptr; Planes H0u;
  // value path
  float* Xv = nullptr; Planes Pv;
  // memory read
  Planes Qn, Pm; float* Sm = nullptr; float* ln_tmp = nullptr; float* sim_scratch = nullptr; int mem_cap = 0;

  // side streams of the DPT heads: the four act_postprocess -> layer_rn chains are independent until refinenet4
  cudaStream_t side[3] = {nullptr, nullptr, nullptr};
  cudaEvent_t ev_fork = nullptr, ev_join[3] = {nullptr, nullptr, nullptr};

  std::map<int, PlanCache> pc_encode;  // keyed by nimg
  PlanCache pc_decode, pc_keys, pc_heads, pc_value;
  // keyed by everything the cached tensor maps bake in: bank length, capacity and BOTH plane base pointers (a new
  // MemoryBank may reuse one address but not the other)
  std::map<std::tuple<long long, long long, const void*, const void*, const void*, const void*>, PlanCache> pc_memread;

  template <typename T>
  T* alloc(size_t n) {
    void* p = nullptr;
    if (cudaMalloc(&p, n * sizeof(T) + 256) != cudaSuccess) {
      set_error("engine: cudaMalloc of %zu bytes failed", n * sizeof(T));
      status = -7;
      return nullptr;
    }
    allocs.push_back(p);
    return reinterpret_cast<T*>(p);
  }
  void release(void* p) {   // cudaFree (synchronising) + forget; null is fine
    if (!p) return;
    for (size_t i = 0; i < allocs.size(); ++i)
      if (allocs[i] == p) {
        cudaFree(p);
        allocs.erase(allocs.begin() + i);
        return;
      }
  }
  Planes alloc_planes(size_t n) {
    Planes p;
    p.hi = alloc<__nv_bfloat16>(n);
    p.lo = alloc<__nv_bfloat16>(n);
    return p;
  }

  int gemm(PlanCache& pc, Planes A, Planes Bw, const Geom& g, const Epi& e, cudaStream_t st) {
    if (pc.building) {
      pc.gemms.emplace_back();
      int r = gemm_plan_init(&pc.gemms.back(), A.hi, A.lo, Bw.hi, Bw.lo, g.groups, g.NB, g.H, g.W, g.Kc, g.taps, g.N,
                             e.epi == EPI_HEADTAIL ? 1128 : g.force_bn, g.lda, g.ldb, g.b_group_rows);
      if (r) return r;
      pc.gemms.back().b_static = (g.b_static && options().prefetch_b) ? 1 : 0;   // decided when the plan is built
    }
    if (pc.gc >= pc.gemms.size()) {
      set_error("engine: plan cache out of sync");
      return -8;
    }
    GemmPlan& p = pc.gemms[pc.gc++];
    GemmArgs& a = p.args;
    a.epi = e.epi; a.act = e.act; a.plane_relu = e.plane_relu;
    a.bias = e.bias; a.res1 = e.res1; a.ldr1 = e.ldr1; a.res2 = e.res2; a.ldr2 = e.ldr2;
    a.out_f32 = e.out; a.ldo = e.ldo; a.out_hi = e.op.hi; a.out_lo = e.op.lo; a.ldp = e.ldp; a.plane_col0 = e.col0;
    if (e.epi == EPI_PIXSHUF) {
      a.ps_s = e.ps_s; a.ps_cout = e.ps_cout;
      a.out_group_rows = (long long)g.NB * g.H * e.ps_s * g.W * e.ps_s;
    } else if (e.epi == EPI_QKV) {
      a.q_C = e.q_C; a.q_role_base = e.q_role_base; a.q_ntok = e.q_ntok; a.q_ntok_pad = e.q_ntok_pad;
      a.q_rope = e.q_rope; a.q_nb = e.q_nb; a.q_pos = e.q_pos; a.q_cs = e.q_cs;
      a.q_out = e.q_out; a.k_out = e.k_out; a.vt_out = e.vt_out; a.q_scale = e.q_scale;
      a.k2_out = e.k2_out; a.vt2_out = e.vt2_out;
    } else if (e.epi == EPI_HEADTAIL) {
      a.ht_w = e.ht_w; a.ht_b = e.ht_b; a.ht_pts = e.ht_pts; a.ht_conf = e.ht_conf;
    }
    a.ln_stats = e.ln_stats; a.ln_np = e.ln_np; a.ln_eps = e.ln_eps; a.ln_cs = e.ln_cs; a.a_swap = e.a_swap;
    a.swap_col0 = e.swap_col0;
    a.stats_out = e.stats_out;
    a.b_static = p.b_static;
    flops += p.flops;
    ++launches;
    if (!profiling) return gemm_launch(p, st);
    Timed t; t.a = get_event(); t.b = get_event(); t.flops = p.flops; t.kind = 0;
    cudaEventRecord(t.a, st);
    int r = gemm_launch(p, st);
    cudaEventRecord(t.b, st);
    timed.push_back(t);
    return r;
  }

  int attention(PlanCache& pc, const float* q, const float* k, const float* vt, int BH, int heads, int nq, int nk,
                Planes out, long long ldo, cudaStream_t st) {
    if (pc.building) {
      pc.attns.emplace_back();
      int r = attn_plan_init(&pc.attns.back(), q, k, vt, BH, heads, nq, nk, Npad);
      if (r) return r;
    }
    if (pc.ac >= pc.attns.size()) {
      set_error("engine: attention plan cache out of sync");
      return -8;
    }
    AttnPlan& p = pc.attns[pc.ac++];
    flops += p.flops;
    ++launches;
    if (!profiling) return attn_launch(p, out.hi, out.lo, nullptr, ldo, st);
    Timed t; t.a = get_event(); t.b = get_event(); t.flops = p.flops; t.kind = 1;
    cudaEventRecord(t.a, st);
    int r = attn_launch(p, out.hi, out.lo, nullptr, ldo, st);
    cudaEventRecord(t.b, st);
    timed.push_back(t);
    return r;
  }

  int ln(const float* x, const s3r_ln& w, long long wb_stride, long long rows_per_group, float eps, long long rows, int C,
         float* out, long long ldo, Planes p, long long ldp, int col0, long long swap, cudaStream_t st) {
    ++launches;
    return launch_layernorm(x, C, w.w, w.b, wb_stride, rows_per_group, eps, rows, C, out, ldo, p.hi, p.lo, ldp, col0,
                            swap, st);
  }

  // ---- ViT blocks on X [nimg*N, D] (in place).  croco/models/blocks.py:127-130 ----
  // LayerNorms are folded into the GEMM that consumes them (s3r_lin.cs): P holds the planes of the block input x and St1
  // its per-row chunk statistics (written by whichever GEMM produced x).  No LayerNorm kernel runs inside a block.
  // Launch structure per block: [qkv of block 0] then, per block, attention, proj, fc1, fc2 and the NEXT block's qkv.
  int vit_qkv(PlanCache& pc, const s3r_block_w& bw, int D, int nimg, bool rope, cudaStream_t st, const int* pos_tab) {
    const int rows = nimg * N;
    Geom g; g.W = rows; g.Kc = D; g.N = 3 * D;
    Epi e; e.epi = EPI_QKV; e.bias = bw.qkv.b; e.q_C = D; e.q_role_base = 0; e.q_ntok = N; e.q_ntok_pad = Npad;
    e.q_rope = rope ? 1 : 0; e.q_nb = nimg; e.q_pos = pos_tab; e.q_cs = (const float2*)w.rope_cs;
    e.q_out = Qb; e.k_out = Kb; e.vt_out = Vtb; e.q_scale = 0.125f;
    e.ln_stats = St1; e.ln_np = D / 32; e.ln_eps = 1e-6f; e.ln_cs = bw.qkv.cs;                       // norm1
    return gemm(pc, P, WP(bw.qkv.w), g, e, st);
  }
  int vit_blocks(PlanCache& pc, const s3r_block_w* blocks, int depth, int D, int nimg, bool rope, float* Xp, cudaStream_t st,
                 const int* pos_tab = nullptr) {
    const int rows = nimg * N, heads = D / 64;
    if (!pos_tab) pos_tab = pos;
    int r;
    if ((r = vit_qkv(pc, blocks[0], D, nimg, rope, st, pos_tab))) return r;
    for (int l = 0; l < depth; ++l) {
      const s3r_block_w& bw = blocks[l];
      if ((r = attention(pc, Qb, Kb, Vtb, nimg * heads, heads, N, N, AO, D, st))) return r;
      {
        Geom g; g.W = rows; g.Kc = D; g.N = D;
        Epi e; e.bias = bw.proj.b; e.res1 = Xp; e.ldr1 = D; e.out = Xp; e.ldo = D;
        e.op = P2; e.ldp = D; e.stats_out = St2;
        if ((r = gemm(pc, AO, WP(bw.proj.w), g, e, st))) return r;
      }
      {
        Geom g; g.W = rows; g.Kc = D; g.N = 4 * D;
        Epi e; e.bias = bw.fc1.b; e.act = ACT_GELU; e.op = Hb; e.ldp = 4 * D;
        e.ln_stats = St2; e.ln_np = D / 32; e.ln_eps = 1e-6f; e.ln_cs = bw.fc1.cs;                       // norm2
        if ((r = gemm(pc, P2, WP(bw.fc1.w), g, e, st))) return r;
      }
      {
        Geom g; g.W = rows; g.Kc = 4 * D; g.N = D;
        Epi e; e.bias = bw.fc2.b; e.res1 = Xp; e.ldr1 = D; e.out = Xp; e.ldo = D;
        e.op = P; e.ldp = D; e.stats_out = St1;
        if ((r = gemm(pc, Hb, WP(bw.fc2.w), g, e, st))) return r;
      }
      if (l + 1 < depth && (r = vit_qkv(pc, blocks[l + 1], D, nimg, rope, st, pos_tab))) return r;
    }
    return 0;
  }
};

// ------------------------------------------------------------------------------------------------
// The library launches on the CURRENT device (stream, cudaFuncSetAttribute and tensor maps are per device): a stage call
// made while another device is current would run on the wrong GPU with this engine's pointers.  Refuse it.
static int engine_device_ok(const s3r_engine* e, const char* what) {
  int cur = -1;
  cudaGetDevice(&cur);
  if (cur == e->device) return 0;
  set_error("%s: the engine lives on device %d but device %d is current (wrap the call in torch.cuda.device(...))", what,
            e->device, cur);
  return -1;
}
#define S3R_ENGINE_DEVICE(e, what) \
  do { if (int r_ = engine_device_ok((e), (what))) return r_; } while (0)

static __global__ void fill_pos_kernel(int* pos, long long rows, int N, int gw) {
  const long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const int t = (int)(r % N);
  pos[2 * r] = t / gw;
  pos[2 * r + 1] = t % gw;
}
static __global__ void bank_bump_kernel(float* count, float* attn, long long ld, int len, int n_new) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (i < len) count[b * ld + i] += 1.0f;           // mem_count += 1   (spann3r/model.py:88)
  else if (i < len + n_new) {                        // new tokens: count = attn = 0   (:89-90)
    count[b * ld + i] = 0.f;
    attn[b * ld + i] = 0.f;
  }
}

extern "C" {

s3r_engine* s3r_engine_create(const s3r_model_w* w, int batch, int height, int width, int max_images) {
  if (!w || batch <= 0 || height % 16 != 0 || width % 16 != 0 || height <= 0 || width <= 0) {
    set_error("s3r_engine_create: need batch > 0 and height, width multiples of 16 (got %d, %dx%d)", batch, height, width);
    return nullptr;
  }
  if (max_images < 2 * batch) max_images = 2 * batch;
  s3r_engine* e = new s3r_engine();
  cudaGetDevice(&e->device);
  e->w = *w;
  e->B = batch; e->H = height; e->W = width;
  e->gh = height / 16; e->gw = width / 16;
  e->N = e->gh * e->gw;
  e->Npad = (e->N + 3) / 4 * 4;
  e->max_images = max_images;
  if (e->gh > w->rope_maxpos || e->gw > w->rope_maxpos) {
    set_error("s3r_engine_create: patch grid %dx%d exceeds the RoPE table (%d positions)", e->gh, e->gw, w->rope_maxpos);
    delete e;
    return nullptr;
  }
  const size_t N = e->N, R = (size_t)batch * N, Mx = (size_t)max_images * N;
  const size_t rows_max = Mx > 2 * R ? Mx : 2 * R;
  e->pos = e->alloc<int>(rows_max * 2);
  e->pos_t = e->alloc<int>(R * 2);
  // encoder / value encoder
  e->X = e->alloc<float>(Mx * 1024);
  e->P = e->alloc_planes(Mx * 1024);
  e->P2 = e->alloc_planes(Mx * 1024);
  e->St1 = e->alloc<float2>(Mx * 32);
  e->St2 = e->alloc<float2>(Mx * 32);
  e->Pim = e->alloc_planes(Mx * 768);
  e->AO = e->alloc_planes(Mx * 1024);
  e->Hb = e->alloc_planes(Mx * 4096);
  e->Qb = e->alloc<float>(Mx * 1024);
  e->Kb = e->alloc<float>(Mx * 1024);
  e->Vtb = e->alloc<float>((size_t)max_images * 16 * 64 * e->Npad);
  // decoder
  e->Xd = e->alloc<float>(2 * R * 768);
  e->Pa = e->alloc_planes(2 * R * 768);
  e->Pb = e->alloc_planes(2 * R * 768);
  e->Pc = e->alloc_planes(2 * R * 768);
  e->Sa = e->alloc<float2>(2 * R * 24);
  e->Sb = e->alloc<float2>(2 * R * 24);
  e->Sc = e->alloc<float2>(2 * R * 24);
  e->AOd = e->alloc_planes(2 * R * 768);
  e->Hd = e->alloc_planes(2 * R * 3072);
  e->E0 = e->alloc_planes(2 * R * 1024);
  e->Hk6 = e->alloc_planes(2 * R * 768);
  e->Hk9 = e->alloc_planes(2 * R * 768);
  e->Hk12 = e->alloc_planes(2 * R * 768);
  e->KH = e->alloc_planes(2 * R * 1792);
  e->KHh = e->alloc_planes(2 * R * 1792);
  e->Qd = e->alloc<float>(2 * R * 768);
  e->Kd = e->alloc<float>(2 * R * 768);
  e->Vtd = e->alloc<float>((size_t)2 * batch * 12 * 64 * e->Npad);
  e->Kd2 = e->alloc<float>(2 * R * 768);
  e->Vtd2 = e->alloc<float>((size_t)2 * batch * 12 * 64 * e->Npad);
  e->D12 = e->alloc<float>(2 * R * 768);
  e->KO = e->alloc<float>(2 * R * 1024);
  // DPT (2 heads as groups, batch images each)
  const size_t gb = 2 * (size_t)batch, g1 = (size_t)e->gh * e->gw;
  const size_t h3 = (e->gh + 1) / 2, w3 = (e->gw + 1) / 2;
  e->T1 = e->alloc_planes(gb * g1 * 96);
  e->A1 = e->alloc_planes(gb * g1 * 16 * 96);
  e->T2 = e->alloc_planes(gb * g1 * 192);
  e->A2 = e->alloc_planes(gb * g1 * 4 * 192);
  e->A3 = e->alloc_planes(gb * g1 * 384);
  e->T4 = e->alloc_planes(gb * g1 * 768);
  e->T4c = e->alloc_planes(gb * h3 * w3 * 9 * 768);
  e->A4 = e->alloc_planes(gb * h3 * w3 * 768);
  const size_t lpix[4] = {g1 * 16, g1 * 4, g1, h3 * w3};
  for (int i = 0; i < 4; ++i) {
    e->Lf[i] = e->alloc<float>(gb * lpix[i] * 256);
    e->Lr[i] = e->alloc_planes(gb * lpix[i] * 256);
  }
  const size_t big = gb * g1 * 16 * 256;  // largest refinenet level (4gh x 4gw)
  e->Ra = e->alloc_planes(big);
  e->Rb = e->alloc_planes(big);
  e->Rf = e->alloc<float>(big);
  e->Rfr = e->alloc_planes(big);
  e->Rlow = e->alloc<float>(big);
  e->Rpath = e->alloc<float>(big);                 // path at the NEXT level's resolution (<= 4gh x 4gw)
  e->P1 = e->alloc_planes(gb * g1 * 64 * 256);     // path_1 at 8gh x 8gw
  e->H0 = e->alloc<float>(gb * g1 * 64 * 128);
  e->H0u = e->alloc_planes(gb * g1 * 256 * 128);   // head.0 output upsampled to H x W
  // value path
  e->Xv = e->alloc<float>(R * 1024);
  e->Pv = e->alloc_planes(R * 1024);
  // memory read
  e->mem_cap = 0;
  e->Qn = e->alloc_planes(R * 1024);
  e->ln_tmp = e->alloc<float>(R * 1024);
  e->sim_scratch = e->alloc<float>((size_t)batch * 8 * N + 64);
  for (int i = 0; i < 3 && !e->status; ++i) {
    if (cudaStreamCreateWithFlags(&e->side[i], cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&e->ev_join[i], cudaEventDisableTiming) != cudaSuccess) {
      set_error("s3r_engine_create: side stream / event creation failed");
      e->status = -7;
    }
  }
  if (!e->status && cudaEventCreateWithFlags(&e->ev_fork, cudaEventDisableTiming) != cudaSuccess) e->status = -7;
  if (e->status) {
    s3r_engine_destroy(e);
    return nullptr;
  }
  fill_pos_kernel<<<(unsigned)((rows_max + 255) / 256), 256>>>(e->pos, (long long)rows_max, e->N, e->gw);
  fill_pos_kernel<<<(unsigned)((R + 255) / 256), 256>>>(e->pos_t, (long long)R, e->N, e->gh);
  if (cudaDeviceSynchronize() != cudaSuccess) {
    set_error("s3r_engine_create: init kernel failed: %s", cudaGetErrorString(cudaGetLastError()));
    s3r_engine_destroy(e);
    return nullptr;
  }
  return e;
}

void s3r_engine_destroy(s3r_engine* e) {
  if (!e) return;
  for (void* p : e->allocs) cudaFree(p);
  for (int i = 0; i < 3; ++i) {
    if (e->side[i]) cudaStreamDestroy(e->side[i]);
    if (e->ev_join[i]) cudaEventDestroy(e->ev_join[i]);
  }
  if (e->ev_fork) cudaEventDestroy(e->ev_fork);
  delete e;
}

double s3r_engine_take_flops(s3r_engine* e) {
  const double f = e->flops;
  e->flops = 0;
  return f;
}
void s3r_engine_profile(s3r_engine* e, int on) { e->profiling = on != 0; }

// Synchronises and copies out the per-launch CUDA-event durations recorded while profiling was on (without
// consuming them: follow with s3r_engine_profile_read).  Returns the number of launches recorded (may exceed cap).
int s3r_engine_profile_list(s3r_engine* e, double* ms, double* flops, int* kind, int cap) {
  if (cudaDeviceSynchronize() != cudaSuccess) {
    set_error("profile_list: %s", cudaGetErrorString(cudaGetLastError()));
    return -6;
  }
  int n = 0;
  for (auto& t : e->timed) {
    if (n < cap) {
      float v = 0.f;
      cudaEventElapsedTime(&v, t.a, t.b);
      ms[n] = v;
      flops[n] = t.flops;
      kind[n] = t.kind;
    }
    ++n;
  }
  return n;
}

// Synchronises, then sums CUDA-event durations of the launches recorded while profiling was on.
// out[0..3] = {gemm_ms, gemm_flops, gemm_launches, attn_ms}, out[4..5] = {attn_flops, attn_launches}
int s3r_engine_profile_read(s3r_engine* e, double* out) {
  for (int i = 0; i < 6; ++i) out[i] = 0;
  if (cudaDeviceSynchronize() != cudaSuccess) {
    set_error("profile_read: %s", cudaGetErrorString(cudaGetLastError()));
    return -6;
  }
  for (auto& t : e->timed) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, t.a, t.b);
    const int o = t.kind == 0 ? 0 : 3;
    out[o] += ms;
    out[o + 1] += t.flops;
    out[o + 2] += 1;
    e->ev_pool.push_back(t.a);
    e->ev_pool.push_back(t.b);
  }
  e->timed.clear();
  return 0;
}

long long s3r_engine_take_launches(s3r_engine* e) {
  const long long n = e->launches;
  e->launches = 0;
  return n;
}

// ------------------------------------------------------------------------------------------------
// encoder: dust3r/model.py:131-154
// ------------------------------------------------------------------------------------------------
int s3r_engine_encode(s3r_engine* e, const float* img, int nimg, float* feat, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  S3R_ENGINE_DEVICE(e, "s3r_engine_encode");
  if (nimg <= 0 || nimg > e->max_images) {
    set_error("s3r_engine_encode: nimg=%d outside [1, %d]", nimg, e->max_images);
    return -1;
  }
  PlanCache& pc = e->pc_encode[nimg];
  pc.begin();
  const int rows = nimg * e->N;
  int r;
  ++e->launches;
  if ((r = launch_im2col_patch16(img, 3LL * e->H * e->W, (long long)e->H * e->W, e->W, 1, nimg, e->gh, e->gw, e->Pim.hi,
                                 e->Pim.lo, st)))
    return r;
  {
    Geom g; g.W = rows; g.Kc = 768; g.N = 1024;
    Epi ep; ep.bias = e->w.patch_embed.b; ep.out = e->X; ep.ldo = 1024;
    ep.op = e->P; ep.ldp = 1024; ep.stats_out = e->St1;   // block 0's folded norm1 reads these
    if ((r = e->gemm(pc, e->Pim, WP(e->w.patch_embed.w), g, ep, st))) return r;
  }
  if ((r = e->vit_blocks(pc, e->w.enc, 24, 1024, nimg, true, e->X, st))) return r;
  if ((r = e->ln(e->X, e->w.enc_norm, 0, 0, 1e-6f, rows, 1024, feat, 1024, Planes(), 0, 0, 0, st))) return r;
  pc.end();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// twin decoder: dust3r/model.py:186-205, croco/models/blocks.py:186-191
// ------------------------------------------------------------------------------------------------
int s3r_engine_decode(s3r_engine* e, const float* f1, const float* f2, float* dec_all, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  S3R_ENGINE_DEVICE(e, "s3r_engine_decode");
  PlanCache& pc = e->pc_decode;
  pc.begin();
  const int N = e->N, B = e->B;
  const long long R = (long long)B * N;
  const float2* cs = (const float2*)e->w.rope_cs;
  int r;
  // hook 0 of the DPT heads = the encoder-dim inputs themselves (dust3r/model.py:187); also the A operand of
  // decoder_embed.  Stream 1 -> group 0, stream 2 -> group 1.
  e->launches += 2;
  if ((r = launch_split(f1, 1024, e->E0.hi, e->E0.lo, 1024, 0, R, 1024, 0, st))) return r;
  if ((r = launch_split(f2, 1024, e->E0.hi + R * 1024, e->E0.lo + R * 1024, 1024, 0, R, 1024, 0, st))) return r;
  {
    Geom g; g.W = (int)(2 * R); g.Kc = 1024; g.N = 768;   // shared weights: one group of 2R rows
    Epi ep; ep.bias = e->w.decoder_embed.b; ep.out = e->Xd; ep.ldo = 768;
    ep.op = e->Pa; ep.ldp = 768; ep.stats_out = e->Sa;
    if ((r = e->gemm(pc, e->E0, WP(e->w.decoder_embed.w), g, ep, st))) return r;
  }
  // All four LayerNorms of a DecoderBlock are folded into the GEMMs that consume them (s3r_lin.cs).  `xin` = planes
  // of the layer input (both streams), Sa its chunk statistics: read by qkv (norm1) and -- with the groups swapped,
  // each stream cross-attends to the OTHER stream's layer input -- by kv (norm_y).  Pb / Sb: x after self attention
  // (norm2 -> q), Pc / Sc: x after cross attention (norm3 -> fc1).  fc2 writes the next layer's xin / Sa.
  // Launch structure: [qkv of layer 0], then per layer: self attention, proj, q, cross attention, cproj, fc1, fc2 and the
  // NEXT layer's qkv.
  auto qkv_launch = [&](int l, Planes xin) {
    // self-attention q, k, v (norm1 folded) and -- same launch, columns >= 2304 reading the OTHER stream's layer
    // input (norm_y folded, group swap) -- the cross-attention k, v
    const s3r_decblock_w& bw = e->w.dec[l];
    Geom g; g.groups = 2; g.W = (int)R; g.Kc = 768; g.N = 3840;
    Epi ep; ep.epi = EPI_QKV; ep.bias = bw.qkv.b; ep.q_C = 768; ep.q_role_base = 0; ep.q_ntok = N; ep.q_ntok_pad = e->Npad;
    ep.q_rope = 1; ep.q_nb = B; ep.q_pos = e->pos; ep.q_cs = cs;
    ep.q_out = e->Qd; ep.k_out = e->Kd; ep.vt_out = e->Vtd; ep.k2_out = e->Kd2; ep.vt2_out = e->Vtd2; ep.q_scale = 0.125f;
    ep.ln_stats = e->Sa; ep.ln_np = 24; ep.ln_eps = 1e-6f; ep.ln_cs = bw.qkv.cs; ep.a_swap = 1; ep.swap_col0 = 2304;
    return e->gemm(pc, xin, WP(bw.qkv.w), g, ep, st);
  };
  Planes xin = e->Pa;
  if ((r = qkv_launch(0, xin))) return r;
  for (int l = 0; l < 12; ++l) {
    const s3r_decblock_w& bw = e->w.dec[l];
    if ((r = e->attention(pc, e->Qd, e->Kd, e->Vtd, 2 * B * 12, 12, N, N, e->AOd, 768, st))) return r;
    {
      Geom g; g.groups = 2; g.W = (int)R; g.Kc = 768; g.N = 768;
      Epi ep; ep.bias = bw.proj.b; ep.res1 = e->Xd; ep.ldr1 = 768; ep.out = e->Xd; ep.ldo = 768;
      ep.op = e->Pb; ep.ldp = 768; ep.stats_out = e->Sb;
      if ((r = e->gemm(pc, e->AOd, WP(bw.proj.w), g, ep, st))) return r;
    }
    // cross attention: q from norm2(x), k/v from norm_y(y), y = the other stream's layer input
    {
      Geom g; g.groups = 2; g.W = (int)R; g.Kc = 768; g.N = 768;
      Epi ep; ep.epi = EPI_QKV; ep.bias = bw.q.b; ep.q_C = 768; ep.q_role_base = 0; ep.q_ntok = N; ep.q_ntok_pad = e->Npad;
      ep.q_rope = 1; ep.q_nb = B; ep.q_pos = e->pos; ep.q_cs = cs;
      ep.q_out = e->Qd; ep.k_out = e->Kd; ep.vt_out = e->Vtd; ep.q_scale = 0.125f;
      ep.ln_stats = e->Sb; ep.ln_np = 24; ep.ln_eps = 1e-6f; ep.ln_cs = bw.q.cs;                        // norm2
      if ((r = e->gemm(pc, e->Pb, WP(bw.q.w), g, ep, st))) return r;
    }
    if ((r = e->attention(pc, e->Qd, e->Kd2, e->Vtd2, 2 * B * 12, 12, N, N, e->AOd, 768, st))) return r;
    {
      Geom g; g.groups = 2; g.W = (int)R; g.Kc = 768; g.N = 768;
      Epi ep; ep.bias = bw.cproj.b; ep.res1 = e->Xd; ep.ldr1 = 768; ep.out = e->Xd; ep.ldo = 768;
      ep.op = e->Pc; ep.ldp = 768; ep.stats_out = e->Sc;
      if ((r = e->gemm(pc, e->AOd, WP(bw.cproj.w), g, ep, st))) return r;
    }
    // MLP
    {
      Geom g; g.groups = 2; g.W = (int)R; g.Kc = 768; g.N = 3072;
      Epi ep; ep.bias = bw.fc1.b; ep.act = ACT_GELU; ep.op = e->Hd; ep.ldp = 3072;
      ep.ln_stats = e->Sc; ep.ln_np = 24; ep.ln_eps = 1e-6f; ep.ln_cs = bw.fc1.cs;                      // norm3
      if ((r = e->gemm(pc, e->Pc, WP(bw.fc1.w), g, ep, st))) return r;
    }
    {
      // the planes of the layer output are the next layer's xin; after layers 6 and 9 they are also DPT hooks
      // (dpt_head.py:108), so those layers write them straight into the hook buffers
      Planes xout = (l == 5) ? e->Hk6 : (l == 8) ? e->Hk9 : e->Pa;
      Geom g; g.groups = 2; g.W = (int)R; g.Kc = 3072; g.N = 768;
      Epi ep; ep.bias = bw.fc2.b; ep.res1 = e->Xd; ep.ldr1 = 768; ep.out = e->Xd; ep.ldo = 768;
      ep.op = xout; ep.ldp = 768; ep.stats_out = e->Sa;
      if ((r = e->gemm(pc, e->Hd, WP(bw.fc2.w), g, ep, st))) return r;
      xin = xout;
    }
    if (l < 11 && (r = qkv_launch(l + 1, xin))) return r;
    if (dec_all && l < 11) {
      ++e->launches;
      cudaMemcpyAsync(dec_all + (size_t)l * 2 * R * 768, e->Xd, (size_t)2 * R * 768 * sizeof(float),
                      cudaMemcpyDeviceToDevice, st);
    }
  }
  // dec_norm on the last pair (dust3r/model.py:203): fp32 for callers, planes as DPT hook 12 and as the
  // right half of the key-head input cat(feat, dec[-1]).
  if ((r = e->ln(e->Xd, e->w.dec_norm, 0, 0, 1e-6f, 2 * R, 768, e->D12, 768, e->Hk12, 768, 0, 0, st))) return r;
  if ((r = e->ln(e->Xd, e->w.dec_norm, 0, 0, 1e-6f, 2 * R, 768, nullptr, 0, e->KH, 1792, 1024, 0, st))) return r;
  if (dec_all) {
    ++e->launches;
    cudaMemcpyAsync(dec_all + (size_t)11 * 2 * R * 768, e->D12, (size_t)2 * R * 768 * sizeof(float),
                    cudaMemcpyDeviceToDevice, st);
  }
  pc.end();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// key heads: spann3r/model.py:299-303 (Linear 1792->1792, GELU, Linear 1792->1024), both heads grouped
// ------------------------------------------------------------------------------------------------
int s3r_engine_keyheads(s3r_engine* e, const float* feat1, const float* feat2, float* k1, float* k2, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  S3R_ENGINE_DEVICE(e, "s3r_engine_keyheads");
  PlanCache& pc = e->pc_keys;
  pc.begin();
  const long long R = (long long)e->B * e->N;
  int r;
  e->launches += 2;
  if ((r = launch_split(feat1, 1024, e->KH.hi, e->KH.lo, 1792, 0, R, 1024, 0, st))) return r;
  if ((r = launch_split(feat2, 1024, e->KH.hi + R * 1792, e->KH.lo + R * 1792, 1792, 0, R, 1024, 0, st))) return r;
  {
    Geom g; g.groups = 2; g.W = (int)R; g.Kc = 1792; g.N = 1792;
    Epi ep; ep.bias = e->w.key_fc1.b; ep.act = ACT_GELU; ep.op = e->KHh; ep.ldp = 1792;
    if ((r = e->gemm(pc, e->KH, WP(e->w.key_fc1.w), g, ep, st))) return r;
  }
  {
    Geom g; g.groups = 2; g.W = (int)R; g.Kc = 1792; g.N = 1024;
    Epi ep; ep.bias = e->w.key_fc2.b; ep.out = e->KO; ep.ldo = 1024;
    if ((r = e->gemm(pc, e->KHh, WP(e->w.key_fc2.w), g, ep, st))) return r;
  }
  e->launches += 2;
  cudaMemcpyAsync(k1, e->KO, (size_t)R * 1024 * sizeof(float), cudaMemcpyDeviceToDevice, st);
  cudaMemcpyAsync(k2, e->KO + R * 1024, (size_t)R * 1024 * sizeof(float), cudaMemcpyDeviceToDevice, st);
  pc.end();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// DPT heads: dust3r/heads/dpt_head.py:34-65 + croco/models/dpt_block.py + postprocess.py, both heads
// as 2 groups.  out_conv (1x1) is applied BEFORE the bilinear x2 upsample of each fusion block:
// both are linear and the interpolation weights sum to 1, so the result is identical up to fp32
// rounding while the 1x1 GEMM runs on 4x fewer pixels.
// ------------------------------------------------------------------------------------------------
int s3r_engine_heads(s3r_engine* e, float* pts, float* conf, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  S3R_ENGINE_DEVICE(e, "s3r_engine_heads");
  PlanCache& pc = e->pc_heads;
  pc.begin();
  const s3r_dpt_w& d = e->w.dpt;
  const int B = e->B, gh = e->gh, gw = e->gw;
  const int h3 = (gh + 1) / 2, w3 = (gw + 1) / 2;
  int r;
  cudaStream_t cur = st;   // stream the next launch goes to
  auto conv1x1 = [&](Planes A, int H, int W, int Cin, const s3r_lin& w, int Cout, Epi ep) {
    Geom g; g.groups = 2; g.NB = B; g.H = H; g.W = W; g.Kc = Cin; g.N = Cout;
    ep.bias = w.b;
    return e->gemm(pc, A, WP(w.w), g, ep, cur);
  };
  auto conv3x3 = [&](Planes A, int H, int W, int Cin, const s3r_lin& w, int Cout, Epi ep) {
    Geom g; g.groups = 2; g.NB = B; g.H = H; g.W = W; g.Kc = Cin; g.taps = 9; g.N = Cout;
    ep.bias = w.b;
    return e->gemm(pc, A, WP(w.w), g, ep, cur);
  };
  const int LH[4] = {4 * gh, 2 * gh, gh, h3}, LW[4] = {4 * gw, 2 * gw, gw, w3}, LC[4] = {96, 192, 384, 768};
  Planes Lin[4] = {e->A1, e->A2, e->A3, e->A4};
  auto layer_rn = [&](int i) {   // layer_rn (3x3, no bias): fp32 (residual) + relu planes (next conv's input)
    Epi ep; ep.out = e->Lf[i]; ep.ldo = 256; ep.op = e->Lr[i]; ep.ldp = 256; ep.plane_relu = 1;
    return conv3x3(Lin[i], LH[i], LW[i], LC[i], d.layer_rn[i], 256, ep);
  };
  // --- act_postprocess (dpt_block.py:356-410) + layer_rn (:33-75): four chains, one per pyramid level, independent
  // until refinenet4.  They are small (2 .. 96 pixel tiles) and latency-bound, so levels 2-4 run on side streams
  // beside level 1 (forked / joined with events; single stream while per-launch profiling is on).  The launch ORDER
  // in the plan cache is the same either way.
  const bool par = !e->profiling;
  if (par) {
    cudaEventRecord(e->ev_fork, st);
    for (int i = 0; i < 3; ++i) cudaStreamWaitEvent(e->side[i], e->ev_fork, 0);
  }
  // level 1 (4gh x 4gw)
  { Epi ep; ep.op = e->T1; ep.ldp = 96; if ((r = conv1x1(e->E0, gh, gw, 1024, d.act1_conv, 96, ep))) return r; }
  { Epi ep; ep.epi = EPI_PIXSHUF; ep.ps_s = 4; ep.ps_cout = 96; ep.op = e->A1; ep.ldp = 96;
    if ((r = conv1x1(e->T1, gh, gw, 96, d.act1_up, 16 * 96, ep))) return r; }
  if ((r = layer_rn(0))) return r;
  // level 2 (2gh x 2gw)
  if (par) cur = e->side[0];
  { Epi ep; ep.op = e->T2; ep.ldp = 192; if ((r = conv1x1(e->Hk6, gh, gw, 768, d.act2_conv, 192, ep))) return r; }
  { Epi ep; ep.epi = EPI_PIXSHUF; ep.ps_s = 2; ep.ps_cout = 192; ep.op = e->A2; ep.ldp = 192;
    if ((r = conv1x1(e->T2, gh, gw, 192, d.act2_up, 4 * 192, ep))) return r; }
  if ((r = layer_rn(1))) return r;
  // level 3 (gh x gw)
  if (par) cur = e->side[1];
  { Epi ep; ep.op = e->A3; ep.ldp = 384; if ((r = conv1x1(e->Hk9, gh, gw, 768, d.act3_conv, 384, ep))) return r; }
  if ((r = layer_rn(2))) return r;
  // level 4 (gh/2 x gw/2): 1x1, then the stride-2 3x3 as im2col + GEMM
  if (par) cur = e->side[2];
  { Epi ep; ep.op = e->T4; ep.ldp = 768; if ((r = conv1x1(e->Hk12, gh, gw, 768, d.act4_conv, 768, ep))) return r; }
  ++e->launches;
  if ((r = launch_im2col_3x3s2(e->T4.hi, e->T4.lo, 2 * B, gh, gw, 768, h3, w3, e->T4c.hi, e->T4c.lo, cur))) return r;
  { Epi ep; ep.op = e->A4; ep.ldp = 768; if ((r = conv1x1(e->T4c, h3, w3, 9 * 768, d.act4_down, 768, ep))) return r; }
  if ((r = layer_rn(3))) return r;
  cur = st;
  if (par) {
    for (int i = 0; i < 3; ++i) {
      cudaEventRecord(e->ev_join[i], e->side[i]);
      cudaStreamWaitEvent(st, e->ev_join[i], 0);
    }
  }
  // --- refinenet4 .. refinenet1 (FeatureFusionBlock_custom, dpt_block.py:189-218) ---
  const float* path = nullptr;  // fp32 path from the coarser level, at this level's resolution
  for (int lvl = 3; lvl >= 0; --lvl) {
    const s3r_fusion_w& f = d.refine[lvl];
    const int Hh = LH[lvl], Ww = LW[lvl];
    const float* xin = e->Lf[lvl];   // input of resConfUnit2 (fp32) ...
    Planes xin_r = e->Lr[lvl];       // ... and its relu planes
    if (path) {
      // output = path + resConfUnit1(layer):  conv1(relu(layer)) -> relu -> conv2 + layer + path
      { Epi ep; ep.act = ACT_RELU; ep.op = e->Ra; ep.ldp = 256; if ((r = conv3x3(e->Lr[lvl], Hh, Ww, 256, f.rcu1.conv1, 256, ep))) return r; }
      { Epi ep; ep.res1 = e->Lf[lvl]; ep.ldr1 = 256; ep.res2 = path; ep.ldr2 = 256; ep.out = e->Rf; ep.ldo = 256;
        ep.op = e->Rfr; ep.ldp = 256; ep.plane_relu = 1;
        if ((r = conv3x3(e->Ra, Hh, Ww, 256, f.rcu1.conv2, 256, ep))) return r; }
      xin = e->Rf;
      xin_r = e->Rfr;
    }
    // resConfUnit2
    { Epi ep; ep.act = ACT_RELU; ep.op = e->Ra; ep.ldp = 256; if ((r = conv3x3(xin_r, Hh, Ww, 256, f.rcu2.conv1, 256, ep))) return r; }
    { Epi ep; ep.res1 = xin; ep.ldr1 = 256; ep.op = e->Rb; ep.ldp = 256; if ((r = conv3x3(e->Ra, Hh, Ww, 256, f.rcu2.conv2, 256, ep))) return r; }
    // out_conv at this resolution, then bilinear x2 (align_corners=True)
    { Epi ep; ep.out = e->Rlow; ep.ldo = 256; if ((r = conv1x1(e->Rb, Hh, Ww, 256, f.out_conv, 256, ep))) return r; }
    ++e->launches;
    if (lvl > 0) {
      // refinenet4's output is cropped to layers[2]'s size when the patch grid is odd (dpt_head.py:56)
      if ((r = launch_upsample2x(e->Rlow, 2 * B, Hh, Ww, 256, e->Rpath, nullptr, nullptr, st, LH[lvl - 1], LW[lvl - 1]))) return r;
      path = e->Rpath;
    } else {
      if ((r = launch_upsample2x(e->Rlow, 2 * B, Hh, Ww, 256, nullptr, e->P1.hi, e->P1.lo, st))) return r;
    }
  }
  // --- head (dpt_block.py:318-324): conv3x3 256->128, x2 bilinear, conv3x3 128->128, ReLU, conv1x1 128->4, postprocess
  { Epi ep; ep.out = e->H0; ep.ldo = 128; if ((r = conv3x3(e->P1, 8 * gh, 8 * gw, 256, d.head0, 128, ep))) return r; }
  ++e->launches;
  if ((r = launch_upsample2x(e->H0, 2 * B, 8 * gh, 8 * gw, 128, nullptr, e->H0u.hi, e->H0u.lo, st))) return r;
  { Epi ep; ep.epi = EPI_HEADTAIL; ep.act = ACT_RELU; ep.ht_w = d.head4_w; ep.ht_b = d.head4_b; ep.ht_pts = pts; ep.ht_conf = conf;
    if ((r = conv3x3(e->H0u, 16 * gh, 16 * gw, 128, d.head2, 128, ep))) return r; }
  pc.end();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// value encoder: spann3r/model.py:305-320 (pos_patch_embed on pts3d, 6 Blocks without RoPE, value_norm,
// value_out) + `cur_v + feat_k1` (:519-521) fused as the residual of value_out.
// ------------------------------------------------------------------------------------------------
int s3r_engine_value(s3r_engine* e, const float* pts3d, const float* feat_k1, int flags, float* out, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  S3R_ENGINE_DEVICE(e, "s3r_engine_value");
  if (flags & ~(S3R_VALUE_PTS_TRANSPOSED | S3R_VALUE_ROPE)) {
    set_error("s3r_engine_value: unknown flags 0x%x", flags);
    return -1;
  }
  const bool tr = (flags & S3R_VALUE_PTS_TRANSPOSED) != 0, rope = (flags & S3R_VALUE_ROPE) != 0;
  // the cached plans do not depend on the flags: same launches, shapes and buffers; the flags only pick the im2col
  // strides and the per-call RoPE switch / position table of the qkv epilogue
  PlanCache& pc = e->pc_value;
  pc.begin();
  const int B = e->B;
  const int rows = B * e->N;
  int r;
  ++e->launches;
  // pts3d is the head's [B, H, W, 3] map: the reference permutes to NCHW first; here the im2col reads it with NHWC
  // strides.  For a portrait frame the landscape wrapper (dust3r/utils/misc.py:66-94) hands encode_cur_value the
  // map with axes 1 and 2 swapped, i.e. an image of W rows x H columns: same memory, row / column strides exchanged,
  // patch grid gw x gh (S3R_VALUE_PTS_TRANSPOSED).
  const long long srow = (long long)e->W * 3, spx = 3;
  if ((r = launch_im2col_patch16(pts3d, (long long)e->H * e->W * 3, 1, tr ? spx : srow, tr ? srow : spx, B,
                                 tr ? e->gw : e->gh, tr ? e->gh : e->gw, e->Pim.hi, e->Pim.lo, st)))
    return r;
  {
    Geom g; g.W = rows; g.Kc = 768; g.N = 1024;
    Epi ep; ep.bias = e->w.pos_patch_embed.b; ep.out = e->Xv; ep.ldo = 1024;
    ep.op = e->P; ep.ldp = 1024; ep.stats_out = e->St1;
    if ((r = e->gemm(pc, e->Pim, WP(e->w.pos_patch_embed.w), g, ep, st))) return r;
  }
  if ((r = e->vit_blocks(pc, e->w.val, 6, 1024, B, rope, e->Xv, st, tr ? e->pos_t : e->pos))) return r;
  if ((r = e->ln(e->Xv, e->w.value_norm, 0, 0, 1e-6f, rows, 1024, nullptr, 0, e->Pv, 1024, 0, 0, st))) return r;
  {
    Geom g; g.W = rows; g.Kc = 1024; g.N = 1024;
    Epi ep; ep.bias = e->w.value_out.b; ep.res1 = feat_k1; ep.ldr1 = 1024; ep.out = out; ep.ldo = 1024;
    if ((r = e->gemm(pc, e->Pv, WP(e->w.value_out.w), g, ep, st))) return r;
  }
  pc.end();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// spatial memory: spann3r/model.py:145-183 (read), :80-95 (append), :97-118 (similarity gate)
// ------------------------------------------------------------------------------------------------
int s3r_engine_memory_read(s3r_engine* e, const s3r_bank* bank, const float* feat, float thresh, float* out,
                           void* stream) {
  return s3r_engine_memory_read_train(e, bank, feat, thresh, 0.f, 0ull, out, stream);
}

// training-mode read (spann3r/model.py:474 attn_thresh = 0, :167-168 dropout on the attention weights): same launches, the
// softmax stage additionally applies the Philox keep-scale of (seed, row * M + column)
int s3r_engine_memory_read_train(s3r_engine* e, const s3r_bank* bank, const float* feat, float thresh, float drop_p,
                                 uint64_t seed, float* out, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  S3R_ENGINE_DEVICE(e, "s3r_engine_memory_read");
  if (!(drop_p >= 0.f && drop_p < 1.f)) {
    set_error("s3r_engine_memory_read: dropout probability %g outside [0, 1)", (double)drop_p);
    return -1;
  }
  const int B = e->B, N = e->N, M = bank->len, cap = bank->cap;
  if (M <= 0 || M > cap || cap % 8 != 0) {
    set_error("s3r_engine_memory_read: bad bank (len=%d cap=%d; cap must be a multiple of 8)", M, cap);
    return -1;
  }
  if (cap > e->mem_cap) {  // (re)size the score / probability scratch for this bank capacity (rare)
    e->release(e->Sm); e->release(e->Pm.hi); e->release(e->Pm.lo);   // the old scratch is dead: no stage is in flight on it
    e->Sm = e->alloc<float>((size_t)B * N * cap);                    // that a later launch of this stream could overtake
    e->Pm = e->alloc_planes((size_t)B * N * cap);
    if (e->status) return e->status;
    e->mem_cap = cap;
    e->pc_memread.clear();
  }
  // plans bake in (len, cap, bank pointers): a process that keeps creating banks at new addresses must not grow the
  // cache without bound (one sequence touches <= 16 distinct lengths)
  if (e->pc_memread.size() > 256) e->pc_memread.clear();
  PlanCache& pc = e->pc_memread[std::make_tuple((long long)M, (long long)cap, (const void*)bank->kn_hi, (const void*)bank->kn_lo,
                                                (const void*)bank->vnt_hi, (const void*)bank->vnt_lo)];
  pc.begin();
  const long long R = (long long)B * N;
  const int Mpad = (M + 7) / 8 * 8;
  int r;
  if ((r = e->ln(feat, e->w.norm_q, 0, 0, 1e-5f, R, 1024, nullptr, 0, e->Qn, 1024, 0, 0, st))) return r;
  {  // S = LN_q(feat) . LN_k(mem_k)^T, one group per batch item (each sequence has its own bank)
    Geom g; g.groups = B; g.W = N; g.Kc = 1024; g.N = M; g.b_group_rows = cap; g.b_static = 0;
    Epi ep; ep.out = e->Sm; ep.ldo = e->mem_cap;
    if ((M + 31) / 32 * 32 > cap) {  // the epilogue writes whole 32-column chunks
      set_error("s3r_engine_memory_read: bank capacity %d must cover len %d rounded up to 32", cap, M);
      return -1;
    }
    Planes Kn; Kn.hi = (__nv_bfloat16*)bank->kn_hi; Kn.lo = (__nv_bfloat16*)bank->kn_lo;
    if ((r = e->gemm(pc, e->Qn, Kn, g, ep, st))) return r;
  }
  e->launches += 3;
  if ((r = launch_mem_softmax(e->Sm, e->mem_cap, R, M, Mpad, 1.0f / 32.0f, thresh, e->Pm.hi, e->Pm.lo, e->mem_cap, st,
                              drop_p, seed)))
    return r;
  // the fp32 scores are dead once the softmax has run: Sm doubles as the [B, chunks, mem_cap] partial-sum scratch
  if ((r = launch_mem_colsum(e->Pm.hi, e->Pm.lo, e->mem_cap, B, N, M, bank->attn, cap, e->Sm, e->mem_cap, st))) return r;
  {  // out = attn . LN_v(mem_v) + feat
    Geom g; g.groups = B; g.W = N; g.Kc = M; g.N = 1024; g.lda = e->mem_cap; g.ldb = cap; g.b_group_rows = 1024; g.b_static = 0;
    Epi ep; ep.res1 = feat; ep.ldr1 = 1024; ep.out = out; ep.ldo = 1024;
    Planes Vt; Vt.hi = (__nv_bfloat16*)bank->vnt_hi; Vt.lo = (__nv_bfloat16*)bank->vnt_lo;
    if ((r = e->gemm(pc, e->Pm, Vt, g, ep, st))) return r;
  }
  pc.end();
  return 0;
}

int s3r_engine_memory_append(s3r_engine* e, const s3r_bank* bank, const float* feat_k, const float* feat_v,
                             void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  S3R_ENGINE_DEVICE(e, "s3r_engine_memory_append");
  const int B = e->B, N = e->N, M = bank->len, cap = bank->cap;
  if (M + N > cap) {
    set_error("s3r_engine_memory_append: bank full (len=%d + %d > cap=%d)", M, N, cap);
    return -1;
  }
  int r;
  Planes Kn; Kn.hi = (__nv_bfloat16*)bank->kn_hi; Kn.lo = (__nv_bfloat16*)bank->kn_lo;
  for (int b = 0; b < B; ++b) {
    const size_t src = (size_t)b * N * 1024, dst = ((size_t)b * cap + M) * 1024;
    // normalised keys straight into the bank rows
    Planes kd; kd.hi = Kn.hi + dst; kd.lo = Kn.lo + dst;
    if ((r = e->ln(feat_k + src, e->w.norm_k, 0, 0, 1e-5f, N, 1024, nullptr, 0, kd, 1024, 0, 0, st))) return r;
    e->launches += 2;
    cudaMemcpyAsync(bank->k_raw + dst, feat_k + src, (size_t)N * 1024 * sizeof(float), cudaMemcpyDeviceToDevice, st);
    cudaMemcpyAsync(bank->v_raw + dst, feat_v + src, (size_t)N * 1024 * sizeof(float), cudaMemcpyDeviceToDevice, st);
  }
  // normalised values -> transposed planes [B, 1024, cap] at columns [M, M+N)
  if ((r = e->ln(feat_v, e->w.norm_v, 0, 0, 1e-5f, (long long)B * N, 1024, e->ln_tmp, 1024, Planes(), 0, 0, 0, st))) return r;
  e->launches += 2;
  if ((r = launch_split_transpose(e->ln_tmp, B, N, 1024, (__nv_bfloat16*)bank->vnt_hi, (__nv_bfloat16*)bank->vnt_lo, cap,
                                  (long long)1024 * cap, M, st)))
    return r;
  dim3 grid((M + N + 255) / 256, B);
  bank_bump_kernel<<<grid, 256, 0, st>>>(bank->count, bank->attn, cap, M, N);
  return cudaGetLastError() == cudaSuccess ? 0 : -6;
}

int s3r_engine_check_sim(s3r_engine* e, const s3r_bank* bank, const float* feat_k, int wm, float* out, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  S3R_ENGINE_DEVICE(e, "s3r_engine_check_sim");
  const int B = e->B, N = e->N;
  if (wm <= 0 || wm > 8 || wm * N > bank->len) {
    set_error("s3r_engine_check_sim: wm=%d invalid for bank len %d", wm, bank->len);
    return -1;
  }
  e->launches += 2;
  const float* wmem = bank->k_raw + (size_t)(bank->len - wm * N) * 1024;  // last wm*N tokens (spann3r/model.py:102-105)
  return launch_check_sim(feat_k, wmem, (long long)bank->cap * 1024, B, wm, N, 1024, e->sim_scratch, out, st);
}

}  // extern "C"
