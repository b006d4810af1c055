// Shared device-side helpers for the sm_90a kernels: mbarrier, TMA, wgmma shared-memory descriptors
// and the split-bf16 ("bf16x3") number format used by every weight GEMM / conv on the path.
//
// Number format (DESIGN.md §3): an fp32 value x is carried as two bf16 planes
//     hi = bf16_rn(x),  lo = bf16_rn(x - hi)          (hi + lo carries ~16 mantissa bits)
// and a product a*b is issued as three tensor-core MMAs into one fp32 register accumulator
//     a_hi*b_hi + a_hi*b_lo + a_lo*b_hi              (the lo*lo term, 2^-16 relative, is dropped)
// which is what keeps the path inside the 1e-3 fp32 parity bar (SURVEY.md §7.3-#1).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdlib>
#include <utility>

namespace s3r {

// ----------------------------------------------------------------------------------------------
// small utilities
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P1;\n\t"
      "elect.sync _|P1, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P1;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// split fp32 -> (hi, lo) bf16
__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(x);
  lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}
// two values at once on the packed converter (F2FP.BF16.PACK_AB, full ALU rate; the scalar F2F.BF16.F32 the single-
// value form compiles to runs on the quarter-rate conversion pipe): hi / lo = packed bf16x2, first value in the low half.
// Bit-identical to split_bf16 on each value.
__device__ __forceinline__ void split2_bf16(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  const uint32_t hu = *reinterpret_cast<const uint32_t*>(&h);
  const float ah = __uint_as_float(hu << 16), bh = __uint_as_float(hu & 0xffff0000u);
  const __nv_bfloat162 l = __floats2bfloat162_rn(a - ah, b - bh);
  hi = hu;
  lo = *reinterpret_cast<const uint32_t*>(&l);
}
__device__ __forceinline__ uint32_t pack_bf16(__nv_bfloat16 a, __nv_bfloat16 b) {
  return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}
// round-to-nearest fp32 -> tf32 (kept in an fp32 container); the tensor core truncates otherwise
__device__ __forceinline__ float to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
// exact-erf GELU (nn.GELU default, croco/models/blocks.py:73-79).  Four values per call, not inlined: one call per
// element serialises ~35 dependent instructions 32 times per chunk (no ILP across calls: measured ~12 us of the
// decoder's fc1 launches), full inlining of 32 copies bloats every epilogue instantiation; four independent chains per
// call hide the FFMA latency at a quarter of the calls.
__device__ __forceinline__ float gelu_erf1(float x) {
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}
static __device__ __noinline__ float4 gelu_erf4(float4 x) {
  return make_float4(gelu_erf1(x.x), gelu_erf1(x.y), gelu_erf1(x.z), gelu_erf1(x.w));
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P1;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P1;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded spin: a descriptor/pipeline bug must not hang the GPU box (a hang is a strike);
// after ~2^28 failed probes the kernel traps, which surfaces as a CUDA error on the host.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 28)) { asm volatile("trap;"); }
  }
}

// ----------------------------------------------------------------------------------------------
// fences
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// ----------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) loads, completion on an mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::
          "r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// Variants on raw shared-memory addresses (warp-uniform producers keep them in uniform registers)
__device__ __forceinline__ void mbar_arrive_expect_tx_u(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_3d_u(uint32_t smem, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::
          "r"(smem),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d_u(uint32_t smem, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2,
                                              int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(smem),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ----------------------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptor for a K-major tile whose rows are exactly one 128-byte
// swizzle span (64 bf16 or 32 tf32) and which is stored as TMA SWIZZLE_128B wrote it:
//   start_address  = addr >> 4                       bits [0,14)
//   leading offset = 1 (ignored for swizzled K-major) bits [16,30)
//   stride offset  = 1024 B >> 4 = 64 (8-row group)   bits [32,46)
//   layout type    = 1 (SWIZZLE_128B)                 bits [62,64)
// Tiles start on 1024-byte boundaries (base offset 0).  Stepping along K inside the 128-byte span = adding
// (bytes >> 4) to the start address; stepping 64 rows = adding 8 KB.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t wgmma_desc_sw128_kmajor(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)64 << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// The same for rows of exactly one 64-byte swizzle span (32 bf16), stored as TMA SWIZZLE_64B wrote it:
//   stride offset  = 8 rows x 64 B = 512 B >> 4 = 32
//   layout type    = 2 (SWIZZLE_64B)
// Tiles start on 512-byte boundaries (base offset 0).  Each k16 step adds 32 bytes (2 in the start field); stepping
// 64 rows = adding 4 KB.
__device__ __forceinline__ uint64_t wgmma_desc_sw64_kmajor(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)32 << 32;
  d |= (uint64_t)2 << 62;
  return d;
}

// ----------------------------------------------------------------------------------------------
// Programmatic dependent launch (PDL): every kernel of the library is launched with
// cudaLaunchAttributeProgrammaticStreamSerialization, signals its dependents at once and waits for
// its prerequisite grid right before touching global memory, so the launch latency, CTA scheduling,
// barrier init and tensor-map prefetch of kernel i+1 overlap the tail of kernel i.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// 128-bit global stores / loads
__device__ __forceinline__ void st_f4(float* p, float a, float b, float c, float d) {
  *reinterpret_cast<float4*>(p) = make_float4(a, b, c, d);
}

// host: "configured once" flags.  cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is a PER-DEVICE attribute, so a
// process that drives several GPUs (Spann3R(...).to('cuda:1') beside one on cuda:0) needs one flag per device ordinal.
struct PerDeviceOnce {
  bool done[64] = {};
  bool& cur() {
    int d = 0;
    cudaGetDevice(&d);
    return done[d & 63];
  }
};

// host: launch with the PDL attribute
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  static const bool use_pdl = (getenv("S3R_NO_PDL") == nullptr);   // debugging switch
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = use_pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

}  // namespace s3r
