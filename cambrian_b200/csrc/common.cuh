// cambrian_b200 — shared device helpers for sm_90a (H100).
//
// Thin inline-PTX wrappers for the Hopper machinery every dense kernel in this library
// uses: mbarrier, TMA (cp.async.bulk.tensor), wgmma (fences, groups, shared-memory
// descriptors; the MMA instructions themselves are in wgmma.cuh).  Nothing here is
// derived from the reference (which ships no native code, SURVEY.md §2a); bit layouts
// follow the PTX ISA (wgmma matrix descriptors, canonical SWIZZLE_128B layouts).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda.h>
#include <stdint.h>
#include "wgmma.cuh"

namespace cb {

typedef __nv_bfloat16 bf16;

// ----------------------------------------------------------------------------------
// error plumbing shared by all translation units (defined in api.cu)
// ----------------------------------------------------------------------------------
int set_error(int code, const char* fmt, ...);
#define CB_OK 0
#define CB_ERR_INVALID 1
#define CB_ERR_CUDA 2
#define CB_ERR_UNSUPPORTED 3

#define CB_CHECK_ARG(cond, ...)                                         \
  do {                                                                  \
    if (!(cond)) return cb::set_error(CB_ERR_INVALID, __VA_ARGS__);     \
  } while (0)

void count_launch();  // api.cu: one increment per kernel launch (cb_launch_count)
#define CB_CUDA_LAUNCH_CHECK(name)                                                    \
  do {                                                                                \
    cb::count_launch();                                                               \
    cudaError_t _e = cudaGetLastError();                                              \
    if (_e != cudaSuccess)                                                            \
      return cb::set_error(CB_ERR_CUDA, "%s: %s", name, cudaGetErrorString(_e));      \
  } while (0)

int device_sm_count();

// ----------------------------------------------------------------------------------
// small math helpers
// ----------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// single MUFU.EX2 (2^-inf = +0, no denormal range fix-up branches): softmax inner loops
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// single MUFU.RCP: __fdividef() adds a range check + rescale sequence (FSETP / FMUL pairs) per element
__device__ __forceinline__ float fast_rcp(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// erf via Abramowitz & Stegun 7.1.26 (|abs err| <= 1.5e-7, far below bf16 resolution): one MUFU.EX2 + one MUFU.RCP +
// 7 FMA instead of erff's ~40-instruction polynomial, which made GELU epilogues the bottleneck of short-K GEMMs
__device__ __forceinline__ float erf_fast(float x) {
  const float ax = fabsf(x);
  const float t = __fdividef(1.0f, fmaf(0.3275911f, ax, 1.0f));
  float y = fmaf(t, 1.061405429f, -1.453152027f);
  y = fmaf(t, y, 1.421413741f);
  y = fmaf(t, y, -0.284496736f);
  y = fmaf(t, y, 0.254829592f);
  const float r = fmaf(-t * y, __expf(-ax * ax), 1.0f);
  return copysignf(r, x);
}
// x * Phi(x) with the same A&S erf, constants folded for z = x / sqrt(2): 14 instructions (2 MUFU) per element —
// GELU epilogues are ALU-bound, so every instruction shows
__device__ __forceinline__ float gelu_erf(float x) {
  const float ax = fabsf(x);
  const float t = fast_rcp(fmaf(0.3275911f * 0.70710678118654752440f, ax, 1.0f));
  float y = fmaf(t, 1.061405429f, -1.453152027f);
  y = fmaf(t, y, 1.421413741f);
  y = fmaf(t, y, -0.284496736f);
  y = fmaf(t, y, 0.254829592f);
  const float e = fast_exp2(x * x * -0.72134752044448170368f);  // exp(-x^2 / 2)
  const float r = fmaf(-(y * t), e, 1.0f);                       // erf(|x| / sqrt(2))
  const float hx = 0.5f * x;
  return fmaf(fabsf(hx), r, hx);                                 // 0.5 x (1 + sign(x) erf(|z|))
}
__device__ __forceinline__ float gelu_erf_grad(float x) {
  const float cdf = 0.5f * (1.0f + erf_fast(x * 0.70710678118654752440f));
  const float pdf = 0.39894228040143267794f * __expf(-0.5f * x * x);
  return cdf + x * pdf;
}
__device__ __forceinline__ float gelu_tanh(float x) {
  const float u = 0.7978845608028654f * (x + 0.044715f * x * x * x);
  return 0.5f * x * (1.0f + tanhf(u));
}
// tanh-GELU with tanh(u) = 1 - 2 / (1 + e^{2u}) on MUFU.EX2 / MUFU.RCP (tanhf's software path is branchy)
__device__ __forceinline__ float gelu_tanh_fast(float x) {
  const float u = 0.7978845608028654f * (x + 0.044715f * x * x * x);
  const float t = 1.0f - 2.0f * fast_rcp(1.0f + fast_exp2(2.0f * 1.44269504088896340736f * u));
  return 0.5f * x * (1.0f + t);
}
// __fdividef: MUFU.RCP + FMUL (2 ulp) instead of the IEEE division's Newton iterations + slow-path branch
__device__ __forceinline__ float quick_gelu(float x) { return x * fast_rcp(1.0f + fast_exp2(-1.702f * 1.44269504088896340736f * x)); }
__device__ __forceinline__ float silu(float x) { return x * fast_rcp(1.0f + fast_exp2(-1.44269504088896340736f * x)); }

// 8 x bf16 <-> 8 x float through one 16-byte register quad
struct alignas(16) bf16x8 {
  __nv_bfloat162 v[4];
};
__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
  const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = __bfloat1622float2(p[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  uint4 u;
  __nv_bfloat162* p = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) p[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return u;
}
// two fp32 -> two e4m3 (round to nearest even, |x| > 448 -> +-448); lo in the low byte (the FP8 row rule of
// quant_fp8.py, shared by every kernel that writes e4m3)
__device__ __forceinline__ uint32_t f8_pack2(float lo, float hi) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}
// 8 fp32 (already scaled by r) -> 8 e4m3 bytes, element 0 in the lowest byte
__device__ __forceinline__ uint2 f8_pack8(const float* v) {
  return make_uint2(f8_pack2(v[0], v[1]) | f8_pack2(v[2], v[3]) << 16, f8_pack2(v[4], v[5]) | f8_pack2(v[6], v[7]) << 16);
}
__device__ __forceinline__ uint4 ldg_nc(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

// ----------------------------------------------------------------------------------
// shared-memory address + mbarrier
// ----------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!done);
}
__device__ __forceinline__ void st_shared_b32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
// generic-proxy writes to smem -> visible to the async proxy (wgmma operand reads, TMA stores)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ----------------------------------------------------------------------------------
// TMA
// ----------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t smem_dst, const CUtensorMap* m, uint32_t bar,
                                            int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5}], [%2];"
      :
      : "r"(smem_dst), "l"(m), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t smem_dst, const CUtensorMap* m, uint32_t bar,
                                            int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5, %6}], [%2];"
      :
      : "r"(smem_dst), "l"(m), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// smem -> global tile store; TMA clips the parts of the box outside the tensor.  Completion is tracked per thread in
// bulk groups: commit after the stores, then wait until their smem source has been read (.read) or fully written out.
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, uint32_t smem_src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               :
               : "l"(m), "r"(smem_src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
// warpgroup-wide register re-allocation: a producer warpgroup gives registers back, consumer warpgroups take them
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
// barrier over a subset of the CTA's warps (id 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// ----------------------------------------------------------------------------------
// wgmma (sm_90a warpgroup MMA): ordering fences and group completion
// ----------------------------------------------------------------------------------
// register accumulators / A fragments written by ordinary instructions -> visible to the next wgmma.mma_async
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int R>
__device__ __forceinline__ void reg_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ----------------------------------------------------------------------------------
// wgmma shared-memory descriptors (SWIZZLE_128B canonical layouts, bf16)
//
// K-major tile (rows = M or N, 64 bf16 = 128 B of K per row, rows packed at 128 B):
//     8-row groups are 1024 B apart -> SBO = 1024, LBO unused.
//     advancing K by 16 elements inside the 128-B swizzle atom = +32 B on the start address.
// MN-major tile (rows = K, 64 bf16 = 128 B of M/N per row; one TMA box = 64(MN) x rows):
//     8-row K groups are 1024 B apart -> SBO = 1024; the next 64-wide MN atom is a whole
//     box away -> LBO = box bytes.  advancing K by 16 rows = +2048 B.
// Tiles start on 1024-byte boundaries, so the swizzle phase is a function of the address (base offset 0).
// ----------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t saddr, uint32_t lbo_bytes,
                                                         uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);              // [0,14)  start address
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;     // [16,30) leading byte offset
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;     // [32,46) stride byte offset
  d |= static_cast<uint64_t>(1) << 62;                              // [62,64) layout: SWIZZLE_128B
  return d;
}

// two fp32 -> one bf16x2 register (low half = first element): the A-fragment format of wgmma with A in registers
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}

}  // namespace cb
