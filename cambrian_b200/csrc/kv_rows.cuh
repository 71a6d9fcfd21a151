// Row helpers shared by the decode KV-cache kernels (fp8.cu: the dense FP8 cache, paged.cu: the paged cache).  Every
// lane owns KV_DPL = 8 consecutive elements of one hd-element head row, so a row is a team of hd / 8 adjacent lanes (16
// at hd 128, 8 at hd 64) and row reductions are xor-shuffles inside the team.
#pragma once
#include "common.cuh"
#include <cuda_fp16.h>
#include <cfloat>

namespace cb {

constexpr int KV_DPL = 8;
constexpr float KV_LOG2E = 1.4426950408889634f;

template <int LPK>
__device__ __forceinline__ float team_max(float v) {
#pragma unroll
  for (int o = LPK / 2; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
template <int LPK>
__device__ __forceinline__ float team_sum(float v) {
#pragma unroll
  for (int o = LPK / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// 8 e4m3 (lowest byte first) -> 8 fp32, exactly: two values per packed cvt to f16x2, then f16 -> f32
__device__ __forceinline__ void e4m3x8_to_f32(uint2 u, float* f) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint16_t pair = (uint16_t)(((i < 2) ? u.x : u.y) >> (16 * (i & 1)));
    uint32_t h2;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h2) : "h"(pair));
    const float2 t = __half22float2(*reinterpret_cast<const __half2*>(&h2));
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
// The row rule of cambrian_b200/kv_fp8.py on a lane's 8 elements f, given the team's amax a: the scale a / 448 and the
// 8 e4m3 bytes of round_satfinite(f * fmin(448 / a, FLT_MAX)).
__device__ __forceinline__ uint2 kv_quant8(const float* f, float a, float* scale) {
  *scale = __fdiv_rn(a, 448.0f);
  const float rr = fminf(__fdiv_rn(448.0f, a), FLT_MAX);
  uint32_t p[2];
#pragma unroll
  for (int i = 0; i < 2; ++i)
    p[i] = f8_pack2(__fmul_rn(f[4 * i], rr), __fmul_rn(f[4 * i + 1], rr)) |
           f8_pack2(__fmul_rn(f[4 * i + 2], rr), __fmul_rn(f[4 * i + 3], rr)) << 16;
  return make_uint2(p[0], p[1]);
}

}  // namespace cb
