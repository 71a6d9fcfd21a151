// cambrian_b200 — AdamW with 8-bit block-wise quantised moments (TrainEngine(optim="adamw_bnb_8bit")).
//
// Format (cambrian_b200/adam8bit.py owns it on the host): blocks of 256 consecutive elements of one parameter; the first
// moment m is coded against the signed dynamic map, the second moment v against the unsigned one, and each block keeps
// one fp32 scale per moment, absmax = max |x| over the block.  Dequantisation: map[code] * absmax, one rounding.
// Quantisation: code = the entry nearest x * (1 / absmax), i.e. the first entry >= that value or the one before it,
// whichever is closer in fp32, the larger on a tie; an all-zero block stores the code of 0.0.
//
// One warp owns one block: lane l holds elements 8l .. 8l + 7 as one 8-element AdamW group with adamw_kernel's arithmetic
// (adamw.cuh), fed the dequantised moments.  The updated m and v stay in registers through the block's absmax (a warp
// max) and are requantised by a binary search over the two maps, which sit in shared memory.  No atomics and no
// communication between warps: the result is the same from run to run and does not depend on the launch shape.
//
//   adamw8_kernel<1>   device state, full-occupancy launch                                 (cb_adamw8)
//   adamw8_kernel<2>   two blocks per warp with every load issued first: the background launch on device state
//                      (cb_adamw8, background = 1) and state in registered host memory (cb_adamw8_host)
#include "adamw.cuh"
#include <algorithm>

namespace cb {

constexpr int A8_BLOCK = 256;
constexpr uint32_t A8_SIGNED_ZERO = 127;   // index of 0.0 in the signed map; the unsigned map starts with 0.0

// bitsandbytes create_dynamic_map(signed=True): 0, 1.0 and +-10^(i-6) * (midpoints of linspace(0.1, 1, 2^i + 1)),
// i = 0..6, in fp32, sorted (nf4.cu's c_dmap)
__constant__ float c_a8_signed[256] = {
    -0x1.fc6666p-1f, -0x1.f53334p-1f, -0x1.eep-1f, -0x1.e6ccccp-1f, -0x1.df999ap-1f, -0x1.d86666p-1f, -0x1.d13334p-1f,
    -0x1.cap-1f, -0x1.c2ccccp-1f, -0x1.bb999ap-1f, -0x1.b46666p-1f, -0x1.ad3334p-1f, -0x1.a6p-1f, -0x1.9eccccp-1f,
    -0x1.97999ap-1f, -0x1.906666p-1f, -0x1.893334p-1f, -0x1.82p-1f, -0x1.7accccp-1f, -0x1.73999ap-1f, -0x1.6c6668p-1f,
    -0x1.653334p-1f, -0x1.5ep-1f, -0x1.56ccccp-1f, -0x1.4f999ap-1f, -0x1.486668p-1f, -0x1.413334p-1f, -0x1.3ap-1f,
    -0x1.32ccccp-1f, -0x1.2b999ap-1f, -0x1.246668p-1f, -0x1.1d3334p-1f, -0x1.16p-1f, -0x1.0eccccp-1f, -0x1.079998p-1f,
    -0x1.006666p-1f, -0x1.f26664p-2f, -0x1.e4p-2f, -0x1.d59998p-2f, -0x1.c73334p-2f, -0x1.b8ccccp-2f, -0x1.aa6666p-2f,
    -0x1.9cp-2f, -0x1.8d9998p-2f, -0x1.7f3334p-2f, -0x1.70ccccp-2f, -0x1.626666p-2f, -0x1.54p-2f, -0x1.459998p-2f,
    -0x1.373334p-2f, -0x1.28ccccp-2f, -0x1.1a6668p-2f, -0x1.0cp-2f, -0x1.fb3332p-3f, -0x1.de6666p-3f, -0x1.c1999ap-3f,
    -0x1.a4ccccp-3f, -0x1.88p-3f, -0x1.6b3334p-3f, -0x1.4e6666p-3f, -0x1.31999ap-3f, -0x1.14ccccp-3f, -0x1.fp-4f,
    -0x1.b66668p-4f, -0x1.93d70ap-4f, -0x1.8851eep-4f, -0x1.7ccccep-4f, -0x1.7147aep-4f, -0x1.65c29p-4f, -0x1.5a3d7p-4f,
    -0x1.4eb854p-4f, -0x1.433334p-4f, -0x1.37ae14p-4f, -0x1.2c28f6p-4f, -0x1.20a3d6p-4f, -0x1.151ebap-4f,
    -0x1.09999ap-4f, -0x1.fc28f6p-5f, -0x1.e51ebap-5f, -0x1.ce147ap-5f, -0x1.b70a3ep-5f, -0x1.ap-5f, -0x1.88f5c2p-5f,
    -0x1.71eb86p-5f, -0x1.5ae146p-5f, -0x1.43d70ap-5f, -0x1.2ccccep-5f, -0x1.15c29p-5f, -0x1.fd70a4p-6f,
    -0x1.cf5c2ap-6f, -0x1.a147aep-6f, -0x1.733334p-6f, -0x1.451ebap-6f, -0x1.170a3ep-6f, -0x1.d1eb86p-7f,
    -0x1.75c29p-7f, -0x1.3e76c8p-7f, -0x1.2c083p-7f, -0x1.19999ap-7f, -0x1.072b02p-7f, -0x1.e978d4p-8f, -0x1.c49ba6p-8f,
    -0x1.9fbe76p-8f, -0x1.7ae148p-8f, -0x1.56041ap-8f, -0x1.3126e8p-8f, -0x1.0c49bap-8f, -0x1.ced914p-9f,
    -0x1.851eb8p-9f, -0x1.3b645ap-9f, -0x1.e353f8p-10f, -0x1.4fdf3ap-10f, -0x1.eecbfep-11f, -0x1.b3d07cp-11f,
    -0x1.78d5p-11f, -0x1.3dd982p-11f, -0x1.02de02p-11f, -0x1.8fc506p-12f, -0x1.19ce0ap-12f, -0x1.47ae16p-13f,
    -0x1.743e96p-14f, -0x1.15df66p-14f, -0x1.6f0068p-15f, -0x1.64840cp-16f, -0x1.040bfep-17f, -0x1.b43528p-19f,
    -0x1.27476ep-21f, 0x0p+0f, 0x1.27476ep-21f, 0x1.b43528p-19f, 0x1.040bfep-17f, 0x1.64840cp-16f, 0x1.6f0068p-15f,
    0x1.15df66p-14f, 0x1.743e96p-14f, 0x1.47ae16p-13f, 0x1.19ce0ap-12f, 0x1.8fc506p-12f, 0x1.02de02p-11f,
    0x1.3dd982p-11f, 0x1.78d5p-11f, 0x1.b3d07cp-11f, 0x1.eecbfep-11f, 0x1.4fdf3ap-10f, 0x1.e353f8p-10f, 0x1.3b645ap-9f,
    0x1.851eb8p-9f, 0x1.ced914p-9f, 0x1.0c49bap-8f, 0x1.3126e8p-8f, 0x1.56041ap-8f, 0x1.7ae148p-8f, 0x1.9fbe76p-8f,
    0x1.c49ba6p-8f, 0x1.e978d4p-8f, 0x1.072b02p-7f, 0x1.19999ap-7f, 0x1.2c083p-7f, 0x1.3e76c8p-7f, 0x1.75c29p-7f,
    0x1.d1eb86p-7f, 0x1.170a3ep-6f, 0x1.451ebap-6f, 0x1.733334p-6f, 0x1.a147aep-6f, 0x1.cf5c2ap-6f, 0x1.fd70a4p-6f,
    0x1.15c29p-5f, 0x1.2ccccep-5f, 0x1.43d70ap-5f, 0x1.5ae146p-5f, 0x1.71eb86p-5f, 0x1.88f5c2p-5f, 0x1.ap-5f,
    0x1.b70a3ep-5f, 0x1.ce147ap-5f, 0x1.e51ebap-5f, 0x1.fc28f6p-5f, 0x1.09999ap-4f, 0x1.151ebap-4f, 0x1.20a3d6p-4f,
    0x1.2c28f6p-4f, 0x1.37ae14p-4f, 0x1.433334p-4f, 0x1.4eb854p-4f, 0x1.5a3d7p-4f, 0x1.65c29p-4f, 0x1.7147aep-4f,
    0x1.7ccccep-4f, 0x1.8851eep-4f, 0x1.93d70ap-4f, 0x1.b66668p-4f, 0x1.fp-4f, 0x1.14ccccp-3f, 0x1.31999ap-3f,
    0x1.4e6666p-3f, 0x1.6b3334p-3f, 0x1.88p-3f, 0x1.a4ccccp-3f, 0x1.c1999ap-3f, 0x1.de6666p-3f, 0x1.fb3332p-3f,
    0x1.0cp-2f, 0x1.1a6668p-2f, 0x1.28ccccp-2f, 0x1.373334p-2f, 0x1.459998p-2f, 0x1.54p-2f, 0x1.626666p-2f,
    0x1.70ccccp-2f, 0x1.7f3334p-2f, 0x1.8d9998p-2f, 0x1.9cp-2f, 0x1.aa6666p-2f, 0x1.b8ccccp-2f, 0x1.c73334p-2f,
    0x1.d59998p-2f, 0x1.e4p-2f, 0x1.f26664p-2f, 0x1.006666p-1f, 0x1.079998p-1f, 0x1.0eccccp-1f, 0x1.16p-1f,
    0x1.1d3334p-1f, 0x1.246668p-1f, 0x1.2b999ap-1f, 0x1.32ccccp-1f, 0x1.3ap-1f, 0x1.413334p-1f, 0x1.486668p-1f,
    0x1.4f999ap-1f, 0x1.56ccccp-1f, 0x1.5ep-1f, 0x1.653334p-1f, 0x1.6c6668p-1f, 0x1.73999ap-1f, 0x1.7accccp-1f,
    0x1.82p-1f, 0x1.893334p-1f, 0x1.906666p-1f, 0x1.97999ap-1f, 0x1.9eccccp-1f, 0x1.a6p-1f, 0x1.ad3334p-1f,
    0x1.b46666p-1f, 0x1.bb999ap-1f, 0x1.c2ccccp-1f, 0x1.cap-1f, 0x1.d13334p-1f, 0x1.d86666p-1f, 0x1.df999ap-1f,
    0x1.e6ccccp-1f, 0x1.eep-1f, 0x1.f53334p-1f, 0x1.fc6666p-1f, 0x1p+0f,
};

// bitsandbytes create_dynamic_map(signed=False): 0, 1.0 and 10^(i-6) * (midpoints of linspace(0.1, 1, 2^(i+1) + 1)),
// i = 0..6, in fp32, sorted
__constant__ float c_a8_unsigned[256] = {
    0x0p+0f, 0x1.5cf754p-22f, 0x1.a0133p-21f, 0x1.1d367p-19f, 0x1.2599ecp-18f, 0x1.bc98a2p-18f, 0x1.29cbaap-17f,
    0x1.0624dcp-16f, 0x1.c2e34p-16f, 0x1.3fd0dp-15f, 0x1.9e3p-15f, 0x1.fc8f34p-15f, 0x1.2d7732p-14f, 0x1.5ca6c8p-14f,
    0x1.8bd662p-14f, 0x1.0cb296p-13f, 0x1.82a994p-13f, 0x1.f8a092p-13f, 0x1.374bc8p-12f, 0x1.724744p-12f,
    0x1.ad42c6p-12f, 0x1.e83e44p-12f, 0x1.119ce2p-11f, 0x1.2f1aap-11f, 0x1.4c986p-11f, 0x1.6a162p-11f, 0x1.8793dep-11f,
    0x1.a511ap-11f, 0x1.c28f5ep-11f, 0x1.e00d1cp-11f, 0x1.fd8adcp-11f, 0x1.2b020cp-10f, 0x1.74bc6ap-10f,
    0x1.be76c8p-10f, 0x1.041894p-9f, 0x1.28f5c2p-9f, 0x1.4dd2fp-9f, 0x1.72b02p-9f, 0x1.978d4ep-9f, 0x1.bc6a8p-9f,
    0x1.e147aep-9f, 0x1.03126ep-8f, 0x1.158104p-8f, 0x1.27ef9ep-8f, 0x1.3a5e34p-8f, 0x1.4cccccp-8f, 0x1.5f3b64p-8f,
    0x1.71a9fap-8f, 0x1.841894p-8f, 0x1.96872ap-8f, 0x1.a8f5c2p-8f, 0x1.bb645cp-8f, 0x1.cdd2fp-8f, 0x1.e0418ap-8f,
    0x1.f2b01ep-8f, 0x1.028f5cp-7f, 0x1.0bc6a8p-7f, 0x1.14fdf2p-7f, 0x1.1e354p-7f, 0x1.276c8ap-7f, 0x1.30a3d6p-7f,
    0x1.39db24p-7f, 0x1.43126ep-7f, 0x1.5eb854p-7f, 0x1.8ccccep-7f, 0x1.bae146p-7f, 0x1.e8f5c4p-7f, 0x1.0b851ep-6f,
    0x1.228f5ep-6f, 0x1.39999ap-6f, 0x1.50a3d6p-6f, 0x1.67ae16p-6f, 0x1.7eb852p-6f, 0x1.95c28ep-6f, 0x1.accccep-6f,
    0x1.c3d70ep-6f, 0x1.dae146p-6f, 0x1.f1eb86p-6f, 0x1.047aep-5f, 0x1.1p-5f, 0x1.1b851ep-5f, 0x1.270a3ep-5f,
    0x1.328f5ep-5f, 0x1.3e147ap-5f, 0x1.49999ap-5f, 0x1.551eb8p-5f, 0x1.60a3d6p-5f, 0x1.6c28f6p-5f, 0x1.77ae14p-5f,
    0x1.833334p-5f, 0x1.8eb85p-5f, 0x1.9a3d7p-5f, 0x1.a5c28ep-5f, 0x1.b147aep-5f, 0x1.bccccep-5f, 0x1.c851eep-5f,
    0x1.d3d70ep-5f, 0x1.df5c2ap-5f, 0x1.eae146p-5f, 0x1.f66666p-5f, 0x1.00f5c4p-4f, 0x1.06b854p-4f, 0x1.0c7ae2p-4f,
    0x1.123d7p-4f, 0x1.18p-4f, 0x1.1dc29p-4f, 0x1.23852p-4f, 0x1.2947aep-4f, 0x1.2f0a3ep-4f, 0x1.34cccep-4f,
    0x1.3a8f5ep-4f, 0x1.4051ecp-4f, 0x1.46147cp-4f, 0x1.4bd70ap-4f, 0x1.51999ap-4f, 0x1.575c2ap-4f, 0x1.5d1eb8p-4f,
    0x1.62e148p-4f, 0x1.68a3d6p-4f, 0x1.6e6666p-4f, 0x1.7428f6p-4f, 0x1.79eb86p-4f, 0x1.7fae16p-4f, 0x1.8570a4p-4f,
    0x1.8b3334p-4f, 0x1.90f5c4p-4f, 0x1.96b852p-4f, 0x1.a8p-4f, 0x1.c4ccccp-4f, 0x1.e1999ap-4f, 0x1.fe6666p-4f,
    0x1.0d9998p-3f, 0x1.1cp-3f, 0x1.2a6668p-3f, 0x1.38ccccp-3f, 0x1.473334p-3f, 0x1.559998p-3f, 0x1.64p-3f,
    0x1.726668p-3f, 0x1.80ccccp-3f, 0x1.8f3334p-3f, 0x1.9d9998p-3f, 0x1.acp-3f, 0x1.ba6668p-3f, 0x1.c8ccccp-3f,
    0x1.d73334p-3f, 0x1.e59998p-3f, 0x1.f4p-3f, 0x1.013332p-2f, 0x1.086666p-2f, 0x1.0f999ap-2f, 0x1.16ccccp-2f,
    0x1.1ep-2f, 0x1.253334p-2f, 0x1.2c6666p-2f, 0x1.339998p-2f, 0x1.3accccp-2f, 0x1.42p-2f, 0x1.493334p-2f,
    0x1.506666p-2f, 0x1.579998p-2f, 0x1.5eccccp-2f, 0x1.66p-2f, 0x1.6d3334p-2f, 0x1.746666p-2f, 0x1.7b9998p-2f,
    0x1.82ccccp-2f, 0x1.8ap-2f, 0x1.913334p-2f, 0x1.986666p-2f, 0x1.9f9998p-2f, 0x1.a6ccccp-2f, 0x1.aep-2f,
    0x1.b53334p-2f, 0x1.bc6666p-2f, 0x1.c39998p-2f, 0x1.caccccp-2f, 0x1.d2p-2f, 0x1.d93334p-2f, 0x1.e06666p-2f,
    0x1.e79998p-2f, 0x1.eeccccp-2f, 0x1.f6p-2f, 0x1.fd3332p-2f, 0x1.023334p-1f, 0x1.05ccccp-1f, 0x1.096666p-1f,
    0x1.0dp-1f, 0x1.109998p-1f, 0x1.143334p-1f, 0x1.17ccccp-1f, 0x1.1b6668p-1f, 0x1.1fp-1f, 0x1.22999ap-1f,
    0x1.263334p-1f, 0x1.29ccccp-1f, 0x1.2d6668p-1f, 0x1.31p-1f, 0x1.34999ap-1f, 0x1.383334p-1f, 0x1.3bccccp-1f,
    0x1.3f6668p-1f, 0x1.43p-1f, 0x1.46999ap-1f, 0x1.4a3334p-1f, 0x1.4dccccp-1f, 0x1.516668p-1f, 0x1.55p-1f,
    0x1.58999ap-1f, 0x1.5c3334p-1f, 0x1.5fccccp-1f, 0x1.636668p-1f, 0x1.67p-1f, 0x1.6a999ap-1f, 0x1.6e3334p-1f,
    0x1.71ccccp-1f, 0x1.756668p-1f, 0x1.79p-1f, 0x1.7c999ap-1f, 0x1.803334p-1f, 0x1.83ccccp-1f, 0x1.876668p-1f,
    0x1.8bp-1f, 0x1.8e9998p-1f, 0x1.923334p-1f, 0x1.95ccccp-1f, 0x1.996668p-1f, 0x1.9dp-1f, 0x1.a09998p-1f,
    0x1.a43334p-1f, 0x1.a7ccccp-1f, 0x1.ab6668p-1f, 0x1.afp-1f, 0x1.b29998p-1f, 0x1.b63334p-1f, 0x1.b9ccccp-1f,
    0x1.bd6668p-1f, 0x1.c1p-1f, 0x1.c49998p-1f, 0x1.c83334p-1f, 0x1.cbccccp-1f, 0x1.cf6668p-1f, 0x1.d3p-1f,
    0x1.d69998p-1f, 0x1.da3334p-1f, 0x1.ddccccp-1f, 0x1.e16668p-1f, 0x1.e5p-1f, 0x1.e89998p-1f, 0x1.ec3334p-1f,
    0x1.efccccp-1f, 0x1.f36668p-1f, 0x1.f7p-1f, 0x1.fa9998p-1f, 0x1.fe3334p-1f, 0x1p+0f,
};

// the code of x: the first of the 256 sorted entries >= x, or the one before it, whichever is closer (the larger on a
// tie).  j counts the entries below x and stops at 255, so x above the last entry also gets 255.
__device__ __forceinline__ uint32_t a8_code(const float* map, float x) {
  int j = 0;
#pragma unroll
  for (int s = 128; s > 0; s >>= 1)
    if (map[j + s - 1] < x) j += s;
  if (j == 0) return 0u;
  return __fsub_rn(map[j], x) <= __fsub_rn(x, map[j - 1]) ? (uint32_t)j : (uint32_t)(j - 1);
}

// 8 values of one block with scale `absmax` -> 8 codes, element 0 in the lowest byte
__device__ __forceinline__ uint2 a8_quant8(const float* map, const float* f, float absmax, uint32_t zero_code) {
  const float inv = __fdiv_rn(1.f, absmax);
  uint32_t w[2] = {0u, 0u};
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const uint32_t c = absmax > 0.f ? a8_code(map, __fmul_rn(f[e], inv)) : zero_code;
    w[e >> 2] |= c << (8 * (e & 3));
  }
  return make_uint2(w[0], w[1]);
}

__device__ __forceinline__ void a8_dequant8(const float* map, uint2 c, float absmax, float* f) {
#pragma unroll
  for (int e = 0; e < 8; ++e) f[e] = __fmul_rn(map[((e < 4 ? c.x : c.y) >> (8 * (e & 3))) & 0xffu], absmax);
}

// p, qm, qv, sm, sv: master, codes and scales (device addresses, possibly of mapped host memory); n % 8 == 0, the last
// block may be partial.  G blocks per warp and iteration: block k of a warp sits k x (warps per CTA) blocks after its first.
template <int G>
__global__ void __launch_bounds__(G == 1 ? 256 : 128, G == 1 ? 1 : 7)
    adamw8_kernel(float* __restrict__ p, uint8_t* __restrict__ qm, uint8_t* __restrict__ qv, float* __restrict__ sm,
                  float* __restrict__ sv, const bf16* __restrict__ g, bf16* __restrict__ p16, long long n, float lr,
                  float b1, float b2, float eps, float wd, float bc1, float bc2, float grad_scale,
                  const float* __restrict__ coef) {
  __shared__ float smap[256], umap[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) smap[i] = c_a8_signed[i], umap[i] = c_a8_unsigned[i];
  __syncthreads();
  const AdamwScalars s = adamw_scalars(lr, wd, bc1, bc2, grad_scale, coef);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
  const long long nvec = n >> 3, nb = (n + A8_BLOCK - 1) / A8_BLOCK;
  const long long stride = (long long)gridDim.x * G * warps;
  for (long long b0 = (long long)blockIdx.x * G * warps + warp; b0 < nb; b0 += stride) {   // warp-uniform trip count
    float pf[G][8], am[G], av[G];
    uint2 cm[G], cv[G];
#pragma unroll
    for (int k = 0; k < G; ++k) {                    // every state read of this iteration is issued here
      const long long b = b0 + (long long)k * warps, i = b * 32 + lane;
      am[k] = av[k] = 0.f;
      cm[k] = cv[k] = make_uint2(0u, 0u);            // pf[k] is read only where it was loaded
      if (b < nb) {
        am[k] = sm[b], av[k] = sv[b];
        if (i < nvec) {
          const float4* pp = reinterpret_cast<const float4*>(p) + 2 * i;
          *reinterpret_cast<float4*>(pf[k]) = pp[0]; *reinterpret_cast<float4*>(pf[k] + 4) = pp[1];
          cm[k] = reinterpret_cast<const uint2*>(qm)[i], cv[k] = reinterpret_cast<const uint2*>(qv)[i];
        }
      }
    }
#pragma unroll
    for (int k = 0; k < G; ++k) {
      const long long b = b0 + (long long)k * warps, i = b * 32 + lane;
      if (b >= nb) break;                            // warp-uniform
      const bool valid = i < nvec;
      float mf[8], vf[8];
      a8_dequant8(smap, cm[k], am[k], mf);
      a8_dequant8(umap, cv[k], av[k], vf);
      if (valid) {
        float gf[8];
        unpack8(ldg_nc(reinterpret_cast<const uint4*>(g) + i), gf);
        adamw_update8(gf, pf[k], mf, vf, b1, b2, eps, s);
        float4* pp = reinterpret_cast<float4*>(p) + 2 * i;
        pp[0] = *reinterpret_cast<float4*>(pf[k]); pp[1] = *reinterpret_cast<float4*>(pf[k] + 4);
        reinterpret_cast<uint4*>(p16)[i] = pack8(pf[k]);
      }
      float mx = 0.f, vx = 0.f;
      if (valid) {
#pragma unroll
        for (int e = 0; e < 8; ++e) mx = fmaxf(mx, fabsf(mf[e])), vx = fmaxf(vx, fabsf(vf[e]));
      }
      mx = warp_max(mx);                             // the new block scales: every lane has read the old ones
      vx = warp_max(vx);
      if (valid) {
        reinterpret_cast<uint2*>(qm)[i] = a8_quant8(smap, mf, mx, A8_SIGNED_ZERO);
        reinterpret_cast<uint2*>(qv)[i] = a8_quant8(umap, vf, vx, 0u);
      }
      if (lane == 0) sm[b] = mx, sv[b] = vx;
    }
  }
}

// ------------------------------------------------------------------------------------------ host
static int adamw8_check(const char* op, float* p, void* qm, void* qv, float* sm, float* sv, const void* g, void* p16,
                        long long n, int step) {
  CB_CHECK_ARG(n >= 0 && n % 8 == 0, "%s: element count must be a non-negative multiple of 8 (got %lld)", op, n);
  CB_CHECK_ARG(step >= 1, "%s: step must be >= 1", op);
  if (n == 0) return CB_OK;
  const struct { const void* ptr; const char* name; int align; } args[] = {
      {p, "p", 16}, {qm, "qm", 8}, {qv, "qv", 8}, {sm, "sm", 4}, {sv, "sv", 4}, {g, "g", 16}, {p16, "p16", 16}};
  for (const auto& a : args) {
    CB_CHECK_ARG(a.ptr != nullptr, "%s: %s is null", op, a.name);
    CB_CHECK_ARG(reinterpret_cast<uintptr_t>(a.ptr) % a.align == 0, "%s: %s must be %d-byte aligned", op, a.name, a.align);
  }
  return CB_OK;
}

static int adamw8_run(int G, int threads, int grid, float* p, void* qm, void* qv, float* sm, float* sv, const void* g,
                      void* p16, long long n, float lr, float b1, float b2, float eps, float wd, int step,
                      float grad_scale, const float* clip_coef, cudaStream_t st) {
  const float bc1 = 1.f - powf(b1, (float)step), bc2 = 1.f - powf(b2, (float)step);   // as adamw_launch
  if (G == 1)
    adamw8_kernel<1><<<grid, threads, 0, st>>>(p, (uint8_t*)qm, (uint8_t*)qv, sm, sv, (const bf16*)g, (bf16*)p16, n, lr,
                                               b1, b2, eps, wd, bc1, bc2, grad_scale, clip_coef);
  else
    adamw8_kernel<2><<<grid, threads, 0, st>>>(p, (uint8_t*)qm, (uint8_t*)qv, sm, sv, (const bf16*)g, (bf16*)p16, n, lr,
                                               b1, b2, eps, wd, bc1, bc2, grad_scale, clip_coef);
  CB_CUDA_LAUNCH_CHECK("adamw8");
  return CB_OK;
}

static bool a8_carveout_set[64] = {false};

// background != 0: one 128-thread block per SM, two blocks per warp in flight, as adamw_launch's background shape: the
// update runs next to a resident persistent GEMM CTA instead of taking every thread slot of the SM.
int adamw8_launch(float* p, void* qm, void* qv, float* sm, float* sv, const void* g, void* p16, long long n, float lr,
                  float b1, float b2, float eps, float wd, int step, float grad_scale, const float* clip_coef,
                  int background, cudaStream_t st) {
  int rc = adamw8_check("adamw8", p, qm, qv, sm, sv, g, p16, n, step);
  if (rc != CB_OK || n == 0) return rc;
  const long long nb = (n + A8_BLOCK - 1) / A8_BLOCK;
  if (background) {
    if ((rc = prefer_max_shared_carveout(adamw8_kernel<2>, a8_carveout_set, "adamw8")) != CB_OK) return rc;
    const int grid = (int)std::min<long long>((nb + 7) / 8, device_sm_count());
    return adamw8_run(2, 128, grid, p, qm, qv, sm, sv, g, p16, n, lr, b1, b2, eps, wd, step, grad_scale, clip_coef, st);
  }
  const int grid = (int)std::min<long long>((nb + 7) / 8, 8LL * device_sm_count());
  return adamw8_run(1, 256, grid, p, qm, qv, sm, sv, g, p16, n, lr, b1, b2, eps, wd, step, grad_scale, clip_coef, st);
}

// Default grid: one 128-thread block per SM, the background shape, which fits beside a resident GEMM CTA.  The fp32
// offload kernel's 4 blocks are far too few here: each warp spends most of a block's time on the requantisation, not
// waiting on PCIe, so more warps must have loads in flight (tools/adam8bit_step.py --kernel sweeps ctas).

int adamw8_host_launch(float* p, void* qm, void* qv, float* sm, float* sv, const void* g, void* p16, long long n,
                       float lr, float b1, float b2, float eps, float wd, int step, float grad_scale,
                       const float* clip_coef, int ctas, cudaStream_t st) {
  CB_CHECK_ARG(ctas >= 0, "adamw8_host: ctas must be >= 0 (0 = default), got %d", ctas);
  int rc = adamw8_check("adamw8_host", p, qm, qv, sm, sv, g, p16, n, step);
  if (rc != CB_OK || n == 0) return rc;
  // every pointer is checked before anything is launched: a misplaced operand is an error code, not a GPU fault
  const long long nb = (n + A8_BLOCK - 1) / A8_BLOCK;
  void *pd = nullptr, *qmd = nullptr, *qvd = nullptr, *smd = nullptr, *svd = nullptr;
  if ((rc = host_state_pointer(p, 4 * n, "adamw8_host", "p", &pd)) != CB_OK) return rc;
  if ((rc = host_state_pointer(qm, n, "adamw8_host", "qm", &qmd)) != CB_OK) return rc;
  if ((rc = host_state_pointer(qv, n, "adamw8_host", "qv", &qvd)) != CB_OK) return rc;
  if ((rc = host_state_pointer(sm, 4 * nb, "adamw8_host", "sm", &smd)) != CB_OK) return rc;
  if ((rc = host_state_pointer(sv, 4 * nb, "adamw8_host", "sv", &svd)) != CB_OK) return rc;
  if ((rc = device_pointer(g, "adamw8_host", "g")) != CB_OK) return rc;
  if ((rc = device_pointer(p16, "adamw8_host", "p16")) != CB_OK) return rc;
  if (clip_coef && (rc = device_pointer(clip_coef, "adamw8_host", "clip_coef")) != CB_OK) return rc;
  if ((rc = prefer_max_shared_carveout(adamw8_kernel<2>, a8_carveout_set, "adamw8_host")) != CB_OK) return rc;
  const int grid = (int)std::min<long long>(ctas > 0 ? ctas : device_sm_count(), (nb + 7) / 8);
  return adamw8_run(2, 128, grid, (float*)pd, qmd, qvd, (float*)smd, (float*)svd, g, p16, n, lr, b1, b2, eps, wd, step,
                    grad_scale, clip_coef, st);
}

}  // namespace cb
