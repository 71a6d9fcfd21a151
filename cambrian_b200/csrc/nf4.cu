// cambrian_b200 — 4-bit NF4 decoder weights with double-quantised scales (`load_4bit`, model/builder.py:37-44).
//
// Format (cambrian_b200/quant.py owns it on the host): blocks of 64 consecutive row-major elements of one HF Linear weight
// W [N, K]; 4-bit codes into the NF4 table, element 2j in the HIGH nibble of byte j; the fp32 block absmax is itself
// quantised to 8 bits against the signed dynamic map, in groups of 256 blocks around the tensor's mean absmax (`offset`).
// Dequantisation, shared by every kernel: absmax_b = map[q_b] * absmax2_g + offset (two roundings, no FMA),
// w~ = bf16(c[code] * absmax_b).
//
//   nf4_codes_kernel / nf4_offset_kernel / nf4_scales_kernel   the quantiser (cb_nf4_quantize), three stream-ordered passes
//   gemv_nf4_kernel<M>                                          decode projections, M <= 8 rows (cb_gemv_nf4)
//   nf4_dequant_kernel                                          W~ in bf16 for the GEMM of larger batches (cb_nf4_dequant)
#include "common.cuh"

namespace cb {

constexpr int NF4_BLOCK = 64;
constexpr int NF4_GROUP = 256;
constexpr int NF4_MAP_ZERO = 127;   // index of 0.0 in the sorted dynamic map
constexpr int NF4_MAX_SEGS = 3;

__constant__ float c_nf4[16] = {
    -1.0f, -0.6961928009986877f, -0.5250730514526367f, -0.39491748809814453f, -0.28444138169288635f,
    -0.18477343022823334f, -0.09105003625154495f, 0.0f, 0.07958029955625534f, 0.16093020141124725f,
    0.24611230194568634f, 0.33791524171829224f, 0.44070982933044434f, 0.5626170039176941f, 0.7229568362236023f, 1.0f};

// bitsandbytes create_dynamic_map(signed=True): 0, 1.0 and +-10^(i-6) * (midpoints of linspace(0.1, 1, 2^i + 1)),
// i = 0..6, in fp32, sorted
__constant__ float c_dmap[256] = {
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

// one row segment of a fused projection: rows [row0, next row0) were quantised as their own tensor
struct Nf4Seg {
  const uint8_t* packed;
  const uint8_t* q;
  const float* a2;
  const float* off;
  int row0;
};
struct Nf4Segs {
  Nf4Seg s[NF4_MAX_SEGS];
  int n;
};

__device__ __forceinline__ Nf4Seg seg_of(const Nf4Segs& t, int row) {
  Nf4Seg g = t.s[0];
  if (t.n > 1 && row >= t.s[1].row0) g = t.s[1];
  if (t.n > 2 && row >= t.s[2].row0) g = t.s[2];
  return g;
}

__device__ __forceinline__ float nf4_block_scale(const float* dmap, uint32_t q, float a2, float off) {
  return __fadd_rn(__fmul_rn(dmap[q], a2), off);
}

// ---------------------------------------------------------------------------------------------------------------------
// quantiser.  Pass 1: 8 lanes per 64-element block, 8 elements (one 16-byte vector) per lane: block absmax (shuffles),
// codes, one 32-bit store of 8 nibbles per lane.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) nf4_codes_kernel(const bf16* __restrict__ w, long long n8, float* __restrict__ absmax,
                                                        uint32_t* __restrict__ packed) {
  float mid[15];
#pragma unroll
  for (int i = 0; i < 15; ++i) mid[i] = __fmul_rn(__fadd_rn(c_nf4[i], c_nf4[i + 1]), 0.5f);
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long base = (long long)blockIdx.x * blockDim.x; base < n8; base += stride) {  // warp-uniform trip count
    const long long i = base + threadIdx.x;
    const bool valid = i < n8;
    float f[8];
    unpack8(valid ? ldg_nc(w + i * 8) : make_uint4(0u, 0u, 0u, 0u), f);
    float a = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) a = fmaxf(a, fabsf(f[e]));
    a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, 1));
    a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, 2));
    a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, 4));
    if (!valid) continue;
    if ((threadIdx.x & 7) == 0) absmax[i >> 3] = a;
    const float inv = __fdiv_rn(1.0f, a);
    uint32_t out = 0u;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      uint32_t code = 7u;
      if (a > 0.f) {
        const float xv = __fmul_rn(f[e], inv);
        code = 0u;
#pragma unroll
        for (int m = 0; m < 15; ++m) code += (mid[m] < xv) ? 1u : 0u;
      }
      out |= code << ((e >> 1) * 8 + ((e & 1) ? 0 : 4));
    }
    packed[i] = out;
  }
}

// Pass 2: offset = mean of the block absmaxes, one CTA, fixed-order fp64 sum (deterministic), rounded once to fp32.
constexpr int NF4_OFF_THREADS = 1024;
__global__ void __launch_bounds__(NF4_OFF_THREADS) nf4_offset_kernel(const float* __restrict__ absmax, long long nb,
                                                                     float* __restrict__ offset) {
  __shared__ double part[NF4_OFF_THREADS];
  double s = 0.0;
  for (long long i = threadIdx.x; i < nb; i += NF4_OFF_THREADS) s += (double)absmax[i];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int h = NF4_OFF_THREADS / 2; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h) part[threadIdx.x] += part[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) offset[0] = (float)(part[0] / (double)nb);
}

// Pass 3: one CTA per group of 256 blocks: absmax2 = max |absmax - offset|, then the nearest dynamic-map entry per block.
__global__ void __launch_bounds__(NF4_GROUP) nf4_scales_kernel(const float* __restrict__ absmax, long long nb,
                                                               const float* __restrict__ offset, uint8_t* __restrict__ qabsmax,
                                                               float* __restrict__ absmax2) {
  __shared__ float dmap[256];
  __shared__ float wmax[NF4_GROUP / 32];
  dmap[threadIdx.x] = c_dmap[threadIdx.x];
  const long long b = (long long)blockIdx.x * NF4_GROUP + threadIdx.x;
  const bool valid = b < nb;
  const float off = offset[0];
  const float dv = valid ? __fsub_rn(absmax[b], off) : 0.f;
  float m = warp_max(fabsf(dv));
  if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = m;
  __syncthreads();
  m = wmax[0];
#pragma unroll
  for (int i = 1; i < NF4_GROUP / 32; ++i) m = fmaxf(m, wmax[i]);
  if (threadIdx.x == 0) absmax2[blockIdx.x] = m;
  if (!valid) return;
  int q = NF4_MAP_ZERO;
  if (m > 0.f) {
    const float v = __fmul_rn(dv, __fdiv_rn(1.0f, m));
    int lo = 0, hi = 256;  // first entry >= v
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (dmap[mid] < v) lo = mid + 1;
      else hi = mid;
    }
    if (lo == 256) q = 255;
    else if (lo == 0) q = 0;
    else q = (__fsub_rn(dmap[lo], v) <= __fsub_rn(v, dmap[lo - 1])) ? lo : lo - 1;  // tie: the larger entry
  }
  qabsmax[b] = (uint8_t)q;
}

int nf4_quantize_launch(const void* w, int N, int K, float* absmax_ws, long long ws_floats, void* packed, void* qabsmax,
                        float* absmax2, float* offset, cudaStream_t st) {
  CB_CHECK_ARG(N > 0 && K > 0 && K % NF4_BLOCK == 0, "nf4_quantize: K=%d must be a positive multiple of %d (N=%d)", K,
               NF4_BLOCK, N);
  CB_CHECK_ARG(w && absmax_ws && packed && qabsmax && absmax2 && offset, "nf4_quantize: null argument");
  CB_CHECK_ARG(((reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(packed)) & 15u) == 0,
               "nf4_quantize: weight and packed output must be 16-byte aligned");
  const long long nb = (long long)N * K / NF4_BLOCK;
  CB_CHECK_ARG(ws_floats >= nb, "nf4_quantize: workspace holds %lld floats, %lld needed", ws_floats, nb);
  const long long n8 = (long long)N * K / 8;
  const long long want = (n8 + 255) / 256;
  const int grid = (int)(want < 16LL * device_sm_count() ? want : 16LL * device_sm_count());
  nf4_codes_kernel<<<grid, 256, 0, st>>>((const bf16*)w, n8, absmax_ws, (uint32_t*)packed);
  CB_CUDA_LAUNCH_CHECK("nf4_codes");
  nf4_offset_kernel<<<1, NF4_OFF_THREADS, 0, st>>>(absmax_ws, nb, offset);
  CB_CUDA_LAUNCH_CHECK("nf4_offset");
  nf4_scales_kernel<<<(unsigned)((nb + NF4_GROUP - 1) / NF4_GROUP), NF4_GROUP, 0, st>>>(absmax_ws, nb, offset,
                                                                                       (uint8_t*)qabsmax, absmax2);
  CB_CUDA_LAUNCH_CHECK("nf4_scales");
  return CB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// decode GEMV: y[M, N] = x[M, K] W~[N, K]^T (+ bias) (+ residual), M <= 8.
//   block = 8 warps, one warp = 2 output columns; K in chunks of 2048, x chunk staged in smem as fp32;
//   per lane and column: two 16-byte packed vectors per chunk (32 weights each, all in one 64-element block), so the
//   block scale is applied once per vector and row: p = sum c[code] x, acc += scale * p.
//   dequantisation: one LDS.64 of a 256-entry float2 table (c[hi nibble], c[lo nibble]) per packed byte.
//   x layout in smem: element (j, lane, word, e) of the chunk at j*1024 + word*256 + (e/4)*128 + lane*4 + e%4, so the
//   two float4 reads of each 8-weight word are contiguous across the warp (no bank conflicts).
// ---------------------------------------------------------------------------------------------------------------------
constexpr int NG_KC = 2048;
constexpr int NG_CPW = 2;
constexpr int NG_WARPS = 8;

template <int M>
__global__ void __launch_bounds__(NG_WARPS * 32)
gemv_nf4_kernel(const bf16* __restrict__ x, void* __restrict__ y, const bf16* __restrict__ bias,
                const bf16* __restrict__ residual, Nf4Segs segs, int N, int K, long long ldx, long long ldy, long long ldr,
                int out_fp32) {
  extern __shared__ __align__(16) float xs[];  // [M][NG_KC], permuted as described above
  __shared__ float2 lut[256];
  __shared__ float dmap[256];
  {
    const int t = threadIdx.x;
    lut[t] = make_float2(c_nf4[t >> 4], c_nf4[t & 15]);
    dmap[t] = c_dmap[t];
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = (blockIdx.x * NG_WARPS + warp) * NG_CPW;
  const uint4* wp[NG_CPW];
  const uint8_t* qs[NG_CPW];
  long long qb0[NG_CPW];
  const float* a2p[NG_CPW];
  float off[NG_CPW];
#pragma unroll
  for (int c = 0; c < NG_CPW; ++c) {
    const int row = min(n0 + c, N - 1);  // a column past N re-reads row N-1 and is never stored
    const Nf4Seg g = seg_of(segs, row);
    const long long r = row - g.row0;
    wp[c] = reinterpret_cast<const uint4*>(g.packed + r * (K / 2));
    qs[c] = g.q;
    qb0[c] = r * (K / NF4_BLOCK);
    a2p[c] = g.a2;
    off[c] = n0 < N ? g.off[0] : 0.f;
  }
  float acc[NG_CPW][M];
#pragma unroll
  for (int c = 0; c < NG_CPW; ++c)
#pragma unroll
    for (int m = 0; m < M; ++m) acc[c][m] = 0.f;
  for (int k0 = 0; k0 < K; k0 += NG_KC) {
    const int kc = min(NG_KC, K - k0);  // multiple of 64
    __syncthreads();
    for (int i = threadIdx.x; i < M * (NG_KC / 8); i += NG_WARPS * 32) {
      const int m = i / (NG_KC / 8), v = i % (NG_KC / 8);
      float f[8];
      unpack8(v * 8 < kc ? *reinterpret_cast<const uint4*>(x + m * ldx + k0 + v * 8) : make_uint4(0u, 0u, 0u, 0u), f);
      const int k = v * 8;
      float* d = xs + m * NG_KC + (k >> 10) * 1024 + ((k >> 3) & 3) * 256 + ((k >> 5) & 31) * 4;
      *reinterpret_cast<float4*>(d) = make_float4(f[0], f[1], f[2], f[3]);
      *reinterpret_cast<float4*>(d + 128) = make_float4(f[4], f[5], f[6], f[7]);
    }
    __syncthreads();
    if (n0 >= N) continue;
    uint4 wv[NG_CPW][NG_KC / 1024];
    float sc[NG_CPW][NG_KC / 1024];
#pragma unroll
    for (int c = 0; c < NG_CPW; ++c)
#pragma unroll
      for (int j = 0; j < NG_KC / 1024; ++j) {
        const int kk = k0 + j * 1024 + lane * 32;
        const bool ok = kk < k0 + kc;
        wv[c][j] = ok ? ldg_nc(wp[c] + kk / 32) : make_uint4(0u, 0u, 0u, 0u);
        const long long gb = qb0[c] + kk / NF4_BLOCK;
        sc[c][j] = ok ? nf4_block_scale(dmap, qs[c][gb], a2p[c][gb / NF4_GROUP], off[c]) : 0.f;
      }
#pragma unroll
    for (int j = 0; j < NG_KC / 1024; ++j) {
      float p[NG_CPW][M];
#pragma unroll
      for (int c = 0; c < NG_CPW; ++c)
#pragma unroll
        for (int m = 0; m < M; ++m) p[c][m] = 0.f;
#pragma unroll
      for (int wd = 0; wd < 4; ++wd) {
        float wf[NG_CPW][8];
#pragma unroll
        for (int c = 0; c < NG_CPW; ++c) {
          const uint32_t word = (&wv[c][j].x)[wd];
#pragma unroll
          for (int b = 0; b < 4; ++b) {
            const float2 t = lut[(word >> (8 * b)) & 0xffu];
            wf[c][2 * b] = t.x;
            wf[c][2 * b + 1] = t.y;
          }
        }
#pragma unroll
        for (int m = 0; m < M; ++m) {
          const float* xr = xs + m * NG_KC + j * 1024 + wd * 256 + lane * 4;
          const float4 xa = *reinterpret_cast<const float4*>(xr);
          const float4 xb = *reinterpret_cast<const float4*>(xr + 128);
          const float xf[8] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
#pragma unroll
          for (int c = 0; c < NG_CPW; ++c)
#pragma unroll
            for (int e = 0; e < 8; ++e) p[c][m] = fmaf(wf[c][e], xf[e], p[c][m]);
        }
      }
#pragma unroll
      for (int c = 0; c < NG_CPW; ++c)
#pragma unroll
        for (int m = 0; m < M; ++m) acc[c][m] = fmaf(sc[c][j], p[c][m], acc[c][m]);
    }
  }
  if (n0 >= N) return;
#pragma unroll
  for (int c = 0; c < NG_CPW; ++c)
#pragma unroll
    for (int m = 0; m < M; ++m) {
      const float s = warp_sum(acc[c][m]);
      const int n = n0 + c;
      if (lane == 0 && n < N) {
        float v = s;
        if (bias) v += __bfloat162float(bias[n]);
        if (residual) v += __bfloat162float(residual[m * ldr + n]);
        if (out_fp32) reinterpret_cast<float*>(y)[m * ldy + n] = v;
        else reinterpret_cast<bf16*>(y)[m * ldy + n] = __float2bfloat16(v);
      }
    }
}

static int fill_segs(Nf4Segs& t, int N, int K, int nseg, const int* row0, const void* const* packed,
                     const void* const* qabsmax, const void* const* absmax2, const void* const* offset, const char* who) {
  CB_CHECK_ARG(N > 0 && K > 0 && K % NF4_BLOCK == 0, "%s: K=%d must be a positive multiple of %d (N=%d)", who, K,
               NF4_BLOCK, N);
  CB_CHECK_ARG(nseg >= 1 && nseg <= NF4_MAX_SEGS && row0 && packed && qabsmax && absmax2 && offset,
               "%s: nseg=%d must be in [1, %d] with host arrays of segment pointers", who, nseg, NF4_MAX_SEGS);
  CB_CHECK_ARG(row0[0] == 0, "%s: the first segment must start at row 0", who);
  t.n = nseg;
  for (int i = 0; i < NF4_MAX_SEGS; ++i) {
    const int j = i < nseg ? i : nseg - 1;
    CB_CHECK_ARG(packed[j] && qabsmax[j] && absmax2[j] && offset[j], "%s: null pointer in segment %d", who, j);
    CB_CHECK_ARG((reinterpret_cast<uintptr_t>(packed[j]) & 15u) == 0, "%s: packed codes of segment %d not 16-byte aligned",
                 who, j);
    if (i < nseg && i > 0)
      CB_CHECK_ARG(row0[i] > row0[i - 1] && row0[i] < N, "%s: segment rows must increase inside [0, N)", who);
    t.s[i] = Nf4Seg{(const uint8_t*)packed[j], (const uint8_t*)qabsmax[j], (const float*)absmax2[j],
                    (const float*)offset[j], i < nseg ? row0[i] : N};
  }
  return CB_OK;
}

template <int M>
static void gemv_nf4_go(int grid, const bf16* x, void* y, const bf16* bias, const bf16* residual, const Nf4Segs& segs, int N,
                        int K, long long ldx, long long ldy, long long ldr, int out_fp32, cudaStream_t st) {
  const int smem = M * NG_KC * (int)sizeof(float);
  static bool attr = false;  // one-time function-attribute cache (dynamic + 3 KB static smem may pass 48 KB from M = 6)
  if (!attr) {
    cudaFuncSetAttribute(gemv_nf4_kernel<M>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    attr = true;
  }
  gemv_nf4_kernel<M><<<grid, NG_WARPS * 32, smem, st>>>(x, y, bias, residual, segs, N, K, ldx, ldy, ldr, out_fp32);
}

int gemv_nf4_launch(const void* x, void* y, int M, int N, int K, long long ldx, long long ldy, int nseg, const int* row0,
                    const void* const* packed, const void* const* qabsmax, const void* const* absmax2,
                    const void* const* offset, const void* bias, const void* residual, long long ldr, int out_fp32,
                    cudaStream_t st) {
  CB_CHECK_ARG(M >= 1 && M <= 8, "gemv_nf4: M=%d must be in [1, 8]", M);
  Nf4Segs segs;
  const int rc = fill_segs(segs, N, K, nseg, row0, packed, qabsmax, absmax2, offset, "gemv_nf4");
  if (rc != CB_OK) return rc;
  CB_CHECK_ARG(x && y && ldx % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15u) == 0,
               "gemv_nf4: x must be 16-byte aligned with a row stride that is a multiple of 8");
  const int grid = (N + NG_WARPS * NG_CPW - 1) / (NG_WARPS * NG_CPW);
  const bf16 *xp = (const bf16*)x, *bp = (const bf16*)bias, *rp = (const bf16*)residual;
#define CB_NG(MM) gemv_nf4_go<MM>(grid, xp, y, bp, rp, segs, N, K, ldx, ldy, ldr, out_fp32, st)
  switch (M) {
    case 1: CB_NG(1); break;
    case 2: CB_NG(2); break;
    case 3: CB_NG(3); break;
    case 4: CB_NG(4); break;
    case 5: CB_NG(5); break;
    case 6: CB_NG(6); break;
    case 7: CB_NG(7); break;
    default: CB_NG(8); break;
  }
#undef CB_NG
  CB_CUDA_LAUNCH_CHECK("gemv_nf4");
  return CB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// dequantiser: W~ (bf16, row-major [N, K]) of a segmented weight; one 16-byte packed vector (32 weights) per item.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) nf4_dequant_kernel(bf16* __restrict__ out, Nf4Segs segs, int N, int K) {
  __shared__ float code[16];
  __shared__ float dmap[256];
  if (threadIdx.x < 16) code[threadIdx.x] = c_nf4[threadIdx.x];
  dmap[threadIdx.x] = c_dmap[threadIdx.x];
  __syncthreads();
  const int per_row = K / 32;
  const long long items = (long long)N * per_row;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < items; i += (long long)gridDim.x * blockDim.x) {
    const int row = (int)(i / per_row);
    const int kk = (int)(i % per_row) * 32;
    const Nf4Seg g = seg_of(segs, row);
    const long long r = row - g.row0;
    const uint4 u = ldg_nc(g.packed + r * (K / 2) + kk / 2);
    const long long blk = r * (K / NF4_BLOCK) + kk / NF4_BLOCK;
    const float s = nf4_block_scale(dmap, g.q[blk], g.a2[blk / NF4_GROUP], g.off[0]);
    uint4 o[4];
    uint32_t* ow = &o[0].x;
#pragma unroll
    for (int wd = 0; wd < 4; ++wd) {
      const uint32_t word = (&u.x)[wd];
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const uint32_t byte = (word >> (8 * b)) & 0xffu;
        ow[wd * 4 + b] = pack_bf16x2(__fmul_rn(code[byte >> 4], s), __fmul_rn(code[byte & 15u], s));
      }
    }
    uint4* dst = reinterpret_cast<uint4*>(out + (long long)row * K + kk);
#pragma unroll
    for (int v = 0; v < 4; ++v) dst[v] = o[v];
  }
}

int nf4_dequant_launch(void* out, int N, int K, int nseg, const int* row0, const void* const* packed,
                       const void* const* qabsmax, const void* const* absmax2, const void* const* offset, cudaStream_t st) {
  Nf4Segs segs;
  const int rc = fill_segs(segs, N, K, nseg, row0, packed, qabsmax, absmax2, offset, "nf4_dequant");
  if (rc != CB_OK) return rc;
  CB_CHECK_ARG(out && (reinterpret_cast<uintptr_t>(out) & 15u) == 0, "nf4_dequant: output must be 16-byte aligned");
  const long long items = (long long)N * (K / 32);
  const long long want = (items + 255) / 256;
  const int grid = (int)(want < 8LL * device_sm_count() ? want : 8LL * device_sm_count());
  nf4_dequant_kernel<<<grid, 256, 0, st>>>((bf16*)out, segs, N, K);
  CB_CUDA_LAUNCH_CHECK("nf4_dequant");
  return CB_OK;
}

}  // namespace cb
