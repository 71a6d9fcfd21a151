// cambrian_b200 — 8-bit LLM.int8 decoder weights (`load_8bit`, model/builder.py:35-36).
//
// Format and arithmetic (cambrian_b200/quant_int8.py owns them on the host and states them in full):
//   weight W [N, K] bf16 -> cb [N, K] int8 = rint(W * (127 / scb[n])) clamped to +-127, scb[n] = max |W[n, :]| (fp32);
//   activation X [M, K] bf16 -> outlier columns O = { j : max_m |X[m, j]| >= tau } (ascending index list + device count),
//     sca[m] = max |X[m, j]| over j not in O, xq [M, K] int8 = rint(X * (127 / sca[m])) off O, 0 on O;
//   output y[m, n] = (float(acc) * (sca[m] * scb[n])) * (1/16129) + o (+ bias[n]) (+ residual[m, n]), acc = sum xq cb
//     exact in int32, o = sum over j in O, ascending, of x[m, j] * (float(cb[n, j]) * (scb[n] * (1/127))).
// Every product and sum of the epilogue is an _rn intrinsic, so FMA contraction cannot reorder it: the tensor-core GEMM
// and the CUDA-core GEMV produce the same int32 sums and therefore the same bits.
//
//   i8_quant_weight_kernel                          cb_int8_quantize_weight, one CTA per row
//   i8_colmax_kernel / i8_outliers_kernel /
//   i8_quant_act_kernel                             cb_int8_quantize_act, three stream-ordered passes, no host sync
//   gemv_int8_kernel<M>                             decode projections, M <= 8 rows (cb_gemv_int8): dp4a
//   gemm_int8_wgmma                                 M > 8 (cb_gemm_int8): TMA ring + wgmma m64n128k32 .s32.s8.s8
#include "common.cuh"
#include <algorithm>
#include <cstring>
#include <cudaTypedefs.h>
#include <mutex>

namespace cb {

constexpr float I8_INV127 = 0x1.020408p-7f;     // 1/127 rounded to fp32
constexpr float I8_INV16129 = 0x1.040c2p-14f;   // 1/16129 = 1/127^2 rounded to fp32

// ---------------------------------------------------------------------------------------------------------------------
// the epilogue, shared by both matmul kernels
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float i8_main(int acc, float sa, float sb) {
  return __fmul_rn(__fmul_rn(__int2float_rn(acc), __fmul_rn(sa, sb)), I8_INV16129);
}
__device__ __forceinline__ float i8_term(float x, int c, float wsc) { return __fmul_rn(x, __fmul_rn(__int2float_rn(c), wsc)); }
__device__ __forceinline__ float i8_finish(float v, float o, const bf16* bias, const bf16* residual, long long r_off, int n) {
  float y = __fadd_rn(v, o);
  if (bias) y = __fadd_rn(y, __bfloat162float(bias[n]));
  if (residual) y = __fadd_rn(y, __bfloat162float(residual[r_off + n]));
  return y;
}

struct I8Epi {
  const float* sca;     // [M]
  const float* scb;     // [N]
  const bf16* x;        // [M, ldx] the bf16 activation (outlier columns)
  long long ldx;
  const int8_t* cb;     // [N, K]
  const int* oidx;      // ascending outlier columns
  const int* ocnt;      // [1] their number (device)
  void* y;
  long long ldy;
  const bf16* bias;     // [N] or null
  const bf16* residual; // [M, ldr] or null
  long long ldr;
  int out_fp32;
};

__device__ __forceinline__ void i8_store(const I8Epi& ep, int m, int n, float v) {
  if (ep.out_fp32) reinterpret_cast<float*>(ep.y)[m * ep.ldy + n] = v;
  else reinterpret_cast<bf16*>(ep.y)[m * ep.ldy + n] = __float2bfloat16(v);
}

// ---------------------------------------------------------------------------------------------------------------------
// weight quantiser: one CTA per row, 8 elements (one 16-byte vector) per thread and step
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) i8_quant_weight_kernel(const bf16* __restrict__ w, int K, long long ldw,
                                                              int8_t* __restrict__ cb, float* __restrict__ scb) {
  __shared__ float red[8];
  const int n = blockIdx.x;
  const bf16* wr = w + (long long)n * ldw;
  float a = 0.f;
  for (int k = threadIdx.x * 8; k < K; k += 256 * 8) {
    float f[8];
    unpack8(*reinterpret_cast<const uint4*>(wr + k), f);
#pragma unroll
    for (int e = 0; e < 8; ++e) a = fmaxf(a, fabsf(f[e]));
  }
  a = warp_max(a);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = a;
  __syncthreads();
  a = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) a = fmaxf(a, red[i]);
  if (threadIdx.x == 0) scb[n] = a;
  const float s = a > 0.f ? __fdiv_rn(127.0f, a) : 0.f;
  int8_t* cr = cb + (long long)n * K;
  for (int k = threadIdx.x * 8; k < K; k += 256 * 8) {
    float f[8];
    unpack8(*reinterpret_cast<const uint4*>(wr + k), f);
    uint32_t p[2] = {0u, 0u};
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int q = max(-127, min(127, __float2int_rn(__fmul_rn(f[e], s))));
      p[e >> 2] |= (uint32_t)(q & 0xff) << (8 * (e & 3));
    }
    *reinterpret_cast<uint2*>(cr + k) = make_uint2(p[0], p[1]);
  }
}

int int8_quantize_weight_launch(const void* w, int N, int K, long long ldw, void* cb, float* scb, cudaStream_t st) {
  CB_CHECK_ARG(N > 0 && K > 0 && K % 16 == 0, "int8_quantize_weight: K=%d must be a positive multiple of 16 (N=%d)", K, N);
  CB_CHECK_ARG(w && cb && scb && ldw >= K && ldw % 8 == 0, "int8_quantize_weight: null argument or bad row stride");
  CB_CHECK_ARG(((reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(cb)) & 15u) == 0,
               "int8_quantize_weight: weight and cb must be 16-byte aligned");
  i8_quant_weight_kernel<<<N, 256, 0, st>>>((const bf16*)w, K, ldw, (int8_t*)cb, scb);
  CB_CUDA_LAUNCH_CHECK("int8_quantize_weight");
  return CB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// activation quantiser.  Pass 1: column max |x| as float bits (non-negative floats order like their bit patterns), one
// thread per 8 columns and up to 32 rows, atomicMax into a zeroed buffer: the max is exact, so any order gives the same.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int I8_CM_ROWS = 32;
__global__ void __launch_bounds__(128) i8_colmax_kernel(const bf16* __restrict__ x, int M, int K, long long ldx,
                                                        unsigned* __restrict__ colmax) {
  const int k = (blockIdx.x * 128 + threadIdx.x) * 8;
  if (k >= K) return;
  const int m0 = blockIdx.y * I8_CM_ROWS, m1 = min(M, m0 + I8_CM_ROWS);
  float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int m = m0; m < m1; ++m) {
    float f[8];
    unpack8(*reinterpret_cast<const uint4*>(x + m * ldx + k), f);
#pragma unroll
    for (int e = 0; e < 8; ++e) a[e] = fmaxf(a[e], fabsf(f[e]));
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) atomicMax(colmax + k + e, __float_as_uint(a[e]));
}

// Pass 2: one CTA compacts the outlier columns in ascending order (block-wide ballot scan per 1024 columns).
__global__ void __launch_bounds__(1024) i8_outliers_kernel(const unsigned* __restrict__ colmax, int K, float thr,
                                                           int* __restrict__ oidx, int* __restrict__ ocnt) {
  __shared__ int wsum[32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int base = 0;
  for (int k0 = 0; k0 < K; k0 += 1024) {
    const int j = k0 + threadIdx.x;
    const bool out = thr > 0.f && j < K && __uint_as_float(colmax[j]) >= thr;
    const unsigned bal = __ballot_sync(0xffffffffu, out);
    if (lane == 0) wsum[warp] = __popc(bal);
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll 4
    for (int w = 0; w < 32; ++w) {
      const int c = wsum[w];
      before += w < warp ? c : 0;
      total += c;
    }
    if (out) oidx[base + before + __popc(bal & ((1u << lane) - 1u))] = j;
    base += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) ocnt[0] = base;
}

// Pass 3: one CTA per row: sca = max |x| off the outlier columns, then xq.
__global__ void __launch_bounds__(256) i8_quant_act_kernel(const bf16* __restrict__ x, int K, long long ldx,
                                                           const unsigned* __restrict__ colmax, float thr,
                                                           int8_t* __restrict__ xq, float* __restrict__ sca) {
  __shared__ float red[8];
  const int m = blockIdx.x;
  const bf16* xr = x + m * ldx;
  auto outlier = [&](int j) { return thr > 0.f && __uint_as_float(colmax[j]) >= thr; };
  float a = 0.f;
  for (int k = threadIdx.x * 8; k < K; k += 256 * 8) {
    float f[8];
    unpack8(*reinterpret_cast<const uint4*>(xr + k), f);
#pragma unroll
    for (int e = 0; e < 8; ++e)
      if (!outlier(k + e)) a = fmaxf(a, fabsf(f[e]));
  }
  a = warp_max(a);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = a;
  __syncthreads();
  a = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) a = fmaxf(a, red[i]);
  if (threadIdx.x == 0) sca[m] = a;
  const float s = a > 0.f ? __fdiv_rn(127.0f, a) : 0.f;
  int8_t* qr = xq + (long long)m * K;
  for (int k = threadIdx.x * 8; k < K; k += 256 * 8) {
    float f[8];
    unpack8(*reinterpret_cast<const uint4*>(xr + k), f);
    uint32_t p[2] = {0u, 0u};
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int q = outlier(k + e) ? 0 : __float2int_rn(__fmul_rn(f[e], s));
      p[e >> 2] |= (uint32_t)(q & 0xff) << (8 * (e & 3));
    }
    *reinterpret_cast<uint2*>(qr + k) = make_uint2(p[0], p[1]);
  }
}

int int8_quantize_act_launch(const void* x, int M, int K, long long ldx, float threshold, void* xq, float* sca,
                             unsigned* colmax_ws, int* oidx, int* ocnt, cudaStream_t st) {
  CB_CHECK_ARG(M > 0 && K > 0 && K % 16 == 0, "int8_quantize_act: K=%d must be a positive multiple of 16 (M=%d)", K, M);
  CB_CHECK_ARG(x && xq && sca && colmax_ws && oidx && ocnt && ldx >= K && ldx % 8 == 0,
               "int8_quantize_act: null argument or bad row stride");
  CB_CHECK_ARG(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(xq)) & 15u) == 0,
               "int8_quantize_act: x and xq must be 16-byte aligned");
  cudaError_t e = cudaMemsetAsync(colmax_ws, 0, (size_t)K * sizeof(unsigned), st);
  if (e != cudaSuccess) return set_error(CB_ERR_CUDA, "int8_quantize_act memset: %s", cudaGetErrorString(e));
  dim3 g1((K / 8 + 127) / 128, (M + I8_CM_ROWS - 1) / I8_CM_ROWS);
  i8_colmax_kernel<<<g1, 128, 0, st>>>((const bf16*)x, M, K, ldx, colmax_ws);
  CB_CUDA_LAUNCH_CHECK("int8_colmax");
  i8_outliers_kernel<<<1, 1024, 0, st>>>(colmax_ws, K, threshold, oidx, ocnt);
  CB_CUDA_LAUNCH_CHECK("int8_outliers");
  i8_quant_act_kernel<<<M, 256, 0, st>>>((const bf16*)x, K, ldx, colmax_ws, threshold, (int8_t*)xq, sca);
  CB_CUDA_LAUNCH_CHECK("int8_quant_act");
  return CB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// decode GEMV, M <= 8 rows: gemv.cu's layout on int8.  block = 8 warps, one warp = 2 output columns; K in chunks of 4096
// bytes (xq chunk: M x 4 KB of smem); per lane and column eight 16-byte cb vectors in flight, 4 dp4a per vector and row
// into exact int32, one integer shuffle tree per (row, column); the epilogue runs on lane c * M + m.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int IG_KC = 4096;
constexpr int IG_CPW = 2;
constexpr int IG_WARPS = 8;

template <int M>
__global__ void __launch_bounds__(IG_WARPS * 32) gemv_int8_kernel(const int8_t* __restrict__ xq, int N, int K, I8Epi ep) {
  __shared__ __align__(16) int8_t xs[M][IG_KC];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = (blockIdx.x * IG_WARPS + warp) * IG_CPW;
  int acc[IG_CPW][M];
#pragma unroll
  for (int c = 0; c < IG_CPW; ++c)
#pragma unroll
    for (int m = 0; m < M; ++m) acc[c][m] = 0;
  for (int k0 = 0; k0 < K; k0 += IG_KC) {
    const int kc = min(IG_KC, K - k0);  // multiple of 16
    __syncthreads();
    for (int i = threadIdx.x; i < M * (IG_KC / 16); i += IG_WARPS * 32) {
      const int m = i / (IG_KC / 16), v = i % (IG_KC / 16);
      uint4 val = make_uint4(0u, 0u, 0u, 0u);
      if (v * 16 < kc) val = *reinterpret_cast<const uint4*>(xq + (long long)m * K + k0 + v * 16);
      *reinterpret_cast<uint4*>(&xs[m][v * 16]) = val;
    }
    __syncthreads();
    if (n0 >= N) continue;
    uint4 wv[IG_CPW][IG_KC / 512];
#pragma unroll
    for (int c = 0; c < IG_CPW; ++c) {
      const int8_t* wp = ep.cb + (long long)min(n0 + c, N - 1) * K + k0;  // a column past N re-reads row N-1, unused
#pragma unroll
      for (int j = 0; j < IG_KC / 512; ++j) {
        const int off = j * 512 + lane * 16;
        wv[c][j] = off < kc ? ldg_nc(wp + off) : make_uint4(0u, 0u, 0u, 0u);
      }
    }
#pragma unroll
    for (int j = 0; j < IG_KC / 512; ++j)
#pragma unroll
      for (int m = 0; m < M; ++m) {
        const uint4 xv = *reinterpret_cast<const uint4*>(&xs[m][j * 512 + lane * 16]);
#pragma unroll
        for (int c = 0; c < IG_CPW; ++c) {
          int s = acc[c][m];
          s = __dp4a((int)wv[c][j].x, (int)xv.x, s);
          s = __dp4a((int)wv[c][j].y, (int)xv.y, s);
          s = __dp4a((int)wv[c][j].z, (int)xv.z, s);
          s = __dp4a((int)wv[c][j].w, (int)xv.w, s);
          acc[c][m] = s;
        }
      }
  }
  if (n0 >= N) return;
  int mine = 0;
#pragma unroll
  for (int c = 0; c < IG_CPW; ++c)
#pragma unroll
    for (int m = 0; m < M; ++m) {
      int s = acc[c][m];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == c * M + m) mine = s;
    }
  if (lane >= IG_CPW * M) return;
  const int c = lane / M, m = lane % M, n = n0 + c;
  if (n >= N) return;
  const float sb = ep.scb[n];
  const float v = i8_main(mine, ep.sca[m], sb);
  const float wsc = __fmul_rn(sb, I8_INV127);
  const int no = *ep.ocnt;
  const int8_t* cr = ep.cb + (long long)n * K;
  const bf16* xr = ep.x + m * ep.ldx;
  float o = 0.f;
  for (int i = 0; i < no; ++i) {
    const int j = ep.oidx[i];
    o = __fadd_rn(o, i8_term(__bfloat162float(xr[j]), cr[j], wsc));
  }
  i8_store(ep, m, n, i8_finish(v, o, ep.bias, ep.residual, m * ep.ldr, n));
}

// ---------------------------------------------------------------------------------------------------------------------
// GEMM, M > 8: gemm.cu's persistent warp-specialised structure on int8.  288 threads: warp 8 is the TMA producer
// (128 x 128-byte boxes of xq and cb into a 6-stage SWIZZLE_128B ring; one k-block = 128 int8 = one swizzle atom), warps
// 0..7 are two consumer warpgroups of 64 rows issuing wgmma m64n128k32 .s32.s8.s8 (4 per k-block, +32 B on the
// descriptor start each) with one k-block group in flight.  The epilogue works from the s32 registers: the int8 term
// per element, then the outlier term read from L2 (x[m, O] and cb[n, O]), then bias / residual and the store.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int QBM = 128, QBN = 128, QBK = 128;
constexpr int Q_STAGES = 6;
constexpr int Q_A_BYTES = QBM * QBK, Q_B_BYTES = QBN * QBK, Q_STAGE_BYTES = Q_A_BYTES + Q_B_BYTES;
constexpr int Q_SMEM_BYTES = Q_STAGES * Q_STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
static_assert(Q_SMEM_BYTES <= 232448, "exceeds the 227 KB of shared memory a CTA may use");
constexpr int Q_GROUP_M = 16;

__device__ __forceinline__ void i8_reg_fence(int32_t (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

__device__ __forceinline__ void i8_tile_to_mn(int r, int m_blocks, int n_blocks, int& mb, int& nb) {
  const int tpg = Q_GROUP_M * n_blocks;
  const int g = r / tpg;
  const int first = g * Q_GROUP_M;
  const int gs = min(Q_GROUP_M, m_blocks - first);
  const int w = r - g * tpg;
  mb = first + w % gs;
  nb = w / gs;
}

__global__ void __launch_bounds__(288, 1)
gemm_int8_wgmma(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, int M, int N, int K,
                int tiles, I8Epi ep) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + Q_STAGES * Q_STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (Q_STAGES + s); };
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int m_blocks = (M + QBM - 1) / QBM;
  const int n_blocks = (N + QBN - 1) / QBN;
  const int num_kb = (K + QBK - 1) / QBK;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < Q_STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int r = blockIdx.x; r < tiles; r += gridDim.x) {
        int mb, nb;
        i8_tile_to_mn(r, m_blocks, n_blocks, mb, nb);
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(empty_bar(stage), phase ^ 1u);
          const uint32_t sa = smem_base + stage * Q_STAGE_BYTES;
          mbar_arrive_expect_tx(full_bar(stage), Q_STAGE_BYTES);
          tma_load_3d(sa, &tmA, full_bar(stage), kb * QBK, mb * QBM, 0);
          tma_load_3d(sa + Q_A_BYTES, &tmB, full_bar(stage), kb * QBK, nb * QBN, 0);
          if (++stage == Q_STAGES) {
            stage = 0;
            phase ^= 1u;
          }
        }
      }
    }
    return;
  }

  const int wg = warp >> 2;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  const int srow = (warp & 3) * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  const int no = *ep.ocnt;
  int32_t acc[64];
  int stage = 0;
  uint32_t phase = 0;
  for (int r = blockIdx.x; r < tiles; r += gridDim.x) {
    int mb, nb;
    i8_tile_to_mn(r, m_blocks, n_blocks, mb, nb);
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0;
    int prev_stage = -1;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(full_bar(stage), phase);
      const uint32_t sa = smem_base + stage * Q_STAGE_BYTES + wg * (64 * QBK);
      const uint32_t sb = smem_base + stage * Q_STAGE_BYTES + Q_A_BYTES;
      i8_reg_fence(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < QBK / 32; ++k)
        WgmmaS8<QBN>::mma(acc, make_smem_desc_sw128(sa + k * 32, 0, 1024), make_smem_desc_sw128(sb + k * 32, 0, 1024), 1u);
      wgmma_commit();
      wgmma_wait<1>();
      i8_reg_fence(acc);
      if (prev_stage >= 0 && wg_leader) mbar_arrive(empty_bar(prev_stage));
      prev_stage = stage;
      if (++stage == Q_STAGES) {
        stage = 0;
        phase ^= 1u;
      }
    }
    wgmma_wait<0>();
    i8_reg_fence(acc);
    if (wg_leader) mbar_arrive(empty_bar(prev_stage));

    // epilogue: acc[4 j + 2 h + e] is row srow + 8 h, column 8 j + cq + e of the warpgroup's 64 x 128 block; one row
    // and a quarter of the thread's columns at a time (the outlier sums of 8 elements in flight, within 168 registers)
    const int n0 = nb * QBN + cq;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = mb * QBM + wg * 64 + srow + 8 * h;
      if (row >= M) continue;
      const float sa = ep.sca[row];
      const bf16* xr = ep.x + row * ep.ldx;
#pragma unroll
      for (int part = 0; part < 4; ++part) {
        float o[8];
#pragma unroll
        for (int t = 0; t < 8; ++t) o[t] = 0.f;
        if (no > 0) {
          float wsc[8];
#pragma unroll
          for (int t = 0; t < 8; ++t) {
            const int col = n0 + 8 * (4 * part + t / 2) + t % 2;
            wsc[t] = col < N ? __fmul_rn(ep.scb[col], I8_INV127) : 0.f;
          }
          for (int i = 0; i < no; ++i) {
            const int jo = ep.oidx[i];
            const float xv = __bfloat162float(xr[jo]);
#pragma unroll
            for (int t = 0; t < 8; ++t) {
              const int col = min(n0 + 8 * (4 * part + t / 2) + t % 2, N - 1);
              o[t] = __fadd_rn(o[t], i8_term(xv, ep.cb[(long long)col * K + jo], wsc[t]));
            }
          }
        }
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          const int j = 4 * part + t / 2, e = t % 2;
          const int col = n0 + 8 * j + e;
          if (col < N) {
            const float v = i8_main(acc[4 * j + 2 * h + e], sa, ep.scb[col]);
            i8_store(ep, row, col, i8_finish(v, o[t], ep.bias, ep.residual, row * ep.ldr, col));
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------
static PFN_cuTensorMapEncodeTiled_v12000 i8_encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  });
  return fn;
}

// int8 [rows, K] row-major (row stride K bytes), box 128 (K) x 128 rows, SWIZZLE_128B; out-of-range elements read as 0
static int make_tmap_i8(CUtensorMap* out, const void* base, uint64_t K, uint64_t rows) {
  auto fn = i8_encode_fn();
  if (!fn) return set_error(CB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[3] = {K, rows, 1};
  cuuint64_t strides[2] = {K, K * rows};
  cuuint32_t box[3] = {QBK, 128, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = CUDA_SUCCESS;
  for (int attempt = 0; attempt < 2; ++attempt) {
    r = fn(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(base), dims, strides, box, estr,
           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_ERROR_INVALID_CONTEXT) break;
    cudaFree(0);  // a thread with no driver context bound yet: bind the primary context and retry
  }
  if (r != CUDA_SUCCESS) return set_error(CB_ERR_CUDA, "cuTensorMapEncodeTiled (int8) failed (%d)", (int)r);
  return CB_OK;
}

static int i8_epi(I8Epi& ep, const char* who, int M, int N, int K, const void* xq, const void* cb, const float* sca,
                  const float* scb, const void* x, long long ldx, const int* oidx, const int* ocnt, void* y,
                  long long ldy, const void* bias, const void* residual, long long ldr, int out_fp32) {
  CB_CHECK_ARG(M > 0 && N > 0 && K > 0 && K % 16 == 0, "%s: K=%d must be a positive multiple of 16 (M=%d N=%d)", who, K, M,
               N);
  CB_CHECK_ARG(xq && cb && sca && scb && x && oidx && ocnt && y, "%s: null argument", who);
  CB_CHECK_ARG(((reinterpret_cast<uintptr_t>(xq) | reinterpret_cast<uintptr_t>(cb)) & 15u) == 0,
               "%s: xq and cb must be 16-byte aligned", who);
  CB_CHECK_ARG(ldx >= K && ldy >= N && (!residual || ldr >= N), "%s: row strides too small", who);
  ep.sca = sca; ep.scb = scb; ep.x = (const bf16*)x; ep.ldx = ldx; ep.cb = (const int8_t*)cb;
  ep.oidx = oidx; ep.ocnt = ocnt; ep.y = y; ep.ldy = ldy;
  ep.bias = (const bf16*)bias; ep.residual = (const bf16*)residual; ep.ldr = ldr; ep.out_fp32 = out_fp32;
  return CB_OK;
}

int gemv_int8_launch(const void* xq, const void* cb, const float* sca, const float* scb, const void* x, long long ldx,
                     const int* oidx, const int* ocnt, void* y, int M, int N, int K, long long ldy, const void* bias,
                     const void* residual, long long ldr, int out_fp32, cudaStream_t st) {
  CB_CHECK_ARG(M >= 1 && M <= 8, "gemv_int8: M=%d must be in [1, 8]", M);
  I8Epi ep;
  const int rc = i8_epi(ep, "gemv_int8", M, N, K, xq, cb, sca, scb, x, ldx, oidx, ocnt, y, ldy, bias, residual, ldr,
                        out_fp32);
  if (rc != CB_OK) return rc;
  const int grid = (N + IG_WARPS * IG_CPW - 1) / (IG_WARPS * IG_CPW);
  const int8_t* q = (const int8_t*)xq;
#define CB_IG(MM) gemv_int8_kernel<MM><<<grid, IG_WARPS * 32, 0, st>>>(q, N, K, ep)
  switch (M) {
    case 1: CB_IG(1); break;
    case 2: CB_IG(2); break;
    case 3: CB_IG(3); break;
    case 4: CB_IG(4); break;
    case 5: CB_IG(5); break;
    case 6: CB_IG(6); break;
    case 7: CB_IG(7); break;
    default: CB_IG(8); break;
  }
#undef CB_IG
  CB_CUDA_LAUNCH_CHECK("gemv_int8");
  return CB_OK;
}

int gemm_int8_launch(const void* xq, const void* cb, const float* sca, const float* scb, const void* x, long long ldx,
                     const int* oidx, const int* ocnt, void* y, int M, int N, int K, long long ldy, const void* bias,
                     const void* residual, long long ldr, int out_fp32, cudaStream_t st) {
  I8Epi ep;
  int rc = i8_epi(ep, "gemm_int8", M, N, K, xq, cb, sca, scb, x, ldx, oidx, ocnt, y, ldy, bias, residual, ldr, out_fp32);
  if (rc != CB_OK) return rc;
  CUtensorMap ta, tb;
  if ((rc = make_tmap_i8(&ta, xq, K, M))) return rc;
  if ((rc = make_tmap_i8(&tb, cb, K, N))) return rc;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(gemm_int8_wgmma, cudaFuncAttributeMaxDynamicSharedMemorySize, Q_SMEM_BYTES);
    if (e != cudaSuccess) return set_error(CB_ERR_CUDA, "gemm_int8 smem attr: %s", cudaGetErrorString(e));
    attr = true;
  }
  const long long tiles = (long long)((M + QBM - 1) / QBM) * ((N + QBN - 1) / QBN);
  CB_CHECK_ARG(tiles < (1LL << 31), "gemm_int8: %lld tiles exceed the grid", tiles);
  const unsigned grid = (unsigned)std::min<long long>(tiles, device_sm_count());
  gemm_int8_wgmma<<<grid, 288, Q_SMEM_BYTES, st>>>(ta, tb, M, N, K, (int)tiles, ep);
  CB_CUDA_LAUNCH_CHECK("gemm_int8_wgmma");
  return CB_OK;
}

}  // namespace cb
