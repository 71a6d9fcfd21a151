// cambrian_b200 — weight-streaming GEMV for decode-shaped projections (M <= 8 rows: one token per sequence of a generate()
// batch, cambrian_llama.py:437-483 -> HF greedy loop).   y[M, N] = x[M, K] W[N, K]^T (+ bias) (+ residual)
//
// With <= 8 rows the 128-row wgmma tile wastes > 93 % of the tensor pipe, and the step is pure weight bandwidth, so this
// kernel does the minimum — every weight byte is loaded exactly once with 16-byte coalesced vectors,
// 16 loads in flight per lane, and multiplied on the FMA pipe against the activation rows held in shared memory.
//   block = 8 warps, one warp = 2 output columns; K is walked in chunks of 2048 (x chunk: M x 4 KB of smem);
//   fp32 accumulation, one shuffle tree per (row, column) at the end.
#include "common.cuh"

namespace cb {

constexpr int GV_KC = 2048;   // K elements per chunk
constexpr int GV_CPW = 2;     // output columns per warp
constexpr int GV_WARPS = 8;

template <int M>
__global__ void __launch_bounds__(GV_WARPS * 32)
gemv_bf16_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w, void* __restrict__ y, const bf16* __restrict__ bias,
                 const bf16* __restrict__ residual, int N, int K, long long ldx, long long ldw, long long ldy, long long ldr,
                 int out_fp32) {
  __shared__ __align__(16) bf16 xs[M][GV_KC];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = (blockIdx.x * GV_WARPS + warp) * GV_CPW;
  float acc[GV_CPW][M];
#pragma unroll
  for (int c = 0; c < GV_CPW; ++c)
#pragma unroll
    for (int m = 0; m < M; ++m) acc[c][m] = 0.f;
  for (int k0 = 0; k0 < K; k0 += GV_KC) {
    const int kc = min(GV_KC, K - k0);  // multiple of 8
    __syncthreads();
    for (int i = threadIdx.x; i < M * (GV_KC / 8); i += GV_WARPS * 32) {
      const int m = i / (GV_KC / 8), v = i % (GV_KC / 8);
      uint4 val = make_uint4(0u, 0u, 0u, 0u);
      if (v * 8 < kc) val = *reinterpret_cast<const uint4*>(x + m * ldx + k0 + v * 8);
      *reinterpret_cast<uint4*>(&xs[m][v * 8]) = val;
    }
    __syncthreads();
    if (n0 < N) {
      // all weight loads of the chunk first (GV_KC / 256 = 8 vectors per column per lane), then the arithmetic
      uint4 wv[GV_CPW][GV_KC / 256];
#pragma unroll
      for (int c = 0; c < GV_CPW; ++c) {
        const bool col_ok = n0 + c < N;
        const bf16* wp = w + static_cast<long long>(col_ok ? n0 + c : n0) * ldw + k0;
#pragma unroll
        for (int j = 0; j < GV_KC / 256; ++j)  // branch-free: past the chunk's end re-read its last vector (x there is 0)
          wv[c][j] = ldg_nc(wp + min(j * 256 + lane * 8, kc - 8));
      }
#pragma unroll
      for (int j = 0; j < GV_KC / 256; ++j) {
        float wf[GV_CPW][8];
#pragma unroll
        for (int c = 0; c < GV_CPW; ++c) unpack8(wv[c][j], wf[c]);
#pragma unroll
        for (int m = 0; m < M; ++m) {
          float xf[8];
          unpack8(*reinterpret_cast<const uint4*>(&xs[m][j * 256 + lane * 8]), xf);
#pragma unroll
          for (int c = 0; c < GV_CPW; ++c)
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[c][m] = fmaf(wf[c][e], xf[e], acc[c][m]);
        }
      }
    }
  }
  if (n0 >= N) return;
#pragma unroll
  for (int c = 0; c < GV_CPW; ++c)
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

int gemv_bf16_launch(const void* x, const void* w, void* y, int M, int N, int K, long long ldx, long long ldw, long long ldy,
                     const void* bias, const void* residual, long long ldr, int out_fp32, cudaStream_t st) {
  CB_CHECK_ARG(M >= 1 && M <= 8 && N > 0 && K > 0, "gemv: M=%d must be in [1, 8] (N=%d K=%d)", M, N, K);
  CB_CHECK_ARG(K % 8 == 0 && ldx % 8 == 0 && ldw % 8 == 0, "gemv: K and the row strides must be multiples of 8");
  CB_CHECK_ARG(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(w)) & 15u) == 0, "gemv: operands must be 16-byte aligned");
  const int grid = (N + GV_WARPS * GV_CPW - 1) / (GV_WARPS * GV_CPW);
  const bf16 *xp = (const bf16*)x, *wp = (const bf16*)w, *bp = (const bf16*)bias, *rp = (const bf16*)residual;
#define CB_GV(MM) gemv_bf16_kernel<MM><<<grid, GV_WARPS * 32, 0, st>>>(xp, wp, y, bp, rp, N, K, ldx, ldw, ldy, ldr, out_fp32)
  if (M == 1) CB_GV(1);
  else if (M == 2) CB_GV(2);
  else if (M <= 4) {
    if (M == 3) CB_GV(3); else CB_GV(4);
  } else if (M <= 6) {
    if (M == 5) CB_GV(5); else CB_GV(6);
  } else {
    if (M == 7) CB_GV(7); else CB_GV(8);
  }
#undef CB_GV
  CB_CUDA_LAUNCH_CHECK("gemv_bf16");
  return CB_OK;
}

}  // namespace cb
