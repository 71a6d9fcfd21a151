// cambrian_b200 — FP8 E4M3 training (`fp8_training`): the transposed weight quantiser of the input-gradient GEMMs.
//
// cambrian_b200/train_fp8.py states the training format; it is the row rule of quant_fp8.py applied to the operands of
// the forward (y = x W^T) and input-gradient (dx = dy W) GEMMs.  f8 wgmma takes only K-major operands, so the dgrad GEMM
// needs W^T [K, N] with one scale per row of W^T, i.e. per input column of W:
//
//   st[k] = amax_k / 448,  r = min(448 / amax_k, FLT_MAX),  wtq[k, n] = e4m3_rn_satfinite(fp32(W[n, k] * r)),
//   amax_k = max_n |W[n, k]|
//
// which is bit for bit cb_fp8_quantize_weight of W.t().contiguous().  The other two new kernels sit next to the bf16
// kernels they must match bit for bit: the E4M3-output RMSNorm in norm.cu and the dual-output SwiGLU backward in
// elementwise.cu.
//
//   f8_colmax_kernel     pass 1: partial column maxima of W over row chunks -> workspace [splits, K] (max is exact, so
//                        the result does not depend on the split count; no atomics)
//   f8_quant_wt_kernel   pass 2: folds the partials of its 64 columns, then transposes a 64 x 64 tile through shared
//                        memory and writes 16 e4m3 bytes of one W^T row per thread
#include "common.cuh"
#include <algorithm>
#include <cfloat>

namespace cb {

constexpr int QT_COLS = 256;   // pass 1: columns per CTA (32 lanes x 8-element vectors), 8 row lanes
constexpr int QT_ROWS = 64;    // pass 1: rows per split are a multiple of this
constexpr int QT_TILE = 64;    // pass 2: 64 (n) x 64 (k) tile
constexpr int QT_LDS = QT_TILE + 2;  // bf16 per shared-memory row: 33 words, so column reads spread over the banks

__global__ void __launch_bounds__(256) f8_colmax_kernel(const bf16* __restrict__ w, int N, int K, long long ldw,
                                                        int rows_per_split, float* __restrict__ part) {
  __shared__ float red[8][QT_COLS + 1];
  const int lane = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int c0 = blockIdx.x * QT_COLS + lane * 8;
  const int n0 = blockIdx.y * rows_per_split;
  const int n1 = min(N, n0 + rows_per_split);
  float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (c0 < K) {
    for (int n = n0 + rl; n < n1; n += 8) {
      float f[8];
      unpack8(ldg_nc(w + (long long)n * ldw + c0), f);
#pragma unroll
      for (int e = 0; e < 8; ++e) a[e] = fmaxf(a[e], fabsf(f[e]));
    }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) red[rl][lane * 8 + e] = a[e];
  __syncthreads();
  const int c = blockIdx.x * QT_COLS + threadIdx.x;
  if (c < K) {
    float t = red[0][threadIdx.x];
#pragma unroll
    for (int i = 1; i < 8; ++i) t = fmaxf(t, red[i][threadIdx.x]);
    part[(long long)blockIdx.y * K + c] = t;
  }
}

__global__ void __launch_bounds__(256) f8_quant_wt_kernel(const bf16* __restrict__ w, int N, int K, long long ldw,
                                                          const float* __restrict__ part, int splits,
                                                          uint8_t* __restrict__ wtq, float* __restrict__ st) {
  __shared__ bf16 tile[QT_TILE][QT_LDS];
  __shared__ float rk[QT_TILE];
  const int k0 = blockIdx.x * QT_TILE, n0 = blockIdx.y * QT_TILE;
  if (threadIdx.x < QT_TILE) {
    const int k = k0 + threadIdx.x;
    float a = 0.f;
    if (k < K)
      for (int i = 0; i < splits; ++i) a = fmaxf(a, part[(long long)i * K + k]);
    if (k < K && blockIdx.y == 0) st[k] = __fdiv_rn(a, 448.0f);
    rk[threadIdx.x] = fminf(__fdiv_rn(448.0f, a), FLT_MAX);  // amax = 0 or below 448 * 2^-128: +inf -> FLT_MAX
  }
  // load W[n0 .. n0 + 64, k0 .. k0 + 64): 8 threads per row, one 16-byte vector each, two passes of 32 rows
#pragma unroll
  for (int p = 0; p < 2; ++p) {
    const int rr = p * 32 + (threadIdx.x >> 3), cv = (threadIdx.x & 7) * 8;
    const int n = n0 + rr, k = k0 + cv;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (n < N && k < K) v = ldg_nc(w + (long long)n * ldw + k);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&tile[rr][cv]);
    dst[0] = v.x;
    dst[1] = v.y;
    dst[2] = v.z;
    dst[3] = v.w;
  }
  __syncthreads();
  // write: thread -> W^T row k0 + (tid >> 2), columns n0 + 16 (tid & 3) .. + 16: a warp stores 8 rows x 64 bytes
  const int kl = threadIdx.x >> 2, nl = (threadIdx.x & 3) * 16;
  const int k = k0 + kl, n = n0 + nl;
  if (k >= K || n >= N) return;  // N % 16 == 0: a chunk is whole or absent
  const float r = rk[kl];
  float f[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) f[j] = __fmul_rn(__bfloat162float(tile[nl + j][kl]), r);
  const uint2 lo = f8_pack8(f), hi = f8_pack8(f + 8);
  *reinterpret_cast<uint4*>(wtq + (long long)k * N + n) = make_uint4(lo.x, lo.y, hi.x, hi.y);
}

// row splits of pass 1: enough CTAs for about four per SM, each split a multiple of QT_ROWS rows
static void wt_splits(int N, int K, int* splits, int* rows_per_split) {
  const int col_blocks = (K + QT_COLS - 1) / QT_COLS;
  const int max_splits = (N + QT_ROWS - 1) / QT_ROWS;
  int s = std::max(1, std::min(max_splits, 4 * device_sm_count() / col_blocks));
  int rps = (N + s - 1) / s;
  rps = (rps + QT_ROWS - 1) / QT_ROWS * QT_ROWS;
  *rows_per_split = rps;
  *splits = (N + rps - 1) / rps;
}

long long fp8_quantize_weight_t_workspace_floats(int N, int K) {
  if (N <= 0 || K <= 0) return 0;
  int s, rps;
  wt_splits(N, K, &s, &rps);
  return (long long)s * K;
}

int fp8_quantize_weight_t_launch(const void* w, int N, int K, long long ldw, void* wtq, float* st, float* ws,
                                 long long ws_floats, cudaStream_t stream) {
  CB_CHECK_ARG(N > 0 && K > 0 && N % 16 == 0 && K % 16 == 0,
               "fp8_quantize_weight_t: N=%d and K=%d must be positive multiples of 16", N, K);
  CB_CHECK_ARG(w && wtq && st && ws && ldw >= K && ldw % 8 == 0, "fp8_quantize_weight_t: null argument or bad row stride");
  CB_CHECK_ARG(((reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(wtq)) & 15u) == 0,
               "fp8_quantize_weight_t: w and wtq must be 16-byte aligned");
  int splits, rps;
  wt_splits(N, K, &splits, &rps);
  CB_CHECK_ARG(ws_floats >= (long long)splits * K, "fp8_quantize_weight_t: workspace too small (%lld < %lld floats)",
               ws_floats, (long long)splits * K);
  f8_colmax_kernel<<<dim3((K + QT_COLS - 1) / QT_COLS, splits), 256, 0, stream>>>((const bf16*)w, N, K, ldw, rps, ws);
  CB_CUDA_LAUNCH_CHECK("f8_colmax_kernel");
  f8_quant_wt_kernel<<<dim3((K + QT_TILE - 1) / QT_TILE, (N + QT_TILE - 1) / QT_TILE), 256, 0, stream>>>(
      (const bf16*)w, N, K, ldw, ws, splits, (uint8_t*)wtq, st);
  CB_CUDA_LAUNCH_CHECK("f8_quant_wt_kernel");
  return CB_OK;
}

}  // namespace cb
