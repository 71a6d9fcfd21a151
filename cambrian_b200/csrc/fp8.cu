// cambrian_b200 — FP8 E4M3 decoder weights for inference (`load_fp8`).
//
// Format and arithmetic (cambrian_b200/quant_fp8.py owns them on the host and states them in full):
//   one row v [K] bf16 (a weight row at load, an activation row per call) -> q [K] e4m3, s fp32:
//     s = amax / 448,  r = min(448 / amax, FLT_MAX),  q[k] = e4m3_rn_satfinite(float(v[k]) * r)
//     (amax = max |v|; each division and product rounded to fp32 on its own; a zero row gives q = +-0, s = 0);
//   output y[m, n] = acc * (sa[m] * sw[n]) (+ bias[n]) (+ residual[m, n]), one rounding to bf16 (or fp32 output), with
//     acc = sum_k float(xq[m, k]) * float(wq[n, k]) in fp32.  The f8 tensor-core MMA keeps fewer than 32 accumulator
//     bits, so every 128-deep k-block is summed by the tensor cores on its own (scale-d = 0 on its first instruction)
//     and added to fp32 registers here.  The summation order is not part of the format: GEMM and GEMV rows agree to
//     fp32 accumulation error, not bit for bit.
//
//   f8_quant_rows_kernel     cb_fp8_quantize_weight / cb_fp8_quantize_act: one CTA per row, amax then q; no atomics
//   gemm_fp8_wgmma           M > 8 (cb_gemm_fp8): bytegemm.cuh's TMA ring, wgmma m64n128k32 .f32.e4m3.e4m3
//   gemv_fp8_wgmma           M <= 8 (cb_gemv_fp8): swap AB, y^T = W x^T as wgmma m64n8k32, K split over a cluster
#include "bytegemm.cuh"
#include <cuda_fp16.h>
#include <algorithm>
#include <cfloat>

namespace cb {

int make_tmap_bf16_3d(CUtensorMap*, const void*, uint64_t, uint64_t, uint64_t, uint64_t, uint64_t, uint32_t);  // gemm.cu

struct F8Epi {
  const float* sa;      // [M]
  const float* sw;      // [N]
  void* y;
  long long ldy;
  const bf16* bias;     // [N] or null
  const bf16* residual; // [M, ldr] or null
  long long ldr;
  int out_fp32;
};

// y = acc * (sa * sw), then + bias, then + residual, each rounded to fp32 on its own
__device__ __forceinline__ float f8_out(const F8Epi& ep, float acc, float sa, float sw, int m, int n) {
  float y = __fmul_rn(acc, __fmul_rn(sa, sw));
  if (ep.bias) y = __fadd_rn(y, __bfloat162float(ep.bias[n]));
  if (ep.residual) y = __fadd_rn(y, __bfloat162float(ep.residual[(long long)m * ep.ldr + n]));
  return y;
}
__device__ __forceinline__ void f8_store(const F8Epi& ep, int m, int n, float v) {
  if (ep.out_fp32) reinterpret_cast<float*>(ep.y)[m * ep.ldy + n] = v;
  else reinterpret_cast<bf16*>(ep.y)[m * ep.ldy + n] = __float2bfloat16(v);
}

// ---------------------------------------------------------------------------------------------------------------------
// quantiser (weights and activations follow the same rule): one CTA per row, 8 elements (one 16-byte vector) per thread
// and step; the row is read twice (amax, then q), the second time from L1 / L2
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) f8_quant_rows_kernel(const bf16* __restrict__ x, int K, long long ldx,
                                                            uint8_t* __restrict__ q, float* __restrict__ s) {
  __shared__ float red[8];
  const int m = blockIdx.x;
  const bf16* xr = x + (long long)m * ldx;
  float a = 0.f;
  for (int k = threadIdx.x * 8; k < K; k += 256 * 8) {
    float f[8];
    unpack8(*reinterpret_cast<const uint4*>(xr + k), f);
#pragma unroll
    for (int e = 0; e < 8; ++e) a = fmaxf(a, fabsf(f[e]));
  }
  a = warp_max(a);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = a;
  __syncthreads();
  a = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) a = fmaxf(a, red[i]);
  if (threadIdx.x == 0) s[m] = __fdiv_rn(a, 448.0f);
  const float r = fminf(__fdiv_rn(448.0f, a), FLT_MAX);  // amax = 0 or below 448 * 2^-128: +inf -> FLT_MAX
  uint8_t* qr = q + (long long)m * K;
  for (int k = threadIdx.x * 8; k < K; k += 256 * 8) {
    float f[8];
    unpack8(*reinterpret_cast<const uint4*>(xr + k), f);
    uint32_t p[2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
      p[h] = f8_pack2(__fmul_rn(f[4 * h], r), __fmul_rn(f[4 * h + 1], r)) |
             f8_pack2(__fmul_rn(f[4 * h + 2], r), __fmul_rn(f[4 * h + 3], r)) << 16;
    *reinterpret_cast<uint2*>(qr + k) = make_uint2(p[0], p[1]);
  }
}

static int f8_quant_rows(const char* who, const void* x, int rows, int K, long long ldx, void* q, float* s,
                         cudaStream_t st) {
  CB_CHECK_ARG(rows > 0 && K > 0 && K % 16 == 0, "%s: K=%d must be a positive multiple of 16 (rows=%d)", who, K, rows);
  CB_CHECK_ARG(x && q && s && ldx >= K && ldx % 8 == 0, "%s: null argument or bad row stride", who);
  CB_CHECK_ARG(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(q)) & 15u) == 0,
               "%s: input and output must be 16-byte aligned", who);
  f8_quant_rows_kernel<<<rows, 256, 0, st>>>((const bf16*)x, K, ldx, (uint8_t*)q, s);
  CB_CUDA_LAUNCH_CHECK(who);
  return CB_OK;
}

int fp8_quantize_weight_launch(const void* w, int N, int K, long long ldw, void* wq, float* sw, cudaStream_t st) {
  return f8_quant_rows("fp8_quantize_weight", w, N, K, ldw, wq, sw, st);
}
int fp8_quantize_act_launch(const void* x, int M, int K, long long ldx, void* xq, float* sa, cudaStream_t st) {
  return f8_quant_rows("fp8_quantize_act", x, M, K, ldx, xq, sa, st);
}

// ---------------------------------------------------------------------------------------------------------------------
// GEMM, M > 8: the int8 GEMM's persistent warp-specialised structure on e4m3.  288 threads: warp 8 runs bytegemm.cuh's
// TMA producer (a 6-stage ring of 128 x 128-byte boxes of xq and wq), warps 0..7 are two consumer warpgroups of 64 rows
// issuing wgmma m64n128k32 .f32.e4m3.e4m3, 4 per k-block, into a fresh partial (scale-d = 0 on the first), then waiting
// for them and adding the partial to the fp32 total before releasing the stage.  While one warpgroup adds, the other
// one's MMAs keep the tensor cores busy.  (Keeping a k-block in flight as well needs a third 64-register set per thread;
// with setmaxnreg on a 384-thread CTA ptxas still allocated 168 registers, spilled and serialised the wgmmas.)
// Epilogue from registers in the order of quant_fp8.py; a bf16 output TMA can address leaves through gemm.cu's swizzled
// staging + TMA store.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int F8_STAGES = 6;
constexpr int F8_STG_BYTES = 64 * 128;  // one 64 x 64 bf16 store sub-tile; two per consumer warpgroup
constexpr int F8_SMEM_BYTES = F8_STAGES * Q_STAGE_BYTES + 4 * F8_STG_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
static_assert(F8_SMEM_BYTES <= 232448, "exceeds the 227 KB of shared memory a CTA may use");

__global__ void __launch_bounds__(288, 1)
gemm_fp8_wgmma(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmC, int M, int N, int K, int tiles, int tma_store, F8Epi ep) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t stg_base = smem_base + F8_STAGES * Q_STAGE_BYTES;
  const uint32_t bar_base = stg_base + 4 * F8_STG_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (F8_STAGES + s); };
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int m_blocks = (M + QBM - 1) / QBM;
  const int n_blocks = (N + QBN - 1) / QBN;
  const int num_kb = (K + QBK - 1) / QBK;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < F8_STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);  // one arrive per consumer warpgroup
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) q_produce<F8_STAGES>(&tmA, &tmB, smem_base, bar_base, M, N, K, tiles);
    return;
  }

  const int wg = warp >> 2;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  const int srow = (warp & 3) * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  const uint32_t stg = stg_base + wg * (2 * F8_STG_BYTES);
  uint32_t q = 0;
  if (wg_leader && tma_store) tma_prefetch_desc(&tmC);

  // gemm.cu's store of one 64 x 64 bf16 sub-tile of the warpgroup's rows: pair(j, h) is the bf16x2 at columns 8 j + cq,
  // + 1 of row srow + 8 h, written to SWIZZLE_128B staging (chunk c of a row at c ^ (row & 7)), stored by TMA, which
  // clips the M / N tails; the two buffers alternate so one drains while the other fills
  auto store_subtile = [&](int x, int y, auto pair) {
    const uint32_t buf = stg + (q & 1u) * F8_STG_BYTES;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = srow + 8 * h;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const __nv_bfloat162 v = pair(j, h);
        st_shared_b32(buf + row * 128 + ((j ^ (row & 7)) << 4) + 2 * cq, *reinterpret_cast<const uint32_t*>(&v));
      }
    }
    fence_proxy_async_smem();
    if (wg_leader) bulk_wait_read<0>();
    named_bar_sync(1 + wg, 128);
    if (wg_leader && x < N && y < M) {
      tma_store_3d(&tmC, buf, x, y, 0);
      bulk_commit();
    }
    ++q;
  };

  float acc[64], part[64];
  int stage = 0;
  uint32_t phase = 0;
  for (int r = blockIdx.x; r < tiles; r += gridDim.x) {
    int mb, nb;
    q_tile_to_mn(r, m_blocks, n_blocks, mb, nb);
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(full_bar(stage), phase);
      const uint32_t sa = smem_base + stage * Q_STAGE_BYTES + wg * (64 * QBK);
      const uint32_t sb = smem_base + stage * Q_STAGE_BYTES + Q_A_BYTES;
      reg_fence(part);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < QBK / 32; ++k)
        WgmmaE4M3<QBN>::mma(part, make_smem_desc_sw128(sa + k * 32, 0, 1024), make_smem_desc_sw128(sb + k * 32, 0, 1024),
                            k > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(part);
      if (wg_leader) mbar_arrive(empty_bar(stage));
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] += part[i];
      if (++stage == F8_STAGES) {
        stage = 0;
        phase ^= 1u;
      }
    }

    // epilogue: acc[4 j + 2 h + e] is row srow + 8 h, column 8 j + cq + e of the warpgroup's 64 x 128 block
    const int y0 = mb * QBM + wg * 64;
    const int n0 = nb * QBN + cq;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = y0 + srow + 8 * h;
      const bool row_ok = row < M;
      const float sa = row_ok ? ep.sa[row] : 0.f;
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = n0 + 8 * j + e;
          float& v = acc[4 * j + 2 * h + e];
          if (row_ok && col < N) {
            v = f8_out(ep, v, sa, ep.sw[col], row, col);
            if (!tma_store) f8_store(ep, row, col, v);
          }
        }
    }
    if (tma_store) {
#pragma unroll
      for (int s = 0; s < 2; ++s)
        store_subtile(nb * QBN + 64 * s, y0, [&](int j, int h) {
          return __floats2bfloat162_rn(acc[4 * (8 * s + j) + 2 * h], acc[4 * (8 * s + j) + 2 * h + 1]);
        });
    }
  }
  if (wg_leader) bulk_wait<0>();  // the CTA's smem must outlive the stores that read it
}

// ---------------------------------------------------------------------------------------------------------------------
// decode GEMV, M <= 8: "swap AB".  y^T [N, M] = W [N, K] * xq^T, so a 64-row W tile is the wgmma A operand and the <= 8
// quantised activation rows are the N = 8 B operand (TMA zero-fills rows past M): wgmma m64n8k32 .f32.e4m3.e4m3, no
// per-weight instruction on the CUDA cores.  160 threads: warp 4 is the TMA producer (per k-block a 64 x 128-byte W box
// and an 8 x 128-byte xq box, 6 stages), warpgroup 0 issues the 4 MMAs of a k-block into a fresh partial (scale-d = 0
// first) and adds it to 4 fp32 registers.  K is split over the CTAs of a cluster (grid.x = splits = cluster size, at
// most 8) so that the narrow projections still fill the SMs; rank 0 adds the ranks' partials in rank order from
// distributed shared memory: deterministic, no atomics, no workspace.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int GV8_STAGES = 6;
constexpr int GV8_A_BYTES = 64 * QBK, GV8_STAGE_BYTES = GV8_A_BYTES + 8 * QBK;  // 9 KB, a multiple of 1024
constexpr int GV8_RED_BYTES = 64 * 8 * 4;
constexpr int GV8_SMEM_BYTES = GV8_STAGES * GV8_STAGE_BYTES + GV8_RED_BYTES + 1024 /*align slack*/ + 128 /*barriers*/;
constexpr int GV8_MAX_SPLITS = 8;  // the portable cluster size

__device__ __forceinline__ uint32_t cluster_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ float ld_cluster_f32(uint32_t local_addr, uint32_t rank) {
  uint32_t remote;
  float v;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local_addr), "r"(rank));
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(remote) : "memory");
  return v;
}

__global__ void __launch_bounds__(160)
gemv_fp8_wgmma(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX, int M, int N, int K,
               int kb_per_split, F8Epi ep) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t red_base = smem_base + GV8_STAGES * GV8_STAGE_BYTES;
  const uint32_t bar_base = red_base + GV8_RED_BYTES;
  float* red = reinterpret_cast<float*>(smem_raw + (red_base - smem_u32(smem_raw)));
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (GV8_STAGES + s); };
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t rank = cluster_rank();
  const int num_kb = (K + QBK - 1) / QBK;
  const int kb0 = (int)rank * kb_per_split;
  const int kb1 = min(num_kb, kb0 + kb_per_split);
  const int n0 = blockIdx.y * 64;

  if (warp == 4 && lane == 0) {
    tma_prefetch_desc(&tmW);
    tma_prefetch_desc(&tmX);
    for (int s = 0; s < GV8_STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 1);
    }
    mbar_fence_init();
  }
  __syncthreads();

  const int srow = (warp & 3) * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  if (warp == 4) {
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(empty_bar(stage), phase ^ 1u);
        const uint32_t s = smem_base + stage * GV8_STAGE_BYTES;
        mbar_arrive_expect_tx(full_bar(stage), GV8_STAGE_BYTES);
        tma_load_3d(s, &tmW, full_bar(stage), kb * QBK, n0, 0);
        tma_load_3d(s + GV8_A_BYTES, &tmX, full_bar(stage), kb * QBK, 0, 0);
        if (++stage == GV8_STAGES) {
          stage = 0;
          phase ^= 1u;
        }
      }
    }
  } else {
    float part[4];
    int stage = 0;
    uint32_t phase = 0;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(full_bar(stage), phase);
      const uint32_t s = smem_base + stage * GV8_STAGE_BYTES;
      reg_fence(part);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < QBK / 32; ++k)
        WgmmaE4M3<8>::mma(part, make_smem_desc_sw128(s + k * 32, 0, 1024),
                          make_smem_desc_sw128(s + GV8_A_BYTES + k * 32, 0, 1024), k > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(part);
      if (threadIdx.x == 0) mbar_arrive(empty_bar(stage));
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[e] += part[e];
      if (++stage == GV8_STAGES) {
        stage = 0;
        phase ^= 1u;
      }
    }
    // acc[e] is W row srow + 8 (e / 2), activation row cq + e % 2 of this rank's k range
#pragma unroll
    for (int e = 0; e < 4; ++e) red[(srow + 8 * (e >> 1)) * 8 + cq + (e & 1)] = acc[e];
  }
  cluster_sync_all();
  if (rank == 0 && warp < 4) {
    const int splits = (num_kb + kb_per_split - 1) / kb_per_split;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int nl = srow + 8 * (e >> 1), m = cq + (e & 1), n = n0 + nl;
      float v = acc[e];
      for (int rr = 1; rr < splits; ++rr) v += ld_cluster_f32(red_base + (nl * 8 + m) * 4, rr);
      if (m < M && n < N) f8_store(ep, m, n, f8_out(ep, v, ep.sa[m], ep.sw[n], m, n));
    }
  }
  cluster_sync_all();  // every rank's partials stay in its shared memory until rank 0 has read them
}

// ---------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------
static int f8_epi(F8Epi& ep, const char* who, int M, int N, int K, const void* xq, const void* wq, const float* sa,
                  const float* sw, void* y, long long ldy, const void* bias, const void* residual, long long ldr,
                  int out_fp32) {
  CB_CHECK_ARG(M > 0 && N > 0 && K > 0 && K % 16 == 0, "%s: K=%d must be a positive multiple of 16 (M=%d N=%d)", who, K, M,
               N);
  CB_CHECK_ARG(xq && wq && sa && sw && y, "%s: null argument", who);
  CB_CHECK_ARG(((reinterpret_cast<uintptr_t>(xq) | reinterpret_cast<uintptr_t>(wq)) & 15u) == 0,
               "%s: xq and wq must be 16-byte aligned", who);
  CB_CHECK_ARG(ldy >= N && (!residual || ldr >= N), "%s: row strides too small", who);
  ep.sa = sa; ep.sw = sw; ep.y = y; ep.ldy = ldy;
  ep.bias = (const bf16*)bias; ep.residual = (const bf16*)residual; ep.ldr = ldr; ep.out_fp32 = out_fp32;
  return CB_OK;
}

int gemv_fp8_launch(const void* xq, const void* wq, const float* sa, const float* sw, void* y, int M, int N, int K,
                    long long ldy, const void* bias, const void* residual, long long ldr, int out_fp32, cudaStream_t st) {
  CB_CHECK_ARG(M >= 1 && M <= 8, "gemv_fp8: M=%d must be in [1, 8]", M);
  F8Epi ep;
  int rc = f8_epi(ep, "gemv_fp8", M, N, K, xq, wq, sa, sw, y, ldy, bias, residual, ldr, out_fp32);
  if (rc != CB_OK) return rc;
  CUtensorMap tw, tx;
  if ((rc = make_tmap_u8(&tw, wq, K, N, 64))) return rc;
  if ((rc = make_tmap_u8(&tx, xq, K, M, 8))) return rc;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(gemv_fp8_wgmma, cudaFuncAttributeMaxDynamicSharedMemorySize, GV8_SMEM_BYTES);
    if (e != cudaSuccess) return set_error(CB_ERR_CUDA, "gemv_fp8 smem attr: %s", cudaGetErrorString(e));
    attr = true;
  }
  // as many K splits as keep about three CTAs (their smem allows three) on every SM, each split at least one k-block
  const int n_tiles = (N + 63) / 64, num_kb = (K + QBK - 1) / QBK;
  int splits = std::max(1, std::min({GV8_MAX_SPLITS, num_kb, 3 * device_sm_count() / n_tiles}));
  const int kps = (num_kb + splits - 1) / splits;
  splits = (num_kb + kps - 1) / kps;
  CB_CHECK_ARG(n_tiles < 65536, "gemv_fp8: N=%d exceeds the grid", N);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(splits, n_tiles, 1);
  cfg.blockDim = dim3(160, 1, 1);
  cfg.dynamicSmemBytes = GV8_SMEM_BYTES;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = splits;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, gemv_fp8_wgmma, tw, tx, M, N, K, kps, ep);
  if (e != cudaSuccess) return set_error(CB_ERR_CUDA, "gemv_fp8 launch: %s", cudaGetErrorString(e));
  CB_CUDA_LAUNCH_CHECK("gemv_fp8_wgmma");
  return CB_OK;
}

int gemm_fp8_launch(const void* xq, const void* wq, const float* sa, const float* sw, void* y, int M, int N, int K,
                    long long ldy, const void* bias, const void* residual, long long ldr, int out_fp32, cudaStream_t st) {
  F8Epi ep;
  int rc = f8_epi(ep, "gemm_fp8", M, N, K, xq, wq, sa, sw, y, ldy, bias, residual, ldr, out_fp32);
  if (rc != CB_OK) return rc;
  CUtensorMap ta, tb, tc;
  if ((rc = make_tmap_u8(&ta, xq, K, M, QBM))) return rc;
  if ((rc = make_tmap_u8(&tb, wq, K, N, QBN))) return rc;
  // bf16 output TMA can address (16-byte aligned base, row stride a multiple of 8): TMA-store epilogue
  const int tma_store = !out_fp32 && (reinterpret_cast<uintptr_t>(y) & 15u) == 0 && ldy % 8 == 0;
  memset(&tc, 0, sizeof(tc));
  if (tma_store && (rc = make_tmap_bf16_3d(&tc, y, N, M, 1, ldy, 0, 64))) return rc;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(gemm_fp8_wgmma, cudaFuncAttributeMaxDynamicSharedMemorySize, F8_SMEM_BYTES);
    if (e != cudaSuccess) return set_error(CB_ERR_CUDA, "gemm_fp8 smem attr: %s", cudaGetErrorString(e));
    attr = true;
  }
  const long long tiles = (long long)((M + QBM - 1) / QBM) * ((N + QBN - 1) / QBN);
  CB_CHECK_ARG(tiles < (1LL << 31), "gemm_fp8: %lld tiles exceed the grid", tiles);
  const unsigned grid = (unsigned)std::min<long long>(tiles, device_sm_count());
  gemm_fp8_wgmma<<<grid, 288, F8_SMEM_BYTES, st>>>(ta, tb, tc, M, N, K, (int)tiles, tma_store, ep);
  CB_CUDA_LAUNCH_CHECK("gemm_fp8_wgmma");
  return CB_OK;
}

}  // namespace cb
