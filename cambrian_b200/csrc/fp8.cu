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
//   kv_fp8_append_kernel     cb_kv_fp8_append: the same row rule on each new K / V head row of the decode KV cache
//   attn_decode_fp8_kernel   cb_attn_decode_fp8: flash-decoding over the FP8 cache (cambrian_b200/kv_fp8.py states it)
#include "bytegemm.cuh"
#include "kv_rows.cuh"
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

// ---------------------------------------------------------------------------------------------------------------------
// FP8 decode KV cache (`kv_cache_dtype="fp8"`).  Per layer kq, vq e4m3 [B, S_max, nkv, hd] and ks, vs fp32
// [B, S_max, nkv]; each (sequence, position, kv head) row of K or V is quantised by the weight / activation rule above.
// Row helpers (one team of hd / 8 lanes per row, the row quantiser) are those of kv_rows.cuh.
// ---------------------------------------------------------------------------------------------------------------------

// cb_kv_fp8_append: team r quantises row r = ((b * S + s) * nkv + h) * 2 + (0: K, 1: V) of the new tokens into position
// offset (+ *offset_dev) + s.  No early exit: every lane of a warp takes part in the team shuffles.
template <int HD>
__global__ void __launch_bounds__(256) kv_fp8_append_kernel(const bf16* __restrict__ k, const bf16* __restrict__ v,
                                                            long long ld, uint8_t* __restrict__ kq, uint8_t* __restrict__ vq,
                                                            float* __restrict__ ks, float* __restrict__ vs, int B, int S,
                                                            int S_max, int nkv, long long offset,
                                                            const long long* __restrict__ offset_dev) {
  constexpr int LPK = HD / KV_DPL;
  const long long rows = 2LL * B * S * nkv;
  const long long r0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / LPK;
  const int sub = threadIdx.x % LPK;
  const bool in_range = r0 < rows;
  const long long r = in_range ? r0 : 0;
  const int which = (int)(r & 1);
  long long t = r >> 1;
  const int h = (int)(t % nkv);
  t /= nkv;
  const int s = (int)(t % S);
  const int b = (int)(t / S);
  const bf16* src = (which ? v : k) + ((long long)b * S + s) * ld + h * HD + sub * KV_DPL;
  float f[8];
  unpack8(*reinterpret_cast<const uint4*>(src), f);
  float a = 0.f;
#pragma unroll
  for (int e = 0; e < 8; ++e) a = fmaxf(a, fabsf(f[e]));
  a = team_max<LPK>(a);
  const long long pos = offset + (offset_dev ? *offset_dev : 0) + s;
  if (!in_range || pos < 0 || pos >= S_max) return;  // a device offset past the buffer writes nothing
  const long long cell = ((long long)b * S_max + pos) * nkv + h;
  float sc;
  const uint2 packed = kv_quant8(f, a, &sc);
  if (sub == 0) (which ? vs : ks)[cell] = sc;
  *reinterpret_cast<uint2*>((which ? vq : kq) + cell * HD + sub * KV_DPL) = packed;
}

// cb_attn_decode_fp8: CTA (split, kv head h, sequence b), 128 threads = TEAMS teams of LPK lanes.  The CTA owns the G
// query heads of kv head h and the key chunk [split * chunk, +chunk) clipped to the valid length L; a chunk wholly past L
// returns before it reads anything.  Each team walks its keys (team, team + TEAMS, ...) BLK at a time: per key one
// 8-byte load of K and of V per lane, G dot products of 8 elements from registers, a team sum, then per head
// score = (dot * ks) * scale and an online softmax in fp32 (one rescale per BLK keys); o += (p * vs) * float(vq).  Keys
// past L or masked out are never loaded.  The teams' (m, l, o) states are merged in team order through shared memory;
// with one split the CTA normalises and stores, otherwise it writes its (m, l, o) to the workspace for
// attn_decode_fp8_combine, which merges the splits in split order.  Fixed orders throughout: bitwise run to run.
constexpr int KVD_THREADS = 128;
constexpr int KVD_MIN_CHUNK = 256;  // keys a split owns at least
constexpr int KVD_MAX_SPLITS = 64;

template <int HD, int G>
__global__ void __launch_bounds__(KVD_THREADS)
attn_decode_fp8_kernel(const bf16* __restrict__ q, long long q_bs, const uint8_t* __restrict__ kq,
                       const uint8_t* __restrict__ vq, const float* __restrict__ ks, const float* __restrict__ vs,
                       const uint8_t* __restrict__ kmask, long long kmask_ld, bf16* __restrict__ o,
                       float* __restrict__ ws, int nkv, int S_max, int chunk, int nsplit, long long length,
                       const long long* __restrict__ length_dev, float scale) {
  constexpr int LPK = HD / KV_DPL;
  constexpr int TEAMS = KVD_THREADS / LPK;
  constexpr int BLK = G <= 4 ? 4 : 2;
  constexpr int ST = HD + 2;  // per-head state: m, l, o[HD]
  __shared__ float red[TEAMS][G][ST];
  const int split = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int nh = nkv * G;
  long long L = length + (length_dev ? *length_dev : 0);
  L = L < (long long)S_max ? L : (long long)S_max;
  const int t0 = split * chunk;
  if (split > 0 && t0 >= L) return;  // split 0 always runs, so an empty cache still yields a defined (zero) output
  const int t1 = (int)(t0 + chunk < L ? t0 + chunk : L);
  const int team = threadIdx.x / LPK, sub = threadIdx.x % LPK;

  float qf[G][8];
#pragma unroll
  for (int g = 0; g < G; ++g)
    unpack8(*reinterpret_cast<const uint4*>(q + (long long)b * q_bs + (h * G + g) * HD + sub * KV_DPL), qf[g]);
  const long long row = (long long)nkv * HD;  // bytes from one position to the next
  const uint8_t* kb = kq + ((long long)b * S_max * nkv + h) * HD + sub * KV_DPL;
  const uint8_t* vb = vq + ((long long)b * S_max * nkv + h) * HD + sub * KV_DPL;
  const float* ksb = ks + (long long)b * S_max * nkv + h;
  const float* vsb = vs + (long long)b * S_max * nkv + h;
  const uint8_t* mb = kmask ? kmask + (long long)b * kmask_ld : nullptr;

  float m[G], l[G], acc[G][8];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    m[g] = -INFINITY;
    l[g] = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[g][e] = 0.f;
  }
  // the trip count is the same for every team (t0, t1 are per CTA), so the team shuffles never diverge
  for (int base = t0; base < t1; base += TEAMS * BLK) {
    uint2 kr[BLK], vr[BLK];
    float ksv[BLK], vsv[BLK];
    unsigned okm = 0u;  // bit j: key j of the block is valid
#pragma unroll
    for (int j = 0; j < BLK; ++j) {
      const int t = base + team + j * TEAMS;
      const bool valid = t < t1 && (!mb || mb[t]);
      okm |= valid ? 1u << j : 0u;
      kr[j] = vr[j] = make_uint2(0u, 0u);
      ksv[j] = vsv[j] = 0.f;
      if (valid) {
        kr[j] = *reinterpret_cast<const uint2*>(kb + t * row);
        vr[j] = *reinterpret_cast<const uint2*>(vb + t * row);
        ksv[j] = ksb[(long long)t * nkv];
        vsv[j] = vsb[(long long)t * nkv];
      }
    }
    float s[BLK][G];
#pragma unroll
    for (int j = 0; j < BLK; ++j) {
      float kf[8];
      e4m3x8_to_f32(kr[j], kf);
#pragma unroll
      for (int g = 0; g < G; ++g) {
        float d = 0.f;
#pragma unroll
        for (int e = 0; e < 8; ++e) d = fmaf(qf[g][e], kf[e], d);
        d = team_sum<LPK>(d);
        s[j][g] = (okm >> j) & 1u ? __fmul_rn(__fmul_rn(d, ksv[j]), scale) : -INFINITY;
      }
    }
    float pv[BLK][G];
#pragma unroll
    for (int g = 0; g < G; ++g) {
      float mx = m[g];
#pragma unroll
      for (int j = 0; j < BLK; ++j) mx = fmaxf(mx, s[j][g]);
      const float c = m[g] == -INFINITY ? 0.f : fast_exp2((m[g] - mx) * KV_LOG2E);
      float ls = __fmul_rn(l[g], c);
#pragma unroll
      for (int j = 0; j < BLK; ++j) {
        const float p = (okm >> j) & 1u ? fast_exp2((s[j][g] - mx) * KV_LOG2E) : 0.f;
        ls += p;
        pv[j][g] = __fmul_rn(p, vsv[j]);
      }
      l[g] = ls;
      m[g] = mx;
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[g][e] = __fmul_rn(acc[g][e], c);
    }
#pragma unroll
    for (int j = 0; j < BLK; ++j) {
      float vf[8];
      e4m3x8_to_f32(vr[j], vf);
#pragma unroll
      for (int g = 0; g < G; ++g)
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[g][e] = fmaf(pv[j][g], vf[e], acc[g][e]);
    }
  }

#pragma unroll
  for (int g = 0; g < G; ++g) {
    if (sub == 0) {
      red[team][g][0] = m[g];
      red[team][g][1] = l[g];
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) red[team][g][2 + sub * KV_DPL + e] = acc[g][e];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < G * HD; i += KVD_THREADS) {
    const int g = i / HD, d = i % HD;
    float M = -INFINITY;
#pragma unroll
    for (int tm = 0; tm < TEAMS; ++tm) M = fmaxf(M, red[tm][g][0]);
    float Ls = 0.f, Os = 0.f;
    if (M != -INFINITY) {
#pragma unroll
      for (int tm = 0; tm < TEAMS; ++tm) {
        const float mt = red[tm][g][0];
        const float w = mt == -INFINITY ? 0.f : fast_exp2((mt - M) * KV_LOG2E);
        Ls = fmaf(red[tm][g][1], w, Ls);
        Os = fmaf(red[tm][g][2 + d], w, Os);
      }
    }
    const long long bh = (long long)b * nh + h * G + g;
    if (nsplit == 1) {
      o[bh * HD + d] = __float2bfloat16(Ls > 0.f ? __fdiv_rn(Os, Ls) : 0.f);
    } else {
      float* w = ws + (bh * nsplit + split) * ST;
      if (d == 0) {
        w[0] = M;
        w[1] = Ls;
      }
      w[2 + d] = Os;
    }
  }
}

// one CTA per (sequence, query head), thread d: the splits that hold valid keys, merged in split order
template <int HD>
__global__ void __launch_bounds__(HD) attn_decode_fp8_combine(const float* __restrict__ ws, bf16* __restrict__ o, int S_max,
                                                              int chunk, int nsplit, long long length,
                                                              const long long* __restrict__ length_dev) {
  constexpr int ST = HD + 2;
  long long L = length + (length_dev ? *length_dev : 0);
  L = L < (long long)S_max ? L : (long long)S_max;
  const int active = L <= 0 ? 0 : (int)((L + chunk - 1) / chunk);
  const long long bh = blockIdx.x;
  const int d = threadIdx.x;
  const float* w = ws + bh * nsplit * ST;
  float M = -INFINITY;
  for (int sp = 0; sp < active; ++sp) M = fmaxf(M, w[sp * ST]);
  float Ls = 0.f, Os = 0.f;
  if (M != -INFINITY) {
    for (int sp = 0; sp < active; ++sp) {
      const float ms = w[sp * ST];
      const float e = ms == -INFINITY ? 0.f : fast_exp2((ms - M) * KV_LOG2E);
      Ls = fmaf(w[sp * ST + 1], e, Ls);
      Os = fmaf(w[sp * ST + 2 + d], e, Os);
    }
  }
  o[bh * HD + d] = __float2bfloat16(Ls > 0.f ? __fdiv_rn(Os, Ls) : 0.f);
}

int kv_fp8_append_launch(const void* k, const void* v, long long ld, void* kq, void* vq, float* ks, float* vs, int B, int S,
                         int S_max, int nkv, int hd, long long offset, const long long* offset_dev, cudaStream_t st) {
  CB_CHECK_ARG(hd == 64 || hd == 128, "kv_fp8_append: hd=%d must be 64 or 128", hd);
  CB_CHECK_ARG(B > 0 && S > 0 && S_max > 0 && nkv > 0, "kv_fp8_append: empty problem (B=%d S=%d S_max=%d nkv=%d)", B, S,
               S_max, nkv);
  CB_CHECK_ARG(k && v && kq && vq && ks && vs, "kv_fp8_append: null argument");
  CB_CHECK_ARG(ld >= (long long)nkv * hd && ld % 8 == 0, "kv_fp8_append: row stride %lld must be >= nkv*hd and a multiple of 8",
               ld);
  CB_CHECK_ARG(((reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v)) & 15u) == 0 &&
                   ((reinterpret_cast<uintptr_t>(kq) | reinterpret_cast<uintptr_t>(vq)) & 7u) == 0 &&
                   ((reinterpret_cast<uintptr_t>(ks) | reinterpret_cast<uintptr_t>(vs)) & 3u) == 0,
               "kv_fp8_append: k, v must be 16-byte aligned, kq, vq 8-byte aligned");
  CB_CHECK_ARG(offset >= 0 && (offset_dev || offset + S <= S_max), "kv_fp8_append: positions [%lld, %lld) outside the cache (%d)",
               offset, offset + S, S_max);
  const long long threads = 2LL * B * S * nkv * (hd / KV_DPL);
  const long long blocks = (threads + 255) / 256;
  CB_CHECK_ARG(blocks < (1LL << 31), "kv_fp8_append: too many rows");
  if (hd == 128)
    kv_fp8_append_kernel<128><<<(unsigned)blocks, 256, 0, st>>>((const bf16*)k, (const bf16*)v, ld, (uint8_t*)kq,
                                                                (uint8_t*)vq, ks, vs, B, S, S_max, nkv, offset, offset_dev);
  else
    kv_fp8_append_kernel<64><<<(unsigned)blocks, 256, 0, st>>>((const bf16*)k, (const bf16*)v, ld, (uint8_t*)kq,
                                                               (uint8_t*)vq, ks, vs, B, S, S_max, nkv, offset, offset_dev);
  CB_CUDA_LAUNCH_CHECK("kv_fp8_append_kernel");
  return CB_OK;
}

// the split count: enough CTAs for about three per SM over (B, nkv), each split at least KVD_MIN_CHUNK keys of S_max
static int kvd_splits(int B, int nkv, int S_max, int* chunk) {
  const long long bk = (long long)B * nkv;
  const long long want = (3LL * device_sm_count() + bk - 1) / bk;
  const long long by_len = (S_max + KVD_MIN_CHUNK - 1) / KVD_MIN_CHUNK;
  int n = (int)std::max(1LL, std::min({want, by_len, (long long)KVD_MAX_SPLITS}));
  *chunk = (S_max + n - 1) / n;
  return (S_max + *chunk - 1) / *chunk;
}

long long attn_decode_fp8_workspace_floats(int B, int nh, int nkv, int S_max, int hd) {
  if (B <= 0 || nh <= 0 || nkv <= 0 || S_max <= 0 || hd <= 0) return 0;
  int chunk;
  const int n = kvd_splits(B, nkv, S_max, &chunk);
  return n > 1 ? (long long)B * nh * n * (hd + 2) : 0;
}

template <int HD>
static void kvd_launch(int G, dim3 grid, cudaStream_t st, const bf16* q, long long q_bs, const uint8_t* kq,
                       const uint8_t* vq, const float* ks, const float* vs, const uint8_t* km, long long km_ld, bf16* o,
                       float* ws, int nkv, int S_max, int chunk, int nsplit, long long length, const long long* length_dev,
                       float scale) {
#define KVD_CASE(GG)                                                                                                     \
  case GG:                                                                                                               \
    attn_decode_fp8_kernel<HD, GG><<<grid, KVD_THREADS, 0, st>>>(q, q_bs, kq, vq, ks, vs, km, km_ld, o, ws, nkv, S_max, \
                                                                 chunk, nsplit, length, length_dev, scale);              \
    break;
  switch (G) {
    KVD_CASE(1) KVD_CASE(2) KVD_CASE(3) KVD_CASE(4) KVD_CASE(5) KVD_CASE(6) KVD_CASE(7) KVD_CASE(8)
  }
#undef KVD_CASE
}

int attn_decode_fp8_launch(const void* q, long long q_bs, const void* kq, const void* vq, const float* ks, const float* vs,
                           const void* kmask, long long kmask_ld, void* o, float* ws, long long ws_floats, int B, int Sq,
                           int nh, int nkv, int S_max, int hd, long long length, const long long* length_dev, float scale,
                           cudaStream_t st) {
  CB_CHECK_ARG(Sq == 1, "attn_decode_fp8: Sq=%d; the decode kernel takes one query per sequence", Sq);
  CB_CHECK_ARG(hd == 64 || hd == 128, "attn_decode_fp8: hd=%d must be 64 or 128", hd);
  CB_CHECK_ARG(B > 0 && B < 65536 && nkv > 0 && nkv < 65536 && S_max > 0, "attn_decode_fp8: bad shape (B=%d nkv=%d S_max=%d)",
               B, nkv, S_max);
  CB_CHECK_ARG(nh % nkv == 0 && nh / nkv >= 1 && nh / nkv <= 8,
               "attn_decode_fp8: nh=%d must be 1..8 times nkv=%d (query heads per kv head)", nh, nkv);
  CB_CHECK_ARG(q && kq && vq && ks && vs && o, "attn_decode_fp8: null argument");
  CB_CHECK_ARG(((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(o)) & 15u) == 0 && q_bs % 8 == 0 &&
                   q_bs >= (long long)nh * hd && ((reinterpret_cast<uintptr_t>(kq) | reinterpret_cast<uintptr_t>(vq)) & 7u) == 0 &&
                   ((reinterpret_cast<uintptr_t>(ks) | reinterpret_cast<uintptr_t>(vs)) & 3u) == 0,
               "attn_decode_fp8: q, o must be 16-byte aligned (q batch stride a multiple of 8), kq, vq 8-byte aligned");
  CB_CHECK_ARG(length >= 0 && (length_dev || length <= S_max), "attn_decode_fp8: length %lld outside the cache (%d)", length,
               S_max);
  CB_CHECK_ARG(!kmask || kmask_ld >= (length_dev ? (long long)S_max : length),
               "attn_decode_fp8: kmask row stride %lld does not cover the valid keys", kmask_ld);
  int chunk;
  const int nsplit = kvd_splits(B, nkv, S_max, &chunk);
  if (nsplit > 1) {
    const long long need = (long long)B * nh * nsplit * (hd + 2);
    CB_CHECK_ARG(ws && ws_floats >= need, "attn_decode_fp8: workspace of %lld floats, %lld needed", ws_floats, need);
  }
  const int G = nh / nkv;
  const dim3 grid(nsplit, nkv, B);
  if (hd == 128)
    kvd_launch<128>(G, grid, st, (const bf16*)q, q_bs, (const uint8_t*)kq, (const uint8_t*)vq, ks, vs, (const uint8_t*)kmask,
                    kmask_ld, (bf16*)o, ws, nkv, S_max, chunk, nsplit, length, length_dev, scale);
  else
    kvd_launch<64>(G, grid, st, (const bf16*)q, q_bs, (const uint8_t*)kq, (const uint8_t*)vq, ks, vs, (const uint8_t*)kmask,
                   kmask_ld, (bf16*)o, ws, nkv, S_max, chunk, nsplit, length, length_dev, scale);
  CB_CUDA_LAUNCH_CHECK("attn_decode_fp8_kernel");
  if (nsplit > 1) {
    if (hd == 128)
      attn_decode_fp8_combine<128><<<B * nh, 128, 0, st>>>(ws, (bf16*)o, S_max, chunk, nsplit, length, length_dev);
    else
      attn_decode_fp8_combine<64><<<B * nh, 64, 0, st>>>(ws, (bf16*)o, S_max, chunk, nsplit, length, length_dev);
    CB_CUDA_LAUNCH_CHECK("attn_decode_fp8_combine");
  }
  return CB_OK;
}

}  // namespace cb
