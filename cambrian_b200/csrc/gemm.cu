// cambrian_b200 — warp-specialised wgmma GEMM for sm_90a (H100).
//
//   C[b] (M x N, row-major)  (+)=  epilogue( alpha * A[b] (M x K) * B[b] (K x N) )
//
// Every dense contraction on the Cambrian hot path goes through this kernel: ViT / ConvNeXt
// linear layers (SURVEY.md §8a A1-A4), the SVA projections (A5, A7), mm_projector (A8), the
// LLaMA q/k/v/o/gate/up/down projections and lm_head (A9, A11) and all of their backward
// GEMMs (dX = dY*W, dW = dY^T*X), which is why both operands can be K-major or MN-major:
//     a_mn = 0 : A stored [M, K] (K contiguous)       a_mn = 1 : A stored [K, M] (M contiguous)
//     b_mn = 0 : B stored [N, K] (nn.Linear weight)   b_mn = 1 : B stored [K, N] (N contiguous)
// wgmma reads either major straight from shared memory (the transpose bits of the instruction), so no layout
// needs a transposed copy.
//
// Structure (persistent: min(tiles, SMs) CTAs of 288 threads, each walking the 128 x BN output tiles
// r = blockIdx.x, + gridDim.x, ...):
//     warp 8      TMA producer   : cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier tx.  The ring's stage and
//                 phase carry across tiles, so the next tile's first k-blocks load while this tile's epilogue runs.
//     warps 0..7  two consumer warpgroups, 64 rows each: wgmma.mma_async 64 x BN x 16 with fp32 accumulators in
//                 registers, one k-block group kept in flight, then bias / act / scale / residual in registers and
//                 the bf16 result through a swizzled smem sub-tile and a TMA store (cp.async.bulk.tensor), which
//                 completes while the warpgroup already runs the next tile's MMAs.
// BN = 64 / 128 / 256 is chosen per problem so that small GEMMs still put a CTA on most of the 132 SMs.
#include "common.cuh"
#include <algorithm>
#include <cstring>
#include <cudaTypedefs.h>
#include <mutex>

namespace cb {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 bf16 = 128 B = one SWIZZLE_128B atom
constexpr int GEMM_THREADS = 288;
constexpr int GROUP_M = 16;  // tile rasterisation: super-rows of 16 m-blocks (2048 rows) keep their A panel L2-resident

struct GemmEpilogue {
  void* C;
  long long ldc, bsc;
  const bf16* bias;      // [N] or null
  const bf16* colscale;  // [N] or null (LayerScale)
  const bf16* residual;  // [M, N] or null
  long long ldr, bsr;
  float alpha;
  int out_fp32;    // C dtype: 0 bf16, 1 fp32
  int accumulate;  // C += result
  int pair_ok;     // two adjacent columns can be loaded / stored as one 4-byte (bf16) / 8-byte (fp32) access
  int tma_store;   // bf16 C addressable by TMA (tmC): stores go through smem; otherwise straight from registers
};
constexpr int ACT_SWIGLU_PAIR = 5;  // the tile's two B halves are BN / 2 gate rows and the matching BN / 2 up rows

// epilogue staging: two 64 x 64 bf16 sub-tiles (SWIZZLE_128B, one TMA store box each) per consumer warpgroup, so one
// can be written while the other's store still reads it
constexpr int STG_BYTES = 64 * 64 * 2;
constexpr int STAGING_BYTES = 2 * 2 * STG_BYTES;

template <int BN>
struct GemmCfg {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = (BN == 256) ? 4 : (BN == 128 ? 6 : 8);  // 192 KB of operands at every BN
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + STAGING_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(SMEM_BYTES <= 232448, "exceeds the 227 KB of shared memory a CTA may use");
};

// activation selected at COMPILE time: a per-element runtime switch (plus slow-path erff / tanhf) made the epilogue of
// short-K GEMMs several times slower than their mainloop
template <int ACT>
__device__ __forceinline__ float apply_act(float v) {
  if constexpr (ACT == 1) return gelu_erf(v);
  else if constexpr (ACT == 2) return gelu_tanh_fast(v);
  else if constexpr (ACT == 3) return quick_gelu(v);
  else if constexpr (ACT == 4) return silu(v);
  else return v;
}

// tile index -> (m block, n block): super-rows of GROUP_M m-blocks (all n-blocks of a super-row before the next one), so
// that a super-row's A panel stays L2-resident while B streams through once per super-row.
__device__ __forceinline__ void tile_to_mn(int r, int m_blocks, int n_blocks, int& mb, int& nb) {
  const int tpg = GROUP_M * n_blocks;
  const int g = r / tpg;
  const int first = g * GROUP_M;
  const int gs = min(GROUP_M, m_blocks - first);
  const int w = r - g * tpg;
  mb = first + w % gs;
  nb = w / gs;
}

// One accumulator row of the tile, this thread's BN / 4 columns (pairs col0 + 8 j, + 1), in place: alpha, bias,
// activation, LayerScale, residual, accumulate (C's old value).  Each fusion is one pass over the row under one test of
// its flag, so that its loads are issued together and no load waits behind a store; the element-wise order of operations
// is the same in every pass, and the caller rounds / stores last.  Needs ep.pair_ok: N is even, so col + 1 < N whenever
// col < N.
template <int BN, int ACT>
__device__ __forceinline__ void fuse_row(const GemmEpilogue& ep, long long c_off, long long r_off, int col0, int N,
                                         float* acc, int h) {
  constexpr int J = BN / 8;
#pragma unroll
  for (int j = 0; j < J; ++j) {
    acc[4 * j + 2 * h] *= ep.alpha;
    acc[4 * j + 2 * h + 1] *= ep.alpha;
  }
  if (ep.bias) {
#pragma unroll
    for (int j = 0; j < J; ++j) {
      const int col = col0 + 8 * j;
      if (col < N) {
        const float2 t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(ep.bias + col));
        acc[4 * j + 2 * h] += t.x;
        acc[4 * j + 2 * h + 1] += t.y;
      }
    }
  }
  if constexpr (ACT != 0) {
#pragma unroll
    for (int j = 0; j < J; ++j) {
      acc[4 * j + 2 * h] = apply_act<ACT>(acc[4 * j + 2 * h]);
      acc[4 * j + 2 * h + 1] = apply_act<ACT>(acc[4 * j + 2 * h + 1]);
    }
  }
  if (ep.colscale) {
#pragma unroll
    for (int j = 0; j < J; ++j) {
      const int col = col0 + 8 * j;
      if (col < N) {
        const float2 t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(ep.colscale + col));
        acc[4 * j + 2 * h] *= t.x;
        acc[4 * j + 2 * h + 1] *= t.y;
      }
    }
  }
  if (ep.residual) {
#pragma unroll
    for (int j = 0; j < J; ++j) {
      const int col = col0 + 8 * j;
      if (col < N) {
        const float2 t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(ep.residual + r_off + col));
        acc[4 * j + 2 * h] += t.x;
        acc[4 * j + 2 * h + 1] += t.y;
      }
    }
  }
  if (ep.accumulate && ep.out_fp32) {
    const float* cr = reinterpret_cast<const float*>(ep.C) + c_off;
#pragma unroll
    for (int j = 0; j < J; ++j) {
      const int col = col0 + 8 * j;
      if (col < N) {
        const float2 o = *reinterpret_cast<const float2*>(cr + col);
        acc[4 * j + 2 * h] += o.x;
        acc[4 * j + 2 * h + 1] += o.y;
      }
    }
  } else if (ep.accumulate) {
    const bf16* cr = reinterpret_cast<const bf16*>(ep.C) + c_off;
#pragma unroll
    for (int j = 0; j < J; ++j) {
      const int col = col0 + 8 * j;
      if (col < N) {
        const float2 o = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(cr + col));
        acc[4 * j + 2 * h] += o.x;
        acc[4 * j + 2 * h + 1] += o.y;
      }
    }
  }
}

// the register-path store of a row fused by fuse_row (fp32 C, or bf16 C that TMA cannot address)
template <int BN>
__device__ __forceinline__ void store_row(const GemmEpilogue& ep, long long c_off, int col0, int N, const float* acc,
                                          int h) {
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = col0 + 8 * j;
    if (col >= N) continue;
    const float x = acc[4 * j + 2 * h], y = acc[4 * j + 2 * h + 1];
    if (ep.out_fp32) *reinterpret_cast<float2*>(reinterpret_cast<float*>(ep.C) + c_off + col) = make_float2(x, y);
    else *reinterpret_cast<__nv_bfloat162*>(reinterpret_cast<bf16*>(ep.C) + c_off + col) = __floats2bfloat162_rn(x, y);
  }
}

// odd N or a misaligned operand: the same operations element by element (columns col, col + 1 of one row)
template <int ACT>
__device__ __forceinline__ void epilogue_elems(const GemmEpilogue& ep, long long c_off, long long r_off, int col, int N,
                                               float v0, float v1) {
  v0 *= ep.alpha;
  v1 *= ep.alpha;
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int c = col + e;
    if (c >= N) break;
    float v = e ? v1 : v0;
    if (ep.bias) v += __bfloat162float(ep.bias[c]);
    v = apply_act<ACT>(v);
    if (ep.colscale) v *= __bfloat162float(ep.colscale[c]);
    if (ep.residual) v += __bfloat162float(ep.residual[r_off + c]);
    if (ep.out_fp32) {
      float* cp = reinterpret_cast<float*>(ep.C) + c_off + c;
      *cp = ep.accumulate ? *cp + v : v;
    } else {
      bf16* cp = reinterpret_cast<bf16*>(ep.C) + c_off + c;
      *cp = __float2bfloat16(ep.accumulate ? __bfloat162float(*cp) + v : v);
    }
  }
}

template <int BN, bool A_MN, bool B_MN, int ACT>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_wgmma(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmAux, int M, int N, int K,
                int tiles, GemmEpilogue ep) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr bool SWIGLU = ACT == ACT_SWIGLU_PAIR;
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B tiles need 1024-byte aligned bases
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t stg_base = smem_base + STAGES * Cfg::STAGE_BYTES;
  const uint32_t bar_base = stg_base + STAGING_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // SwiGLU: N = 2F columns, one tile = BN / 2 features (BN / 2 gate + BN / 2 up columns)
  const int m_blocks = (M + BM - 1) / BM;
  const int n_blocks = SWIGLU ? (N / 2) / (BN / 2) : (N + BN - 1) / BN;
  const int tiles_per_batch = m_blocks * n_blocks;
  const int num_kb = (K + BK - 1) / BK;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);  // one arrive per consumer warpgroup
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ============================ TMA producer ============================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int r = blockIdx.x; r < tiles; r += gridDim.x) {
        const int b = r / tiles_per_batch;
        int mb, nb;
        tile_to_mn(r - b * tiles_per_batch, m_blocks, n_blocks, mb, nb);
        const int m0 = mb * BM;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(empty_bar(stage), phase ^ 1u);
          const uint32_t sa = smem_base + stage * Cfg::STAGE_BYTES;
          const uint32_t sb = sa + Cfg::A_BYTES;
          mbar_arrive_expect_tx(full_bar(stage), Cfg::STAGE_BYTES);
          const int k0 = kb * BK;
          if (!A_MN) {
            tma_load_3d(sa, &tmA, full_bar(stage), k0, m0, b);
          } else {
#pragma unroll
            for (int i = 0; i < BM / 64; ++i)
              tma_load_3d(sa + i * (64 * BK * 2), &tmA, full_bar(stage), m0 + 64 * i, k0, b);
          }
          if (SWIGLU) {  // gate rows [nb BN/2, +BN/2) and up rows [F + nb BN/2, +BN/2)
            tma_load_3d(sb, &tmB, full_bar(stage), k0, nb * (BN / 2), 0);
            tma_load_3d(sb + (BN / 2) * BK * 2, &tmB, full_bar(stage), k0, N / 2 + nb * (BN / 2), 0);
          } else if (!B_MN) {
            tma_load_3d(sb, &tmB, full_bar(stage), k0, nb * BN, b);
          } else {
#pragma unroll
            for (int i = 0; i < BN / 64; ++i)
              tma_load_3d(sb + i * (64 * BK * 2), &tmB, full_bar(stage), nb * BN + 64 * i, k0, b);
          }
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1u;
          }
        }
      }
    }
    return;
  }

  // ============================ consumer warpgroups ============================
  const int wg = warp >> 2;  // rows [64 wg, +64) of the tile
  const bool wg_leader = (threadIdx.x & 127) == 0;
  const int srow = (warp & 3) * 16 + (lane >> 2);  // this thread's first row within the warpgroup's 64
  const int cq = 2 * (lane & 3);
  const uint32_t stg = stg_base + wg * (2 * STG_BYTES);
  uint32_t q = 0;  // sub-tiles this warpgroup has staged: selects the buffer
  if (wg_leader && ep.tma_store) {
    tma_prefetch_desc(&tmC);
    if (SWIGLU) tma_prefetch_desc(&tmAux);
  }

  // One 64 x 64 bf16 sub-tile of the warpgroup's rows through smem: pair(j, h) is the bf16x2 at columns 8 j + cq, + 1
  // of the thread's row srow + 8 h.  SWIZZLE_128B puts a row's 16-byte chunk c at c ^ (row & 7), so the 8 rows x 4
  // quads of one warp write hit all 32 banks once.  The other buffer's store must have read it out before the barrier
  // lets anyone write there; stores with a box wholly outside C (x >= x_end, y >= M) are skipped.
  auto store_subtile = [&](const CUtensorMap* map, int x, int x_end, int y, int z, auto pair) {
    const uint32_t buf = stg + (q & 1u) * STG_BYTES;
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
    if (wg_leader && x < x_end && y < M) {
      tma_store_3d(map, buf, x, y, z);
      bulk_commit();
    }
    ++q;
  };

  float acc[BN / 2];
  int stage = 0;
  uint32_t phase = 0;
  for (int r = blockIdx.x; r < tiles; r += gridDim.x) {
    const int b = r / tiles_per_batch;
    int mb, nb;
    tile_to_mn(r - b * tiles_per_batch, m_blocks, n_blocks, mb, nb);
    const int m0 = mb * BM;
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int prev_stage = -1;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(full_bar(stage), phase);
      const uint32_t sa = smem_base + stage * Cfg::STAGE_BYTES + wg * (64 * 128);
      const uint32_t sb = smem_base + stage * Cfg::STAGE_BYTES + Cfg::A_BYTES;
      reg_fence(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        const uint64_t adesc = A_MN ? make_smem_desc_sw128(sa + k * 2048, 64 * BK * 2, 1024)
                                    : make_smem_desc_sw128(sa + k * 32, 0, 1024);
        const uint64_t bdesc = B_MN ? make_smem_desc_sw128(sb + k * 2048, 64 * BK * 2, 1024)
                                    : make_smem_desc_sw128(sb + k * 32, 0, 1024);
        WgmmaSS<BN, A_MN ? 1 : 0, B_MN ? 1 : 0>::mma(acc, adesc, bdesc, 1u);
      }
      wgmma_commit();
      wgmma_wait<1>();  // the previous k-block's MMAs have retired: its stage can be refilled
      reg_fence(acc);
      if (prev_stage >= 0 && wg_leader) mbar_arrive(empty_bar(prev_stage));
      prev_stage = stage;
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1u;
      }
    }
    wgmma_wait<0>();
    reg_fence(acc);
    if (wg_leader) mbar_arrive(empty_bar(prev_stage));  // the producer is already filling it with the next tile

    // ============================ epilogue ============================
    const int y0 = m0 + wg * 64;
    if constexpr (SWIGLU) {
      // accumulator columns [0, BN/2) = gate, [BN/2, BN) = up of the same BN/2 features: write both pre-activations
      // (saved for backward) and silu(gate) * up without a second pass over the [M, 2F] tensor
      constexpr int JH = BN / 16;  // 8-column groups per half
      const int F = N >> 1;
      const int f0 = nb * (BN / 2);
#pragma unroll
      for (int s = 0; s < BN / 128; ++s)
        store_subtile(&tmC, f0 + 64 * s, N, y0, 0, [&](int j, int h) {
          return __floats2bfloat162_rn(acc[4 * (8 * s + j) + 2 * h], acc[4 * (8 * s + j) + 2 * h + 1]);
        });
#pragma unroll
      for (int s = 0; s < BN / 128; ++s)
        store_subtile(&tmC, F + f0 + 64 * s, N, y0, 0, [&](int j, int h) {
          return __floats2bfloat162_rn(acc[4 * (JH + 8 * s + j) + 2 * h], acc[4 * (JH + 8 * s + j) + 2 * h + 1]);
        });
#pragma unroll
      for (int s = 0; s < BN / 128; ++s)
        store_subtile(&tmAux, f0 + 64 * s, F, y0, 0, [&](int j, int h) {
          // round to bf16 first: the separate kernels (and the reference) apply silu to the STORED pre-activations
          const float2 g = __bfloat1622float2(
              __floats2bfloat162_rn(acc[4 * (8 * s + j) + 2 * h], acc[4 * (8 * s + j) + 2 * h + 1]));
          const float2 u = __bfloat1622float2(
              __floats2bfloat162_rn(acc[4 * (JH + 8 * s + j) + 2 * h], acc[4 * (JH + 8 * s + j) + 2 * h + 1]));
          return __floats2bfloat162_rn(silu(g.x) * u.x, silu(g.y) * u.y);
        });
    } else {
      const int n0 = nb * BN;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = y0 + srow + 8 * h;
        if (row >= M) continue;
        const long long c_off = static_cast<long long>(b) * ep.bsc + static_cast<long long>(row) * ep.ldc;
        const long long r_off = static_cast<long long>(b) * ep.bsr + static_cast<long long>(row) * ep.ldr;
        if (ep.pair_ok) {
          fuse_row<BN, ACT>(ep, c_off, r_off, n0 + cq, N, acc, h);
          if (!ep.tma_store) store_row<BN>(ep, c_off, n0 + cq, N, acc, h);
          continue;
        }
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          if (n0 + 8 * j >= N) break;
          epilogue_elems<ACT>(ep, c_off, r_off, n0 + 8 * j + cq, N, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
      }
      if (ep.tma_store) {
#pragma unroll
        for (int s = 0; s < BN / 64; ++s)
          store_subtile(&tmC, n0 + 64 * s, N, y0, b, [&](int j, int h) {
            return __floats2bfloat162_rn(acc[4 * (8 * s + j) + 2 * h], acc[4 * (8 * s + j) + 2 * h + 1]);
          });
      }
    }
  }
  if (wg_leader) bulk_wait<0>();  // the CTA's smem must outlive the stores that read it
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
static PFN_cuTensorMapEncodeTiled_v12000 get_encode_fn() {
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

// 3-D bf16 tensor map: dims (inner, rows, batch), box (64, box_rows, 1), SWIZZLE_128B
int make_tmap_bf16_3d(CUtensorMap* out, const void* base, uint64_t inner, uint64_t rows, uint64_t batch,
                      uint64_t ld_elems, uint64_t batch_stride_elems, uint32_t box_rows) {
  auto fn = get_encode_fn();
  if (!fn) return set_error(CB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  if ((reinterpret_cast<uintptr_t>(base) & 15u) != 0)
    return set_error(CB_ERR_INVALID, "TMA operand base must be 16-byte aligned");
  if ((ld_elems % 8) != 0 || (batch > 1 && (batch_stride_elems % 8) != 0))
    return set_error(CB_ERR_INVALID, "TMA operand strides must be multiples of 8 elements (ld=%llu)",
                     (unsigned long long)ld_elems);
  cuuint64_t dims[3] = {inner, rows, batch};
  cuuint64_t bs = (batch > 1) ? batch_stride_elems * 2 : ld_elems * 2 * (rows ? rows : 1);
  cuuint64_t strides[2] = {ld_elems * 2, bs};
  cuuint32_t box[3] = {64, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box,
                  estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r == CUDA_ERROR_INVALID_CONTEXT) {
    // a thread that has only used the runtime lazily (e.g. PyTorch's autograd worker) has no driver context bound yet:
    // bind the primary context of its current device and retry
    cudaFree(0);
    r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  if (r != CUDA_SUCCESS) return set_error(CB_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
  return CB_OK;
}

// operand maps (A, B) and, for the TMA-store epilogue, the output maps (C, SwiGLU's second output); 64 x 64 store boxes
struct GemmMaps {
  CUtensorMap a, b, c, aux;
};

template <int BN, bool A_MN, bool B_MN, int ACT>
static int launch_gemm(const GemmMaps& tm, int M, int N, int K, int batch, const GemmEpilogue& ep,
                       cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  auto kern = gemm_bf16_wgmma<BN, A_MN, B_MN, ACT>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
    if (e != cudaSuccess) return set_error(CB_ERR_CUDA, "gemm smem attr: %s", cudaGetErrorString(e));
    attr_set = true;
  }
  const int n_blocks = (ACT == ACT_SWIGLU_PAIR) ? (N / 2) / (BN / 2) : (N + BN - 1) / BN;
  const long long tiles = (long long)((M + BM - 1) / BM) * n_blocks * batch;
  CB_CHECK_ARG(tiles < (1LL << 31), "gemm: %lld tiles exceed the grid", tiles);
  const unsigned grid = (unsigned)std::min<long long>(tiles, device_sm_count());
  kern<<<grid, GEMM_THREADS, Cfg::SMEM_BYTES, stream>>>(tm.a, tm.b, tm.c, tm.aux, M, N, K, (int)tiles, ep);
  CB_CUDA_LAUNCH_CHECK("gemm_bf16_wgmma");
  return CB_OK;
}

template <int BN>
static int dispatch_major(int a_mn, int b_mn, int act, const GemmMaps& tm, int M, int N, int K, int batch,
                          const GemmEpilogue& ep, cudaStream_t stream) {
  if (!a_mn && !b_mn) {
    switch (act) {
      case 1: return launch_gemm<BN, false, false, 1>(tm, M, N, K, batch, ep, stream);
      case 2: return launch_gemm<BN, false, false, 2>(tm, M, N, K, batch, ep, stream);
      case 3: return launch_gemm<BN, false, false, 3>(tm, M, N, K, batch, ep, stream);
      case 4: return launch_gemm<BN, false, false, 4>(tm, M, N, K, batch, ep, stream);
      default: return launch_gemm<BN, false, false, 0>(tm, M, N, K, batch, ep, stream);
    }
  }
  if (!a_mn && b_mn) return launch_gemm<BN, false, true, 0>(tm, M, N, K, batch, ep, stream);
  if (a_mn && !b_mn) return launch_gemm<BN, true, false, 0>(tm, M, N, K, batch, ep, stream);
  return launch_gemm<BN, true, true, 0>(tm, M, N, K, batch, ep, stream);
}

int gemm_bf16(const void* A, const void* B, void* C, int M, int N, int K, int batch, long long lda,
              long long ldb, long long ldc, long long bsa, long long bsb, long long bsc, int a_mn, int b_mn,
              const void* bias, const void* colscale, const void* residual, long long ldr, long long bsr,
              float alpha, int act, int out_fp32, int accumulate, int force_bn, cudaStream_t stream) {
  CB_CHECK_ARG(M > 0 && N > 0 && K > 0 && batch > 0, "gemm: empty problem M=%d N=%d K=%d batch=%d", M, N, K,
               batch);
  CB_CHECK_ARG(A && B && C, "gemm: null operand");
  CB_CHECK_ARG(act >= 0 && act <= 4, "gemm: unknown activation %d", act);
  CB_CHECK_ARG(act == 0 || (!a_mn && !b_mn), "gemm: a fused activation needs K-major operands (forward layout)");
  CB_CHECK_ARG(force_bn == 0 || force_bn == 64 || force_bn == 128 || force_bn == 256, "gemm: bad BLOCK_N %d", force_bn);
  int bn = force_bn;
  if (bn == 0) {
    // the widest tile that still gives most SMs a CTA: wide tiles halve the operand traffic per FLOP, but a GEMM of
    // fewer tiles than SMs leaves the rest of the chip idle
    const int sms = device_sm_count();
    const long long mb = (M + BM - 1) / BM;
    auto tiles = [&](int b_n) { return mb * ((N + b_n - 1) / b_n) * batch; };
    if (N > 128 && tiles(256) >= (long long)(sms * 7) / 10) bn = 256;
    else if (N > 64 && tiles(128) >= (long long)(sms * 6) / 10) bn = 128;
    else if (N > 128 && tiles(64) > 2LL * sms) bn = 128;
    else bn = 64;
  }
  GemmMaps tm;
  std::memset(&tm, 0, sizeof(tm));
  int rc;
  if (!a_mn) rc = make_tmap_bf16_3d(&tm.a, A, K, M, batch, lda, bsa, BM);
  else       rc = make_tmap_bf16_3d(&tm.a, A, M, K, batch, lda, bsa, BK);
  if (rc) return rc;
  if (!b_mn) rc = make_tmap_bf16_3d(&tm.b, B, K, N, batch, ldb, bsb, bn);
  else       rc = make_tmap_bf16_3d(&tm.b, B, N, K, batch, ldb, bsb, BK);
  if (rc) return rc;
  GemmEpilogue ep;
  ep.C = C; ep.ldc = ldc; ep.bsc = bsc;
  ep.bias = static_cast<const bf16*>(bias);
  ep.colscale = static_cast<const bf16*>(colscale);
  ep.residual = static_cast<const bf16*>(residual);
  ep.ldr = ldr; ep.bsr = bsr;
  ep.alpha = alpha; ep.out_fp32 = out_fp32; ep.accumulate = accumulate;
  const unsigned calign = out_fp32 ? 7u : 3u;
  bool pair = (N % 2 == 0) && (ldc % 2 == 0) && (bsc % 2 == 0) && ((reinterpret_cast<uintptr_t>(C) & calign) == 0);
  if (residual)
    pair = pair && (ldr % 2 == 0) && (bsr % 2 == 0) && ((reinterpret_cast<uintptr_t>(residual) & 3u) == 0);
  if (bias) pair = pair && ((reinterpret_cast<uintptr_t>(bias) & 3u) == 0);
  if (colscale) pair = pair && ((reinterpret_cast<uintptr_t>(colscale) & 3u) == 0);
  ep.pair_ok = pair ? 1 : 0;
  // bf16 C whose base and strides TMA can address takes the smem + TMA-store epilogue; fp32 C, and views at an odd
  // element offset or stride, store from registers
  const bool tma = pair && !out_fp32 && ((reinterpret_cast<uintptr_t>(C) & 15u) == 0) && ldc % 8 == 0 &&
                   (batch == 1 || (bsc > 0 && bsc % 8 == 0));
  if (tma && (rc = make_tmap_bf16_3d(&tm.c, C, N, M, batch, ldc, bsc, 64))) return rc;
  ep.tma_store = tma ? 1 : 0;
  switch (bn) {
    case 256: return dispatch_major<256>(a_mn, b_mn, act, tm, M, N, K, batch, ep, stream);
    case 128: return dispatch_major<128>(a_mn, b_mn, act, tm, M, N, K, batch, ep, stream);
    default:  return dispatch_major<64>(a_mn, b_mn, act, tm, M, N, K, batch, ep, stream);
  }
}

// gate/up projection + SwiGLU in one GEMM.  A [M, K] (lda), W = [gate_proj; up_proj] [2F, K] (ldw);
// gu_out [M, 2F] (ld_gu) receives the bf16 pre-activations, act_out [M, F] (ld_act) silu(gate) * up.
int gemm_swiglu_bf16(const void* A, const void* W, void* gu_out, void* act_out, int M, int F, int K, long long lda,
                     long long ldw, long long ld_gu, long long ld_act, cudaStream_t stream) {
  CB_CHECK_ARG(M > 0 && F > 0 && K > 0, "gemm_swiglu: empty problem M=%d F=%d K=%d", M, F, K);
  CB_CHECK_ARG(A && W && gu_out && act_out, "gemm_swiglu: null operand");
  CB_CHECK_ARG(F % 128 == 0, "gemm_swiglu: F=%d must be a multiple of 128 (whole 128-feature tiles, 16-byte aligned halves)", F);
  CB_CHECK_ARG(ld_gu % 8 == 0 && ld_act % 8 == 0 && ((reinterpret_cast<uintptr_t>(gu_out) & 15u) == 0) &&
                   ((reinterpret_cast<uintptr_t>(act_out) & 15u) == 0),
               "gemm_swiglu: outputs must be 16-byte aligned with ld %% 8 == 0");
  const int N = 2 * F;
  // 128 gate + 128 up features per tile: the same 128 x 256 tile and operand traffic per FLOP as the generic BN = 256
  // kernel (a 64 + 64 tile reads 32 KB of operands per 64-deep k-block for half the FLOPs of a 48 KB 128 x 256 k-block)
  constexpr int BN = 256;
  GemmMaps tm;
  int rc;
  if ((rc = make_tmap_bf16_3d(&tm.a, A, K, M, 1, lda, 0, BM))) return rc;
  if ((rc = make_tmap_bf16_3d(&tm.b, W, K, N, 1, ldw, 0, BN / 2))) return rc;
  if ((rc = make_tmap_bf16_3d(&tm.c, gu_out, N, M, 1, ld_gu, 0, 64))) return rc;
  if ((rc = make_tmap_bf16_3d(&tm.aux, act_out, F, M, 1, ld_act, 0, 64))) return rc;
  GemmEpilogue ep;
  ep.C = gu_out; ep.ldc = ld_gu; ep.bsc = 0;
  ep.bias = nullptr; ep.colscale = nullptr; ep.residual = nullptr; ep.ldr = 0; ep.bsr = 0;
  ep.alpha = 1.0f; ep.out_fp32 = 0; ep.accumulate = 0; ep.pair_ok = 1; ep.tma_store = 1;
  return launch_gemm<BN, false, false, ACT_SWIGLU_PAIR>(tm, M, N, K, 1, ep, stream);
}

}  // namespace cb
