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
// Structure (one CTA per 128 x BN output tile, 288 threads):
//     warp 8      TMA producer   : cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier tx
//     warps 0..7  two consumer warpgroups, 64 rows each: wgmma.mma_async 64 x BN x 16 with fp32 accumulators in
//                 registers, one k-block group kept in flight, then bias / act / scale / residual -> HBM
// BN = 64 / 128 / 256 is chosen per problem so that small GEMMs still put a CTA on most of the 132 SMs.
#include "common.cuh"
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
  void* aux;       // fused SwiGLU: second output, silu(gate) * up, [M, N / 2] bf16
  long long ld_aux;
};
constexpr int ACT_SWIGLU_PAIR = 5;  // the tile's two B halves are 64 gate rows and the matching 64 up rows

template <int BN>
struct GemmCfg {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = (BN == 256) ? 4 : (BN == 128 ? 6 : 8);
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
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

// one output element pair (columns col, col + 1 of one row): alpha, bias, activation, LayerScale, residual, accumulate
template <int ACT>
__device__ __forceinline__ void epilogue_pair(const GemmEpilogue& ep, long long c_off, long long r_off, int col, int N,
                                              float v0, float v1) {
  v0 *= ep.alpha;
  v1 *= ep.alpha;
  if (ep.pair_ok) {
    if (col >= N) return;  // N is even here, so col + 1 < N as well
    if (ep.bias) {
      const float2 t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(ep.bias + col));
      v0 += t.x;
      v1 += t.y;
    }
    v0 = apply_act<ACT>(v0);
    v1 = apply_act<ACT>(v1);
    if (ep.colscale) {
      const float2 t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(ep.colscale + col));
      v0 *= t.x;
      v1 *= t.y;
    }
    if (ep.residual) {
      const float2 t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(ep.residual + r_off + col));
      v0 += t.x;
      v1 += t.y;
    }
    if (ep.out_fp32) {
      float2* cp = reinterpret_cast<float2*>(reinterpret_cast<float*>(ep.C) + c_off + col);
      if (ep.accumulate) {
        const float2 o = *cp;
        v0 += o.x;
        v1 += o.y;
      }
      *cp = make_float2(v0, v1);
    } else {
      __nv_bfloat162* cp = reinterpret_cast<__nv_bfloat162*>(reinterpret_cast<bf16*>(ep.C) + c_off + col);
      if (ep.accumulate) {
        const float2 o = __bfloat1622float2(*cp);
        v0 += o.x;
        v1 += o.y;
      }
      *cp = __floats2bfloat162_rn(v0, v1);
    }
    return;
  }
#pragma unroll
  for (int e = 0; e < 2; ++e) {  // odd N or a misaligned operand: element by element
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
gemm_bf16_wgmma(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, int M, int N, int K,
                GemmEpilogue ep) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr bool SWIGLU = ACT == ACT_SWIGLU_PAIR;
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B tiles need 1024-byte aligned bases
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + STAGES * Cfg::STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // SwiGLU: N = 2F columns, one tile = 64 features (64 gate + 64 up columns)
  const int m_blocks = (M + BM - 1) / BM;
  const int n_blocks = SWIGLU ? (N / 2) / 64 : (N + BN - 1) / BN;
  const int tiles_per_batch = m_blocks * n_blocks;
  const int b = blockIdx.x / tiles_per_batch;
  int mb, nb;
  tile_to_mn(blockIdx.x - b * tiles_per_batch, m_blocks, n_blocks, mb, nb);
  const int m0 = mb * BM;
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
          for (int i = 0; i < BM / 64; ++i) tma_load_3d(sa + i * (64 * BK * 2), &tmA, full_bar(stage), m0 + 64 * i, k0, b);
        }
        if (SWIGLU) {  // gate rows [64 nb, +64) and up rows [F + 64 nb, +64)
          tma_load_3d(sb, &tmB, full_bar(stage), k0, nb * 64, 0);
          tma_load_3d(sb + 64 * BK * 2, &tmB, full_bar(stage), k0, N / 2 + nb * 64, 0);
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
    return;
  }

  // ============================ consumer warpgroups ============================
  const int wg = warp >> 2;  // rows [64 wg, +64) of the tile
  const bool wg_leader = (threadIdx.x & 127) == 0;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  int stage = 0;
  uint32_t phase = 0;
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

  // ============================ epilogue ============================
  const int r_lo = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  if constexpr (SWIGLU) {
    // accumulator columns [0, 64) = gate, [64, 128) = up of the same 64 features: write both pre-activations (saved for
    // backward) and silu(gate) * up without a second pass over the [M, 2F] tensor
    const int F = N >> 1;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = r_lo + 8 * h;
      if (row >= M) continue;
      bf16* gu = reinterpret_cast<bf16*>(ep.C) + static_cast<long long>(row) * ep.ldc;
      bf16* ao = reinterpret_cast<bf16*>(ep.aux) + static_cast<long long>(row) * ep.ld_aux;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int f = nb * 64 + 8 * j + cq;
        // round to bf16 first: the separate kernels (and the reference) apply silu to the STORED bf16 pre-activations
        const __nv_bfloat162 g2 = __floats2bfloat162_rn(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        const __nv_bfloat162 u2 = __floats2bfloat162_rn(acc[4 * (j + 8) + 2 * h], acc[4 * (j + 8) + 2 * h + 1]);
        const float2 g = __bfloat1622float2(g2), u = __bfloat1622float2(u2);
        *reinterpret_cast<__nv_bfloat162*>(gu + f) = g2;
        *reinterpret_cast<__nv_bfloat162*>(gu + F + f) = u2;
        *reinterpret_cast<__nv_bfloat162*>(ao + f) = __floats2bfloat162_rn(silu(g.x) * u.x, silu(g.y) * u.y);
      }
    }
  } else {
    const int n0 = nb * BN;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = r_lo + 8 * h;
      if (row >= M) continue;
      const long long c_off = static_cast<long long>(b) * ep.bsc + static_cast<long long>(row) * ep.ldc;
      const long long r_off = static_cast<long long>(b) * ep.bsr + static_cast<long long>(row) * ep.ldr;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = n0 + 8 * j + cq;
        if (n0 + 8 * j >= N) break;
        epilogue_pair<ACT>(ep, c_off, r_off, col, N, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
      }
    }
  }
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

template <int BN, bool A_MN, bool B_MN, int ACT>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, int M, int N, int K, int batch,
                       const GemmEpilogue& ep, cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  auto kern = gemm_bf16_wgmma<BN, A_MN, B_MN, ACT>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
    if (e != cudaSuccess) return set_error(CB_ERR_CUDA, "gemm smem attr: %s", cudaGetErrorString(e));
    attr_set = true;
  }
  const int n_blocks = (ACT == ACT_SWIGLU_PAIR) ? (N / 2) / 64 : (N + BN - 1) / BN;
  const long long tiles = (long long)((M + BM - 1) / BM) * n_blocks * batch;
  CB_CHECK_ARG(tiles < (1LL << 31), "gemm: %lld tiles exceed the grid", tiles);
  kern<<<(unsigned)tiles, GEMM_THREADS, Cfg::SMEM_BYTES, stream>>>(tmA, tmB, M, N, K, ep);
  CB_CUDA_LAUNCH_CHECK("gemm_bf16_wgmma");
  return CB_OK;
}

template <int BN>
static int dispatch_major(int a_mn, int b_mn, int act, const CUtensorMap& tmA, const CUtensorMap& tmB, int M, int N,
                          int K, int batch, const GemmEpilogue& ep, cudaStream_t stream) {
  if (!a_mn && !b_mn) {
    switch (act) {
      case 1: return launch_gemm<BN, false, false, 1>(tmA, tmB, M, N, K, batch, ep, stream);
      case 2: return launch_gemm<BN, false, false, 2>(tmA, tmB, M, N, K, batch, ep, stream);
      case 3: return launch_gemm<BN, false, false, 3>(tmA, tmB, M, N, K, batch, ep, stream);
      case 4: return launch_gemm<BN, false, false, 4>(tmA, tmB, M, N, K, batch, ep, stream);
      default: return launch_gemm<BN, false, false, 0>(tmA, tmB, M, N, K, batch, ep, stream);
    }
  }
  if (!a_mn && b_mn) return launch_gemm<BN, false, true, 0>(tmA, tmB, M, N, K, batch, ep, stream);
  if (a_mn && !b_mn) return launch_gemm<BN, true, false, 0>(tmA, tmB, M, N, K, batch, ep, stream);
  return launch_gemm<BN, true, true, 0>(tmA, tmB, M, N, K, batch, ep, stream);
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
  CUtensorMap tmA, tmB;
  int rc;
  if (!a_mn) rc = make_tmap_bf16_3d(&tmA, A, K, M, batch, lda, bsa, BM);
  else       rc = make_tmap_bf16_3d(&tmA, A, M, K, batch, lda, bsa, BK);
  if (rc) return rc;
  if (!b_mn) rc = make_tmap_bf16_3d(&tmB, B, K, N, batch, ldb, bsb, bn);
  else       rc = make_tmap_bf16_3d(&tmB, B, N, K, batch, ldb, bsb, BK);
  if (rc) return rc;
  GemmEpilogue ep;
  ep.C = C; ep.ldc = ldc; ep.bsc = bsc;
  ep.bias = static_cast<const bf16*>(bias);
  ep.colscale = static_cast<const bf16*>(colscale);
  ep.residual = static_cast<const bf16*>(residual);
  ep.ldr = ldr; ep.bsr = bsr;
  ep.alpha = alpha; ep.out_fp32 = out_fp32; ep.accumulate = accumulate;
  ep.aux = nullptr; ep.ld_aux = 0;
  const unsigned calign = out_fp32 ? 7u : 3u;
  bool pair = (N % 2 == 0) && (ldc % 2 == 0) && (bsc % 2 == 0) && ((reinterpret_cast<uintptr_t>(C) & calign) == 0);
  if (residual)
    pair = pair && (ldr % 2 == 0) && (bsr % 2 == 0) && ((reinterpret_cast<uintptr_t>(residual) & 3u) == 0);
  if (bias) pair = pair && ((reinterpret_cast<uintptr_t>(bias) & 3u) == 0);
  if (colscale) pair = pair && ((reinterpret_cast<uintptr_t>(colscale) & 3u) == 0);
  ep.pair_ok = pair ? 1 : 0;
  switch (bn) {
    case 256: return dispatch_major<256>(a_mn, b_mn, act, tmA, tmB, M, N, K, batch, ep, stream);
    case 128: return dispatch_major<128>(a_mn, b_mn, act, tmA, tmB, M, N, K, batch, ep, stream);
    default:  return dispatch_major<64>(a_mn, b_mn, act, tmA, tmB, M, N, K, batch, ep, stream);
  }
}

// gate/up projection + SwiGLU in one GEMM.  A [M, K] (lda), W = [gate_proj; up_proj] [2F, K] (ldw);
// gu_out [M, 2F] (ld_gu) receives the bf16 pre-activations, act_out [M, F] (ld_act) silu(gate) * up.
int gemm_swiglu_bf16(const void* A, const void* W, void* gu_out, void* act_out, int M, int F, int K, long long lda,
                     long long ldw, long long ld_gu, long long ld_act, cudaStream_t stream) {
  CB_CHECK_ARG(M > 0 && F > 0 && K > 0, "gemm_swiglu: empty problem M=%d F=%d K=%d", M, F, K);
  CB_CHECK_ARG(A && W && gu_out && act_out, "gemm_swiglu: null operand");
  CB_CHECK_ARG(F % 128 == 0, "gemm_swiglu: F=%d must be a multiple of 128 (whole 64-feature tiles, 16-byte aligned halves)", F);
  CB_CHECK_ARG(ld_gu % 8 == 0 && ld_act % 8 == 0 && ((reinterpret_cast<uintptr_t>(gu_out) & 15u) == 0) &&
                   ((reinterpret_cast<uintptr_t>(act_out) & 15u) == 0),
               "gemm_swiglu: outputs must be 16-byte aligned with ld %% 8 == 0");
  const int N = 2 * F;
  CUtensorMap tmA, tmB;
  int rc;
  if ((rc = make_tmap_bf16_3d(&tmA, A, K, M, 1, lda, 0, BM))) return rc;
  if ((rc = make_tmap_bf16_3d(&tmB, W, K, N, 1, ldw, 0, 64))) return rc;
  GemmEpilogue ep;
  ep.C = gu_out; ep.ldc = ld_gu; ep.bsc = 0;
  ep.bias = nullptr; ep.colscale = nullptr; ep.residual = nullptr; ep.ldr = 0; ep.bsr = 0;
  ep.alpha = 1.0f; ep.out_fp32 = 0; ep.accumulate = 0; ep.pair_ok = 1;
  ep.aux = act_out; ep.ld_aux = ld_act;
  return launch_gemm<128, false, false, ACT_SWIGLU_PAIR>(tmA, tmB, M, N, K, 1, ep, stream);
}

}  // namespace cb
