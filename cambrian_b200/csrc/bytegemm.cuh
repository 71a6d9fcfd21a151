// cambrian_b200 — the operand side shared by the 8-bit tensor-core matmuls (int8.cu: LLM.int8, fp8.cu: FP8 E4M3).
//
// Both take row-major one-byte operands [rows, K] (the nn.Linear layout, K-major as the 8-bit wgmma forms require), so
// one k-block of 128 elements is one 128-byte SWIZZLE_128B atom per row and the tensor maps, the persistent tile order
// and the TMA producer loop are the same for both element types.  What the consumers do with the ring (s32 sums, fp32
// promotion) stays in each kernel.
#pragma once
#include "common.cuh"
#include <cudaTypedefs.h>
#include <mutex>

namespace cb {

constexpr int QBM = 128, QBN = 128, QBK = 128;
constexpr int Q_A_BYTES = QBM * QBK, Q_B_BYTES = QBN * QBK, Q_STAGE_BYTES = Q_A_BYTES + Q_B_BYTES;
constexpr int Q_GROUP_M = 16;

// persistent tile r -> (m block, n block): super-rows of Q_GROUP_M m blocks, so neighbouring CTAs share operand tiles in L2
__device__ __forceinline__ void q_tile_to_mn(int r, int m_blocks, int n_blocks, int& mb, int& nb) {
  const int tpg = Q_GROUP_M * n_blocks;
  const int g = r / tpg;
  const int first = g * Q_GROUP_M;
  const int gs = min(Q_GROUP_M, m_blocks - first);
  const int w = r - g * tpg;
  mb = first + w % gs;
  nb = w / gs;
}

// One thread fills the ring: per k-block of every tile this CTA owns (r = blockIdx.x, + gridDim.x, ...), a 128 x 128-byte
// box of A then of B into stage `stage` (A at +0, B at +Q_A_BYTES).  full_bar(s) = bars + 8 s, empty_bar(s) = bars +
// 8 (STAGES + s); the consumers release a stage by arriving on its empty barrier.
template <int STAGES>
__device__ __forceinline__ void q_produce(const CUtensorMap* tmA, const CUtensorMap* tmB, uint32_t smem_base, uint32_t bars,
                                          int M, int N, int K, int tiles) {
  const int m_blocks = (M + QBM - 1) / QBM;
  const int n_blocks = (N + QBN - 1) / QBN;
  const int num_kb = (K + QBK - 1) / QBK;
  int stage = 0;
  uint32_t phase = 0;
  for (int r = blockIdx.x; r < tiles; r += gridDim.x) {
    int mb, nb;
    q_tile_to_mn(r, m_blocks, n_blocks, mb, nb);
    for (int kb = 0; kb < num_kb; ++kb) {
      const uint32_t full = bars + 8u * stage, empty = bars + 8u * (STAGES + stage);
      mbar_wait(empty, phase ^ 1u);
      const uint32_t sa = smem_base + stage * Q_STAGE_BYTES;
      mbar_arrive_expect_tx(full, Q_STAGE_BYTES);
      tma_load_3d(sa, tmA, full, kb * QBK, mb * QBM, 0);
      tma_load_3d(sa + Q_A_BYTES, tmB, full, kb * QBK, nb * QBN, 0);
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1u;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------
static PFN_cuTensorMapEncodeTiled_v12000 q_encode_fn() {
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

// one-byte [rows, K] row-major (row stride K bytes), box 128 (K) x box_rows, SWIZZLE_128B; out-of-range elements read as 0
static int make_tmap_u8(CUtensorMap* out, const void* base, uint64_t K, uint64_t rows, uint32_t box_rows) {
  auto fn = q_encode_fn();
  if (!fn) return set_error(CB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[3] = {K, rows, 1};
  cuuint64_t strides[2] = {K, K * rows};
  cuuint32_t box[3] = {QBK, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = CUDA_SUCCESS;
  for (int attempt = 0; attempt < 2; ++attempt) {
    r = fn(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(base), dims, strides, box, estr,
           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_ERROR_INVALID_CONTEXT) break;
    cudaFree(0);  // a thread with no driver context bound yet: bind the primary context and retry
  }
  if (r != CUDA_SUCCESS) return set_error(CB_ERR_CUDA, "cuTensorMapEncodeTiled (8-bit operand) failed (%d)", (int)r);
  return CB_OK;
}

}  // namespace cb
