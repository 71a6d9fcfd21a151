// cambrian_b200 — LayerNorm / RMSNorm forward + backward (HBM-bound row kernels).
//
// Used by: ViT / ConvNeXt LayerNorms (SURVEY.md §8a A1-A4), the SVA q/k/v LayerNorms and
// `norm` (vision_sampler.py:170-175,258), mm_projector_aux LayerNorm (cambrian_arch.py:56) and
// the LLaMA RMSNorm (A9).  RMSNorm follows the training-time variant the reference patches in
// (train_fsdp.py:1429-1435): y = (w * (x_fp32 * rsqrt(mean(x^2)+eps))).to(dtype); hf_cast=1
// gives the stock HF order (cast x_hat to bf16, then multiply).
//
// One row is handled by TPR threads (32..512) holding <= 4 x 16 B vectors each, so every row is
// read exactly once from HBM with 16-byte coalesced loads; statistics are two-pass in fp32.
// The SVA "latents + pos_embed[window position]" add (vision_sampler.py:304-309) is fused into
// the LayerNorm load: pos is indexed by the position of the grid cell inside its r x r window.
#include "common.cuh"
#include <cfloat>

namespace cb {

constexpr int NORM_VPT = 4;

template <int TPR>
__device__ __forceinline__ float row_sum(float v, float* red, int row_slot) {
  v = warp_sum(v);
  if (TPR > 32) {
    constexpr int W = TPR / 32;
    const int wid = (threadIdx.x % TPR) >> 5;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[row_slot * W + wid] = v;
    __syncthreads();
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < W; ++i) t += red[row_slot * W + i];
    v = t;
  }
  return v;
}

struct PosAdd {
  const bf16* pos;  // [r*r, C] or null
  int side, r;
};
__device__ __forceinline__ int pos_index(const PosAdd& p, long long row) {
  if (p.side == 0) return (int)(row % ((long long)p.r * p.r));  // window-rearranged layout [N, r*r, C]
  const int cell = (int)(row % ((long long)p.side * p.side));
  const int y = cell / p.side, x = cell - y * p.side;
  return (y % p.r) * p.r + (x % p.r);
}

template <int TPR>
__device__ __forceinline__ float row_max(float v, float* red, int row_slot) {
  v = warp_max(v);
  if (TPR > 32) {
    constexpr int W = TPR / 32;
    const int wid = (threadIdx.x % TPR) >> 5;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[row_slot * W + wid] = v;
    __syncthreads();
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < W; ++i) t = fmaxf(t, red[row_slot * W + i]);
    v = t;
  }
  return v;
}

// E4M3 output of the RMSNorm (F8 = true, `fp8_training`): the row y is rounded to bf16 exactly as the bf16 output is,
// then quantised by the row rule of quant_fp8.py into q [rows, C] e4m3 and s [rows] fp32; Y is not written
struct F8Rows {
  uint8_t* q;
  float* s;
};

template <int TPR, bool RMS, bool F8 = false>
__global__ void __launch_bounds__(TPR < 256 ? 256 : TPR)
norm_fwd_kernel(const bf16* __restrict__ X, const bf16* __restrict__ gamma, const bf16* __restrict__ beta,
                bf16* __restrict__ Y, float* __restrict__ mean_out, float* __restrict__ rstd_out,
                long long rows, int C, float eps, int hf_cast, PosAdd pa, F8Rows f8 = {}) {
  constexpr int RPB = TPR < 256 ? 256 / TPR : 1;
  __shared__ float red[RPB * (TPR / 32) + 1];
  const int slot = threadIdx.x / TPR, tir = threadIdx.x % TPR;
  const long long row = (long long)blockIdx.x * RPB + slot;
  const bool active = row < rows;  // inactive rows still take part in __syncthreads
  const int nvec = C >> 3;
  float x[NORM_VPT][8];
  float s = 0.f;
  const uint4* xp = reinterpret_cast<const uint4*>(X + (active ? row : 0) * C);
  const uint4* pp = nullptr;
  if (pa.pos && active) pp = reinterpret_cast<const uint4*>(pa.pos + (size_t)pos_index(pa, row) * C);
#pragma unroll
  for (int i = 0; i < NORM_VPT; ++i) {
    const int vi = tir + i * TPR;
    if (active && vi < nvec) {
      unpack8(ldg_nc(xp + vi), x[i]);
      if (pp) {
        float t[8];
        unpack8(pp[vi], t);
#pragma unroll
        for (int e = 0; e < 8; ++e) x[i][e] = __bfloat162float(__float2bfloat16(x[i][e] + t[e]));
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) s += RMS ? x[i][e] * x[i][e] : x[i][e];
    }
  }
  float mean = 0.f, rstd;
  if (RMS) {
    const float ss = row_sum<TPR>(s, red, slot);
    rstd = rsqrtf(ss / C + eps);
  } else {
    mean = row_sum<TPR>(s, red, slot) / C;
    float v = 0.f;
#pragma unroll
    for (int i = 0; i < NORM_VPT; ++i) {
      const int vi = tir + i * TPR;
      if (active && vi < nvec) {
#pragma unroll
        for (int e = 0; e < 8; ++e) { const float d = x[i][e] - mean; v += d * d; }
      }
    }
    v = row_sum<TPR>(v, red, slot);
    rstd = rsqrtf(v / C + eps);
  }
  if constexpr (F8) {
    static_assert(RMS, "the E4M3 output exists for the RMSNorm only");
    // y as the bf16 path computes and rounds it, kept in x; then amax, s, r and q of quant_fp8.py
    const uint4* gp = reinterpret_cast<const uint4*>(gamma);
    float a = 0.f;
#pragma unroll
    for (int i = 0; i < NORM_VPT; ++i) {
      const int vi = tir + i * TPR;
      if (active && vi < nvec) {
        float g[8], o[8];
        unpack8(gp[vi], g);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          float xh = x[i][e] * rstd;
          if (hf_cast) xh = __bfloat162float(__float2bfloat16(xh));
          o[e] = g[e] * xh;
        }
        unpack8(pack8(o), x[i]);
#pragma unroll
        for (int e = 0; e < 8; ++e) a = fmaxf(a, fabsf(x[i][e]));
      }
    }
    a = row_max<TPR>(a, red, slot);
    if (!active) return;
    if (tir == 0) {
      if (rstd_out) rstd_out[row] = rstd;
      f8.s[row] = __fdiv_rn(a, 448.0f);
    }
    const float r = fminf(__fdiv_rn(448.0f, a), FLT_MAX);  // amax = 0 or below 448 * 2^-128: +inf -> FLT_MAX
    uint2* qp = reinterpret_cast<uint2*>(f8.q + row * C);
#pragma unroll
    for (int i = 0; i < NORM_VPT; ++i) {
      const int vi = tir + i * TPR;
      if (vi < nvec) {
        float t[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) t[e] = __fmul_rn(x[i][e], r);
        qp[vi] = f8_pack8(t);
      }
    }
    return;
  }
  if (!active) return;
  if (tir == 0) {
    if (mean_out) mean_out[row] = mean;
    if (rstd_out) rstd_out[row] = rstd;
  }
  uint4* yp = reinterpret_cast<uint4*>(Y + row * C);
  const uint4* gp = reinterpret_cast<const uint4*>(gamma);
  const uint4* bp = reinterpret_cast<const uint4*>(beta);
#pragma unroll
  for (int i = 0; i < NORM_VPT; ++i) {
    const int vi = tir + i * TPR;
    if (vi < nvec) {
      float g[8], o[8];
      unpack8(gp[vi], g);
      if (RMS) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          float xh = x[i][e] * rstd;
          if (hf_cast) xh = __bfloat162float(__float2bfloat16(xh));
          o[e] = g[e] * xh;
        }
      } else {
        float bt[8];
        if (bp) unpack8(bp[vi], bt);
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] = (x[i][e] - mean) * rstd * g[e] + (bp ? bt[e] : 0.f);
      }
      yp[vi] = pack8(o);
    }
  }
}

// backward: dx per row; per-block partial sums of dgamma / dbeta into part_g / part_b [P, C] (fp32)
template <int TPR, bool RMS, int VPT>
__global__ void __launch_bounds__(TPR < 256 ? 256 : TPR)
norm_bwd_kernel(const bf16* __restrict__ dY, const bf16* __restrict__ X, const bf16* __restrict__ gamma,
                const float* __restrict__ mean_in, const float* __restrict__ rstd_in, bf16* __restrict__ dX,
                const bf16* __restrict__ dRes, float* __restrict__ part_g, float* __restrict__ part_b, long long rows,
                int C, PosAdd pa) {
  constexpr int RPB = TPR < 256 ? 256 / TPR : 1;
  __shared__ float red[RPB * (TPR / 32) + 1];
  const int slot = threadIdx.x / TPR, tir = threadIdx.x % TPR;
  const int nvec = C >> 3;
  float g[VPT][8], ag[VPT][8], ab[VPT][8];
  const uint4* gp = reinterpret_cast<const uint4*>(gamma);
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int vi = tir + i * TPR;
#pragma unroll
    for (int e = 0; e < 8; ++e) { ag[i][e] = 0.f; ab[i][e] = 0.f; g[i][e] = 0.f; }
    if (vi < nvec) unpack8(gp[vi], g[i]);
  }
  const long long row_stride = (long long)gridDim.x * RPB;
  const long long iters = (rows + row_stride - 1) / row_stride;
  for (long long it = 0; it < iters; ++it) {
    const long long row = it * row_stride + (long long)blockIdx.x * RPB + slot;
    const bool active = row < rows;
    float x[VPT][8], dy[VPT][8];
    const float mean = (!RMS && active) ? mean_in[row] : 0.f;
    const float rstd = active ? rstd_in[row] : 0.f;
    const uint4* xp = reinterpret_cast<const uint4*>(X + (active ? row : 0) * C);
    const uint4* dp = reinterpret_cast<const uint4*>(dY + (active ? row : 0) * C);
    const uint4* pp = nullptr;
    if (pa.pos && active) pp = reinterpret_cast<const uint4*>(pa.pos + (size_t)pos_index(pa, row) * C);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int vi = tir + i * TPR;
      if (active && vi < nvec) {
        unpack8(ldg_nc(xp + vi), x[i]);
        unpack8(ldg_nc(dp + vi), dy[i]);
        if (pp) {
          float t[8];
          unpack8(pp[vi], t);
#pragma unroll
          for (int e = 0; e < 8; ++e) x[i][e] = __bfloat162float(__float2bfloat16(x[i][e] + t[e]));
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float xh = (x[i][e] - mean) * rstd;
          const float gd = g[i][e] * dy[i][e];
          s1 += gd;
          s2 += gd * xh;
          ag[i][e] += dy[i][e] * xh;
          ab[i][e] += dy[i][e];
          x[i][e] = xh;   // keep x_hat
          dy[i][e] = gd;  // keep gamma*dy
        }
      }
    }
    if (!RMS) s1 = row_sum<TPR>(s1, red, slot) / C;
    s2 = row_sum<TPR>(s2, red, slot) / C;
    if (active) {
      uint4* dxp = reinterpret_cast<uint4*>(dX + row * C);
#pragma unroll
      for (int i = 0; i < VPT; ++i) {
        const int vi = tir + i * TPR;
        if (vi < nvec) {
          float o[8];
#pragma unroll
          for (int e = 0; e < 8; ++e)
            o[e] = RMS ? rstd * (dy[i][e] - x[i][e] * s2) : rstd * (dy[i][e] - s1 - x[i][e] * s2);
          if (dRes) {  // fused residual-stream gradient: dx = d_residual + d_norm_input
            float t[8];
            unpack8(ldg_nc(reinterpret_cast<const uint4*>(dRes + row * C) + vi), t);
#pragma unroll
            for (int e = 0; e < 8; ++e) o[e] += t[e];
          }
          dxp[vi] = pack8(o);
        }
      }
    }
  }
  const size_t prow = (size_t)blockIdx.x * RPB + slot;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int vi = tir + i * TPR;
    if (vi < nvec) {
      float4* pg = reinterpret_cast<float4*>(part_g + prow * C + (size_t)vi * 8);
      pg[0] = make_float4(ag[i][0], ag[i][1], ag[i][2], ag[i][3]);
      pg[1] = make_float4(ag[i][4], ag[i][5], ag[i][6], ag[i][7]);
      if (!RMS && part_b) {
        float4* pb = reinterpret_cast<float4*>(part_b + prow * C + (size_t)vi * 8);
        pb[0] = make_float4(ab[i][0], ab[i][1], ab[i][2], ab[i][3]);
        pb[1] = make_float4(ab[i][4], ab[i][5], ab[i][6], ab[i][7]);
      }
    }
  }
}

// out[c] = sum_p part[p, c]  (deterministic fixed-order column reduction)
// 32 columns x 32 row-lanes per block: coalesced 128 B reads, fixed-order (deterministic) tree over the row lanes.
// (The first version used one thread per column over all P partial rows: 16 blocks for C = 4096 -> 135 us per call,
//  7.5% of the whole training step in the r01 launch list.)
__global__ void __launch_bounds__(1024)
colsum_kernel(const float* __restrict__ part, int P, int C, bf16* __restrict__ out_bf16, float* __restrict__ out_f32) {
  __shared__ float red[32][33];
  const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cx;
  float s = 0.f;
  if (c < C)
    for (int p = ry; p < P; p += 32) s += part[(size_t)p * C + c];
  red[ry][cx] = s;
  __syncthreads();
  if (ry == 0 && c < C) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 32; ++k) t += red[k][cx];
    if (out_bf16) out_bf16[c] = __float2bfloat16(t);
    if (out_f32) out_f32[c] = t;
  }
}

static int pick_tpr(int C, int vpt = NORM_VPT) {
  const int need = (C / 8 + vpt - 1) / vpt;
  if (need <= 32) return 32;
  if (need <= 64) return 64;
  if (need <= 128) return 128;
  if (need <= 256) return 256;
  if (need <= 512) return 512;
  return 0;
}

template <bool RMS>
static int norm_fwd_t(const void* x, const void* gamma, const void* beta, void* y, float* mean, float* rstd,
                      long long rows, int C, float eps, int hf_cast, PosAdd pa, cudaStream_t st) {
  const int tpr = pick_tpr(C);
  CB_CHECK_ARG(C % 8 == 0 && tpr != 0, "norm: C=%d must be a multiple of 8 and <= 16384", C);
  CB_CHECK_ARG(rows > 0, "norm: rows=%lld", rows);
  const bf16 *X = (const bf16*)x, *G = (const bf16*)gamma, *Bt = (const bf16*)beta;
  bf16* Y = (bf16*)y;
#define CB_NORM_FWD(T)                                                                              \
  {                                                                                                 \
    constexpr int RPB = T < 256 ? 256 / T : 1;                                                      \
    const unsigned grid = (unsigned)((rows + RPB - 1) / RPB);                                       \
    norm_fwd_kernel<T, RMS><<<grid, T < 256 ? 256 : T, 0, st>>>(X, G, Bt, Y, mean, rstd, rows, C,  \
                                                                 eps, hf_cast, pa);                 \
  }
  switch (tpr) {
    case 32: CB_NORM_FWD(32) break;
    case 64: CB_NORM_FWD(64) break;
    case 128: CB_NORM_FWD(128) break;
    case 256: CB_NORM_FWD(256) break;
    default: CB_NORM_FWD(512) break;
  }
#undef CB_NORM_FWD
  CB_CUDA_LAUNCH_CHECK("norm_fwd");
  return CB_OK;
}

// backward keeps x_hat, gamma*dy and two partial-sum arrays live: 2 vectors per thread (instead of 4) halves the
// register footprint (196 -> ~110) so 2-3 blocks fit per SM; rows wider than 512*2 vectors fall back to 4.
static void bwd_cfg(int C, int* tpr, int* vpt) {
  *vpt = (C / 8 <= 1024) ? 2 : 4;
  *tpr = pick_tpr(C, *vpt);
}

template <bool RMS>
static int norm_bwd_t(const void* dy, const void* x, const void* gamma, const float* mean, const float* rstd,
                      void* dx, const void* dres, void* dgamma, void* dbeta, float* workspace, long long ws_floats,
                      long long rows, int C, PosAdd pa, cudaStream_t st) {
  int tpr, vpt;
  bwd_cfg(C, &tpr, &vpt);
  CB_CHECK_ARG(C % 8 == 0 && tpr != 0, "norm bwd: C=%d must be a multiple of 8 and <= 16384", C);
  CB_CHECK_ARG(rows > 0, "norm bwd: rows=%lld", rows);
  const int rpb = tpr < 256 ? 256 / tpr : 1;
  long long grid = (rows + rpb - 1) / rpb;
  const long long cap = 2LL * device_sm_count();
  if (grid > cap) grid = cap;
  const long long P = grid * rpb;
  CB_CHECK_ARG(workspace && ws_floats >= 2 * P * C, "norm bwd: workspace too small (%lld < %lld floats)",
               ws_floats, 2 * P * C);
  float* part_g = workspace;
  float* part_b = workspace + P * C;
#define CB_NORM_BWD(T, V)                                                                                   \
  norm_bwd_kernel<T, RMS, V><<<(unsigned)grid, T < 256 ? 256 : T, 0, st>>>(                                \
      (const bf16*)dy, (const bf16*)x, (const bf16*)gamma, mean, rstd, (bf16*)dx, (const bf16*)dres, part_g, part_b, \
      rows, C, pa);
  if (vpt == 2) {
    switch (tpr) {
      case 32: CB_NORM_BWD(32, 2) break;
      case 64: CB_NORM_BWD(64, 2) break;
      case 128: CB_NORM_BWD(128, 2) break;
      case 256: CB_NORM_BWD(256, 2) break;
      default: CB_NORM_BWD(512, 2) break;
    }
  } else {
    CB_NORM_BWD(512, 4)
  }
#undef CB_NORM_BWD
  CB_CUDA_LAUNCH_CHECK("norm_bwd");
  colsum_kernel<<<(C + 31) / 32, 1024, 0, st>>>(part_g, (int)P, C, (bf16*)dgamma, nullptr);
  if (!RMS && dbeta) colsum_kernel<<<(C + 31) / 32, 1024, 0, st>>>(part_b, (int)P, C, (bf16*)dbeta, nullptr);
  CB_CUDA_LAUNCH_CHECK("norm_bwd colsum");
  return CB_OK;
}

// RMSNorm forward with an E4M3 output (`fp8_training`): the pick_tpr / row layout of norm_fwd_t, so rstd and the bf16
// rounding of y match rmsnorm_fwd bit for bit; q [rows, C] e4m3, s [rows] fp32 by the quant_fp8.py row rule
int rmsnorm_fwd_fp8(const void* x, const void* gamma, void* q, float* s, float* rstd, long long rows, int C, float eps,
                    int hf_cast, cudaStream_t st) {
  const int tpr = pick_tpr(C);
  CB_CHECK_ARG(C % 16 == 0 && tpr != 0, "rmsnorm_fwd_fp8: C=%d must be a multiple of 16 and <= 16384", C);
  CB_CHECK_ARG(rows > 0, "rmsnorm_fwd_fp8: rows=%lld", rows);
  CB_CHECK_ARG(x && gamma && q && s, "rmsnorm_fwd_fp8: null argument");
  CB_CHECK_ARG(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(gamma) | reinterpret_cast<uintptr_t>(q)) &
                15u) == 0, "rmsnorm_fwd_fp8: x, gamma and q must be 16-byte aligned");
  const PosAdd pa{nullptr, 1, 1};
  const F8Rows f8{(uint8_t*)q, s};
#define CB_NORM_FWD_F8(T)                                                                                     \
  {                                                                                                           \
    constexpr int RPB = T < 256 ? 256 / T : 1;                                                                \
    const unsigned grid = (unsigned)((rows + RPB - 1) / RPB);                                                 \
    norm_fwd_kernel<T, true, true><<<grid, T < 256 ? 256 : T, 0, st>>>((const bf16*)x, (const bf16*)gamma,    \
                                                                      nullptr, nullptr, nullptr, rstd, rows, C, \
                                                                      eps, hf_cast, pa, f8);                   \
  }
  switch (tpr) {
    case 32: CB_NORM_FWD_F8(32) break;
    case 64: CB_NORM_FWD_F8(64) break;
    case 128: CB_NORM_FWD_F8(128) break;
    case 256: CB_NORM_FWD_F8(256) break;
    default: CB_NORM_FWD_F8(512) break;
  }
#undef CB_NORM_FWD_F8
  CB_CUDA_LAUNCH_CHECK("rmsnorm_fwd_fp8");
  return CB_OK;
}

int layernorm_fwd(const void* x, const void* gamma, const void* beta, void* y, float* mean, float* rstd,
                  long long rows, int C, float eps, const void* pos, int side, int r, cudaStream_t st) {
  PosAdd pa{(const bf16*)pos, side >= 0 ? side : 0, r > 0 ? r : 1};
  return norm_fwd_t<false>(x, gamma, beta, y, mean, rstd, rows, C, eps, 0, pa, st);
}
int layernorm_bwd(const void* dy, const void* x, const void* gamma, const float* mean, const float* rstd,
                  void* dx, const void* dres, void* dgamma, void* dbeta, float* ws, long long ws_floats, long long rows,
                  int C, const void* pos, int side, int r, cudaStream_t st) {
  PosAdd pa{(const bf16*)pos, side >= 0 ? side : 0, r > 0 ? r : 1};
  return norm_bwd_t<false>(dy, x, gamma, mean, rstd, dx, dres, dgamma, dbeta, ws, ws_floats, rows, C, pa, st);
}
int rmsnorm_fwd(const void* x, const void* gamma, void* y, float* rstd, long long rows, int C, float eps,
                int hf_cast, cudaStream_t st) {
  PosAdd pa{nullptr, 1, 1};
  return norm_fwd_t<true>(x, gamma, nullptr, y, nullptr, rstd, rows, C, eps, hf_cast, pa, st);
}
int rmsnorm_bwd(const void* dy, const void* x, const void* gamma, const float* rstd, void* dx, const void* dres,
                void* dgamma, float* ws, long long ws_floats, long long rows, int C, cudaStream_t st) {
  PosAdd pa{nullptr, 1, 1};
  return norm_bwd_t<true>(dy, x, gamma, nullptr, rstd, dx, dres, dgamma, nullptr, ws, ws_floats, rows, C, pa, st);
}
long long norm_bwd_workspace_floats(long long rows, int C) {
  int tpr, vpt;
  bwd_cfg(C, &tpr, &vpt);
  if (!tpr) return 0;
  const int rpb = tpr < 256 ? 256 / tpr : 1;
  long long grid = (rows + rpb - 1) / rpb;
  const long long cap = 2LL * device_sm_count();
  if (grid > cap) grid = cap;
  return 2 * grid * rpb * (long long)C;
}

}  // namespace cb
