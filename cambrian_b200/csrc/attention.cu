// cambrian_b200 — wgmma flash attention (forward + backward) for sm_90a (H100).
//
// Covers the two softmax-attention shapes of the hot path (SURVEY.md §8a):
//   * ViT towers (A1-A3): non-causal, head_dim 64 (CLIP, DINOv2) / 72 (SigLIP), 577 / 729 tokens, fwd only
//   * LLaMA decoder (A9): causal + key-padding mask, GQA, head_dim 128, S = 2048, fwd + bwd
// replacing torch SDPA as called by HF CLIP/DINOv2/Llama attention and timm Attention.
//
// Layout: q/k/v/o are addressed as (b, s, head, d) with arbitrary batch / row strides and heads packed along the
// row, so the fused QKV GEMM output [B*S, (nh + 2 nkv) * hd] is consumed in place (no permute / contiguous).
//
// Forward (one CTA = 128 query rows of one head; 288 threads):
//   warp 8     TMA producer : Q once, then K_j / V_j tiles through an mbarrier ring
//   warps 0-7  two consumer warpgroups of 64 query rows: S_j = Q K_j^T (wgmma, fp32 in registers), online softmax in
//              the log2 domain (rows are spread over the 4 lanes of a quad), P_j re-packed in registers as the bf16
//              A operand of O += P_j V_j (wgmma with A from registers, V read MN-major from shared memory).
// Backward, two kernels so that every output element has exactly one writer (no atomics: bit-identical run to run):
//   dK / dV: one CTA = 128 keys of one KV head, two warpgroups of 64 keys, looping over the query heads of the GQA group
//     and the 64-row query tiles, which a producer warp streams (with their lse / delta slices) through an mbarrier
//     ring: S^T = K Q^T and dP^T = V dO^T in registers; P^T and dS^T are re-packed in registers as the A operands of
//     dV += P^T dO and dK += dS^T Q.
//   dQ: one CTA = 128 queries of one head (same layout as the forward), looping over 64-key tiles: S = Q K^T and
//     dP = dO V^T in registers, dS re-packed as the A operand of dQ += dS K; dQ x scale is stored once per element, as
//     bf16, into the caller's view.
// Tiles that every (query, key) pair of a warp can see skip the per-element masking; grids are 1-D, heaviest causal
// tiles first.
#include "common.cuh"
#include <cudaTypedefs.h>
#include <type_traits>

namespace cb {

int make_tmap_bf16_4d(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t d3,
                      uint64_t s1, uint64_t s2, uint64_t s3, uint32_t box_rows);

constexpr float LOG2E = 1.4426950408889634f;

struct AttnParams {
  bf16* o;
  long long o_bs, o_ss;  // element strides of O (batch, row); heads packed at hd
  float* lse;            // [B, nh, Sq] log2-domain, may be null
  const uint8_t* kmask;  // [B, Skv] 1 = attend, may be null
  int B, nh, nkv, Sq, Skv, hd, causal;
  float scale_log2;      // softmax scale * log2(e)
};

// true iff every key of [k0, k0 + N) is set in the key mask (the caller checks k0 + N <= Skv): N / 32 bytes per lane in
// one load where aligned, and a warp vote, so the result is warp-uniform.  Tiles that pass skip the per-element masking.
template <int N>
__device__ __forceinline__ bool keys_all_valid(const uint8_t* km, int k0) {
  constexpr int PER = N / 32;
  static_assert(PER == 2 || PER == 4, "64- or 128-key tiles");
  const uint8_t* kp = km + k0 + PER * (threadIdx.x & 31);
  uint32_t w = 0;
  if (!(reinterpret_cast<uintptr_t>(kp) & (PER - 1))) {
    w = PER == 4 ? *reinterpret_cast<const uint32_t*>(kp) : *reinterpret_cast<const uint16_t*>(kp);
  } else {
#pragma unroll
    for (int i = 0; i < PER; ++i) w |= (uint32_t)kp[i] << (8 * i);
  }
  bool ok = true;
#pragma unroll
  for (int i = 0; i < PER; ++i) ok = ok && ((w >> (8 * i)) & 0xffu);
  return __all_sync(0xffffffffu, ok);
}

// Grids are 1-D with the tile index slowest, so the first wave holds the heaviest causal tiles of every (head, batch)
// and the light ones fill the tail.
struct TileIdx {
  int t, h, b;
};
__device__ __forceinline__ TileIdx tile_index(int heads, int B) {
  const int hb = heads * B;
  const int rem = (int)blockIdx.x % hb;
  return {(int)blockIdx.x / hb, rem % heads, rem / heads};
}

template <int HDP>
struct FwdCfg {
  static constexpr int ATOMS = (HDP + 63) / 64;
  static constexpr int TILE = ATOMS * 16384;         // one [128 x hd] operand tile, 64-column SWIZZLE_128B atoms
  static constexpr int STAGES = 3;                   // hd 128: 32 KB Q + 3 x 64 KB K / V
  static constexpr int SMEM = TILE * (1 + 2 * STAGES) + 1024 + 256;
};

template <int HDP>
__global__ void __launch_bounds__(288, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, AttnParams p) {
  using Cfg = FwdCfg<HDP>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sQ = base;
  const uint32_t sK = sQ + Cfg::TILE;
  const uint32_t sV = sK + STAGES * Cfg::TILE;
  const uint32_t bars = sV + STAGES * Cfg::TILE;
  const uint32_t q_full = bars;
  auto k_full = [&](int s) { return bars + 8u * (1 + s); };
  auto v_full = [&](int s) { return bars + 8u * (1 + STAGES + s); };
  auto kv_empty = [&](int s) { return bars + 8u * (1 + 2 * STAGES + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q_tiles = (p.Sq + 127) / 128;
  const TileIdx ti = tile_index(p.nh, p.B);
  const int qt = q_tiles - 1 - ti.t;  // heavy (late) causal tiles first
  const int h = ti.h, b = ti.b;
  const int hk = h / (p.nh / p.nkv);
  const int q0 = qt * 128;
  const int kv_tiles_all = (p.Skv + 127) / 128;
  // causal: keys <= query index (+ offset when Skv > Sq, e.g. a prefilled cache)
  const int coff = p.Skv - p.Sq;
  int n_tiles = kv_tiles_all;
  if (p.causal) {
    const int last_key = q0 + 127 + coff;
    n_tiles = min(kv_tiles_all, last_key / 128 + 1);
    if (n_tiles < 1) n_tiles = 1;
  }

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(k_full(s), 1);
      mbar_init(v_full(s), 1);
      mbar_init(kv_empty(s), 2);  // one arrive per consumer warpgroup
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ================================ TMA producer ================================
    if (lane == 0) {
      mbar_arrive_expect_tx(q_full, Cfg::TILE);
#pragma unroll
      for (int a = 0; a < Cfg::ATOMS; ++a) tma_load_4d(sQ + a * 16384, &tmQ, q_full, a * 64, h, q0, b);
      int st = 0;
      uint32_t ph = 0;
      for (int j = 0; j < n_tiles; ++j) {
        mbar_wait(kv_empty(st), ph ^ 1u);
        mbar_arrive_expect_tx(k_full(st), Cfg::TILE);
#pragma unroll
        for (int a = 0; a < Cfg::ATOMS; ++a)
          tma_load_4d(sK + st * Cfg::TILE + a * 16384, &tmK, k_full(st), a * 64, hk, j * 128, b);
        mbar_arrive_expect_tx(v_full(st), Cfg::TILE);
#pragma unroll
        for (int a = 0; a < Cfg::ATOMS; ++a)
          tma_load_4d(sV + st * Cfg::TILE + a * 16384, &tmV, v_full(st), a * 64, hk, j * 128, b);
        if (++st == STAGES) { st = 0; ph ^= 1u; }
      }
    }
    return;
  }

  // ================================ consumer warpgroups ================================
  const int wg = warp >> 2;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  const int rloc = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's rows: rloc and rloc + 8
  const int cq = 2 * (lane & 3);                             // and columns 8 j + cq, + 1 of every 8-column block
  const uint8_t* km = p.kmask ? p.kmask + (size_t)b * p.Skv : nullptr;
  float o[HDP / 2];
#pragma unroll
  for (int i = 0; i < HDP / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  mbar_wait(q_full, 0);
  int st = 0;
  uint32_t ph = 0;
  for (int j = 0; j < n_tiles; ++j) {
    const int k0 = j * 128;
    float s[64];
    mbar_wait(k_full(st), ph);
    const uint32_t kb = sK + st * Cfg::TILE;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < HDP / 16; ++kk) {
      const uint32_t off = (kk >> 2) * 16384 + (kk & 3) * 32;
      WgmmaSS<128, 0, 0>::mma(s, make_smem_desc_sw128(sQ + wg * 8192 + off, 0, 1024),
                              make_smem_desc_sw128(kb + off, 0, 1024), kk ? 1u : 0u);
    }
    wgmma_commit();
    // masking (keys past Skv, past the diagonal, padded keys) -> -inf; scores into the log2 domain.  A tile inside Skv,
    // below the diagonal for all 64 rows of the warpgroup, whose keys are all valid keeps every score as it is.
    bool full_tile = k0 + 128 <= p.Skv && (!p.causal || k0 + 127 <= q0 + wg * 64 + coff);
    if (full_tile && km) full_tile = keys_all_valid<128>(km, k0);
    wgmma_wait<0>();
    reg_fence(s);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float v = s[4 * jj + e] * p.scale_log2;
        if (!full_tile) {
          const int key = k0 + 8 * jj + cq + (e & 1);
          const int qi = q0 + rloc + 8 * (e >> 1);
          const bool ok = key < p.Skv && (!p.causal || key <= qi + coff) && (!km || km[key]);
          v = ok ? v : -INFINITY;
        }
        s[4 * jj + e] = v;
        mx[e >> 1] = fmaxf(mx[e >> 1], v);
      }
    }
    float corr[2], mref[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float m_new = fmaxf(m_run[r], mx[r]);
      mref[r] = m_new == -INFINITY ? 0.f : m_new;  // fully masked so far: exp2(-inf - 0) = 0 keeps everything finite
      corr[r] = fast_exp2(m_run[r] - mref[r]);
      m_run[r] = m_new;
      l_run[r] *= corr[r];
    }
#pragma unroll
    for (int jj = 0; jj < HDP / 8; ++jj) {
#pragma unroll
      for (int e = 0; e < 4; ++e) o[4 * jj + e] *= corr[e >> 1];
    }
    // P = exp2(s - m): row sums (per thread; the quad is summed once at the end) and the bf16 A fragments of P V
    uint32_t pa[8][4];
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
      float pv[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        pv[e] = fast_exp2(s[4 * jj + e] - mref[e >> 1]);
        l_run[e >> 1] += pv[e];
      }
      pa[jj >> 1][(jj & 1) * 2 + 0] = pack_bf16x2(pv[0], pv[1]);
      pa[jj >> 1][(jj & 1) * 2 + 1] = pack_bf16x2(pv[2], pv[3]);
    }
    mbar_wait(v_full(st), ph);
    const uint32_t vb = sV + st * Cfg::TILE;
    reg_fence(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)
      WgmmaRS<HDP, 1>::mma(o, pa[kk], make_smem_desc_sw128(vb + kk * 2048, 16384, 1024), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
    if (wg_leader) mbar_arrive(kv_empty(st));
    if (++st == STAGES) { st = 0; ph ^= 1u; }
  }
  // ---- epilogue: O / l -> bf16 -> HBM
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float l = l_run[r];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int qi = q0 + rloc + 8 * r;
    if (qi >= p.Sq) continue;
    const float inv = l > 0.f ? 1.f / l : 0.f;
    bf16* op = p.o + (long long)b * p.o_bs + (long long)qi * p.o_ss + (long long)h * p.hd;
#pragma unroll
    for (int jj = 0; jj < HDP / 8; ++jj) {
      const int d = 8 * jj + cq;
      if (d < p.hd)
        *reinterpret_cast<__nv_bfloat162*>(op + d) = __floats2bfloat162_rn(o[4 * jj + 2 * r] * inv, o[4 * jj + 2 * r + 1] * inv);
    }
    if (p.lse && (lane & 3) == 0)
      p.lse[((long long)b * p.nh + h) * p.Sq + qi] = l > 0.f ? m_run[r] + log2f(l) : INFINITY;
  }
}

// ------------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------------
// delta[b, h, s] = sum_d dO[b,s,h,d] * O[b,s,h,d]   (fp32).  hd / 8 lanes (one 16-byte vector each) per (b, s, h), so a
// warp covers 32 / (hd / 8) heads: with one warp per head only hd / 8 of the 32 lanes had work (2.2 TB/s).
__global__ void attn_delta_kernel(const bf16* __restrict__ o, const bf16* __restrict__ d_o, float* __restrict__ delta,
                                  int B, int S, int nh, int hd, long long o_bs, long long o_ss, long long do_bs,
                                  long long do_ss) {
  const int lph = hd >> 3;                       // lanes per head: 16 (hd 128) or 8 (hd 64)
  const int hpw = 32 / lph;                      // heads per warp
  const long long w = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const long long total = (long long)B * S * nh;
  const long long idx = w * hpw + lane / lph;    // (b, s, h) handled by this lane group
  const int sub = lane % lph;
  float acc = 0.f;
  if (idx < total) {
    const int h = (int)(idx % nh);
    const long long t = idx / nh;
    const int s = (int)(t % S);
    const int b = (int)(t / S);
    const bf16* op = o + b * o_bs + s * o_ss + (long long)h * hd + sub * 8;
    const bf16* gp = d_o + b * do_bs + s * do_ss + (long long)h * hd + sub * 8;
    float a[8], g[8];
    unpack8(ldg_nc(op), a);
    unpack8(ldg_nc(gp), g);
#pragma unroll
    for (int e = 0; e < 8; ++e) acc += a[e] * g[e];
  }
  for (int off = lph >> 1; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if (idx < total && sub == 0) {
    const int h = (int)(idx % nh);
    const long long t = idx / nh;
    delta[((long long)(t / S) * nh + h) * S + (t % S)] = acc;
  }
}

struct AttnBwdParams {
  bf16* dq;                 // (b, s, head, d) with strides below: dS K x softmax scale, every element written once
  bf16* dk;                 // (b, s, kv head, d)
  bf16* dv;
  long long dq_bs, dq_ss, dk_bs, dk_ss, dv_bs, dv_ss;
  const float* lse;         // [B, nh, Sq] log2 domain
  const float* delta;       // [B, nh, Sq]
  const uint8_t* kmask;
  int B, nh, nkv, Sq, Skv, hd, causal;
  float scale_log2, scale;
};

template <int HDP>
struct BwdCfg {
  static constexpr int ATOMS = HDP / 64;
  static constexpr int KTILE = ATOMS * 16384;  // [128 keys x hd]
  static constexpr int QTILE = ATOMS * 8192;   // [64 queries x hd]
  static constexpr int STAGES = 4;             // Q / dO ring; each stage also holds the tile's lse[64] and delta[64]
  static constexpr int SMEM = 2 * KTILE + 2 * STAGES * QTILE + STAGES * 512 + 1024 + 256;
};

// 384 threads: warpgroups 0-1 consume (dK and dV alone hold HDP fp32 per thread), warp 8 of warpgroup 2 produces.
// Registers are allocated per 4 warps, so a 288-thread CTA would cap every thread at 168; setmaxnreg moves the
// producer warpgroup's share to the consumers instead (128 x 24 + 256 x 240 <= 64 K).
template <int HDP>
__global__ void __launch_bounds__(384, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO, AttnBwdParams p) {
  using Cfg = BwdCfg<HDP>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sK = base;
  const uint32_t sV = sK + Cfg::KTILE;
  const uint32_t sQ = sV + Cfg::KTILE;
  const uint32_t sdO = sQ + STAGES * Cfg::QTILE;
  const uint32_t sLD = sdO + STAGES * Cfg::QTILE;
  const uint32_t bars = sLD + STAGES * 512;
  const uint32_t kv_full = bars;
  auto qd_full = [&](int s) { return bars + 8u * (1 + s); };
  auto qd_empty = [&](int s) { return bars + 8u * (1 + STAGES + s); };
  float* ld_stage = reinterpret_cast<float*>(smem_raw + (sLD - smem_u32(smem_raw)));  // [STAGES][lse 64 | delta 64]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const TileIdx ti = tile_index(p.nkv, p.B);
  const int jt = ti.t, g = ti.h, b = ti.b;  // key tile 0 is seen by every query: heavy tiles first
  const int G = p.nh / p.nkv;
  const int k0 = jt * 128;
  const int q_tiles = (p.Sq + 63) / 64;
  const int coff = p.Skv - p.Sq;
  // causal: query i attends key k iff k <= i + coff  ->  first query tile that can see key k0
  int i_begin = 0;
  if (p.causal) {
    const int first_q = k0 - coff;
    i_begin = first_q > 0 ? first_q / 64 : 0;
  }
  const int n_i = q_tiles > i_begin ? q_tiles - i_begin : 0;
  const int n_iter = n_i * G;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    tma_prefetch_desc(&tmdO);
    mbar_init(kv_full, 1);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(qd_full(s), 1 + 32);  // the TMA transaction arrive + one per producer lane after its lse / delta stores
      mbar_init(qd_empty(s), 8);      // one arrive per consumer warp
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // ================================ producer warp ================================
    setmaxnreg_dec<24>();
    if (warp > 8) return;
    if (lane == 0) {
      mbar_arrive_expect_tx(kv_full, 2 * Cfg::KTILE);
#pragma unroll
      for (int a = 0; a < Cfg::ATOMS; ++a) {
        tma_load_4d(sK + a * 16384, &tmK, kv_full, a * 64, g, k0, b);
        tma_load_4d(sV + a * 16384, &tmV, kv_full, a * 64, g, k0, b);
      }
    }
    int st = 0;
    uint32_t ph = 0;
    for (int it = 0; it < n_iter; ++it) {
      const int h = g * G + it / n_i;
      const int qi0 = (i_begin + it % n_i) * 64;
      mbar_wait(qd_empty(st), ph ^ 1u);
      if (lane == 0) {
        mbar_arrive_expect_tx(qd_full(st), 2 * Cfg::QTILE);
#pragma unroll
        for (int a = 0; a < Cfg::ATOMS; ++a) {
          tma_load_4d(sQ + st * Cfg::QTILE + a * 8192, &tmQ, qd_full(st), a * 64, h, qi0, b);
          tma_load_4d(sdO + st * Cfg::QTILE + a * 8192, &tmdO, qd_full(st), a * 64, h, qi0, b);
        }
      }
      const float* lse = p.lse + ((long long)b * p.nh + h) * p.Sq;
      const float* dlt = p.delta + ((long long)b * p.nh + h) * p.Sq;
      float* ld = ld_stage + st * 128;
#pragma unroll
      for (int i = lane; i < 64; i += 32) {
        const int qi = qi0 + i;
        ld[i] = qi < p.Sq ? __ldg(lse + qi) : 0.f;
        ld[64 + i] = qi < p.Sq ? __ldg(dlt + qi) : 0.f;
      }
      mbar_arrive(qd_full(st));
      if (++st == STAGES) { st = 0; ph ^= 1u; }
    }
    return;
  }

  // ================================ consumer warpgroups ================================
  setmaxnreg_inc<240>();
  const int wg = warp >> 2;
  const int kr = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's key rows kr, kr + 8 (S^T, dK, dV)
  const int cq = 2 * (lane & 3);
  const int wk0 = k0 + wg * 64 + (warp & 3) * 16;          // this warp's 16 key rows start here
  bool key_ok[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int kidx = k0 + kr + 8 * r;
    key_ok[r] = kidx < p.Skv && (!p.kmask || p.kmask[(size_t)b * p.Skv + kidx]);
  }
  const bool warp_keys_ok = __all_sync(0xffffffffu, key_ok[0] && key_ok[1]);
  float dv[HDP / 2], dk[HDP / 2];
#pragma unroll
  for (int i = 0; i < HDP / 2; ++i) dv[i] = dk[i] = 0.f;
  mbar_wait(kv_full, 0);
  int st = 0;
  uint32_t ph = 0;
  for (int it = 0; it < n_iter; ++it) {
    const int qi0 = (i_begin + it % n_i) * 64;
    const uint32_t qb = sQ + st * Cfg::QTILE, dob = sdO + st * Cfg::QTILE;
    mbar_wait(qd_full(st), ph);
    float sT[32], dpT[32];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < HDP / 16; ++kk) {
      const uint32_t koff = (kk >> 2) * 16384 + (kk & 3) * 32, qoff = (kk >> 2) * 8192 + (kk & 3) * 32;
      WgmmaSS<64, 0, 0>::mma(sT, make_smem_desc_sw128(sK + wg * 8192 + koff, 0, 1024),
                             make_smem_desc_sw128(qb + qoff, 0, 1024), kk ? 1u : 0u);
    }
#pragma unroll
    for (int kk = 0; kk < HDP / 16; ++kk) {
      const uint32_t koff = (kk >> 2) * 16384 + (kk & 3) * 32, qoff = (kk >> 2) * 8192 + (kk & 3) * 32;
      WgmmaSS<64, 0, 0>::mma(dpT, make_smem_desc_sw128(sV + wg * 8192 + koff, 0, 1024),
                             make_smem_desc_sw128(dob + qoff, 0, 1024), kk ? 1u : 0u);
    }
    wgmma_commit();
    // every (key, query) pair of the tile is visible to this warp: all 64 queries exist, the warp's 16 keys are valid
    // and none lies past the diagonal of the tile's first query
    const bool full = warp_keys_ok && qi0 + 64 <= p.Sq && (!p.causal || wk0 + 15 <= qi0 + coff);
    const float* ld = ld_stage + st * 128;
    wgmma_wait<0>();
    reg_fence(sT);
    reg_fence(dpT);
    // P^T = exp2(S^T * scale - lse) on visible (key, query) pairs, dS^T = P^T * (dP^T - delta): bf16 A fragments of
    // dV += P^T dO and dK += dS^T Q
    uint32_t pa[4][4], da[4][4];
    auto grads = [&](auto full_tile) {
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        float pv[4], dsv[4];
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int qc = 8 * jj + cq + c;
          const float L = ld[qc], D = ld[64 + qc];
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const int e = 2 * r + c;
            bool vis = true;
            if (!decltype(full_tile)::value)
              vis = qi0 + qc < p.Sq && key_ok[r] && (!p.causal || k0 + kr + 8 * r <= qi0 + qc + coff);
            const float pe = vis ? fast_exp2(fmaf(sT[4 * jj + e], p.scale_log2, -L)) : 0.f;
            pv[e] = pe;
            dsv[e] = pe * (dpT[4 * jj + e] - D);
          }
        }
        pa[jj >> 1][(jj & 1) * 2 + 0] = pack_bf16x2(pv[0], pv[1]);
        pa[jj >> 1][(jj & 1) * 2 + 1] = pack_bf16x2(pv[2], pv[3]);
        da[jj >> 1][(jj & 1) * 2 + 0] = pack_bf16x2(dsv[0], dsv[1]);
        da[jj >> 1][(jj & 1) * 2 + 1] = pack_bf16x2(dsv[2], dsv[3]);
      }
    };
    if (full)
      grads(std::true_type());
    else
      grads(std::false_type());
    reg_fence(dv);
    reg_fence(dk);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {  // K = 64 queries
      WgmmaRS<HDP, 1>::mma(dv, pa[kk], make_smem_desc_sw128(dob + kk * 2048, 8192, 1024), 1u);
      WgmmaRS<HDP, 1>::mma(dk, da[kk], make_smem_desc_sw128(qb + kk * 2048, 8192, 1024), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(dv);
    reg_fence(dk);
    if (lane == 0) mbar_arrive(qd_empty(st));  // this warp no longer reads the stage (wgmma operands, lse / delta)
    if (++st == STAGES) { st = 0; ph ^= 1u; }
  }
  // ---- epilogue: dK (x softmax scale), dV -> bf16 (zeros for keys no query sees)
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int kidx = k0 + kr + 8 * r;
    if (kidx >= p.Skv) continue;
    bf16* dkp = p.dk + (long long)b * p.dk_bs + (long long)kidx * p.dk_ss + (long long)g * p.hd;
    bf16* dvp = p.dv + (long long)b * p.dv_bs + (long long)kidx * p.dv_ss + (long long)g * p.hd;
#pragma unroll
    for (int jj = 0; jj < HDP / 8; ++jj) {
      const int d = 8 * jj + cq;
      *reinterpret_cast<__nv_bfloat162*>(dkp + d) =
          __floats2bfloat162_rn(dk[4 * jj + 2 * r] * p.scale, dk[4 * jj + 2 * r + 1] * p.scale);
      *reinterpret_cast<__nv_bfloat162*>(dvp + d) = __floats2bfloat162_rn(dv[4 * jj + 2 * r], dv[4 * jj + 2 * r + 1]);
    }
  }
}

template <int HDP>
struct DqCfg {
  static constexpr int ATOMS = HDP / 64;
  static constexpr int QTILE = ATOMS * 16384;  // [128 queries x hd]
  static constexpr int KTILE = ATOMS * 8192;   // [64 keys x hd]
  static constexpr int STAGES = 4;
  static constexpr int SMEM = 2 * QTILE + 2 * STAGES * KTILE + 1024 + 256;
};

template <int HDP>
__global__ void __launch_bounds__(288, 1)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                   const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO, AttnBwdParams p) {
  using Cfg = DqCfg<HDP>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sQ = base;
  const uint32_t sdO = sQ + Cfg::QTILE;
  const uint32_t sK = sdO + Cfg::QTILE;
  const uint32_t sV = sK + STAGES * Cfg::KTILE;
  const uint32_t bars = sV + STAGES * Cfg::KTILE;
  const uint32_t q_full = bars;
  auto kv_full = [&](int s) { return bars + 8u * (1 + s); };
  auto kv_empty = [&](int s) { return bars + 8u * (1 + STAGES + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q_tiles = (p.Sq + 127) / 128;
  const TileIdx ti = tile_index(p.nh, p.B);
  const int qt = q_tiles - 1 - ti.t;  // heavy (late) causal tiles first
  const int h = ti.h, b = ti.b;
  const int hk = h / (p.nh / p.nkv);
  const int q0 = qt * 128;
  const int coff = p.Skv - p.Sq;
  const int kv_tiles_all = (p.Skv + 63) / 64;
  int n_tiles = kv_tiles_all;
  if (p.causal) n_tiles = max(1, min(kv_tiles_all, (q0 + 127 + coff) / 64 + 1));

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    tma_prefetch_desc(&tmdO);
    mbar_init(q_full, 1);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(kv_full(s), 1);
      mbar_init(kv_empty(s), 2);  // one arrive per consumer warpgroup
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ================================ TMA producer ================================
    if (lane == 0) {
      mbar_arrive_expect_tx(q_full, 2 * Cfg::QTILE);
#pragma unroll
      for (int a = 0; a < Cfg::ATOMS; ++a) {
        tma_load_4d(sQ + a * 16384, &tmQ, q_full, a * 64, h, q0, b);
        tma_load_4d(sdO + a * 16384, &tmdO, q_full, a * 64, h, q0, b);
      }
      int st = 0;
      uint32_t ph = 0;
      for (int j = 0; j < n_tiles; ++j) {
        mbar_wait(kv_empty(st), ph ^ 1u);
        mbar_arrive_expect_tx(kv_full(st), 2 * Cfg::KTILE);
#pragma unroll
        for (int a = 0; a < Cfg::ATOMS; ++a) {
          tma_load_4d(sK + st * Cfg::KTILE + a * 8192, &tmK, kv_full(st), a * 64, hk, j * 64, b);
          tma_load_4d(sV + st * Cfg::KTILE + a * 8192, &tmV, kv_full(st), a * 64, hk, j * 64, b);
        }
        if (++st == STAGES) { st = 0; ph ^= 1u; }
      }
    }
    return;
  }

  // ================================ consumer warpgroups ================================
  const int wg = warp >> 2;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  const int rloc = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's query rows: rloc and rloc + 8
  const int cq = 2 * (lane & 3);
  const int wq0 = q0 + wg * 64 + (warp & 3) * 16;             // this warp's 16 query rows start here
  const uint8_t* km = p.kmask ? p.kmask + (size_t)b * p.Skv : nullptr;
  const float* lse = p.lse + ((long long)b * p.nh + h) * p.Sq;
  const float* dlt = p.delta + ((long long)b * p.nh + h) * p.Sq;
  int qi[2];
  float L[2], D[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    qi[r] = q0 + rloc + 8 * r;
    L[r] = qi[r] < p.Sq ? __ldg(lse + qi[r]) : 0.f;
    D[r] = qi[r] < p.Sq ? __ldg(dlt + qi[r]) : 0.f;
  }
  float dq[HDP / 2];
#pragma unroll
  for (int i = 0; i < HDP / 2; ++i) dq[i] = 0.f;
  mbar_wait(q_full, 0);
  int st = 0;
  uint32_t ph = 0;
  for (int j = 0; j < n_tiles; ++j) {
    const int k0 = j * 64;
    mbar_wait(kv_full(st), ph);
    const uint32_t kb = sK + st * Cfg::KTILE, vb = sV + st * Cfg::KTILE;
    float s[32], dp[32];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < HDP / 16; ++kk) {
      const uint32_t qoff = wg * 8192 + (kk >> 2) * 16384 + (kk & 3) * 32, koff = (kk >> 2) * 8192 + (kk & 3) * 32;
      WgmmaSS<64, 0, 0>::mma(s, make_smem_desc_sw128(sQ + qoff, 0, 1024), make_smem_desc_sw128(kb + koff, 0, 1024),
                             kk ? 1u : 0u);
    }
#pragma unroll
    for (int kk = 0; kk < HDP / 16; ++kk) {
      const uint32_t qoff = wg * 8192 + (kk >> 2) * 16384 + (kk & 3) * 32, koff = (kk >> 2) * 8192 + (kk & 3) * 32;
      WgmmaSS<64, 0, 0>::mma(dp, make_smem_desc_sw128(sdO + qoff, 0, 1024), make_smem_desc_sw128(vb + koff, 0, 1024),
                             kk ? 1u : 0u);
    }
    wgmma_commit();
    // every (query, key) pair of the tile is visible to this warp: the 64 keys lie inside Skv, at or before the
    // diagonal of the warp's first query, and are all valid; the warp's 16 queries exist
    bool full = k0 + 64 <= p.Skv && wq0 + 16 <= p.Sq && (!p.causal || k0 + 63 <= wq0 + coff);
    if (full && km) full = keys_all_valid<64>(km, k0);
    wgmma_wait<0>();
    reg_fence(s);
    reg_fence(dp);
    // dS = P * (dP - delta), P = exp2(S * scale - lse) on visible (query, key) pairs: bf16 A fragments of dQ += dS K
    uint32_t da[4][4];
    auto grads = [&](auto full_tile) {
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        float dsv[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int r = e >> 1, key = k0 + 8 * jj + cq + (e & 1);
          bool vis = true;
          if (!decltype(full_tile)::value)
            vis = qi[r] < p.Sq && key < p.Skv && (!p.causal || key <= qi[r] + coff) && (!km || km[key]);
          const float pe = vis ? fast_exp2(fmaf(s[4 * jj + e], p.scale_log2, -L[r])) : 0.f;
          dsv[e] = pe * (dp[4 * jj + e] - D[r]);
        }
        da[jj >> 1][(jj & 1) * 2 + 0] = pack_bf16x2(dsv[0], dsv[1]);
        da[jj >> 1][(jj & 1) * 2 + 1] = pack_bf16x2(dsv[2], dsv[3]);
      }
    };
    if (full)
      grads(std::true_type());
    else
      grads(std::false_type());
    reg_fence(dq);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)  // K = 64 keys; K read MN-major (hd contiguous)
      WgmmaRS<HDP, 1>::mma(dq, da[kk], make_smem_desc_sw128(kb + kk * 2048, 8192, 1024), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(dq);
    if (wg_leader) mbar_arrive(kv_empty(st));
    if (++st == STAGES) { st = 0; ph ^= 1u; }
  }
  // ---- epilogue: dQ x softmax scale in fp32, rounded once to bf16 (the caller's view may be a packed dQKV buffer)
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (qi[r] >= p.Sq) continue;
    bf16* dqp = p.dq + (long long)b * p.dq_bs + (long long)qi[r] * p.dq_ss + (long long)h * p.hd;
#pragma unroll
    for (int jj = 0; jj < HDP / 8; ++jj)
      *reinterpret_cast<__nv_bfloat162*>(dqp + 8 * jj + cq) =
          __floats2bfloat162_rn(dq[4 * jj + 2 * r] * p.scale, dq[4 * jj + 2 * r + 1] * p.scale);
  }
}

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
static PFN_cuTensorMapEncodeTiled_v12000 encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(ptr);
  }
  return fn;
}

// dims (d0 = head_dim contiguous, d1 = heads, d2 = sequence, d3 = batch); strides in elements
int make_tmap_bf16_4d(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t d3,
                      uint64_t s1, uint64_t s2, uint64_t s3, uint32_t box_rows) {
  auto fn = encode_fn();
  if (!fn) return set_error(CB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  if ((reinterpret_cast<uintptr_t>(base) & 15u) || (s1 % 8) || (s2 % 8) || (d3 > 1 && (s3 % 8)))
    return set_error(CB_ERR_INVALID, "attention: operands must be 16-byte aligned with strides %% 8 == 0");
  cuuint64_t dims[4] = {d0, d1, d2, d3};
  cuuint64_t strides[3] = {s1 * 2, s2 * 2, (d3 > 1 ? s3 : s2 * d2) * 2};
  cuuint32_t box[4] = {64, 1, box_rows, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r == CUDA_ERROR_INVALID_CONTEXT) {  // see gemm.cu: bind the primary context on lazily-initialised threads
    cudaFree(0);
    r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  if (r != CUDA_SUCCESS) return set_error(CB_ERR_CUDA, "cuTensorMapEncodeTiled(4d) failed (%d)", (int)r);
  return CB_OK;
}

static int hd_padded(int hd) { return (hd + 15) / 16 * 16; }

template <int HDP>
static int launch_fwd(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const AttnParams& p,
                      cudaStream_t st) {
  using Cfg = FwdCfg<HDP>;
  auto kern = attn_fwd_kernel<HDP>;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM);
    if (e != cudaSuccess) return set_error(CB_ERR_CUDA, "attn fwd smem attr: %s", cudaGetErrorString(e));
    attr = true;
  }
  kern<<<(p.Sq + 127) / 128 * p.nh * p.B, 288, Cfg::SMEM, st>>>(tq, tk, tv, p);
  CB_CUDA_LAUNCH_CHECK("attn_fwd");
  return CB_OK;
}

int attn_fwd_launch(const void* q, const void* k, const void* v, void* o, float* lse, const void* kmask, int B,
                    int nh, int nkv, int Sq, int Skv, int hd, long long q_bs, long long q_ss, long long k_bs,
                    long long k_ss, long long v_bs, long long v_ss, long long o_bs, long long o_ss, float scale,
                    int causal, cudaStream_t st) {
  CB_CHECK_ARG(B > 0 && nh > 0 && nkv > 0 && Sq > 0 && Skv > 0, "attention: empty problem");
  CB_CHECK_ARG(nh % nkv == 0, "attention: nh=%d not a multiple of nkv=%d", nh, nkv);
  CB_CHECK_ARG(hd % 8 == 0 && hd <= 128, "attention: head_dim=%d must be a multiple of 8 and <= 128", hd);
  CB_CHECK_ARG(o_ss % 8 == 0 && o_bs % 8 == 0 && !(reinterpret_cast<uintptr_t>(o) & 15u),
               "attention: output must be 16-byte aligned with strides %% 8 == 0");
  CUtensorMap tq, tk, tv;
  int rc;
  if ((rc = make_tmap_bf16_4d(&tq, q, hd, nh, Sq, B, hd, q_ss, q_bs, 128))) return rc;
  if ((rc = make_tmap_bf16_4d(&tk, k, hd, nkv, Skv, B, hd, k_ss, k_bs, 128))) return rc;
  if ((rc = make_tmap_bf16_4d(&tv, v, hd, nkv, Skv, B, hd, v_ss, v_bs, 128))) return rc;
  AttnParams p;
  p.o = (bf16*)o; p.o_bs = o_bs; p.o_ss = o_ss; p.lse = lse; p.kmask = (const uint8_t*)kmask;
  p.B = B; p.nh = nh; p.nkv = nkv; p.Sq = Sq; p.Skv = Skv; p.hd = hd; p.causal = causal;
  p.scale_log2 = scale * LOG2E;
  const int hdp = hd_padded(hd);
  if (hdp <= 64) return launch_fwd<64>(tq, tk, tv, p, st);
  if (hdp <= 80) return launch_fwd<80>(tq, tk, tv, p, st);
  if (hdp <= 96) return launch_fwd<96>(tq, tk, tv, p, st);
  return launch_fwd<128>(tq, tk, tv, p, st);
}

template <int HDP>
static int launch_bwd(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const CUtensorMap& tdo,
                      const AttnBwdParams& p, cudaStream_t st) {
  using Cfg = BwdCfg<HDP>;
  auto kern = attn_bwd_kernel<HDP>;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM);
    if (e != cudaSuccess) return set_error(CB_ERR_CUDA, "attn bwd smem attr: %s", cudaGetErrorString(e));
    attr = true;
  }
  kern<<<(p.Skv + 127) / 128 * p.nkv * p.B, 384, Cfg::SMEM, st>>>(tq, tk, tv, tdo, p);
  CB_CUDA_LAUNCH_CHECK("attn_bwd");
  return CB_OK;
}

template <int HDP>
static int launch_bwd_dq(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const CUtensorMap& tdo,
                         const AttnBwdParams& p, cudaStream_t st) {
  using Cfg = DqCfg<HDP>;
  auto kern = attn_bwd_dq_kernel<HDP>;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM);
    if (e != cudaSuccess) return set_error(CB_ERR_CUDA, "attn bwd dq smem attr: %s", cudaGetErrorString(e));
    attr = true;
  }
  kern<<<(p.Sq + 127) / 128 * p.nh * p.B, 288, Cfg::SMEM, st>>>(tq, tk, tv, tdo, p);
  CB_CUDA_LAUNCH_CHECK("attn_bwd_dq");
  return CB_OK;
}

int attn_bwd_launch(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                    float* delta, void* dq, void* dk, void* dv, const void* kmask, int B, int nh, int nkv,
                    int Sq, int Skv, int hd, long long q_bs, long long q_ss, long long k_bs, long long k_ss,
                    long long v_bs, long long v_ss, long long o_bs, long long o_ss, long long do_bs, long long do_ss,
                    long long dq_bs, long long dq_ss, long long dk_bs, long long dk_ss, long long dv_bs,
                    long long dv_ss, float scale, int causal, cudaStream_t st) {
  CB_CHECK_ARG(B > 0 && nh > 0 && nkv > 0 && Sq > 0 && Skv > 0, "attention bwd: empty problem");
  CB_CHECK_ARG(nh % nkv == 0, "attention bwd: nh=%d not a multiple of nkv=%d", nh, nkv);
  CB_CHECK_ARG(hd == 64 || hd == 128, "attention bwd: head_dim=%d unsupported (64 or 128)", hd);
  CB_CHECK_ARG(lse && delta && dq && dk && dv, "attention bwd: lse / delta / dq / dk / dv buffers are required");
  CB_CHECK_ARG(!(reinterpret_cast<uintptr_t>(dq) & 3u) && dq_bs % 2 == 0 && dq_ss % 2 == 0,
               "attention bwd: dq must be 4-byte aligned with even strides");
  {
    const long long warps = ((long long)B * Sq * nh + (256 / hd) - 1) / (256 / hd);   // 32 / (hd / 8) heads per warp
    attn_delta_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, st>>>((const bf16*)o, (const bf16*)d_o, delta, B,
                                                                           Sq, nh, hd, o_bs, o_ss, do_bs, do_ss);
    CB_CUDA_LAUNCH_CHECK("attn_delta");
  }
  CUtensorMap tq, tk, tv, tdo;
  int rc;
  if ((rc = make_tmap_bf16_4d(&tq, q, hd, nh, Sq, B, hd, q_ss, q_bs, 64))) return rc;
  if ((rc = make_tmap_bf16_4d(&tk, k, hd, nkv, Skv, B, hd, k_ss, k_bs, 128))) return rc;
  if ((rc = make_tmap_bf16_4d(&tv, v, hd, nkv, Skv, B, hd, v_ss, v_bs, 128))) return rc;
  if ((rc = make_tmap_bf16_4d(&tdo, d_o, hd, nh, Sq, B, hd, do_ss, do_bs, 64))) return rc;
  AttnBwdParams p;
  p.dq = (bf16*)dq; p.dk = (bf16*)dk; p.dv = (bf16*)dv;
  p.dq_bs = dq_bs; p.dq_ss = dq_ss; p.dk_bs = dk_bs; p.dk_ss = dk_ss; p.dv_bs = dv_bs; p.dv_ss = dv_ss;
  p.lse = lse; p.delta = delta; p.kmask = (const uint8_t*)kmask;
  p.B = B; p.nh = nh; p.nkv = nkv; p.Sq = Sq; p.Skv = Skv; p.hd = hd; p.causal = causal;
  p.scale_log2 = scale * LOG2E; p.scale = scale;
  // the dQ kernel streams 64-key K / V tiles against 128-query Q / dO tiles
  CUtensorMap tq128, tk64, tv64, tdo128;
  if ((rc = make_tmap_bf16_4d(&tq128, q, hd, nh, Sq, B, hd, q_ss, q_bs, 128))) return rc;
  if ((rc = make_tmap_bf16_4d(&tk64, k, hd, nkv, Skv, B, hd, k_ss, k_bs, 64))) return rc;
  if ((rc = make_tmap_bf16_4d(&tv64, v, hd, nkv, Skv, B, hd, v_ss, v_bs, 64))) return rc;
  if ((rc = make_tmap_bf16_4d(&tdo128, d_o, hd, nh, Sq, B, hd, do_ss, do_bs, 128))) return rc;
  if (hd == 64) {
    if ((rc = launch_bwd<64>(tq, tk, tv, tdo, p, st))) return rc;
    return launch_bwd_dq<64>(tq128, tk64, tv64, tdo128, p, st);
  }
  if ((rc = launch_bwd<128>(tq, tk, tv, tdo, p, st))) return rc;
  return launch_bwd_dq<128>(tq128, tk64, tv64, tdo128, p, st);
}

}  // namespace cb
