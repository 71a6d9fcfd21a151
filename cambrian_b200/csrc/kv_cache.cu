// cambrian_b200 — the decode KV caches: the dense FP8 cache of `generate(kv_cache_dtype="fp8")` and the paged cache of
// continuous batching (cambrian_b200/serving.py).
//
// Formats (the host modules own them and state them in full):
//   dense FP8 (cambrian_b200/kv_fp8.py): per layer kq, vq e4m3 [B, S_max, nkv, hd] and ks, vs fp32 [B, S_max, nkv];
//   paged (cambrian_b200/paged_kv.py): per layer K and V pages [num_pages, page_size, nkv, hd], bf16 or e4m3 with fp32
//     scales [num_pages, page_size, nkv]; a block table int32 [rows, table_ld] maps (row, position >> log2(page_size)) to
//     a page, and lens int32 [rows] holds each row's cached length, negative for an inactive (padding) row.
// Both store one position's nkv head rows in one cell: the row of (cell, kv head h) starts (cell * nkv + h) * hd
// elements in, its scale sits at cell * nkv + h, and the FP8 rows follow kv_fp8.py's row rule.  The caches differ only
// in which cell holds a position, which rows take part and how long each is, and that is all DenseCells and PagedCells
// say; the kernels below are written once over them, so the two caches share their bytes and their decode arithmetic.
//
//   kv_append_kernel    cb_kv_fp8_append, cb_paged_kv_append: new K / V head rows into their cells (bf16: a copy; FP8:
//                       the row rule)
//   kv_decode_kernel    cb_attn_decode_fp8, cb_attn_decode_paged: flash-decoding, one query per row, keys split over CTAs
//   kv_decode_combine   merges a row's splits in split order (no atomics) and rounds once to bf16
#include "common.cuh"
#include <cuda_fp16.h>
#include <algorithm>
#include <cfloat>

namespace cb {

// Every lane owns KV_DPL = 8 consecutive elements of one hd-element head row, so a row is a team of hd / 8 adjacent lanes
// (16 at hd 128, 8 at hd 64) and row reductions are xor-shuffles inside the team.
constexpr int KV_DPL = 8;
constexpr float KV_LOG2E = 1.4426950408889634f;

template <int LPK>
__device__ __forceinline__ float team_max(float v) {
#pragma unroll
  for (int o = LPK / 2; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
template <int LPK>
__device__ __forceinline__ float team_sum(float v) {
#pragma unroll
  for (int o = LPK / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// 8 e4m3 (lowest byte first) -> 8 fp32, exactly: two values per packed cvt to f16x2, then f16 -> f32
__device__ __forceinline__ void e4m3x8_to_f32(uint2 u, float* f) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint16_t pair = (uint16_t)(((i < 2) ? u.x : u.y) >> (16 * (i & 1)));
    uint32_t h2;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h2) : "h"(pair));
    const float2 t = __half22float2(*reinterpret_cast<const __half2*>(&h2));
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}

// Merges n (m, l, o[]) states in order, state i at s + i * stride: M = max m_i and, with w_i = exp(m_i - M) (0 for an
// empty state), Ls = sum l_i w_i and Os = sum o_i[d] w_i.
__device__ __forceinline__ void kv_merge(const float* s, int n, int stride, int d, float& M, float& Ls, float& Os) {
  M = -INFINITY;
  for (int i = 0; i < n; ++i) M = fmaxf(M, s[i * stride]);
  Ls = Os = 0.f;
  if (M == -INFINITY) return;
  for (int i = 0; i < n; ++i) {
    const float mi = s[i * stride];
    const float w = mi == -INFINITY ? 0.f : fast_exp2((mi - M) * KV_LOG2E);
    Ls = fmaf(s[i * stride + 1], w, Ls);
    Os = fmaf(s[i * stride + 2 + d], w, Os);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Cell addressing, for row b of a launch: active(b) (an inactive row is neither written nor read); base(b) (an append's
// first position, or a decode's valid length before the kernels clip it to cap); cell(b, t) for 0 <= t < cap (the cell
// of position t, -1 when there is none); key_mask(b) (a decode's key mask row, null for none); kDirect (a decode of one
// split normalises and stores o itself, without the combine).
// ---------------------------------------------------------------------------------------------------------------------

// The dense FP8 cache: position t of sequence b is cell b * S_max + t; base = pos (+ *pos_dev, the device slot of the
// graph-replayed step).
struct DenseCells {
  long long cap;  // S_max
  long long pos;
  const long long* pos_dev;
  const uint8_t* kmask;
  long long kmask_ld;
  static constexpr bool kDirect = true;
  __device__ bool active(int) const { return true; }
  __device__ long long base(int) const { return pos + (pos_dev ? *pos_dev : 0); }
  __device__ long long cell(int b, long long t) const { return b * cap + t; }
  __device__ const uint8_t* key_mask(int b) const { return kmask ? kmask + b * kmask_ld : nullptr; }
};

// The paged cache: position t of row b is slot t % page_size of page table[b, t / page_size], none when that entry is
// not a page of the pool; base = pos (+ lens[b] with from_lens, which a decode always sets).  Its key mask is null at
// compile time, so its decode carries no mask test.
struct PagedCells {
  long long cap;  // max_pages * page_size
  long long pos;
  const int* lens;
  int from_lens;
  const int* table;
  long long table_ld;
  int lg_ps, num_pages;
  static constexpr bool kDirect = false;
  __device__ bool active(int b) const { return !lens || lens[b] >= 0; }
  __device__ long long base(int b) const { return pos + (from_lens ? lens[b] : 0); }
  __device__ long long cell(int b, long long t) const {
    const int page = table[b * table_ld + (t >> lg_ps)];
    if (page < 0 || page >= num_pages) return -1;
    return ((long long)page << lg_ps) | (t & ((1LL << lg_ps) - 1));
  }
  __device__ const uint8_t* key_mask(int) const { return nullptr; }
};

// ---------------------------------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------------------------------

// Team r handles row r = ((b * S + s) * nkv + h) * 2 + (0: K, 1: V) of the new tokens, written at position base(b) + s;
// a position outside [0, cap) or without a cell writes nothing.  No early exit before the team reduction: every lane of
// a warp takes part in the shuffles.
template <int HD, bool F8, class Cells>
__global__ void __launch_bounds__(256)
kv_append_kernel(const bf16* __restrict__ k, const bf16* __restrict__ v, long long ld, void* __restrict__ kc,
                 void* __restrict__ vc, float* __restrict__ ksc, float* __restrict__ vsc, Cells cells, int B, int S,
                 int nkv) {
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
  const uint4 raw = *reinterpret_cast<const uint4*>(src);
  float f[8];
  float a = 0.f;
  if (F8) {
    unpack8(raw, f);
#pragma unroll
    for (int e = 0; e < 8; ++e) a = fmaxf(a, fabsf(f[e]));
    a = team_max<LPK>(a);
  }
  if (!in_range || !cells.active(b)) return;
  const long long pos = cells.base(b) + s;
  if (pos < 0 || pos >= cells.cap) return;
  const long long cell = cells.cell(b, pos);
  if (cell < 0) return;
  const long long dst = (cell * nkv + h) * HD + sub * KV_DPL;
  if (F8) {
    // the row rule of kv_fp8.py: scale a / 448, bytes round_satfinite(f * fmin(448 / a, FLT_MAX))
    const float rr = fminf(__fdiv_rn(448.0f, a), FLT_MAX);
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = __fmul_rn(f[e], rr);
    if (sub == 0) (which ? vsc : ksc)[cell * nkv + h] = __fdiv_rn(a, 448.0f);
    *reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(which ? vc : kc) + dst) = f8_pack8(f);
  } else {
    *reinterpret_cast<uint4*>(reinterpret_cast<bf16*>(which ? vc : kc) + dst) = raw;
  }
}

// CTA (split, kv head h, row b), KVD_THREADS threads = TEAMS teams of LPK lanes.  The CTA owns the G query heads of
// kv head h and keys [split * chunk, +chunk) clipped to the row's valid length L; an inactive row, or a split
// wholly past L, returns before it reads anything, except split 0 of the dense cache, which always runs so that a
// single split stores zeros for an empty cache.  Each team walks its keys (team, team + TEAMS, ...) BLK at a time:
// per key one load of K and of V per lane (16 bytes bf16, 8 bytes e4m3), G dot products of 8 elements from
// registers, a team sum, then per head the score (bf16: dot * scale; FP8: (dot * ks) * scale) and an online softmax
// in fp32 (one rescale per BLK keys); o += p * v (FP8: (p * vs) * float(vq)).  Keys without a cell or masked out are
// never loaded.  The teams' (m, l, o) states are merged in team order through shared memory; in a dense launch of
// one split the CTA normalises and stores, otherwise it writes its state to the workspace slot (row, query head,
// split) for kv_decode_combine.  Fixed orders throughout: bitwise run to run.
constexpr int KVD_THREADS = 128;
constexpr int KVD_MIN_CHUNK = 256;    // dense: keys a split owns at least
constexpr int KVD_MAX_SPLITS = 64;    // dense: splits at most
constexpr int KVD_PAGED_CHUNK = 256;  // paged: keys per split, a constant, never a function of the batch or the SM count

template <int HD, int G, bool F8, class Cells>
__global__ void __launch_bounds__(KVD_THREADS)
kv_decode_kernel(const bf16* __restrict__ q, long long q_bs, const void* __restrict__ kc, const void* __restrict__ vc,
                 const float* __restrict__ ksc, const float* __restrict__ vsc, Cells cells, bf16* __restrict__ o,
                 float* __restrict__ ws, int nkv, int chunk, int nsplit, float scale) {
  constexpr int LPK = HD / KV_DPL;
  constexpr int TEAMS = KVD_THREADS / LPK;
  constexpr int BLK = G <= 4 ? 4 : 2;
  constexpr int ST = HD + 2;  // per-head state: m, l, o[HD]
  __shared__ float red[TEAMS][G][ST];
  const int split = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int nh = nkv * G;
  if (!cells.active(b)) return;
  const long long L = min(cells.base(b), cells.cap);
  const int t0 = split * chunk;  // key positions fit in int: L < 2^31 in both caches
  if (t0 >= L && (split > 0 || !Cells::kDirect)) return;
  const int t1 = (int)min((long long)t0 + chunk, L);
  const int team = threadIdx.x / LPK, sub = threadIdx.x % LPK;
  const uint8_t* mb = cells.key_mask(b);

  float qf[G][8];
#pragma unroll
  for (int g = 0; g < G; ++g)
    unpack8(*reinterpret_cast<const uint4*>(q + (long long)b * q_bs + (h * G + g) * HD + sub * KV_DPL), qf[g]);

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
    uint4 kr[BLK], vr[BLK];
    float ksv[BLK], vsv[BLK];
    unsigned okm = 0u;  // bit j: key j of the block is valid
#pragma unroll
    for (int j = 0; j < BLK; ++j) {
      const int t = base + team + j * TEAMS;
      long long cell = t < t1 ? cells.cell(b, t) : -1;
      if (mb && t < t1 && !mb[t]) cell = -1;  // the mask byte and the cell load independently of each other
      okm |= cell >= 0 ? 1u << j : 0u;
      kr[j] = vr[j] = make_uint4(0u, 0u, 0u, 0u);
      ksv[j] = vsv[j] = 0.f;
      if (cell >= 0) {
        const long long off = (cell * nkv + h) * HD + sub * KV_DPL;
        if (F8) {
          const uint2 k2 = *reinterpret_cast<const uint2*>(reinterpret_cast<const uint8_t*>(kc) + off);
          const uint2 v2 = *reinterpret_cast<const uint2*>(reinterpret_cast<const uint8_t*>(vc) + off);
          kr[j] = make_uint4(k2.x, k2.y, 0u, 0u);
          vr[j] = make_uint4(v2.x, v2.y, 0u, 0u);
          ksv[j] = ksc[cell * nkv + h];
          vsv[j] = vsc[cell * nkv + h];
        } else {
          kr[j] = *reinterpret_cast<const uint4*>(reinterpret_cast<const bf16*>(kc) + off);
          vr[j] = *reinterpret_cast<const uint4*>(reinterpret_cast<const bf16*>(vc) + off);
        }
      }
    }
    float s[BLK][G];
#pragma unroll
    for (int j = 0; j < BLK; ++j) {
      float kf[8];
      if (F8)
        e4m3x8_to_f32(make_uint2(kr[j].x, kr[j].y), kf);
      else
        unpack8(kr[j], kf);
#pragma unroll
      for (int g = 0; g < G; ++g) {
        float d = 0.f;
#pragma unroll
        for (int e = 0; e < 8; ++e) d = fmaf(qf[g][e], kf[e], d);
        d = team_sum<LPK>(d);
        const float sc = F8 ? __fmul_rn(__fmul_rn(d, ksv[j]), scale) : __fmul_rn(d, scale);
        s[j][g] = (okm >> j) & 1u ? sc : -INFINITY;
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
        pv[j][g] = F8 ? __fmul_rn(p, vsv[j]) : p;
      }
      l[g] = ls;
      m[g] = mx;
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[g][e] = __fmul_rn(acc[g][e], c);
    }
#pragma unroll
    for (int j = 0; j < BLK; ++j) {
      float vf[8];
      if (F8)
        e4m3x8_to_f32(make_uint2(vr[j].x, vr[j].y), vf);
      else
        unpack8(vr[j], vf);
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
    float M, Ls, Os;
    kv_merge(&red[0][g][0], TEAMS, G * ST, d, M, Ls, Os);
    const long long bh = (long long)b * nh + h * G + g;
    if (Cells::kDirect && nsplit == 1) {
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

// one CTA per (row, query head), thread d: the splits below the row's valid length, merged in split order; an inactive
// or empty row gets zeros
template <int HD, class Cells>
__global__ void __launch_bounds__(HD) kv_decode_combine(const float* __restrict__ ws, bf16* __restrict__ o, Cells cells,
                                                        int nh, int chunk, int nsplit) {
  constexpr int ST = HD + 2;
  const long long bh = blockIdx.x;
  const int b = (int)(bh / nh);
  const long long L = cells.active(b) ? min(cells.base(b), cells.cap) : 0;
  const int active = L <= 0 ? 0 : (int)(((unsigned)L + chunk - 1) / (unsigned)chunk);  // L < 2^31 in both caches
  const int d = threadIdx.x;
  float M, Ls, Os;
  kv_merge(ws + bh * nsplit * ST, active, ST, d, M, Ls, Os);
  o[bh * HD + d] = __float2bfloat16(Ls > 0.f ? __fdiv_rn(Os, Ls) : 0.f);
}

// ---------------------------------------------------------------------------------------------------------------------
// host side: the launches both caches share, then each cache's entry points (their checks, cells and split policy)
// ---------------------------------------------------------------------------------------------------------------------
template <bool F8, class Cells>
static int kv_append(const char* who, const Cells& cells, const void* k, const void* v, long long ld, void* kc, void* vc,
                     float* ksc, float* vsc, int B, int S, int nkv, int hd, cudaStream_t st) {
  const long long blocks = (2LL * B * S * nkv * (hd / KV_DPL) + 255) / 256;
  CB_CHECK_ARG(blocks < (1LL << 31), "%s: too many rows", who);
  (hd == 128 ? kv_append_kernel<128, F8, Cells> : kv_append_kernel<64, F8, Cells>)<<<(unsigned)blocks, 256, 0, st>>>(
      (const bf16*)k, (const bf16*)v, ld, kc, vc, ksc, vsc, cells, B, S, nkv);
  CB_CUDA_LAUNCH_CHECK("kv_append_kernel");
  return CB_OK;
}

// The split kernel over grid (nsplit, nkv, rows), then the combine, which a dense launch of one split does not need.
template <bool F8, class Cells>
static int kv_decode(const Cells& cells, int hd, const void* q, long long q_bs, const void* kc, const void* vc,
                     const float* ksc, const float* vsc, void* o, float* ws, int rows, int nh, int nkv, int chunk,
                     int nsplit, float scale, cudaStream_t st) {
#define KVD_G(HD)                                                                                              \
  {kv_decode_kernel<HD, 1, F8, Cells>, kv_decode_kernel<HD, 2, F8, Cells>, kv_decode_kernel<HD, 3, F8, Cells>, \
   kv_decode_kernel<HD, 4, F8, Cells>, kv_decode_kernel<HD, 5, F8, Cells>, kv_decode_kernel<HD, 6, F8, Cells>, \
   kv_decode_kernel<HD, 7, F8, Cells>, kv_decode_kernel<HD, 8, F8, Cells>}
  static decltype(&kv_decode_kernel<64, 1, F8, Cells>) const kernels[2][8] = {KVD_G(64), KVD_G(128)};
#undef KVD_G
  kernels[hd == 128][nh / nkv - 1]<<<dim3(nsplit, nkv, rows), KVD_THREADS, 0, st>>>(
      (const bf16*)q, q_bs, kc, vc, ksc, vsc, cells, (bf16*)o, ws, nkv, chunk, nsplit, scale);
  CB_CUDA_LAUNCH_CHECK("kv_decode_kernel");
  if (Cells::kDirect && nsplit == 1) return CB_OK;
  (hd == 128 ? kv_decode_combine<128, Cells> : kv_decode_combine<64, Cells>)<<<rows * nh, hd, 0, st>>>(
      ws, (bf16*)o, cells, nh, chunk, nsplit);
  CB_CUDA_LAUNCH_CHECK("kv_decode_combine");
  return CB_OK;
}

// ---- the dense FP8 cache ----

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
  const DenseCells cells{S_max, offset, offset_dev, nullptr, 0};
  return kv_append<true>("kv_fp8_append", cells, k, v, ld, kq, vq, ks, vs, B, S, nkv, hd, st);
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
  const long long need = attn_decode_fp8_workspace_floats(B, nh, nkv, S_max, hd);
  CB_CHECK_ARG(need == 0 || (ws && ws_floats >= need), "attn_decode_fp8: workspace of %lld floats, %lld needed", ws_floats,
               need);
  const DenseCells cells{S_max, length, length_dev, (const uint8_t*)kmask, kmask_ld};
  return kv_decode<true>(cells, hd, q, q_bs, kq, vq, ks, vs, o, ws, B, nh, nkv, chunk, nsplit, scale, st);
}

// ---- the paged cache ----

// the checks both entry points share: the page geometry and the block table's host-visible shape
static int paged_geometry(const char* who, int rows, int nkv, int hd, int page_size, int num_pages, int max_pages,
                          long long table_ld) {
  CB_CHECK_ARG(hd == 64 || hd == 128, "%s: hd=%d must be 64 or 128", who, hd);
  CB_CHECK_ARG(page_size >= 16 && page_size <= (1 << 20) && (page_size & (page_size - 1)) == 0,
               "%s: page_size=%d must be a power of two >= 16", who, page_size);
  CB_CHECK_ARG(rows > 0 && rows < 65536 && nkv > 0 && nkv < 65536, "%s: bad shape (rows=%d nkv=%d)", who, rows, nkv);
  CB_CHECK_ARG(num_pages > 0 && max_pages > 0, "%s: empty page pool or table (num_pages=%d max_pages=%d)", who, num_pages,
               max_pages);
  CB_CHECK_ARG(table_ld >= max_pages, "%s: block table row stride %lld is below max_pages=%d", who, table_ld, max_pages);
  CB_CHECK_ARG((long long)max_pages * page_size < (1LL << 31), "%s: max_pages * page_size exceeds 2^31 positions", who);
  return CB_OK;
}

int paged_kv_append_launch(const void* k, const void* v, long long ld, void* kp, void* vp, float* ksc, float* vsc, int fp8,
                           const int* table, long long table_ld, const int* lens, int rows, int S, int nkv, int hd,
                           int page_size, int num_pages, int max_pages, long long offset, int from_lens, cudaStream_t st) {
  int rc = paged_geometry("paged_kv_append", rows, nkv, hd, page_size, num_pages, max_pages, table_ld);
  if (rc != CB_OK) return rc;
  CB_CHECK_ARG(S > 0, "paged_kv_append: S=%d new rows per sequence", S);
  CB_CHECK_ARG(k && v && kp && vp && table && (!fp8 || (ksc && vsc)), "paged_kv_append: null argument");
  CB_CHECK_ARG(!from_lens || lens, "paged_kv_append: the start position comes from lens, but lens is null");
  CB_CHECK_ARG(ld >= (long long)nkv * hd && ld % 8 == 0,
               "paged_kv_append: row stride %lld must be >= nkv*hd and a multiple of 8", ld);
  CB_CHECK_ARG(((reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v)) & 15u) == 0 &&
                   ((reinterpret_cast<uintptr_t>(kp) | reinterpret_cast<uintptr_t>(vp)) & 15u) == 0 &&
                   ((reinterpret_cast<uintptr_t>(ksc) | reinterpret_cast<uintptr_t>(vsc)) & 3u) == 0,
               "paged_kv_append: k, v and the pages must be 16-byte aligned");
  const long long max_pos = (long long)max_pages * page_size;
  CB_CHECK_ARG(offset >= 0 && (from_lens || offset + S <= max_pos),
               "paged_kv_append: positions [%lld, %lld) outside the table (%lld)", offset, offset + S, max_pos);
  const PagedCells cells{max_pos, offset, lens, from_lens, table, table_ld, __builtin_ctz(page_size), num_pages};
  if (fp8) return kv_append<true>("paged_kv_append", cells, k, v, ld, kp, vp, ksc, vsc, rows, S, nkv, hd, st);
  return kv_append<false>("paged_kv_append", cells, k, v, ld, kp, vp, ksc, vsc, rows, S, nkv, hd, st);
}

static long long paged_splits(int max_pages, int page_size) {
  return ((long long)max_pages * page_size + KVD_PAGED_CHUNK - 1) / KVD_PAGED_CHUNK;
}

long long attn_decode_paged_workspace_floats(int rows, int nh, int max_pages, int page_size, int hd) {
  if (rows <= 0 || nh <= 0 || max_pages <= 0 || page_size <= 0 || hd <= 0) return 0;
  return (long long)rows * nh * paged_splits(max_pages, page_size) * (hd + 2);
}

int attn_decode_paged_launch(const void* q, long long q_bs, const void* kp, const void* vp, const float* ksc,
                             const float* vsc, int fp8, const int* table, long long table_ld, const int* lens, int len_add,
                             void* o, float* ws, long long ws_floats, int rows, int nh, int nkv, int hd, int page_size,
                             int num_pages, int max_pages, float scale, cudaStream_t st) {
  int rc = paged_geometry("attn_decode_paged", rows, nkv, hd, page_size, num_pages, max_pages, table_ld);
  if (rc != CB_OK) return rc;
  CB_CHECK_ARG(nh % nkv == 0 && nh / nkv >= 1 && nh / nkv <= 8,
               "attn_decode_paged: nh=%d must be 1..8 times nkv=%d (query heads per kv head)", nh, nkv);
  CB_CHECK_ARG(q && kp && vp && table && lens && o && ws && (!fp8 || (ksc && vsc)), "attn_decode_paged: null argument");
  CB_CHECK_ARG(len_add >= 0, "attn_decode_paged: len_add=%d must be >= 0", len_add);
  CB_CHECK_ARG(((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(o)) & 15u) == 0 && q_bs % 8 == 0 &&
                   q_bs >= (long long)nh * hd &&
                   ((reinterpret_cast<uintptr_t>(kp) | reinterpret_cast<uintptr_t>(vp)) & 15u) == 0 &&
                   ((reinterpret_cast<uintptr_t>(ksc) | reinterpret_cast<uintptr_t>(vsc)) & 3u) == 0,
               "attn_decode_paged: q, o and the pages must be 16-byte aligned (q row stride a multiple of 8, >= nh*hd)");
  const long long nsplit = paged_splits(max_pages, page_size);
  const long long need = attn_decode_paged_workspace_floats(rows, nh, max_pages, page_size, hd);
  CB_CHECK_ARG(ws_floats >= need, "attn_decode_paged: workspace of %lld floats, %lld needed", ws_floats, need);
  CB_CHECK_ARG(nsplit < (1LL << 31), "attn_decode_paged: too many splits");
  // every split is combined, even a single one, so a row's result never depends on the other rows or the grid
  const PagedCells cells{(long long)max_pages * page_size, len_add, lens, 1, table, table_ld, __builtin_ctz(page_size),
                         num_pages};
  if (fp8)
    return kv_decode<true>(cells, hd, q, q_bs, kp, vp, ksc, vsc, o, ws, rows, nh, nkv, KVD_PAGED_CHUNK, (int)nsplit, scale,
                           st);
  return kv_decode<false>(cells, hd, q, q_bs, kp, vp, ksc, vsc, o, ws, rows, nh, nkv, KVD_PAGED_CHUNK, (int)nsplit, scale,
                          st);
}

}  // namespace cb
