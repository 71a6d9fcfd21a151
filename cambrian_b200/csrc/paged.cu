// cambrian_b200 — paged decode KV cache for continuous batching (cambrian_b200/serving.py).
//
// Format (cambrian_b200/paged_kv.py owns it on the host and states it in full): per layer K and V pages
// [num_pages, page_size, nkv, hd], bf16 or e4m3 with fp32 scales [num_pages, page_size, nkv] (the row rule of kv_fp8.py);
// a block table int32 [rows, table_ld] maps (row, position >> log2(page_size)) to a page; lens int32 [rows] holds each
// row's cached length, negative for an inactive (padding) row.
//
//   paged_append_kernel   cb_paged_kv_append: new K / V head rows into their pages (bf16: a copy; FP8: the row rule,
//                         bit for bit what kv_fp8_append_kernel writes)
//   paged_decode_kernel   cb_attn_decode_paged: flash-decoding over each row's pages, one query per row; every split
//                         covers PD_CHUNK key positions, so a row's result never depends on the other rows or the grid
//   paged_decode_combine  merges a row's splits in split order (no atomics) and rounds once to bf16
#include "common.cuh"
#include "kv_rows.cuh"
#include <algorithm>

namespace cb {

constexpr int PD_THREADS = 128;
constexpr int PD_CHUNK = 256;  // key positions per split: a constant, never a function of the batch or the SM count

// Page cell of position t of row b (the index of its (page, slot) pair in [num_pages * page_size]), or -1 when the
// table holds no valid page there.
__device__ __forceinline__ long long paged_cell(const int* __restrict__ table, long long table_ld, int b, long long t,
                                                int lg_ps, int num_pages) {
  const int page = table[(long long)b * table_ld + (t >> lg_ps)];
  if (page < 0 || page >= num_pages) return -1;
  return ((long long)page << lg_ps) | (t & ((1LL << lg_ps) - 1));
}

// Team r handles row r = ((b * S + s) * nkv + h) * 2 + (0: K, 1: V) of the new tokens, written at position
// offset (+ lens[b]) + s.  No early exit before the team reduction: every lane of a warp takes part in the shuffles.
template <int HD, bool F8>
__global__ void __launch_bounds__(256)
paged_append_kernel(const bf16* __restrict__ k, const bf16* __restrict__ v, long long ld, void* __restrict__ kp,
                    void* __restrict__ vp, float* __restrict__ ksc, float* __restrict__ vsc, const int* __restrict__ table,
                    long long table_ld, const int* __restrict__ lens, int rows_b, int S, int nkv, int lg_ps, int num_pages,
                    long long max_pos, long long offset, int from_lens) {
  constexpr int LPK = HD / KV_DPL;
  const long long rows = 2LL * rows_b * S * nkv;
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
  if (!in_range) return;
  const int len = lens ? lens[b] : 0;
  if (len < 0) return;  // inactive row
  const long long pos = offset + (from_lens ? len : 0) + s;
  if (pos < 0 || pos >= max_pos) return;
  const long long cell = paged_cell(table, table_ld, b, pos, lg_ps, num_pages);
  if (cell < 0) return;
  const long long dst = (cell * nkv + h) * HD + sub * KV_DPL;
  if (F8) {
    float sc;
    const uint2 packed = kv_quant8(f, a, &sc);
    if (sub == 0) (which ? vsc : ksc)[cell * nkv + h] = sc;
    *reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(which ? vp : kp) + dst) = packed;
  } else {
    *reinterpret_cast<uint4*>(reinterpret_cast<bf16*>(which ? vp : kp) + dst) = raw;
  }
}

// CTA (split, kv head h, row b), PD_THREADS threads = TEAMS teams of LPK lanes.  The CTA owns the G query heads of kv
// head h and keys [split * PD_CHUNK, +PD_CHUNK) clipped to the row's valid length L = lens[b] + len_add; a split wholly
// past L (or an inactive row) returns before it reads anything.  Each team walks its keys (team, team + TEAMS, ...) BLK
// at a time: per key one load of K and of V per lane (16 bytes bf16, 8 bytes e4m3) through the block table, G dot
// products of 8 elements from registers, a team sum, then per head the score (bf16: dot * scale; FP8: (dot * ks) *
// scale) and an online softmax in fp32; o += p * v (FP8: (p * vs) * float(vq)).  The teams' (m, l, o) states are merged
// in team order through shared memory and written to the workspace slot (row, query head, split).
template <int HD, int G, bool F8>
__global__ void __launch_bounds__(PD_THREADS)
paged_decode_kernel(const bf16* __restrict__ q, long long q_bs, const void* __restrict__ kp, const void* __restrict__ vp,
                    const float* __restrict__ ksc, const float* __restrict__ vsc, const int* __restrict__ table,
                    long long table_ld, const int* __restrict__ lens, int len_add, float* __restrict__ ws, int nkv,
                    int lg_ps, int num_pages, long long max_pos, int nsplit, float scale) {
  constexpr int LPK = HD / KV_DPL;
  constexpr int TEAMS = PD_THREADS / LPK;
  constexpr int BLK = G <= 4 ? 4 : 2;
  constexpr int ST = HD + 2;  // per-head state: m, l, o[HD]
  __shared__ float red[TEAMS][G][ST];
  const int split = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int nh = nkv * G;
  const int len = lens[b];
  if (len < 0) return;
  long long L = (long long)len + len_add;
  L = L < max_pos ? L : max_pos;
  const long long t0 = (long long)split * PD_CHUNK;
  if (t0 >= L) return;
  const long long t1 = t0 + PD_CHUNK < L ? t0 + PD_CHUNK : L;
  const int team = threadIdx.x / LPK, sub = threadIdx.x % LPK;

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
  for (long long base = t0; base < t1; base += TEAMS * BLK) {
    uint4 kr[BLK], vr[BLK];
    float ksv[BLK], vsv[BLK];
    unsigned okm = 0u;  // bit j: key j of the block is valid
#pragma unroll
    for (int j = 0; j < BLK; ++j) {
      const long long t = base + team + j * TEAMS;
      const long long cell = t < t1 ? paged_cell(table, table_ld, b, t, lg_ps, num_pages) : -1;
      okm |= cell >= 0 ? 1u << j : 0u;
      kr[j] = vr[j] = make_uint4(0u, 0u, 0u, 0u);
      ksv[j] = vsv[j] = 0.f;
      if (cell >= 0) {
        const long long off = (cell * nkv + h) * HD + sub * KV_DPL;
        if (F8) {
          const uint2 k2 = *reinterpret_cast<const uint2*>(reinterpret_cast<const uint8_t*>(kp) + off);
          const uint2 v2 = *reinterpret_cast<const uint2*>(reinterpret_cast<const uint8_t*>(vp) + off);
          kr[j] = make_uint4(k2.x, k2.y, 0u, 0u);
          vr[j] = make_uint4(v2.x, v2.y, 0u, 0u);
          ksv[j] = ksc[cell * nkv + h];
          vsv[j] = vsc[cell * nkv + h];
        } else {
          kr[j] = *reinterpret_cast<const uint4*>(reinterpret_cast<const bf16*>(kp) + off);
          vr[j] = *reinterpret_cast<const uint4*>(reinterpret_cast<const bf16*>(vp) + off);
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
  for (int i = threadIdx.x; i < G * HD; i += PD_THREADS) {
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
    float* w = ws + (((long long)b * nh + h * G + g) * nsplit + split) * ST;
    if (d == 0) {
      w[0] = M;
      w[1] = Ls;
    }
    w[2 + d] = Os;
  }
}

// one CTA per (row, query head), thread d: the splits below the row's valid length, merged in split order; an inactive
// or empty row gets zeros
template <int HD>
__global__ void __launch_bounds__(HD)
paged_decode_combine(const float* __restrict__ ws, bf16* __restrict__ o, const int* __restrict__ lens, int len_add, int nh,
                     long long max_pos, int nsplit) {
  constexpr int ST = HD + 2;
  const long long bh = blockIdx.x;
  const int len = lens[bh / nh];
  long long L = len < 0 ? 0 : (long long)len + len_add;
  L = L < max_pos ? L : max_pos;
  const int active = L <= 0 ? 0 : (int)((L + PD_CHUNK - 1) / PD_CHUNK);
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

static int log2_page(int page_size) {
  int lg = 0;
  while ((1 << lg) < page_size) ++lg;
  return lg;
}

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
  const long long threads = 2LL * rows * S * nkv * (hd / KV_DPL);
  const long long blocks = (threads + 255) / 256;
  CB_CHECK_ARG(blocks < (1LL << 31), "paged_kv_append: too many rows");
  const int lg = log2_page(page_size);
#define PA_LAUNCH(HD, F8)                                                                                          \
  paged_append_kernel<HD, F8><<<(unsigned)blocks, 256, 0, st>>>((const bf16*)k, (const bf16*)v, ld, kp, vp, ksc, vsc, \
                                                                table, table_ld, lens, rows, S, nkv, lg, num_pages,   \
                                                                max_pos, offset, from_lens)
  if (hd == 128) {
    if (fp8) PA_LAUNCH(128, true); else PA_LAUNCH(128, false);
  } else {
    if (fp8) PA_LAUNCH(64, true); else PA_LAUNCH(64, false);
  }
#undef PA_LAUNCH
  CB_CUDA_LAUNCH_CHECK("paged_append_kernel");
  return CB_OK;
}

static long long paged_splits(int max_pages, int page_size) {
  return ((long long)max_pages * page_size + PD_CHUNK - 1) / PD_CHUNK;
}

long long attn_decode_paged_workspace_floats(int rows, int nh, int max_pages, int page_size, int hd) {
  if (rows <= 0 || nh <= 0 || max_pages <= 0 || page_size <= 0 || hd <= 0) return 0;
  return (long long)rows * nh * paged_splits(max_pages, page_size) * (hd + 2);
}

template <int HD, bool F8>
static void pd_launch(int G, dim3 grid, cudaStream_t st, const bf16* q, long long q_bs, const void* kp, const void* vp,
                      const float* ksc, const float* vsc, const int* table, long long table_ld, const int* lens,
                      int len_add, float* ws, int nkv, int lg, int num_pages, long long max_pos, int nsplit, float scale) {
#define PD_CASE(GG)                                                                                                 \
  case GG:                                                                                                          \
    paged_decode_kernel<HD, GG, F8><<<grid, PD_THREADS, 0, st>>>(q, q_bs, kp, vp, ksc, vsc, table, table_ld, lens,   \
                                                                 len_add, ws, nkv, lg, num_pages, max_pos, nsplit, \
                                                                 scale);                                            \
    break;
  switch (G) {
    PD_CASE(1) PD_CASE(2) PD_CASE(3) PD_CASE(4) PD_CASE(5) PD_CASE(6) PD_CASE(7) PD_CASE(8)
  }
#undef PD_CASE
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
  const long long need = (long long)rows * nh * nsplit * (hd + 2);
  CB_CHECK_ARG(ws_floats >= need, "attn_decode_paged: workspace of %lld floats, %lld needed", ws_floats, need);
  CB_CHECK_ARG(nsplit < (1LL << 31), "attn_decode_paged: too many splits");
  const int G = nh / nkv, lg = log2_page(page_size);
  const long long max_pos = (long long)max_pages * page_size;
  const dim3 grid((unsigned)nsplit, nkv, rows);
  const bf16* qb = (const bf16*)q;
  if (hd == 128) {
    if (fp8) pd_launch<128, true>(G, grid, st, qb, q_bs, kp, vp, ksc, vsc, table, table_ld, lens, len_add, ws, nkv, lg,
                                  num_pages, max_pos, (int)nsplit, scale);
    else pd_launch<128, false>(G, grid, st, qb, q_bs, kp, vp, ksc, vsc, table, table_ld, lens, len_add, ws, nkv, lg,
                               num_pages, max_pos, (int)nsplit, scale);
  } else {
    if (fp8) pd_launch<64, true>(G, grid, st, qb, q_bs, kp, vp, ksc, vsc, table, table_ld, lens, len_add, ws, nkv, lg,
                                 num_pages, max_pos, (int)nsplit, scale);
    else pd_launch<64, false>(G, grid, st, qb, q_bs, kp, vp, ksc, vsc, table, table_ld, lens, len_add, ws, nkv, lg,
                              num_pages, max_pos, (int)nsplit, scale);
  }
  CB_CUDA_LAUNCH_CHECK("paged_decode_kernel");
  if (hd == 128)
    paged_decode_combine<128><<<rows * nh, 128, 0, st>>>(ws, (bf16*)o, lens, len_add, nh, max_pos, (int)nsplit);
  else
    paged_decode_combine<64><<<rows * nh, 64, 0, st>>>(ws, (bf16*)o, lens, len_add, nh, max_pos, (int)nsplit);
  CB_CUDA_LAUNCH_CHECK("paged_decode_combine");
  return CB_OK;
}

}  // namespace cb
