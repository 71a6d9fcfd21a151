// cambrian_b200 — token sampling for generate(do_sample=True) and the continuous-batching server: one token per row of
// fp32 logits [rows, V] under each row's own temperature, top-k and top-p, drawn by a Gumbel-max race over Philox4x32-10
// uniforms.  The rule (the host docstring in cambrian_b200/generation.py states it for users):
//
//   scores   s_i = x_i when T == 1, else x_i / T (IEEE division)
//   top-k    0 < k < V: keep s_i >= the k-th largest score (ties kept)
//   top-p    p < 1: over the top-k set, keep i iff G(i) < p * Z, with m_j = rint(expf(s_j - max) * 2^40) as an integer,
//            G(i) = sum of m_j over kept j with s_j > s_i, Z = sum of all kept m_j (compared in fp64).  The sums are exact
//            integers, so they do not depend on any summation order.  The maximum always has G = 0 and is kept.
//   draw     the kept i maximising s_i - logf(-logf(u_i)), the lowest index on a tie; u_i from Philox4x32-10 with key =
//            the row's 64-bit seed, counter = (i >> 2, step lo32, step hi32, 0), output word i & 3 = w, and
//            u_i = ((w >> 9) + 0.5) * 2^-23, exact in fp32 and strictly inside (0, 1).
//
// One CTA per row, no global atomics and no float atomics: shared-memory integer counters only, whose totals do not depend
// on their order.  So a row's token is a function of its logits, parameters, seed and step alone, bitwise run to run and
// independent of the other rows, the grid and the SM count.
//
// Paths.  With top-k on and at most SMP_CAP scores at or above the k-th (the usual case: HF applies top_k = 50 whenever it
// samples), a radix select finds the k-th score in four histogram passes over the row (which stays in L2 between passes)
// and one more pass gathers the candidates into shared memory; top-p and the race then run on them.  Otherwise top-p
// runs as a radix search over the whole row on the mass histogram, and the race is one more pass over the row.
#include "common.cuh"
#include <cfloat>
#include <climits>

namespace cb {

constexpr int SMP_THREADS = 512;
constexpr int SMP_WARPS = SMP_THREADS / 32;
constexpr int SMP_CAP = 2048;                      // top-k candidates held in shared memory
constexpr float SMP_MASS_SCALE = 1099511627776.0f;  // 2^40: Z <= V * 2^40 < 2^63 for V < 2^23
constexpr int SMP_MAX_V = 1 << 23;

__host__ __device__ __forceinline__ uint32_t mulhi32(uint32_t a, uint32_t b) {
  return (uint32_t)(((uint64_t)a * b) >> 32);
}

// Philox4x32-10 (Salmon et al., SC'11; the Random123 constants)
__host__ __device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    const uint32_t hi0 = mulhi32(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = mulhi32(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
  }
  return c;
}

__device__ __forceinline__ uint32_t smp_word(int i, uint64_t seed, int64_t step) {
  const uint4 r = philox4x32_10(make_uint4((uint32_t)(i >> 2), (uint32_t)step, (uint32_t)((uint64_t)step >> 32), 0u),
                                (uint32_t)seed, (uint32_t)(seed >> 32));
  const int w = i & 3;
  return w == 0 ? r.x : w == 1 ? r.y : w == 2 ? r.z : r.w;
}

__device__ __forceinline__ float race_key(float s, uint32_t w) {
  const float u = ((float)(w >> 9) + 0.5f) * 1.1920928955078125e-07f;  // 2^-23
  return s - logf(-logf(u));
}

// order-preserving map of a float to uint32 (-0 is first folded onto +0, so equal scores get equal keys)
__device__ __forceinline__ uint32_t ord_key(float s) {
  const uint32_t u = __float_as_uint(s + 0.0f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ unsigned long long smp_mass(float s, float m) {
  return __float2ull_rn(expf(s - m) * SMP_MASS_SCALE);
}

struct SampleSmem {
  uint32_t hist[256];
  unsigned long long mass[256];
  float cs[SMP_CAP];
  int ci[SMP_CAP];
  unsigned long long cm[SMP_CAP];
  unsigned long long red_u[SMP_WARPS];
  float red_f[SMP_WARPS];
  int red_i[SMP_WARPS];
  uint32_t n, prefix, above, cnt_ge;
  unsigned long long above_m;
};

// Visits every score of the row: each thread takes 4 consecutive elements per trip and every thread makes the same number
// of trips (f is called with valid = false past the end), so warp collectives inside f are uniform.
template <class F>
__device__ __forceinline__ void smp_for_row(const float* row, int V, float T, F&& f) {
  const int ng = (V + 3) >> 2;
  for (int g0 = 0; g0 < ng; g0 += SMP_THREADS) {
    const int g = g0 + (int)threadIdx.x;
    float s[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int i = 4 * g + u;
      const float x = i < V ? row[i] : 0.0f;
      s[u] = T == 1.0f ? x : x / T;
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) f(4 * g + u, s[u], 4 * g + u < V);
  }
}

__device__ __forceinline__ float block_max(float v, SampleSmem& sm) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sm.red_f[threadIdx.x >> 5] = v;
  __syncthreads();
  v = sm.red_f[0];
#pragma unroll
  for (int w = 1; w < SMP_WARPS; ++w) v = fmaxf(v, sm.red_f[w]);
  return v;
}

__device__ __forceinline__ unsigned long long block_sum(unsigned long long v, SampleSmem& sm) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sm.red_u[threadIdx.x >> 5] = v;
  __syncthreads();
  v = 0;
#pragma unroll
  for (int w = 0; w < SMP_WARPS; ++w) v += sm.red_u[w];
  return v;
}

__device__ __forceinline__ bool race_better(float k, int i, float bk, int bi) { return k > bk || (k == bk && i < bi); }

// the race winner over the block: the largest key, the lowest index on a tie
__device__ __forceinline__ int block_race(float k, int i, SampleSmem& sm) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ok = __shfl_xor_sync(0xffffffffu, k, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (race_better(ok, oi, k, i)) k = ok, i = oi;
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sm.red_f[threadIdx.x >> 5] = k, sm.red_i[threadIdx.x >> 5] = i;
  __syncthreads();
  k = sm.red_f[0];
  i = sm.red_i[0];
#pragma unroll
  for (int w = 1; w < SMP_WARPS; ++w)
    if (race_better(sm.red_f[w], sm.red_i[w], k, i)) k = sm.red_f[w], i = sm.red_i[w];
  return i;
}

// one histogram count per warp and digit (digit 256: nothing to count)
__device__ __forceinline__ void hist_add(uint32_t* hist, uint32_t digit) {
  const uint32_t peers = __match_any_sync(0xffffffffu, digit);
  if (digit < 256 && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&hist[digit], (uint32_t)__popc(peers));
}

__global__ void __launch_bounds__(SMP_THREADS)
sample_tokens_kernel(const float* __restrict__ logits, long long ld, int V, const float* __restrict__ temperature,
                     const int* __restrict__ top_k, const float* __restrict__ top_p, const uint64_t* __restrict__ seed,
                     const int64_t* __restrict__ step, int64_t* __restrict__ out) {
  __shared__ SampleSmem sm;
  const int b = blockIdx.x;
  const int tid = threadIdx.x;
  const float* row = logits + (long long)b * ld;
  const float T = temperature[b];
  const int k = top_k[b];
  const float p = top_p[b];
  const uint64_t sd = seed[b];
  const int64_t st = step[b];
  const bool use_k = k > 0 && k < V;
  const bool use_p = p < 1.0f;

  // ---- top-k: the k-th largest key by a radix select, 8 bits per pass from the top
  uint32_t thr = 0;                  // kept iff ord_key(s) >= thr
  uint32_t cnt_ge = (uint32_t)V;     // how many scores have a key >= thr
  if (use_k) {
    uint32_t prefix = 0, pmask = 0, above = 0;
    for (int shift = 24; shift >= 0; shift -= 8) {
      for (int d = tid; d < 256; d += SMP_THREADS) sm.hist[d] = 0;
      __syncthreads();
      smp_for_row(row, V, T, [&](int, float s, bool valid) {
        const uint32_t key = ord_key(s);
        hist_add(sm.hist, valid && (key & pmask) == prefix ? (key >> shift) & 255u : 256u);
      });
      __syncthreads();
      if (tid == 0) {
        uint32_t cum = above;
        int d = 255;
        for (; d > 0; --d) {
          if (cum + sm.hist[d] >= (uint32_t)k) break;
          cum += sm.hist[d];
        }
        sm.prefix = prefix | ((uint32_t)d << shift);
        sm.above = cum;
        sm.cnt_ge = cum + sm.hist[d];
      }
      __syncthreads();
      prefix = sm.prefix;
      above = sm.above;
      pmask |= 255u << shift;
      __syncthreads();
    }
    thr = prefix;
    cnt_ge = sm.cnt_ge;
  }

  if (use_k && cnt_ge <= (uint32_t)SMP_CAP) {
    // ---- candidates: the cnt_ge scores at or above the k-th, gathered into shared memory in any order
    if (tid == 0) sm.n = 0;
    __syncthreads();
    smp_for_row(row, V, T, [&](int i, float s, bool valid) {
      if (valid && ord_key(s) >= thr) {
        const uint32_t slot = atomicAdd(&sm.n, 1u);
        sm.cs[slot] = s;
        sm.ci[slot] = i;
      }
    });
    __syncthreads();
    const int n = (int)sm.n;
    if (use_p) {
      float m = -INFINITY;
      for (int j = tid; j < n; j += SMP_THREADS) m = fmaxf(m, sm.cs[j]);
      m = block_max(m, sm);
      unsigned long long z = 0;
      for (int j = tid; j < n; j += SMP_THREADS) z += (sm.cm[j] = smp_mass(sm.cs[j], m));
      z = block_sum(z, sm);   // its barriers also publish cm[]
      const double pz = (double)p * (double)z;
      for (int j = tid; j < n; j += SMP_THREADS) {
        const float s = sm.cs[j];
        unsigned long long g = 0;
        for (int q = 0; q < n; ++q) g += sm.cs[q] > s ? sm.cm[q] : 0ull;
        if (!((double)g < pz)) sm.ci[j] = -1 - sm.ci[j];   // dropped by top-p
      }
      __syncthreads();
    }
    float bk = -INFINITY;
    int bi = INT_MAX;
    for (int j = tid; j < n; j += SMP_THREADS) {
      const int i = sm.ci[j];
      if (i >= 0) {
        const float key = race_key(sm.cs[j], smp_word(i, sd, st));
        if (race_better(key, i, bk, bi)) bk = key, bi = i;
      }
    }
    const int win = block_race(bk, bi, sm);
    if (tid == 0) out[b] = win;
    return;
  }

  // ---- top-p over the whole row: a radix search of the mass histogram for the lowest kept key
  if (use_p) {
    float m = -INFINITY;
    smp_for_row(row, V, T, [&](int, float s, bool valid) {
      if (valid && ord_key(s) >= thr) m = fmaxf(m, s);
    });
    m = block_max(m, sm);
    unsigned long long z = 0;
    smp_for_row(row, V, T, [&](int, float s, bool valid) {
      if (valid && ord_key(s) >= thr) z += smp_mass(s, m);
    });
    z = block_sum(z, sm);
    const double pz = (double)p * (double)z;
    uint32_t prefix = 0, pmask = 0;
    unsigned long long above = 0;   // mass of the kept-by-k scores above the prefix's key range
    for (int shift = 24; shift >= 0; shift -= 8) {
      for (int d = tid; d < 256; d += SMP_THREADS) sm.hist[d] = 0, sm.mass[d] = 0;
      __syncthreads();
      smp_for_row(row, V, T, [&](int, float s, bool valid) {
        const uint32_t key = ord_key(s);
        const bool in = valid && key >= thr && (key & pmask) == prefix;
        const uint32_t digit = in ? (key >> shift) & 255u : 256u;
        hist_add(sm.hist, digit);
        if (in) {
          const unsigned long long ms = smp_mass(s, m);
          if (ms) atomicAdd(&sm.mass[digit], ms);
        }
      });
      __syncthreads();
      if (tid == 0) {
        // the largest key of digit d has exactly G = above + the mass of the digits above d: the cut is in the lowest
        // non-empty digit where that is < p * Z
        unsigned long long run = above, run_sel = above;
        int sel = -1;
        for (int d = 255; d >= 0; --d) {
          if (!((double)run < pz)) break;
          if (sm.hist[d]) sel = d, run_sel = run;
          run += sm.mass[d];
        }
        sel = sel < 0 ? 255 : sel;   // not reached: the largest kept score always has G = 0 < p * Z
        sm.prefix = prefix | ((uint32_t)sel << shift);
        sm.above_m = run_sel;
      }
      __syncthreads();
      prefix = sm.prefix;
      above = sm.above_m;
      pmask |= 255u << shift;
      __syncthreads();
    }
    thr = max(thr, prefix);
  }

  // ---- the race over the whole row
  float bk = -INFINITY;
  int bi = INT_MAX;
  const int ng = (V + 3) >> 2;
  for (int g = tid; g < ng; g += SMP_THREADS) {
    float s[4];
    bool any = false;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int i = 4 * g + u;
      const float x = i < V ? row[i] : -INFINITY;
      s[u] = T == 1.0f ? x : x / T;
      any |= i < V && ord_key(s[u]) >= thr;
    }
    if (!any) continue;
    const uint4 r = philox4x32_10(make_uint4((uint32_t)g, (uint32_t)st, (uint32_t)((uint64_t)st >> 32), 0u),
                                  (uint32_t)sd, (uint32_t)(sd >> 32));
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int i = 4 * g + u;
      if (i < V && ord_key(s[u]) >= thr) {
        const float key = race_key(s[u], w[u]);
        if (race_better(key, i, bk, bi)) bk = key, bi = i;
      }
    }
  }
  const int win = block_race(bk, bi, sm);
  if (tid == 0) out[b] = win;
}

long long sample_tokens_workspace_floats(int rows, int V) {
  (void)rows;
  (void)V;
  return 0;
}

int sample_tokens_launch(const float* logits, long long ld, int rows, int V, const float* temperature, const int* top_k,
                         const float* top_p, const uint64_t* seed, const int64_t* step, int64_t* out, float* ws,
                         long long ws_floats, cudaStream_t st) {
  CB_CHECK_ARG(rows >= 1, "sample_tokens: rows=%d must be >= 1", rows);
  CB_CHECK_ARG(V >= 1 && V < SMP_MAX_V, "sample_tokens: V=%d must be in [1, %d)", V, SMP_MAX_V);
  CB_CHECK_ARG(ld >= V, "sample_tokens: row stride %lld must be >= V=%d", ld, V);
  CB_CHECK_ARG(logits && temperature && top_k && top_p && seed && step && out, "sample_tokens: null argument");
  CB_CHECK_ARG(((reinterpret_cast<uintptr_t>(logits) | reinterpret_cast<uintptr_t>(temperature) |
                 reinterpret_cast<uintptr_t>(top_k) | reinterpret_cast<uintptr_t>(top_p)) & 3u) == 0 &&
                   ((reinterpret_cast<uintptr_t>(seed) | reinterpret_cast<uintptr_t>(step) |
                     reinterpret_cast<uintptr_t>(out)) & 7u) == 0,
               "sample_tokens: logits, temperature, top_k and top_p must be 4-byte aligned, seed, step and out 8-byte");
  const long long need = sample_tokens_workspace_floats(rows, V);
  CB_CHECK_ARG(ws_floats >= need && (need == 0 || ws), "sample_tokens: workspace of %lld floats, %lld needed", ws_floats,
               need);
  sample_tokens_kernel<<<rows, SMP_THREADS, 0, st>>>(logits, ld, V, temperature, top_k, top_p, seed, step, out);
  CB_CUDA_LAUNCH_CHECK("sample_tokens_kernel");
  return CB_OK;
}

}  // namespace cb
