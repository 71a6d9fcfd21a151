// cambrian_b200 — image preprocessing on the GPU (SURVEY.md §8f rank 4).
//
// Replaces, per tower, the host pipeline of `process_images` (mm_utils.py:186-201):
//     expand2square(img, int(mean*255))  ->  PIL Image.resize((R, R))  ->  processor.preprocess (x/255, (x-mean)/std)
// `Image.resize` defaults to BICUBIC with antialiasing and works on uint8 in two passes (horizontal, then vertical) with
// 22-bit fixed-point coefficients and a round-to-uint8 between the passes (Pillow `src/libImaging/Resample.c`, a
// third-party dependency of the reference: restated here from its published algorithm; the tests compare against the
// installed Pillow bit for bit).  The pad of expand2square is never materialised: the horizontal pass reads a virtual
// square whose out-of-image pixels are the pad colour.
#include "common.cuh"

#include <algorithm>
#include <cmath>
#include <vector>

namespace cb {

static constexpr int PRECISION_BITS = 32 - 8 - 2;

static double bicubic_filter(double x) {
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}

// Resample.c precompute_coeffs + normalize_coeffs_8bpc for the whole-image box [0, in_size)
int resample_ksize(int in_size, int out_size) {
  double filterscale = (double)in_size / out_size;
  if (filterscale < 1.0) filterscale = 1.0;
  const double support = 2.0 * filterscale;
  return (int)ceil(support) * 2 + 1;
}
void resample_coeffs(int in_size, int out_size, int* bounds, int* kk) {
  const double scale = (double)in_size / out_size;
  double filterscale = scale;
  if (filterscale < 1.0) filterscale = 1.0;
  const double support = 2.0 * filterscale;
  const int ksize = (int)ceil(support) * 2 + 1;
  std::vector<double> pre(ksize);
  for (int xx = 0; xx < out_size; ++xx) {
    const double center = (xx + 0.5) * scale;
    double ww = 0.0;
    const double ss = 1.0 / filterscale;
    int xmin = (int)(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5);
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    for (int x = 0; x < xmax; ++x) {
      const double w = bicubic_filter((x + xmin - center + 0.5) * ss);
      pre[x] = w;
      ww += w;
    }
    for (int x = 0; x < xmax; ++x)
      if (ww != 0.0) pre[x] /= ww;
    int* k = kk + (size_t)xx * ksize;
    for (int x = 0; x < ksize; ++x) {
      if (x >= xmax) {
        k[x] = 0;
      } else if (pre[x] < 0) {
        k[x] = (int)(-0.5 + pre[x] * (1 << PRECISION_BITS));
      } else {
        k[x] = (int)(0.5 + pre[x] * (1 << PRECISION_BITS));
      }
    }
    bounds[xx * 2] = xmin;
    bounds[xx * 2 + 1] = xmax;
  }
}

__device__ __forceinline__ int clip8(int v) {
  v >>= PRECISION_BITS;  // arithmetic shift, like the reference's table lookup index
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

// horizontal pass over the virtual S x S square: tmp[y][xx][c], y in [0, S), xx in [0, R)
__global__ void resample_h_kernel(const uint8_t* __restrict__ img, int H, int W, int S, int off_y, int off_x, int R,
                                  const int* __restrict__ bounds, const int* __restrict__ kk, int ksize, int pad_r,
                                  int pad_g, int pad_b, uint8_t* __restrict__ tmp) {
  const long long total = (long long)S * R;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int xx = (int)(i % R), y = (int)(i / R);
    const int xmin = bounds[xx * 2], xmax = bounds[xx * 2 + 1];
    const int* k = kk + (size_t)xx * ksize;
    int s0 = 1 << (PRECISION_BITS - 1), s1 = s0, s2 = s0;
    const int iy = y - off_y;
    const bool row_in = iy >= 0 && iy < H;
    for (int x = 0; x < xmax; ++x) {
      const int ix = x + xmin - off_x;
      int r = pad_r, g = pad_g, b = pad_b;
      if (row_in && ix >= 0 && ix < W) {
        const uint8_t* p = img + ((size_t)iy * W + ix) * 3;
        r = p[0];
        g = p[1];
        b = p[2];
      }
      const int c = k[x];
      s0 += r * c;
      s1 += g * c;
      s2 += b * c;
    }
    uint8_t* o = tmp + (size_t)i * 3;
    o[0] = (uint8_t)clip8(s0);
    o[1] = (uint8_t)clip8(s1);
    o[2] = (uint8_t)clip8(s2);
  }
}

// vertical pass + normalisation: out[c][yy][xx] = (u8 / 255 - mean[c]) / std[c]
__global__ void resample_v_norm_kernel(const uint8_t* __restrict__ tmp, int R, const int* __restrict__ bounds,
                                       const int* __restrict__ kk, int ksize, float m0, float m1, float m2, float is0,
                                       float is1, float is2, bf16* __restrict__ out, uint8_t* __restrict__ out_u8) {
  const long long total = (long long)R * R;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int xx = (int)(i % R), yy = (int)(i / R);
    const int ymin = bounds[yy * 2], ymax = bounds[yy * 2 + 1];
    const int* k = kk + (size_t)yy * ksize;
    int s0 = 1 << (PRECISION_BITS - 1), s1 = s0, s2 = s0;
    for (int y = 0; y < ymax; ++y) {
      const uint8_t* p = tmp + ((size_t)(y + ymin) * R + xx) * 3;
      const int c = k[y];
      s0 += p[0] * c;
      s1 += p[1] * c;
      s2 += p[2] * c;
    }
    const int v0 = clip8(s0), v1 = clip8(s1), v2 = clip8(s2);
    if (out_u8) {
      out_u8[i * 3] = (uint8_t)v0;
      out_u8[i * 3 + 1] = (uint8_t)v1;
      out_u8[i * 3 + 2] = (uint8_t)v2;
    }
    const float inv255 = 1.0f / 255.0f;
    out[i] = __float2bfloat16((v0 * inv255 - m0) * is0);
    out[total + i] = __float2bfloat16((v1 * inv255 - m1) * is1);
    out[2 * total + i] = __float2bfloat16((v2 * inv255 - m2) * is2);
  }
}

static size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

long long preprocess_workspace_bytes(int H, int W, int R) {
  const int S = H > W ? H : W;
  const int ksize = resample_ksize(S, R);
  return (long long)(align256((size_t)S * R * 3) + 2 * align256((size_t)R * 2 * sizeof(int)) +
                     align256((size_t)R * ksize * sizeof(int)));
}

int preprocess_launch(const uint8_t* img, int H, int W, int R, const int* pad_rgb, const float* mean, const float* std_,
                      void* out, uint8_t* out_u8, void* ws, long long ws_bytes, cudaStream_t st) {
  CB_CHECK_ARG(H > 0 && W > 0 && R > 0, "preprocess: bad sizes %d x %d -> %d", H, W, R);
  CB_CHECK_ARG(ws_bytes >= preprocess_workspace_bytes(H, W, R), "preprocess: workspace too small");
  const int S = H > W ? H : W;
  // expand2square (mm_utils.py:153-164): paste at ((S - W) // 2, 0) or (0, (S - H) // 2)
  const int off_x = W < H ? (H - W) / 2 : 0, off_y = W > H ? (W - H) / 2 : 0;
  const int ksize = resample_ksize(S, R);
  // the square is resized in both directions by the same factor: one coefficient table serves both passes
  std::vector<int> bounds((size_t)R * 2), kk((size_t)R * ksize);
  resample_coeffs(S, R, bounds.data(), kk.data());
  uint8_t* base = (uint8_t*)ws;
  uint8_t* tmp = base;
  int* d_bounds = (int*)(base + align256((size_t)S * R * 3));
  int* d_kk = (int*)((uint8_t*)d_bounds + 2 * align256((size_t)R * 2 * sizeof(int)));
  // pageable-source cudaMemcpyAsync stages the data before returning, so the vectors may die with this frame
  if (cudaMemcpyAsync(d_bounds, bounds.data(), bounds.size() * sizeof(int), cudaMemcpyHostToDevice, st) != cudaSuccess ||
      cudaMemcpyAsync(d_kk, kk.data(), kk.size() * sizeof(int), cudaMemcpyHostToDevice, st) != cudaSuccess)
    return set_error(CB_ERR_CUDA, "preprocess: coefficient upload failed: %s", cudaGetErrorString(cudaGetLastError()));
  const int threads = 256;
  long long nb = ((long long)S * R + threads - 1) / threads;
  resample_h_kernel<<<(unsigned)std::min<long long>(nb, device_sm_count() * 32LL), threads, 0, st>>>(
      img, H, W, S, off_y, off_x, R, d_bounds, d_kk, ksize, pad_rgb[0], pad_rgb[1], pad_rgb[2], tmp);
  CB_CUDA_LAUNCH_CHECK("resample_h");
  nb = ((long long)R * R + threads - 1) / threads;
  resample_v_norm_kernel<<<(unsigned)std::min<long long>(nb, device_sm_count() * 32LL), threads, 0, st>>>(
      tmp, R, d_bounds, d_kk, ksize, mean[0], mean[1], mean[2], 1.0f / std_[0], 1.0f / std_[1], 1.0f / std_[2],
      (bf16*)out, out_u8);
  CB_CUDA_LAUNCH_CHECK("resample_v_norm");
  return CB_OK;
}

}  // namespace cb
