// cambrian_b200 — HBM-bound elementwise / gather / reduction kernels of the hot path.
//
// All kernels use 16-byte vector accesses on the contiguous channel dimension (C % 8 == 0), fp32 math,
// grid-stride loops sized in multiples of the SM count.  Reference call sites are cited per kernel.
#include "common.cuh"
#include <cfloat>
#include <climits>

namespace cb {

static inline unsigned grid_for(long long work_items, int threads, int per_sm = 8) {
  long long blocks = (work_items + threads - 1) / threads;
  const long long cap = (long long)device_sm_count() * per_sm;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (unsigned)blocks;
}

__device__ __forceinline__ float act_fwd(float v, int act) {
  switch (act) {
    case 1: return gelu_erf(v);
    case 2: return gelu_tanh(v);
    case 3: return quick_gelu(v);
    case 4: return silu(v);
    default: return v;
  }
}
__device__ __forceinline__ float act_grad(float x, int act) {
  switch (act) {
    case 1: return gelu_erf_grad(x);
    case 2: {
      const float u = 0.7978845608028654f * (x + 0.044715f * x * x * x);
      const float t = tanhf(u);
      return 0.5f * (1.f + t) + 0.5f * x * (1.f - t * t) * 0.7978845608028654f * (1.f + 3.f * 0.044715f * x * x);
    }
    case 3: {
      const float s = 1.f / (1.f + __expf(-1.702f * x));
      return s + 1.702f * x * s * (1.f - s);
    }
    case 4: {
      const float s = 1.f / (1.f + __expf(-x));
      return s * (1.f + x * (1.f - s));
    }
    default: return 1.f;
  }
}

// ---------------------------------------------------------------------------------- activations
// y = act(x)                         (nn.GELU in vision_sampler.py:241, cambrian_arch.py:49,56)
__global__ void act_fwd_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, long long nvec, int act) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float f[8];
    unpack8(ldg_nc(x + i), f);
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = act_fwd(f[e], act);
    y[i] = pack8(f);
  }
}
// dx = dy * act'(x)
__global__ void act_bwd_kernel(const uint4* __restrict__ dy, const uint4* __restrict__ x, uint4* __restrict__ dx,
                               long long nvec, int act) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float f[8], g[8];
    unpack8(ldg_nc(x + i), f);
    unpack8(ldg_nc(dy + i), g);
#pragma unroll
    for (int e = 0; e < 8; ++e) g[e] *= act_grad(f[e], act);
    dx[i] = pack8(g);
  }
}

// ------------------------------------------------------------------------------------- SwiGLU
// out = silu(gate) * up        HF LlamaMLP: down_proj(act_fn(gate_proj(x)) * up_proj(x))
// gate/up rows may live in one fused [rows, 2*I] buffer: pass ld (elements) and the two base pointers.
__global__ void swiglu_fwd_kernel(const bf16* __restrict__ gate, const bf16* __restrict__ up, bf16* __restrict__ out,
                                  long long rows, int I, long long ld_in, long long ld_out) {
  const int vpr = I >> 3;
  const long long total = rows * vpr;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / vpr;
    const int c = (int)(i - r * vpr) << 3;
    float g[8], u[8];
    unpack8(ldg_nc(gate + r * ld_in + c), g);
    unpack8(ldg_nc(up + r * ld_in + c), u);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      // HF computes silu in bf16 then multiplies in bf16: round the intermediate like the reference does
      const float s = __bfloat162float(__float2bfloat16(silu(g[e])));
      g[e] = s * u[e];
    }
    *reinterpret_cast<uint4*>(out + r * ld_out + c) = pack8(g);
  }
}
// d / dgate and d / dup of out = silu(gate) * up for 8 elements (the swiglu_bwd kernels share it, so both give the
// same bits)
__device__ __forceinline__ void swiglu_grad8(const float* d, const float* g, const float* u, float* dg, float* du) {
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float s = 1.f / (1.f + __expf(-g[e]));
    du[e] = d[e] * g[e] * s;
    dg[e] = d[e] * u[e] * s * (1.f + g[e] * (1.f - s));
  }
}
__global__ void swiglu_bwd_kernel(const bf16* __restrict__ dout, const bf16* __restrict__ gate,
                                  const bf16* __restrict__ up, bf16* __restrict__ dgate, bf16* __restrict__ dup,
                                  long long rows, int I, long long ld_in, long long ld_dout, long long ld_dgu) {
  const int vpr = I >> 3;
  const long long total = rows * vpr;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / vpr;
    const int c = (int)(i - r * vpr) << 3;
    float g[8], u[8], d[8], dg[8], du[8];
    unpack8(ldg_nc(gate + r * ld_in + c), g);
    unpack8(ldg_nc(up + r * ld_in + c), u);
    unpack8(ldg_nc(dout + r * ld_dout + c), d);
    swiglu_grad8(d, g, u, dg, du);
    *reinterpret_cast<uint4*>(dgate + r * ld_dgu + c) = pack8(dg);
    *reinterpret_cast<uint4*>(dup + r * ld_dgu + c) = pack8(du);
  }
}
// The same gradients with a second, E4M3 output (`fp8_training`): one CTA per row writes dgate / dup in bf16 exactly as
// swiglu_bwd_kernel does, takes the amax of the rounded [dgate | dup] row, then reads its own bf16 stores back (the
// same thread wrote them, so plain loads see them) and writes q [rows, 2I] e4m3 (dgate in columns [0, I), dup in
// [I, 2I)) and s [rows] by the row rule of quant_fp8.py.  No atomics.
__global__ void __launch_bounds__(256) swiglu_bwd_fp8_kernel(const bf16* __restrict__ dout, const bf16* __restrict__ gate,
                                                             const bf16* __restrict__ up, bf16* dgate, bf16* dup,
                                                             uint8_t* __restrict__ q, float* __restrict__ s_out, int I,
                                                             long long ld_in, long long ld_dout, long long ld_dgu) {
  __shared__ float red[8];
  const long long r = blockIdx.x;
  float a = 0.f;
  for (int c = threadIdx.x * 8; c < I; c += 256 * 8) {
    float g[8], u[8], d[8], dg[8], du[8];
    unpack8(ldg_nc(gate + r * ld_in + c), g);
    unpack8(ldg_nc(up + r * ld_in + c), u);
    unpack8(ldg_nc(dout + r * ld_dout + c), d);
    swiglu_grad8(d, g, u, dg, du);
    const uint4 pg = pack8(dg), pu = pack8(du);
    *reinterpret_cast<uint4*>(dgate + r * ld_dgu + c) = pg;
    *reinterpret_cast<uint4*>(dup + r * ld_dgu + c) = pu;
    unpack8(pg, dg);
    unpack8(pu, du);
#pragma unroll
    for (int e = 0; e < 8; ++e) a = fmaxf(a, fmaxf(fabsf(dg[e]), fabsf(du[e])));
  }
  a = warp_max(a);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = a;
  __syncthreads();
  a = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) a = fmaxf(a, red[i]);
  if (threadIdx.x == 0) s_out[r] = __fdiv_rn(a, 448.0f);
  const float rr = fminf(__fdiv_rn(448.0f, a), FLT_MAX);  // amax = 0 or below 448 * 2^-128: +inf -> FLT_MAX
  uint8_t* qr = q + r * 2 * I;
  for (int c = threadIdx.x * 8; c < I; c += 256 * 8) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float f[8];
      unpack8(*reinterpret_cast<const uint4*>((h ? dup : dgate) + r * ld_dgu + c), f);
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] = __fmul_rn(f[e], rr);
      *reinterpret_cast<uint2*>(qr + h * I + c) = f8_pack8(f);
    }
  }
}

// --------------------------------------------------------------------------------------- RoPE
// In-place rotary embedding on the q and k heads of a packed [rows, ld] buffer (HF apply_rotary_pos_emb,
// rotate_half convention; called inside LlamaAttention from cambrian_llama.py:142-164).  cos/sin tables are
// [max_pos, hd/2] fp32 built on the host exactly as HF does; like HF they are rounded to bf16 before use and
// every product / sum is rounded to bf16.  inverse=1 applies the transposed rotation (backward).
__global__ void rope_kernel(bf16* __restrict__ buf, const long long* __restrict__ pos, const float* __restrict__ cos_t,
                            const float* __restrict__ sin_t, long long rows, int n_heads, int hd, long long ld,
                            int max_pos, int inverse) {
  const int half = hd >> 1;
  const int vph = half >> 3;  // vectors per half head
  const long long total = rows * n_heads * vph;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vph);
    const long long t = i / vph;
    const int h = (int)(t % n_heads);
    const long long r = t / n_heads;
    long long p = pos[r];
    if (p < 0) p = 0;
    if (p >= max_pos) p = max_pos - 1;
    bf16* base = buf + r * ld + (long long)h * hd + v * 8;
    float x1[8], x2[8], o1[8], o2[8];
    unpack8(*reinterpret_cast<const uint4*>(base), x1);
    unpack8(*reinterpret_cast<const uint4*>(base + half), x2);
    const float* cp = cos_t + p * half + v * 8;
    const float* sp = sin_t + p * half + v * 8;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float c = __bfloat162float(__float2bfloat16(cp[e]));
      float s = __bfloat162float(__float2bfloat16(sp[e]));
      if (inverse) s = -s;
      const float a1 = __bfloat162float(__float2bfloat16(x1[e] * c));
      const float b1 = __bfloat162float(__float2bfloat16(-x2[e] * s));
      const float a2 = __bfloat162float(__float2bfloat16(x2[e] * c));
      const float b2 = __bfloat162float(__float2bfloat16(x1[e] * s));
      o1[e] = a1 + b1;
      o2[e] = a2 + b2;
    }
    *reinterpret_cast<uint4*>(base) = pack8(o1);
    *reinterpret_cast<uint4*>(base + half) = pack8(o2);
  }
}

// ------------------------------------------------------------------------- embedding + image splice
// out[b, s] = image token?  (newline column ? newline : img[b, row*q + col])  :  embed[max(ids[b,s],0)]
// Static-shape splice of cambrian_arch.py:413-420 (newline append) + :457-490 (embed + replace): the image span
// [start, start + q*(q+1)) of sample b begins at the position of its IMAGE_TOKEN_INDEX (-200) id.
__global__ void embed_splice_kernel(const long long* __restrict__ ids, const int* __restrict__ img_start,
                                    const bf16* __restrict__ embed, const bf16* __restrict__ img,
                                    const bf16* __restrict__ newline, bf16* __restrict__ out, int B, int S, int H,
                                    int q_side, long long vocab) {
  const int vpr = H >> 3;
  const long long total = (long long)B * S * vpr;
  const int span = q_side * (q_side + 1);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    const long long t = i / vpr;
    const int s = (int)(t % S);
    const int b = (int)(t / S);
    const int st = img ? img_start[b] : -1;
    const bf16* src;
    if (st >= 0 && s >= st && s < st + span) {
      const int k = s - st, row = k / (q_side + 1), col = k - row * (q_side + 1);
      src = (col == q_side) ? newline : img + ((long long)b * q_side * q_side + row * q_side + col) * H;
    } else {
      long long id = ids[t];
      if (id < 0 || id >= vocab) id = 0;
      src = embed + id * H;
    }
    reinterpret_cast<uint4*>(out + t * H)[v] = ldg_nc(reinterpret_cast<const uint4*>(src) + v);
  }
}
// backward: d_img gathers its rows; text rows are scatter-added (bf16x2 atomics) into d_embed (pre-zeroed by
// the caller); newline rows are copied to d_newline_rows [B*q, H] for a column sum.
__global__ void embed_splice_bwd_kernel(const bf16* __restrict__ dout, const long long* __restrict__ ids,
                                        const int* __restrict__ img_start, bf16* __restrict__ d_embed,
                                        bf16* __restrict__ d_img, bf16* __restrict__ d_nl_rows, int B, int S, int H,
                                        int q_side, long long vocab) {
  const int vpr = H >> 3;
  const long long total = (long long)B * S * vpr;
  const int span = q_side * (q_side + 1);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    const long long t = i / vpr;
    const int s = (int)(t % S);
    const int b = (int)(t / S);
    const int st = d_img ? img_start[b] : -1;
    const uint4 g = ldg_nc(reinterpret_cast<const uint4*>(dout + t * H) + v);
    if (st >= 0 && s >= st && s < st + span) {
      const int k = s - st, row = k / (q_side + 1), col = k - row * (q_side + 1);
      if (col == q_side) {
        if (d_nl_rows) reinterpret_cast<uint4*>(d_nl_rows + ((long long)b * q_side + row) * H)[v] = g;
      } else {
        reinterpret_cast<uint4*>(d_img + ((long long)b * q_side * q_side + row * q_side + col) * H)[v] = g;
      }
    } else if (d_embed) {
      long long id = ids[t];
      if (id < 0 || id >= vocab) id = 0;
      __nv_bfloat162* dst = reinterpret_cast<__nv_bfloat162*>(d_embed + id * H + v * 8);
      const __nv_bfloat162* gg = reinterpret_cast<const __nv_bfloat162*>(&g);
#pragma unroll
      for (int e = 0; e < 4; ++e) atomicAdd(dst + e, gg[e]);
    }
  }
}

// Deterministic embedding-row gradient: the rows of `dout` that belong to the same token id are summed by ONE block in
// position order (fp32) and written once, instead of racing bf16x2 atomics whose rounding depends on arrival order.
// keys[t] = token id of flattened position t, or >= vocab for positions that carry no embedding gradient (image span);
// order = positions stably sorted by key.  d_embed += (single writer per row: still deterministic); ids that do not occur
// are not touched.
__global__ void __launch_bounds__(128)
embed_grad_sorted_kernel(const bf16* __restrict__ dout, const long long* __restrict__ keys, const int* __restrict__ order,
                         bf16* __restrict__ d_embed, long long n, int H, long long vocab) {
  const long long p = blockIdx.x;
  const long long key = keys[order[p]];
  if (key < 0 || key >= vocab) return;
  if (p > 0 && keys[order[p - 1]] == key) return;  // not the first position of this id's segment
  const int vpr = H >> 3;
  for (int v = threadIdx.x; v < vpr; v += blockDim.x) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (long long q = p; q < n; ++q) {
      const long long t = order[q];
      if (keys[t] != key) break;
      float f[8];
      unpack8(ldg_nc(reinterpret_cast<const uint4*>(dout + t * H) + v), f);
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] += f[e];
    }
    uint4* dst = reinterpret_cast<uint4*>(d_embed + key * H) + v;
    float old[8];
    unpack8(*dst, old);  // += : zero on the first micro-batch of a step, the running sum under gradient accumulation
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] += old[e];
    *dst = pack8(acc);
  }
}

// --------------------------------------------------------------------------- ViT token assembly
// out[b, 0] = cls + pos[0] (if cls);  out[b, c + i] = patch[b, i] + pos[c + i]
// (HF CLIPVisionEmbeddings / Dinov2Embeddings / timm _pos_embed, reached from clip_encoder.py:104 etc.)
__global__ void add_pos_tokens_kernel(const bf16* __restrict__ patch, const bf16* __restrict__ cls,
                                      const bf16* __restrict__ pos, bf16* __restrict__ out, int B, int N, int C) {
  const int vpr = C >> 3;
  const int T = N + (cls ? 1 : 0);
  const long long total = (long long)B * T * vpr;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    const long long t = i / vpr;
    const int tok = (int)(t % T);
    const int b = (int)(t / T);
    float a[8], p[8];
    if (cls && tok == 0) unpack8(reinterpret_cast<const uint4*>(cls)[v], a);
    else unpack8(ldg_nc(reinterpret_cast<const uint4*>(patch + ((long long)b * N + tok - (cls ? 1 : 0)) * C) + v), a);
    unpack8(reinterpret_cast<const uint4*>(pos + (long long)tok * C)[v], p);
#pragma unroll
    for (int e = 0; e < 8; ++e) a[e] += p[e];
    reinterpret_cast<uint4*>(out + t * C)[v] = pack8(a);
  }
}

// ------------------------------------------------------------------------------- bilinear resize
// tokens [B, h, w, C] -> [B, th, tw, C], fp32 interpolation, align_corners=False (F.interpolate bilinear as used
// by clip_encoder.py:83-88, siglip_encoder.py:80-85, dino_encoder.py:141-146, clip_convnext_encoder.py:112-117).
// in_off / in_row_stride let the source skip a CLS token or read a wider buffer.
__global__ void bilinear_kernel(const bf16* __restrict__ in, bf16* __restrict__ out, int B, int h, int w, int th,
                                int tw, int C, long long in_batch_stride, long long out_batch_stride, int out_ld,
                                int out_col0) {
  const int vpr = C >> 3;
  const long long total = (long long)B * th * tw * vpr;
  const float sy = (float)h / th, sx = (float)w / tw;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    long long t = i / vpr;
    const int ox = (int)(t % tw);
    t /= tw;
    const int oy = (int)(t % th);
    const int b = (int)(t / th);
    float fy = ((float)oy + 0.5f) * sy - 0.5f, fx = ((float)ox + 0.5f) * sx - 0.5f;
    if (fy < 0.f) fy = 0.f;
    if (fx < 0.f) fx = 0.f;
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = min(y0 + 1, h - 1), x1 = min(x0 + 1, w - 1);
    const float ly = fy - y0, lx = fx - x0;
    const bf16* base = in + (long long)b * in_batch_stride;
    float a[8], bb[8], c[8], d[8], o[8];
    unpack8(ldg_nc(reinterpret_cast<const uint4*>(base + ((long long)y0 * w + x0) * C) + v), a);
    unpack8(ldg_nc(reinterpret_cast<const uint4*>(base + ((long long)y0 * w + x1) * C) + v), bb);
    unpack8(ldg_nc(reinterpret_cast<const uint4*>(base + ((long long)y1 * w + x0) * C) + v), c);
    unpack8(ldg_nc(reinterpret_cast<const uint4*>(base + ((long long)y1 * w + x1) * C) + v), d);
#pragma unroll
    for (int e = 0; e < 8; ++e)
      o[e] = (1.f - ly) * ((1.f - lx) * a[e] + lx * bb[e]) + ly * ((1.f - lx) * c[e] + lx * d[e]);
    bf16* op = out + (long long)b * out_batch_stride + ((long long)oy * tw + ox) * out_ld + out_col0;
    reinterpret_cast<uint4*>(op)[v] = pack8(o);
  }
}

// ---------------------------------------------------------------------------------- patchify
// NCHW image [B, Cin, R, R] -> rows [B*g*g, Kpad], K index = (c, py, px) (conv weight [D, Cin, p, p] flattened);
// columns >= Cin*p*p are zero (TMA needs K % 8 == 0: 3*14*14 = 588 -> 592).  Replaces the strided Conv2d patch
// embedding of HF CLIP / DINOv2 / timm PatchEmbed and the ConvNeXt 4x4 stem by an im2col feeding the GEMM.
__global__ void patchify_nchw_kernel(const bf16* __restrict__ img, bf16* __restrict__ out, int B, int Cin, int R,
                                     int p, int Kpad) {
  const int g = R / p;
  const long long total = (long long)B * g * g * Kpad;
  const int K = Cin * p * p;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(i % Kpad);
    long long t = i / Kpad;
    const int gx = (int)(t % g);
    t /= g;
    const int gy = (int)(t % g);
    const int b = (int)(t / g);
    bf16 val = __float2bfloat16(0.f);
    if (k < K) {
      const int c = k / (p * p), rem = k - c * p * p, py = rem / p, px = rem - py * p;
      val = img[(((long long)b * Cin + c) * R + gy * p + py) * R + gx * p + px];
    }
    out[i] = val;
  }
}
// NHWC feature map [B, H, W, C] -> rows [B*(H/p)*(W/p), p*p*C], K index = (py, px, c)
// (ConvNeXt downsample conv2x2/2; weights are permuted to (py, px, c) order at load time)
__global__ void patchify_nhwc_kernel(const bf16* __restrict__ in, bf16* __restrict__ out, int B, int H, int W, int C,
                                     int p) {
  const int vpr = C >> 3, gh = H / p, gw = W / p;
  const long long total = (long long)B * gh * gw * p * p * vpr;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    long long t = i / vpr;
    const int pp = (int)(t % (p * p));
    t /= (p * p);
    const int gx = (int)(t % gw);
    t /= gw;
    const int gy = (int)(t % gh);
    const int b = (int)(t / gh);
    const int py = pp / p, px = pp - py * p;
    const uint4 val = ldg_nc(reinterpret_cast<const uint4*>(in + (((long long)b * H + gy * p + py) * W + gx * p + px) * C) + v);
    reinterpret_cast<uint4*>(out)[i] = val;
  }
}

// ------------------------------------------------------------------------ depthwise 7x7 conv (NHWC)
// y[b,y,x,c] = bias[c] + sum_{dy,dx} w[dy,dx,c] * x[b, y+dy-3, x+dx-3, c]     (timm ConvNeXtBlock.conv_dw,
// reached from clip_convnext_encoder.py:121-144).  Weights pre-permuted to [7,7,C].  Each thread owns 8 channels
// of one output pixel; neighbouring threads share input rows through L1/L2 (bandwidth-bound, 49 taps).
// Register-tiled: each thread owns 8 channels of a 2 x 4 patch of output pixels and walks the 8 input rows the patch
// needs once (10 input vectors per row), so every loaded input vector feeds up to 2 x 7 taps.
// Block = 16 channel-vectors (128 channels) x 8 patches covering an 8 x 8 pixel region; the block's 49 x 128 weights
// are converted to fp32 ONCE into shared memory (25 KB) and the block then walks down a column strip, so (a) the
// per-tap weight fetch is two conflict-free LDS.128 instead of an L2-latency LDG + 8 unpack ops (C = 1536: 150 KB of
// weights never fit L1 next to the streamed input), (b) vertically adjacent steps re-hit their halo rows in L1.
constexpr int DW_TY = 2, DW_TX = 4, DW_CV = 16;
#ifndef CB_DW_MINB
#define CB_DW_MINB 3
#endif
__global__ void __launch_bounds__(128, CB_DW_MINB)
dwconv7_kernel(const bf16* __restrict__ in, const bf16* __restrict__ w, const bf16* __restrict__ bias,
               bf16* __restrict__ out, int B, int H, int W, int C, int ysplit) {
  // [tap][half][cv][4]: lanes read consecutive 16-byte words (a [cv][8] layout makes LDS.128 2-way bank-conflicted)
  __shared__ __align__(16) float sw[49][2][DW_CV * 4];
  __shared__ __align__(16) float sb[DW_CV * 8];
  const int vpr = C >> 3;
  const int nchunk = (vpr + DW_CV - 1) / DW_CV;
  const int strips = (W + 7) / 8;
  int bid = blockIdx.x;
  const int chunk = bid % nchunk;
  bid /= nchunk;
  const int ys = bid % ysplit;
  bid /= ysplit;
  const int strip = bid % strips;
  const int b = bid / strips;
  const int c_base = chunk * DW_CV * 8;
  for (int i = threadIdx.x; i < 49 * DW_CV * 8; i += blockDim.x) {
    const int tap = i / (DW_CV * 8), c = i - tap * (DW_CV * 8);
    sw[tap][(c >> 2) & 1][(c >> 3) * 4 + (c & 3)] =
        (c_base + c < C) ? __bfloat162float(w[(long long)tap * C + c_base + c]) : 0.f;
  }
  for (int i = threadIdx.x; i < DW_CV * 8; i += blockDim.x)
    sb[i] = (bias && c_base + i < C) ? __bfloat162float(bias[c_base + i]) : 0.f;
  __syncthreads();
  const int cv = threadIdx.x & (DW_CV - 1), st = threadIdx.x / DW_CV;
  const int v = chunk * DW_CV + cv;
  if (v >= vpr) return;
  const int steps = (H + 7) / 8, per = (steps + ysplit - 1) / ysplit;
  const int s_end = min(steps, (ys + 1) * per);
  const int x0 = strip * 8 + (st & 1) * DW_TX;
  if (x0 >= W) return;
  for (int s = ys * per; s < s_end; ++s) {
    const int y0 = s * 8 + (st >> 1) * DW_TY;
    if (y0 >= H) break;
    float acc[DW_TY][DW_TX][8];
#pragma unroll
    for (int oy = 0; oy < DW_TY; ++oy)
#pragma unroll
      for (int ox = 0; ox < DW_TX; ++ox)
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[oy][ox][e] = sb[cv * 8 + e];
    const bf16* img = in + (long long)b * H * W * C + v * 8;
#pragma unroll 1
    for (int r = 0; r < DW_TY + 6; ++r) {
      const int iy = y0 + r - 3;
      if (iy < 0 || iy >= H) continue;
      // branch-free halo: clamp the address, select zeros afterwards — conditional loads compiled to a branch per
      // vector and serialised the ten load latencies (ncu source view: every first use stalled on its own LDG)
      uint4 raw[DW_TX + 6];
      const bf16* rowp = img + (long long)iy * W * C;
#pragma unroll
      for (int c = 0; c < DW_TX + 6; ++c) {
        const int ix = x0 + c - 3;
        const int ixc = min(max(ix, 0), W - 1);
        raw[c] = *reinterpret_cast<const uint4*>(rowp + (long long)ixc * C);
      }
      float row[DW_TX + 6][8];
#pragma unroll
      for (int c = 0; c < DW_TX + 6; ++c) {
        const int ix = x0 + c - 3;
        const bool ok = ix >= 0 && ix < W;
        uint4 v4 = raw[c];
        v4.x = ok ? v4.x : 0u;
        v4.y = ok ? v4.y : 0u;
        v4.z = ok ? v4.z : 0u;
        v4.w = ok ? v4.w : 0u;
        unpack8(v4, row[c]);
      }
#pragma unroll
      for (int oy = 0; oy < DW_TY; ++oy) {
        const int ky = r - oy;
        if (ky < 0 || ky > 6) continue;
#pragma unroll
        for (int kx = 0; kx < 7; ++kx) {
          const float4 k0 = *reinterpret_cast<const float4*>(&sw[ky * 7 + kx][0][cv * 4]);
          const float4 k1 = *reinterpret_cast<const float4*>(&sw[ky * 7 + kx][1][cv * 4]);
          const float k[8] = {k0.x, k0.y, k0.z, k0.w, k1.x, k1.y, k1.z, k1.w};
#pragma unroll
          for (int ox = 0; ox < DW_TX; ++ox)
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[oy][ox][e] = fmaf(row[ox + kx][e], k[e], acc[oy][ox][e]);
        }
      }
    }
#pragma unroll
    for (int oy = 0; oy < DW_TY; ++oy)
#pragma unroll
      for (int ox = 0; ox < DW_TX; ++ox) {
        const int y = y0 + oy, x = x0 + ox;
        if (y < H && x < W)
          *reinterpret_cast<uint4*>(out + (((long long)b * H + y) * W + x) * C + v * 8) = pack8(acc[oy][ox]);
      }
  }
}

// ------------------------------------------------------------------------ dynamic-shape (inference) helpers
// rearrange_vision_tower_features_inference (cambrian_arch.py:289-330): feat [B, side, side, C] with side = q * r
// -> windows [B * (y1-y0) * (x1-x0), r*r, C] for the query rows [y0, y1) x columns [x0, x1) (the crop `unpad_image`
// applies to the q x q window grid; full range = the train-time rearrangement :271-287).
__global__ void window_gather_kernel(const bf16* __restrict__ feat, bf16* __restrict__ out, int B, int q, int r, int C,
                                     int y0, int y1, int x0, int x1) {
  const int vpr = C >> 3;
  const int hh = y1 - y0, ww = x1 - x0, side = q * r;
  const long long total = (long long)B * hh * ww * r * r * vpr;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    long long t = i / vpr;
    const int wx = (int)(t % r);
    t /= r;
    const int wy = (int)(t % r);
    t /= r;
    const int qx = (int)(t % ww) + x0;
    t /= ww;
    const int qy = (int)(t % hh) + y0;
    const int b = (int)(t / hh);
    const long long src = (((long long)b * side + qy * r + wy) * side + qx * r + wx) * C;
    reinterpret_cast<uint4*>(out)[i] = ldg_nc(reinterpret_cast<const uint4*>(feat + src) + v);
  }
}

// Ragged embedding + image splice (cambrian_arch.py:493-609): out[row] = embed[src] (src >= 0) | zeros (src == -1,
// padding) | newline (src == INT_MIN) | img[-2 - src] (image feature row).  The row map is built on the host from the
// ids, attention mask and per-sample unpadded grid sizes.
__global__ void embed_splice_ragged_kernel(bf16* __restrict__ out, const bf16* __restrict__ embed,
                                           const bf16* __restrict__ img, const bf16* __restrict__ newline,
                                           const int* __restrict__ src, long long rows, int H) {
  const int vpr = H >> 3;
  const long long total = rows * vpr;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    const long long row = i / vpr;
    const int s = src[row];
    uint4 val = make_uint4(0, 0, 0, 0);
    if (s >= 0) val = ldg_nc(reinterpret_cast<const uint4*>(embed + (long long)s * H) + v);
    else if (s == INT_MIN) val = ldg_nc(reinterpret_cast<const uint4*>(newline) + v);
    else if (s <= -2) val = ldg_nc(reinterpret_cast<const uint4*>(img + (long long)(-2 - s) * H) + v);
    reinterpret_cast<uint4*>(out)[i] = val;
  }
}

// ---------------------------------------------------------------------------- small reductions
// dst += src (bf16), used where a tensor feeds several consumers in hand-written backward passes
__global__ void add_inplace_kernel(uint4* __restrict__ dst, const uint4* __restrict__ src, long long nvec) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float a[8], b[8];
    unpack8(dst[i], a);
    unpack8(ldg_nc(src + i), b);
#pragma unroll
    for (int e = 0; e < 8; ++e) a[e] += b[e];
    dst[i] = pack8(a);
  }
}
// out[g, c] = scale * sum_{r < rows_per_group} x[g*rows_per_group + r, c]   (fp32 accumulate, fixed order)
//   - global context = mean over tower-0 tokens (cambrian_arch.py:377): groups = B, scale = 1/N
//   - bias / newline / vision_query gradients: groups = 1, scale = 1
// one block per (group, 256-column slab); threads stride rows, then a shared-memory tree over row lanes.
__global__ void group_colsum_kernel(const bf16* __restrict__ x, bf16* __restrict__ out_bf16, float* __restrict__ out_f32,
                                    long long rows_per_group, int C, float scale, int accumulate) {
  __shared__ float red[8][33];
  const int g = blockIdx.y;
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  const int lane_r = threadIdx.x >> 5;  // 8 row lanes
  float s = 0.f;
  if (c < C) {
    const bf16* p = x + (long long)g * rows_per_group * C + c;
    for (long long r = lane_r; r < rows_per_group; r += 8) s += __bfloat162float(p[r * C]);
  }
  red[lane_r][threadIdx.x & 31] = s;
  __syncthreads();
  if (lane_r == 0 && c < C) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += red[k][threadIdx.x & 31];
    t *= scale;
    const long long o = (long long)g * C + c;
    if (out_bf16) out_bf16[o] = __float2bfloat16(accumulate ? __bfloat162float(out_bf16[o]) + t : t);
    if (out_f32) out_f32[o] = accumulate ? out_f32[o] + t : t;
  }
}
// dx[g*rows + r, c] (+)= scale * dmean[g, c]   (backward of the token mean)
__global__ void group_broadcast_kernel(const bf16* __restrict__ dmean, bf16* __restrict__ dx, long long rows_per_group,
                                       int C, int groups, float scale, int accumulate) {
  const int vpr = C >> 3;
  const long long total = (long long)groups * rows_per_group * vpr;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    const long long row = i / vpr;
    const int g = (int)(row / rows_per_group);
    float m[8];
    unpack8(reinterpret_cast<const uint4*>(dmean + (long long)g * C)[v], m);
#pragma unroll
    for (int e = 0; e < 8; ++e) m[e] *= scale;
    if (accumulate) {
      float o[8];
      unpack8(reinterpret_cast<uint4*>(dx)[i], o);
#pragma unroll
      for (int e = 0; e < 8; ++e) m[e] += o[e];
    }
    reinterpret_cast<uint4*>(dx)[i] = pack8(m);
  }
}
// d_pos[w, c] = sum over grid cells whose window position is w of dx[cell, c]   (pos_embed gradient,
// backward of vision_sampler.py:304-309 on the natural grid layout)
__global__ void pos_grad_kernel(const bf16* __restrict__ dx, bf16* __restrict__ dpos, int B, int side, int r, int C,
                                int accumulate) {
  const int w = blockIdx.y;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const int wy = w / r, wx = w - wy * r, q = side / r;
  float s = 0.f;
  for (int b = 0; b < B; ++b)
    for (int qy = 0; qy < q; ++qy)
      for (int qx = 0; qx < q; ++qx)
        s += __bfloat162float(dx[(((long long)b * side + qy * r + wy) * side + qx * r + wx) * C + c]);
  const long long o = (long long)w * C + c;
  dpos[o] = __float2bfloat16(accumulate ? __bfloat162float(dpos[o]) + s : s);
}
// in: contiguous [rows, cols] fp32;  out: bf16 rows at stride out_ld (>= cols) — lets dQ land inside a packed dQKV buffer
__global__ void f32_to_bf16_kernel(const float4* __restrict__ in, bf16* __restrict__ out, long long nvec, int vpr,
                                   long long out_ld, float scale) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    const float4 a = in[2 * i], b = in[2 * i + 1];
    float f[8] = {a.x * scale, a.y * scale, a.z * scale, a.w * scale, b.x * scale, b.y * scale, b.z * scale, b.w * scale};
    const long long r = i / vpr;
    const int c = (int)(i - r * vpr) << 3;
    *reinterpret_cast<uint4*>(out + r * out_ld + c) = pack8(f);
  }
}

// ------------------------------------------------------------------- in-LLM SVA latent gather / scatter
// cambrian_llama.py:168-207 (static branch): the q*(q+1) image positions [start, start + q*(q+1)) of the residual
// stream hold q rows of (q latent queries + 1 newline token).  gather copies the q*q latent rows into a dense
// [B*q*q, H] buffer; scatter writes (updated) latent rows back in place.  Newline rows are never touched.
__global__ void span_gather_kernel(const bf16* __restrict__ hidden, bf16* __restrict__ lat, int B, int S, int H, int start,
                                   int q_h, int q_side) {
  const int vpr = H >> 3;
  const long long total = (long long)B * q_h * q_side * vpr;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    long long t = i / vpr;
    const int col = (int)(t % q_side);
    t /= q_side;
    const int row = (int)(t % q_h);
    const int b = (int)(t / q_h);
    const long long src = ((long long)b * S + start + row * (q_side + 1) + col) * H;
    reinterpret_cast<uint4*>(lat)[i] = ldg_nc(reinterpret_cast<const uint4*>(hidden + src) + v);
  }
}
__global__ void span_scatter_kernel(bf16* __restrict__ hidden, const bf16* __restrict__ lat, int B, int S, int H, int start,
                                    int q_h, int q_side) {
  const int vpr = H >> 3;
  const long long total = (long long)B * q_h * q_side * vpr;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % vpr);
    long long t = i / vpr;
    const int col = (int)(t % q_side);
    t /= q_side;
    const int row = (int)(t % q_h);
    const int b = (int)(t / q_h);
    const long long dst = ((long long)b * S + start + row * (q_side + 1) + col) * H;
    reinterpret_cast<uint4*>(hidden + dst)[v] = ldg_nc(reinterpret_cast<const uint4*>(lat) + i);
  }
}

// -------------------------------------------------------------------------------- cross entropy
// One block per row of bf16 logits [rows, V]: loss_row = logsumexp(fp32(logits)) - logit[label]; rows with
// label == ignore_index contribute 0.  If dlogits != null the row is overwritten IN PLACE with
// (softmax - onehot) * grad_scale (bf16) for the backward GEMMs (cambrian_llama.py:408-422: logits.float(),
// shift, CrossEntropyLoss mean over non-ignored; the shift is done by the caller's label pointer).
__global__ void __launch_bounds__(1024)
cross_entropy_kernel(bf16* __restrict__ logits, const long long* __restrict__ labels, float* __restrict__ loss_rows,
                     long long V, long long ld, float grad_scale, const float* __restrict__ scale_dev, int write_grad,
                     long long ignore_index) {
  __shared__ float red_m[32], red_s[32];
  if (scale_dev) grad_scale *= __ldg(scale_dev);  // e.g. 1 / (number of valid labels), counted on the device: no host sync
  const long long row = blockIdx.x;
  bf16* lp = logits + row * ld;
  const long long label = labels[row];
  const bool ignored = (label == ignore_index) || label < 0 || label >= V;
  if (ignored && !write_grad) {
    if (threadIdx.x == 0) loss_rows[row] = 0.f;
    return;
  }
  const long long nvec = V >> 3;  // V % 8 == 0 required
  float m = -INFINITY, s = 0.f;
  if (!ignored) {
    for (long long i = threadIdx.x; i < nvec; i += blockDim.x) {
      float f[8];
      unpack8(reinterpret_cast<const uint4*>(lp)[i], f);
      float lm = f[0];
#pragma unroll
      for (int e = 1; e < 8; ++e) lm = fmaxf(lm, f[e]);
      const float mn = fmaxf(m, lm);
      float acc = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) acc += __expf(f[e] - mn);
      s = s * __expf(m - mn) + acc;
      m = mn;
    }
    // block combine (max, sum)
    const float wm = warp_max(m);
    s = (m == -INFINITY) ? 0.f : s * __expf(m - wm);  // threads without elements (V/8 < blockDim) hold (-inf, 0)
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) { red_m[threadIdx.x >> 5] = wm; red_s[threadIdx.x >> 5] = s; }
    __syncthreads();
    const int nw = blockDim.x >> 5;
    float bm = -INFINITY;
    for (int k = 0; k < nw; ++k) bm = fmaxf(bm, red_m[k]);
    float bs = 0.f;
    for (int k = 0; k < nw; ++k) bs += (red_m[k] == -INFINITY) ? 0.f : red_s[k] * __expf(red_m[k] - bm);
    m = bm;
    s = bs;
    if (threadIdx.x == 0) loss_rows[row] = (m + logf(s)) - __bfloat162float(lp[label]);
    __syncthreads();
  } else if (threadIdx.x == 0) {
    loss_rows[row] = 0.f;
  }
  if (write_grad) {
    const float inv = ignored ? 0.f : grad_scale / s;
    for (long long i = threadIdx.x; i < nvec; i += blockDim.x) {
      float f[8];
      if (ignored) {
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = 0.f;
      } else {
        unpack8(reinterpret_cast<const uint4*>(lp)[i], f);
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = __expf(f[e] - m) * inv;
        const long long c0 = i << 3;
        if (label >= c0 && label < c0 + 8) f[label - c0] -= grad_scale;
      }
      reinterpret_cast<uint4*>(lp)[i] = pack8(f);
    }
  }
}
// sum of loss rows and count of non-ignored labels -> out[0] += sum, out[1] += count (single block, fixed order)
__global__ void loss_reduce_kernel(const float* __restrict__ loss_rows, const long long* __restrict__ labels,
                                   long long rows, long long V, long long ignore_index, float* __restrict__ out) {
  __shared__ float rs[32], rc[32];
  float s = 0.f, c = 0.f;
  for (long long i = threadIdx.x; i < rows; i += blockDim.x) {
    const long long l = labels[i];
    if (l != ignore_index && l >= 0 && l < V) { s += loss_rows[i]; c += 1.f; }
  }
  s = warp_sum(s);
  c = warp_sum(c);
  if ((threadIdx.x & 31) == 0) { rs[threadIdx.x >> 5] = s; rc[threadIdx.x >> 5] = c; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float ts = 0.f, tc = 0.f;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) { ts += rs[k]; tc += rc[k]; }
    out[0] += ts;
    out[1] += tc;
  }
}

// -------------------------------------------------------------------------------------- AdamW
// fp32 master weights + fp32 moments, bf16 gradients in, bf16 compute copy out (torch.optim.AdamW semantics,
// decoupled weight decay; the reference trains with HF Trainer's AdamW: cambrian_trainer.py:242-381).
// `coef` (optional, device): gradient scale computed on the device by clip_coef_kernel (1/world x clip factor) — the
// clipped update needs no host round trip.  `grad_scale` is used when coef is null.
template <int UNROLL>
__global__ void adamw_kernel(float* __restrict__ p, float* __restrict__ m, float* __restrict__ v,
                             const bf16* __restrict__ g, bf16* __restrict__ p16, long long n, float lr, float b1,
                             float b2, float eps, float wd, float bc1, float bc2, float grad_scale,
                             const float* __restrict__ coef) {
  const long long nvec = n >> 3;
  const float gs = coef ? __ldg(coef) : grad_scale;
  const float inv_sqrt_bc2 = rsqrtf(bc2), step_size = lr / bc1, decay = 1.f - lr * wd;
  const long long stride = (long long)gridDim.x * blockDim.x;
#pragma unroll UNROLL
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec; i += stride) {
    float gf[8];
    unpack8(ldg_nc(reinterpret_cast<const uint4*>(g) + i), gf);
    float4* pp = reinterpret_cast<float4*>(p) + 2 * i;
    float4* mp = reinterpret_cast<float4*>(m) + 2 * i;
    float4* vp = reinterpret_cast<float4*>(v) + 2 * i;
    float pf[8], mf[8], vf[8];
    *reinterpret_cast<float4*>(pf) = pp[0]; *reinterpret_cast<float4*>(pf + 4) = pp[1];
    *reinterpret_cast<float4*>(mf) = mp[0]; *reinterpret_cast<float4*>(mf + 4) = mp[1];
    *reinterpret_cast<float4*>(vf) = vp[0]; *reinterpret_cast<float4*>(vf + 4) = vp[1];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float gg = gf[e] * gs;
      pf[e] *= decay;
      mf[e] = b1 * mf[e] + (1.f - b1) * gg;
      vf[e] = b2 * vf[e] + (1.f - b2) * gg * gg;
      const float denom = sqrtf(vf[e]) * inv_sqrt_bc2 + eps;
      pf[e] -= step_size * (mf[e] / denom);
    }
    pp[0] = *reinterpret_cast<float4*>(pf); pp[1] = *reinterpret_cast<float4*>(pf + 4);
    mp[0] = *reinterpret_cast<float4*>(mf); mp[1] = *reinterpret_cast<float4*>(mf + 4);
    vp[0] = *reinterpret_cast<float4*>(vf); vp[1] = *reinterpret_cast<float4*>(vf + 4);
    reinterpret_cast<uint4*>(p16)[i] = pack8(pf);
  }
}

// ---------------------------------------------------------------------------- gradient clipping
// Sum of squares of a bf16 gradient range, deterministic: per-block partials in `ws`, then one block adds them to *acc in
// a fixed order (torch.nn.utils.clip_grad_norm_ as HF Trainer calls it with max_grad_norm = 1.0 in every reference script).
__global__ void sumsq_partial_kernel(const uint4* __restrict__ g, long long nvec, float* __restrict__ ws) {
  float s = 0.f;
#pragma unroll 8
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float f[8];
    unpack8(ldg_nc(g + i), f);
#pragma unroll
    for (int e = 0; e < 8; ++e) s = fmaf(f[e], f[e], s);
  }
  __shared__ float red[32];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) t += red[k];
    ws[blockIdx.x] = t;
  }
}
__global__ void sumsq_final_kernel(const float* __restrict__ ws, int nblocks, float* __restrict__ acc) {
  // one warp, fixed order: lane l sums ws[l], ws[l + 32], ... then a shuffle tree
  float t = 0.f;
  for (int i = threadIdx.x; i < nblocks; i += 32) t += ws[i];
  t = warp_sum(t);
  if (threadIdx.x == 0) acc[0] += t;
}
// coef[0] = inv_world * min(1, max_norm / (norm + 1e-6)),  coef[1] = norm  with norm = sqrt(sumsq) * inv_world (the L2 norm
// of the rank-averaged gradient);  sumsq is reset for the next step.
__global__ void clip_coef_kernel(float* __restrict__ sumsq, float max_norm, float inv_world, float* __restrict__ coef) {
  const float norm = sqrtf(sumsq[0]) * inv_world;
  coef[0] = inv_world * fminf(1.f, max_norm / (norm + 1e-6f));
  coef[1] = norm;
  sumsq[0] = 0.f;
}

// ------------------------------------------------------------------------------------------ host
#define VEC_CHECK(n, what) CB_CHECK_ARG((n) % 8 == 0, what ": element count / channel dim must be a multiple of 8")

int act_fwd_launch(const void* x, void* y, long long n, int act, cudaStream_t st) {
  VEC_CHECK(n, "act_fwd");
  if (n == 0) return CB_OK;
  act_fwd_kernel<<<grid_for(n / 8, 256), 256, 0, st>>>((const uint4*)x, (uint4*)y, n / 8, act);
  CB_CUDA_LAUNCH_CHECK("act_fwd");
  return CB_OK;
}
int act_bwd_launch(const void* dy, const void* x, void* dx, long long n, int act, cudaStream_t st) {
  VEC_CHECK(n, "act_bwd");
  if (n == 0) return CB_OK;
  act_bwd_kernel<<<grid_for(n / 8, 256), 256, 0, st>>>((const uint4*)dy, (const uint4*)x, (uint4*)dx, n / 8, act);
  CB_CUDA_LAUNCH_CHECK("act_bwd");
  return CB_OK;
}
int swiglu_fwd_launch(const void* gate, const void* up, void* out, long long rows, int I, long long ld_in,
                      long long ld_out, cudaStream_t st) {
  VEC_CHECK(I, "swiglu_fwd");
  CB_CHECK_ARG(ld_in % 8 == 0 && ld_out % 8 == 0, "swiglu: strides must be multiples of 8");
  swiglu_fwd_kernel<<<grid_for(rows * (I / 8), 256), 256, 0, st>>>((const bf16*)gate, (const bf16*)up, (bf16*)out, rows,
                                                                  I, ld_in, ld_out);
  CB_CUDA_LAUNCH_CHECK("swiglu_fwd");
  return CB_OK;
}
int swiglu_bwd_launch(const void* dout, const void* gate, const void* up, void* dgate, void* dup, long long rows, int I,
                      long long ld_in, long long ld_dout, long long ld_dgu, cudaStream_t st) {
  VEC_CHECK(I, "swiglu_bwd");
  CB_CHECK_ARG(ld_in % 8 == 0 && ld_dout % 8 == 0 && ld_dgu % 8 == 0, "swiglu: strides must be multiples of 8");
  swiglu_bwd_kernel<<<grid_for(rows * (I / 8), 256), 256, 0, st>>>((const bf16*)dout, (const bf16*)gate, (const bf16*)up,
                                                                  (bf16*)dgate, (bf16*)dup, rows, I, ld_in, ld_dout,
                                                                  ld_dgu);
  CB_CUDA_LAUNCH_CHECK("swiglu_bwd");
  return CB_OK;
}
int swiglu_bwd_fp8_launch(const void* dout, const void* gate, const void* up, void* dgate, void* dup, void* q, float* s,
                          long long rows, int I, long long ld_in, long long ld_dout, long long ld_dgu, cudaStream_t st) {
  CB_CHECK_ARG(rows > 0 && rows < (1LL << 31) && I > 0 && I % 8 == 0, "swiglu_bwd_fp8: rows=%lld, I=%d must be a "
               "multiple of 8", rows, I);
  CB_CHECK_ARG(dout && gate && up && dgate && dup && q && s, "swiglu_bwd_fp8: null argument");
  CB_CHECK_ARG(ld_in % 8 == 0 && ld_dout % 8 == 0 && ld_dgu % 8 == 0, "swiglu: strides must be multiples of 8");
  CB_CHECK_ARG(((reinterpret_cast<uintptr_t>(dout) | reinterpret_cast<uintptr_t>(gate) | reinterpret_cast<uintptr_t>(up) |
                 reinterpret_cast<uintptr_t>(dgate) | reinterpret_cast<uintptr_t>(dup) | reinterpret_cast<uintptr_t>(q)) &
                15u) == 0, "swiglu_bwd_fp8: every operand must be 16-byte aligned");
  swiglu_bwd_fp8_kernel<<<(unsigned)rows, 256, 0, st>>>((const bf16*)dout, (const bf16*)gate, (const bf16*)up,
                                                        (bf16*)dgate, (bf16*)dup, (uint8_t*)q, s, I, ld_in, ld_dout,
                                                        ld_dgu);
  CB_CUDA_LAUNCH_CHECK("swiglu_bwd_fp8");
  return CB_OK;
}
int rope_launch(void* buf, const long long* pos, const float* cos_t, const float* sin_t, long long rows, int n_heads,
                int hd, long long ld, int max_pos, int inverse, cudaStream_t st) {
  CB_CHECK_ARG(hd % 16 == 0 && ld % 8 == 0, "rope: head_dim must be a multiple of 16 and ld of 8");
  rope_kernel<<<grid_for(rows * n_heads * (hd / 16), 256), 256, 0, st>>>((bf16*)buf, pos, cos_t, sin_t, rows, n_heads, hd,
                                                                        ld, max_pos, inverse);
  CB_CUDA_LAUNCH_CHECK("rope");
  return CB_OK;
}
int embed_splice_launch(const long long* ids, const int* img_start, const void* embed, const void* img,
                        const void* newline, void* out, int B, int S, int H, int q_side, long long vocab,
                        cudaStream_t st) {
  VEC_CHECK(H, "embed_splice");
  embed_splice_kernel<<<grid_for((long long)B * S * (H / 8), 256), 256, 0, st>>>(
      ids, img_start, (const bf16*)embed, (const bf16*)img, (const bf16*)newline, (bf16*)out, B, S, H, q_side, vocab);
  CB_CUDA_LAUNCH_CHECK("embed_splice");
  return CB_OK;
}
int embed_splice_bwd_launch(const void* dout, const long long* ids, const int* img_start, void* d_embed, void* d_img,
                            void* d_nl_rows, int B, int S, int H, int q_side, long long vocab, cudaStream_t st) {
  VEC_CHECK(H, "embed_splice_bwd");
  embed_splice_bwd_kernel<<<grid_for((long long)B * S * (H / 8), 256), 256, 0, st>>>(
      (const bf16*)dout, ids, img_start, (bf16*)d_embed, (bf16*)d_img, (bf16*)d_nl_rows, B, S, H, q_side, vocab);
  CB_CUDA_LAUNCH_CHECK("embed_splice_bwd");
  return CB_OK;
}
int embed_grad_sorted_launch(const void* dout, const long long* keys, const int* order, void* d_embed, long long n, int H,
                             long long vocab, cudaStream_t st) {
  VEC_CHECK(H, "embed_grad_sorted");
  CB_CHECK_ARG(dout && keys && order && d_embed && n > 0 && vocab > 0, "embed_grad_sorted: bad arguments");
  embed_grad_sorted_kernel<<<(unsigned)n, 128, 0, st>>>((const bf16*)dout, keys, order, (bf16*)d_embed, n, H, vocab);
  CB_CUDA_LAUNCH_CHECK("embed_grad_sorted");
  return CB_OK;
}
int add_pos_tokens_launch(const void* patch, const void* cls, const void* pos, void* out, int B, int N, int C,
                          cudaStream_t st) {
  VEC_CHECK(C, "add_pos_tokens");
  add_pos_tokens_kernel<<<grid_for((long long)B * (N + 1) * (C / 8), 256), 256, 0, st>>>(
      (const bf16*)patch, (const bf16*)cls, (const bf16*)pos, (bf16*)out, B, N, C);
  CB_CUDA_LAUNCH_CHECK("add_pos_tokens");
  return CB_OK;
}
int bilinear_launch(const void* in, void* out, int B, int h, int w, int th, int tw, int C, long long in_bs,
                    long long out_bs, int out_ld, int out_col0, cudaStream_t st) {
  VEC_CHECK(C, "bilinear");
  CB_CHECK_ARG(out_ld % 8 == 0 && out_col0 % 8 == 0, "bilinear: output stride / column offset must be multiples of 8");
  bilinear_kernel<<<grid_for((long long)B * th * tw * (C / 8), 256), 256, 0, st>>>((const bf16*)in, (bf16*)out, B, h, w, th,
                                                                                  tw, C, in_bs, out_bs, out_ld, out_col0);
  CB_CUDA_LAUNCH_CHECK("bilinear");
  return CB_OK;
}
int patchify_nchw_launch(const void* img, void* out, int B, int Cin, int R, int p, int Kpad, cudaStream_t st) {
  // R need not be a multiple of p: like a stride-p convolution, the trailing R % p pixels are dropped
  // (SigLIP 384 / 14 -> 27 x 27 patches)
  CB_CHECK_ARG(R >= p && Kpad >= Cin * p * p && Kpad % 8 == 0, "patchify: image smaller than the patch or bad Kpad");
  const int g = R / p;
  patchify_nchw_kernel<<<grid_for((long long)B * g * g * Kpad, 256), 256, 0, st>>>((const bf16*)img, (bf16*)out, B, Cin, R,
                                                                                  p, Kpad);
  CB_CUDA_LAUNCH_CHECK("patchify_nchw");
  return CB_OK;
}
int patchify_nhwc_launch(const void* in, void* out, int B, int H, int W, int C, int p, cudaStream_t st) {
  VEC_CHECK(C, "patchify_nhwc");
  CB_CHECK_ARG(H >= p && W >= p, "patchify_nhwc: feature map smaller than the patch");  // remainder rows/cols are dropped (conv stride semantics)
  patchify_nhwc_kernel<<<grid_for((long long)B * H * W * (C / 8), 256), 256, 0, st>>>((const bf16*)in, (bf16*)out, B, H, W,
                                                                                     C, p);
  CB_CUDA_LAUNCH_CHECK("patchify_nhwc");
  return CB_OK;
}
int dwconv7_launch(const void* in, const void* w, const void* bias, void* out, int B, int H, int W, int C,
                   cudaStream_t st) {
  VEC_CHECK(C, "dwconv7");
  const int nchunk = (C / 8 + DW_CV - 1) / DW_CV, strips = (W + 7) / 8, steps = (H + 7) / 8;
  const long long base = (long long)nchunk * strips * B;
  // >= ~4 waves of (SMs x 3 resident blocks) when the image is tall enough, so the tail wave stays small
  const long long want = (4LL * CB_DW_MINB * device_sm_count() + base - 1) / base;
  const int ysplit = (int)std::max(1LL, std::min<long long>(steps, want));
  dwconv7_kernel<<<(unsigned)(base * ysplit), 128, 0, st>>>((const bf16*)in, (const bf16*)w, (const bf16*)bias,
                                                            (bf16*)out, B, H, W, C, ysplit);
  CB_CUDA_LAUNCH_CHECK("dwconv7");
  return CB_OK;
}
int add_inplace_launch(void* dst, const void* src, long long n, cudaStream_t st) {
  VEC_CHECK(n, "add_inplace");
  if (n == 0) return CB_OK;
  add_inplace_kernel<<<grid_for(n / 8, 256), 256, 0, st>>>((uint4*)dst, (const uint4*)src, n / 8);
  CB_CUDA_LAUNCH_CHECK("add_inplace");
  return CB_OK;
}
int group_colsum_launch(const void* x, void* out_bf16, float* out_f32, int groups, long long rows_per_group, int C,
                        float scale, int accumulate, cudaStream_t st) {
  CB_CHECK_ARG(groups > 0 && rows_per_group > 0 && C > 0, "group_colsum: empty input");
  dim3 grid((C + 31) / 32, groups);
  group_colsum_kernel<<<grid, 256, 0, st>>>((const bf16*)x, (bf16*)out_bf16, out_f32, rows_per_group, C, scale, accumulate);
  CB_CUDA_LAUNCH_CHECK("group_colsum");
  return CB_OK;
}
int group_broadcast_launch(const void* dmean, void* dx, int groups, long long rows_per_group, int C, float scale,
                           int accumulate, cudaStream_t st) {
  VEC_CHECK(C, "group_broadcast");
  group_broadcast_kernel<<<grid_for((long long)groups * rows_per_group * (C / 8), 256), 256, 0, st>>>(
      (const bf16*)dmean, (bf16*)dx, rows_per_group, C, groups, scale, accumulate);
  CB_CUDA_LAUNCH_CHECK("group_broadcast");
  return CB_OK;
}
int pos_grad_launch(const void* dx, void* dpos, int B, int side, int r, int C, int accumulate, cudaStream_t st) {
  CB_CHECK_ARG(r >= 1 && side % r == 0, "pos_grad: side must be a multiple of r");
  dim3 grid((C + 127) / 128, r * r);
  pos_grad_kernel<<<grid, 128, 0, st>>>((const bf16*)dx, (bf16*)dpos, B, side, r, C, accumulate);
  CB_CUDA_LAUNCH_CHECK("pos_grad");
  return CB_OK;
}
int f32_to_bf16_launch(const float* in, void* out, long long rows, int cols, long long out_ld, float scale,
                       cudaStream_t st) {
  VEC_CHECK(cols, "f32_to_bf16");
  CB_CHECK_ARG(out_ld % 8 == 0 && out_ld >= cols, "f32_to_bf16: out_ld must be a multiple of 8 and >= cols");
  const long long n = rows * cols;
  if (n == 0) return CB_OK;
  f32_to_bf16_kernel<<<grid_for(n / 8, 256), 256, 0, st>>>((const float4*)in, (bf16*)out, n / 8, cols / 8, out_ld, scale);
  CB_CUDA_LAUNCH_CHECK("f32_to_bf16");
  return CB_OK;
}
int window_gather_launch(const void* feat, void* out, int B, int q, int r, int C, int y0, int y1, int x0, int x1,
                         cudaStream_t st) {
  VEC_CHECK(C, "window_gather");
  CB_CHECK_ARG(q > 0 && r > 0 && 0 <= y0 && y0 < y1 && y1 <= q && 0 <= x0 && x0 < x1 && x1 <= q,
               "window_gather: crop [%d,%d)x[%d,%d) outside the %dx%d query grid", y0, y1, x0, x1, q, q);
  window_gather_kernel<<<grid_for((long long)B * (y1 - y0) * (x1 - x0) * r * r * (C / 8), 256), 256, 0, st>>>(
      (const bf16*)feat, (bf16*)out, B, q, r, C, y0, y1, x0, x1);
  CB_CUDA_LAUNCH_CHECK("window_gather");
  return CB_OK;
}
int embed_splice_ragged_launch(void* out, const void* embed, const void* img, const void* newline, const int* src,
                               long long rows, int H, cudaStream_t st) {
  VEC_CHECK(H, "embed_splice_ragged");
  CB_CHECK_ARG(rows > 0, "embed_splice_ragged: no rows");
  embed_splice_ragged_kernel<<<grid_for(rows * (H / 8), 256), 256, 0, st>>>((bf16*)out, (const bf16*)embed, (const bf16*)img,
                                                                          (const bf16*)newline, src, rows, H);
  CB_CUDA_LAUNCH_CHECK("embed_splice_ragged");
  return CB_OK;
}
int span_gather_launch(const void* hidden, void* lat, int B, int S, int H, int start, int q_h, int q_side, cudaStream_t st) {
  VEC_CHECK(H, "span_gather");
  CB_CHECK_ARG(q_h > 0 && q_side > 0 && start >= 0 && start + q_h * (q_side + 1) <= S,
               "span_gather: image span [%d, +%d) outside sequence %d", start, q_h * (q_side + 1), S);
  span_gather_kernel<<<grid_for((long long)B * q_h * q_side * (H / 8), 256), 256, 0, st>>>((const bf16*)hidden, (bf16*)lat,
                                                                                         B, S, H, start, q_h, q_side);
  CB_CUDA_LAUNCH_CHECK("span_gather");
  return CB_OK;
}
int span_scatter_launch(void* hidden, const void* lat, int B, int S, int H, int start, int q_h, int q_side, cudaStream_t st) {
  VEC_CHECK(H, "span_scatter");
  CB_CHECK_ARG(q_h > 0 && q_side > 0 && start >= 0 && start + q_h * (q_side + 1) <= S,
               "span_scatter: image span [%d, +%d) outside sequence %d", start, q_h * (q_side + 1), S);
  span_scatter_kernel<<<grid_for((long long)B * q_h * q_side * (H / 8), 256), 256, 0, st>>>((bf16*)hidden, (const bf16*)lat,
                                                                                          B, S, H, start, q_h, q_side);
  CB_CUDA_LAUNCH_CHECK("span_scatter");
  return CB_OK;
}
int cross_entropy_launch(void* logits, const long long* labels, float* loss_rows, float* loss_acc, long long rows,
                         long long V, long long ld, float grad_scale, const float* scale_dev, int write_grad,
                         long long ignore_index, cudaStream_t st) {
  CB_CHECK_ARG(V % 8 == 0 && ld % 8 == 0, "cross_entropy: vocab and ld must be multiples of 8");
  CB_CHECK_ARG(rows > 0, "cross_entropy: no rows");
  cross_entropy_kernel<<<(unsigned)rows, 1024, 0, st>>>((bf16*)logits, labels, loss_rows, V, ld, grad_scale, scale_dev,
                                                       write_grad, ignore_index);
  CB_CUDA_LAUNCH_CHECK("cross_entropy");
  if (loss_acc) {
    loss_reduce_kernel<<<1, 1024, 0, st>>>(loss_rows, labels, rows, V, ignore_index, loss_acc);
    CB_CUDA_LAUNCH_CHECK("loss_reduce");
  }
  return CB_OK;
}
// background != 0: ONE 128-thread block per SM (72 registers x 4 warps = 9.2 K of the 11.8 K registers a resident GEMM CTA
// — 320 threads x 168 registers, ~200 KB smem — leaves free; no shared memory) so the grid fits NEXT TO a persistent GEMM
// CTA on every SM: the HBM-bound update then runs underneath tensor-core-bound work instead of taking all 2048 thread
// slots of each SM and serialising with it (r01: the GEMMs launched behind an 8-blocks/SM AdamW grid ran at ~1000 instead
// of ~1480 TFLOP/s because their CTAs had to wait).  4 independent 112-byte load groups per thread keep ~57 KB per SM in
// flight, enough for a few TB/s; it only has to finish under the pass it hides in.
int adamw_launch(float* p, float* m, float* v, const void* g, void* p16, long long n, float lr, float b1, float b2,
                 float eps, float wd, int step, float grad_scale, const float* clip_coef, int background,
                 cudaStream_t st) {
  VEC_CHECK(n, "adamw");
  CB_CHECK_ARG(step >= 1, "adamw: step must be >= 1");
  if (n == 0) return CB_OK;
  const float bc1 = 1.f - powf(b1, (float)step), bc2 = 1.f - powf(b2, (float)step);
  if (background)
    adamw_kernel<4><<<grid_for(n / 8, 128, 1), 128, 0, st>>>(p, m, v, (const bf16*)g, (bf16*)p16, n, lr, b1, b2, eps, wd,
                                                            bc1, bc2, grad_scale, clip_coef);
  else
    adamw_kernel<1><<<grid_for(n / 8, 256), 256, 0, st>>>(p, m, v, (const bf16*)g, (bf16*)p16, n, lr, b1, b2, eps, wd, bc1,
                                                         bc2, grad_scale, clip_coef);
  CB_CUDA_LAUNCH_CHECK("adamw");
  return CB_OK;
}
int sumsq_launch(const void* g, long long n, float* acc, float* ws, long long ws_floats, int background, cudaStream_t st) {
  VEC_CHECK(n, "sumsq");
  CB_CHECK_ARG(acc && ws, "sumsq: null accumulator / workspace");
  if (n == 0) return CB_OK;
  const int threads = background ? 128 : 256;
  const unsigned grid = grid_for(n / 8, threads, background ? 1 : 8);
  CB_CHECK_ARG((long long)grid <= ws_floats, "sumsq: workspace too small (%lld < %u floats)", ws_floats, grid);
  sumsq_partial_kernel<<<grid, threads, 0, st>>>((const uint4*)g, n / 8, ws);
  CB_CUDA_LAUNCH_CHECK("sumsq_partial");
  sumsq_final_kernel<<<1, 32, 0, st>>>(ws, (int)grid, acc);
  CB_CUDA_LAUNCH_CHECK("sumsq_final");
  return CB_OK;
}
int clip_coef_launch(float* sumsq, float max_norm, float inv_world, float* coef, cudaStream_t st) {
  CB_CHECK_ARG(sumsq && coef && max_norm > 0.f && inv_world > 0.f, "clip_coef: bad arguments");
  clip_coef_kernel<<<1, 1, 0, st>>>(sumsq, max_norm, inv_world, coef);
  CB_CUDA_LAUNCH_CHECK("clip_coef");
  return CB_OK;
}

}  // namespace cb
