// cambrian_b200 — extern "C" entry points (the drop-in boundary, include/cambrian_b200.h).
#include "common.cuh"
#include "../../include/cambrian_b200.h"
#include <cstdarg>
#include <cstdio>
#include <atomic>

namespace cb {

static thread_local char g_err[512] = "";

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

static std::atomic<long long> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
long long launch_count() { return g_launches.load(std::memory_order_relaxed); }

int device_sm_count() {
  static int sms[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (sms[dev] == 0) {
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
    sms[dev] = v;
  }
  return sms[dev];
}

// implemented in the kernel translation units
int gemm_bf16(const void*, const void*, void*, int, int, int, int, long long, long long, long long, long long,
              long long, long long, int, int, const void*, const void*, const void*, long long, long long, float,
              int, int, int, int, cudaStream_t);
int sva_window_attn_fwd_launch(const void*, void*, float*, int, const void* const*, const void* const*,
                               const void* const*, const int*, int, int, int, int, cudaStream_t);
int sva_window_attn_bwd_launch(const void*, const void*, const void*, const float*, void*, int,
                               const void* const*, const void* const*, const void* const*, void* const*,
                               void* const*, const int*, int, int, int, int, cudaStream_t);
int layernorm_fwd(const void*, const void*, const void*, void*, float*, float*, long long, int, float,
                  const void*, int, int, cudaStream_t);
int layernorm_bwd(const void*, const void*, const void*, const float*, const float*, void*, const void*, void*, void*,
                  float*, long long, long long, int, const void*, int, int, cudaStream_t);
int rmsnorm_fwd(const void*, const void*, void*, float*, long long, int, float, int, cudaStream_t);
int rmsnorm_bwd(const void*, const void*, const void*, const float*, void*, const void*, void*, float*, long long,
                long long, int, cudaStream_t);
long long norm_bwd_workspace_floats(long long, int);

int attn_fwd_launch(const void*, const void*, const void*, void*, float*, const void*, int, int, int, int, int, int,
                    long long, long long, long long, long long, long long, long long, long long, long long, float, int,
                    int, cudaStream_t);
int attn_bwd_launch(const void*, const void*, const void*, const void*, const void*, const float*, float*, void*, void*,
                    void*, const void*, int, int, int, int, int, int, long long, long long, long long, long long,
                    long long, long long, long long, long long, long long, long long, long long, long long, long long,
                    long long, long long, long long, float, int, int, cudaStream_t);
int act_fwd_launch(const void*, void*, long long, int, cudaStream_t);
int act_bwd_launch(const void*, const void*, void*, long long, int, cudaStream_t);
int swiglu_fwd_launch(const void*, const void*, void*, long long, int, long long, long long, cudaStream_t);
int swiglu_bwd_launch(const void*, const void*, const void*, void*, void*, long long, int, long long, long long,
                      long long, cudaStream_t);
int rope_launch(void*, const long long*, const float*, const float*, long long, int, int, long long, int, int,
                cudaStream_t);
int embed_splice_launch(const long long*, const int*, const void*, const void*, const void*, void*, int, int, int, int,
                        long long, cudaStream_t);
int embed_splice_bwd_launch(const void*, const long long*, const int*, void*, void*, void*, int, int, int, int,
                            long long, cudaStream_t);
int embed_grad_sorted_launch(const void*, const long long*, const int*, void*, long long, int, long long, cudaStream_t);
int add_pos_tokens_launch(const void*, const void*, const void*, void*, int, int, int, cudaStream_t);
int bilinear_launch(const void*, void*, int, int, int, int, int, int, long long, long long, int, int, cudaStream_t);
int patchify_nchw_launch(const void*, void*, int, int, int, int, int, cudaStream_t);
int patchify_nhwc_launch(const void*, void*, int, int, int, int, int, cudaStream_t);
int dwconv7_launch(const void*, const void*, const void*, void*, int, int, int, int, cudaStream_t);
int add_inplace_launch(void*, const void*, long long, cudaStream_t);
int group_colsum_launch(const void*, void*, float*, int, long long, int, float, int, cudaStream_t);
int group_broadcast_launch(const void*, void*, int, long long, int, float, int, cudaStream_t);
int pos_grad_launch(const void*, void*, int, int, int, int, int, cudaStream_t);
int f32_to_bf16_launch(const float*, void*, long long, int, long long, float, cudaStream_t);
int cross_entropy_launch(void*, const long long*, float*, float*, long long, long long, long long, float, const float*,
                         int, long long, cudaStream_t);
int adamw_launch(float*, float*, float*, const void*, void*, long long, float, float, float, float, float, int, float,
                 const float*, int, cudaStream_t);
int adamw_host_launch(float*, float*, float*, const void*, void*, long long, float, float, float, float, float, int, float,
                      const float*, int, cudaStream_t);
int adamw8_launch(float*, void*, void*, float*, float*, const void*, void*, long long, float, float, float, float, float, int,
                  float, const float*, int, cudaStream_t);
int adamw8_host_launch(float*, void*, void*, float*, float*, const void*, void*, long long, float, float, float, float, float,
                       int, float, const float*, int, cudaStream_t);
int sumsq_launch(const void*, long long, float*, float*, long long, int, cudaStream_t);
int gemv_bf16_launch(const void*, const void*, void*, int, int, int, long long, long long, long long, const void*, const void*,
                     long long, int, cudaStream_t);
int allreduce_symm_launch(unsigned long long, const unsigned long long*, const unsigned long long*, long long, long long, int,
                          int, unsigned int, int, cudaStream_t);
int clip_coef_launch(float*, float, float, float*, cudaStream_t);
int span_gather_launch(const void*, void*, int, int, int, int, int, int, cudaStream_t);
int span_scatter_launch(void*, const void*, int, int, int, int, int, int, cudaStream_t);
int gemm_swiglu_bf16(const void*, const void*, void*, void*, int, int, int, long long, long long, long long, long long,
                     cudaStream_t);
int resample_ksize(int, int);
void resample_coeffs(int, int, int*, int*);
long long preprocess_workspace_bytes(int, int, int);
int preprocess_launch(const uint8_t*, int, int, int, const int*, const float*, const float*, void*, uint8_t*, void*, long long,
                      cudaStream_t);
int window_gather_launch(const void*, void*, int, int, int, int, int, int, int, int, cudaStream_t);
int embed_splice_ragged_launch(void*, const void*, const void*, const void*, const int*, long long, int, cudaStream_t);
int tower_combine_fwd_launch(const void*, int, const void* const*, const void*, void*, long long, int, int, cudaStream_t);
int tower_combine_bwd_launch(const void*, int, const void* const*, const void*, void* const*, void*, long long, int, int,
                             cudaStream_t);
int bilinear_bwd_launch(const void*, void*, int, int, int, int, int, int, cudaStream_t);
int nf4_quantize_launch(const void*, int, int, float*, long long, void*, void*, float*, float*, cudaStream_t);
int gemv_nf4_launch(const void*, void*, int, int, int, long long, long long, int, const int*, const void* const*,
                    const void* const*, const void* const*, const void* const*, const void*, const void*, long long, int,
                    cudaStream_t);
int nf4_dequant_launch(void*, int, int, int, const int*, const void* const*, const void* const*, const void* const*,
                       const void* const*, cudaStream_t);
int int8_quantize_weight_launch(const void*, int, int, long long, void*, float*, cudaStream_t);
int int8_quantize_act_launch(const void*, int, int, long long, float, void*, float*, unsigned*, int*, int*, cudaStream_t);
int gemv_int8_launch(const void*, const void*, const float*, const float*, const void*, long long, const int*, const int*,
                     void*, int, int, int, long long, const void*, const void*, long long, int, cudaStream_t);
int gemm_int8_launch(const void*, const void*, const float*, const float*, const void*, long long, const int*, const int*,
                     void*, int, int, int, long long, const void*, const void*, long long, int, cudaStream_t);
int fp8_quantize_weight_launch(const void*, int, int, long long, void*, float*, cudaStream_t);
int fp8_quantize_act_launch(const void*, int, int, long long, void*, float*, cudaStream_t);
int gemv_fp8_launch(const void*, const void*, const float*, const float*, void*, int, int, int, long long, const void*,
                    const void*, long long, int, cudaStream_t);
int gemm_fp8_launch(const void*, const void*, const float*, const float*, void*, int, int, int, long long, const void*,
                    const void*, long long, int, cudaStream_t);
int kv_fp8_append_launch(const void*, const void*, long long, void*, void*, float*, float*, int, int, int, int, int, long long,
                         const long long*, cudaStream_t);
long long attn_decode_fp8_workspace_floats(int, int, int, int, int);
int attn_decode_fp8_launch(const void*, long long, const void*, const void*, const float*, const float*, const void*, long long,
                           void*, float*, long long, int, int, int, int, int, int, long long, const long long*, float,
                           cudaStream_t);
long long fp8_quantize_weight_t_workspace_floats(int, int);
int fp8_quantize_weight_t_launch(const void*, int, int, long long, void*, float*, float*, long long, cudaStream_t);
int rmsnorm_fwd_fp8(const void*, const void*, void*, float*, float*, long long, int, float, int, cudaStream_t);
int swiglu_bwd_fp8_launch(const void*, const void*, const void*, void*, void*, void*, float*, long long, int, long long,
                          long long, long long, cudaStream_t);
int paged_kv_append_launch(const void*, const void*, long long, void*, void*, float*, float*, int, const int*, long long,
                           const int*, int, int, int, int, int, int, int, long long, int, cudaStream_t);
long long attn_decode_paged_workspace_floats(int, int, int, int, int);
int attn_decode_paged_launch(const void*, long long, const void*, const void*, const float*, const float*, int, const int*,
                             long long, const int*, int, void*, float*, long long, int, int, int, int, int, int, int, float,
                             cudaStream_t);
int paged_kv_gather_launch(const void*, const void*, const float*, const float*, int, const int*, int, int, int, int, int,
                           long long, void*, void*, long long, cudaStream_t);
long long sample_tokens_workspace_floats(int, int);
int sample_tokens_launch(const float*, long long, int, int, const float*, const int*, const float*, const uint64_t*,
                         const int64_t*, int64_t*, float*, long long, cudaStream_t);

}  // namespace cb

#define ST(s) static_cast<cudaStream_t>(s)

extern "C" {

int cb_version(void) { return 1; }
const char* cb_last_error(void) { return cb::g_err; }
int cb_sm_count(void) { return cb::device_sm_count(); }
int64_t cb_launch_count(void) { return cb::launch_count(); }

int cb_gemm_bf16(const void* A, const void* B, void* C, int M, int N, int K, int batch, int64_t lda,
                 int64_t ldb, int64_t ldc, int64_t bsa, int64_t bsb, int64_t bsc, int a_mn, int b_mn,
                 const void* bias, const void* colscale, const void* residual, int64_t ldr, int64_t bsr,
                 float alpha, int act, int out_fp32, int accumulate, int force_bn, void* stream) {
  return cb::gemm_bf16(A, B, C, M, N, K, batch, lda, ldb, ldc, bsa, bsb, bsc, a_mn, b_mn, bias, colscale,
                       residual, ldr, bsr, alpha, act, out_fp32, accumulate, force_bn, ST(stream));
}

int cb_sva_window_attn_fwd(const void* q, void* out, float* lse, int num_towers, const void* const* k,
                           const void* const* v, const void* const* mask, const int* r, int batch,
                           int q_side, int hidden, int windowed, void* stream) {
  return cb::sva_window_attn_fwd_launch(q, out, lse, num_towers, k, v, mask, r, batch, q_side, hidden, windowed,
                                        ST(stream));
}
int cb_sva_window_attn_bwd(const void* q, const void* out, const void* dout, const float* lse, void* dq,
                           int num_towers, const void* const* k, const void* const* v,
                           const void* const* mask, void* const* dk, void* const* dv, const int* r,
                           int batch, int q_side, int hidden, int windowed, void* stream) {
  return cb::sva_window_attn_bwd_launch(q, out, dout, lse, dq, num_towers, k, v, mask, dk, dv, r, batch,
                                        q_side, hidden, windowed, ST(stream));
}

int cb_layernorm_fwd(const void* x, const void* gamma, const void* beta, void* y, float* mean, float* rstd,
                     int64_t rows, int C, float eps, const void* pos, int side, int r, void* stream) {
  return cb::layernorm_fwd(x, gamma, beta, y, mean, rstd, rows, C, eps, pos, side, r, ST(stream));
}
int cb_layernorm_bwd(const void* dy, const void* x, const void* gamma, const float* mean, const float* rstd,
                     void* dx, const void* dres, void* dgamma, void* dbeta, float* workspace,
                     int64_t workspace_floats, int64_t rows, int C, const void* pos, int side, int r, void* stream) {
  return cb::layernorm_bwd(dy, x, gamma, mean, rstd, dx, dres, dgamma, dbeta, workspace, workspace_floats, rows, C,
                           pos, side, r, ST(stream));
}
int cb_rmsnorm_fwd(const void* x, const void* gamma, void* y, float* rstd, int64_t rows, int C, float eps,
                   int hf_cast, void* stream) {
  return cb::rmsnorm_fwd(x, gamma, y, rstd, rows, C, eps, hf_cast, ST(stream));
}
int cb_rmsnorm_bwd(const void* dy, const void* x, const void* gamma, const float* rstd, void* dx,
                   const void* dres, void* dgamma, float* workspace, int64_t workspace_floats, int64_t rows, int C,
                   void* stream) {
  return cb::rmsnorm_bwd(dy, x, gamma, rstd, dx, dres, dgamma, workspace, workspace_floats, rows, C, ST(stream));
}
int64_t cb_norm_bwd_workspace_floats(int64_t rows, int C) { return cb::norm_bwd_workspace_floats(rows, C); }

int cb_attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, const void* kmask, int B, int nh,
                int nkv, int Sq, int Skv, int hd, int64_t q_bs, int64_t q_ss, int64_t k_bs, int64_t k_ss,
                int64_t v_bs, int64_t v_ss, int64_t o_bs, int64_t o_ss, float scale, int causal, void* stream) {
  return cb::attn_fwd_launch(q, k, v, o, lse, kmask, B, nh, nkv, Sq, Skv, hd, q_bs, q_ss, k_bs, k_ss, v_bs, v_ss, o_bs,
                             o_ss, scale, causal, 0, ST(stream));
}
int cb_attn_fwd_window(const void* q, const void* k, const void* v, void* o, float* lse, const void* kmask, int B,
                       int nh, int nkv, int Sq, int Skv, int hd, int64_t q_bs, int64_t q_ss, int64_t k_bs, int64_t k_ss,
                       int64_t v_bs, int64_t v_ss, int64_t o_bs, int64_t o_ss, float scale, int causal, int window,
                       void* stream) {
  return cb::attn_fwd_launch(q, k, v, o, lse, kmask, B, nh, nkv, Sq, Skv, hd, q_bs, q_ss, k_bs, k_ss, v_bs, v_ss, o_bs,
                             o_ss, scale, causal, window, ST(stream));
}
int cb_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                float* delta, void* dq, void* dk, void* dv, const void* kmask, int B, int nh, int nkv, int Sq,
                int Skv, int hd, int64_t q_bs, int64_t q_ss, int64_t k_bs, int64_t k_ss, int64_t v_bs, int64_t v_ss,
                int64_t o_bs, int64_t o_ss, int64_t do_bs, int64_t do_ss, int64_t dq_bs, int64_t dq_ss,
                int64_t dk_bs, int64_t dk_ss, int64_t dv_bs, int64_t dv_ss, float scale, int causal, void* stream) {
  return cb::attn_bwd_launch(q, k, v, o, d_o, lse, delta, dq, dk, dv, kmask, B, nh, nkv, Sq, Skv, hd, q_bs, q_ss,
                             k_bs, k_ss, v_bs, v_ss, o_bs, o_ss, do_bs, do_ss, dq_bs, dq_ss, dk_bs, dk_ss, dv_bs, dv_ss,
                             scale, causal, 0, ST(stream));
}
int cb_attn_bwd_window(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                       float* delta, void* dq, void* dk, void* dv, const void* kmask, int B, int nh, int nkv, int Sq,
                       int Skv, int hd, int64_t q_bs, int64_t q_ss, int64_t k_bs, int64_t k_ss, int64_t v_bs,
                       int64_t v_ss, int64_t o_bs, int64_t o_ss, int64_t do_bs, int64_t do_ss, int64_t dq_bs,
                       int64_t dq_ss, int64_t dk_bs, int64_t dk_ss, int64_t dv_bs, int64_t dv_ss, float scale,
                       int causal, int window, void* stream) {
  return cb::attn_bwd_launch(q, k, v, o, d_o, lse, delta, dq, dk, dv, kmask, B, nh, nkv, Sq, Skv, hd, q_bs, q_ss,
                             k_bs, k_ss, v_bs, v_ss, o_bs, o_ss, do_bs, do_ss, dq_bs, dq_ss, dk_bs, dk_ss, dv_bs, dv_ss,
                             scale, causal, window, ST(stream));
}
int cb_act_fwd(const void* x, void* y, int64_t n, int act, void* stream) {
  return cb::act_fwd_launch(x, y, n, act, ST(stream));
}
int cb_act_bwd(const void* dy, const void* x, void* dx, int64_t n, int act, void* stream) {
  return cb::act_bwd_launch(dy, x, dx, n, act, ST(stream));
}
int cb_swiglu_fwd(const void* gate, const void* up, void* out, int64_t rows, int I, int64_t ld_in, int64_t ld_out,
                  void* stream) {
  return cb::swiglu_fwd_launch(gate, up, out, rows, I, ld_in, ld_out, ST(stream));
}
int cb_swiglu_bwd(const void* dout, const void* gate, const void* up, void* dgate, void* dup, int64_t rows, int I,
                  int64_t ld_in, int64_t ld_dout, int64_t ld_dgu, void* stream) {
  return cb::swiglu_bwd_launch(dout, gate, up, dgate, dup, rows, I, ld_in, ld_dout, ld_dgu, ST(stream));
}
int cb_rope(void* buf, const int64_t* pos, const float* cos_t, const float* sin_t, int64_t rows, int n_heads, int hd,
            int64_t ld, int max_pos, int inverse, void* stream) {
  return cb::rope_launch(buf, reinterpret_cast<const long long*>(pos), cos_t, sin_t, rows, n_heads, hd, ld, max_pos,
                         inverse, ST(stream));
}
int cb_embed_splice(const int64_t* ids, const int32_t* img_start, const void* embed, const void* img,
                    const void* newline, void* out, int B, int S, int H, int q_side, int64_t vocab, void* stream) {
  return cb::embed_splice_launch(reinterpret_cast<const long long*>(ids), img_start, embed, img, newline, out, B, S, H,
                                 q_side, vocab, ST(stream));
}
int cb_embed_splice_bwd(const void* dout, const int64_t* ids, const int32_t* img_start, void* d_embed, void* d_img,
                        void* d_newline_rows, int B, int S, int H, int q_side, int64_t vocab, void* stream) {
  return cb::embed_splice_bwd_launch(dout, reinterpret_cast<const long long*>(ids), img_start, d_embed, d_img,
                                     d_newline_rows, B, S, H, q_side, vocab, ST(stream));
}
int cb_add_pos_tokens(const void* patch, const void* cls, const void* pos, void* out, int B, int N, int C,
                      void* stream) {
  return cb::add_pos_tokens_launch(patch, cls, pos, out, B, N, C, ST(stream));
}
int cb_bilinear(const void* in, void* out, int B, int h, int w, int th, int tw, int C, int64_t in_bs, int64_t out_bs,
                int out_ld, int out_col0, void* stream) {
  return cb::bilinear_launch(in, out, B, h, w, th, tw, C, in_bs, out_bs, out_ld, out_col0, ST(stream));
}
int cb_patchify_nchw(const void* img, void* out, int B, int Cin, int R, int p, int Kpad, void* stream) {
  return cb::patchify_nchw_launch(img, out, B, Cin, R, p, Kpad, ST(stream));
}
int cb_patchify_nhwc(const void* in, void* out, int B, int H, int W, int C, int p, void* stream) {
  return cb::patchify_nhwc_launch(in, out, B, H, W, C, p, ST(stream));
}
int cb_dwconv7(const void* in, const void* w, const void* bias, void* out, int B, int H, int W, int C, void* stream) {
  return cb::dwconv7_launch(in, w, bias, out, B, H, W, C, ST(stream));
}
int cb_add_inplace(void* dst, const void* src, int64_t n, void* stream) {
  return cb::add_inplace_launch(dst, src, n, ST(stream));
}
int cb_group_colsum(const void* x, void* out_bf16, float* out_f32, int groups, int64_t rows_per_group, int C,
                    float scale, int accumulate, void* stream) {
  return cb::group_colsum_launch(x, out_bf16, out_f32, groups, rows_per_group, C, scale, accumulate, ST(stream));
}
int cb_group_broadcast(const void* dmean, void* dx, int groups, int64_t rows_per_group, int C, float scale,
                       int accumulate, void* stream) {
  return cb::group_broadcast_launch(dmean, dx, groups, rows_per_group, C, scale, accumulate, ST(stream));
}
int cb_pos_grad(const void* dx, void* dpos, int B, int side, int r, int C, int accumulate, void* stream) {
  return cb::pos_grad_launch(dx, dpos, B, side, r, C, accumulate, ST(stream));
}
int cb_f32_to_bf16(const float* in, void* out, int64_t rows, int cols, int64_t out_ld, float scale, void* stream) {
  return cb::f32_to_bf16_launch(in, out, rows, cols, out_ld, scale, ST(stream));
}
int cb_cross_entropy(void* logits, const int64_t* labels, float* loss_rows, float* loss_acc, int64_t rows, int64_t V,
                     int64_t ld, float grad_scale, int write_grad, int64_t ignore_index, void* stream) {
  return cb::cross_entropy_launch(logits, reinterpret_cast<const long long*>(labels), loss_rows, loss_acc, rows, V, ld,
                                  grad_scale, nullptr, write_grad, ignore_index, ST(stream));
}
int cb_cross_entropy_ex(void* logits, const int64_t* labels, float* loss_rows, float* loss_acc, int64_t rows, int64_t V,
                        int64_t ld, float grad_scale, const float* grad_scale_dev, int write_grad, int64_t ignore_index,
                        void* stream) {
  return cb::cross_entropy_launch(logits, reinterpret_cast<const long long*>(labels), loss_rows, loss_acc, rows, V, ld,
                                  grad_scale, grad_scale_dev, write_grad, ignore_index, ST(stream));
}
int cb_span_gather(const void* hidden, void* lat, int B, int S, int H, int start, int q_side, void* stream) {
  return cb::span_gather_launch(hidden, lat, B, S, H, start, q_side, q_side, ST(stream));
}
int cb_span_gather_hw(const void* hidden, void* lat, int B, int S, int H, int start, int q_h, int q_w, void* stream) {
  return cb::span_gather_launch(hidden, lat, B, S, H, start, q_h, q_w, ST(stream));
}
int cb_span_scatter_hw(void* hidden, const void* lat, int B, int S, int H, int start, int q_h, int q_w, void* stream) {
  return cb::span_scatter_launch(hidden, lat, B, S, H, start, q_h, q_w, ST(stream));
}
int cb_window_gather(const void* feat, void* out, int B, int q_side, int r, int C, int y0, int y1, int x0, int x1,
                     void* stream) {
  return cb::window_gather_launch(feat, out, B, q_side, r, C, y0, y1, x0, x1, ST(stream));
}
int cb_embed_splice_ragged(void* out, const void* embed, const void* img, const void* newline, const int32_t* src,
                           int64_t rows, int H, void* stream) {
  return cb::embed_splice_ragged_launch(out, embed, img, newline, src, rows, H, ST(stream));
}
int cb_span_scatter(void* hidden, const void* lat, int B, int S, int H, int start, int q_side, void* stream) {
  return cb::span_scatter_launch(hidden, lat, B, S, H, start, q_side, q_side, ST(stream));
}
int cb_gemm_swiglu_bf16(const void* A, const void* W, void* gu_out, void* act_out, int M, int F, int K, int64_t lda,
                        int64_t ldw, int64_t ld_gu, int64_t ld_act, void* stream) {
  return cb::gemm_swiglu_bf16(A, W, gu_out, act_out, M, F, K, lda, ldw, ld_gu, ld_act, ST(stream));
}
int cb_resample_ksize(int in_size, int out_size) {
  if (in_size <= 0 || out_size <= 0) return 0;
  return cb::resample_ksize(in_size, out_size);
}
int cb_resample_coeffs(int in_size, int out_size, int32_t* bounds, int32_t* kk) {
  if (in_size <= 0 || out_size <= 0 || !bounds || !kk) return cb::set_error(CB_ERR_INVALID, "resample_coeffs: bad arguments");
  cb::resample_coeffs(in_size, out_size, bounds, kk);
  return CB_OK;
}
int64_t cb_preprocess_workspace_bytes(int H, int W, int R) {
  if (H <= 0 || W <= 0 || R <= 0) return 0;
  return cb::preprocess_workspace_bytes(H, W, R);
}
int cb_preprocess_image(const uint8_t* img, int H, int W, int R, const int32_t* pad_rgb, const float* mean,
                        const float* std, void* out, uint8_t* out_u8, void* workspace, int64_t workspace_bytes,
                        void* stream) {
  if (!img || !pad_rgb || !mean || !std || !out || !workspace)
    return cb::set_error(CB_ERR_INVALID, "preprocess_image: null argument");
  return cb::preprocess_launch(img, H, W, R, pad_rgb, mean, std, out, out_u8, workspace, workspace_bytes, ST(stream));
}
int cb_adamw(float* p, float* m, float* v, const void* g, void* p16, int64_t n, float lr, float beta1, float beta2,
             float eps, float weight_decay, int step, float grad_scale, void* stream) {
  return cb::adamw_launch(p, m, v, g, p16, n, lr, beta1, beta2, eps, weight_decay, step, grad_scale, nullptr, 0, ST(stream));
}
int cb_adamw_ex(float* p, float* m, float* v, const void* g, void* p16, int64_t n, float lr, float beta1, float beta2,
                float eps, float weight_decay, int step, float grad_scale, const float* clip_coef, int background,
                void* stream) {
  return cb::adamw_launch(p, m, v, g, p16, n, lr, beta1, beta2, eps, weight_decay, step, grad_scale, clip_coef, background,
                          ST(stream));
}
int cb_adamw_host(float* p, float* m, float* v, const void* g, void* p16, int64_t n, float lr, float beta1, float beta2,
                  float eps, float weight_decay, int step, float grad_scale, const float* clip_coef, int ctas, void* stream) {
  return cb::adamw_host_launch(p, m, v, g, p16, n, lr, beta1, beta2, eps, weight_decay, step, grad_scale, clip_coef, ctas,
                               ST(stream));
}
int cb_adamw8(float* p, uint8_t* qm, uint8_t* qv, float* sm, float* sv, const void* g, void* p16, int64_t n, float lr,
              float beta1, float beta2, float eps, float weight_decay, int step, float grad_scale, const float* clip_coef,
              int background, void* stream) {
  return cb::adamw8_launch(p, qm, qv, sm, sv, g, p16, n, lr, beta1, beta2, eps, weight_decay, step, grad_scale, clip_coef,
                           background, ST(stream));
}
int cb_adamw8_host(float* p, uint8_t* qm, uint8_t* qv, float* sm, float* sv, const void* g, void* p16, int64_t n,
                   float lr, float beta1, float beta2, float eps, float weight_decay, int step, float grad_scale,
                   const float* clip_coef, int ctas, void* stream) {
  return cb::adamw8_host_launch(p, qm, qv, sm, sv, g, p16, n, lr, beta1, beta2, eps, weight_decay, step, grad_scale,
                                clip_coef, ctas, ST(stream));
}
int cb_embed_grad_sorted(const void* dout, const int64_t* keys, const int32_t* order, void* d_embed, int64_t n, int H,
                         int64_t vocab, void* stream) {
  return cb::embed_grad_sorted_launch(dout, reinterpret_cast<const long long*>(keys), order, d_embed, n, H, vocab,
                                      ST(stream));
}
int cb_allreduce_symm_bf16(uint64_t multicast_base, const uint64_t* buffer_ptrs, const uint64_t* signal_pad_ptrs,
                           int64_t offset_bytes, int64_t nbytes, int rank, int world, uint32_t epoch, int ctas, void* stream) {
  return cb::allreduce_symm_launch(multicast_base, reinterpret_cast<const unsigned long long*>(buffer_ptrs),
                                   reinterpret_cast<const unsigned long long*>(signal_pad_ptrs), offset_bytes, nbytes, rank,
                                   world, epoch, ctas, ST(stream));
}
int cb_gemv_bf16(const void* x, const void* w, void* y, int M, int N, int K, int64_t ldx, int64_t ldw, int64_t ldy,
                 const void* bias, const void* residual, int64_t ldr, int out_fp32, void* stream) {
  return cb::gemv_bf16_launch(x, w, y, M, N, K, ldx, ldw, ldy, bias, residual, ldr, out_fp32, ST(stream));
}
int cb_sumsq_bf16(const void* g, int64_t n, float* acc, float* workspace, int64_t workspace_floats, int background,
                  void* stream) {
  return cb::sumsq_launch(g, n, acc, workspace, workspace_floats, background, ST(stream));
}
int cb_clip_coef(float* sumsq, float max_norm, float inv_world, float* coef, void* stream) {
  return cb::clip_coef_launch(sumsq, max_norm, inv_world, coef, ST(stream));
}
int cb_tower_combine_fwd(const void* logits, int ld_logits, const void* const* aggs, const void* q_in, void* out, int64_t N,
                         int C, int num_towers, void* stream) {
  return cb::tower_combine_fwd_launch(logits, ld_logits, aggs, q_in, out, N, C, num_towers, ST(stream));
}
int cb_tower_combine_bwd(const void* logits, int ld_logits, const void* const* aggs, const void* dout, void* const* daggs,
                         void* dlogits, int64_t N, int C, int num_towers, void* stream) {
  return cb::tower_combine_bwd_launch(logits, ld_logits, aggs, dout, daggs, dlogits, N, C, num_towers, ST(stream));
}
int cb_bilinear_bwd(const void* dout, void* din, int B, int h, int w, int th, int tw, int C, void* stream) {
  return cb::bilinear_bwd_launch(dout, din, B, h, w, th, tw, C, ST(stream));
}
int cb_nf4_quantize(const void* w, int N, int K, float* absmax_ws, int64_t ws_floats, void* packed, void* qabsmax,
                    float* absmax2, float* offset, void* stream) {
  return cb::nf4_quantize_launch(w, N, K, absmax_ws, ws_floats, packed, qabsmax, absmax2, offset, ST(stream));
}
int cb_gemv_nf4(const void* x, void* y, int M, int N, int K, int64_t ldx, int64_t ldy, int nseg, const int32_t* seg_row0,
                const void* const* packed, const void* const* qabsmax, const void* const* absmax2, const void* const* offset,
                const void* bias, const void* residual, int64_t ldr, int out_fp32, void* stream) {
  return cb::gemv_nf4_launch(x, y, M, N, K, ldx, ldy, nseg, seg_row0, packed, qabsmax, absmax2, offset, bias, residual, ldr,
                             out_fp32, ST(stream));
}
int cb_nf4_dequant(void* out, int N, int K, int nseg, const int32_t* seg_row0, const void* const* packed,
                   const void* const* qabsmax, const void* const* absmax2, const void* const* offset, void* stream) {
  return cb::nf4_dequant_launch(out, N, K, nseg, seg_row0, packed, qabsmax, absmax2, offset, ST(stream));
}
int cb_int8_quantize_weight(const void* w, int N, int K, int64_t ldw, void* cb, float* scb, void* stream) {
  return cb::int8_quantize_weight_launch(w, N, K, ldw, cb, scb, ST(stream));
}
int cb_int8_quantize_act(const void* x, int M, int K, int64_t ldx, float threshold, void* xq, float* sca,
                         uint32_t* colmax_ws, int32_t* outlier_idx, int32_t* n_outlier, void* stream) {
  return cb::int8_quantize_act_launch(x, M, K, ldx, threshold, xq, sca, colmax_ws, outlier_idx, n_outlier, ST(stream));
}
int cb_gemv_int8(const void* xq, const void* cb, const float* sca, const float* scb, const void* x, int64_t ldx,
                 const int32_t* outlier_idx, const int32_t* n_outlier, void* y, int M, int N, int K, int64_t ldy,
                 const void* bias, const void* residual, int64_t ldr, int out_fp32, void* stream) {
  return cb::gemv_int8_launch(xq, cb, sca, scb, x, ldx, outlier_idx, n_outlier, y, M, N, K, ldy, bias, residual, ldr,
                              out_fp32, ST(stream));
}
int cb_gemm_int8(const void* xq, const void* cb, const float* sca, const float* scb, const void* x, int64_t ldx,
                 const int32_t* outlier_idx, const int32_t* n_outlier, void* y, int M, int N, int K, int64_t ldy,
                 const void* bias, const void* residual, int64_t ldr, int out_fp32, void* stream) {
  return cb::gemm_int8_launch(xq, cb, sca, scb, x, ldx, outlier_idx, n_outlier, y, M, N, K, ldy, bias, residual, ldr,
                              out_fp32, ST(stream));
}
int cb_fp8_quantize_weight(const void* w, int N, int K, int64_t ldw, void* wq, float* sw, void* stream) {
  return cb::fp8_quantize_weight_launch(w, N, K, ldw, wq, sw, ST(stream));
}
int cb_fp8_quantize_act(const void* x, int M, int K, int64_t ldx, void* xq, float* sa, void* stream) {
  return cb::fp8_quantize_act_launch(x, M, K, ldx, xq, sa, ST(stream));
}
int cb_gemv_fp8(const void* xq, const void* wq, const float* sa, const float* sw, void* y, int M, int N, int K,
                int64_t ldy, const void* bias, const void* residual, int64_t ldr, int out_fp32, void* stream) {
  return cb::gemv_fp8_launch(xq, wq, sa, sw, y, M, N, K, ldy, bias, residual, ldr, out_fp32, ST(stream));
}
int cb_gemm_fp8(const void* xq, const void* wq, const float* sa, const float* sw, void* y, int M, int N, int K,
                int64_t ldy, const void* bias, const void* residual, int64_t ldr, int out_fp32, void* stream) {
  return cb::gemm_fp8_launch(xq, wq, sa, sw, y, M, N, K, ldy, bias, residual, ldr, out_fp32, ST(stream));
}
int cb_kv_fp8_append(const void* k, const void* v, int64_t ld, void* kq, void* vq, float* ks, float* vs, int B, int S,
                     int S_max, int nkv, int hd, int64_t offset, const int64_t* offset_dev, void* stream) {
  return cb::kv_fp8_append_launch(k, v, ld, kq, vq, ks, vs, B, S, S_max, nkv, hd, offset,
                                  reinterpret_cast<const long long*>(offset_dev), ST(stream));
}
int64_t cb_attn_decode_fp8_workspace_floats(int B, int nh, int nkv, int S_max, int hd) {
  return cb::attn_decode_fp8_workspace_floats(B, nh, nkv, S_max, hd);
}
int cb_attn_decode_fp8(const void* q, int64_t q_bs, const void* kq, const void* vq, const float* ks, const float* vs,
                       const void* kmask, int64_t kmask_ld, void* o, float* workspace, int64_t workspace_floats, int B, int Sq,
                       int nh, int nkv, int S_max, int hd, int64_t length, const int64_t* length_dev, float scale,
                       void* stream) {
  return cb::attn_decode_fp8_launch(q, q_bs, kq, vq, ks, vs, kmask, kmask_ld, o, workspace, workspace_floats, B, Sq, nh, nkv,
                                    S_max, hd, length, reinterpret_cast<const long long*>(length_dev), scale, ST(stream));
}
int64_t cb_fp8_quantize_weight_t_workspace_floats(int N, int K) {
  return cb::fp8_quantize_weight_t_workspace_floats(N, K);
}
int cb_fp8_quantize_weight_t(const void* w, int N, int K, int64_t ldw, void* wtq, float* st, float* workspace,
                             int64_t workspace_floats, void* stream) {
  return cb::fp8_quantize_weight_t_launch(w, N, K, ldw, wtq, st, workspace, workspace_floats, ST(stream));
}
int cb_rmsnorm_fwd_fp8(const void* x, const void* gamma, void* xq, float* sa, float* rstd, int64_t rows, int C, float eps,
                       int hf_cast, void* stream) {
  return cb::rmsnorm_fwd_fp8(x, gamma, xq, sa, rstd, rows, C, eps, hf_cast, ST(stream));
}
int cb_swiglu_bwd_fp8(const void* dout, const void* gate, const void* up, void* dgate, void* dup, void* dguq, float* sdgu,
                      int64_t rows, int I, int64_t ld_in, int64_t ld_dout, int64_t ld_dgu, void* stream) {
  return cb::swiglu_bwd_fp8_launch(dout, gate, up, dgate, dup, dguq, sdgu, rows, I, ld_in, ld_dout, ld_dgu, ST(stream));
}
int cb_paged_kv_append(const void* k, const void* v, int64_t ld, void* k_pages, void* v_pages, float* k_scales,
                       float* v_scales, int fp8, const int* block_table, int64_t table_ld, const int* lens, int rows, int S,
                       int nkv, int hd, int page_size, int num_pages, int max_pages, int64_t offset, int offset_from_lens,
                       void* stream) {
  return cb::paged_kv_append_launch(k, v, ld, k_pages, v_pages, k_scales, v_scales, fp8, block_table, table_ld, lens, rows,
                                    S, nkv, hd, page_size, num_pages, max_pages, offset, offset_from_lens, ST(stream));
}
int64_t cb_attn_decode_paged_workspace_floats(int rows, int nh, int max_pages, int page_size, int hd) {
  return cb::attn_decode_paged_workspace_floats(rows, nh, max_pages, page_size, hd);
}
int cb_attn_decode_paged(const void* q, int64_t q_bs, const void* k_pages, const void* v_pages, const float* k_scales,
                         const float* v_scales, int fp8, const int* block_table, int64_t table_ld, const int* lens,
                         int len_add, void* o, float* workspace, int64_t workspace_floats, int rows, int nh, int nkv, int hd,
                         int page_size, int num_pages, int max_pages, float scale, void* stream) {
  return cb::attn_decode_paged_launch(q, q_bs, k_pages, v_pages, k_scales, v_scales, fp8, block_table, table_ld, lens,
                                      len_add, o, workspace, workspace_floats, rows, nh, nkv, hd, page_size, num_pages,
                                      max_pages, scale, ST(stream));
}
int cb_paged_kv_gather(const void* k_pages, const void* v_pages, const float* k_scales, const float* v_scales, int fp8,
                       const int* block_table_row, int nkv, int hd, int page_size, int num_pages, int max_pages, int64_t P,
                       void* out_k, void* out_v, int64_t out_ld, void* stream) {
  return cb::paged_kv_gather_launch(k_pages, v_pages, k_scales, v_scales, fp8, block_table_row, nkv, hd, page_size,
                                    num_pages, max_pages, P, out_k, out_v, out_ld, ST(stream));
}
int64_t cb_sample_tokens_workspace_floats(int rows, int V) { return cb::sample_tokens_workspace_floats(rows, V); }
int cb_sample_tokens(const float* logits, int64_t ld, int rows, int V, const float* temperature, const int* top_k,
                     const float* top_p, const uint64_t* seed, const int64_t* step, int64_t* out, float* workspace,
                     int64_t workspace_floats, void* stream) {
  return cb::sample_tokens_launch(logits, ld, rows, V, temperature, top_k, top_p, seed, step, out, workspace,
                                  workspace_floats, ST(stream));
}

}  // extern "C"
