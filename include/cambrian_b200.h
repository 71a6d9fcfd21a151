/* cambrian_b200 — C ABI of the H100-native (sm_90a) Cambrian-1 hot-path kernels (libcambrian_b200.so).
 *
 * The reference (cambrian-mllm/cambrian) has NO FFI / plugin layer: its hot path is Python
 * nn.Modules that dispatch torch ops (SURVEY.md §2a, §8b).  This header therefore declares the
 * boundary a maintainer binds from Python with ctypes (see INTEGRATION.md): one entry point per
 * operator the reference modules execute, each citing the reference call site it replaces.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer owned by the caller (torch allocations); the library never
 *     allocates, frees or retains memory (SURVEY.md §8b "Memory ownership");
 *   - `stream` is the caller's cudaStream_t (torch.cuda.current_stream().cuda_stream) passed as void*;
 *   - all entry points are re-entrant per stream, keep no global mutable state besides one-time
 *     function-attribute caches, and return 0 on success or a CB_ERR_* code; cb_last_error()
 *     returns a thread-local message.  The Python wrappers re-raise ValueError / RuntimeError as
 *     the reference modules do (vision_sampler.py:202-206, builder.py:147);
 *   - activations and parameters are bf16 (uint16 storage) unless a parameter says otherwise;
 *     statistics, LSE and losses are fp32; token ids / labels / positions are int64.
 */
#ifndef CAMBRIAN_B200_H
#define CAMBRIAN_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CB_OK 0
#define CB_ERR_INVALID 1
#define CB_ERR_CUDA 2
#define CB_ERR_UNSUPPORTED 3

/* activation codes for cb_gemm_bf16 / cb_act_* */
#define CB_ACT_NONE 0
#define CB_ACT_GELU_ERF 1   /* nn.GELU()            vision_sampler.py:241, cambrian_arch.py:49,56 */
#define CB_ACT_GELU_TANH 2  /* gelu(approximate='tanh') (SigLIP HF variant)                       */
#define CB_ACT_QUICK_GELU 3 /* CLIP quick_gelu      clip_encoder.py:47 -> HF CLIPMLP              */
#define CB_ACT_SILU 4       /* LLaMA SwiGLU gate    cambrian_llama.py:142-164 -> HF LlamaMLP      */

int cb_version(void);
const char* cb_last_error(void);
int cb_sm_count(void);
/* number of kernels this library has launched in this process (bench.py reports the per-step delta as gpu_launches) */
int64_t cb_launch_count(void);

/* ---- dense contraction: wgmma + TMA GEMM ----------------------------------------------------
 * C[b] (M x N row-major, ldc)  (+)=  epi( alpha * opA(A[b]) (M x K) * opB(B[b]) (K x N) )
 *   a_mn = 0: A is [M, K] with K contiguous (lda);  a_mn = 1: A is [K, M] with M contiguous
 *   b_mn = 0: B is [N, K] with K contiguous (ldb) — the nn.Linear weight layout;  b_mn = 1: [K, N]
 *   epi(v) = act(v + bias[n]) * colscale[n] + residual[m, n]; each of bias/colscale/residual may be NULL
 *   out_fp32: C is fp32 instead of bf16; accumulate: C += epi(..)
 *   force_bn: 0 = heuristic tile width, else 64 / 128 / 256
 * Replaces every nn.Linear / matmul of the hot path: HF CLIP/DINOv2/LLaMA linears, timm SigLIP /
 * ConvNeXt linears, vision_sampler.py:170-175,254-257 (q/k/v/o/proj_* Linear), cambrian_arch.py:49,56
 * (mm_projector, mm_projector_aux), cambrian_llama.py:402-409 (lm_head), and their autograd backward.
 * Requires lda/ldb and the batch strides to be multiples of 8 elements and 16-byte aligned bases (TMA). */
int cb_gemm_bf16(const void* A, const void* B, void* C, int M, int N, int K, int batch,
                 int64_t lda, int64_t ldb, int64_t ldc, int64_t bsa, int64_t bsb, int64_t bsc,
                 int a_mn, int b_mn, const void* bias, const void* colscale, const void* residual,
                 int64_t ldr, int64_t bsr, float alpha, int act, int out_fp32, int accumulate,
                 int force_bn, void* stream);

/* ---- SVA window attention (SURVEY.md §8a A6) -------------------------------------------------
 * Fused replacement of rearrange_vision_tower_features_train (cambrian_arch.py:271-287) + the SDPA
 * inside MultiKVCrossAttention.forward (vision_sampler.py:191-230).
 *   q, out : [batch*q_side*q_side, hidden] bf16 (hidden = 1024 = 16 heads x 64)
 *   k[t], v[t] : [batch, (r[t]*q_side)^2, hidden] bf16 projected key/value grids in natural layout
 *   mask[t] : [batch*q_side*q_side, r[t]*r[t]] bool (1 byte) or NULL (= all true); `mask` itself may be NULL
 *   lse : [batch*q_side*q_side, 16] fp32 log2-domain log-sum-exp, needed by the backward (may be NULL)
 *   windowed = 1: k/v are the reference's window-rearranged [N, r*r, hidden] tensors (vision_sampler.py API);
 *   windowed = 0: natural grid layout (the fast path used by cambrian_arch: no permute/contiguous copies)
 *   A query whose keys are masked in every tower attends to nothing: the forward writes out = 0 and LSE = +inf for it
 *   (not NaN), and the backward writes dq = 0 for it.  The backward writes every dk / dv row of every tower: masked keys,
 *   including all keys of such a query, get exact zero rows. */
int cb_sva_window_attn_fwd(const void* q, void* out, float* lse, int num_towers, const void* const* k,
                           const void* const* v, const void* const* mask, const int* r, int batch,
                           int q_side, int hidden, int windowed, void* stream);
int cb_sva_window_attn_bwd(const void* q, const void* out, const void* dout, const float* lse, void* dq,
                           int num_towers, const void* const* k, const void* const* v,
                           const void* const* mask, void* const* dk, void* const* dv, const int* r,
                           int batch, int q_side, int hidden, int windowed, void* stream);

/* ---- normalisation ----------------------------------------------------------------------------
 * LayerNorm over the last dim C (nn.LayerNorm, eps in fp32 statistics).  `pos` (may be NULL) is the
 * SVA pos_embed [r*r, C] added to row x BEFORE normalising, indexed by the cell's position in its
 * r x r window of a side x side grid (vision_sampler.py:304-309 fused with :170-175).
 * mean/rstd [rows] fp32 are written when non-NULL (needed by the backward). */
int cb_layernorm_fwd(const void* x, const void* gamma, const void* beta, void* y, float* mean, float* rstd,
                     int64_t rows, int C, float eps, const void* pos, int side, int r, void* stream);
/* dres (may be NULL): gradient arriving on the residual branch, fused as dx = dres + d(norm input).
 * side = 0 selects the window-rearranged layout [N, r*r, C] for `pos` (row % (r*r)); side > 0 the natural grid. */
int cb_layernorm_bwd(const void* dy, const void* x, const void* gamma, const float* mean, const float* rstd,
                     void* dx, const void* dres, void* dgamma, void* dbeta, float* workspace,
                     int64_t workspace_floats, int64_t rows, int C, const void* pos, int side, int r, void* stream);
/* LLaMA RMSNorm.  hf_cast = 0: (w * x_hat_fp32).to(bf16) — the variant the reference trains with
 * (train_fsdp.py:1429-1435);  hf_cast = 1: w * x_hat.to(bf16) — stock HF LlamaRMSNorm (inference). */
int cb_rmsnorm_fwd(const void* x, const void* gamma, void* y, float* rstd, int64_t rows, int C, float eps,
                   int hf_cast, void* stream);
int cb_rmsnorm_bwd(const void* dy, const void* x, const void* gamma, const float* rstd, void* dx,
                   const void* dres, void* dgamma, float* workspace, int64_t workspace_floats, int64_t rows, int C,
                   void* stream);
int64_t cb_norm_bwd_workspace_floats(int64_t rows, int C);

/* ---- softmax attention: wgmma flash attention --------------------------------------------------
 * q/k/v/o element (b, s, head, d) lives at base + b*bs + s*ss + head*hd + d (element strides), so the packed
 * QKV GEMM output is consumed in place.  nh % nkv == 0 (GQA).  kmask [B, Skv] bool (1 byte, 1 = attend) or NULL.
 * causal: key k visible to query i iff k <= i + (Skv - Sq).  lse [B, nh, Sq] fp32 (log2 domain) may be NULL.
 * Replaces torch SDPA inside HF CLIPAttention / Dinov2SelfAttention / timm Attention (clip_encoder.py:104,
 * dino_encoder.py:159, siglip_encoder.py:97) and HF LlamaSdpaAttention with the 4-D causal+padding mask of
 * cambrian_llama.py:123-128.  head_dim: any multiple of 8 up to 128 (fwd); 64, 96 or 128 (bwd). */
int cb_attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, const void* kmask, int B, int nh,
                int nkv, int Sq, int Skv, int hd, int64_t q_bs, int64_t q_ss, int64_t k_bs, int64_t k_ss,
                int64_t v_bs, int64_t v_ss, int64_t o_bs, int64_t o_ss, float scale, int causal, void* stream);
/* cb_attn_fwd with a causal sliding window (Phi-3): key slot j is visible from query slot i (i = query row + Skv - Sq)
 * iff 0 <= i - j < window, on top of the key mask.  window = 0 means none and is cb_attn_fwd exactly; window > 0 needs
 * causal = 1.  Key tiles before the window of a whole warpgroup are skipped, not masked. */
int cb_attn_fwd_window(const void* q, const void* k, const void* v, void* o, float* lse, const void* kmask, int B,
                       int nh, int nkv, int Sq, int Skv, int hd, int64_t q_bs, int64_t q_ss, int64_t k_bs, int64_t k_ss,
                       int64_t v_bs, int64_t v_ss, int64_t o_bs, int64_t o_ss, float scale, int causal, int window,
                       void* stream);
/* delta [B, nh, Sq] fp32 scratch; dq/dk/dv written (bf16, strided, heads packed at hd: dq may be a view into a packed
 * dQKV buffer).  Every output element has one writer (no atomics), so the results are bit-identical from run to run. */
int cb_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                float* delta, void* dq, void* dk, void* dv, const void* kmask, int B, int nh, int nkv, int Sq,
                int Skv, int hd, int64_t q_bs, int64_t q_ss, int64_t k_bs, int64_t k_ss, int64_t v_bs, int64_t v_ss,
                int64_t o_bs, int64_t o_ss, int64_t do_bs, int64_t do_ss, int64_t dq_bs, int64_t dq_ss,
                int64_t dk_bs, int64_t dk_ss, int64_t dv_bs, int64_t dv_ss, float scale, int causal, void* stream);
/* cb_attn_bwd with the causal sliding window of cb_attn_fwd_window (pass the same window and the lse it wrote): query
 * tiles past the window of a whole warpgroup's keys, and key tiles before the window of a whole warpgroup's queries,
 * are skipped.  window = 0 means none and is cb_attn_bwd exactly; window > 0 needs causal = 1.  A query row that sees no
 * key (lse = +inf) gets dq = 0. */
int cb_attn_bwd_window(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                       float* delta, void* dq, void* dk, void* dv, const void* kmask, int B, int nh, int nkv, int Sq,
                       int Skv, int hd, int64_t q_bs, int64_t q_ss, int64_t k_bs, int64_t k_ss, int64_t v_bs,
                       int64_t v_ss, int64_t o_bs, int64_t o_ss, int64_t do_bs, int64_t do_ss, int64_t dq_bs,
                       int64_t dq_ss, int64_t dk_bs, int64_t dk_ss, int64_t dv_bs, int64_t dv_ss, float scale,
                       int causal, int window, void* stream);

/* ---- elementwise / gather / reduction kernels (HBM-bound) -------------------------------------- */
/* y = act(x), dx = dy * act'(x); n elements (n % 8 == 0).  nn.GELU of vision_sampler.py:241, cambrian_arch.py:49,56 */
int cb_act_fwd(const void* x, void* y, int64_t n, int act, void* stream);
int cb_act_bwd(const void* dy, const void* x, void* dx, int64_t n, int act, void* stream);
/* out = silu(gate) * up (HF LlamaMLP); gate/up rows may live in one [rows, 2I] buffer (ld_in) */
int cb_swiglu_fwd(const void* gate, const void* up, void* out, int64_t rows, int I, int64_t ld_in, int64_t ld_out,
                  void* stream);
int cb_swiglu_bwd(const void* dout, const void* gate, const void* up, void* dgate, void* dup, int64_t rows, int I,
                  int64_t ld_in, int64_t ld_dout, int64_t ld_dgu, void* stream);
/* in-place rotary embedding of the first n_heads heads of each row of a packed [rows, ld] buffer;
 * pos int64 [rows]; cos/sin fp32 [max_pos, hd/2]; inverse = 1 applies the transpose (backward).
 * HF apply_rotary_pos_emb as used by LlamaAttention (cambrian_llama.py:142-164). */
int cb_rope(void* buf, const int64_t* pos, const float* cos_t, const float* sin_t, int64_t rows, int n_heads, int hd,
            int64_t ld, int max_pos, int inverse, void* stream);
/* inputs_embeds [B,S,H]: embed_tokens gather + image-span replace + image_newline column
 * (cambrian_arch.py:413-420, :457-490).  img [B, q*q, H] or NULL (text only); img_start int32 [B] (<0: no image) */
int cb_embed_splice(const int64_t* ids, const int32_t* img_start, const void* embed, const void* img,
                    const void* newline, void* out, int B, int S, int H, int q_side, int64_t vocab, void* stream);
int cb_embed_splice_bwd(const void* dout, const int64_t* ids, const int32_t* img_start, void* d_embed, void* d_img,
                        void* d_newline_rows, int B, int S, int H, int q_side, int64_t vocab, void* stream);
/* ViT token assembly: out[b] = [cls + pos[0]] ++ (patch[b] + pos[1:])  (cls may be NULL: SigLIP) */
int cb_add_pos_tokens(const void* patch, const void* cls, const void* pos, void* out, int B, int N, int C,
                      void* stream);
/* fp32 bilinear token-grid resize, align_corners=False (clip_encoder.py:83-88 and siblings, cambrian_arch.py:397-400)
 * in: [B, h, w, C] rows at in_bs batch stride; out row (b, oy, ox) at out + b*out_bs + (oy*tw+ox)*out_ld + out_col0 */
int cb_bilinear(const void* in, void* out, int B, int h, int w, int th, int tw, int C, int64_t in_bs, int64_t out_bs,
                int out_ld, int out_col0, void* stream);
/* im2col for strided patch convolutions feeding cb_gemm_bf16 */
int cb_patchify_nchw(const void* img, void* out, int B, int Cin, int R, int p, int Kpad, void* stream);
int cb_patchify_nhwc(const void* in, void* out, int B, int H, int W, int C, int p, void* stream);
/* depthwise 7x7 conv, NHWC, weights [7,7,C] (timm ConvNeXtBlock.conv_dw via clip_convnext_encoder.py:121-144) */
int cb_dwconv7(const void* in, const void* w, const void* bias, void* out, int B, int H, int W, int C, void* stream);
int cb_add_inplace(void* dst, const void* src, int64_t n, void* stream);
/* out[g, c] = scale * sum_r x[g*rows_per_group + r, c]; either output may be NULL (cambrian_arch.py:377 mean; bias grads) */
int cb_group_colsum(const void* x, void* out_bf16, float* out_f32, int groups, int64_t rows_per_group, int C,
                    float scale, int accumulate, void* stream);
int cb_group_broadcast(const void* dmean, void* dx, int groups, int64_t rows_per_group, int C, float scale,
                       int accumulate, void* stream);
/* d pos_embed [r*r, C] from the gradient of the (x + pos) rows on the natural grid layout */
int cb_pos_grad(const void* dx, void* dpos, int B, int side, int r, int C, int accumulate, void* stream);
/* fp32 [rows, cols] contiguous -> bf16 rows at stride out_ld, times scale (dQ of cb_attn_bwd into a packed dQKV buffer) */
int cb_f32_to_bf16(const float* in, void* out, int64_t rows, int cols, int64_t out_ld, float scale, void* stream);
/* per-row cross entropy on bf16 logits [rows, V] (fp32 math, cambrian_llama.py:408-422); loss_rows [rows];
 * loss_acc (may be NULL) += {sum of losses, number of non-ignored rows}; write_grad overwrites the logits in place
 * with (softmax - onehot) * grad_scale. */
int cb_cross_entropy(void* logits, const int64_t* labels, float* loss_rows, float* loss_acc, int64_t rows, int64_t V,
                     int64_t ld, float grad_scale, int write_grad, int64_t ignore_index, void* stream);
/* same, with an additional gradient scale read from DEVICE memory (grad_scale_dev[0], may be NULL): the mean over
 * non-ignored labels (cambrian_llama.py:411-422) without counting them on the host */
int cb_cross_entropy_ex(void* logits, const int64_t* labels, float* loss_rows, float* loss_acc, int64_t rows, int64_t V,
                        int64_t ld, float grad_scale, const float* grad_scale_dev, int write_grad, int64_t ignore_index,
                        void* stream);
/* in-LLM SVA site (cambrian_llama.py:168-207): gather the q*q latent rows of the image span [start, start+q*(q+1))
 * of hidden [B,S,H] into lat [B*q*q, H] / scatter updated rows back in place (newline rows untouched) */
int cb_span_gather(const void* hidden, void* lat, int B, int S, int H, int start, int q_side, void* stream);
int cb_span_scatter(void* hidden, const void* lat, int B, int S, int H, int start, int q_side, void* stream);
/* Dynamic-shape (per-sample, non-square) variant of the two above: the span holds q_h rows of (q_w queries + 1 newline)
 * (cambrian_llama.py:208-253, final_vision_feature_size[b] = (q_h, q_w)). */
int cb_span_gather_hw(const void* hidden, void* lat, int B, int S, int H, int start, int q_h, int q_w, void* stream);
int cb_span_scatter_hw(void* hidden, const void* lat, int B, int S, int H, int start, int q_h, int q_w, void* stream);
/* Window rearrangement with the `unpad_image` crop of the q x q window grid
 * (rearrange_vision_tower_features_inference, cambrian_arch.py:289-330; full range = _train, :271-287):
 * feat [B, q*r, q*r, C] -> out [B*(y1-y0)*(x1-x0), r*r, C] for query rows [y0,y1) x columns [x0,x1). */
int cb_window_gather(const void* feat, void* out, int B, int q_side, int r, int C, int y0, int y1, int x0, int x1,
                     void* stream);
/* Ragged embed + splice of the dynamic branch (cambrian_arch.py:493-609): out[row] = embed[src[row]] if src >= 0,
 * zeros if src == -1 (padding), newline if src == INT32_MIN, img[-2 - src] otherwise; rows = B * max_len. */
int cb_embed_splice_ragged(void* out, const void* embed, const void* img, const void* newline, const int32_t* src,
                           int64_t rows, int H, void* stream);
/* LLaMA MLP first half in one launch (HF LlamaMLP, reached from cambrian_llama.py:142-166): W = [gate_proj; up_proj]
 * [2F, K]; gu_out [M, 2F] = A W^T (bf16 pre-activations, saved for backward), act_out [M, F] = silu(gate) * up.
 * F % 128 == 0.  wgmma GEMM whose tile pairs 64 gate columns with the matching 64 up columns. */
int cb_gemm_swiglu_bf16(const void* A, const void* W, void* gu_out, void* act_out, int M, int F, int K, int64_t lda,
                        int64_t ldw, int64_t ld_gu, int64_t ld_act, void* stream);
/* Image preprocessing on the GPU (SURVEY.md 8f rank 4) — replaces, per tower, the host chain of `process_images`
 * (mm_utils.py:186-201): expand2square(img, int(mean*255)) -> PIL Image.resize((R,R)) [bicubic, antialiased, uint8,
 * bit-exact with Pillow's Resample.c] -> x/255 -> (x-mean)/std.  img: device uint8 [H,W,3] RGB; out: bf16 [3,R,R];
 * out_u8 (optional, may be NULL): the resized uint8 image [R,R,3]; pad_rgb / mean / std: HOST arrays of 3.
 * cb_resample_ksize / cb_resample_coeffs are the host-side coefficient generator (bounds [out,2], kk [out,ksize],
 * 22-bit fixed point) exposed for tests. */
int cb_resample_ksize(int in_size, int out_size);
int cb_resample_coeffs(int in_size, int out_size, int32_t* bounds, int32_t* kk);
int64_t cb_preprocess_workspace_bytes(int H, int W, int R);
int cb_preprocess_image(const uint8_t* img, int H, int W, int R, const int32_t* pad_rgb, const float* mean,
                        const float* std, void* out, uint8_t* out_u8, void* workspace, int64_t workspace_bytes,
                        void* stream);
/* AdamW on fp32 master weights / moments with bf16 gradients, writing the bf16 compute copy */
int cb_adamw(float* p, float* m, float* v, const void* g, void* p16, int64_t n, float lr, float beta1, float beta2,
             float eps, float weight_decay, int step, float grad_scale, void* stream);
/* cb_adamw with (a) the gradient scale read from DEVICE memory (clip_coef[0], written by cb_clip_coef; null = use
 * grad_scale) so a clipped step needs no host sync, and (b) a background launch shape (one small block per SM) that
 * co-resides with a persistent GEMM CTA on every SM.  Replaces HF Trainer's clip_grad_norm_ + AdamW.step
 * (cambrian_trainer.py:242-381; transformers Trainer max_grad_norm default 1.0). */
int cb_adamw_ex(float* p, float* m, float* v, const void* g, void* p16, int64_t n, float lr, float beta1, float beta2,
                float eps, float weight_decay, int step, float grad_scale, const float* clip_coef, int background,
                void* stream);
/* cb_adamw_ex with the fp32 state in HOST memory (DeepSpeed's `offload_optimizer`, scripts/zero3_offload.json), the
 * arithmetic still on the GPU and bitwise equal to cb_adamw_ex: p, m, v are host memory registered with CUDA and mapped
 * (cudaHostRegister with cudaHostRegisterMapped), read and written over PCIe in one pass; g, p16 (and clip_coef) are
 * device memory.  The one exception to "every pointer is a device pointer".  Every pointer's placement is checked before
 * the launch: a pointer in the wrong kind of memory returns CB_ERR_INVALID naming the argument.  ctas: blocks of the
 * PCIe-bound grid (0 = default); 128-thread blocks without shared memory that fit next to a resident GEMM CTA. */
int cb_adamw_host(float* p, float* m, float* v, const void* g, void* p16, int64_t n, float lr, float beta1, float beta2,
                  float eps, float weight_decay, int step, float grad_scale, const float* clip_coef, int ctas, void* stream);
/* cb_adamw_ex with 8-bit block-wise quantised moments (HF `optim="adamw_bnb_8bit"`, cambrian_trainer.py:365-367): m and v
 * are one uint8 code per element (qm against the signed dynamic map, qv against the unsigned one) and one fp32 absmax per
 * 256-element block (sm, sv; ceil(n / 256) each); p stays the fp32 master.  Per element: dequantise (map[code] * absmax),
 * update with cb_adamw_ex's arithmetic, write p and p16; then per block requantise m and v against their new absmax.
 * n % 8 == 0; the last block may be partial.  No atomics: bit-reproducible.  Alignment: p, g, p16 16 B; qm, qv 8 B. */
int cb_adamw8(float* p, uint8_t* qm, uint8_t* qv, float* sm, float* sv, const void* g, void* p16, int64_t n, float lr,
              float beta1, float beta2, float eps, float weight_decay, int step, float grad_scale, const float* clip_coef,
              int background, void* stream);
/* cb_adamw8 with p, qm, qv, sm, sv in registered, mapped host memory (offload_optimizer), bitwise equal to cb_adamw8; g,
 * p16 (and clip_coef) are device memory.  Placement is checked as cb_adamw_host checks it, before any launch.  ctas:
 * blocks of the PCIe-bound grid (0 = default). */
int cb_adamw8_host(float* p, uint8_t* qm, uint8_t* qv, float* sm, float* sv, const void* g, void* p16, int64_t n,
                   float lr, float beta1, float beta2, float eps, float weight_decay, int step, float grad_scale,
                   const float* clip_coef, int ctas, void* stream);
/* Deterministic gradient of the embedding rows (backward of embed_tokens inside cb_embed_splice): rows of dout [n, H] with
 * equal keys[t] (token id; >= vocab = no gradient, e.g. the image span) are summed in position order by one block and
 * written once to d_embed [vocab, H] (pre-zeroed).  `order` = positions stably sorted by key.  Replaces the racing
 * bf16x2 atomics of cb_embed_splice_bwd (pass d_embed = NULL there). */
int cb_embed_grad_sorted(const void* dout, const int64_t* keys, const int32_t* order, void* d_embed, int64_t n, int H,
                         int64_t vocab, void* stream);
/* Decode-shaped projection, M <= 8 rows: y[M,N] = x[M,K] W[N,K]^T (+ bias[N]) (+ residual[M,N]); W in nn.Linear layout.
 * Weight-streaming CUDA-core kernel (each weight byte read once, fp32 accumulation) used by the KV-cache decode step of
 * generate() (cambrian_llama.py:437-483) where a 128-row tensor-core tile would idle; y bf16 or fp32 (lm_head logits). */
int cb_gemv_bf16(const void* x, const void* w, void* y, int M, int N, int K, int64_t ldx, int64_t ldw, int64_t ldy,
                 const void* bias, const void* residual, int64_t ldr, int out_fp32, void* stream);
/* In-place sum all-reduce of the bf16 range [offset_bytes, +nbytes) of a SYMMETRIC buffer (same offset on every rank) —
 * the bucketed gradient reduction of the data-parallel step (reference: inside torch_xla FSDP; explicit helper
 * cambrian_trainer.py:181-190).  multicast_base != 0: NVLS path (multimem.ld_reduce / multimem.st, the NVSwitch adds and
 * fans out); 0: peer loads / stores over NVLink.  buffer_ptrs / signal_pad_ptrs: HOST arrays of `world` peer-mapped device
 * addresses (this rank's own included).  epoch: strictly increasing across launches on all ranks alike, advance by 2 per
 * call.  nbytes % (16 * world) == 0.  Every rank must issue the same calls in the same order. */
int cb_allreduce_symm_bf16(uint64_t multicast_base, const uint64_t* buffer_ptrs, const uint64_t* signal_pad_ptrs,
                           int64_t offset_bytes, int64_t nbytes, int rank, int world, uint32_t epoch, int ctas, void* stream);
/* acc[0] += sum of squares of n bf16 values (deterministic two-stage reduction; workspace >= grid floats, 4096 suffices) */
int cb_sumsq_bf16(const void* g, int64_t n, float* acc, float* workspace, int64_t workspace_floats, int background,
                  void* stream);
/* coef[0] = inv_world * min(1, max_norm / (sqrt(sumsq[0]) * inv_world + 1e-6)); coef[1] = that norm; sumsq[0] = 0
 * (torch.nn.utils.clip_grad_norm_ on the rank-averaged gradient, all on the device) */
int cb_clip_coef(float* sumsq, float max_norm, float inv_world, float* coef, void* stream);
/* `sep` aggregator layer (VisionAggregationLayer.forward, vision_sampler.py:368-398): per-query softmax over the towers
 * of the weight_mlp logits and the weighted sum of the per-tower aggregates added to the query stream,
 *   out[n,:] = q_in[n,:] + sum_t softmax(logits[n,:T])[t] * aggs[t][n,:]        (replaces .softmax(-1), torch.stack,
 * (agg * weight).sum(2) and the residual add).  logits [N, ld_logits >= T] bf16 (columns >= T are padding), aggs = HOST
 * array of T device pointers to [N, C] bf16.  Backward: daggs[t] = w_t * dout, dlogits = softmax adjoint of
 * g_t = <dout, agg_t> (padding columns zeroed); d q_in = dout. */
int cb_tower_combine_fwd(const void* logits, int ld_logits, const void* const* aggs, const void* q_in, void* out, int64_t N,
                         int C, int num_towers, void* stream);
int cb_tower_combine_bwd(const void* logits, int ld_logits, const void* const* aggs, const void* dout, void* const* daggs,
                         void* dlogits, int64_t N, int C, int num_towers, void* stream);
/* adjoint of cb_bilinear on contiguous grids: dout [B, th, tw, C] -> din [B, h, w, C] (backward of the query-grid resize
 * cambrian_arch.py:394-401 and of the towers' token interpolation, clip_encoder.py:83-88 and siblings); deterministic */
int cb_bilinear_bwd(const void* dout, void* din, int B, int h, int w, int th, int tw, int C, void* stream);
/* 4-bit NF4 decoder weights with double-quantised scales, the `load_4bit` path of model/builder.py:37-44 (bitsandbytes
 * NF4 + double quantisation there; the format is defined in cambrian_b200/quant.py).  Blocks of 64 row-major elements of
 * one Linear weight W [N, K] (K % 64 == 0); packed [N, K/2] uint8 codes (element 2j in the high nibble), qabsmax [N*K/64]
 * uint8 indices into the signed dynamic map, absmax2 [ceil(N*K/64 / 256)] fp32 group scales, offset [1] fp32.
 * Dequantised weight: w~ = bf16(c[code] * (map[qabsmax] * absmax2 + offset)), no FMA contraction.
 *
 * cb_nf4_quantize: quantise one bf16 W [N, K] on the device; absmax_ws is caller-provided fp32 scratch of >= N*K/64
 * floats.  Deterministic (fixed-order reductions), no host synchronisation. */
int cb_nf4_quantize(const void* w, int N, int K, float* absmax_ws, int64_t ws_floats, void* packed, void* qabsmax,
                    float* absmax2, float* offset, void* stream);
/* Decode-shaped projection on NF4 weights, M <= 8 rows: y[M,N] = x[M,K] W~[N,K]^T (+ bias[N]) (+ residual[M,N]), y bf16 or
 * fp32, fp32 accumulation — the NF4 counterpart of cb_gemv_bf16 for the KV-cache decode step.  W~ may be a fused
 * projection (q|k|v, gate|up) of up to 3 separately quantised row segments: HOST arrays of nseg entries, segment i covers
 * rows [seg_row0[i], seg_row0[i+1]) (seg_row0[0] = 0) and carries its own packed / qabsmax / absmax2 / offset. */
int cb_gemv_nf4(const void* x, void* y, int M, int N, int K, int64_t ldx, int64_t ldy, int nseg, const int32_t* seg_row0,
                const void* const* packed, const void* const* qabsmax, const void* const* absmax2, const void* const* offset,
                const void* bias, const void* residual, int64_t ldr, int out_fp32, void* stream);
/* W~ of a segmented NF4 weight (same segment table as cb_gemv_nf4) written as bf16 [N, K] into caller-provided scratch,
 * bitwise equal to the definition above: the larger-batch path runs the bf16 GEMM on it. */
int cb_nf4_dequant(void* out, int N, int K, int nseg, const int32_t* seg_row0, const void* const* packed,
                   const void* const* qabsmax, const void* const* absmax2, const void* const* offset, void* stream);
/* 8-bit LLM.int8 decoder weights, the `load_8bit` path of model/builder.py:35-36 (bitsandbytes LLM.int8 with
 * llm_int8_threshold = 6.0 there; the format and the exact order of the epilogue are defined in
 * cambrian_b200/quant_int8.py).  Per-row absmax scales on both sides, K % 16 == 0:
 *   weight:     scb[n] = max |W[n,:]|, cb[n,k] = clamp(rint(W[n,k] * (127 / scb[n])), -127, 127), int8 [N, K];
 *   activation: outlier columns O = { j : max_m |x[m,j]| >= threshold } (none when threshold <= 0), sca[m] = max |x[m,j]|
 *               over j not in O, xq[m,j] = rint(x[m,j] * (127 / sca[m])) off O and 0 on O, int8 [M, K];
 *   output:     y = (float(sum xq cb) * (sca * scb)) * (1/16129) + sum_{j in O, ascending} x[m,j] * (float(cb[n,j]) *
 *               (scb[n] * (1/127))) (+ bias[n]) (+ residual[m,n]), every operation rounded on its own (no FMA).
 *
 * cb_int8_quantize_weight: one bf16 W [N, K] (row stride ldw) -> cb (row stride K), scb; deterministic, no host sync. */
int cb_int8_quantize_weight(const void* w, int N, int K, int64_t ldw, void* cb, float* scb, void* stream);
/* x [M, K] bf16 (row stride ldx) -> xq [M, K] int8, sca [M] fp32, outlier_idx [<= K] int32 ascending, n_outlier [1]
 * int32 on the device; colmax_ws is caller-provided scratch of K uint32.  No host synchronisation (graph-capturable). */
int cb_int8_quantize_act(const void* x, int M, int K, int64_t ldx, float threshold, void* xq, float* sca,
                         uint32_t* colmax_ws, int32_t* outlier_idx, int32_t* n_outlier, void* stream);
/* y[M,N] (bf16 or fp32, row stride ldy) from the quantised activation (xq, sca, outliers; x is the bf16 activation it
 * came from) and weight (cb, scb) — M <= 8 rows (decode): CUDA-core dp4a GEMV; any M: int8 tensor-core GEMM
 * (wgmma .s32.s8.s8).  Both are bitwise equal to the definition above, so to each other. */
int cb_gemv_int8(const void* xq, const void* cb, const float* sca, const float* scb, const void* x, int64_t ldx,
                 const int32_t* outlier_idx, const int32_t* n_outlier, void* y, int M, int N, int K, int64_t ldy,
                 const void* bias, const void* residual, int64_t ldr, int out_fp32, void* stream);
int cb_gemm_int8(const void* xq, const void* cb, const float* sca, const float* scb, const void* x, int64_t ldx,
                 const int32_t* outlier_idx, const int32_t* n_outlier, void* y, int M, int N, int K, int64_t ldy,
                 const void* bias, const void* residual, int64_t ldr, int out_fp32, void* stream);
/* FP8 E4M3 decoder weights for inference (`load_fp8`).  The reference has no FP8 path: these replace the same seven
 * decoder projections as the two entries above (`F.linear` in the LlamaDecoderLayer that model/builder.py:29-175 builds),
 * with the format and the exact order of the epilogue defined in cambrian_b200/quant_fp8.py.  Per-row scales on both
 * sides, K % 16 == 0; the same rule quantises a weight row at load and an activation row per call:
 *   s = amax / 448, r = min(448 / amax, FLT_MAX), q[k] = e4m3_rn_satfinite(v[k] * r)   (every operation fp32-rounded);
 *   output: y = acc * (sa[m] * sw[n]) (+ bias[n]) (+ residual[m,n]), acc = sum_k xq[m,k] * wq[n,k] in fp32, every
 *   128-deep k-block summed on the tensor cores on its own and added in fp32 registers.
 *
 * cb_fp8_quantize_weight: one bf16 W [N, K] (row stride ldw) -> wq e4m3 [N, K] (row stride K), sw fp32 [N];
 * deterministic, no host sync. */
int cb_fp8_quantize_weight(const void* w, int N, int K, int64_t ldw, void* wq, float* sw, void* stream);
/* x [M, K] bf16 (row stride ldx) -> xq e4m3 [M, K], sa fp32 [M]: one pass per row, no atomics, no host synchronisation
 * (graph-capturable). */
int cb_fp8_quantize_act(const void* x, int M, int K, int64_t ldx, void* xq, float* sa, void* stream);
/* y[M,N] (bf16 or fp32, row stride ldy) from the quantised activation (xq, sa) and weight (wq, sw) — M <= 8 rows
 * (decode): wgmma m64n8k32 with W as the A operand, K split over a thread-block cluster and reduced in rank order; any
 * M: tensor-core GEMM (wgmma m64n128k32 .f32.e4m3.e4m3).  Both deterministic run to run; their summation orders
 * differ, so they agree to fp32 accumulation error, not bit for bit. */
int cb_gemv_fp8(const void* xq, const void* wq, const float* sa, const float* sw, void* y, int M, int N, int K,
                int64_t ldy, const void* bias, const void* residual, int64_t ldr, int out_fp32, void* stream);
int cb_gemm_fp8(const void* xq, const void* wq, const float* sa, const float* sw, void* y, int M, int N, int K,
                int64_t ldy, const void* bias, const void* residual, int64_t ldr, int out_fp32, void* stream);
/* FP8 E4M3 decode KV cache (`generate(..., kv_cache_dtype="fp8")`; the format and the decode arithmetic are defined in
 * cambrian_b200/kv_fp8.py).  The reference keeps HF's bf16 DynamicCache behind LlamaSdpaAttention (the decode steps of
 * cambrian_llama.py:437-483 through GenerationMixin.generate); these replace its cache update and the decode-step SDPA.
 * Per layer: kq, vq e4m3 [B, S_max, nkv, hd] and ks, vs fp32 [B, S_max, nkv]; every (sequence, position, kv head) row of
 * K or V is quantised by the cb_fp8_quantize_act rule (s = amax / 448, q = e4m3_rn_satfinite(x * r)).  hd 64 or 128.
 *
 * cb_kv_fp8_append: the new rows k, v (element (b, s, h, d) at base + (b * S + s) * ld + h * hd + d: the K and V heads of
 * the packed post-RoPE qkv rows, read in place) go to positions offset + s, plus *offset_dev when offset_dev is not NULL
 * (the device write slot of the graph-replayed decode step; a position past S_max is then skipped). */
int cb_kv_fp8_append(const void* k, const void* v, int64_t ld, void* kq, void* vq, float* ks, float* vs, int B, int S,
                     int S_max, int nkv, int hd, int64_t offset, const int64_t* offset_dev, void* stream);
/* fp32 workspace cb_attn_decode_fp8 needs for this shape on the current device (0: one split, no workspace) */
int64_t cb_attn_decode_fp8_workspace_floats(int B, int nh, int nkv, int S_max, int hd);
/* Decode attention over the FP8 cache (flash-decoding), one query per sequence (Sq == 1): q element (b, h, d) at
 * q + b * q_bs + h * hd + d (a view of the packed qkv row), o [B, nh, hd] bf16 contiguous.  Valid keys: positions below
 * length (+ *length_dev when not NULL), clipped to S_max, and with kmask [B, kmask_ld] (1 byte, 1 = attend; may be NULL)
 * set.  One CTA per (key split, kv head, sequence) serves the nh / nkv (1..8) query heads of that kv head, so each cache
 * byte is read once per call, and only below the valid length.  The split count is a function of (B, nkv, S_max, SM
 * count); with more than one split the partial results are merged in split order through `workspace` (no atomics):
 * bit-identical from run to run. */
int cb_attn_decode_fp8(const void* q, int64_t q_bs, const void* kq, const void* vq, const float* ks, const float* vs,
                       const void* kmask, int64_t kmask_ld, void* o, float* workspace, int64_t workspace_floats, int B, int Sq,
                       int nh, int nkv, int S_max, int hd, int64_t length, const int64_t* length_dev, float scale,
                       void* stream);
/* FP8 E4M3 training of the decoder projections (`config.fp8_training`; the format is defined in
 * cambrian_b200/train_fp8.py).  The four forward GEMMs (y = x W^T) and the four input-gradient GEMMs (dx = dy W) of a
 * decoder layer run on cb_gemm_fp8 with the row rule above; the weight-gradient GEMMs stay bf16.  Every scale is constant
 * along the reduction dimension: per token on the activation / gradient side, per row of W in forward and per row of
 * W^T (per input column of W) in the input-gradient GEMM.
 *
 * cb_fp8_quantize_weight_t: bf16 W [N, K] (row stride ldw) -> wtq e4m3 [K, N] (row stride N), st fp32 [K], bit for bit
 * cb_fp8_quantize_weight of W^T; N % 16 == 0, K % 16 == 0.  Column maxima go through `workspace` (at least
 * cb_fp8_quantize_weight_t_workspace_floats(N, K) floats on the current device); no atomics. */
int64_t cb_fp8_quantize_weight_t_workspace_floats(int N, int K);
int cb_fp8_quantize_weight_t(const void* w, int N, int K, int64_t ldw, void* wtq, float* st, float* workspace,
                             int64_t workspace_floats, void* stream);
/* cb_rmsnorm_fwd with an E4M3 output: y is computed and rounded to bf16 as cb_rmsnorm_fwd does, then quantised per row
 * into xq e4m3 [rows, C] and sa fp32 [rows]; rstd [rows] as cb_rmsnorm_fwd writes it (may be NULL).  Bit for bit
 * cb_fp8_quantize_act(cb_rmsnorm_fwd(x)).  C % 16 == 0. */
int cb_rmsnorm_fwd_fp8(const void* x, const void* gamma, void* xq, float* sa, float* rstd, int64_t rows, int C, float eps,
                       int hf_cast, void* stream);
/* cb_swiglu_bwd with a second output: dgate / dup bf16 exactly as cb_swiglu_bwd writes them, plus dguq e4m3 [rows, 2I]
 * (contiguous; dgate in columns [0, I), dup in [I, 2I)) and sdgu fp32 [rows] by the row rule over the whole [dgate | dup]
 * row: bit for bit cb_fp8_quantize_act of the [rows, 2I] gradient.  I % 8 == 0; one CTA per row, no atomics. */
int cb_swiglu_bwd_fp8(const void* dout, const void* gate, const void* up, void* dgate, void* dup, void* dguq, float* sdgu,
                      int64_t rows, int I, int64_t ld_in, int64_t ld_dout, int64_t ld_dgu, void* stream);
/* Paged decode KV cache for continuous batching (cambrian_b200/serving.py; the format is defined in
 * cambrian_b200/paged_kv.py).  The reference serves many requests at once through SGLang (serve/sglang_worker.py) and
 * keeps HF's per-call cache behind LlamaSdpaAttention (the cache update and decode-step SDPA of cambrian_llama.py:437-483
 * through GenerationMixin.generate); these replace that cache update and decode SDPA for a batch of independent
 * sequences.  Per layer K and V pages [num_pages, page_size, nkv, hd] (position-major inside a page), bf16 (fp8 == 0) or
 * e4m3 with fp32 scales [num_pages, page_size, nkv] by the row rule of cb_kv_fp8_append (fp8 == 1).  block_table int32
 * [rows, table_ld]: entry (b, p) is the page holding positions [p * page_size, (p + 1) * page_size) of row b (only the
 * first max_pages columns are read).  lens int32 [rows]: row b's cached length; a negative length marks an inactive
 * (padding) row.  page_size is a power of two >= 16; hd 64 or 128.  A table entry outside [0, num_pages) is skipped.
 *
 * cb_paged_kv_append: the new rows k, v (element (b, s, h, d) at base + (b * S + s) * ld + h * hd + d: the K and V heads
 * of the packed post-RoPE qkv rows, read in place) go to position offset + s, plus lens[b] when offset_from_lens (the
 * graph-replayed decode step).  lens may be NULL when !offset_from_lens; an inactive row writes nothing.  FP8 pages get
 * bit for bit the bytes and scales cb_kv_fp8_append writes for the same rows. */
int cb_paged_kv_append(const void* k, const void* v, int64_t ld, void* k_pages, void* v_pages, float* k_scales,
                       float* v_scales, int fp8, const int* block_table, int64_t table_ld, const int* lens, int rows, int S,
                       int nkv, int hd, int page_size, int num_pages, int max_pages, int64_t offset, int offset_from_lens,
                       void* stream);
/* fp32 workspace cb_attn_decode_paged needs: rows * nh * ceil(max_pages * page_size / 256) * (hd + 2) */
int64_t cb_attn_decode_paged_workspace_floats(int rows, int nh, int max_pages, int page_size, int hd);
/* Decode attention over the pages (flash-decoding), one query per row: q element (b, h, d) at q + b * q_bs + h * hd + d
 * (a view of the packed qkv row), o [rows, nh, hd] bf16 contiguous.  Valid keys of row b: positions below
 * lens[b] + len_add (len_add = 1 counts the row appended just before).  One CTA per (key split, kv head, row) serves the
 * nh / nkv (1..8) query heads of that kv head, so each cached byte is read once per call, and only below the valid
 * length.  Every split covers 256 key positions, independent of rows, bucket and SM count; the grid is sized from
 * max_pages and splits past a row's length exit.  Partials are merged in split order through `workspace` (no atomics),
 * so a row's output is bitwise independent of the other rows of the launch.  bf16 pages: scores and the PV sum in fp32,
 * one rounding to bf16; FP8 pages: the decode arithmetic of cb_attn_decode_fp8.  A row of length <= 0 gets zeros. */
int cb_attn_decode_paged(const void* q, int64_t q_bs, const void* k_pages, const void* v_pages, const float* k_scales,
                         const float* v_scales, int fp8, const int* block_table, int64_t table_ld, const int* lens,
                         int len_add, void* o, float* workspace, int64_t workspace_floats, int rows, int nh, int nkv, int hd,
                         int page_size, int num_pages, int max_pages, float scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CAMBRIAN_B200_H */
