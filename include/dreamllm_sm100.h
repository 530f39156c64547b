/* libdreamllm_sm100.so — C ABI of the H100-native (sm_90a) DreamLLM hot path.
 *
 * The reference (RunpeiDong/DreamLLM) is pure Python and has no FFI of its own (SURVEY.md §8b); these entry points
 * are what a ctypes / cffi binding inside `omni/models/dreamllm` calls in place of the torch ops the reference
 * issues.  Each function cites the reference call site it replaces
 * (paths relative to /root/reference/omni/models/dreamllm/).
 *
 * Conventions: plain device pointers + sizes, no torch types; bf16 unless noted; row-major; `ld*` = row stride in
 * ELEMENTS; every call is asynchronous on `stream` (a cudaStream_t passed as void*), allocates nothing, never
 * synchronises; returns 0 or a negative DLLM_ERR_* code.  Thread-safe for distinct streams.
 */
#ifndef DREAMLLM_SM100_H
#define DREAMLLM_SM100_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define DLLM_OK 0
#define DLLM_ERR_SHAPE (-1)
#define DLLM_ERR_ALIGN (-2)
#define DLLM_ERR_DRIVER (-3)
#define DLLM_ERR_TMAP (-4)
#define DLLM_ERR_LAUNCH (-5)
#define DLLM_ERR_UNSUPPORTED (-6)

int dllm_version(void);
const char* dllm_error_string(int code);
/* Leave `n` SMs out of the persistent GEMM grids (for an overlapped NCCL all-reduce; data-parallel training only). */
int dllm_set_reserved_sms(int n);
int dllm_get_reserved_sms(void);

/* Dense contraction on wgmma tensor cores: C[M,N] = op(A) * op(B), fp32 accumulate in registers.
 *   a_mn = 0: A is [M,K] row-major; a_mn = 1: A is stored [K,M] row-major (i.e. A^T, used for wgrad)
 *   b_mn = 0: B is [N,K] row-major (an nn.Linear weight); b_mn = 1: B is stored [K,N] row-major
 *   out_fp32: C dtype (0 = bf16, 1 = fp32).  cta_pair: accepted for compatibility, no effect (one CTA per tile).
 * Replaces F.linear / nn.Linear and their autograd dgrad/wgrad:
 *   modeling_dreamllm.py:336-338, :395 (q/k/v/o_proj), :237 (gate/up/down_proj), :1452 (lm_head),
 *   omni/models/projector/mlp_projector.py:11-50 (projectors). */
int dllm_gemm_bf16(const void* A, const void* B, void* C, int M, int N, int K, long lda, long ldb, long ldc,
                   int a_mn, int b_mn, int out_fp32, int cta_pair, void* stream);

/* DreamLLMRMSNorm.forward (modeling_dreamllm.py:86-91), optionally fused with the preceding residual add
 * (:638, :644): if `add` != NULL, x_out = bf16(x + add) is written and normalised.  rstd[T] (fp32) is saved for bwd. */
int dllm_rmsnorm_fwd(const void* x, const void* add, const void* weight, void* x_out, void* y, float* rstd, int T,
                     int H, float eps, void* stream);
size_t dllm_rmsnorm_bwd_workspace_bytes(int T, int H);
/* dx = d(norm)/dx (+ dres if != NULL); dweight (=|+=) column sums (bf16). */
int dllm_rmsnorm_bwd(const void* dy, const void* x, const void* weight, const float* rstd, const void* dres, void* dx,
                     void* dweight, int dweight_accumulate, void* workspace, size_t workspace_bytes, int T, int H,
                     void* stream);

/* apply_rotary_pos_emb (modeling_dreamllm.py:184-209) in place on `heads_total` heads laid side by side in a
 * [T, ld] buffer (q and k blocks of the fused qkv projection); cos/sin tables [max_pos, head_dim] bf16 (:126-127),
 * pos[T] int32.  mode = +1 forward, -1 backward. */
int dllm_rope_inplace(void* buf, const void* cos_table, const void* sin_table, const int* pos, long ld, int T,
                      int heads_total, int head_dim, int mode, void* stream);

/* DreamLLMMLP activation (modeling_dreamllm.py:237): act = silu(gate) * up on the fused [T, 2I] gate|up buffer. */
int dllm_swiglu_fwd(const void* gate_up, void* act, long ld_gate_up, int T, int I, void* stream);
int dllm_swiglu_bwd(const void* dact, const void* gate_up, void* dgate_up, long ld_gate_up, int T, int I, void* stream);

int dllm_add_bf16(const void* a, const void* b, void* out, long n, void* stream);

/* Shifted masked-mean cross entropy (modeling_dreamllm.py:1453-1470). labels[T] int64, already shifted, -100 =
 * ignore. loss[1] fp32.  If write_grad, logits are overwritten in place by dloss * d(loss)/d(logits) (bf16).
 * workspace: (T + 2) floats. */
int dllm_cross_entropy(void* logits, const long long* labels, float* loss, float dloss, void* workspace, long ld,
                       int T, int V, int write_grad, void* stream);

/* embed_tokens lookup (modeling_dreamllm.py:1066-1067) and its deterministic gradient (sorted segment sums). */
int dllm_embedding_fwd(const long long* ids, const void* weight, void* out, int T, int H, void* stream);
int dllm_embedding_bwd(const long long* sorted_ids, const long long* order, const void* dy, void* dweight, int T,
                       int H, int accumulate, void* stream);

/* Causal / full flash attention on wgmma tensor cores (replaces flash_attn_func / flash_attn_varlen_func,
 * modeling_dreamllm.py:500-551, and the eager path :357-379).
 * q,k,v: [B, S, nh, d] views with row stride ld_qkv (elements) between consecutive tokens — the fused qkv GEMM
 * output is consumed directly, no transposes.  out: [B, S, nh*d] (ld_o).  lse: [B, nh, S] fp32.
 * seqlens: int32[B] valid (right-padded) lengths or NULL.  Rows >= seqlens[b] are written as zeros (pad_input). */
int dllm_attn_fwd(const void* q, const void* k, const void* v, void* out, float* lse, const int* seqlens, int B,
                  int S, int nh, int d, long ld_qkv, long ld_o, int causal, float scale, void* stream);
size_t dllm_attn_bwd_workspace_bytes(int B, int S, int nh, int d);
int dllm_attn_bwd(const void* dout, const void* q, const void* k, const void* v, const void* out, const float* lse,
                  void* dq, void* dk, void* dv, const int* seqlens, void* workspace, size_t workspace_bytes, int B,
                  int S, int nh, int d, long ld_qkv, long ld_o, long ld_dqkv, int causal, float scale, void* stream);

/* GEMM with fused epilogue: out = act(bf16(acc + bias[col])) (+ residual[row, col]); act 0 none, 1 quick_gelu
 * (CLIP MLP, transformers activations.QuickGELU), 2 gelu-erf (MLPProjector, mlp_projector.py:30-50), 3 silu.
 * Replaces nn.Linear(bias=True) + activation + residual add in the CLIP tower / projectors / UNet transformer blocks. */
int dllm_gemm_bf16_ex(const void* A, const void* B, void* C, int M, int N, int K, long lda, long ldb, long ldc,
                      int a_mn, int b_mn, int out_fp32, int cta_pair, const void* bias, const void* residual, long ldr,
                      int act, void* stream);

/* nn.LayerNorm forward (CLIP layer_norm1/2 + pre_layrnorm, modeling_plugins.py:321 -> transformers CLIPVisionModel). */
int dllm_layernorm_fwd(const void* x, const void* weight, const void* bias, void* y, int T, int H, float eps, void* stream);

/* CLIP patch embedding (Conv2d k=s=patch, no bias) as unfold + GEMM, and CLS/position-embedding assembly. */
int dllm_clip_patchify(const void* images_nchw, void* out, int N, int R, int patch, int Kpad, void* stream);
int dllm_clip_assemble(const void* patches, const void* cls, const void* pos, void* out, int N, int P, int C, void* stream);

/* Index-driven row copies: the embedding splice of DreamLLMModel.forward (modeling_dreamllm.py:1082-1141) and the
 * dream-query conditioning gather (:1401-1418).  mode 0: dst[dst_idx[r]] = src[src_idx[r]]; mode 1: += (unique dst). */
int dllm_copy_rows(void* dst, const int* dst_idx, const void* src, const int* src_idx, int R, int H, int mode, void* stream);
int dllm_segment_sum_rows(void* dst, const void* src, const int* seg, const int* rows, int Q, int H, void* stream);
int dllm_zero_rows(void* dst, const int* idx, int R, int H, void* stream);

/* ---- Stable-Diffusion-2.1 UNet denoising step (reference: StableDiffusionHead.pipeline, modeling_plugins.py:809-833;
 * arithmetic = diffusers 0.24 UNet2DConditionModel / DDPMScheduler / DDIM, restated in oracle/unet_oracle.py). NHWC bf16. ---- */

/* attention with separate kv length (UNet cross-attention on the dream-query conditioning: Skv = 64 / 77). */
int dllm_attn_fwd_ex(const void* q, const void* k, const void* v, void* out, float* lse, const int* seqlens, int B, int Sq,
                     int Skv, int nh, int d, long ld_q, long ld_kv, long ld_o, int causal, float scale, void* stream);
/* kv-cache attention (reference :344-355, :444-449 concat past k/v): k/v live in a preallocated [B, kv_rows, nh*d] cache with Skv valid
 * rows; causal uses the bottom-right aligned mask (query i is at absolute position Skv - Sq + i). */
int dllm_attn_fwd_cache(const void* q, const void* k, const void* v, void* out, float* lse, int B, int Sq, int Skv, int kv_rows, int nh,
                        int d, long ld_q, long ld_kv, long ld_o, int causal, float scale, void* stream);
/* same, for a PADDED prompt batch held in the cache: kv_mask [B, mask_ld] bytes, 0 = pad key (the 2-D `attention_mask` HF `generate` keeps
 * extending, modeling_dreamllm.py:1511-1547; the reference's flash path drops those tokens with `_upad_input`, :553-583).  Pad QUERY rows
 * whose keys are all masked come back as zeros, as `pad_input` re-inserts them (:545).  mask_ld % 16 == 0, >= round_up(Skv, 64). */
int dllm_attn_fwd_cache_mask(const void* q, const void* k, const void* v, void* out, float* lse, const void* kv_mask, int mask_ld, int B,
                             int Sq, int Skv, int kv_rows, int nh, int d, long ld_q, long ld_kv, long ld_o, int causal, float scale,
                             void* stream);
/* grouped-query attention (reference repeat_kv, modeling_dreamllm.py:242-252; flash_attn_func takes the narrow K/V directly, :485):
 * k, v: [B, kv_rows, nkv, d] with nkv dividing nh; q head h attends with kv head h / (nh / nkv).  Covers every case of the forward
 * entries above: cache rows (kv_rows >= Skv), right-padded `seqlens` (NULL = none) and the cache key mask `kv_mask` (NULL = none).
 * nkv == nh is multi-head attention, and the entries above are exactly that call.  nkv <= 0 or nh % nkv != 0: invalid shape. */
int dllm_attn_fwd_gqa(const void* q, const void* k, const void* v, void* out, float* lse, const int* seqlens, const void* kv_mask,
                      int mask_ld, int B, int Sq, int Skv, int kv_rows, int nh, int nkv, int d, long ld_q, long ld_kv, long ld_o, int causal,
                      float scale, void* stream);
/* Attention probabilities of dllm_attn_fwd_gqa (output_attentions, the eager path's weights, modeling_dreamllm.py:357-378): probs is a
 * dense bf16 [B, nh, Sq, Skv] (row stride Skv, 16-byte aligned base), lse the [B, nh, Sq] output of the dllm_attn_fwd_gqa call with the
 * same q, k, masks and shapes.  Every element is written: masked keys are 0, a right-padded query row (row >= seqlens[b]) is a softmax
 * over the sample's keys < seqlens[b], a row with no visible key is uniform 1/Skv.  Same shape / alignment rules as dllm_attn_fwd_gqa. */
int dllm_attn_probs_gqa(const void* q, const void* k, const float* lse, void* probs, const int* seqlens, const void* kv_mask, int mask_ld,
                        int B, int Sq, int Skv, int kv_rows, int nh, int nkv, int d, long ld_q, long ld_kv, int causal, float scale,
                        void* stream);
/* backward of dllm_attn_fwd_gqa (no kv-cache): dk, dv are [B, Skv, nkv, d] (token stride ld_dkv); the gradient of kv head hk is the sum
 * over its group of q heads, in a fixed order (bitwise repeatable).  Workspace: dllm_attn_bwd_workspace_bytes(B, Sq, nh, d). */
int dllm_attn_bwd_gqa(const void* dout, const void* q, const void* k, const void* v, const void* out, const float* lse, void* dq,
                      void* dk, void* dv, const int* seqlens, void* workspace, size_t workspace_bytes, int B, int Sq, int Skv, int nh,
                      int nkv, int d, long ld_q, long ld_kv, long ld_o, long ld_dq, long ld_dkv, int causal, float scale, void* stream);
/* Packed (unpadded) batches, the layout of flash_attn_varlen_func (reference modeling_dreamllm.py:532, :553-583): B samples laid end to
 * end as T = sum(len_b) tokens.  q: [T, nh, d], k, v: [T, nkv, d] views (token strides ld_q / ld_kv), out: [T, nh*d] (ld_o), lse:
 * [nh, T] fp32.  cu_seqlens: device int32 [B + 1], non-decreasing, cu[0] = 0, cu[B] = T; sample b owns rows cu[b] .. cu[b+1] - 1 and
 * attends only to itself (zero-length samples are legal).  max_seqlen (host) bounds every length and sizes the grid.  cu_seqlens and
 * max_seqlen are trusted: validate them on the host.  Every row of out / lse is written exactly once, and the rows of sample b equal,
 * bit for bit, dllm_attn_fwd_gqa on that sample alone (B = 1, Sq = Skv = len_b).  NULL cu_seqlens, max_seqlen <= 0 or > T: invalid
 * shape. */
int dllm_attn_fwd_varlen(const void* q, const void* k, const void* v, void* out, float* lse, const int* cu_seqlens, int B, int T,
                         int max_seqlen, int nh, int nkv, int d, long ld_q, long ld_kv, long ld_o, int causal, float scale, void* stream);
/* backward of dllm_attn_fwd_varlen: dq [T, nh, d] (ld_dq), dk, dv [T, nkv, d] (ld_dkv), each row written exactly once; deterministic, and
 * bit-identical per sample to dllm_attn_bwd_gqa on that sample alone.  The workspace holds delta and lse * log2(e) as two [nh, T_pad]
 * fp32 planes, T_pad = round_up(T, 64) + 64 (the backward reads whole 64-row tiles: the slack after row T is written as zeros). */
size_t dllm_attn_bwd_varlen_workspace_bytes(int T, int nh, int d);
int dllm_attn_bwd_varlen(const void* dout, const void* q, const void* k, const void* v, const void* out, const float* lse, void* dq,
                         void* dk, void* dv, const int* cu_seqlens, void* workspace, size_t workspace_bytes, int B, int T, int max_seqlen,
                         int nh, int nkv, int d, long ld_q, long ld_kv, long ld_o, long ld_dq, long ld_dkv, int causal, float scale,
                         void* stream);
/* ResnetBlock2D / Upsample2D conv: implicit-GEMM 3x3 stride-1 pad-1 on wgmma tensor cores (4-D TMA im2col, zero-fill padding).
 * y = conv(x, w) + bias[c] + rowbias[n, c] (+ residual);  w is [Cout, 3, 3, Cin]. */
int dllm_conv3x3_nhwc(const void* x, const void* w, void* y, int N, int H, int W, int Cin, int Cout, const void* bias,
                      const void* rowbias, const void* residual, void* stream);
size_t dllm_groupnorm_workspace_bytes(int N, int HW, int G);
int dllm_groupnorm_nhwc(const void* x, const void* w, const void* b, void* y, void* workspace, size_t ws_bytes, int N, int HW,
                        int C, int G, float eps, int silu, void* stream);
int dllm_geglu(const void* in, void* out, int T, int I, void* stream);
int dllm_upsample2x_nhwc(const void* x, void* y, int N, int H, int W, int C, void* stream);
/* pad = 1: UNet Downsample2D; pad = 0: VAE downsample (F.pad (0,1,0,1) + padding-0 conv) */
int dllm_im2col_s2_nhwc(const void* x, void* out, int N, int H, int W, int C, int pad, void* stream);
int dllm_copy_cols(const void* src, void* dst, long rows, int Cs, int Cd, int col0, void* stream);
/* latents x_nchw [Bsrc,Cin,H,W] fp32 -> y_nhwc [B,H,W,Cout]; image n reads latents[n % Bsrc] (CFG duplication, plugins:811) */
int dllm_conv_in(const float* x_nchw, const void* w, const void* bias, void* y_nhwc, int B, int Bsrc, int Cin, int H, int W, int Cout,
                 void* stream);
int dllm_conv_out(const void* x_nhwc, const void* w, const void* bias, float* y_nchw, int B, int C, int H, int W, int Cout, void* stream);
/* Split-K forms for small-M shapes (stage-1 steps run the UNet on 4 samples: an 8x8 plane is 256 GEMM rows and would occupy 5 of 74 CTA
 * pairs).  `*_workspace_bytes` returns 0 when the shape is not worth splitting; otherwise pass that many bytes of 16-byte aligned scratch:
 * the GEMM writes fp32 K-slice partials there and a reduce kernel applies bias / row-group bias / activation / residual with the fused
 * epilogue's rounding points.  C = act(bf16(A B^T + bias)) (+ residual) for b_mn = 0 (nn.Linear forward), C = A B for b_mn = 1 (dgrad). */
size_t dllm_gemm_splitk_workspace_bytes(int M, int N, int K);
/* N-tile width (128, 160, 192, 224 or 256) that dllm_gemm_bf16_ws uses for this shape when given its workspace: the split-K width when
 * the shape is split, otherwise the width the tile planner picks (b_mn = 1 is the dgrad NN form).  Pure host code. */
int dllm_gemm_tile_n(int M, int N, int K, int b_mn);
int dllm_gemm_bf16_ws(const void* A, const void* B, void* C, int M, int N, int K, long lda, long ldb, long ldc, int b_mn, const void* bias,
                      const void* residual, long ldr, int act, void* ws, size_t ws_bytes, void* stream);
size_t dllm_conv3x3_splitk_workspace_bytes(int N, int H, int W, int Cin, int Cout);
int dllm_conv3x3_nhwc_ws(const void* x, const void* w, void* y, int N, int H, int W, int Cin, int Cout, const void* bias,
                         const void* rowbias, const void* residual, void* ws, size_t ws_bytes, void* stream);
/* UNet FeedForward-in projection with GEGLU in the GEMM epilogue (diffusers `GEGLU.forward`: h, gate = proj(x).chunk(2); h * gelu(gate)):
 * out[M, N/2] = h * gelu(gate) where [h | gate] = A @ W^T + b and Wp / bias_p hold W / b with rows permuted to [64 h rows | 64 gate rows]
 * per 128-row group; the [M, N] projection is never written.  N % 128 == 0. */
int dllm_gemm_bf16_geglu(const void* A, const void* Wp, const void* bias_p, void* out, int M, int N, int K, long lda, long ldb, long ldc,
                         void* stream);
/* tensor-core forms of the two tiny-channel convolutions (conv_in: Conv2d(4|3, C, 3, pad 1) of UNet2DConditionModel / AutoencoderKL;
 * conv_out: Conv2d(C, 4|8|3, 3, pad 1)):
 *   cols [B*H*W, 64] bf16 = im2col(x_nchw fp32), k = (c*3 + r)*3 + s zero-padded to 64  ->  dllm_gemm_bf16_ex(cols, Wk [Cout, 64], bias)
 *   y8 [N*H*W, 8] bf16 = dllm_conv3x3_nhwc(x, W8 [8, 9*C])                                ->  out fp32 NCHW [N, Cout, H*W] (first Cout channels) */
int dllm_im2col_in(const float* x_nchw, void* cols, int B, int Bsrc, int Cin, int H, int W, void* stream);
int dllm_nhwc_to_nchw_f32(const void* y_nhwc8, float* out_nchw, int N, int HW, int Cp, int Cout, void* stream);
/* timestep = timesteps[*step] (device-side schedule so one captured CUDA graph serves every step) */
int dllm_timestep_embedding(const int* timesteps, const int* step, void* out, int B, int dim, void* stream);
int dllm_timestep_embedding_batch(const int* t_per_sample, void* out, int B, int dim, void* stream);
/* fused CFG combine + DDIM (mode 0) / DDPM (mode 1) update; coef[step] = {sqrt(a_t), sqrt(1-a_t), c_x0, c_eps|c_xt, sigma};
 * advances *step. */
int dllm_sampler_step(const float* eps, float* latents, const float* noise, const float* coef, int* step, float guidance,
                      int use_cfg, int mode, long n, void* stream);

/* ---- input-gradient (dgrad-only) backward of the frozen UNet + diffusion loss plumbing: StableDiffusionHead.forward,
 * modeling_plugins.py:493-577 (add_noise :536, unet(...) :556, MSE :559). ---- */
int dllm_attn_bwd_ex(const void* dout, const void* q, const void* k, const void* v, const void* out, const float* lse, void* dq,
                     void* dk, void* dv, const int* seqlens, void* workspace, size_t workspace_bytes, int B, int Sq, int Skv, int nh,
                     int d, long ld_q, long ld_kv, long ld_o, long ld_dq, long ld_dkv, int causal, float scale, void* stream);
int dllm_groupnorm_stats(const void* x, float* stats, void* workspace, size_t ws_bytes, int N, int HW, int C, int G, float eps, void* stream);
int dllm_groupnorm_apply(const void* x, const void* w, const void* b, const float* stats, void* y, int N, int HW, int C, int G, int silu,
                         void* stream);
int dllm_groupnorm_bwd_nhwc(const void* dy, const void* x, const void* w, const void* b, const float* stats, const void* dres, void* dx,
                            void* workspace, size_t ws_bytes, int N, int HW, int C, int G, int silu, void* stream);
int dllm_layernorm_bwd(const void* dy, const void* x, const void* w, const void* dres, void* dx, int T, int H, float eps, void* stream);
/* ---- CLIP vision tower training (freeze_clip_vision_model=False / freeze_embedding_layers=False, modeling_plugins.py:248-257) ----
 * LayerNorm backward with the affine gradients: dx (+ dres) exactly as dllm_layernorm_bwd computes it (same bits), and
 * dgamma[h] = sum_t dy[t, h] * xhat[t, h], dbeta[h] = sum_t dy[t, h] in fp32, written as bf16.  The sums are per-CTA fp32 partials in the
 * caller's workspace (>= dllm_layernorm_bwd_affine_workspace_bytes(T, H)), added in a fixed order: no atomics, the bits depend only on
 * the inputs and (T, H).  H % 8 == 0, H <= 1536; dy, x, w, dres, dx and the workspace 16-byte aligned (dgamma / dbeta are written
 * element by element). */
size_t dllm_layernorm_bwd_affine_workspace_bytes(int T, int H);
int dllm_layernorm_bwd_affine(const void* dy, const void* x, const void* w, const void* dres, void* dx, void* dgamma, void* dbeta,
                              void* workspace, size_t workspace_bytes, int T, int H, float eps, void* stream);
/* y = x * sigmoid(1.702 x) (transformers QuickGELU) and dx = dy * (s + 1.702 x s (1 - s)), s = sigmoid(1.702 x): bf16 in and out, fp32
 * arithmetic, one rounding, n % 8 == 0, 16-byte aligned pointers.  The forward uses the fused GEMM epilogue's formula. */
int dllm_quick_gelu(const void* x, void* y, long n, void* stream);
int dllm_quick_gelu_bwd(const void* dy, const void* x, void* dx, long n, void* stream);
int dllm_geglu_bwd(const void* dout, const void* in, void* din, int T, int I, void* stream);
int dllm_upsample2x_bwd_nhwc(const void* dy, void* dx, int N, int H, int W, int C, void* stream);
int dllm_col2im_s2_nhwc(const void* dcols, void* dx, int N, int H, int W, int C, void* stream);
int dllm_copy_cols2(const void* src, void* dst, long rows, int Cs, int Cd, int scol0, int dcol0, int ncols, void* stream);
int dllm_conv_out_bwd(const float* dy_nchw, const void* w, void* dx_nhwc, int B, int C, int H, int W, int Cout, void* stream);
int dllm_add_noise(const float* x0, const float* noise, const int* t, const float* alphas_cumprod, float* out, int B, long per_sample,
                   void* stream);
int dllm_mse_fwd_bwd(const float* pred, const float* target, float* loss, float* dpred, long n, void* stream);
/* min-SNR weighted MSE (modeling_plugins.py:561-572 with `_compute_snr` :468-491): w_b = min(snr(t_b), gamma) / snr(t_b) */
int dllm_mse_minsnr_fwd_bwd(const float* pred, const float* target, const int* t, const float* alphas_cumprod, float snr_gamma,
                            float* loss, float* dpred, int B, long per_sample, void* stream);

/* ---- VAE encoder helpers (AutoencoderKL.encode(...).latent_dist.sample() * scaling_factor, modeling_plugins.py:511-512) ---- */
int dllm_softmax_rows(void* x, long rows, int cols, float scale, void* stream);
int dllm_vae_sample(const float* h, const void* wq, const void* bq, const float* z, float* out, int B, int L, long plane, float scaling,
                    void* stream);

/* ---- data-parallel optimizer shard (SURVEY §8f row 4) ----
 * Replaces torch.optim.AdamW (`optim="adamw_torch"`, projects/dreamllm/configs/stage1/base.py:85, stage2/base.py:95) applied to this
 * rank's shard of a flat bf16 gradient bucket under FSDP shard_grad_op (stage2/base.py:91-94), with the gradient clipping of
 * omni/train/trainer.py:800-807 folded in: the step scales grads by min(1, max_grad_norm / (sqrt(*grad_sumsq) + 1e-6)) when
 * grad_sumsq != NULL and max_grad_norm > 0 (grad_sumsq = global sum of squares, device pointer, read at kernel time: no host sync).
 * n % 8 == 0, 16-byte aligned pointers.  bf16_state = 0: master / exp_avg / exp_avg_sq are fp32 shards, `param` (bf16) is written from
 * the updated master.  bf16_state = 1: `param`, exp_avg, exp_avg_sq are bf16 and every ATen op of the reference optimizer's
 * single-tensor path rounds to bf16 (bit-for-bit the arithmetic the reference runs on its bf16-loaded model); master is ignored.
 * `step` is the 1-based step count used for the bias corrections.  Hyper-parameters are doubles: Python computes 1 - beta1, lr / (1 - beta1^t)
 * ... in double before ATen narrows them to the fp32 opmath type, and the kernel's scalars are derived the same way. */
int dllm_adamw_step(const void* grad, void* master, void* exp_avg, void* exp_avg_sq, void* param, long n, int bf16_state, double lr,
                    double beta1, double beta2, double eps, double weight_decay, int step, const float* grad_sumsq,
                    double max_grad_norm,
                    void* stream);
/* sum of squares of a bf16 vector in fp32 (deterministic two-stage reduction); *out = (accumulate ? *out : 0) + sum(x^2) */
size_t dllm_sumsq_workspace_bytes(void);
int dllm_sumsq_bf16(const void* x, long n, float* out, int accumulate, void* workspace, size_t workspace_bytes, void* stream);

/* ---- SDXL UNet addition embedding (diffusers UNet2DConditionModel, addition_embed_type "text_time") and the gradient that reaches the
 * pooled conditioning through it: omni/models/dreamllm_sdxl/modeling_plugins.py:197-215 (global_projector(mean(1)), unet(...,
 * added_cond_kwargs)), :344-395 (pipeline). ----
 * out[n, c] = scale * sum_{hw < HW} x[n, hw, c] for x [N, HW, C] bf16 (C % 8 == 0), fp32 accumulate, written as fp32 (out_bf16 = 0) or
 * bf16 into row n of out (row stride ldo >= C elements: a column slice of a wider buffer).  Deterministic: per-CTA partials, then a
 * fixed-order pass, no atomics.  Used for each resnet's time_emb_proj bias gradient (sum over pixels of the conv1 output gradient)
 * and for the mean over the dream queries (scale = 1/Q, bf16: torch.mean's single rounding). */
size_t dllm_channel_sum_workspace_bytes(int N, int HW, int C);
int dllm_channel_sum_nhwc(const void* x, void* out, long ldo, int out_bf16, float scale, int N, int HW, int C, void* workspace,
                          size_t workspace_bytes, void* stream);
/* Timesteps(dim, flip_sin_to_cos=True, shift 0) of fp32 ids [B, n_ids] -> bf16 [cos | sin] per id, id-major, into row b of out
 * (row stride ldo elements, >= n_ids * dim): SDXL's add_time_proj(time_ids) written straight into columns 1280.. of add_embeds. */
int dllm_time_ids_embedding(const float* ids, void* out, long ldo, int B, int n_ids, int dim, void* stream);
/* y = silu(x) and dx = dy * silu'(x), bf16, n % 8 == 0. */
int dllm_silu_bf16(const void* x, void* y, long n, void* stream);
int dllm_silu_bwd_bf16(const void* dy, const void* x, void* dx, long n, void* stream);
/* dst[b, r, :] = scale * src[b, :] for src [B, H], dst [B, R, H] bf16 (H % 8 == 0): backward of a mean over R rows. */
int dllm_broadcast_rows(const void* src, void* dst, int B, int R, int H, float scale, void* stream);

/* ---- One-token decode step over the kv-cache (dreamllm_b200/decode.py captures it in a CUDA graph).  The cache length is read from
 * the device (`kv_len`, one int32 for the whole batch), so a captured launch stays valid as the cache grows. ----
 * Split planner: the kv rows [0, max_len) are cut into n_splits ranges of split_len rows (a multiple of 64).  split_len depends on
 * (B, nkv, sms) only; max_len only sets n_splits, and the last split starts below max_len.  sms <= 0: the current device's SM count. */
int dllm_attn_decode_plan(int B, int nkv, int max_len, int sms, int* n_splits, int* split_len);
/* fp32 partials of one dllm_attn_decode call with these sizes (the same sms): n_splits * B * nh * (d + 2) * 4 bytes. */
size_t dllm_attn_decode_workspace_bytes(int B, int nh, int nkv, int d, int max_len, int sms);
/* out[b, h * d : (h + 1) * d] = softmax(q[b, h] . K[b, :kv_len, h / g]^T * scale + mask) . V[b, :kv_len, h / g]  (g = nh / nkv in
 * {1, 2, 4, 8}, d 64 or 128).  q: row b at q + b * ld_q (16-byte aligned, ld_q % 8 == 0), heads of d contiguous (the q columns of
 * the fused qkv row).  k_cache / v_cache:
 * contiguous [B, max_len, nkv, d].  kv_mask (nullable): uint8 [B, mask_ld >= max_len], 0 = padded key.  Every key below *kv_len is
 * visible (the query is the newest token).  out row stride ld_o.  Splits at or past *kv_len write a neutral partial; a combine kernel
 * merges the partials in fixed order (deterministic, no atomics). */
int dllm_attn_decode(const void* q, long ld_q, const void* k_cache, const void* v_cache, const int* kv_len, const void* kv_mask,
                     int mask_ld, void* out, long ld_o, void* workspace, size_t workspace_bytes, int B, int max_len, int nh, int nkv, int d,
                     float scale, int sms, void* stream);
/* qkv [B, (nh + 2 nkv) d] (row stride ld): q and k heads rotated in place at positions pos[B] (int32) with the bf16 cos / sin tables
 * of dllm_rope_inplace (same arithmetic, same bits); the rotated k and the v of row b are written to row *kv_len of k_cache / v_cache
 * [B, max_len, nkv, d].  Nothing is written to the cache when *kv_len >= max_len. */
int dllm_rope_append_kv(void* qkv, long ld, const void* cos_table, const void* sin_table, const int* pos, void* k_cache, void* v_cache,
                        const int* kv_len, int max_len, int B, int nh, int nkv, int d, void* stream);

#ifdef __cplusplus
}
#endif
#endif
