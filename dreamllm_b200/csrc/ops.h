// Internal C++ declarations of the non-GEMM ops (definitions: elementwise.cu, attn_sm90.cu).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace dllm {
int rmsnorm_fwd(const void* x, const void* add, const void* w, void* x_out, void* y, float* rstd, int T, int H, float eps,
                cudaStream_t s);
size_t rmsnorm_bwd_workspace(int T, int H);
int rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd, const void* dres, void* dx, void* dw,
                int dw_accumulate, void* workspace, size_t workspace_bytes, int T, int H, cudaStream_t s);
int rope_inplace(void* buf, const void* cos_t, const void* sin_t, const int* pos, long ld, int T, int heads_total,
                 int head_dim, int mode, cudaStream_t s);
int swiglu_fwd(const void* gu, void* act, long ld_gu, int T, int I, cudaStream_t s);
int swiglu_bwd(const void* dact, const void* gu, void* dgu, long ld_gu, int T, int I, cudaStream_t s);
int add_bf16(const void* a, const void* b, void* o, long n, cudaStream_t s);
int cross_entropy(void* logits, const long long* labels, float* loss, float dloss, void* workspace, long ld, int T, int V,
                  int write_grad, cudaStream_t s);
int embedding_fwd(const long long* ids, const void* W, void* out, int T, int H, cudaStream_t s);
int embedding_bwd(const long long* sorted_ids, const long long* order, const void* dy, void* dW, int T, int H,
                  int accumulate, cudaStream_t s);
int layernorm_fwd(const void* x, const void* w, const void* b, void* y, int T, int H, float eps, cudaStream_t s);
int clip_patchify(const void* img, void* out, int N, int R, int patch, int Kpad, cudaStream_t s);
int clip_assemble(const void* patches, const void* cls, const void* pos, void* out, int N, int P, int C, cudaStream_t s);
int copy_rows(void* dst, const int* dst_idx, const void* src, const int* src_idx, int R, int H, int mode, cudaStream_t s);
int segment_sum_rows(void* dst, const void* src, const int* seg, const int* rows, int Q, int H, cudaStream_t s);
int zero_rows(void* dst, const int* idx, int R, int H, cudaStream_t s);
int attn_fwd(const void* q, const void* k, const void* v, void* out, float* lse, const int* seqlens, int B, int S, int nh,
             int d, long ld_qkv, long ld_o, int causal, float scale, cudaStream_t s);
int attn_fwd_ex(const void* q, const void* k, const void* v, void* out, float* lse, const int* seqlens, int B, int S, int Skv,
                int nh, int d, long ld_q, long ld_kv, long ld_o, int causal, float scale, cudaStream_t s);
int attn_fwd_cache(const void* q, const void* k, const void* v, void* out, float* lse, const int* seqlens, int B, int S, int Skv,
                   int kv_rows, int nh, int d, long ld_q, long ld_kv, long ld_o, int causal, float scale, cudaStream_t s);
int attn_fwd_cache_mask(const void* q, const void* k, const void* v, void* out, float* lse, const int* seqlens, const void* kv_mask,
                        int mask_ld, int B, int S, int Skv, int kv_rows, int nh, int d, long ld_q, long ld_kv, long ld_o, int causal,
                        float scale, cudaStream_t st);
int attn_fwd_gqa(const void* q, const void* k, const void* v, void* out, float* lse, const int* seqlens, const void* kv_mask,
                 int mask_ld, int B, int S, int Skv, int kv_rows, int nh, int nkv, int d, long ld_q, long ld_kv, long ld_o, int causal,
                 float scale, cudaStream_t st);
int attn_fwd_varlen(const void* q, const void* k, const void* v, void* out, float* lse, const int* cu_seqlens, int B, int T,
                    int max_seqlen, int nh, int nkv, int d, long ld_q, long ld_kv, long ld_o, int causal, float scale, cudaStream_t st);
int attn_probs_gqa(const void* q, const void* k, const float* lse, void* probs, const int* seqlens, const void* kv_mask, int mask_ld,
                   int B, int S, int Skv, int kv_rows, int nh, int nkv, int d, long ld_q, long ld_kv, int causal, float scale,
                   cudaStream_t st);
size_t groupnorm_workspace(int N, int HW, int G);
int groupnorm_nhwc(const void* x, const void* w, const void* b, void* y, void* workspace, size_t ws_bytes, int N, int HW, int C,
                   int G, float eps, int silu, cudaStream_t s);
int geglu(const void* in, void* out, int T, int I, cudaStream_t s);
int upsample2x_nhwc(const void* x, void* y, int N, int H, int W, int C, cudaStream_t s);
int im2col_s2_nhwc(const void* x, void* out, int N, int H, int W, int C, int pad, cudaStream_t s);
int copy_cols(const void* src, void* dst, long rows, int Cs, int Cd, int col0, cudaStream_t s);
int conv_in_nchw_to_nhwc(const float* x, const void* w, const void* bias, void* y, int B, int Bsrc, int Cin, int H, int W,
                         int Cout, cudaStream_t s);
int conv_out_nhwc_to_nchw(const void* x, const void* w, const void* bias, float* y, int B, int C, int H, int W, int Cout,
                          cudaStream_t s);
int im2col_in(const float* x, void* cols, int B, int Bsrc, int Cin, int H, int W, cudaStream_t s);
int nhwc_to_nchw_f32(const void* y, float* out, int N, int HW, int Cp, int Cout, cudaStream_t s);
int timestep_embedding(const int* timesteps, const int* step, void* out, int B, int dim, cudaStream_t s);
int timestep_embedding_batch(const int* t, void* out, int B, int dim, cudaStream_t s);
int sampler_step(const float* eps, float* latents, const float* noise, const float* coef, int* step, float guidance, int use_cfg,
                 int mode, long n, cudaStream_t s);
size_t attn_bwd_workspace(int B, int S, int nh, int d);
int attn_bwd(const void* dout, const void* q, const void* k, const void* v, const void* out, const float* lse, void* dq,
             void* dk, void* dv, const int* seqlens, void* workspace, size_t workspace_bytes, int B, int S, int nh, int d,
             long ld_qkv, long ld_o, long ld_dqkv, int causal, float scale, cudaStream_t s);
int attn_bwd_ex(const void* dout, const void* q, const void* k, const void* v, const void* out, const float* lse, void* dq,
                void* dk, void* dv, const int* seqlens, void* workspace, size_t workspace_bytes, int B, int S, int Skv, int nh,
                int d, long ld_q, long ld_kv, long ld_o, long ld_dq, long ld_dkv, int causal, float scale, cudaStream_t s);
int attn_bwd_gqa(const void* dout, const void* q, const void* k, const void* v, const void* out, const float* lse, void* dq,
                 void* dk, void* dv, const int* seqlens, void* workspace, size_t workspace_bytes, int B, int S, int Skv, int nh,
                 int nkv, int d, long ld_q, long ld_kv, long ld_o, long ld_dq, long ld_dkv, int causal, float scale, cudaStream_t s);
size_t attn_bwd_varlen_workspace(int T, int nh, int d);
int attn_bwd_varlen(const void* dout, const void* q, const void* k, const void* v, const void* out, const float* lse, void* dq,
                    void* dk, void* dv, const int* cu_seqlens, void* workspace, size_t workspace_bytes, int B, int T, int max_seqlen,
                    int nh, int nkv, int d, long ld_q, long ld_kv, long ld_o, long ld_dq, long ld_dkv, int causal, float scale,
                    cudaStream_t s);
int groupnorm_bwd_nhwc(const void* dy, const void* x, const void* w, const void* b, const float* stats, const void* dres, void* dx,
                       void* workspace, size_t ws_bytes, int N, int HW, int C, int G, int silu, cudaStream_t s);
int groupnorm_stats(const void* x, float* stats, void* workspace, size_t ws_bytes, int N, int HW, int C, int G, float eps, cudaStream_t s);
int groupnorm_apply(const void* x, const void* w, const void* b, const float* stats, void* y, int N, int HW, int C, int G, int silu,
                    cudaStream_t s);
int layernorm_bwd(const void* dy, const void* x, const void* w, const void* dres, void* dx, int T, int H, float eps, cudaStream_t s);
size_t layernorm_bwd_affine_workspace(int T, int H);
int layernorm_bwd_affine(const void* dy, const void* x, const void* w, const void* dres, void* dx, void* dgamma, void* dbeta,
                         void* workspace, size_t ws_bytes, int T, int H, float eps, cudaStream_t s);
int quick_gelu(const void* x, void* y, long n, cudaStream_t s);
int quick_gelu_bwd(const void* dy, const void* x, void* dx, long n, cudaStream_t s);
int geglu_bwd(const void* dout, const void* in, void* din, int T, int I, cudaStream_t s);
int upsample2x_bwd_nhwc(const void* dy, void* dx, int N, int H, int W, int C, cudaStream_t s);
int col2im_s2_nhwc(const void* dcols, void* dx, int N, int H, int W, int C, cudaStream_t s);
int copy_cols2(const void* src, void* dst, long rows, int Cs, int Cd, int scol0, int dcol0, int ncols, cudaStream_t s);
int conv_out_bwd(const float* dy, const void* w, void* dx, int B, int C, int H, int W, int Cout, cudaStream_t s);
int add_noise(const float* x0, const float* noise, const int* t, const float* ac, float* out, int B, long per_sample, cudaStream_t s);
int mse_fwd_bwd(const float* pred, const float* target, float* loss, float* dpred, long n, cudaStream_t s);
int mse_minsnr_fwd_bwd(const float* pred, const float* target, const int* t, const float* ac, float gamma, float* loss, float* dpred,
                       int B, long per_sample, cudaStream_t s);
int softmax_rows(void* x, long rows, int cols, float scale, cudaStream_t s);
int vae_sample(const float* h, const void* wq, const void* bq, const float* z, float* out, int B, int L, long plane, float scaling,
               cudaStream_t s);
// optim.cu — sharded AdamW + grad-norm (SURVEY §8f row 4)
int adamw_step(const void* grad, void* master, void* mom, void* var, void* param, long n, int bf16_state, double lr, double beta1,
               double beta2, double eps, double weight_decay, int step, const float* sumsq, double max_norm, cudaStream_t s);
size_t sumsq_workspace();
int sumsq_bf16(const void* x, long n, float* out, int accumulate, void* workspace, size_t ws_bytes, cudaStream_t s);
// sdxl_ops.cu: addition embedding of the SDXL UNet and its gradient path
size_t channel_sum_workspace(int N, int HW, int C);
int channel_sum_nhwc(const void* x, void* out, long ldo, int out_bf16, float scale, int N, int HW, int C, void* workspace,
                     size_t ws_bytes, cudaStream_t s);
int time_ids_embedding(const float* ids, void* out, long ldo, int B, int n_ids, int dim, cudaStream_t s);
int silu_bf16(const void* x, void* y, long n, cudaStream_t s);
int silu_bwd_bf16(const void* dy, const void* x, void* dx, long n, cudaStream_t s);
int broadcast_rows(const void* src, void* dst, int B, int R, int H, float scale, cudaStream_t s);
// decode_sm90.cu: one-token decode attention over the kv-cache (split-KV, cache length on the device) and the RoPE + cache append
int attn_decode_plan(int B, int nkv, int max_len, int sms, int* n_splits, int* split_len);
size_t attn_decode_workspace(int B, int nh, int nkv, int d, int max_len, int sms);
int attn_decode(const void* q, long ld_q, const void* k_cache, const void* v_cache, const int* kv_len, const void* kv_mask, int mask_ld,
                void* out, long ld_o, void* workspace, size_t ws_bytes, int B, int max_len, int nh, int nkv, int d, float scale, int sms,
                cudaStream_t s);
int rope_append_kv(void* qkv, long ld, const void* cos_t, const void* sin_t, const int* pos, void* k_cache, void* v_cache,
                   const int* kv_len, int max_len, int B, int nh, int nkv, int d, cudaStream_t s);
}  // namespace dllm
