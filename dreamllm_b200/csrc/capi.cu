// extern "C" boundary of libdreamllm_sm100.so — see include/dreamllm_sm100.h for the contract.
#include "../../include/dreamllm_sm100.h"
#include "gemm_sm90.h"
#include "ops.h"

using namespace dllm;

static inline cudaStream_t S(void* s) { return static_cast<cudaStream_t>(s); }

// Autograd may call us on a worker thread that has never touched CUDA (observed: cuTensorMapEncodeTiled ->
// CUDA_ERROR_INVALID_CONTEXT when the first CUDA work of the engine's device thread is one of our Functions).  Bind the
// context that owns the caller's buffer — never "device 0" — before any driver/runtime call.
typedef CUresult (*PFN_ctxGetCurrent)(CUcontext*);
typedef CUresult (*PFN_ctxSetCurrent)(CUcontext);
typedef CUresult (*PFN_ptrGetAttr)(void*, CUpointer_attribute, CUdeviceptr);
static void ensure_context(const void* dev_ptr) {
  static PFN_ctxGetCurrent get_cur = nullptr;
  static PFN_ctxSetCurrent set_cur = nullptr;
  static PFN_ptrGetAttr ptr_attr = nullptr;
  static bool resolved = false;
  if (!resolved) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuCtxGetCurrent", &p, cudaEnableDefault, &q) == cudaSuccess) get_cur = (PFN_ctxGetCurrent)p;
    if (cudaGetDriverEntryPoint("cuCtxSetCurrent", &p, cudaEnableDefault, &q) == cudaSuccess) set_cur = (PFN_ctxSetCurrent)p;
    if (cudaGetDriverEntryPoint("cuPointerGetAttribute", &p, cudaEnableDefault, &q) == cudaSuccess) ptr_attr = (PFN_ptrGetAttr)p;
    resolved = true;
  }
  if (!get_cur || !set_cur || !ptr_attr || !dev_ptr) return;
  CUcontext cur = nullptr;
  if (get_cur(&cur) == CUDA_SUCCESS && cur) return;
  CUcontext owner = nullptr;
  if (ptr_attr(&owner, CU_POINTER_ATTRIBUTE_CONTEXT, reinterpret_cast<CUdeviceptr>(dev_ptr)) == CUDA_SUCCESS && owner) set_cur(owner);
}

extern "C" {

int dllm_version(void) { return 100; }
int dllm_set_reserved_sms(int n) { set_reserved_sms(n); return 0; }
int dllm_get_reserved_sms(void) { return reserved_sms(); }

const char* dllm_error_string(int code) {
  switch (code) {
    case 0: return "ok";
    case DLLM_ERR_SHAPE: return "invalid shape / size";
    case DLLM_ERR_ALIGN: return "pointer or stride not 16-byte aligned";
    case DLLM_ERR_DRIVER: return "cuTensorMapEncodeTiled unavailable (no CUDA driver)";
    case DLLM_ERR_TMAP: return "tensor map encode failed";
    case DLLM_ERR_LAUNCH: return "kernel launch failed";
    case DLLM_ERR_UNSUPPORTED: return "unsupported configuration";
    default: return "unknown error";
  }
}

int dllm_gemm_bf16(const void* A, const void* B, void* C, int M, int N, int K, long lda, long ldb, long ldc, int a_mn,
                   int b_mn, int out_fp32, int cta_pair, void* stream) {
  ensure_context(A);
  return gemm_bf16(A, B, C, M, N, K, lda, ldb, ldc, a_mn, b_mn, out_fp32, cta_pair, S(stream));
}

int dllm_rmsnorm_fwd(const void* x, const void* add, const void* weight, void* x_out, void* y, float* rstd, int T, int H,
                     float eps, void* stream) {
  ensure_context(x);
  return rmsnorm_fwd(x, add, weight, x_out, y, rstd, T, H, eps, S(stream));
}
size_t dllm_rmsnorm_bwd_workspace_bytes(int T, int H) { return rmsnorm_bwd_workspace(T, H); }
int dllm_rmsnorm_bwd(const void* dy, const void* x, const void* weight, const float* rstd, const void* dres, void* dx,
                     void* dweight, int dweight_accumulate, void* workspace, size_t workspace_bytes, int T, int H,
                     void* stream) {
  ensure_context(dy);
  return rmsnorm_bwd(dy, x, weight, rstd, dres, dx, dweight, dweight_accumulate, workspace, workspace_bytes, T, H, S(stream));
}
int dllm_rope_inplace(void* buf, const void* cos_table, const void* sin_table, const int* pos, long ld, int T,
                      int heads_total, int head_dim, int mode, void* stream) {
  ensure_context(buf);
  return rope_inplace(buf, cos_table, sin_table, pos, ld, T, heads_total, head_dim, mode, S(stream));
}
int dllm_swiglu_fwd(const void* gate_up, void* act, long ld, int T, int I, void* stream) {
  ensure_context(gate_up);
  return swiglu_fwd(gate_up, act, ld, T, I, S(stream));
}
int dllm_swiglu_bwd(const void* dact, const void* gate_up, void* dgate_up, long ld, int T, int I, void* stream) {
  ensure_context(dact);
  return swiglu_bwd(dact, gate_up, dgate_up, ld, T, I, S(stream));
}
int dllm_add_bf16(const void* a, const void* b, void* out, long n, void* stream) {
  ensure_context(a);
  return add_bf16(a, b, out, n, S(stream));
}
int dllm_cross_entropy(void* logits, const long long* labels, float* loss, float dloss, void* workspace, long ld, int T,
                       int V, int write_grad, void* stream) {
  ensure_context(logits);
  return cross_entropy(logits, labels, loss, dloss, workspace, ld, T, V, write_grad, S(stream));
}
int dllm_embedding_fwd(const long long* ids, const void* weight, void* out, int T, int H, void* stream) {
  ensure_context(weight);
  return embedding_fwd(ids, weight, out, T, H, S(stream));
}
int dllm_embedding_bwd(const long long* sorted_ids, const long long* order, const void* dy, void* dweight, int T, int H,
                       int accumulate, void* stream) {
  ensure_context(dy);
  return embedding_bwd(sorted_ids, order, dy, dweight, T, H, accumulate, S(stream));
}
int dllm_attn_fwd(const void* q, const void* k, const void* v, void* out, float* lse, const int* seqlens, int B, int Sq,
                  int nh, int d, long ld_qkv, long ld_o, int causal, float scale, void* stream) {
  ensure_context(q);
  return attn_fwd(q, k, v, out, lse, seqlens, B, Sq, nh, d, ld_qkv, ld_o, causal, scale, S(stream));
}
size_t dllm_attn_bwd_workspace_bytes(int B, int Sq, int nh, int d) { return attn_bwd_workspace(B, Sq, nh, d); }
int dllm_attn_bwd(const void* dout, const void* q, const void* k, const void* v, const void* out, const float* lse,
                  void* dq, void* dk, void* dv, const int* seqlens, void* workspace, size_t workspace_bytes, int B,
                  int Sq, int nh, int d, long ld_qkv, long ld_o, long ld_dqkv, int causal, float scale, void* stream) {
  ensure_context(dout);
  return attn_bwd(dout, q, k, v, out, lse, dq, dk, dv, seqlens, workspace, workspace_bytes, B, Sq, nh, d, ld_qkv, ld_o,
                  ld_dqkv, causal, scale, S(stream));
}

int dllm_gemm_bf16_ex(const void* A, const void* B, void* C, int M, int N, int K, long lda, long ldb, long ldc, int a_mn,
                      int b_mn, int out_fp32, int cta_pair, const void* bias, const void* residual, long ldr, int act,
                      void* stream) {
  ensure_context(A);
  return gemm_bf16_ex(A, B, C, M, N, K, lda, ldb, ldc, a_mn, b_mn, out_fp32, cta_pair, bias, residual, ldr, act, S(stream));
}
int dllm_layernorm_fwd(const void* x, const void* weight, const void* bias, void* y, int T, int H, float eps, void* stream) {
  ensure_context(x);
  return layernorm_fwd(x, weight, bias, y, T, H, eps, S(stream));
}
int dllm_clip_patchify(const void* images, void* out, int N, int R, int patch, int Kpad, void* stream) {
  ensure_context(images);
  return clip_patchify(images, out, N, R, patch, Kpad, S(stream));
}
int dllm_clip_assemble(const void* patches, const void* cls, const void* pos, void* out, int N, int P, int C, void* stream) {
  ensure_context(patches);
  return clip_assemble(patches, cls, pos, out, N, P, C, S(stream));
}
int dllm_copy_rows(void* dst, const int* dst_idx, const void* src, const int* src_idx, int R, int H, int mode, void* stream) {
  ensure_context(dst);
  return copy_rows(dst, dst_idx, src, src_idx, R, H, mode, S(stream));
}
int dllm_segment_sum_rows(void* dst, const void* src, const int* seg, const int* rows, int Q, int H, void* stream) {
  ensure_context(dst);
  return segment_sum_rows(dst, src, seg, rows, Q, H, S(stream));
}
int dllm_zero_rows(void* dst, const int* idx, int R, int H, void* stream) {
  ensure_context(dst);
  return zero_rows(dst, idx, R, H, S(stream));
}

int dllm_attn_fwd_ex(const void* q, const void* k, const void* v, void* out, float* lse, const int* seqlens, int B, int Sq,
                     int Skv, int nh, int d, long ld_q, long ld_kv, long ld_o, int causal, float scale, void* stream) {
  ensure_context(q);
  return attn_fwd_ex(q, k, v, out, lse, seqlens, B, Sq, Skv, nh, d, ld_q, ld_kv, ld_o, causal, scale, S(stream));
}
int dllm_attn_fwd_cache(const void* q, const void* k, const void* v, void* out, float* lse, int B, int Sq, int Skv, int kv_rows, int nh,
                        int d, long ld_q, long ld_kv, long ld_o, int causal, float scale, void* stream) {
  ensure_context(q);
  return attn_fwd_cache(q, k, v, out, lse, nullptr, B, Sq, Skv, kv_rows, nh, d, ld_q, ld_kv, ld_o, causal, scale, S(stream));
}
int dllm_attn_fwd_cache_mask(const void* q, const void* k, const void* v, void* out, float* lse, const void* kv_mask, int mask_ld, int B,
                             int Sq, int Skv, int kv_rows, int nh, int d, long ld_q, long ld_kv, long ld_o, int causal, float scale,
                             void* stream) {
  return attn_fwd_cache_mask(q, k, v, out, lse, nullptr, kv_mask, mask_ld, B, Sq, Skv, kv_rows, nh, d, ld_q, ld_kv, ld_o, causal, scale,
                             S(stream));
}
int dllm_attn_fwd_gqa(const void* q, const void* k, const void* v, void* out, float* lse, const int* seqlens, const void* kv_mask,
                      int mask_ld, int B, int Sq, int Skv, int kv_rows, int nh, int nkv, int d, long ld_q, long ld_kv, long ld_o, int causal,
                      float scale, void* stream) {
  ensure_context(q);
  return attn_fwd_gqa(q, k, v, out, lse, seqlens, kv_mask, mask_ld, B, Sq, Skv, kv_rows, nh, nkv, d, ld_q, ld_kv, ld_o, causal, scale,
                      S(stream));
}
int dllm_attn_probs_gqa(const void* q, const void* k, const float* lse, void* probs, const int* seqlens, const void* kv_mask, int mask_ld,
                        int B, int Sq, int Skv, int kv_rows, int nh, int nkv, int d, long ld_q, long ld_kv, int causal, float scale,
                        void* stream) {
  ensure_context(q);
  return attn_probs_gqa(q, k, lse, probs, seqlens, kv_mask, mask_ld, B, Sq, Skv, kv_rows, nh, nkv, d, ld_q, ld_kv, causal, scale,
                        S(stream));
}
int dllm_attn_bwd_gqa(const void* dout, const void* q, const void* k, const void* v, const void* out, const float* lse, void* dq,
                      void* dk, void* dv, const int* seqlens, void* workspace, size_t workspace_bytes, int B, int Sq, int Skv, int nh,
                      int nkv, int d, long ld_q, long ld_kv, long ld_o, long ld_dq, long ld_dkv, int causal, float scale, void* stream) {
  ensure_context(dout);
  return attn_bwd_gqa(dout, q, k, v, out, lse, dq, dk, dv, seqlens, workspace, workspace_bytes, B, Sq, Skv, nh, nkv, d, ld_q, ld_kv,
                      ld_o, ld_dq, ld_dkv, causal, scale, S(stream));
}
int dllm_attn_fwd_varlen(const void* q, const void* k, const void* v, void* out, float* lse, const int* cu_seqlens, int B, int T,
                         int max_seqlen, int nh, int nkv, int d, long ld_q, long ld_kv, long ld_o, int causal, float scale, void* stream) {
  ensure_context(q);
  return attn_fwd_varlen(q, k, v, out, lse, cu_seqlens, B, T, max_seqlen, nh, nkv, d, ld_q, ld_kv, ld_o, causal, scale, S(stream));
}
size_t dllm_attn_bwd_varlen_workspace_bytes(int T, int nh, int d) { return attn_bwd_varlen_workspace(T, nh, d); }
int dllm_attn_bwd_varlen(const void* dout, const void* q, const void* k, const void* v, const void* out, const float* lse, void* dq,
                         void* dk, void* dv, const int* cu_seqlens, void* workspace, size_t workspace_bytes, int B, int T, int max_seqlen,
                         int nh, int nkv, int d, long ld_q, long ld_kv, long ld_o, long ld_dq, long ld_dkv, int causal, float scale,
                         void* stream) {
  ensure_context(dout);
  return attn_bwd_varlen(dout, q, k, v, out, lse, dq, dk, dv, cu_seqlens, workspace, workspace_bytes, B, T, max_seqlen, nh, nkv, d, ld_q,
                         ld_kv, ld_o, ld_dq, ld_dkv, causal, scale, S(stream));
}
int dllm_conv3x3_nhwc(const void* x, const void* w, void* y, int N, int H, int W, int Cin, int Cout, const void* bias,
                      const void* rowbias, const void* residual, void* stream) {
  ensure_context(x);
  return conv3x3_nhwc(x, w, y, N, H, W, Cin, Cout, bias, rowbias, residual, S(stream));
}
size_t dllm_groupnorm_workspace_bytes(int N, int HW, int G) { return groupnorm_workspace(N, HW, G); }
int dllm_groupnorm_nhwc(const void* x, const void* w, const void* b, void* y, void* workspace, size_t ws_bytes, int N, int HW,
                        int C, int G, float eps, int silu, void* stream) {
  ensure_context(x);
  return groupnorm_nhwc(x, w, b, y, workspace, ws_bytes, N, HW, C, G, eps, silu, S(stream));
}
int dllm_geglu(const void* in, void* out, int T, int I, void* stream) { ensure_context(in); return geglu(in, out, T, I, S(stream)); }
int dllm_upsample2x_nhwc(const void* x, void* y, int N, int H, int W, int C, void* stream) {
  ensure_context(x);
  return upsample2x_nhwc(x, y, N, H, W, C, S(stream));
}
int dllm_im2col_s2_nhwc(const void* x, void* out, int N, int H, int W, int C, int pad, void* stream) {
  ensure_context(x);
  return im2col_s2_nhwc(x, out, N, H, W, C, pad, S(stream));
}
int dllm_copy_cols(const void* src, void* dst, long rows, int Cs, int Cd, int col0, void* stream) {
  ensure_context(src);
  return copy_cols(src, dst, rows, Cs, Cd, col0, S(stream));
}
int dllm_conv_in(const float* x, const void* w, const void* bias, void* y, int B, int Bsrc, int Cin, int H, int W, int Cout,
                 void* stream) {
  ensure_context(x);
  return conv_in_nchw_to_nhwc(x, w, bias, y, B, Bsrc, Cin, H, W, Cout, S(stream));
}
int dllm_conv_out(const void* x, const void* w, const void* bias, float* y, int B, int C, int H, int W, int Cout, void* stream) {
  ensure_context(x);
  return conv_out_nhwc_to_nchw(x, w, bias, y, B, C, H, W, Cout, S(stream));
}
size_t dllm_gemm_splitk_workspace_bytes(int M, int N, int K) { return gemm_splitk_workspace(M, N, K); }
int dllm_gemm_tile_n(int M, int N, int K, int b_mn) { return gemm_tile_bn(M, N, K, b_mn); }
int dllm_gemm_bf16_ws(const void* A, const void* B, void* C, int M, int N, int K, long lda, long ldb, long ldc, int b_mn, const void* bias,
                      const void* residual, long ldr, int act, void* ws, size_t ws_bytes, void* stream) {
  ensure_context(A);
  return gemm_bf16_ws(A, B, C, M, N, K, lda, ldb, ldc, b_mn, bias, residual, ldr, act, ws, ws_bytes, S(stream));
}
size_t dllm_conv3x3_splitk_workspace_bytes(int N, int H, int W, int Cin, int Cout) { return conv3x3_splitk_workspace(N, H, W, Cin, Cout); }
int dllm_conv3x3_nhwc_ws(const void* x, const void* w, void* y, int N, int H, int W, int Cin, int Cout, const void* bias,
                         const void* rowbias, const void* residual, void* ws, size_t ws_bytes, void* stream) {
  ensure_context(x);
  return conv3x3_nhwc_ws(x, w, y, N, H, W, Cin, Cout, bias, rowbias, residual, ws, ws_bytes, S(stream));
}
int dllm_gemm_bf16_geglu(const void* A, const void* Wp, const void* bias_p, void* out, int M, int N, int K, long lda, long ldb, long ldc,
                         void* stream) {
  ensure_context(A);
  return gemm_bf16_geglu(A, Wp, bias_p, out, M, N, K, lda, ldb, ldc, S(stream));
}
int dllm_im2col_in(const float* x, void* cols, int B, int Bsrc, int Cin, int H, int W, void* stream) {
  ensure_context(cols);
  return im2col_in(x, cols, B, Bsrc, Cin, H, W, S(stream));
}
int dllm_nhwc_to_nchw_f32(const void* y, float* out, int N, int HW, int Cp, int Cout, void* stream) {
  ensure_context(y);
  return nhwc_to_nchw_f32(y, out, N, HW, Cp, Cout, S(stream));
}
int dllm_timestep_embedding(const int* timesteps, const int* step, void* out, int B, int dim, void* stream) {
  ensure_context(out);
  return timestep_embedding(timesteps, step, out, B, dim, S(stream));
}
int dllm_timestep_embedding_batch(const int* t, void* out, int B, int dim, void* stream) {
  ensure_context(out);
  return timestep_embedding_batch(t, out, B, dim, S(stream));
}
int dllm_sampler_step(const float* eps, float* latents, const float* noise, const float* coef, int* step, float guidance,
                      int use_cfg, int mode, long n, void* stream) {
  ensure_context(eps);
  return sampler_step(eps, latents, noise, coef, step, guidance, use_cfg, mode, n, S(stream));
}
int dllm_attn_bwd_ex(const void* dout, const void* q, const void* k, const void* v, const void* out, const float* lse, void* dq,
                     void* dk, void* dv, const int* seqlens, void* workspace, size_t workspace_bytes, int B, int Sq, int Skv, int nh,
                     int d, long ld_q, long ld_kv, long ld_o, long ld_dq, long ld_dkv, int causal, float scale, void* stream) {
  ensure_context(dout);
  return attn_bwd_ex(dout, q, k, v, out, lse, dq, dk, dv, seqlens, workspace, workspace_bytes, B, Sq, Skv, nh, d, ld_q, ld_kv, ld_o,
                     ld_dq, ld_dkv, causal, scale, S(stream));
}
int dllm_groupnorm_stats(const void* x, float* stats, void* workspace, size_t ws_bytes, int N, int HW, int C, int G, float eps, void* stream) {
  ensure_context(x);
  return groupnorm_stats(x, stats, workspace, ws_bytes, N, HW, C, G, eps, S(stream));
}
int dllm_groupnorm_apply(const void* x, const void* w, const void* b, const float* stats, void* y, int N, int HW, int C, int G, int silu,
                         void* stream) {
  ensure_context(x);
  return groupnorm_apply(x, w, b, stats, y, N, HW, C, G, silu, S(stream));
}
int dllm_groupnorm_bwd_nhwc(const void* dy, const void* x, const void* w, const void* b, const float* stats, const void* dres, void* dx,
                            void* workspace, size_t ws_bytes, int N, int HW, int C, int G, int silu, void* stream) {
  ensure_context(dy);
  return groupnorm_bwd_nhwc(dy, x, w, b, stats, dres, dx, workspace, ws_bytes, N, HW, C, G, silu, S(stream));
}
int dllm_layernorm_bwd(const void* dy, const void* x, const void* w, const void* dres, void* dx, int T, int H, float eps, void* stream) {
  ensure_context(dy);
  return layernorm_bwd(dy, x, w, dres, dx, T, H, eps, S(stream));
}
size_t dllm_layernorm_bwd_affine_workspace_bytes(int T, int H) { return layernorm_bwd_affine_workspace(T, H); }
int dllm_layernorm_bwd_affine(const void* dy, const void* x, const void* w, const void* dres, void* dx, void* dgamma, void* dbeta,
                              void* workspace, size_t workspace_bytes, int T, int H, float eps, void* stream) {
  ensure_context(dy);
  return layernorm_bwd_affine(dy, x, w, dres, dx, dgamma, dbeta, workspace, workspace_bytes, T, H, eps, S(stream));
}
int dllm_quick_gelu(const void* x, void* y, long n, void* stream) {
  ensure_context(x);
  return quick_gelu(x, y, n, S(stream));
}
int dllm_quick_gelu_bwd(const void* dy, const void* x, void* dx, long n, void* stream) {
  ensure_context(dy);
  return quick_gelu_bwd(dy, x, dx, n, S(stream));
}
int dllm_geglu_bwd(const void* dout, const void* in, void* din, int T, int I, void* stream) {
  ensure_context(dout);
  return geglu_bwd(dout, in, din, T, I, S(stream));
}
int dllm_upsample2x_bwd_nhwc(const void* dy, void* dx, int N, int H, int W, int C, void* stream) {
  ensure_context(dy);
  return upsample2x_bwd_nhwc(dy, dx, N, H, W, C, S(stream));
}
int dllm_col2im_s2_nhwc(const void* dcols, void* dx, int N, int H, int W, int C, void* stream) {
  ensure_context(dcols);
  return col2im_s2_nhwc(dcols, dx, N, H, W, C, S(stream));
}
int dllm_copy_cols2(const void* src, void* dst, long rows, int Cs, int Cd, int scol0, int dcol0, int ncols, void* stream) {
  ensure_context(src);
  return copy_cols2(src, dst, rows, Cs, Cd, scol0, dcol0, ncols, S(stream));
}
int dllm_conv_out_bwd(const float* dy, const void* w, void* dx, int B, int C, int H, int W, int Cout, void* stream) {
  ensure_context(dy);
  return conv_out_bwd(dy, w, dx, B, C, H, W, Cout, S(stream));
}
int dllm_add_noise(const float* x0, const float* noise, const int* t, const float* alphas_cumprod, float* out, int B, long per_sample,
                   void* stream) {
  ensure_context(x0);
  return add_noise(x0, noise, t, alphas_cumprod, out, B, per_sample, S(stream));
}
int dllm_mse_fwd_bwd(const float* pred, const float* target, float* loss, float* dpred, long n, void* stream) {
  ensure_context(pred);
  return mse_fwd_bwd(pred, target, loss, dpred, n, S(stream));
}
int dllm_mse_minsnr_fwd_bwd(const float* pred, const float* target, const int* t, const float* alphas_cumprod, float snr_gamma,
                            float* loss, float* dpred, int B, long per_sample, void* stream) {
  ensure_context(pred);
  return mse_minsnr_fwd_bwd(pred, target, t, alphas_cumprod, snr_gamma, loss, dpred, B, per_sample, S(stream));
}

int dllm_softmax_rows(void* x, long rows, int cols, float scale, void* stream) {
  ensure_context(x);
  return softmax_rows(x, rows, cols, scale, S(stream));
}
int dllm_vae_sample(const float* h, const void* wq, const void* bq, const float* z, float* out, int B, int L, long plane, float scaling,
                    void* stream) {
  ensure_context(h);
  return vae_sample(h, wq, bq, z, out, B, L, plane, scaling, S(stream));
}


int dllm_adamw_step(const void* grad, void* master, void* exp_avg, void* exp_avg_sq, void* param, long n, int bf16_state, double lr,
                    double beta1, double beta2, double eps, double weight_decay, int step, const float* grad_sumsq,
                    double max_grad_norm,
                    void* stream) {
  ensure_context(grad);
  return adamw_step(grad, master, exp_avg, exp_avg_sq, param, n, bf16_state, lr, beta1, beta2, eps, weight_decay, step, grad_sumsq,
                    max_grad_norm, S(stream));
}
size_t dllm_sumsq_workspace_bytes(void) { return sumsq_workspace(); }
int dllm_sumsq_bf16(const void* x, long n, float* out, int accumulate, void* workspace, size_t workspace_bytes, void* stream) {
  ensure_context(out);
  return sumsq_bf16(x, n, out, accumulate, workspace, workspace_bytes, S(stream));
}

size_t dllm_channel_sum_workspace_bytes(int N, int HW, int C) { return channel_sum_workspace(N, HW, C); }
int dllm_channel_sum_nhwc(const void* x, void* out, long ldo, int out_bf16, float scale, int N, int HW, int C, void* workspace,
                          size_t workspace_bytes, void* stream) {
  ensure_context(x);
  return channel_sum_nhwc(x, out, ldo, out_bf16, scale, N, HW, C, workspace, workspace_bytes, S(stream));
}
int dllm_time_ids_embedding(const float* ids, void* out, long ldo, int B, int n_ids, int dim, void* stream) {
  ensure_context(out);
  return time_ids_embedding(ids, out, ldo, B, n_ids, dim, S(stream));
}
int dllm_silu_bf16(const void* x, void* y, long n, void* stream) {
  ensure_context(x);
  return silu_bf16(x, y, n, S(stream));
}
int dllm_silu_bwd_bf16(const void* dy, const void* x, void* dx, long n, void* stream) {
  ensure_context(dy);
  return silu_bwd_bf16(dy, x, dx, n, S(stream));
}
int dllm_broadcast_rows(const void* src, void* dst, int B, int R, int H, float scale, void* stream) {
  ensure_context(src);
  return broadcast_rows(src, dst, B, R, H, scale, S(stream));
}
int dllm_attn_decode_plan(int B, int nkv, int max_len, int sms, int* n_splits, int* split_len) {
  return attn_decode_plan(B, nkv, max_len, sms, n_splits, split_len);
}
size_t dllm_attn_decode_workspace_bytes(int B, int nh, int nkv, int d, int max_len, int sms) {
  return attn_decode_workspace(B, nh, nkv, d, max_len, sms);
}
int dllm_attn_decode(const void* q, long ld_q, const void* k_cache, const void* v_cache, const int* kv_len, const void* kv_mask,
                     int mask_ld, void* out, long ld_o, void* workspace, size_t workspace_bytes, int B, int max_len, int nh, int nkv, int d,
                     float scale, int sms, void* stream) {
  ensure_context(q);
  return attn_decode(q, ld_q, k_cache, v_cache, kv_len, kv_mask, mask_ld, out, ld_o, workspace, workspace_bytes, B, max_len, nh, nkv, d,
                     scale, sms, S(stream));
}
int dllm_rope_append_kv(void* qkv, long ld, const void* cos_table, const void* sin_table, const int* pos, void* k_cache, void* v_cache,
                        const int* kv_len, int max_len, int B, int nh, int nkv, int d, void* stream) {
  ensure_context(qkv);
  return rope_append_kv(qkv, ld, cos_table, sin_table, pos, k_cache, v_cache, kv_len, max_len, B, nh, nkv, d, S(stream));
}

}  // extern "C"
