// Internal (C++) declarations shared between the kernels and the C-ABI layer.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define DLLM_OK 0
#define DLLM_ERR_SHAPE (-1)
#define DLLM_ERR_ALIGN (-2)
#define DLLM_ERR_DRIVER (-3)
#define DLLM_ERR_TMAP (-4)
#define DLLM_ERR_LAUNCH (-5)
#define DLLM_ERR_UNSUPPORTED (-6)

namespace dllm {

int num_sms();
void set_reserved_sms(int n);
int reserved_sms();
int make_tmap_2d(CUtensorMap* map, const void* ptr, int elem_bytes, uint64_t rows, uint64_t cols, uint64_t ld,
                 uint32_t box_rows, uint32_t box_cols);

// C[M,N] = op(A) op(B); see gemm_sm90.cu for the operand conventions. ld* are row strides in elements.
int gemm_bf16(const void* A, const void* B, void* C, int M, int N, int K, long lda, long ldb, long ldc, int a_mn,
              int b_mn, int out_fp32, int cta_pair, cudaStream_t stream);

// same, with the fused epilogue out = act(bf16(acc + bias)) (+ residual); act: 0 none, 1 quick_gelu, 2 gelu(erf), 3 silu
int gemm_bf16_ex(const void* A, const void* B, void* C, int M, int N, int K, long lda, long ldb, long ldc, int a_mn,
                 int b_mn, int out_fp32, int cta_pair, const void* bias, const void* residual, long ldr, int act,
                 cudaStream_t stream);

// split-K variants for small-M shapes (workspace sized by the *_workspace query; 0 = the shape is not split)
size_t gemm_splitk_workspace(int M, int N, int K);
// N-tile width a bf16-output GEMM with K-major A uses when run with that workspace: the split-K width, or the tile planner's
int gemm_tile_bn(int M, int N, int K, int b_mn);
int gemm_bf16_ws(const void* A, const void* B, void* C, int M, int N, int K, long lda, long ldb, long ldc, int b_mn, const void* bias,
                 const void* residual, long ldr, int act, void* ws, size_t ws_bytes, cudaStream_t stream);
size_t conv3x3_splitk_workspace(int Nimg, int H, int W, int Cin, int Cout);
int conv3x3_nhwc_ws(const void* x, const void* w, void* y, int Nimg, int H, int W, int Cin, int Cout, const void* bias,
                    const void* rowbias, const void* residual, void* ws, size_t ws_bytes, cudaStream_t stream);

// FeedForward-in projection with the GEGLU fused into the epilogue (weight rows pre-permuted: [64 value | 64 gate] per 128-row group)
int gemm_bf16_geglu(const void* A, const void* Wp, const void* bias_p, void* out, int M, int N, int K, long lda, long ldb, long ldc,
                    cudaStream_t stream);

// implicit-GEMM 3x3 stride-1 pad-1 convolution, NHWC bf16 (see gemm_sm90.cu)
int conv3x3_nhwc(const void* x, const void* w, void* y, int Nimg, int H, int W, int Cin, int Cout, const void* bias,
                 const void* rowbias, const void* residual, cudaStream_t stream);

}  // namespace dllm
