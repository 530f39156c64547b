// Kernels of the SDXL UNet's addition embedding ("text_time", diffusers 0.24 UNet2DConditionModel) and of the gradient that reaches
// the pooled conditioning through it (sm_90a).  HBM-bound or tiny; bf16 data, fp32 arithmetic, one rounding per output.
//   channel_sum_nhwc   : out[n, c] = scale * sum_hw x[n, hw, c]   (time_emb_proj bias gradient of every resnet; mean over dream queries)
//   time_ids_embedding : Timesteps(256, flip_sin_to_cos=True, shift 0) of float ids, written into a column slice of add_embeds
//   silu / silu_bwd    : the SiLU between temb and the resnets' time_emb_proj, and inside add_embedding
//   broadcast_rows     : dst[b, r, :] = scale * src[b, :]          (backward of the mean over dream queries)
#include "common.cuh"
#include "ops.h"
#include "../../include/dreamllm_sm100.h"

namespace dllm {
namespace {

__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[i]));
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
    w[i] = *reinterpret_cast<const uint32_t*>(&h);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// ---- channel sum.  Pass 1: CTA (chunk, column tile, n) sums `rows` rows of a 512-channel tile: 64 threads per row, one 16-byte vector
// each, 4 row groups; the groups are added in a fixed order through shared memory and the CTA writes one fp32 partial row.  Pass 2 adds
// the partials of each (n, c) in chunk order.  No atomics: the result depends only on (N, HW, C), never on scheduling.
constexpr int kCsVecs = 64;
constexpr int kCsGroups = 4;
constexpr int kCsTargetCtas = 528;   // 4 per SM of a 132-SM H100

__global__ void __launch_bounds__(kCsVecs * kCsGroups) channel_sum_partial_kernel(const bf16* __restrict__ x, float* __restrict__ partial,
                                                                                   int HW, int C, int rows, int chunks) {
  __shared__ float sm[kCsGroups][8][kCsVecs];
  const int n = blockIdx.z, chunk = blockIdx.x;
  const int col = threadIdx.x % kCsVecs, grp = threadIdx.x / kCsVecs;
  const int nv = C >> 3;
  const int v = blockIdx.y * kCsVecs + col;
  const int r0 = chunk * rows, r1 = min(HW, r0 + rows);
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (v < nv) {
    const uint4* base = reinterpret_cast<const uint4*>(x + static_cast<size_t>(n) * HW * C) + v;
    for (int r = r0 + grp; r < r1; r += kCsGroups) {
      float f[8];
      unpack8(base[static_cast<size_t>(r) * nv], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += f[j];
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) sm[grp][j][col] = acc[j];
  __syncthreads();
  if (grp == 0 && v < nv) {
    float s[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] = ((sm[0][j][col] + sm[1][j][col]) + sm[2][j][col]) + sm[3][j][col];
    float4* dst = reinterpret_cast<float4*>(partial + (static_cast<size_t>(n) * chunks + chunk) * C + static_cast<size_t>(v) * 8);
    dst[0] = make_float4(s[0], s[1], s[2], s[3]);
    dst[1] = make_float4(s[4], s[5], s[6], s[7]);
  }
}

__global__ void __launch_bounds__(256) channel_sum_final_kernel(const float* __restrict__ partial, void* __restrict__ out, long ldo,
                                                                int out_bf16, float scale, int C, int chunks) {
  const int n = blockIdx.y;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float* p = partial + static_cast<size_t>(n) * chunks * C + c;
  float s = 0.f;
  for (int k = 0; k < chunks; ++k) s += p[static_cast<size_t>(k) * C];
  s *= scale;
  if (out_bf16)
    static_cast<bf16*>(out)[n * ldo + c] = __float2bfloat16_rn(s);
  else
    static_cast<float*>(out)[n * ldo + c] = s;
}

void channel_sum_plan(int N, int HW, int C, int* rows, int* chunks) {
  const int tiles = (C / 8 + kCsVecs - 1) / kCsVecs;
  int want = (kCsTargetCtas + N * tiles - 1) / (N * tiles);
  want = want < 1 ? 1 : want;
  int r = (HW + want - 1) / want;
  r = r < kCsGroups ? kCsGroups : r;                  // at least one row per group
  *rows = r;
  *chunks = (HW + r - 1) / r;
}

// ---- Timesteps(dim, flip_sin_to_cos=True, downscale_freq_shift=0) of float ids (diffusers get_timestep_embedding, fp32):
// emb[b, i*dim + k] = cos(id * f_k), emb[b, i*dim + half + k] = sin(id * f_k), f_k = exp(-ln(10000) k / half).  exp / cos / sin run
// in double (the library is built with --use_fast_math, whose single-precision sin / cos lose accuracy at arguments ~1e3), the
// argument id * f_k is formed in fp32 as torch forms it, and each value is rounded to bf16 once.
__global__ void time_ids_embedding_kernel(const float* __restrict__ ids, bf16* __restrict__ out, long ldo, int B, int n_ids, int dim) {
  const int half = dim / 2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * n_ids * half) return;
  const int k = i % half;
  const int bi = i / half;
  const int b = bi / n_ids, id = bi - b * n_ids;
  const float expo = -9.210340371976184f * static_cast<float>(k) / static_cast<float>(half);
  const float f = static_cast<float>(exp(static_cast<double>(expo)));
  const float a = ids[b * n_ids + id] * f;
  bf16* o = out + b * ldo + id * dim;
  o[k] = __float2bfloat16_rn(static_cast<float>(cos(static_cast<double>(a))));
  o[half + k] = __float2bfloat16_rn(static_cast<float>(sin(static_cast<double>(a))));
}

// ---- SiLU and its input gradient, 8 elements per thread.  Forward: the GEMM epilogue's formula (x / (1 + exp(-x))), so a separate
// SiLU rounds exactly as a fused one.  Backward: dx = dy * s * (1 + x (1 - s)), s = sigmoid(x) (torch's silu_backward).
__global__ void silu_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, long nvec) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= nvec) return;
  float f[8];
  unpack8(x[i], f);
#pragma unroll
  for (int j = 0; j < 8; ++j) f[j] = f[j] / (1.f + expf(-f[j]));
  y[i] = pack8(f);
}
__global__ void silu_bwd_kernel(const uint4* __restrict__ dy, const uint4* __restrict__ x, uint4* __restrict__ dx, long nvec) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= nvec) return;
  float g[8], f[8];
  unpack8(dy[i], g);
  unpack8(x[i], f);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float s = 1.f / (1.f + expf(-f[j]));
    g[j] = g[j] * (s * (1.f + f[j] * (1.f - s)));
  }
  dx[i] = pack8(g);
}

__global__ void broadcast_rows_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, int R, int nv, float scale, long total) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long v = i % nv;
  const long b = i / (static_cast<long>(R) * nv);
  float f[8];
  unpack8(src[b * nv + v], f);
#pragma unroll
  for (int j = 0; j < 8; ++j) f[j] *= scale;
  dst[i] = pack8(f);
}

}  // namespace

size_t channel_sum_workspace(int N, int HW, int C) {
  if (N <= 0 || HW <= 0 || C <= 0 || C % 8) return 0;
  int rows, chunks;
  channel_sum_plan(N, HW, C, &rows, &chunks);
  return static_cast<size_t>(N) * chunks * C * sizeof(float);
}

int channel_sum_nhwc(const void* x, void* out, long ldo, int out_bf16, float scale, int N, int HW, int C, void* workspace,
                     size_t ws_bytes, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(x, workspace);
  if (N <= 0 || HW <= 0 || C <= 0 || C % 8 || ldo < C || !out) return DLLM_ERR_SHAPE;
  if (ws_bytes < channel_sum_workspace(N, HW, C)) return DLLM_ERR_SHAPE;
  int rows, chunks;
  channel_sum_plan(N, HW, C, &rows, &chunks);
  float* partial = static_cast<float*>(workspace);
  const int tiles = (C / 8 + kCsVecs - 1) / kCsVecs;
  channel_sum_partial_kernel<<<dim3(chunks, tiles, N), kCsVecs * kCsGroups, 0, s>>>((const bf16*)x, partial, HW, C, rows, chunks);
  channel_sum_final_kernel<<<dim3((C + 255) / 256, N), 256, 0, s>>>(partial, out, ldo, out_bf16, scale, C, chunks);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

int time_ids_embedding(const float* ids, void* out, long ldo, int B, int n_ids, int dim, cudaStream_t s) {
  if (B <= 0 || n_ids <= 0 || dim <= 0 || dim % 2 || ldo < static_cast<long>(n_ids) * dim || !ids || !out) return DLLM_ERR_SHAPE;
  const int total = B * n_ids * (dim / 2);
  time_ids_embedding_kernel<<<(total + 127) / 128, 128, 0, s>>>(ids, (bf16*)out, ldo, B, n_ids, dim);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

int silu_bf16(const void* x, void* y, long n, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(x, y);
  if (n <= 0 || n % 8) return DLLM_ERR_SHAPE;
  const long nvec = n / 8;
  silu_kernel<<<static_cast<unsigned>((nvec + 255) / 256), 256, 0, s>>>((const uint4*)x, (uint4*)y, nvec);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

int silu_bwd_bf16(const void* dy, const void* x, void* dx, long n, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(dy, x, dx);
  if (n <= 0 || n % 8) return DLLM_ERR_SHAPE;
  const long nvec = n / 8;
  silu_bwd_kernel<<<static_cast<unsigned>((nvec + 255) / 256), 256, 0, s>>>((const uint4*)dy, (const uint4*)x, (uint4*)dx, nvec);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

int broadcast_rows(const void* src, void* dst, int B, int R, int H, float scale, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(src, dst);
  if (B <= 0 || R <= 0 || H <= 0 || H % 8) return DLLM_ERR_SHAPE;
  const long total = static_cast<long>(B) * R * (H / 8);
  broadcast_rows_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>((const uint4*)src, (uint4*)dst, R, H / 8, scale, total);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

}  // namespace dllm
