// Sharded AdamW step + gradient sum-of-squares for the data-parallel optimizer (SURVEY.md §8f row 4; sm_90a).
//
// Replaces, for one rank's shard of a flat gradient bucket, what the reference gets from HF Trainer:
//   `optim="adamw_torch"` (projects/dreamllm/configs/stage1/base.py:85, stage2/base.py:95) on a model loaded in bf16
//   (projects/dreamllm/train.py:68-70, :138) under FSDP `shard_grad_op` (stage2/base.py:91-94), with
//   `clip_grad_norm_(max_grad_norm)` before the step (omni/train/trainer.py:800-807).
//
// Both kernels are HBM-bound streaming passes (no reuse): 128-bit vector accesses, grid-stride over 132 x 8 CTAs (one H100 SXM).
//   adamw_kernel<false>: fp32 master / m / v shard, bf16 grad in, bf16 param out : 14 B read + 14 B written per element
//   adamw_kernel<true> : bf16 param / m / v (the reference's arithmetic: every ATen op of torch.optim.AdamW's
//                        single-tensor path rounds its result to bf16)          :  8 B read +  6 B written per element
//   sumsq: 2 B read per element, deterministic two-stage reduction (per-CTA partials -> one CTA), accumulates into *out.
// Arithmetic uses the _rn intrinsics so --use_fast_math cannot contract or approximate it (parity with the CPU optimizer).
#include "common.cuh"
#include "ops.h"

#include "../../include/dreamllm_sm100.h"

namespace dllm {

namespace {
struct alignas(16) BVec8 {
  __nv_bfloat162 v[4];
};
__device__ __forceinline__ void bunpack8(const BVec8& p, float* f) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(p.v[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ BVec8 bpack8(const float* f) {
  BVec8 p;
#pragma unroll
  for (int i = 0; i < 4; ++i) p.v[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return p;
}
// 128-bit accesses spelled as uint4: a struct copy of BVec8 compiles to four 32-bit LDG/STG (checked in SASS)
__device__ __forceinline__ BVec8 ld8(const BVec8* p) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  return *reinterpret_cast<const BVec8*>(&u);
}
__device__ __forceinline__ void st8(BVec8* p, const BVec8& v) { *reinterpret_cast<uint4*>(p) = *reinterpret_cast<const uint4*>(&v); }
__device__ __forceinline__ float rbf(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

struct AdamWArgs {
  float decay;      // 1 - lr * weight_decay
  float w1;         // 1 - beta1
  float beta2;
  float w2;         // 1 - beta2
  float bc2_sqrt;   // sqrt(1 - beta2^t)
  float eps;
  float neg_step;   // -lr / (1 - beta1^t)
  float max_norm;   // <= 0: no clipping
};

// clip coefficient of torch.nn.utils.clip_grad_norm_: min(1, max_norm / (total_norm + 1e-6))
__device__ __forceinline__ float clip_coef(const float* __restrict__ sumsq, float max_norm) {
  if (sumsq == nullptr || !(max_norm > 0.f)) return 1.f;
  const float norm = __fsqrt_rn(*sumsq);
  return fminf(1.f, __fdiv_rn(max_norm, __fadd_rn(norm, 1e-6f)));
}

// One element of torch.optim.AdamW (single-tensor path, torch/optim/adamw.py `_single_tensor_adamw`):
//   p.mul_(1 - lr*wd); m.lerp_(g, 1-b1); v.mul_(b2).addcmul_(g, g, value=1-b2);
//   denom = (v.sqrt() / bias_correction2_sqrt).add_(eps); p.addcdiv_(m, denom, value=-lr/bias_correction1)
// kRound = true rounds after every ATen op (bf16 tensors); false keeps fp32 throughout (fp32 master weights).
template <bool kRound>
__device__ __forceinline__ void adamw_elem(float g, float& p, float& m, float& v, const AdamWArgs& a) {
  auto R = [](float x) { return kRound ? rbf(x) : x; };
  p = R(__fmul_rn(p, a.decay));
  m = R(__fadd_rn(m, __fmul_rn(a.w1, __fsub_rn(g, m))));                 // lerp, weight < 0.5 branch
  v = R(__fmul_rn(v, a.beta2));
  v = R(__fadd_rn(v, __fmul_rn(__fmul_rn(a.w2, g), g)));                 // addcmul: self + (value * t1) * t2
  float d = R(__fsqrt_rn(v));
  d = R(__fdiv_rn(d, a.bc2_sqrt));
  d = R(__fadd_rn(d, a.eps));
  p = R(__fadd_rn(p, __fdiv_rn(__fmul_rn(a.neg_step, m), d)));           // addcdiv: self + (value * t1) / t2
}

template <bool kBf16State>
__global__ void __launch_bounds__(256) adamw_kernel(const BVec8* __restrict__ grad, void* __restrict__ master, void* __restrict__ mom,
                                                    void* __restrict__ var, BVec8* __restrict__ param, long nvec, AdamWArgs a,
                                                    const float* __restrict__ sumsq) {
  const float coef = clip_coef(sumsq, a.max_norm);
  const long stride = static_cast<long>(gridDim.x) * blockDim.x;
  for (long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += stride) {
    float g[8], p[8], m[8], v[8];
    bunpack8(ld8(grad + i), g);
    if constexpr (kBf16State) {
      bunpack8(ld8(param + i), p);
      bunpack8(ld8(reinterpret_cast<const BVec8*>(mom) + i), m);
      bunpack8(ld8(reinterpret_cast<const BVec8*>(var) + i), v);
    } else {
      const float4* w4 = reinterpret_cast<const float4*>(master) + 2 * i;
      const float4* m4 = reinterpret_cast<const float4*>(mom) + 2 * i;
      const float4* v4 = reinterpret_cast<const float4*>(var) + 2 * i;
      *reinterpret_cast<float4*>(p) = w4[0];
      *reinterpret_cast<float4*>(p + 4) = w4[1];
      *reinterpret_cast<float4*>(m) = m4[0];
      *reinterpret_cast<float4*>(m + 4) = m4[1];
      *reinterpret_cast<float4*>(v) = v4[0];
      *reinterpret_cast<float4*>(v + 4) = v4[1];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float gj = g[j];
      if (coef != 1.f) gj = kBf16State ? rbf(__fmul_rn(gj, coef)) : __fmul_rn(gj, coef);   // clip_grad_norm_: g.mul_(coef)
      adamw_elem<kBf16State>(gj, p[j], m[j], v[j], a);
    }
    if constexpr (kBf16State) {
      st8(reinterpret_cast<BVec8*>(mom) + i, bpack8(m));
      st8(reinterpret_cast<BVec8*>(var) + i, bpack8(v));
    } else {
      float4* w4 = reinterpret_cast<float4*>(master) + 2 * i;
      float4* m4 = reinterpret_cast<float4*>(mom) + 2 * i;
      float4* v4 = reinterpret_cast<float4*>(var) + 2 * i;
      w4[0] = *reinterpret_cast<float4*>(p);
      w4[1] = *reinterpret_cast<float4*>(p + 4);
      m4[0] = *reinterpret_cast<float4*>(m);
      m4[1] = *reinterpret_cast<float4*>(m + 4);
      v4[0] = *reinterpret_cast<float4*>(v);
      v4[1] = *reinterpret_cast<float4*>(v + 4);
    }
    st8(param + i, bpack8(p));
  }
}

constexpr int kSumsqBlocks = 132 * 4;   // 4 CTAs per H100 SM

__global__ void __launch_bounds__(256) sumsq_partial_kernel(const BVec8* __restrict__ x, long nvec, float* __restrict__ partials) {
  __shared__ float red[8];
  float acc = 0.f;
  const long stride = static_cast<long>(gridDim.x) * blockDim.x;
  for (long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += stride) {
    float f[8];
    bunpack8(ld8(x + i), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc = fmaf(f[j], f[j], acc);
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < 8 ? red[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0) partials[blockIdx.x] = t;
  }
}
__global__ void __launch_bounds__(1024) sumsq_final_kernel(const float* __restrict__ partials, int n, float* __restrict__ out,
                                                           int accumulate) {
  __shared__ float red[32];
  float acc = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) acc += partials[i];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = red[threadIdx.x];
    t = warp_sum(t);
    if (threadIdx.x == 0) out[0] = accumulate ? out[0] + t : t;
  }
}
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
}  // namespace

int adamw_step(const void* grad, void* master, void* mom, void* var, void* param, long n, int bf16_state, double lr, double beta1,
               double beta2, double eps, double weight_decay, int step, const float* sumsq, double max_norm, cudaStream_t s) {
  if (n < 0 || (n & 7) || step < 1) return DLLM_ERR_SHAPE;
  if (n == 0) return 0;
  if (!grad || !mom || !var || !param || (!bf16_state && !master)) return DLLM_ERR_SHAPE;
  if (!aligned16(grad) || !aligned16(mom) || !aligned16(var) || !aligned16(param) || (!bf16_state && !aligned16(master)))
    return DLLM_ERR_ALIGN;
  // scalars in double, as Python computes them in torch/optim/adamw.py, then narrowed once to the fp32 opmath type
  const double bc1 = 1.0 - pow(beta1, step);
  const double bc2 = 1.0 - pow(beta2, step);
  AdamWArgs a;
  a.decay = static_cast<float>(1.0 - lr * weight_decay);
  a.w1 = static_cast<float>(1.0 - beta1);
  a.beta2 = static_cast<float>(beta2);
  a.w2 = static_cast<float>(1.0 - beta2);
  a.bc2_sqrt = static_cast<float>(sqrt(bc2));
  a.eps = static_cast<float>(eps);
  a.neg_step = static_cast<float>(-(lr / bc1));
  a.max_norm = static_cast<float>(max_norm);
  const long nvec = n >> 3;
  const int blocks = static_cast<int>(std::min<long>((nvec + 255) / 256, 132L * 8));
  if (bf16_state)
    adamw_kernel<true><<<blocks, 256, 0, s>>>(reinterpret_cast<const BVec8*>(grad), nullptr, mom, var, reinterpret_cast<BVec8*>(param),
                                              nvec, a, sumsq);
  else
    adamw_kernel<false><<<blocks, 256, 0, s>>>(reinterpret_cast<const BVec8*>(grad), master, mom, var, reinterpret_cast<BVec8*>(param),
                                               nvec, a, sumsq);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

size_t sumsq_workspace() { return static_cast<size_t>(kSumsqBlocks) * sizeof(float); }

int sumsq_bf16(const void* x, long n, float* out, int accumulate, void* workspace, size_t ws_bytes, cudaStream_t s) {
  if (n < 0 || (n & 7) || !out) return DLLM_ERR_SHAPE;
  if (ws_bytes < sumsq_workspace() || !workspace) return DLLM_ERR_SHAPE;
  if (n > 0 && !aligned16(x)) return DLLM_ERR_ALIGN;
  const long nvec = n >> 3;
  const int blocks = static_cast<int>(std::max<long>(1, std::min<long>((nvec + 255) / 256, kSumsqBlocks)));
  sumsq_partial_kernel<<<blocks, 256, 0, s>>>(reinterpret_cast<const BVec8*>(x), nvec, reinterpret_cast<float*>(workspace));
  sumsq_final_kernel<<<1, 1024, 0, s>>>(reinterpret_cast<const float*>(workspace), blocks, out, accumulate);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

}  // namespace dllm
