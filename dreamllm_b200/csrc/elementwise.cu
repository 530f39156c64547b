// HBM-bound kernels of the DreamLLM decoder path (sm_90a): RMSNorm fwd/bwd (+fused residual add),
// RoPE (in place on the fused qkv buffer), SwiGLU fwd/bwd, shifted masked cross-entropy (fwd + in-place
// dlogits), embedding gather / sorted segment scatter, bf16 add.
// All move 8-element (16-byte) vectors per thread (128-bit LDG/STG, see the Vec8 note below), fp32 math, warp-shuffle reductions; rounding points follow the
// reference's bf16 eager path (cited per kernel) so bf16-vs-bf16 parity holds to the last place where cheap.
#include "common.cuh"
#include "gemm_sm90.h"

namespace dllm {

// 8 bf16 = one 16-byte vector.  The single uint4 member makes every copy of the struct one LDG.E.128 / STG.E.128; the earlier
// `__nv_bfloat162 v[4]` layout was split by nvcc into four 32-bit accesses (4x the LSU / L1 wavefronts: rmsnorm 0.62 -> 0.75, rope
// 0.63 -> 0.68, layernorm 0.47 -> 0.67 of the HBM copy peak on the same box, profiles/r02_ab_hbm_flags.txt).  Row starts must be 16-byte
// aligned (true for every caller: widths and strides are multiples of 8 elements); the host wrappers check the base pointers.
struct alignas(16) Vec8 {
  uint4 u;
  __device__ __forceinline__ __nv_bfloat162 get(int i) const {
    const uint32_t w = (i == 0) ? u.x : (i == 1) ? u.y : (i == 2) ? u.z : u.w;
    return *reinterpret_cast<const __nv_bfloat162*>(&w);
  }
  __device__ __forceinline__ void set(int i, __nv_bfloat162 h) {
    const uint32_t w = *reinterpret_cast<const uint32_t*>(&h);
    if (i == 0) u.x = w; else if (i == 1) u.y = w; else if (i == 2) u.z = w; else u.w = w;
  }
};
__device__ __forceinline__ void unpack8(const Vec8 p, float* f) {   // by value: one 128-bit load per vector
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = __bfloat1622float2(p.get(i));
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ Vec8 pack8(const float* f) {
  Vec8 p;
#pragma unroll
  for (int i = 0; i < 4; ++i) p.set(i, __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]));
  return p;
}
__device__ __forceinline__ float bf16r(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

template <int NT>
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();  // protect `red` from the previous use
  if (l == 0) red[w] = v;
  __syncthreads();
  float t = (l < NT / 32) ? red[l] : 0.f;
  return warp_sum(t);  // every warp reduces the same NT/32 partials -> identical result in all threads
}

// ------------------------------------------------------------------------------------------------ RMSNorm
// reference: DreamLLMRMSNorm.forward, modeling_dreamllm.py:86-91
//   y = w * bf16( x32 * rsqrt(mean(x32^2) + eps) )        (cast BEFORE the weight multiply, :91)
// fused option: x <- x + add (bf16 add as the residual `residual + hidden_states`, :638/:644) written to x_out.
constexpr int kNormThreads = 256;
constexpr int kNormMaxV = 4;  // hidden <= 256 * 4 * 8 = 8192

__global__ void __launch_bounds__(kNormThreads) rmsnorm_fwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ add,
                                                                   const bf16* __restrict__ w, bf16* __restrict__ x_out,
                                                                   bf16* __restrict__ y, float* __restrict__ rstd_out,
                                                                   int H, float eps) {
  __shared__ float red[kNormThreads / 32];
  const int row = blockIdx.x;
  const int nvec = H >> 3;
  const Vec8* xr = reinterpret_cast<const Vec8*>(x + static_cast<size_t>(row) * H);
  const Vec8* ar = add ? reinterpret_cast<const Vec8*>(add + static_cast<size_t>(row) * H) : nullptr;
  float xv[kNormMaxV][8];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < kNormMaxV; ++i) {
    const int v = threadIdx.x + i * kNormThreads;
    if (v < nvec) {
      unpack8(xr[v], xv[i]);
      if (ar) {
        float a[8];
        unpack8(ar[v], a);
#pragma unroll
        for (int j = 0; j < 8; ++j) xv[i][j] = bf16r(xv[i][j] + a[j]);
        if (x_out) reinterpret_cast<Vec8*>(x_out + static_cast<size_t>(row) * H)[v] = pack8(xv[i]);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) ss += xv[i][j] * xv[i][j];
    }
  }
  ss = block_sum<kNormThreads>(ss, red);
  const float rstd = rsqrtf(ss / static_cast<float>(H) + eps);
  if (threadIdx.x == 0 && rstd_out) rstd_out[row] = rstd;
  const Vec8* wr = reinterpret_cast<const Vec8*>(w);
  Vec8* yr = reinterpret_cast<Vec8*>(y + static_cast<size_t>(row) * H);
#pragma unroll
  for (int i = 0; i < kNormMaxV; ++i) {
    const int v = threadIdx.x + i * kNormThreads;
    if (v < nvec) {
      float wf[8], o[8];
      unpack8(wr[v], wf);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = wf[j] * bf16r(xv[i][j] * rstd);
      yr[v] = pack8(o);
    }
  }
}

// backward, two kernels (the first fused version kept dw partials in registers: 161 regs, 12 % occupancy, 18 % of DRAM
// peak in ncu — profiles/r01_ncu_full_summary.csv):
//   dx kernel : one CTA per row.  g = bf16(dy*w); dx = rstd*(g - xhat*mean(g*xhat)) (+ dres)
//   dw kernel : 2-D grid (256-column blocks x row splits); dw_partial[split, h] = sum_rows dy * bf16(x*rstd)
__global__ void __launch_bounds__(kNormThreads) rmsnorm_bwd_dx_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                                                                      const bf16* __restrict__ w, const float* __restrict__ rstd,
                                                                      const bf16* __restrict__ dres, bf16* __restrict__ dx, int H) {
  __shared__ float red[kNormThreads / 32];
  const int row = blockIdx.x;
  const int nvec = H >> 3;
  const size_t off = static_cast<size_t>(row) * H;
  const float rs = rstd[row];
  float g[kNormMaxV][8], xh[kNormMaxV][8];
  float dot = 0.f;
#pragma unroll
  for (int i = 0; i < kNormMaxV; ++i) {
    const int v = threadIdx.x + i * kNormThreads;
    if (v < nvec) {
      float d[8], xx[8], wf[8];
      unpack8(reinterpret_cast<const Vec8*>(dy + off)[v], d);
      unpack8(reinterpret_cast<const Vec8*>(x + off)[v], xx);
      unpack8(reinterpret_cast<const Vec8*>(w)[v], wf);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        xh[i][j] = xx[j] * rs;
        g[i][j] = bf16r(d[j] * wf[j]);
        dot += g[i][j] * xh[i][j];
      }
    }
  }
  dot = block_sum<kNormThreads>(dot, red) / static_cast<float>(H);
#pragma unroll
  for (int i = 0; i < kNormMaxV; ++i) {
    const int v = threadIdx.x + i * kNormThreads;
    if (v < nvec) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = rs * (g[i][j] - xh[i][j] * dot);
      if (dres) {
        float r[8];
        unpack8(reinterpret_cast<const Vec8*>(dres + off)[v], r);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] += r[j];
      }
      reinterpret_cast<Vec8*>(dx + off)[v] = pack8(o);
    }
  }
}

constexpr int kDwSplits = 64;
__global__ void __launch_bounds__(256) rmsnorm_bwd_dw_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                                                             const float* __restrict__ rstd, float* __restrict__ dw_partial,
                                                             int T, int H) {
  __shared__ float sm[8][32][9];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int v = blockIdx.x * 32 + tx;  // 8-column vector index
  const int nvec = H >> 3;
  const int rows_per = (T + kDwSplits - 1) / kDwSplits;
  const int r0 = blockIdx.y * rows_per;
  const int r1 = min(T, r0 + rows_per);
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (v < nvec) {
#pragma unroll 4
    for (int r = r0 + ty; r < r1; r += 8) {
      const size_t off = static_cast<size_t>(r) * H;
      float d[8], xx[8];
      unpack8(reinterpret_cast<const Vec8*>(dy + off)[v], d);
      unpack8(reinterpret_cast<const Vec8*>(x + off)[v], xx);
      const float rs = __ldg(rstd + r);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += d[j] * bf16r(xx[j] * rs);
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) sm[ty][tx][j] = acc[j];
  __syncthreads();
  if (ty == 0 && v < nvec) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float s = 0.f;
#pragma unroll
      for (int y = 0; y < 8; ++y) s += sm[y][tx][j];
      dw_partial[static_cast<size_t>(blockIdx.y) * H + v * 8 + j] = s;
    }
  }
}

// dw[h] (+)= sum_p partial[p, h]
__global__ void colsum_partials_kernel(const float* __restrict__ partial, bf16* __restrict__ dw, int P, int H,
                                       int accumulate) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= H) return;
  float s = 0.f;
  for (int p = 0; p < P; ++p) s += partial[static_cast<size_t>(p) * H + h];
  if (accumulate) s += __bfloat162float(dw[h]);
  dw[h] = __float2bfloat16_rn(s);
}

int rmsnorm_fwd(const void* x, const void* add, const void* w, void* x_out, void* y, float* rstd, int T, int H,
                float eps, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(x, add, w, x_out, y);
  if (H % 8 || H > kNormThreads * kNormMaxV * 8 || T <= 0) return DLLM_ERR_SHAPE;
  rmsnorm_fwd_kernel<<<T, kNormThreads, 0, s>>>((const bf16*)x, (const bf16*)add, (const bf16*)w, (bf16*)x_out, (bf16*)y,
                                                rstd, H, eps);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

size_t rmsnorm_bwd_workspace(int T, int H) { return static_cast<size_t>(kDwSplits) * H * sizeof(float); }

int rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd, const void* dres, void* dx, void* dw,
                int dw_accumulate, void* workspace, size_t workspace_bytes, int T, int H, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(dy, x, w, dres, dx);
  if (H % 8 || H > kNormThreads * kNormMaxV * 8 || T <= 0) return DLLM_ERR_SHAPE;
  if (dw && workspace_bytes < rmsnorm_bwd_workspace(T, H)) return DLLM_ERR_SHAPE;
  rmsnorm_bwd_dx_kernel<<<T, kNormThreads, 0, s>>>((const bf16*)dy, (const bf16*)x, (const bf16*)w, rstd, (const bf16*)dres,
                                                   (bf16*)dx, H);
  if (dw) {
    dim3 grid((H / 8 + 31) / 32, kDwSplits);
    rmsnorm_bwd_dw_kernel<<<grid, 256, 0, s>>>((const bf16*)dy, (const bf16*)x, rstd, (float*)workspace, T, H);
    colsum_partials_kernel<<<(H + 255) / 256, 256, 0, s>>>((const float*)workspace, (bf16*)dw, kDwSplits, H, dw_accumulate);
  }
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// ------------------------------------------------------------------------------------------------ RoPE
// reference: apply_rotary_pos_emb / rotate_half, modeling_dreamllm.py:176-209 (half-split), tables rounded to the
// model dtype (:126-127).  In place on `n_tensors` consecutive [T, nh*d] column blocks of a row-major buffer with row
// stride ld (the fused qkv buffer: q at column 0, k at column nh*d).  mode +1 = forward, -1 = backward (transpose).
template <int D>
__global__ void rope_kernel(bf16* __restrict__ buf, const bf16* __restrict__ cos_t, const bf16* __restrict__ sin_t,
                            const int* __restrict__ pos, long ld, int T, int heads_total, int mode) {
  constexpr int VPH = D / 16;  // threads per head: each handles 8 elements of the first half + their partners
  const long gid = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long total = static_cast<long>(T) * heads_total * VPH;
  if (gid >= total) return;
  const int vi = static_cast<int>(gid % VPH);
  const long th = gid / VPH;
  const int head = static_cast<int>(th % heads_total);
  const int t = static_cast<int>(th / heads_total);
  const int p = pos[t];
  bf16* base = buf + static_cast<size_t>(t) * ld + static_cast<size_t>(head) * D + vi * 8;
  float a[8], b[8], c1[8], c2[8], s1[8], s2[8];
  const Vec8 va{*reinterpret_cast<const uint4*>(base)}, vb{*reinterpret_cast<const uint4*>(base + D / 2)};   // whole-vector loads
  unpack8(va, a);
  unpack8(vb, b);
  unpack8(*reinterpret_cast<const Vec8*>(cos_t + static_cast<size_t>(p) * D + vi * 8), c1);
  unpack8(*reinterpret_cast<const Vec8*>(cos_t + static_cast<size_t>(p) * D + D / 2 + vi * 8), c2);
  unpack8(*reinterpret_cast<const Vec8*>(sin_t + static_cast<size_t>(p) * D + vi * 8), s1);
  unpack8(*reinterpret_cast<const Vec8*>(sin_t + static_cast<size_t>(p) * D + D / 2 + vi * 8), s2);
  float o1[8], o2[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    if (mode > 0) {
      // q'[i] = q[i] cos[i] + (-q[i+D/2]) sin[i];   q'[i+D/2] = q[i+D/2] cos[i+D/2] + q[i] sin[i+D/2]
      o1[j] = bf16r(a[j] * c1[j]) + bf16r(-b[j] * s1[j]);
      o2[j] = bf16r(b[j] * c2[j]) + bf16r(a[j] * s2[j]);
    } else {
      // dq[i] = g[i] cos[i] + g[i+D/2] sin[i+D/2];  dq[i+D/2] = g[i+D/2] cos[i+D/2] - g[i] sin[i]
      o1[j] = bf16r(a[j] * c1[j]) + bf16r(b[j] * s2[j]);
      o2[j] = bf16r(b[j] * c2[j]) + bf16r(-a[j] * s1[j]);
    }
  }
  *reinterpret_cast<Vec8*>(base) = pack8(o1);
  *reinterpret_cast<Vec8*>(base + D / 2) = pack8(o2);
}

int rope_inplace(void* buf, const void* cos_t, const void* sin_t, const int* pos, long ld, int T, int heads_total,
                 int head_dim, int mode, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(buf, cos_t, sin_t);
  if (T <= 0 || heads_total <= 0 || (ld % 8)) return DLLM_ERR_SHAPE;
  const int vph = head_dim / 16;
  const long total = static_cast<long>(T) * heads_total * vph;
  const int nt = 256;
  const unsigned grid = static_cast<unsigned>((total + nt - 1) / nt);
  if (head_dim == 128)
    rope_kernel<128><<<grid, nt, 0, s>>>((bf16*)buf, (const bf16*)cos_t, (const bf16*)sin_t, pos, ld, T, heads_total, mode);
  else if (head_dim == 64)
    rope_kernel<64><<<grid, nt, 0, s>>>((bf16*)buf, (const bf16*)cos_t, (const bf16*)sin_t, pos, ld, T, heads_total, mode);
  else
    return DLLM_ERR_UNSUPPORTED;
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// ------------------------------------------------------------------------------------------------ SwiGLU
// reference: DreamLLMMLP.forward, modeling_dreamllm.py:237: act = bf16( bf16(silu(g)) * u )
// gu is the fused gate|up GEMM output [T, 2I] (gate at column 0, up at column I), row stride ld_gu.
__global__ void swiglu_fwd_kernel(const bf16* __restrict__ gu, bf16* __restrict__ act, long ld_gu, int T, int I) {
  const int nvec = I >> 3;
  const long gid = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (gid >= static_cast<long>(T) * nvec) return;
  const int v = static_cast<int>(gid % nvec);
  const long t = gid / nvec;
  float g[8], u[8], o[8];
  unpack8(*reinterpret_cast<const Vec8*>(gu + t * ld_gu + v * 8), g);
  unpack8(*reinterpret_cast<const Vec8*>(gu + t * ld_gu + I + v * 8), u);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float s = bf16r(g[j] / (1.f + expf(-g[j])));
    o[j] = s * u[j];
  }
  *reinterpret_cast<Vec8*>(act + t * static_cast<long>(I) + v * 8) = pack8(o);
}

// d_gu[:, :I] = bf16(dact*u) * silu'(g);  d_gu[:, I:] = dact * bf16(silu(g))
__global__ void swiglu_bwd_kernel(const bf16* __restrict__ dact, const bf16* __restrict__ gu, bf16* __restrict__ dgu,
                                  long ld_gu, int T, int I) {
  const int nvec = I >> 3;
  const long gid = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (gid >= static_cast<long>(T) * nvec) return;
  const int v = static_cast<int>(gid % nvec);
  const long t = gid / nvec;
  float g[8], u[8], d[8], og[8], ou[8];
  unpack8(*reinterpret_cast<const Vec8*>(gu + t * ld_gu + v * 8), g);
  unpack8(*reinterpret_cast<const Vec8*>(gu + t * ld_gu + I + v * 8), u);
  unpack8(*reinterpret_cast<const Vec8*>(dact + t * static_cast<long>(I) + v * 8), d);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float sig = 1.f / (1.f + expf(-g[j]));
    const float s = bf16r(g[j] * sig);
    const float ds = bf16r(d[j] * u[j]);
    og[j] = ds * (sig * (1.f + g[j] * (1.f - sig)));
    ou[j] = d[j] * s;
  }
  *reinterpret_cast<Vec8*>(dgu + t * ld_gu + v * 8) = pack8(og);
  *reinterpret_cast<Vec8*>(dgu + t * ld_gu + I + v * 8) = pack8(ou);
}

int swiglu_fwd(const void* gu, void* act, long ld_gu, int T, int I, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(gu, act);
  if (I % 8 || ld_gu % 8 || T <= 0) return DLLM_ERR_SHAPE;
  const long total = static_cast<long>(T) * (I / 8);
  swiglu_fwd_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>((const bf16*)gu, (bf16*)act, ld_gu, T, I);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}
int swiglu_bwd(const void* dact, const void* gu, void* dgu, long ld_gu, int T, int I, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(dact, gu, dgu);
  if (I % 8 || ld_gu % 8 || T <= 0) return DLLM_ERR_SHAPE;
  const long total = static_cast<long>(T) * (I / 8);
  swiglu_bwd_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>((const bf16*)dact, (const bf16*)gu, (bf16*)dgu,
                                                                          ld_gu, T, I);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// ------------------------------------------------------------------------------------------------ add
__global__ void add_kernel(const bf16* __restrict__ a, const bf16* __restrict__ b, bf16* __restrict__ o, long nvec) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= nvec) return;
  float x[8], y[8];
  unpack8(reinterpret_cast<const Vec8*>(a)[i], x);
  unpack8(reinterpret_cast<const Vec8*>(b)[i], y);
#pragma unroll
  for (int j = 0; j < 8; ++j) x[j] += y[j];
  reinterpret_cast<Vec8*>(o)[i] = pack8(x);
}
int add_bf16(const void* a, const void* b, void* o, long n, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(a, b, o);
  if (n % 8 || n <= 0) return DLLM_ERR_SHAPE;
  const long nvec = n / 8;
  add_kernel<<<static_cast<unsigned>((nvec + 255) / 256), 256, 0, s>>>((const bf16*)a, (const bf16*)b, (bf16*)o, nvec);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// ------------------------------------------------------------------------------------------------ cross entropy
// reference: DreamLLMForCausalMLM.forward, modeling_dreamllm.py:1453-1470: logits.float(); shift; CE(reduction none);
// masked mean over labels != -100 (0 when there is no valid label).  `labels` here are ALREADY shifted by the host
// (labels[t] = target of row t, -100 for the last position of every sequence and for ignored targets).
// One CTA per row: online max/sum-exp in fp32, then dlogits written IN PLACE over the bf16 logits:
//   dlogits = (softmax - onehot) * dloss / n_valid.
constexpr int kCeThreads = 256;

__global__ void ce_count_kernel(const long long* __restrict__ labels, int T, float* __restrict__ inv_count) {
  __shared__ float red[kCeThreads / 32];
  float c = 0.f;
  for (int i = threadIdx.x; i < T; i += kCeThreads) c += (labels[i] != -100) ? 1.f : 0.f;
  c = block_sum<kCeThreads>(c, red);
  if (threadIdx.x == 0) {
    inv_count[0] = c > 0.f ? 1.f / c : 0.f;
    inv_count[1] = c;
  }
}

__global__ void __launch_bounds__(kCeThreads) ce_fwd_bwd_kernel(bf16* __restrict__ logits, const long long* __restrict__ labels,
                                                                 float* __restrict__ row_loss, const float* __restrict__ inv_count,
                                                                 float dloss, long ld, int V, int write_grad) {
  __shared__ float red[kCeThreads / 32];
  __shared__ float red2[kCeThreads / 32];
  const int row = blockIdx.x;
  const long long label = labels[row];
  bf16* lr = logits + static_cast<size_t>(row) * ld;
  const int nvec = V >> 3;
  if (label == -100) {
    if (threadIdx.x == 0) row_loss[row] = 0.f;
    if (write_grad) {
      Vec8 z;
#pragma unroll
      for (int i = 0; i < 4; ++i) z.set(i, __floats2bfloat162_rn(0.f, 0.f));
      for (int v = threadIdx.x; v < nvec; v += kCeThreads) reinterpret_cast<Vec8*>(lr)[v] = z;
    }
    return;
  }
  // pass 1: online logsumexp
  float m = -INFINITY, ssum = 0.f;
  for (int v = threadIdx.x; v < nvec; v += kCeThreads) {
    float f[8];
    unpack8(reinterpret_cast<const Vec8*>(lr)[v], f);
    float mx = f[0];
#pragma unroll
    for (int j = 1; j < 8; ++j) mx = fmaxf(mx, f[j]);
    const float mn = fmaxf(m, mx);
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc += expf(f[j] - mn);
    ssum = ssum * expf(m - mn) + acc;
    m = mn;
  }
  // block combine (max then rescaled sums)
  float wm = warp_max(m);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) red[w] = wm;
  __syncthreads();
  float bm = (l < kCeThreads / 32) ? red[l] : -INFINITY;
  bm = warp_max(bm);
  float sc = (m == -INFINITY) ? 0.f : ssum * expf(m - bm);
  sc = warp_sum(sc);
  if (l == 0) red2[w] = sc;
  __syncthreads();
  float bs = (l < kCeThreads / 32) ? red2[l] : 0.f;
  bs = warp_sum(bs);
  const float lse = bm + logf(bs);
  if (threadIdx.x == 0) row_loss[row] = lse - __bfloat162float(lr[label]);
  if (!write_grad) return;
  __syncthreads();  // everyone has read lr[label] / finished pass 1 before it is overwritten
  const float scale = dloss * inv_count[0];
  for (int v = threadIdx.x; v < nvec; v += kCeThreads) {
    float f[8];
    unpack8(reinterpret_cast<const Vec8*>(lr)[v], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float p = expf(f[j] - lse);
      if (v * 8 + j == label) p -= 1.f;
      f[j] = p * scale;
    }
    reinterpret_cast<Vec8*>(lr)[v] = pack8(f);
  }
}

__global__ void ce_reduce_kernel(const float* __restrict__ row_loss, int T, const float* __restrict__ inv_count,
                                 float* __restrict__ loss) {
  __shared__ float red[kCeThreads / 32];
  float s = 0.f;
  for (int i = threadIdx.x; i < T; i += kCeThreads) s += row_loss[i];
  s = block_sum<kCeThreads>(s, red);
  if (threadIdx.x == 0) loss[0] = s * inv_count[0];
}

// workspace: float[T + 2] (row losses, then {1/n_valid, n_valid})
int cross_entropy(void* logits, const long long* labels, float* loss, float dloss, void* workspace, long ld, int T,
                  int V, int write_grad, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(logits);
  if (V % 8 || ld % 8 || T <= 0) return DLLM_ERR_SHAPE;
  float* row_loss = static_cast<float*>(workspace);
  float* inv_count = row_loss + T;
  ce_count_kernel<<<1, kCeThreads, 0, s>>>(labels, T, inv_count);
  ce_fwd_bwd_kernel<<<T, kCeThreads, 0, s>>>((bf16*)logits, labels, row_loss, inv_count, dloss, ld, V, write_grad);
  ce_reduce_kernel<<<1, kCeThreads, 0, s>>>(row_loss, T, inv_count, loss);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// ------------------------------------------------------------------------------------------------ embedding
// reference: embed_tokens lookup, modeling_dreamllm.py:1066-1067 (index path: bit-exact row copies)
__global__ void embedding_fwd_kernel(const long long* __restrict__ ids, const bf16* __restrict__ W, bf16* __restrict__ out,
                                     int T, int H) {
  const int nvec = H >> 3;
  const long gid = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (gid >= static_cast<long>(T) * nvec) return;
  const int v = static_cast<int>(gid % nvec);
  const long t = gid / nvec;
  const long long id = ids[t];
  reinterpret_cast<uint4*>(out + t * H)[v] = reinterpret_cast<const uint4*>(W + static_cast<size_t>(id) * H)[v];
}
// Deterministic scatter-add: `order` is the argsort of ids, `sorted_ids` = ids[order]. Block p handles the segment
// that STARTS at sorted position p (others exit): dW[id] (+)= sum over the segment of dy[order[q]] (fp32 accumulate).
__global__ void embedding_bwd_kernel(const long long* __restrict__ sorted_ids, const long long* __restrict__ order,
                                     const bf16* __restrict__ dy, bf16* __restrict__ dW, int T, int H, int accumulate) {
  const int p = blockIdx.x;
  const long long id = sorted_ids[p];
  if (p > 0 && sorted_ids[p - 1] == id) return;
  const int nvec = H >> 3;
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    for (int q = p; q < T && sorted_ids[q] == id; ++q) {
      float f[8];
      unpack8(reinterpret_cast<const Vec8*>(dy + static_cast<size_t>(order[q]) * H)[v], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += f[j];
    }
    Vec8* dst = reinterpret_cast<Vec8*>(dW + static_cast<size_t>(id) * H) + v;
    if (accumulate) {
      float f[8];
      unpack8(*dst, f);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += f[j];
    }
    *dst = pack8(acc);
  }
}
int embedding_fwd(const long long* ids, const void* W, void* out, int T, int H, cudaStream_t s) {
  if (H % 8 || T <= 0) return DLLM_ERR_SHAPE;
  const long total = static_cast<long>(T) * (H / 8);
  embedding_fwd_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>(ids, (const bf16*)W, (bf16*)out, T, H);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}
int embedding_bwd(const long long* sorted_ids, const long long* order, const void* dy, void* dW, int T, int H,
                  int accumulate, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(dy, dW);
  if (H % 8 || T <= 0) return DLLM_ERR_SHAPE;
  embedding_bwd_kernel<<<T, 128, 0, s>>>(sorted_ids, order, (const bf16*)dy, (bf16*)dW, T, H, accumulate);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}


// ------------------------------------------------------------------------------------------------ LayerNorm (fwd)
// CLIP ViT / UNet transformer blocks (transformers CLIPEncoderLayer.layer_norm1/2, pre_layrnorm; diffusers
// BasicTransformerBlock.norm1-3): y = (x - mean) * rsqrt(var + eps) * w + b, fp32 statistics, one rounding to bf16.
// Frozen towers on this path (modeling_plugins.py:235-236 freeze CLIP; UNet frozen) -> forward only.
__global__ void __launch_bounds__(kNormThreads) layernorm_fwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                                                                     const bf16* __restrict__ b, bf16* __restrict__ y, int H,
                                                                     float eps) {
  __shared__ float red[kNormThreads / 32];
  const int row = blockIdx.x;
  const int nvec = H >> 3;
  const Vec8* xr = reinterpret_cast<const Vec8*>(x + static_cast<size_t>(row) * H);
  float xv[kNormMaxV][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < kNormMaxV; ++i) {
    const int v = threadIdx.x + i * kNormThreads;
    if (v < nvec) {
      unpack8(xr[v], xv[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += xv[i][j];
    }
  }
  const float mean = block_sum<kNormThreads>(sum, red) / static_cast<float>(H);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < kNormMaxV; ++i) {
    const int v = threadIdx.x + i * kNormThreads;
    if (v < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float d = xv[i][j] - mean; sq += d * d; }
    }
  }
  const float rstd = rsqrtf(block_sum<kNormThreads>(sq, red) / static_cast<float>(H) + eps);
  Vec8* yr = reinterpret_cast<Vec8*>(y + static_cast<size_t>(row) * H);
#pragma unroll
  for (int i = 0; i < kNormMaxV; ++i) {
    const int v = threadIdx.x + i * kNormThreads;
    if (v < nvec) {
      float wf[8], bf[8], o[8];
      unpack8(reinterpret_cast<const Vec8*>(w)[v], wf);
      unpack8(reinterpret_cast<const Vec8*>(b)[v], bf);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (xv[i][j] - mean) * rstd * wf[j] + bf[j];
      yr[v] = pack8(o);
    }
  }
}
// Small rows (UNet C = 320/640/1280, CLIP 1024): one WARP per row, no block barriers (the CTA-per-row version ran at 130 us
// for 84 MB of traffic on the UNet's [131072, 320] LayerNorms — profiles/r01_unet_launch_list_summary.md).
template <int VPL>  // 8-element vectors per lane
__global__ void __launch_bounds__(256) layernorm_fwd_warp_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                                                                 const bf16* __restrict__ b, bf16* __restrict__ y, int T, int H,
                                                                 float eps) {
  const int lane = threadIdx.x & 31;
  const long row = (static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (row >= T) return;
  const int nvec = H >> 3;
  const Vec8* xr = reinterpret_cast<const Vec8*>(x + row * H);
  float xv[VPL][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int v = lane + i * 32;
    if (v < nvec) {
      unpack8(xr[v], xv[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += xv[i][j];
    }
  }
  const float mean = warp_sum(sum) / static_cast<float>(H);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int v = lane + i * 32;
    if (v < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float d = xv[i][j] - mean; sq += d * d; }
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) / static_cast<float>(H) + eps);
  Vec8* yr = reinterpret_cast<Vec8*>(y + row * H);
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int v = lane + i * 32;
    if (v < nvec) {
      float wf[8], bf[8], o[8];
      unpack8(reinterpret_cast<const Vec8*>(w)[v], wf);
      unpack8(reinterpret_cast<const Vec8*>(b)[v], bf);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (xv[i][j] - mean) * rstd * wf[j] + bf[j];
      yr[v] = pack8(o);
    }
  }
}

int layernorm_fwd(const void* x, const void* w, const void* b, void* y, int T, int H, float eps, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(x, w, b, y);
  if (H % 8 || H > kNormThreads * kNormMaxV * 8 || T <= 0) return DLLM_ERR_SHAPE;
  const int nvec = H / 8;
  if (nvec <= 32 * 6) {
    const unsigned grid = static_cast<unsigned>((static_cast<long>(T) * 32 + 255) / 256);
    if (nvec <= 64)
      layernorm_fwd_warp_kernel<2><<<grid, 256, 0, s>>>((const bf16*)x, (const bf16*)w, (const bf16*)b, (bf16*)y, T, H, eps);
    else if (nvec <= 128)
      layernorm_fwd_warp_kernel<4><<<grid, 256, 0, s>>>((const bf16*)x, (const bf16*)w, (const bf16*)b, (bf16*)y, T, H, eps);
    else
      layernorm_fwd_warp_kernel<6><<<grid, 256, 0, s>>>((const bf16*)x, (const bf16*)w, (const bf16*)b, (bf16*)y, T, H, eps);
    return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
  }
  layernorm_fwd_kernel<<<T, kNormThreads, 0, s>>>((const bf16*)x, (const bf16*)w, (const bf16*)b, (bf16*)y, H, eps);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// ------------------------------------------------------------------------------------------------ CLIP patch embedding
// transformers CLIPVisionEmbeddings: Conv2d(3, C, k=s=patch, bias=False) == GEMM over unfolded patches.
// patchify: images [N,3,R,R] (NCHW bf16) -> rows [N*G*G, Kpad], k = (c*patch + ky)*patch + kx (the conv weight's
// flatten order), zero-padded to Kpad (multiple of 8 so the row stride is 16-byte aligned for TMA).
__global__ void patchify_kernel(const bf16* __restrict__ img, bf16* __restrict__ out, int N, int R, int patch, int G,
                                int Kpad) {
  const long gid = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long total = static_cast<long>(N) * G * G * Kpad;
  if (gid >= total) return;
  const int k = static_cast<int>(gid % Kpad);
  const long pr = gid / Kpad;
  const int gx = static_cast<int>(pr % G);
  const int gy = static_cast<int>((pr / G) % G);
  const int n = static_cast<int>(pr / (static_cast<long>(G) * G));
  bf16 v = __float2bfloat16_rn(0.f);
  if (k < 3 * patch * patch) {
    const int kx = k % patch, ky = (k / patch) % patch, c = k / (patch * patch);
    v = img[((static_cast<size_t>(n) * 3 + c) * R + gy * patch + ky) * R + gx * patch + kx];
  }
  out[gid] = v;
}
// x[n, 0] = cls + pos[0];  x[n, 1+p] = patch[n, p] + pos[1+p]   (bf16 adds as torch.cat + position_embedding)
__global__ void clip_assemble_kernel(const bf16* __restrict__ patches, const bf16* __restrict__ cls,
                                     const bf16* __restrict__ pos, bf16* __restrict__ out, int N, int P, int C) {
  const int nvec = C >> 3;
  const long gid = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long total = static_cast<long>(N) * (P + 1) * nvec;
  if (gid >= total) return;
  const int v = static_cast<int>(gid % nvec);
  const long tr = gid / nvec;
  const int t = static_cast<int>(tr % (P + 1));
  const long n = tr / (P + 1);
  float a[8], b[8];
  if (t == 0) unpack8(reinterpret_cast<const Vec8*>(cls)[v], a);
  else unpack8(reinterpret_cast<const Vec8*>(patches + (n * P + (t - 1)) * C)[v], a);
  unpack8(reinterpret_cast<const Vec8*>(pos + static_cast<size_t>(t) * C)[v], b);
#pragma unroll
  for (int j = 0; j < 8; ++j) a[j] += b[j];
  reinterpret_cast<Vec8*>(out + tr * C)[v] = pack8(a);
}
int clip_patchify(const void* img, void* out, int N, int R, int patch, int Kpad, cudaStream_t s) {
  if (N <= 0 || R % patch || Kpad % 8 || Kpad < 3 * patch * patch) return DLLM_ERR_SHAPE;
  const int G = R / patch;
  const long total = static_cast<long>(N) * G * G * Kpad;
  patchify_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>((const bf16*)img, (bf16*)out, N, R, patch, G, Kpad);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}
int clip_assemble(const void* patches, const void* cls, const void* pos, void* out, int N, int P, int C, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(patches, cls, pos, out);
  if (N <= 0 || P <= 0 || C % 8) return DLLM_ERR_SHAPE;
  const long total = static_cast<long>(N) * (P + 1) * (C / 8);
  clip_assemble_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>((const bf16*)patches, (const bf16*)cls,
                                                                                (const bf16*)pos, (bf16*)out, N, P, C);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// ------------------------------------------------------------------------------------------------ row gather / scatter
// Index paths of DreamLLMModel.forward's embedding splice (modeling_dreamllm.py:1082-1141) and the dream-query
// conditioning gather (:1401-1418): bit-exact row copies driven by a host-built (dst_row, src_row) map.
//   mode 0: dst[dst_idx[r]]  = src[src_idx[r]]          (splice / gather; duplicates in src_idx allowed)
//   mode 1: dst[dst_idx[r]] += src[src_idx[r]]          (gradient of a gather with UNIQUE dst rows per launch)
__global__ void copy_rows_kernel(bf16* __restrict__ dst, const int* __restrict__ dst_idx, const bf16* __restrict__ src,
                                 const int* __restrict__ src_idx, int R, int H, int mode) {
  const int nvec = H >> 3;
  const long gid = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (gid >= static_cast<long>(R) * nvec) return;
  const int v = static_cast<int>(gid % nvec);
  const int r = static_cast<int>(gid / nvec);
  const Vec8 sv = reinterpret_cast<const Vec8*>(src + static_cast<size_t>(src_idx[r]) * H)[v];
  Vec8* d = reinterpret_cast<Vec8*>(dst + static_cast<size_t>(dst_idx[r]) * H) + v;
  if (mode == 0) {
    *d = sv;
  } else {
    float a[8], b[8];
    unpack8(*d, a);
    unpack8(sv, b);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] += b[j];
    *d = pack8(a);
  }
}
// dst[q] = sum over the CSR segment [seg[q], seg[q+1]) of src[rows[i]]   (fp32 accumulate, deterministic):
// gradient of the dream-query broadcast (every <dream_start> occurrence reads the same Q rows).
__global__ void segment_sum_rows_kernel(bf16* __restrict__ dst, const bf16* __restrict__ src, const int* __restrict__ seg,
                                        const int* __restrict__ rows, int H) {
  const int q = blockIdx.x;
  const int nvec = H >> 3;
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    for (int i = seg[q]; i < seg[q + 1]; ++i) {
      float f[8];
      unpack8(reinterpret_cast<const Vec8*>(src + static_cast<size_t>(rows[i]) * H)[v], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += f[j];
    }
    reinterpret_cast<Vec8*>(dst + static_cast<size_t>(q) * H)[v] = pack8(acc);
  }
}
__global__ void zero_rows_kernel(bf16* __restrict__ dst, const int* __restrict__ idx, int R, int H) {
  const int nvec = H >> 3;
  const long gid = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (gid >= static_cast<long>(R) * nvec) return;
  Vec8 z;
#pragma unroll
  for (int i = 0; i < 4; ++i) z.set(i, __floats2bfloat162_rn(0.f, 0.f));
  reinterpret_cast<Vec8*>(dst + static_cast<size_t>(idx[gid / nvec]) * H)[gid % nvec] = z;
}
int copy_rows(void* dst, const int* dst_idx, const void* src, const int* src_idx, int R, int H, int mode, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(dst, src);
  if (H % 8 || R < 0) return DLLM_ERR_SHAPE;
  if (R == 0) return 0;
  const long total = static_cast<long>(R) * (H / 8);
  copy_rows_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>((bf16*)dst, dst_idx, (const bf16*)src, src_idx, R, H, mode);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}
int segment_sum_rows(void* dst, const void* src, const int* seg, const int* rows, int Q, int H, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(dst, src);
  if (H % 8 || Q <= 0) return DLLM_ERR_SHAPE;
  segment_sum_rows_kernel<<<Q, 128, 0, s>>>((bf16*)dst, (const bf16*)src, seg, rows, H);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}
int zero_rows(void* dst, const int* idx, int R, int H, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(dst);
  if (H % 8 || R < 0) return DLLM_ERR_SHAPE;
  if (R == 0) return 0;
  const long total = static_cast<long>(R) * (H / 8);
  zero_rows_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>((bf16*)dst, idx, R, H);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

}  // namespace dllm
