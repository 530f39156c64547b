// HBM-bound kernels of the SD-2.1 UNet denoising step (sm_90a), NHWC bf16 activations.
// Reference call sites: StableDiffusionHead.pipeline, modeling_plugins.py:809-833 (unet(...) -> CFG combine ->
// scheduler.step), whose arithmetic is diffusers 0.24 (ResnetBlock2D GroupNorm+SiLU, GEGLU, Upsample2D, Downsample2D,
// Timesteps, DDIM/DDPM step) — restated in oracle/unet_oracle.py.
#include "common.cuh"
#include "gemm_sm90.h"
#include "ops.h"

namespace dllm {

// 8 bf16 = one 16-byte vector.  The single uint4 member makes every copy of the struct one LDG.E.128 / STG.E.128; the earlier
// `__nv_bfloat162 v[4]` layout was split by nvcc into four 32-bit accesses (4x the LSU / L1 wavefronts: rmsnorm 0.62 -> 0.75, rope
// 0.63 -> 0.68, layernorm 0.47 -> 0.67 of the HBM copy peak on the same box, profiles/r02_ab_hbm_flags.txt).  Row starts must be 16-byte
// aligned (true for every caller: widths and strides are multiples of 8 elements); the host wrappers check the base pointers.
struct alignas(16) V8 {
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
__device__ __forceinline__ void up8(const V8& p, float* f) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(p.get(i));
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ V8 pk8(const float* f) {
  V8 p;
#pragma unroll
  for (int i = 0; i < 4; ++i) p.set(i, __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]));
  return p;
}
__device__ __forceinline__ float r16(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// ------------------------------------------------------------------------------------------------ GroupNorm (+SiLU)
// x [N, HW, C]; G groups of C/G channels.  All four kernels (forward statistics / apply, backward sums / apply) share one thread mapping:
// a CTA owns `rows` consecutive pixel rows of one image and runs RL * (C/8) threads — thread (rl, v) keeps the 8 channels of vector v
// in registers (weight, bias, the <= 2 group records they belong to) and walks rows rl, rl + RL, ... with four independent 16-byte
// loads in flight, so there is no per-element integer division and every lane of the CTA carries data (r01's mapping left 216 of 256
// threads idle at C = 320 and issued one load per thread per trip: 0.13-0.25 of the HBM peak, profiles/r02_ab_hbm_flags.txt).
// Reductions are two-stage and order-fixed (per-thread registers -> smem [RL][C] -> one thread per group -> global partials ->
// finalize), i.e. deterministic: graph replays stay bit-identical to eager launches.
constexpr int kGnMaxThreads = 512;
template <bool kBwd>
struct GnUnroll { static constexpr int v = kBwd ? 2 : 4; };   // rows in flight per thread (the backward kernels carry twice the state)

struct GnMap {
  int nvec, RL, threads;
};
static inline GnMap gn_map(int C) {
  GnMap m;
  m.nvec = C >> 3;
  m.RL = kGnMaxThreads / m.nvec;
  if (m.RL < 1) m.RL = 1;
  if (m.RL > 32) m.RL = 32;
  m.threads = m.RL * m.nvec;
  return m;
}

// the (at most two) groups the 8 channels [8v, 8v+8) fall into: channels j < split belong to g0, the rest to g0 + 1 (cpg >= 8);
// for cpg < 8 (VAE: 128 channels / 32 groups) `gidx` lists the group of every channel instead
struct GnVecGroups {
  int g0, split;
  bool two;
  int gidx[8];
};
__device__ __forceinline__ GnVecGroups gn_vec_groups(int v, int cpg, int G) {
  GnVecGroups r;
  r.two = cpg >= 8;
  r.g0 = (v * 8) / cpg;
  r.split = r.two ? min(8, (r.g0 + 1) * cpg - v * 8) : 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) r.gidx[j] = r.two ? min(r.g0 + (j >= r.split ? 1 : 0), G - 1) : (v * 8 + j) / cpg;
  return r;
}

// forward statistics partials (kBwd = false): per (n, chunk, g) {sum x, sum x^2}
// backward partials          (kBwd = true ): per (n, chunk, g) {sum g, sum g * xhat} with g = dy * silu'(y) * w
template <bool kBwd>
__global__ void __launch_bounds__(kGnMaxThreads) gn_partial_kernel(const bf16* __restrict__ x, const bf16* __restrict__ dy,
                                                                   const bf16* __restrict__ w, const bf16* __restrict__ b,
                                                                   const float* __restrict__ stats, float* __restrict__ partial, int HW,
                                                                   int C, int G, int rows_per_cta, int RL, int silu) {
  extern __shared__ float sm[];  // [RL][2][C]
  const int n = blockIdx.y, chunk = blockIdx.x, nchunks = gridDim.x;
  const int nvec = C >> 3, cpg = C / G;
  const int v = threadIdx.x % nvec, rl = threadIdx.x / nvec;
  const int r0 = chunk * rows_per_cta, r1 = min(HW, r0 + rows_per_cta);
  float s[8], q[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) s[j] = q[j] = 0.f;
  float wf[8], bf_[8], mean[8], rstd[8];
  if constexpr (kBwd) {
    up8(reinterpret_cast<const V8*>(w)[v], wf);
    up8(reinterpret_cast<const V8*>(b)[v], bf_);
    const GnVecGroups gg = gn_vec_groups(v, cpg, G);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float2 st = *reinterpret_cast<const float2*>(stats + (static_cast<size_t>(n) * G + gg.gidx[j]) * 2);
      mean[j] = st.x;
      rstd[j] = st.y;
    }
  }
  const size_t base = static_cast<size_t>(n) * HW * C;
  const V8* xb = reinterpret_cast<const V8*>(x + base) + v;
  const V8* db = kBwd ? reinterpret_cast<const V8*>(dy + base) + v : nullptr;
  constexpr int kGnUnroll = GnUnroll<kBwd>::v;
  for (int r = r0 + rl; r < r1; r += RL * kGnUnroll) {
    V8 xv[kGnUnroll], dv[kGnUnroll];
#pragma unroll
    for (int u = 0; u < kGnUnroll; ++u) {
      const int rr = r + u * RL;
      if (rr < r1) {
        xv[u] = xb[static_cast<size_t>(rr) * nvec];
        if constexpr (kBwd) dv[u] = db[static_cast<size_t>(rr) * nvec];
      }
    }
#pragma unroll
    for (int u = 0; u < kGnUnroll; ++u) {
      const int rr = r + u * RL;
      if (rr < r1) {
        float f[8];
        up8(xv[u], f);
        if constexpr (!kBwd) {
#pragma unroll
          for (int j = 0; j < 8; ++j) { s[j] += f[j]; q[j] += f[j] * f[j]; }
        } else {
          float d[8];
          up8(dv[u], d);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float xh = (f[j] - mean[j]) * rstd[j];
            float gq = d[j];
            if (silu) {
              const float y = r16(xh * wf[j] + bf_[j]);
              const float sg = 1.f / (1.f + expf(-y));
              gq *= sg * (1.f + y * (1.f - sg));
            }
            gq *= wf[j];
            s[j] += gq;
            q[j] += gq * xh;
          }
        }
      }
    }
  }
  float* sm_s = sm + (static_cast<size_t>(rl) * 2) * C + v * 8;
#pragma unroll
  for (int j = 0; j < 8; ++j) { sm_s[j] = s[j]; sm_s[C + j] = q[j]; }
  __syncthreads();
  // stage 1: one thread per (stat, channel) sums the RL row-lane partials (order-fixed, conflict-free: consecutive threads read
  // consecutive floats); stage 2: one thread per (group, stat) sums its cpg channels.  (A single thread per group walking RL x cpg
  // values cost ~7k cycles per CTA — more than streaming the CTA's rows.)
  for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) {
    float a = 0.f;
    for (int l = 0; l < RL; ++l) a += sm[static_cast<size_t>(l) * 2 * C + i];
    sm[i] = a;                                   // row-lane 0's slot doubles as the reduced vector (each i touched by one thread only)
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * G; i += blockDim.x) {
    const int g = i >> 1, which = i & 1;
    const float* p0 = sm + which * C + g * cpg;
    float a = 0.f;
    for (int c = 0; c < cpg; ++c) a += p0[c];
    partial[((static_cast<size_t>(n) * nchunks + chunk) * G + g) * 2 + which] = a;
  }
}
// forward: stats[n, g] = {mean, rstd};  backward (eps < 0, x unused): sums[n, g] = {sum g / count, sum g xhat / count}
// One WARP per (n, g): lanes stride over the chunk partials, then a fixed-order shuffle tree (deterministic).  (One thread walking up
// to 128 partials serially cost 17 us per GroupNorm on the VAE's 512x512 planes.)
// The variance E[x^2] - mean^2 of the partials cancels in fp32 when |mean| >> std: at mean / std = 64 and 128 it put rstd off by 3e-4
// to 9e-4 (H100, 700 W; tests/test_tower_kernels_gpu.py).  When mean^2 > kGnRecomputeRatio * var the warp re-reads the group and takes
// the variance about the mean, sum (x - mean)^2 / count less the (sum (x - mean))^2 / count^2 correction: rstd then within 6e-5 at
// mean / std = 128 on a 256 x 256 plane.  Below that ratio (|mean| < 11.3 std) the one-pass rstd is good to ~3e-5 and is kept bit for
// bit, so ordinary activations pay nothing and compute what they computed before.
constexpr float kGnRecomputeRatio = 128.f;
__global__ void gn_finalize_kernel(const float* __restrict__ partial, const bf16* __restrict__ x, float* __restrict__ stats, int nchunks,
                                   int G, int HW, int C, float count, float eps, int total) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;  // n * G + g
  const int lane = threadIdx.x & 31;
  if (i >= total) return;
  const int n = i / G, g = i - n * G;
  float a = 0.f, b = 0.f;
  for (int c = lane; c < nchunks; c += 32) {
    const float2 p = *reinterpret_cast<const float2*>(partial + ((static_cast<size_t>(n) * nchunks + c) * G + g) * 2);
    a += p.x;
    b += p.y;
  }
  a = warp_sum(a);
  b = warp_sum(b);
  if (eps < 0.f) {
    if (lane != 0) return;
    stats[2 * i] = a / count;
    stats[2 * i + 1] = b / count;
    return;
  }
  const float mean = a / count;
  float var = fmaxf(b / count - mean * mean, 0.f);
  if (mean * mean > kGnRecomputeRatio * var) {   // the whole warp takes this branch (a, b are warp-uniform)
    const int cpg = C / G;
    const bf16* xg = x + static_cast<size_t>(n) * HW * C + static_cast<size_t>(g) * cpg;
    float s1 = 0.f, s2 = 0.f;
    for (int r = lane; r < HW; r += 32)
      for (int c = 0; c < cpg; ++c) {
        const float d = __bfloat162float(xg[static_cast<size_t>(r) * C + c]) - mean;
        s1 += d;
        s2 += d * d;
      }
    s1 = warp_sum(s1);
    s2 = warp_sum(s2);
    var = fmaxf((s2 - s1 * s1 / count) / count, 0.f);
  }
  if (lane != 0) return;
  stats[2 * i] = mean;
  stats[2 * i + 1] = rsqrtf(var + eps);
}
// forward  (kBwd = false): y  = silu?( bf16( (x - mean) * rstd * w + b ) )
// backward (kBwd = true ): dx = rstd * (g - mean_g(g) - xhat * mean_g(g * xhat)) (+ dres),   g = dy * silu'(y) * w
template <bool kBwd>
__global__ void __launch_bounds__(kGnMaxThreads) gn_apply_kernel(const bf16* __restrict__ x, const bf16* __restrict__ dy,
                                                                 const bf16* __restrict__ w, const bf16* __restrict__ b,
                                                                 const float* __restrict__ stats, const float* __restrict__ sums,
                                                                 const bf16* __restrict__ dres, bf16* __restrict__ out, int HW, int C, int G,
                                                                 int rows_per_cta, int RL, int silu) {
  const int n = blockIdx.y, chunk = blockIdx.x;
  const int nvec = C >> 3, cpg = C / G;
  const int v = threadIdx.x % nvec, rl = threadIdx.x / nvec;
  const int r0 = chunk * rows_per_cta, r1 = min(HW, r0 + rows_per_cta);
  float wf[8], bf_[8], mean[8], rstd[8], m1[8], m2[8];
  up8(reinterpret_cast<const V8*>(w)[v], wf);
  up8(reinterpret_cast<const V8*>(b)[v], bf_);
  const GnVecGroups gg = gn_vec_groups(v, cpg, G);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const size_t si = (static_cast<size_t>(n) * G + gg.gidx[j]) * 2;
    const float2 st = *reinterpret_cast<const float2*>(stats + si);
    mean[j] = st.x;
    rstd[j] = st.y;
    if constexpr (kBwd) {
      const float2 sm2 = *reinterpret_cast<const float2*>(sums + si);
      m1[j] = sm2.x;
      m2[j] = sm2.y;
    }
  }
  const size_t base = static_cast<size_t>(n) * HW * C;
  const V8* xb = reinterpret_cast<const V8*>(x + base) + v;
  const V8* db = kBwd ? reinterpret_cast<const V8*>(dy + base) + v : nullptr;
  const V8* rb = (kBwd && dres) ? reinterpret_cast<const V8*>(dres + base) + v : nullptr;
  V8* ob = reinterpret_cast<V8*>(out + base) + v;
  constexpr int kGnUnroll = GnUnroll<kBwd>::v;
  for (int r = r0 + rl; r < r1; r += RL * kGnUnroll) {
    V8 xv[kGnUnroll], dv[kGnUnroll], rv[kGnUnroll];
#pragma unroll
    for (int u = 0; u < kGnUnroll; ++u) {
      const int rr = r + u * RL;
      if (rr < r1) {
        xv[u] = xb[static_cast<size_t>(rr) * nvec];
        if constexpr (kBwd) {
          dv[u] = db[static_cast<size_t>(rr) * nvec];
          if (rb) rv[u] = rb[static_cast<size_t>(rr) * nvec];
        }
      }
    }
#pragma unroll
    for (int u = 0; u < kGnUnroll; ++u) {
      const int rr = r + u * RL;
      if (rr < r1) {
        float f[8], o[8];
        up8(xv[u], f);
        if constexpr (!kBwd) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            float t = r16((f[j] - mean[j]) * rstd[j] * wf[j] + bf_[j]);
            if (silu) t = t / (1.f + expf(-t));
            o[j] = t;
          }
        } else {
          float d[8], rs[8];
          up8(dv[u], d);
          if (rb) up8(rv[u], rs);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float xh = (f[j] - mean[j]) * rstd[j];
            float gq = d[j];
            if (silu) {
              const float y = r16(xh * wf[j] + bf_[j]);
              const float sg = 1.f / (1.f + expf(-y));
              gq *= sg * (1.f + y * (1.f - sg));
            }
            gq *= wf[j];
            float t = rstd[j] * (gq - m1[j] - xh * m2[j]);
            if (rb) t += rs[j];
            o[j] = t;
          }
        }
        ob[static_cast<size_t>(rr) * nvec] = pk8(o);
      }
    }
  }
}

// pixel rows per partial-sum CTA: 64 for the big UNet planes, more for the VAE's 512x512 planes so that the finalize pass never walks
// more than 128 partials, fewer for small planes so that the grid still covers every SM
static inline int gn_rows(int HW, int N) {
  int rows = 256;                                  // enough rows per CTA to amortise the per-CTA prologue / reduction epilogue ...
  while ((HW + rows - 1) / rows > 128) rows *= 2;
  while (rows > 8 && static_cast<long>(N) * ((HW + rows - 1) / rows) < 4 * num_sms() && (HW + rows / 2 - 1) / (rows / 2) <= 128) rows /= 2;   // ... but >= 4 CTAs / SM
  return rows;
}
size_t groupnorm_workspace(int N, int HW, int G) {
  const int rows = gn_rows(HW, N);
  const int nchunks = (HW + rows - 1) / rows;
  return (static_cast<size_t>(N) * nchunks * G * 2 + static_cast<size_t>(N) * G * 2) * sizeof(float);
}
static int gn_check(int N, int HW, int C, int G, size_t ws_bytes) {
  if (C % 8 || C % G || (C >> 3) > kGnMaxThreads || N <= 0 || HW <= 0) return DLLM_ERR_SHAPE;
  if (ws_bytes < groupnorm_workspace(N, HW, G)) return DLLM_ERR_SHAPE;
  return 0;
}
static int gn_launch_stats(const bf16* x, float* stats, float* partial, int N, int HW, int C, int G, float eps, cudaStream_t s) {
  const GnMap m = gn_map(C);
  const int rows = gn_rows(HW, N);
  const int nchunks = (HW + rows - 1) / rows;
  gn_partial_kernel<false><<<dim3(nchunks, N), m.threads, static_cast<size_t>(m.RL) * 2 * C * sizeof(float), s>>>(
      x, nullptr, nullptr, nullptr, nullptr, partial, HW, C, G, rows, m.RL, 0);
  gn_finalize_kernel<<<(N * G * 32 + 255) / 256, 256, 0, s>>>(partial, x, stats, nchunks, G, HW, C, static_cast<float>(HW) * (C / G), eps,
                                                               N * G);
  return 0;
}
static void gn_launch_apply(const bf16* x, const bf16* w, const bf16* b, const float* stats, bf16* y, int N, int HW, int C, int G, int silu,
                            cudaStream_t s) {
  const GnMap m = gn_map(C);
  int rows = 128;
  while (rows > m.RL && static_cast<long>(N) * ((HW + rows - 1) / rows) < 4 * num_sms()) rows /= 2;
  gn_apply_kernel<false><<<dim3((HW + rows - 1) / rows, N), m.threads, 0, s>>>(x, nullptr, w, b, stats, nullptr, nullptr, y, HW, C, G, rows,
                                                                                m.RL, silu);
}
int groupnorm_nhwc(const void* x, const void* w, const void* b, void* y, void* workspace, size_t ws_bytes, int N, int HW, int C,
                   int G, float eps, int silu, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(x, w, b, y);
  if (int rc = gn_check(N, HW, C, G, ws_bytes)) return rc;
  float* partial = static_cast<float*>(workspace);
  const int rows = gn_rows(HW, N);
  float* stats = partial + static_cast<size_t>(N) * ((HW + rows - 1) / rows) * G * 2;
  gn_launch_stats((const bf16*)x, stats, partial, N, HW, C, G, eps, s);
  gn_launch_apply((const bf16*)x, (const bf16*)w, (const bf16*)b, stats, (bf16*)y, N, HW, C, G, silu, s);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// ------------------------------------------------------------------------------------------------ GEGLU
// diffusers GEGLU: h, gate = proj(x).chunk(2); out = h * gelu(gate)      in [T, 2I] -> out [T, I]
// grid = (ceil(I/8 / 256), T / kGegluRows): a thread keeps its column vector and walks kGegluRows token rows with all loads of two rows
// issued before the erf math (no 64-bit index division, 4 x 16 B in flight per thread)
constexpr int kGegluRows = 4;
__global__ void __launch_bounds__(256) geglu_kernel(const bf16* __restrict__ in, bf16* __restrict__ out, int T, int I) {
  const int nvec = I >> 3;
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nvec) return;
  const int t0 = blockIdx.y * kGegluRows;
#pragma unroll
  for (int tt = 0; tt < kGegluRows; tt += 2) {
    V8 av[2], gv[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const long t = t0 + tt + u;
      if (t < T) {
        av[u] = *reinterpret_cast<const V8*>(in + t * 2 * I + v * 8);
        gv[u] = *reinterpret_cast<const V8*>(in + t * 2 * I + I + v * 8);
      }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const long t = t0 + tt + u;
      if (t < T) {
        float a[8], g[8];
        up8(av[u], a);
        up8(gv[u], g);
#pragma unroll
        for (int j = 0; j < 8; ++j) a[j] *= r16(0.5f * g[j] * (1.f + erff(g[j] * 0.70710678118654752f)));
        *reinterpret_cast<V8*>(out + t * I + v * 8) = pk8(a);
      }
    }
  }
}
int geglu(const void* in, void* out, int T, int I, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(in, out);
  if (I % 8 || T <= 0) return DLLM_ERR_SHAPE;
  const int nvec = I / 8;
  const int bt = ((nvec < 256 ? nvec : 256) + 31) / 32 * 32;      // no idle lanes when I/8 < 256 (I = 1280: 160 threads)
  const long rows = (static_cast<long>(T) + kGegluRows - 1) / kGegluRows;
  if (rows > 65535L * 32768L) return DLLM_ERR_SHAPE;
  // blockIdx.y is limited to 65535: fold the excess into more columns per launch is not needed for T <= 262 140
  if (rows > 65535) {
    for (long r0 = 0; r0 < T; r0 += 65535L * kGegluRows) {
      const int Tc = static_cast<int>(T - r0 < 65535L * kGegluRows ? T - r0 : 65535L * kGegluRows);
      geglu_kernel<<<dim3((nvec + bt - 1) / bt, (Tc + kGegluRows - 1) / kGegluRows), bt, 0, s>>>((const bf16*)in + r0 * 2 * I,
                                                                                                 (bf16*)out + r0 * I, Tc, I);
    }
  } else {
    geglu_kernel<<<dim3((nvec + bt - 1) / bt, static_cast<unsigned>(rows)), bt, 0, s>>>((const bf16*)in, (bf16*)out, T, I);
  }
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// ------------------------------------------------------------------------------------------------ spatial data movement
// nearest 2x upsample (Upsample2D's F.interpolate), NHWC
__global__ void upsample2x_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, int N, int H, int W, int C) {
  const int nvec = C >> 3;
  const long gid = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long total = static_cast<long>(N) * 4 * H * W * nvec;
  if (gid >= total) return;
  const int v = static_cast<int>(gid % nvec);
  long p = gid / nvec;
  const int wo = static_cast<int>(p % (2 * W)); p /= 2 * W;
  const int ho = static_cast<int>(p % (2 * H));
  const int n = static_cast<int>(p / (2 * H));
  reinterpret_cast<uint4*>(y)[gid] = reinterpret_cast<const uint4*>(x + ((static_cast<size_t>(n) * H + ho / 2) * W + wo / 2) * C)[v];
}
// im2col for the stride-2 3x3 pad-1 Downsample2D conv: out [N*Ho*Wo, 9*C], k = (r, s, c)
__global__ void im2col_s2_kernel(const bf16* __restrict__ x, bf16* __restrict__ out, int N, int H, int W, int C, int pad) {
  const int nvec = C >> 3;
  const int Ho = H / 2, Wo = W / 2;
  const long gid = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long total = static_cast<long>(N) * Ho * Wo * 9 * nvec;
  if (gid >= total) return;
  const int v = static_cast<int>(gid % nvec);
  long p = gid / nvec;
  const int tap = static_cast<int>(p % 9); p /= 9;
  const int wo = static_cast<int>(p % Wo); p /= Wo;
  const int ho = static_cast<int>(p % Ho);
  const int n = static_cast<int>(p / Ho);
  // pad = 1: UNet Downsample2D (symmetric padding 1); pad = 0: VAE downsample (F.pad (0,1,0,1) then padding 0)
  const int h = 2 * ho + tap / 3 - pad, w = 2 * wo + tap % 3 - pad;
  uint4 val = make_uint4(0, 0, 0, 0);
  if (h >= 0 && h < H && w >= 0 && w < W) val = reinterpret_cast<const uint4*>(x + ((static_cast<size_t>(n) * H + h) * W + w) * C)[v];
  reinterpret_cast<uint4*>(out)[gid] = val;
}
// dst[:, col0 : col0 + Cs] = src  (channel concat of skip connections, NHWC => a strided 2-D copy)
__global__ void copy_cols_kernel(const bf16* __restrict__ src, bf16* __restrict__ dst, long rows, int Cs, int Cd, int col0) {
  const int nvec = Cs >> 3;
  const long gid = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (gid >= rows * nvec) return;
  const int v = static_cast<int>(gid % nvec);
  const long r = gid / nvec;
  *reinterpret_cast<uint4*>(dst + r * Cd + col0 + v * 8) = reinterpret_cast<const uint4*>(src + r * Cs)[v];
}
int upsample2x_nhwc(const void* x, void* y, int N, int H, int W, int C, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(x, y);
  if (C % 8) return DLLM_ERR_SHAPE;
  const long total = static_cast<long>(N) * 4 * H * W * (C / 8);
  upsample2x_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>((const bf16*)x, (bf16*)y, N, H, W, C);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}
int im2col_s2_nhwc(const void* x, void* out, int N, int H, int W, int C, int pad, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(x, out);
  if (C % 8 || H % 2 || W % 2) return DLLM_ERR_SHAPE;
  const long total = static_cast<long>(N) * (H / 2) * (W / 2) * 9 * (C / 8);
  im2col_s2_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>((const bf16*)x, (bf16*)out, N, H, W, C, pad);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}
int copy_cols(const void* src, void* dst, long rows, int Cs, int Cd, int col0, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(src, dst);
  if (Cs % 8 || Cd % 8 || col0 % 8 || rows <= 0) return DLLM_ERR_SHAPE;
  const long total = rows * (Cs / 8);
  copy_cols_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>((const bf16*)src, (bf16*)dst, rows, Cs, Cd, col0);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// ------------------------------------------------------------------------------------------------ conv_in / conv_out
// conv_in: latents fp32 NCHW [B,Cin(=4),H,W] (rounded to bf16 as the bf16 pipeline feeds them) -> NHWC bf16 [B,H,W,Cout];
// w [Cout, Cin, 3, 3] bf16 (diffusers layout).  One thread = one pixel x 8 output channels.
__global__ void __launch_bounds__(128) conv_in_kernel(const float* __restrict__ x, const bf16* __restrict__ w,
                                                      const bf16* __restrict__ bias, bf16* __restrict__ y, int B, int Bsrc, int Cin,
                                                      int H, int W, int Cout) {
  // weights staged once per CTA as fp32 [Cin*9][Cout] so the inner loop reads 8 consecutive output channels
  extern __shared__ float wsm[];
  const int K = Cin * 9;
  for (int i = threadIdx.x; i < K * Cout; i += blockDim.x) {
    const int o = i % Cout, k = i / Cout;  // k = (c*3 + r)*3 + s, the conv weight's own flatten order
    wsm[i] = __bfloat162float(w[static_cast<size_t>(o) * K + k]);
  }
  __syncthreads();
  const int nvec = Cout >> 3;
  const long total = static_cast<long>(B) * H * W * nvec;
  for (long gid = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; gid < total; gid += static_cast<long>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(gid % nvec);
    long p = gid / nvec;
    const int wx = static_cast<int>(p % W); p /= W;
    const int hy = static_cast<int>(p % H);
    const int nb = static_cast<int>(p / H);
    const int n = nb % Bsrc;  // CFG: the same latents feed the uncond and cond halves (:811)
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = __bfloat162float(bias[v * 8 + j]);
    for (int c = 0; c < Cin; ++c)
      for (int r = 0; r < 3; ++r)
        for (int sx = 0; sx < 3; ++sx) {
          const int h = hy + r - 1, ww = wx + sx - 1;
          if (h < 0 || h >= H || ww < 0 || ww >= W) continue;
          const float xv = r16(x[((static_cast<size_t>(n) * Cin + c) * H + h) * W + ww]);
          const float* wk = wsm + ((c * 3 + r) * 3 + sx) * Cout + v * 8;
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] += xv * wk[j];
        }
    reinterpret_cast<V8*>(y)[gid] = pk8(acc);
  }
}
// conv_out: NHWC bf16 [B,H,W,C] -> fp32 NCHW [B,Cout(=4),H,W]; w [Cout, C, 3, 3] bf16.  One warp = one pixel.
template <int COUT>
__global__ void conv_out_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w, const bf16* __restrict__ bias,
                                float* __restrict__ y, int B, int C, int H, int W) {
  const long warp = (static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= static_cast<long>(B) * H * W) return;
  const int wx = static_cast<int>(warp % W);
  const int hy = static_cast<int>((warp / W) % H);
  const int n = static_cast<int>(warp / (static_cast<long>(W) * H));
  float acc[COUT];
#pragma unroll
  for (int o = 0; o < COUT; ++o) acc[o] = 0.f;
  for (int r = 0; r < 3; ++r)
    for (int sx = 0; sx < 3; ++sx) {
      const int h = hy + r - 1, ww = wx + sx - 1;
      if (h < 0 || h >= H || ww < 0 || ww >= W) continue;
      const bf16* xp = x + ((static_cast<size_t>(n) * H + h) * W + ww) * C;
      for (int c = lane; c < C; c += 32) {
        const float xv = __bfloat162float(xp[c]);
#pragma unroll
        for (int o = 0; o < COUT; ++o) acc[o] += xv * __bfloat162float(w[((static_cast<size_t>(o) * C + c) * 3 + r) * 3 + sx]);
      }
    }
#pragma unroll
  for (int o = 0; o < COUT; ++o) acc[o] = warp_sum(acc[o]);
  if (lane == 0)
#pragma unroll
    for (int o = 0; o < COUT; ++o)
      y[((static_cast<size_t>(n) * COUT + o) * H + hy) * W + wx] = r16(acc[o] + __bfloat162float(bias[o]));
}
int conv_in_nchw_to_nhwc(const float* x, const void* w, const void* bias, void* y, int B, int Bsrc, int Cin, int H, int W,
                         int Cout, cudaStream_t s) {
  if (Cout % 8 || Bsrc <= 0) return DLLM_ERR_SHAPE;
  const size_t smem = static_cast<size_t>(Cin) * 9 * Cout * sizeof(float);
  if (smem > 96 * 1024) return DLLM_ERR_UNSUPPORTED;
  static bool once = false;
  if (!once) { cudaFuncSetAttribute(conv_in_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024); once = true; }
  conv_in_kernel<<<num_sms() * 4, 128, smem, s>>>(x, (const bf16*)w, (const bf16*)bias, (bf16*)y, B, Bsrc, Cin, H, W, Cout);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}
int conv_out_nhwc_to_nchw(const void* x, const void* w, const void* bias, float* y, int B, int C, int H, int W, int Cout,
                          cudaStream_t s) {
  if (Cout != 4 && Cout != 8 && Cout != 3) return DLLM_ERR_UNSUPPORTED;
  const long warps = static_cast<long>(B) * H * W;
  if (Cout == 3)
    conv_out_kernel<3><<<static_cast<unsigned>((warps * 32 + 255) / 256), 256, 0, s>>>((const bf16*)x, (const bf16*)w, (const bf16*)bias, y, B, C, H, W);
  else if (Cout == 4)
    conv_out_kernel<4><<<static_cast<unsigned>((warps * 32 + 255) / 256), 256, 0, s>>>((const bf16*)x, (const bf16*)w, (const bf16*)bias, y, B, C, H, W);
  else
    conv_out_kernel<8><<<static_cast<unsigned>((warps * 32 + 255) / 256), 256, 0, s>>>((const bf16*)x, (const bf16*)w, (const bf16*)bias, y, B, C, H, W);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// ---- conv_in / conv_out on the tensor cores (round 2).  The direct kernels above cost 1.36 ms (conv_in, 4 -> 320 @ 64x64 x 32) and
// 0.68 ms (conv_out) of a 42 ms UNet step, and 0.95 ms per VAE conv_in at 512x512 (profiles/r02d_unet_launch_list_summary.md):
//   conv_in  = im2col of the tiny-Cin fp32 NCHW input into bf16 rows [M, 64] (k = (c*3 + r)*3 + s, zero padded to one 64-wide K block)
//              + the wgmma GEMM with the bias epilogue against the [Cout, 64] weight matrix          (dllm_im2col_in + dllm_gemm_bf16_ex)
//   conv_out = the implicit-GEMM conv3x3 with Cout zero-padded to 8 + a channel-slicing NHWC bf16 -> NCHW fp32 pass
//                                                                                                    (dllm_conv3x3_nhwc + dllm_nhwc_to_nchw_f32)
__global__ void im2col_in_kernel(const float* __restrict__ x, bf16* __restrict__ cols, long total_vec, int Bsrc, int Cin, int H, int W) {
  const long gid = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (gid >= total_vec) return;
  const int v = static_cast<int>(gid & 7);
  long p = gid >> 3;
  const int wx = static_cast<int>(p % W); p /= W;
  const int hy = static_cast<int>(p % H);
  const int n = static_cast<int>(p / H) % Bsrc;        // CFG: image n reads latents[n % Bsrc]
  const int K = Cin * 9;
  float f[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int k = v * 8 + j;
    float val = 0.f;
    if (k < K) {
      const int c = k / 9, rs = k - 9 * c, r = rs / 3, sx = rs - 3 * r;
      const int h = hy + r - 1, ww = wx + sx - 1;
      if (h >= 0 && h < H && ww >= 0 && ww < W) val = x[((static_cast<size_t>(n) * Cin + c) * H + h) * W + ww];
    }
    f[j] = val;
  }
  reinterpret_cast<V8*>(cols)[gid] = pk8(f);
}
int im2col_in(const float* x, void* cols, int B, int Bsrc, int Cin, int H, int W, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(cols);
  if (B <= 0 || Bsrc <= 0 || Cin * 9 > 64) return DLLM_ERR_SHAPE;
  const long total = static_cast<long>(B) * H * W * 8;
  im2col_in_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>(x, (bf16*)cols, total, Bsrc, Cin, H, W);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}
// y [N*HW, Cp] bf16 (Cp = 8: one 16-byte vector per pixel) -> out fp32 NCHW [N, Cout, HW], Cout <= Cp
__global__ void nhwc_to_nchw_f32_kernel(const bf16* __restrict__ y, float* __restrict__ out, long total, int HW, int Cout) {
  const long gid = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (gid >= total) return;
  const long n = gid / HW;
  const int p = static_cast<int>(gid - n * HW);
  float f[8];
  up8(reinterpret_cast<const V8*>(y)[gid], f);
#pragma unroll
  for (int o = 0; o < 8; ++o)
    if (o < Cout) out[(static_cast<size_t>(n) * Cout + o) * HW + p] = f[o];
}
int nhwc_to_nchw_f32(const void* y, float* out, int N, int HW, int Cp, int Cout, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(y);
  if (Cp != 8 || Cout > 8 || Cout <= 0 || N <= 0) return DLLM_ERR_SHAPE;
  const long total = static_cast<long>(N) * HW;
  nhwc_to_nchw_f32_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>((const bf16*)y, out, total, HW, Cout);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// ------------------------------------------------------------------------------------------------ time embedding / sampler
// Timesteps(320, flip_sin_to_cos=True, shift 0): emb[b] = [cos(t*f_i) | sin(t*f_i)], f_i = exp(-ln(10000) i / half).
// t is read from the device-side schedule: timesteps[*step] (so one captured CUDA graph serves every step).
__global__ void timestep_embedding_kernel(const int* __restrict__ timesteps, const int* __restrict__ step, bf16* __restrict__ out,
                                          int B, int dim) {
  const int half = dim / 2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * half) return;
  const int b = i / half, k = i - b * half;
  const float t = static_cast<float>(timesteps[*step]);
  const float f = expf(-logf(10000.f) * static_cast<float>(k) / static_cast<float>(half));
  out[b * dim + k] = __float2bfloat16_rn(cosf(t * f));
  out[b * dim + half + k] = __float2bfloat16_rn(sinf(t * f));
}
// training flavour: one timestep per sample (t ~ U{0..999}, modeling_plugins.py:528)
__global__ void timestep_embedding_batch_kernel(const int* __restrict__ t, bf16* __restrict__ out, int B, int dim) {
  const int half = dim / 2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * half) return;
  const int b = i / half, k = i - b * half;
  const float tv = static_cast<float>(t[b]);
  const float f = expf(-logf(10000.f) * static_cast<float>(k) / static_cast<float>(half));
  out[b * dim + k] = __float2bfloat16_rn(cosf(tv * f));
  out[b * dim + half + k] = __float2bfloat16_rn(sinf(tv * f));
}
int timestep_embedding_batch(const int* t, void* out, int B, int dim, cudaStream_t s) {
  timestep_embedding_batch_kernel<<<(B * dim / 2 + 127) / 128, 128, 0, s>>>(t, (bf16*)out, B, dim);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}
int timestep_embedding(const int* timesteps, const int* step, void* out, int B, int dim, cudaStream_t s) {
  timestep_embedding_kernel<<<(B * dim / 2 + 127) / 128, 128, 0, s>>>(timesteps, step, (bf16*)out, B, dim);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// One sampler update, fused: CFG combine (modeling_plugins.py:824-830) + scheduler.step (:833), then advance the device-side
// step counter.  eps [2B,...] = [uncond | cond] (guidance > 1, as the reference's torch.cat order :774-784) or [B,...].
// coef[step] = {sqrt(a_t), sqrt(1-a_t), c_x0, c_xt_or_eps, sigma}:
//   DDIM (eta 0): x' = c_x0 * x0 + c_eps * eps             (c_x0 = sqrt(a_prev), c_eps = sqrt(1-a_prev), sigma = 0)
//   DDPM        : x' = c_x0 * x0 + c_xt * x_t + sigma * z  (mode 1)
__global__ void sampler_step_kernel(const float* __restrict__ eps, float* __restrict__ latents, const float* __restrict__ noise,
                                    const float* __restrict__ coef, int* __restrict__ step, float guidance, int use_cfg, int mode,
                                    long n) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int st = *step;
  if (i < n) {
    const float* c = coef + st * 5;
    float e = eps[i];
    if (use_cfg) e = e + guidance * (eps[n + i] - e);
    const float xt = latents[i];
    const float x0 = (xt - c[1] * e) / c[0];
    float out = (mode == 0) ? c[2] * x0 + c[3] * e : c[2] * x0 + c[3] * xt + (noise ? c[4] * noise[static_cast<size_t>(st) * n + i] : 0.f);
    latents[i] = out;
  }
}
__global__ void advance_step_kernel(int* step) { *step += 1; }
int sampler_step(const float* eps, float* latents, const float* noise, const float* coef, int* step, float guidance, int use_cfg,
                 int mode, long n, cudaStream_t s) {
  sampler_step_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(eps, latents, noise, coef, step, guidance, use_cfg, mode, n);
  advance_step_kernel<<<1, 1, 0, s>>>(step);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}


// ================================================================================================ backward (input gradients only)
// StableDiffusionHead.forward trains through a FROZEN UNet (modeling_plugins.py:493-577, freeze_unet=True): gradients must reach the
// dream-query conditioning, so every op needs d/d(input) but no weight gradients (SURVEY §7 "Backward through frozen towers").

// ---- GroupNorm(+SiLU) backward.  g = dy * silu'(y_gn) * w;  dx = rstd * (g - mean_g(g) - xhat * mean_g(g * xhat))
// (kernels: gn_partial_kernel<true> / gn_finalize_kernel(eps < 0) / gn_apply_kernel<true> above)
// stats: [N, G, 2] {mean, rstd} from the forward (groupnorm_stats); workspace as in the forward
int groupnorm_bwd_nhwc(const void* dy, const void* x, const void* w, const void* b, const float* stats, const void* dres, void* dx,
                       void* workspace, size_t ws_bytes, int N, int HW, int C, int G, int silu, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(dy, x, w, b, dres, dx);
  if (int rc = gn_check(N, HW, C, G, ws_bytes)) return rc;
  const GnMap m = gn_map(C);
  const int rows = gn_rows(HW, N);
  const int nchunks = (HW + rows - 1) / rows;
  float* partial = static_cast<float*>(workspace);
  float* sums = partial + static_cast<size_t>(N) * nchunks * G * 2;
  gn_partial_kernel<true><<<dim3(nchunks, N), m.threads, static_cast<size_t>(m.RL) * 2 * C * sizeof(float), s>>>(
      (const bf16*)x, (const bf16*)dy, (const bf16*)w, (const bf16*)b, stats, partial, HW, C, G, rows, m.RL, silu);
  gn_finalize_kernel<<<(N * G * 32 + 255) / 256, 256, 0, s>>>(partial, nullptr, sums, nchunks, G, HW, C, static_cast<float>(HW) * (C / G),
                                                               -1.f, N * G);
  int arows = 128;
  while (arows > m.RL && static_cast<long>(N) * ((HW + arows - 1) / arows) < 4 * num_sms()) arows /= 2;
  gn_apply_kernel<true><<<dim3((HW + arows - 1) / arows, N), m.threads, 0, s>>>((const bf16*)x, (const bf16*)dy, (const bf16*)w,
                                                                                (const bf16*)b, stats, sums, (const bf16*)dres, (bf16*)dx,
                                                                                HW, C, G, arows, m.RL, silu);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}
// forward statistics only ([N, G, 2]) — kept by the training path for the backward
int groupnorm_stats(const void* x, float* stats, void* workspace, size_t ws_bytes, int N, int HW, int C, int G, float eps, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(x);
  if (int rc = gn_check(N, HW, C, G, ws_bytes)) return rc;
  gn_launch_stats((const bf16*)x, stats, static_cast<float*>(workspace), N, HW, C, G, eps, s);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}
int groupnorm_apply(const void* x, const void* w, const void* b, const float* stats, void* y, int N, int HW, int C, int G, int silu,
                    cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(x, w, b, y);
  if (C % 8 || C % G || (C >> 3) > kGnMaxThreads || N <= 0) return DLLM_ERR_SHAPE;
  gn_launch_apply((const bf16*)x, (const bf16*)w, (const bf16*)b, stats, (bf16*)y, N, HW, C, G, silu, s);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// ---- LayerNorm backward (dx only), warp per row, statistics recomputed:  dx = rstd * (g - mean(g) - xhat * mean(g * xhat)) (+ dres)
// kStats (the affine backward below): lane 0 also stores the row's (mean, rstd) for the weight-gradient pass; dx is computed by the same
// code either way, so the two entries give the same dx bits.
template <int VPL, bool kStats = false>
__global__ void __launch_bounds__(256) layernorm_bwd_warp_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                                                                 const bf16* __restrict__ w, const bf16* __restrict__ dres,
                                                                 bf16* __restrict__ dx, int T, int H, float eps,
                                                                 float2* __restrict__ stats = nullptr) {
  const int lane = threadIdx.x & 31;
  const long row = (static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (row >= T) return;
  const int nvec = H >> 3;
  float xv[VPL][8], gv[VPL][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int v = lane + i * 32;
    if (v < nvec) {
      up8(reinterpret_cast<const V8*>(x + row * H)[v], xv[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += xv[i][j];
    }
  }
  const float mean = warp_sum(sum) / static_cast<float>(H);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int v = lane + i * 32;
    if (v < nvec)
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float d = xv[i][j] - mean; sq += d * d; }
  }
  const float rstd = rsqrtf(warp_sum(sq) / static_cast<float>(H) + eps);
  if constexpr (kStats) {
    if (lane == 0) stats[row] = make_float2(mean, rstd);
  }
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int v = lane + i * 32;
    if (v < nvec) {
      float d[8], wf[8];
      up8(reinterpret_cast<const V8*>(dy + row * H)[v], d);
      up8(reinterpret_cast<const V8*>(w)[v], wf);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        xv[i][j] = (xv[i][j] - mean) * rstd;
        gv[i][j] = d[j] * wf[j];
        s1 += gv[i][j];
        s2 += gv[i][j] * xv[i][j];
      }
    }
  }
  s1 = warp_sum(s1) / static_cast<float>(H);
  s2 = warp_sum(s2) / static_cast<float>(H);
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int v = lane + i * 32;
    if (v < nvec) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = rstd * (gv[i][j] - s1 - xv[i][j] * s2);
      if (dres) {
        float r[8];
        up8(reinterpret_cast<const V8*>(dres + row * H)[v], r);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] += r[j];
      }
      reinterpret_cast<V8*>(dx + row * H)[v] = pk8(o);
    }
  }
}
int layernorm_bwd(const void* dy, const void* x, const void* w, const void* dres, void* dx, int T, int H, float eps, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(dy, x, w, dres, dx);
  const int nvec = H / 8;
  if (H % 8 || nvec > 32 * 6 || T <= 0) return DLLM_ERR_SHAPE;
  const unsigned grid = static_cast<unsigned>((static_cast<long>(T) * 32 + 255) / 256);
  if (nvec <= 64) layernorm_bwd_warp_kernel<2><<<grid, 256, 0, s>>>((const bf16*)dy, (const bf16*)x, (const bf16*)w, (const bf16*)dres, (bf16*)dx, T, H, eps);
  else if (nvec <= 128) layernorm_bwd_warp_kernel<4><<<grid, 256, 0, s>>>((const bf16*)dy, (const bf16*)x, (const bf16*)w, (const bf16*)dres, (bf16*)dx, T, H, eps);
  else layernorm_bwd_warp_kernel<6><<<grid, 256, 0, s>>>((const bf16*)dy, (const bf16*)x, (const bf16*)w, (const bf16*)dres, (bf16*)dx, T, H, eps);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// ---- LayerNorm backward with the affine gradients (CLIP tower training).  dx: the warp kernel above with kStats, so it is bit-identical
// to layernorm_bwd.  dgamma[h] = sum_t dy[t, h] * xhat[t, h], dbeta[h] = sum_t dy[t, h] (xhat = (x - mean) * rstd in fp32, as the dx
// kernel forms it): the rmsnorm_bwd_dw pattern — CTA (32 column vectors, row split) keeps 8 row groups of fp32 sums, adds them through
// shared memory in group order and writes one partial row per split; a second kernel adds the kLnSplits partials in split order.  No
// atomics: the bits depend only on the inputs and (T, H).
constexpr int kLnSplits = 64;
__global__ void __launch_bounds__(256) layernorm_bwd_dwb_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                                                                const float2* __restrict__ stats, float* __restrict__ partial, int T,
                                                                int H) {
  __shared__ float sg[8][32][9], sb[8][32][9];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int v = blockIdx.x * 32 + tx;
  const int nvec = H >> 3;
  const int rows_per = (T + kLnSplits - 1) / kLnSplits;
  const int r0 = blockIdx.y * rows_per;
  const int r1 = min(T, r0 + rows_per);
  float ag[8], ab[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) ag[j] = ab[j] = 0.f;
  if (v < nvec) {
#pragma unroll 2
    for (int r = r0 + ty; r < r1; r += 8) {
      const long off = static_cast<long>(r) * H;
      float d[8], xx[8];
      up8(reinterpret_cast<const V8*>(dy + off)[v], d);
      up8(reinterpret_cast<const V8*>(x + off)[v], xx);
      const float2 st = stats[r];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        ag[j] += d[j] * ((xx[j] - st.x) * st.y);
        ab[j] += d[j];
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    sg[ty][tx][j] = ag[j];
    sb[ty][tx][j] = ab[j];
  }
  __syncthreads();
  if (ty == 0 && v < nvec) {
    float* pg = partial + static_cast<size_t>(blockIdx.y) * 2 * H;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float g = 0.f, b = 0.f;
#pragma unroll
      for (int y = 0; y < 8; ++y) {
        g += sg[y][tx][j];
        b += sb[y][tx][j];
      }
      pg[v * 8 + j] = g;
      pg[H + v * 8 + j] = b;
    }
  }
}
__global__ void __launch_bounds__(256) layernorm_dwb_final_kernel(const float* __restrict__ partial, bf16* __restrict__ dgamma,
                                                                  bf16* __restrict__ dbeta, int H) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= H) return;
  float g = 0.f, b = 0.f;
  for (int p = 0; p < kLnSplits; ++p) {
    g += partial[static_cast<size_t>(p) * 2 * H + h];
    b += partial[static_cast<size_t>(p) * 2 * H + H + h];
  }
  dgamma[h] = __float2bfloat16_rn(g);
  dbeta[h] = __float2bfloat16_rn(b);
}

size_t layernorm_bwd_affine_workspace(int T, int H) {
  if (T <= 0 || H <= 0) return 0;
  return static_cast<size_t>(T) * sizeof(float2) + static_cast<size_t>(kLnSplits) * 2 * H * sizeof(float);
}

int layernorm_bwd_affine(const void* dy, const void* x, const void* w, const void* dres, void* dx, void* dgamma, void* dbeta,
                         void* workspace, size_t ws_bytes, int T, int H, float eps, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(dy, x, w, dres, dx, workspace);
  const int nvec = H / 8;
  if (H % 8 || nvec > 32 * 6 || T <= 0 || !dgamma || !dbeta || !dx) return DLLM_ERR_SHAPE;
  if (ws_bytes < layernorm_bwd_affine_workspace(T, H)) return DLLM_ERR_SHAPE;
  float2* stats = static_cast<float2*>(workspace);
  float* partial = reinterpret_cast<float*>(static_cast<char*>(workspace) + static_cast<size_t>(T) * sizeof(float2));
  const unsigned grid = static_cast<unsigned>((static_cast<long>(T) * 32 + 255) / 256);
  if (nvec <= 64)
    layernorm_bwd_warp_kernel<2, true><<<grid, 256, 0, s>>>((const bf16*)dy, (const bf16*)x, (const bf16*)w, (const bf16*)dres, (bf16*)dx, T, H, eps, stats);
  else if (nvec <= 128)
    layernorm_bwd_warp_kernel<4, true><<<grid, 256, 0, s>>>((const bf16*)dy, (const bf16*)x, (const bf16*)w, (const bf16*)dres, (bf16*)dx, T, H, eps, stats);
  else
    layernorm_bwd_warp_kernel<6, true><<<grid, 256, 0, s>>>((const bf16*)dy, (const bf16*)x, (const bf16*)w, (const bf16*)dres, (bf16*)dx, T, H, eps, stats);
  layernorm_bwd_dwb_kernel<<<dim3((nvec + 31) / 32, kLnSplits), 256, 0, s>>>((const bf16*)dy, (const bf16*)x, stats, partial, T, H);
  layernorm_dwb_final_kernel<<<(H + 255) / 256, 256, 0, s>>>(partial, (bf16*)dgamma, (bf16*)dbeta, H);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// ---- Quick-GELU (CLIP MLP, transformers activations.QuickGELU) for the trainable tower, whose backward needs the pre-activation: fc1
// runs as a bias-only GEMM and this kernel applies y = x * sigmoid(1.702 x) with the GEMM epilogue's formula (x / (1 + exp(-1.702 x))),
// fp32, one rounding.  Backward: dx = dy * (s + 1.702 x s (1 - s)), s = sigmoid(1.702 x).  8 elements (one 16-byte vector) per thread.
__global__ void quick_gelu_kernel(const V8* __restrict__ x, V8* __restrict__ y, long nvec) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= nvec) return;
  float f[8];
  up8(x[i], f);
#pragma unroll
  for (int j = 0; j < 8; ++j) f[j] = f[j] / (1.f + expf(-1.702f * f[j]));
  y[i] = pk8(f);
}
__global__ void quick_gelu_bwd_kernel(const V8* __restrict__ dy, const V8* __restrict__ x, V8* __restrict__ dx, long nvec) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= nvec) return;
  float g[8], f[8];
  up8(dy[i], g);
  up8(x[i], f);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float sg = 1.f / (1.f + expf(-1.702f * f[j]));
    g[j] = g[j] * (sg + 1.702f * f[j] * sg * (1.f - sg));
  }
  dx[i] = pk8(g);
}
int quick_gelu(const void* x, void* y, long n, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(x, y);
  if (n <= 0 || n % 8 || !x || !y) return DLLM_ERR_SHAPE;
  const long nvec = n / 8;
  quick_gelu_kernel<<<static_cast<unsigned>((nvec + 255) / 256), 256, 0, s>>>((const V8*)x, (V8*)y, nvec);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}
int quick_gelu_bwd(const void* dy, const void* x, void* dx, long n, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(dy, x, dx);
  if (n <= 0 || n % 8 || !dy || !x || !dx) return DLLM_ERR_SHAPE;
  const long nvec = n / 8;
  quick_gelu_bwd_kernel<<<static_cast<unsigned>((nvec + 255) / 256), 256, 0, s>>>((const V8*)dy, (const V8*)x, (V8*)dx, nvec);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// ---- GEGLU backward: d_h = dout * gelu(g);  d_g = dout * h * gelu'(g)
__global__ void geglu_bwd_kernel(const bf16* __restrict__ dout, const bf16* __restrict__ in, bf16* __restrict__ din, int T, int I) {
  const int nvec = I >> 3;
  const long gid = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (gid >= static_cast<long>(T) * nvec) return;
  const int v = static_cast<int>(gid % nvec);
  const long t = gid / nvec;
  float a[8], g[8], d[8], oa[8], og[8];
  up8(*reinterpret_cast<const V8*>(in + t * 2 * I + v * 8), a);
  up8(*reinterpret_cast<const V8*>(in + t * 2 * I + I + v * 8), g);
  up8(*reinterpret_cast<const V8*>(dout + t * I + v * 8), d);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float cdf = 0.5f * (1.f + erff(g[j] * 0.70710678118654752f));
    const float pdf = 0.3989422804014327f * expf(-0.5f * g[j] * g[j]);
    oa[j] = d[j] * r16(g[j] * cdf);
    og[j] = d[j] * a[j] * (cdf + g[j] * pdf);
  }
  *reinterpret_cast<V8*>(din + t * 2 * I + v * 8) = pk8(oa);
  *reinterpret_cast<V8*>(din + t * 2 * I + I + v * 8) = pk8(og);
}
int geglu_bwd(const void* dout, const void* in, void* din, int T, int I, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(dout, in, din);
  if (I % 8 || T <= 0) return DLLM_ERR_SHAPE;
  const long total = static_cast<long>(T) * (I / 8);
  geglu_bwd_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>((const bf16*)dout, (const bf16*)in, (bf16*)din, T, I);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// ---- spatial backward helpers
// nearest-2x upsample backward: dx[n,h,w] = sum of the 4 children
__global__ void upsample2x_bwd_kernel(const bf16* __restrict__ dy, bf16* __restrict__ dx, int N, int H, int W, int C) {
  const int nvec = C >> 3;
  const long gid = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (gid >= static_cast<long>(N) * H * W * nvec) return;
  const int v = static_cast<int>(gid % nvec);
  long p = gid / nvec;
  const int w = static_cast<int>(p % W); p /= W;
  const int h = static_cast<int>(p % H);
  const int n = static_cast<int>(p / H);
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      float f[8];
      up8(reinterpret_cast<const V8*>(dy + ((static_cast<size_t>(n) * 2 * H + 2 * h + i) * 2 * W + 2 * w + j) * C)[v], f);
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] += f[e];
    }
  reinterpret_cast<V8*>(dx)[gid] = pk8(acc);
}
// col2im of the stride-2 3x3 pad-1 conv: dx[n,h,w,c] = sum_{r,s: (h-r+1), (w-s+1) even, in range} dcols[n, (h-r+1)/2, (w-s+1)/2, (r,s,c)]
__global__ void col2im_s2_kernel(const bf16* __restrict__ dcols, bf16* __restrict__ dx, int N, int H, int W, int C) {
  const int nvec = C >> 3;
  const int Ho = H / 2, Wo = W / 2;
  const long gid = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (gid >= static_cast<long>(N) * H * W * nvec) return;
  const int v = static_cast<int>(gid % nvec);
  long p = gid / nvec;
  const int w = static_cast<int>(p % W); p /= W;
  const int h = static_cast<int>(p % H);
  const int n = static_cast<int>(p / H);
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int r = 0; r < 3; ++r) {
    const int hh = h - r + 1;
    if (hh < 0 || (hh & 1) || hh / 2 >= Ho) continue;
    for (int sx = 0; sx < 3; ++sx) {
      const int ww = w - sx + 1;
      if (ww < 0 || (ww & 1) || ww / 2 >= Wo) continue;
      float f[8];
      up8(reinterpret_cast<const V8*>(dcols + (((static_cast<size_t>(n) * Ho + hh / 2) * Wo + ww / 2) * 9 + r * 3 + sx) * C)[v], f);
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] += f[e];
    }
  }
  reinterpret_cast<V8*>(dx)[gid] = pk8(acc);
}
// general column-block copy: dst[:, dcol0 : dcol0+n] = src[:, scol0 : scol0+n]
__global__ void copy_cols2_kernel(const bf16* __restrict__ src, bf16* __restrict__ dst, long rows, int Cs, int Cd, int scol0, int dcol0, int ncols) {
  const int nvec = ncols >> 3;
  const long gid = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (gid >= rows * nvec) return;
  const int v = static_cast<int>(gid % nvec);
  const long r = gid / nvec;
  *reinterpret_cast<uint4*>(dst + r * Cd + dcol0 + v * 8) = *reinterpret_cast<const uint4*>(src + r * Cs + scol0 + v * 8);
}
int upsample2x_bwd_nhwc(const void* dy, void* dx, int N, int H, int W, int C, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(dy, dx);
  if (C % 8) return DLLM_ERR_SHAPE;
  const long total = static_cast<long>(N) * H * W * (C / 8);
  upsample2x_bwd_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>((const bf16*)dy, (bf16*)dx, N, H, W, C);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}
int col2im_s2_nhwc(const void* dcols, void* dx, int N, int H, int W, int C, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(dcols, dx);
  if (C % 8 || H % 2 || W % 2) return DLLM_ERR_SHAPE;
  const long total = static_cast<long>(N) * H * W * (C / 8);
  col2im_s2_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>((const bf16*)dcols, (bf16*)dx, N, H, W, C);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}
int copy_cols2(const void* src, void* dst, long rows, int Cs, int Cd, int scol0, int dcol0, int ncols, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(src, dst);
  if (Cs % 8 || Cd % 8 || scol0 % 8 || dcol0 % 8 || ncols % 8 || rows <= 0) return DLLM_ERR_SHAPE;
  const long total = rows * (ncols / 8);
  copy_cols2_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>((const bf16*)src, (bf16*)dst, rows, Cs, Cd, scol0, dcol0, ncols);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// ---- conv_out backward: deps fp32 NCHW [B,4,H,W] -> dx NHWC bf16 [B,H,W,C]; w [4, C, 3, 3]
template <int COUT>
__global__ void conv_out_bwd_kernel(const float* __restrict__ dy, const bf16* __restrict__ w, bf16* __restrict__ dx, int B, int C, int H, int W) {
  const int nvec = C >> 3;
  const long gid = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (gid >= static_cast<long>(B) * H * W * nvec) return;
  const int v = static_cast<int>(gid % nvec);
  long p = gid / nvec;
  const int wx = static_cast<int>(p % W); p /= W;
  const int hy = static_cast<int>(p % H);
  const int n = static_cast<int>(p / H);
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int r = 0; r < 3; ++r) {
    const int h = hy - r + 1;
    if (h < 0 || h >= H) continue;
    for (int sx = 0; sx < 3; ++sx) {
      const int ww = wx - sx + 1;
      if (ww < 0 || ww >= W) continue;
#pragma unroll
      for (int o = 0; o < COUT; ++o) {
        const float g = dy[((static_cast<size_t>(n) * COUT + o) * H + h) * W + ww];
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] += g * __bfloat162float(w[((static_cast<size_t>(o) * C + v * 8 + e) * 3 + r) * 3 + sx]);
      }
    }
  }
  reinterpret_cast<V8*>(dx)[gid] = pk8(acc);
}
int conv_out_bwd(const float* dy, const void* w, void* dx, int B, int C, int H, int W, int Cout, cudaStream_t s) {
  if (Cout != 4 || C % 8) return DLLM_ERR_UNSUPPORTED;
  const long total = static_cast<long>(B) * H * W * (C / 8);
  conv_out_bwd_kernel<4><<<static_cast<unsigned>((total + 127) / 128), 128, 0, s>>>(dy, (const bf16*)w, (bf16*)dx, B, C, H, W);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// ---- diffusion loss plumbing (StableDiffusionHead.forward, modeling_plugins.py:520-559)
// noisy = sqrt(ac[t_n]) * x0 + sqrt(1 - ac[t_n]) * noise     (DDPMScheduler.add_noise), per-sample timestep
__global__ void add_noise_kernel(const float* __restrict__ x0, const float* __restrict__ noise, const int* __restrict__ t,
                                 const float* __restrict__ alphas_cumprod, float* __restrict__ out, long per_sample, long total) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const float a = alphas_cumprod[t[i / per_sample]];
  out[i] = sqrtf(a) * x0[i] + sqrtf(1.f - a) * noise[i];
}
int add_noise(const float* x0, const float* noise, const int* t, const float* ac, float* out, int B, long per_sample, cudaStream_t s) {
  const long total = static_cast<long>(B) * per_sample;
  add_noise_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>(x0, noise, t, ac, out, per_sample, total);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}
// loss = mean((pred - target)^2) in fp32 (:559), dpred = 2 (pred - target) / n   (single CTA: n = B*4*64*64 is tiny)
__global__ void mse_fwd_bwd_kernel(const float* __restrict__ pred, const float* __restrict__ target, float* __restrict__ loss,
                                   float* __restrict__ dpred, long n) {
  __shared__ float red[32];
  float acc = 0.f;
  const float inv = 1.f / static_cast<float>(n);
  for (long i = threadIdx.x; i < n; i += blockDim.x) {
    const float d = pred[i] - target[i];
    acc += d * d;
    dpred[i] = 2.f * d * inv;
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = (threadIdx.x < (blockDim.x >> 5)) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) loss[0] = v * inv;
  }
}
int mse_fwd_bwd(const float* pred, const float* target, float* loss, float* dpred, long n, cudaStream_t s) {
  mse_fwd_bwd_kernel<<<1, 1024, 0, s>>>(pred, target, loss, dpred, n);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}
// min-SNR weighted variant (reference modeling_plugins.py:561-572, `_compute_snr` :468-491):
//   snr_b = (sqrt(ac[t_b]) / sqrt(1 - ac[t_b]))^2,  w_b = min(snr_b, gamma) / snr_b,
//   loss = mean_b( w_b * mean_chw((pred - target)^2) ),  dpred = 2 w_b (pred - target) / n.
__global__ void mse_minsnr_fwd_bwd_kernel(const float* __restrict__ pred, const float* __restrict__ target, const int* __restrict__ t,
                                          const float* __restrict__ alphas_cumprod, float gamma, float* __restrict__ loss,
                                          float* __restrict__ dpred, long per_sample, long n) {
  __shared__ float red[32];
  float acc = 0.f;
  const float inv = 1.f / static_cast<float>(n);
  for (long i = threadIdx.x; i < n; i += blockDim.x) {
    const float ac = alphas_cumprod[t[i / per_sample]];
    const float r = sqrtf(ac) / sqrtf(1.f - ac);
    const float snr = r * r;
    const float w = fminf(snr, gamma) / snr;
    const float d = pred[i] - target[i];
    acc += w * d * d;
    dpred[i] = 2.f * w * d * inv;
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = (threadIdx.x < (blockDim.x >> 5)) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) loss[0] = v * inv;
  }
}
int mse_minsnr_fwd_bwd(const float* pred, const float* target, const int* t, const float* ac, float gamma, float* loss, float* dpred,
                       int B, long per_sample, cudaStream_t s) {
  if (B <= 0 || per_sample <= 0 || !(gamma > 0.f)) return DLLM_ERR_SHAPE;
  mse_minsnr_fwd_bwd_kernel<<<1, 1024, 0, s>>>(pred, target, t, ac, gamma, loss, dpred, per_sample, static_cast<long>(B) * per_sample);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}


// ================================================================================================ VAE encoder helpers
// AutoencoderKL mid-block attention is ONE head of dim 512 (SURVEY A.3): run as GEMM -> row softmax -> GEMM.
// In-place row softmax of bf16 scores with fp32 math: p = softmax(x * scale).
__global__ void __launch_bounds__(256) softmax_rows_kernel(bf16* __restrict__ x, int cols, float scale) {
  __shared__ float red[8];
  bf16* row = x + static_cast<size_t>(blockIdx.x) * cols;
  const int nvec = cols >> 3;
  float m = -INFINITY;
  for (int v = threadIdx.x; v < nvec; v += 256) {
    float f[8];
    up8(reinterpret_cast<const V8*>(row)[v], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) m = fmaxf(m, f[j]);
  }
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int v = threadIdx.x; v < nvec; v += 256) {
    float f[8];
    up8(reinterpret_cast<const V8*>(row)[v], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) sum += expf((f[j] - m) * scale);
  }
  sum = warp_sum(sum);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) sum += red[i];
  const float inv = 1.f / sum;
  for (int v = threadIdx.x; v < nvec; v += 256) {
    float f[8];
    up8(reinterpret_cast<const V8*>(row)[v], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = expf((f[j] - m) * scale) * inv;
    reinterpret_cast<V8*>(row)[v] = pk8(f);
  }
}
int softmax_rows(void* x, long rows, int cols, float scale, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(x);
  if (cols % 8 || rows <= 0) return DLLM_ERR_SHAPE;
  softmax_rows_kernel<<<static_cast<unsigned>(rows), 256, 0, s>>>((bf16*)x, cols, scale);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}
// quant_conv (1x1, 2L -> 2L) + DiagonalGaussianDistribution.sample() + scaling_factor (modeling_plugins.py:511-512):
//   moments = Wq h + bq; mean, logvar = chunk(moments); latents = (mean + exp(0.5 * clamp(logvar, -30, 20)) * z) * scaling
__global__ void vae_sample_kernel(const float* __restrict__ h, const bf16* __restrict__ wq, const bf16* __restrict__ bq,
                                  const float* __restrict__ z, float* __restrict__ out, int B, int L, long plane, float scaling) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long>(B) * plane) return;
  const int n = static_cast<int>(i / plane);
  const long p = i - n * plane;
  float hv[16];
  for (int c = 0; c < 2 * L; ++c) hv[c] = h[(static_cast<size_t>(n) * 2 * L + c) * plane + p];
  for (int o = 0; o < L; ++o) {
    float mean = __bfloat162float(bq[o]), logvar = __bfloat162float(bq[L + o]);
    for (int c = 0; c < 2 * L; ++c) {
      mean += __bfloat162float(wq[o * 2 * L + c]) * hv[c];
      logvar += __bfloat162float(wq[(L + o) * 2 * L + c]) * hv[c];
    }
    mean = r16(mean);
    logvar = fminf(fmaxf(r16(logvar), -30.f), 20.f);
    out[(static_cast<size_t>(n) * L + o) * plane + p] = (mean + expf(0.5f * logvar) * z[(static_cast<size_t>(n) * L + o) * plane + p]) * scaling;
  }
}
int vae_sample(const float* h, const void* wq, const void* bq, const float* z, float* out, int B, int L, long plane, float scaling,
               cudaStream_t s) {
  if (L > 8) return DLLM_ERR_UNSUPPORTED;
  const long total = static_cast<long>(B) * plane;
  vae_sample_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>(h, (const bf16*)wq, (const bf16*)bq, z, out, B, L, plane, scaling);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

}  // namespace dllm
