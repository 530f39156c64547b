// One-token decode step of the kv-cache (sm_90a): split-KV attention whose cache length is read from the device, and the RoPE + cache
// append that precedes it.  Neither kernel takes a host value that changes from token to token, so a captured launch stays valid while
// the cache grows (dreamllm_b200/decode.py replays the whole decode step as one CUDA graph).
//
//   attn_decode_kernel  : CTA = (kv split, kv head, batch), one warpgroup.  The group's q heads (1, 2, 4 or 8) are the first rows of a
//                         zero-padded 64-row wgmma tile, so K/V are read once per group; 64-row K/V chunks stream through a TMA ring
//                         (S = Q K^T from two shared-memory operands, P.V with P from registers, as attn_fwd_kernel).  Each split
//                         writes one fp32 partial (o, running max, sum) per q head.
//   attn_decode_combine : one CTA per (q head, batch) merges the partials in fixed split order -> bf16 out.  No atomics.
//   rope_append_kv      : rope_kernel's arithmetic on the new token's q and k at device positions, plus the k/v write to cache row *kv_len.
#include "common.cuh"
#include "gemm_sm90.h"
#include "ops.h"
#include "wgmma.cuh"

namespace dllm {
namespace {

constexpr int kDecChunk = 64;               // kv rows per ring stage (the N of the S = Q K^T wgmma)
constexpr int kDecRefLen = 2048;            // planner: cache length at which the grid should hold ~2 CTAs per SM
constexpr float kLog2e = 1.4426950408889634f;

template <int D>
struct DecSmem {
  static constexpr int NCH = D / 64;                    // 64-column (128-byte) swizzle chunks of a row
  static constexpr int kStages = D == 128 ? 2 : 4;      // 16 + 64 / 8 + 64 KB: two (d 128) or three (d 64) CTAs per SM
  static constexpr int kTile = NCH * 64 * 128;          // Q, or one K (or V) chunk: [NCH][64 rows][128 B]
  static constexpr int kStage = 2 * kTile;
  static constexpr int oQ = 0, oRing = kTile, oBar = oRing + kStages * kStage;
  static constexpr int kBytes = oBar + 8 * kStages + 1024 /*align slack*/;
};

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
// K step ks (16 columns) of a K-major [NCH][64 rows][128 B] tile; 16 rows (one MN-major K step) of a V chunk
__device__ __forceinline__ uint64_t kmajor_desc(uint32_t base, int ks) {
  return make_smem_desc(base + (ks >> 2) * (64 * 128) + (ks & 3) * 32u, 16u, 1024u);
}
__device__ __forceinline__ uint64_t mnmajor_desc(uint32_t base, int kk) { return make_smem_desc(base + kk * 2048u, 64 * 128, 1024u); }

// The arithmetic of attn_fwd_kernel (attn_sm90.cu) on a 64-key chunk: S = q.k in fp32, masked keys -inf, p = exp2(S * scale log2e - m)
// rounded to bf16 for P.V, the running sum over the unrounded p.  Only the order of the sums differs (per split, merged by the combine).
// m64nN accumulator: element 4j + 2h + e of thread t sits at row 16 (t / 32) + (t % 32) / 4 + 8h, column 8j + 2 (t % 4) + e, so the
// group's rows (< 8) are the h = 0 elements of warp 0; the other rows are zero-q padding and are never stored.
// part_o [n_splits, B, nh, D], part_ml [n_splits, B, nh, 2].
template <int D>
__global__ void __launch_bounds__(128) attn_decode_kernel(const __grid_constant__ CUtensorMap tk, const __grid_constant__ CUtensorMap tv,
                                                          const bf16* __restrict__ q, long ld_q, const int* __restrict__ kv_len_ptr,
                                                          const uint8_t* __restrict__ kv_mask, int mask_ld, int max_len,
                                                          float* __restrict__ part_o, float* __restrict__ part_ml, int B, int nh,
                                                          int group, int split_len, float scale_log2) {
  using L = DecSmem<D>;
  constexpr int ST = L::kStages;
  constexpr int NJ = kDecChunk / 8;
  const int split = blockIdx.x, hk = blockIdx.y, b = blockIdx.z;
  const int t = threadIdx.x;
  const int row_t = 16 * (t >> 5) + ((t & 31) >> 2), c_in = 2 * (t & 3);
  const int kv_len = *kv_len_ptr;
  const int start = split * split_len;
  const int end = min(start + split_len, kv_len);
  const int n_chunks = end > start ? (end - start + kDecChunk - 1) / kDecChunk : 0;

  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

  if (n_chunks > 0) {   // otherwise the split starts at or past kv_len: a neutral partial (m -inf, l 0, o 0)
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + L::oBar);
    const int row_base = b * max_len + start;    // the maps are [B * max_len, nkv * D]
    auto load = [&](int j) {
      const int st = j % ST;
      uint8_t* dst = smem + L::oRing + st * L::kStage;
      mbar_arrive_expect_tx(&full[st], 2 * kDecChunk * D * 2);
#pragma unroll
      for (int c = 0; c < L::NCH; ++c) {
        tma_load_2d(dst + c * 64 * 128, &tk, &full[st], hk * D + c * 64, row_base + j * kDecChunk);
        tma_load_2d(dst + L::kTile + c * 64 * 128, &tv, &full[st], hk * D + c * 64, row_base + j * kDecChunk);
      }
    };
    if (t == 0) {
      tma_prefetch_desc(&tk);
      tma_prefetch_desc(&tv);
      for (int s = 0; s < ST; ++s) mbar_init(&full[s], 1);
      fence_mbar_init();
      for (int j = 0; j < ST && j < n_chunks; ++j) load(j);
    }
    // Q tile in the TMA box's 128B-swizzled layout: 16-byte unit u of row r at unit u ^ (r & 7); rows >= group are zero
    for (int u = t; u < 64 * (D / 8); u += 128) {
      const int r = u / (D / 8), cu = u % (D / 8);
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (r < group) v = *reinterpret_cast<const uint4*>(q + static_cast<size_t>(b) * ld_q + static_cast<size_t>(hk * group + r) * D + cu * 8);
      *reinterpret_cast<uint4*>(smem + L::oQ + (cu >> 3) * (64 * 128) + r * 128 + (((cu & 7) ^ (r & 7)) << 4)) = v;
    }
    fence_proxy_async_smem();   // generic-proxy writes of Q before the wgmma (async proxy) reads them
    __syncthreads();            // and the barrier init before any wait

    const uint32_t sQ = smem_u32(smem + L::oQ);
    const uint8_t* mrow = kv_mask ? kv_mask + static_cast<size_t>(b) * mask_ld : nullptr;
    for (int j = 0; j < n_chunks; ++j) {
      const int st = j % ST;
      mbar_wait(&full[st], (j / ST) & 1, 1);
      const uint32_t sK = smem_u32(smem + L::oRing + st * L::kStage), sV = sK + L::kTile;
      float s[kDecChunk / 2];
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < D / 16; ++ks) wgmma_ss<kDecChunk, 0, 0>(s, kmajor_desc(sQ, ks), kmajor_desc(sK, ks), ks > 0);
      wgmma_commit();
      wgmma_wait<0>();
      const int kv0 = start + j * kDecChunk;
#pragma unroll
      for (int jj = 0; jj < NJ; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int kvi = kv0 + 8 * jj + c_in + e;
          bool ok = kvi < end;
          if (ok && mrow != nullptr) ok = mrow[kvi] != 0;
          if (!ok) s[4 * jj + e] = s[4 * jj + 2 + e] = -INFINITY;
        }
      float alpha[2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        float mx = -INFINITY;
#pragma unroll
        for (int jj = 0; jj < NJ; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * hh], s[4 * jj + 2 * hh + 1]));
        mx = quad_max(mx);
        const float m_new = fmaxf(m_run[hh], mx * scale_log2);
        alpha[hh] = (m_run[hh] == -INFINITY) ? 0.f : exp2f(m_run[hh] - m_new);
        m_run[hh] = m_new;
        const float m_use = (m_new == -INFINITY) ? 0.f : m_new;
        float ls = 0.f;
#pragma unroll
        for (int jj = 0; jj < NJ; ++jj)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float p = exp2f(s[4 * jj + 2 * hh + e] * scale_log2 - m_use);
            s[4 * jj + 2 * hh + e] = p;
            ls += p;
          }
        l_run[hh] = l_run[hh] * alpha[hh] + ls;
      }
#pragma unroll
      for (int jj = 0; jj < D / 8; ++jj) {
        o[4 * jj + 0] *= alpha[0]; o[4 * jj + 1] *= alpha[0];
        o[4 * jj + 2] *= alpha[1]; o[4 * jj + 3] *= alpha[1];
      }
      // the m64nN accumulator's 16-column slice kk, rounded to bf16, is the m64k16 A fragment of a register-A wgmma
      uint32_t pf[kDecChunk / 16][4];
#pragma unroll
      for (int kk = 0; kk < kDecChunk / 16; ++kk) {
        pf[kk][0] = pack_bf16(s[8 * kk + 0], s[8 * kk + 1]);
        pf[kk][1] = pack_bf16(s[8 * kk + 2], s[8 * kk + 3]);
        pf[kk][2] = pack_bf16(s[8 * kk + 4], s[8 * kk + 5]);
        pf[kk][3] = pack_bf16(s[8 * kk + 6], s[8 * kk + 7]);
      }
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kDecChunk / 16; ++kk) wgmma_rs<D, 1>(o, pf[kk], mnmajor_desc(sV, kk), 1);
      wgmma_commit();
      wgmma_wait<0>();
      __syncthreads();   // the warpgroup is done with stage st
      if (t == 0 && j + ST < n_chunks) load(j + ST);
    }
    l_run[0] = quad_sum(l_run[0]);
  }
  if (row_t < group) {   // warp 0, h = 0
    const size_t prow = (static_cast<size_t>(split) * B + b) * nh + hk * group + row_t;
    float* po = part_o + prow * D + c_in;
#pragma unroll
    for (int jj = 0; jj < D / 8; ++jj) *reinterpret_cast<float2*>(po + 8 * jj) = make_float2(o[4 * jj], o[4 * jj + 1]);
    if ((t & 3) == 0) *reinterpret_cast<float2*>(part_ml + prow * 2) = make_float2(m_run[0], l_run[0]);
  }
}

// out[b, h * D + c] = sum_s w_s o_s[c] / sum_s w_s l_s, w_s = exp2(m_s - max m), partials taken in index order
template <int D>
__global__ void __launch_bounds__(D) attn_decode_combine_kernel(const float* __restrict__ part_o, const float* __restrict__ part_ml,
                                                                bf16* __restrict__ out, long ld_o, int B, int nh, int n_sub) {
  const int h = blockIdx.x, b = blockIdx.y, c = threadIdx.x;
  const size_t stride = static_cast<size_t>(B) * nh;
  const size_t row0 = static_cast<size_t>(b) * nh + h;
  float M = -INFINITY;
  for (int s = 0; s < n_sub; ++s) M = fmaxf(M, part_ml[(s * stride + row0) * 2]);
  float acc = 0.f, l = 0.f;
  if (M != -INFINITY) {
    for (int s = 0; s < n_sub; ++s) {
      const float2 ml = *reinterpret_cast<const float2*>(part_ml + (s * stride + row0) * 2);
      const float w = ml.x == -INFINITY ? 0.f : exp2f(ml.x - M);
      l += w * ml.y;
      acc += w * part_o[(s * stride + row0) * D + c];
    }
  }
  const float inv = l > 0.f ? 1.f / l : 0.f;
  out[static_cast<size_t>(b) * ld_o + static_cast<size_t>(h) * D + c] = __float2bfloat16_rn(acc * inv);
}

// ------------------------------------------------------------------------------------------------ RoPE + append
// rope_kernel<D> (elementwise.cu) with mode +1 on the q and k heads of one token per row, at positions pos[b]; the rotated k heads and the
// v heads are also written to cache row *kv_len.  Threads of the v heads only copy.
__device__ __forceinline__ void unpack8(const uint4 u, float* f) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[i]));
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  return make_uint4(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]), pack_bf16(f[6], f[7]));
}
__device__ __forceinline__ float bf16r(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

template <int D>
__global__ void rope_append_kv_kernel(bf16* __restrict__ qkv, long ld, const bf16* __restrict__ cos_t, const bf16* __restrict__ sin_t,
                                      const int* __restrict__ pos, bf16* __restrict__ k_cache, bf16* __restrict__ v_cache,
                                      const int* __restrict__ kv_len_ptr, int max_len, int B, int nh, int nkv) {
  constexpr int VPH = D / 16;
  const int heads = nh + 2 * nkv;
  const long gid = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (gid >= static_cast<long>(B) * heads * VPH) return;
  const int vi = static_cast<int>(gid % VPH);
  const long th = gid / VPH;
  const int head = static_cast<int>(th % heads);
  const int b = static_cast<int>(th / heads);
  const int row = *kv_len_ptr;
  bf16* base = qkv + static_cast<size_t>(b) * ld + static_cast<size_t>(head) * D + vi * 8;
  uint4 o1v = *reinterpret_cast<const uint4*>(base), o2v = *reinterpret_cast<const uint4*>(base + D / 2);
  if (head < nh + nkv) {
    const int p = pos[b];
    float a[8], bb[8], c1[8], c2[8], s1[8], s2[8], o1[8], o2[8];
    unpack8(o1v, a);
    unpack8(o2v, bb);
    unpack8(*reinterpret_cast<const uint4*>(cos_t + static_cast<size_t>(p) * D + vi * 8), c1);
    unpack8(*reinterpret_cast<const uint4*>(cos_t + static_cast<size_t>(p) * D + D / 2 + vi * 8), c2);
    unpack8(*reinterpret_cast<const uint4*>(sin_t + static_cast<size_t>(p) * D + vi * 8), s1);
    unpack8(*reinterpret_cast<const uint4*>(sin_t + static_cast<size_t>(p) * D + D / 2 + vi * 8), s2);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o1[j] = bf16r(a[j] * c1[j]) + bf16r(-bb[j] * s1[j]);
      o2[j] = bf16r(bb[j] * c2[j]) + bf16r(a[j] * s2[j]);
    }
    o1v = pack8(o1);
    o2v = pack8(o2);
    *reinterpret_cast<uint4*>(base) = o1v;
    *reinterpret_cast<uint4*>(base + D / 2) = o2v;
    if (head < nh) return;
  }
  if (row < 0 || row >= max_len) return;   // the host refuses an overflowing step; never write past the cache
  const bool is_k = head < nh + nkv;
  const int hk = is_k ? head - nh : head - nh - nkv;
  bf16* dst = (is_k ? k_cache : v_cache) + (static_cast<size_t>(b) * max_len + row) * nkv * D + static_cast<size_t>(hk) * D + vi * 8;
  *reinterpret_cast<uint4*>(dst) = o1v;
  *reinterpret_cast<uint4*>(dst + D / 2) = o2v;
}

}  // namespace

// Split planner: the split LENGTH depends on (B, nkv, SMs) only, so that the splits a cache row falls into (and with them the bits of the
// result) do not depend on how long the cache was allocated; max_len only sets how many splits cover it.  The length is chosen so that
// at kDecRefLen cached rows B * nkv * splits is about two CTAs per SM, and is never below one 64-row chunk.
int attn_decode_plan(int B, int nkv, int max_len, int sms, int* n_splits, int* split_len) {
  if (B <= 0 || nkv <= 0 || max_len <= 0) return DLLM_ERR_SHAPE;
  if (sms <= 0) sms = num_sms();
  const long want = static_cast<long>(kDecRefLen) * B * nkv / (2L * sms);
  long len = (want + kDecChunk - 1) / kDecChunk * kDecChunk;
  if (len < kDecChunk) len = kDecChunk;
  *split_len = static_cast<int>(len);
  *n_splits = static_cast<int>((max_len + len - 1) / len);
  return 0;
}

size_t attn_decode_workspace(int B, int nh, int nkv, int d, int max_len, int sms) {
  int ns = 0, sl = 0;
  if (attn_decode_plan(B, nkv, max_len, sms, &ns, &sl) != 0) return 0;
  return static_cast<size_t>(ns) * B * nh * (d + 2) * sizeof(float);
}

int attn_decode(const void* q, long ld_q, const void* k_cache, const void* v_cache, const int* kv_len, const void* kv_mask, int mask_ld,
                void* out, long ld_o, void* workspace, size_t ws_bytes, int B, int max_len, int nh, int nkv, int d, float scale, int sms,
                cudaStream_t s) {
  if (B <= 0 || nh <= 0 || nkv <= 0 || max_len <= 0 || nh % nkv) return DLLM_ERR_SHAPE;
  const int group = nh / nkv;
  if (group != 1 && group != 2 && group != 4 && group != 8) return DLLM_ERR_UNSUPPORTED;
  if (d != 64 && d != 128) return DLLM_ERR_UNSUPPORTED;
  if (kv_mask && mask_ld < max_len) return DLLM_ERR_SHAPE;
  if ((reinterpret_cast<uintptr_t>(q) & 15) || (ld_q & 7) || (reinterpret_cast<uintptr_t>(workspace) & 15)) return DLLM_ERR_ALIGN;
  int ns = 0, sl = 0;
  if (attn_decode_plan(B, nkv, max_len, sms, &ns, &sl) != 0) return DLLM_ERR_SHAPE;
  if (ws_bytes < attn_decode_workspace(B, nh, nkv, d, max_len, sms)) return DLLM_ERR_SHAPE;
  CUtensorMap tk, tv;
  const uint64_t rows = static_cast<uint64_t>(B) * max_len, cols = static_cast<uint64_t>(nkv) * d;
  int rc = make_tmap_2d(&tk, k_cache, 2, rows, cols, cols, kDecChunk, 64);
  if (rc) return rc;
  rc = make_tmap_2d(&tv, v_cache, 2, rows, cols, cols, kDecChunk, 64);
  if (rc) return rc;
  float* part_o = static_cast<float*>(workspace);
  float* part_ml = part_o + static_cast<size_t>(ns) * B * nh * d;
  const float scale_log2 = scale * kLog2e;
  const dim3 grid(ns, nkv, B);
  if (d == 128) {
    static bool attr = false;
    if (!attr) {
      if (cudaFuncSetAttribute(attn_decode_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, DecSmem<128>::kBytes) != cudaSuccess) {
        cudaGetLastError();
        return DLLM_ERR_LAUNCH;
      }
      attr = true;
    }
    attn_decode_kernel<128><<<grid, 128, DecSmem<128>::kBytes, s>>>(
        tk, tv, static_cast<const bf16*>(q), ld_q, kv_len, static_cast<const uint8_t*>(kv_mask), mask_ld, max_len, part_o, part_ml, B, nh,
        group, sl, scale_log2);
    attn_decode_combine_kernel<128><<<dim3(nh, B), 128, 0, s>>>(part_o, part_ml, static_cast<bf16*>(out), ld_o, B, nh, ns);
  } else {
    static bool attr = false;
    if (!attr) {
      if (cudaFuncSetAttribute(attn_decode_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, DecSmem<64>::kBytes) != cudaSuccess) {
        cudaGetLastError();
        return DLLM_ERR_LAUNCH;
      }
      attr = true;
    }
    attn_decode_kernel<64><<<grid, 128, DecSmem<64>::kBytes, s>>>(
        tk, tv, static_cast<const bf16*>(q), ld_q, kv_len, static_cast<const uint8_t*>(kv_mask), mask_ld, max_len, part_o, part_ml, B, nh,
        group, sl, scale_log2);
    attn_decode_combine_kernel<64><<<dim3(nh, B), 64, 0, s>>>(part_o, part_ml, static_cast<bf16*>(out), ld_o, B, nh, ns);
  }
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

int rope_append_kv(void* qkv, long ld, const void* cos_t, const void* sin_t, const int* pos, void* k_cache, void* v_cache,
                   const int* kv_len, int max_len, int B, int nh, int nkv, int d, cudaStream_t s) {
  DLLM_REQUIRE_ALIGN16(qkv, cos_t, sin_t, k_cache, v_cache);
  if (B <= 0 || nh <= 0 || nkv <= 0 || max_len <= 0 || (ld % 8) || ld < static_cast<long>(nh + 2 * nkv) * d) return DLLM_ERR_SHAPE;
  const long total = static_cast<long>(B) * (nh + 2 * nkv) * (d / 16);
  const int nt = 256;
  const unsigned grid = static_cast<unsigned>((total + nt - 1) / nt);
  if (d == 128)
    rope_append_kv_kernel<128><<<grid, nt, 0, s>>>((bf16*)qkv, ld, (const bf16*)cos_t, (const bf16*)sin_t, pos, (bf16*)k_cache,
                                                   (bf16*)v_cache, kv_len, max_len, B, nh, nkv);
  else if (d == 64)
    rope_append_kv_kernel<64><<<grid, nt, 0, s>>>((bf16*)qkv, ld, (const bf16*)cos_t, (const bf16*)sin_t, pos, (bf16*)k_cache,
                                                  (bf16*)v_cache, kv_len, max_len, B, nh, nkv);
  else
    return DLLM_ERR_UNSUPPORTED;
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

}  // namespace dllm
