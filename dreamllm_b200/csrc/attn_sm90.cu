// wgmma flash attention for sm_90a: forward, and backward split in two deterministic kernels (dK/dV, dQ).
//
// Replaces flash_attn_func / flash_attn_varlen_func (reference modeling_dreamllm.py:500-551) and the eager
// softmax(QK^T/sqrt(d) + mask)V path (:357-379).  q/k/v are read straight out of the fused qkv projection buffer
// ([B, S, heads, d] views with a shared token stride) through 3-D TMA maps — no transposes, no .contiguous().
//
// Common structure of the three kernels (256 threads = two warpgroups, one CTA per (tile, head, batch)):
//   * thread 0 issues the TMA loads: the CTA's own 128-row tile once, the streamed tiles through a two-stage ring (mbarrier complete_tx);
//   * each warpgroup owns 64 rows of the CTA's tile and runs its tile-GEMMs as wgmma.mma_async with the accumulators in registers;
//     S / dP come from two shared-memory operands, P / dS are fed to the next wgmma straight from registers (the m64nN accumulator
//     fragment of a 16-column slice is the m64k16 A-operand fragment, so no shuffle or shared-memory round trip is needed);
//   * the ring stage of tile j is refilled with tile j + 2 once both warpgroups have passed the CTA barrier at the end of iteration j.
// Grouped-query attention: k/v carry nkv = nh / group heads and q head h reads kv head h / group (reference repeat_kv, :242-252).  The
// forward and dQ kernels only remap the K/V column they load; the dK/dV kernel runs one CTA per kv head and sums the group's q heads.
// Packed batches (kVarlen instantiations, flash_attn_varlen_func's layout): the B samples lie end to end in one [T, cols] sequence and
// `seqlens` carries cu_seqlens [B + 1].  The tensor maps are [1, T, cols]; the CTA of (tile i, sample b) loads rows from cu[b] + 128 i, so
// tiles are aligned to the start of each sample exactly as in the padded layout and the arithmetic of a sample is that of a B = 1 call on
// it alone.  A tile's tail holds the next sample's rows (or TMA zero fill past T): they are masked as keys and as query rows like the
// padded layout's pad rows, and never stored; a CTA whose tile starts at or past its sample's length exits before it touches a barrier.
#include <stdlib.h>

#include "common.cuh"
#include "gemm_sm90.h"
#include "ops.h"
#include "wgmma.cuh"

namespace dllm {

constexpr int kAttnThreads = 256;
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

typedef CUresult (*PFN_encodeTiled3)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                     CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// [B, S, cols] bf16 view: token stride ld (elements), batch stride S*ld; box = [1, box_rows, 64 cols], 128B swizzle
static int make_tmap_bsc(CUtensorMap* map, const void* ptr, int B, int S, int cols, long ld, int box_rows) {
  static PFN_encodeTiled3 enc = nullptr;
  if (!enc) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p)
      return DLLM_ERR_DRIVER;
    enc = reinterpret_cast<PFN_encodeTiled3>(p);
  }
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || ((ld * 2) & 15)) return DLLM_ERR_ALIGN;
  cuuint64_t gdim[3] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(S), static_cast<cuuint64_t>(B)};
  cuuint64_t gstr[2] = {static_cast<cuuint64_t>(ld) * 2, static_cast<cuuint64_t>(S) * ld * 2};
  cuuint32_t box[3] = {64, static_cast<cuuint32_t>(box_rows), 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), gdim, gstr, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : DLLM_ERR_TMAP;
}

// ------------------------------------------------------------------------------------------------ fragment helpers
// m64nN fp32 accumulator of a warpgroup: element 4j + 2h + e sits at row 16 * (t / 32) + (t % 32) / 4 + 8h and column 8j + 2 (t % 4) + e
// (t = thread index in the warpgroup).  Its 16-column slice kk, rounded to bf16, is exactly the m64k16 A fragment of a register-A wgmma.
__device__ __forceinline__ void acc_to_afrag(const float* s, int kk, uint32_t* a) {
  a[0] = pack_bf16(s[8 * kk + 0], s[8 * kk + 1]);
  a[1] = pack_bf16(s[8 * kk + 2], s[8 * kk + 3]);
  a[2] = pack_bf16(s[8 * kk + 4], s[8 * kk + 5]);
  a[3] = pack_bf16(s[8 * kk + 6], s[8 * kk + 7]);
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
// Descriptors are built once per tile base and stepped with a plain add (the start-address field counts 16-byte units and no tile
// crosses the 256 KB its 14 bits span); with the K loops unrolled every step is the tile's descriptor plus a constant, so a tile's
// wgmma issue back to back instead of each behind its own descriptor arithmetic.
// K-major operand: K step ks of a tile stored as [K/64 chunks][rows][128 B] (chunk_bytes apart)
__device__ __forceinline__ uint64_t kmajor_desc0(uint32_t base) { return make_smem_desc(base, 16u, 1024u); }
__device__ __forceinline__ uint64_t kmajor_step(uint64_t d0, uint32_t chunk_bytes, int ks) {
  return d0 + (((ks >> 2) * chunk_bytes + (ks & 3) * 32u) >> 4);
}
// MN-major operand: K step ks (16 lines) of a tile stored as [MN/64 chunks][K lines][128 B]
__device__ __forceinline__ uint64_t mnmajor_desc0(uint32_t base, uint32_t chunk_bytes) { return make_smem_desc(base, chunk_bytes, 1024u); }
__device__ __forceinline__ uint64_t mnmajor_step(uint64_t d0, int ks) { return d0 + ((ks * 2048u) >> 4); }
// acc [64 rows x D] of warpgroup rows (row_t + 8h) -> bf16 * mul at dst[(base + row) * ld + col0 + col], rows < n_rows only
// (base, n_rows) = (b * S, S) in the padded layout, (cu[b], the sample's length) in the packed one
template <int D>
__device__ __forceinline__ void store_rows(const float* acc, bf16* dst, long ld, size_t base, int n_rows, int row_t, int col0, int c_in,
                                           const float* mul) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row_t + 8 * h;
    if (row >= n_rows) continue;
    bf16* p = dst + (base + row) * ld + col0 + c_in;
#pragma unroll
    for (int j = 0; j < D / 8; ++j)
      *reinterpret_cast<uint32_t*>(p + 8 * j) = pack_bf16(acc[4 * j + 2 * h] * mul[h], acc[4 * j + 2 * h + 1] * mul[h]);
  }
}

// ================================================================================================ forward
// CTA = 128 query rows of one (head, batch); KV tiles of kBKV = 128 rows stream through a two-stage ring.
constexpr int kBKV = 128;
template <int D>
struct FwdSmem {
  static constexpr int NCH = D / 64;
  static constexpr int kQ = NCH * 16384;         // [NCH][128][128B]
  static constexpr int kKV = NCH * kBKV * 128;   // [NCH][kBKV][128B]
  static constexpr int oQ = 0, oK = kQ, oV = oK + 2 * kKV, oBar = oV + 2 * kKV;
  static constexpr int kBytes = oBar + 64 + 1024 /*align slack*/;
};

template <int D, bool kCausal, bool kVarlen>
__global__ void __launch_bounds__(kAttnThreads, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk,
                const __grid_constant__ CUtensorMap tv, bf16* __restrict__ out, long ld_o, float* __restrict__ lse,
                const int* __restrict__ seqlens, int S, int Skv, int nh, int group, float scale_log2,
                const uint8_t* __restrict__ kv_mask, int mask_ld) {
  // kv_mask (nullable): [B, mask_ld] bytes, 0 = padded key position that no query may attend to — the 2-D `attention_mask` of a padded
  // batch living inside a kv-cache (reference :553-583 drops those tokens with `_upad_input`; HF left-pads decoder-only prompts)
  // causal with Skv > S = kv-cache decode / continuation (reference :344-355, :444-449): query i sits at absolute position
  // (Skv - S) + i, i.e. the mask is bottom-right aligned:  kv <= q + coff
  using L = FwdSmem<D>;
  constexpr int NCH = L::NCH;
  constexpr int NJ = kBKV / 8;                    // accumulator column blocks of S
  const int coff = kCausal ? (Skv - S) : 0;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* q_full = reinterpret_cast<uint64_t*>(smem + L::oBar);
  uint64_t* kv_full = q_full + 1;                 // [2]

  const int h = blockIdx.y, b = blockIdx.z;
  // packed: sample b is rows row0 .. row0 + len - 1 of batch entry 0 (S = Skv = T); the grid is sized for the longest sample
  const int row0 = kVarlen ? seqlens[b] : 0, bz = kVarlen ? 0 : b;
  const int len = kVarlen ? seqlens[b + 1] - row0 : 0;
  const int n_qt = kVarlen ? (len + 127) / 128 : gridDim.x;
  if (kVarlen && static_cast<int>(blockIdx.x) >= n_qt) return;
  // causal: q tile i has i + 1 KV tiles of work; launch the heaviest first so the grid's tail is made of short CTAs (LPT order)
  const int q0 = (kCausal ? (n_qt - 1 - blockIdx.x) : blockIdx.x) * 128;
  const int hkv = h / group;
  const int kv_len = kVarlen ? len : (seqlens ? min(seqlens[b], Skv) : Skv);   // Skv != S only for cross-attention (non-causal)
  const int q_len = kVarlen ? len : (seqlens ? kv_len : S);                    // right-padded self-attention: rows >= len are padding
  const int n_rows = kVarlen ? len : S;                                        // rows of out / lse this sample owns
  const int kv_end = kCausal ? min(kv_len, q0 + 128 + coff) : kv_len;
  const int n_kv = kv_end > 0 ? (kv_end + kBKV - 1) / kBKV : 0;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    mbar_init(&kv_full[0], 1);
    mbar_init(&kv_full[1], 1);
    fence_mbar_init();
  }
  __syncthreads();
  auto load_kv = [&](int j) {
    const int st = j & 1;
    mbar_arrive_expect_tx(&kv_full[st], 2 * kBKV * D * 2);
    for (int c = 0; c < NCH; ++c) {
      tma_load_3d(smem + L::oK + st * L::kKV + c * kBKV * 128, &tk, &kv_full[st], hkv * D + c * 64, row0 + j * kBKV, bz);
      tma_load_3d(smem + L::oV + st * L::kKV + c * kBKV * 128, &tv, &kv_full[st], hkv * D + c * 64, row0 + j * kBKV, bz);
    }
  };
  if (threadIdx.x == 0 && n_kv > 0) {
    mbar_arrive_expect_tx(q_full, 128 * D * 2);
    for (int c = 0; c < NCH; ++c) tma_load_3d(smem + L::oQ + c * 16384, &tq, q_full, h * D + c * 64, row0 + q0, bz);
    load_kv(0);
    if (n_kv > 1) load_kv(1);
  }

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int r_in = 16 * (t >> 5) + ((t & 31) >> 2), c_in = 2 * (t & 3);
  const int row_t = q0 + wg * 64 + r_in;          // + 8h
  const uint32_t sQ = smem_u32(smem + L::oQ) + wg * 8192;
  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  if (n_kv > 0) mbar_wait(q_full, 0, 1);
  for (int j = 0; j < n_kv; ++j) {
    const int st = j & 1;
    mbar_wait(&kv_full[st], (j >> 1) & 1, 2);
    const uint32_t sK = smem_u32(smem + L::oK + st * L::kKV), sV = smem_u32(smem + L::oV + st * L::kKV);
    float s[kBKV / 2];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < D / 16; ++ks) wgmma_ss<kBKV, 0, 0>(s, kmajor_step(kmajor_desc0(sQ), 16384, ks), kmajor_step(kmajor_desc0(sK), kBKV * 128, ks), ks > 0);
    wgmma_commit();
    wgmma_wait<0>();

    const int kv0 = j * kBKV;
    const bool need_mask = (kCausal && kv0 + kBKV - 1 > q0 + coff) || (kv0 + kBKV > kv_len) || (kv_mask != nullptr);
    if (need_mask) {
#pragma unroll
      for (int jj = 0; jj < NJ; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int kvi = kv0 + 8 * jj + c_in + e;
          bool ok = kvi < kv_len;
          if (ok && kv_mask != nullptr) ok = kv_mask[static_cast<size_t>(b) * mask_ld + kvi] != 0;
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const bool okr = ok && (!kCausal || kvi <= row_t + 8 * hh + coff);
            if (!okr) s[4 * jj + 2 * hh + e] = -INFINITY;
          }
        }
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
    uint32_t pf[kBKV / 16][4];
#pragma unroll
    for (int kk = 0; kk < kBKV / 16; ++kk) acc_to_afrag(s, kk, pf[kk]);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kBKV / 16; ++kk) wgmma_rs<D, 1>(o, pf[kk], mnmajor_step(mnmajor_desc0(sV, kBKV * 128), kk), 1);
    wgmma_commit();
    wgmma_wait<0>();
    __syncthreads();                                   // both warpgroups are done with ring stage st
    if (threadIdx.x == 0 && j + 2 < n_kv) load_kv(j + 2);
  }

  float inv[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const float l = quad_sum(l_run[hh]);
    const int row = row_t + 8 * hh;
    const bool valid_row = (row < q_len) && l > 0.f;
    inv[hh] = valid_row ? 1.f / l : 0.f;
    if (row < n_rows && (t & 3) == 0)
      lse[(static_cast<size_t>(bz) * nh + h) * S + row0 + row] = valid_row ? (m_run[hh] + log2f(l)) * kLn2 : INFINITY;
  }
  store_rows<D>(o, out, ld_o, static_cast<size_t>(bz) * S + row0, n_rows, row_t, h * D, c_in, inv);
}

// ================================================================================================ backward prep
// delta[b,h,s] = sum_d dO*O ; lse2 = lse*log2(e).
// Output layout is padded to [B, nh, S_pad] (S_pad = S rounded up to 64, pad entries = 0) so the backward kernels may read a whole
// 64-row q tile's values without a bound check.  A packed batch runs it as B = 1, S = T with S_pad >= T + 64: the backward kernels read
// a sample's last q tile up to 63 rows past the sample, i.e. the next sample's (masked) values or, after the last sample, the zero pad.
// A block owns 32 consecutive tokens of one batch entry and all heads: rows (token, head) are read 16 bytes per thread with four row
// groups in flight (contiguous: heads are adjacent in memory), the dot products are parked in shared memory as [head][token], and the
// outputs leave as 128-byte runs along the token axis.
template <int D>
__global__ void __launch_bounds__(256) attn_bwd_prep_kernel(const bf16* __restrict__ dout, const bf16* __restrict__ out,
                                                            const float* __restrict__ lse, float* __restrict__ delta,
                                                            float* __restrict__ lse2, int B, int S, int S_pad, int nh, long ld_o) {
  constexpr int GS = D / 8;          // lanes per row
  constexpr int RPP = 256 / GS;      // rows per block pass
  constexpr int U = 4;               // passes in flight
  constexpr int TOK = 32;
  extern __shared__ float sacc[];    // [nh][TOK]
  const int tiles_per_b = S_pad / TOK;
  const int b = blockIdx.x / tiles_per_b, s0 = (blockIdx.x - b * tiles_per_b) * TOK;
  const int ntok = max(0, min(TOK, S - s0));
  const int nrows = ntok * nh;
  const int sub = threadIdx.x / GS, li = threadIdx.x % GS;
  const size_t base = (static_cast<size_t>(b) * S + s0) * ld_o;
  for (int r0 = 0; r0 < nrows; r0 += RPP * U) {
    uint4 a[U], g[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int r = r0 + u * RPP + sub;
      a[u] = g[u] = make_uint4(0u, 0u, 0u, 0u);
      if (r < nrows) {
        const int tok = r / nh, h = r - tok * nh;
        const size_t off = base + static_cast<size_t>(tok) * ld_o + h * D + li * 8;
        a[u] = __ldg(reinterpret_cast<const uint4*>(out + off));
        g[u] = __ldg(reinterpret_cast<const uint4*>(dout + off));
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int r = r0 + u * RPP + sub;
      const __nv_bfloat162* pa = reinterpret_cast<const __nv_bfloat162*>(&a[u]);
      const __nv_bfloat162* pg = reinterpret_cast<const __nv_bfloat162*>(&g[u]);
      float acc = 0.f;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 x = __bfloat1622float2(pa[e]), y = __bfloat1622float2(pg[e]);
        acc += x.x * y.x + x.y * y.y;
      }
#pragma unroll
      for (int o = GS / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (li == 0 && r < nrows) {
        const int tok = r / nh, h = r - tok * nh;
        sacc[h * TOK + tok] = acc;
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nh * TOK; i += 256) {
    const int h = i / TOK, tk = i - h * TOK, sq = s0 + tk;
    const size_t idxp = (static_cast<size_t>(b) * nh + h) * S_pad + sq;
    const bool real = sq < S;
    delta[idxp] = real ? sacc[i] : 0.f;
    lse2[idxp] = real ? lse[(static_cast<size_t>(b) * nh + h) * S + sq] * kLog2e : 0.f;
  }
}

// ================================================================================================ backward: dK, dV
// CTA = one 128-row kv tile of one (b, kv head hk) (64 kv rows per warpgroup); 64-row q tiles (Q and dO) stream through the ring.
//   S^T = K Q^T, dP^T = V dO^T (both operands from shared memory), P^T = exp2(S^T * scale log2e - lse2[q]), dS^T = P^T (dP^T - delta[q]),
//   dV += P^T dO and dK += dS^T Q with P^T / dS^T as register A operands and dO / Q read MN-major.
// Under GQA the CTA walks the flattened sequence (q head hk * group + g) x (q tile i), g outer, and keeps summing into the same register
// accumulators: the group's sum has one fixed order (no atomics, no workspace), and the ring runs on across head boundaries.
template <int D>
struct BwdKVSmem {
  static constexpr int NCH = D / 64;
  static constexpr int kKV = NCH * 16384;        // K, V: [NCH][128][128B]
  static constexpr int kQT = NCH * 8192;         // Q, dO tile: [NCH][64][128B]
  static constexpr int oK = 0, oV = kKV, oQ = 2 * kKV, oDO = oQ + 2 * kQT, oBar = oDO + 2 * kQT;
  static constexpr int kBytes = oBar + 64 + 1024;
};

template <int D, bool kCausal, bool kVarlen>
__global__ void __launch_bounds__(kAttnThreads, 1)
attn_bwd_dkdv_kernel(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk,
                     const __grid_constant__ CUtensorMap tv, const __grid_constant__ CUtensorMap tdo, bf16* __restrict__ dk,
                     bf16* __restrict__ dv, long ld_dkv, const float* __restrict__ lse2, const float* __restrict__ delta,
                     const int* __restrict__ seqlens, int S, int Skv, int Sp, int nh, int group, float scale, float scale_log2) {
  using L = BwdKVSmem<D>;
  constexpr int NCH = L::NCH;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* kv_full = reinterpret_cast<uint64_t*>(smem + L::oBar);
  uint64_t* q_full = kv_full + 1;                 // [2]

  const int kv0 = blockIdx.x * 128, hk = blockIdx.y, b = blockIdx.z;
  const int row0 = kVarlen ? seqlens[b] : 0, bz = kVarlen ? 0 : b;      // packed: see attn_fwd_kernel
  const int len = kVarlen ? seqlens[b + 1] - row0 : 0;
  if (kVarlen && kv0 >= len) return;
  const int kv_len = kVarlen ? len : (seqlens ? min(seqlens[b], Skv) : Skv);
  const int q_len = kVarlen ? len : (seqlens ? kv_len : S);
  const int i0 = kCausal ? kv0 / 64 : 0;           // first q tile that can see this kv tile
  const int i1 = (kv0 < kv_len) ? (q_len + 63) / 64 : 0;
  const int n_q = max(0, i1 - i0);
  const int n_items = n_q * group;                 // item it = (q head hk * group + it / n_q, q tile i0 + it % n_q)

  if (threadIdx.x == 0) {
    mbar_init(kv_full, 1);
    mbar_init(&q_full[0], 1);
    mbar_init(&q_full[1], 1);
    fence_mbar_init();
  }
  __syncthreads();
  auto load_q = [&](int it) {
    const int st = it & 1, g = it / n_q, i = i0 + (it - g * n_q), col = (hk * group + g) * D;
    mbar_arrive_expect_tx(&q_full[st], 2 * 64 * D * 2);
    for (int c = 0; c < NCH; ++c) {
      tma_load_3d(smem + L::oQ + st * L::kQT + c * 8192, &tq, &q_full[st], col + c * 64, row0 + i * 64, bz);
      tma_load_3d(smem + L::oDO + st * L::kQT + c * 8192, &tdo, &q_full[st], col + c * 64, row0 + i * 64, bz);
    }
  };
  if (threadIdx.x == 0 && n_items > 0) {
    mbar_arrive_expect_tx(kv_full, 2 * 128 * D * 2);
    for (int c = 0; c < NCH; ++c) {
      tma_load_3d(smem + L::oK + c * 16384, &tk, kv_full, hk * D + c * 64, row0 + kv0, bz);
      tma_load_3d(smem + L::oV + c * 16384, &tv, kv_full, hk * D + c * 64, row0 + kv0, bz);
    }
    load_q(0);
    if (n_items > 1) load_q(1);
  }

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int r_in = 16 * (t >> 5) + ((t & 31) >> 2), c_in = 2 * (t & 3);
  const int row_t = kv0 + wg * 64 + r_in;          // kv row of accumulator element (h = 0); + 8 for h = 1
  const uint32_t sK = smem_u32(smem + L::oK) + wg * 8192, sV = smem_u32(smem + L::oV) + wg * 8192;
  float dka[D / 2], dva[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) dka[i] = dva[i] = 0.f;
  if (n_items > 0) mbar_wait(kv_full, 0, 3);
  for (int it = 0; it < n_items; ++it) {
    const int st = it & 1, g = it / n_q, i = i0 + (it - g * n_q);
    const float* lse_bh = lse2 + (static_cast<size_t>(bz) * nh + hk * group + g) * Sp + row0;
    const float* del_bh = delta + (static_cast<size_t>(bz) * nh + hk * group + g) * Sp + row0;
    mbar_wait(&q_full[st], (it >> 1) & 1, 4);
    const uint32_t sQ = smem_u32(smem + L::oQ + st * L::kQT), sDO = smem_u32(smem + L::oDO + st * L::kQT);
    float sa[32], dpa[32];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < D / 16; ++ks) wgmma_ss<64, 0, 0>(sa, kmajor_step(kmajor_desc0(sK), 16384, ks), kmajor_step(kmajor_desc0(sQ), 8192, ks), ks > 0);
#pragma unroll
    for (int ks = 0; ks < D / 16; ++ks) wgmma_ss<64, 0, 0>(dpa, kmajor_step(kmajor_desc0(sV), 16384, ks), kmajor_step(kmajor_desc0(sDO), 8192, ks), ks > 0);
    wgmma_commit();
    wgmma_wait<0>();
    const int q0 = i * 64;
    const bool need_mask = (kCausal && q0 < kv0 + 127) || (q0 + 64 > q_len) || (kv0 + 128 > kv_len);
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int q = q0 + 8 * jj + c_in + e;
        const float l2 = lse_bh[q], dl = del_bh[q];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int kv = row_t + 8 * hh;
          const int x = 4 * jj + 2 * hh + e;
          const bool ok = !need_mask || (q < q_len && kv < kv_len && (!kCausal || kv <= q));
          const float p = ok ? exp2f(sa[x] * scale_log2 - l2) : 0.f;
          sa[x] = p;
          dpa[x] = p * (dpa[x] - dl);
        }
      }
    uint32_t pf[4][4], df[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) { acc_to_afrag(sa, kk, pf[kk]); acc_to_afrag(dpa, kk, df[kk]); }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_rs<D, 1>(dva, pf[kk], mnmajor_step(mnmajor_desc0(sDO, 8192), kk), 1);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_rs<D, 1>(dka, df[kk], mnmajor_step(mnmajor_desc0(sQ, 8192), kk), 1);
    wgmma_commit();
    wgmma_wait<0>();
    __syncthreads();                                   // both warpgroups are done with ring stage st
    if (threadIdx.x == 0 && it + 2 < n_items) load_q(it + 2);
  }
  const float ms[2] = {scale, scale}, one[2] = {1.f, 1.f};
  const size_t base = static_cast<size_t>(bz) * Skv + row0;
  store_rows<D>(dka, dk, ld_dkv, base, kVarlen ? len : Skv, row_t, hk * D, c_in, ms);
  store_rows<D>(dva, dv, ld_dkv, base, kVarlen ? len : Skv, row_t, hk * D, c_in, one);
}

// ================================================================================================ backward: dQ
// CTA = one 128-row q tile of one (b, h) (64 q rows per warpgroup); 64-row kv tiles (K and V) stream through the ring.
//   S = Q K^T, dP = dO V^T, P = exp2(S * scale log2e - lse2[q]), dS = P (dP - delta[q]), dQ += dS K (dS from registers, K read MN-major).
template <int D>
struct BwdQSmem {
  static constexpr int NCH = D / 64;
  static constexpr int kQ = NCH * 16384;         // Q, dO: [NCH][128][128B]
  static constexpr int kKT = NCH * 8192;         // K, V tile: [NCH][64][128B]
  static constexpr int oQ = 0, oDO = kQ, oK = 2 * kQ, oV = oK + 2 * kKT, oBar = oV + 2 * kKT;
  static constexpr int kBytes = oBar + 64 + 1024;
};

template <int D, bool kCausal, bool kVarlen>
__global__ void __launch_bounds__(kAttnThreads, 1)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk,
                   const __grid_constant__ CUtensorMap tv, const __grid_constant__ CUtensorMap tdo, bf16* __restrict__ dq,
                   long ld_dq, const float* __restrict__ lse2, const float* __restrict__ delta, const int* __restrict__ seqlens,
                   int S, int Skv, int Sp, int nh, int group, float scale, float scale_log2) {
  using L = BwdQSmem<D>;
  constexpr int NCH = L::NCH;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* q_full = reinterpret_cast<uint64_t*>(smem + L::oBar);
  uint64_t* kv_full = q_full + 1;                 // [2]

  const int h = blockIdx.y, b = blockIdx.z;
  const int row0 = kVarlen ? seqlens[b] : 0, bz = kVarlen ? 0 : b;      // packed: see attn_fwd_kernel
  const int len = kVarlen ? seqlens[b + 1] - row0 : 0;
  const int n_qt = kVarlen ? (len + 127) / 128 : gridDim.x;
  if (kVarlen && static_cast<int>(blockIdx.x) >= n_qt) return;
  const int q0 = (kCausal ? (n_qt - 1 - blockIdx.x) : blockIdx.x) * 128;
  const int hkv = h / group;
  const int kv_len = kVarlen ? len : (seqlens ? min(seqlens[b], Skv) : Skv);
  const int q_len = kVarlen ? len : (seqlens ? kv_len : S);
  const int kv_end = (q0 < q_len) ? (kCausal ? min(kv_len, q0 + 128) : kv_len) : 0;
  const int n_kv = kv_end > 0 ? (kv_end + 63) / 64 : 0;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    mbar_init(&kv_full[0], 1);
    mbar_init(&kv_full[1], 1);
    fence_mbar_init();
  }
  __syncthreads();
  auto load_kv = [&](int j) {
    const int st = j & 1;
    mbar_arrive_expect_tx(&kv_full[st], 2 * 64 * D * 2);
    for (int c = 0; c < NCH; ++c) {
      tma_load_3d(smem + L::oK + st * L::kKT + c * 8192, &tk, &kv_full[st], hkv * D + c * 64, row0 + j * 64, bz);
      tma_load_3d(smem + L::oV + st * L::kKT + c * 8192, &tv, &kv_full[st], hkv * D + c * 64, row0 + j * 64, bz);
    }
  };
  if (threadIdx.x == 0 && n_kv > 0) {
    mbar_arrive_expect_tx(q_full, 2 * 128 * D * 2);
    for (int c = 0; c < NCH; ++c) {
      tma_load_3d(smem + L::oQ + c * 16384, &tq, q_full, h * D + c * 64, row0 + q0, bz);
      tma_load_3d(smem + L::oDO + c * 16384, &tdo, q_full, h * D + c * 64, row0 + q0, bz);
    }
    load_kv(0);
    if (n_kv > 1) load_kv(1);
  }

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int r_in = 16 * (t >> 5) + ((t & 31) >> 2), c_in = 2 * (t & 3);
  const int row_t = q0 + wg * 64 + r_in;
  const uint32_t sQ = smem_u32(smem + L::oQ) + wg * 8192, sDO = smem_u32(smem + L::oDO) + wg * 8192;
  const float* lse_bh = lse2 + (static_cast<size_t>(bz) * nh + h) * Sp;
  const float* del_bh = delta + (static_cast<size_t>(bz) * nh + h) * Sp;
  float l2[2], dl[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int row = min(row0 + row_t + 8 * hh, Sp - 1);
    l2[hh] = lse_bh[row];
    dl[hh] = del_bh[row];
  }
  float dqa[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) dqa[i] = 0.f;
  if (n_kv > 0) mbar_wait(q_full, 0, 5);
  for (int j = 0; j < n_kv; ++j) {
    const int st = j & 1;
    mbar_wait(&kv_full[st], (j >> 1) & 1, 6);
    const uint32_t sK = smem_u32(smem + L::oK + st * L::kKT), sV = smem_u32(smem + L::oV + st * L::kKT);
    float sa[32], dpa[32];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < D / 16; ++ks) wgmma_ss<64, 0, 0>(sa, kmajor_step(kmajor_desc0(sQ), 16384, ks), kmajor_step(kmajor_desc0(sK), 8192, ks), ks > 0);
#pragma unroll
    for (int ks = 0; ks < D / 16; ++ks) wgmma_ss<64, 0, 0>(dpa, kmajor_step(kmajor_desc0(sDO), 16384, ks), kmajor_step(kmajor_desc0(sV), 8192, ks), ks > 0);
    wgmma_commit();
    wgmma_wait<0>();
    const int kv0 = j * 64;
    const bool need_mask = (kCausal && kv0 + 63 > q0) || (kv0 + 64 > kv_len) || (q0 + 128 > q_len);
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int kv = kv0 + 8 * jj + c_in + e;
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int q = row_t + 8 * hh;
          const int x = 4 * jj + 2 * hh + e;
          const bool ok = !need_mask || (q < q_len && kv < kv_len && (!kCausal || kv <= q));
          const float p = ok ? exp2f(sa[x] * scale_log2 - l2[hh]) : 0.f;
          dpa[x] = p * (dpa[x] - dl[hh]);
        }
      }
    uint32_t df[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) acc_to_afrag(dpa, kk, df[kk]);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_rs<D, 1>(dqa, df[kk], mnmajor_step(mnmajor_desc0(sK, 8192), kk), 1);
    wgmma_commit();
    wgmma_wait<0>();
    __syncthreads();                                   // both warpgroups are done with ring stage st
    if (threadIdx.x == 0 && j + 2 < n_kv) load_kv(j + 2);
  }
  const float ms[2] = {scale, scale};
  store_rows<D>(dqa, dq, ld_dq, static_cast<size_t>(bz) * S + row0, kVarlen ? len : S, row_t, h * D, c_in, ms);
}

// ================================================================================================ attention probabilities
// P = softmax(Q K^T * scale + mask) as a dense bf16 [B, nh, S, Skv] (the eager path's attention weights, reference :357-378), from the
// forward's lse: one QK^T pass, P = exp2(S * scale log2e - lse log2e), no V and no PV product.  CTA = 128 query rows of one (head, batch),
// the forward's grid and layout (two warpgroups of 64 rows, K tiles through a two-stage TMA ring).  Row semantics, as the reference's:
//   * rows with a finite lse: the forward's own statistics;
//   * right-padded rows (row >= seqlens[b]): the reference masks keys only, so they are a softmax over keys < len.  The forward stores
//     lse = +inf there, so a CTA holding such rows first runs a statistics pass over K (the forward's online max / sum);
//   * rows with no visible key (a left-padded prompt position, a length-0 sample): the reference clamps every score to finfo.min, so
//     the row is uniform, bf16(1 / Skv) in every column.
// Every element of the output is written exactly once: tiles past the last one with a visible key get no MMA and are written as
// zeros (or the uniform value).  P tiles are staged in shared memory with each row shifted by its global misalignment, so the rows of
// an arbitrary width Skv leave as 16-byte stores except for the partial chunk at either end.
template <int D>
struct ProbsSmem {
  static constexpr int NCH = D / 64;
  static constexpr int kQ = NCH * 16384;         // [NCH][128][128B]
  static constexpr int kK = NCH * kBKV * 128;    // [NCH][kBKV][128B]
  static constexpr int kPitch = kBKV + 16;       // staging row (elements): 128 columns + up to 7 of shift, 16-byte multiple
  static constexpr int oQ = 0, oK = kQ, oP = oK + 2 * kK, oBar = oP + 128 * kPitch * 2;
  static constexpr int kBytes = oBar + 64 + 1024;
};

template <int D, bool kCausal>
__global__ void __launch_bounds__(kAttnThreads, 1)
attn_probs_kernel(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk, const float* __restrict__ lse,
                  bf16* __restrict__ probs, const int* __restrict__ seqlens, int S, int Skv, int nh, int group, float scale_log2,
                  const uint8_t* __restrict__ kv_mask, int mask_ld) {
  using L = ProbsSmem<D>;
  constexpr int NCH = L::NCH;
  constexpr int NJ = kBKV / 8;
  constexpr int P = L::kPitch;
  const int coff = kCausal ? (Skv - S) : 0;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* q_full = reinterpret_cast<uint64_t*>(smem + L::oBar);
  uint64_t* k_full = q_full + 1;                  // [2]
  bf16* stage = reinterpret_cast<bf16*>(smem + L::oP);

  const int q0 = (kCausal ? (gridDim.x - 1 - blockIdx.x) : blockIdx.x) * 128, h = blockIdx.y, b = blockIdx.z;
  const int hkv = h / group;
  const int kv_len = seqlens ? min(seqlens[b], Skv) : Skv;
  const int q_len = seqlens ? kv_len : S;
  const int kv_end = kCausal ? min(kv_len, q0 + 128 + coff) : kv_len;
  const int n_kv = kv_end > 0 ? (kv_end + kBKV - 1) / kBKV : 0;   // tiles with a visible key for some row of the CTA
  const int n_tiles = (Skv + kBKV - 1) / kBKV;
  const bool stats_pass = min(S, q0 + 128) > q_len;             // the tile holds right-padded rows
  const int n_items = (stats_pass ? 2 : 1) * n_kv;               // K tiles through the ring: [statistics pass,] write pass

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    mbar_init(&k_full[0], 1);
    mbar_init(&k_full[1], 1);
    fence_mbar_init();
  }
  __syncthreads();
  auto load_k = [&](int it) {
    const int st = it & 1, j = it % n_kv;
    mbar_arrive_expect_tx(&k_full[st], kBKV * D * 2);
    for (int c = 0; c < NCH; ++c)
      tma_load_3d(smem + L::oK + st * L::kK + c * kBKV * 128, &tk, &k_full[st], hkv * D + c * 64, j * kBKV, b);
  };
  if (threadIdx.x == 0 && n_items > 0) {
    mbar_arrive_expect_tx(q_full, 128 * D * 2);
    for (int c = 0; c < NCH; ++c) tma_load_3d(smem + L::oQ + c * 16384, &tq, q_full, h * D + c * 64, q0, b);
    load_k(0);
    if (n_items > 1) load_k(1);
  }

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int r_in = 16 * (t >> 5) + ((t & 31) >> 2), c_in = 2 * (t & 3);
  const int row_t = q0 + wg * 64 + r_in;          // + 8h
  const uint32_t sQ = smem_u32(smem + L::oQ) + wg * 8192;

  // S = Q K^T of ring item `it` into s, then release its ring stage
  auto qk = [&](int it, float* s) {
    const int st = it & 1;
    mbar_wait(&k_full[st], (it >> 1) & 1, 7);
    const uint32_t sK = smem_u32(smem + L::oK + st * L::kK);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < D / 16; ++ks) wgmma_ss<kBKV, 0, 0>(s, kmajor_step(kmajor_desc0(sQ), 16384, ks), kmajor_step(kmajor_desc0(sK), kBKV * 128, ks), ks > 0);
    wgmma_commit();
    wgmma_wait<0>();
    __syncthreads();                                   // both warpgroups are done with ring stage st
    if (threadIdx.x == 0 && it + 2 < n_items) load_k(it + 2);
  };
  // the forward's mask: -inf where the key is past kv_len, padded in kv_mask or (causal) after the query
  auto mask_tile = [&](float* s, int kv0) {
    if (!((kCausal && kv0 + kBKV - 1 > q0 + coff) || (kv0 + kBKV > kv_len) || (kv_mask != nullptr))) return;
#pragma unroll
    for (int jj = 0; jj < NJ; ++jj)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int kvi = kv0 + 8 * jj + c_in + e;
        bool ok = kvi < kv_len;
        if (ok && kv_mask != nullptr) ok = kv_mask[static_cast<size_t>(b) * mask_ld + kvi] != 0;
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
          if (!(ok && (!kCausal || kvi <= row_t + 8 * hh + coff))) s[4 * jj + 2 * hh + e] = -INFINITY;
      }
  };

  // per row: lse in log2 units, or uniform (no visible key)
  const float* lse_bh = lse + (static_cast<size_t>(b) * nh + h) * S;
  float l2[2];
  bool uni[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int row = row_t + 8 * hh;
    const float v = row < min(S, q_len) ? lse_bh[row] : INFINITY;
    uni[hh] = v == INFINITY;
    l2[hh] = v * kLog2e;
  }
  if (n_items > 0) mbar_wait(q_full, 0, 8);
  int it = 0;
  if (stats_pass) {
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    for (int j = 0; j < n_kv; ++j, ++it) {
      float s[kBKV / 2];
      qk(it, s);
      mask_tile(s, j * kBKV);
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        float mx = -INFINITY;
#pragma unroll
        for (int jj = 0; jj < NJ; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * hh], s[4 * jj + 2 * hh + 1]));
        mx = quad_max(mx);
        const float m_new = fmaxf(m_run[hh], mx * scale_log2);
        const float alpha = (m_run[hh] == -INFINITY) ? 0.f : exp2f(m_run[hh] - m_new);
        m_run[hh] = m_new;
        const float m_use = (m_new == -INFINITY) ? 0.f : m_new;
        float ls = 0.f;
#pragma unroll
        for (int jj = 0; jj < NJ; ++jj)
#pragma unroll
          for (int e = 0; e < 2; ++e) ls += exp2f(s[4 * jj + 2 * hh + e] * scale_log2 - m_use);
        l_run[hh] = l_run[hh] * alpha + ls;
      }
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const float l = quad_sum(l_run[hh]);
      if (row_t + 8 * hh >= q_len) {
        uni[hh] = !(l > 0.f);
        l2[hh] = m_run[hh] + log2f(l);
      }
    }
  }

  const float uval = __frcp_rn(static_cast<float>(Skv));   // the reference's fp32 softmax over Skv equal scores
  const size_t plane = (static_cast<size_t>(b) * nh + h) * S;
  for (int j = 0; j < n_tiles; ++j) {
    const int kv0 = j * kBKV;
    float s[kBKV / 2];
    if (j < n_kv) {
      qk(it++, s);
      mask_tile(s, kv0);
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int jj = 0; jj < NJ; ++jj)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float& x = s[4 * jj + 2 * hh + e];
            x = uni[hh] ? uval : exp2f(x * scale_log2 - l2[hh]);
          }
    } else {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int jj = 0; jj < NJ; ++jj) s[4 * jj + 2 * hh] = s[4 * jj + 2 * hh + 1] = uni[hh] ? uval : 0.f;
    }
    // registers -> staging rows, each shifted by m = (its global element index) % 8 so that 16-byte global chunks are 16-byte aligned here
    named_bar_sync(1 + wg, 128);                       // this warpgroup's previous tile has left the staging rows
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int R = wg * 64 + r_in + 8 * hh;
      const int m = static_cast<int>(((plane + q0 + R) * Skv + kv0) & 7);
      bf16* srow = stage + R * P + m;
#pragma unroll
      for (int jj = 0; jj < NJ; ++jj) {
        const float a = s[4 * jj + 2 * hh], c = s[4 * jj + 2 * hh + 1];
        if ((m & 1) == 0) {
          *reinterpret_cast<uint32_t*>(srow + 8 * jj + c_in) = pack_bf16(a, c);
        } else {
          srow[8 * jj + c_in] = __float2bfloat16_rn(a);
          srow[8 * jj + c_in + 1] = __float2bfloat16_rn(c);
        }
      }
    }
    named_bar_sync(1 + wg, 128);
    // staging -> global: a half-warp per row, lane k of it owns 16-byte chunks k and k + 16 of the row's span
    const int n = min(kBKV, Skv - kv0), lane16 = t & 15;
    for (int rr = t >> 4; rr < 64; rr += 8) {
      const int R = wg * 64 + rr;
      if (q0 + R >= S) break;
      const size_t e0 = (plane + q0 + R) * Skv + kv0;
      const int m = static_cast<int>(e0 & 7);
      bf16* g = probs + (e0 - m);
      const bf16* srow = stage + R * P;
      const int nch = (m + n + 7) >> 3;
      for (int k = lane16; k < nch; k += 16) {
        const int lo = 8 * k;
        if (lo >= m && lo + 8 <= m + n) {
          *reinterpret_cast<uint4*>(g + lo) = *reinterpret_cast<const uint4*>(srow + lo);
        } else {
          for (int c = max(lo, m); c < min(lo + 8, m + n); ++c) g[c] = srow[c];
        }
      }
    }
  }
}

// ================================================================================================ host
template <typename K>
static int set_smem(K kern, int bytes) {
  return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// grid_rows: rows the grid's tile axis covers (S; packed: the longest sample, with S = Skv = T and seqlens = cu_seqlens)
template <int D, bool C, bool V = false>
static int launch_fwd(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, void* out, long ld_o, float* lse,
                      const int* seqlens, int B, int S, int Skv, int nh, int group, float scale_log2, cudaStream_t st,
                      const uint8_t* kv_mask, int mask_ld, int grid_rows) {
  auto kern = attn_fwd_kernel<D, C, V>;
  static bool once = false;
  if (!once) {
    if (set_smem(kern, FwdSmem<D>::kBytes)) return DLLM_ERR_LAUNCH;
    once = true;
  }
  dim3 grid((grid_rows + 127) / 128, nh, B);
  kern<<<grid, kAttnThreads, FwdSmem<D>::kBytes, st>>>(tq, tk, tv, static_cast<bf16*>(out), ld_o, lse, seqlens, S, Skv, nh, group,
                                                       scale_log2, kv_mask, mask_ld);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

int attn_fwd(const void* q, const void* k, const void* v, void* out, float* lse, const int* seqlens, int B, int S, int nh,
             int d, long ld_qkv, long ld_o, int causal, float scale, cudaStream_t st) {
  return attn_fwd_gqa(q, k, v, out, lse, seqlens, nullptr, 0, B, S, S, S, nh, nh, d, ld_qkv, ld_qkv, ld_o, causal, scale, st);
}

// q: [B, S, nh, d] (token stride ld_q); k, v: [B, Skv, nh, d] (token stride ld_kv).  Skv != S = cross-attention.
int attn_fwd_ex(const void* q, const void* k, const void* v, void* out, float* lse, const int* seqlens, int B, int S, int Skv,
                int nh, int d, long ld_q, long ld_kv, long ld_o, int causal, float scale, cudaStream_t st) {
  return attn_fwd_gqa(q, k, v, out, lse, seqlens, nullptr, 0, B, S, Skv, Skv, nh, nh, d, ld_q, ld_kv, ld_o, causal, scale, st);
}

// kv_rows = rows allocated per batch entry in the k/v buffers (>= Skv): lets a preallocated kv-cache [B, max_len, nh*d] be read in
// place with Skv valid rows.  causal with Skv > S uses the bottom-right aligned mask (decode / continuation).
int attn_fwd_cache(const void* q, const void* k, const void* v, void* out, float* lse, const int* seqlens, int B, int S, int Skv,
                   int kv_rows, int nh, int d, long ld_q, long ld_kv, long ld_o, int causal, float scale, cudaStream_t st) {
  return attn_fwd_gqa(q, k, v, out, lse, seqlens, nullptr, 0, B, S, Skv, kv_rows, nh, nh, d, ld_q, ld_kv, ld_o, causal, scale, st);
}

// + kv_mask [B, mask_ld] bytes (0 = padded key): a padded prompt batch inside the kv-cache.  mask_ld must cover whole 64-key tiles
// (mask_ld % 16 == 0, mask_ld >= round_up(Skv, 64)).
int attn_fwd_cache_mask(const void* q, const void* k, const void* v, void* out, float* lse, const int* seqlens, const void* kv_mask,
                        int mask_ld, int B, int S, int Skv, int kv_rows, int nh, int d, long ld_q, long ld_kv, long ld_o, int causal,
                        float scale, cudaStream_t st) {
  return attn_fwd_gqa(q, k, v, out, lse, seqlens, kv_mask, mask_ld, B, S, Skv, kv_rows, nh, nh, d, ld_q, ld_kv, ld_o, causal, scale, st);
}

// The one forward entry every variant above funnels into.  k, v: [B, kv_rows, nkv, d] with nkv dividing nh (grouped-query attention;
// nkv == nh is multi-head attention).
int attn_fwd_gqa(const void* q, const void* k, const void* v, void* out, float* lse, const int* seqlens, const void* kv_mask,
                 int mask_ld, int B, int S, int Skv, int kv_rows, int nh, int nkv, int d, long ld_q, long ld_kv, long ld_o, int causal,
                 float scale, cudaStream_t st) {
  if (B <= 0 || S <= 0 || Skv <= 0 || nh <= 0 || kv_rows < Skv) return DLLM_ERR_SHAPE;
  if (nkv <= 0 || nh % nkv != 0) return DLLM_ERR_SHAPE;
  if (kv_mask && ((mask_ld & 15) || mask_ld < (Skv + 63) / 64 * 64 || (reinterpret_cast<uintptr_t>(kv_mask) & 15))) return DLLM_ERR_ALIGN;
  const uint8_t* km = static_cast<const uint8_t*>(kv_mask);
  if (d != 128 && d != 64) return DLLM_ERR_UNSUPPORTED;
  if (S != Skv && seqlens) return DLLM_ERR_UNSUPPORTED;
  if (causal && Skv < S) return DLLM_ERR_SHAPE;
  if ((reinterpret_cast<uintptr_t>(out) & 15) || (ld_o & 7)) return DLLM_ERR_ALIGN;
  CUtensorMap tq, tk, tv;
  int rc;
  if ((rc = make_tmap_bsc(&tq, q, B, S, nh * d, ld_q, 128))) return rc;
  if ((rc = make_tmap_bsc(&tk, k, B, kv_rows, nkv * d, ld_kv, kBKV))) return rc;
  if ((rc = make_tmap_bsc(&tv, v, B, kv_rows, nkv * d, ld_kv, kBKV))) return rc;
  const float sl2 = scale * kLog2e;
  const int g = nh / nkv;
  if (d == 128) return causal ? launch_fwd<128, true>(tq, tk, tv, out, ld_o, lse, seqlens, B, S, Skv, nh, g, sl2, st, km, mask_ld, S)
                              : launch_fwd<128, false>(tq, tk, tv, out, ld_o, lse, seqlens, B, S, Skv, nh, g, sl2, st, km, mask_ld, S);
  return causal ? launch_fwd<64, true>(tq, tk, tv, out, ld_o, lse, seqlens, B, S, Skv, nh, g, sl2, st, km, mask_ld, S)
                : launch_fwd<64, false>(tq, tk, tv, out, ld_o, lse, seqlens, B, S, Skv, nh, g, sl2, st, km, mask_ld, S);
}

// Packed batch: q [T, nh, d], k / v [T, nkv, d], out [T, nh * d], lse [nh, T]; cu_seqlens int32 [B + 1] on the device, non-decreasing
// with cu[0] = 0 and cu[B] = T (trusted, as is max_seqlen >= every length: the Python layer checks them on the host).  Self-attention
// inside each sample; sample b's rows equal attn_fwd_gqa on that sample alone, bit for bit.
int attn_fwd_varlen(const void* q, const void* k, const void* v, void* out, float* lse, const int* cu_seqlens, int B, int T,
                    int max_seqlen, int nh, int nkv, int d, long ld_q, long ld_kv, long ld_o, int causal, float scale, cudaStream_t st) {
  if (B <= 0 || T <= 0 || nh <= 0 || max_seqlen <= 0 || max_seqlen > T || !cu_seqlens) return DLLM_ERR_SHAPE;
  if (nkv <= 0 || nh % nkv != 0) return DLLM_ERR_SHAPE;
  if (d != 128 && d != 64) return DLLM_ERR_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(out) & 15) || (ld_o & 7)) return DLLM_ERR_ALIGN;
  CUtensorMap tq, tk, tv;
  int rc;
  if ((rc = make_tmap_bsc(&tq, q, 1, T, nh * d, ld_q, 128))) return rc;
  if ((rc = make_tmap_bsc(&tk, k, 1, T, nkv * d, ld_kv, kBKV))) return rc;
  if ((rc = make_tmap_bsc(&tv, v, 1, T, nkv * d, ld_kv, kBKV))) return rc;
  const float sl2 = scale * kLog2e;
  const int g = nh / nkv;
#define DLLM_FWDV(DD, CC) \
  return launch_fwd<DD, CC, true>(tq, tk, tv, out, ld_o, lse, cu_seqlens, B, T, T, nh, g, sl2, st, nullptr, 0, max_seqlen)
  if (d == 128) { if (causal) DLLM_FWDV(128, true); else DLLM_FWDV(128, false); }
  if (causal) DLLM_FWDV(64, true); else DLLM_FWDV(64, false);
#undef DLLM_FWDV
}

template <int D, bool C>
static int launch_probs(const CUtensorMap& tq, const CUtensorMap& tk, const float* lse, void* probs, const int* seqlens, int B, int S,
                        int Skv, int nh, int group, float scale_log2, cudaStream_t st, const uint8_t* kv_mask, int mask_ld) {
  auto kern = attn_probs_kernel<D, C>;
  static bool once = false;
  if (!once) {
    if (set_smem(kern, ProbsSmem<D>::kBytes)) return DLLM_ERR_LAUNCH;
    once = true;
  }
  dim3 grid((S + 127) / 128, nh, B);
  kern<<<grid, kAttnThreads, ProbsSmem<D>::kBytes, st>>>(tq, tk, lse, static_cast<bf16*>(probs), seqlens, S, Skv, nh, group, scale_log2,
                                                         kv_mask, mask_ld);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// Attention probabilities [B, nh, S, Skv] bf16 (dense, row-major) of the attention attn_fwd_gqa computed with the same q, k, masks and
// shapes; `lse` is that call's output.
int attn_probs_gqa(const void* q, const void* k, const float* lse, void* probs, const int* seqlens, const void* kv_mask, int mask_ld,
                   int B, int S, int Skv, int kv_rows, int nh, int nkv, int d, long ld_q, long ld_kv, int causal, float scale,
                   cudaStream_t st) {
  if (B <= 0 || S <= 0 || Skv <= 0 || nh <= 0 || kv_rows < Skv) return DLLM_ERR_SHAPE;
  if (nkv <= 0 || nh % nkv != 0) return DLLM_ERR_SHAPE;
  if (kv_mask && ((mask_ld & 15) || mask_ld < (Skv + 63) / 64 * 64 || (reinterpret_cast<uintptr_t>(kv_mask) & 15))) return DLLM_ERR_ALIGN;
  const uint8_t* km = static_cast<const uint8_t*>(kv_mask);
  if (d != 128 && d != 64) return DLLM_ERR_UNSUPPORTED;
  if (S != Skv && seqlens) return DLLM_ERR_UNSUPPORTED;
  if (causal && Skv < S) return DLLM_ERR_SHAPE;
  if (reinterpret_cast<uintptr_t>(probs) & 15) return DLLM_ERR_ALIGN;
  CUtensorMap tq, tk;
  int rc;
  if ((rc = make_tmap_bsc(&tq, q, B, S, nh * d, ld_q, 128))) return rc;
  if ((rc = make_tmap_bsc(&tk, k, B, kv_rows, nkv * d, ld_kv, kBKV))) return rc;
  const float sl2 = scale * kLog2e;
  const int g = nh / nkv;
  if (d == 128) return causal ? launch_probs<128, true>(tq, tk, lse, probs, seqlens, B, S, Skv, nh, g, sl2, st, km, mask_ld)
                              : launch_probs<128, false>(tq, tk, lse, probs, seqlens, B, S, Skv, nh, g, sl2, st, km, mask_ld);
  return causal ? launch_probs<64, true>(tq, tk, lse, probs, seqlens, B, S, Skv, nh, g, sl2, st, km, mask_ld)
                : launch_probs<64, false>(tq, tk, lse, probs, seqlens, B, S, Skv, nh, g, sl2, st, km, mask_ld);
}

static inline int s_pad(int S) { return (S + 63) / 64 * 64; }
size_t attn_bwd_workspace(int B, int S, int nh, int) { return static_cast<size_t>(B) * s_pad(S) * nh * 2 * sizeof(float); }

// packed: one [nh, T_pad] plane each for delta and lse2, T_pad = T rounded up to 64 plus one 64-row tile of zeros (see the prep kernel)
static inline int t_pad(int T) { return s_pad(T) + 64; }
size_t attn_bwd_varlen_workspace(int T, int nh, int) { return static_cast<size_t>(t_pad(T)) * nh * 2 * sizeof(float); }

// packed (V): S = Skv = T, seqlens = cu_seqlens and max_seqlen sizes the tile axis of both grids; Sp = row pitch of delta / lse2
template <int D, bool C, bool V = false>
static int launch_bwd(const CUtensorMap& tq64, const CUtensorMap& tq128, const CUtensorMap& tk64, const CUtensorMap& tk128,
                      const CUtensorMap& tv64, const CUtensorMap& tv128, const CUtensorMap& tdo64, const CUtensorMap& tdo128,
                      const bf16* dout, const bf16* out, const float* lse, float* delta, float* lse2, const int* seqlens, bf16* dq,
                      bf16* dk, bf16* dv, long ld_dq, long ld_dkv, int B, int S, int Skv, int nh, int nkv, long ld_o,
                      float scale, cudaStream_t st, int max_seqlen, int Sp) {
  auto k1 = attn_bwd_dkdv_kernel<D, C, V>;
  auto k2 = attn_bwd_dq_kernel<D, C, V>;
  static bool once = false;
  if (!once) {
    if (set_smem(k1, BwdKVSmem<D>::kBytes) || set_smem(k2, BwdQSmem<D>::kBytes)) return DLLM_ERR_LAUNCH;
    once = true;
  }
  if (nh > 384) return DLLM_ERR_SHAPE;   // prep kernel parks nh x 32 floats in (default-limit) shared memory
  attn_bwd_prep_kernel<D><<<static_cast<unsigned>(static_cast<long>(V ? 1 : B) * (Sp / 32)), 256, static_cast<size_t>(nh) * 32 * sizeof(float), st>>>(
      dout, out, lse, delta, lse2, V ? 1 : B, S, Sp, nh, ld_o);
  const int group = nh / nkv;
  dim3 grid_kv(((V ? max_seqlen : Skv) + 127) / 128, nkv, B), grid_q(((V ? max_seqlen : S) + 127) / 128, nh, B);
  k1<<<grid_kv, kAttnThreads, BwdKVSmem<D>::kBytes, st>>>(tq64, tk128, tv128, tdo64, dk, dv, ld_dkv, lse2, delta, seqlens, S, Skv, Sp,
                                                           nh, group, scale, scale * kLog2e);
  k2<<<grid_q, kAttnThreads, BwdQSmem<D>::kBytes, st>>>(tq128, tk64, tv64, tdo128, dq, ld_dq, lse2, delta, seqlens, S, Skv, Sp, nh, group,
                                                        scale, scale * kLog2e);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

int attn_bwd(const void* dout, const void* q, const void* k, const void* v, const void* out, const float* lse, void* dq,
             void* dk, void* dv, const int* seqlens, void* workspace, size_t workspace_bytes, int B, int S, int nh, int d,
             long ld_qkv, long ld_o, long ld_dqkv, int causal, float scale, cudaStream_t st) {
  return attn_bwd_ex(dout, q, k, v, out, lse, dq, dk, dv, seqlens, workspace, workspace_bytes, B, S, S, nh, d, ld_qkv, ld_qkv, ld_o,
                     ld_dqkv, ld_dqkv, causal, scale, st);
}

int attn_bwd_ex(const void* dout, const void* q, const void* k, const void* v, const void* out, const float* lse, void* dq,
                void* dk, void* dv, const int* seqlens, void* workspace, size_t workspace_bytes, int B, int S, int Skv, int nh,
                int d, long ld_q, long ld_kv, long ld_o, long ld_dq, long ld_dkv, int causal, float scale, cudaStream_t st) {
  return attn_bwd_gqa(dout, q, k, v, out, lse, dq, dk, dv, seqlens, workspace, workspace_bytes, B, S, Skv, nh, nh, d, ld_q, ld_kv, ld_o,
                      ld_dq, ld_dkv, causal, scale, st);
}

// k, v, dk, dv: [B, Skv, nkv, d], nkv dividing nh.  dK / dV of kv head hk sum the group's q heads hk * group .. hk * group + group - 1.
int attn_bwd_gqa(const void* dout, const void* q, const void* k, const void* v, const void* out, const float* lse, void* dq,
                 void* dk, void* dv, const int* seqlens, void* workspace, size_t workspace_bytes, int B, int S, int Skv, int nh,
                 int nkv, int d, long ld_q, long ld_kv, long ld_o, long ld_dq, long ld_dkv, int causal, float scale, cudaStream_t st) {
  if (B <= 0 || S <= 0 || Skv <= 0 || nh <= 0) return DLLM_ERR_SHAPE;
  if (nkv <= 0 || nh % nkv != 0) return DLLM_ERR_SHAPE;
  if (d != 128 && d != 64) return DLLM_ERR_UNSUPPORTED;
  if (S != Skv && (causal || seqlens)) return DLLM_ERR_UNSUPPORTED;
  if (workspace_bytes < attn_bwd_workspace(B, S, nh, d)) return DLLM_ERR_SHAPE;
  if ((reinterpret_cast<uintptr_t>(dq) & 15) || (reinterpret_cast<uintptr_t>(dk) & 15) || (reinterpret_cast<uintptr_t>(dv) & 15) ||
      (reinterpret_cast<uintptr_t>(out) & 15) || (reinterpret_cast<uintptr_t>(dout) & 15) || (ld_dq & 7) || (ld_dkv & 7) || (ld_o & 7))
    return DLLM_ERR_ALIGN;
  float* delta = static_cast<float*>(workspace);
  float* lse2 = delta + static_cast<size_t>(B) * s_pad(S) * nh;
  CUtensorMap tq64, tq128, tk64, tk128, tv64, tv128, tdo64, tdo128;
  int rc;
  const int C = nh * d, Ckv = nkv * d;
  if ((rc = make_tmap_bsc(&tq64, q, B, S, C, ld_q, 64))) return rc;
  if ((rc = make_tmap_bsc(&tq128, q, B, S, C, ld_q, 128))) return rc;
  if ((rc = make_tmap_bsc(&tk64, k, B, Skv, Ckv, ld_kv, 64))) return rc;
  if ((rc = make_tmap_bsc(&tk128, k, B, Skv, Ckv, ld_kv, 128))) return rc;
  if ((rc = make_tmap_bsc(&tv64, v, B, Skv, Ckv, ld_kv, 64))) return rc;
  if ((rc = make_tmap_bsc(&tv128, v, B, Skv, Ckv, ld_kv, 128))) return rc;
  if ((rc = make_tmap_bsc(&tdo64, dout, B, S, C, ld_o, 64))) return rc;
  if ((rc = make_tmap_bsc(&tdo128, dout, B, S, C, ld_o, 128))) return rc;
#define DLLM_BWD(DD, CC)                                                                                                    \
  return launch_bwd<DD, CC>(tq64, tq128, tk64, tk128, tv64, tv128, tdo64, tdo128, (const bf16*)dout, (const bf16*)out, lse, delta, \
                            lse2, seqlens, (bf16*)dq, (bf16*)dk, (bf16*)dv, ld_dq, ld_dkv, B, S, Skv, nh, nkv, ld_o, scale, st, 0, s_pad(S))
  if (d == 128) { if (causal) DLLM_BWD(128, true); else DLLM_BWD(128, false); }
  if (causal) DLLM_BWD(64, true); else DLLM_BWD(64, false);
#undef DLLM_BWD
}

// Backward of attn_fwd_varlen: dq [T, nh, d], dk / dv [T, nkv, d]; every row is written exactly once, by its own sample's CTAs, and
// sample b's rows equal attn_bwd_gqa on that sample alone, bit for bit.  Workspace: attn_bwd_varlen_workspace(T, nh, d).
int attn_bwd_varlen(const void* dout, const void* q, const void* k, const void* v, const void* out, const float* lse, void* dq,
                    void* dk, void* dv, const int* cu_seqlens, void* workspace, size_t workspace_bytes, int B, int T, int max_seqlen,
                    int nh, int nkv, int d, long ld_q, long ld_kv, long ld_o, long ld_dq, long ld_dkv, int causal, float scale,
                    cudaStream_t st) {
  if (B <= 0 || T <= 0 || nh <= 0 || max_seqlen <= 0 || max_seqlen > T || !cu_seqlens) return DLLM_ERR_SHAPE;
  if (nkv <= 0 || nh % nkv != 0) return DLLM_ERR_SHAPE;
  if (d != 128 && d != 64) return DLLM_ERR_UNSUPPORTED;
  if (workspace_bytes < attn_bwd_varlen_workspace(T, nh, d)) return DLLM_ERR_SHAPE;
  if ((reinterpret_cast<uintptr_t>(dq) & 15) || (reinterpret_cast<uintptr_t>(dk) & 15) || (reinterpret_cast<uintptr_t>(dv) & 15) ||
      (reinterpret_cast<uintptr_t>(out) & 15) || (reinterpret_cast<uintptr_t>(dout) & 15) || (ld_dq & 7) || (ld_dkv & 7) || (ld_o & 7))
    return DLLM_ERR_ALIGN;
  const int Tp = t_pad(T);
  float* delta = static_cast<float*>(workspace);
  float* lse2 = delta + static_cast<size_t>(Tp) * nh;
  CUtensorMap tq64, tq128, tk64, tk128, tv64, tv128, tdo64, tdo128;
  int rc;
  const int C = nh * d, Ckv = nkv * d;
  if ((rc = make_tmap_bsc(&tq64, q, 1, T, C, ld_q, 64))) return rc;
  if ((rc = make_tmap_bsc(&tq128, q, 1, T, C, ld_q, 128))) return rc;
  if ((rc = make_tmap_bsc(&tk64, k, 1, T, Ckv, ld_kv, 64))) return rc;
  if ((rc = make_tmap_bsc(&tk128, k, 1, T, Ckv, ld_kv, 128))) return rc;
  if ((rc = make_tmap_bsc(&tv64, v, 1, T, Ckv, ld_kv, 64))) return rc;
  if ((rc = make_tmap_bsc(&tv128, v, 1, T, Ckv, ld_kv, 128))) return rc;
  if ((rc = make_tmap_bsc(&tdo64, dout, 1, T, C, ld_o, 64))) return rc;
  if ((rc = make_tmap_bsc(&tdo128, dout, 1, T, C, ld_o, 128))) return rc;
#define DLLM_BWDV(DD, CC)                                                                                                          \
  return launch_bwd<DD, CC, true>(tq64, tq128, tk64, tk128, tv64, tv128, tdo64, tdo128, (const bf16*)dout, (const bf16*)out, lse, \
                                  delta, lse2, cu_seqlens, (bf16*)dq, (bf16*)dk, (bf16*)dv, ld_dq, ld_dkv, B, T, T, nh, nkv, ld_o, \
                                  scale, st, max_seqlen, Tp)
  if (d == 128) { if (causal) DLLM_BWDV(128, true); else DLLM_BWDV(128, false); }
  if (causal) DLLM_BWDV(64, true); else DLLM_BWDV(64, false);
#undef DLLM_BWDV
}

}  // namespace dllm
