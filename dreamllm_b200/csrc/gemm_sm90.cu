// Persistent warp-specialised wgmma GEMM for sm_90a (bf16 x bf16 -> fp32 accumulators in registers -> bf16|fp32).
//
//   C[M,N] = op(A) * op(B)      A "K-major":  memory [M, K] row-major        (x, dY)
//                               A "MN-major": memory [K, M] row-major        (dY^T for wgrad)
//                               B "K-major":  memory [N, K] row-major        (nn.Linear weight, fwd)
//                               B "MN-major": memory [K, N] row-major        (weight for dgrad, x for wgrad)
//
// This single kernel serves every dense contraction on the DreamLLM hot path (reference call sites:
// modeling_dreamllm.py:336-338, :395 (q/k/v/o_proj), :237 (gate/up/down_proj), :1452 (lm_head), and their
// autograd dgrad/wgrad), replacing the cuBLAS calls torch makes for nn.Linear.
//
// Structure (one CTA of 384 threads per SM, persistent over a static tile list: CTA c takes tiles c, c + grid, ...):
//   warpgroup 0     TMA producer (one elected thread): global -> 128B-swizzled smem stages, mbarrier complete_tx
//   warpgroups 1-2  consumers: each issues wgmma.mma_async (m64 x kBN x k16) for its 64 rows of the 128-row tile, keeps the fp32
//                   accumulator in registers and runs the epilogue.  bf16 outputs are staged in shared memory 64 columns at a time
//                   and leave as TMA bulk tensor stores that drain while the warpgroup goes on (kStaged); fp32 outputs, and bf16
//                   views no tensor map can describe, are stored from registers.  The producer keeps filling stages for the next
//                   tile meanwhile.
//   setmaxnreg moves registers from the producer warpgroup to the consumers (a 64 x 256 fp32 accumulator is 128 registers a thread).
#include <stdlib.h>

#include "common.cuh"
#include "gemm_sm90.h"
#include "wgmma.cuh"

namespace dllm {

constexpr int BM = 128;  // A rows per CTA (two consumer warpgroups x 64)
constexpr int BN = 256;  // widest N tile (kBN 128 / 160 / 192 / 224 are instantiated for outputs whose width tiles badly by 256: see plan_bn)
constexpr int BK = 64;   // 64 bf16 = one 128-byte swizzle line
constexpr int kGemmThreads = 384;

template <int kBN = BN, bool kStaged = false>
struct GemmCfg {
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = kBN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kBarBytes = 256;
  // staged epilogue: two 8 KB buffers (64 rows x 64 bf16 columns) per consumer warpgroup, one being filled while the other drains
  static constexpr int kOutBufBytes = 64 * 64 * 2;
  static constexpr int kOutBytes = kStaged ? 2 * 2 * kOutBufBytes : 0;
  // operand stages + staging + barriers <= 227 KB (every stage size is a multiple of the 1 KB the 128-byte swizzle needs as alignment):
  //   kBN        256  224  192  160  128
  //   direct       4    5    5    6    7
  //   staged       4    4    4    5    6
  static constexpr int kStagesFit = (227 * 1024 - kBarBytes - 1024 - kOutBytes) / kStageBytes;
  static constexpr int kStages = kStagesFit > 8 ? 8 : kStagesFit;
  static constexpr int kSmemBytes = kStages * kStageBytes + kOutBytes + kBarBytes + 1024 /*align slack*/;
  // a staging buffer leaves as one 64-column box (128-byte swizzle); widths that end in half a buffer (160, 224) use 32-column boxes
  // (64-byte swizzle), two to a buffer, so that the last one stops at the tile's edge
  static constexpr int kBoxCols = (kBN % 64) ? 32 : 64;
};

// Fused epilogue:  out = act( bf16(acc + bias[col]) ) (+ residual[row, col])   — rounding points as the reference's
// unfused bf16 sequence (Linear output rounded, activation rounded, residual add rounded).
struct GemmEpi {
  const bf16* bias;      // [N] or nullptr
  const bf16* residual;  // [M, ldr] or nullptr
  long ldr;
  int act;               // 0 none, 1 quick_gelu x*sigmoid(1.702x), 2 gelu (erf), 3 silu
  const bf16* rowbias;   // [M / rows_per_group, N] or nullptr: per-row-group bias (ResnetBlock2D's time-embedding add)
  int rows_per_group;
};

// Implicit-GEMM 3x3 / stride 1 / pad 1 convolution on NHWC activations: A[m, k] = x[n, h + r - 1, w + s - 1, c] with
// m = (n, h, w), k = (r, s, c).  A 128-row tile is the 4-D TMA box {64 c, Wb, Hb, Nb} (Wb*Hb*Nb = 128) fetched at
// coordinates (c0, s - 1, h0 + r - 1, n0): out-of-range rows/columns are zero-filled by TMA == the conv's zero padding.
struct ConvGeom {
  int cpt;       // Cin / 64: K blocks per filter tap
  int W, H;      // plane
  int HW;
};

__device__ __forceinline__ float epi_act(float x, int act) {
  if (act == 1) return x / (1.f + expf(-1.702f * x));
  if (act == 2) return 0.5f * x * (1.f + erff(x * 0.70710678118654752f));
  if (act == 3) return x / (1.f + expf(-x));
  return x;
}

__device__ __forceinline__ float2 ld_bf16x2(const bf16* p) {
  return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p));
}
__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// two adjacent output columns (col, col + 1) of row `row`; `pair` = both in range and the pair is naturally aligned
template <typename OutT>
__device__ __forceinline__ void store2(OutT* C, long ldc, int row, int col, int N, bool pair, float x0, float x1) {
  OutT* p = C + static_cast<size_t>(row) * ldc + col;
  if constexpr (sizeof(OutT) == 4) {
    if (pair) { *reinterpret_cast<float2*>(p) = make_float2(x0, x1); return; }
    p[0] = x0;
    if (col + 1 < N) p[1] = x1;
  } else {
    if (pair) { *reinterpret_cast<uint32_t*>(p) = pack_bf16(x0, x1); return; }
    p[0] = __float2bfloat16_rn(x0);
    if (col + 1 < N) p[1] = __float2bfloat16_rn(x1);
  }
}

__device__ __forceinline__ float2 bf16x2_f(uint32_t v) { return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v)); }
__device__ __forceinline__ uint32_t ld_u32(const bf16* p) { return *reinterpret_cast<const uint32_t*>(p); }

// The fused epilogue's arithmetic on two adjacent columns, shared by the direct and the staged store paths (kEpi 1 / 2).
template <int kEpi>
__device__ __forceinline__ void epi_apply(float& x0, float& x1, float2 bb, bool has_rb, float2 rb, int act, bool has_rs, float2 rs) {
  x0 += bb.x;
  x1 += bb.y;
  if (has_rb) {
    x0 += rb.x;
    x1 += rb.y;
  }
  if constexpr (kEpi == 2) {
    x0 = bf16_round(x0);
    x1 = bf16_round(x1);
    if (act == 1) {
      x0 = x0 / (1.f + __expf(-1.702f * x0));
      x1 = x1 / (1.f + __expf(-1.702f * x1));
    } else if (act == 2) {
      x0 = 0.5f * x0 * (1.f + erff(x0 * 0.70710678118654752f));
      x1 = 0.5f * x1 * (1.f + erff(x1 * 0.70710678118654752f));
    } else {
      x0 = x0 / (1.f + __expf(-x0));
      x1 = x1 / (1.f + __expf(-x1));
    }
  }
  if (has_rs) {
    x0 = bf16_round(x0) + rs.x;
    x1 = bf16_round(x1) + rs.y;
  }
}
// GEGLU on one element: value and gate pre-activations (accumulator + bias) -> h * gelu(gate), each factor rounded to bf16
__device__ __forceinline__ float epi_geglu(float a, float g) {
  a = bf16_round(a);
  g = bf16_round(g);
  return a * bf16_round(0.5f * g * (1.f + erff(g * 0.70710678118654752f)));
}

// kEpi: 0 = plain store, 1 = + bias / row-group bias / residual, 2 = 1 + activation, 3 = GEGLU.  Compile-time so that the plain and
// the bias-only epilogues carry none of the (inlined expf / erff) activation code.
//
// ksplit > 1 (split-K, small-M shapes that would leave most SMs idle): a work unit is (output tile, K slice); unit u covers K blocks
// [ks * kb_per, min(num_kb, (ks + 1) * kb_per)) of tile u / ksplit and stores its fp32 partial at rows ks * Mp + ... of C (the
// workspace; Mp = M rounded up to whole tiles); splitk_reduce_kernel sums the slices and applies the epilogue.
//
// kStaged (bf16 outputs): the epilogue's results go to shared memory and leave through tma_c, the tensor map of the output view
// ([M, N] at pitch ldc; [M, N / 2] for GEGLU), which clips at the view's extents: no row or column test guards a store.
template <bool kAMN, bool kBMN, typename OutT, bool kConv = false, int kEpi = 0, int kBN = BN, bool kStaged = false>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
            const __grid_constant__ CUtensorMap tma_c, OutT* __restrict__ C, long ldc, int M, int N, int K, int group_m, GemmEpi epi,
            ConvGeom cg, int ksplit) {
  static_assert(!kStaged || sizeof(OutT) == 2, "staged epilogue: bf16 out");
  using Cfg = GemmCfg<kBN, kStaged>;
  constexpr int kStages = Cfg::kStages;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* out_s = smem + kStages * Cfg::kStageBytes;   // staging buffers [warpgroup][2] (kStaged)
  uint64_t* bars = reinterpret_cast<uint64_t*>(out_s + Cfg::kOutBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kStages;

  const int warp_idx = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    if constexpr (kStaged) tma_prefetch_desc(&tma_c);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);   // one arrive per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  // ---- tile schedule (identical sequence in every role) ----
  const int num_m_tiles = (M + BM - 1) / BM;
  const int num_n_tiles = (N + kBN - 1) / kBN;
  const int num_tiles = num_m_tiles * num_n_tiles * ksplit;       // work units
  const int num_kb = (K + BK - 1) / BK;
  const int kb_per = (num_kb + ksplit - 1) / ksplit;
  const int split_rows = num_m_tiles * BM;                          // Mp: row pitch between K slices in the partial workspace
  const int tiles_per_group = group_m * num_n_tiles;
  auto tile_coords = [&](int tile, int& m_blk, int& n_blk) {
    const int g = tile / tiles_per_group;
    const int first_m = g * group_m;
    const int gsize = min(group_m, num_m_tiles - first_m);
    const int r = tile - g * tiles_per_group;
    m_blk = first_m + r % gsize;
    n_blk = r / gsize;
  };

  if (warp_idx < 4) {
    // ======================= TMA producer =======================
    setmaxnreg_dec<40>();
    if (warp_idx == 0 && elect_one_sync()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int m_blk, n_blk;
        tile_coords(tile / ksplit, m_blk, n_blk);
        const int ks = tile % ksplit;
        const int m0 = m_blk * BM, n0 = n_blk * kBN;
        for (int kb = ks * kb_per; kb < min(num_kb, (ks + 1) * kb_per); ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1, 1);
          uint8_t* a_s = smem + stage * Cfg::kStageBytes;
          uint8_t* b_s = a_s + Cfg::kABytes;
          const int k0 = kb * BK;
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          if constexpr (kConv) {
            // implicit-conv coordinates of this 128-pixel tile and this K block's filter tap
            const int tap = kb / cg.cpt;
            const int cv_c = (kb - tap * cg.cpt) * BK;
            const int r = tap / 3, sx = tap - 3 * r;
            const int cv_n = m0 / cg.HW;
            const int rem = m0 - cv_n * cg.HW;
            const int h0 = rem / cg.W;
            const int cv_h = h0 + r - 1;
            const int cv_w = (rem - h0 * cg.W) + sx - 1;   // non-zero only for planes wider than one 128-pixel tile
            tma_load_4d(a_s, &tma_a, &full_bar[stage], cv_c, cv_w, cv_h, cv_n);
          } else if constexpr (!kAMN) {
            tma_load_2d(a_s, &tma_a, &full_bar[stage], k0, m0);
          } else {
#pragma unroll
            for (int i = 0; i < BM / 64; ++i) tma_load_2d(a_s + i * 8192, &tma_a, &full_bar[stage], m0 + i * 64, k0);
          }
          if constexpr (!kBMN) {
            tma_load_2d(b_s, &tma_b, &full_bar[stage], k0, n0);
          } else {
#pragma unroll
            for (int i = 0; i < kBN / 64; ++i) tma_load_2d(b_s + i * 8192, &tma_b, &full_bar[stage], n0 + i * 64, k0);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ======================= consumers: wgmma + epilogue =======================
    setmaxnreg_inc<232>();
    const int wg = (threadIdx.x >> 7) - 1;   // 0 / 1: rows [64 wg, 64 wg + 64) of the tile
    const int t = threadIdx.x & 127;
    // accumulator fragment of m64nN: element 4j + 2h + e sits at row 16 * (t / 32) + (t % 32) / 4 + 8h, column 8j + 2 (t % 4) + e
    const int r_in = 16 * (t >> 5) + ((t & 31) >> 2);
    const int c_in = 2 * (t & 3);
    float acc[kBN / 2];
    // stage-0 descriptors; every other (stage, K step) is that plus a compile-time byte offset (the start-address field counts 16-byte
    // units and no tile crosses the 256 KB its 14 bits span, so a plain add is exact).  Hoisted, the K block's four wgmma issue back to back.
    const uint32_t a_s0 = smem_u32(smem) + wg * 8192;   // 64 K-major rows, or MN-major box wg
    const uint32_t b_s0 = smem_u32(smem) + Cfg::kABytes;
    const uint64_t adesc0 = kAMN ? make_smem_desc(a_s0, 8192, 1024) : make_smem_desc(a_s0, 16, 1024);
    const uint64_t bdesc0 = kBMN ? make_smem_desc(b_s0, 8192, 1024) : make_smem_desc(b_s0, 16, 1024);
    constexpr uint32_t a_step = kAMN ? 2048u : 32u, b_step = kBMN ? 2048u : 32u;   // bytes per K = 16 step
    const uint32_t a_lo = __shfl_sync(0xffffffffu, static_cast<uint32_t>(adesc0), 0), a_hi = static_cast<uint32_t>(adesc0 >> 32);
    const uint32_t b_lo = __shfl_sync(0xffffffffu, static_cast<uint32_t>(bdesc0), 0), b_hi = static_cast<uint32_t>(bdesc0 >> 32);
    // staged epilogue: stmatrix.x4 writes four 8 x 8 blocks (two 8-column groups x two 8-row halves) of the warp's 16 rows; lane l
    // supplies the address of row l % 8 of block l / 8.  A buffer row is 128 bytes (64 in the 32-column boxes) and its 16-byte chunks
    // are XOR-swizzled by the row as the TMA box expects, which also spreads the 8 rows of a block over all 32 banks.
    const int st_r = 16 * (t >> 5) + 8 * ((lane >> 3) & 1) + (lane & 7);
    const uint32_t st_row = st_r * (Cfg::kBoxCols == 64 ? 128 : 64);
    const uint32_t st_xor = ((lane >> 4) ^ (Cfg::kBoxCols == 64 ? (st_r & 7) : ((st_r >> 1) & 3))) << 4;
    int sbuf = 0;   // staging buffer the next 64 columns go to
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int m_blk, n_blk;
      tile_coords(tile / ksplit, m_blk, n_blk);
      const int ks = tile % ksplit;
      const int kb0 = ks * kb_per, kb1 = min(num_kb, kb0 + kb_per);
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase, 3);
        // only the low word of a descriptor (start address, leading offset) changes with the stage and the K step, and the sum never
        // carries out of it.  The words are broadcast from lane 0, which tells the compiler they are the same across the warp: the
        // adds run on the uniform datapath, where wgmma takes its descriptors from, and the group's MMAs issue back to back.
        const uint32_t soff = __shfl_sync(0xffffffffu, static_cast<uint32_t>((stage * Cfg::kStageBytes) >> 4), 0);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          const uint64_t da = (static_cast<uint64_t>(a_hi) << 32) | (a_lo + soff + ((k * a_step) >> 4));
          const uint64_t db = (static_cast<uint64_t>(b_hi) << 32) | (b_lo + soff + ((k * b_step) >> 4));
          wgmma_ss<kBN, kAMN ? 1 : 0, kBMN ? 1 : 0>(acc, da, db, (kb != kb0 || k != 0) ? 1 : 0);
        }
        wgmma_commit();
        wgmma_wait<1>();   // the previous K block's MMAs have retired: its stage can be refilled
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      const int row_t = m_blk * BM + wg * 64 + r_in;        // + 8h
      const int col_t = n_blk * kBN + c_in;                 // + 8j
      if constexpr (kStaged) {
        // ---- epilogue: registers -> swizzled staging buffer -> TMA store, one buffer (64 output columns, 8 groups of 8) at a time ----
        constexpr int kJ = (kEpi == 3) ? kBN / 16 : kBN / 8;        // 8-column groups of the output tile
        constexpr int kBufs = (kJ + 7) / 8;
        const int ncols = (kEpi == 3) ? (N >> 1) : N;
        const int ocol0 = (kEpi == 3) ? n_blk * (kBN / 2) : n_blk * kBN;
        const int orow0 = m_blk * BM + wg * 64;
        const bool live = orow0 < M;                                 // the same for the whole warpgroup
        const bool has_rb = kEpi > 0 && epi.rowbias != nullptr, has_rs = kEpi > 0 && epi.residual != nullptr;
        const bf16* rbp[2] = {nullptr, nullptr};
        const bf16* rsp[2] = {nullptr, nullptr};
        if constexpr (kEpi == 1 || kEpi == 2) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = row_t + 8 * h;
            if (has_rb && row < M) rbp[h] = epi.rowbias + static_cast<size_t>(row / epi.rows_per_group) * N;
            if (has_rs && row < M) rsp[h] = epi.residual + static_cast<size_t>(row) * epi.ldr;
          }
        }
        // the epilogue's operands of the two 8-column groups jj, jj + 1 of buffer u, as raw bf16 pairs: bias (GEGLU: value bias),
        // row-group bias (GEGLU: gate bias in rb[0]), residual.  The first two groups' are fetched while the last K blocks retire (kEarly);
        // the rest are independent loads the compiler is free to issue ahead of the arithmetic (stmatrix does not order them).
        struct EpiIn { uint32_t b[2], rb[2][2], rs[2][2]; };
        auto epi_load = [&](int u, int jj0, EpiIn& in) {
          if constexpr (kEpi != 0) {
#pragma unroll
            for (int dj = 0; dj < 2; ++dj) {
              if constexpr (kEpi == 3) {
                const int col = col_t + 128 * u + 8 * (jj0 + dj);  // value column in the permuted N space (gate at + 64)
                const bool ok = epi.bias != nullptr && col < N;
                in.b[dj] = ok ? ld_u32(epi.bias + col) : 0u;
                in.rb[0][dj] = ok ? ld_u32(epi.bias + col + 64) : 0u;
              } else {
                const int col = col_t + 64 * u + 8 * (jj0 + dj);
                const bool ok = col < N;                             // fused epilogues require N % 8 == 0
                in.b[dj] = (ok && epi.bias != nullptr) ? ld_u32(epi.bias + col) : 0u;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  in.rb[h][dj] = (ok && rbp[h] != nullptr) ? ld_u32(rbp[h] + col) : 0u;
                  in.rs[h][dj] = (ok && rsp[h] != nullptr) ? ld_u32(rsp[h] + col) : 0u;
                }
              }
            }
          }
        };
        constexpr bool kEarly = kBN <= 192;   // the 224 / 256-wide accumulators leave no registers to hold operands across the wait
        EpiIn first;
        if (kEarly && live) epi_load(0, 0, first);
        wgmma_wait<0>();
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        if (live) {
#pragma unroll
          for (int u = 0; u < kBufs; ++u) {
            const int c0 = ocol0 + 64 * u;
            if (c0 >= ncols) break;
            uint8_t* buf = out_s + (wg * 2 + sbuf) * Cfg::kOutBufBytes;
            const uint32_t buf_u32 = smem_u32(buf);
#pragma unroll
            for (int jj = 0; jj < 8; jj += 2) {
              if (8 * u + jj >= kJ) continue;
              EpiIn cur;
              if (kEarly && u == 0 && jj == 0) cur = first;
              else epi_load(u, jj, cur);
              uint32_t r[4];                                         // matrices (jj, h 0), (jj, h 1), (jj + 1, h 0), (jj + 1, h 1)
#pragma unroll
              for (int dj = 0; dj < 2; ++dj) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  float x0, x1;
                  if constexpr (kEpi == 3) {
                    const int j = 16 * u + jj + dj;
                    const float2 bv = bf16x2_f(cur.b[dj]), bg = bf16x2_f(cur.rb[0][dj]);
                    x0 = epi_geglu(acc[4 * j + 2 * h] + bv.x, acc[4 * (j + 8) + 2 * h] + bg.x);
                    x1 = epi_geglu(acc[4 * j + 2 * h + 1] + bv.y, acc[4 * (j + 8) + 2 * h + 1] + bg.y);
                  } else {
                    const int j = 8 * u + jj + dj;
                    x0 = acc[4 * j + 2 * h];
                    x1 = acc[4 * j + 2 * h + 1];
                    if constexpr (kEpi > 0)
                      epi_apply<kEpi>(x0, x1, bf16x2_f(cur.b[dj]), has_rb, bf16x2_f(cur.rb[h][dj]), epi.act, has_rs,
                                      bf16x2_f(cur.rs[h][dj]));
                  }
                  r[2 * dj + h] = pack_bf16(x0, x1);
                }
              }
              const uint32_t off = Cfg::kBoxCols == 64 ? st_row + ((jj << 4) ^ st_xor)
                                                       : (jj >> 2) * 4096 + st_row + (((jj & 3) << 4) ^ st_xor);
              stmatrix_x4(buf_u32 + off, r[0], r[1], r[2], r[3]);
            }
            // every thread's writes become visible to the TMA engine; thread 0 has seen the previous store (the other buffer) read
            // its source, so past the barrier that buffer is free for u + 1
            fence_proxy_async_smem();
            if (t == 0) tma_store_wait_read<0>();
            named_bar_sync(1 + wg, 128);
            if (t == 0) {
              if constexpr (Cfg::kBoxCols == 64) {
                tma_store_2d(&tma_c, buf, c0, orow0);
              } else {
#pragma unroll
                for (int k = 0; k < 2; ++k)
                  if (8 * u + 4 * k < kJ && c0 + 32 * k < ncols) tma_store_2d(&tma_c, buf + 4096 * k, c0 + 32 * k, orow0);
              }
              tma_store_commit();
            }
            sbuf ^= 1;
          }
        }
      } else {
      wgmma_wait<0>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);

      // ---- epilogue: registers -> global (fp32 outputs; bf16 views whose base or pitch a tensor map cannot take) ----
      const long row_off = (ksplit > 1) ? static_cast<long>(ks) * split_rows : 0;
      const bool pair_ok = (ldc & 1) == 0 && (reinterpret_cast<uintptr_t>(C) & (2 * sizeof(OutT) - 1)) == 0;
      if constexpr (kEpi == 3) {
        // GEGLU epilogue (diffusers FeedForward: h, gate = proj(x).chunk(2); out = h * gelu(gate)).  The weight rows were permuted at
        // load time so that every 128-column group of this GEMM's N space is [64 value columns | their 64 gate columns]; a thread
        // holds value column c and its gate column c + 64 of the same rows and writes column c of the [M, N/2] output — the [M, N]
        // projection is never written.  Rounding points = the unfused sequence (Linear output to bf16, gelu(gate) to bf16, product to
        // bf16): bit-identical results.
        static_assert(kEpi != 3 || sizeof(OutT) == 2, "GEGLU epilogue: bf16 out");
#pragma unroll
        for (int pr = 0; pr < kBN / 128; ++pr) {
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int j = pr * 16 + jj;
            const int col = col_t + 8 * j;                  // value column in the permuted N space (gate at + 64)
            if (col >= N) continue;
            float2 bv = make_float2(0.f, 0.f), bg = make_float2(0.f, 0.f);
            if (epi.bias != nullptr) { bv = ld_bf16x2(epi.bias + col); bg = ld_bf16x2(epi.bias + col + 64); }
            const int ocol = (n_blk * kBN >> 1) + pr * 64 + 8 * jj + c_in;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = row_t + 8 * h;
              if (row >= M) continue;
              const float o0 = epi_geglu(acc[4 * j + 2 * h] + bv.x, acc[4 * (j + 8) + 2 * h] + bg.x);
              const float o1 = epi_geglu(acc[4 * j + 2 * h + 1] + bv.y, acc[4 * (j + 8) + 2 * h + 1] + bg.y);
              store2<OutT>(C, ldc, row, ocol, N >> 1, pair_ok, o0, o1);
            }
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < kBN / 8; ++j) {
          const int col = col_t + 8 * j;
          if (col >= N) continue;
          const bool pair = pair_ok && col + 1 < N;
          float2 bb = make_float2(0.f, 0.f);
          if (kEpi > 0 && epi.bias != nullptr) bb = ld_bf16x2(epi.bias + col);   // fused epilogues require N % 8 == 0
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = row_t + 8 * h;
            if (row >= M) continue;
            float x0 = acc[4 * j + 2 * h], x1 = acc[4 * j + 2 * h + 1];
            if constexpr (kEpi > 0) {
              float2 rb = make_float2(0.f, 0.f), rs = make_float2(0.f, 0.f);
              if (epi.rowbias != nullptr) rb = ld_bf16x2(epi.rowbias + static_cast<size_t>(row / epi.rows_per_group) * N + col);
              if (epi.residual != nullptr) rs = ld_bf16x2(epi.residual + static_cast<size_t>(row) * epi.ldr + col);
              epi_apply<kEpi>(x0, x1, bb, epi.rowbias != nullptr, rb, epi.act, epi.residual != nullptr, rs);
            }
            store2<OutT>(C, ldc, static_cast<int>(row + row_off), col, N, pair, x0, x1);
          }
        }
      }
      }
    }
    if constexpr (kStaged) {
      if (t == 0) tma_store_wait_all<0>();   // the last stores have left shared memory and reached global memory before the CTA exits
    }
  }
}

// ------------------------------------------------------------------------------------------------ host
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess || !p) return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

// 2D row-major tensor [rows, cols] with row stride `ld` elements; box = [box_rows, box_cols]; 128B swizzle.
int make_tmap_2d(CUtensorMap* map, const void* ptr, int elem_bytes, uint64_t rows, uint64_t cols, uint64_t ld,
                 uint32_t box_rows, uint32_t box_cols) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return DLLM_ERR_DRIVER;
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || ((ld * elem_bytes) & 15)) return DLLM_ERR_ALIGN;
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstr[1] = {ld * elem_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUtensorMapDataType dt = elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  CUresult r = enc(map, dt, 2, const_cast<void*>(ptr), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    fprintf(stderr, "dllm: cuTensorMapEncodeTiled failed (CUresult %d): ptr=%p elem=%d rows=%llu cols=%llu ld=%llu box=[%u x %u]\n",
            (int)r, ptr, elem_bytes, (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld, box_rows, box_cols);
  return r == CUDA_SUCCESS ? 0 : DLLM_ERR_TMAP;
}

// Output view [rows, cols] of bf16 at pitch `ld`, written in boxes of 64 rows x 32 | 64 columns (64- | 128-byte swizzle).  The extents
// are the view's, not the allocation's: the TMA store clips at them, and that is all that keeps a tile's tail rows and columns from
// being written.
static int make_tmap_out(CUtensorMap* map, void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_cols) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return DLLM_ERR_DRIVER;
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstr[1] = {ld * 2};
  cuuint32_t box[2] = {box_cols, 64};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, ptr, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   box_cols == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    fprintf(stderr, "dllm: cuTensorMapEncodeTiled(out) failed (CUresult %d): ptr=%p rows=%llu cols=%llu ld=%llu box=[64 x %u]\n", (int)r,
            ptr, (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld, box_cols);
  return r == CUDA_SUCCESS ? 0 : DLLM_ERR_TMAP;
}

// SMs left free for a concurrently running collective (NCCL all-reduce overlapped with backward): a persistent GEMM that
// asks for every SM would have the CTAs that cannot be scheduled wait for the collective kernel to finish and then run
// their whole static tile list alone.  See dreamllm_b200/ddp.py.
static int g_reserved_sms = 0;
void set_reserved_sms(int n) { g_reserved_sms = n < 0 ? 0 : n; }
int reserved_sms() { return g_reserved_sms; }

int num_sms() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
      cudaGetLastError();
      n = 0;
      return 132;   // no device visible (build host): plan for an H100 SXM so the workspace queries stay meaningful
    }
  }
  return n;
}

// N-tile width of split-K launches (plan_split) and of the launches that have no intermediate width (MN-major A, fp32 out): 256 (the
// widest wgmma, half the A re-reads from shared memory per MMA of a 128-wide tile) except for outputs that fit ONE 128-wide tile, where a
// 256-wide tile would be half padding.
static inline int pick_bn(int N) { return N <= 128 ? 128 : 256; }

// Tile planner of the unsplit bf16-output launches with K-major A (forward NT, dgrad NN, conv): the N width that minimises
// ceil(tiles / SMs) x t(width), t being the per-tile time relative to 256 (DESIGN §4 has the measurement).  A width that fits N exactly
// computes no padding columns (UNet C = 320 / 640 / 960), and a narrower tile can fill the last wave of a small-M launch (LLM M = 400).
// MN-major B is fetched in 64-column boxes, so its widths are multiples of 64.  t varies by about +-15 % from shape to shape, so costs
// within 5 % of the least count as a tie, and ties go to the wider tile (widest first below): on many-wave launches (7B training at
// 8192 tokens) the wave counts of all widths come out nearly even and 256, the most efficient per column, stays.
struct BnCost {
  int bn;
  float t;
};
static constexpr BnCost kBnKMajor[] = {{256, 1.f}, {224, 0.861f}, {192, 0.781f}, {160, 0.645f}, {128, 0.536f}};
static constexpr BnCost kBnMNMajor[] = {{256, 1.f}, {192, 0.781f}, {128, 0.536f}};

// DLLM_GEMM_BN=<width> pins the planner's choice (scripts/gemm_shapes.py times every width this way); other widths are ignored.
static int forced_bn() {
  static const int bn = [] {
    const char* s = getenv("DLLM_GEMM_BN");
    return s ? atoi(s) : 0;
  }();
  return bn;
}

static int plan_bn(int M, int N, int a_mn, int b_mn, bool bf16_out) {
  if (a_mn || !bf16_out) return pick_bn(N);
  const BnCost* w = b_mn ? kBnMNMajor : kBnKMajor;
  const int nw = b_mn ? sizeof(kBnMNMajor) / sizeof(BnCost) : sizeof(kBnKMajor) / sizeof(BnCost);
  for (int i = 0; i < nw; ++i)
    if (w[i].bn == forced_bn()) return w[i].bn;
  int slots = num_sms() - g_reserved_sms;
  if (slots < 1) slots = 1;
  const long mt = (M + BM - 1) / BM;
  float cost[8], least = 0.f;
  for (int i = 0; i < nw; ++i) {
    const long tiles = mt * ((N + w[i].bn - 1) / w[i].bn);
    cost[i] = static_cast<float>((tiles + slots - 1) / slots) * w[i].t;
    if (i == 0 || cost[i] < least) least = cost[i];
  }
  for (int i = 0; i < nw; ++i)
    if (cost[i] <= 1.05f * least) return w[i].bn;
  return w[0].bn;
}

template <bool kAMN, bool kBMN, typename OutT, bool kConv = false, int kEpi = 0, int kBN = BN, bool kStaged = false>
static int launch_gemm_bn(const CUtensorMap& ta, const CUtensorMap& tb, void* C, long ldc, int M, int N, int K, const GemmEpi& epi,
                          cudaStream_t stream, ConvGeom cg = ConvGeom{1, 1, 1, 1}, int ksplit = 1) {
  using Cfg = GemmCfg<kBN, kStaged>;
  auto kern = gemm_kernel<kAMN, kBMN, OutT, kConv, kEpi, kBN, kStaged>;
  CUtensorMap tc{};
  if constexpr (kStaged) {
    if (int rc = make_tmap_out(&tc, C, M, kEpi == 3 ? N / 2 : N, ldc, Cfg::kBoxCols)) return rc;
  }
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes) != cudaSuccess)
      return DLLM_ERR_LAUNCH;
    attr_set = true;
  }
  const int num_tiles = ((M + BM - 1) / BM) * ((N + kBN - 1) / kBN) * ksplit;
  int avail = num_sms() - g_reserved_sms;
  if (avail < 1) avail = 1;
  const int grid = num_tiles < avail ? num_tiles : avail;
  kern<<<grid, kGemmThreads, Cfg::kSmemBytes, stream>>>(ta, tb, tc, static_cast<OutT*>(C), ldc, M, N, K, 16, epi, cg, ksplit);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}
// bf16 outputs take the staged (TMA store) epilogue whenever a tensor map can describe the view: base 16-byte aligned, row pitch a
// multiple of 16 bytes.  Any other bf16 view, and every fp32 output, is stored from registers.
template <bool kAMN, bool kBMN, typename OutT, bool kConv, int kEpi, int kBN>
static int launch_gemm_out(const CUtensorMap& ta, const CUtensorMap& tb, void* C, long ldc, int M, int N, int K, const GemmEpi& epi,
                           cudaStream_t stream, ConvGeom cg) {
  if constexpr (sizeof(OutT) == 2) {
    if (!(reinterpret_cast<uintptr_t>(C) & 15) && !(ldc & 7))
      return launch_gemm_bn<kAMN, kBMN, OutT, kConv, kEpi, kBN, true>(ta, tb, C, ldc, M, N, K, epi, stream, cg);
  }
  return launch_gemm_bn<kAMN, kBMN, OutT, kConv, kEpi, kBN, false>(ta, tb, C, ldc, M, N, K, epi, stream, cg);
}
// `bn` must be the value the B tensor map's box was built for (plan_bn); only the widths plan_bn can return are instantiated
template <bool kAMN, bool kBMN, typename OutT, bool kConv = false, int kEpi = 0>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, void* C, long ldc, int M, int N, int K, const GemmEpi& epi,
                       cudaStream_t stream, ConvGeom cg, int bn) {
  if constexpr (!kAMN && sizeof(OutT) == 2) {
    if (bn == 192) return launch_gemm_out<kAMN, kBMN, OutT, kConv, kEpi, 192>(ta, tb, C, ldc, M, N, K, epi, stream, cg);
    if constexpr (!kBMN) {
      if (bn == 160) return launch_gemm_out<kAMN, kBMN, OutT, kConv, kEpi, 160>(ta, tb, C, ldc, M, N, K, epi, stream, cg);
      if (bn == 224) return launch_gemm_out<kAMN, kBMN, OutT, kConv, kEpi, 224>(ta, tb, C, ldc, M, N, K, epi, stream, cg);
    }
  }
  if (bn == 128) return launch_gemm_out<kAMN, kBMN, OutT, kConv, kEpi, 128>(ta, tb, C, ldc, M, N, K, epi, stream, cg);
  if (bn == 256) return launch_gemm_out<kAMN, kBMN, OutT, kConv, kEpi, 256>(ta, tb, C, ldc, M, N, K, epi, stream, cg);
  return DLLM_ERR_UNSUPPORTED;
}

// ------------------------------------------------------------------------------------------------ split-K (small-M shapes)
// A [256 x 1280] output over K = 11520 (UNet conv 1280 -> 1280 on the 8x8 plane of 4 samples) is 10 tiles: 10 of 132 SMs busy for
// 180 K blocks each.  Split-K hands every (tile, K slice) to its own CTA, writes fp32 partials to a caller-provided workspace and lets
// one small kernel sum them and apply the epilogue with the usual rounding points.
struct SplitPlan {
  int bn, ksplit, mp;   // mp = M rounded up to whole tiles
  size_t ws_bytes;
};
static SplitPlan plan_split(int M, int N, int K) {
  SplitPlan p;
  p.bn = pick_bn(N);
  const int mt = (M + BM - 1) / BM, nt = (N + p.bn - 1) / p.bn;
  const int tiles = mt * nt, num_kb = (K + BK - 1) / BK;
  int slots = num_sms() - g_reserved_sms;
  if (slots < 1) slots = 1;
  int ks = 1;
  if (tiles > 0 && tiles * 2 <= slots && num_kb >= 8) {   // (an empty output plans no split: its entry points refuse the shape)
    ks = slots / tiles;
    if (ks > num_kb / 4) ks = num_kb / 4;    // at least 4 K blocks per slice
    if (ks > 16) ks = 16;
    if (ks < 2) ks = 1;
    // no empty slice: the kernel gives every slice ceil(num_kb / ks) K blocks, so the last of e.g. 16 slices of 90 blocks would start
    // past the end and store an accumulator no MMA ever initialised
    if (ks > 1) { const int per = (num_kb + ks - 1) / ks; ks = (num_kb + per - 1) / per; }
  }
  p.ksplit = ks;
  p.mp = mt * BM;
  p.ws_bytes = ks > 1 ? static_cast<size_t>(ks) * p.mp * N * sizeof(float) : 0;
  return p;
}
size_t gemm_splitk_workspace(int M, int N, int K) { return plan_split(M, N, K).ws_bytes; }
int gemm_tile_bn(int M, int N, int K, int b_mn) {
  const SplitPlan p = plan_split(M, N, K);
  return p.ksplit > 1 ? p.bn : plan_bn(M, N, 0, b_mn, true);
}

// out[m, n] = epilogue( sum_ks ws[ks * mp + m, n] ): bias / row-group bias added in fp32, rounded to bf16, optional activation (rounded),
// optional residual add (rounded) — the rounding points of gemm_kernel's fused epilogues.  One thread = 8 columns.
__global__ void splitk_reduce_kernel(const float* __restrict__ ws, bf16* __restrict__ out, long ldc, int M, int N, int mp, int ksplit,
                                     GemmEpi epi) {
  const int nvec = N >> 3;
  const long gid = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (gid >= static_cast<long>(M) * nvec) return;
  const int v = static_cast<int>(gid % nvec);
  const int m = static_cast<int>(gid / nvec);
  float x[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) x[e] = 0.f;
  for (int ks = 0; ks < ksplit; ++ks) {
    const float4* p = reinterpret_cast<const float4*>(ws + (static_cast<size_t>(ks) * mp + m) * N + v * 8);
    const float4 a = p[0], b = p[1];
    x[0] += a.x; x[1] += a.y; x[2] += a.z; x[3] += a.w; x[4] += b.x; x[5] += b.y; x[6] += b.z; x[7] += b.w;
  }
  auto add8 = [&](const bf16* src) {
    const uint4 q = __ldg(reinterpret_cast<const uint4*>(src));
    const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&q);
#pragma unroll
    for (int e = 0; e < 4; ++e) { const float2 f = __bfloat1622float2(h2[e]); x[2 * e] += f.x; x[2 * e + 1] += f.y; }
  };
  if (epi.bias) add8(epi.bias + v * 8);
  if (epi.rowbias) add8(epi.rowbias + static_cast<size_t>(m / epi.rows_per_group) * N + v * 8);
  if (epi.act) {
#pragma unroll
    for (int e = 0; e < 8; ++e) x[e] = epi_act(__bfloat162float(__float2bfloat16_rn(x[e])), epi.act);
  }
  if (epi.residual) {
    const uint4 q = *reinterpret_cast<const uint4*>(epi.residual + static_cast<size_t>(m) * epi.ldr + v * 8);
    const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&q);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = __bfloat1622float2(h2[e]);
      x[2 * e] = __bfloat162float(__float2bfloat16_rn(x[2 * e])) + f.x;
      x[2 * e + 1] = __bfloat162float(__float2bfloat16_rn(x[2 * e + 1])) + f.y;
    }
  }
  uint4 o;
  o.x = pack_bf16(x[0], x[1]); o.y = pack_bf16(x[2], x[3]); o.z = pack_bf16(x[4], x[5]); o.w = pack_bf16(x[6], x[7]);
  *reinterpret_cast<uint4*>(out + static_cast<size_t>(m) * ldc + v * 8) = o;
}
static int launch_splitk_reduce(const void* ws, void* out, long ldc, int M, int N, const SplitPlan& p, const GemmEpi& epi, cudaStream_t st) {
  const long total = static_cast<long>(M) * (N / 8);
  splitk_reduce_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>((const float*)ws, (bf16*)out, ldc, M, N, p.mp, p.ksplit, epi);
  return cudaGetLastError() == cudaSuccess ? 0 : DLLM_ERR_LAUNCH;
}

// bf16-output GEMM (fwd NT or dgrad NN) with the fused-epilogue operands, run as split-K when the shape calls for it and a workspace of
// gemm_splitk_workspace(M, N, K) bytes is given; otherwise identical to gemm_bf16_ex.
int gemm_bf16_ws(const void* A, const void* B, void* C, int M, int N, int K, long lda, long ldb, long ldc, int b_mn, const void* bias,
                 const void* residual, long ldr, int act, void* ws, size_t ws_bytes, cudaStream_t stream) {
  const SplitPlan p = plan_split(M, N, K);
  // (the reduce kernel writes 16 bytes at a time: an output view it cannot write that way runs unsplit)
  if (p.ksplit <= 1 || !ws || ws_bytes < p.ws_bytes || (N % 8) || (reinterpret_cast<uintptr_t>(ws) & 15) || (ldc % 8) ||
      (reinterpret_cast<uintptr_t>(C) & 15))
    return gemm_bf16_ex(A, B, C, M, N, K, lda, ldb, ldc, 0, b_mn, 0, -1, bias, residual, ldr, act, stream);
  if (residual && ((reinterpret_cast<uintptr_t>(residual) & 15) || ((ldr * 2) & 15))) return DLLM_ERR_ALIGN;
  if (bias && (reinterpret_cast<uintptr_t>(bias) & 15)) return DLLM_ERR_ALIGN;
  CUtensorMap ta, tb;
  int rc;
  if ((rc = make_tmap_2d(&ta, A, 2, M, K, lda, BM, BK))) return rc;
  if (!b_mn) rc = make_tmap_2d(&tb, B, 2, N, K, ldb, p.bn, BK);
  else rc = make_tmap_2d(&tb, B, 2, K, N, ldb, BK, 64);
  if (rc) return rc;
  GemmEpi none{nullptr, nullptr, 0, 0, nullptr, 1};
  const ConvGeom nocg{1, 1, 1, 1};
  if (!b_mn) rc = (p.bn == 128) ? launch_gemm_bn<false, false, float, false, 0, 128>(ta, tb, ws, N, M, N, K, none, stream, nocg, p.ksplit)
                                : launch_gemm_bn<false, false, float, false, 0, 256>(ta, tb, ws, N, M, N, K, none, stream, nocg, p.ksplit);
  else rc = (p.bn == 128) ? launch_gemm_bn<false, true, float, false, 0, 128>(ta, tb, ws, N, M, N, K, none, stream, nocg, p.ksplit)
                          : launch_gemm_bn<false, true, float, false, 0, 256>(ta, tb, ws, N, M, N, K, none, stream, nocg, p.ksplit);
  if (rc) return rc;
  GemmEpi epi{static_cast<const bf16*>(bias), static_cast<const bf16*>(residual), ldr, act, nullptr, 1};
  return launch_splitk_reduce(ws, C, ldc, M, N, p, epi, stream);
}

int gemm_bf16(const void* A, const void* B, void* C, int M, int N, int K, long lda, long ldb, long ldc, int a_mn,
              int b_mn, int out_fp32, int cta_pair, cudaStream_t stream) {
  return gemm_bf16_ex(A, B, C, M, N, K, lda, ldb, ldc, a_mn, b_mn, out_fp32, cta_pair, nullptr, nullptr, 0, 0, stream);
}

// cta_pair: kept in the ABI for callers written against two-CTA builds; every tile here is computed by one CTA, so it has no effect.
int gemm_bf16_ex(const void* A, const void* B, void* C, int M, int N, int K, long lda, long ldb, long ldc, int a_mn,
                 int b_mn, int out_fp32, int cta_pair, const void* bias, const void* residual, long ldr, int act,
                 cudaStream_t stream) {
  (void)cta_pair;
  if (M <= 0 || N <= 0 || K <= 0 || act < 0 || act > 3) return DLLM_ERR_SHAPE;
  if ((bias || residual) && (N % 8)) return DLLM_ERR_SHAPE;
  if (residual && ((reinterpret_cast<uintptr_t>(residual) & 15) || ((ldr * 2) & 15))) return DLLM_ERR_ALIGN;
  if (bias && (reinterpret_cast<uintptr_t>(bias) & 15)) return DLLM_ERR_ALIGN;
  if (reinterpret_cast<uintptr_t>(C) & (out_fp32 ? 15 : 1)) return DLLM_ERR_ALIGN;   // bf16: see launch_gemm_out
  GemmEpi epi{static_cast<const bf16*>(bias), static_cast<const bf16*>(residual), ldr, act, nullptr, 1};
  const int bn = plan_bn(M, N, a_mn, b_mn, !out_fp32);
  const ConvGeom nocg{1, 1, 1, 1};
  CUtensorMap ta, tb;
  int rc;
  // A
  if (!a_mn) rc = make_tmap_2d(&ta, A, 2, M, K, lda, BM, BK);
  else rc = make_tmap_2d(&ta, A, 2, K, M, lda, BK, 64);
  if (rc) return rc;
  // B
  if (!b_mn) rc = make_tmap_2d(&tb, B, 2, N, K, ldb, bn, BK);
  else rc = make_tmap_2d(&tb, B, 2, K, N, ldb, BK, 64);
  if (rc) return rc;

  const int emode = (act != 0) ? 2 : ((bias || residual) ? 1 : 0);
  if (emode != 0) {
    // fused epilogues exist for the forward (NT, bf16 out) contraction only
    if (a_mn || b_mn || out_fp32) return DLLM_ERR_UNSUPPORTED;
    return emode == 2 ? launch_gemm<false, false, bf16, false, 2>(ta, tb, C, ldc, M, N, K, epi, stream, nocg, bn)
                      : launch_gemm<false, false, bf16, false, 1>(ta, tb, C, ldc, M, N, K, epi, stream, nocg, bn);
  }
#define DLLM_GEMM_CASE(AMN, BMN)                                                                           \
  if ((a_mn != 0) == AMN && (b_mn != 0) == BMN) {                                                          \
    return out_fp32 ? launch_gemm<AMN, BMN, float>(ta, tb, C, ldc, M, N, K, epi, stream, nocg, bn)         \
                    : launch_gemm<AMN, BMN, bf16>(ta, tb, C, ldc, M, N, K, epi, stream, nocg, bn);         \
  }
  DLLM_GEMM_CASE(false, false)
  DLLM_GEMM_CASE(false, true)
  DLLM_GEMM_CASE(true, true)
  DLLM_GEMM_CASE(true, false)
#undef DLLM_GEMM_CASE
  return DLLM_ERR_SHAPE;
}

// out[M, N/2] = GEGLU(A @ Wp^T + bias_p): Wp / bias_p are the FeedForward's `proj` weight / bias with rows permuted so that every
// 128-row group is [64 value rows | the 64 matching gate rows] (dreamllm_b200/unet.py builds them once per frozen UNet).
int gemm_bf16_geglu(const void* A, const void* Wp, const void* bias_p, void* out, int M, int N, int K, long lda, long ldb, long ldc,
                    cudaStream_t stream) {
  if (M <= 0 || N <= 0 || K <= 0 || (N % 128)) return DLLM_ERR_SHAPE;
  if (bias_p && (reinterpret_cast<uintptr_t>(bias_p) & 15)) return DLLM_ERR_ALIGN;
  if (reinterpret_cast<uintptr_t>(out) & 1) return DLLM_ERR_ALIGN;
  GemmEpi epi{static_cast<const bf16*>(bias_p), nullptr, 0, 2, nullptr, 1};
  CUtensorMap ta, tb;
  int rc;
  if ((rc = make_tmap_2d(&ta, A, 2, M, K, lda, BM, BK))) return rc;
  if ((rc = make_tmap_2d(&tb, Wp, 2, N, K, ldb, BN, BK))) return rc;
  return launch_gemm_out<false, false, bf16, false, 3, 256>(ta, tb, out, ldc, M, N, K, epi, stream, ConvGeom{1, 1, 1, 1});
}

// 4-D NHWC activation map: dims {C, W, H, N}, box {64, Wb, Hb, Nb}, 128B swizzle.
static int make_tmap_nhwc(CUtensorMap* map, const void* ptr, int Nimg, int H, int W, int C, int Wb, int Hb, int Nb) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return DLLM_ERR_DRIVER;
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (C % 8)) return DLLM_ERR_ALIGN;
  cuuint64_t gdim[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)Nimg};
  cuuint64_t gstr[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[4] = {64, (cuuint32_t)Wb, (cuuint32_t)Hb, (cuuint32_t)Nb};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), gdim, gstr, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) fprintf(stderr, "dllm: cuTensorMapEncodeTiled(4D) failed (CUresult %d)\n", (int)r);
  return r == CUDA_SUCCESS ? 0 : DLLM_ERR_TMAP;
}

size_t conv3x3_splitk_workspace(int Nimg, int H, int W, int Cin, int Cout) {
  const int M = Nimg * H * W;
  return plan_split(M, Cout, 9 * Cin).ws_bytes;
}
int conv3x3_nhwc(const void* x, const void* w, void* y, int Nimg, int H, int W, int Cin, int Cout, const void* bias,
                 const void* rowbias, const void* residual, cudaStream_t stream) {
  return conv3x3_nhwc_ws(x, w, y, Nimg, H, W, Cin, Cout, bias, rowbias, residual, nullptr, 0, stream);
}
// y[n,h,w,:] = conv3x3(x, w) + bias + rowbias[n] (+ residual);  x NHWC [Nimg,H,W,Cin], w [Cout, 3,3,Cin] (K-major), y NHWC.
// With a workspace of conv3x3_splitk_workspace() bytes small planes run split-K (see plan_split).
int conv3x3_nhwc_ws(const void* x, const void* w, void* y, int Nimg, int H, int W, int Cin, int Cout, const void* bias,
                    const void* rowbias, const void* residual, void* ws, size_t ws_bytes, cudaStream_t stream) {
  if (Nimg <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cin % 64 || Cout <= 0 || Cout % 8) return DLLM_ERR_SHAPE;
  if (W > 128 ? (W % 128) : (128 % W)) return DLLM_ERR_SHAPE;
  if (reinterpret_cast<uintptr_t>(y) & 1) return DLLM_ERR_ALIGN;
  const int HW = H * W;
  int Wb = W > 128 ? 128 : W, Hb = W > 128 ? 1 : 128 / W, Nb = 1;
  if (Hb > H) {  // small planes: the 128-pixel tile spans several whole images
    if (Hb % H) return DLLM_ERR_SHAPE;
    Nb = Hb / H;
    Hb = H;
  } else if (H % Hb) {
    return DLLM_ERR_SHAPE;
  }
  const int M = Nimg * HW, K = 9 * Cin;
  const SplitPlan sp = plan_split(M, Cout, K);
  const bool split = sp.ksplit > 1 && ws && ws_bytes >= sp.ws_bytes && !(reinterpret_cast<uintptr_t>(ws) & 15) &&
                     !(reinterpret_cast<uintptr_t>(y) & 15);
  const int bn = split ? sp.bn : plan_bn(M, Cout, 0, 0, true);
  CUtensorMap ta, tb;
  int rc;
  if ((rc = make_tmap_nhwc(&ta, x, Nimg, H, W, Cin, Wb, Hb, Nb))) return rc;
  if ((rc = make_tmap_2d(&tb, w, 2, Cout, K, K, bn, BK))) return rc;
  GemmEpi epi{static_cast<const bf16*>(bias), static_cast<const bf16*>(residual), Cout, 0, static_cast<const bf16*>(rowbias), HW};
  ConvGeom cg{Cin / 64, W, H, HW};
  if (split) {
    GemmEpi none{nullptr, nullptr, 0, 0, nullptr, 1};
    rc = (bn == 128) ? launch_gemm_bn<false, false, float, true, 0, 128>(ta, tb, ws, Cout, M, Cout, K, none, stream, cg, sp.ksplit)
                     : launch_gemm_bn<false, false, float, true, 0, 256>(ta, tb, ws, Cout, M, Cout, K, none, stream, cg, sp.ksplit);
    if (rc) return rc;
    return launch_splitk_reduce(ws, y, Cout, M, Cout, sp, epi, stream);
  }
  const bool any_epi = bias || rowbias || residual;
  return any_epi ? launch_gemm<false, false, bf16, true, 1>(ta, tb, y, Cout, M, Cout, K, epi, stream, cg, bn)
                 : launch_gemm<false, false, bf16, true, 0>(ta, tb, y, Cout, M, Cout, K, epi, stream, cg, bn);
}

}  // namespace dllm
