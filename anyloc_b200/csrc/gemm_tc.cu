// wgmma GEMM engine:  C[M,N] = (A_hi+A_lo)[M,K] . (B_hi+B_lo)[N,K]^T  + fused epilogue,
// fp32-equivalent accuracy through the 3-term split
//      A.B ~= A_hi.B_hi + A_lo.B_hi + A_hi.B_lo
// where (hi, lo) are tf32 pairs (two fp32 words, consumed as tf32), fp16 pairs of s*x or bf16 pairs of x (not
// fp32-equivalent: about 16 significant bits), materialised by the producer kernels (LayerNorm / previous epilogue /
// weight prep).
//
// Structure (one persistent CTA per SM, 3 warpgroups = 384 threads, CTA tile 128 x 128):
//   warpgroup 0 : TMA producer -- one thread streams cp.async.bulk.tensor 2D, 128B-swizzled K-major boxes of 128 bytes
//                 of K ({A_hi, A_lo, B_hi, B_lo} per stage) into a ring guarded by full / empty mbarriers.
//   warpgroups 1-2 : consumers -- each owns 64 rows x 128 columns: wgmma.mma_async m64n128 (k16 fp16 / k8 tf32) straight
//                 from shared memory into registers.  The tensor core's fp32 accumulation is not round-to-nearest, a
//                 bias that grows with K, so the wgmmas only accumulate a CHUNK of k-blocks; each chunk is then added
//                 (round-to-nearest) into a second register accumulator that holds the whole 64 x 128 sub-tile.  After
//                 the last chunk: bias / GELU / SwiGLU / LayerScale+residual / pair split, staged in shared memory
//                 subtile by subtile and stored with TMA (epilogue_staged), so the stores drain behind the next
//                 tile's mainloop.  The hi-only coarse passes, and outputs TMA cannot store, are stored from registers.
// The single formats (formats.cuh) run one wgmma per k-step through the same pipeline with hi-only stages and the staged
// epilogue, a third of the 3-term MMAs, not fp32-equivalent: single bf16 (ANYLOC_PAIR_BF16), single fp16
// (ANYLOC_PAIR_F16X1, the hi array of the fp16 pairs alone), and single e4m3 (ANYLOC_PAIR_FP8: A = e4m3 rows with one
// power-of-two scale per row, B = one e4m3 matrix; 128-element k-blocks on UINT8 tensor maps, the accumulator of row m
// multiplied by A's row scale before the epilogue).  Their SPLIT outputs are one array in Fmt<FMT>::OUT.
// Tiles are rastered in bands of BAND_N column blocks, n-fastest inside a band: the resident CTAs share a few A row
// panels and one band of B that stays in L2 while the outputs stream through.
#include <cuda.h>
#include <stdlib.h>
#include "epilogue.cuh"
#include "tc_common.cuh"

namespace anyloc {

namespace tc {

constexpr int BM = 128, BN = 128;
constexpr int KSTEPS = 4;                  // wgmma k-steps per 128-byte k-block (32 B each: 8 tf32 or 16 fp16)
constexpr int A_BYTES = BM * 128;          // 16 KB: 128 rows x 128 B
constexpr int B_BYTES = BN * 128;          // 16 KB
constexpr int THREADS = 384;
constexpr int STG_BYTES = 8192;            // one epilogue staging buffer (see epilogue_staged)

// LO = true : stages hold {A_hi, A_lo, B_hi, B_lo} (3-term split, 64 KB).  LO = false: hi-only single pass (coarse
// scores): {A_hi, B_hi} = 32 KB per stage -> twice the pipeline depth in the same shared memory.
// LOM (lo operands present): bit 0 = A_lo, bit 1 = B_lo; a compile-time mask keeps the wgmma sequence branch-free.
// STG: the staged epilogue is compiled in -- the 3-term passes and the single formats (hi-only, so 6 stages of 32 KB
// plus 4 x 8 KB staging = 231 424 B of H100's 232 448 B opt-in), not the hi-only coarse passes (below).
template <bool LO, bool STG = LO> struct Cfg {
  static constexpr int STAGE_BYTES = (LO ? 2 : 1) * (A_BYTES + B_BYTES);
  static constexpr int B_OFF = (LO ? 2 : 1) * A_BYTES;
  static constexpr int STAGES = LO ? 3 : 6;
  static constexpr int BAR_OFF = STAGES * STAGE_BYTES;          // mbarriers (< 256 B)
  static constexpr int SMEM_BYTES = BAR_OFF + 256 + 1024 /*align*/;
  // epilogue staging buffers (2 per consumer warpgroup), 3-term passes only.  The hi-only coarse passes keep the
  // register epilogue, a small share of their time: with the staged path compiled in, their mainloop ran slower
  // (H100, retrieval coarse pass with the epilogue discarded: 2.46 -> 2.65 ms).  A launch that does not stage asks
  // for SMEM_BYTES only, the staged ones for SMEM_BYTES_STAGED.
  static constexpr bool STAGED = STG;
  static constexpr int STG_OFF = BAR_OFF + 1024;
  static constexpr int SMEM_BYTES_STAGED = STG_OFF + 4 * STG_BYTES + 1024 /*align*/;
};
constexpr int BAND_N = 16;                 // column blocks per raster band
constexpr int CHUNK_KB_TF32 = 2;          // k-blocks accumulated by the tensor core between two round-to-nearest adds
constexpr int CHUNK_KB_F16 = 8;            // (24 / 96 wgmma k-steps per chunk)
// The single-bf16 pass keeps the round-to-nearest chunks of the fp16 pairs (CHUNK_KB_F16: 32 wgmmas per chunk).  Its
// second 64-register accumulator fits without spills (ptxas -v), the chunk add is 64 FADDs per thread per 32 wgmmas,
// and it keeps the accumulation term of the error (c u sqrt(K) |A||B|, u = 2^-24) that of the f16x3 GEMMs, so the
// operands' own bf16 rounding (2^-8 relative) is the only new error term.  The bf16 pairs (ANYLOC_PAIR_BF16X3) take the
// same chunks with the fp16 pairs' 96 wgmmas each, so their error over the fp16 pairs' is that of the operands' split.
constexpr int CHUNK_KB_COARSE = 32;        // hi-only fp16 coarse pass (retrieval): <= 128 k-steps per chunk, the bound
                                           // topk.cu re-scores against
// The e4m3 pass promotes the tensor core's partial sums into the round-to-nearest fp32 accumulator every k-block (128
// elements, 4 wgmmas): the fp8 wgmma is not known to accumulate in full fp32 (DESIGN §4.9 states what was measured).
constexpr int CHUNK_KB_FP8 = 1;

__device__ __forceinline__ void tile_coords(int tile, int num_m, int num_n, int band_n, int& m_blk, int& n_blk) {
  const int per_band = num_m * band_n;
  const int band = tile / per_band, r = tile - band * per_band;
  const int w = min(band_n, num_n - band * band_n);       // width of this (possibly last, narrower) band
  m_blk = r / w;
  n_blk = band * band_n + (r - m_blk * w);
}

// SPLIT outputs of elements o, o + 1 (o even) in the format OUT; and as epi_store_split chooses it
template <int OUT>
__device__ __forceinline__ void split_put2(const EpiParams& ep, size_t o, float a, float b) {
  typedef typename Fmt<OUT>::T T;
  put2<OUT>(reinterpret_cast<T*>(ep.out), reinterpret_cast<T*>(ep.out_lo), o, a, b);
}
template <int FMT = ANYLOC_PAIR_TF32>
__device__ __forceinline__ void store_split2(const EpiParams& ep, size_t o, float a, float b) {
  if constexpr (fixed_out<FMT>()) split_put2<Fmt<FMT>::OUT>(ep, o, a, b);
  else if (ep.out_fmt != ANYLOC_PAIR_TF32) split_put2<ANYLOC_PAIR_F16>(ep, o, a, b);
  else split_put2<ANYLOC_PAIR_TF32>(ep, o, a, b);
}

// epilogue of two adjacent accumulator columns (n even, n+1) of row m
template <int FMT = ANYLOC_PAIR_TF32>
__device__ __forceinline__ void epi_pair(const EpiParams& ep, int m, int n, int N, float v0, float v1) {
  const int mode = ep.mode;
  if (mode < 0) return;                    // diagnostic: discard (ANYLOC_GEMM_DEBUG_SKIP_EPI)
  if (mode == ANYLOC_EPI_SWIGLU_SPLIT) {   // (x1_j, x2_j) = columns (2j, 2j+1); N is even
    epi_store_pair<FMT>(ep, m, n, v0, v1);
    return;
  }
  if (n + 1 >= N || (ep.ldo & 1)) {
    epi_store1<FMT>(ep, m, n, v0);
    if (n + 1 < N) epi_store1<FMT>(ep, m, n + 1, v1);
    return;
  }
  const float al = ep.alpha;
  float2 b = make_float2(0.f, 0.f);
  if (ep.bias) b = __ldg(reinterpret_cast<const float2*>(ep.bias + n));
  const float x0 = v0 * al + b.x, x1 = v1 * al + b.y;
  const size_t o = (size_t)m * ep.ldo + n;
  if (mode == ANYLOC_EPI_BIAS) {
    *reinterpret_cast<float2*>(ep.out + o) = make_float2(x0, x1);
  } else if (mode == ANYLOC_EPI_LS_RESID) {
    const float2 g = __ldg(reinterpret_cast<const float2*>(ep.gamma + n));
    const float2 r = *reinterpret_cast<const float2*>(ep.resid + o);
    *reinterpret_cast<float2*>(ep.out + o) = make_float2(r.x + g.x * x0, r.y + g.y * x1);
  } else if (mode == ANYLOC_EPI_GELU_SPLIT) {
    store_split2<FMT>(ep, o, gelu_erf(x0), gelu_erf(x1));
  } else {                                 // BIAS_SPLIT
    store_split2<FMT>(ep, o, x0, x1);
  }
}

// Register epilogue of the 3-term passes that do not stage (gated launches, outputs TMA cannot store: see
// make_epi_maps) of one consumer thread's part of a 64 x 128 sub-tile: rows r0 and r0 + 8, column pairs nq + 8j (j < 16), accumulators in the wgmma layout,
// applied and stored pair by pair.
template <int FMT = ANYLOC_PAIR_TF32>
__device__ __forceinline__ void epilogue_pairs(const EpiParams& ep, int r0, int nq, int M, int N, const float* sum) {
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int n = nq + j * 8;
    if (n >= N) continue;
    if (r0 < M) epi_pair<FMT>(ep, r0, n, N, sum[4 * j], sum[4 * j + 1]);
    if (r0 + 8 < M) epi_pair<FMT>(ep, r0 + 8, n, N, sum[4 * j + 2], sum[4 * j + 3]);
  }
}

// Register epilogue of the hi-only passes (the VLAD and retrieval coarse scores): where every column pair of the tile
// lies inside N (and, except for SwiGLU, ldo is even), the bias / gamma / residual loads of 2 column pairs (both rows)
// are issued together ahead of their stores -- 8 memory round trips per thread and tile instead of 32 -- otherwise
// pair by pair.  Same values, same arithmetic as epilogue_pairs.  (Groups of 4 or 8 pairs spill.)
__device__ __forceinline__ void epilogue_regs_batched(const EpiParams& ep, int r0, int nq, int M, int N, const float* sum) {
  const int mode = ep.mode;
  if (mode < 0) return;                    // diagnostic: discard (ANYLOC_GEMM_DEBUG_SKIP_EPI)
  const int n0 = nq & ~(BN - 1);
  const bool swiglu = mode == ANYLOC_EPI_SWIGLU_SPLIT, resid = mode == ANYLOC_EPI_LS_RESID;
  if (n0 + BN > N || (!swiglu && (ep.ldo & 1))) {
    epilogue_pairs(ep, r0, nq, M, N, sum);
    return;
  }
  const bool row0 = r0 < M, row1 = r0 + 8 < M;
  const size_t o0 = (size_t)r0 * ep.ldo, o1 = (size_t)(r0 + 8) * ep.ldo;
  const float al = ep.alpha;
#pragma unroll
  for (int j0 = 0; j0 < 16; j0 += 2) {
    float2 b[2], g[2], ra[2], rb[2];
#pragma unroll
    for (int jj = 0; jj < 2; ++jj) {
      const int n = nq + (j0 + jj) * 8;
      b[jj] = ep.bias ? __ldg(reinterpret_cast<const float2*>(ep.bias + n)) : make_float2(0.f, 0.f);
      if (resid) {
        g[jj] = __ldg(reinterpret_cast<const float2*>(ep.gamma + n));
        if (row0) ra[jj] = *reinterpret_cast<const float2*>(ep.resid + o0 + n);
        if (row1) rb[jj] = *reinterpret_cast<const float2*>(ep.resid + o1 + n);
      }
    }
#pragma unroll
    for (int jj = 0; jj < 2; ++jj) {
      const int j = j0 + jj, n = nq + j * 8;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!(h ? row1 : row0)) continue;
        const float v0 = sum[4 * j + 2 * h], v1 = sum[4 * j + 2 * h + 1];
        const size_t ro = h ? o1 : o0;
        if (swiglu) {                      // (x1_j, x2_j) = columns (n, n+1) -> column n/2
          const float x1 = v0 * al + b[jj].x, x2 = v1 * al + b[jj].y;
          epi_store_split(ep, ro + (n >> 1), silu(x1) * x2);
          continue;
        }
        const float x0 = v0 * al + b[jj].x, x1 = v1 * al + b[jj].y;
        const size_t o = ro + n;
        if (mode == ANYLOC_EPI_BIAS) {
          *reinterpret_cast<float2*>(ep.out + o) = make_float2(x0, x1);
        } else if (resid) {
          const float2 r = h ? rb[jj] : ra[jj];
          *reinterpret_cast<float2*>(ep.out + o) = make_float2(r.x + g[jj].x * x0, r.y + g[jj].y * x1);
        } else if (mode == ANYLOC_EPI_GELU_SPLIT) {
          store_split2(ep, o, gelu_erf(x0), gelu_erf(x1));
        } else {                           // BIAS_SPLIT
          store_split2(ep, o, x0, x1);
        }
      }
    }
  }
}

// ------------------------------------------------------------------ staged epilogue
// Output formats of the staged path: the SPLIT output format OUT (ANYLOC_PAIR_*), or OUT_F32 (BIAS / LS_RESID).  A
// subtile is 64 rows x COLS output columns; one 8 KB staging buffer holds it: 64 x 32 fp32, the hi and lo halves (4 KB
// each) of 64 x 32 fp16 or 64 x 16 fp32 pairs, or 64 x 64 single bf16 or single fp16.
constexpr int OUT_F32 = -1;
constexpr int STG_HALF = STG_BYTES / 2;    // offset of the lo array (pair formats)
constexpr int STG_ROWS = 64;               // TMA box rows of the output maps: one consumer warpgroup's rows

template <int OUT> constexpr bool stage_lo() {
  if constexpr (OUT == OUT_F32) return false;
  else return Fmt<OUT>::LO;
}
template <int OUT> constexpr int stage_esz() {
  if constexpr (OUT == OUT_F32) return 4;
  else return (int)sizeof(typename Fmt<OUT>::T);
}
template <int OUT>
struct StageFmt {
  static constexpr bool LO = stage_lo<OUT>();                        // a lo array in the buffer's second half
  static constexpr int ESZ = stage_esz<OUT>();
  static constexpr int ROW_BYTES = STG_BYTES / STG_ROWS / (LO ? 2 : 1);   // 128 or 64 bytes per row of one array
  static constexpr int COLS = ROW_BYTES / ESZ;                       // output columns per subtile
  static constexpr uint32_t SWZ = ROW_BYTES == 128 ? 7 : 3;          // TMA SWIZZLE_128B / SWIZZLE_64B
};

// Byte offset of byte b of staging row `row`, placed as TMA's SWIZZLE_128B / _64B expects it: the 16-byte chunk index
// XOR offset bits 7.. .  The 8 rows that one warp's store instruction covers land in distinct banks.
template <int OUT>
__device__ __forceinline__ uint32_t stg_off(int row, int b) {
  const uint32_t o = (uint32_t)(row * StageFmt<OUT>::ROW_BYTES + b);
  return o ^ (((o >> 7) & StageFmt<OUT>::SWZ) << 4);
}

// bias / gamma of columns (n, n+1); columns at or past N (which TMA clips) read nothing
__device__ __forceinline__ float2 ldg_col_pair(const float* p, int n, int N) {
  if (n + 1 < N) return __ldg(reinterpret_cast<const float2*>(p + n));
  return make_float2(n < N ? __ldg(p + n) : 0.f, 0.f);
}

// TMA load of the residual subtile (64 rows from m0, 32 fp32 columns from oc) into a staging buffer
__device__ __forceinline__ void resid_load(const CUtensorMap* tm, uint8_t* buf, uint64_t* bar, int oc, int m0) {
  mbar_expect_tx(smem_u32(bar), STG_BYTES);
  tma_load_2d(smem_u32(buf), tm, smem_u32(bar), oc, m0);
}

// Staged epilogue of one consumer warpgroup's 64 x 128 sub-tile (rows from m0, accumulator columns from n0), one
// subtile at a time: every thread applies the epilogue to its accumulators of the subtile and writes the results into
// the warpgroup's staging buffer -- for LS_RESID the buffer already holds the TMA-loaded residual and is updated in
// place -- then, after a proxy fence and the warpgroup's named barrier, one thread stores the buffer with TMA, which
// clips the M and N tails.  The stores drain while the warpgroup works on the next subtile and the next tile's
// mainloop.  Two buffers alternate (running subtile count `cnt`); a buffer is rewritten only once the store issued
// from it has read it (waited before the barrier of the subtile in between).  Same arithmetic as epi_pair.
template <int OUT, bool SWIGLU, bool RESID>
__device__ __forceinline__ void epilogue_staged(const EpiParams& ep, const CUtensorMap* tm_out, const CUtensorMap* tm_lo,
                                                const CUtensorMap* tm_resid, uint8_t* stg, uint64_t* rbar,
                                                uint32_t& rphase, uint32_t& cnt, int wg, int t, int m0, int n0, int N,
                                                const float* sum) {
  using F = StageFmt<OUT>;
  constexpr int ACC = SWIGLU ? 2 * F::COLS : F::COLS;    // accumulator columns per subtile
  constexpr int JS = ACC / 8;                             // 8-column accumulator groups per subtile
  const int lane = t & 31, q = lane & 3, row = (t >> 5) * 16 + (lane >> 2);
  const int n_out = SWIGLU ? N >> 1 : N;
  const int oc_base = SWIGLU ? n0 >> 1 : n0;
  const bool gelu = ep.mode == ANYLOC_EPI_GELU_SPLIT;
  const float al = ep.alpha;
#pragma unroll
  for (int s = 0; s < BN / ACC; ++s) {
    const int oc0 = oc_base + s * F::COLS;
    if (oc0 >= n_out) break;
    const uint32_t b = cnt & 1;
    uint8_t* buf = stg + b * STG_BYTES;
    if (RESID) { mbar_wait(smem_u32(rbar + b), (rphase >> b) & 1); rphase ^= 1u << b; }
#pragma unroll
    for (int jj = 0; jj < JS; ++jj) {
      const int j = s * JS + jj, n = n0 + j * 8 + 2 * q;
      const float2 bb = ep.bias ? ldg_col_pair(ep.bias, n, N) : make_float2(0.f, 0.f);
      float2 g;
      if (RESID) g = ldg_col_pair(ep.gamma, n, N);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = row + 8 * h;
        const float x0 = sum[4 * j + 2 * h] * al + bb.x, x1 = sum[4 * j + 2 * h + 1] * al + bb.y;
        if constexpr (SWIGLU) {            // (x1_j, x2_j) = columns (n, n+1) -> output column n/2
          typedef typename Fmt<OUT>::T E;
          const float v = silu(x0) * x1;
          const uint32_t o = stg_off<OUT>(r, (4 * jj + q) * F::ESZ);
          E hi, lo;
          Fmt<OUT>::split1(v, hi, lo);
          *reinterpret_cast<E*>(buf + o) = hi;
          if constexpr (F::LO) *reinterpret_cast<E*>(buf + STG_HALF + o) = lo;
          continue;
        }
        const uint32_t o = stg_off<OUT>(r, (8 * jj + 2 * q) * F::ESZ);
        if constexpr (OUT == OUT_F32) {
          float2* p = reinterpret_cast<float2*>(buf + o);
          if (RESID) {
            const float2 rr = *p;
            *p = make_float2(rr.x + g.x * x0, rr.y + g.y * x1);
          } else {
            *p = make_float2(x0, x1);
          }
        } else {
          typedef typename Fmt<OUT>::W2 W;
          const float y0 = gelu ? gelu_erf(x0) : x0, y1 = gelu ? gelu_erf(x1) : x1;
          W hi, lo;
          Fmt<OUT>::split2(y0, y1, hi, lo);
          *reinterpret_cast<W*>(buf + o) = hi;
          if constexpr (F::LO) *reinterpret_cast<W*>(buf + STG_HALF + o) = lo;
        }
      }
    }
    fence_proxy_async_smem();
    if (t == 0) bulk_wait_read<0>();       // the previous subtile's store has read the other buffer: free after the barrier
    if (wg == 1) named_bar_sync<1>(128);    // the warpgroup's own barrier (0 is __syncthreads')
    else named_bar_sync<2>(128);
    if (t == 0) {
      tma_store_2d(tm_out, smem_u32(buf), oc0, m0);
      if (F::LO) tma_store_2d(tm_lo, smem_u32(buf + STG_HALF), oc0, m0);
      bulk_commit();
      if (RESID && s + 2 < BN / ACC && oc0 + 2 * F::COLS < n_out) {
        // residual of subtile s + 2 into this buffer, once the store has read it
        bulk_wait_read<0>();
        resid_load(tm_resid, buf, rbar + b, oc0 + 2 * F::COLS, m0);
      }
    }
    ++cnt;
  }
}

// FMT: the operand format (ANYLOC_PAIR_*); every k-block is 128 bytes of K: 32 tf32, 64 fp16 or bf16, 128 e4m3
// elements.  LOM != 0 (lo operands) for the pair formats only.  The single formats run one wgmma per k-step and write
// their SPLIT outputs in Fmt<FMT>::OUT; single e4m3 takes A's row scales in ep.row_scale.
// ep.gate (nullable): the kernel returns at once when *gate == 0 (conditional fallbacks without a host sync).
// staged != 0: the epilogue goes through shared memory and TMA stores (tm_out, tm_out_lo for the pair formats,
// tm_resid for LS_RESID: (n_out, M) maps with 64-row boxes); 0: stored pair by pair from registers.
template <int FMT, int LOM>
__global__ void __launch_bounds__(THREADS, 1)
gemm_tc3_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                const __grid_constant__ CUtensorMap tm_b_hi, const __grid_constant__ CUtensorMap tm_b_lo,
                const __grid_constant__ CUtensorMap tm_out, const __grid_constant__ CUtensorMap tm_out_lo,
                const __grid_constant__ CUtensorMap tm_resid, int staged,
                int M, int N, int K, int band_n, int chunk_kb, EpiParams ep) {
  constexpr bool LO = LOM != 0, has_a_lo = (LOM & 1) != 0, has_b_lo = (LOM & 2) != 0;
  static_assert(LOM == 0 || Fmt<FMT>::LO, "lo operands belong to the pair formats");
  using C = Cfg<LO, LO || !Fmt<FMT>::LO>;
  if (ep.gate != nullptr && *reinterpret_cast<const volatile int*>(ep.gate) == 0) return;   // uniform over the grid
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + C::BAR_OFF);                    // [STAGES]
  uint64_t* empty_bar = full_bar + C::STAGES;                                             // [STAGES]
  uint64_t* resid_bar = empty_bar + C::STAGES;                   // [2 per consumer warpgroup]: residual subtile landed

  const int wg = threadIdx.x >> 7;
  const int num_m = (M + BM - 1) / BM, num_n = (N + BN - 1) / BN;
  const int num_tiles = num_m * num_n;
  constexpr int BKE = 128 / (int)sizeof(typename Fmt<FMT>::T);   // elements per k-block (128 bytes)
  const int num_k = (K + BKE - 1) / BKE;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_a_hi) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_b_hi) : "memory");
    for (int s = 0; s < C::STAGES; ++s) { mbar_init(smem_u32(full_bar + s), 1); mbar_init(smem_u32(empty_bar + s), 2); }
    if (C::STAGED)
      for (int i = 0; i < 4; ++i) mbar_init(smem_u32(resid_bar + i), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    if (threadIdx.x == 0) {
      // ------------------------------------------------ TMA producer
      const uint32_t tx_bytes = A_BYTES * (1 + ((LO && has_a_lo) ? 1 : 0)) + B_BYTES * (1 + ((LO && has_b_lo) ? 1 : 0));
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int mb, nb; tile_coords(tile, num_m, num_n, band_n, mb, nb);
        const int m0 = mb * BM, n0 = nb * BN;
        for (int kb = 0; kb < num_k; ++kb) {
          mbar_wait(smem_u32(empty_bar + stage), phase ^ 1);
          const uint32_t fb = smem_u32(full_bar + stage);
          mbar_expect_tx(fb, tx_bytes);
          const uint32_t sbase = smem_u32(smem + stage * C::STAGE_BYTES);
          tma_load_2d(sbase, &tm_a_hi, fb, kb * BKE, m0);
          if (LO && has_a_lo) tma_load_2d(sbase + A_BYTES, &tm_a_lo, fb, kb * BKE, m0);
          tma_load_2d(sbase + C::B_OFF, &tm_b_hi, fb, kb * BKE, n0);
          if (LO && has_b_lo) tma_load_2d(sbase + C::B_OFF + B_BYTES, &tm_b_lo, fb, kb * BKE, n0);
          if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ---------------------------------------- consumers: rows [64 (wg-1), +64) of the tile
  const int t = threadIdx.x & 127, warp = t >> 5, lane = t & 31;
  const uint32_t a_sub = (uint32_t)(wg - 1) * 64 * 128;       // byte offset of this warpgroup's 64 A rows
  uint8_t* stg = smem + C::STG_OFF + (wg - 1) * 2 * STG_BYTES;  // this warpgroup's two staging buffers
  uint64_t* rbar = resid_bar + (wg - 1) * 2;
  const int mode = ep.mode;
  staged = C::STAGED && staged;
  const bool resid_staged = staged && mode == ANYLOC_EPI_LS_RESID;
  uint32_t stg_cnt = 0, rphase = 0;                           // staged subtiles so far; resid_bar parities
  int stage = 0; uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    int mb, nb; tile_coords(tile, num_m, num_n, band_n, mb, nb);
    const int m0 = mb * BM + (wg - 1) * 64, n0 = nb * BN;
    float sum[64], acc[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) { sum[j] = 0.f; acc[j] = 0.f; }
    int prev_stage = -1;
    for (int kb0 = 0; kb0 < num_k; kb0 += chunk_kb) {
      const int kb1 = min(num_k, kb0 + chunk_kb);
      if (resid_staged && kb1 == num_k && t == 0 && m0 < M) {
        // the last chunk starts: fetch the residual of the first two subtiles into the staging buffers, which the
        // previous tile's stores have finished reading by now
        bulk_wait_read<0>();
        for (int i = 0; i < 2; ++i) {
          const uint32_t b = (stg_cnt + i) & 1;
          const int oc = n0 + i * StageFmt<OUT_F32>::COLS;
          if (oc < N) resid_load(&tm_resid, stg + b * STG_BYTES, rbar + b, oc, m0);
        }
      }
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(smem_u32(full_bar + stage), phase);
        const uint32_t sbase = smem_u32(smem + stage * C::STAGE_BYTES);
        const uint64_t a_hi = make_desc(sbase + a_sub), a_lo = make_desc(sbase + A_BYTES + a_sub);
        const uint64_t b_hi = make_desc(sbase + C::B_OFF), b_lo = make_desc(sbase + C::B_OFF + B_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < KSTEPS; ++k) {
          const uint64_t adv = (uint64_t)((k * 32) >> 4);      // +32 B per k-step inside the atom (both types)
          wgmma_m64n128<FMT>(acc, a_hi + adv, b_hi + adv, (kb != kb0 || k != 0) ? 1u : 0u);
          if (has_a_lo) wgmma_m64n128<FMT>(acc, a_lo + adv, b_hi + adv, 1u);
          if (has_b_lo) wgmma_m64n128<FMT>(acc, a_hi + adv, b_lo + adv, 1u);
        }
        wgmma_commit();
        // the previous k-block's wgmmas have retired once at most this one is in flight: free its stage
        wgmma_wait<1>();
        if (prev_stage >= 0 && t == 0) mbar_arrive(smem_u32(empty_bar + prev_stage));
        prev_stage = stage;
        if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
      }
      // end of a chunk: add the tensor core's partial sums with round-to-nearest fp32 adds
      wgmma_wait<0>();
      fence_regs<64>(acc);
#pragma unroll
      for (int j = 0; j < 64; ++j) sum[j] += acc[j];
    }
    if (t == 0) mbar_arrive(smem_u32(empty_bar + prev_stage));
    if (mode < 0 || m0 >= M) continue;       // discard (ANYLOC_GEMM_DEBUG_SKIP_EPI) / no rows for this warpgroup
    if constexpr (FMT == ANYLOC_PAIR_FP8) {  // dequantise A: row m's sums times its power-of-two scale (exact)
      const int r = m0 + warp * 16 + (lane >> 2);
      const float s0 = r < M ? __ldg(ep.row_scale + r) : 0.f, s1 = r + 8 < M ? __ldg(ep.row_scale + r + 8) : 0.f;
#pragma unroll
      for (int j = 0; j < 16; ++j) { sum[4 * j] *= s0; sum[4 * j + 1] *= s0; sum[4 * j + 2] *= s1; sum[4 * j + 3] *= s1; }
    }
    if constexpr (!C::STAGED) {
      epilogue_regs_batched(ep, m0 + warp * 16 + (lane >> 2), n0 + 2 * (lane & 3), M, N, sum);
      continue;
    }
    if (!staged) {
      epilogue_pairs<FMT>(ep, m0 + warp * 16 + (lane >> 2), n0 + 2 * (lane & 3), M, N, sum);
      continue;
    }
#define ANYLOC_EPI_STAGED(OUT_, SWIGLU_, RESID_)                                                                    \
  epilogue_staged<OUT_, SWIGLU_, RESID_>(ep, &tm_out, &tm_out_lo, &tm_resid, stg, rbar, rphase, stg_cnt, wg, t, m0,  \
                                         n0, N, sum)
    if (mode == ANYLOC_EPI_BIAS) ANYLOC_EPI_STAGED(OUT_F32, false, false);
    else if (mode == ANYLOC_EPI_LS_RESID) ANYLOC_EPI_STAGED(OUT_F32, false, true);
    else if constexpr (fixed_out<FMT>()) {   // BIAS_SPLIT / GELU_SPLIT / SWIGLU_SPLIT -> the format's own output
      if (mode == ANYLOC_EPI_SWIGLU_SPLIT) ANYLOC_EPI_STAGED(Fmt<FMT>::OUT, true, false);
      else ANYLOC_EPI_STAGED(Fmt<FMT>::OUT, false, false);
    } else if (mode == ANYLOC_EPI_SWIGLU_SPLIT) {    // -> tf32 or fp16 pairs, as ep.out_fmt says
      if (ep.out_fmt != ANYLOC_PAIR_TF32) ANYLOC_EPI_STAGED(ANYLOC_PAIR_F16, true, false);
      else ANYLOC_EPI_STAGED(ANYLOC_PAIR_TF32, true, false);
    } else {                                 // BIAS_SPLIT / GELU_SPLIT
      if (ep.out_fmt != ANYLOC_PAIR_TF32) ANYLOC_EPI_STAGED(ANYLOC_PAIR_F16, false, false);
      else ANYLOC_EPI_STAGED(ANYLOC_PAIR_TF32, false, false);
    }
#undef ANYLOC_EPI_STAGED
  }
  if (staged && t == 0) bulk_wait<0>();     // the last stores complete before the CTA exits
}

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return nullptr;
    fn = (EncodeTiledFn)p;
  }
  return fn;
}

// tensor-map element type of fmt's arrays (the tf32 pairs' are fp32 words)
static CUtensorMapDataType map_dtype(int fmt) {
  switch (fmt) {
    case ANYLOC_PAIR_FP8: return CU_TENSOR_MAP_DATA_TYPE_UINT8;
    case ANYLOC_PAIR_BF16: case ANYLOC_PAIR_BF16X3: return CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    case ANYLOC_PAIR_F16: case ANYLOC_PAIR_F16X1: return CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    default: return CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  }
}

int make_map(CUtensorMap* map, const void* ptr, int rows, int K, int ld, int box_rows, int fmt) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { set_error("gemm_tc: cuTensorMapEncodeTiled unavailable"); return ANYLOC_ERR_CUDA; }
  const int esz = format_info(fmt).esz;
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * esz};
  cuuint32_t box[2] = {(cuuint32_t)(128 / esz), (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, map_dtype(fmt), 2, (void*)ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("gemm_tc: cuTensorMapEncodeTiled failed (%d) rows=%d K=%d ld=%d", (int)r, rows, K, ld); return ANYLOC_ERR_CUDA; }
  return ANYLOC_OK;
}

int make_map_3d16(CUtensorMap* map, const void* ptr, int imgs, int rows, int cols, int box_rows, int fmt) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { set_error("tensor map: cuTensorMapEncodeTiled unavailable"); return ANYLOC_ERR_CUDA; }
  cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)imgs};
  cuuint64_t strides[2] = {(cuuint64_t)cols * 2, (cuuint64_t)rows * cols * 2};
  cuuint32_t box[3] = {64, (cuuint32_t)box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, map_dtype(fmt), 3, (void*)ptr, dims,
                   strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("tensor map: cuTensorMapEncodeTiled failed (%d) imgs=%d rows=%d cols=%d", (int)r, imgs, rows, cols); return ANYLOC_ERR_CUDA; }
  return ANYLOC_OK;
}

// output map of the staged epilogue: [rows, cols] of fmt's elements (ANYLOC_PAIR_TF32: fp32), row pitch ld, boxes of
// 64 rows x box_cols swizzled as stg_off places them.  TMA clips the boxes at rows and cols, so the ld padding is never
// written.
static int make_out_map(CUtensorMap* map, const void* ptr, int rows, int cols, int ld, int fmt, int box_cols) {
  const int esz = format_info(fmt).esz;
  EncodeTiledFn enc = get_encode();
  if (!enc) { set_error("gemm_tc: cuTensorMapEncodeTiled unavailable"); return ANYLOC_ERR_CUDA; }
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * esz};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)STG_ROWS};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, map_dtype(fmt), 2, (void*)ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   box_cols * esz == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("gemm_tc: cuTensorMapEncodeTiled failed (%d) for the output: rows=%d cols=%d ld=%d", (int)r, rows, cols, ld); return ANYLOC_ERR_CUDA; }
  return ANYLOC_OK;
}

// Output maps of the staged epilogue.  *staged = false (maps zeroed) where the result is discarded or TMA cannot
// store the output: row pitch or row length not a multiple of 16 bytes (the start addresses are 16-byte aligned by
// gemm_tc_supported).  The row-length condition is conservative: in one H100 run of the staged-path test without it,
// a 68-column fp16 output (136 bytes per row) came back with its ldo padding columns 68..71 written, as if the store
// clipped columns only to 16-byte units.  Not reproduced since (the condition keeps such shapes off the staged path).
// out: the SPLIT output format (ANYLOC_PAIR_*).
static int make_epi_maps(const EpiParams& ep, int out, int M, int N, CUtensorMap* m_out, CUtensorMap* m_lo,
                         CUtensorMap* m_resid, bool* staged) {
  memset(m_out, 0, sizeof(*m_out)); memset(m_lo, 0, sizeof(*m_lo)); memset(m_resid, 0, sizeof(*m_resid));
  const bool split = ep.mode == ANYLOC_EPI_BIAS_SPLIT || ep.mode == ANYLOC_EPI_GELU_SPLIT ||
                     ep.mode == ANYLOC_EPI_SWIGLU_SPLIT;
  const int fmt = split ? out : ANYLOC_PAIR_TF32;      // BIAS / LS_RESID: fp32
  const FormatInfo& f = format_info(fmt);
  const int esz = f.esz;
  const int n_out = ep.mode == ANYLOC_EPI_SWIGLU_SPLIT ? N / 2 : N;
  *staged = ep.mode >= 0 && ((long long)ep.ldo * esz) % 16 == 0 && ((long long)n_out * esz) % 16 == 0;
  if (!*staged) return ANYLOC_OK;
  const bool lo = split && f.lo;
  const int cols = STG_BYTES / STG_ROWS / (lo ? 2 : 1) / esz;     // StageFmt<out or OUT_F32>::COLS
  int rc;
  if ((rc = make_out_map(m_out, ep.out, M, n_out, ep.ldo, fmt, cols))) return rc;
  if (lo && (rc = make_out_map(m_lo, ep.out_lo, M, n_out, ep.ldo, fmt, cols))) return rc;
  if (ep.mode == ANYLOC_EPI_LS_RESID && (rc = make_out_map(m_resid, ep.resid, M, n_out, ep.ldo, fmt, cols))) return rc;
  return ANYLOC_OK;
}

}  // namespace tc

bool gemm_tc_supported(const void* a_hi, const void* a_lo, int lda, const void* b_hi, const void* b_lo, int ldb,
                       int M, int N, int K, const EpiParams& ep, int fmt) {
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  const int q = 16 / format_info(fmt).esz;   // elements per 16 bytes
  if (M < 1 || N < 1 || K < q) return false;
  if ((K % q) || (lda % q) || (ldb % q)) return false;
  if (!al16(a_hi) || !al16(b_hi) || (a_lo && !al16(a_lo)) || (b_lo && !al16(b_lo))) return false;
  if (!al16(ep.out) || (ep.out_lo && !al16(ep.out_lo)) || (ep.resid && !al16(ep.resid))) return false;
  if (ep.bias && !al16(ep.bias)) return false;
  if (ep.gamma && !al16(ep.gamma)) return false;
  return true;
}

// epilogue of this host thread's last launch (anyloc_gemm_tc_last_staged)
static thread_local int g_last_staged = -1;

template <int FMT, int LOM>
static int launch_impl(const void* a_hi, const void* a_lo, int lda, const void* b_hi, const void* b_lo, int ldb, int M,
                       int N, int K, const EpiParams& ep, int chunk, cudaStream_t st) {
  using namespace tc;
  constexpr bool LO = LOM != 0;
  using CF = Cfg<LO, LO || !Fmt<FMT>::LO>;
  static_assert(CF::SMEM_BYTES_STAGED <= 232448, "GEMM over H100's shared-memory opt-in");
  CUtensorMap ma_hi, ma_lo, mb_hi, mb_lo;
  int rc;
  if ((rc = make_map(&ma_hi, a_hi, M, K, lda, BM, FMT))) return rc;
  if ((rc = make_map(&ma_lo, a_lo ? a_lo : a_hi, M, K, lda, BM, FMT))) return rc;
  if ((rc = make_map(&mb_hi, b_hi, N, K, ldb, BN, FMT))) return rc;
  if ((rc = make_map(&mb_lo, b_lo ? b_lo : b_hi, N, K, ldb, BN, FMT))) return rc;
  CUtensorMap mo, mo_lo, mr;
  bool staged = false;
  memset(&mo, 0, sizeof(mo)); memset(&mo_lo, 0, sizeof(mo_lo)); memset(&mr, 0, sizeof(mr));
  // A gated launch is a conditional fallback that usually returns at once: it keeps the register epilogue, so it
  // encodes no output maps and asks for the same shared memory as the coarse pass it follows (a launch that asked
  // for more would make the SM switch its shared-memory configuration back and forth).
  const int out = fixed_out<FMT>() ? Fmt<FMT>::OUT : (ep.out_fmt != ANYLOC_PAIR_TF32 ? ANYLOC_PAIR_F16 : ANYLOC_PAIR_TF32);
  if (CF::STAGED && ep.gate == nullptr && (rc = make_epi_maps(ep, out, M, N, &mo, &mo_lo, &mr, &staged))) return rc;
  const int smem = staged ? CF::SMEM_BYTES_STAGED : CF::SMEM_BYTES;
  g_last_staged = staged ? 1 : 0;
  static unsigned long long attr_seen = 0;
  if (first_use_on_this_device(&attr_seen)) {
    ANYLOC_CHECK_CUDA(cudaFuncSetAttribute(gemm_tc3_kernel<FMT, LOM>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           CF::STAGED ? CF::SMEM_BYTES_STAGED : CF::SMEM_BYTES));
  }
  const int tiles = cdiv(M, BM) * cdiv(N, BN);
  const int grid = std::min(tiles, device_sm_count());
  gemm_tc3_kernel<FMT, LOM><<<grid, THREADS, smem, st>>>(
      ma_hi, ma_lo, mb_hi, mb_lo, mo, mo_lo, mr, staged ? 1 : 0, M, N, K, std::min(BAND_N, cdiv(N, BN)), chunk, ep);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}

// ANYLOC_GEMM_CHUNK: k-blocks per round-to-nearest chunk of the 3-term and e4m3 GEMMs (A/B knob; 0 = default)
static int gemm_chunk_env() {
  static int chunk_env = -1;
  if (chunk_env < 0) { const char* e = getenv("ANYLOC_GEMM_CHUNK"); chunk_env = e ? atoi(e) : 0; }
  return chunk_env;
}

// C = A . B^T + epilogue of fmt operands.  The tf32 and fp16 pairs take lo operands (a_lo, b_lo nullable), the bf16
// pairs both of them (the caller checks); the single formats take none, except single e4m3, whose a_lo holds A's fp32
// row scales [M].  The bf16 pairs run the fp16 pairs' 3-term pipeline with the bf16 wgmma and their chunks.  The single bf16 and fp16 GEMMs accumulate
// in the fp16 pairs' round-to-nearest chunks (CHUNK_KB_F16), single e4m3 promotes every CHUNK_KB_FP8 k-blocks.  The
// single formats have their own instantiations, so the hi-only coarse passes (<F16 | TF32, 0>) keep their register
// epilogue and shared memory.
int gemm_tc_launch(const void* a_hi, const void* a_lo, int lda, const void* b_hi, const void* b_lo, int ldb, int M,
                   int N, int K, const EpiParams& ep_in, int fmt, cudaStream_t st) {
  const int chunk_env = gemm_chunk_env();
  EpiParams ep = ep_in;
  switch (fmt) {
    case ANYLOC_PAIR_BF16:
      return launch_impl<ANYLOC_PAIR_BF16, 0>(a_hi, nullptr, lda, b_hi, nullptr, ldb, M, N, K, ep, tc::CHUNK_KB_F16, st);
    case ANYLOC_PAIR_F16X1:
      return launch_impl<ANYLOC_PAIR_F16X1, 0>(a_hi, nullptr, lda, b_hi, nullptr, ldb, M, N, K, ep, tc::CHUNK_KB_F16,
                                               st);
    case ANYLOC_PAIR_FP8:
      ep.row_scale = static_cast<const float*>(a_lo);
      return launch_impl<ANYLOC_PAIR_FP8, 0>(a_hi, nullptr, lda, b_hi, nullptr, ldb, M, N, K, ep,
                                             chunk_env > 0 ? chunk_env : tc::CHUNK_KB_FP8, st);
    default: break;
  }
  // diagnostic only (tools/, never set by the product): bit m set -> GEMMs with epilogue mode m discard their result,
  // which exposes how much of a GEMM's time is its epilogue
  static int skip_epi = -1;
  if (skip_epi < 0) { const char* e = getenv("ANYLOC_GEMM_DEBUG_SKIP_EPI"); skip_epi = e ? atoi(e) : 0; }
  if (skip_epi && ((skip_epi >> ep_in.mode) & 1)) ep.mode = -1;
  if (fmt == ANYLOC_PAIR_BF16X3)
    return launch_impl<ANYLOC_PAIR_BF16X3, 3>(a_hi, a_lo, lda, b_hi, b_lo, ldb, M, N, K, ep,
                                              chunk_env > 0 ? chunk_env : tc::CHUNK_KB_F16, st);
  const bool f16 = fmt == ANYLOC_PAIR_F16;
  const int lom = (a_lo ? 1 : 0) | (b_lo ? 2 : 0);
  // hi-only fp16 pass = the retrieval's coarse scores, whose error bound allows long chunks
  const int chunk = lom == 0 ? (f16 ? tc::CHUNK_KB_COARSE : tc::CHUNK_KB_TF32)
                             : chunk_env > 0 ? chunk_env : (f16 ? tc::CHUNK_KB_F16 : tc::CHUNK_KB_TF32);
#define ANYLOC_GEMM_LAUNCH(FMT_, LOM_) launch_impl<FMT_, LOM_>(a_hi, a_lo, lda, b_hi, b_lo, ldb, M, N, K, ep, chunk, st)
  switch (lom + (f16 ? 4 : 0)) {
    case 0: return ANYLOC_GEMM_LAUNCH(ANYLOC_PAIR_TF32, 0);
    case 1: return ANYLOC_GEMM_LAUNCH(ANYLOC_PAIR_TF32, 1);
    case 2: return ANYLOC_GEMM_LAUNCH(ANYLOC_PAIR_TF32, 2);
    case 3: return ANYLOC_GEMM_LAUNCH(ANYLOC_PAIR_TF32, 3);
    case 4: return ANYLOC_GEMM_LAUNCH(ANYLOC_PAIR_F16, 0);
    case 5: return ANYLOC_GEMM_LAUNCH(ANYLOC_PAIR_F16, 1);
    case 6: return ANYLOC_GEMM_LAUNCH(ANYLOC_PAIR_F16, 2);
    default: return ANYLOC_GEMM_LAUNCH(ANYLOC_PAIR_F16, 3);
  }
#undef ANYLOC_GEMM_LAUNCH
}

}  // namespace anyloc

extern "C" int anyloc_gemm_tc_last_staged(void) { return anyloc::g_last_staged; }
