// wgmma flash attention, softmax(Q K^T / 8) V per head (head_dim 64), for the 2-byte formats FMT:
//   ANYLOC_PAIR_F16  : q, k, v are fp16 pairs (hi, lo) of 8*x in the row-major qkv buffer [B*T, 3D] (q | k | v thirds,
//                      written by the qkv GEMM's split epilogue); both products are 3-term
//                      X.Y ~= X_hi.Y_hi + X_lo.Y_hi + X_hi.Y_lo; output fp16 pairs of 8*o.
//   ANYLOC_PAIR_BF16 : q, k, v are one bf16 array bf16_rn(x); one term per product, P rounded once to bf16; one bf16
//                      output.
//   ANYLOC_PAIR_F16X1: q, k, v are one fp16 array, the hi half of the fp16 pairs of 8*x; one term per product, the
//                      pairs' scales (1/64 in the logit scale, P = 1024 p rounded once to its hi half); output the hi of
//                      8*o.
//   ANYLOC_PAIR_BF16X3: q, k, v are bf16 pairs (hi, lo) of x, no scale; both products 3-term as for the fp16 pairs, P
//                      (unscaled) split into bf16 pairs; output bf16 pairs of o.
// The arithmetic is that of the mma.sync kernel it replaced (attention_tc.cu keeps it for tf32 pairs): P = 1024 p split
// into fp16 pairs, 1/kActScale^2 and log2(e) folded into the logit scale, ex2.approx, and each 64-key block's P.V
// accumulated from zero by the tensor core and then added to the running output with round-to-nearest fp32 adds.
//
// CTA = (128-query tile, head, image), three warpgroups:
//   warpgroup 0   : producer -- one thread issues TMA loads (3-D tensor maps over (columns, rows, image), 64 x 64 boxes,
//                   128B swizzle): Q (hi, lo) of all 128 rows once, then K and V blocks of 64 keys (hi, lo) through a
//                   STAGES-deep full / empty mbarrier ring shared by both consumers.  Gives its registers away
//                   (setmaxnreg).
//   warpgroups 1-2: consumers -- each owns 64 query rows.  S = Q K^T is wgmma m64n64k16 SS (Q and K K-major); the S
//                   accumulator is the register A fragment of P.V, wgmma m64n64k16 RS with V as the transposed
//                   (MN-major) B operand.  Block j+1's S wgmmas are issued before block j's softmax, so the softmax
//                   runs under them, and the other consumer's MMAs fill the rest.  A consumer whose 64 rows all lie
//                   at or beyond T does nothing (the empty barriers count only the active consumers), so a tile count
//                   per image that is odd costs no padded MMAs.
// Keys at or beyond T read zeros (past the image in the 3-D map) or the next image's rows (the packed map) and are
// masked to p = 0 exactly; in the packed kernel the consumers also zero those V rows of the last key block before P.V,
// so a non-finite row of another image cannot reach O_j.  Query rows at or beyond T are computed and never written.
#include <stdlib.h>
#include "tc_common.cuh"

namespace anyloc {
namespace awg {

using namespace tc;

__device__ __forceinline__ float ex2(float x) {
  float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y;
}

constexpr int BQ = 128, BKV = 64, HD = 64, THREADS = 384, STAGES = 4;
constexpr int TILE_BYTES = 64 * 128;            // one 64-row x 64-column (128 B) box

template <int FMT> struct Cfg {
  static constexpr int NT = Fmt<FMT>::LO ? 2 : 1;   // arrays per operand: (hi, lo), or one
  static constexpr int Q_BYTES = NT * 2 * TILE_BYTES;                   // 128 rows
  static constexpr int K_OFF = 0, V_OFF = NT * TILE_BYTES;              // inside a stage; lo at + TILE_BYTES
  static constexpr int STAGE_BYTES = 2 * NT * TILE_BYTES;
  static constexpr int BAR_OFF = Q_BYTES + STAGES * STAGE_BYTES;
  static constexpr int SMEM_BYTES = BAR_OFF + 256 + 1024 /*align*/;
};

template <int FMT, bool VARLEN>
__device__ __forceinline__ void attention_wg_cta(const CUtensorMap* tm_hi, const CUtensorMap* tm_lo, int T, int D,
                                                 void* __restrict__ o_hi_, void* __restrict__ o_lo_,
                                                 const VarlenAttnTable* tab) {
  using C = Cfg<FMT>;
  using F = Fmt<FMT>;
  constexpr bool PAIRS = F::LO;                 // three terms per product
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + C::BAR_OFF);    // [STAGES]
  uint64_t* empty_bar = full_bar + STAGES;                                // [STAGES]
  uint64_t* q_bar = empty_bar + STAGES;

  int qt = blockIdx.x;
  const int h = blockIdx.y;
  int img = blockIdx.z, row0 = 0;               // map coordinates: (column, row0 + row, img)
  size_t out0 = (size_t)blockIdx.z * T;         // first output row of the image
  if constexpr (VARLEN) {
    int lo = 0, hi = tab->n - 1;                // the last entry with tile0 <= qt
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (tab->tile0[mid] <= qt) lo = mid; else hi = mid - 1;
    }
    qt -= tab->tile0[lo]; T = tab->len[lo]; row0 = tab->row0[lo]; img = 0; out0 = (size_t)row0;
  }
  const int nblk = (T + BKV - 1) / BKV;
  const int active = min(2, (T - qt * BQ + 63) / 64);      // consumers with at least one row below T
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(tm_hi) : "memory");
    for (int s = 0; s < STAGES; ++s) { mbar_init(smem_u32(full_bar + s), 1); mbar_init(smem_u32(empty_bar + s), active); }
    mbar_init(smem_u32(q_bar), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------------------------ TMA producer
    setmaxnreg_dec<24>();
    if (threadIdx.x == 0) {
      const uint32_t qb = smem_u32(q_bar);
      mbar_expect_tx(qb, C::Q_BYTES);
      for (int a = 0; a < C::NT; ++a)
        for (int r = 0; r < 2; ++r)
          tma_load_3d(smem_u32(smem + (2 * a + r) * TILE_BYTES), a ? tm_lo : tm_hi, qb, h * HD,
                      row0 + qt * BQ + 64 * r, img);
      for (int j = 0; j < nblk; ++j) {
        const int stage = j % STAGES;
        mbar_wait(smem_u32(empty_bar + stage), ((j / STAGES) & 1) ^ 1);
        const uint32_t fb = smem_u32(full_bar + stage);
        mbar_expect_tx(fb, C::STAGE_BYTES);
        const uint32_t sb = smem_u32(smem + C::Q_BYTES + stage * C::STAGE_BYTES);
        for (int a = 0; a < C::NT; ++a) {
          tma_load_3d(sb + C::K_OFF + a * TILE_BYTES, a ? tm_lo : tm_hi, fb, D + h * HD, row0 + j * BKV, img);
          tma_load_3d(sb + C::V_OFF + a * TILE_BYTES, a ? tm_lo : tm_hi, fb, 2 * D + h * HD, row0 + j * BKV, img);
        }
      }
    }
    return;
  }

  // ---------------------------------------- consumers: query rows [64 cw, +64) of the tile
  setmaxnreg_inc<240>();
  const int cw = wg - 1;
  if (qt * BQ + cw * 64 >= T) return;           // no rows below T: not counted by the empty barriers
  const int t = threadIdx.x & 127, warp = t >> 5, lane = t & 31, g = lane >> 2, t4 = lane & 3;
  constexpr bool SCALED = F::SCALED;            // fp16 operands carry s = kActScale and P is scaled into fp16's range
  const float P_SCALE = SCALED ? 1024.0f : 1.0f;
  // S holds (s q).(s k), s = kActScale for fp16 pairs: fold 1/s^2 into the 1/sqrt(64) * log2(e) scale
  const float kScale = 0.125f * 1.4426950408889634f * (SCALED ? 1.0f / (kActScale * kActScale) : 1.0f);
  // The scaled logit of a live key.  fp16 operands cannot overflow the fp32 sum (|S| < 64 * 65504^2), so an infinite S
  // means an operand overflowed fp16.  A key whose operand is +-Inf against a query of the opposite sign gives
  // S = -Inf (single fp16 has no lo term to meet it; the pairs' lo term may have the same sign), and the softmax would
  // drop that key with p = 0 while every output stays finite.  s * 0 turns such an S into NaN, which reaches the
  // outputs and the fp16-range guard; for finite s it is a zero of s's sign, so the sum is s * kScale bit for bit.
  auto logit = [&](float s) {
    if constexpr (SCALED) return fmaf(s, kScale, s * 0.0f);
    else return s * kScale;
  };

  const uint32_t q_base = smem_u32(smem) + cw * TILE_BYTES;
  const uint64_t dq_hi = make_desc(q_base), dq_lo = make_desc(q_base + 2 * TILE_BYTES);
  auto stage_addr = [&](int j) { return smem_u32(smem + C::Q_BYTES + (j % STAGES) * C::STAGE_BYTES); };

  // S = Q K^T (3-term; bf16 and single fp16: one term) of block j into s, committed as one wgmma group
  auto issue_s = [&](float* s, int j) {
    const uint32_t sb = stage_addr(j);
    const uint64_t dk_hi = make_desc(sb + C::K_OFF), dk_lo = make_desc(sb + C::K_OFF + TILE_BYTES);
    fence_regs<32>(s);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint64_t adv = (uint64_t)((k * 32) >> 4);          // +32 B per k16 step inside the 128 B row
      wgmma_m64n64_ss<FMT>(s, dq_hi + adv, dk_hi + adv, k != 0 ? 1u : 0u);
      if constexpr (PAIRS) {
        wgmma_m64n64_ss<FMT>(s, dq_lo + adv, dk_hi + adv, 1u);
        wgmma_m64n64_ss<FMT>(s, dq_hi + adv, dk_lo + adv, 1u);
      }
    }
    wgmma_commit();
    fence_regs<32>(s);
  };

  float o[32];                 // [4 nd + c]: rows g / g+8 (c >= 2) of this warp's 16, dims 8 nd + 2 t4 + (c & 1)
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

  // one key block: S of block j is complete in sc; S of block j + 1 goes into sn under this block's softmax
  auto block = [&](float* sc, float* sn, int j) {
    if (j + 1 < nblk) {
      mbar_wait(smem_u32(full_bar + (j + 1) % STAGES), ((j + 1) / STAGES) & 1);
      issue_s(sn, j + 1);
    }
    // ---- online softmax (rows g and g+8; a row's 64 keys are spread over the 4 threads of a quad)
    float p[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) p[i] = sc[i];
    float mx0 = m0, mx1 = m1;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int key = j * BKV + nt * 8 + 2 * t4;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const bool live = key + e < T;
        p[4 * nt + e] = live ? logit(p[4 * nt + e]) : -INFINITY;
        p[4 * nt + 2 + e] = live ? logit(p[4 * nt + 2 + e]) : -INFINITY;
        mx0 = fmaxf(mx0, p[4 * nt + e]); mx1 = fmaxf(mx1, p[4 * nt + 2 + e]);
      }
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float alpha0 = ex2(m0 - mx0), alpha1 = ex2(m1 - mx1);
    m0 = mx0; m1 = mx1;
    float r0 = 0.f, r1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      p[4 * nt + 0] = ex2(p[4 * nt + 0] - mx0); p[4 * nt + 1] = ex2(p[4 * nt + 1] - mx0);
      p[4 * nt + 2] = ex2(p[4 * nt + 2] - mx1); p[4 * nt + 3] = ex2(p[4 * nt + 3] - mx1);
      r0 += p[4 * nt + 0] + p[4 * nt + 1]; r1 += p[4 * nt + 2] + p[4 * nt + 3];
    }
    l0 = l0 * alpha0 + r0; l1 = l1 * alpha1 + r1;

    // ---- P as the A fragments of P.V: k16 step ks = S column groups 2ks, 2ks + 1
    uint32_t ph[4][4], pl[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        F::pack2(p[8 * ks + 2 * i] * P_SCALE, p[8 * ks + 2 * i + 1] * P_SCALE, ph[ks][i], pl[ks][i]);
      }
    }
    // ---- O_j = P V (3-term), accumulated from zero, then o = alpha o + O_j (round-to-nearest)
    const uint32_t sb = stage_addr(j);
    if constexpr (VARLEN) {
      // The last key block of a packed image ends inside the stage, and its V rows from T on are the next image's
      // (or whatever lies between images): p = 0 there, but 0 * Inf or NaN would still reach O_j.  The active
      // consumers zero those rows (a 128 B swizzled row stays within its own 128 B), as the padded kernel reads them.
      const int rem = T - j * BKV;                      // keys of this block below T
      if (rem < BKV) {
        const int pieces = (BKV - rem) * 8;             // 16 B pieces per V tile
        for (int i = cw * 128 + t; i < C::NT * pieces; i += active * 128) {
          const int a = i / pieces, r = rem + (i % pieces) / 8;
          asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(sb + C::V_OFF + a * TILE_BYTES + r * 128 +
                                                                          (i % 8) * 16), "r"(0u) : "memory");
        }
        fence_proxy_async_smem();                       // before P.V's wgmma reads them
        named_bar_sync<1>(active * 128);
      }
    }
    const uint64_t dv_hi = make_desc_mn(sb + C::V_OFF), dv_lo = make_desc_mn(sb + C::V_OFF + TILE_BYTES);
    float pv[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) pv[i] = 0.f;
    fence_regs<32>(pv);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const uint64_t adv = (uint64_t)((ks * 2048) >> 4);       // 16 keys = two 8-row atoms
      wgmma_m64n64_rs_tb<FMT>(pv, ph[ks], dv_hi + adv, ks != 0 ? 1u : 0u);
      if constexpr (PAIRS) {
        wgmma_m64n64_rs_tb<FMT>(pv, pl[ks], dv_hi + adv, 1u);
        wgmma_m64n64_rs_tb<FMT>(pv, ph[ks], dv_lo + adv, 1u);
      }
    }
    wgmma_commit();
    fence_regs<32>(pv);
    wgmma_wait<0>();           // S of block j + 1 and O_j
    fence_regs<32>(pv);
    fence_regs<32>(sn);
    if (t == 0) mbar_arrive(smem_u32(empty_bar + j % STAGES));   // K_j and V_j are no longer read
#pragma unroll
    for (int nd = 0; nd < 8; ++nd) {
      o[4 * nd + 0] = o[4 * nd + 0] * alpha0 + pv[4 * nd + 0]; o[4 * nd + 1] = o[4 * nd + 1] * alpha0 + pv[4 * nd + 1];
      o[4 * nd + 2] = o[4 * nd + 2] * alpha1 + pv[4 * nd + 2]; o[4 * nd + 3] = o[4 * nd + 3] * alpha1 + pv[4 * nd + 3];
    }
  };

  float sa[32], sb[32];
  mbar_wait(smem_u32(q_bar), 0);
  mbar_wait(smem_u32(full_bar), 0);
  issue_s(sa, 0);
  wgmma_wait<0>();
  fence_regs<32>(sa);
  for (int j = 0; j < nblk; j += 2) {
    block(sa, sb, j);
    if (j + 1 < nblk) block(sb, sa, j + 1);
  }

  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  // o holds (P_SCALE p) . (s v) and fp16 outputs are pairs of s*o, so only P_SCALE and the softmax denominator remain
  const float inv0 = 1.0f / (l0 * P_SCALE), inv1 = 1.0f / (l1 * P_SCALE);
  const int q0 = qt * BQ + cw * 64 + warp * 16 + g;
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int q = q0 + 8 * half;
    if (q >= T) continue;
    const float inv = half ? inv1 : inv0;
    const size_t off = (out0 + q) * (size_t)D + (size_t)h * HD + 2 * t4;
#pragma unroll
    for (int nd = 0; nd < 8; ++nd) {
      uint32_t hh, ll;           // o is already scaled: the words of the values as they are
      F::pack2(o[4 * nd + 2 * half] * inv, o[4 * nd + 2 * half + 1] * inv, hh, ll);
      *reinterpret_cast<uint32_t*>(reinterpret_cast<typename F::T*>(o_hi_) + off + nd * 8) = hh;
      if constexpr (F::LO) *reinterpret_cast<uint32_t*>(reinterpret_cast<typename F::T*>(o_lo_) + off + nd * 8) = ll;
    }
  }
}

// B images of T tokens each: grid (128-query tiles, heads, B); maps over (3D columns, T rows, B images)
template <int FMT>
__global__ void __launch_bounds__(THREADS, 1)
attention_wg_kernel(const __grid_constant__ CUtensorMap tm_hi, const __grid_constant__ CUtensorMap tm_lo, int T, int D,
                    void* __restrict__ o_hi, void* __restrict__ o_lo) {
  attention_wg_cta<FMT, false>(&tm_hi, &tm_lo, T, D, o_hi, o_lo, nullptr);
}

// Images of different lengths packed row after row: grid (sum of every image's 128-query tiles, heads); maps over
// (3D columns, all packed rows, 1).  The host lists the images longest first, so the CTAs with the longest key loops
// start first and short images fill the tail.
template <int FMT>
__global__ void __launch_bounds__(THREADS, 1)
attention_wg_varlen_kernel(const __grid_constant__ CUtensorMap tm_hi, const __grid_constant__ CUtensorMap tm_lo,
                           const __grid_constant__ VarlenAttnTable tab, int D, void* __restrict__ o_hi,
                           void* __restrict__ o_lo) {
  attention_wg_cta<FMT, true>(&tm_hi, &tm_lo, 0, D, o_hi, o_lo, &tab);
}

// Launches the padded (tab == nullptr: B images of T tokens) or the packed kernel of fmt over the maps of qkv_{hi,lo}
static int launch(const void* qkv_hi, const void* qkv_lo, int imgs, int rows, int T, const VarlenAttnTable* tab,
                  dim3 grid, int D, void* o_hi, void* o_lo, int fmt, cudaStream_t st) {
  CUtensorMap m_hi, m_lo;
  int rc;
  if ((rc = tc::make_map_3d16(&m_hi, qkv_hi, imgs, rows, 3 * D, 64, fmt))) return rc;
  if ((rc = tc::make_map_3d16(&m_lo, format_info(fmt).lo ? qkv_lo : qkv_hi, imgs, rows, 3 * D, 64, fmt))) return rc;
  return fmt_switch(fmt, [&](auto c) {
    constexpr int FMT = decltype(c)::value;
    if constexpr (sizeof(typename Fmt<FMT>::T) != 2) {
      set_error("attention_wg: format %d is not a 2-byte format", fmt);
      return (int)ANYLOC_ERR_ARG;
    } else {
      static unsigned long long seen = 0;
      if (first_use_on_this_device(&seen)) {
        ANYLOC_CHECK_CUDA(cudaFuncSetAttribute(attention_wg_kernel<FMT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               Cfg<FMT>::SMEM_BYTES));
        ANYLOC_CHECK_CUDA(cudaFuncSetAttribute(attention_wg_varlen_kernel<FMT>,
                                               cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<FMT>::SMEM_BYTES));
      }
      if (tab)
        attention_wg_varlen_kernel<FMT><<<grid, THREADS, Cfg<FMT>::SMEM_BYTES, st>>>(m_hi, m_lo, *tab, D, o_hi, o_lo);
      else
        attention_wg_kernel<FMT><<<grid, THREADS, Cfg<FMT>::SMEM_BYTES, st>>>(m_hi, m_lo, T, D, o_hi, o_lo);
      ANYLOC_CHECK_LAUNCH();
      return (int)ANYLOC_OK;
    }
  });
}

}  // namespace awg

// qkv_{hi,lo}: [B*T, 3D] in the format fmt: fp16 pairs of 8*x (ANYLOC_PAIR_F16), bf16 pairs of x (_BF16X3), or one
// array (qkv_lo and o_lo unused) of bf16 (_BF16) or of the hi halves of those fp16 pairs (_F16X1); o_{hi,lo}: [B*T, D]
// of the same kind.
// 16-byte aligned (the caller checks).
int attention_wg_launch(const void* qkv_hi, const void* qkv_lo, int B, int T, int D, int heads, void* o_hi, void* o_lo,
                        int fmt, cudaStream_t st) {
  using namespace awg;
  return launch(qkv_hi, qkv_lo, B, T, T, nullptr, dim3(cdiv(T, BQ), heads, B), D, o_hi, o_lo, fmt, st);
}

// the same over images of different lengths packed into one [rows, 3D] qkv buffer, rows = the end of the last image;
// tab lists them with their first 64-query tiles, which become 128-query tiles here (same order)
int attention_wg_varlen_launch(const void* qkv_hi, const void* qkv_lo, const VarlenAttnTable& tab, int D, int heads,
                               void* o_hi, void* o_lo, int fmt, cudaStream_t st) {
  using namespace awg;
  VarlenAttnTable t = tab;
  int tiles = 0, rows = 0;
  for (int k = 0; k < t.n; ++k) {
    t.tile0[k] = tiles;
    tiles += cdiv(t.len[k], BQ);
    if (t.row0[k] + t.len[k] > rows) rows = t.row0[k] + t.len[k];
  }
  return launch(qkv_hi, qkv_lo, 1, rows, 0, &t, dim3(tiles, heads), D, o_hi, o_lo, fmt, st);
}

}  // namespace anyloc
