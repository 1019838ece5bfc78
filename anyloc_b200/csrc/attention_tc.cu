// Tensor-core flash attention, softmax(Q K^T / 8) V per head (head_dim 64), tf32 pairs: q, k, v are tf32 pairs (two
// fp32 arrays) in the row-major qkv buffer [B*T, 3D] (q | k | v thirds); mma.sync m16n8k8 (tf32); output tf32 pairs.
// Both GEMMs use the 3-term split  X.Y ~= X_hi.Y_hi + X_lo.Y_hi + X_hi.Y_lo  (fp32-equivalent accuracy), and each key
// block's P.V partial is accumulated from zero and then added to the running output with round-to-nearest fp32 adds.
// The 2-byte formats (fp16 pairs, single bf16, single fp16) run the wgmma kernel of attention_wg.cu instead: wgmma's
// transposed B operand, which P.V needs for V, exists for 16-bit types only.
//
// CTA = (64-query tile, head, image), 4 warps; warp w owns query rows [16w, 16w+16) of the tile and keeps its Q
// fragments (hi, lo) in registers for the whole key loop.  K and V blocks of 64 keys (hi and lo) are streamed through a
// double-buffered shared-memory ring with cp.async (rows beyond T are zero-filled and masked to -inf in S).  The S
// accumulator fragments are exactly the A-operand fragments of P.V (the key order inside a k8 step is permuted to match
// and V is read in the same order), so P never leaves registers.
#include <stdlib.h>
#include "common.cuh"

namespace anyloc {
namespace atc {

constexpr int BQ = 64, BKV = 64, HD = 64, WARPS = 4, THREADS = WARPS * 32;

struct Cfg {
  using T = float;
  static constexpr int PITCH = HD + 4;                                 // elements per smem row (bank-conflict-free reads)
  static constexpr int MAT = BKV * PITCH;                              // elements of one [64 keys x 64 dims] tile
  static constexpr int NMAT = 4;                                       // K_hi, K_lo, V_hi, V_lo
  static constexpr int STAGE = NMAT * MAT;
  static constexpr int SMEM_BYTES = 2 * STAGE * (int)sizeof(T);
  static constexpr int CHUNKS_PER_ROW = HD * (int)sizeof(T) / 16;     // 16-byte cp.async pieces per 64-dim row
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void mma_tf32(float* d, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ float ex2(float x) {
  float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y;
}
__device__ __forceinline__ uint32_t f2u(float x) { return __float_as_uint(x); }

// One CTA's work.  Uniform (VARLEN = false): blockIdx = (query tile, head, image) over B images of T tokens.  VARLEN:
// blockIdx = (tile of the packed grid, head); the table gives the image's first row, its length T and its first tile.
template <bool VARLEN>
__device__ __forceinline__ void attention_cta(const void* __restrict__ qkv_hi_, const void* __restrict__ qkv_lo_, int T,
                                              int D, void* __restrict__ o_hi_, void* __restrict__ o_lo_,
                                              const VarlenAttnTable* tab) {
  using C = Cfg;
  using E = typename C::T;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  E* smem = reinterpret_cast<E*>(smem_raw);
  const E* qkv_hi = reinterpret_cast<const E*>(qkv_hi_);
  const E* qkv_lo = reinterpret_cast<const E*>(qkv_lo_);
  int qt = blockIdx.x;
  const int h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t4 = lane & 3;
  const size_t ld = 3 * (size_t)D;
  size_t img0 = (size_t)b * T;
  if constexpr (VARLEN) {
    int lo = 0, hi = tab->n - 1;          // the last entry with tile0 <= qt
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (tab->tile0[mid] <= qt) lo = mid; else hi = mid - 1;
    }
    qt -= tab->tile0[lo]; T = tab->len[lo]; img0 = (size_t)tab->row0[lo];
  }
  const int nblk = (T + BKV - 1) / BKV;
  const float kScale = 0.125f * 1.4426950408889634f;     // 1/sqrt(64) * log2(e)

  // ---- K/V block loader: 64 rows x {K_hi, K_lo, V_hi, V_lo}, 16-byte pieces, rows >= T zero-filled
  auto load_block = [&](int j, int buf) {
    E* st = smem + buf * C::STAGE;
    constexpr int PIECES = C::NMAT * BKV * C::CHUNKS_PER_ROW;
    for (int p = threadIdx.x; p < PIECES; p += THREADS) {
      const int mat = p / (BKV * C::CHUNKS_PER_ROW), r = (p / C::CHUNKS_PER_ROW) % BKV, c = p % C::CHUNKS_PER_ROW;
      const int key = j * BKV + r;
      const bool valid = key < T;
      const E* src = (mat & 1) ? qkv_lo : qkv_hi;
      const bool is_k = mat < 2;
      const size_t col = (size_t)(is_k ? D : 2 * D) + (size_t)h * HD + (size_t)c * (16 / sizeof(E));
      const E* gp = src + (valid ? (img0 + key) * ld + col : 0);
      cp_async16((uint32_t)__cvta_generic_to_shared(st + mat * C::MAT + r * C::PITCH + c * (16 / sizeof(E))), gp, valid);
    }
    cp_async_commit();
  };
  load_block(0, 0);

  // ---- Q fragments of this warp's 16 rows (hi, lo), zero beyond T
  const int q0 = qt * BQ + warp * 16 + g, q1 = q0 + 8;
  constexpr int QK_STEPS = HD / 8;
  uint32_t qa_hi[QK_STEPS][4], qa_lo[QK_STEPS][4];
  {
    const size_t r0 = (img0 + q0) * ld + (size_t)h * HD, r1 = (img0 + q1) * ld + (size_t)h * HD;
    const bool v0 = q0 < T, v1 = q1 < T;
#pragma unroll
    for (int ks = 0; ks < QK_STEPS; ++ks) {
      const int c0 = ks * 8 + t4, c1 = c0 + 4;
      qa_hi[ks][0] = v0 ? f2u(qkv_hi[r0 + c0]) : 0u; qa_hi[ks][1] = v1 ? f2u(qkv_hi[r1 + c0]) : 0u;
      qa_hi[ks][2] = v0 ? f2u(qkv_hi[r0 + c1]) : 0u; qa_hi[ks][3] = v1 ? f2u(qkv_hi[r1 + c1]) : 0u;
      qa_lo[ks][0] = v0 ? f2u(qkv_lo[r0 + c0]) : 0u; qa_lo[ks][1] = v1 ? f2u(qkv_lo[r1 + c0]) : 0u;
      qa_lo[ks][2] = v0 ? f2u(qkv_lo[r0 + c1]) : 0u; qa_lo[ks][3] = v1 ? f2u(qkv_lo[r1 + c1]) : 0u;
    }
  }

  float o[8][4];                 // [dim tile][c0..c3]: rows g / g+8, dims 8 nd + 2 t4 + {0,1}
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
#pragma unroll
  for (int nd = 0; nd < 8; ++nd) o[nd][0] = o[nd][1] = o[nd][2] = o[nd][3] = 0.f;

  for (int j = 0; j < nblk; ++j) {
    const int buf = j & 1;
    if (j + 1 < nblk) { load_block(j + 1, buf ^ 1); cp_async_wait<1>(); }
    else cp_async_wait<0>();
    __syncthreads();
    const E* sK_hi = smem + buf * C::STAGE;
    const E* sK_lo = sK_hi + C::MAT;
    const E* sV_hi = sK_hi + 2 * C::MAT;
    const E* sV_lo = sK_hi + 3 * C::MAT;

    // ---- S = Q K^T (3-term) for this warp's 16 rows x 64 keys
    float s[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float* kh = sK_hi + (nt * 8 + g) * C::PITCH;
      const float* kl = sK_lo + (nt * 8 + g) * C::PITCH;
#pragma unroll
      for (int ks = 0; ks < QK_STEPS; ++ks) {
        const uint32_t bh0 = f2u(kh[ks * 8 + t4]), bh1 = f2u(kh[ks * 8 + t4 + 4]);
        const uint32_t bl0 = f2u(kl[ks * 8 + t4]), bl1 = f2u(kl[ks * 8 + t4 + 4]);
        mma_tf32(s[nt], qa_hi[ks], bh0, bh1);
        mma_tf32(s[nt], qa_lo[ks], bh0, bh1);
        mma_tf32(s[nt], qa_hi[ks], bl0, bl1);
      }
    }

    // ---- online softmax (rows g and g+8; a row's 64 keys are spread over the 4 threads of a quad)
    float mx0 = m0, mx1 = m1;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int key = j * BKV + nt * 8 + 2 * t4;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const bool live = key + e < T;
        s[nt][e] = live ? s[nt][e] * kScale : -INFINITY;
        s[nt][2 + e] = live ? s[nt][2 + e] * kScale : -INFINITY;
        mx0 = fmaxf(mx0, s[nt][e]); mx1 = fmaxf(mx1, s[nt][2 + e]);
      }
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float alpha0 = ex2(m0 - mx0), alpha1 = ex2(m1 - mx1);
    m0 = mx0; m1 = mx1;
    float r0 = 0.f, r1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      s[nt][0] = ex2(s[nt][0] - mx0); s[nt][1] = ex2(s[nt][1] - mx0);
      s[nt][2] = ex2(s[nt][2] - mx1); s[nt][3] = ex2(s[nt][3] - mx1);
      r0 += s[nt][0] + s[nt][1]; r1 += s[nt][2] + s[nt][3];
    }
    l0 = l0 * alpha0 + r0; l1 = l1 * alpha1 + r1;

    // ---- O_j = P V (3-term), accumulated from zero, then o = alpha o + O_j (round-to-nearest)
    float pv[8][4];
#pragma unroll
    for (int nd = 0; nd < 8; ++nd) pv[nd][0] = pv[nd][1] = pv[nd][2] = pv[nd][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {          // 8 keys per step = S tile ks; A slot t4 <-> key 2 t4, slot t4+4 <-> 2 t4 + 1
      uint32_t ph[4], pl[4];
      float hh, ll;
      split_tf32(s[ks][0], hh, ll); ph[0] = f2u(hh); pl[0] = f2u(ll);
      split_tf32(s[ks][2], hh, ll); ph[1] = f2u(hh); pl[1] = f2u(ll);
      split_tf32(s[ks][1], hh, ll); ph[2] = f2u(hh); pl[2] = f2u(ll);
      split_tf32(s[ks][3], hh, ll); ph[3] = f2u(hh); pl[3] = f2u(ll);
      const float* vh0 = sV_hi + (ks * 8 + 2 * t4) * C::PITCH;
      const float* vl0 = sV_lo + (ks * 8 + 2 * t4) * C::PITCH;
#pragma unroll
      for (int nd = 0; nd < 8; ++nd) {
        const uint32_t bh0 = f2u(vh0[nd * 8 + g]), bh1 = f2u(vh0[C::PITCH + nd * 8 + g]);
        const uint32_t bl0 = f2u(vl0[nd * 8 + g]), bl1 = f2u(vl0[C::PITCH + nd * 8 + g]);
        mma_tf32(pv[nd], ph, bh0, bh1);
        mma_tf32(pv[nd], pl, bh0, bh1);
        mma_tf32(pv[nd], ph, bl0, bl1);
      }
    }
#pragma unroll
    for (int nd = 0; nd < 8; ++nd) {
      o[nd][0] = o[nd][0] * alpha0 + pv[nd][0]; o[nd][1] = o[nd][1] * alpha0 + pv[nd][1];
      o[nd][2] = o[nd][2] * alpha1 + pv[nd][2]; o[nd][3] = o[nd][3] * alpha1 + pv[nd][3];
    }
    __syncthreads();             // every warp is done with this buffer before it is refilled
  }

  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int q = half ? q1 : q0;
    if (q >= T) continue;
    const float inv = half ? inv1 : inv0;
    const size_t off = (img0 + q) * (size_t)D + (size_t)h * HD + 2 * t4;
#pragma unroll
    for (int nd = 0; nd < 8; ++nd) {
      const float a = o[nd][2 * half] * inv, c = o[nd][2 * half + 1] * inv;
      float2 hh, ll;
      split_tf32(a, hh.x, ll.x); split_tf32(c, hh.y, ll.y);
      *reinterpret_cast<float2*>(reinterpret_cast<float*>(o_hi_) + off + nd * 8) = hh;
      *reinterpret_cast<float2*>(reinterpret_cast<float*>(o_lo_) + off + nd * 8) = ll;
    }
  }
}

// B images of T tokens each: grid (query tiles, heads, B)
__global__ void __launch_bounds__(THREADS)
attention_tc_kernel(const void* __restrict__ qkv_hi_, const void* __restrict__ qkv_lo_, int T, int D,
                    void* __restrict__ o_hi_, void* __restrict__ o_lo_) {
  attention_cta<false>(qkv_hi_, qkv_lo_, T, D, o_hi_, o_lo_, nullptr);
}

// Images of different lengths packed row after row: grid (sum of every image's query tiles, heads).  The host lists
// the images longest first, so the CTAs with the longest key loops start first and short images fill the tail.
__global__ void __launch_bounds__(THREADS)
attention_tc_varlen_kernel(const void* __restrict__ qkv_hi_, const void* __restrict__ qkv_lo_,
                           const __grid_constant__ VarlenAttnTable tab, int D, void* __restrict__ o_hi_,
                           void* __restrict__ o_lo_) {
  attention_cta<true>(qkv_hi_, qkv_lo_, 0, D, o_hi_, o_lo_, &tab);
}

// fp32 (hi,lo) qkv pairs -> fp16 pairs of 8*x (same [M,3D] layout).  Standalone building-block path only.
__global__ void __launch_bounds__(256)
qkv_to_f16_kernel(const float* __restrict__ qkv_hi, const float* __restrict__ qkv_lo, size_t n, __half* __restrict__ q16_hi,
                  __half* __restrict__ q16_lo) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    __half hh, ll; split_f16((qkv_hi[i] + qkv_lo[i]) * kActScale, hh, ll);
    q16_hi[i] = hh; q16_lo[i] = ll;
  }
}

}  // namespace atc

int attention_wg_launch(const void* qkv_hi, const void* qkv_lo, int B, int T, int D, int heads, void* o_hi, void* o_lo,
                        int fmt, cudaStream_t st);
int attention_wg_varlen_launch(const void* qkv_hi, const void* qkv_lo, const VarlenAttnTable& tab, int D, int heads,
                               void* o_hi, void* o_lo, int fmt, cudaStream_t st);

// qkv_{hi,lo}: [B*T, 3D] in the format fmt (ANYLOC_PAIR_*: tf32 pairs, fp16 pairs of 8*x, bf16 pairs, or single bf16 or
// single fp16 with qkv_lo unused); o_{hi,lo}: [B*T, D] of the same kind (single formats: o_hi only).  The 2-byte formats
// run attention_wg.cu's kernel; the mma.sync kernel here takes the tf32 pairs only.
int attention_tc_launch(const void* qkv_hi, const void* qkv_lo, int B, int T, int D, int heads, void* o_hi, void* o_lo,
                        int fmt, cudaStream_t st) {
  using namespace atc;
  ANYLOC_REQUIRE(D == heads * HD, "attention_tc: head_dim must be 64 (D=%d heads=%d)", D, heads);
  ANYLOC_REQUIRE(B <= 65535 && heads <= 65535, "attention_tc: grid too large (B=%d heads=%d)", B, heads);
  if (fmt == ANYLOC_PAIR_BF16 || fmt == ANYLOC_PAIR_F16 || fmt == ANYLOC_PAIR_F16X1 || fmt == ANYLOC_PAIR_BF16X3)
    return attention_wg_launch(qkv_hi, qkv_lo, B, T, D, heads, o_hi, o_lo, fmt, st);
  static unsigned long long attr_seen = 0;
  if (first_use_on_this_device(&attr_seen))
    ANYLOC_CHECK_CUDA(cudaFuncSetAttribute(attention_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           Cfg::SMEM_BYTES));
  const dim3 grid(cdiv(T, BQ), heads, B);
  attention_tc_kernel<<<grid, THREADS, Cfg::SMEM_BYTES, st>>>(qkv_hi, qkv_lo, T, D, o_hi, o_lo);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}

// the same over images of different lengths packed into one [sum T_i, 3D] qkv buffer; tab.tile0 (64-query tiles) runs
// to n_tiles
int attention_tc_varlen_launch(const void* qkv_hi, const void* qkv_lo, const VarlenAttnTable& tab, int n_tiles, int D,
                               int heads, void* o_hi, void* o_lo, int fmt, cudaStream_t st) {
  using namespace atc;
  ANYLOC_REQUIRE(D == heads * HD, "attention_tc: head_dim must be 64 (D=%d heads=%d)", D, heads);
  ANYLOC_REQUIRE(heads <= 65535, "attention_tc: grid too large (heads=%d)", heads);
  if (fmt == ANYLOC_PAIR_BF16 || fmt == ANYLOC_PAIR_F16 || fmt == ANYLOC_PAIR_F16X1 || fmt == ANYLOC_PAIR_BF16X3)
    return attention_wg_varlen_launch(qkv_hi, qkv_lo, tab, D, heads, o_hi, o_lo, fmt, st);
  static unsigned long long attr_seen = 0;
  if (first_use_on_this_device(&attr_seen))
    ANYLOC_CHECK_CUDA(cudaFuncSetAttribute(attention_tc_varlen_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           Cfg::SMEM_BYTES));
  const dim3 grid(n_tiles, heads);
  attention_tc_varlen_kernel<<<grid, THREADS, Cfg::SMEM_BYTES, st>>>(qkv_hi, qkv_lo, tab, D, o_hi, o_lo);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}

// standalone fp16-pair attention on fp32 (hi,lo) qkv: converts into the fp16 operand layout in a stream-ordered
// temporary first
int attention_tc16_standalone(const float* qkv_hi, const float* qkv_lo, int B, int T, int D, int heads, void* o_hi,
                              void* o_lo, cudaStream_t st) {
  const size_t nq = (size_t)B * T * 3 * D;
  __half* buf = nullptr;
  ANYLOC_CHECK_CUDA(cudaMallocAsync((void**)&buf, 2 * nq * sizeof(__half), st));
  const int blocks = (int)std::min<size_t>((nq + 255) / 256, (size_t)device_sm_count() * 16);
  atc::qkv_to_f16_kernel<<<blocks, 256, 0, st>>>(qkv_hi, qkv_lo, nq, buf, buf + nq);
  ANYLOC_CHECK_LAUNCH();
  int rc = attention_tc_launch(buf, buf + nq, B, T, D, heads, o_hi, o_lo, ANYLOC_PAIR_F16, st);
  cudaFreeAsync(buf, st);
  return rc;
}

}  // namespace anyloc
