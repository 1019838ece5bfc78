// Shared GEMM epilogue (used by the SIMT and the tensor-core GEMM kernels).
#pragma once
#include "formats.cuh"

namespace anyloc {

struct EpiParams {
  int mode;
  const float* bias;    // [N] nullable
  const float* gamma;   // [N] (LS_RESID)
  const float* resid;   // [M,ldo] (LS_RESID; may alias out)
  float* out;           // [M,ldo]
  float* out_lo;        // [M,ldo] (SPLIT modes)
  int ldo;
  float alpha = 1.0f;   // accumulator scale (1/(s_A*s_B) for fp16-pair inputs, else 1)
  int out_fmt = ANYLOC_PAIR_TF32;   // SPLIT output format (ANYLOC_PAIR_*): the tf32 and fp16 pair GEMMs write tf32 or
                                    // fp16 pairs by it at run time; the other formats write Fmt<FMT>::OUT
  const int* gate = nullptr;   // device flag (nullable): tensor-core GEMM kernels return immediately when *gate == 0 (conditional fallbacks without a host sync)
  const float* row_scale = nullptr;   // [M] e4m3 A operand's row scales (single e4m3 GEMM only): acc of row m times row_scale[m]
};

// SPLIT output v of element o in the format OUT
template <int OUT>
__device__ __forceinline__ void split_put1(const EpiParams& p, size_t o, float v) {
  typedef typename Fmt<OUT>::T T;
  put1<OUT>(reinterpret_cast<T*>(p.out), reinterpret_cast<T*>(p.out_lo), o, v);
}
// SPLIT output of a GEMM on FMT inputs (the SIMT engine's pair GEMMs take the default): Fmt<FMT>::OUT, or for the tf32
// and fp16 pair inputs the pair format ep.out_fmt names, chosen at run time (fixed_out)
template <int FMT = ANYLOC_PAIR_TF32>
__device__ __forceinline__ void epi_store_split(const EpiParams& p, size_t o, float v) {
  if constexpr (fixed_out<FMT>()) split_put1<Fmt<FMT>::OUT>(p, o, v);
  else if (p.out_fmt != ANYLOC_PAIR_TF32) split_put1<ANYLOC_PAIR_F16>(p, o, v);
  else split_put1<ANYLOC_PAIR_TF32>(p, o, v);
}

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
__device__ __forceinline__ float silu(float x) { return x / (1.0f + expf(-x)); }
// Same function on the special-function unit: e = 2^(-x log2 e) (ex2.approx, 2^-22 relative), 1/(1+e) by rcp.approx +
// one Newton step.  |error| <= ~3e-7 |silu(x)|; 7 instructions instead of ~35 (the SwiGLU epilogue runs it 4 M times
// per GEMM).  x -> -inf: e = inf, 1/(1+e) = 0 -> -0;  NaN propagates.
__device__ __forceinline__ float silu_fast(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
  const float d = 1.0f + e;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(d));
  r = (d < 3.0e38f) ? fmaf(r, fmaf(-d, r, 1.0f), r) : r;     // Newton step (skipped when d overflowed: r = 0)
  return x * r;
}

// Apply the epilogue to one accumulator element (m, n).  For SWIGLU the caller passes the PAIR
// (acc0 at column n even, acc1 at column n+1) and the result lands in column n/2.
template <int FMT = ANYLOC_PAIR_TF32>
__device__ __forceinline__ void epi_store1(const EpiParams& p, int m, int n, float acc) {
  float v = acc * p.alpha + (p.bias ? __ldg(p.bias + n) : 0.f);
  size_t o = (size_t)m * p.ldo + n;
  switch (p.mode) {
    case ANYLOC_EPI_BIAS: p.out[o] = v; break;
    case ANYLOC_EPI_BIAS_SPLIT: epi_store_split<FMT>(p, o, v); break;
    case ANYLOC_EPI_GELU_SPLIT: epi_store_split<FMT>(p, o, gelu_erf(v)); break;
    case ANYLOC_EPI_LS_RESID: p.out[o] = p.resid[o] + __ldg(p.gamma + n) * v; break;
    default: break;
  }
}
template <int FMT = ANYLOC_PAIR_TF32>
__device__ __forceinline__ void epi_store_pair(const EpiParams& p, int m, int n_even, float acc0, float acc1) {
  // SWIGLU: columns (n_even, n_even+1) = (x1_j, x2_j), j = n_even/2
  float x1 = acc0 * p.alpha + (p.bias ? __ldg(p.bias + n_even) : 0.f);
  float x2 = acc1 * p.alpha + (p.bias ? __ldg(p.bias + n_even + 1) : 0.f);
  epi_store_split<FMT>(p, (size_t)m * p.ldo + (n_even >> 1), silu(x1) * x2);
}

}  // namespace anyloc
