// The GEMM-input formats (ANYLOC_PAIR_*), each described once: Fmt<FMT> for the kernels, format_info(fmt) for the
// host.  A new format adds a Fmt specialisation (element type, LO, SCALED, OUT and its stores), a row in
// format_info's table and a case in fmt_switch.
#pragma once
#include <type_traits>
#include "common.cuh"

namespace anyloc {

// Fmt<FMT>:
//   T       element type of the hi (and lo) array; W2 the word of two adjacent elements
//   LO      the format has a lo array
//   SCALED  it stores kActScale x for an activation x (split1, split2 and put4 scale)
//   OUT     the format that SPLIT epilogues and the attention write for these inputs
//   split1 / split2: the stored hi (and lo) of one value, or the words of two adjacent values (`a` first); lo is left
//           untouched without a lo array.  put1 / put2 below store them.
//   put4    stores 4 values at elements 4 i .. 4 i + 3 of hi (and lo)
//   pack2   (2-byte formats) the words of a and b as given, unscaled
template <int FMT> struct Fmt;

template <> struct Fmt<ANYLOC_PAIR_TF32> {    // tf32 pairs: hi = rna_tf32(x), lo = x - hi
  typedef float T;
  static constexpr bool LO = true, SCALED = false;
  typedef float2 W2;
  static constexpr int OUT = ANYLOC_PAIR_TF32;
  static __device__ __forceinline__ void split1(float x, T& h, T& l) { split_tf32(x, h, l); }
  static __device__ __forceinline__ void split2(float a, float b, W2& h, W2& l) {
    split_tf32(a, h.x, l.x); split_tf32(b, h.y, l.y);
  }
  static __device__ __forceinline__ void put4(T* hi, T* lo, size_t i, float a, float b, float c, float d) {
    float4 h, l;
    split_tf32(a, h.x, l.x); split_tf32(b, h.y, l.y); split_tf32(c, h.z, l.z); split_tf32(d, h.w, l.w);
    reinterpret_cast<float4*>(hi)[i] = h; reinterpret_cast<float4*>(lo)[i] = l;
  }
};

template <> struct Fmt<ANYLOC_PAIR_F16> {     // fp16 pairs of kActScale x (split_f16)
  typedef __half T;
  static constexpr bool LO = true, SCALED = true;
  typedef uint32_t W2;
  static constexpr int OUT = ANYLOC_PAIR_F16;
  static __device__ __forceinline__ void split1(float x, T& h, T& l) { split_f16(x * kActScale, h, l); }
  static __device__ __forceinline__ void split2(float a, float b, W2& h, W2& l) {
    split_f16x2(a * kActScale, b * kActScale, h, l);
  }
  static __device__ __forceinline__ void pack2(float a, float b, uint32_t& h, uint32_t& l) { split_f16x2(a, b, h, l); }
  static __device__ __forceinline__ void put4(T* hi, T* lo, size_t i, float a, float b, float c, float d) {
    uint2 h, l;
    split_f16x2(a * kActScale, b * kActScale, h.x, l.x);
    split_f16x2(c * kActScale, d * kActScale, h.y, l.y);
    reinterpret_cast<uint2*>(hi)[i] = h; reinterpret_cast<uint2*>(lo)[i] = l;
  }
};

template <> struct Fmt<ANYLOC_PAIR_BF16> {    // single bf16: bf16_rn(x), no lo, no scale
  typedef __nv_bfloat16 T;
  static constexpr bool LO = false, SCALED = false;
  typedef uint32_t W2;
  static constexpr int OUT = ANYLOC_PAIR_BF16;
  static __device__ __forceinline__ void split1(float x, T& h, T&) { h = __float2bfloat16_rn(x); }
  static __device__ __forceinline__ void split2(float a, float b, W2& h, W2&) { h = pack_bf16x2(a, b); }
  static __device__ __forceinline__ void pack2(float a, float b, uint32_t& h, uint32_t&) { h = pack_bf16x2(a, b); }
  static __device__ __forceinline__ void put4(T* hi, T*, size_t i, float a, float b, float c, float d) {
    reinterpret_cast<uint2*>(hi)[i] = make_uint2(pack_bf16x2(a, b), pack_bf16x2(c, d));
  }
};

template <> struct Fmt<ANYLOC_PAIR_F16X1> {   // single fp16: the hi of Fmt<ANYLOC_PAIR_F16>'s pair, bit for bit
  typedef __half T;
  static constexpr bool LO = false, SCALED = true;
  typedef uint32_t W2;
  static constexpr int OUT = ANYLOC_PAIR_F16X1;
  static __device__ __forceinline__ void split1(float x, T& h, T&) { h = f16_hi(x * kActScale); }
  static __device__ __forceinline__ void split2(float a, float b, W2& h, W2&) {
    h = pack_f16x2_hi(a * kActScale, b * kActScale);
  }
  static __device__ __forceinline__ void pack2(float a, float b, uint32_t& h, uint32_t&) { h = pack_f16x2_hi(a, b); }
  static __device__ __forceinline__ void put4(T* hi, T*, size_t i, float a, float b, float c, float d) {
    reinterpret_cast<uint2*>(hi)[i] =
        make_uint2(pack_f16x2_hi(a * kActScale, b * kActScale), pack_f16x2_hi(c * kActScale, d * kActScale));
  }
};

template <> struct Fmt<ANYLOC_PAIR_BF16X3> {  // bf16 pairs: hi = bf16_rn(x), lo = bf16_rn(x - hi), no scale
  typedef __nv_bfloat16 T;
  static constexpr bool LO = true, SCALED = false;
  typedef uint32_t W2;
  static constexpr int OUT = ANYLOC_PAIR_BF16X3;
  static __device__ __forceinline__ void split1(float x, T& h, T& l) {
    h = __float2bfloat16_rn(x);
    l = __float2bfloat16_rn(x - __bfloat162float(h));
  }
  static __device__ __forceinline__ void split2(float a, float b, W2& h, W2& l) { split_bf16x2(a, b, h, l); }
  static __device__ __forceinline__ void pack2(float a, float b, uint32_t& h, uint32_t& l) { split_bf16x2(a, b, h, l); }
  static __device__ __forceinline__ void put4(T* hi, T* lo, size_t i, float a, float b, float c, float d) {
    uint2 h, l;
    split_bf16x2(a, b, h.x, l.x);
    split_bf16x2(c, d, h.y, l.y);
    reinterpret_cast<uint2*>(hi)[i] = h; reinterpret_cast<uint2*>(lo)[i] = l;
  }
};

// single e4m3: sizes only.  Its writers (LayerNorm's row scale, the quantisers) scale by a power of two per row or
// tensor, a different kind of store; the A operand's lo slot holds those fp32 row scales.
template <> struct Fmt<ANYLOC_PAIR_FP8> {
  typedef uint8_t T;
  static constexpr bool LO = false, SCALED = false;
  static constexpr int OUT = ANYLOC_PAIR_BF16;
};

// One value, or two adjacent values (i even), stored at element i of hi (and lo) in the format FMT
template <int FMT>
__device__ __forceinline__ void put1(typename Fmt<FMT>::T* hi, typename Fmt<FMT>::T* lo, size_t i, float x) {
  typename Fmt<FMT>::T h, l;
  Fmt<FMT>::split1(x, h, l);
  hi[i] = h;
  if constexpr (Fmt<FMT>::LO) lo[i] = l;
}
template <int FMT>
__device__ __forceinline__ void put2(typename Fmt<FMT>::T* hi, typename Fmt<FMT>::T* lo, size_t i, float a, float b) {
  typename Fmt<FMT>::W2 h, l;
  Fmt<FMT>::split2(a, b, h, l);
  *reinterpret_cast<typename Fmt<FMT>::W2*>(hi + i) = h;
  if constexpr (Fmt<FMT>::LO) *reinterpret_cast<typename Fmt<FMT>::W2*>(lo + i) = l;
}

// "no format": the qkv tap writes no attention operands
constexpr int FMT_NONE = -1;

// Host: f(std::integral_constant<int, FMT>()) for the run-time format fmt; other values run the tf32 pairs
template <class F>
inline auto fmt_switch(int fmt, F&& f) {
  switch (fmt) {
    case ANYLOC_PAIR_F16: return f(std::integral_constant<int, ANYLOC_PAIR_F16>());
    case ANYLOC_PAIR_BF16: return f(std::integral_constant<int, ANYLOC_PAIR_BF16>());
    case ANYLOC_PAIR_FP8: return f(std::integral_constant<int, ANYLOC_PAIR_FP8>());
    case ANYLOC_PAIR_F16X1: return f(std::integral_constant<int, ANYLOC_PAIR_F16X1>());
    case ANYLOC_PAIR_BF16X3: return f(std::integral_constant<int, ANYLOC_PAIR_BF16X3>());
    default: return f(std::integral_constant<int, ANYLOC_PAIR_TF32>());
  }
}

// The SPLIT output format of a GEMM on FMT inputs is Fmt<FMT>::OUT, fixed at compile time -- except for the tf32 and
// fp16 pairs, whose GEMMs write either of those two pair formats as EpiParams::out_fmt says at run time
template <int FMT> __host__ __device__ constexpr bool fixed_out() { return !Fmt<FMT>::LO || FMT == ANYLOC_PAIR_BF16X3; }

// Host-side facts of a format
struct FormatInfo {
  const char* name;        // in error messages
  const char* id;          // its ANYLOC_PAIR_* name
  int esz;                 // bytes per element of the activations and of the weights
  bool lo;                 // lo arrays
  bool row_scales;         // A's lo slot holds fp32 row scales
  bool tc_only;            // runs on the tensor-core engine only
  int out;                 // format of the SPLIT outputs and of the attention
  int patch;               // format of the patch embedding
};
inline const FormatInfo& format_info(int fmt) {
  static const FormatInfo table[] = {
      {"tf32-pair", "ANYLOC_PAIR_TF32", 4, true, false, false, ANYLOC_PAIR_TF32, ANYLOC_PAIR_TF32},
      {"fp16-pair", "ANYLOC_PAIR_F16", 2, true, false, false, ANYLOC_PAIR_F16, ANYLOC_PAIR_F16},
      {"single-bf16", "ANYLOC_PAIR_BF16", 2, false, false, true, ANYLOC_PAIR_BF16, ANYLOC_PAIR_BF16},
      {"single-e4m3", "ANYLOC_PAIR_FP8", 1, false, true, true, ANYLOC_PAIR_BF16, ANYLOC_PAIR_BF16},
      {"single-fp16", "ANYLOC_PAIR_F16X1", 2, false, false, true, ANYLOC_PAIR_F16X1, ANYLOC_PAIR_F16X1},
      {"bf16-pair", "ANYLOC_PAIR_BF16X3", 2, true, false, true, ANYLOC_PAIR_BF16X3, ANYLOC_PAIR_BF16X3},
  };
  return table[fmt >= ANYLOC_PAIR_TF32 && fmt <= ANYLOC_PAIR_BF16X3 ? fmt : ANYLOC_PAIR_TF32];
}

}  // namespace anyloc
