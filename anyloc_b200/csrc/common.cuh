// Shared helpers for libanyloc_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <math.h>
#include "../../include/anyloc_b200.h"

namespace anyloc {

void set_error(const char* fmt, ...);

#define ANYLOC_CHECK_CUDA(expr)                                                        \
  do {                                                                                 \
    cudaError_t _e = (expr);                                                           \
    if (_e != cudaSuccess) {                                                           \
      anyloc::set_error("%s:%d CUDA error %s: %s", __FILE__, __LINE__,                 \
                        cudaGetErrorName(_e), cudaGetErrorString(_e));                 \
      return ANYLOC_ERR_CUDA;                                                          \
    }                                                                                  \
  } while (0)

#define ANYLOC_CHECK_LAUNCH()                                                          \
  do {                                                                                 \
    anyloc::count_launch();                                                            \
    ANYLOC_CHECK_CUDA(cudaGetLastError());                                             \
  } while (0)

#define ANYLOC_REQUIRE(cond, ...)                                                      \
  do {                                                                                 \
    if (!(cond)) {                                                                     \
      anyloc::set_error(__VA_ARGS__);                                                  \
      return ANYLOC_ERR_ARG;                                                           \
    }                                                                                  \
  } while (0)

// Refuses a pointer that is not a multiple of `bytes` (a power of two): "<who>: <name> must be <bytes>-byte aligned
// (<why>)".  A null pointer passes; the entries' null checks are their own.
#define ANYLOC_REQUIRE_ALIGNED(p, bytes, who, name, why)                               \
  ANYLOC_REQUIRE((reinterpret_cast<uintptr_t>(p) & ((uintptr_t)(bytes) - 1)) == 0,     \
                 "%s: %s must be %d-byte aligned (%s)", who, name, (int)(bytes), why)

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
static inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// bump allocator over a caller-owned workspace
struct Workspace {
  char* base; size_t size; size_t off;
  Workspace(void* p, size_t n) : base((char*)p), size(n), off(0) {}
  template <typename T> T* take(size_t count) {
    size_t bytes = align_up(count * sizeof(T), 256);
    if (off + bytes > size) return nullptr;
    T* r = (T*)(base + off); off += bytes; return r;
  }
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// fp32 -> (hi, lo): hi = round-to-nearest tf32 (10 explicit mantissa bits, low 13 bits zero),
// lo = x - hi (exact in fp32).  hi + lo == x exactly.
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  hi = __uint_as_float(u & 0xffffe000u);
  lo = x - hi;
}

// fp16 pair format (engine TC3H): a GEMM input x is stored as (hi, lo) = (fp16(s*x), fp16(s*x - hi)), s a power
// of two; hi+lo carries ~22 significant bits of s*x like the tf32 pair, at half the bytes and on the 2x faster
// kind::f16 tensor path.  Activations use the fixed scale kActScale, weights a per-tensor scale (see vit.py);
// the GEMM epilogue multiplies the accumulator by alpha = 1/(s_A*s_B) (exact).
constexpr float kActScale = 8.0f;
// f32 <-> f16 conversions run on the 16-lane/clk conversion path (measured: they, not the FMAs, bounded the softmax
// warps of the attention kernel), so the hi part is rounded to 11 significant bits with Veltkamp's splitting on the
// FMA pipe (t = x*(2^13+1); hi = t - (t - x), round-to-nearest) and only the final packs use cvt -- one
// cvt.rn.f16x2.f32 per TWO elements in the packed variant.
__device__ __forceinline__ float veltkamp_hi11(float x) {
  const float t = __fmul_rn(x, 8193.0f);
  return __fsub_rn(t, __fsub_rn(t, x));
}
__device__ __forceinline__ void split_f16(float xs, __half& hi, __half& lo) {
  const float h = veltkamp_hi11(xs);
  hi = __float2half_rn(h);                       // exact (11 significant bits) inside the fp16 normal range
  lo = __float2half_rn(__fsub_rn(xs, h));
}
// two values -> packed (hi, lo) words; `a` lands in the low 16 bits (element k), `b` in the high 16 bits (k+1)
__device__ __forceinline__ void split_f16x2(float a, float b, uint32_t& hi2, uint32_t& lo2) {
  const float ha = veltkamp_hi11(a), hb = veltkamp_hi11(b);
  const float la = __fsub_rn(a, ha), lb = __fsub_rn(b, hb);
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(hi2) : "f"(hb), "f"(ha));
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(lo2) : "f"(lb), "f"(la));
}

// Single fp16 format (ANYLOC_PAIR_F16X1): the hi half of the fp16 pair alone, bit for bit what split_f16 /
// split_f16x2 write into hi for the same (scaled) input.  Two values -> one packed word; `a` in the low 16 bits.
__device__ __forceinline__ uint32_t pack_f16x2_hi(float a, float b) {
  const float ha = veltkamp_hi11(a), hb = veltkamp_hi11(b);
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hb), "f"(ha));
  return r;
}
__device__ __forceinline__ __half f16_hi(float xs) { return __float2half_rn(veltkamp_hi11(xs)); }

// Single bf16 format (ANYLOC_PAIR_BF16): one array of bf16_rn(x), no lo word and no scale.  Two values -> one packed
// word; `a` lands in the low 16 bits (element k), `b` in the high 16 bits (k+1).
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
// bf16 pair format (ANYLOC_PAIR_BF16X3): hi = bf16_rn(x), lo = bf16_rn(x - hi); x - hi is exact in fp32 (hi keeps x's
// leading 8 bits, so the difference fits in 24).  Two values -> packed (hi, lo) words; `a` in the low 16 bits.
__device__ __forceinline__ void split_bf16x2(float a, float b, uint32_t& hi2, uint32_t& lo2) {
  hi2 = pack_bf16x2(a, b);
  lo2 = pack_bf16x2(a - __uint_as_float(hi2 << 16), b - __uint_as_float(hi2 & 0xffff0000u));
}

// Single e4m3 format (ANYLOC_PAIR_FP8): a row (activations) or a matrix (weights) is one e4m3 array q = e4m3_rn(x / s)
// with one power-of-two scale s, x ~ q s.  s = 2^k with k the smallest integer that puts max|x| / s <= 448 (e4m3's
// largest finite value), at least -126 so that s and 1/s are normal fp32 numbers; s = 1 for an all-zero (or NaN) row.
// Scaling by a power of two is exact, so e4m3_rn is the only rounding.  448 = 0.875 2^9: with max|x| = m 2^e, m in
// [0.5, 1), k = e - 9, or e - 8 when m > 0.875.  Activation rows that hold an Inf get a NaN scale (fp8_row_scale).
__host__ __device__ inline int fp8_scale_exp(float amax) {
  if (!(amax > 0.f) || amax > 3.402823466e38f) return 0;
  int e;
  const float m = frexpf(amax, &e);
  const int k = e - 9 + (m > 0.875f ? 1 : 0);
  return k < -126 ? -126 : k;
}
// 2^k for k in [-126, 127]
__host__ __device__ inline float pow2f(int k) {
  union { uint32_t u; float f; } v;
  v.u = (uint32_t)(127 + k) << 23;
  return v.f;
}
// The scale s and its inverse of a row of e4m3 activations whose max |x| (NaNs dropped, as fmaxf drops them) is amax.
// A row that holds an Inf gets s = 1/s = NaN: q = e4m3_rn(x / s) is then NaN throughout, where satfinite would have
// clamped the Inf to +-448 and left a finite, wrong row, and the GEMM's dequantisation by s makes the consumer's output
// row NaN.
__device__ __forceinline__ void fp8_row_scale(float amax, float& s, float& inv) {
  const int k = fp8_scale_exp(amax);
  const bool inf = !(amax <= 3.402823466e38f);
  s = inf ? __int_as_float(0x7fffffff) : pow2f(k);
  inv = inf ? __int_as_float(0x7fffffff) : pow2f(-k);
}
// e4m3_rn of two values (satfinite: beyond +-448 clamps, NaN stays NaN) -> `a` in the low byte, `b` in the high byte
__device__ __forceinline__ uint32_t pack_e4m3x2(float a, float b) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(b), "f"(a));
  return r;
}
__device__ __forceinline__ uint32_t pack_e4m3x4(float a, float b, float c, float d) {
  return pack_e4m3x2(a, b) | (pack_e4m3x2(c, d) << 16);
}

// Per-image geometry of a packed batch of differently sized images (anyloc_vit_extract_varlen).  The tables reach the
// kernels by value as __grid_constant__ parameters: the launch copies them, so a call neither synchronises with the
// host nor keeps a host pointer, and each stays under the classic 4 KB kernel-parameter limit.
constexpr int kVarlenMaxB = ANYLOC_VIT_VARLEN_MAX_B;
// im2col, token assembly and the facet slice.  Image i has tokens [tok0[i], tok0[i] + 1 + nreg + gh[i]*gw[i]) of the
// packed sequence (cls, nreg registers, patches), patch rows from tok0[i] - (1 + nreg) * i and, without the cls token,
// output rows from tok0[i] - i.
struct VarlenImgTable {
  int n;
  int tok0[kVarlenMaxB];
  int gh[kVarlenMaxB], gw[kVarlenMaxB];
  const float* ptr[kVarlenMaxB];        // the image [3, gh*P, gw*P] (im2col) or its positional table (assembly)
  int nreg;                             // register tokens per image (last: the fields above keep their offsets)
};
static_assert(sizeof(VarlenImgTable) <= 4096, "kernel parameter over 4 KB");
// the last image i whose first row tok0[i] - skip*i (skip = rows the kernel's grid omits per image) is <= row
__device__ __forceinline__ int varlen_image_of(const VarlenImgTable& t, int row, int skip) {
  int lo = 0, hi = t.n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (t.tok0[mid] - skip * mid <= row) lo = mid; else hi = mid - 1;
  }
  return lo;
}
// the attention: one entry per image, in any order; tile0 ascending, tile0[0] = 0
struct VarlenAttnTable {
  int n;
  int tile0[kVarlenMaxB];               // first 64-query tile of the entry in the grid
  int row0[kVarlenMaxB];                // first token row of the image
  int len[kVarlenMaxB];                 // its tokens
};
static_assert(sizeof(VarlenAttnTable) <= 4096, "kernel parameter over 4 KB");

// Where an aggregation kernel finds image b's rows.  A padded batch [B,N,D] keeps image b at rows b*N.., of which the
// first min(N, n_valid[b]) count (all N without n_valid); a packed list [R,D] keeps it at rows row0[b] .. + len[b]
// (device arrays, checked on the host by varlen_rows_check).  The kernels take either, so the padded instantiations
// compile to the code they had before the packed ones existed.
struct PaddedRows {
  const int32_t* n_valid; int N;
  __device__ __forceinline__ size_t first(int b) const { return (size_t)b * N; }
  __device__ __forceinline__ int count(int b) const { return n_valid ? min(N, n_valid[b]) : N; }
};
struct PackedRows {
  const int64_t* row0; const int32_t* len;
  __device__ __forceinline__ size_t first(int b) const { return (size_t)row0[b]; }
  __device__ __forceinline__ int count(int b) const { return len[b]; }
};
// The host side of a packed list's table: copies row0 / len [B] from the device (a synchronisation of `st`) and
// checks that every len >= 0, row0 >= 0, row0 + len <= R and that no two images share a row (an empty image shares
// none).  -> ANYLOC_OK with the largest len in *max_len, else ANYLOC_ERR_ARG / _CUDA naming `who`.
int varlen_rows_check(const int64_t* row0, const int32_t* len, int B, int64_t R, cudaStream_t st, const char* who,
                      int* max_len);

// where the qkv tap kernel writes the q, k and v facet rows of one layer (null: that facet is not tapped)
struct QkvTapOuts {
  float* out[3];
};

int device_sm_count();
// true the first time it is called on the CURRENT device for this flag word: cudaFuncSetAttribute is per device, so a
// process that drives several GPUs must repeat it on each of them (one bit per device ordinal; atomic because two host
// threads may race on the word).  A failing cudaFuncSetAttribute is reported to the caller by ANYLOC_CHECK_CUDA; the
// launch that follows a failed attribute set fails loudly as well (dynamic shared memory over the default limit).
static inline bool first_use_on_this_device(unsigned long long* seen) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return true;
  const unsigned long long bit = 1ull << dev;
  const unsigned long long old = __atomic_fetch_or(seen, bit, __ATOMIC_RELAXED);
  return (old & bit) == 0;
}
void count_launch();

// Optional per-category device timing (cudaEvents on the launching stream), see anyloc_profile_*.
enum ProfCat { PC_GEMM_TC = 0, PC_GEMM_SIMT, PC_ATTENTION, PC_LAYERNORM, PC_VIT_MISC, PC_VLAD, PC_TOPK, PC_COUNT };
struct ProfScope {
  int slot; cudaStream_t st;
  ProfScope(int cat, cudaStream_t stream, double work);
  ~ProfScope();
};

}  // namespace anyloc
