// C ABI of libanyloc_b200.so: error plumbing, building-block wrappers, GEMM engine dispatch and the
// DINOv2 forward orchestration (early exit at the hooked module; reference
// /root/reference/utilities.py:245-252,263-285 + upstream DinoVisionTransformer).
#include <stdarg.h>
#include <string.h>
#include <algorithm>
#include <array>
#include <atomic>
#include <vector>
#include "epilogue.cuh"

namespace anyloc {

static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof(g_err), fmt, ap); va_end(ap);
}

static std::atomic<long long> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

namespace {
struct ProfRec { cudaEvent_t a, b; int cat; double work; };
bool g_prof_on = false;
std::vector<ProfRec> g_prof;
size_t g_prof_used = 0;
}  // namespace
ProfScope::ProfScope(int cat, cudaStream_t stream, double work) : slot(-1), st(stream) {
  if (!g_prof_on) return;
  if (g_prof_used == g_prof.size()) {
    ProfRec r{};
    if (cudaEventCreate(&r.a) != cudaSuccess || cudaEventCreate(&r.b) != cudaSuccess) return;
    g_prof.push_back(r);
  }
  slot = (int)g_prof_used++;
  g_prof[slot].cat = cat; g_prof[slot].work = work;
  cudaEventRecord(g_prof[slot].a, st);
}
ProfScope::~ProfScope() { if (slot >= 0) cudaEventRecord(g_prof[slot].b, st); }

int device_sm_count() {
  // per device ordinal: one process may drive several (possibly non-identical / MIG) devices
  static std::atomic<int> cached[64];
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 148;
  n = cached[dev].load(std::memory_order_relaxed);
  if (n > 0) return n;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 148;
  cached[dev].store(n, std::memory_order_relaxed);
  return n;
}

// engines (defined in gemm_simt.cu / gemm_tc.cu)
int gemm_simt_launch(const void*, const void*, int, const void*, const void*, int, int, int, int,
                     const EpiParams&, bool f16, cudaStream_t);
int gemm_tc_launch(const void*, const void*, int, const void*, const void*, int, int, int, int,
                   const EpiParams&, int fmt, cudaStream_t);
bool gemm_tc_supported(const void* a_hi, const void* a_lo, int lda, const void* b_hi, const void* b_lo,
                       int ldb, int M, int N, int K, const EpiParams& ep, int fmt);
// vit_ops.cu / attention.cu
int launch_split(const float*, float*, float*, size_t, cudaStream_t);
int launch_split_f16(const float*, void*, void*, size_t, float, cudaStream_t);
int launch_split_bf16(const float*, void*, size_t, cudaStream_t);
int launch_im2col(const float*, int, int, int, int, int, void*, void*, int, cudaStream_t);
int launch_assemble(const float*, const float*, const float*, const float*, int, int, int, int, float*, cudaStream_t);
int launch_layernorm(const float*, const float*, const float*, int, int, float, void*, void*, int, cudaStream_t);
int launch_quantize_fp8_rows(const void*, int, int, void*, float*, cudaStream_t);
int launch_quantize_fp8_tensor(const float*, size_t, void*, float*, cudaStream_t);
int launch_facet_out(const float*, int, int, int64_t, int, int, int, int, float*, cudaStream_t);
int launch_l2norm(const float*, int64_t, int, int64_t, float*, cudaStream_t);
int attention_launch(const float*, const float*, int, int, int, int, void*, void*, bool, cudaStream_t);
int attention_tc_launch(const void*, const void*, int, int, int, int, void*, void*, int, cudaStream_t);
int attention_tc16_standalone(const float*, const float*, int, int, int, int, void*, void*, cudaStream_t);
int attention_tc_varlen_launch(const void*, const void*, const VarlenAttnTable&, int, int, int, void*, void*, int,
                               cudaStream_t);
int launch_im2col_varlen(const VarlenImgTable&, int, int, int, void*, void*, int, cudaStream_t);
int launch_assemble_varlen(const float*, const float*, const float*, const VarlenImgTable&, int, int, float*,
                           cudaStream_t);
int launch_facet_out_varlen(const float*, const VarlenImgTable&, int, int64_t, int, int, int, int, float*, cudaStream_t);
int launch_qkv_tap(const float*, int, int, const VarlenImgTable*, int, int, void*, void*, const QkvTapOuts&, int, int,
                   cudaStream_t);
// pca.cu
size_t pca_colsum_workspace_bytes(int64_t, int);
int pca_colsum_launch(const float*, int64_t, int64_t, int, double*, double*, cudaStream_t);
int pca_atb_launch(int, const float*, int64_t, const double*, const double*, int64_t, int64_t, int, int, double*,
                   int64_t, cudaStream_t);
int pca_mirror_launch(double*, int, int64_t, cudaStream_t);

// fmt: ANYLOC_PAIR_* of the operands.  The single formats and the bf16 pairs run on the tensor cores only: they run
// the wgmma kernel at every M (no SIMT route, so a row's result never depends on how many rows share the call) and
// refuse the SIMT engine.  Single e4m3's a_lo holds A's fp32 row scales; the bf16 pairs need both lo operands.
static int gemm_dispatch(const void* a_hi, const void* a_lo, int lda, const void* b_hi, const void* b_lo,
                         int ldb, int M, int N, int K, const EpiParams& ep, int engine, int fmt, cudaStream_t st) {
  if (M == 0 || N == 0) return ANYLOC_OK;
  const FormatInfo& f = format_info(fmt);
  const double flops = 2.0 * M * N * K;
  if (f.tc_only) {
    const bool a_lo_ok = f.row_scales ? a_lo && (reinterpret_cast<uintptr_t>(a_lo) & 3) == 0 : f.lo ? a_lo != nullptr
                                                                                                 : !a_lo;
    const bool b_lo_ok = f.lo ? b_lo != nullptr : !b_lo;
    if (engine == ANYLOC_GEMM_SIMT || !a_lo_ok || !b_lo_ok ||
        !gemm_tc_supported(a_hi, f.lo ? a_lo : nullptr, lda, b_hi, b_lo, ldb, M, N, K, ep, fmt)) {
      set_error("gemm: the %s format runs on the tensor-core engine only, with 16-byte aligned operands, K, lda and "
                "ldb multiples of %d%s (M=%d N=%d K=%d lda=%d ldb=%d engine=%d)", f.name, 16 / f.esz,
                f.row_scales ? ", A's row scales and no B lo operand" : f.lo ? " and both lo operands"
                                                                          : " and no lo operands", M, N, K, lda, ldb,
                engine);
      return ANYLOC_ERR_UNSUPPORTED;
    }
    ProfScope ps(PC_GEMM_TC, st, flops);
    return gemm_tc_launch(a_hi, a_lo, lda, b_hi, b_lo, ldb, M, N, K, ep, fmt, st);
  }
  bool tc_ok = gemm_tc_supported(a_hi, a_lo, lda, b_hi, b_lo, ldb, M, N, K, ep, fmt);
  if (engine == ANYLOC_GEMM_TC3 && !tc_ok) {
    set_error("gemm: tensor-core engine does not support this shape/alignment (M=%d N=%d K=%d lda=%d ldb=%d f16=%d)",
              M, N, K, lda, ldb, (int)(fmt == ANYLOC_PAIR_F16));
    return ANYLOC_ERR_UNSUPPORTED;
  }
  if (engine == ANYLOC_GEMM_TC3 || (engine == ANYLOC_GEMM_AUTO && tc_ok && M >= 32)) {
    ProfScope ps(PC_GEMM_TC, st, flops);
    return gemm_tc_launch(a_hi, a_lo, lda, b_hi, b_lo, ldb, M, N, K, ep, fmt, st);
  }
  ProfScope ps(PC_GEMM_SIMT, st, flops);
  return gemm_simt_launch(a_hi, a_lo, lda, b_hi, b_lo, ldb, M, N, K, ep, fmt == ANYLOC_PAIR_F16, st);
}

}  // namespace anyloc

using namespace anyloc;

extern "C" const char* anyloc_last_error(void) { return g_err; }
extern "C" int anyloc_version(void) { return 101; }
extern "C" long long anyloc_launch_count(void) { return g_launches.load(); }
extern "C" int anyloc_profile_enable(int on) { g_prof_on = on != 0; g_prof_used = 0; return ANYLOC_OK; }
extern "C" int anyloc_profile_read(double* ms, long long* groups, double* work) {
  ANYLOC_REQUIRE(ms && groups && work, "profile_read: null pointer");
  for (int c = 0; c < PC_COUNT; ++c) { ms[c] = 0.0; groups[c] = 0; work[c] = 0.0; }
  for (size_t i = 0; i < g_prof_used; ++i) {
    float t = 0.f;
    ANYLOC_CHECK_CUDA(cudaEventSynchronize(g_prof[i].b));
    ANYLOC_CHECK_CUDA(cudaEventElapsedTime(&t, g_prof[i].a, g_prof[i].b));
    ms[g_prof[i].cat] += t; groups[g_prof[i].cat] += 1; work[g_prof[i].cat] += g_prof[i].work;
  }
  g_prof_used = 0;
  return ANYLOC_OK;
}

extern "C" int anyloc_device_info(int* sm_count, size_t* smem_optin_bytes) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) {
    cudaGetLastError();
    set_error("no CUDA device visible (libanyloc_b200 has no CPU fallback)");
    return ANYLOC_ERR_CUDA;
  }
  int dev = 0; cudaDeviceProp p;
  ANYLOC_CHECK_CUDA(cudaGetDevice(&dev));
  ANYLOC_CHECK_CUDA(cudaGetDeviceProperties(&p, dev));
  if (sm_count) *sm_count = p.multiProcessorCount;
  if (smem_optin_bytes) *smem_optin_bytes = p.sharedMemPerBlockOptin;
  return p.major * 10 + p.minor;
}

extern "C" int anyloc_gemm_nt(const void* a_hi, const void* a_lo, int lda, const void* b_hi, const void* b_lo,
                              int ldb, int M, int N, int K, int in_dtype, float alpha, int epilogue,
                              const float* bias, const float* gamma, const float* resid, void* out, void* out_lo,
                              int ldo, int out_dtype, int engine, void* stream) {
  ANYLOC_REQUIRE(a_hi && b_hi && out, "gemm_nt: null pointer");
  ANYLOC_REQUIRE(M >= 0 && N >= 0 && K > 0, "gemm_nt: bad dims");
  ANYLOC_REQUIRE(in_dtype >= ANYLOC_PAIR_TF32 && in_dtype <= ANYLOC_PAIR_BF16X3, "gemm_nt: bad in_dtype %d", in_dtype);
  ANYLOC_REQUIRE(out_dtype >= ANYLOC_PAIR_TF32 && out_dtype <= ANYLOC_PAIR_BF16X3 && out_dtype != ANYLOC_PAIR_FP8,
                 "gemm_nt: bad out_dtype %d", out_dtype);
  ANYLOC_REQUIRE(epilogue >= ANYLOC_EPI_BIAS && epilogue <= ANYLOC_EPI_LS_RESID, "gemm_nt: bad epilogue %d", epilogue);
  const FormatInfo& f = format_info(in_dtype);
  const bool either_pair = f.lo && !f.tc_only;     // tf32 or fp16 pair inputs write either of those pairs
  ANYLOC_REQUIRE(either_pair ? out_dtype == ANYLOC_PAIR_TF32 || out_dtype == ANYLOC_PAIR_F16 : out_dtype == f.out,
                 "gemm_nt: %s inputs write %s outputs (in_dtype=%d out_dtype=%d)", f.name,
                 either_pair ? "tf32-pair or fp16-pair" : format_info(f.out).name, in_dtype, out_dtype);
  if (f.lo && f.tc_only)
    ANYLOC_REQUIRE(a_lo && b_lo, "gemm_nt: the %s format needs both lo operands (a_lo and b_lo)", f.name);
  if (f.row_scales)
    ANYLOC_REQUIRE(a_lo && !b_lo && !out_lo, "gemm_nt: %s inputs take A's row scales in a_lo, no b_lo and no out_lo",
                   f.name);
  else if (!f.lo)
    ANYLOC_REQUIRE(!a_lo && !b_lo && !out_lo, "gemm_nt: the %s format has no lo arrays (a_lo, b_lo, out_lo must be "
                   "NULL)", f.name);
  else if (epilogue == ANYLOC_EPI_BIAS_SPLIT || epilogue == ANYLOC_EPI_GELU_SPLIT || epilogue == ANYLOC_EPI_SWIGLU_SPLIT)
    ANYLOC_REQUIRE(out_lo, "gemm_nt: split epilogue needs out_lo");
  if (epilogue == ANYLOC_EPI_SWIGLU_SPLIT) ANYLOC_REQUIRE(N % 2 == 0, "gemm_nt: swiglu needs even N");
  if (epilogue == ANYLOC_EPI_LS_RESID) ANYLOC_REQUIRE(gamma && resid, "gemm_nt: LS_RESID needs gamma and resid");
  EpiParams ep{epilogue, bias, gamma, resid, (float*)out, (float*)out_lo, ldo};
  ep.alpha = alpha;
  ep.out_fmt = out_dtype;
  return gemm_dispatch(a_hi, a_lo, lda, b_hi, b_lo, ldb, M, N, K, ep, engine, in_dtype, (cudaStream_t)stream);
}

// internal (topk.cu): plain-store GEMM with a device gate; not part of the public header
extern "C" int anyloc_gemm_nt_gated(const void* a_hi, const void* a_lo, int lda, const void* b_hi, const void* b_lo, int ldb,
                                    int M, int N, int K, int in_dtype, float alpha, float* out, int ldo, const int* gate,
                                    void* stream) {
  EpiParams ep{ANYLOC_EPI_BIAS, nullptr, nullptr, nullptr, out, nullptr, ldo};
  ep.alpha = alpha;
  ep.gate = gate;
  cudaStream_t st = (cudaStream_t)stream;
  const int fmt = in_dtype == ANYLOC_PAIR_F16 ? ANYLOC_PAIR_F16 : ANYLOC_PAIR_TF32;
  if (gate) {      // conditional fallback: tensor-core engine only (its kernels test the device flag), nothing recorded
    if (!gemm_tc_supported(a_hi, a_lo, lda, b_hi, b_lo, ldb, M, N, K, ep, fmt)) {
      set_error("gemm_nt_gated: shape outside the tensor-core engine's contract");
      return ANYLOC_ERR_UNSUPPORTED;
    }
    return gemm_tc_launch(a_hi, a_lo, lda, b_hi, b_lo, ldb, M, N, K, ep, fmt, st);
  }
  return gemm_dispatch(a_hi, a_lo, lda, b_hi, b_lo, ldb, M, N, K, ep, ANYLOC_GEMM_AUTO, fmt, st);
}

extern "C" int anyloc_split_tf32(const float* x, float* hi, float* lo, size_t n, void* stream) {
  ANYLOC_REQUIRE(x && hi && lo, "split_tf32: null pointer");
  if (n == 0) return ANYLOC_OK;
  return launch_split(x, hi, lo, n, (cudaStream_t)stream);
}

extern "C" int anyloc_split_f16(const float* x, void* hi, void* lo, size_t n, float scale, void* stream) {
  ANYLOC_REQUIRE(x && hi && lo, "split_f16: null pointer");
  if (n == 0) return ANYLOC_OK;
  return launch_split_f16(x, hi, lo, n, scale, (cudaStream_t)stream);
}

extern "C" int anyloc_split_bf16(const float* x, void* y, size_t n, void* stream) {
  ANYLOC_REQUIRE(x && y, "split_bf16: null pointer");
  if (n == 0) return ANYLOC_OK;
  return launch_split_bf16(x, y, n, (cudaStream_t)stream);
}

extern "C" int anyloc_layernorm_split(const float* x, const float* w, const float* b, int M, int D,
                                      float eps, void* y_hi, void* y_lo, int out_dtype, void* stream) {
  const FormatInfo& f = format_info(out_dtype);
  const bool has_lo = f.lo || f.row_scales;      // y_lo: the lo array, or e4m3's row scales
  ANYLOC_REQUIRE(x && w && b && y_hi && (y_lo || !has_lo), "layernorm: null pointer");
  ANYLOC_REQUIRE(has_lo || !y_lo, "layernorm: the %s output has no lo array (y_lo must be NULL)", f.name);
  ANYLOC_REQUIRE(M >= 0 && D > 0 && D % 4 == 0 && D <= 2048, "layernorm: M=%d D=%d (M >= 0, D a multiple of 4 in "
                 "[4, 2048])", M, D);
  // float4 loads of x, w and b; y_hi and y_lo are stored 4 elements at a time (16, 8 or 4 bytes); e4m3's y_lo holds
  // fp32 scales
  const uintptr_t hi_align = 4 * f.esz - 1, lo_align = f.row_scales ? 3 : hi_align;
  ANYLOC_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(b)) &
                  15) == 0 && (reinterpret_cast<uintptr_t>(y_hi) & hi_align) == 0 &&
                 (reinterpret_cast<uintptr_t>(y_lo) & lo_align) == 0,
                 "layernorm: x, w and b must be 16-byte aligned, y_hi and y_lo aligned to 4 of their elements (fp8: "
                 "y_hi 4-byte, y_lo 4-byte)");
  if (M == 0) return ANYLOC_OK;
  return launch_layernorm(x, w, b, M, D, eps, y_hi, y_lo, out_dtype, (cudaStream_t)stream);
}

extern "C" float anyloc_fp8_scale(float amax) { return pow2f(fp8_scale_exp(amax)); }

extern "C" int anyloc_quantize_fp8_rows(const void* x, int M, int K, void* q, float* scales, void* stream) {
  ANYLOC_REQUIRE(x && q && scales, "quantize_fp8_rows: null pointer");
  ANYLOC_REQUIRE(M >= 0 && K > 0 && K % 8 == 0, "quantize_fp8_rows: M=%d K=%d (K a positive multiple of 8)", M, K);
  ANYLOC_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(q) & 7) == 0 &&
                 (reinterpret_cast<uintptr_t>(scales) & 3) == 0,
                 "quantize_fp8_rows: x must be 16-byte, q 8-byte and scales 4-byte aligned");
  if (M == 0) return ANYLOC_OK;
  return launch_quantize_fp8_rows(x, M, K, q, scales, (cudaStream_t)stream);
}

extern "C" int anyloc_quantize_fp8_tensor(const float* x, void* q, size_t n, float* scale_host, void* stream) {
  ANYLOC_REQUIRE(x && q && scale_host, "quantize_fp8_tensor: null pointer");
  ANYLOC_REQUIRE(n > 0, "quantize_fp8_tensor: empty tensor");
  return launch_quantize_fp8_tensor(x, n, q, scale_host, (cudaStream_t)stream);
}

// qkv_f16: qkv_{hi,lo} already hold fp16 pairs of 8*x for all three thirds (the ViT's qkv epilogue wrote them).
static int attention_dispatch(const float* qkv_hi, const float* qkv_lo, int B, int T, int D, int heads, void* o_hi,
                              void* o_lo, bool out_f16, int engine, cudaStream_t st, bool qkv_f16 = false) {
  ProfScope ps(PC_ATTENTION, st, 4.0 * B * (double)T * T * D);
  const bool tc_ok = qkv_lo != nullptr && (D % 4) == 0 &&
                     (reinterpret_cast<uintptr_t>(qkv_hi) & 15) == 0 && (reinterpret_cast<uintptr_t>(qkv_lo) & 15) == 0;
  if (engine == ANYLOC_GEMM_TC3 && !tc_ok) {
    set_error("attention: the tensor-core engine needs the (hi,lo) qkv pair, 16-byte aligned");
    return ANYLOC_ERR_UNSUPPORTED;
  }
  if (engine == ANYLOC_GEMM_SIMT || !tc_ok)
    return attention_launch(qkv_hi, qkv_lo, B, T, D, heads, o_hi, o_lo, out_f16, st);
  if (out_f16) {     // fp16-pair precision: operands are fp16 pairs too (inside the ViT the qkv epilogue wrote them)
    if (qkv_f16) return attention_tc_launch(qkv_hi, qkv_lo, B, T, D, heads, o_hi, o_lo, ANYLOC_PAIR_F16, st);
    return attention_tc16_standalone(qkv_hi, qkv_lo, B, T, D, heads, o_hi, o_lo, st);
  }
  return attention_tc_launch(qkv_hi, qkv_lo, B, T, D, heads, o_hi, o_lo, ANYLOC_PAIR_TF32, st);
}

extern "C" int anyloc_attention(const float* qkv_hi, const float* qkv_lo, int B, int T, int D, int heads,
                                void* o_hi, void* o_lo, int out_dtype, int engine, void* stream) {
  const FormatInfo& f = format_info(out_dtype);
  if (f.tc_only && f.out == out_dtype) {     // a tensor-core-only format in and out: one the qkv epilogue writes
    ANYLOC_REQUIRE(qkv_hi && o_hi, "attention: null pointer");
    if (f.lo)
      ANYLOC_REQUIRE(qkv_lo && o_lo, "attention: the %s format needs qkv_lo and o_lo", f.name);
    else
      ANYLOC_REQUIRE(!qkv_lo && !o_lo, "attention: the %s format has no lo arrays (qkv_lo, o_lo must be NULL)", f.name);
    ANYLOC_REQUIRE(D == heads * 64, "attention: head_dim must be 64 (D=%d heads=%d)", D, heads);
    ANYLOC_REQUIRE_ALIGNED(o_hi, 8, "attention", "o_hi", "64-bit stores of the tensor-core epilogue");
    ANYLOC_REQUIRE_ALIGNED(o_lo, 8, "attention", "o_lo", "64-bit stores of the tensor-core epilogue");
    if (engine == ANYLOC_GEMM_SIMT || (reinterpret_cast<uintptr_t>(qkv_hi) & 15) != 0 ||
        (reinterpret_cast<uintptr_t>(qkv_lo) & 15) != 0) {
      set_error("attention: the %s format runs on the tensor-core engine only, with a 16-byte aligned qkv", f.name);
      return ANYLOC_ERR_UNSUPPORTED;
    }
    if (B == 0 || T == 0) return ANYLOC_OK;
    ProfScope ps(PC_ATTENTION, (cudaStream_t)stream, 4.0 * B * (double)T * T * D);
    return attention_tc_launch(qkv_hi, qkv_lo, B, T, D, heads, o_hi, o_lo, out_dtype, (cudaStream_t)stream);
  }
  ANYLOC_REQUIRE(qkv_hi && o_hi && o_lo, "attention: null pointer");
  ANYLOC_REQUIRE(D == heads * 64, "attention: head_dim must be 64 (D=%d heads=%d)", D, heads);
  ANYLOC_REQUIRE_ALIGNED(o_hi, 8, "attention", "o_hi", "64-bit stores of the tensor-core epilogue");
  ANYLOC_REQUIRE_ALIGNED(o_lo, 8, "attention", "o_lo", "64-bit stores of the tensor-core epilogue");
  if (B == 0 || T == 0) return ANYLOC_OK;
  return attention_dispatch(qkv_hi, qkv_lo, B, T, D, heads, o_hi, o_lo, out_dtype == ANYLOC_PAIR_F16, engine,
                            (cudaStream_t)stream);
}

// The attention table of n packed images (image i: rows [row0[i], row0[i] + len[i])): entries longest first, so the
// longest key loops start first, ties in input order; each entry's first 64-query tile.  Returns the tile count.  The
// ViT's list calls and anyloc_attention_varlen both build their tables here.
static int varlen_attn_table(int n, const int* row0, const int* len, VarlenAttnTable* t) {
  int order[kVarlenMaxB];
  for (int i = 0; i < n; ++i) order[i] = i;
  std::stable_sort(order, order + n, [&](int a, int b) { return len[a] > len[b]; });
  int tiles = 0;
  t->n = n;
  for (int k = 0; k < n; ++k) {
    const int i = order[k];
    t->tile0[k] = tiles; t->row0[k] = row0[i]; t->len[k] = len[i];
    tiles += cdiv(len[i], 64);
  }
  return tiles;
}

extern "C" int anyloc_attention_varlen(const void* qkv_hi, const void* qkv_lo, int n, const int32_t* row0,
                                       const int32_t* len, int D, int heads, void* o_hi, void* o_lo, int fmt,
                                       void* stream) {
  ANYLOC_REQUIRE(fmt == ANYLOC_PAIR_TF32 || fmt == ANYLOC_PAIR_F16 || fmt == ANYLOC_PAIR_BF16 ||
                 fmt == ANYLOC_PAIR_F16X1 || fmt == ANYLOC_PAIR_BF16X3, "attention_varlen: bad fmt %d", fmt);
  const FormatInfo& f = format_info(fmt);
  ANYLOC_REQUIRE(qkv_hi && o_hi && row0 && len, "attention_varlen: null pointer");
  if (!f.lo)
    ANYLOC_REQUIRE(!qkv_lo && !o_lo, "attention_varlen: the %s format has no lo arrays (qkv_lo, o_lo must be NULL)",
                   f.name);
  else
    ANYLOC_REQUIRE(qkv_lo && o_lo, "attention_varlen: the pair formats need qkv_lo and o_lo");
  ANYLOC_REQUIRE(n >= 1 && n <= ANYLOC_VIT_VARLEN_MAX_B, "attention_varlen: n=%d out of range [1,%d]", n,
                 ANYLOC_VIT_VARLEN_MAX_B);
  ANYLOC_REQUIRE(heads >= 1 && D == heads * 64, "attention_varlen: head_dim must be 64 (D=%d heads=%d)", D, heads);
  int by_row[ANYLOC_VIT_VARLEN_MAX_B];
  for (int i = 0; i < n; ++i) {
    ANYLOC_REQUIRE(len[i] >= 1 && row0[i] >= 0 && (int64_t)row0[i] + len[i] <= INT32_MAX,
                   "attention_varlen: image %d has row0=%d len=%d", i, row0[i], len[i]);
    by_row[i] = i;
  }
  std::sort(by_row, by_row + n, [&](int a, int b) { return row0[a] < row0[b]; });
  for (int k = 1; k < n; ++k)
    ANYLOC_REQUIRE(row0[by_row[k - 1]] + len[by_row[k - 1]] <= row0[by_row[k]],
                   "attention_varlen: images %d and %d overlap", by_row[k - 1], by_row[k]);
  ANYLOC_REQUIRE_ALIGNED(o_hi, 8, "attention_varlen", "o_hi", "64-bit stores of the tensor-core epilogue");
  ANYLOC_REQUIRE_ALIGNED(o_lo, 8, "attention_varlen", "o_lo", "64-bit stores of the tensor-core epilogue");
  if ((reinterpret_cast<uintptr_t>(qkv_hi) & 15) != 0 || (reinterpret_cast<uintptr_t>(qkv_lo) & 15) != 0) {
    set_error("attention_varlen: qkv_hi and qkv_lo must be 16-byte aligned (TMA and cp.async)");
    return ANYLOC_ERR_UNSUPPORTED;
  }
  VarlenAttnTable tab;
  const int tiles = varlen_attn_table(n, row0, len, &tab);
  double flops = 0.0;
  for (int i = 0; i < n; ++i) flops += 4.0 * (double)len[i] * len[i] * D;
  ProfScope ps(PC_ATTENTION, (cudaStream_t)stream, flops);
  return attention_tc_varlen_launch(qkv_hi, qkv_lo, tab, tiles, D, heads, o_hi, o_lo, fmt, (cudaStream_t)stream);
}

extern "C" int anyloc_l2_normalize_rows(const float* x, int64_t rows, int D, int64_t ld_in, float* y,
                                        void* stream) {
  ANYLOC_REQUIRE(x && y && D % 4 == 0 && ld_in % 4 == 0, "l2_normalize_rows: bad args");
  ANYLOC_REQUIRE(rows >= 0 && D > 0 && ld_in >= D, "l2_normalize_rows: rows=%lld D=%d ld_in=%lld (rows >= 0, D > 0, "
                 "ld_in >= D)", (long long)rows, D, (long long)ld_in);
  ANYLOC_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0,
                 "l2_normalize_rows: x and y must be 16-byte aligned (float4 access)");
  if (rows == 0) return ANYLOC_OK;
  return launch_l2norm(x, rows, D, ld_in, y, (cudaStream_t)stream);
}

// ------------------------------------------------------------------ streamed PCA fit (pca.cu)
extern "C" size_t anyloc_pca_colsum_workspace_bytes(int64_t rows, int cols) {
  return pca_colsum_workspace_bytes(rows, cols);
}

extern "C" int anyloc_pca_colsum(const float* x, int64_t ld, int64_t rows, int cols, double* sum, void* ws,
                                 size_t ws_bytes, void* stream) {
  ANYLOC_REQUIRE(x && sum && ws, "pca_colsum: null pointer");
  // the PCA kernels read and write one element at a time: natural alignment is the whole contract, for any ld
  ANYLOC_REQUIRE_ALIGNED(x, 4, "pca_colsum", "x", "fp32 access");
  ANYLOC_REQUIRE_ALIGNED(sum, 8, "pca_colsum", "sum", "fp64 access");
  ANYLOC_REQUIRE_ALIGNED(ws, 8, "pca_colsum", "ws", "fp64 access");
  ANYLOC_REQUIRE(rows >= 0 && cols >= 0 && ld >= cols, "pca_colsum: rows=%lld cols=%d ld=%lld (rows >= 0, cols >= 0, "
                 "ld >= cols)", (long long)rows, cols, (long long)ld);
  if (ws_bytes < pca_colsum_workspace_bytes(rows, cols)) {
    set_error("pca_colsum: workspace too small (%zu given, %zu needed)", ws_bytes,
              pca_colsum_workspace_bytes(rows, cols));
    return ANYLOC_ERR_WORKSPACE;
  }
  return pca_colsum_launch(x, ld, rows, cols, sum, (double*)ws, (cudaStream_t)stream);
}

extern "C" int anyloc_pca_accumulate(int mode, const float* x, int64_t ld, int64_t rows, int cols, const double* mu,
                                     const double* u, int64_t ld_u, int k, double* out, int64_t ld_out, void* stream) {
  ANYLOC_REQUIRE(mode == ANYLOC_PCA_COV || mode == ANYLOC_PCA_GRAM || mode == ANYLOC_PCA_VT ||
                 mode == ANYLOC_PCA_SKETCH, "pca_accumulate: unknown mode %d", mode);
  const bool uses_u = mode == ANYLOC_PCA_VT || mode == ANYLOC_PCA_SKETCH;
  ANYLOC_REQUIRE(x && mu && out && (!uses_u || u || k == 0), "pca_accumulate: null pointer");
  ANYLOC_REQUIRE_ALIGNED(x, 4, "pca_accumulate", "x", "fp32 access");
  ANYLOC_REQUIRE_ALIGNED(mu, 8, "pca_accumulate", "mu", "fp64 access");
  ANYLOC_REQUIRE_ALIGNED(u, 8, "pca_accumulate", "u", "fp64 access");
  ANYLOC_REQUIRE_ALIGNED(out, 8, "pca_accumulate", "out", "fp64 access");
  ANYLOC_REQUIRE(rows >= 0 && cols >= 0 && ld >= cols, "pca_accumulate: rows=%lld cols=%d ld=%lld (rows >= 0, "
                 "cols >= 0, ld >= cols)", (long long)rows, cols, (long long)ld);
  // out [M, N] += sum over K of A(kk, i) B(kk, j)
  int64_t M = cols, N = cols, K = rows;
  if (mode == ANYLOC_PCA_GRAM) {
    M = N = rows;
    K = cols;
  } else if (uses_u) {
    ANYLOC_REQUIRE(k >= 0 && ld_u >= k, "pca_accumulate: k=%d ld_u=%lld (k >= 0, ld_u >= k)", k, (long long)ld_u);
    if (mode == ANYLOC_PCA_VT) {
      M = k;
    } else {
      M = rows;
      N = k;
      K = cols;
    }
  }
  ANYLOC_REQUIRE(M <= (1 << 20) && ld_out >= N, "pca_accumulate: output [%lld, %lld] with ld_out=%lld (at most 2^20 "
                 "rows, ld_out >= columns)", (long long)M, (long long)N, (long long)ld_out);
  return pca_atb_launch(mode, x, ld, mu, u, ld_u, K, (int)M, (int)N, out, ld_out, (cudaStream_t)stream);
}

extern "C" int anyloc_pca_mirror(double* a, int m, int64_t ld, void* stream) {
  ANYLOC_REQUIRE(a && m >= 0 && m <= 65535 * 32 && ld >= m, "pca_mirror: a=%p m=%d ld=%lld (0 <= m <= 65535*32, "
                 "ld >= m)", (void*)a, m, (long long)ld);
  ANYLOC_REQUIRE_ALIGNED(a, 8, "pca_mirror", "a", "fp64 access");
  return pca_mirror_launch(a, m, ld, (cudaStream_t)stream);
}

// ------------------------------------------------------------------ ViT forward
extern "C" int anyloc_vit_patch_k(int patch) { return (int)align_up((size_t)3 * patch * patch, 32); }

namespace {
struct VitBuffers {
  float *pa_hi, *pa_lo, *ptmp, *x, *y_hi, *y_lo, *qkv, *qkv_lo, *h_hi, *h_lo;
  float* qkv32;     // [M, 3D] fp32 rows of a tapped layer's qkv GEMM (null unless the tap list needs them)
  void* h8;         // single e4m3: the FFN hidden layer quantised [M, H] and its row scales [M] (else null)
  float* h8_s;
};
// n_patch patch rows and M token rows in all; the fp32 qkv rows only when `qkv32`.  Each buffer is sized by the format
// that fills it (format_info): the patch rows pa [n_patch, Kp] in the patch embedding's format, the LayerNorm rows y
// [M, D] in pair_dtype, q, k, v [M, 3D] (which also hold the fp32 [M, D] output of a lone q/k/v tap) and the hidden
// layer h [M, H] in the SPLIT output format; lo arrays where the format has them.  The tf32 and fp16 pairs' buffers
// hold fp32 words, so that either pair format fits (the SIMT attention of the fp16-pair precision takes tf32 pairs); the
// bf16 pairs' hold bf16.  Single
// e4m3 adds the LayerNorm rows' scales [M] in y_lo and the e4m3 hidden layer h8 [M, H] with its row scales [M], and its
// attention writes its bf16 output [M, D] into h.
size_t vit_carve(const AnylocVitCfg* c, size_t n_patch, size_t M, bool qkv32, void* ws, size_t ws_bytes,
                 VitBuffers* out) {
  const int D = c->embed_dim, Kp = anyloc_vit_patch_k(c->patch), H = c->ffn_hidden;
  const FormatInfo& f = format_info(c->pair_dtype);
  const FormatInfo &pf = format_info(f.patch), &of = format_info(f.out);
  Workspace w(ws ? ws : (void*)256, ws ? ws_bytes : (size_t)-1 / 2);
  // n elements of fi's arrays: hi, and lo (or null)
  auto take = [&](const FormatInfo& fi, size_t n, float** hi, float** lo) {
    const size_t esz = fi.lo && !fi.tc_only ? sizeof(float) : fi.esz;     // tf32 / fp16 pairs: fp32 words
    *hi = (float*)w.take<uint8_t>(n * esz);
    *lo = fi.lo ? (float*)w.take<uint8_t>(n * esz) : nullptr;
  };
  VitBuffers b;
  take(pf, n_patch * Kp, &b.pa_hi, &b.pa_lo);
  b.ptmp = w.take<float>(n_patch * D);
  b.x = w.take<float>(M * D);
  take(f, M * D, &b.y_hi, &b.y_lo);
  if (f.row_scales) b.y_lo = w.take<float>(M);
  take(of, M * 3 * D, &b.qkv, &b.qkv_lo);
  take(of, M * H, &b.h_hi, &b.h_lo);
  b.h8 = f.row_scales ? w.take<uint8_t>(M * H) : nullptr;
  b.h8_s = f.row_scales ? w.take<float>(M) : nullptr;
  b.qkv32 = qkv32 ? w.take<float>(M * 3 * D) : nullptr;
  if (out) *out = b;
  if (ws && (!b.pa_hi || !b.ptmp || !b.x || !b.y_hi || !b.qkv || !b.h_hi || (qkv32 && !b.qkv32) ||
             (f.row_scales && (!b.y_lo || !b.h8 || !b.h8_s)) ||
             (f.lo && (!b.pa_lo || !b.y_lo || !b.qkv_lo || !b.h_lo))))
    return 0;
  return w.off;
}

// The sequences the attention runs over: B images of T tokens each, or (tab != nullptr) the packed images of a
// variable-length call, n_tiles 64-query tiles in all, whose output rows img maps
struct VitSeqs {
  int B, T;
  const VarlenAttnTable* tab;
  int n_tiles;
  double attn_flops;
  const VarlenImgTable* img;
};

// The taps of one call by layer: bit f of mask[l] set = facet f (ANYLOC_FACET_*) of layer l is returned, into
// out[l][f].  Layers 0..l_max run, each once.
struct TapPlan {
  int l_max;
  std::vector<uint8_t> mask;
  std::vector<std::array<float*, 4>> out;
  bool qkv32;          // some layer's fp32 qkv rows are kept (see vit_trunk)
  int use_cls, norm_descs;
};
int popcount3(int m) { return (m & 1) + ((m >> 1) & 1) + ((m >> 2) & 1); }
// false (with the error text set) on R < 0 or on R > 0 register tokens without their weights
bool registers_ok(const char* fn, const AnylocVitCfg* cfg, const AnylocVitWeights* w) {
  if (cfg->num_registers < 0) { set_error("%s: num_registers=%d < 0", fn, cfg->num_registers); return false; }
  if (cfg->num_registers > 0 && !w->register_tokens) {
    set_error("%s: num_registers=%d but register_tokens is null", fn, cfg->num_registers);
    return false;
  }
  return true;
}
// The operand format of the weights: ANYLOC_OK, or (error text set) ANYLOC_ERR_ARG for a single format's weights with
// a non-null lo matrix or bf16-pair weights with a null one, ANYLOC_ERR_UNSUPPORTED for either on the SIMT engine
int format_check(const char* fn, const AnylocVitCfg* cfg, const AnylocVitWeights* w, int engine) {
  const FormatInfo& f = format_info(cfg->pair_dtype);
  if (!f.tc_only) return ANYLOC_OK;
  bool lo = w->patch_w_lo != nullptr, no_lo = w->patch_w_lo == nullptr;
  for (int l = 0; l < cfg->depth && w->blocks; ++l) {
    const AnylocVitBlock& b = w->blocks[l];
    lo = lo || b.qkv_w_lo || b.proj_w_lo || b.in_w_lo || b.out_w_lo;
    no_lo = no_lo || !b.qkv_w_lo || !b.proj_w_lo || !b.in_w_lo || !b.out_w_lo;
  }
  if (f.lo && no_lo) {
    set_error("%s: pair_dtype %s takes %s weights; every *_w_lo must be non-NULL", fn, f.id, f.name);
    return ANYLOC_ERR_ARG;
  }
  if (!f.lo && lo) {
    set_error("%s: pair_dtype %s takes %s block weights and %s patch weights; every *_w_lo must be NULL", fn, f.id,
              f.name, format_info(f.patch).name);
    return ANYLOC_ERR_ARG;
  }
  if (engine == ANYLOC_GEMM_SIMT) {
    set_error("%s: the %s format runs on the tensor-core engine only (gemm_engine auto or tc3, not simt)", fn, f.name);
    return ANYLOC_ERR_UNSUPPORTED;
  }
  return ANYLOC_OK;
}
// The alignment of every device pointer a forward reads or writes: ANYLOC_OK, or ANYLOC_ERR_ARG naming the pointer.
// Whatever reaches the GEMM (weights, biases, LayerScale gammas) needs gemm_tc_supported's 16 bytes, so that an
// accepted pointer never moves a GEMM off the tensor cores; the LayerNorm gains and biases are float4 loads, the outputs
// float4 stores; ws needs what its strictest carved buffer needs (TMA), since Workspace::take aligns offsets, not
// addresses.  The images, positional tables, cls and register tokens are read one fp32 at a time.  n_img images img[i]
// and tables pos[i] (named img / pos_embed unless `list`), n_taps outputs taps[i].out (named out unless `taps_named`).
int vit_alignment(const char* fn, const AnylocVitCfg* cfg, const AnylocVitWeights* w, int n_img,
                  const float* const* img, const float* const* pos, bool list, const AnylocVitTap* taps, int n_taps,
                  bool taps_named, const void* ws) {
  char name[64];
  const char* gemm = "tensor-core GEMM operand";
  ANYLOC_REQUIRE_ALIGNED(ws, 16, fn, "ws", "TMA and float4 access of the buffers carved from it");
  ANYLOC_REQUIRE_ALIGNED(w->patch_w_hi, 16, fn, "w.patch_w_hi", gemm);
  ANYLOC_REQUIRE_ALIGNED(w->patch_w_lo, 16, fn, "w.patch_w_lo", gemm);
  ANYLOC_REQUIRE_ALIGNED(w->patch_b, 16, fn, "w.patch_b", gemm);
  ANYLOC_REQUIRE_ALIGNED(w->cls_token, 4, fn, "w.cls_token", "fp32 access");
  if (cfg->num_registers > 0) ANYLOC_REQUIRE_ALIGNED(w->register_tokens, 4, fn, "w.register_tokens", "fp32 access");
  for (int l = 0; l < cfg->depth && w->blocks; ++l) {
    const AnylocVitBlock& b = w->blocks[l];
    const struct { const void* p; const char* field; int bytes; const char* why; } ptrs[] = {
        {b.ln1_w, "ln1_w", 16, "float4 access"}, {b.ln1_b, "ln1_b", 16, "float4 access"},
        {b.qkv_w_hi, "qkv_w_hi", 16, gemm}, {b.qkv_w_lo, "qkv_w_lo", 16, gemm}, {b.qkv_b, "qkv_b", 16, gemm},
        {b.proj_w_hi, "proj_w_hi", 16, gemm}, {b.proj_w_lo, "proj_w_lo", 16, gemm}, {b.proj_b, "proj_b", 16, gemm},
        {b.ls1, "ls1", 16, gemm}, {b.ln2_w, "ln2_w", 16, "float4 access"}, {b.ln2_b, "ln2_b", 16, "float4 access"},
        {b.in_w_hi, "in_w_hi", 16, gemm}, {b.in_w_lo, "in_w_lo", 16, gemm}, {b.in_b, "in_b", 16, gemm},
        {b.out_w_hi, "out_w_hi", 16, gemm}, {b.out_w_lo, "out_w_lo", 16, gemm}, {b.out_b, "out_b", 16, gemm},
        {b.ls2, "ls2", 16, gemm}};
    for (const auto& q : ptrs) {
      snprintf(name, sizeof(name), "blocks[%d].%s", l, q.field);
      ANYLOC_REQUIRE_ALIGNED(q.p, q.bytes, fn, name, q.why);
    }
  }
  for (int i = 0; i < n_img; ++i) {
    snprintf(name, sizeof(name), list ? "img[%d]" : "img", i);
    ANYLOC_REQUIRE_ALIGNED(img[i], 4, fn, name, "fp32 access");
    snprintf(name, sizeof(name), list ? "pos_embed[%d]" : "pos_embed", i);
    ANYLOC_REQUIRE_ALIGNED(pos[i], 4, fn, name, "fp32 access");
  }
  for (int i = 0; i < n_taps; ++i) {
    snprintf(name, sizeof(name), taps_named ? "taps[%d].out" : "out", i);
    ANYLOC_REQUIRE_ALIGNED(taps[i].out, 16, fn, name, "float4 stores");
  }
  return ANYLOC_OK;
}
// Returns false (with the error text set) on an empty list, a bad layer or facet, a repeated tap or (need_out) a null
// output.
bool tap_plan(const char* fn, const AnylocVitCfg* cfg, const AnylocVitTap* taps, int n_taps, bool need_out,
              TapPlan* p) {
  if (!taps || n_taps < 1) { set_error("%s: no taps", fn); return false; }
  p->l_max = -1;
  p->mask.assign(cfg->depth, 0);
  p->out.assign(cfg->depth, std::array<float*, 4>{});
  for (int i = 0; i < n_taps; ++i) {
    const int l = taps[i].layer, f = taps[i].facet;
    if (l < 0 || l >= cfg->depth) { set_error("%s: tap %d: layer %d out of range [0,%d)", fn, i, l, cfg->depth); return false; }
    if (f < ANYLOC_FACET_QUERY || f > ANYLOC_FACET_TOKEN) { set_error("%s: tap %d: bad facet %d", fn, i, f); return false; }
    if (p->mask[l] & (1 << f)) { set_error("%s: tap %d: layer %d facet %d is requested twice", fn, i, l, f); return false; }
    if (need_out && !taps[i].out) { set_error("%s: tap %d: null output", fn, i); return false; }
    p->mask[l] |= 1 << f;
    p->out[l][f] = taps[i].out;
    p->l_max = std::max(p->l_max, l);
  }
  // the fp32 rows are needed at a q/k/v-tapped layer the forward continues through, and at the last layer when it
  // returns two or three of q, k, v (one alone takes that third's own GEMM)
  const int last = p->mask[p->l_max];
  p->qkv32 = (last & 8) ? (last & 7) != 0 : popcount3(last) >= 2;
  for (int l = 0; l < p->l_max; ++l) p->qkv32 = p->qkv32 || (p->mask[l] & 7) != 0;
  return true;
}
}  // namespace

extern "C" size_t anyloc_vit_workspace_bytes(const AnylocVitCfg* cfg, int B, int H, int W) {
  if (!cfg || cfg->num_registers < 0 || B <= 0 || H < cfg->patch || W < cfg->patch) return 0;
  const size_t N = (size_t)(H / cfg->patch) * (W / cfg->patch);
  return vit_carve(cfg, B * N, B * (N + 1 + cfg->num_registers), false, nullptr, 0, nullptr) + 4096;
}

extern "C" size_t anyloc_vit_taps_workspace_bytes(const AnylocVitCfg* cfg, int B, int H, int W, const AnylocVitTap* taps,
                                                  int n_taps) {
  TapPlan tp;
  if (!cfg || cfg->num_registers < 0 || B <= 0 || H < cfg->patch || W < cfg->patch ||
      !tap_plan("vit_taps_workspace_bytes", cfg, taps, n_taps, false, &tp))
    return 0;
  const size_t N = (size_t)(H / cfg->patch) * (W / cfg->patch);
  return vit_carve(cfg, B * N, B * (N + 1 + cfg->num_registers), tp.qkv32, nullptr, 0, nullptr) + 4096;
}

// the facet slice of the M token rows in src (row stride ld) -> out
static int facet_out(const VitSeqs& sq, int M, const float* src, int64_t ld, int D, const TapPlan& tp, float* out,
                     cudaStream_t st) {
  if (sq.img)
    return launch_facet_out_varlen(src, *sq.img, M - (tp.use_cls ? 0 : sq.B), ld, 0, D, tp.use_cls, tp.norm_descs, out,
                                   st);
  return launch_facet_out(src, sq.B, sq.T, ld, 0, D, tp.use_cls, tp.norm_descs, out, st);
}

// the fp32 qkv rows of layer l in bf.qkv32 -> the facets of l the plan asks for and, unless attn_fmt is FMT_NONE, the
// attention's operands in bf.qkv / bf.qkv_lo in the format attn_fmt
static int qkv_tap(const AnylocVitCfg* c, const VitBuffers& bf, int M, const VitSeqs& sq, const TapPlan& tp, int l,
                   int attn_fmt, cudaStream_t st) {
  const int D = c->embed_dim, m = tp.mask[l];
  const QkvTapOuts o{{(m & 1) ? tp.out[l][0] : nullptr, (m & 2) ? tp.out[l][1] : nullptr,
                      (m & 4) ? tp.out[l][2] : nullptr}};
  const bool pairs = attn_fmt != FMT_NONE;
  const FormatInfo& f = format_info(attn_fmt);
  const double rows_out = (double)M - (tp.use_cls ? 0 : sq.B);
  const double bytes = 12.0 * M * D + (pairs ? 3.0 * f.esz * (f.lo ? 2 : 1) * M * D : 0.0) +
                       4.0 * rows_out * D * popcount3(m);
  ProfScope ps(PC_VIT_MISC, st, bytes);
  return launch_qkv_tap(bf.qkv32, M, sq.T, sq.img, D, attn_fmt, pairs ? bf.qkv : nullptr, pairs ? bf.qkv_lo : nullptr,
                        o, tp.use_cls, tp.norm_descs, st);
}

// One transformer block over the M token rows in bf.x, in place.  With tp (layer l has q/k/v taps) the qkv GEMM
// writes fp32 rows and the tap kernel derives the attention's operands and the tapped facets from them.
static int vit_block(const AnylocVitCfg* c, const AnylocVitBlock& wb, const VitBuffers& bf, int M, const VitSeqs& sq,
                     int engine, cudaStream_t st, const TapPlan* tp = nullptr, int l = 0) {
  const int D = c->embed_dim, Hf = c->ffn_hidden;
  const int fmt = c->pair_dtype;
  const FormatInfo& f = format_info(fmt);
  int rc;
  const double ln_bytes = (4.0 + f.esz * (f.lo ? 2 : 1)) * M * D;
  { ProfScope ps(PC_LAYERNORM, st, ln_bytes);
    if ((rc = launch_layernorm(bf.x, wb.ln1_w, wb.ln1_b, M, D, 1e-6f, bf.y_hi, bf.y_lo, fmt, st))) return rc; }
  // q, k and v leave the qkv GEMM row-major through the plain split epilogue, in the attention's operand format: the
  // SPLIT output format, except that the SIMT attention of the fp16-pair precision takes tf32 pairs
  const int attn_fmt = fmt == ANYLOC_PAIR_F16 && engine == ANYLOC_GEMM_SIMT ? ANYLOC_PAIR_TF32 : f.out;
  if (tp) {
    EpiParams e_qkv{ANYLOC_EPI_BIAS, wb.qkv_b, nullptr, nullptr, bf.qkv32, nullptr, 3 * D};
    e_qkv.alpha = wb.qkv_alpha;
    if ((rc = gemm_dispatch(bf.y_hi, bf.y_lo, D, wb.qkv_w_hi, wb.qkv_w_lo, D, M, 3 * D, D, e_qkv, engine, fmt, st))) return rc;
    if ((rc = qkv_tap(c, bf, M, sq, *tp, l, attn_fmt, st))) return rc;
  } else {
    EpiParams e_qkv{ANYLOC_EPI_BIAS_SPLIT, wb.qkv_b, nullptr, nullptr, bf.qkv, bf.qkv_lo, 3 * D};
    e_qkv.out_fmt = attn_fmt;
    e_qkv.alpha = wb.qkv_alpha;
    if ((rc = gemm_dispatch(bf.y_hi, bf.y_lo, D, wb.qkv_w_hi, wb.qkv_w_lo, D, M, 3 * D, D, e_qkv, engine, fmt, st))) return rc;
  }
  // single e4m3: the bf16 attention output goes to h and is quantised to the proj GEMM's e4m3 rows and their scales
  float* o_hi = f.row_scales ? bf.h_hi : bf.y_hi;
  float* o_lo = format_info(attn_fmt).lo ? bf.y_lo : nullptr;
  if (sq.tab) {
    ProfScope ps(PC_ATTENTION, st, sq.attn_flops);
    if ((rc = attention_tc_varlen_launch(bf.qkv, bf.qkv_lo, *sq.tab, sq.n_tiles, D, c->num_heads, o_hi, o_lo, attn_fmt,
                                         st)))
      return rc;
  } else if (f.tc_only) {
    ProfScope ps(PC_ATTENTION, st, 4.0 * sq.B * (double)sq.T * sq.T * D);
    if ((rc = attention_tc_launch(bf.qkv, bf.qkv_lo, sq.B, sq.T, D, c->num_heads, o_hi, o_lo, attn_fmt, st))) return rc;
  } else if ((rc = attention_dispatch(bf.qkv, bf.qkv_lo, sq.B, sq.T, D, c->num_heads, bf.y_hi, bf.y_lo,
                                      fmt == ANYLOC_PAIR_F16, engine, st, attn_fmt == ANYLOC_PAIR_F16))) {
    return rc;
  }
  if (f.row_scales) {
    ProfScope ps(PC_VIT_MISC, st, 3.0 * M * D);
    if ((rc = launch_quantize_fp8_rows(bf.h_hi, M, D, bf.y_hi, bf.y_lo, st))) return rc;
  }
  EpiParams e_proj{ANYLOC_EPI_LS_RESID, wb.proj_b, wb.ls1, bf.x, bf.x, nullptr, D};
  e_proj.alpha = wb.proj_alpha;
  if ((rc = gemm_dispatch(bf.y_hi, bf.y_lo, D, wb.proj_w_hi, wb.proj_w_lo, D, M, D, D, e_proj, engine, fmt, st))) return rc;
  { ProfScope ps(PC_LAYERNORM, st, ln_bytes);
    if ((rc = launch_layernorm(bf.x, wb.ln2_w, wb.ln2_b, M, D, 1e-6f, bf.y_hi, bf.y_lo, fmt, st))) return rc; }
  EpiParams e_in{c->ffn_kind == ANYLOC_FFN_MLP ? ANYLOC_EPI_GELU_SPLIT : ANYLOC_EPI_SWIGLU_SPLIT, wb.in_b, nullptr,
                 nullptr, bf.h_hi, bf.h_lo, Hf};
  e_in.alpha = wb.in_alpha; e_in.out_fmt = f.out;
  const int n_in = c->ffn_kind == ANYLOC_FFN_MLP ? Hf : 2 * Hf;
  if ((rc = gemm_dispatch(bf.y_hi, bf.y_lo, D, wb.in_w_hi, wb.in_w_lo, D, M, n_in, D, e_in, engine, fmt, st))) return rc;
  if (f.row_scales) {
    ProfScope ps(PC_VIT_MISC, st, 3.0 * M * Hf);
    if ((rc = launch_quantize_fp8_rows(bf.h_hi, M, Hf, bf.h8, bf.h8_s, st))) return rc;
  }
  EpiParams e_out{ANYLOC_EPI_LS_RESID, wb.out_b, wb.ls2, bf.x, bf.x, nullptr, D};
  e_out.alpha = wb.out_alpha;
  return gemm_dispatch(f.row_scales ? bf.h8 : bf.h_hi, f.row_scales ? bf.h8_s : bf.h_lo, Hf, wb.out_w_hi,
                       wb.out_w_lo, Hf, M, D, Hf, e_out, engine, fmt, st);
}

// Blocks 0..l_max over the M assembled token rows in bf.x, each run once, writing every tap of the plan:
//  - a layer with q/k/v taps that the forward continues through runs its qkv GEMM into fp32 rows (bf.qkv32), from
//    which the tap kernel writes the attention's operand pairs and the tapped facets; other layers run unchanged;
//  - a token tap of layer l is the facet slice of x after block l, before block l + 1 overwrites it;
//  - the last layer without a token tap exits early after norm1 and what its q/k/v taps need: one facet alone is that
//    third's own N = D GEMM and the facet slice, two or three are the N = 3D GEMM and the tap kernel without pairs.
static int vit_trunk(const AnylocVitCfg* cfg, const AnylocVitWeights* w, const VitBuffers& bf, int M, const VitSeqs& sq,
                     const TapPlan& tp, int gemm_engine, cudaStream_t st) {
  const int D = cfg->embed_dim, fmt = cfg->pair_dtype;
  const size_t wsz = format_info(fmt).esz;
  int rc;
  for (int l = 0; l <= tp.l_max; ++l) {
    const AnylocVitBlock& wb = w->blocks[l];
    const int qkv = tp.mask[l] & 7;
    const bool token = (tp.mask[l] & 8) != 0;
    if (l == tp.l_max && !token) {
      if ((rc = launch_layernorm(bf.x, wb.ln1_w, wb.ln1_b, M, D, 1e-6f, bf.y_hi, bf.y_lo, fmt, st))) return rc;
      if (popcount3(qkv) == 1) {
        const int facet = qkv == 1 ? 0 : qkv == 2 ? 1 : 2;
        const size_t woff = (size_t)facet * D * D * wsz;  // bytes: weights are e4m3, __half/bf16 or float
        EpiParams e_f{ANYLOC_EPI_BIAS, wb.qkv_b + (size_t)facet * D, nullptr, nullptr, bf.qkv, nullptr, D};
        e_f.alpha = wb.qkv_alpha;
        if ((rc = gemm_dispatch(bf.y_hi, bf.y_lo, D, (const char*)wb.qkv_w_hi + woff,
                                wb.qkv_w_lo ? (const char*)wb.qkv_w_lo + woff : nullptr, D, M, D, D, e_f, gemm_engine,
                                fmt, st)))
          return rc;
        return facet_out(sq, M, bf.qkv, D, D, tp, tp.out[l][facet], st);
      }
      EpiParams e_qkv{ANYLOC_EPI_BIAS, wb.qkv_b, nullptr, nullptr, bf.qkv32, nullptr, 3 * D};
      e_qkv.alpha = wb.qkv_alpha;
      if ((rc = gemm_dispatch(bf.y_hi, bf.y_lo, D, wb.qkv_w_hi, wb.qkv_w_lo, D, M, 3 * D, D, e_qkv, gemm_engine, fmt,
                              st)))
        return rc;
      return qkv_tap(cfg, bf, M, sq, tp, l, FMT_NONE, st);
    }
    if ((rc = vit_block(cfg, wb, bf, M, sq, gemm_engine, st, qkv ? &tp : nullptr, l))) return rc;
    if (token && (rc = facet_out(sq, M, bf.x, D, D, tp, tp.out[l][ANYLOC_FACET_TOKEN], st))) return rc;
  }
  return ANYLOC_OK;
}

static int vit_extract_taps(const char* fn, const AnylocVitCfg* cfg, const AnylocVitWeights* w, const float* img, int B,
                            int H, int W, const float* pos_embed, const AnylocVitTap* taps, int n_taps, int use_cls,
                            int norm_descs, void* ws, size_t ws_bytes, int gemm_engine, cudaStream_t st,
                            bool taps_named) {
  ANYLOC_REQUIRE(cfg && w && img && pos_embed && ws, "%s: null pointer", fn);
  ANYLOC_REQUIRE(cfg->patch > 0 && H % cfg->patch == 0 && W % cfg->patch == 0 && H > 0 && W > 0,
                 "%s: H=%d W=%d must be positive multiples of the patch size %d", fn, H, W, cfg->patch);
  TapPlan tp;
  if (!tap_plan(fn, cfg, taps, n_taps, true, &tp)) return ANYLOC_ERR_ARG;
  tp.use_cls = use_cls; tp.norm_descs = norm_descs;
  ANYLOC_REQUIRE(cfg->embed_dim == cfg->num_heads * 64, "%s: head_dim must be 64", fn);
  ANYLOC_REQUIRE(B > 0, "%s: empty batch", fn);
  if (!registers_ok(fn, cfg, w)) return ANYLOC_ERR_ARG;
  int rc;
  if ((rc = format_check(fn, cfg, w, gemm_engine))) return rc;
  if ((rc = vit_alignment(fn, cfg, w, 1, &img, &pos_embed, false, taps, n_taps, taps_named, ws))) return rc;
  const int R = cfg->num_registers;
  const int P = cfg->patch, N = (H / P) * (W / P), T = N + 1 + R, D = cfg->embed_dim, Kp = anyloc_vit_patch_k(P);
  const int M = B * T;
  VitBuffers bf;
  if (!vit_carve(cfg, (size_t)B * N, (size_t)M, tp.qkv32, ws, ws_bytes, &bf)) {
    set_error("%s: workspace too small (%zu given, %zu needed)", fn, ws_bytes,
              vit_carve(cfg, (size_t)B * N, (size_t)M, tp.qkv32, nullptr, 0, nullptr) + 4096);
    return ANYLOC_ERR_WORKSPACE;
  }
  const int fmt = format_info(cfg->pair_dtype).patch;
  if ((rc = launch_im2col(img, B, H, W, P, Kp, bf.pa_hi, bf.pa_lo, fmt, st))) return rc;
  EpiParams e_pe{ANYLOC_EPI_BIAS, w->patch_b, nullptr, nullptr, bf.ptmp, nullptr, D};
  e_pe.alpha = w->patch_alpha;
  if ((rc = gemm_dispatch(bf.pa_hi, bf.pa_lo, Kp, w->patch_w_hi, w->patch_w_lo, Kp, B * N, D, Kp, e_pe,
                          gemm_engine, fmt, st))) return rc;
  if ((rc = launch_assemble(bf.ptmp, w->cls_token, w->register_tokens, pos_embed, B, N, R, D, bf.x, st))) return rc;
  const VitSeqs sq{B, T, nullptr, 0, 0.0, nullptr};
  return vit_trunk(cfg, w, bf, M, sq, tp, gemm_engine, st);
}

extern "C" int anyloc_vit_extract(const AnylocVitCfg* cfg, const AnylocVitWeights* w, const float* img,
                                  int B, int H, int W, const float* pos_embed, int layer, int facet,
                                  int use_cls, int norm_descs, float* out, void* ws, size_t ws_bytes,
                                  int gemm_engine, void* stream) {
  ANYLOC_REQUIRE(cfg && out, "vit_extract: null pointer");
  const AnylocVitTap tap{layer, facet, out};
  return vit_extract_taps("vit_extract", cfg, w, img, B, H, W, pos_embed, &tap, 1, use_cls, norm_descs, ws, ws_bytes,
                          gemm_engine, (cudaStream_t)stream, false);
}

extern "C" int anyloc_vit_extract_taps(const AnylocVitCfg* cfg, const AnylocVitWeights* w, const float* img, int B, int H,
                                       int W, const float* pos_embed, const AnylocVitTap* taps, int n_taps, int use_cls,
                                       int norm_descs, void* ws, size_t ws_bytes, int gemm_engine, void* stream) {
  ANYLOC_REQUIRE(cfg, "vit_extract_taps: null pointer");
  return vit_extract_taps("vit_extract_taps", cfg, w, img, B, H, W, pos_embed, taps, n_taps, use_cls, norm_descs, ws,
                          ws_bytes, gemm_engine, (cudaStream_t)stream, true);
}

namespace {
struct VarlenPlan {
  VarlenImgTable img;         // img.ptr: the images for im2col, then the positional tables for the assembly
  VarlenAttnTable attn;
  int n_patch, n_tok, n_tiles;
  double attn_flops;
};
// Geometry of a variable-length batch, from the host arrays of anyloc_vit_extract_varlen.  Returns false (with the
// error text set) on a bad B or size.
bool varlen_plan(const AnylocVitCfg* cfg, int B, const int32_t* hw, VarlenPlan* p) {
  if (!cfg || cfg->patch <= 0) { set_error("vit_extract_varlen: null or bad config"); return false; }
  if (cfg->num_registers < 0) { set_error("vit_extract_varlen: num_registers=%d < 0", cfg->num_registers); return false; }
  if (B < 1 || B > ANYLOC_VIT_VARLEN_MAX_B) {
    set_error("vit_extract_varlen: B=%d out of range [1,%d]", B, ANYLOC_VIT_VARLEN_MAX_B);
    return false;
  }
  if (!hw) { set_error("vit_extract_varlen: null hw"); return false; }
  const int P = cfg->patch, R = cfg->num_registers;
  int64_t tok = 0, patches = 0;
  double flops = 0.0;
  p->img.n = B; p->img.nreg = R;
  int len[ANYLOC_VIT_VARLEN_MAX_B];
  for (int i = 0; i < B; ++i) {
    const int H = hw[2 * i], W = hw[2 * i + 1];
    if (H <= 0 || W <= 0 || H % P || W % P) {
      set_error("vit_extract_varlen: image %d is %dx%d; H and W must be positive multiples of the patch size %d", i, H,
                W, P);
      return false;
    }
    const int64_t n = (int64_t)(H / P) * (W / P);
    if (tok + n + 1 + R > (int64_t)INT32_MAX / 32) {     // the row-per-warp kernels index threads in 32 bits
      set_error("vit_extract_varlen: too many tokens in one call");
      return false;
    }
    p->img.tok0[i] = (int)tok;
    p->img.gh[i] = H / P; p->img.gw[i] = W / P;
    p->img.ptr[i] = nullptr;
    tok += n + 1 + R; patches += n;
    flops += 4.0 * (double)(n + 1 + R) * (n + 1 + R) * cfg->embed_dim;
    len[i] = (int)n + 1 + R;
  }
  p->n_tiles = varlen_attn_table(B, p->img.tok0, len, &p->attn);
  p->n_patch = (int)patches; p->n_tok = (int)tok; p->attn_flops = flops;
  return true;
}
}  // namespace

extern "C" size_t anyloc_vit_varlen_workspace_bytes(const AnylocVitCfg* cfg, int B, const int32_t* hw) {
  VarlenPlan p;
  if (!varlen_plan(cfg, B, hw, &p)) return 0;
  return vit_carve(cfg, (size_t)p.n_patch, (size_t)p.n_tok, false, nullptr, 0, nullptr) + 4096;
}

extern "C" size_t anyloc_vit_taps_varlen_workspace_bytes(const AnylocVitCfg* cfg, int B, const int32_t* hw,
                                                         const AnylocVitTap* taps, int n_taps) {
  VarlenPlan p;
  TapPlan tp;
  if (!varlen_plan(cfg, B, hw, &p) || !tap_plan("vit_taps_varlen_workspace_bytes", cfg, taps, n_taps, false, &tp))
    return 0;
  return vit_carve(cfg, (size_t)p.n_patch, (size_t)p.n_tok, tp.qkv32, nullptr, 0, nullptr) + 4096;
}

static int vit_extract_taps_varlen(const char* fn, const AnylocVitCfg* cfg, const AnylocVitWeights* w, int B,
                                   const float* const* img, const int32_t* hw, const float* const* pos_embed,
                                   const AnylocVitTap* taps, int n_taps, int use_cls, int norm_descs, void* ws,
                                   size_t ws_bytes, int gemm_engine, cudaStream_t st, bool taps_named) {
  ANYLOC_REQUIRE(cfg && w && img && pos_embed && ws, "%s: null pointer", fn);
  TapPlan tp;
  if (!tap_plan(fn, cfg, taps, n_taps, true, &tp)) return ANYLOC_ERR_ARG;
  tp.use_cls = use_cls; tp.norm_descs = norm_descs;
  ANYLOC_REQUIRE(cfg->embed_dim == cfg->num_heads * 64, "%s: head_dim must be 64", fn);
  if (gemm_engine == ANYLOC_GEMM_SIMT) {
    set_error("%s: needs the tensor-core attention (gemm_engine auto or tc3, not simt)", fn);
    return ANYLOC_ERR_UNSUPPORTED;
  }
  ANYLOC_REQUIRE(gemm_engine == ANYLOC_GEMM_AUTO || gemm_engine == ANYLOC_GEMM_TC3, "%s: bad gemm_engine %d", fn,
                 gemm_engine);
  if (!registers_ok(fn, cfg, w)) return ANYLOC_ERR_ARG;
  int rc;
  if ((rc = format_check(fn, cfg, w, gemm_engine))) return rc;
  VarlenPlan p;
  if (!varlen_plan(cfg, B, hw, &p)) return ANYLOC_ERR_ARG;
  for (int i = 0; i < B; ++i)
    ANYLOC_REQUIRE(img[i] && pos_embed[i], "%s: null image or positional table %d", fn, i);
  if ((rc = vit_alignment(fn, cfg, w, B, img, pos_embed, true, taps, n_taps, taps_named, ws))) return rc;
  const int P = cfg->patch, D = cfg->embed_dim, Kp = anyloc_vit_patch_k(P), M = p.n_tok;
  VitBuffers bf;
  if (!vit_carve(cfg, (size_t)p.n_patch, (size_t)M, tp.qkv32, ws, ws_bytes, &bf)) {
    set_error("%s: workspace too small (%zu given, %zu needed)", fn, ws_bytes,
              vit_carve(cfg, (size_t)p.n_patch, (size_t)M, tp.qkv32, nullptr, 0, nullptr) + 4096);
    return ANYLOC_ERR_WORKSPACE;
  }
  const int fmt = format_info(cfg->pair_dtype).patch;
  for (int i = 0; i < B; ++i) p.img.ptr[i] = img[i];
  if ((rc = launch_im2col_varlen(p.img, p.n_patch, P, Kp, bf.pa_hi, bf.pa_lo, fmt, st))) return rc;
  EpiParams e_pe{ANYLOC_EPI_BIAS, w->patch_b, nullptr, nullptr, bf.ptmp, nullptr, D};
  e_pe.alpha = w->patch_alpha;
  if ((rc = gemm_dispatch(bf.pa_hi, bf.pa_lo, Kp, w->patch_w_hi, w->patch_w_lo, Kp, p.n_patch, D, Kp, e_pe,
                          gemm_engine, fmt, st))) return rc;
  for (int i = 0; i < B; ++i) p.img.ptr[i] = pos_embed[i];
  if ((rc = launch_assemble_varlen(bf.ptmp, w->cls_token, w->register_tokens, p.img, M, D, bf.x, st))) return rc;
  const VitSeqs sq{B, 0, &p.attn, p.n_tiles, p.attn_flops, &p.img};
  return vit_trunk(cfg, w, bf, M, sq, tp, gemm_engine, st);
}

extern "C" int anyloc_vit_extract_varlen(const AnylocVitCfg* cfg, const AnylocVitWeights* w, int B,
                                         const float* const* img, const int32_t* hw, const float* const* pos_embed,
                                         int layer, int facet, int use_cls, int norm_descs, float* out, void* ws,
                                         size_t ws_bytes, int gemm_engine, void* stream) {
  ANYLOC_REQUIRE(cfg && out, "vit_extract_varlen: null pointer");
  const AnylocVitTap tap{layer, facet, out};
  return vit_extract_taps_varlen("vit_extract_varlen", cfg, w, B, img, hw, pos_embed, &tap, 1, use_cls, norm_descs, ws,
                                 ws_bytes, gemm_engine, (cudaStream_t)stream, false);
}

extern "C" int anyloc_vit_extract_taps_varlen(const AnylocVitCfg* cfg, const AnylocVitWeights* w, int B,
                                              const float* const* img, const int32_t* hw,
                                              const float* const* pos_embed, const AnylocVitTap* taps, int n_taps,
                                              int use_cls, int norm_descs, void* ws, size_t ws_bytes, int gemm_engine,
                                              void* stream) {
  ANYLOC_REQUIRE(cfg, "vit_extract_taps_varlen: null pointer");
  return vit_extract_taps_varlen("vit_extract_taps_varlen", cfg, w, B, img, hw, pos_embed, taps, n_taps, use_cls,
                                 norm_descs, ws, ws_bytes, gemm_engine, (cudaStream_t)stream, true);
}
