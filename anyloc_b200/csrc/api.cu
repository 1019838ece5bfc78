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
                   const EpiParams&, bool f16, cudaStream_t);
bool gemm_tc_supported(const void* a_hi, const void* a_lo, int lda, const void* b_hi, const void* b_lo,
                       int ldb, int M, int N, int K, const EpiParams& ep, bool f16);
// vit_ops.cu / attention.cu
int launch_split(const float*, float*, float*, size_t, cudaStream_t);
int launch_split_f16(const float*, void*, void*, size_t, float, cudaStream_t);
int launch_im2col(const float*, int, int, int, int, int, void*, void*, bool, cudaStream_t);
int launch_assemble(const float*, const float*, const float*, const float*, int, int, int, int, float*, cudaStream_t);
int launch_layernorm(const float*, const float*, const float*, int, int, float, void*, void*, bool, cudaStream_t);
int launch_facet_out(const float*, int, int, int64_t, int, int, int, int, float*, cudaStream_t);
int launch_l2norm(const float*, int64_t, int, int64_t, float*, cudaStream_t);
int attention_launch(const float*, const float*, int, int, int, int, void*, void*, bool, cudaStream_t);
int attention_tc_launch(const void*, const void*, int, int, int, int, void*, void*, bool, cudaStream_t);
int attention_tc16_standalone(const float*, const float*, int, int, int, int, void*, void*, cudaStream_t);
int attention_tc_varlen_launch(const void*, const void*, const VarlenAttnTable&, int, int, int, void*, void*, bool,
                               cudaStream_t);
int launch_im2col_varlen(const VarlenImgTable&, int, int, int, void*, void*, bool, cudaStream_t);
int launch_assemble_varlen(const float*, const float*, const float*, const VarlenImgTable&, int, int, float*,
                           cudaStream_t);
int launch_facet_out_varlen(const float*, const VarlenImgTable&, int, int64_t, int, int, int, int, float*, cudaStream_t);
int launch_qkv_tap(const float*, int, int, const VarlenImgTable*, int, int, void*, void*, const QkvTapOuts&, int, int,
                   cudaStream_t);

static int gemm_dispatch(const void* a_hi, const void* a_lo, int lda, const void* b_hi, const void* b_lo,
                         int ldb, int M, int N, int K, const EpiParams& ep, int engine, bool f16, cudaStream_t st) {
  if (M == 0 || N == 0) return ANYLOC_OK;
  bool tc_ok = gemm_tc_supported(a_hi, a_lo, lda, b_hi, b_lo, ldb, M, N, K, ep, f16);
  if (engine == ANYLOC_GEMM_TC3 && !tc_ok) {
    set_error("gemm: tensor-core engine does not support this shape/alignment (M=%d N=%d K=%d lda=%d ldb=%d f16=%d)",
              M, N, K, lda, ldb, (int)f16);
    return ANYLOC_ERR_UNSUPPORTED;
  }
  const double flops = 2.0 * M * N * K;
  if (engine == ANYLOC_GEMM_TC3 || (engine == ANYLOC_GEMM_AUTO && tc_ok && M >= 32)) {
    ProfScope ps(PC_GEMM_TC, st, flops);
    return gemm_tc_launch(a_hi, a_lo, lda, b_hi, b_lo, ldb, M, N, K, ep, f16, st);
  }
  ProfScope ps(PC_GEMM_SIMT, st, flops);
  return gemm_simt_launch(a_hi, a_lo, lda, b_hi, b_lo, ldb, M, N, K, ep, f16, st);
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
  ANYLOC_REQUIRE(in_dtype == ANYLOC_PAIR_TF32 || in_dtype == ANYLOC_PAIR_F16, "gemm_nt: bad in_dtype %d", in_dtype);
  ANYLOC_REQUIRE(out_dtype == ANYLOC_PAIR_TF32 || out_dtype == ANYLOC_PAIR_F16, "gemm_nt: bad out_dtype %d", out_dtype);
  ANYLOC_REQUIRE(epilogue >= ANYLOC_EPI_BIAS && epilogue <= ANYLOC_EPI_LS_RESID, "gemm_nt: bad epilogue %d", epilogue);
  if (epilogue == ANYLOC_EPI_BIAS_SPLIT || epilogue == ANYLOC_EPI_GELU_SPLIT || epilogue == ANYLOC_EPI_SWIGLU_SPLIT)
    ANYLOC_REQUIRE(out_lo, "gemm_nt: split epilogue needs out_lo");
  if (epilogue == ANYLOC_EPI_SWIGLU_SPLIT) ANYLOC_REQUIRE(N % 2 == 0, "gemm_nt: swiglu needs even N");
  if (epilogue == ANYLOC_EPI_LS_RESID) ANYLOC_REQUIRE(gamma && resid, "gemm_nt: LS_RESID needs gamma and resid");
  EpiParams ep{epilogue, bias, gamma, resid, (float*)out, (float*)out_lo, ldo};
  ep.alpha = alpha;
  ep.out_f16 = out_dtype == ANYLOC_PAIR_F16;
  return gemm_dispatch(a_hi, a_lo, lda, b_hi, b_lo, ldb, M, N, K, ep, engine, in_dtype == ANYLOC_PAIR_F16,
                       (cudaStream_t)stream);
}

// internal (topk.cu): plain-store GEMM with a device gate; not part of the public header
extern "C" int anyloc_gemm_nt_gated(const void* a_hi, const void* a_lo, int lda, const void* b_hi, const void* b_lo, int ldb,
                                    int M, int N, int K, int in_dtype, float alpha, float* out, int ldo, const int* gate,
                                    void* stream) {
  EpiParams ep{ANYLOC_EPI_BIAS, nullptr, nullptr, nullptr, out, nullptr, ldo};
  ep.alpha = alpha;
  ep.gate = gate;
  cudaStream_t st = (cudaStream_t)stream;
  const bool f16 = in_dtype == ANYLOC_PAIR_F16;
  if (gate) {      // conditional fallback: tensor-core engine only (its kernels test the device flag), nothing recorded
    if (!gemm_tc_supported(a_hi, a_lo, lda, b_hi, b_lo, ldb, M, N, K, ep, f16)) {
      set_error("gemm_nt_gated: shape outside the tensor-core engine's contract");
      return ANYLOC_ERR_UNSUPPORTED;
    }
    return gemm_tc_launch(a_hi, a_lo, lda, b_hi, b_lo, ldb, M, N, K, ep, f16, st);
  }
  return gemm_dispatch(a_hi, a_lo, lda, b_hi, b_lo, ldb, M, N, K, ep, ANYLOC_GEMM_AUTO, f16, st);
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

extern "C" int anyloc_layernorm_split(const float* x, const float* w, const float* b, int M, int D,
                                      float eps, void* y_hi, void* y_lo, int out_dtype, void* stream) {
  ANYLOC_REQUIRE(x && w && b && y_hi && y_lo, "layernorm: null pointer");
  if (M == 0) return ANYLOC_OK;
  return launch_layernorm(x, w, b, M, D, eps, y_hi, y_lo, out_dtype == ANYLOC_PAIR_F16, (cudaStream_t)stream);
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
    if (qkv_f16) return attention_tc_launch(qkv_hi, qkv_lo, B, T, D, heads, o_hi, o_lo, true, st);
    return attention_tc16_standalone(qkv_hi, qkv_lo, B, T, D, heads, o_hi, o_lo, st);
  }
  return attention_tc_launch(qkv_hi, qkv_lo, B, T, D, heads, o_hi, o_lo, false, st);
}

extern "C" int anyloc_attention(const float* qkv_hi, const float* qkv_lo, int B, int T, int D, int heads,
                                void* o_hi, void* o_lo, int out_dtype, int engine, void* stream) {
  ANYLOC_REQUIRE(qkv_hi && o_hi && o_lo, "attention: null pointer");
  ANYLOC_REQUIRE(D == heads * 64, "attention: head_dim must be 64 (D=%d heads=%d)", D, heads);
  if (B == 0 || T == 0) return ANYLOC_OK;
  return attention_dispatch(qkv_hi, qkv_lo, B, T, D, heads, o_hi, o_lo, out_dtype == ANYLOC_PAIR_F16, engine,
                            (cudaStream_t)stream);
}

extern "C" int anyloc_l2_normalize_rows(const float* x, int64_t rows, int D, int64_t ld_in, float* y,
                                        void* stream) {
  ANYLOC_REQUIRE(x && y && D % 4 == 0 && ld_in % 4 == 0, "l2_normalize_rows: bad args");
  if (rows == 0) return ANYLOC_OK;
  return launch_l2norm(x, rows, D, ld_in, y, (cudaStream_t)stream);
}

// ------------------------------------------------------------------ ViT forward
extern "C" int anyloc_vit_patch_k(int patch) { return (int)align_up((size_t)3 * patch * patch, 32); }

namespace {
struct VitBuffers {
  float *pa_hi, *pa_lo, *ptmp, *x, *y_hi, *y_lo, *qkv, *qkv_lo, *h_hi, *h_lo;
  float* qkv32;     // [M, 3D] fp32 rows of a tapped layer's qkv GEMM (null unless the tap list needs them)
};
// n_patch patch rows and M token rows in all; the fp32 qkv rows only when `qkv32`
size_t vit_carve(const AnylocVitCfg* c, size_t n_patch, size_t M, bool qkv32, void* ws, size_t ws_bytes,
                 VitBuffers* out) {
  const int D = c->embed_dim, Kp = anyloc_vit_patch_k(c->patch);
  Workspace w(ws ? ws : (void*)256, ws ? ws_bytes : (size_t)-1 / 2);
  VitBuffers b;
  b.pa_hi = w.take<float>(n_patch * Kp); b.pa_lo = w.take<float>(n_patch * Kp);
  b.ptmp = w.take<float>(n_patch * D);
  b.x = w.take<float>(M * D);
  b.y_hi = w.take<float>(M * D); b.y_lo = w.take<float>(M * D);
  b.qkv = w.take<float>(M * 3 * D); b.qkv_lo = w.take<float>(M * 3 * D);
  b.h_hi = w.take<float>(M * c->ffn_hidden); b.h_lo = w.take<float>(M * c->ffn_hidden);
  b.qkv32 = qkv32 ? w.take<float>(M * 3 * D) : nullptr;
  if (out) *out = b;
  if (ws && (!b.pa_hi || !b.pa_lo || !b.ptmp || !b.x || !b.y_hi || !b.y_lo || !b.qkv || !b.qkv_lo || !b.h_hi || !b.h_lo ||
             (qkv32 && !b.qkv32)))
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

// the fp32 qkv rows of layer l in bf.qkv32 -> the facets of l the plan asks for and, when `pairs`, the attention's
// (hi, lo) operands in bf.qkv / bf.qkv_lo (fp16 pairs when f16_attn, else tf32 pairs)
static int qkv_tap(const AnylocVitCfg* c, const VitBuffers& bf, int M, const VitSeqs& sq, const TapPlan& tp, int l,
                   bool pairs, bool f16_attn, cudaStream_t st) {
  const int D = c->embed_dim, m = tp.mask[l];
  const QkvTapOuts o{{(m & 1) ? tp.out[l][0] : nullptr, (m & 2) ? tp.out[l][1] : nullptr,
                      (m & 4) ? tp.out[l][2] : nullptr}};
  const int pair = pairs ? (f16_attn ? 2 : 1) : 0;
  const double rows_out = (double)M - (tp.use_cls ? 0 : sq.B);
  const double bytes = 12.0 * M * D + (pair ? (pair == 2 ? 12.0 : 24.0) * M * D : 0.0) + 4.0 * rows_out * D * popcount3(m);
  ProfScope ps(PC_VIT_MISC, st, bytes);
  return launch_qkv_tap(bf.qkv32, M, sq.T, sq.img, D, pair, pairs ? bf.qkv : nullptr, pairs ? bf.qkv_lo : nullptr, o,
                        tp.use_cls, tp.norm_descs, st);
}

// One transformer block over the M token rows in bf.x, in place.  With tp (layer l has q/k/v taps) the qkv GEMM
// writes fp32 rows and the tap kernel derives the attention's operands and the tapped facets from them.
static int vit_block(const AnylocVitCfg* c, const AnylocVitBlock& wb, const VitBuffers& bf, int M, const VitSeqs& sq,
                     int engine, cudaStream_t st, const TapPlan* tp = nullptr, int l = 0) {
  const int D = c->embed_dim, Hf = c->ffn_hidden;
  const bool f16 = c->pair_dtype == ANYLOC_PAIR_F16;
  int rc;
  const double ln_bytes = (f16 ? 8.0 : 12.0) * M * D;
  { ProfScope ps(PC_LAYERNORM, st, ln_bytes);
    if ((rc = launch_layernorm(bf.x, wb.ln1_w, wb.ln1_b, M, D, 1e-6f, bf.y_hi, bf.y_lo, f16, st))) return rc; }
  // q, k and v leave the qkv GEMM row-major through the plain split epilogue; for the tensor-core attention in the
  // fp16-pair precision they are fp16 pairs of 8*x, the attention kernel's operand format
  const bool f16_attn = engine != ANYLOC_GEMM_SIMT && f16;
  if (tp) {
    EpiParams e_qkv{ANYLOC_EPI_BIAS, wb.qkv_b, nullptr, nullptr, bf.qkv32, nullptr, 3 * D};
    e_qkv.alpha = wb.qkv_alpha;
    if ((rc = gemm_dispatch(bf.y_hi, bf.y_lo, D, wb.qkv_w_hi, wb.qkv_w_lo, D, M, 3 * D, D, e_qkv, engine, f16, st))) return rc;
    if ((rc = qkv_tap(c, bf, M, sq, *tp, l, true, f16_attn, st))) return rc;
  } else {
    EpiParams e_qkv{ANYLOC_EPI_BIAS_SPLIT, wb.qkv_b, nullptr, nullptr, bf.qkv, bf.qkv_lo, 3 * D};
    e_qkv.out_f16 = f16_attn;
    e_qkv.alpha = wb.qkv_alpha;
    if ((rc = gemm_dispatch(bf.y_hi, bf.y_lo, D, wb.qkv_w_hi, wb.qkv_w_lo, D, M, 3 * D, D, e_qkv, engine, f16, st))) return rc;
  }
  if (sq.tab) {
    ProfScope ps(PC_ATTENTION, st, sq.attn_flops);
    if ((rc = attention_tc_varlen_launch(bf.qkv, bf.qkv_lo, *sq.tab, sq.n_tiles, D, c->num_heads, bf.y_hi, bf.y_lo,
                                         f16, st)))
      return rc;
  } else if ((rc = attention_dispatch(bf.qkv, bf.qkv_lo, sq.B, sq.T, D, c->num_heads, bf.y_hi, bf.y_lo, f16, engine,
                                      st, f16_attn))) {
    return rc;
  }
  EpiParams e_proj{ANYLOC_EPI_LS_RESID, wb.proj_b, wb.ls1, bf.x, bf.x, nullptr, D};
  e_proj.alpha = wb.proj_alpha;
  if ((rc = gemm_dispatch(bf.y_hi, bf.y_lo, D, wb.proj_w_hi, wb.proj_w_lo, D, M, D, D, e_proj, engine, f16, st))) return rc;
  { ProfScope ps(PC_LAYERNORM, st, ln_bytes);
    if ((rc = launch_layernorm(bf.x, wb.ln2_w, wb.ln2_b, M, D, 1e-6f, bf.y_hi, bf.y_lo, f16, st))) return rc; }
  EpiParams e_in{c->ffn_kind == ANYLOC_FFN_MLP ? ANYLOC_EPI_GELU_SPLIT : ANYLOC_EPI_SWIGLU_SPLIT, wb.in_b, nullptr,
                 nullptr, bf.h_hi, bf.h_lo, Hf};
  e_in.alpha = wb.in_alpha; e_in.out_f16 = f16;
  const int n_in = c->ffn_kind == ANYLOC_FFN_MLP ? Hf : 2 * Hf;
  if ((rc = gemm_dispatch(bf.y_hi, bf.y_lo, D, wb.in_w_hi, wb.in_w_lo, D, M, n_in, D, e_in, engine, f16, st))) return rc;
  EpiParams e_out{ANYLOC_EPI_LS_RESID, wb.out_b, wb.ls2, bf.x, bf.x, nullptr, D};
  e_out.alpha = wb.out_alpha;
  return gemm_dispatch(bf.h_hi, bf.h_lo, Hf, wb.out_w_hi, wb.out_w_lo, Hf, M, D, Hf, e_out, engine, f16, st);
}

// Blocks 0..l_max over the M assembled token rows in bf.x, each run once, writing every tap of the plan:
//  - a layer with q/k/v taps that the forward continues through runs its qkv GEMM into fp32 rows (bf.qkv32), from
//    which the tap kernel writes the attention's operand pairs and the tapped facets; other layers run unchanged;
//  - a token tap of layer l is the facet slice of x after block l, before block l + 1 overwrites it;
//  - the last layer without a token tap exits early after norm1 and what its q/k/v taps need: one facet alone is that
//    third's own N = D GEMM and the facet slice, two or three are the N = 3D GEMM and the tap kernel without pairs.
static int vit_trunk(const AnylocVitCfg* cfg, const AnylocVitWeights* w, const VitBuffers& bf, int M, const VitSeqs& sq,
                     const TapPlan& tp, int gemm_engine, cudaStream_t st) {
  const int D = cfg->embed_dim;
  const bool f16 = cfg->pair_dtype == ANYLOC_PAIR_F16;
  int rc;
  for (int l = 0; l <= tp.l_max; ++l) {
    const AnylocVitBlock& wb = w->blocks[l];
    const int qkv = tp.mask[l] & 7;
    const bool token = (tp.mask[l] & 8) != 0;
    if (l == tp.l_max && !token) {
      if ((rc = launch_layernorm(bf.x, wb.ln1_w, wb.ln1_b, M, D, 1e-6f, bf.y_hi, bf.y_lo, f16, st))) return rc;
      if (popcount3(qkv) == 1) {
        const int facet = qkv == 1 ? 0 : qkv == 2 ? 1 : 2;
        const size_t woff = (size_t)facet * D * D * (f16 ? 2 : 4);      // bytes: weights are __half or float
        EpiParams e_f{ANYLOC_EPI_BIAS, wb.qkv_b + (size_t)facet * D, nullptr, nullptr, bf.qkv, nullptr, D};
        e_f.alpha = wb.qkv_alpha;
        if ((rc = gemm_dispatch(bf.y_hi, bf.y_lo, D, (const char*)wb.qkv_w_hi + woff, (const char*)wb.qkv_w_lo + woff,
                                D, M, D, D, e_f, gemm_engine, f16, st)))
          return rc;
        return facet_out(sq, M, bf.qkv, D, D, tp, tp.out[l][facet], st);
      }
      EpiParams e_qkv{ANYLOC_EPI_BIAS, wb.qkv_b, nullptr, nullptr, bf.qkv32, nullptr, 3 * D};
      e_qkv.alpha = wb.qkv_alpha;
      if ((rc = gemm_dispatch(bf.y_hi, bf.y_lo, D, wb.qkv_w_hi, wb.qkv_w_lo, D, M, 3 * D, D, e_qkv, gemm_engine, f16,
                              st)))
        return rc;
      return qkv_tap(cfg, bf, M, sq, tp, l, false, false, st);
    }
    if ((rc = vit_block(cfg, wb, bf, M, sq, gemm_engine, st, qkv ? &tp : nullptr, l))) return rc;
    if (token && (rc = facet_out(sq, M, bf.x, D, D, tp, tp.out[l][ANYLOC_FACET_TOKEN], st))) return rc;
  }
  return ANYLOC_OK;
}

static int vit_extract_taps(const char* fn, const AnylocVitCfg* cfg, const AnylocVitWeights* w, const float* img, int B,
                            int H, int W, const float* pos_embed, const AnylocVitTap* taps, int n_taps, int use_cls,
                            int norm_descs, void* ws, size_t ws_bytes, int gemm_engine, cudaStream_t st) {
  ANYLOC_REQUIRE(cfg && w && img && pos_embed && ws, "%s: null pointer", fn);
  ANYLOC_REQUIRE(cfg->patch > 0 && H % cfg->patch == 0 && W % cfg->patch == 0 && H > 0 && W > 0,
                 "%s: H=%d W=%d must be positive multiples of the patch size %d", fn, H, W, cfg->patch);
  TapPlan tp;
  if (!tap_plan(fn, cfg, taps, n_taps, true, &tp)) return ANYLOC_ERR_ARG;
  tp.use_cls = use_cls; tp.norm_descs = norm_descs;
  ANYLOC_REQUIRE(cfg->embed_dim == cfg->num_heads * 64, "%s: head_dim must be 64", fn);
  ANYLOC_REQUIRE(B > 0, "%s: empty batch", fn);
  if (!registers_ok(fn, cfg, w)) return ANYLOC_ERR_ARG;
  const int R = cfg->num_registers;
  const int P = cfg->patch, N = (H / P) * (W / P), T = N + 1 + R, D = cfg->embed_dim, Kp = anyloc_vit_patch_k(P);
  const int M = B * T;
  VitBuffers bf;
  if (!vit_carve(cfg, (size_t)B * N, (size_t)M, tp.qkv32, ws, ws_bytes, &bf)) {
    set_error("%s: workspace too small (%zu given, %zu needed)", fn, ws_bytes,
              vit_carve(cfg, (size_t)B * N, (size_t)M, tp.qkv32, nullptr, 0, nullptr) + 4096);
    return ANYLOC_ERR_WORKSPACE;
  }
  int rc;
  const bool f16 = cfg->pair_dtype == ANYLOC_PAIR_F16;
  if ((rc = launch_im2col(img, B, H, W, P, Kp, bf.pa_hi, bf.pa_lo, f16, st))) return rc;
  EpiParams e_pe{ANYLOC_EPI_BIAS, w->patch_b, nullptr, nullptr, bf.ptmp, nullptr, D};
  e_pe.alpha = w->patch_alpha;
  if ((rc = gemm_dispatch(bf.pa_hi, bf.pa_lo, Kp, w->patch_w_hi, w->patch_w_lo, Kp, B * N, D, Kp, e_pe,
                          gemm_engine, f16, st))) return rc;
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
                          gemm_engine, (cudaStream_t)stream);
}

extern "C" int anyloc_vit_extract_taps(const AnylocVitCfg* cfg, const AnylocVitWeights* w, const float* img, int B, int H,
                                       int W, const float* pos_embed, const AnylocVitTap* taps, int n_taps, int use_cls,
                                       int norm_descs, void* ws, size_t ws_bytes, int gemm_engine, void* stream) {
  ANYLOC_REQUIRE(cfg, "vit_extract_taps: null pointer");
  return vit_extract_taps("vit_extract_taps", cfg, w, img, B, H, W, pos_embed, taps, n_taps, use_cls, norm_descs, ws,
                          ws_bytes, gemm_engine, (cudaStream_t)stream);
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
  int64_t tok = 0, patches = 0, tiles = 0;
  double flops = 0.0;
  p->img.n = B; p->img.nreg = R; p->attn.n = B;
  int order[ANYLOC_VIT_VARLEN_MAX_B];
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
    order[i] = i;
  }
  // attention entries longest first (the longest key loops start first); ties keep the input order
  std::stable_sort(order, order + B, [&](int a, int b) { return p->img.gh[a] * p->img.gw[a] > p->img.gh[b] * p->img.gw[b]; });
  for (int k = 0; k < B; ++k) {
    const int i = order[k], T = p->img.gh[i] * p->img.gw[i] + 1 + R;
    p->attn.tile0[k] = (int)tiles; p->attn.row0[k] = p->img.tok0[i]; p->attn.len[k] = T;
    tiles += cdiv(T, 64);
  }
  p->n_patch = (int)patches; p->n_tok = (int)tok; p->n_tiles = (int)tiles; p->attn_flops = flops;
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
                                   size_t ws_bytes, int gemm_engine, cudaStream_t st) {
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
  VarlenPlan p;
  if (!varlen_plan(cfg, B, hw, &p)) return ANYLOC_ERR_ARG;
  for (int i = 0; i < B; ++i)
    ANYLOC_REQUIRE(img[i] && pos_embed[i], "%s: null image or positional table %d", fn, i);
  const int P = cfg->patch, D = cfg->embed_dim, Kp = anyloc_vit_patch_k(P), M = p.n_tok;
  VitBuffers bf;
  if (!vit_carve(cfg, (size_t)p.n_patch, (size_t)M, tp.qkv32, ws, ws_bytes, &bf)) {
    set_error("%s: workspace too small (%zu given, %zu needed)", fn, ws_bytes,
              vit_carve(cfg, (size_t)p.n_patch, (size_t)M, tp.qkv32, nullptr, 0, nullptr) + 4096);
    return ANYLOC_ERR_WORKSPACE;
  }
  int rc;
  const bool f16 = cfg->pair_dtype == ANYLOC_PAIR_F16;
  for (int i = 0; i < B; ++i) p.img.ptr[i] = img[i];
  if ((rc = launch_im2col_varlen(p.img, p.n_patch, P, Kp, bf.pa_hi, bf.pa_lo, f16, st))) return rc;
  EpiParams e_pe{ANYLOC_EPI_BIAS, w->patch_b, nullptr, nullptr, bf.ptmp, nullptr, D};
  e_pe.alpha = w->patch_alpha;
  if ((rc = gemm_dispatch(bf.pa_hi, bf.pa_lo, Kp, w->patch_w_hi, w->patch_w_lo, Kp, p.n_patch, D, Kp, e_pe,
                          gemm_engine, f16, st))) return rc;
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
                                 ws_bytes, gemm_engine, (cudaStream_t)stream);
}

extern "C" int anyloc_vit_extract_taps_varlen(const AnylocVitCfg* cfg, const AnylocVitWeights* w, int B,
                                              const float* const* img, const int32_t* hw,
                                              const float* const* pos_embed, const AnylocVitTap* taps, int n_taps,
                                              int use_cls, int norm_descs, void* ws, size_t ws_bytes, int gemm_engine,
                                              void* stream) {
  ANYLOC_REQUIRE(cfg, "vit_extract_taps_varlen: null pointer");
  return vit_extract_taps_varlen("vit_extract_taps_varlen", cfg, w, B, img, hw, pos_embed, taps, n_taps, use_cls,
                                 norm_descs, ws, ws_bytes, gemm_engine, (cudaStream_t)stream);
}
