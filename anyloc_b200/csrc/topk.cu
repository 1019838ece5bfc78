// Query->database retrieval (reference: /root/reference/utilities.py:435-450, faiss IndexFlatIP /
// IndexFlatL2 exact search).  normalise rows -> score GEMM (fp32-equivalent) -> k-best per query,
// best first, lowest database index first among equal scores.
#include <float.h>
#include <algorithm>
#include "common.cuh"

// internal (api.cu): the plain-store 3-term GEMM with an optional device gate (*gate == 0 -> the kernels return at once);
// when gated, no algorithmic work is recorded (the coarse pass already accounted for the product)
extern "C" int anyloc_gemm_nt_gated(const void* a_hi, const void* a_lo, int lda, const void* b_hi, const void* b_lo, int ldb,
                                    int M, int N, int K, int in_dtype, float alpha, float* out, int ldo, const int* gate,
                                    void* stream);

namespace anyloc {

// fp16-pair scale of unit-norm rows: |s y| <= 4096 < 65504, and s*y - hi stays far above the fp16 subnormal step for
// every element that matters (an element below 2^-12 of the row norm contributes < 2^-36 to a unit dot product).
constexpr float kRetrievalScale = 4096.0f;

// y = x / max(|x|, 1e-12) written as a tf32 (hi,lo) pair (hi+lo == fp32 value); also |y|^2 per row
// (needed by the L2 metric).  One CTA per row.
template <bool F16>
__global__ void __launch_bounds__(256)
normalize_rows_split_kernel(const float* __restrict__ x, int D, int do_norm, void* __restrict__ hi_v,
                            void* __restrict__ lo_v, float* __restrict__ sq, float* __restrict__ dn /* nullable, F16 only */,
                            int* __restrict__ dn_max_bits /* nullable */, int n_rows) {
  // grid-stride over the rows with a grid of ~3 CTAs per SM: a row (196 KB at Dv = 49152) is read twice (norm pass,
  // split pass) and the second read must still find it in L2 -- with one CTA per row ~1200 rows (230 MB) were in
  // flight and both passes went to DRAM (ncu, round 2: 3.93 GB read for a 1.97 GB database)
  for (size_t row = blockIdx.x; row < (size_t)n_rows; row += gridDim.x) {
  __syncthreads();
  const float4* xr = reinterpret_cast<const float4*>(x + row * D);
  const int D4 = D >> 2;
  float ss = 0.f;
  for (int d = threadIdx.x; d < D4; d += blockDim.x) {
    float4 v = __ldg(xr + d);
    ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  __shared__ float red[8];
  __shared__ float tot;
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  if (threadIdx.x == 0) { float t = 0.f; for (int w = 0; w < 8; ++w) t += red[w]; tot = t; }
  __syncthreads();
  const float nrm = fmaxf(sqrtf(tot), 1e-12f);
  float4* h4 = reinterpret_cast<float4*>(reinterpret_cast<float*>(hi_v) + row * D);
  float4* l4 = reinterpret_cast<float4*>(reinterpret_cast<float*>(lo_v) + row * D);
  uint2* h2 = reinterpret_cast<uint2*>(reinterpret_cast<__half*>(hi_v) + row * D);   // 4 halves = 8 bytes
  uint2* l2 = reinterpret_cast<uint2*>(reinterpret_cast<__half*>(lo_v) + row * D);
  float ss2 = 0.f, dd2 = 0.f;
  for (int d = threadIdx.x; d < D4; d += blockDim.x) {
    float4 v = __ldg(xr + d);
    if (do_norm) { v.x = v.x / nrm; v.y = v.y / nrm; v.z = v.z / nrm; v.w = v.w / nrm; }
    ss2 += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    if constexpr (F16) {
      uint2 h, l;
      const float a0 = v.x * kRetrievalScale, a1 = v.y * kRetrievalScale, a2 = v.z * kRetrievalScale, a3 = v.w * kRetrievalScale;
      split_f16x2(a0, a1, h.x, l.x);
      split_f16x2(a2, a3, h.y, l.y);
      h2[d] = h; l2[d] = l;
      // what a hi-only product drops of this row: s*y - hi (exact in fp32: hi is s*y rounded to 11 significant bits)
      const float e0 = a0 - veltkamp_hi11(a0), e1 = a1 - veltkamp_hi11(a1), e2 = a2 - veltkamp_hi11(a2), e3 = a3 - veltkamp_hi11(a3);
      dd2 += e0 * e0 + e1 * e1 + e2 * e2 + e3 * e3;
    } else {
      float4 h, l;
      split_tf32(v.x, h.x, l.x); split_tf32(v.y, h.y, l.y);
      split_tf32(v.z, h.z, l.z); split_tf32(v.w, h.w, l.w);
      h4[d] = h; l4[d] = l;
    }
  }
  if (sq) {
    ss2 = warp_sum(ss2);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss2;
    __syncthreads();
    if (threadIdx.x == 0) { float t = 0.f; for (int w = 0; w < 8; ++w) t += red[w]; sq[row] = t; }
  }
  if (F16 && dn) {
    // |s*y - hi| / s, rounded UP (1 + 2^-10), plus the fp16 subnormal slack sqrt(D) * 2^-25 / s (elements of |s*y| < 2^-14
    // are rounded to the 2^-24 grid) -- a rigorous bound on what the hi-only (coarse) score ignores of this row
    dd2 = warp_sum(dd2);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = dd2;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f; for (int w = 0; w < 8; ++w) t += red[w];
      const float b = (sqrtf(t) * 1.001f + sqrtf((float)D) * 2.98e-8f) / kRetrievalScale;
      dn[row] = b;
      // positive floats order like their bit patterns.  A row holding a NaN or an Inf (b = NaN) stays out of the header:
      // a NaN there would make every query's threshold NaN, i.e. no candidates and an empty answer.  The row's own
      // coarse scores are NaN, so it is never a candidate, as it is never selected on the exact route.
      if (dn_max_bits && b <= FLT_MAX) atomicMax(dn_max_bits, __float_as_int(b));
    }
  }
  }
}

// Single-pass form for rows that fit the registers of a 1024-thread CTA (D <= 16 * 4096 floats): the row is loaded ONCE
// (NV float4 per thread, the whole row in flight), reduced, normalised, split and stored -- 4 B read + 4 B (fp16 pairs) or
// 8 B (tf32 pairs) written per element, instead of reading the row twice.  Same arithmetic, except that |x|^2 is summed in
// the order of this thread layout (fp32 rounding of the norm only).
template <bool F16, int NV>
__global__ void __launch_bounds__(1024, 1)
normalize_rows_split_reg_kernel(const float* __restrict__ x, int D, int do_norm, void* __restrict__ hi_v,
                                void* __restrict__ lo_v, float* __restrict__ sq, float* __restrict__ dn,
                                int* __restrict__ dn_max_bits, int n_rows) {
  const int D4 = D >> 2;
  __shared__ float red[32];
  __shared__ float s_tot;
  for (size_t row = blockIdx.x; row < (size_t)n_rows; row += gridDim.x) {
    const float4* xr = reinterpret_cast<const float4*>(x + row * D);
    float4 v[NV];
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int d = threadIdx.x + j * 1024;
      v[j] = d < D4 ? __ldg(xr + d) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int j = 0; j < NV; ++j) ss += v[j].x * v[j].x + v[j].y * v[j].y + v[j].z * v[j].z + v[j].w * v[j].w;
    ss = warp_sum(ss);
    __syncthreads();                                   // red / s_tot of the previous row have been consumed
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    if (threadIdx.x == 0) { float t = 0.f; for (int w = 0; w < 32; ++w) t += red[w]; s_tot = t; }
    __syncthreads();
    const float nrm = fmaxf(sqrtf(s_tot), 1e-12f);
    float ss2 = 0.f, dd2 = 0.f;
    uint2* h2 = reinterpret_cast<uint2*>(reinterpret_cast<__half*>(hi_v) + row * D);
    uint2* l2 = reinterpret_cast<uint2*>(reinterpret_cast<__half*>(lo_v) + row * D);
    float4* h4 = reinterpret_cast<float4*>(reinterpret_cast<float*>(hi_v) + row * D);
    float4* l4 = reinterpret_cast<float4*>(reinterpret_cast<float*>(lo_v) + row * D);
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int d = threadIdx.x + j * 1024;
      if (d >= D4) continue;
      float4 y = v[j];
      if (do_norm) { y.x = y.x / nrm; y.y = y.y / nrm; y.z = y.z / nrm; y.w = y.w / nrm; }
      ss2 += y.x * y.x + y.y * y.y + y.z * y.z + y.w * y.w;
      if constexpr (F16) {
        uint2 h, l;
        const float a0 = y.x * kRetrievalScale, a1 = y.y * kRetrievalScale, a2 = y.z * kRetrievalScale, a3 = y.w * kRetrievalScale;
        split_f16x2(a0, a1, h.x, l.x);
        split_f16x2(a2, a3, h.y, l.y);
        h2[d] = h; l2[d] = l;
        const float e0 = a0 - veltkamp_hi11(a0), e1 = a1 - veltkamp_hi11(a1), e2 = a2 - veltkamp_hi11(a2), e3 = a3 - veltkamp_hi11(a3);
        dd2 += e0 * e0 + e1 * e1 + e2 * e2 + e3 * e3;
      } else {
        float4 h, l;
        split_tf32(y.x, h.x, l.x); split_tf32(y.y, h.y, l.y); split_tf32(y.z, h.z, l.z); split_tf32(y.w, h.w, l.w);
        h4[d] = h; l4[d] = l;
      }
    }
    ss2 = warp_sum(ss2); dd2 = warp_sum(dd2);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss2;
    __syncthreads();
    if (threadIdx.x == 0 && sq) { float t = 0.f; for (int w = 0; w < 32; ++w) t += red[w]; sq[row] = t; }
    if (F16 && dn) {
      __syncthreads();
      if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = dd2;
      __syncthreads();
      if (threadIdx.x == 0) {
        float t = 0.f; for (int w = 0; w < 32; ++w) t += red[w];
        const float b = (sqrtf(t) * 1.001f + sqrtf((float)D) * 2.98e-8f) / kRetrievalScale;
        dn[row] = b;
        if (dn_max_bits && b <= FLT_MAX) atomicMax(dn_max_bits, __float_as_int(b));     // finite rows only, as above
      }
    }
  }
}

// host dispatch of the two forms
template <bool F16>
static cudaError_t launch_normalize_rows(const float* x, int n_rows, int D, int do_norm, void* hi, void* lo, float* sq, float* dn,
                                         int* dn_max_bits, cudaStream_t st) {
  const int D4 = D >> 2, sms = device_sm_count();
  if (D4 > 2 * 1024 && D4 <= 16 * 1024) {            // long rows: the single-pass register form, one CTA per SM
    const int grid = std::min(n_rows, sms);
    if (D4 <= 4 * 1024) normalize_rows_split_reg_kernel<F16, 4><<<grid, 1024, 0, st>>>(x, D, do_norm, hi, lo, sq, dn, dn_max_bits, n_rows);
    else if (D4 <= 8 * 1024) normalize_rows_split_reg_kernel<F16, 8><<<grid, 1024, 0, st>>>(x, D, do_norm, hi, lo, sq, dn, dn_max_bits, n_rows);
    else if (D4 <= 12 * 1024) normalize_rows_split_reg_kernel<F16, 12><<<grid, 1024, 0, st>>>(x, D, do_norm, hi, lo, sq, dn, dn_max_bits, n_rows);
    else normalize_rows_split_reg_kernel<F16, 16><<<grid, 1024, 0, st>>>(x, D, do_norm, hi, lo, sq, dn, dn_max_bits, n_rows);
  } else {
    normalize_rows_split_kernel<F16><<<std::min(n_rows, 8 * sms), 256, 0, st>>>(x, D, do_norm, hi, lo, sq, dn, dn_max_bits, n_rows);
  }
  return cudaGetLastError();
}

// k-best selection per query row, best first, lowest index first among equal scores (metric IP: larger is better;
// metric L2: key := -(qq - 2 s + dd)).  O(n_db) per query:
//   A: every thread keeps the best score of its strided share of the row;
//   B: tau = the k-th best of the 1024 thread bests (k rounds of block arg-best over 1024 values): those are k DISTINCT
//      row elements, so the row's true k-th best is >= tau and every member of the true top-k is >= tau;
//   C: second sweep, the elements >= tau (usually k .. a few k of them) are compacted into a shared-memory list;
//   D: k rounds of arg-best over the list (score descending, lowest index first among equal scores).
// More than SEL_CAP candidates (a row with thousands of equal scores) -> k ordered sweeps over the row (read-only).
// MERGE (streamed search, k <= SEL_CAP): the row is a piece of the database holding global rows [row0, row0 + n_db),
// and dist / idx hold the running k best of the rows before it.  Those k enter the list first (slots 0 .. k-1, so they
// stay in shared memory through the sweeps) and the k best of the union are written back in place.  tau is still taken
// over the piece alone: the union's k-th best is at least the piece's, so every union top-k member of the piece is >= tau.
constexpr int SEL_CAP = 4096;
__device__ __forceinline__ bool better(float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); }

__device__ __forceinline__ void block_argbest(float& best, int& besti, float* bv, int* bi) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    float ov = __shfl_xor_sync(0xffffffffu, best, o);
    int oi = __shfl_xor_sync(0xffffffffu, besti, o);
    if (better(ov, oi, best, besti)) { best = ov; besti = oi; }
  }
  if ((threadIdx.x & 31) == 0) { bv[threadIdx.x >> 5] = best; bi[threadIdx.x >> 5] = besti; }
  __syncthreads();
  if (threadIdx.x < 32) {
    const int nw = blockDim.x >> 5;
    best = threadIdx.x < nw ? bv[threadIdx.x] : -INFINITY;
    besti = threadIdx.x < nw ? bi[threadIdx.x] : 0x7fffffff;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      float ov = __shfl_xor_sync(0xffffffffu, best, o);
      int oi = __shfl_xor_sync(0xffffffffu, besti, o);
      if (better(ov, oi, best, besti)) { best = ov; besti = oi; }
    }
    if (threadIdx.x == 0) { bv[32] = best; bi[32] = besti; }
  }
  __syncthreads();
  best = bv[32]; besti = bi[32];
  __syncthreads();
}

template <bool MERGE>
__global__ void __launch_bounds__(1024)
topk_select2_kernel(const float* __restrict__ scores, int n_db, int64_t ld, int k, int metric,
                    const float* __restrict__ qq, const float* __restrict__ dd,
                    float* __restrict__ dist, int64_t* __restrict__ idx, const int* __restrict__ gate /* nullable */,
                    int row0 /* MERGE only */) {
  if (gate != nullptr && *reinterpret_cast<const volatile int*>(gate) == 0) return;
  const int q = blockIdx.x;
  const float* s = scores + (size_t)q * ld;
  const bool l2 = metric == ANYLOC_METRIC_L2;
  const float a = l2 ? qq[q] : 0.f;
  auto key = [&](int j) { const float v = s[j]; return l2 ? -((a - 2.0f * v) + dd[j]) : v; };   // larger = better
  auto gid = [&](int j) { return MERGE ? row0 + j : j; };                                         // global row index
  __shared__ float bv[33];
  __shared__ int bi[33];
  __shared__ float cv[SEL_CAP];
  __shared__ int ci[SEL_CAP];
  __shared__ int count;
  if constexpr (MERGE) {
    // the running list (read before anything is written back); its -1 pads can never be selected
    for (int r = threadIdx.x; r < k; r += blockDim.x) {
      const int64_t i = idx[(size_t)q * k + r];
      const float d = dist[(size_t)q * k + r];
      cv[r] = i >= 0 ? (l2 ? -d : d) : -INFINITY;
      ci[r] = i >= 0 ? (int)i : 0x7fffffff;
    }
    if (threadIdx.x == 0) count = k;
  } else {
    if (threadIdx.x == 0) count = 0;
  }
  // A
  float mine = -INFINITY; int minei = 0x7fffffff;
  for (int j = threadIdx.x; j < n_db; j += blockDim.x) {
    const float v = key(j);
    if (better(v, gid(j), mine, minei)) { mine = v; minei = gid(j); }
  }
  // B
  float tau = -INFINITY;
  {
    float v = mine; int vi = minei;
    for (int r = 0; r < k; ++r) {
      float b = v; int bidx = vi;
      block_argbest(b, bidx, bv, bi);
      if (bidx == 0x7fffffff) { tau = -INFINITY; break; }   // fewer than k elements in the row
      tau = b;
      if (vi == bidx) { v = -INFINITY; vi = 0x7fffffff; }    // the winner leaves the pool
    }
  }
  __syncthreads();
  // C
  for (int j = threadIdx.x; j < n_db; j += blockDim.x) {
    const float v = key(j);
    if (v >= tau) {
      const int slot = atomicAdd(&count, 1);
      if (slot < SEL_CAP) { cv[slot] = v; ci[slot] = gid(j); }
    }
  }
  __syncthreads();
  const int n_c = count;
  if (n_c > SEL_CAP) {
    // thousands of (near-)equal scores: k ordered sweeps over the row itself -- round r takes the best element that
    // comes strictly after round r-1's winner in (score descending, index ascending) order
    float pv = INFINITY; int pj = -1;
    for (int r = 0; r < k; ++r) {
      float b = -INFINITY; int bidx = 0x7fffffff;
      for (int j = threadIdx.x; j < n_db; j += blockDim.x) {
        const float v = key(j);
        if ((v < pv || (v == pv && gid(j) > pj)) && better(v, gid(j), b, bidx)) { b = v; bidx = gid(j); }
      }
      if constexpr (MERGE) {             // the running list, still in slots 0 .. k-1
        for (int c = threadIdx.x; c < k; c += blockDim.x) {
          const float v = cv[c]; const int i = ci[c];
          if ((v < pv || (v == pv && i > pj)) && better(v, i, b, bidx)) { b = v; bidx = i; }
        }
      }
      block_argbest(b, bidx, bv, bi);
      if (threadIdx.x == 0) {
        dist[(size_t)q * k + r] = bidx != 0x7fffffff ? (l2 ? -b : b) : (l2 ? INFINITY : -INFINITY);
        idx[(size_t)q * k + r] = bidx != 0x7fffffff ? bidx : -1;
      }
      pv = b; pj = bidx;
      if (bidx == 0x7fffffff) pv = -INFINITY;      // exhausted: every later round pads
    }
    return;
  }
  // D
  for (int r = 0; r < k; ++r) {
    float b = -INFINITY; int bidx = 0x7fffffff; int bslot = -1;
    for (int c = threadIdx.x; c < n_c; c += blockDim.x)
      if (better(cv[c], ci[c], b, bidx)) { b = cv[c]; bidx = ci[c]; bslot = c; }
    float wb = b; int wi = bidx;
    block_argbest(wb, wi, bv, bi);
    if (bslot >= 0 && wi == bidx && wi != 0x7fffffff) { cv[bslot] = -INFINITY; ci[bslot] = 0x7fffffff; }
    if (threadIdx.x == 0) {
      if (wi != 0x7fffffff) {
        dist[(size_t)q * k + r] = l2 ? -wb : wb;
        idx[(size_t)q * k + r] = wi;
      } else {
        dist[(size_t)q * k + r] = l2 ? INFINITY : -INFINITY;
        idx[(size_t)q * k + r] = -1;          // faiss pads with -1 when k > ntotal
      }
    }
    __syncthreads();
  }
}


// ---------------------------------------------------------------------------------------------------------------------
// Coarse retrieval (inner product on an fp16-pair index).  One hi-only tensor-core pass gives S~ = hi_q . hi_d / s^2 with
//   |S~ - S| <= eps_q = (dn_q + DN + dn_q DN) (1 + 2^-10) + 3e-5
// (dn_* = |s y - hi| / s per row, measured when the pairs were written; DN = max over the database; Cauchy-Schwarz per
// dropped term, |y| <= 1 + 1e-6; 3e-5 covers the fp32 accumulation: <= 128 truncating steps per tensor-core chunk + 24
// round-to-nearest chunk adds).  With tau = the k-th best S~ of a query, every member of its exact top-k has
// S~ >= tau - 2 eps_q, so those candidates (usually k .. 3k of 10^4-10^5 rows) are re-scored EXACTLY from the (hi,lo)
// pairs in fp32 and the k best of them -- score descending, lowest index first -- are the answer: identical to the
// 3-term path up to fp32 rounding of the scores, at a third of the tensor-core work.  A query with more than CAND_MAX
// candidates raises a device flag that switches on the 3-term fallback (launched behind it, gated, no host sync).
// MERGE (streamed search): the rows are one piece of the database and run_dist holds the k best EXACT scores of the
// rows before it (-inf while fewer than k).  Its k-th, R, is a second lower bound: a row of this piece enters the final
// top-k only by beating all k running entries (their indices are lower, so a tie loses), i.e. with S > R, and then
// S~ >= S - eps_q > R - eps_q.  The threshold is max(tau, R) - 2 eps_q: R - eps_q would do, the second eps_q leaves the
// same margin for the fp32 rounding of the re-scored S that tau - 2 eps_q leaves.
constexpr int CAND_MAX = 256;

template <bool MERGE>
__global__ void __launch_bounds__(1024)
topk_candidates_kernel(const float* __restrict__ scores, int n_db, int64_t ld, int k, const float* __restrict__ dn_q,
                       const int* __restrict__ dn_max_bits, int32_t* __restrict__ cand /* [n_q, CAND_MAX] */,
                       int32_t* __restrict__ cand_n /* [n_q] */, int* __restrict__ overflow,
                       const float* __restrict__ run_dist /* MERGE only: [n_q, k] */) {
  const int q = blockIdx.x;
  const float* s = scores + (size_t)q * ld;
  __shared__ float bv[33];
  __shared__ int bi[33];
  __shared__ int ci[SEL_CAP];
  __shared__ int count;
  if (threadIdx.x == 0) count = 0;
  float mine = -INFINITY; int minei = 0x7fffffff;
  for (int j = threadIdx.x; j < n_db; j += blockDim.x) {
    const float v = s[j];
    if (better(v, j, mine, minei)) { mine = v; minei = j; }
  }
  float tau = -INFINITY;
  {
    float v = mine; int vi = minei;
    for (int r = 0; r < k; ++r) {
      float b = v; int bidx = vi;
      block_argbest(b, bidx, bv, bi);
      if (bidx == 0x7fffffff) { tau = -INFINITY; break; }
      tau = b;
      if (vi == bidx) { v = -INFINITY; vi = 0x7fffffff; }
    }
  }
  const float DN = __int_as_float(*dn_max_bits), dq = dn_q[q];
  const float eps = (dq + DN + dq * DN) * 1.001f + 3.0e-5f;
  float thr;
  if constexpr (MERGE) thr = fmaxf(tau, run_dist[(size_t)q * k + k - 1]) - 2.0f * eps;
  else thr = tau - 2.0f * eps;
  __syncthreads();
  for (int j = threadIdx.x; j < n_db; j += blockDim.x) {
    if (s[j] >= thr) {
      const int slot = atomicAdd(&count, 1);
      if (slot < SEL_CAP) ci[slot] = j;
    }
  }
  __syncthreads();
  const int n_c = count;
  if (n_c > CAND_MAX) {
    if (threadIdx.x == 0) { cand_n[q] = 0; atomicExch(overflow, 1); }
    return;
  }
  for (int c = threadIdx.x; c < n_c; c += blockDim.x) cand[(size_t)q * CAND_MAX + c] = ci[c];
  if (threadIdx.x == 0) cand_n[q] = n_c;
}

// CTA per query: exact fp32 scores of its candidates from the fp16 (hi,lo) pairs, then the k best of them.
__device__ __forceinline__ float2 h2f(uint32_t u) {
  return __half22float2(*reinterpret_cast<const __half2*>(&u));
}
constexpr int RS_CHUNK = 4096;          // query elements staged per pass (fp32: 16 KB of shared memory)
constexpr int COARSE_K_MAX = 64;        // the coarse route's largest k
// MERGE (streamed search): the candidates are rows of a piece holding global rows [row0, ...), and dist / idx hold the
// running k best of the rows before it; those join the re-scored candidates and the k best of both go back in place.
template <bool MERGE>
__global__ void __launch_bounds__(256)
topk_rescore_kernel(const __half* __restrict__ db_hi, const __half* __restrict__ db_lo, const __half* __restrict__ qu_hi,
                    const __half* __restrict__ qu_lo, int Dv, int k, const int32_t* __restrict__ cand,
                    const int32_t* __restrict__ cand_n, const int* __restrict__ overflow, float* __restrict__ dist,
                    int64_t* __restrict__ idx, int row0 /* MERGE only */) {
  if (*reinterpret_cast<const volatile int*>(overflow) != 0) return;       // the 3-term fallback answers every query
  const int q = blockIdx.x, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  constexpr int LIST = CAND_MAX + (MERGE ? COARSE_K_MAX : 0);
  __shared__ __align__(16) float xq[RS_CHUNK];      // this pass' slice of the query, hi + lo (exact: 22 significant bits)
  __shared__ float cv[LIST];
  __shared__ int ci[LIST];
  __shared__ float bv[33];
  __shared__ int bi[33];
  const int n_c = cand_n[q];
  for (int c = threadIdx.x; c < n_c; c += blockDim.x) { cv[c] = 0.f; ci[c] = cand[(size_t)q * CAND_MAX + c]; }
  // The query is read ONCE per CTA (slice by slice into shared memory); every candidate row is streamed once, in
  // 8 KB pieces per array.  Warp w owns candidates w, w + 8, ...; partial sums are added slice by slice in slice order.
  for (int d0 = 0; d0 < Dv; d0 += RS_CHUNK) {
    const int len = min(RS_CHUNK, Dv - d0);          // multiple of 8
    __syncthreads();
    for (int t = threadIdx.x; t < (len >> 3); t += blockDim.x) {
      const uint4 xh = __ldg(reinterpret_cast<const uint4*>(qu_hi + (size_t)q * Dv + d0) + t);
      const uint4 xl = __ldg(reinterpret_cast<const uint4*>(qu_lo + (size_t)q * Dv + d0) + t);
      const uint32_t hw[4] = {xh.x, xh.y, xh.z, xh.w}, lw[4] = {xl.x, xl.y, xl.z, xl.w};
      float o[8];
#pragma unroll
      for (int e = 0; e < 4; ++e) { const float2 a = h2f(hw[e]), b2 = h2f(lw[e]); o[2 * e] = a.x + b2.x; o[2 * e + 1] = a.y + b2.y; }
      *reinterpret_cast<float4*>(xq + t * 8) = make_float4(o[0], o[1], o[2], o[3]);
      *reinterpret_cast<float4*>(xq + t * 8 + 4) = make_float4(o[4], o[5], o[6], o[7]);
    }
    __syncthreads();
    for (int c = w; c < n_c; c += 8) {
      const size_t roff = (size_t)ci[c] * Dv + d0;
      const uint4* dh = reinterpret_cast<const uint4*>(db_hi + roff);
      const uint4* dl = reinterpret_cast<const uint4*>(db_lo + roff);
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
      for (int t = lane; t < (len >> 3); t += 32) {
        const uint4 yh = __ldg(dh + t), yl = __ldg(dl + t);
        const float4 x0 = *reinterpret_cast<const float4*>(xq + t * 8), x1 = *reinterpret_cast<const float4*>(xq + t * 8 + 4);
        const float2 h0 = h2f(yh.x), l0 = h2f(yl.x), h1 = h2f(yh.y), l1 = h2f(yl.y);
        const float2 h2 = h2f(yh.z), l2 = h2f(yl.z), h3 = h2f(yh.w), l3 = h2f(yl.w);
        a0 = fmaf(x0.x, h0.x + l0.x, a0); a1 = fmaf(x0.y, h0.y + l0.y, a1);
        a2 = fmaf(x0.z, h1.x + l1.x, a2); a3 = fmaf(x0.w, h1.y + l1.y, a3);
        a0 = fmaf(x1.x, h2.x + l2.x, a0); a1 = fmaf(x1.y, h2.y + l2.y, a1);
        a2 = fmaf(x1.z, h3.x + l3.x, a2); a3 = fmaf(x1.w, h3.y + l3.y, a3);
      }
      const float part = warp_sum((a0 + a1) + (a2 + a3));
      if (lane == 0) cv[c] += part;
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < n_c; c += blockDim.x) cv[c] *= 1.0f / (kRetrievalScale * kRetrievalScale);
  __syncthreads();
  int n_l = n_c;
  if constexpr (MERGE) {
    for (int c = threadIdx.x; c < n_c; c += blockDim.x) ci[c] += row0;
    for (int r = threadIdx.x; r < k; r += blockDim.x) {      // -1 pads can never be selected
      const int64_t i = idx[(size_t)q * k + r];
      cv[n_c + r] = i >= 0 ? dist[(size_t)q * k + r] : -INFINITY;
      ci[n_c + r] = i >= 0 ? (int)i : 0x7fffffff;
    }
    __syncthreads();
    n_l = n_c + k;
  }
  for (int r = 0; r < k; ++r) {
    float b = -INFINITY; int bidx = 0x7fffffff; int bslot = -1;
    for (int c = threadIdx.x; c < n_l; c += blockDim.x)
      if (better(cv[c], ci[c], b, bidx)) { b = cv[c]; bidx = ci[c]; bslot = c; }
    float wb = b; int wi = bidx;
    block_argbest(wb, wi, bv, bi);
    if (bslot >= 0 && wi == bidx && wi != 0x7fffffff) { cv[bslot] = -INFINITY; ci[bslot] = 0x7fffffff; }
    if (threadIdx.x == 0) {
      dist[(size_t)q * k + r] = wi != 0x7fffffff ? wb : -INFINITY;
      idx[(size_t)q * k + r] = wi != 0x7fffffff ? wi : -1;
    }
    __syncthreads();
  }
}

}  // namespace anyloc

using namespace anyloc;


// ---- prepared database ("index"): what faiss' index.add(db) leaves behind (utilities.py:449).
// Layout of the caller-owned blob for `capacity` rows of Dv columns:
//   hi [capacity, Dv] | lo [capacity, Dv] | sq [capacity] fp32 (|y|^2 per row, the L2 metric needs it) |
//   dn [capacity] fp32 (|s y - hi| / s per row: what a hi-only product ignores; fp16 layout only) | header (256 B: max dn)
// with hi/lo either fp16 pairs of 4096*y (unit rows: normalize != 0, Dv % 8 == 0 -- the 2x faster kind::f16 tensor
// path) or tf32 pairs of y (rows of unknown range).
static bool index_uses_f16(int Dv, int normalize) { return normalize && (Dv % 8) == 0; }
struct IndexView { void* hi; void* lo; float* sq; float* dn; int* hdr; bool f16; size_t pair_bytes_per_row; };
// split: the device blob of a split index (fp16 pairs; lo lives in host memory), hi | sq | dn | header
static bool carve_index(void* blob, size_t bytes, int64_t capacity, int Dv, int normalize, IndexView* v,
                        bool split = false) {
  v->f16 = index_uses_f16(Dv, normalize);
  const size_t esz = v->f16 ? 2 : 4;
  v->pair_bytes_per_row = (size_t)Dv * esz;
  Workspace w(blob, bytes);
  v->hi = w.take<char>((size_t)capacity * Dv * esz);
  v->lo = split ? nullptr : w.take<char>((size_t)capacity * Dv * esz);
  v->sq = w.take<float>((size_t)capacity);
  v->dn = w.take<float>((size_t)capacity);
  v->hdr = w.take<int>(64);
  return v->hi && (split || v->lo) && v->sq && v->dn && v->hdr;
}

// An index blob (resident or split, and a split index's host lo array) is written as float4 / uint2 rows, read by the
// score GEMM's TMA (gemm_tc_supported's 16-byte test) and as uint4 by the rescoring and the split gather: every entry
// that takes one requires 16 bytes, so a blob one of them would refuse is refused by all.
#define ANYLOC_REQUIRE_BLOB(p, who, name) ANYLOC_REQUIRE_ALIGNED(p, 16, who, name, "float4, uint4 and TMA access")
// a search's outputs: fp32 distances and int64 indices, one element at a time
static int search_out_alignment(const char* who, const float* dist, const int64_t* idx) {
  ANYLOC_REQUIRE_ALIGNED(dist, 4, who, "dist", "fp32 access");
  ANYLOC_REQUIRE_ALIGNED(idx, 8, who, "idx", "int64 access");
  return ANYLOC_OK;
}

extern "C" size_t anyloc_index_bytes(int64_t capacity, int Dv, int normalize) {
  const size_t esz = index_uses_f16(Dv, normalize) ? 2 : 4;
  return 2 * align_up((size_t)capacity * Dv * esz, 256) + 2 * align_up((size_t)capacity * 4, 256) + 256 + 256;
}

// A fresh blob must be initialised once (clears the header) before the first anyloc_index_add.
extern "C" int anyloc_index_init(void* index, size_t index_bytes, int64_t capacity, int Dv, int normalize, void* stream) {
  ANYLOC_REQUIRE(index, "index_init: null pointer");
  ANYLOC_REQUIRE_BLOB(index, "index_init", "index");
  IndexView v;
  if (!carve_index(index, index_bytes, capacity, Dv, normalize, &v)) { set_error("index_init: blob too small"); return ANYLOC_ERR_WORKSPACE; }
  ANYLOC_CHECK_CUDA(cudaMemsetAsync(v.hdr, 0, 256, (cudaStream_t)stream));
  return ANYLOC_OK;
}

extern "C" int anyloc_index_add(void* index, size_t index_bytes, int64_t capacity, int64_t row_offset, const float* rows,
                                int n_rows, int Dv, int normalize, void* stream) {
  ANYLOC_REQUIRE(index && (rows || n_rows == 0), "index_add: null pointer");
  ANYLOC_REQUIRE(n_rows >= 0 && Dv > 0 && Dv % 4 == 0 && row_offset >= 0 && row_offset + n_rows <= capacity,
                 "index_add: bad dims n_rows=%d Dv=%d offset=%lld capacity=%lld", n_rows, Dv, (long long)row_offset,
                 (long long)capacity);
  ANYLOC_REQUIRE_BLOB(index, "index_add", "index");
  ANYLOC_REQUIRE_ALIGNED(rows, 16, "index_add", "rows", "float4 access");
  IndexView v;
  if (!carve_index(index, index_bytes, capacity, Dv, normalize, &v)) {
    set_error("index_add: blob too small (%zu given, %zu needed)", index_bytes, anyloc_index_bytes(capacity, Dv, normalize));
    return ANYLOC_ERR_WORKSPACE;
  }
  if (n_rows == 0) return ANYLOC_OK;
  cudaStream_t st = (cudaStream_t)stream;
  ProfScope ps(PC_TOPK, st, (v.f16 ? 8.0 : 12.0) * (double)n_rows * Dv);
  const size_t off = (size_t)row_offset * Dv;
  if (v.f16)
    ANYLOC_CHECK_CUDA(launch_normalize_rows<true>(rows, n_rows, Dv, normalize, (__half*)v.hi + off, (__half*)v.lo + off,
                                                  v.sq + row_offset, v.dn + row_offset, v.hdr, st));
  else
    ANYLOC_CHECK_CUDA(launch_normalize_rows<false>(rows, n_rows, Dv, normalize, (float*)v.hi + off, (float*)v.lo + off,
                                                   v.sq + row_offset, nullptr, nullptr, st));
  count_launch();
  return ANYLOC_OK;
}

// Growth: the first n_rows rows of every section (and the header) of `src` -> `dst` (a larger blob of the same Dv / normalize).
extern "C" int anyloc_index_copy(void* dst, size_t dst_bytes, int64_t dst_capacity, const void* src, size_t src_bytes,
                                 int64_t src_capacity, int64_t n_rows, int Dv, int normalize, void* stream) {
  ANYLOC_REQUIRE(dst && src && n_rows >= 0 && n_rows <= src_capacity && n_rows <= dst_capacity, "index_copy: bad arguments");
  ANYLOC_REQUIRE_BLOB(dst, "index_copy", "dst");
  ANYLOC_REQUIRE_BLOB(src, "index_copy", "src");
  IndexView d, s;
  if (!carve_index(dst, dst_bytes, dst_capacity, Dv, normalize, &d) ||
      !carve_index(const_cast<void*>(src), src_bytes, src_capacity, Dv, normalize, &s)) {
    set_error("index_copy: blob too small");
    return ANYLOC_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const size_t pb = (size_t)n_rows * d.pair_bytes_per_row;
  ANYLOC_CHECK_CUDA(cudaMemcpyAsync(d.hi, s.hi, pb, cudaMemcpyDeviceToDevice, st));
  ANYLOC_CHECK_CUDA(cudaMemcpyAsync(d.lo, s.lo, pb, cudaMemcpyDeviceToDevice, st));
  ANYLOC_CHECK_CUDA(cudaMemcpyAsync(d.sq, s.sq, (size_t)n_rows * 4, cudaMemcpyDeviceToDevice, st));
  ANYLOC_CHECK_CUDA(cudaMemcpyAsync(d.dn, s.dn, (size_t)n_rows * 4, cudaMemcpyDeviceToDevice, st));
  ANYLOC_CHECK_CUDA(cudaMemcpyAsync(d.hdr, s.hdr, 256, cudaMemcpyDeviceToDevice, st));
  return ANYLOC_OK;
}

// workspace of one search: query pairs + |q|^2 + dn_q + the [n_q, n_db] score matrix + candidate lists + flags
extern "C" size_t anyloc_index_search_workspace_bytes(int64_t n_db, int n_q, int Dv, int normalize) {
  const size_t esz = index_uses_f16(Dv, normalize) ? 2 : 4;
  return 2 * align_up((size_t)n_q * Dv * esz, 256) + 2 * align_up((size_t)n_q * 4, 256) +
         align_up((size_t)n_q * (size_t)n_db * 4, 256) + align_up((size_t)n_q * CAND_MAX * 4, 256) +
         align_up((size_t)n_q * 4, 256) + 256 + 1024;
}

struct SearchWs { void* qu_hi; void* qu_lo; float* qq; float* dnq; float* scores; int32_t* cand; int32_t* cand_n; int* flags; };
static bool carve_search(void* ws, size_t ws_bytes, int64_t n_db, int n_q, int Dv, size_t esz, SearchWs* s) {
  Workspace w(ws, ws_bytes);
  s->qu_hi = w.take<char>((size_t)n_q * Dv * esz);
  s->qu_lo = w.take<char>((size_t)n_q * Dv * esz);
  s->qq = w.take<float>(n_q);
  s->dnq = w.take<float>(n_q);
  s->scores = w.take<float>((size_t)n_q * (size_t)n_db);
  s->cand = w.take<int32_t>((size_t)n_q * CAND_MAX);
  s->cand_n = w.take<int32_t>(n_q);
  s->flags = w.take<int>(64);
  return s->qu_hi && s->qu_lo && s->qq && s->dnq && s->scores && s->cand && s->cand_n && s->flags;
}

// The search of rows [first, first + n_db) of a carved index.  Resident (MERGE = false, first = row0 = 0, n_total = n_db):
// the k best are written to dist / idx.  Continuation (MERGE): those rows are global rows [row0, row0 + n_db) of a
// database of n_total rows, and their k best are merged into the running list dist / idx.  The route follows n_total,
// so that every piece is answered by the product the resident search of the whole database would use.
template <bool MERGE>
static int search_rows(const IndexView& v0, int64_t first, int64_t n_db, int64_t row0, int64_t n_total, const float* qu,
                       int n_q, int Dv, int k, int metric, int normalize, float* dist, int64_t* idx, void* ws,
                       size_t ws_bytes, cudaStream_t st) {
  void* stream = st;
  const size_t esz = v0.f16 ? 2 : 4;
  IndexView v = v0;
  if constexpr (MERGE) {
    v.hi = (char*)v0.hi + (size_t)first * Dv * esz;
    v.lo = (char*)v0.lo + (size_t)first * Dv * esz;
    v.sq = v0.sq + first;
  } else {
    (void)first; (void)row0; (void)n_total;
  }
  SearchWs s;
  if (!carve_search(ws, ws_bytes, n_db, n_q, Dv, esz, &s)) {
    set_error("index_search: workspace too small (%zu given, %zu needed)", ws_bytes,
              anyloc_index_search_workspace_bytes(n_db, n_q, Dv, normalize));
    return ANYLOC_ERR_WORKSPACE;
  }
  void *qu_hi = s.qu_hi, *qu_lo = s.qu_lo;
  float *qq = s.qq, *dnq = s.dnq, *scores = s.scores;
  int32_t *cand = s.cand, *cand_n = s.cand_n;
  int* flags = s.flags;
  int rc;
  {
    ProfScope ps(PC_TOPK, st, (v.f16 ? 8.0 : 12.0) * (double)n_q * Dv);
    if (v.f16) ANYLOC_CHECK_CUDA(launch_normalize_rows<true>(qu, n_q, Dv, normalize, qu_hi, qu_lo, qq, dnq, nullptr, st));
    else ANYLOC_CHECK_CUDA(launch_normalize_rows<false>(qu, n_q, Dv, normalize, qu_hi, qu_lo, qq, nullptr, nullptr, st));
    count_launch();
  }
  const float alpha = v.f16 ? 1.0f / (kRetrievalScale * kRetrievalScale) : 1.0f;
  const int pair = v.f16 ? ANYLOC_PAIR_F16 : ANYLOC_PAIR_TF32;
  // ---- coarse pass + exact re-scoring of the candidates (inner product, fp16 index)
  const bool coarse = v.f16 && metric == ANYLOC_METRIC_IP && k <= COARSE_K_MAX && (MERGE ? n_total : n_db) >= 1024 &&
                      n_q >= 32;
  const int* gate = nullptr;
  if (coarse) {
    ANYLOC_CHECK_CUDA(cudaMemsetAsync(flags, 0, 256, st));
    // hi-only GEMM: a_lo = b_lo = nullptr selects the single-pass kernels of the tensor-core engine (recorded under PC_GEMM_TC
    // with the FULL 2*n_q*n_db*Dv algorithmic FLOPs: the coarse pass + re-scoring replace the whole product)
    rc = anyloc_gemm_nt(qu_hi, nullptr, Dv, v.hi, nullptr, Dv, n_q, (int)n_db, Dv, pair, alpha, ANYLOC_EPI_BIAS, nullptr,
                        nullptr, nullptr, scores, nullptr, (int)n_db, ANYLOC_PAIR_TF32, ANYLOC_GEMM_TC3, stream);
    if (rc) return rc;
    ProfScope ps(PC_TOPK, st, 8.0 * (double)n_q * (double)n_db);
    topk_candidates_kernel<MERGE><<<n_q, 1024, 0, st>>>(scores, (int)n_db, n_db, k, dnq, v.hdr, cand, cand_n, flags,
                                                        dist);
    ANYLOC_CHECK_LAUNCH();
    topk_rescore_kernel<MERGE><<<n_q, 256, 0, st>>>((const __half*)v.hi, (const __half*)v.lo, (const __half*)qu_hi,
                                                    (const __half*)qu_lo, Dv, k, cand, cand_n, flags, dist, idx,
                                                    (int)row0);
    ANYLOC_CHECK_LAUNCH();
    gate = flags;            // the exact path below only runs (on the device) if a candidate list overflowed
  }
  // ---- exact path: 3-term score GEMM on the tensor-core engine (gemm_dispatch records it under PC_GEMM_TC) + selection
  rc = anyloc_gemm_nt_gated(qu_hi, qu_lo, Dv, v.hi, v.lo, Dv, n_q, (int)n_db, Dv, pair, alpha, scores, (int)n_db, gate, stream);
  if (rc) return rc;
  {
    ProfScope ps(PC_TOPK, st, gate ? 0.0 : 8.0 * (double)n_q * (double)n_db);
    topk_select2_kernel<MERGE><<<n_q, 1024, 0, st>>>(scores, (int)n_db, n_db, k, metric, qq, v.sq, dist, idx, gate,
                                                     (int)row0);
    ANYLOC_CHECK_LAUNCH();
  }
  return ANYLOC_OK;
}

extern "C" int anyloc_index_search(const void* index, size_t index_bytes, int64_t capacity, int64_t n_db, const float* qu,
                                   int n_q, int Dv, int k, int metric, int normalize, float* dist, int64_t* idx, void* ws,
                                   size_t ws_bytes, void* stream) {
  ANYLOC_REQUIRE(index && qu && dist && idx && ws, "index_search: null pointer");
  ANYLOC_REQUIRE(n_db > 0 && n_db <= capacity && n_db < (1ll << 31) && n_q >= 0 && Dv > 0 && k > 0,
                 "index_search: bad dims n_db=%lld n_q=%d Dv=%d k=%d", (long long)n_db, n_q, Dv, k);
  ANYLOC_REQUIRE(Dv % 4 == 0, "index_search: Dv=%d must be a multiple of 4", Dv);
  ANYLOC_REQUIRE(metric == ANYLOC_METRIC_IP || metric == ANYLOC_METRIC_L2, "index_search: unknown metric %d", metric);
  ANYLOC_REQUIRE_BLOB(index, "index_search", "index");
  ANYLOC_REQUIRE_ALIGNED(qu, 16, "index_search", "qu", "float4 access");
  ANYLOC_REQUIRE_BLOB(ws, "index_search", "ws");
  const int rc = search_out_alignment("index_search", dist, idx);
  if (rc) return rc;
  if (n_q == 0) return ANYLOC_OK;
  IndexView v;
  if (!carve_index(const_cast<void*>(index), index_bytes, capacity, Dv, normalize, &v)) {
    set_error("index_search: index blob too small");
    return ANYLOC_ERR_WORKSPACE;
  }
  return search_rows<false>(v, 0, n_db, 0, n_db, qu, n_q, Dv, k, metric, normalize, dist, idx, ws, ws_bytes,
                            (cudaStream_t)stream);
}

extern "C" int anyloc_index_search_continue(const void* index, size_t index_bytes, int64_t capacity, int64_t first,
                                            int64_t n_rows, int64_t row0, int64_t n_total, const float* qu, int n_q,
                                            int Dv, int k, int metric, int normalize, float* dist, int64_t* idx,
                                            void* ws, size_t ws_bytes, void* stream) {
  ANYLOC_REQUIRE(index && qu && dist && idx && ws, "index_search_continue: null pointer");
  ANYLOC_REQUIRE(n_rows > 0 && first >= 0 && first + n_rows <= capacity && row0 >= 0 && row0 + n_rows <= n_total &&
                 n_total < (1ll << 31) && n_q >= 0 && Dv > 0 && k > 0,
                 "index_search_continue: bad dims first=%lld n_rows=%lld row0=%lld n_total=%lld capacity=%lld n_q=%d "
                 "Dv=%d k=%d", (long long)first, (long long)n_rows, (long long)row0, (long long)n_total,
                 (long long)capacity, n_q, Dv, k);
  ANYLOC_REQUIRE(k <= SEL_CAP, "index_search_continue: k=%d above %d (the running list is merged in shared memory)", k,
                 SEL_CAP);
  ANYLOC_REQUIRE(Dv % 4 == 0, "index_search_continue: Dv=%d must be a multiple of 4", Dv);
  ANYLOC_REQUIRE(metric == ANYLOC_METRIC_IP || metric == ANYLOC_METRIC_L2, "index_search_continue: unknown metric %d",
                 metric);
  ANYLOC_REQUIRE_BLOB(index, "index_search_continue", "index");
  ANYLOC_REQUIRE_ALIGNED(qu, 16, "index_search_continue", "qu", "float4 access");
  ANYLOC_REQUIRE_BLOB(ws, "index_search_continue", "ws");
  const int rc = search_out_alignment("index_search_continue", dist, idx);
  if (rc) return rc;
  if (n_q == 0) return ANYLOC_OK;
  IndexView v;
  if (!carve_index(const_cast<void*>(index), index_bytes, capacity, Dv, normalize, &v)) {
    set_error("index_search_continue: index blob too small");
    return ANYLOC_ERR_WORKSPACE;
  }
  return search_rows<true>(v, first, n_rows, row0, n_total, qu, n_q, Dv, k, metric, normalize, dist, idx, ws, ws_bytes,
                           (cudaStream_t)stream);
}

// ---- split index: an fp16-pair index (normalize = 1, Dv % 8 == 0) whose lo halves live in caller-owned page-locked
// host memory, lo [capacity, Dv] fp16, and whose device blob is hi | sq | dn | header (carve_index(split = true)).  Every
// value is the one the resident index holds (the same kernel writes them); only where lo lives differs.
static bool split_carve(const void* blob, size_t bytes, int64_t capacity, int Dv, IndexView* v) {
  return carve_index(const_cast<void*>(blob), bytes, capacity, Dv, 1, v, true);
}

// the device address of the host lo array (page-locked memory is mapped into the unified address space)
static __half* split_lo(const void* lo, const char* what) {
  cudaPointerAttributes a;
  if (!lo || cudaPointerGetAttributes(&a, lo) != cudaSuccess || a.type != cudaMemoryTypeHost || !a.devicePointer) {
    cudaGetLastError();
    set_error("%s: lo must be page-locked host memory (cudaHostAlloc, torch pin_memory)", what);
    return nullptr;
  }
  return (__half*)a.devicePointer;
}

extern "C" size_t anyloc_index_split_bytes(int64_t capacity, int Dv) {
  return align_up((size_t)capacity * Dv * 2, 256) + 2 * align_up((size_t)capacity * 4, 256) + 256 + 256;
}

extern "C" int anyloc_index_split_init(void* index, size_t index_bytes, int64_t capacity, int Dv, void* stream) {
  ANYLOC_REQUIRE(index && capacity >= 0 && Dv > 0 && Dv % 8 == 0,
                 "index_split_init: bad arguments (capacity=%lld, Dv=%d must be a positive multiple of 8)",
                 (long long)capacity, Dv);
  ANYLOC_REQUIRE_BLOB(index, "index_split_init", "index");
  IndexView v;
  if (!split_carve(index, index_bytes, capacity, Dv, &v)) { set_error("index_split_init: blob too small"); return ANYLOC_ERR_WORKSPACE; }
  ANYLOC_CHECK_CUDA(cudaMemsetAsync(v.hdr, 0, 256, (cudaStream_t)stream));
  return ANYLOC_OK;
}

extern "C" int anyloc_index_split_copy(void* dst, size_t dst_bytes, int64_t dst_capacity, const void* src,
                                       size_t src_bytes, int64_t src_capacity, int64_t n_rows, int Dv, void* stream) {
  ANYLOC_REQUIRE(dst && src && n_rows >= 0 && n_rows <= src_capacity && n_rows <= dst_capacity && Dv > 0 && Dv % 8 == 0,
                 "index_split_copy: bad arguments");
  ANYLOC_REQUIRE_BLOB(dst, "index_split_copy", "dst");
  ANYLOC_REQUIRE_BLOB(src, "index_split_copy", "src");
  IndexView d, s;
  if (!split_carve(dst, dst_bytes, dst_capacity, Dv, &d) || !split_carve(src, src_bytes, src_capacity, Dv, &s)) {
    set_error("index_split_copy: blob too small");
    return ANYLOC_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  ANYLOC_CHECK_CUDA(cudaMemcpyAsync(d.hi, s.hi, (size_t)n_rows * d.pair_bytes_per_row, cudaMemcpyDeviceToDevice, st));
  ANYLOC_CHECK_CUDA(cudaMemcpyAsync(d.sq, s.sq, (size_t)n_rows * 4, cudaMemcpyDeviceToDevice, st));
  ANYLOC_CHECK_CUDA(cudaMemcpyAsync(d.dn, s.dn, (size_t)n_rows * 4, cudaMemcpyDeviceToDevice, st));
  ANYLOC_CHECK_CUDA(cudaMemcpyAsync(d.hdr, s.hdr, 256, cudaMemcpyDeviceToDevice, st));
  return ANYLOC_OK;
}

extern "C" int anyloc_index_split_add(void* index, size_t index_bytes, int64_t capacity, void* lo, int64_t row_offset,
                                      const float* rows, int n_rows, int Dv, void* stream) {
  ANYLOC_REQUIRE(index && (rows || n_rows == 0), "index_split_add: null pointer");
  ANYLOC_REQUIRE(n_rows >= 0 && Dv > 0 && Dv % 8 == 0 && row_offset >= 0 && row_offset + n_rows <= capacity,
                 "index_split_add: bad dims n_rows=%d Dv=%d (a multiple of 8) offset=%lld capacity=%lld", n_rows, Dv,
                 (long long)row_offset, (long long)capacity);
  ANYLOC_REQUIRE_BLOB(index, "index_split_add", "index");
  ANYLOC_REQUIRE_BLOB(lo, "index_split_add", "lo");
  ANYLOC_REQUIRE_ALIGNED(rows, 16, "index_split_add", "rows", "float4 access");
  IndexView v;
  if (!split_carve(index, index_bytes, capacity, Dv, &v)) {
    set_error("index_split_add: blob too small (%zu given, %zu needed)", index_bytes, anyloc_index_split_bytes(capacity, Dv));
    return ANYLOC_ERR_WORKSPACE;
  }
  __half* lo_d = split_lo(lo, "index_split_add");
  if (!lo_d) return ANYLOC_ERR_ARG;
  if (n_rows == 0) return ANYLOC_OK;
  cudaStream_t st = (cudaStream_t)stream;
  ProfScope ps(PC_TOPK, st, 8.0 * (double)n_rows * Dv);
  const size_t off = (size_t)row_offset * Dv;
  ANYLOC_CHECK_CUDA(launch_normalize_rows<true>(rows, n_rows, Dv, 1, (__half*)v.hi + off, lo_d + off, v.sq + row_offset,
                                                v.dn + row_offset, v.hdr, st));
  count_launch();
  return ANYLOC_OK;
}

extern "C" int anyloc_index_split_piece(void* dst, size_t dst_bytes, int64_t dst_capacity, const void* index,
                                        size_t index_bytes, int64_t capacity, const void* lo, int64_t first,
                                        int64_t n_rows, int Dv, void* stream) {
  ANYLOC_REQUIRE(dst && index && first >= 0 && n_rows >= 0 && first + n_rows <= capacity && n_rows <= dst_capacity &&
                 Dv > 0 && Dv % 8 == 0, "index_split_piece: bad arguments first=%lld n_rows=%lld capacity=%lld "
                 "dst_capacity=%lld Dv=%d", (long long)first, (long long)n_rows, (long long)capacity,
                 (long long)dst_capacity, Dv);
  ANYLOC_REQUIRE_BLOB(dst, "index_split_piece", "dst");
  ANYLOC_REQUIRE_BLOB(index, "index_split_piece", "index");
  ANYLOC_REQUIRE_BLOB(lo, "index_split_piece", "lo");
  IndexView d, s;
  if (!carve_index(dst, dst_bytes, dst_capacity, Dv, 1, &d) || !split_carve(index, index_bytes, capacity, Dv, &s)) {
    set_error("index_split_piece: blob too small");
    return ANYLOC_ERR_WORKSPACE;
  }
  const __half* lo_d = split_lo(lo, "index_split_piece");
  if (!lo_d) return ANYLOC_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t pb = (size_t)n_rows * d.pair_bytes_per_row;
  ANYLOC_CHECK_CUDA(cudaMemcpyAsync(d.hi, (const __half*)s.hi + (size_t)first * Dv, pb, cudaMemcpyDeviceToDevice, st));
  ANYLOC_CHECK_CUDA(cudaMemcpyAsync(d.lo, lo_d + (size_t)first * Dv, pb, cudaMemcpyDefault, st));
  ANYLOC_CHECK_CUDA(cudaMemcpyAsync(d.sq, s.sq + first, (size_t)n_rows * 4, cudaMemcpyDeviceToDevice, st));
  ANYLOC_CHECK_CUDA(cudaMemcpyAsync(d.dn, s.dn + first, (size_t)n_rows * 4, cudaMemcpyDeviceToDevice, st));
  ANYLOC_CHECK_CUDA(cudaMemcpyAsync(d.hdr, s.hdr, 256, cudaMemcpyDeviceToDevice, st));
  return ANYLOC_OK;
}

// The coarse route of a split index.  The candidates' lo rows reach the unchanged topk_rescore_kernel through a staging
// blob: the chunk's candidate rows are de-duplicated on the device and given staging slots in ascending row order (so
// the rescore's (score desc, index asc) order over slots is its order over rows), their hi (HBM) and lo (host memory)
// rows are gathered into the slots, the lists are remapped to slots, and the k best are mapped back to rows.
namespace anyloc {
// every candidate row of the chunk: slot[row] = 1; cnt[1] += the candidates of the query
__global__ void __launch_bounds__(256)
split_mark_kernel(const int32_t* __restrict__ cand, const int32_t* __restrict__ cand_n, int32_t* __restrict__ slot,
                  int* __restrict__ cnt) {
  const int q = blockIdx.x, n = cand_n[q];
  for (int c = threadIdx.x; c < n; c += blockDim.x) slot[cand[(size_t)q * CAND_MAX + c]] = 1;
  if (threadIdx.x == 0 && n) atomicAdd(cnt + 1, n);
}

// one CTA: each marked row gets slot[row] = its rank among the marked rows, row_of[rank] = row; cnt[0] = their count
__global__ void __launch_bounds__(1024)
split_scan_kernel(int32_t* __restrict__ slot, int n_db, int32_t* __restrict__ row_of, int* __restrict__ cnt) {
  __shared__ int wsum[32];
  const int per = (n_db + blockDim.x - 1) / blockDim.x;
  const int b = min(n_db, (int)threadIdx.x * per), e = min(n_db, b + per);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int own = 0;
  for (int j = b; j < e; ++j) own += slot[j];
  int x = own;                                           // inclusive scan over the block, warp by warp
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  if (lane == 31) wsum[w] = x;
  __syncthreads();
  if (w == 0) {
    int t = lane < (int)(blockDim.x >> 5) ? wsum[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, t, o); if (lane >= o) t += y; }
    wsum[lane] = t;
  }
  __syncthreads();
  int r = x - own + (w ? wsum[w - 1] : 0);
  for (int j = b; j < e; ++j)
    if (slot[j]) { row_of[r] = j; slot[j] = r++; }
  if (threadIdx.x == blockDim.x - 1) cnt[0] = r;
}

// staging slot blockIdx.x <- database row row_of[slot]: hi from the device blob, lo from host memory through its
// unified address.  16-byte loads, 4 per thread and array issued before any store, so that ~1000 resident CTAs keep
// thousands of host reads in flight.
__global__ void __launch_bounds__(256)
split_gather_kernel(const uint4* __restrict__ hi, const uint4* __restrict__ lo, const int32_t* __restrict__ row_of,
                    int n16, uint4* __restrict__ st_hi, uint4* __restrict__ st_lo) {
  const size_t src = (size_t)row_of[blockIdx.x] * n16, dst = (size_t)blockIdx.x * n16;
  for (int t0 = threadIdx.x; t0 < n16; t0 += 4 * blockDim.x) {
    uint4 l[4], h[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int t = t0 + u * blockDim.x;
      if (t < n16) { l[u] = __ldg(lo + src + t); h[u] = __ldg(hi + src + t); }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int t = t0 + u * blockDim.x;
      if (t < n16) { st_lo[dst + t] = l[u]; st_hi[dst + t] = h[u]; }
    }
  }
}

__global__ void __launch_bounds__(256)
split_remap_kernel(int32_t* __restrict__ cand, const int32_t* __restrict__ cand_n, const int32_t* __restrict__ slot) {
  const int q = blockIdx.x;
  for (int c = threadIdx.x; c < cand_n[q]; c += blockDim.x) {
    int32_t* p = cand + (size_t)q * CAND_MAX + c;
    *p = slot[*p];
  }
}

__global__ void __launch_bounds__(256)
split_unmap_kernel(int64_t* __restrict__ idx, int64_t n, const int32_t* __restrict__ row_of) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && idx[i] >= 0) idx[i] = row_of[idx[i]];
}
}  // namespace anyloc

// the search workspace, then slot [n_db] and row_of [n_q * CAND_MAX]
struct SplitWs { SearchWs s; int32_t* slot; int32_t* row_of; };
static bool carve_split_search(void* ws, size_t ws_bytes, int64_t n_db, int n_q, int Dv, SplitWs* w) {
  const size_t head = anyloc_index_search_workspace_bytes(n_db, n_q, Dv, 1);
  if (!carve_search(ws, ws_bytes, n_db, n_q, Dv, 2, &w->s) || ws_bytes < head) return false;
  Workspace t((char*)ws + head, ws_bytes - head);
  w->slot = t.take<int32_t>((size_t)n_db);
  w->row_of = t.take<int32_t>((size_t)n_q * CAND_MAX);
  return w->slot && w->row_of;
}

extern "C" size_t anyloc_index_split_search_workspace_bytes(int64_t n_db, int n_q, int Dv) {
  return anyloc_index_search_workspace_bytes(n_db, n_q, Dv, 1) + align_up((size_t)n_db * 4, 256) +
         align_up((size_t)n_q * CAND_MAX * 4, 256);
}

extern "C" size_t anyloc_index_split_stage_bytes(int64_t rows, int Dv) {
  return 2 * align_up((size_t)rows * Dv * 2, 256);
}

extern "C" int anyloc_index_split_search(const void* index, size_t index_bytes, int64_t capacity, int64_t n_db,
                                         const float* qu, int n_q, int Dv, int k, void* ws, size_t ws_bytes,
                                         int64_t* counts, void* stream) {
  ANYLOC_REQUIRE(index && qu && ws && counts, "index_split_search: null pointer");
  ANYLOC_REQUIRE_BLOB(index, "index_split_search", "index");
  ANYLOC_REQUIRE_ALIGNED(qu, 16, "index_split_search", "qu", "float4 access");
  ANYLOC_REQUIRE_BLOB(ws, "index_split_search", "ws");
  ANYLOC_REQUIRE_ALIGNED(counts, 8, "index_split_search", "counts", "int64 host array");
  counts[0] = -1; counts[1] = 0;
  ANYLOC_REQUIRE(n_db > 0 && n_db <= capacity && n_db < (1ll << 31) && n_q >= 0 && Dv > 0 && Dv % 8 == 0 && k > 0,
                 "index_split_search: bad dims n_db=%lld n_q=%d Dv=%d (a multiple of 8) k=%d", (long long)n_db, n_q,
                 Dv, k);
  IndexView v;
  if (!split_carve(index, index_bytes, capacity, Dv, &v)) {
    set_error("index_split_search: index blob too small");
    return ANYLOC_ERR_WORKSPACE;
  }
  if (!(k <= COARSE_K_MAX && n_db >= 1024 && n_q >= 32)) return ANYLOC_OK;    // the resident search's route test
  SplitWs w;
  if (!carve_split_search(ws, ws_bytes, n_db, n_q, Dv, &w)) {
    set_error("index_split_search: workspace too small (%zu given, %zu needed)", ws_bytes,
              anyloc_index_split_search_workspace_bytes(n_db, n_q, Dv));
    return ANYLOC_ERR_WORKSPACE;
  }
  const SearchWs& s = w.s;
  cudaStream_t st = (cudaStream_t)stream;
  {
    ProfScope ps(PC_TOPK, st, 8.0 * (double)n_q * Dv);
    ANYLOC_CHECK_CUDA(launch_normalize_rows<true>(qu, n_q, Dv, 1, s.qu_hi, s.qu_lo, s.qq, s.dnq, nullptr, st));
    count_launch();
  }
  ANYLOC_CHECK_CUDA(cudaMemsetAsync(s.flags, 0, 256, st));
  int rc = anyloc_gemm_nt(s.qu_hi, nullptr, Dv, v.hi, nullptr, Dv, n_q, (int)n_db, Dv, ANYLOC_PAIR_F16,
                          1.0f / (kRetrievalScale * kRetrievalScale), ANYLOC_EPI_BIAS, nullptr, nullptr, nullptr,
                          s.scores, nullptr, (int)n_db, ANYLOC_PAIR_TF32, ANYLOC_GEMM_TC3, stream);
  if (rc) return rc;
  ProfScope ps(PC_TOPK, st, 8.0 * (double)n_q * (double)n_db);
  topk_candidates_kernel<false><<<n_q, 1024, 0, st>>>(s.scores, (int)n_db, n_db, k, s.dnq, v.hdr, s.cand, s.cand_n,
                                                      s.flags, nullptr);
  ANYLOC_CHECK_LAUNCH();
  // flags[0]: overflow (topk_candidates_kernel), flags[1]: unique candidate rows, flags[2]: candidate rows
  ANYLOC_CHECK_CUDA(cudaMemsetAsync(w.slot, 0, (size_t)n_db * 4, st));
  split_mark_kernel<<<n_q, 256, 0, st>>>(s.cand, s.cand_n, w.slot, s.flags + 1);
  ANYLOC_CHECK_LAUNCH();
  split_scan_kernel<<<1, 1024, 0, st>>>(w.slot, (int)n_db, w.row_of, s.flags + 1);
  ANYLOC_CHECK_LAUNCH();
  int f[3];
  ANYLOC_CHECK_CUDA(cudaMemcpyAsync(f, s.flags, sizeof(f), cudaMemcpyDeviceToHost, st));
  ANYLOC_CHECK_CUDA(cudaStreamSynchronize(st));
  if (!f[0]) { counts[0] = f[1]; counts[1] = f[2]; }
  return ANYLOC_OK;
}

extern "C" int anyloc_index_split_rescore(const void* index, size_t index_bytes, int64_t capacity, const void* lo,
                                          int64_t n_db, int n_q, int Dv, int k, void* ws, size_t ws_bytes,
                                          int64_t n_unique, void* stage, size_t stage_bytes, float* dist, int64_t* idx,
                                          void* stream) {
  ANYLOC_REQUIRE(index && ws && dist && idx, "index_split_rescore: null pointer");
  ANYLOC_REQUIRE(n_db > 0 && n_db <= capacity && n_db < (1ll << 31) && n_q >= 32 && Dv > 0 && Dv % 8 == 0 && k > 0 &&
                 k <= COARSE_K_MAX && n_unique >= 0 && n_unique <= std::min<int64_t>(n_db, (int64_t)n_q * CAND_MAX),
                 "index_split_rescore: bad dims n_db=%lld n_q=%d Dv=%d k=%d n_unique=%lld", (long long)n_db, n_q, Dv,
                 k, (long long)n_unique);
  ANYLOC_REQUIRE_BLOB(index, "index_split_rescore", "index");
  ANYLOC_REQUIRE_BLOB(lo, "index_split_rescore", "lo");
  ANYLOC_REQUIRE_BLOB(ws, "index_split_rescore", "ws");
  ANYLOC_REQUIRE_BLOB(stage, "index_split_rescore", "stage");
  const int rc = search_out_alignment("index_split_rescore", dist, idx);
  if (rc) return rc;
  IndexView v;
  SplitWs w;
  if (!split_carve(index, index_bytes, capacity, Dv, &v) || !carve_split_search(ws, ws_bytes, n_db, n_q, Dv, &w)) {
    set_error("index_split_rescore: index blob or workspace too small");
    return ANYLOC_ERR_WORKSPACE;
  }
  const __half* lo_d = split_lo(lo, "index_split_rescore");
  if (!lo_d) return ANYLOC_ERR_ARG;
  const SearchWs& s = w.s;
  cudaStream_t st = (cudaStream_t)stream;
  ProfScope ps(PC_TOPK, st, 4.0 * (double)n_unique * Dv);
  const __half *db_hi = (const __half*)v.hi, *db_lo = lo_d;
  if (stage) {
    ANYLOC_REQUIRE(stage_bytes >= anyloc_index_split_stage_bytes(n_unique, Dv),
                   "index_split_rescore: stage too small (%zu given, %zu needed)", stage_bytes,
                   anyloc_index_split_stage_bytes(n_unique, Dv));
    __half* st_hi = (__half*)stage;
    __half* st_lo = (__half*)((char*)stage + align_up((size_t)n_unique * Dv * 2, 256));
    if (n_unique) {
      split_gather_kernel<<<(unsigned)n_unique, 256, 0, st>>>((const uint4*)v.hi, (const uint4*)lo_d, w.row_of, Dv / 8,
                                                              (uint4*)st_hi, (uint4*)st_lo);
      ANYLOC_CHECK_LAUNCH();
    }
    split_remap_kernel<<<n_q, 256, 0, st>>>(s.cand, s.cand_n, w.slot);
    ANYLOC_CHECK_LAUNCH();
    db_hi = st_hi; db_lo = st_lo;
  }
  topk_rescore_kernel<false><<<n_q, 256, 0, st>>>(db_hi, db_lo, (const __half*)s.qu_hi, (const __half*)s.qu_lo, Dv, k,
                                                  s.cand, s.cand_n, s.flags, dist, idx, 0);
  ANYLOC_CHECK_LAUNCH();
  if (stage) {
    const int64_t n = (int64_t)n_q * k;
    split_unmap_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(idx, n, w.row_of);
    ANYLOC_CHECK_LAUNCH();
  }
  return ANYLOC_OK;
}

// One-shot form (get_top_k_recall builds the index and searches it once, utilities.py:449-450): a temporary index in
// the caller's workspace, then the search above.
extern "C" size_t anyloc_topk_workspace_bytes(int n_db, int n_q, int Dv, int k) {
  (void)k;
  // sized for the larger (tf32-pair) layout so that the same buffer serves normalize = 0 / 1
  return anyloc_index_bytes(n_db, (int)align_up((size_t)Dv, 4), 0) +
         anyloc_index_search_workspace_bytes(n_db, n_q, (int)align_up((size_t)Dv, 4), 0) + 512;
}

extern "C" int anyloc_topk(const float* db, const float* qu, int n_db, int n_q, int Dv, int k, int metric,
                           int normalize, float* dist, int64_t* idx, void* ws, size_t ws_bytes,
                           void* stream) {
  ANYLOC_REQUIRE(db && qu && dist && idx && ws, "topk: null pointer");
  ANYLOC_REQUIRE(n_db > 0 && n_q >= 0 && Dv > 0 && k > 0, "topk: bad dims n_db=%d n_q=%d Dv=%d k=%d", n_db, n_q, Dv, k);
  ANYLOC_REQUIRE(Dv % 4 == 0, "topk: Dv=%d must be a multiple of 4", Dv);
  ANYLOC_REQUIRE(metric == ANYLOC_METRIC_IP || metric == ANYLOC_METRIC_L2, "topk: unknown metric %d", metric);
  ANYLOC_REQUIRE_ALIGNED(db, 16, "topk", "db", "float4 access");
  ANYLOC_REQUIRE_ALIGNED(qu, 16, "topk", "qu", "float4 access");
  ANYLOC_REQUIRE_BLOB(ws, "topk", "ws");
  int rc = search_out_alignment("topk", dist, idx);
  if (rc) return rc;
  if (n_q == 0) return ANYLOC_OK;
  const size_t ib = anyloc_index_bytes(n_db, Dv, normalize);
  // the documented size, whichever pair format this call picks (it covers the carve below in every case)
  const size_t need = anyloc_topk_workspace_bytes(n_db, n_q, Dv, k);
  if (ws_bytes < need) {
    set_error("topk: workspace too small (%zu given, %zu needed)", ws_bytes, need);
    return ANYLOC_ERR_WORKSPACE;
  }
  rc = anyloc_index_init(ws, ib, n_db, Dv, normalize, stream);
  if (rc) return rc;
  if ((rc = anyloc_index_add(ws, ib, n_db, 0, db, n_db, Dv, normalize, stream))) return rc;
  char* rest = (char*)ws + align_up(ib, 256);
  return anyloc_index_search(ws, ib, n_db, n_db, qu, n_q, Dv, k, metric, normalize, dist, idx, rest,
                             ws_bytes - align_up(ib, 256), stream);
}
