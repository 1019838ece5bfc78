// Hard-assignment VLAD (reference: /root/reference/utilities.py:819-926, residuals :956-962,
// assignment fpk.KMeans.predict :849).  See include/anyloc_b200.h for the contract.
//
// Hard VLAD per call:
//   centre_prep : c^_k = c_k/(|c_k|+1e-8) (cosine) or c_k with bias -|c_k|^2/2 (euclid), plus a tf32-rounded copy
//                 (once per vocabulary with anyloc_vlad_prepare)
//   coarse      : S~[R,K] = X . c^T on the tensor-core (wgmma) GEMM engine, single tf32 pass straight from the raw fp32
//                 features (no conversion pass; the tensor core truncates) -- HBM-bound, reads X once
//   rescore     : warp per row: |x|, candidate set {k : S~_k >= max - 2 eps} with the rigorous tf32 bound
//                 eps = 2^-9 |x| max|c^|, exact fp32 dot products only for the candidates (row held in registers),
//                 first-max argmax -> labels identical to an exact fp32 evaluation; 1/max(|x|,1e-12)
//   accumulate3 : CTA per (128-column slice, image): rows sorted by label, sum_{label=k}(x^ - c_k) in registers, then
//                 the intra + global L2 normalisation in the same kernel.  Images of more rows than its shared memory
//                 holds take accumulate2 (shared-memory accumulators) + the normalise launch.
//   sorted      : (anyloc_vlad_generate_sorted, the shapes neither holds) accumulate3's order with its per-image tables
//                 in the workspace: sort, accumulate, combine and normalise launches.
// (The FFMA assignment kernel serves D > 2048, calls of fewer than 256 rows and workspaces without room for the
// coarse scores, at any K.)
#include <algorithm>
#include <vector>
#include "epilogue.cuh"

namespace anyloc {

// ------------------------------------------------------------------ centre prep
__global__ void vlad_centre_prep_kernel(const float* __restrict__ c, int K, int D, int dist_mode,
                                        float* __restrict__ chat, float* __restrict__ cbias,
                                        float* __restrict__ chat_tf32, float* __restrict__ cnorm,
                                        int32_t* __restrict__ tickets, int n_tickets) {
  // the accumulate3 tickets of this call are cleared here (saves a memset node)
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_tickets; i += gridDim.x * blockDim.x) tickets[i] = 0;
  int k = blockIdx.x;
  const float* row = c + (size_t)k * D;
  float ss = 0.f;
  for (int d = threadIdx.x; d < D; d += blockDim.x) { float v = row[d]; ss += v * v; }
  __shared__ float red[32];
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) red[0] = v;
  }
  __syncthreads();
  ss = red[0];
  if (dist_mode == ANYLOC_DIST_COSINE) {
    const float den = sqrtf(ss) + 1e-8f;            // fpk cos_sim: b / (|b| + 1e-8)
    for (int d = threadIdx.x; d < D; d += blockDim.x) {
      float v = row[d] / den, h, l;
      chat[(size_t)k * D + d] = v;
      if (chat_tf32) { split_tf32(v, h, l); chat_tf32[(size_t)k * D + d] = h; }
    }
    if (threadIdx.x == 0) { cbias[k] = 0.f; if (cnorm) cnorm[k] = sqrtf(ss) / den; }
  } else {
    // argmax_k 2 x.c_k - |x|^2 - |c_k|^2  ==  argmax_k (x.c_k - |c_k|^2/2)
    for (int d = threadIdx.x; d < D; d += blockDim.x) {
      float v = row[d], h, l;
      chat[(size_t)k * D + d] = v;
      if (chat_tf32) { split_tf32(v, h, l); chat_tf32[(size_t)k * D + d] = h; }
    }
    if (threadIdx.x == 0) { cbias[k] = -0.5f * ss; if (cnorm) cnorm[k] = sqrtf(ss); }
  }
}

// ------------------------------------------------------------------ assign
// One warp handles ROWS rows at a time; lanes stride the feature dimension in float4.
template <int ROWS>
__global__ void __launch_bounds__(256)
vlad_assign_kernel(const float* __restrict__ x, const int32_t* __restrict__ n_valid, int N_per_img,
                   int64_t R, int D, int K, const float* __restrict__ chat,
                   const float* __restrict__ cbias, int32_t* __restrict__ labels,
                   float* __restrict__ inv_norm) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int D4 = D >> 2;
  for (int64_t r0 = warp * ROWS; r0 < R; r0 += nwarps * ROWS) {
    const float4* xr[ROWS];
    bool valid[ROWS];
#pragma unroll
    for (int i = 0; i < ROWS; ++i) {
      int64_t r = r0 + i;
      valid[i] = r < R;
      if (valid[i] && n_valid) {
        int b = (int)(r / N_per_img), n = (int)(r % N_per_img);
        valid[i] = n < n_valid[b];
      }
      xr[i] = reinterpret_cast<const float4*>(x + (valid[i] ? r : r0) * (int64_t)D);
      if (r0 + i >= R) xr[i] = reinterpret_cast<const float4*>(x + r0 * (int64_t)D);
    }
    float ss[ROWS];
#pragma unroll
    for (int i = 0; i < ROWS; ++i) ss[i] = 0.f;
    for (int d = lane; d < D4; d += 32) {
#pragma unroll
      for (int i = 0; i < ROWS; ++i) {
        float4 v = __ldg(xr[i] + d);
        ss[i] += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
      }
    }
    float best[ROWS]; int bestk[ROWS];
#pragma unroll
    for (int i = 0; i < ROWS; ++i) { ss[i] = warp_sum(ss[i]); best[i] = -INFINITY; bestk[i] = 0; }
    for (int k = 0; k < K; ++k) {
      const float4* cr = reinterpret_cast<const float4*>(chat + (size_t)k * D);
      float acc[ROWS];
#pragma unroll
      for (int i = 0; i < ROWS; ++i) acc[i] = 0.f;
      for (int d = lane; d < D4; d += 32) {
        float4 c = __ldg(cr + d);
#pragma unroll
        for (int i = 0; i < ROWS; ++i) {
          float4 v = __ldg(xr[i] + d);     // L1-resident after the norm pass
          acc[i] = fmaf(v.x, c.x, acc[i]); acc[i] = fmaf(v.y, c.y, acc[i]);
          acc[i] = fmaf(v.z, c.z, acc[i]); acc[i] = fmaf(v.w, c.w, acc[i]);
        }
      }
      float bk = cbias[k];
#pragma unroll
      for (int i = 0; i < ROWS; ++i) {
        float s = warp_sum(acc[i]) + bk;
        if (s > best[i]) { best[i] = s; bestk[i] = k; }   // strict >: lowest index wins ties
      }
    }
    if (lane == 0) {
#pragma unroll
      for (int i = 0; i < ROWS; ++i) {
        int64_t r = r0 + i;
        if (r < R) {
          labels[r] = valid[i] ? bestk[i] : -1;
          if (inv_norm) inv_norm[r] = 1.0f / fmaxf(sqrtf(ss[i]), 1e-12f);
        }
      }
    }
  }
}

// ------------------------------------------------------------------ rescore (exact labels from coarse scores)
// One warp per row.  The row (D <= 2048) lives in registers; only the candidates whose coarse tf32 score is within
// 2*eps of the row maximum are re-evaluated exactly (fp32 FMA, same c^ as the exact path), so the label equals the
// exact-fp32 argmax (lowest index among exact ties).
template <int MAXV>      // float4 per lane: D <= 128 * MAXV
__global__ void __launch_bounds__(256)
vlad_rescore_kernel(const float* __restrict__ x, const int32_t* __restrict__ n_valid, int N_per_img, int64_t R,
                    int D, int K, const float* __restrict__ chat, const float* __restrict__ cbias,
                    const float* __restrict__ cnorm, const float* __restrict__ coarse /*[R,K]*/,
                    int32_t* __restrict__ labels, float* __restrict__ inv_norm) {
  const int lane = threadIdx.x & 31;
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= R) return;
  bool valid = true;
  if (n_valid) { int b = (int)(row / N_per_img), n = (int)(row % N_per_img); valid = n < n_valid[b]; }
  const int D4 = D >> 2;
  const float4* xr = reinterpret_cast<const float4*>(x + row * (int64_t)D);
  float4 v[MAXV];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    int d = lane + i * 32;
    if (d < D4) { v[i] = __ldg(xr + d); ss += v[i].x * v[i].x + v[i].y * v[i].y + v[i].z * v[i].z + v[i].w * v[i].w; }
  }
  ss = warp_sum(ss);
  const float xn = sqrtf(ss);
  // coarse maximum and the largest centre norm (lanes stride over k)
  float smax = -INFINITY, cmax = 0.f;
  for (int k = lane; k < K; k += 32) {
    smax = fmaxf(smax, coarse[row * K + k]);
    cmax = fmaxf(cmax, cnorm[k]);
  }
  smax = warp_max(smax); cmax = warp_max(cmax);
  // |S~_k - S_k| <= (2^-10 + 2^-11) sum|x_i c_i| <= 1.5 * 2^-10 |x||c_k| < 2^-9 |x||c_k|  (truncated x, rounded c)
  const float thresh = smax - 2.0f * (0.001953125f * xn * cmax) - 1e-30f;
  float best = -INFINITY; int bestk = 0;
  for (int k0 = 0; k0 < K; k0 += 32) {
    const int k = k0 + lane;
    const bool cand = k < K && coarse[row * K + k] >= thresh;
    unsigned mask = __ballot_sync(0xffffffffu, cand);
    while (mask) {
      // up to four candidates at a time (independent accumulators hide the L1/L2 latency of the centre rows)
      int kk[4]; int n = 0;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (mask) { kk[q] = k0 + __ffs(mask) - 1; mask &= mask - 1; ++n; } else kk[q] = kk[0];
      }
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int i = 0; i < MAXV; ++i) {
        int d = lane + i * 32;
        if (d < D4) {
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            float4 c = __ldg(reinterpret_cast<const float4*>(chat + (size_t)kk[q] * D) + d);
            acc[q] = fmaf(v[i].x, c.x, acc[q]); acc[q] = fmaf(v[i].y, c.y, acc[q]);
            acc[q] = fmaf(v[i].z, c.z, acc[q]); acc[q] = fmaf(v[i].w, c.w, acc[q]);
          }
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float sc = warp_sum(acc[q]) + cbias[kk[q]];
        if (q < n && sc > best) { best = sc; bestk = kk[q]; }   // ascending k, strict >: lowest index wins exact ties
      }
    }
  }
  if (lane == 0) {
    labels[row] = valid ? bestk : -1;
    if (inv_norm) inv_norm[row] = 1.0f / fmaxf(xn, 1e-12f);
  }
}

// Several vocabularies' labels from one read of each row (anyloc_vlad_assign_multi).  load_row and rescore_row restate
// vlad_rescore_kernel's row load and its per-row body operation for operation (the same loads, FMAs, reductions and
// candidate order), so each vocabulary's label is the one that kernel computes; vlad_rescore_kernel keeps its own text
// because calling the shared body from it changes its register allocation.
// rescore_row: the label of one row (warp-wide); v holds the row's float4s, xn = |x|, crow its K coarse scores.
template <int MAXV>
__device__ __forceinline__ int rescore_row(const float4 (&v)[MAXV], float xn, int lane, int D, int K,
                                           const float* __restrict__ crow, const float* __restrict__ chat,
                                           const float* __restrict__ cbias, const float* __restrict__ cnorm) {
  const int D4 = D >> 2;
  // coarse maximum and the largest centre norm (lanes stride over k)
  float smax = -INFINITY, cmax = 0.f;
  for (int k = lane; k < K; k += 32) {
    smax = fmaxf(smax, crow[k]);
    cmax = fmaxf(cmax, cnorm[k]);
  }
  smax = warp_max(smax); cmax = warp_max(cmax);
  // |S~_k - S_k| <= (2^-10 + 2^-11) sum|x_i c_i| <= 1.5 * 2^-10 |x||c_k| < 2^-9 |x||c_k|  (truncated x, rounded c)
  const float thresh = smax - 2.0f * (0.001953125f * xn * cmax) - 1e-30f;
  float best = -INFINITY; int bestk = 0;
  for (int k0 = 0; k0 < K; k0 += 32) {
    const int k = k0 + lane;
    const bool cand = k < K && crow[k] >= thresh;
    unsigned mask = __ballot_sync(0xffffffffu, cand);
    while (mask) {
      // up to four candidates at a time (independent accumulators hide the L1/L2 latency of the centre rows)
      int kk[4]; int n = 0;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (mask) { kk[q] = k0 + __ffs(mask) - 1; mask &= mask - 1; ++n; } else kk[q] = kk[0];
      }
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int i = 0; i < MAXV; ++i) {
        int d = lane + i * 32;
        if (d < D4) {
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            float4 c = __ldg(reinterpret_cast<const float4*>(chat + (size_t)kk[q] * D) + d);
            acc[q] = fmaf(v[i].x, c.x, acc[q]); acc[q] = fmaf(v[i].y, c.y, acc[q]);
            acc[q] = fmaf(v[i].z, c.z, acc[q]); acc[q] = fmaf(v[i].w, c.w, acc[q]);
          }
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float sc = warp_sum(acc[q]) + cbias[kk[q]];
        if (q < n && sc > best) { best = sc; bestk = kk[q]; }   // ascending k, strict >: lowest index wins exact ties
      }
    }
  }
  return bestk;
}

template <int MAXV>      // float4 per lane: D <= 128 * MAXV
__device__ __forceinline__ float load_row(const float* __restrict__ x, int64_t row, int D, int lane, float4 (&v)[MAXV]) {
  const int D4 = D >> 2;
  const float4* xr = reinterpret_cast<const float4*>(x + row * (int64_t)D);
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    int d = lane + i * 32;
    if (d < D4) { v[i] = __ldg(xr + d); ss += v[i].x * v[i].x + v[i].y * v[i].y + v[i].z * v[i].z + v[i].w * v[i].w; }
  }
  return sqrtf(warp_sum(ss));
}

// The coarse scores [R, ldc] hold the vocabularies side by side, segment s in columns [koff[s], koff[s] + k[s]) of the scores and rows of the prepared
// centres.  Each segment's candidates, threshold and argmax are vlad_rescore_kernel's for that vocabulary alone.
constexpr int ASSIGN_MULTI_SEGS = 32;      // segments per rescoring launch
struct RescoreSegs {
  int n;
  int koff[ASSIGN_MULTI_SEGS], k[ASSIGN_MULTI_SEGS];
  int32_t* labels[ASSIGN_MULTI_SEGS];      // the segment's labels of this launch's first row
};

template <int MAXV>
__global__ void __launch_bounds__(256)
vlad_rescore_multi_kernel(const float* __restrict__ x, int64_t R, int D, int ldc, const float* __restrict__ chat,
                          const float* __restrict__ cbias, const float* __restrict__ cnorm,
                          const float* __restrict__ coarse /*[R,ldc]*/, const RescoreSegs segs) {
  const int lane = threadIdx.x & 31;
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= R) return;
  float4 v[MAXV];
  const float xn = load_row<MAXV>(x, row, D, lane, v);
  for (int s = 0; s < segs.n; ++s) {
    const int k0 = segs.koff[s];
    const int bestk = rescore_row<MAXV>(v, xn, lane, D, segs.k[s], coarse + row * ldc + k0, chat + (size_t)k0 * D,
                                        cbias + k0, cnorm + k0);
    if (lane == 0) segs.labels[s][row] = bestk;
  }
}

// ------------------------------------------------------------------ accumulate v2
// CTA = (image, 128-column slice); WARPS warps split the rows; lane owns 4 consecutive columns (float4).
// Per-warp accumulators [K][128] in shared memory (no conflicts: a warp touches 512 contiguous bytes per row),
// reduced across warps at the end in a fixed order -> deterministic.
// Image b is rows.count(b) rows from rows.first(b) of x, labels and inv_norm (PaddedRows / PackedRows, common.cuh).
template <class Rows>
__device__ __forceinline__ void accumulate2_image(const float* __restrict__ x, const int32_t* __restrict__ labels,
                                                  const float* __restrict__ inv_norm, const float* __restrict__ centers,
                                                  Rows rows, int D, int K, int norm_descs, int warps,
                                                  float* __restrict__ vlad, float* __restrict__ partial_ss) {
  extern __shared__ float sm[];
  float* cen = sm;                                        // [K][128]
  float* acc = sm + (size_t)K * 128;                      // [warps][K][128]
  const int b = blockIdx.y, slice = blockIdx.x, t = threadIdx.x, lane = t & 31, w = t >> 5;
  const int N = rows.count(b);
  const int col = slice * 128 + lane * 4;
  const bool colok = col < D;                             // D % 4 == 0
  for (int i = t; i < K * 32; i += blockDim.x) {
    const int k = i >> 5, c4 = (i & 31) * 4, gc = slice * 128 + c4;
    float4 cv = gc < D ? __ldg(reinterpret_cast<const float4*>(centers + (size_t)k * D + gc)) : make_float4(0.f, 0.f, 0.f, 0.f);
    *reinterpret_cast<float4*>(cen + k * 128 + c4) = cv;
  }
  for (int i = t; i < warps * K * 32; i += blockDim.x) reinterpret_cast<float4*>(acc)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  __syncthreads();
  if (w < warps && colok) {
    float* my = acc + (size_t)w * K * 128 + lane * 4;
    const float* xb = x + rows.first(b) * D + col;
    const int32_t* lb = labels + rows.first(b);
    const float* ib = inv_norm + rows.first(b);
    constexpr int U = 16;                                 // rows in flight per warp (latency hiding)
    for (int n0 = w; n0 < N; n0 += U * warps) {
      float4 v[U]; int lab[U]; float sc[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int n = n0 + u * warps;
        lab[u] = n < N ? lb[n] : -1;
        sc[u] = (n < N && norm_descs) ? ib[n] : 1.0f;
        v[u] = lab[u] >= 0 ? __ldg(reinterpret_cast<const float4*>(xb + (size_t)n * D)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (lab[u] >= 0) {
          float4 a = *reinterpret_cast<float4*>(my + lab[u] * 128);
          const float4 c = *reinterpret_cast<const float4*>(cen + lab[u] * 128 + lane * 4);
          a.x += v[u].x * sc[u] - c.x; a.y += v[u].y * sc[u] - c.y; a.z += v[u].z * sc[u] - c.z; a.w += v[u].w * sc[u] - c.w;
          *reinterpret_cast<float4*>(my + lab[u] * 128) = a;
        }
      }
    }
  }
  __syncthreads();
  // reduce the warps' partials (fixed order), write V and the per-slice sums of squares
  const int nslices = gridDim.x;
  for (int k = w; k < K; k += blockDim.x >> 5) {          // one warp per cluster row
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int q = 0; q < warps; ++q) {
      float4 p = *reinterpret_cast<const float4*>(acc + ((size_t)q * K + k) * 128 + lane * 4);
      a.x += p.x; a.y += p.y; a.z += p.z; a.w += p.w;
    }
    float ss = 0.f;
    if (colok) {
      *reinterpret_cast<float4*>(vlad + ((size_t)b * K + k) * D + col) = a;
      ss = a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w;
    }
    ss = warp_sum(ss);
    if (lane == 0) partial_ss[((size_t)b * K + k) * nslices + slice] = ss;
  }
}

__global__ void __launch_bounds__(256, 2)
vlad_accumulate2_kernel(const float* __restrict__ x, const int32_t* __restrict__ labels,
                        const float* __restrict__ inv_norm, const float* __restrict__ centers,
                        int N, int D, int K, int norm_descs, int warps, float* __restrict__ vlad,
                        float* __restrict__ partial_ss /* [B,K,nslices] */) {
  accumulate2_image(x, labels, inv_norm, centers, PaddedRows{nullptr, N}, D, K, norm_descs, warps, vlad, partial_ss);
}

// packed images: image b is rows [row0[b], row0[b] + len[b]) of x, labels and inv_norm
__global__ void __launch_bounds__(256, 2)
vlad_accumulate2_varlen_kernel(const float* __restrict__ x, const int32_t* __restrict__ labels,
                               const float* __restrict__ inv_norm, const float* __restrict__ centers,
                               const int64_t* __restrict__ row0, const int32_t* __restrict__ len, int D, int K,
                               int norm_descs, int warps, float* __restrict__ vlad, float* __restrict__ partial_ss) {
  accumulate2_image(x, labels, inv_norm, centers, PackedRows{row0, len}, D, K, norm_descs, warps, vlad, partial_ss);
}

// ------------------------------------------------------------------ normalisation factors
// Image b's intra-normalisation scales scale[k] = 1/max(|V_k|,1e-12) (1 without intra_norm) and its global factor
// 1/max(|(scale_k V_k)_k|,1e-12), from the per-slice sums of squares partial_ss [B,K,nslices], in one fixed order
// (slices in order, then clusters in order), so every CTA that derives them gets the same bits.  scale and sq are [K]
// in shared memory; the block's threads stride over k.  __ldcg: within accumulate3 the sums come from other CTAs of
// the running kernel.  Every thread of the block must call it; it returns the global factor to all of them.
__device__ __forceinline__ float vlad_norm_factors(const float* partial_ss, int b, int K, int nslices, int intra_norm,
                                                   float* scale, float* sq) {
  __shared__ float s_gnorm;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    float ss = 0.f;
    for (int s = 0; s < nslices; ++s) ss += __ldcg(partial_ss + ((size_t)b * K + k) * nslices + s);
    const float nk = sqrtf(ss);
    const float sc = intra_norm ? 1.0f / fmaxf(nk, 1e-12f) : 1.0f;
    scale[k] = sc;
    const float nb = nk * sc;                               // norm of the block after intra-normalisation
    sq[k] = nb * nb;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float tot = 0.f;
    for (int k = 0; k < K; ++k) tot += sq[k];
    s_gnorm = 1.0f / fmaxf(sqrtf(tot), 1e-12f);
  }
  __syncthreads();
  return s_gnorm;
}

// ------------------------------------------------------------------ accumulate v3 (+ fused normalisation)
// CTA = (128-column slice, image), 8 warps, 4-5 CTAs per SM (one wave at the BASELINE shapes).  The image's rows are
// counting-sorted by label in shared memory (stable: rows of a cluster stay in row order), the sorted list is cut into
// tasks of <= 64 rows of ONE cluster, and warps grab tasks dynamically: 8 independent 512-byte row segments in flight
// per warp, the partial sum lives in registers (lane = 4 columns) -- no shared-memory accumulators, no
// read-modify-write chains, and a skewed vocabulary (one cluster holding a third of the image) no longer serialises on
// one warp.  Clusters of several tasks are combined from shared-memory slots in task order, so every sum has ONE fixed
// order: bitwise reproducible, batch == single image.  The last CTA of an image to finish (global ticket) applies the
// intra- and global L2 normalisation to that image's descriptor while it is still in L2 (no separate launch).
constexpr int ACC3_WARPS = 8;
constexpr int ACC3_SEG = 64;
static inline int acc3_max_tasks(int N, int K) { return N / ACC3_SEG + K + 1; }
__device__ __forceinline__ int acc3_max_tasks_dev(int N, int K) { return N / ACC3_SEG + K + 1; }
static inline int acc3_max_slots(int N) { return 2 * (N / ACC3_SEG) + 2; }
static inline size_t acc3_smem_bytes(int N, int K) {
  return ((size_t)4 * N + 3 * (size_t)(K + 1) + (size_t)ACC3_WARPS * K + 2 * (size_t)K + acc3_max_tasks(N, K) + 4) * 4 +
         (size_t)acc3_max_slots(N) * 512;
}

// One task's sum in this lane's 4 columns: sum over the sorted positions [s, e) of one cluster of x * (1/|x|) - c.
// xb points at the columns in the image's first row, ck at the cluster's centre; ooff / inv_s hold each row's offset
// n * D and 1/|x| in sorted order (int in accumulate3's shared memory, int64_t in the sorted route's workspace).  Zero
// for columns past D (colok false).  accumulate3 and the sorted route both sum their tasks here, so their descriptors
// are bitwise equal.  The in-flight bytes live in registers (8 x 16 B per lane = 4 KB per warp; 4 CTAs x 8 warps ->
// 128 KB per SM), so the loop is kept lean: row offsets and 1/|x| were laid out in sorted order by the placement pass.
template <class Off>
__device__ __forceinline__ float4 task_sum(bool colok, const float* ck, const float* xb, const Off* ooff,
                                           const float* inv_s, int s, int e) {
  const float4 c = colok ? __ldg(reinterpret_cast<const float4*>(ck)) : make_float4(0.f, 0.f, 0.f, 0.f);
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  if (colok) {
    constexpr int U = 8;
    int i = s;
    for (; i + U <= e; i += U) {
      float4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) v[u] = __ldg(reinterpret_cast<const float4*>(xb + ooff[i + u]));
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const float sc = inv_s[i + u];
        a.x += v[u].x * sc - c.x; a.y += v[u].y * sc - c.y; a.z += v[u].z * sc - c.z; a.w += v[u].w * sc - c.w;
      }
    }
    if (i < e) {                                             // tail: < U rows, same order
      float4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) if (i + u < e) v[u] = __ldg(reinterpret_cast<const float4*>(xb + ooff[i + u]));
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (i + u < e) {
          const float sc = inv_s[i + u];
          a.x += v[u].x * sc - c.x; a.y += v[u].y * sc - c.y; a.z += v[u].z * sc - c.z; a.w += v[u].w * sc - c.w;
        }
      }
    }
  }
  return a;
}

// A lane's share of a cluster's sum of squares: x*x, then y, z and w by fma.  accumulate3 and the sorted accumulate
// spell it out because a sum of products leaves the fused pair to the compiler, which picks it per kernel, and their
// descriptors must agree bit for bit.  vlad_sorted_combine_kernel still writes the sum of products (sum_sq there costs
// it a register); it compiles to this order today, and test_vlad_large_k_gpu's multi-task layouts hold it there.
__device__ __forceinline__ float sum_sq(float4 a) { return fmaf(a.w, a.w, fmaf(a.z, a.z, fmaf(a.y, a.y, a.x * a.x))); }

// Image b is rows.count(b) <= N rows from rows.first(b) of x, labels and inv_norm (PaddedRows / PackedRows,
// common.cuh); N sizes the shared-memory layout.
template <class Rows>
__device__ __forceinline__ void accumulate3_image(const float* __restrict__ x, const int32_t* __restrict__ labels,
                                                  const float* __restrict__ inv_norm, const float* __restrict__ centers,
                                                  Rows rows, int N, int D, int K, int norm_descs, int intra_norm,
                                                  float* vlad, float* partial_ss, int32_t* done, int wait_all) {
  extern __shared__ __align__(16) int sm3[];
  int* ooff = sm3;                                          // [N] n * D of the rows, sorted by label (stable)
  int* lab = ooff + N;                                      // [N]
  float* inv_s = reinterpret_cast<float*>(lab + N);         // [N] 1/|x| in the same sorted order
  int* start = reinterpret_cast<int*>(inv_s + N);           // [K+1] first sorted position of cluster k
  int* tstart = start + K + 1;                              // [K+1] first task of cluster k
  int* sbase = tstart + K + 1;                              // [K+1] first partial-sum slot of a multi-task cluster
  int* cntw = sbase + K + 1;                                // [ACC3_WARPS][K]
  float* kss = reinterpret_cast<float*>(cntw + ACC3_WARPS * K);   // [K]
  float* ksq = kss + K;                                     // [K]
  int* task_k = reinterpret_cast<int*>(ksq + K);            // [max_tasks]
  float* inv = reinterpret_cast<float*>(task_k + acc3_max_tasks_dev(N, K));   // [N] 1/|x| in row order (prologue only)
  float* slots = reinterpret_cast<float*>(sm3) +
                 (((size_t)4 * N + 3 * (size_t)(K + 1) + (size_t)ACC3_WARPS * K + 2 * (size_t)K + acc3_max_tasks_dev(N, K) + 3) & ~(size_t)3);
  __shared__ int next_task, s_last;
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  // images in reverse order: the assignment pass streamed them in ascending order, so the last ones are the most
  // likely to still sit in L2 when this kernel starts
  const int b = (int)gridDim.y - 1 - (int)blockIdx.y, slice = blockIdx.x, nslices = gridDim.x;
  const int nr = rows.count(b);
  const int col = slice * 128 + lane * 4;
  const bool colok = col < D;                               // D % 4 == 0
  for (int n = t; n < nr; n += blockDim.x) {
    lab[n] = labels[rows.first(b) + n];
    inv[n] = norm_descs ? inv_norm[rows.first(b) + n] : 1.0f;
  }
  for (int i = t; i < ACC3_WARPS * K; i += blockDim.x) cntw[i] = 0;
  if (t == 0) next_task = 0;
  __syncthreads();
  // per-warp histograms over contiguous row chunks
  const int chunk = (((nr + ACC3_WARPS - 1) / ACC3_WARPS) + 31) & ~31;
  const int r0 = min(nr, w * chunk), r1 = min(nr, r0 + chunk);
  for (int n = r0 + lane; n < r1; n += 32) { const int l = lab[n]; if (l >= 0) atomicAdd(&cntw[w * K + l], 1); }
  __syncthreads();
  for (int k = t; k < K; k += blockDim.x) {                 // exclusive prefix over the warps, cluster totals
    int tot = 0;
    for (int ww = 0; ww < ACC3_WARPS; ++ww) { const int c = cntw[ww * K + k]; cntw[ww * K + k] = tot; tot += c; }
    start[k] = tot;
  }
  __syncthreads();
  if (w == 0) {                                             // exclusive scans: rows, tasks, partial-sum slots
    int run_r = 0, run_t = 0, run_s = 0;
    for (int k0 = 0; k0 < K; k0 += 32) {
      const int k = k0 + lane;
      const int c = k < K ? start[k] : 0;
      const int nt = k < K ? max(1, (c + ACC3_SEG - 1) / ACC3_SEG) : 0;
      const int ns = nt > 1 ? nt : 0;
      int ir = c, it = nt, is = ns;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int yr = __shfl_up_sync(0xffffffffu, ir, o), yt = __shfl_up_sync(0xffffffffu, it, o),
                  ys = __shfl_up_sync(0xffffffffu, is, o);
        if (lane >= o) { ir += yr; it += yt; is += ys; }
      }
      if (k < K) { start[k] = run_r + ir - c; tstart[k] = run_t + it - nt; sbase[k] = run_s + is - ns; }
      run_r += __shfl_sync(0xffffffffu, ir, 31);
      run_t += __shfl_sync(0xffffffffu, it, 31);
      run_s += __shfl_sync(0xffffffffu, is, 31);
    }
    if (lane == 0) { start[K] = run_r; tstart[K] = run_t; sbase[K] = run_s; }
  }
  __syncthreads();
  for (int k = t; k < K; k += blockDim.x)                   // task table
    for (int q = tstart[k]; q < tstart[k + 1]; ++q) task_k[q] = k;
  for (int n0 = r0; n0 < r1; n0 += 32) {                    // stable placement
    const int n = n0 + lane;
    const int l = n < r1 ? lab[n] : -1;
    const bool active = l >= 0;
    const float iv = active ? inv[n] : 1.0f;
    const unsigned am = __ballot_sync(0xffffffffu, active);
    unsigned peers = 0; int rank = 0;
    if (active) {
      peers = __match_any_sync(am, l);
      rank = __popc(peers & ((1u << lane) - 1u));
      const int pos = start[l] + cntw[w * K + l] + rank;
      ooff[pos] = n * D;
      inv_s[pos] = iv;
    }
    __syncwarp();
    if (active && rank == 0) cntw[w * K + l] += __popc(peers);
    __syncwarp();
  }
  __syncthreads();
  // tasks -> registers.  Every warp grabs its NEXT task one task early.
  const float* xb = x + rows.first(b) * D + col;
  const int ntasks = tstart[K];
  auto grab = [&]() { int q = 0; if (lane == 0) q = atomicAdd(&next_task, 1); return __shfl_sync(0xffffffffu, q, 0); };
  int q = grab();
  while (q < ntasks) {
    const int qn = grab();
    const int k = task_k[q];
    const int seg = q - tstart[k], nt = tstart[k + 1] - tstart[k];
    const int s = start[k] + seg * ACC3_SEG, e = min(start[k + 1], s + ACC3_SEG);
    const float4 a = task_sum(colok, centers + (size_t)k * D + col, xb, ooff, inv_s, s, e);
    if (nt == 1) {
      if (colok) *reinterpret_cast<float4*>(vlad + ((size_t)b * K + k) * D + col) = a;
      const float ss = warp_sum(sum_sq(a));
      if (lane == 0) kss[k] = ss;
    } else {
      *reinterpret_cast<float4*>(slots + (size_t)(sbase[k] + seg) * 128 + lane * 4) = a;
    }
    q = qn;
  }
  __syncthreads();
  for (int k = w; k < K; k += ACC3_WARPS) {                 // clusters of several tasks: combine in task order
    const int nt = tstart[k + 1] - tstart[k];
    if (nt <= 1) continue;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int q = 0; q < nt; ++q) {
      const float4 p = *reinterpret_cast<const float4*>(slots + (size_t)(sbase[k] + q) * 128 + lane * 4);
      a.x += p.x; a.y += p.y; a.z += p.z; a.w += p.w;
    }
    if (colok) *reinterpret_cast<float4*>(vlad + ((size_t)b * K + k) * D + col) = a;
    const float ss = warp_sum(sum_sq(a));
    if (lane == 0) kss[k] = ss;
  }
  __syncthreads();
  for (int k = t; k < K; k += blockDim.x) partial_ss[((size_t)b * K + k) * nslices + slice] = kss[k];
  __syncthreads();
  if (t == 0) {
    __threadfence();      // cumulative: orders every write the barrier above made visible to this thread (the pattern of
                          // cooperative-groups grid sync), instead of 256 per-thread fences
    s_last = (atomicAdd(&done[b], 1) == nslices - 1);
  }
  __syncthreads();
  if (wait_all) {
    // Whole grid co-resident (checked on the host): every slice-CTA waits until all slices of its image have published
    // their sums of squares, derives the SAME scales in the same order, and normalises ITS OWN 128-column slice -- the
    // normalisation is spread over all CTAs of the image instead of serialising K*D elements behind the last one
    // (measured tail of the last-CTA variant: 10 us of 41 at c2, 30-40 us of 130 at c5).
    if (t == 0) {
      const long long t0 = clock64();
      for (;;) {
        int v;
        asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(done + b) : "memory");
        if (v >= nslices) break;
        __nanosleep(64);
        if (clock64() - t0 > 8000000000LL) __trap();      // never hang the GPU
      }
    }
    __syncthreads();
    const float g = vlad_norm_factors(partial_ss, b, K, nslices, intra_norm, kss, ksq);
    const int nq = K * 32;                                  // float4 elements of this slice
    constexpr int UW = 8;
    for (int i0 = t; i0 < nq; i0 += blockDim.x * UW) {
      float4 v[UW];
#pragma unroll
      for (int u = 0; u < UW; ++u) {
        const int i = i0 + u * blockDim.x, c4 = slice * 128 + (i & 31) * 4;
        if (i < nq && c4 < D) v[u] = __ldcg(reinterpret_cast<const float4*>(vlad + ((size_t)b * K + (i >> 5)) * D + c4));
      }
#pragma unroll
      for (int u = 0; u < UW; ++u) {
        const int i = i0 + u * blockDim.x, c4 = slice * 128 + (i & 31) * 4;
        if (i < nq && c4 < D) {
          const float sc = kss[i >> 5];
          v[u].x = (v[u].x * sc) * g; v[u].y = (v[u].y * sc) * g; v[u].z = (v[u].z * sc) * g; v[u].w = (v[u].w * sc) * g;
          *reinterpret_cast<float4*>(vlad + ((size_t)b * K + (i >> 5)) * D + c4) = v[u];
        }
      }
    }
    return;
  }
  if (!s_last) return;
  // ---- last CTA of this image: intra- and global normalisation (same factors as vlad_normalize_kernel)
  __threadfence();
  if (t == 0) done[b] = 0;
  const float g = vlad_norm_factors(partial_ss, b, K, nslices, intra_norm, kss, ksq);
  float4* vb = reinterpret_cast<float4*>(vlad + (size_t)b * K * D);
  const int D4 = D >> 2, total4 = K * D4;
  constexpr int UN = 8;                                     // loads batched ahead of the stores (L2 latency chain)
  for (int i0 = t; i0 < total4; i0 += blockDim.x * UN) {
    float4 v[UN];
#pragma unroll
    for (int u = 0; u < UN; ++u) {
      const int i = i0 + u * blockDim.x;
      if (i < total4) v[u] = __ldcg(vb + i);
    }
#pragma unroll
    for (int u = 0; u < UN; ++u) {
      const int i = i0 + u * blockDim.x;
      if (i < total4) {
        const float sc = kss[i / D4];
        // two separate multiplications like F.normalize(intra) then F.normalize(global)
        v[u].x = (v[u].x * sc) * g; v[u].y = (v[u].y * sc) * g; v[u].z = (v[u].z * sc) * g; v[u].w = (v[u].w * sc) * g;
        vb[i] = v[u];
      }
    }
  }
}

__global__ void __launch_bounds__(ACC3_WARPS * 32, 4)
vlad_accumulate3_kernel(const float* __restrict__ x, const int32_t* __restrict__ labels,
                        const float* __restrict__ inv_norm, const float* __restrict__ centers, int N, int D, int K,
                        int norm_descs, int intra_norm, float* vlad, float* partial_ss /* [B,K,nslices] */,
                        int32_t* done /* [B], zero on entry */, int wait_all) {
  accumulate3_image(x, labels, inv_norm, centers, PaddedRows{nullptr, N}, N, D, K, norm_descs, intra_norm, vlad,
                    partial_ss, done, wait_all);
}

// packed images: image b is rows [row0[b], row0[b] + len[b]) of x, labels and inv_norm, and N >= every len[b] sizes
// the shared-memory layout.  The stable label order, the tasks and their sums depend on the image's rows alone, not on
// N or on the row chunks of the histogram pass: an image's descriptor is bitwise accumulate3's for the same rows.
__global__ void __launch_bounds__(ACC3_WARPS * 32, 4)
vlad_accumulate3_varlen_kernel(const float* __restrict__ x, const int32_t* __restrict__ labels,
                               const float* __restrict__ inv_norm, const float* __restrict__ centers,
                               const int64_t* __restrict__ row0, const int32_t* __restrict__ len, int N, int D, int K,
                               int norm_descs, int intra_norm, float* vlad, float* partial_ss, int32_t* done,
                               int wait_all) {
  accumulate3_image(x, labels, inv_norm, centers, PackedRows{row0, len}, N, D, K, norm_descs, intra_norm, vlad,
                    partial_ss, done, wait_all);
}

// columns per slice: every VLAD path cuts D into 128-column slices (one thread per column in the kernels below)
constexpr int ACC_COLS = 128;

// ------------------------------------------------------------------ soft assignment (utilities.py:862-887)
// a[r,k] = softmax_k(temp * cos(x_r, c_k)) with F.cosine_similarity's clamps (each norm clamped at 1e-8).
// One warp handles ROWS rows per pass over the centres (rows stay L1-resident); scores are staged in shared memory.
template <int ROWS>
__global__ void __launch_bounds__(256)
vlad_soft_assign_kernel(const float* __restrict__ x, const int32_t* __restrict__ n_valid, int N_per_img, int64_t R,
                        int D, int K, const float* __restrict__ chat /* c / max(|c|, 1e-8) */, float temp,
                        float* __restrict__ assign /*[R,K]*/, float* __restrict__ inv_norm) {
  extern __shared__ float sc_smem[];                 // [warps][ROWS][K]
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  float* sc = sc_smem + (size_t)wib * ROWS * K;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int D4 = D >> 2;
  for (int64_t r0 = warp * ROWS; r0 < R; r0 += nwarps * ROWS) {
    const float4* xr[ROWS];
    bool valid[ROWS];
#pragma unroll
    for (int i = 0; i < ROWS; ++i) {
      int64_t r = r0 + i;
      valid[i] = r < R;
      if (valid[i] && n_valid) valid[i] = (int)(r % N_per_img) < n_valid[(int)(r / N_per_img)];
      xr[i] = reinterpret_cast<const float4*>(x + (r < R ? r : r0) * (int64_t)D);
    }
    float ss[ROWS];
#pragma unroll
    for (int i = 0; i < ROWS; ++i) ss[i] = 0.f;
    for (int d = lane; d < D4; d += 32) {
#pragma unroll
      for (int i = 0; i < ROWS; ++i) {
        float4 v = __ldg(xr[i] + d);
        ss[i] += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
      }
    }
    float rx[ROWS];
#pragma unroll
    for (int i = 0; i < ROWS; ++i) { ss[i] = sqrtf(warp_sum(ss[i])); rx[i] = temp / fmaxf(ss[i], 1e-8f); }
    for (int k = 0; k < K; ++k) {
      const float4* cr = reinterpret_cast<const float4*>(chat + (size_t)k * D);
      float acc[ROWS];
#pragma unroll
      for (int i = 0; i < ROWS; ++i) acc[i] = 0.f;
      for (int d = lane; d < D4; d += 32) {
        float4 c = __ldg(cr + d);
#pragma unroll
        for (int i = 0; i < ROWS; ++i) {
          float4 v = __ldg(xr[i] + d);
          acc[i] = fmaf(v.x, c.x, acc[i]); acc[i] = fmaf(v.y, c.y, acc[i]);
          acc[i] = fmaf(v.z, c.z, acc[i]); acc[i] = fmaf(v.w, c.w, acc[i]);
        }
      }
#pragma unroll
      for (int i = 0; i < ROWS; ++i) {
        float s = warp_sum(acc[i]) * rx[i];
        if (lane == 0) sc[i * K + k] = s;
      }
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < ROWS; ++i) {
      int64_t r = r0 + i;
      if (r >= R) continue;
      if (!valid[i]) {        // padded row of a ragged batch: exactly 0, whatever it holds (its scores may be NaN)
        for (int k = lane; k < K; k += 32) assign[r * K + k] = 0.f;
        if (lane == 0 && inv_norm) inv_norm[r] = 0.f;
        continue;
      }
      float m = -INFINITY;
      for (int k = lane; k < K; k += 32) m = fmaxf(m, sc[i * K + k]);
      m = warp_max(m);
      float z = 0.f;
      for (int k = lane; k < K; k += 32) { float e = expf(sc[i * K + k] - m); sc[i * K + k] = e; z += e; }
      z = warp_sum(z);
      const float iz = 1.0f / z;
      for (int k = lane; k < K; k += 32) assign[r * K + k] = sc[i * K + k] * iz;
      if (lane == 0 && inv_norm) inv_norm[r] = 1.0f / fmaxf(ss[i], 1e-12f);
    }
    __syncwarp();
  }
}

// V[b,k,:] = sum_q a[q,k] * sum_c (x^_q - c_c) = K * sum_q a[q,k] x^_q - (sum_q a[q,k]) * sum_c c_c
// (the reference sums cluster k's weight over the residuals to ALL centres, utilities.py:881-884).
// CTA = (128-column slice, image); thread = column; KC cluster accumulators in registers per pass.  Only the image's
// first n_valid[b] rows are read: a padded row's weight is 0, but 0 * NaN would not be.
constexpr int SOFT_KC = 32, SOFT_QT = 64;
// the padded soft batch: image b's first min(N, max(0, n_valid[b])) rows of b*N.. (all N without n_valid)
struct SoftPaddedRows {
  const int32_t* n_valid; int N;
  __device__ __forceinline__ size_t first(int b) const { return (size_t)b * N; }
  __device__ __forceinline__ int count(int b) const { return n_valid ? min(N, max(0, n_valid[b])) : N; }
};
template <class Rows>
__device__ __forceinline__ void soft_accumulate_image(const float* __restrict__ x, Rows rows,
                                                      const float* __restrict__ assign,
                                                      const float* __restrict__ inv_norm,
                                                      const float* __restrict__ centers, int D, int K, int norm_descs,
                                                      float* __restrict__ vlad, float* __restrict__ partial_ss) {
  __shared__ __align__(16) float a_tile[SOFT_QT][SOFT_KC];
  __shared__ float inv_tile[SOFT_QT];
  __shared__ float red[ACC_COLS / 32][SOFT_KC];
  const int t = threadIdx.x, slice = blockIdx.x, b = blockIdx.y, nslices = gridDim.x;
  const int col = slice * ACC_COLS + t;
  const bool colok = col < D;
  const int N = rows.count(b);
  const float* xb = x + rows.first(b) * D;
  const float* ab = assign + rows.first(b) * K;
  float csum = 0.f;
  if (colok) for (int c = 0; c < K; ++c) csum += __ldg(centers + (size_t)c * D + col);
  for (int k0 = 0; k0 < K; k0 += SOFT_KC) {
    const int kc = min(SOFT_KC, K - k0);
    float acc[SOFT_KC];
#pragma unroll
    for (int j = 0; j < SOFT_KC; ++j) acc[j] = 0.f;
    float wsum = 0.f;                         // thread j < kc: sum_q a[q, k0 + j]
    for (int q0 = 0; q0 < N; q0 += SOFT_QT) {
      const int qn = min(SOFT_QT, N - q0);
      __syncthreads();
      for (int i = t; i < SOFT_QT * SOFT_KC; i += ACC_COLS) {
        int q = i / SOFT_KC, j = i % SOFT_KC;
        a_tile[q][j] = (q < qn && j < kc) ? __ldg(ab + (size_t)(q0 + q) * K + k0 + j) : 0.f;
      }
      for (int q = t; q < SOFT_QT; q += ACC_COLS)
        inv_tile[q] = (q < qn) ? (norm_descs ? inv_norm[rows.first(b) + q0 + q] : 1.0f) : 0.f;
      __syncthreads();
      if (t < SOFT_KC) for (int q = 0; q < qn; ++q) wsum += a_tile[q][t];
      if (colok) {
#pragma unroll 4
        for (int q = 0; q < qn; ++q) {
          const float xv = __ldg(xb + (size_t)(q0 + q) * D + col) * inv_tile[q];
          const float4* ar = reinterpret_cast<const float4*>(a_tile[q]);
#pragma unroll
          for (int j4 = 0; j4 < SOFT_KC / 4; ++j4) {
            float4 a = ar[j4];
            acc[4 * j4 + 0] = fmaf(a.x, xv, acc[4 * j4 + 0]); acc[4 * j4 + 1] = fmaf(a.y, xv, acc[4 * j4 + 1]);
            acc[4 * j4 + 2] = fmaf(a.z, xv, acc[4 * j4 + 2]); acc[4 * j4 + 3] = fmaf(a.w, xv, acc[4 * j4 + 3]);
          }
        }
      }
    }
    // epilogue for this cluster chunk: values, then per-(image, cluster, slice) sums of squares
    __syncthreads();
    if (t < SOFT_KC) inv_tile[t] = wsum;      // SOFT_KC <= SOFT_QT: reuse as the weight sums
    __syncthreads();
#pragma unroll
    for (int j = 0; j < SOFT_KC; ++j) {
      float v = 0.f;
      if (colok && j < kc) {
        v = (float)K * acc[j] - inv_tile[j] * csum;
        vlad[((size_t)b * K + k0 + j) * D + col] = v;
      }
      float sq = warp_sum(v * v);
      if ((t & 31) == 0) red[t >> 5][j] = sq;
    }
    __syncthreads();
    if (t < kc) {
      float tot = 0.f;
      for (int w = 0; w < ACC_COLS / 32; ++w) tot += red[w][t];
      partial_ss[((size_t)b * K + k0 + t) * nslices + slice] = tot;
    }
  }
}

__global__ void __launch_bounds__(ACC_COLS)
vlad_soft_accumulate_kernel(const float* __restrict__ x, const int32_t* __restrict__ n_valid,
                            const float* __restrict__ assign, const float* __restrict__ inv_norm,
                            const float* __restrict__ centers, int N_per_img, int D, int K, int norm_descs,
                            float* __restrict__ vlad, float* __restrict__ partial_ss) {
  soft_accumulate_image(x, SoftPaddedRows{n_valid, N_per_img}, assign, inv_norm, centers, D, K, norm_descs, vlad,
                        partial_ss);
}

// packed images: image b is rows [row0[b], row0[b] + len[b]) of x, assign [R,K] and inv_norm
__global__ void __launch_bounds__(ACC_COLS)
vlad_soft_accumulate_varlen_kernel(const float* __restrict__ x, const int64_t* __restrict__ row0,
                                   const int32_t* __restrict__ len, const float* __restrict__ assign,
                                   const float* __restrict__ inv_norm, const float* __restrict__ centers, int D, int K,
                                   int norm_descs, float* __restrict__ vlad, float* __restrict__ partial_ss) {
  soft_accumulate_image(x, PackedRows{row0, len}, assign, inv_norm, centers, D, K, norm_descs, vlad, partial_ss);
}

// ------------------------------------------------------------------ normalise
__global__ void __launch_bounds__(256)
vlad_normalize_kernel(float* __restrict__ vlad, const float* __restrict__ partial_ss, int D, int K,
                      int nslices, int intra_norm) {
  extern __shared__ float scale[];   // [2K]: scales, then the blocks' squared norms
  const int b = blockIdx.x;
  const float gnorm = vlad_norm_factors(partial_ss, b, K, nslices, intra_norm, scale, scale + K);
  float* v = vlad + (size_t)b * K * D;
  const size_t total = (size_t)K * D;
  for (size_t i = (size_t)blockIdx.y * blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.y * blockDim.x) {
    int k = (int)(i / D);
    // two separate multiplications like F.normalize(intra) then F.normalize(global)
    v[i] = (v[i] * scale[k]) * gnorm;
  }
}

// ------------------------------------------------------------------ sorted route (any K, any N)
// accumulate3's summation order with its per-image tables in the workspace instead of shared memory, so no (N, K) is
// out of reach.  vlad_sort_kernel (CTA per image) builds the stable label order of the rows, the tasks of <= 64 rows
// of one cluster and the slot bases of multi-task clusters exactly as accumulate3's prologue does;
// vlad_sorted_accumulate_kernel sums each task in registers with accumulate3's task_sum; vlad_sorted_combine_kernel adds
// the slots of multi-task clusters in task order; vlad_normalize_kernel then applies the factors of vlad_norm_factors.
// Every sum has accumulate3's order, so the descriptors are bitwise those of accumulate3 wherever it runs.
constexpr int SORTED_TASKS_PER_CTA = 64;
static inline int sorted_max_slots(int N) { return 2 * (N / ACC3_SEG) + 2; }
struct SortedTables {
  int64_t* ooff;     // [B,N] row offsets n * D in label order (stable)
  float* inv_s;      // [B,N] 1/|x| in the same order
  int* cntw;         // [B,ACC3_WARPS,K] per-warp histograms, then placement cursors
  int* start;        // [B,K+1] first sorted position of cluster k
  int* tstart;       // [B,K+1] first task of cluster k
  int* sbase;        // [B,K+1] first slot of a multi-task cluster
  int* task_k;       // [B,max_tasks] cluster of each task
  float* slots;      // [B,max_slots,D] partial sums of multi-task clusters
};

// Image b is rows.count(b) <= N rows from rows.first(b) of labels and inv_norm; N sizes the tables.
template <class Rows>
__device__ __forceinline__ void sort_image(const int32_t* __restrict__ labels, const float* __restrict__ inv_norm,
                                           Rows rows, int N, int D, int K, int norm_descs, SortedTables tb) {
  const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, w = t >> 5;
  const int nr = rows.count(b);
  const int maxT = acc3_max_tasks_dev(N, K);
  const int32_t* lab = labels + rows.first(b);
  int64_t* ooff = tb.ooff + (size_t)b * N;
  float* inv_s = tb.inv_s + (size_t)b * N;
  int* cntw = tb.cntw + (size_t)b * ACC3_WARPS * K;
  int* start = tb.start + (size_t)b * (K + 1);
  int* tstart = tb.tstart + (size_t)b * (K + 1);
  int* sbase = tb.sbase + (size_t)b * (K + 1);
  int* task_k = tb.task_k + (size_t)b * maxT;
  for (int i = t; i < ACC3_WARPS * K; i += blockDim.x) cntw[i] = 0;
  __syncthreads();
  const int chunk = (((nr + ACC3_WARPS - 1) / ACC3_WARPS) + 31) & ~31;
  const int r0 = min(nr, w * chunk), r1 = min(nr, r0 + chunk);
  for (int n = r0 + lane; n < r1; n += 32) { const int l = lab[n]; if (l >= 0) atomicAdd(&cntw[w * K + l], 1); }
  __syncthreads();
  for (int k = t; k < K; k += blockDim.x) {
    int tot = 0;
    for (int ww = 0; ww < ACC3_WARPS; ++ww) { const int c = cntw[ww * K + k]; cntw[ww * K + k] = tot; tot += c; }
    start[k] = tot;
  }
  __syncthreads();
  if (w == 0) {
    int run_r = 0, run_t = 0, run_s = 0;
    for (int k0 = 0; k0 < K; k0 += 32) {
      const int k = k0 + lane;
      const int c = k < K ? start[k] : 0;
      const int nt = k < K ? max(1, (c + ACC3_SEG - 1) / ACC3_SEG) : 0;
      const int ns = nt > 1 ? nt : 0;
      int ir = c, it = nt, is = ns;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int yr = __shfl_up_sync(0xffffffffu, ir, o), yt = __shfl_up_sync(0xffffffffu, it, o),
                  ys = __shfl_up_sync(0xffffffffu, is, o);
        if (lane >= o) { ir += yr; it += yt; is += ys; }
      }
      if (k < K) { start[k] = run_r + ir - c; tstart[k] = run_t + it - nt; sbase[k] = run_s + is - ns; }
      run_r += __shfl_sync(0xffffffffu, ir, 31);
      run_t += __shfl_sync(0xffffffffu, it, 31);
      run_s += __shfl_sync(0xffffffffu, is, 31);
    }
    if (lane == 0) { start[K] = run_r; tstart[K] = run_t; sbase[K] = run_s; }
  }
  __syncthreads();
  for (int k = t; k < K; k += blockDim.x)
    for (int q = tstart[k]; q < tstart[k + 1]; ++q) task_k[q] = k;
  for (int n0 = r0; n0 < r1; n0 += 32) {
    const int n = n0 + lane;
    const int l = n < r1 ? lab[n] : -1;
    const bool active = l >= 0;
    const unsigned am = __ballot_sync(0xffffffffu, active);
    unsigned peers = 0; int rank = 0;
    if (active) {
      peers = __match_any_sync(am, l);
      rank = __popc(peers & ((1u << lane) - 1u));
      const int pos = start[l] + cntw[w * K + l] + rank;
      ooff[pos] = (int64_t)n * D;
      inv_s[pos] = norm_descs ? inv_norm[rows.first(b) + n] : 1.0f;
    }
    __syncwarp();
    if (active && rank == 0) cntw[w * K + l] += __popc(peers);
    __syncwarp();
  }
}

__global__ void __launch_bounds__(ACC3_WARPS * 32)
vlad_sort_kernel(const int32_t* __restrict__ labels, const float* __restrict__ inv_norm, int N, int D, int K,
                 int norm_descs, SortedTables tb) {
  sort_image(labels, inv_norm, PaddedRows{nullptr, N}, N, D, K, norm_descs, tb);
}

__global__ void __launch_bounds__(ACC3_WARPS * 32)
vlad_sort_varlen_kernel(const int32_t* __restrict__ labels, const float* __restrict__ inv_norm,
                        const int64_t* __restrict__ row0, const int32_t* __restrict__ len, int N, int D, int K,
                        int norm_descs, SortedTables tb) {
  sort_image(labels, inv_norm, PackedRows{row0, len}, N, D, K, norm_descs, tb);
}

// CTA = (128-column slice, image, range of SORTED_TASKS_PER_CTA tasks); warps grab the range's tasks dynamically.  A
// single-task cluster's sum goes straight to the descriptor with its sum of squares; a multi-task cluster's to its
// slot.  Image b's rows start at rows.first(b) of x; N sizes the tables.
template <class Rows>
__device__ __forceinline__ void sorted_accumulate_image(const float* __restrict__ x, const float* __restrict__ centers,
                                                        Rows rows, int N, int D, int K, SortedTables tb,
                                                        float* __restrict__ vlad, float* __restrict__ partial_ss) {
  __shared__ int next_task;
  const int b = blockIdx.y, slice = blockIdx.x, nslices = gridDim.x, lane = threadIdx.x & 31;
  const int maxT = acc3_max_tasks_dev(N, K), maxS = 2 * (N / ACC3_SEG) + 2;
  const int* start = tb.start + (size_t)b * (K + 1);
  const int* tstart = tb.tstart + (size_t)b * (K + 1);
  const int* sbase = tb.sbase + (size_t)b * (K + 1);
  const int* task_k = tb.task_k + (size_t)b * maxT;
  const int64_t* ooff = tb.ooff + (size_t)b * N;
  const float* inv_s = tb.inv_s + (size_t)b * N;
  const int q0 = blockIdx.z * SORTED_TASKS_PER_CTA, q1 = min(tstart[K], q0 + SORTED_TASKS_PER_CTA);
  if (q0 >= q1) return;
  if (threadIdx.x == 0) next_task = q0;
  __syncthreads();
  const int col = slice * 128 + lane * 4;
  const bool colok = col < D;
  const float* xb = x + rows.first(b) * D + col;
  auto grab = [&]() { int q = 0; if (lane == 0) q = atomicAdd(&next_task, 1); return __shfl_sync(0xffffffffu, q, 0); };
  int q = grab();
  while (q < q1) {
    const int qn = grab();
    const int k = task_k[q];
    const int seg = q - tstart[k], nt = tstart[k + 1] - tstart[k];
    const int s = start[k] + seg * ACC3_SEG, e = min(start[k + 1], s + ACC3_SEG);
    const float4 a = task_sum(colok, centers + (size_t)k * D + col, xb, ooff, inv_s, s, e);
    if (nt == 1) {
      if (colok) *reinterpret_cast<float4*>(vlad + ((size_t)b * K + k) * D + col) = a;
      const float ss = warp_sum(sum_sq(a));
      if (lane == 0) partial_ss[((size_t)b * K + k) * nslices + slice] = ss;
    } else if (colok) {
      *reinterpret_cast<float4*>(tb.slots + ((size_t)b * maxS + sbase[k] + seg) * D + col) = a;
    }
    q = qn;
  }
}

__global__ void __launch_bounds__(ACC3_WARPS * 32)
vlad_sorted_accumulate_kernel(const float* __restrict__ x, const float* __restrict__ centers, int N, int D, int K,
                              SortedTables tb, float* __restrict__ vlad, float* __restrict__ partial_ss) {
  sorted_accumulate_image(x, centers, PaddedRows{nullptr, N}, N, D, K, tb, vlad, partial_ss);
}

__global__ void __launch_bounds__(ACC3_WARPS * 32)
vlad_sorted_accumulate_varlen_kernel(const float* __restrict__ x, const float* __restrict__ centers,
                                     const int64_t* __restrict__ row0, const int32_t* __restrict__ len, int N, int D,
                                     int K, SortedTables tb, float* __restrict__ vlad, float* __restrict__ partial_ss) {
  sorted_accumulate_image(x, centers, PackedRows{row0, len}, N, D, K, tb, vlad, partial_ss);
}

// CTA = (128-column slice, image): clusters of several tasks, their slots added in task order (accumulate3's combine)
__global__ void __launch_bounds__(ACC3_WARPS * 32)
vlad_sorted_combine_kernel(int N, int D, int K, SortedTables tb, float* __restrict__ vlad,
                           float* __restrict__ partial_ss) {
  const int b = blockIdx.y, slice = blockIdx.x, nslices = gridDim.x, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int maxS = 2 * (N / ACC3_SEG) + 2;
  const int* tstart = tb.tstart + (size_t)b * (K + 1);
  const int* sbase = tb.sbase + (size_t)b * (K + 1);
  const int col = slice * 128 + lane * 4;
  const bool colok = col < D;
  for (int k = w; k < K; k += ACC3_WARPS) {
    const int nt = tstart[k + 1] - tstart[k];
    if (nt <= 1) continue;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int q = 0; q < nt; ++q) {
      const float4 p = colok ? *reinterpret_cast<const float4*>(tb.slots + ((size_t)b * maxS + sbase[k] + q) * D + col)
                             : make_float4(0.f, 0.f, 0.f, 0.f);
      a.x += p.x; a.y += p.y; a.z += p.z; a.w += p.w;
    }
    if (colok) *reinterpret_cast<float4*>(vlad + ((size_t)b * K + k) * D + col) = a;
    const float ss = warp_sum(a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w);
    if (lane == 0) partial_ss[((size_t)b * K + k) * nslices + slice] = ss;
  }
}

// ------------------------------------------------------------------ k-means update
// Deterministic: every (column slice, row chunk) CTA writes ITS partial sums / counts, the finalize kernel adds the
// chunks in chunk order -- no floating-point atomics, so a fitted vocabulary is bit-reproducible for a fixed seed
// (like the reference's single-threaded mask @ X).
// x holds one ROUND: chunk c's piece is rows [c*piece, min(R, (c+1)*piece)) of x.  The in-memory update is one round
// of whole chunks (piece = rows_per).  A streamed fit feeds each chunk's rows in several rounds; with `resume` the
// running sums continue from psums / pcounts, and a sequential fp32 sum continued from a stored partial is the same
// sum, so the partials after the last round are bit-identical to the in-memory ones.
__global__ void kmeans_accumulate_kernel(const float* __restrict__ x, const int32_t* __restrict__ labels,
                                         int64_t R, int64_t piece, int D, int K, int resume,
                                         float* __restrict__ psums /* [chunks,K,D] */,
                                         float* __restrict__ pcounts /* [chunks,K] */) {
  // grid (D/128 slices, row-chunks); shared [K][128] partial sums
  extern __shared__ float acc[];
  const int t = threadIdx.x, col = blockIdx.x * ACC_COLS + t;
  const bool colok = col < D;
  float* ps = psums + (size_t)blockIdx.y * K * D;
  for (int k = 0; k < K; ++k) acc[k * ACC_COLS + t] = resume && colok ? ps[(size_t)k * D + col] : 0.f;
  float* cnt = acc + (size_t)K * ACC_COLS;
  for (int k = t; k < K; k += ACC_COLS) cnt[k] = resume && blockIdx.x == 0 ? pcounts[(size_t)blockIdx.y * K + k] : 0.f;
  __syncthreads();
  int64_t r0 = (int64_t)blockIdx.y * piece, r1 = min(R, r0 + piece);
  for (int64_t r = r0; r < r1; ++r) {
    int l = labels[r];
    if (l < 0) continue;
    if (colok) acc[l * ACC_COLS + t] += __ldg(x + r * D + col);
    if (blockIdx.x == 0 && t == 0) cnt[l] += 1.f;
  }
  __syncthreads();
  for (int k = 0; k < K; ++k)
    if (colok) ps[(size_t)k * D + col] = acc[k * ACC_COLS + t];
  if (blockIdx.x == 0)
    for (int k = t; k < K; k += ACC_COLS) pcounts[(size_t)blockIdx.y * K + k] = cnt[k];
}

// The same partials for any K: grid (D/128 slices, row-chunks, cluster tiles); a CTA keeps the 128-column sums of the
// k_tile clusters [k0, k0 + k_tile) in shared memory and adds only the rows labelled inside its tile, in row order --
// every (cluster, column) sum is kmeans_accumulate_kernel's sequential sum, so the partials are bitwise equal.
__global__ void kmeans_accumulate_tiled_kernel(const float* __restrict__ x, const int32_t* __restrict__ labels,
                                               int64_t R, int64_t piece, int D, int K, int k_tile, int resume,
                                               float* __restrict__ psums /* [chunks,K,D] */,
                                               float* __restrict__ pcounts /* [chunks,K] */) {
  extern __shared__ float acc[];                          // [k_tile][128] sums, then [k_tile] counts
  const int t = threadIdx.x, col = blockIdx.x * ACC_COLS + t;
  const bool colok = col < D;
  const int k0 = blockIdx.z * k_tile, kt = min(k_tile, K - k0);
  float* ps = psums + (size_t)blockIdx.y * K * D + (size_t)k0 * D;
  for (int k = 0; k < kt; ++k) acc[k * ACC_COLS + t] = resume && colok ? ps[(size_t)k * D + col] : 0.f;
  float* cnt = acc + (size_t)k_tile * ACC_COLS;
  for (int k = t; k < kt; k += ACC_COLS) cnt[k] = resume && blockIdx.x == 0 ? pcounts[(size_t)blockIdx.y * K + k0 + k] : 0.f;
  __syncthreads();
  int64_t r0 = (int64_t)blockIdx.y * piece, r1 = min(R, r0 + piece);
  for (int64_t r = r0; r < r1; ++r) {
    const int l = labels[r] - k0;
    if (l < 0 || l >= kt) continue;
    if (colok) acc[l * ACC_COLS + t] += __ldg(x + r * D + col);
    if (blockIdx.x == 0 && t == 0) cnt[l] += 1.f;
  }
  __syncthreads();
  for (int k = 0; k < kt; ++k)
    if (colok) ps[(size_t)k * D + col] = acc[k * ACC_COLS + t];
  if (blockIdx.x == 0)
    for (int k = t; k < kt; k += ACC_COLS) pcounts[(size_t)blockIdx.y * K + k0 + k] = cnt[k];
}

// The same partials for several vocabularies fitted on the same rows (anyloc_kmeans_accumulate_round_multi): a CTA
// keeps every vocabulary's [K][128] sums and [K] counts in shared memory, reads each row's 128 columns once and adds
// them to every vocabulary's cluster, in row order -- each vocabulary's sums are kmeans_accumulate_kernel's.
constexpr int KMEANS_MULTI_SET = 32;       // vocabularies per launch
struct AccumSet {
  int n;
  int k[KMEANS_MULTI_SET], off[KMEANS_MULTI_SET];      // off: the vocabulary's first shared-memory float
  const int32_t* labels[KMEANS_MULTI_SET];
  float *psums[KMEANS_MULTI_SET], *pcounts[KMEANS_MULTI_SET];
};

__global__ void kmeans_accumulate_multi_kernel(const float* __restrict__ x, int64_t R, int64_t piece, int D, int resume,
                                               const AccumSet set) {
  extern __shared__ float acc[];                          // per vocabulary: [K][128] sums, then [K] counts
  const int t = threadIdx.x, col = blockIdx.x * ACC_COLS + t;
  const bool colok = col < D;
  for (int v = 0; v < set.n; ++v) {
    const int K = set.k[v];
    float* a = acc + set.off[v];
    const float* ps = set.psums[v] + (size_t)blockIdx.y * K * D;
    for (int k = 0; k < K; ++k) a[k * ACC_COLS + t] = resume && colok ? ps[(size_t)k * D + col] : 0.f;
    for (int k = t; k < K; k += ACC_COLS)
      a[K * ACC_COLS + k] = resume && blockIdx.x == 0 ? set.pcounts[v][(size_t)blockIdx.y * K + k] : 0.f;
  }
  __syncthreads();
  int64_t r0 = (int64_t)blockIdx.y * piece, r1 = min(R, r0 + piece);
  for (int64_t r = r0; r < r1; ++r) {
    const float xv = colok ? __ldg(x + r * D + col) : 0.f;
    for (int v = 0; v < set.n; ++v) {
      const int l = set.labels[v][r];
      if (l < 0) continue;
      float* a = acc + set.off[v];
      if (colok) a[l * ACC_COLS + t] += xv;
      if (blockIdx.x == 0 && t == 0) a[set.k[v] * ACC_COLS + l] += 1.f;
    }
  }
  __syncthreads();
  for (int v = 0; v < set.n; ++v) {
    const int K = set.k[v];
    const float* a = acc + set.off[v];
    float* ps = set.psums[v] + (size_t)blockIdx.y * K * D;
    for (int k = 0; k < K; ++k)
      if (colok) ps[(size_t)k * D + col] = a[k * ACC_COLS + t];
    if (blockIdx.x == 0)
      for (int k = t; k < K; k += ACC_COLS) set.pcounts[v][(size_t)blockIdx.y * K + k] = a[K * ACC_COLS + k];
  }
}

__global__ void __launch_bounds__(256)
kmeans_finalize_kernel(const float* __restrict__ psums, const float* __restrict__ pcounts, int chunks,
                       const float* __restrict__ old_c, int D, int K, float* __restrict__ new_c,
                       float* __restrict__ perr /* [gridDim.x] */) {
  // grid-stride over the K*D centre elements; per-block squared shift -> perr[block] (summed in order by the last kernel)
  float e = 0.f;
  const size_t total = (size_t)K * D;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(i / D);
    float c = 0.f, sm = 0.f;
    for (int ch = 0; ch < chunks; ++ch) { c += pcounts[(size_t)ch * K + k]; sm += psums[(size_t)ch * total + i]; }
    const float v = c > 0.f ? sm / c : 0.f;    // NaN -> 0 for empty clusters (fpk)
    new_c[i] = v;
    const float d = v - old_c[i];
    e += d * d;
  }
  __shared__ float red[8];
  e = warp_sum(e);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = e;
  __syncthreads();
  if (threadIdx.x == 0) {
    float tot = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
    perr[blockIdx.x] = tot;
  }
}

__global__ void kmeans_err_kernel(const float* __restrict__ perr, int n, float* __restrict__ err) {
  if (threadIdx.x == 0 && blockIdx.x == 0) { float t = 0.f; for (int i = 0; i < n; ++i) t += perr[i]; err[0] = t; }
}

}  // namespace anyloc

using namespace anyloc;

namespace anyloc {
// GEMM engines (gemm_tc.cu)
int gemm_tc_launch(const void*, const void*, int, const void*, const void*, int, int, int, int, const EpiParams&, int,
                   cudaStream_t);
bool gemm_tc_supported(const void*, const void*, int, const void*, const void*, int, int, int, int, const EpiParams&,
                       int);
}  // namespace anyloc

namespace {
struct AssignBufs {
  float *chat, *chat_tf32, *cbias, *cnorm, *coarse;
  int32_t* done = nullptr; int n_done = 0;                                           // accumulate3 tickets (optional)
};

// labels (+ 1/|x|) for R rows: tensor-core coarse scores + exact rescoring when the shape allows it, else the
// FFMA kernel
int launch_assign(const float* feats, const int32_t* n_valid, int N_per_img, int64_t R, int D, int K,
                  const float* centers, int dist_mode, const AssignBufs& ab, int32_t* labels, float* inv_norm,
                  cudaStream_t st, bool prepared = false, int64_t R_route = -1) {
  if (prepared) {    // c^, tf32 copy, bias and norms already sit in ab (anyloc_vlad_prepare); only the tickets need zeroing
    if (ab.done) ANYLOC_CHECK_CUDA(cudaMemsetAsync(ab.done, 0, (size_t)ab.n_done * sizeof(int32_t), st));
  } else {
    vlad_centre_prep_kernel<<<K, 256, 0, st>>>(centers, K, D, dist_mode, ab.chat, ab.cbias, ab.chat_tf32, ab.cnorm,
                                               ab.done, ab.done ? ab.n_done : 0);
    ANYLOC_CHECK_LAUNCH();
  }
  EpiParams ep{ANYLOC_EPI_BIAS, ab.cbias, nullptr, nullptr, ab.coarse, nullptr, K};
  // R_route: the rows of the padded batch a packed list stands for, so both take the same kernels
  const bool fast = ab.coarse != nullptr && D <= 2048 && (R_route < 0 ? R : R_route) >= 256 && R < (1ll << 31) &&
                    gemm_tc_supported(feats, nullptr, D, ab.chat_tf32, nullptr, D, (int)R, K, D, ep, ANYLOC_PAIR_TF32);
  if (fast) {
    int rc = gemm_tc_launch(feats, nullptr, D, ab.chat_tf32, nullptr, D, (int)R, K, D, ep, ANYLOC_PAIR_TF32, st);
    if (rc) return rc;
    const int blocks = (int)((R + 7) / 8);
    if (D <= 512)
      vlad_rescore_kernel<4><<<blocks, 256, 0, st>>>(feats, n_valid, N_per_img, R, D, K, ab.chat, ab.cbias, ab.cnorm,
                                                     ab.coarse, labels, inv_norm);
    else if (D <= 1024)
      vlad_rescore_kernel<8><<<blocks, 256, 0, st>>>(feats, n_valid, N_per_img, R, D, K, ab.chat, ab.cbias, ab.cnorm,
                                                     ab.coarse, labels, inv_norm);
    else
      vlad_rescore_kernel<16><<<blocks, 256, 0, st>>>(feats, n_valid, N_per_img, R, D, K, ab.chat, ab.cbias, ab.cnorm,
                                                      ab.coarse, labels, inv_norm);
    ANYLOC_CHECK_LAUNCH();
    return ANYLOC_OK;
  }
  int sms = device_sm_count();
  int64_t warps_needed = (R + 1) / 2;
  int blocks = (int)std::min<int64_t>((warps_needed + 7) / 8, (int64_t)sms * 8);
  if (blocks < 1) blocks = 1;
  vlad_assign_kernel<2><<<blocks, 256, 0, st>>>(feats, n_valid, N_per_img, R, D, K, ab.chat, ab.cbias, labels,
                                               inv_norm);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}

bool take_assign_bufs(Workspace& w, int64_t R, int D, int K, AssignBufs* ab) {
  ab->chat = w.take<float>((size_t)K * D);
  ab->chat_tf32 = w.take<float>((size_t)K * D);
  ab->cbias = w.take<float>(K);
  ab->cnorm = w.take<float>(K);
  ab->coarse = w.take<float>((size_t)R * K);        // may be null when the caller's workspace is the small one
  return ab->chat && ab->chat_tf32 && ab->cbias && ab->cnorm;
}

// The hard path's workspace: labels, 1/|x|, per-slice sums of squares, the assignment buffers and, with `tickets`,
// the accumulate3 tickets.  It is a superset of the soft path's carve (1/|x|, sums of squares, c^ and the [R,K]
// assignment in the coarse scores' place) and of anyloc_vlad_assign's, so anyloc_vlad_workspace_bytes sizes all
// three.  R rows of features (B * N padded), B images.  With ws == nullptr it is a dry run; returns the bytes taken,
// 0 when the workspace is too small.
struct HardBufs { int32_t* labels; float *inv_norm, *partial; AssignBufs ab; };
size_t carve_hard(void* ws, size_t ws_bytes, size_t R, int B, int D, int K, bool tickets, HardBufs* hb) {
  Workspace w(ws ? ws : (void*)256, ws ? ws_bytes : (size_t)-1 / 2);
  hb->labels = w.take<int32_t>(R);
  hb->inv_norm = w.take<float>(R);
  hb->partial = w.take<float>((size_t)B * K * cdiv(D, ACC_COLS));
  const bool ok = hb->labels && hb->inv_norm && hb->partial && take_assign_bufs(w, (int64_t)R, D, K, &hb->ab);
  if (tickets) { hb->ab.done = w.take<int32_t>((size_t)B); hb->ab.n_done = B; }
  return ok ? w.off : 0;
}

// intra- and global L2 normalisation of B descriptors [B,K*D] in place, from their per-slice sums of squares
int launch_normalize(float* vlad, const float* partial, int B, int D, int K, int intra_norm, cudaStream_t st) {
  const int ysplit = std::max(1, std::min(64, (int)(((size_t)K * D + 256 * 16 - 1) / (256 * 16))));
  vlad_normalize_kernel<<<dim3(B, ysplit), 256, 2 * K * sizeof(float), st>>>(vlad, partial, D, K, cdiv(D, ACC_COLS),
                                                                           intra_norm);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}

// The pointers every hard assignment hands its kernels.  feats and the workspace (c^, its tf32 copy, the bias and the
// coarse scores) must pass gemm_tc_supported's 16-byte test, so that the route -- and with it the labels at near-ties --
// never depends on where an accepted buffer sits; the FFMA and rescoring kernels read feats and c^ as float4 too.
static int assign_alignment(const char* who, const float* feats, const int32_t* labels, const void* ws) {
  ANYLOC_REQUIRE_ALIGNED(feats, 16, who, "feats", "float4 and TMA access");
  ANYLOC_REQUIRE_ALIGNED(labels, 4, who, "labels", "int32 access");
  ANYLOC_REQUIRE_ALIGNED(ws, 16, who, "ws", "float4 and TMA access");
  return ANYLOC_OK;
}

// The hard generates add the accumulations' float4 reads of the centres and float4 stores of the descriptors; a
// prepared blob stands in for the workspace's c^ and tf32 copy, so it needs what the workspace needs.
static int generate_alignment(const char* who, const float* feats, const int32_t* n_valid, const float* centers,
                              const void* prepared, const float* vlad, const int32_t* labels_out, const void* ws) {
  ANYLOC_REQUIRE_ALIGNED(feats, 16, who, "feats", "float4 and TMA access");
  ANYLOC_REQUIRE_ALIGNED(n_valid, 4, who, "n_valid", "int32 access");
  ANYLOC_REQUIRE_ALIGNED(centers, 16, who, "centers", "float4 access");
  ANYLOC_REQUIRE_ALIGNED(prepared, 16, who, "prepared", "float4 and TMA access");
  ANYLOC_REQUIRE_ALIGNED(vlad, 16, who, "vlad", "float4 access");
  ANYLOC_REQUIRE_ALIGNED(labels_out, 4, who, "labels", "int32 access");
  ANYLOC_REQUIRE_ALIGNED(ws, 16, who, "ws", "float4 and TMA access");
  return ANYLOC_OK;
}
}  // namespace

extern "C" size_t anyloc_vlad_workspace_bytes(int B, int N, int D, int K) {
  HardBufs hb;
  return carve_hard(nullptr, 0, (size_t)B * N, B, D, K, true, &hb);
}

extern "C" int anyloc_vlad_assign(const float* feats, const float* centers, int R, int D, int K,
                                  int dist_mode, int32_t* labels, void* ws, size_t ws_bytes,
                                  void* stream) {
  ANYLOC_REQUIRE(feats && centers && labels && ws, "vlad_assign: null pointer");
  ANYLOC_REQUIRE(R >= 0 && D > 0 && K > 0 && D % 4 == 0, "vlad_assign: bad dims R=%d D=%d K=%d", R, D, K);
  int rc = assign_alignment("vlad_assign", feats, labels, ws);
  if (rc) return rc;
  ANYLOC_REQUIRE_ALIGNED(centers, 4, "vlad_assign", "centers", "fp32 access");
  if (R == 0) return ANYLOC_OK;
  Workspace w(ws, ws_bytes);
  AssignBufs ab;
  if (!take_assign_bufs(w, R, D, K, &ab)) { set_error("vlad_assign: workspace too small"); return ANYLOC_ERR_WORKSPACE; }
  return launch_assign(feats, nullptr, R, R, D, K, centers, dist_mode, ab, labels, nullptr, (cudaStream_t)stream);
}

// anyloc_vlad_assign_multi: the rows of one coarse slice, bounding its [rows, sum K] scores to 2^26 floats (256 MB)
constexpr int64_t ASSIGN_MULTI_COARSE = 1ll << 26;
static int64_t assign_multi_slice(int64_t R, int64_t Ksum) {
  return std::min<int64_t>(R, std::max<int64_t>(256, ASSIGN_MULTI_COARSE / Ksum / 256 * 256));
}

// the prepared centres of all vocabularies side by side ([sum K, D], tf32 copy, bias, norms) and, where the coarse
// route can run at all (D <= 2048, R >= 256), one slice of coarse scores.  ws == nullptr: dry run.
static size_t carve_assign_multi(void* ws, size_t ws_bytes, int64_t R, int D, int64_t Ksum, AssignBufs* ab) {
  Workspace w(ws ? ws : (void*)256, ws ? ws_bytes : (size_t)-1 / 2);
  ab->chat = w.take<float>((size_t)Ksum * D);
  ab->chat_tf32 = w.take<float>((size_t)Ksum * D);
  ab->cbias = w.take<float>(Ksum);
  ab->cnorm = w.take<float>(Ksum);
  ab->coarse = D <= 2048 && R >= 256 ? w.take<float>((size_t)assign_multi_slice(R, Ksum) * Ksum) : nullptr;
  const bool ok = ab->chat && ab->chat_tf32 && ab->cbias && ab->cnorm && (ab->coarse || D > 2048 || R < 256);
  return ok ? w.off : 0;
}

static int64_t assign_multi_ksum(int V, const int* K) {
  int64_t s = 0;
  for (int v = 0; v < V; ++v) s += K[v];
  return s;
}

extern "C" size_t anyloc_vlad_assign_multi_workspace_bytes(int64_t R, int D, int V, const int* K) {
  if (!K || V <= 0 || D <= 0) return 0;
  const int64_t Ksum = assign_multi_ksum(V, K);
  AssignBufs ab;
  return Ksum > 0 ? carve_assign_multi(nullptr, 0, R, D, Ksum, &ab) : 0;
}

extern "C" int anyloc_vlad_assign_multi(const float* feats, int64_t R, int D, int V, const float* const* centers,
                                        const int* K, int dist_mode, int32_t* labels, void* ws, size_t ws_bytes,
                                        void* stream) {
  ANYLOC_REQUIRE(feats && centers && K && labels && ws, "vlad_assign_multi: null pointer");
  ANYLOC_REQUIRE(R >= 0 && R < (1ll << 31) && D > 0 && D % 4 == 0 && V > 0,
                 "vlad_assign_multi: bad dims R=%lld D=%d V=%d", (long long)R, D, V);
  ANYLOC_REQUIRE(dist_mode == ANYLOC_DIST_COSINE || dist_mode == ANYLOC_DIST_EUCLIDEAN,
                 "vlad_assign_multi: unknown dist_mode %d", dist_mode);
  for (int v = 0; v < V; ++v) {
    ANYLOC_REQUIRE(K[v] > 0 && centers[v], "vlad_assign_multi: vocabulary %d has K=%d or no centres", v, K[v]);
    ANYLOC_REQUIRE((reinterpret_cast<uintptr_t>(centers[v]) & 3) == 0,
                   "vlad_assign_multi: centers[%d] must be 4-byte aligned (fp32 access)", v);
  }
  const int rc0 = assign_alignment("vlad_assign_multi", feats, labels, ws);
  if (rc0) return rc0;
  const int64_t Ksum = assign_multi_ksum(V, K);
  ANYLOC_REQUIRE(Ksum < (1ll << 31), "vlad_assign_multi: %lld centres in all", (long long)Ksum);
  if (R == 0) return ANYLOC_OK;
  AssignBufs ab;
  if (!carve_assign_multi(ws, ws_bytes, R, D, Ksum, &ab)) {
    set_error("vlad_assign_multi: workspace too small (%zu given, %zu needed)", ws_bytes,
              anyloc_vlad_assign_multi_workspace_bytes(R, D, V, K));
    return ANYLOC_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  // Each vocabulary takes the route anyloc_vlad_assign takes for it alone: its buffers there are 256-byte aligned like
  // these, so the GEMM shape check with N = K_v gives the same answer.  The FFMA and rescoring kernels may break
  // near-ties differently, so a vocabulary that would take the FFMA kernel alone takes it here too.
  std::vector<int> koff(V), fast(V);
  bool any_fast = false;
  for (int v = 0, off = 0; v < V; off += K[v], ++v) {
    koff[v] = off;
    vlad_centre_prep_kernel<<<K[v], 256, 0, st>>>(centers[v], K[v], D, dist_mode, ab.chat + (size_t)off * D,
                                                  ab.cbias + off, ab.chat_tf32 + (size_t)off * D, ab.cnorm + off,
                                                  nullptr, 0);
    ANYLOC_CHECK_LAUNCH();
    const EpiParams ep{ANYLOC_EPI_BIAS, ab.cbias, nullptr, nullptr, ab.coarse, nullptr, K[v]};
    fast[v] = ab.coarse != nullptr && D <= 2048 && R >= 256 &&
              gemm_tc_supported(feats, nullptr, D, ab.chat_tf32, nullptr, D, (int)R, K[v], D, ep, ANYLOC_PAIR_TF32);
    any_fast = any_fast || fast[v];
    if (!fast[v]) {
      const int sms = device_sm_count();
      const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>(((R + 1) / 2 + 7) / 8, (int64_t)sms * 8));
      vlad_assign_kernel<2><<<blocks, 256, 0, st>>>(feats, nullptr, (int)R, R, D, K[v], ab.chat + (size_t)off * D,
                                                    ab.cbias + off, labels + (size_t)v * R, nullptr);
      ANYLOC_CHECK_LAUNCH();
    }
  }
  if (!any_fast) return ANYLOC_OK;
  // one tf32 GEMM over all sum K prepared centres per slice of rows, then the segmented rescoring, 32 vocabularies at
  // a time
  const int64_t S = assign_multi_slice(R, Ksum);
  const EpiParams ep{ANYLOC_EPI_BIAS, ab.cbias, nullptr, nullptr, ab.coarse, nullptr, (int)Ksum};
  for (int64_t r0 = 0; r0 < R; r0 += S) {
    const int m = (int)std::min<int64_t>(S, R - r0);
    const float* xs = feats + r0 * D;
    int rc = gemm_tc_launch(xs, nullptr, D, ab.chat_tf32, nullptr, D, m, (int)Ksum, D, ep, ANYLOC_PAIR_TF32, st);
    if (rc) return rc;
    RescoreSegs segs;
    segs.n = 0;
    for (int v = 0; v < V; ++v) {
      if (fast[v]) {
        segs.koff[segs.n] = koff[v];
        segs.k[segs.n] = K[v];
        segs.labels[segs.n] = labels + (size_t)v * R + r0;
        ++segs.n;
      }
      if (segs.n == ASSIGN_MULTI_SEGS || (v == V - 1 && segs.n > 0)) {
        const int blocks = (m + 7) / 8;
        if (D <= 512)
          vlad_rescore_multi_kernel<4><<<blocks, 256, 0, st>>>(xs, m, D, (int)Ksum, ab.chat, ab.cbias, ab.cnorm,
                                                               ab.coarse, segs);
        else if (D <= 1024)
          vlad_rescore_multi_kernel<8><<<blocks, 256, 0, st>>>(xs, m, D, (int)Ksum, ab.chat, ab.cbias, ab.cnorm,
                                                               ab.coarse, segs);
        else
          vlad_rescore_multi_kernel<16><<<blocks, 256, 0, st>>>(xs, m, D, (int)Ksum, ab.chat, ab.cbias, ab.cnorm,
                                                                ab.coarse, segs);
        ANYLOC_CHECK_LAUNCH();
        segs.n = 0;
      }
    }
  }
  return ANYLOC_OK;
}

// Prepared vocabulary blob (anyloc_vlad_prepare): c^ [K,D] | tf32(c^) [K,D] | bias [K] | |c^| [K].  Everything the
// per-call centre-prep launch would produce.  With blob == nullptr a dry run; returns the bytes taken, 0 when the blob
// is too small.
struct PreparedView { float *chat, *chat_tf32, *cbias, *cnorm; };
static size_t carve_prepared(void* blob, size_t bytes, int D, int K, PreparedView* pv) {
  Workspace w(blob ? blob : (void*)256, blob ? bytes : (size_t)-1 / 2);
  pv->chat = w.take<float>((size_t)K * D);
  pv->chat_tf32 = w.take<float>((size_t)K * D);
  pv->cbias = w.take<float>(K);
  pv->cnorm = w.take<float>(K);
  return pv->chat && pv->chat_tf32 && pv->cbias && pv->cnorm ? w.off : 0;
}

// A prepared vocabulary stands in for the per-call centre prep: its c^, tf32 copy, bias and norms replace the
// workspace's in ab.  -> false (ab untouched) without a blob or when the blob is too small for (D, K).
static bool use_prepared(void* prepared, size_t prepared_bytes, int D, int K, AssignBufs* ab) {
  PreparedView pv;
  if (!prepared || !carve_prepared(prepared, prepared_bytes, D, K, &pv)) return false;
  ab->chat = pv.chat; ab->chat_tf32 = pv.chat_tf32; ab->cbias = pv.cbias; ab->cnorm = pv.cnorm;
  return true;
}

extern "C" size_t anyloc_vlad_prepared_bytes(int D, int K) {
  PreparedView pv;
  return carve_prepared(nullptr, 0, D, K, &pv);
}

extern "C" int anyloc_vlad_prepare(const float* centers, int D, int K, int dist_mode, void* prepared,
                                   size_t prepared_bytes, void* stream) {
  ANYLOC_REQUIRE(centers && prepared, "vlad_prepare: null pointer");
  ANYLOC_REQUIRE(D > 0 && K > 0 && D % 4 == 0, "vlad_prepare: bad dims D=%d K=%d", D, K);
  ANYLOC_REQUIRE(dist_mode == ANYLOC_DIST_COSINE || dist_mode == ANYLOC_DIST_EUCLIDEAN,
                 "vlad_prepare: unknown dist_mode %d", dist_mode);
  // the blob's readers (the generates' assignment) need 16 bytes, so a blob they would refuse is refused here
  ANYLOC_REQUIRE_ALIGNED(centers, 4, "vlad_prepare", "centers", "fp32 access");
  ANYLOC_REQUIRE_ALIGNED(prepared, 16, "vlad_prepare", "prepared", "float4 and TMA access");
  PreparedView pv;
  if (!carve_prepared(prepared, prepared_bytes, D, K, &pv)) { set_error("vlad_prepare: blob too small"); return ANYLOC_ERR_WORKSPACE; }
  vlad_centre_prep_kernel<<<K, 256, 0, (cudaStream_t)stream>>>(centers, K, D, dist_mode, pv.chat, pv.cbias, pv.chat_tf32,
                                                               pv.cnorm, nullptr, 0);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}

// accumulate2's row-splitting warps: as many as shared memory allows ((1 + warps) * K * 128 floats), at most 4 when
// two CTAs then fit per SM, else what fits in one (signed: K > 200 leaves none)
static int acc2_warps(int K) {
  return (int)std::min<long long>(4, (long long)((200 * 1024) / ((size_t)K * 128 * 4)) - 1);
}

// The one predicate that picks the hard-VLAD accumulation: accumulate3 when its shared memory fits 100 KB, else
// accumulate2 when one row-splitting warp fits, else the sorted route (anyloc_vlad_generate_sorted), which
// vlad_generate_impl refuses.
static int vlad_route(int N, int D, int K) {
  if (acc3_smem_bytes(N, K) <= 100 * 1024 && (int64_t)N * D < (1ll << 31)) return ANYLOC_VLAD_ROUTE_ACC3;
  return acc2_warps(K) >= 1 ? ANYLOC_VLAD_ROUTE_ACC2 : ANYLOC_VLAD_ROUTE_SORTED;
}

// The accumulation and normalisation of B images of up to N rows (N > 0) from their labels (or soft weights) and 1/|x|,
// padded (image b at rows b * N; n_valid for the soft accumulate) or packed (row0 / len).  route is the hard
// accumulation's (ANYLOC_VLAD_ROUTE_*; -1 with soft weights) and partial, done (ACC3: the tickets, zero on entry) and
// tb (sorted: the tables) the workspace it needs.  Every generate and accumulate entry launches its accumulation here.
template <bool PACKED>
static int launch_accumulate(const float* feats, const int32_t* n_valid, const int64_t* row0, const int32_t* len,
                             const int32_t* labels, const float* assign, const float* inv_norm, const float* centers,
                             int B, int N, int D, int K, int norm_descs, int intra_norm, float* vlad, int route,
                             float* partial, int32_t* done, const SortedTables* tb, cudaStream_t st) {
  const int nslices = cdiv(D, ACC_COLS);
  if (assign) {
    if (PACKED)
      vlad_soft_accumulate_varlen_kernel<<<dim3(nslices, B), ACC_COLS, 0, st>>>(feats, row0, len, assign, inv_norm,
                                                                               centers, D, K, norm_descs, vlad, partial);
    else
      vlad_soft_accumulate_kernel<<<dim3(nslices, B), ACC_COLS, 0, st>>>(feats, n_valid, assign, inv_norm, centers, N,
                                                                        D, K, norm_descs, vlad, partial);
    ANYLOC_CHECK_LAUNCH();
    return launch_normalize(vlad, partial, B, D, K, intra_norm, st);
  }
  if (route == ANYLOC_VLAD_ROUTE_ACC3) {
    const size_t smem3 = acc3_smem_bytes(N, K);
    static unsigned long long attr_seen = 0;         // one flag word per instantiation, so per kernel
    if (first_use_on_this_device(&attr_seen)) {
      if (PACKED)
        ANYLOC_CHECK_CUDA(cudaFuncSetAttribute(vlad_accumulate3_varlen_kernel,
                                               cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
      else
        ANYLOC_CHECK_CUDA(cudaFuncSetAttribute(vlad_accumulate3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               100 * 1024));
    }
    // all CTAs co-resident -> the slice-CTAs of an image may wait for each other (distributed normalisation);
    // otherwise the image's last CTA normalises alone
    int occ = 0;
    if (PACKED)
      ANYLOC_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, vlad_accumulate3_varlen_kernel,
                                                                      ACC3_WARPS * 32, smem3));
    else
      ANYLOC_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, vlad_accumulate3_kernel, ACC3_WARPS * 32,
                                                                      smem3));
    const int wait_all = (long long)nslices * B <= (long long)occ * device_sm_count() ? 1 : 0;
    if (PACKED)
      vlad_accumulate3_varlen_kernel<<<dim3(nslices, B), ACC3_WARPS * 32, smem3, st>>>(
          feats, labels, inv_norm, centers, row0, len, N, D, K, norm_descs, intra_norm, vlad, partial, done, wait_all);
    else
      vlad_accumulate3_kernel<<<dim3(nslices, B), ACC3_WARPS * 32, smem3, st>>>(
          feats, labels, inv_norm, centers, N, D, K, norm_descs, intra_norm, vlad, partial, done, wait_all);
    ANYLOC_CHECK_LAUNCH();
    return ANYLOC_OK;
  }
  if (route == ANYLOC_VLAD_ROUTE_ACC2) {
    const int warps = acc2_warps(K);
    const size_t smem = (size_t)(1 + warps) * K * 128 * 4;
    if (PACKED) {
      ANYLOC_CHECK_CUDA(cudaFuncSetAttribute(vlad_accumulate2_varlen_kernel,
                                             cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      vlad_accumulate2_varlen_kernel<<<dim3(nslices, B), 128, smem, st>>>(feats, labels, inv_norm, centers, row0, len,
                                                                          D, K, norm_descs, warps, vlad, partial);
    } else {
      ANYLOC_CHECK_CUDA(cudaFuncSetAttribute(vlad_accumulate2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)smem));
      vlad_accumulate2_kernel<<<dim3(nslices, B), 128, smem, st>>>(feats, labels, inv_norm, centers, N, D, K,
                                                                   norm_descs, warps, vlad, partial);
    }
    ANYLOC_CHECK_LAUNCH();
    return launch_normalize(vlad, partial, B, D, K, intra_norm, st);
  }
  const int ztasks = cdiv(acc3_max_tasks(N, K), SORTED_TASKS_PER_CTA);
  if (PACKED) {
    vlad_sort_varlen_kernel<<<B, ACC3_WARPS * 32, 0, st>>>(labels, inv_norm, row0, len, N, D, K, norm_descs, *tb);
    ANYLOC_CHECK_LAUNCH();
    vlad_sorted_accumulate_varlen_kernel<<<dim3(nslices, B, ztasks), ACC3_WARPS * 32, 0, st>>>(
        feats, centers, row0, len, N, D, K, *tb, vlad, partial);
  } else {
    vlad_sort_kernel<<<B, ACC3_WARPS * 32, 0, st>>>(labels, inv_norm, N, D, K, norm_descs, *tb);
    ANYLOC_CHECK_LAUNCH();
    vlad_sorted_accumulate_kernel<<<dim3(nslices, B, ztasks), ACC3_WARPS * 32, 0, st>>>(feats, centers, N, D, K, *tb,
                                                                                        vlad, partial);
  }
  ANYLOC_CHECK_LAUNCH();
  vlad_sorted_combine_kernel<<<dim3(nslices, B), ACC3_WARPS * 32, 0, st>>>(N, D, K, *tb, vlad, partial);
  ANYLOC_CHECK_LAUNCH();
  return launch_normalize(vlad, partial, B, D, K, intra_norm, st);
}

static int vlad_generate_impl(const float* feats, const int32_t* n_valid, const float* centers, void* prepared,
                              size_t prepared_bytes, int B, int N, int D, int K, int dist_mode, int norm_descs,
                              int intra_norm, float* vlad, int32_t* labels_out, void* ws, size_t ws_bytes, void* stream) {
  ANYLOC_REQUIRE(feats && centers && vlad && ws, "vlad_generate: null pointer");
  ANYLOC_REQUIRE(B >= 0 && N >= 0 && D > 0 && K > 0, "vlad_generate: bad dims");
  ANYLOC_REQUIRE(D % 4 == 0, "vlad_generate: D=%d must be a multiple of 4", D);
  ANYLOC_REQUIRE(dist_mode == ANYLOC_DIST_COSINE || dist_mode == ANYLOC_DIST_EUCLIDEAN,
                 "vlad_generate: unknown dist_mode %d", dist_mode);
  int rc = generate_alignment(prepared ? "vlad_generate_prepared" : "vlad_generate", feats, n_valid, centers, prepared,
                              vlad, labels_out, ws);
  if (rc) return rc;
  if (B == 0) return ANYLOC_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (N == 0) { ANYLOC_CHECK_CUDA(cudaMemsetAsync(vlad, 0, (size_t)B * K * D * 4, st)); return ANYLOC_OK; }
  const size_t R = (size_t)B * N;
  const size_t smem3 = acc3_smem_bytes(N, K);
  const bool fits3 = vlad_route(N, D, K) == ANYLOC_VLAD_ROUTE_ACC3;
  HardBufs hb;
  if (!carve_hard(ws, ws_bytes, R, B, D, K, fits3, &hb)) {
    set_error("vlad_generate: workspace too small (%zu bytes given)", ws_bytes);
    return ANYLOC_ERR_WORKSPACE;
  }
  AssignBufs& ab = hb.ab;
  const bool acc3 = ab.done != nullptr;             // fits3 and room for the tickets
  // else accumulate2; shapes neither serves belong to anyloc_vlad_generate_sorted
  const int warps = acc2_warps(K);
  ANYLOC_REQUIRE(acc3 || warps >= 1, "vlad_generate: K=%d N=%d needs %zu B shared memory (accumulate3 has 100 KB)", K,
                 N, smem3);
  // a prepared vocabulary replaces the per-call centre prep on every route
  const bool use_prep = use_prepared(prepared, prepared_bytes, D, K, &ab);
  ProfScope ps(PC_VLAD, st, 4.0 * ((double)B * N * D + (double)B * K * D + (double)K * D));
  rc = launch_assign(feats, n_valid, N, (int64_t)R, D, K, centers, dist_mode, ab, hb.labels, hb.inv_norm, st, use_prep);
  if (rc) return rc;
  // the assignment cleared the tickets
  rc = launch_accumulate<false>(feats, nullptr, nullptr, nullptr, hb.labels, nullptr, hb.inv_norm, centers, B, N, D, K,
                                norm_descs, intra_norm, vlad, acc3 ? ANYLOC_VLAD_ROUTE_ACC3 : ANYLOC_VLAD_ROUTE_ACC2,
                                hb.partial, ab.done, nullptr, st);
  if (rc) return rc;
  if (labels_out)
    ANYLOC_CHECK_CUDA(cudaMemcpyAsync(labels_out, hb.labels, R * 4, cudaMemcpyDeviceToDevice, st));
  return ANYLOC_OK;
}

extern "C" int anyloc_vlad_generate(const float* feats, const int32_t* n_valid, const float* centers,
                                    int B, int N, int D, int K, int dist_mode, int norm_descs,
                                    int intra_norm, float* vlad, int32_t* labels_out, void* ws,
                                    size_t ws_bytes, void* stream) {
  return vlad_generate_impl(feats, n_valid, centers, nullptr, 0, B, N, D, K, dist_mode, norm_descs, intra_norm, vlad,
                            labels_out, ws, ws_bytes, stream);
}

extern "C" int anyloc_vlad_generate_prepared(const float* feats, const int32_t* n_valid, const float* centers,
                                             void* prepared, size_t prepared_bytes, int B, int N, int D, int K,
                                             int dist_mode, int norm_descs, int intra_norm, float* vlad,
                                             int32_t* labels_out, void* ws, size_t ws_bytes, void* stream) {
  ANYLOC_REQUIRE(prepared, "vlad_generate_prepared: null prepared blob");
  return vlad_generate_impl(feats, n_valid, centers, prepared, prepared_bytes, B, N, D, K, dist_mode, norm_descs,
                            intra_norm, vlad, labels_out, ws, ws_bytes, stream);
}

extern "C" int anyloc_vlad_generate_route(int B, int N, int D, int K) {
  ANYLOC_REQUIRE(B >= 0 && N >= 0 && D > 0 && K > 0, "vlad_generate_route: bad dims");
  return vlad_route(N, D, K);
}

// The sorted route's per-image tables of B images of up to N rows, taken from w; false when w is too small.
static bool take_sorted_tables(Workspace& w, int B, int N, int D, int K, SortedTables* tb) {
  const size_t R = (size_t)B * N, K1 = (size_t)B * (K + 1);
  tb->ooff = w.take<int64_t>(R);
  tb->inv_s = w.take<float>(R);
  tb->cntw = w.take<int>((size_t)B * ACC3_WARPS * K);
  tb->start = w.take<int>(K1);
  tb->tstart = w.take<int>(K1);
  tb->sbase = w.take<int>(K1);
  tb->task_k = w.take<int>((size_t)B * acc3_max_tasks(N, K));
  tb->slots = w.take<float>((size_t)B * sorted_max_slots(N) * D);
  return tb->ooff && tb->inv_s && tb->cntw && tb->start && tb->tstart && tb->sbase && tb->task_k && tb->slots;
}

// The sorted route's workspace: carve_hard's buffers for R feature rows without the tickets, then the per-image tables
// of B images of up to N rows.  With ws == nullptr a dry run; returns the bytes taken, 0 when the workspace is too small.
static size_t carve_sorted(void* ws, size_t ws_bytes, size_t R_feats, int B, int N, int D, int K, HardBufs* hb,
                           SortedTables* tb) {
  const size_t off = carve_hard(ws, ws_bytes, R_feats, B, D, K, false, hb);
  if (!off) return 0;
  Workspace w(ws ? (void*)((char*)ws + off) : (void*)256, ws ? ws_bytes - off : (size_t)-1 / 2);
  return take_sorted_tables(w, B, N, D, K, tb) ? off + w.off : 0;
}

extern "C" size_t anyloc_vlad_sorted_workspace_bytes(int B, int N, int D, int K) {
  HardBufs hb;
  SortedTables tb;
  return carve_sorted(nullptr, 0, (size_t)B * N, B, N, D, K, &hb, &tb);
}

extern "C" int anyloc_vlad_generate_sorted(const float* feats, const int32_t* n_valid, const float* centers,
                                           void* prepared, size_t prepared_bytes, int B, int N, int D, int K,
                                           int dist_mode, int norm_descs, int intra_norm, float* vlad,
                                           int32_t* labels_out, void* ws, size_t ws_bytes, void* stream) {
  ANYLOC_REQUIRE(feats && centers && prepared && vlad && ws, "vlad_generate_sorted: null pointer");
  ANYLOC_REQUIRE(B >= 0 && N >= 0 && D > 0 && K > 0, "vlad_generate_sorted: bad dims");
  ANYLOC_REQUIRE(D % 4 == 0, "vlad_generate_sorted: D=%d must be a multiple of 4", D);
  ANYLOC_REQUIRE(dist_mode == ANYLOC_DIST_COSINE || dist_mode == ANYLOC_DIST_EUCLIDEAN,
                 "vlad_generate_sorted: unknown dist_mode %d", dist_mode);
  const int ztasks = cdiv(acc3_max_tasks(N, K), SORTED_TASKS_PER_CTA);
  ANYLOC_REQUIRE(B <= 65535 && ztasks <= 65535, "vlad_generate_sorted: B=%d N=%d K=%d exceed the launch grid", B, N, K);
  int rc = generate_alignment("vlad_generate_sorted", feats, n_valid, centers, prepared, vlad, labels_out, ws);
  if (rc) return rc;
  if (B == 0) return ANYLOC_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (N == 0) { ANYLOC_CHECK_CUDA(cudaMemsetAsync(vlad, 0, (size_t)B * K * D * 4, st)); return ANYLOC_OK; }
  HardBufs hb;
  SortedTables tb;
  if (!carve_sorted(ws, ws_bytes, (size_t)B * N, B, N, D, K, &hb, &tb)) {
    set_error("vlad_generate_sorted: workspace too small (%zu bytes given, %zu needed)", ws_bytes,
              anyloc_vlad_sorted_workspace_bytes(B, N, D, K));
    return ANYLOC_ERR_WORKSPACE;
  }
  const bool use_prep = use_prepared(prepared, prepared_bytes, D, K, &hb.ab);
  const size_t R = (size_t)B * N;
  ProfScope ps(PC_VLAD, st, 4.0 * ((double)B * N * D + (double)B * K * D + (double)K * D));
  rc = launch_assign(feats, n_valid, N, (int64_t)R, D, K, centers, dist_mode, hb.ab, hb.labels, hb.inv_norm, st,
                     use_prep);
  if (rc) return rc;
  rc = launch_accumulate<false>(feats, nullptr, nullptr, nullptr, hb.labels, nullptr, hb.inv_norm, centers, B, N, D, K,
                                norm_descs, intra_norm, vlad, ANYLOC_VLAD_ROUTE_SORTED, hb.partial, nullptr, &tb, st);
  if (rc) return rc;
  if (labels_out)
    ANYLOC_CHECK_CUDA(cudaMemcpyAsync(labels_out, hb.labels, R * 4, cudaMemcpyDeviceToDevice, st));
  return ANYLOC_OK;
}

// Centres for F.cosine_similarity: c / max(|c|, 1e-8)
namespace anyloc {
__global__ void vlad_soft_centre_prep_kernel(const float* __restrict__ c, int K, int D, float* __restrict__ chat) {
  int k = blockIdx.x;
  const float* row = c + (size_t)k * D;
  float ss = 0.f;
  for (int d = threadIdx.x; d < D; d += blockDim.x) { float v = row[d]; ss += v * v; }
  __shared__ float red[32];
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) red[0] = v;
  }
  __syncthreads();
  const float den = fmaxf(sqrtf(red[0]), 1e-8f);
  for (int d = threadIdx.x; d < D; d += blockDim.x) chat[(size_t)k * D + d] = row[d] / den;
}
}  // namespace anyloc

extern "C" int anyloc_vlad_generate_soft(const float* feats, const int32_t* n_valid, const float* centers,
                                         int B, int N, int D, int K, float soft_temp, int norm_descs,
                                         int intra_norm, float* vlad, float* assign_out, void* ws,
                                         size_t ws_bytes, void* stream) {
  ANYLOC_REQUIRE(feats && centers && vlad && ws, "vlad_generate_soft: null pointer");
  ANYLOC_REQUIRE(B >= 0 && N >= 0 && D > 0 && K > 0, "vlad_generate_soft: bad dims");
  ANYLOC_REQUIRE(D % 4 == 0, "vlad_generate_soft: D=%d must be a multiple of 4", D);
  ANYLOC_REQUIRE(K <= 2048, "vlad_generate_soft: K=%d > 2048", K);
  // the soft assignment reads feats and c^ (workspace) as float4; the accumulation reads the centres and writes the
  // descriptors one fp32 at a time
  ANYLOC_REQUIRE_ALIGNED(feats, 16, "vlad_generate_soft", "feats", "float4 access");
  ANYLOC_REQUIRE_ALIGNED(n_valid, 4, "vlad_generate_soft", "n_valid", "int32 access");
  ANYLOC_REQUIRE_ALIGNED(centers, 4, "vlad_generate_soft", "centers", "fp32 access");
  ANYLOC_REQUIRE_ALIGNED(vlad, 4, "vlad_generate_soft", "vlad", "fp32 access");
  ANYLOC_REQUIRE_ALIGNED(assign_out, 4, "vlad_generate_soft", "assign", "fp32 access");
  ANYLOC_REQUIRE_ALIGNED(ws, 16, "vlad_generate_soft", "ws", "float4 access");
  if (B == 0) return ANYLOC_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (N == 0) { ANYLOC_CHECK_CUDA(cudaMemsetAsync(vlad, 0, (size_t)B * K * D * 4, st)); return ANYLOC_OK; }
  Workspace w(ws, ws_bytes);
  const size_t R = (size_t)B * N;
  const int nslices = cdiv(D, ACC_COLS);
  float* inv_norm = w.take<float>(R);
  float* partial = w.take<float>((size_t)B * K * nslices);
  float* chat = w.take<float>((size_t)K * D);
  float* assign = w.take<float>(R * K);
  if (!inv_norm || !partial || !chat || !assign) {
    set_error("vlad_generate_soft: workspace too small (%zu bytes given)", ws_bytes);
    return ANYLOC_ERR_WORKSPACE;
  }
  ProfScope ps(PC_VLAD, st, 4.0 * ((double)B * N * D + (double)B * K * D + (double)K * D));
  vlad_soft_centre_prep_kernel<<<K, 256, 0, st>>>(centers, K, D, chat);
  ANYLOC_CHECK_LAUNCH();
  constexpr int ROWS = 2;
  const size_t smem = (size_t)8 * ROWS * K * 4;
  ANYLOC_CHECK_CUDA(cudaFuncSetAttribute(vlad_soft_assign_kernel<ROWS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem));
  int blocks = (int)std::min<int64_t>(((int64_t)(R + ROWS - 1) / ROWS + 7) / 8, (int64_t)device_sm_count() * 8);
  vlad_soft_assign_kernel<ROWS><<<std::max(blocks, 1), 256, smem, st>>>(feats, n_valid, N, (int64_t)R, D, K, chat,
                                                                       soft_temp, assign, inv_norm);
  ANYLOC_CHECK_LAUNCH();
  int rc = launch_accumulate<false>(feats, n_valid, nullptr, nullptr, nullptr, assign, inv_norm, centers, B, N, D, K,
                                   norm_descs, intra_norm, vlad, -1, partial, nullptr, nullptr, st);
  if (rc) return rc;
  if (assign_out)
    ANYLOC_CHECK_CUDA(cudaMemcpyAsync(assign_out, assign, R * K * 4, cudaMemcpyDeviceToDevice, st));
  return ANYLOC_OK;
}

// ====================================================================================================================
// Packed lists (anyloc_vlad_generate_varlen / _soft_varlen): image b is rows [row0[b], row0[b] + len[b]) of feats
// [R,D].  The per-row passes (assignment, 1/|x|) run over all R rows with the padded path's kernels; the accumulations
// take the *_varlen instantiations, which find an image's rows through the table and otherwise run the padded
// kernels' code at the padded shape (N = the longest len), so each descriptor is bitwise the padded call's.
// ====================================================================================================================
namespace anyloc {
// dst rows of image b = src rows of image b (width 32-bit words per row); CTA per image.  The per-row outputs
// (labels, soft assignment) of the rows that belong to an image; the caller has filled the others.
__global__ void __launch_bounds__(256)
varlen_copy_rows_kernel(const uint32_t* __restrict__ src, const int64_t* __restrict__ row0,
                        const int32_t* __restrict__ len, int width, uint32_t* __restrict__ dst) {
  const int b = blockIdx.x;
  const size_t off = (size_t)row0[b] * width, n = (size_t)len[b] * width;
  for (size_t i = threadIdx.x; i < n; i += blockDim.x) dst[off + i] = src[off + i];
}
}  // namespace anyloc

namespace {
// the refusals every packed entry shares, before anything is read or launched
int varlen_args(const char* who, const float* feats, int64_t R, const int64_t* row0, const int32_t* len, int B,
                int D, int K, const float* vlad) {
  ANYLOC_REQUIRE(B >= 0 && B <= 65535 && R >= 0 && R < (1ll << 31) && D > 0 && K > 0 && D % 4 == 0,
                 "%s: bad dims B=%d R=%lld D=%d K=%d (B <= 65535, R < 2^31, D a multiple of 4)", who, B, (long long)R,
                 D, K);
  ANYLOC_REQUIRE(feats && row0 && len && vlad, "%s: null pointer", who);
  ANYLOC_REQUIRE_ALIGNED(feats, 16, who, "feats", "float4 access");
  ANYLOC_REQUIRE_ALIGNED(row0, 8, who, "row0", "int64 access");
  ANYLOC_REQUIRE_ALIGNED(len, 4, who, "len", "int32 access");
  ANYLOC_REQUIRE_ALIGNED(vlad, 16, who, "vlad", "float4 access");
  return ANYLOC_OK;
}

// labels_out / assign_out [R, width]: fill (every byte `fill`), then each image's rows from the workspace copy
int varlen_rows_out(const void* src, const int64_t* row0, const int32_t* len, int B, int64_t R, int width, int fill,
                    void* dst, cudaStream_t st) {
  ANYLOC_CHECK_CUDA(cudaMemsetAsync(dst, fill, (size_t)R * width * 4, st));
  if (!src) return ANYLOC_OK;
  varlen_copy_rows_kernel<<<B, 256, 0, st>>>((const uint32_t*)src, row0, len, width, (uint32_t*)dst);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}
}  // namespace

extern "C" size_t anyloc_vlad_varlen_workspace_bytes(int64_t R, int B, int max_len, int D, int K) {
  HardBufs hb;
  SortedTables tb;
  if (vlad_route(max_len, D, K) == ANYLOC_VLAD_ROUTE_SORTED)
    return carve_sorted(nullptr, 0, (size_t)R, B, max_len, D, K, &hb, &tb);
  return carve_hard(nullptr, 0, (size_t)R, B, D, K, true, &hb);
}

extern "C" int anyloc_vlad_generate_varlen(const float* feats, int64_t R, const int64_t* row0, const int32_t* len,
                                           int B, const float* centers, void* prepared, size_t prepared_bytes, int D,
                                           int K, int dist_mode, int norm_descs, int intra_norm, float* vlad,
                                           int32_t* labels_out, void* ws, size_t ws_bytes, void* stream) {
  int rc = varlen_args("vlad_generate_varlen", feats, R, row0, len, B, D, K, vlad);
  if (rc) return rc;
  ANYLOC_REQUIRE(centers && ws, "vlad_generate_varlen: null pointer");
  ANYLOC_REQUIRE(dist_mode == ANYLOC_DIST_COSINE || dist_mode == ANYLOC_DIST_EUCLIDEAN,
                 "vlad_generate_varlen: unknown dist_mode %d", dist_mode);
  rc = generate_alignment("vlad_generate_varlen", feats, nullptr, centers, prepared, vlad, labels_out, ws);
  if (rc) return rc;
  if (B == 0) return ANYLOC_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int N = 0;                                        // the padded batch's row count: the longest image
  rc = varlen_rows_check(row0, len, B, R, st, "vlad_generate_varlen", &N);
  if (rc) return rc;
  const int route = vlad_route(N, D, K);
  const int ztasks = cdiv(acc3_max_tasks(N, K), SORTED_TASKS_PER_CTA);
  ANYLOC_REQUIRE(route != ANYLOC_VLAD_ROUTE_SORTED || ztasks <= 65535,
                 "vlad_generate_varlen: N=%d K=%d exceed the launch grid", N, K);
  HardBufs hb;
  SortedTables tb;
  const size_t got = route == ANYLOC_VLAD_ROUTE_SORTED
                         ? carve_sorted(ws, ws_bytes, (size_t)R, B, N, D, K, &hb, &tb)
                         : carve_hard(ws, ws_bytes, (size_t)R, B, D, K, route == ANYLOC_VLAD_ROUTE_ACC3, &hb);
  if (!got || (route == ANYLOC_VLAD_ROUTE_ACC3 && !hb.ab.done)) {
    set_error("vlad_generate_varlen: workspace too small (%zu bytes given, %zu needed)", ws_bytes,
              anyloc_vlad_varlen_workspace_bytes(R, B, N, D, K));
    return ANYLOC_ERR_WORKSPACE;
  }
  if (N == 0) {                                     // every image empty: zero descriptors, like the padded call
    ANYLOC_CHECK_CUDA(cudaMemsetAsync(vlad, 0, (size_t)B * K * D * 4, st));
    return labels_out ? varlen_rows_out(nullptr, row0, len, B, R, 1, 0xff, labels_out, st) : ANYLOC_OK;
  }
  const bool use_prep = use_prepared(prepared, prepared_bytes, D, K, &hb.ab);
  ProfScope ps(PC_VLAD, st, 4.0 * ((double)R * D + (double)B * K * D + (double)K * D));
  rc = launch_assign(feats, nullptr, 0, R, D, K, centers, dist_mode, hb.ab, hb.labels, hb.inv_norm, st, use_prep,
                     (int64_t)B * N);
  if (rc) return rc;
  // the assignment cleared the tickets of the ACC3 route
  rc = launch_accumulate<true>(feats, nullptr, row0, len, hb.labels, nullptr, hb.inv_norm, centers, B, N, D, K,
                               norm_descs, intra_norm, vlad, route, hb.partial, hb.ab.done, &tb, st);
  if (rc) return rc;
  return labels_out ? varlen_rows_out(hb.labels, row0, len, B, R, 1, 0xff, labels_out, st) : ANYLOC_OK;
}

// inv_norm [R] | partial [B,K,nslices] | c^ [K,D] | assign [R,K]: anyloc_vlad_generate_soft's carve for R packed rows
static size_t carve_soft_varlen(void* ws, size_t ws_bytes, int64_t R, int B, int D, int K, float** inv_norm,
                                float** partial, float** chat, float** assign) {
  Workspace w(ws ? ws : (void*)256, ws ? ws_bytes : (size_t)-1 / 2);
  *inv_norm = w.take<float>((size_t)R);
  *partial = w.take<float>((size_t)B * K * cdiv(D, ACC_COLS));
  *chat = w.take<float>((size_t)K * D);
  *assign = w.take<float>((size_t)R * K);
  return *inv_norm && *partial && *chat && *assign ? w.off : 0;
}

extern "C" size_t anyloc_vlad_soft_varlen_workspace_bytes(int64_t R, int B, int D, int K) {
  float *a, *b, *c, *d;
  return carve_soft_varlen(nullptr, 0, R, B, D, K, &a, &b, &c, &d);
}

extern "C" int anyloc_vlad_generate_soft_varlen(const float* feats, int64_t R, const int64_t* row0, const int32_t* len,
                                                int B, const float* centers, int D, int K, float soft_temp,
                                                int norm_descs, int intra_norm, float* vlad, float* assign_out,
                                                void* ws, size_t ws_bytes, void* stream) {
  int rc = varlen_args("vlad_generate_soft_varlen", feats, R, row0, len, B, D, K, vlad);
  if (rc) return rc;
  ANYLOC_REQUIRE(centers && ws, "vlad_generate_soft_varlen: null pointer");
  ANYLOC_REQUIRE(K <= 2048, "vlad_generate_soft_varlen: K=%d > 2048", K);
  ANYLOC_REQUIRE_ALIGNED(centers, 4, "vlad_generate_soft_varlen", "centers", "fp32 access");
  ANYLOC_REQUIRE_ALIGNED(assign_out, 4, "vlad_generate_soft_varlen", "assign", "fp32 access");
  ANYLOC_REQUIRE_ALIGNED(ws, 16, "vlad_generate_soft_varlen", "ws", "float4 access");
  if (B == 0) return ANYLOC_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int N = 0;
  rc = varlen_rows_check(row0, len, B, R, st, "vlad_generate_soft_varlen", &N);
  if (rc) return rc;
  float *inv_norm, *partial, *chat, *assign;
  if (!carve_soft_varlen(ws, ws_bytes, R, B, D, K, &inv_norm, &partial, &chat, &assign)) {
    set_error("vlad_generate_soft_varlen: workspace too small (%zu bytes given, %zu needed)", ws_bytes,
              anyloc_vlad_soft_varlen_workspace_bytes(R, B, D, K));
    return ANYLOC_ERR_WORKSPACE;
  }
  if (N == 0) {
    ANYLOC_CHECK_CUDA(cudaMemsetAsync(vlad, 0, (size_t)B * K * D * 4, st));
    return assign_out ? varlen_rows_out(nullptr, row0, len, B, R, K, 0, assign_out, st) : ANYLOC_OK;
  }
  ProfScope ps(PC_VLAD, st, 4.0 * ((double)R * D + (double)B * K * D + (double)K * D));
  vlad_soft_centre_prep_kernel<<<K, 256, 0, st>>>(centers, K, D, chat);
  ANYLOC_CHECK_LAUNCH();
  constexpr int ROWS = 2;
  const size_t smem = (size_t)8 * ROWS * K * 4;
  ANYLOC_CHECK_CUDA(cudaFuncSetAttribute(vlad_soft_assign_kernel<ROWS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem));
  int blocks = (int)std::min<int64_t>(((int64_t)(R + ROWS - 1) / ROWS + 7) / 8, (int64_t)device_sm_count() * 8);
  vlad_soft_assign_kernel<ROWS><<<std::max(blocks, 1), 256, smem, st>>>(feats, nullptr, 0, R, D, K, chat, soft_temp,
                                                                       assign, inv_norm);
  ANYLOC_CHECK_LAUNCH();
  rc = launch_accumulate<true>(feats, nullptr, row0, len, nullptr, assign, inv_norm, centers, B, N, D, K, norm_descs,
                               intra_norm, vlad, -1, partial, nullptr, nullptr, st);
  if (rc) return rc;
  return assign_out ? varlen_rows_out(assign, row0, len, B, R, K, 0, assign_out, st) : ANYLOC_OK;
}

// The fixed row partition of the k-means update: at most 64 contiguous chunks, enough (column slice, chunk) CTAs to
// fill the device, at least 256 rows per chunk.  Its summation order is what a fitted vocabulary's bits depend on.
static int kmeans_chunks(int64_t R, int D) {
  const int nslices = cdiv(D, ACC_COLS);
  const int64_t fill = 4 * device_sm_count() / std::max(1, nslices);
  return (int)std::max<int64_t>(1, std::min<int64_t>(std::min<int64_t>((R + 255) / 256, fill), 64));
}
constexpr int KMEANS_FIN_BLOCKS = 64;

namespace {
// Every k-means kernel reads and writes one fp32 or int32 at a time, the workspace's sums and counts included, so 4
// bytes is the whole contract.  Null pointers are the ones the entry does not take.
int kmeans_alignment(const char* who, const float* x, const int32_t* labels, const float* old_centers,
                     const float* new_centers, const float* err_out, const void* ws) {
  ANYLOC_REQUIRE_ALIGNED(x, 4, who, "x", "fp32 access");
  ANYLOC_REQUIRE_ALIGNED(labels, 4, who, "labels", "int32 access");
  ANYLOC_REQUIRE_ALIGNED(old_centers, 4, who, "old_centers", "fp32 access");
  ANYLOC_REQUIRE_ALIGNED(new_centers, 4, who, "new_centers", "fp32 access");
  ANYLOC_REQUIRE_ALIGNED(err_out, 4, who, "err_out", "fp32 access");
  ANYLOC_REQUIRE_ALIGNED(ws, 4, who, "ws", "fp32 access");
  return ANYLOC_OK;
}

struct KmeansBufs { float *psums, *pcounts, *perr; int chunks; };
bool take_kmeans_bufs(void* ws, size_t ws_bytes, int64_t R, int D, int K, KmeansBufs* b) {
  b->chunks = kmeans_chunks(R, D);
  Workspace w(ws, ws_bytes);
  b->psums = w.take<float>((size_t)b->chunks * K * D);
  b->pcounts = w.take<float>((size_t)b->chunks * K);
  b->perr = w.take<float>(KMEANS_FIN_BLOCKS);
  return b->psums && b->pcounts && b->perr;
}
}  // namespace

extern "C" int anyloc_kmeans_partition(int64_t R, int D, int* chunks, int64_t* rows_per) {
  ANYLOC_REQUIRE(chunks && rows_per, "kmeans_partition: null pointer");
  ANYLOC_REQUIRE(R >= 0 && D > 0, "kmeans_partition: bad dims R=%lld D=%d", (long long)R, D);
  *chunks = kmeans_chunks(R, D);
  *rows_per = (R + *chunks - 1) / *chunks;
  return ANYLOC_OK;
}

extern "C" size_t anyloc_kmeans_round_workspace_bytes(int64_t R, int D, int K) {
  const size_t chunks = (size_t)kmeans_chunks(R, D);
  return align_up(chunks * K * D * 4, 256) + align_up(chunks * K * 4, 256) + align_up(KMEANS_FIN_BLOCKS * 4, 256) + 256;
}

extern "C" size_t anyloc_kmeans_workspace_bytes(int R, int D, int K) {
  return anyloc_kmeans_round_workspace_bytes(R, D, K);
}

extern "C" int anyloc_kmeans_accumulate_round(const float* x, const int32_t* labels, int64_t R, int64_t round_rows,
                                              int64_t piece_rows, int D, int K, int resume, void* ws, size_t ws_bytes,
                                              void* stream) {
  ANYLOC_REQUIRE(x && labels && ws, "kmeans_accumulate_round: null pointer");
  int rc = kmeans_alignment("kmeans_accumulate_round", x, labels, nullptr, nullptr, nullptr, ws);
  if (rc) return rc;
  ANYLOC_REQUIRE(R >= 0 && D > 0 && K > 0 && piece_rows >= 0 && round_rows >= 0,
                 "kmeans_accumulate_round: bad dims R=%lld D=%d K=%d", (long long)R, D, K);
  KmeansBufs b;
  if (!take_kmeans_bufs(ws, ws_bytes, R, D, K, &b)) {
    set_error("kmeans_accumulate_round: workspace too small (%zu given, %zu needed)", ws_bytes,
              anyloc_kmeans_round_workspace_bytes(R, D, K));
    return ANYLOC_ERR_WORKSPACE;
  }
  ANYLOC_REQUIRE(round_rows <= (int64_t)b.chunks * piece_rows,
                 "kmeans_accumulate_round: %lld rows do not fit %d pieces of %lld", (long long)round_rows, b.chunks,
                 (long long)piece_rows);
  cudaStream_t st = (cudaStream_t)stream;
  size_t smem = ((size_t)K * ACC_COLS + K) * 4;
  ANYLOC_REQUIRE(smem <= 220 * 1024, "kmeans_accumulate_round: K=%d too large", K);
  ANYLOC_CHECK_CUDA(cudaFuncSetAttribute(kmeans_accumulate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem));
  int nslices = cdiv(D, ACC_COLS);
  kmeans_accumulate_kernel<<<dim3(nslices, b.chunks), ACC_COLS, smem, st>>>(x, labels, round_rows, piece_rows, D, K,
                                                                            resume, b.psums, b.pcounts);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}

extern "C" int anyloc_kmeans_finalize(const float* old_centers, int64_t R, int D, int K, float* new_centers,
                                      float* err_out, void* ws, size_t ws_bytes, void* stream) {
  ANYLOC_REQUIRE(old_centers && new_centers && err_out && ws, "kmeans_finalize: null pointer");
  int rc = kmeans_alignment("kmeans_finalize", nullptr, nullptr, old_centers, new_centers, err_out, ws);
  if (rc) return rc;
  KmeansBufs b;
  if (!take_kmeans_bufs(ws, ws_bytes, R, D, K, &b)) {
    set_error("kmeans_finalize: workspace too small (%zu given, %zu needed)", ws_bytes,
              anyloc_kmeans_round_workspace_bytes(R, D, K));
    return ANYLOC_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  kmeans_finalize_kernel<<<KMEANS_FIN_BLOCKS, 256, 0, st>>>(b.psums, b.pcounts, b.chunks, old_centers, D, K,
                                                            new_centers, b.perr);
  ANYLOC_CHECK_LAUNCH();
  kmeans_err_kernel<<<1, 32, 0, st>>>(b.perr, KMEANS_FIN_BLOCKS, err_out);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}

extern "C" int anyloc_kmeans_update(const float* x, const int32_t* labels, const float* old_centers,
                                    int R, int D, int K, float* new_centers, float* err_out, void* ws,
                                    size_t ws_bytes, void* stream) {
  ANYLOC_REQUIRE(x && labels && old_centers && new_centers && err_out && ws, "kmeans_update: null pointer");
  int rc = kmeans_alignment("kmeans_update", x, labels, old_centers, new_centers, err_out, ws);
  if (rc) return rc;
  int chunks;
  int64_t rows_per;
  rc = anyloc_kmeans_partition(R, D, &chunks, &rows_per);
  if (!rc) rc = anyloc_kmeans_accumulate_round(x, labels, R, R, rows_per, D, K, 0, ws, ws_bytes, stream);
  if (!rc) rc = anyloc_kmeans_finalize(old_centers, R, D, K, new_centers, err_out, ws, ws_bytes, stream);
  return rc;
}

// clusters per CTA of kmeans_accumulate_tiled_kernel: (k_tile * 128 + k_tile) * 4 bytes within the same 220 KB
constexpr int KMEANS_MAX_TILE = 220 * 1024 / ((ACC_COLS + 1) * 4);

extern "C" int anyloc_kmeans_accumulate_round_tiled(const float* x, const int32_t* labels, int64_t R, int64_t round_rows,
                                                    int64_t piece_rows, int D, int K, int k_tile, int resume, void* ws,
                                                    size_t ws_bytes, void* stream) {
  ANYLOC_REQUIRE(x && labels && ws, "kmeans_accumulate_round_tiled: null pointer");
  int rc = kmeans_alignment("kmeans_accumulate_round_tiled", x, labels, nullptr, nullptr, nullptr, ws);
  if (rc) return rc;
  ANYLOC_REQUIRE(R >= 0 && D > 0 && K > 0 && piece_rows >= 0 && round_rows >= 0,
                 "kmeans_accumulate_round_tiled: bad dims R=%lld D=%d K=%d", (long long)R, D, K);
  ANYLOC_REQUIRE(k_tile >= 0 && k_tile <= KMEANS_MAX_TILE, "kmeans_accumulate_round_tiled: k_tile=%d not in [0, %d]",
                 k_tile, KMEANS_MAX_TILE);
  KmeansBufs b;
  if (!take_kmeans_bufs(ws, ws_bytes, R, D, K, &b)) {
    set_error("kmeans_accumulate_round_tiled: workspace too small (%zu given, %zu needed)", ws_bytes,
              anyloc_kmeans_round_workspace_bytes(R, D, K));
    return ANYLOC_ERR_WORKSPACE;
  }
  ANYLOC_REQUIRE(round_rows <= (int64_t)b.chunks * piece_rows,
                 "kmeans_accumulate_round_tiled: %lld rows do not fit %d pieces of %lld", (long long)round_rows,
                 b.chunks, (long long)piece_rows);
  const int tile = std::min(K, k_tile == 0 ? KMEANS_MAX_TILE : k_tile);
  const int ntiles = cdiv(K, tile);
  ANYLOC_REQUIRE(ntiles <= 65535, "kmeans_accumulate_round_tiled: K=%d needs %d tiles of %d", K, ntiles, tile);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t smem = ((size_t)tile * ACC_COLS + tile) * 4;
  ANYLOC_CHECK_CUDA(cudaFuncSetAttribute(kmeans_accumulate_tiled_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem));
  kmeans_accumulate_tiled_kernel<<<dim3(cdiv(D, ACC_COLS), b.chunks, ntiles), ACC_COLS, smem, st>>>(
      x, labels, round_rows, piece_rows, D, K, tile, resume, b.psums, b.pcounts);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}

extern "C" int anyloc_kmeans_update_tiled(const float* x, const int32_t* labels, const float* old_centers, int64_t R,
                                          int D, int K, int k_tile, float* new_centers, float* err_out, void* ws,
                                          size_t ws_bytes, void* stream) {
  ANYLOC_REQUIRE(x && labels && old_centers && new_centers && err_out && ws, "kmeans_update_tiled: null pointer");
  int rc = kmeans_alignment("kmeans_update_tiled", x, labels, old_centers, new_centers, err_out, ws);
  if (rc) return rc;
  int chunks;
  int64_t rows_per;
  rc = anyloc_kmeans_partition(R, D, &chunks, &rows_per);
  if (!rc) rc = anyloc_kmeans_accumulate_round_tiled(x, labels, R, R, rows_per, D, K, k_tile, 0, ws, ws_bytes, stream);
  if (!rc) rc = anyloc_kmeans_finalize(old_centers, R, D, K, new_centers, err_out, ws, ws_bytes, stream);
  return rc;
}

extern "C" int anyloc_kmeans_accumulate_round_multi(const float* x, int V, const int32_t* const* labels, const int* K,
                                                    int64_t R, int64_t round_rows, int64_t piece_rows, int D,
                                                    int resume, void* const* ws, const size_t* ws_bytes,
                                                    void* stream) {
  ANYLOC_REQUIRE(x && labels && K && ws && ws_bytes, "kmeans_accumulate_round_multi: null pointer");
  ANYLOC_REQUIRE_ALIGNED(x, 4, "kmeans_accumulate_round_multi", "x", "fp32 access");
  ANYLOC_REQUIRE(V > 0 && R >= 0 && D > 0 && piece_rows >= 0 && round_rows >= 0,
                 "kmeans_accumulate_round_multi: bad dims V=%d R=%lld D=%d", V, (long long)R, D);
  for (int v = 0; v < V; ++v) {
    ANYLOC_REQUIRE((reinterpret_cast<uintptr_t>(labels[v]) & 3) == 0,
                   "kmeans_accumulate_round_multi: labels[%d] must be 4-byte aligned (int32 access)", v);
    ANYLOC_REQUIRE((reinterpret_cast<uintptr_t>(ws[v]) & 3) == 0,
                   "kmeans_accumulate_round_multi: ws[%d] must be 4-byte aligned (fp32 access)", v);
  }
  std::vector<KmeansBufs> b(V);
  for (int v = 0; v < V; ++v) {
    ANYLOC_REQUIRE(labels[v] && K[v] > 0, "kmeans_accumulate_round_multi: vocabulary %d has K=%d or no labels", v, K[v]);
    ANYLOC_REQUIRE(((size_t)K[v] * ACC_COLS + K[v]) * 4 <= 220 * 1024,
                   "kmeans_accumulate_round_multi: vocabulary %d has K=%d, beyond the untiled update's shared memory",
                   v, K[v]);
    if (!take_kmeans_bufs(ws[v], ws_bytes[v], R, D, K[v], &b[v])) {
      set_error("kmeans_accumulate_round_multi: vocabulary %d's workspace is too small (%zu given, %zu needed)", v,
                ws_bytes[v], anyloc_kmeans_round_workspace_bytes(R, D, K[v]));
      return ANYLOC_ERR_WORKSPACE;
    }
  }
  ANYLOC_REQUIRE(round_rows <= (int64_t)b[0].chunks * piece_rows,
                 "kmeans_accumulate_round_multi: %lld rows do not fit %d pieces of %lld", (long long)round_rows,
                 b[0].chunks, (long long)piece_rows);
  cudaStream_t st = (cudaStream_t)stream;
  ANYLOC_CHECK_CUDA(cudaFuncSetAttribute(kmeans_accumulate_multi_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         220 * 1024));
  // consecutive vocabularies share a launch while their sums and counts fit the 220 KB
  AccumSet set;
  set.n = 0;
  int used = 0;
  for (int v = 0; v <= V; ++v) {
    const int need = v < V ? (K[v] * ACC_COLS + K[v]) : 0;
    if (set.n > 0 && (v == V || set.n == KMEANS_MULTI_SET || (size_t)(used + need) * 4 > 220 * 1024)) {
      kmeans_accumulate_multi_kernel<<<dim3(cdiv(D, ACC_COLS), b[0].chunks), ACC_COLS, (size_t)used * 4, st>>>(
          x, round_rows, piece_rows, D, resume, set);
      ANYLOC_CHECK_LAUNCH();
      set.n = 0;
      used = 0;
    }
    if (v == V) break;
    set.k[set.n] = K[v];
    set.off[set.n] = used;
    set.labels[set.n] = labels[v];
    set.psums[set.n] = b[v].psums;
    set.pcounts[set.n] = b[v].pcounts;
    ++set.n;
    used += need;
  }
  return ANYLOC_OK;
}

// ====================================================================================================================
// Residual tensors and the per-image cache path (utilities.py:928-972, :843-852, :864-878).  Off the hot path: the
// reference materialises x^ - c for ALL (patch, centre) pairs ([N,K,D] fp32, 104 MB per image at c2) and, with a
// cache directory, re-builds descriptors from cached residuals / labels / soft assignments without the features.
// ====================================================================================================================
namespace anyloc {

// out[q,k,:] = x_q / max(|x_q|, 1e-12) - c_k (F.normalize when norm_descs, utilities.py:959-962).  CTA per row;
// HBM-bound on the N*K*D*4 bytes written.
__global__ void __launch_bounds__(256)
vlad_residuals_kernel(const float* __restrict__ x, const float* __restrict__ centers, int D, int K, int norm_descs,
                      float* __restrict__ out) {
  const size_t q = blockIdx.x;
  const float4* xr = reinterpret_cast<const float4*>(x + q * D);
  const int D4 = D >> 2;
  __shared__ float red[8];
  __shared__ float s_nrm;
  float ss = 0.f;
  if (norm_descs) {
    for (int d = threadIdx.x; d < D4; d += blockDim.x) { float4 v = __ldg(xr + d); ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w; }
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    if (threadIdx.x == 0) { float t = 0.f; for (int w = 0; w < 8; ++w) t += red[w]; s_nrm = fmaxf(sqrtf(t), 1e-12f); }
    __syncthreads();
  }
  const float nrm = norm_descs ? s_nrm : 1.0f;
  float4* o = reinterpret_cast<float4*>(out + q * (size_t)K * D);
  for (int d = threadIdx.x; d < D4; d += blockDim.x) {
    float4 v = __ldg(xr + d);
    if (norm_descs) { v.x /= nrm; v.y /= nrm; v.z /= nrm; v.w /= nrm; }
    for (int k = 0; k < K; ++k) {
      const float4 c = __ldg(reinterpret_cast<const float4*>(centers + (size_t)k * D) + d);
      o[(size_t)k * D4 + d] = make_float4(v.x - c.x, v.y - c.y, v.z - c.z, v.w - c.w);
    }
  }
}

// hard: V[k,col] = sum_{q: label_q = k} R[q,k,col] (utilities.py:858); CTA = (column slice, cluster), thread = column,
// rows in index order.  Unused clusters stay zero (:840).
__global__ void __launch_bounds__(ACC_COLS)
vlad_from_residuals_hard_kernel(const float* __restrict__ resid, const int32_t* __restrict__ labels, int N, int D, int K,
                                float* __restrict__ vlad, float* __restrict__ partial_ss) {
  const int slice = blockIdx.x, k = blockIdx.y, t = threadIdx.x, nslices = gridDim.x;
  const int col = slice * ACC_COLS + t;
  const bool colok = col < D;
  float acc = 0.f;
  for (int q = 0; q < N; ++q)
    if (__ldg(labels + q) == k && colok) acc += __ldg(resid + ((size_t)q * K + k) * D + col);
  if (colok) vlad[(size_t)k * D + col] = acc;
  __shared__ float red[ACC_COLS / 32];
  const float s = warp_sum(colok ? acc * acc : 0.f);
  if ((t & 31) == 0) red[t >> 5] = s;
  __syncthreads();
  if (t == 0) { float tot = 0.f; for (int w = 0; w < ACC_COLS / 32; ++w) tot += red[w]; partial_ss[(size_t)k * nslices + slice] = tot; }
}

// soft: V[k,col] = sum_q a[q,k] * sum_c R[q,c,col] (utilities.py:879-884: cluster k's weight on the residuals to ALL
// centres).  CTA = column slice, thread = column, 32 cluster accumulators per pass.
__global__ void __launch_bounds__(ACC_COLS)
vlad_from_residuals_soft_kernel(const float* __restrict__ resid, const float* __restrict__ assign, int N, int D, int K,
                                float* __restrict__ vlad, float* __restrict__ partial_ss) {
  const int slice = blockIdx.x, t = threadIdx.x, nslices = gridDim.x;
  const int col = slice * ACC_COLS + t;
  const bool colok = col < D;
  __shared__ float red[ACC_COLS / 32][32];
  for (int k0 = 0; k0 < K; k0 += 32) {
    const int kc = min(32, K - k0);
    float acc[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[j] = 0.f;
    if (colok) {
      for (int q = 0; q < N; ++q) {
        float s = 0.f;
        for (int c = 0; c < K; ++c) s += __ldg(resid + ((size_t)q * K + c) * D + col);
#pragma unroll
        for (int j = 0; j < 32; ++j) if (j < kc) acc[j] = fmaf(__ldg(assign + (size_t)q * K + k0 + j), s, acc[j]);
      }
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      float v = (colok && j < kc) ? acc[j] : 0.f;
      if (colok && j < kc) vlad[(size_t)(k0 + j) * D + col] = v;
      const float sq = warp_sum(v * v);
      if ((t & 31) == 0) red[t >> 5][j] = sq;
    }
    __syncthreads();
    if (t < kc) {
      float tot = 0.f;
      for (int w = 0; w < ACC_COLS / 32; ++w) tot += red[w][t];
      partial_ss[(size_t)(k0 + t) * nslices + slice] = tot;
    }
  }
}

}  // namespace anyloc

extern "C" int anyloc_vlad_residuals(const float* feats, const float* centers, int N, int D, int K, int norm_descs,
                                     float* out, void* stream) {
  ANYLOC_REQUIRE(feats && centers && out, "vlad_residuals: null pointer");
  ANYLOC_REQUIRE(N >= 0 && D > 0 && K > 0 && D % 4 == 0, "vlad_residuals: bad dims N=%d D=%d K=%d", N, D, K);
  ANYLOC_REQUIRE_ALIGNED(feats, 16, "vlad_residuals", "feats", "float4 access");
  ANYLOC_REQUIRE_ALIGNED(centers, 16, "vlad_residuals", "centers", "float4 access");
  ANYLOC_REQUIRE_ALIGNED(out, 16, "vlad_residuals", "out", "float4 access");
  if (N == 0) return ANYLOC_OK;
  cudaStream_t st = (cudaStream_t)stream;
  ProfScope ps(PC_VLAD, st, 4.0 * ((double)N * D + (double)K * D + (double)N * K * D));
  vlad_residuals_kernel<<<N, 256, 0, st>>>(feats, centers, D, K, norm_descs, out);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}

extern "C" size_t anyloc_vlad_from_residuals_workspace_bytes(int D, int K) {
  return align_up((size_t)K * cdiv(D, ACC_COLS) * 4, 256) + 256;
}

extern "C" int anyloc_vlad_from_residuals(const float* resid, const int32_t* labels, const float* assign, int N, int D,
                                          int K, int intra_norm, float* vlad, void* ws, size_t ws_bytes, void* stream) {
  ANYLOC_REQUIRE(resid && vlad && ws, "vlad_from_residuals: null pointer");
  ANYLOC_REQUIRE((labels != nullptr) != (assign != nullptr), "vlad_from_residuals: pass labels (hard) OR assign (soft)");
  ANYLOC_REQUIRE(N >= 0 && D > 0 && K > 0, "vlad_from_residuals: bad dims N=%d D=%d K=%d", N, D, K);
  // scalar kernels throughout (the normalisation included)
  ANYLOC_REQUIRE_ALIGNED(resid, 4, "vlad_from_residuals", "resid", "fp32 access");
  ANYLOC_REQUIRE_ALIGNED(labels, 4, "vlad_from_residuals", "labels", "int32 access");
  ANYLOC_REQUIRE_ALIGNED(assign, 4, "vlad_from_residuals", "assign", "fp32 access");
  ANYLOC_REQUIRE_ALIGNED(vlad, 4, "vlad_from_residuals", "vlad", "fp32 access");
  ANYLOC_REQUIRE_ALIGNED(ws, 4, "vlad_from_residuals", "ws", "fp32 access");
  cudaStream_t st = (cudaStream_t)stream;
  const int nslices = cdiv(D, ACC_COLS);
  Workspace w(ws, ws_bytes);
  float* partial = w.take<float>((size_t)K * nslices);
  if (!partial) { set_error("vlad_from_residuals: workspace too small"); return ANYLOC_ERR_WORKSPACE; }
  ProfScope ps(PC_VLAD, st, 4.0 * ((double)N * K * D + (double)K * D));
  if (labels) vlad_from_residuals_hard_kernel<<<dim3(nslices, K), ACC_COLS, 0, st>>>(resid, labels, N, D, K, vlad, partial);
  else vlad_from_residuals_soft_kernel<<<nslices, ACC_COLS, 0, st>>>(resid, assign, N, D, K, vlad, partial);
  ANYLOC_CHECK_LAUNCH();
  return launch_normalize(vlad, partial, 1, D, K, intra_norm, st);
}

// ====================================================================================================================
// Several vocabularies' descriptors from one read of the features (generate_vocabularies).  The per-row passes are
// shared: anyloc_vlad_label_multi labels each row against every hard vocabulary and writes its 1/|x| once, and
// anyloc_vlad_soft_assign_multi writes every soft vocabulary's assignment from one read of each row.  Each member's
// accumulation then runs alone from those per-row results (anyloc_vlad_accumulate / _varlen) with the kernels, route
// and normalisation its own generate call takes (launch_accumulate, which launches every generate call's
// accumulation), so every descriptor is bitwise that call's.
// ====================================================================================================================
namespace anyloc {

// vlad_rescore_multi_kernel plus what the assignment of a generate call also writes: label -1 for the rows n_valid
// leaves out of their image (row g of the call is row g % N_per_img of image g / N_per_img) and 1/max(|x|,1e-12).  x,
// the labels of each segment and inv_norm point at row r0 of the call; R rows from there.
template <int MAXV>
__global__ void __launch_bounds__(256)
vlad_rescore_multi_norm_kernel(const float* __restrict__ x, const int32_t* __restrict__ n_valid, int N_per_img,
                               int64_t r0, int64_t R, int D, int ldc, const float* __restrict__ chat,
                               const float* __restrict__ cbias, const float* __restrict__ cnorm,
                               const float* __restrict__ coarse /*[R,ldc]*/, const RescoreSegs segs,
                               float* __restrict__ inv_norm) {
  const int lane = threadIdx.x & 31;
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= R) return;
  bool valid = true;
  if (n_valid) {
    const int64_t g = r0 + row;
    valid = (int)(g % N_per_img) < n_valid[(int)(g / N_per_img)];
  }
  float4 v[MAXV];
  const float xn = load_row<MAXV>(x, row, D, lane, v);
  for (int s = 0; s < segs.n; ++s) {
    const int k0 = segs.koff[s];
    const int bestk = rescore_row<MAXV>(v, xn, lane, D, segs.k[s], coarse + row * ldc + k0, chat + (size_t)k0 * D,
                                        cbias + k0, cnorm + k0);
    if (lane == 0) segs.labels[s][row] = valid ? bestk : -1;
  }
  if (lane == 0 && inv_norm) inv_norm[row] = 1.0f / fmaxf(xn, 1e-12f);
}

// Soft assignment of several vocabularies whose normalised centres c / max(|c|, 1e-8) sit side by side in chat
// [sum K, D]: segment s is columns [koff[s], koff[s] + k[s]) with temperature temp[s], written to assign[s] [R, k[s]].
// It restates vlad_soft_assign_kernel operation for operation: the dot products x.c^ are taken once for all segments
// (the same FMAs and warp_sum), each segment's temp / max(|x|, 1e-8) multiplies them afterwards, and the max, the
// exp-sum and the scaling run lane-strided over the segment exactly as over a single vocabulary, so each segment's
// probabilities are that kernel's bits.  Rows n_valid leaves out get exactly 0 (and inv_norm 0).
constexpr int SOFT_MULTI_SEGS = 32;
constexpr int SOFT_MULTI_ROWS = 2;
constexpr int SOFT_MULTI_SMEM = 232448;                  // H100's opt-in shared memory per block
struct SoftSegs {
  int n;
  int koff[SOFT_MULTI_SEGS], k[SOFT_MULTI_SEGS];
  float temp[SOFT_MULTI_SEGS];
  float* assign[SOFT_MULTI_SEGS];
};

template <int ROWS>
__global__ void __launch_bounds__(256)
vlad_soft_assign_multi_kernel(const float* __restrict__ x, const int32_t* __restrict__ n_valid, int N_per_img,
                              int64_t R, int D, int ksum, const float* __restrict__ chat, const SoftSegs segs,
                              float* __restrict__ inv_norm) {
  extern __shared__ float scm_smem[];                  // [warps][ROWS][ksum] raw dot products, then probabilities
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  float* sc = scm_smem + (size_t)wib * ROWS * ksum;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int D4 = D >> 2;
  for (int64_t r0 = warp * ROWS; r0 < R; r0 += nwarps * ROWS) {
    const float4* xr[ROWS];
    bool valid[ROWS];
#pragma unroll
    for (int i = 0; i < ROWS; ++i) {
      int64_t r = r0 + i;
      valid[i] = r < R;
      if (valid[i] && n_valid) valid[i] = (int)(r % N_per_img) < n_valid[(int)(r / N_per_img)];
      xr[i] = reinterpret_cast<const float4*>(x + (r < R ? r : r0) * (int64_t)D);
    }
    float ss[ROWS];
#pragma unroll
    for (int i = 0; i < ROWS; ++i) ss[i] = 0.f;
    for (int d = lane; d < D4; d += 32) {
#pragma unroll
      for (int i = 0; i < ROWS; ++i) {
        float4 v = __ldg(xr[i] + d);
        ss[i] += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
      }
    }
#pragma unroll
    for (int i = 0; i < ROWS; ++i) ss[i] = sqrtf(warp_sum(ss[i]));
    for (int k = 0; k < ksum; ++k) {
      const float4* cr = reinterpret_cast<const float4*>(chat + (size_t)k * D);
      float acc[ROWS];
#pragma unroll
      for (int i = 0; i < ROWS; ++i) acc[i] = 0.f;
      for (int d = lane; d < D4; d += 32) {
        float4 c = __ldg(cr + d);
#pragma unroll
        for (int i = 0; i < ROWS; ++i) {
          float4 v = __ldg(xr[i] + d);
          acc[i] = fmaf(v.x, c.x, acc[i]); acc[i] = fmaf(v.y, c.y, acc[i]);
          acc[i] = fmaf(v.z, c.z, acc[i]); acc[i] = fmaf(v.w, c.w, acc[i]);
        }
      }
#pragma unroll
      for (int i = 0; i < ROWS; ++i) {
        const float s = warp_sum(acc[i]);
        if (lane == 0) sc[i * ksum + k] = s;
      }
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < ROWS; ++i) {
      int64_t r = r0 + i;
      if (r >= R) continue;
      if (!valid[i]) {        // padded row of a ragged batch: exactly 0, whatever it holds (its scores may be NaN)
        for (int s = 0; s < segs.n; ++s)
          for (int k = lane; k < segs.k[s]; k += 32) segs.assign[s][r * segs.k[s] + k] = 0.f;
        if (lane == 0 && inv_norm) inv_norm[r] = 0.f;
        continue;
      }
      for (int s = 0; s < segs.n; ++s) {
        const int K = segs.k[s];
        float* row = sc + i * ksum + segs.koff[s];
        const float rx = segs.temp[s] / fmaxf(ss[i], 1e-8f);
        float m = -INFINITY;
        for (int k = lane; k < K; k += 32) { const float v = row[k] * rx; row[k] = v; m = fmaxf(m, v); }
        m = warp_max(m);
        float z = 0.f;
        for (int k = lane; k < K; k += 32) { float e = expf(row[k] - m); row[k] = e; z += e; }
        z = warp_sum(z);
        const float iz = 1.0f / z;
        float* a = segs.assign[s] + r * K;
        for (int k = lane; k < K; k += 32) a[k] = row[k] * iz;
      }
      if (lane == 0 && inv_norm) inv_norm[r] = 1.0f / fmaxf(ss[i], 1e-12f);
    }
    __syncwarp();
  }
}

}  // namespace anyloc

namespace {
// anyloc_vlad_label_multi's workspace: the prepared centres of all vocabularies side by side ([sum K, D] c^, its tf32
// copy, bias, norms) and, for D <= 2048, one slice of coarse scores.  Unlike anyloc_vlad_assign_multi's, the slice is
// there for R < 256 too: a member's route rows, not R, decide whether it takes the tensor-core route.  ws == nullptr:
// dry run.
size_t carve_label_multi(void* ws, size_t ws_bytes, int64_t R, int D, int64_t Ksum, AssignBufs* ab) {
  Workspace w(ws ? ws : (void*)256, ws ? ws_bytes : (size_t)-1 / 2);
  ab->chat = w.take<float>((size_t)Ksum * D);
  ab->chat_tf32 = w.take<float>((size_t)Ksum * D);
  ab->cbias = w.take<float>(Ksum);
  ab->cnorm = w.take<float>(Ksum);
  const bool coarse = D <= 2048 && R > 0;
  ab->coarse = coarse ? w.take<float>((size_t)assign_multi_slice(R, Ksum) * Ksum) : nullptr;
  const bool ok = ab->chat && ab->chat_tf32 && ab->cbias && ab->cnorm && (ab->coarse || !coarse);
  return ok ? w.off : 0;
}

// anyloc_vlad_accumulate(_varlen)'s workspace for B images of up to N rows: the per-slice sums of squares, the
// accumulate3 tickets on that route and the sorted route's per-image tables on that one (route < 0: soft, the sums
// alone).  ws == nullptr: dry run.
size_t carve_accumulate(void* ws, size_t ws_bytes, int B, int N, int D, int K, int route, float** partial,
                        int32_t** done, SortedTables* tb) {
  Workspace w(ws ? ws : (void*)256, ws ? ws_bytes : (size_t)-1 / 2);
  *partial = w.take<float>((size_t)B * K * cdiv(D, ACC_COLS));
  *done = route == ANYLOC_VLAD_ROUTE_ACC3 ? w.take<int32_t>((size_t)B) : nullptr;
  bool ok = *partial && (route != ANYLOC_VLAD_ROUTE_ACC3 || *done);
  if (route == ANYLOC_VLAD_ROUTE_SORTED) ok = take_sorted_tables(w, B, N, D, K, tb) && ok;
  return ok ? w.off : 0;
}

// The pointers of both accumulate entries: the hard routes read feats and the centres and write the descriptors as
// float4 (the sorted route's tables hold int64 and float4 slots); labels, soft weights, n_valid and 1/|x| are read one
// 32-bit word at a time.
int accumulate_alignment(const char* who, const float* feats, const int32_t* labels, const float* assign,
                         const float* inv_norm, const float* centers, const float* vlad, const void* ws) {
  ANYLOC_REQUIRE_ALIGNED(feats, 16, who, "feats", "float4 access");
  ANYLOC_REQUIRE_ALIGNED(labels, 4, who, "labels", "int32 access");
  ANYLOC_REQUIRE_ALIGNED(assign, 4, who, "assign", "fp32 access");
  ANYLOC_REQUIRE_ALIGNED(inv_norm, 4, who, "inv_norm", "fp32 access");
  ANYLOC_REQUIRE_ALIGNED(centers, 16, who, "centers", "float4 access");
  ANYLOC_REQUIRE_ALIGNED(vlad, 16, who, "vlad", "float4 access");
  ANYLOC_REQUIRE_ALIGNED(ws, 16, who, "ws", "float4 access");
  return ANYLOC_OK;
}

// anyloc_vlad_accumulate(_varlen) after their refusals: the route, the workspace and the tickets, then the launches
template <bool PACKED>
int accumulate_call(const float* feats, const int32_t* n_valid, const int64_t* row0, const int32_t* len,
                    const int32_t* labels, const float* assign, const float* inv_norm, const float* centers, int B,
                    int N, int D, int K, int norm_descs, int intra_norm, float* vlad, void* ws, size_t ws_bytes,
                    const char* who, cudaStream_t st) {
  const int route = assign ? -1 : vlad_route(N, D, K);
  const int ztasks = cdiv(acc3_max_tasks(N, K), SORTED_TASKS_PER_CTA);
  ANYLOC_REQUIRE(route != ANYLOC_VLAD_ROUTE_SORTED || ztasks <= 65535, "%s: N=%d K=%d exceed the launch grid", who, N,
                 K);
  float* partial;
  int32_t* done;
  SortedTables tb;
  if (!carve_accumulate(ws, ws_bytes, B, N, D, K, route, &partial, &done, &tb)) {
    size_t need = carve_accumulate(nullptr, 0, B, N, D, K, route, &partial, &done, &tb);
    set_error("%s: workspace too small (%zu bytes given, %zu needed)", who, ws_bytes, need);
    return ANYLOC_ERR_WORKSPACE;
  }
  if (N == 0) {                                     // every image empty: zero descriptors, like the generate calls
    ANYLOC_CHECK_CUDA(cudaMemsetAsync(vlad, 0, (size_t)B * K * D * 4, st));
    return ANYLOC_OK;
  }
  ProfScope ps(PC_VLAD, st, 4.0 * ((double)B * N * D + (double)B * K * D));
  if (done) ANYLOC_CHECK_CUDA(cudaMemsetAsync(done, 0, (size_t)B * sizeof(int32_t), st));
  return launch_accumulate<PACKED>(feats, n_valid, row0, len, labels, assign, inv_norm, centers, B, N, D, K, norm_descs,
                                   intra_norm, vlad, route, partial, done, &tb, st);
}
}  // namespace

extern "C" size_t anyloc_vlad_label_multi_workspace_bytes(int64_t R, int D, int V, const int* K) {
  if (!K || V <= 0 || D <= 0 || R < 0) return 0;
  for (int v = 0; v < V; ++v)
    if (K[v] <= 0) return 0;
  AssignBufs ab;
  return carve_label_multi(nullptr, 0, R, D, assign_multi_ksum(V, K), &ab);
}

extern "C" int anyloc_vlad_label_multi(const float* feats, const int32_t* n_valid, int N, int64_t R,
                                       const int64_t* route_rows, int D, int V, const float* const* centers,
                                       void* const* prepared, const size_t* prepared_bytes, const int* K,
                                       int dist_mode, int32_t* labels, float* inv_norm, void* ws, size_t ws_bytes,
                                       void* stream) {
  const char* who = "vlad_label_multi";
  ANYLOC_REQUIRE(feats && centers && K && labels && inv_norm && ws, "%s: null pointer", who);
  ANYLOC_REQUIRE(R >= 0 && R < (1ll << 31) && D > 0 && D % 4 == 0 && V > 0 && (!n_valid || (N > 0 && R % N == 0)),
                 "%s: bad dims R=%lld N=%d D=%d V=%d (R < 2^31, D a multiple of 4, R a multiple of N with n_valid)",
                 who, (long long)R, N, D, V);
  ANYLOC_REQUIRE(dist_mode == ANYLOC_DIST_COSINE || dist_mode == ANYLOC_DIST_EUCLIDEAN, "%s: unknown dist_mode %d",
                 who, dist_mode);
  ANYLOC_REQUIRE(!prepared || prepared_bytes, "%s: prepared blobs without their sizes", who);
  for (int v = 0; v < V; ++v) {
    ANYLOC_REQUIRE(K[v] > 0 && centers[v], "%s: vocabulary %d has K=%d or no centres", who, v, K[v]);
    ANYLOC_REQUIRE(!route_rows || route_rows[v] >= 0, "%s: route_rows[%d] = %lld", who, v,
                   (long long)route_rows[v]);
    ANYLOC_REQUIRE((reinterpret_cast<uintptr_t>(centers[v]) & 3) == 0,
                   "%s: centers[%d] must be 4-byte aligned (fp32 access)", who, v);
    ANYLOC_REQUIRE(!prepared || (reinterpret_cast<uintptr_t>(prepared[v]) & 15) == 0,
                   "%s: prepared[%d] must be 16-byte aligned (float4 and TMA access)", who, v);
  }
  int rc = assign_alignment(who, feats, labels, ws);
  if (rc) return rc;
  ANYLOC_REQUIRE_ALIGNED(n_valid, 4, who, "n_valid", "int32 access");
  ANYLOC_REQUIRE_ALIGNED(inv_norm, 4, who, "inv_norm", "fp32 access");
  const int64_t Ksum = assign_multi_ksum(V, K);
  ANYLOC_REQUIRE(Ksum < (1ll << 31), "%s: %lld centres in all", who, (long long)Ksum);
  if (R == 0) return ANYLOC_OK;
  AssignBufs ab;
  if (!carve_label_multi(ws, ws_bytes, R, D, Ksum, &ab)) {
    set_error("%s: workspace too small (%zu given, %zu needed)", who, ws_bytes,
              anyloc_vlad_label_multi_workspace_bytes(R, D, V, K));
    return ANYLOC_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  ProfScope ps(PC_VLAD, st, 4.0 * ((double)R * D + (double)Ksum * D));
  // each vocabulary's centres from its prepared blob where one is given (what its own generate call reads), else
  // prepared here by the same kernel
  std::vector<int> koff(V), fast(V);
  bool any_fast = false;
  for (int v = 0, off = 0; v < V; off += K[v], ++v) {
    koff[v] = off;
    PreparedView pv;
    if (prepared && prepared[v] && carve_prepared(prepared[v], prepared_bytes[v], D, K[v], &pv)) {
      const size_t kd = (size_t)K[v] * D * 4, k4 = (size_t)K[v] * 4;
      ANYLOC_CHECK_CUDA(cudaMemcpyAsync(ab.chat + (size_t)off * D, pv.chat, kd, cudaMemcpyDeviceToDevice, st));
      ANYLOC_CHECK_CUDA(cudaMemcpyAsync(ab.chat_tf32 + (size_t)off * D, pv.chat_tf32, kd, cudaMemcpyDeviceToDevice, st));
      ANYLOC_CHECK_CUDA(cudaMemcpyAsync(ab.cbias + off, pv.cbias, k4, cudaMemcpyDeviceToDevice, st));
      ANYLOC_CHECK_CUDA(cudaMemcpyAsync(ab.cnorm + off, pv.cnorm, k4, cudaMemcpyDeviceToDevice, st));
    } else {
      vlad_centre_prep_kernel<<<K[v], 256, 0, st>>>(centers[v], K[v], D, dist_mode, ab.chat + (size_t)off * D,
                                                    ab.cbias + off, ab.chat_tf32 + (size_t)off * D, ab.cnorm + off,
                                                    nullptr, 0);
      ANYLOC_CHECK_LAUNCH();
    }
    // launch_assign's test, with the rows of the member's own call (route_rows[v]) where it takes the route from
    const EpiParams ep{ANYLOC_EPI_BIAS, ab.cbias, nullptr, nullptr, ab.coarse, nullptr, K[v]};
    const int64_t rr = route_rows ? route_rows[v] : R;
    fast[v] = ab.coarse != nullptr && D <= 2048 && rr >= 256 &&
              gemm_tc_supported(feats, nullptr, D, ab.chat_tf32, nullptr, D, (int)R, K[v], D, ep, ANYLOC_PAIR_TF32);
    any_fast = any_fast || fast[v];
  }
  // the FFMA members; the first writes 1/|x| when no member rescores (the rescoring writes it otherwise)
  float* inv_ffma = any_fast ? nullptr : inv_norm;
  for (int v = 0; v < V; ++v) {
    if (fast[v]) continue;
    const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>(((R + 1) / 2 + 7) / 8, (int64_t)device_sm_count() * 8));
    vlad_assign_kernel<2><<<blocks, 256, 0, st>>>(feats, n_valid, n_valid ? N : (int)R, R, D, K[v],
                                                  ab.chat + (size_t)koff[v] * D, ab.cbias + koff[v],
                                                  labels + (size_t)v * R, inv_ffma);
    ANYLOC_CHECK_LAUNCH();
    inv_ffma = nullptr;
  }
  if (!any_fast) return ANYLOC_OK;
  const int64_t S = assign_multi_slice(R, Ksum);
  const EpiParams ep{ANYLOC_EPI_BIAS, ab.cbias, nullptr, nullptr, ab.coarse, nullptr, (int)Ksum};
  for (int64_t r0 = 0; r0 < R; r0 += S) {
    const int m = (int)std::min<int64_t>(S, R - r0);
    const float* xs = feats + r0 * D;
    rc = gemm_tc_launch(xs, nullptr, D, ab.chat_tf32, nullptr, D, m, (int)Ksum, D, ep, ANYLOC_PAIR_TF32, st);
    if (rc) return rc;
    RescoreSegs segs;
    segs.n = 0;
    float* inv = inv_norm + r0;                      // written by the slice's first rescoring launch
    for (int v = 0; v < V; ++v) {
      if (fast[v]) {
        segs.koff[segs.n] = koff[v];
        segs.k[segs.n] = K[v];
        segs.labels[segs.n] = labels + (size_t)v * R + r0;
        ++segs.n;
      }
      if (segs.n == ASSIGN_MULTI_SEGS || (v == V - 1 && segs.n > 0)) {
        const int blocks = (m + 7) / 8;
        const int Nn = n_valid ? N : 1;
        if (D <= 512)
          vlad_rescore_multi_norm_kernel<4><<<blocks, 256, 0, st>>>(xs, n_valid, Nn, r0, m, D, (int)Ksum, ab.chat,
                                                                    ab.cbias, ab.cnorm, ab.coarse, segs, inv);
        else if (D <= 1024)
          vlad_rescore_multi_norm_kernel<8><<<blocks, 256, 0, st>>>(xs, n_valid, Nn, r0, m, D, (int)Ksum, ab.chat,
                                                                    ab.cbias, ab.cnorm, ab.coarse, segs, inv);
        else
          vlad_rescore_multi_norm_kernel<16><<<blocks, 256, 0, st>>>(xs, n_valid, Nn, r0, m, D, (int)Ksum, ab.chat,
                                                                     ab.cbias, ab.cnorm, ab.coarse, segs, inv);
        ANYLOC_CHECK_LAUNCH();
        segs.n = 0;
        inv = nullptr;
      }
    }
  }
  return ANYLOC_OK;
}

extern "C" size_t anyloc_vlad_soft_assign_multi_workspace_bytes(int D, int V, const int* K) {
  if (!K || V <= 0 || D <= 0) return 0;
  for (int v = 0; v < V; ++v)
    if (K[v] <= 0) return 0;
  return align_up((size_t)assign_multi_ksum(V, K) * D * 4, 256);
}

extern "C" int anyloc_vlad_soft_assign_multi(const float* feats, const int32_t* n_valid, int N, int64_t R, int D, int V,
                                             const float* const* centers, const int* K, const float* soft_temp,
                                             float* const* assign, float* inv_norm, void* ws, size_t ws_bytes,
                                             void* stream) {
  const char* who = "vlad_soft_assign_multi";
  ANYLOC_REQUIRE(feats && centers && K && soft_temp && assign && inv_norm && ws, "%s: null pointer", who);
  ANYLOC_REQUIRE(R >= 0 && R < (1ll << 31) && D > 0 && D % 4 == 0 && V > 0 && (!n_valid || (N > 0 && R % N == 0)),
                 "%s: bad dims R=%lld N=%d D=%d V=%d (R < 2^31, D a multiple of 4, R a multiple of N with n_valid)",
                 who, (long long)R, N, D, V);
  for (int v = 0; v < V; ++v) {
    ANYLOC_REQUIRE(K[v] > 0 && K[v] <= 2048 && centers[v] && assign[v],
                   "%s: vocabulary %d has K=%d (1..2048), no centres or no assignment", who, v, K[v]);
    ANYLOC_REQUIRE((reinterpret_cast<uintptr_t>(centers[v]) & 3) == 0,
                   "%s: centers[%d] must be 4-byte aligned (fp32 access)", who, v);
    ANYLOC_REQUIRE((reinterpret_cast<uintptr_t>(assign[v]) & 3) == 0,
                   "%s: assign[%d] must be 4-byte aligned (fp32 access)", who, v);
  }
  ANYLOC_REQUIRE_ALIGNED(feats, 16, who, "feats", "float4 access");
  ANYLOC_REQUIRE_ALIGNED(n_valid, 4, who, "n_valid", "int32 access");
  ANYLOC_REQUIRE_ALIGNED(inv_norm, 4, who, "inv_norm", "fp32 access");
  ANYLOC_REQUIRE_ALIGNED(ws, 16, who, "ws", "float4 access");
  if (R == 0) return ANYLOC_OK;
  Workspace w(ws, ws_bytes);
  const int64_t Ksum = assign_multi_ksum(V, K);
  float* chat = w.take<float>((size_t)Ksum * D);
  if (!chat) {
    set_error("%s: workspace too small (%zu given, %zu needed)", who, ws_bytes,
              anyloc_vlad_soft_assign_multi_workspace_bytes(D, V, K));
    return ANYLOC_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  ProfScope ps(PC_VLAD, st, 4.0 * ((double)R * D + (double)Ksum * D));
  for (int v = 0, off = 0; v < V; off += K[v], ++v) {
    vlad_soft_centre_prep_kernel<<<K[v], 256, 0, st>>>(centers[v], K[v], D, chat + (size_t)off * D);
    ANYLOC_CHECK_LAUNCH();
  }
  // consecutive members share a launch while their scores fit a warp's share of shared memory (and at most
  // SOFT_MULTI_SEGS of them); a launch of wider scores runs fewer warps per block
  constexpr int ROWS = SOFT_MULTI_ROWS;
  float* inv = inv_norm;                             // written by the first launch
  for (int v0 = 0, off0 = 0; v0 < V;) {
    SoftSegs segs;
    segs.n = 0;
    int ksum = 0;
    while (v0 + segs.n < V && segs.n < SOFT_MULTI_SEGS &&
           (size_t)(ksum + K[v0 + segs.n]) * ROWS * 4 <= (size_t)SOFT_MULTI_SMEM) {
      const int v = v0 + segs.n;
      segs.koff[segs.n] = ksum;
      segs.k[segs.n] = K[v];
      segs.temp[segs.n] = soft_temp[v];
      segs.assign[segs.n] = assign[v];
      ksum += K[v];
      ++segs.n;
    }
    const int warps = (int)std::min<size_t>(8, (size_t)SOFT_MULTI_SMEM / ((size_t)ROWS * ksum * 4));
    const size_t smem = (size_t)warps * ROWS * ksum * 4;
    ANYLOC_CHECK_CUDA(cudaFuncSetAttribute(vlad_soft_assign_multi_kernel<ROWS>,
                                           cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t blocks = std::min<int64_t>(((R + ROWS - 1) / ROWS + warps - 1) / warps,
                                             (int64_t)device_sm_count() * 64 / warps);
    vlad_soft_assign_multi_kernel<ROWS><<<(int)std::max<int64_t>(blocks, 1), warps * 32, smem, st>>>(
        feats, n_valid, n_valid ? N : 1, R, D, ksum, chat + (size_t)off0 * D, segs, inv);
    ANYLOC_CHECK_LAUNCH();
    inv = nullptr;
    v0 += segs.n;
    off0 += ksum;
  }
  return ANYLOC_OK;
}

extern "C" size_t anyloc_vlad_accumulate_workspace_bytes(int B, int N, int D, int K, int soft) {
  if (B < 0 || N < 0 || D <= 0 || K <= 0) return 0;
  float* partial;
  int32_t* done;
  SortedTables tb;
  return carve_accumulate(nullptr, 0, B, N, D, K, soft ? -1 : vlad_route(N, D, K), &partial, &done, &tb);
}

extern "C" int anyloc_vlad_accumulate(const float* feats, const int32_t* n_valid, const int32_t* labels,
                                      const float* assign, const float* inv_norm, const float* centers, int B, int N,
                                      int D, int K, int norm_descs, int intra_norm, float* vlad, void* ws,
                                      size_t ws_bytes, void* stream) {
  const char* who = "vlad_accumulate";
  ANYLOC_REQUIRE(feats && inv_norm && centers && vlad && ws, "%s: null pointer", who);
  ANYLOC_REQUIRE((labels != nullptr) != (assign != nullptr), "%s: pass labels (hard) OR assign (soft)", who);
  ANYLOC_REQUIRE(B >= 0 && B <= 65535 && N >= 0 && D > 0 && K > 0 && D % 4 == 0 && (int64_t)B * N < (1ll << 31),
                 "%s: bad dims B=%d N=%d D=%d K=%d (B <= 65535, B * N < 2^31, D a multiple of 4)", who, B, N, D, K);
  int rc = accumulate_alignment(who, feats, labels, assign, inv_norm, centers, vlad, ws);
  if (rc) return rc;
  ANYLOC_REQUIRE_ALIGNED(n_valid, 4, who, "n_valid", "int32 access");
  if (B == 0) return ANYLOC_OK;
  return accumulate_call<false>(feats, assign ? n_valid : nullptr, nullptr, nullptr, labels, assign, inv_norm, centers,
                                B, N, D, K, norm_descs, intra_norm, vlad, ws, ws_bytes, who, (cudaStream_t)stream);
}

extern "C" int anyloc_vlad_accumulate_varlen(const float* feats, int64_t R, const int64_t* row0, const int32_t* len,
                                             int B, const int32_t* labels, const float* assign, const float* inv_norm,
                                             const float* centers, int D, int K, int norm_descs, int intra_norm,
                                             float* vlad, void* ws, size_t ws_bytes, void* stream) {
  const char* who = "vlad_accumulate_varlen";
  int rc = varlen_args(who, feats, R, row0, len, B, D, K, vlad);
  if (rc) return rc;
  ANYLOC_REQUIRE(inv_norm && centers && ws, "%s: null pointer", who);
  ANYLOC_REQUIRE((labels != nullptr) != (assign != nullptr), "%s: pass labels (hard) OR assign (soft)", who);
  rc = accumulate_alignment(who, feats, labels, assign, inv_norm, centers, vlad, ws);
  if (rc) return rc;
  if (B == 0) return ANYLOC_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int N = 0;                                        // the padded batch's row count: the longest image
  rc = varlen_rows_check(row0, len, B, R, st, who, &N);
  if (rc) return rc;
  return accumulate_call<true>(feats, nullptr, row0, len, labels, assign, inv_norm, centers, B, N, D, K, norm_descs,
                               intra_norm, vlad, ws, ws_bytes, who, st);
}
