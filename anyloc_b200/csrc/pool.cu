// Sibling aggregators on the same patch features (SURVEY 8f rank 3): GeM (scripts/dino_v2_gem.py:170-189) and
// average / max pooling (scripts/dino_v2_gp.py:130-135) over the patch axis of [B,N,D] features -> [B,D].
//   average : mean_n x                      max : max_n x
//   gem     : m = mean_n x^p (|x|^p with use_abs);  out = sign(m) |m|^(1/p)   (the reference takes the complex
//             root and restores the sign; with use_abs it is the plain real root)
// One read of the features (HBM-bound, 4 B per element).  CTA = (128-column slice, image): 8 row groups x 32 lanes
// x float4 columns, fixed-order shared-memory reduction across the row groups -> deterministic.  An image with no
// valid rows (n_valid[b] <= 0) is written NaN in every mode: torch's mean of an empty set, and max has no value.
#include <algorithm>
#include <vector>
#include "common.cuh"

namespace anyloc {

enum { POOL_AVG = 0, POOL_MAX = 1, POOL_GEM = 2 };

__device__ __forceinline__ float gem_pow(float x, float p, int ip, bool use_abs) {
  if (use_abs) x = fabsf(x);
  if (ip > 0) {                       // integer exponent: repeated products like torch.pow(x, 3)
    float r = x;
    for (int i = 1; i < ip; ++i) r *= x;
    return r;
  }
  return powf(x, p);                  // NaN for negative x and fractional p, as in the reference
}

// torch.max propagates NaN (fmaxf drops it)
__device__ __forceinline__ float nanmax(float a, float b) { return (a != a) ? a : ((b != b) ? b : fmaxf(a, b)); }

// Image b's rows: `rows.first(b)` is its first row in x, `rows.count(b)` how many of them it pools (common.cuh).
template <int MODE, class Rows>
__device__ __forceinline__ void pool_image(const float* __restrict__ x, Rows rows, int D, float p, int ip, int use_abs,
                                           float* __restrict__ out) {
  __shared__ float4 part[8][32];
  const int lane = threadIdx.x & 31, grp = threadIdx.x >> 5;
  const int b = blockIdx.y, col = blockIdx.x * 128 + lane * 4;
  const int n = rows.count(b);
  const bool colok = col < D;
  float4 acc = MODE == POOL_MAX ? make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY) : make_float4(0.f, 0.f, 0.f, 0.f);
  if (colok) {
    const float* xb = x + rows.first(b) * D + col;
    for (int r = grp; r < n; r += 8) {
      float4 v = __ldg(reinterpret_cast<const float4*>(xb + (size_t)r * D));
      if (MODE == POOL_MAX) {
        acc.x = nanmax(acc.x, v.x); acc.y = nanmax(acc.y, v.y); acc.z = nanmax(acc.z, v.z); acc.w = nanmax(acc.w, v.w);
      } else if (MODE == POOL_GEM) {
        acc.x += gem_pow(v.x, p, ip, use_abs); acc.y += gem_pow(v.y, p, ip, use_abs);
        acc.z += gem_pow(v.z, p, ip, use_abs); acc.w += gem_pow(v.w, p, ip, use_abs);
      } else {
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
    }
  }
  part[grp][lane] = acc;
  __syncthreads();
  if (grp == 0 && colok) {
    float r[4] = {acc.x, acc.y, acc.z, acc.w};
    for (int g = 1; g < 8; ++g) {
      float4 o = part[g][lane];
      float q[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (MODE == POOL_MAX) r[i] = nanmax(r[i], q[i]);
        else r[i] += q[i];
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (MODE != POOL_MAX) r[i] = r[i] / (float)n;
      if (MODE == POOL_GEM) {
        const float m = r[i];
        const float root = powf(fabsf(m), 1.0f / p);
        r[i] = use_abs ? root : (m > 0.f ? root : (m < 0.f ? -root : (m == 0.f ? 0.f : m)));
      }
      if (n <= 0) r[i] = __int_as_float(0x7fc00000);
    }
    *reinterpret_cast<float4*>(out + (size_t)b * D + col) = make_float4(r[0], r[1], r[2], r[3]);
  }
}

template <int MODE>
__global__ void __launch_bounds__(256)
pool_kernel(const float* __restrict__ x, const int32_t* __restrict__ n_valid, int N, int D, float p, int ip,
            int use_abs, float* __restrict__ out) {
  pool_image<MODE>(x, PaddedRows{n_valid, N}, D, p, ip, use_abs, out);
}

// packed images: image b is rows [row0[b], row0[b] + len[b]) of x
template <int MODE>
__global__ void __launch_bounds__(256)
pool_varlen_kernel(const float* __restrict__ x, const int64_t* __restrict__ row0, const int32_t* __restrict__ len,
                   int D, float p, int ip, int use_abs, float* __restrict__ out) {
  pool_image<MODE>(x, PackedRows{row0, len}, D, p, ip, use_abs, out);
}

}  // namespace anyloc

using namespace anyloc;

extern "C" int anyloc_pool(const float* feats, const int32_t* n_valid, int B, int N, int D, int mode, float gem_p,
                           int gem_use_abs, float* out, void* stream) {
  ANYLOC_REQUIRE(feats && out, "pool: null pointer");
  ANYLOC_REQUIRE(B >= 0 && N > 0 && D > 0 && D % 4 == 0, "pool: bad dims B=%d N=%d D=%d (D multiple of 4)", B, N, D);
  ANYLOC_REQUIRE(B <= 65535, "pool: B=%d exceeds the grid limit", B);
  ANYLOC_REQUIRE(mode >= POOL_AVG && mode <= POOL_GEM, "pool: unknown mode %d", mode);
  ANYLOC_REQUIRE(mode != POOL_GEM || gem_p != 0.f, "pool: gem_p must be non-zero");
  ANYLOC_REQUIRE_ALIGNED(feats, 16, "pool", "feats", "float4 access");
  ANYLOC_REQUIRE_ALIGNED(out, 16, "pool", "out", "float4 access");
  ANYLOC_REQUIRE_ALIGNED(n_valid, 4, "pool", "n_valid", "int32 access");
  if (B == 0) return ANYLOC_OK;
  cudaStream_t st = (cudaStream_t)stream;
  dim3 grid(cdiv(D, 128), B);
  const int ip = (gem_p == floorf(gem_p) && gem_p >= 1.f && gem_p <= 16.f) ? (int)gem_p : 0;
  if (mode == POOL_AVG) pool_kernel<POOL_AVG><<<grid, 256, 0, st>>>(feats, n_valid, N, D, gem_p, ip, gem_use_abs, out);
  else if (mode == POOL_MAX) pool_kernel<POOL_MAX><<<grid, 256, 0, st>>>(feats, n_valid, N, D, gem_p, ip, gem_use_abs, out);
  else pool_kernel<POOL_GEM><<<grid, 256, 0, st>>>(feats, n_valid, N, D, gem_p, ip, gem_use_abs, out);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}

namespace anyloc {
int varlen_rows_check(const int64_t* row0, const int32_t* len, int B, int64_t R, cudaStream_t st, const char* who,
                      int* max_len) {
  std::vector<int64_t> r0(B);
  std::vector<int32_t> n(B);
  ANYLOC_CHECK_CUDA(cudaMemcpyAsync(r0.data(), row0, (size_t)B * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  ANYLOC_CHECK_CUDA(cudaMemcpyAsync(n.data(), len, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  ANYLOC_CHECK_CUDA(cudaStreamSynchronize(st));
  int m = 0;
  std::vector<int> by_row;
  by_row.reserve(B);
  for (int i = 0; i < B; ++i) {
    ANYLOC_REQUIRE(n[i] >= 0 && r0[i] >= 0 && r0[i] <= R - n[i], "%s: image %d has row0=%lld len=%d (R=%lld rows)", who,
                   i, (long long)r0[i], n[i], (long long)R);
    m = std::max(m, n[i]);
    if (n[i] > 0) by_row.push_back(i);
  }
  std::sort(by_row.begin(), by_row.end(), [&](int a, int b) { return r0[a] < r0[b]; });
  for (size_t k = 1; k < by_row.size(); ++k)
    ANYLOC_REQUIRE(r0[by_row[k - 1]] + n[by_row[k - 1]] <= r0[by_row[k]], "%s: images %d and %d overlap", who,
                   by_row[k - 1], by_row[k]);
  *max_len = m;
  return ANYLOC_OK;
}
}  // namespace anyloc

extern "C" int anyloc_pool_varlen(const float* feats, int64_t R, const int64_t* row0, const int32_t* len, int B, int D,
                                  int mode, float gem_p, int gem_use_abs, float* out, void* stream) {
  ANYLOC_REQUIRE(B >= 0 && B <= 65535 && R >= 0 && D > 0 && D % 4 == 0,
                 "pool_varlen: bad dims B=%d R=%lld D=%d (B <= 65535, D multiple of 4)", B, (long long)R, D);
  ANYLOC_REQUIRE(mode >= POOL_AVG && mode <= POOL_GEM, "pool_varlen: unknown mode %d", mode);
  ANYLOC_REQUIRE(mode != POOL_GEM || gem_p != 0.f, "pool_varlen: gem_p must be non-zero");
  ANYLOC_REQUIRE_ALIGNED(feats, 16, "pool_varlen", "feats", "float4 access");
  ANYLOC_REQUIRE_ALIGNED(row0, 8, "pool_varlen", "row0", "int64 access");
  ANYLOC_REQUIRE_ALIGNED(len, 4, "pool_varlen", "len", "int32 access");
  ANYLOC_REQUIRE_ALIGNED(out, 16, "pool_varlen", "out", "float4 access");
  if (B == 0) return ANYLOC_OK;
  ANYLOC_REQUIRE(feats && row0 && len && out, "pool_varlen: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  int max_len = 0;
  const int rc = varlen_rows_check(row0, len, B, R, st, "pool_varlen", &max_len);
  if (rc) return rc;
  dim3 grid(cdiv(D, 128), B);
  const int ip = (gem_p == floorf(gem_p) && gem_p >= 1.f && gem_p <= 16.f) ? (int)gem_p : 0;
  if (mode == POOL_AVG) pool_varlen_kernel<POOL_AVG><<<grid, 256, 0, st>>>(feats, row0, len, D, gem_p, ip, gem_use_abs, out);
  else if (mode == POOL_MAX) pool_varlen_kernel<POOL_MAX><<<grid, 256, 0, st>>>(feats, row0, len, D, gem_p, ip, gem_use_abs, out);
  else pool_varlen_kernel<POOL_GEM><<<grid, 256, 0, st>>>(feats, row0, len, D, gem_p, ip, gem_use_abs, out);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}
