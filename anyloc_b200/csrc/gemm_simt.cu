// fp32 FFMA GEMM  C[M,N] = (A_hi+A_lo)[M,K] . (B_hi+B_lo)[N,K]^T  + epilogue.
// Validation engine and the engine for shapes the tensor-core (wgmma) kernel does not take.
// 128x128x16 CTA tile, 256 threads, 8x8 register micro-tile, double-buffered shared memory.
#include "epilogue.cuh"

namespace anyloc {

constexpr int BM = 128, BN = 128, BK = 16;

template <typename T> __device__ __forceinline__ float4 load4(const T* p);
template <> __device__ __forceinline__ float4 load4<float>(const float* p) {
  return __ldg(reinterpret_cast<const float4*>(p));
}
template <> __device__ __forceinline__ float4 load4<__half>(const __half* p) {
  uint2 raw = __ldg(reinterpret_cast<const uint2*>(p));
  const __half2* h = reinterpret_cast<const __half2*>(&raw);
  float2 a = __half22float2(h[0]), b = __half22float2(h[1]);
  return make_float4(a.x, a.y, b.x, b.y);
}

// T = float: (hi,lo) tf32 pairs; T = __half: fp16 pairs (scaled; ep.alpha undoes the scale)
template <typename T>
__global__ void __launch_bounds__(256)
gemm_simt_kernel(const T* __restrict__ a_hi, const T* __restrict__ a_lo, int lda,
                 const T* __restrict__ b_hi, const T* __restrict__ b_lo, int ldb,
                 int M, int N, int K, EpiParams ep) {
  __shared__ float As[2][BK][BM + 4];
  __shared__ float Bs[2][BK][BN + 4];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  // loader mapping: each thread loads 2 float4 of A and 2 of B per k-tile (128 rows x 16 k)
  const int lrow = tid >> 2;          // 0..63
  const int lk = (tid & 3) * 4;       // 0,4,8,12
  const int tx = tid & 15, ty = tid >> 4;   // 16x16 threads; micro tile rows ty*4 + {0..3, 64..67}, cols likewise
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  float4 ra[2], rb[2];
  auto gload = [&](int k0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      int r = lrow + h * 64;
      int gm = m0 + r, gn = n0 + r, gk = k0 + lk;
      float4 va = make_float4(0.f, 0.f, 0.f, 0.f), vb = va;
      if (gm < M && gk < K) {
        va = load4<T>(a_hi + (size_t)gm * lda + gk);
        if (a_lo) { float4 l = load4<T>(a_lo + (size_t)gm * lda + gk);
                    va.x += l.x; va.y += l.y; va.z += l.z; va.w += l.w; }
      }
      if (gn < N && gk < K) {
        vb = load4<T>(b_hi + (size_t)gn * ldb + gk);
        if (b_lo) { float4 l = load4<T>(b_lo + (size_t)gn * ldb + gk);
                    vb.x += l.x; vb.y += l.y; vb.z += l.z; vb.w += l.w; }
      }
      ra[h] = va; rb[h] = vb;
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      int r = lrow + h * 64;
      As[buf][lk + 0][r] = ra[h].x; As[buf][lk + 1][r] = ra[h].y;
      As[buf][lk + 2][r] = ra[h].z; As[buf][lk + 3][r] = ra[h].w;
      Bs[buf][lk + 0][r] = rb[h].x; Bs[buf][lk + 1][r] = rb[h].y;
      Bs[buf][lk + 2][r] = rb[h].z; Bs[buf][lk + 3][r] = rb[h].w;
    }
  };
  const int nk = (K + BK - 1) / BK;
  gload(0); sstore(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) gload((kt + 1) * BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
      float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4 + 64]);
      float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
      float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4 + 64]);
      float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (kt + 1 < nk) sstore(buf ^ 1);
    __syncthreads();
  }
  // epilogue
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int m = m0 + ty * 4 + (i & 3) + (i >> 2) * 64;
    if (m >= M) continue;
    if (ep.mode == ANYLOC_EPI_SWIGLU_SPLIT) {
#pragma unroll
      for (int j = 0; j < 8; j += 2) {
        int n = n0 + tx * 4 + (j & 3) + (j >> 2) * 64;
        if (n + 1 < N) epi_store_pair(ep, m, n, acc[i][j], acc[i][j + 1]);
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        int n = n0 + tx * 4 + (j & 3) + (j >> 2) * 64;
        if (n < N) epi_store1(ep, m, n, acc[i][j]);
      }
    }
  }
}

int gemm_simt_launch(const void* a_hi, const void* a_lo, int lda, const void* b_hi, const void* b_lo,
                     int ldb, int M, int N, int K, const EpiParams& ep, bool f16, cudaStream_t st) {
  ANYLOC_REQUIRE(K % 4 == 0 && lda % 4 == 0 && ldb % 4 == 0, "gemm_simt: K/lda/ldb must be multiples of 4");
  // load4 reads 4 elements at once: 16-byte (fp32) / 8-byte (fp16) aligned operands
  const uintptr_t amask = f16 ? 7 : 15;
  auto aligned = [&](const void* p) { return (reinterpret_cast<uintptr_t>(p) & amask) == 0; };
  ANYLOC_REQUIRE(aligned(a_hi) && aligned(a_lo) && aligned(b_hi) && aligned(b_lo),
                 "gemm_simt: operands must be %d-byte aligned", (int)amask + 1);
  dim3 grid(cdiv(N, BN), cdiv(M, BM));
  if (f16)
    gemm_simt_kernel<__half><<<grid, 256, 0, st>>>((const __half*)a_hi, (const __half*)a_lo, lda, (const __half*)b_hi,
                                                   (const __half*)b_lo, ldb, M, N, K, ep);
  else
    gemm_simt_kernel<float><<<grid, 256, 0, st>>>((const float*)a_hi, (const float*)a_lo, lda, (const float*)b_hi,
                                                  (const float*)b_lo, ldb, M, N, K, ep);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}

}  // namespace anyloc
