// Streamed PCA fit of reduce_pca (utilities.py:522-586) for rows that do not fit on the device: the fp64 column sums
// of the mean pass and the centred A^T.B products of the Gram / covariance matrix and of vt, accumulated piece by
// piece into caller-owned fp64 outputs; and the two products of the randomized fit's power iterations, (X - mu).W
// (sketch) and W^T.(X - mu) (vt).  The rows arrive as fp32 and are centred in fp64 registers on the way to
// shared memory; no centred or fp64 copy of them is ever written.  The products run on the FP64 tensor cores
// (mma.sync m16n8k4 .f64, DMMA: wgmma has no fp64 shape).
#include <algorithm>
#include <type_traits>
#include "common.cuh"

namespace anyloc {

namespace {

constexpr int PCA_BM = 64, PCA_BK = 16, PCA_THREADS = 128;
constexpr int PCA_LDS = PCA_BM + 4;     // 68 doubles: the 4 k-rows a fragment load touches fall in distinct banks
constexpr int COLSUM_THREADS = 256, COLSUM_MAX_CHUNKS = 32, COLSUM_MIN_ROWS = 64;

__device__ __forceinline__ void dmma_16x8x4(double (&c)[4], double a0, double a1, double b0) {
  asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
               : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
               : "d"(a0), "d"(a1), "d"(b0));
}

// The k-tiles [PCA_BK x PCA_BM] of one operand, op(kk, i) for kk in [k0, k0+BK), i in [i0, i0+BM), 8 values per
// thread, zero outside [0, K) x [0, M).  MN-major (contracting over rows): op(kk, i) = x[kk*ld + i] - mu[i], a warp
// reads 32 consecutive columns of one row.  K-major (contracting over columns): op(kk, i) = x[i*ld + kk] - mu[kk], a
// warp reads 16 consecutive columns of two rows.  mu == nullptr: x is taken as it is (the fp64 u operand).
template <bool KMAJOR, typename T>
struct TileLoader {
  using Elem = T;
  const T* p;           // this thread's element 0 of k-tile 0
  int64_t ld;
  const double* mu;
  double m;             // MN-major: the centre of this thread's column, the same in every k-tile
  int koff;             // this thread's first kk within a k-tile
  unsigned ok;          // bit e: element e's row / column lies inside [0, M)

  __device__ __forceinline__ TileLoader(const T* x, int64_t ld_, const double* mu_, int64_t i0, int64_t M)
      : ld(ld_), mu(mu_), m(0.0), ok(0) {
    const int t = threadIdx.x;
    if (!KMAJOR) {
      const int64_t i = i0 + (t & 63);
      koff = t >> 6;
      p = x + (int64_t)koff * ld + (i < M ? i : 0);
      if (i < M) {
        ok = 0xffu;
        if (mu) m = mu[i];
      }
    } else {
      koff = t & 15;
      const int64_t i = i0 + (t >> 4);
      p = x + (i < M ? i : 0) * ld + koff;
#pragma unroll
      for (int e = 0; e < 8; ++e) ok |= (i + 8 * e < M) ? 1u << e : 0u;
    }
  }
  __device__ __forceinline__ void load(double (&v)[8], int64_t k0, int64_t K) const {
    const int64_t rem = K - k0 - koff;       // elements at kk offsets < rem lie inside [0, K)
    if (!KMAJOR) {
      const T* q = p + k0 * ld;
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = ((ok >> e & 1u) && 2 * e < rem) ? (double)q[2 * e * ld] - m : 0.0;
    } else {
      const T* q = p + k0;
      const double c = (rem > 0 && mu) ? mu[k0 + koff] : 0.0;
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = ((ok >> e & 1u) && rem > 0) ? (double)q[8 * e * ld] - c : 0.0;
    }
  }
};

template <bool KMAJOR>
__device__ __forceinline__ void store_tile(double (*s)[PCA_LDS], const double (&v)[8]) {
  const int t = threadIdx.x;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    if (!KMAJOR) s[(t >> 6) + 2 * e][t & 63] = v[e];
    else s[t & 15][(t >> 4) + 8 * e] = v[e];
  }
}

// out[i, j] += sum_kk A(kk, i) B(kk, j) over one 64x64 output tile per CTA, kk in [0, K) in ascending k-tiles, so a
// given call sums every element in the same order on every run.  Four warps of 32x32, each 2 x 4 m16n8k4 DMMAs per
// k-step.  Only elements inside [0, M) x [0, N) are read or written.
//   ANYLOC_PCA_COV : A = B = x - mu (MN-major, rows [K, M]);  lower-triangle tiles only (out [M, M]).
//   ANYLOC_PCA_GRAM: A = B = (x - mu)^T (K-major, x [M, K]);  lower-triangle tiles only (out [M, M]).
//   ANYLOC_PCA_VT  : A = u (fp64 [K, M], not centred), B = x - mu (x [K, N]); every tile (out [M, N]).
//   ANYLOC_PCA_SKETCH: A = (x - mu)^T (K-major, x [M, K]), B = u (fp64 [K, N], not centred); every tile (out [M, N]).
template <int MODE>
__global__ void __launch_bounds__(PCA_THREADS) pca_atb_kernel(const float* __restrict__ x, int64_t ldx,
                                                              const double* __restrict__ mu,
                                                              const double* __restrict__ u, int64_t ldu, int64_t K,
                                                              int M, int N, double* __restrict__ out, int64_t ldo) {
  constexpr bool TRI = MODE == ANYLOC_PCA_COV || MODE == ANYLOC_PCA_GRAM;
  constexpr bool A_KMAJOR = MODE == ANYLOC_PCA_GRAM || MODE == ANYLOC_PCA_SKETCH;
  constexpr bool B_KMAJOR = MODE == ANYLOC_PCA_GRAM;
  __shared__ double As[PCA_BK][PCA_LDS];
  __shared__ double Bs[PCA_BK][PCA_LDS];

  int64_t tm, tn;
  if (TRI) {        // blockIdx.x -> (tm, tn), tn <= tm, row by row
    const int64_t b = blockIdx.x;
    tm = (int64_t)((sqrt(8.0 * (double)b + 1.0) - 1.0) * 0.5);
    while (tm * (tm + 1) / 2 > b) --tm;
    while ((tm + 1) * (tm + 2) / 2 <= b) ++tm;
    tn = b - tm * (tm + 1) / 2;
  } else {
    tm = blockIdx.y;
    tn = blockIdx.x;
  }
  const int64_t m0 = tm * PCA_BM, n0 = tn * PCA_BM;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tg = lane & 3;
  const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;

  double acc[2][4][4];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[a][b][c] = 0.0;

  using ALoader = TileLoader<A_KMAJOR, typename std::conditional<MODE == ANYLOC_PCA_VT, double, float>::type>;
  using BLoader = TileLoader<B_KMAJOR, typename std::conditional<MODE == ANYLOC_PCA_SKETCH, double, float>::type>;
  const ALoader la = MODE == ANYLOC_PCA_VT ? ALoader((const typename ALoader::Elem*)u, ldu, nullptr, m0, M)
                                           : ALoader((const typename ALoader::Elem*)x, ldx, mu, m0, M);
  const BLoader lb = MODE == ANYLOC_PCA_SKETCH ? BLoader((const typename BLoader::Elem*)u, ldu, nullptr, n0, N)
                                               : BLoader((const typename BLoader::Elem*)x, ldx, mu, n0, N);
  double va[8], vb[8];
  auto load = [&](int64_t k0) {
    la.load(va, k0, K);
    lb.load(vb, k0, K);
  };
  const int64_t nk = (K + PCA_BK - 1) / PCA_BK;
  load(0);
  for (int64_t kt = 0; kt < nk; ++kt) {
    store_tile<A_KMAJOR>(As, va);
    store_tile<B_KMAJOR>(Bs, vb);
    __syncthreads();
    if (kt + 1 < nk) load((kt + 1) * PCA_BK);     // the next tile's global loads fly under this tile's DMMAs
#pragma unroll
    for (int ks = 0; ks < PCA_BK; ks += 4) {
      double a[2][2], b[4];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        a[mi][0] = As[ks + tg][wm + mi * 16 + g];
        a[mi][1] = As[ks + tg][wm + mi * 16 + g + 8];
      }
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) b[ni] = Bs[ks + tg][wn + ni * 8 + g];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) dmma_16x8x4(acc[mi][ni], a[mi][0], a[mi][1], b[ni]);
    }
    __syncthreads();
  }

#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int64_t i = m0 + wm + mi * 16 + g + 8 * (c >> 1), j = n0 + wn + ni * 8 + 2 * tg + (c & 1);
        if (i < M && j < N) out[i * ldo + j] += acc[mi][ni][c];
      }
}

// part[chunk, c] = sum of x[r, c] over the chunk's rows, in row order
__global__ void __launch_bounds__(COLSUM_THREADS) pca_colsum_kernel(const float* __restrict__ x, int64_t ld,
                                                                    int64_t rows, int cols, int64_t rows_per,
                                                                    double* __restrict__ part) {
  const int c = blockIdx.x * COLSUM_THREADS + threadIdx.x;
  if (c >= cols) return;
  const int64_t r0 = blockIdx.y * rows_per, r1 = min(rows, r0 + rows_per);
  double s = 0.0;
#pragma unroll 8
  for (int64_t r = r0; r < r1; ++r) s += (double)x[r * ld + c];
  part[(int64_t)blockIdx.y * cols + c] = s;
}

// sum[c] += the chunks' partial sums, in chunk order
__global__ void __launch_bounds__(COLSUM_THREADS) pca_colsum_finish_kernel(const double* __restrict__ part,
                                                                           int chunks, int cols,
                                                                           double* __restrict__ sum) {
  const int c = blockIdx.x * COLSUM_THREADS + threadIdx.x;
  if (c >= cols) return;
  double s = 0.0;
  for (int k = 0; k < chunks; ++k) s += part[(int64_t)k * cols + c];
  sum[c] += s;
}

// a[i, j] = a[j, i] for j > i: the strict upper triangle from the lower one, through a 32x32 shared-memory tile
__global__ void __launch_bounds__(256) pca_mirror_kernel(double* __restrict__ a, int m, int64_t lda) {
  __shared__ double t[32][33];
  const int ti = blockIdx.y, tj = blockIdx.x;     // destination tile (ti, tj), tj >= ti
  if (tj < ti) return;
  for (int r = threadIdx.y; r < 32; r += 8) {     // source tile (tj, ti): rows tj*32+r, columns ti*32+x
    const int64_t i = (int64_t)tj * 32 + r, j = (int64_t)ti * 32 + threadIdx.x;
    if (i < m && j < m) t[r][threadIdx.x] = a[i * lda + j];
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int64_t i = (int64_t)ti * 32 + r, j = (int64_t)tj * 32 + threadIdx.x;
    if (i < m && j < m && j > i) a[i * lda + j] = t[threadIdx.x][r];
  }
}

int colsum_chunks(int64_t rows) {
  const int64_t c = (rows + COLSUM_MIN_ROWS - 1) / COLSUM_MIN_ROWS;
  return (int)std::min<int64_t>(std::max<int64_t>(c, 1), COLSUM_MAX_CHUNKS);
}

}  // namespace

size_t pca_colsum_workspace_bytes(int64_t rows, int cols) {
  return (size_t)colsum_chunks(rows) * (size_t)std::max(cols, 0) * sizeof(double);
}

int pca_colsum_launch(const float* x, int64_t ld, int64_t rows, int cols, double* sum, double* part,
                      cudaStream_t st) {
  if (rows == 0 || cols == 0) return ANYLOC_OK;
  const int chunks = colsum_chunks(rows);
  const int64_t rows_per = (rows + chunks - 1) / chunks;
  const dim3 grid(cdiv(cols, COLSUM_THREADS), chunks);
  pca_colsum_kernel<<<grid, COLSUM_THREADS, 0, st>>>(x, ld, rows, cols, rows_per, part);
  ANYLOC_CHECK_LAUNCH();
  pca_colsum_finish_kernel<<<cdiv(cols, COLSUM_THREADS), COLSUM_THREADS, 0, st>>>(part, chunks, cols, sum);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}

int pca_atb_launch(int mode, const float* x, int64_t ldx, const double* mu, const double* u, int64_t ldu, int64_t K,
                   int M, int N, double* out, int64_t ldo, cudaStream_t st) {
  if (M == 0 || N == 0) return ANYLOC_OK;
  const int64_t tm = (M + PCA_BM - 1) / PCA_BM, tn = (N + PCA_BM - 1) / PCA_BM;
  if (mode == ANYLOC_PCA_VT) {
    pca_atb_kernel<ANYLOC_PCA_VT><<<dim3((unsigned)tn, (unsigned)tm), PCA_THREADS, 0, st>>>(x, ldx, mu, u, ldu, K, M,
                                                                                           N, out, ldo);
  } else if (mode == ANYLOC_PCA_SKETCH) {
    pca_atb_kernel<ANYLOC_PCA_SKETCH><<<dim3((unsigned)tn, (unsigned)tm), PCA_THREADS, 0, st>>>(x, ldx, mu, u, ldu, K,
                                                                                               M, N, out, ldo);
  } else {
    const unsigned tiles = (unsigned)(tm * (tm + 1) / 2);
    if (mode == ANYLOC_PCA_COV)
      pca_atb_kernel<ANYLOC_PCA_COV><<<tiles, PCA_THREADS, 0, st>>>(x, ldx, mu, u, ldu, K, M, N, out, ldo);
    else
      pca_atb_kernel<ANYLOC_PCA_GRAM><<<tiles, PCA_THREADS, 0, st>>>(x, ldx, mu, u, ldu, K, M, N, out, ldo);
  }
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}

int pca_mirror_launch(double* a, int m, int64_t lda, cudaStream_t st) {
  if (m == 0) return ANYLOC_OK;
  const int t = cdiv(m, 32);
  pca_mirror_kernel<<<dim3(t, t), dim3(32, 8), 0, st>>>(a, m, lda);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}

}  // namespace anyloc
