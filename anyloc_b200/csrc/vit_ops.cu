// Element-wise / row-wise pieces of the DINOv2 forward (upstream dinov2 DinoVisionTransformer,
// reached from /root/reference/utilities.py:269): im2col for the 14x14/s14 patch embedding,
// token assembly (+cls, +pos-embed), LayerNorm (eps 1e-6) fused with the tf32 (hi,lo) split
// that feeds the tensor-core GEMMs, the facet slice + F.normalize epilogue of
// DinoV2ExtractFeatures.__call__ (utilities.py:270-283), and the qkv tap that keeps the q/k/v facets of a layer the
// forward continues through.
#include "common.cuh"

namespace anyloc {

__global__ void split_tf32_kernel(const float* __restrict__ x, float* __restrict__ hi,
                                  float* __restrict__ lo, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) { float h, l; split_tf32(x[i], h, l); hi[i] = h; lo[i] = l; }
}

// x -> fp16 pair of scale*x
__global__ void split_f16_kernel(const float* __restrict__ x, __half* __restrict__ hi, __half* __restrict__ lo,
                                 size_t n, float scale) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) { __half h, l; split_f16(x[i] * scale, h, l); hi[i] = h; lo[i] = l; }
}

template <bool F16> struct PairOut;
template <> struct PairOut<false> {
  typedef float T;
  static __device__ __forceinline__ void put(float* hi, float* lo, size_t i, float v) { float h, l; split_tf32(v, h, l); hi[i] = h; lo[i] = l; }
};
template <> struct PairOut<true> {
  typedef __half T;
  static __device__ __forceinline__ void put(__half* hi, __half* lo, size_t i, float v) { __half h, l; split_f16(v * kActScale, h, l); hi[i] = h; lo[i] = l; }
};

// patch pi of image b of img [B,3,H,W] -> patch row `row` of (hi,lo), column order (c, ky, kx) like conv
// weight.flatten(1)
template <bool F16>
__device__ __forceinline__ void im2col_row(const float* __restrict__ img, int b, int H, int W, int P, int Kp, size_t row,
                                           int pi, typename PairOut<F16>::T* __restrict__ hi,
                                           typename PairOut<F16>::T* __restrict__ lo) {
  const int gw = W / P;
  const int py = pi / gw, px = pi % gw;
  const int Kreal = 3 * P * P;
  for (int c = threadIdx.x; c < Kp; c += blockDim.x) {
    float v = 0.f;
    if (c < Kreal) {
      int ch = c / (P * P), rem = c % (P * P), ky = rem / P, kx = rem % P;
      v = __ldg(img + (((size_t)b * 3 + ch) * H + (py * P + ky)) * W + (px * P + kx));
    }
    PairOut<F16>::put(hi, lo, row * Kp + c, v);
  }
}

// img [B,3,H,W] -> patches (hi,lo) [B*gh*gw, Kp]
template <bool F16>
__global__ void im2col_split_kernel(const float* __restrict__ img, int B, int H, int W, int P, int Kp,
                                    typename PairOut<F16>::T* __restrict__ hi, typename PairOut<F16>::T* __restrict__ lo) {
  const int gh = H / P, gw = W / P;
  const size_t row = blockIdx.x;               // patch index
  const int b = (int)(row / (gh * gw)), pi = (int)(row % (gh * gw));
  im2col_row<F16>(img, b, H, W, P, Kp, row, pi, hi, lo);
}

// images of different sizes, one block per patch row of the packed [sum gh_i*gw_i, Kp] output
template <bool F16>
__global__ void im2col_split_varlen_kernel(const __grid_constant__ VarlenImgTable tab, int P, int Kp,
                                           typename PairOut<F16>::T* __restrict__ hi,
                                           typename PairOut<F16>::T* __restrict__ lo) {
  const int skip = 1 + tab.nreg, row = blockIdx.x, i = varlen_image_of(tab, row, skip);
  im2col_row<F16>(tab.ptr[i], 0, tab.gh[i] * P, tab.gw[i] * P, P, Kp, row, row - (tab.tok0[i] - skip * i), hi, lo);
}

// x[row,:] = cls + pos[0] (t = 0), reg[t-1] (1 <= t <= R: no positional embedding) or patch[b*N + p,:] + pos[1+p]
// (t = 1 + R + p)     (prepare_tokens)
__device__ __forceinline__ void assemble_row(const float* __restrict__ patch, const float* __restrict__ cls,
                                             const float* __restrict__ reg, const float* __restrict__ pos, int b, int N,
                                             int R, int D, size_t row, int t, float* __restrict__ x) {
  if (t >= 1 && t <= R) {
    const float* r = reg + (size_t)(t - 1) * D;
    for (int d = threadIdx.x; d < D; d += blockDim.x) x[row * D + d] = r[d];
    return;
  }
  const int tp = t == 0 ? 0 : t - R;     // the token's row of the positional table
  const float* src = tp == 0 ? cls : patch + ((size_t)b * N + (tp - 1)) * D;
  const float* pe = pos + (size_t)tp * D;
  for (int d = threadIdx.x; d < D; d += blockDim.x) x[row * D + d] = src[d] + pe[d];
}

__global__ void assemble_tokens_kernel(const float* __restrict__ patch, const float* __restrict__ cls,
                                       const float* __restrict__ reg, const float* __restrict__ pos, int B, int N,
                                       int R, int D, float* __restrict__ x) {
  const size_t row = blockIdx.x;     // over B*T, T = 1 + R + N
  const int T = N + 1 + R;
  const int b = (int)(row / T), t = (int)(row % T);
  assemble_row(patch, cls, reg, pos, b, N, R, D, row, t, x);
}

// images of different sizes, one block per token row of the packed sequence; image i reads its own positional table
__global__ void assemble_tokens_varlen_kernel(const float* __restrict__ patch, const float* __restrict__ cls,
                                              const float* __restrict__ reg, const __grid_constant__ VarlenImgTable tab,
                                              int D, float* __restrict__ x) {
  const int row = blockIdx.x, i = varlen_image_of(tab, row, 0);
  assemble_row(patch + (size_t)(tab.tok0[i] - (1 + tab.nreg) * i) * D, cls, reg, tab.ptr[i], 0, 0, tab.nreg, D, row,
               row - tab.tok0[i], x);
}

// LayerNorm over the last dim (biased variance, eps inside sqrt) -> (hi,lo). One warp per row.
template <int MAXV, bool F16>   // float4 per lane
__global__ void __launch_bounds__(256)
layernorm_split_kernel(const float* __restrict__ x, const float* __restrict__ w,
                       const float* __restrict__ b, int M, int D, float eps,
                       typename PairOut<F16>::T* __restrict__ y_hi, typename PairOut<F16>::T* __restrict__ y_lo) {
  const int lane = threadIdx.x & 31;
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= M) return;
  const int D4 = D >> 2;
  const float4* xr = reinterpret_cast<const float4*>(x + (size_t)row * D);
  float4 v[MAXV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    int d = lane + i * 32;
    if (d < D4) { v[i] = xr[d]; s += (v[i].x + v[i].y) + (v[i].z + v[i].w); }
  }
  const float mean = warp_sum(s) / (float)D;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    int d = lane + i * 32;
    if (d < D4) {
      float a = v[i].x - mean, bb = v[i].y - mean, c = v[i].z - mean, e = v[i].w - mean;
      q += (a * a + bb * bb) + (c * c + e * e);
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / (float)D + eps);
  const float4* w4 = reinterpret_cast<const float4*>(w);
  const float4* b4 = reinterpret_cast<const float4*>(b);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    int d = lane + i * 32;
    if (d < D4) {
      float4 ww = __ldg(w4 + d), bb = __ldg(b4 + d);
      const float y0 = (v[i].x - mean) * rstd * ww.x + bb.x, y1 = (v[i].y - mean) * rstd * ww.y + bb.y;
      const float y2 = (v[i].z - mean) * rstd * ww.z + bb.z, y3 = (v[i].w - mean) * rstd * ww.w + bb.w;
      if constexpr (F16) {
        uint2 h, l;
        split_f16x2(y0 * kActScale, y1 * kActScale, h.x, l.x);
        split_f16x2(y2 * kActScale, y3 * kActScale, h.y, l.y);
        reinterpret_cast<uint2*>(y_hi + (size_t)row * D)[d] = h;
        reinterpret_cast<uint2*>(y_lo + (size_t)row * D)[d] = l;
      } else {
        float4 h, l;
        split_tf32(y0, h.x, l.x); split_tf32(y1, h.y, l.y); split_tf32(y2, h.z, l.z); split_tf32(y3, h.w, l.w);
        reinterpret_cast<float4*>(y_hi + (size_t)row * D)[d] = h;
        reinterpret_cast<float4*>(y_lo + (size_t)row * D)[d] = l;
      }
    }
  }
}

// y[r,:] = x[r, 0:D] / max(|x[r]|,1e-12) (or plain copy), x rows strided by ld_in. One warp per row.
__global__ void __launch_bounds__(256)
l2norm_rows_kernel(const float* __restrict__ x, int64_t rows, int D, int64_t ld_in, int do_norm,
                   float* __restrict__ y) {
  const int lane = threadIdx.x & 31;
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= rows) return;
  const float4* xr = reinterpret_cast<const float4*>(x + row * ld_in);
  float4* yr = reinterpret_cast<float4*>(y + row * D);
  const int D4 = D >> 2;
  float ss = 0.f;
  for (int d = lane; d < D4; d += 32) { float4 v = xr[d]; ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w; }
  const float nrm = fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
  for (int d = lane; d < D4; d += 32) {
    float4 v = xr[d];
    if (do_norm) { v.x /= nrm; v.y /= nrm; v.z /= nrm; v.w /= nrm; }
    yr[d] = v;
  }
}

// the arithmetic of the facet slice's F.normalize, shared by facet_row and the qkv tap: each lane sums the squares
// of its float4s d = lane, lane + 32, ... in that order, then every element is divided by max(|x|, 1e-12)
__device__ __forceinline__ float sumsq_add(float ss, float4 v) { return ss + (v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w); }
__device__ __forceinline__ float4 div4(float4 v, float nrm) { v.x /= nrm; v.y /= nrm; v.z /= nrm; v.w /= nrm; return v; }

// one token row -> one output row (normalised if do_norm), one warp
__device__ __forceinline__ void facet_row(int lane, const float* __restrict__ x, int D, int do_norm,
                                          float* __restrict__ y) {
  const float4* xr = reinterpret_cast<const float4*>(x);
  float4* yr = reinterpret_cast<float4*>(y);
  const int D4 = D >> 2;
  float ss = 0.f;
  for (int d = lane; d < D4; d += 32) ss = sumsq_add(ss, xr[d]);
  const float nrm = fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
  for (int d = lane; d < D4; d += 32) {
    float4 v = xr[d];
    if (do_norm) v = div4(v, nrm);
    yr[d] = v;
  }
}

// One fp32 row [q | k | v] of a tapped layer's qkv GEMM (3D columns, one warp, each element read once) -> the
// attention's operand pairs of the row, in the format the qkv GEMM's split epilogue writes (pair: 0 none, 1 tf32
// pairs, 2 fp16 pairs of kActScale*x; epi_store_split's split), and the rows of the requested facets (out[f] != null),
// through facet_row's arithmetic.
template <int MAXV>     // float4 per lane and third: D <= 128 * MAXV
__device__ __forceinline__ void qkv_tap_row(int lane, const float* __restrict__ src, int D, int pair, void* hi,
                                            void* lo, const QkvTapOuts& o, int64_t orow, int do_norm) {
  const int D4 = D >> 2;
#pragma unroll 1
  for (int f = 0; f < 3; ++f) {
    const float4* xr = reinterpret_cast<const float4*>(src + (size_t)f * D);
    float4 v[MAXV];
#pragma unroll
    for (int i = 0; i < MAXV; ++i)
      if (lane + i * 32 < D4) v[i] = xr[lane + i * 32];
    if (pair == 2) {
      uint2* h2 = reinterpret_cast<uint2*>(reinterpret_cast<__half*>(hi) + (size_t)f * D);
      uint2* l2 = reinterpret_cast<uint2*>(reinterpret_cast<__half*>(lo) + (size_t)f * D);
#pragma unroll
      for (int i = 0; i < MAXV; ++i) {
        const int d = lane + i * 32;
        if (d < D4) {
          uint2 h, l;
          split_f16x2(v[i].x * kActScale, v[i].y * kActScale, h.x, l.x);
          split_f16x2(v[i].z * kActScale, v[i].w * kActScale, h.y, l.y);
          h2[d] = h; l2[d] = l;
        }
      }
    } else if (pair == 1) {
      float4* h4 = reinterpret_cast<float4*>(reinterpret_cast<float*>(hi) + (size_t)f * D);
      float4* l4 = reinterpret_cast<float4*>(reinterpret_cast<float*>(lo) + (size_t)f * D);
#pragma unroll
      for (int i = 0; i < MAXV; ++i) {
        const int d = lane + i * 32;
        if (d < D4) {
          float4 h, l;
          split_tf32(v[i].x, h.x, l.x); split_tf32(v[i].y, h.y, l.y); split_tf32(v[i].z, h.z, l.z); split_tf32(v[i].w, h.w, l.w);
          h4[d] = h; l4[d] = l;
        }
      }
    }
    float* out = f == 0 ? o.out[0] : f == 1 ? o.out[1] : o.out[2];     // (not o.out[f]: no local-memory copy)
    if (out == nullptr || orow < 0) continue;
    float4* yr = reinterpret_cast<float4*>(out + orow * D);
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i)
      if (lane + i * 32 < D4) ss = sumsq_add(ss, v[i]);
    const float nrm = fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
#pragma unroll
    for (int i = 0; i < MAXV; ++i)
      if (lane + i * 32 < D4) yr[lane + i * 32] = do_norm ? div4(v[i], nrm) : v[i];
  }
}

// B images of T tokens: token row r -> output row r (use_cls) or r - b - 1 (its cls row has none)
template <int MAXV>
__global__ void __launch_bounds__(256)
qkv_tap_kernel(const float* __restrict__ src, int M, int T, int D, int pair, void* hi, void* lo, const QkvTapOuts o,
               int use_cls, int do_norm) {
  const int lane = threadIdx.x & 31;
  const int row = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (row >= M) return;
  const int b = row / T, t = row - b * T;
  const int64_t orow = use_cls ? row : (t == 0 ? -1 : row - b - 1);
  const size_t e = (size_t)row * 3 * D * (pair == 2 ? 2 : 4);     // byte offset of the row's pairs
  qkv_tap_row<MAXV>(lane, src + (size_t)row * 3 * D, D, pair, pair ? (char*)hi + e : nullptr,
                    pair ? (char*)lo + e : nullptr, o, orow, do_norm);
}

// images of different sizes packed row after row: image i's tokens from tab.tok0[i]
template <int MAXV>
__global__ void __launch_bounds__(256)
qkv_tap_varlen_kernel(const float* __restrict__ src, const __grid_constant__ VarlenImgTable tab, int M, int D, int pair,
                      void* hi, void* lo, const QkvTapOuts o, int use_cls, int do_norm) {
  const int lane = threadIdx.x & 31;
  const int row = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (row >= M) return;
  const int i = varlen_image_of(tab, row, 0);
  const int64_t orow = use_cls ? row : (row == tab.tok0[i] ? -1 : row - i - 1);
  const size_t e = (size_t)row * 3 * D * (pair == 2 ? 2 : 4);
  qkv_tap_row<MAXV>(lane, src + (size_t)row * 3 * D, D, pair, pair ? (char*)hi + e : nullptr,
                    pair ? (char*)lo + e : nullptr, o, orow, do_norm);
}

// gather token rows [B, T, ld] (skipping cls unless use_cls, column offset col0) -> [B, T', D] then normalise
__global__ void __launch_bounds__(256)
facet_out_kernel(const float* __restrict__ src, int B, int T, int64_t ld, int col0, int D, int use_cls,
                 int do_norm, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int Tout = use_cls ? T : T - 1;
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= (int64_t)B * Tout) return;
  const int b = (int)(row / Tout), t = (int)(row % Tout) + (use_cls ? 0 : 1);
  facet_row(lane, src + ((int64_t)b * T + t) * ld + col0, D, do_norm, out + row * D);
}

// images of different sizes packed row after row: `rows` output rows, image i's from tok0[i] (- i without cls)
__global__ void __launch_bounds__(256)
facet_out_varlen_kernel(const float* __restrict__ src, const __grid_constant__ VarlenImgTable tab, int rows, int64_t ld,
                        int col0, int D, int use_cls, int do_norm, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int row = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (row >= rows) return;
  const int skip = use_cls ? 0 : 1, i = varlen_image_of(tab, row, skip);
  const int tok = row + skip * (i + 1);         // the token row: every earlier image and this one skipped their cls
  facet_row(lane, src + (int64_t)tok * ld + col0, D, do_norm, out + (int64_t)row * D);
}

int launch_split(const float* x, float* hi, float* lo, size_t n, cudaStream_t st) {
  int blocks = (int)std::min<size_t>((n + 255) / 256, (size_t)device_sm_count() * 16);
  if (blocks < 1) blocks = 1;
  split_tf32_kernel<<<blocks, 256, 0, st>>>(x, hi, lo, n);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}
int launch_split_f16(const float* x, void* hi, void* lo, size_t n, float scale, cudaStream_t st) {
  int blocks = (int)std::min<size_t>((n + 255) / 256, (size_t)device_sm_count() * 16);
  if (blocks < 1) blocks = 1;
  split_f16_kernel<<<blocks, 256, 0, st>>>(x, (__half*)hi, (__half*)lo, n, scale);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}
int launch_im2col(const float* img, int B, int H, int W, int P, int Kp, void* hi, void* lo, bool f16, cudaStream_t st) {
  if (f16) im2col_split_kernel<true><<<B * (H / P) * (W / P), 128, 0, st>>>(img, B, H, W, P, Kp, (__half*)hi, (__half*)lo);
  else im2col_split_kernel<false><<<B * (H / P) * (W / P), 128, 0, st>>>(img, B, H, W, P, Kp, (float*)hi, (float*)lo);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}
int launch_assemble(const float* patch, const float* cls, const float* reg, const float* pos, int B, int N, int R, int D,
                    float* x, cudaStream_t st) {
  assemble_tokens_kernel<<<B * (N + 1 + R), 256, 0, st>>>(patch, cls, reg, pos, B, N, R, D, x);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}
template <bool F16>
static void ln_launch(const float* x, const float* w, const float* b, int M, int D, float eps, void* y_hi, void* y_lo,
                      cudaStream_t st) {
  typedef typename PairOut<F16>::T T;
  int blocks = cdiv(M, 8);
  if (D <= 512) layernorm_split_kernel<4, F16><<<blocks, 256, 0, st>>>(x, w, b, M, D, eps, (T*)y_hi, (T*)y_lo);
  else if (D <= 1024) layernorm_split_kernel<8, F16><<<blocks, 256, 0, st>>>(x, w, b, M, D, eps, (T*)y_hi, (T*)y_lo);
  else layernorm_split_kernel<16, F16><<<blocks, 256, 0, st>>>(x, w, b, M, D, eps, (T*)y_hi, (T*)y_lo);
}
int launch_layernorm(const float* x, const float* w, const float* b, int M, int D, float eps, void* y_hi,
                     void* y_lo, bool f16, cudaStream_t st) {
  ANYLOC_REQUIRE(D % 4 == 0 && D <= 2048, "layernorm: D=%d unsupported (multiple of 4, <= 2048)", D);
  if (f16) ln_launch<true>(x, w, b, M, D, eps, y_hi, y_lo, st);
  else ln_launch<false>(x, w, b, M, D, eps, y_hi, y_lo, st);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}
int launch_facet_out(const float* src, int B, int T, int64_t ld, int col0, int D, int use_cls, int do_norm,
                     float* out, cudaStream_t st) {
  int64_t rows = (int64_t)B * (use_cls ? T : T - 1);
  facet_out_kernel<<<(int)((rows + 7) / 8), 256, 0, st>>>(src, B, T, ld, col0, D, use_cls, do_norm, out);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}
// packed batches of differently sized images: tab.ptr holds the images (im2col) or the positional tables (assembly)
int launch_im2col_varlen(const VarlenImgTable& tab, int n_patches, int P, int Kp, void* hi, void* lo, bool f16,
                         cudaStream_t st) {
  if (f16) im2col_split_varlen_kernel<true><<<n_patches, 128, 0, st>>>(tab, P, Kp, (__half*)hi, (__half*)lo);
  else im2col_split_varlen_kernel<false><<<n_patches, 128, 0, st>>>(tab, P, Kp, (float*)hi, (float*)lo);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}
int launch_assemble_varlen(const float* patch, const float* cls, const float* reg, const VarlenImgTable& tab,
                           int n_tokens, int D, float* x, cudaStream_t st) {
  assemble_tokens_varlen_kernel<<<n_tokens, 256, 0, st>>>(patch, cls, reg, tab, D, x);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}
int launch_facet_out_varlen(const float* src, const VarlenImgTable& tab, int rows, int64_t ld, int col0, int D,
                            int use_cls, int do_norm, float* out, cudaStream_t st) {
  facet_out_varlen_kernel<<<(rows + 7) / 8, 256, 0, st>>>(src, tab, rows, ld, col0, D, use_cls, do_norm, out);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}
// the fp32 qkv rows [M, 3D] of a tapped layer -> pairs (hi, lo; null: none) and facet rows; tab: packed images, else
// B images of T tokens
template <int MAXV>
static void qkv_tap_launch(const float* src, int M, int T, const VarlenImgTable* tab, int D, int pair, void* hi,
                           void* lo, const QkvTapOuts& o, int use_cls, int do_norm, cudaStream_t st) {
  if (tab) qkv_tap_varlen_kernel<MAXV><<<cdiv(M, 8), 256, 0, st>>>(src, *tab, M, D, pair, hi, lo, o, use_cls, do_norm);
  else qkv_tap_kernel<MAXV><<<cdiv(M, 8), 256, 0, st>>>(src, M, T, D, pair, hi, lo, o, use_cls, do_norm);
}
int launch_qkv_tap(const float* src, int M, int T, const VarlenImgTable* tab, int D, int pair, void* hi, void* lo,
                   const QkvTapOuts& o, int use_cls, int do_norm, cudaStream_t st) {
  ANYLOC_REQUIRE(D % 4 == 0 && D <= 2048, "qkv_tap: D=%d unsupported (multiple of 4, <= 2048)", D);
  if (D <= 512) qkv_tap_launch<4>(src, M, T, tab, D, pair, hi, lo, o, use_cls, do_norm, st);
  else if (D <= 1024) qkv_tap_launch<8>(src, M, T, tab, D, pair, hi, lo, o, use_cls, do_norm, st);
  else qkv_tap_launch<16>(src, M, T, tab, D, pair, hi, lo, o, use_cls, do_norm, st);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}
int launch_l2norm(const float* x, int64_t rows, int D, int64_t ld_in, float* y, cudaStream_t st) {
  l2norm_rows_kernel<<<(int)((rows + 7) / 8), 256, 0, st>>>(x, rows, D, ld_in, 1, y);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}

}  // namespace anyloc
