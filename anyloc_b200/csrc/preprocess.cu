// Image pre-processing on the device (SURVEY 8f rank 2): the reference's `base_transform`
// (dvgl_benchmark/datasets_ws.py:20-23: ToTensor + Normalize(mean, std)) followed by the centre crop to a multiple of
// the patch size (scripts/dino_v2_vlad.py:174-176, demo/anyloc_vlad_generate.py:178-181), fused into one pass:
//   out[b,c,y,x] = ((float)img[b, top+y, left+x, c] / 255 - mean[c]) / std[c]
// Same operation order as torchvision (div, sub, div; IEEE round-to-nearest each) -> bit-identical results.
// HBM-bound: 3 B read + 12 B written per pixel.
#include <algorithm>
#include "common.cuh"

namespace anyloc {

__global__ void __launch_bounds__(256)
preprocess_u8_kernel(const uint8_t* __restrict__ img, int H, int W, int top, int left, int Hc, int Wc,
                     float m0, float m1, float m2, float s0, float s1, float s2, float* __restrict__ out) {
  // grid (ceil(Wc/2 / 256), Hc, B); a thread converts two neighbouring pixels and writes one float2 per plane
  const int x = (blockIdx.x * blockDim.x + threadIdx.x) * 2;
  const int y = blockIdx.y, b = blockIdx.z;
  if (x >= Wc) return;
  const uint8_t* src = img + (((size_t)b * H + top + y) * W + left + x) * 3;
  const bool two = x + 1 < Wc;
  float p[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) p[i] = (i < 3 || two) ? __fdiv_rn((float)__ldg(src + i), 255.0f) : 0.f;
  const float mean[3] = {m0, m1, m2}, sd[3] = {s0, s1, s2};
  const size_t plane = (size_t)Hc * Wc;
  float* dst = out + (size_t)b * 3 * plane + (size_t)y * Wc + x;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float a = __fdiv_rn(__fsub_rn(p[c], mean[c]), sd[c]);
    float bb = __fdiv_rn(__fsub_rn(p[3 + c], mean[c]), sd[c]);
    if (two && ((Wc & 1) == 0)) *reinterpret_cast<float2*>(dst + c * plane) = make_float2(a, bb);
    else { dst[c * plane] = a; if (two) dst[c * plane + 1] = bb; }
  }
}


// ToTensor + Normalize + ANTIALIASED resize + centre crop in one pass (dvgl_benchmark/datasets_ws.py:222-239:
// `T.functional.resize(base_transform(img), [480, 640])`, bilinear; demo/anyloc_vlad_generate.py:165-177:
// `T.resize(img_pt, (h, w), InterpolationMode.BICUBIC)` of over-sized images).  On float tensors torchvision's resize is
// torch.nn.functional.interpolate(..., align_corners=False, antialias=True): per output index i,
//   scale = in / out; support = (taps/2) * max(scale, 1); centre = scale * (i + 0.5);
//   first = max(int(centre - support + 0.5), 0); n = min(int(centre + support + 0.5), in) - first;
//   w_j = filter((j + first - centre + 0.5) / max(scale, 1)), normalised to sum 1
// with the triangle filter (bilinear, 2 taps) or Keys' cubic with a = -0.5 (bicubic, 4 taps).  A thread owns one
// output pixel (all 3 channels): horizontal sums per source row, weighted by the vertical filter -- the order of the
// separable ATen CPU kernel (horizontal pass first).  Reads 3 B per tap, writes 12 B per pixel.
__device__ __forceinline__ float aa_filter(float x, int cubic) {
  x = fabsf(x);
  if (!cubic) return x < 1.0f ? 1.0f - x : 0.0f;
  const float a = -0.5f;
  if (x < 1.0f) return ((a + 2.0f) * x - (a + 3.0f)) * x * x + 1.0f;
  if (x < 2.0f) return (((x - 5.0f) * x + 8.0f) * x - 4.0f) * a;
  return 0.0f;
}
struct AaSpan { int first, n; float scale_inv, centre; };
__device__ __forceinline__ AaSpan aa_span(int i, int in_size, int out_size, int cubic) {
  const float scale = (float)in_size / (float)out_size;
  const float support = (cubic ? 2.0f : 1.0f) * (scale >= 1.0f ? scale : 1.0f);
  AaSpan s;
  s.centre = scale * ((float)i + 0.5f);
  s.scale_inv = scale >= 1.0f ? 1.0f / scale : 1.0f;
  s.first = max((int)(s.centre - support + 0.5f), 0);
  s.n = min((int)(s.centre + support + 0.5f), in_size) - s.first;
  return s;
}
constexpr int AA_MAX_TAPS = 64;      // covers down-scaling by up to 16x (bicubic) / 32x (bilinear)

__global__ void __launch_bounds__(128)
preprocess_resize_u8_kernel(const uint8_t* __restrict__ img, int H, int W, int Hr, int Wr, int cubic, int top, int left,
                            int Hc, int Wc, float m0, float m1, float m2, float s0, float s1, float s2,
                            float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, b = blockIdx.z;
  if (x >= Wc) return;
  const AaSpan sx = aa_span(left + x, W, Wr, cubic), sy = aa_span(top + y, H, Hr, cubic);
  float wx[AA_MAX_TAPS];
  float totx = 0.f;
  for (int j = 0; j < sx.n; ++j) { wx[j] = aa_filter(((float)(j + sx.first) - sx.centre + 0.5f) * sx.scale_inv, cubic); totx += wx[j]; }
  for (int j = 0; j < sx.n; ++j) wx[j] /= totx;
  float toty = 0.f;
  for (int j = 0; j < sy.n; ++j) toty += aa_filter(((float)(j + sy.first) - sy.centre + 0.5f) * sy.scale_inv, cubic);
  const float mean[3] = {m0, m1, m2}, sd[3] = {s0, s1, s2};
  float acc[3] = {0.f, 0.f, 0.f};
  for (int jy = 0; jy < sy.n; ++jy) {
    const float wy = aa_filter(((float)(jy + sy.first) - sy.centre + 0.5f) * sy.scale_inv, cubic) / toty;
    const uint8_t* row = img + (((size_t)b * H + sy.first + jy) * W + sx.first) * 3;
    float h[3] = {0.f, 0.f, 0.f};
    for (int jx = 0; jx < sx.n; ++jx) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float v = __fdiv_rn(__fsub_rn(__fdiv_rn((float)__ldg(row + jx * 3 + c), 255.0f), mean[c]), sd[c]);
        h[c] = fmaf(wx[jx], v, h[c]);
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) acc[c] = fmaf(wy, h[c], acc[c]);
  }
  const size_t plane = (size_t)Hc * Wc;
  float* dst = out + (size_t)b * 3 * plane + (size_t)y * Wc + x;
#pragma unroll
  for (int c = 0; c < 3; ++c) dst[c * plane] = acc[c];
}

// ---------------------------------------------------------------- a list of differently sized images in one launch
// Per-image geometry, passed by value as a __grid_constant__ parameter (no host sync, no host pointer kept; the
// pattern of VarlenImgTable).  Image i's output [3, Hc, Wc] starts at out + off[i]; its output tiles are
// [tile0[i], tile0[i+1]) of the flat grid (tile0[n] = the grid size).
constexpr int kPreN = ANYLOC_PREPROCESS_VARLEN_BATCH;
constexpr int PRE_TW = 32, PRE_TH = 8;               // output tile: 32 columns x 8 rows, one pixel per thread
struct PreVarlenTable {
  int n, cubic;
  float mean[3], sd[3];
  const uint8_t* src[kPreN];
  long long off[kPreN];
  int H[kPreN], W[kPreN], Hr[kPreN], Wr[kPreN], top[kPreN], left[kPreN], Hc[kPreN], Wc[kPreN];
  int tile0[kPreN + 1];
};
static_assert(sizeof(PreVarlenTable) <= 4096, "kernel parameter over 4 KB");

struct PreTile { int img, x0, y0; };
// the last image whose first tile is <= blockIdx.x, and the tile's first output column / row in it
__device__ __forceinline__ PreTile pre_tile_of(const PreVarlenTable& t) {
  const int b = blockIdx.x;
  int lo = 0, hi = t.n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (t.tile0[mid] <= b) lo = mid; else hi = mid - 1;
  }
  const int k = b - t.tile0[lo], tx = (t.Wc[lo] + PRE_TW - 1) / PRE_TW;
  return {lo, (k % tx) * PRE_TW, (k / tx) * PRE_TH};
}

// The crop-only path: anyloc_preprocess_u8's operations per pixel, so each image is bit-identical to it.
__global__ void __launch_bounds__(PRE_TW * PRE_TH)
preprocess_u8_varlen_kernel(const __grid_constant__ PreVarlenTable t, float* __restrict__ out) {
  const PreTile p = pre_tile_of(t);
  const int i = p.img, x = p.x0 + threadIdx.x % PRE_TW, y = p.y0 + threadIdx.x / PRE_TW;
  const int Hc = t.Hc[i], Wc = t.Wc[i];
  if (x >= Wc || y >= Hc) return;
  const uint8_t* src = t.src[i] + ((size_t)(t.top[i] + y) * t.W[i] + t.left[i] + x) * 3;
  const size_t plane = (size_t)Hc * Wc;
  float* dst = out + t.off[i] + (size_t)y * Wc + x;
#pragma unroll
  for (int c = 0; c < 3; ++c)
    dst[c * plane] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)__ldg(src + c), 255.0f), t.mean[c]), t.sd[c]);
}

// aa_span and the filter argument with every rounding spelled out: the operations, in the order and with the
// roundings, that nvcc gives preprocess_resize_u8_kernel (centre = scale * (i + 0.5) rounded once; the product
// taps * max(scale, 1) is exact, so its fusion into centre +- support there changes nothing).  Written with _rn
// intrinsics so that no FMA contraction in this kernel can differ from that one.
__device__ __forceinline__ AaSpan aa_span_rn(int i, int in_size, int out_size, int cubic) {
  const float scale = __fdiv_rn((float)in_size, (float)out_size);
  const float support = __fmul_rn(cubic ? 2.0f : 1.0f, scale >= 1.0f ? scale : 1.0f);
  AaSpan s;
  s.centre = __fmul_rn(scale, __fadd_rn((float)i, 0.5f));
  s.scale_inv = scale >= 1.0f ? __fdiv_rn(1.0f, scale) : 1.0f;
  s.first = max((int)__fadd_rn(__fsub_rn(s.centre, support), 0.5f), 0);
  s.n = min((int)__fadd_rn(__fadd_rn(s.centre, support), 0.5f), in_size) - s.first;
  return s;
}
__device__ __forceinline__ float aa_weight_rn(int j, const AaSpan& s, int cubic) {
  return aa_filter(__fmul_rn(__fadd_rn(__fsub_rn((float)j, s.centre), 0.5f), s.scale_inv), cubic);
}

// The resize path, tiled and separable.  A CTA owns PRE_TW x PRE_TH output pixels of one image and walks the source
// rows they read in chunks of R rows: (a) normalise each source pixel of the chunk's rows x the tile's source columns
// once into shared memory; (b) form each horizontal sum once per (source row, output column); (c) add each row's sum
// into the output pixels whose vertical window holds it.  Per output pixel these are preprocess_resize_u8_kernel's
// operations in its order -- the same normalisation chain, fmaf over jx ascending with weights wx[jx] / totx, then
// fmaf over jy ascending with weights filter / toty (chunks and rows ascending) -- so the result is bit-identical.
constexpr int PRE_VS_FLOATS = 6144;                  // normalised source chunk, 3 planes: 24 KB
constexpr int PRE_RMAX = 16;                          // source rows per chunk at most
__global__ void __launch_bounds__(PRE_TW * PRE_TH)
preprocess_resize_u8_varlen_kernel(const __grid_constant__ PreVarlenTable t, float* __restrict__ out) {
  __shared__ float wxs[AA_MAX_TAPS][PRE_TW];          // wx[jx] / totx of each output column
  __shared__ int fxs[PRE_TW], nxs[PRE_TW];
  __shared__ float vs[PRE_VS_FLOATS];
  __shared__ float hs[3][PRE_RMAX][PRE_TW];
  const PreTile p = pre_tile_of(t);
  const int i = p.img, cubic = t.cubic;
  const int H = t.H[i], W = t.W[i], Hr = t.Hr[i], Wr = t.Wr[i], Hc = t.Hc[i], Wc = t.Wc[i];
  const int tx = threadIdx.x % PRE_TW, ty = threadIdx.x / PRE_TW;
  const int nx = min(PRE_TW, Wc - p.x0), ny = min(PRE_TH, Hc - p.y0);    // valid columns / rows of the tile
  // source columns [cx0, cx1) and rows [ry0, ry1) the tile reads (first and first + n do not decrease with i)
  const AaSpan sx0 = aa_span_rn(t.left[i] + p.x0, W, Wr, cubic), sx1 = aa_span_rn(t.left[i] + p.x0 + nx - 1, W, Wr, cubic);
  const AaSpan sy0 = aa_span_rn(t.top[i] + p.y0, H, Hr, cubic), sy1 = aa_span_rn(t.top[i] + p.y0 + ny - 1, H, Hr, cubic);
  const int cx0 = sx0.first, ncols = sx1.first + sx1.n - cx0;
  const int ry0 = sy0.first, ry1 = sy1.first + sy1.n;
  if (threadIdx.x < nx) {
    const AaSpan sx = aa_span_rn(t.left[i] + p.x0 + threadIdx.x, W, Wr, cubic);
    float totx = 0.f;
    for (int j = 0; j < sx.n; ++j) {
      const float w = aa_weight_rn(j + sx.first, sx, cubic);
      wxs[j][threadIdx.x] = w;
      totx = __fadd_rn(totx, w);
    }
    for (int j = 0; j < sx.n; ++j) wxs[j][threadIdx.x] = __fdiv_rn(wxs[j][threadIdx.x], totx);
    fxs[threadIdx.x] = sx.first - cx0;
    nxs[threadIdx.x] = sx.n;
  }
  // this thread's output row: its vertical window and weight total
  const bool live = tx < nx && ty < ny;
  const AaSpan sy = aa_span_rn(t.top[i] + p.y0 + min(ty, ny - 1), H, Hr, cubic);
  float toty = 0.f;
  for (int j = 0; j < sy.n; ++j) toty = __fadd_rn(toty, aa_weight_rn(j + sy.first, sy, cubic));
  // >= 1: under the host's tap-window check (taps * max(W / Wr, 1) + 2 <= AA_MAX_TAPS) a column's window spans at most
  // AA_MAX_TAPS columns and 31 columns' first taps at most 31 * 31 + 1 more, so ncols <= 1026
  const int R = min(PRE_RMAX, PRE_VS_FLOATS / (3 * ncols));
  const int plane_vs = R * ncols;
  const uint8_t* img = t.src[i];
  float acc[3] = {0.f, 0.f, 0.f};
  __syncthreads();
  for (int r0 = ry0; r0 < ry1; r0 += R) {
    const int rows = min(R, ry1 - r0);
    // (a) normalised source pixels, planar [c][row][col]
    for (int e = threadIdx.x; e < rows * ncols; e += blockDim.x) {
      const int rr = e / ncols, col = e - rr * ncols;
      const uint8_t* s = img + ((size_t)(r0 + rr) * W + cx0 + col) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c)
        vs[c * plane_vs + e] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)__ldg(s + c), 255.0f), t.mean[c]), t.sd[c]);
    }
    __syncthreads();
    // (b) horizontal sums of each (source row, output column)
    for (int e = threadIdx.x; e < rows * PRE_TW; e += blockDim.x) {
      const int rr = e / PRE_TW, x = e % PRE_TW;
      if (x >= nx) continue;
      const float* v = vs + rr * ncols + fxs[x];
      float h[3] = {0.f, 0.f, 0.f};
      for (int jx = 0; jx < nxs[x]; ++jx) {
        const float w = wxs[jx][x];
#pragma unroll
        for (int c = 0; c < 3; ++c) h[c] = fmaf(w, v[c * plane_vs + jx], h[c]);
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) hs[c][rr][x] = h[c];
    }
    __syncthreads();
    // (c) vertical weights of the chunk's rows inside this output row's window.  The next chunk's (a) writes only vs,
    // and its (b) overwrites hs after the barrier that follows (a).
    if (live) {
      const int ja = max(r0, sy.first), jb = min(r0 + rows, sy.first + sy.n);
      for (int r = ja; r < jb; ++r) {
        const float wy = __fdiv_rn(aa_weight_rn(r, sy, cubic), toty);
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[c] = fmaf(wy, hs[c][r - r0][tx], acc[c]);
      }
    }
  }
  if (!live) return;
  const size_t plane = (size_t)Hc * Wc;
  float* dst = out + t.off[i] + (size_t)(p.y0 + ty) * Wc + p.x0 + tx;
#pragma unroll
  for (int c = 0; c < 3; ++c) dst[c * plane] = acc[c];
}

}  // namespace anyloc

using namespace anyloc;

extern "C" int anyloc_preprocess_u8(const uint8_t* img, int B, int H, int W, int top, int left, int Hc, int Wc,
                                    const float* mean3, const float* std3, float* out, void* stream) {
  ANYLOC_REQUIRE(img && out && mean3 && std3, "preprocess_u8: null pointer");
  ANYLOC_REQUIRE(B >= 0 && H > 0 && W > 0 && Hc > 0 && Wc > 0 && top >= 0 && left >= 0 && top + Hc <= H &&
                     left + Wc <= W,
                 "preprocess_u8: crop [%d+%d, %d+%d] outside the %dx%d image", top, Hc, left, Wc, H, W);
  ANYLOC_REQUIRE(Hc <= 65535 && B <= 65535, "preprocess_u8: Hc=%d / B=%d exceed the grid limits", Hc, B);
  ANYLOC_REQUIRE(std3[0] != 0.f && std3[1] != 0.f && std3[2] != 0.f, "preprocess_u8: zero std");
  // an even Wc keeps every row's pairs at even element offsets, which the kernel stores as float2
  ANYLOC_REQUIRE((reinterpret_cast<uintptr_t>(out) & ((Wc & 1) ? 3 : 7)) == 0,
                 "preprocess_u8: out must be 4-byte aligned, and 8-byte aligned when Wc is even (float2 stores)");
  if (B == 0) return ANYLOC_OK;
  dim3 grid(cdiv(cdiv(Wc, 2), 256), Hc, B);
  preprocess_u8_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(img, H, W, top, left, Hc, Wc, mean3[0], mean3[1], mean3[2],
                                                              std3[0], std3[1], std3[2], out);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}

// interpolation: 0 = bilinear, 1 = bicubic (both antialiased, torchvision's defaults for tensors).  The image is
// resized to Hr x Wr, then the window [top, top+Hc) x [left, left+Wc) of the RESIZED image is written.
extern "C" int anyloc_preprocess_resize_u8(const uint8_t* img, int B, int H, int W, int Hr, int Wr, int interpolation,
                                           int top, int left, int Hc, int Wc, const float* mean3, const float* std3,
                                           float* out, void* stream) {
  ANYLOC_REQUIRE(img && out && mean3 && std3, "preprocess_resize_u8: null pointer");
  ANYLOC_REQUIRE(interpolation == 0 || interpolation == 1, "preprocess_resize_u8: unknown interpolation %d", interpolation);
  ANYLOC_REQUIRE(B >= 0 && H > 0 && W > 0 && Hr > 0 && Wr > 0 && Hc > 0 && Wc > 0 && top >= 0 && left >= 0 &&
                     top + Hc <= Hr && left + Wc <= Wr,
                 "preprocess_resize_u8: crop [%d+%d, %d+%d] outside the resized %dx%d image", top, Hc, left, Wc, Hr, Wr);
  ANYLOC_REQUIRE(Hc <= 65535 && B <= 65535, "preprocess_resize_u8: Hc=%d / B=%d exceed the grid limits", Hc, B);
  ANYLOC_REQUIRE(std3[0] != 0.f && std3[1] != 0.f && std3[2] != 0.f, "preprocess_resize_u8: zero std");
  ANYLOC_REQUIRE((reinterpret_cast<uintptr_t>(out) & 3) == 0, "preprocess_resize_u8: out must be 4-byte aligned");
  const float taps = interpolation ? 4.0f : 2.0f;
  const float sxm = std::max((float)W / Wr, 1.0f), sym = std::max((float)H / Hr, 1.0f);
  ANYLOC_REQUIRE(taps * sxm + 2.0f <= AA_MAX_TAPS && taps * sym + 2.0f <= 1.0e9f,
                 "preprocess_resize_u8: horizontal down-scaling factor %.1f exceeds the %d-tap window", sxm, AA_MAX_TAPS);
  if (B == 0) return ANYLOC_OK;
  dim3 grid(cdiv(Wc, 128), Hc, B);
  preprocess_resize_u8_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(img, H, W, Hr, Wr, interpolation, top, left, Hc, Wc,
                                                                      mean3[0], mean3[1], mean3[2], std3[0], std3[1],
                                                                      std3[2], out);
  ANYLOC_CHECK_LAUNCH();
  return ANYLOC_OK;
}

// A list of n images in ceil(n / ANYLOC_PREPROCESS_VARLEN_BATCH) launches on one stream; every argument of every image
// is checked before the first launch, so a refusal writes nothing.  interpolation -1: no resize (Hr, Wr unused).
extern "C" int anyloc_preprocess_u8_varlen(int n, const uint8_t* const* imgs, const int* H, const int* W, const int* Hr,
                                           const int* Wr, int interpolation, const int* top, const int* left,
                                           const int* Hc, const int* Wc, const float* mean3, const float* std3,
                                           float* out, const int64_t* out_offset, void* stream) {
  const bool resize = interpolation >= 0;
  ANYLOC_REQUIRE(n >= 0, "preprocess_u8_varlen: n=%d", n);
  ANYLOC_REQUIRE(interpolation >= -1 && interpolation <= 1, "preprocess_u8_varlen: unknown interpolation %d",
                 interpolation);
  ANYLOC_REQUIRE(imgs && H && W && top && left && Hc && Wc && mean3 && std3 && out && out_offset &&
                     (!resize || (Hr && Wr)),
                 "preprocess_u8_varlen: null pointer");
  ANYLOC_REQUIRE(std3[0] != 0.f && std3[1] != 0.f && std3[2] != 0.f, "preprocess_u8_varlen: zero std");
  ANYLOC_REQUIRE((reinterpret_cast<uintptr_t>(out) & 3) == 0, "preprocess_u8_varlen: out must be 4-byte aligned");
  for (int i = 0; i < n; ++i) {
    const int hr = resize ? Hr[i] : H[i], wr = resize ? Wr[i] : W[i];
    ANYLOC_REQUIRE(imgs[i], "preprocess_u8_varlen: null pointer (image %d)", i);
    ANYLOC_REQUIRE(H[i] > 0 && W[i] > 0 && hr > 0 && wr > 0 && Hc[i] > 0 && Wc[i] > 0 && top[i] >= 0 && left[i] >= 0 &&
                       top[i] + Hc[i] <= hr && left[i] + Wc[i] <= wr,
                   "preprocess_u8_varlen: image %d: crop [%d+%d, %d+%d] outside the %s%dx%d image", i, top[i], Hc[i],
                   left[i], Wc[i], resize ? "resized " : "", hr, wr);
    ANYLOC_REQUIRE(out_offset[i] >= 0, "preprocess_u8_varlen: image %d: negative output offset", i);
    if (resize) {
      const float taps = interpolation ? 4.0f : 2.0f, sxm = std::max((float)W[i] / wr, 1.0f);
      ANYLOC_REQUIRE(taps * sxm + 2.0f <= AA_MAX_TAPS,
                     "preprocess_u8_varlen: image %d: horizontal down-scaling factor %.1f exceeds the %d-tap window", i,
                     sxm, AA_MAX_TAPS);
    }
  }
  // grid limit per launch: the tiles of kPreN images
  for (int b0 = 0; b0 < n; b0 += kPreN) {
    long long tiles = 0;
    for (int i = b0; i < std::min(n, b0 + kPreN); ++i)
      tiles += (long long)cdiv(Wc[i], PRE_TW) * cdiv(Hc[i], PRE_TH);
    ANYLOC_REQUIRE(tiles <= 0x7fffffffLL, "preprocess_u8_varlen: %lld output tiles in images %d.. exceed the grid limit",
                   tiles, b0);
  }
  for (int b0 = 0; b0 < n; b0 += kPreN) {
    PreVarlenTable t;
    t.n = std::min(n - b0, kPreN);
    t.cubic = interpolation == 1;
    for (int c = 0; c < 3; ++c) t.mean[c] = mean3[c], t.sd[c] = std3[c];
    int tiles = 0;
    for (int k = 0; k < t.n; ++k) {
      const int i = b0 + k;
      t.src[k] = imgs[i];
      t.off[k] = out_offset[i];
      t.H[k] = H[i], t.W[k] = W[i], t.Hr[k] = resize ? Hr[i] : H[i], t.Wr[k] = resize ? Wr[i] : W[i];
      t.top[k] = top[i], t.left[k] = left[i], t.Hc[k] = Hc[i], t.Wc[k] = Wc[i];
      t.tile0[k] = tiles;
      tiles += cdiv(Wc[i], PRE_TW) * cdiv(Hc[i], PRE_TH);
    }
    t.tile0[t.n] = tiles;
    if (resize) preprocess_resize_u8_varlen_kernel<<<tiles, PRE_TW * PRE_TH, 0, (cudaStream_t)stream>>>(t, out);
    else preprocess_u8_varlen_kernel<<<tiles, PRE_TW * PRE_TH, 0, (cudaStream_t)stream>>>(t, out);
    ANYLOC_CHECK_LAUNCH();
  }
  return ANYLOC_OK;
}
