// The ConvNeXt backbone's own kernels (models/convnext.py:45-335, upstream DINOv3's ConvNeXt): everything around the two
// pointwise GEMMs of a block, which run on gemm_tc.cu (pwconv1 with the erf-GELU epilogue, pwconv2 with bias, LayerScale
// and the residual add), and around the stride-2 / stride-4 convolutions, which are GEMMs over patchified pixels.
//   dwconv7_ln_kernel    depthwise 7x7 conv (padding 3, bias) + the block's per-pixel LayerNorm -> bf16 pwconv1 operand
//   ln_patchify2_kernel  a downsampling layer's per-pixel LayerNorm, written into the 2x2 conv's im2col operand
//   pool_tokens_kernel   the pooled "class token" (mean over H x W, fixed summation order) + the token rows
//   resize_bilinear_aa_kernel  antialiased bilinear resize of a stage's map to the ViT patch grid
// The LayerNorms use layernorm.cuh's row statistics and normalisation: every normalised pixel has the bits
// d3_layernorm_fwd gives for that row.
#include "ptx.cuh"
#include "d3_internal.h"
#include "layernorm.cuh"

namespace d3 {

#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

// ------------------------------------------------------------------------------------------------ dwconv 7x7 + LayerNorm
// A CTA owns a TH x 8 tile of output pixels of one image, across all C channels.  Phase 1: a work item is one output
// row of the tile in one channel, items numbered row-major so that a warp's loads are consecutive channels.  The 7 input
// rows under it, 14 values each (zero outside the map), go into registers and are multiplied into the row's 8
// accumulators with the channel's 7 taps of that kernel row.  All 98 loads of an item can be in flight together; the rows neighbouring
// items share come again from L1, the halo re-reads between neighbouring tiles from L2.  The conv outputs (+ bias) go to
// shared memory as fp32 rows of C.  Phase 2: one warp per pixel, ln_row_stats / ln_store_row on the staged row, bf16
// out.  TH is the largest of 8, 4, 2 that keeps the staged rows within DW_SMEM_MAX, halved further (down to 1) while
// the grid would not fill every SM twice (the small maps of the late stages).
constexpr int DW_TW = 8;
constexpr int DW_THREADS_MAX = 256;
constexpr int DW_SMEM_MAX = 96 * 1024;     // two CTAs per SM

// Two CTAs per SM (128 registers a thread), except for the generic-width and the 1536-wide LayerNorm, which need a few
// more registers than that and get them (one CTA per SM) rather than spill.
template <int VPL>
__global__ void __launch_bounds__(DW_THREADS_MAX, VPL == 0 || VPL == 12 ? 1 : 2)
dwconv7_ln_kernel(const float* __restrict__ X, const float* __restrict__ wt, const float* __restrict__ wb,
                  const float* __restrict__ scale, const float* __restrict__ bias, __nv_bfloat16* __restrict__ Y, int H,
                  int W, int C, int TH, int tiles_h, int tiles_w, float eps) {
  extern __shared__ float4 dw_smem[];
  float* const s = reinterpret_cast<float*>(dw_smem);    // [TH * DW_TW][C]
  constexpr int TW = DW_TW;
  const int tw = blockIdx.x % tiles_w, th = (blockIdx.x / tiles_w) % tiles_h, b = blockIdx.x / (tiles_w * tiles_h);
  const int h0 = th * TH, w0 = tw * TW;
  const float* const xb = X + (size_t)b * H * W * C;
  const int rows = min(TH, H - h0);
  for (int item = threadIdx.x; item < rows * C; item += blockDim.x) {
    const int i = item / C, c = item - i * C;
    float acc[TW];
#pragma unroll
    for (int j = 0; j < TW; ++j) acc[j] = 0.f;
#pragma unroll
    for (int kh = 0; kh < 7; ++kh) {
      const int ih = h0 + i + kh - 3;
      const bool row_in = ih >= 0 && ih < H;
      float xin[TW + 6], k[7];
#pragma unroll
      for (int j = 0; j < TW + 6; ++j) {
        const int iw = w0 - 3 + j;
        xin[j] = row_in && iw >= 0 && iw < W ? __ldg(xb + ((size_t)ih * W + iw) * C + c) : 0.f;
      }
#pragma unroll
      for (int kw = 0; kw < 7; ++kw) k[kw] = __ldg(wt + (size_t)(kh * 7 + kw) * C + c);
#pragma unroll
      for (int kw = 0; kw < 7; ++kw)
#pragma unroll
        for (int j = 0; j < TW; ++j) acc[j] = fmaf(k[kw], xin[j + kw], acc[j]);
    }
    const float bc = __ldg(wb + c);
#pragma unroll
    for (int j = 0; j < TW; ++j) s[(size_t)(i * TW + j) * C + c] = acc[j] + bc;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, warps = blockDim.x >> 5;
  for (int p = warp; p < TH * TW; p += warps) {
    const int h = h0 + p / TW, w = w0 + p % TW;
    if (h >= H || w >= W) continue;     // uniform over the warp
    const float4* xr = reinterpret_cast<const float4*>(s + (size_t)p * C);
    float4 v[VPL > 0 ? VPL : 1];
    float mean, rstd;
    ln_row_stats<VPL>(xr, lane, C, eps, v, mean, rstd);
    ln_store_row<VPL>(Y + (((size_t)b * H + h) * W + w) * C, xr, lane, C, v, scale, bias, mean, rstd);
  }
}

// ------------------------------------------------------------------------------------------------ LayerNorm + 2x2 patchify
// Downsampling layer i = 1..3 (models/convnext.py:168-177): LayerNorm of every pixel of X [n, H, W, C], then Conv 2x2
// stride 2 = a GEMM over [n * H/2 * W/2, 4C] rows whose column (kh * 2 + kw) * C + c is pixel (2i + kh, 2j + kw)'s
// normalised channel c (the HWIO kernel [2, 2, C, C'] viewed as [4C, C']).  One warp per input pixel, written straight
// into its slot: the same bits as d3_layernorm_fwd followed by the permutation.
template <int VPL>
__global__ void __launch_bounds__(256)
ln_patchify2_kernel(const float* __restrict__ X, const float* __restrict__ scale, const float* __restrict__ bias,
                    __nv_bfloat16* __restrict__ Y, long T, int H, int W, int C, float eps) {
  const int warps = blockDim.x >> 5, lane = threadIdx.x & 31;
  for (long row = (long)blockIdx.x * warps + (threadIdx.x >> 5); row < T; row += (long)gridDim.x * warps) {
    const int w = (int)(row % W), h = (int)((row / W) % H);
    const long b = row / ((long)W * H);
    __nv_bfloat16* dst = Y + (((size_t)b * (H / 2) + h / 2) * (W / 2) + w / 2) * 4 * C + ((h & 1) * 2 + (w & 1)) * C;
    const float4* xr = reinterpret_cast<const float4*>(X + row * (long)C);
    float4 v[VPL > 0 ? VPL : 1];
    float mean, rstd;
    ln_row_stats<VPL>(xr, lane, C, eps, v, mean, rstd);
    ln_store_row<VPL>(dst, xr, lane, C, v, scale, bias, mean, rstd);
  }
}

// ------------------------------------------------------------------------------------------------ pooled class token
// models/convnext.py:223,254 x_pool = mean over H x W.  A CTA takes 64 channels (16 float4 columns) of one image:
// row group g of PT_GROUPS sums the rows p = g, g + PT_GROUPS, ... in that order, then thread g = 0 adds the groups'
// partial sums in group order and divides by P: the same bits every run, whatever the schedule.  With copy, every row
// is also written to row 1 + p of the image's [rows = 1 + P, C] block of `out` as it is read (X read once).
constexpr int PT_GROUPS = 16;
constexpr int PT_QUADS = 16;
__global__ void __launch_bounds__(PT_GROUPS * PT_QUADS)
pool_tokens_kernel(const float* __restrict__ X, float* __restrict__ out, int P, int C, int rows, int copy) {
  __shared__ float4 part[PT_GROUPS][PT_QUADS];
  const int q = threadIdx.x % PT_QUADS, g = threadIdx.x / PT_QUADS;
  const int c4 = blockIdx.x * PT_QUADS + q, b = blockIdx.y;
  const bool on = c4 < C / 4;
  const float4* xb = reinterpret_cast<const float4*>(X + (size_t)b * P * C);
  float4* ob = reinterpret_cast<float4*>(out + (size_t)b * rows * C);
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  if (on) {
#pragma unroll 4
    for (int p = g; p < P; p += PT_GROUPS) {
      const float4 v = xb[(size_t)p * (C / 4) + c4];
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
      if (copy) ob[(size_t)(1 + p) * (C / 4) + c4] = v;
    }
  }
  part[g][q] = s;
  __syncthreads();
  if (g == 0 && on) {
    float4 t = part[0][q];
#pragma unroll
    for (int k = 1; k < PT_GROUPS; ++k) {
      const float4 u = part[k][q];
      t.x += u.x; t.y += u.y; t.z += u.z; t.w += u.w;
    }
    ob[c4] = make_float4(t.x / P, t.y / P, t.z / P, t.w / P);
  }
}

// ------------------------------------------------------------------------------------------------ bilinear resize
// models/convnext.py:256-261 (upstream: F.interpolate(mode="bilinear", antialias=True)): torch's
// _upsample_bilinear2d_aa arithmetic, separable taps with support max(scale, 1) around the centre scale (o + 0.5), the
// triangle filter stretched by max(scale, 1), weights normalised over the taps inside the map.  fp32 maps
// [n, Hs, Ws, C] -> rows prefix .. prefix + Hd*Wd - 1 of each image's [prefix + Hd*Wd, C] block of dst (the token layout
// of d3_layernorm_tokens_out, row 0 the pooled class token).  One CTA per output pixel, one float4 of channels per
// thread.
constexpr int BL_TAPS = 16;
__device__ __forceinline__ int bilinear_aa_taps(int o, int in, int out, int* idx, float* w) {
  const float scale = (float)in / (float)out;
  const float sup = fmaxf(scale, 1.f), inv = 1.f / fmaxf(scale, 1.f);
  const float c = scale * (o + 0.5f);
  const int lo = max((int)(c - sup + 0.5f), 0), hi = min((int)(c + sup + 0.5f), in);
  int n = 0;
  float tot = 0.f;
  for (int x = lo; x < hi && n < BL_TAPS; ++x, ++n) {
    idx[n] = x;
    w[n] = fmaxf(0.f, 1.f - fabsf((x - c + 0.5f) * inv));
    tot += w[n];
  }
  for (int k = 0; k < n; ++k) w[k] /= tot;
  return n;
}
__global__ void resize_bilinear_aa_kernel(const float* __restrict__ src, float* __restrict__ dst, int Hs, int Ws, int Hd,
                                          int Wd, int C, int prefix) {
  const int ox = blockIdx.x % Wd, oy = (blockIdx.x / Wd) % Hd, n = blockIdx.x / (Wd * Hd);
  int ix[BL_TAPS], iy[BL_TAPS];
  float wx[BL_TAPS], wy[BL_TAPS];
  const int nx = bilinear_aa_taps(ox, Ws, Wd, ix, wx), ny = bilinear_aa_taps(oy, Hs, Hd, iy, wy);
  const float* base = src + (size_t)n * Hs * Ws * C;
  float* out = dst + ((size_t)n * (prefix + Hd * Wd) + prefix + (size_t)oy * Wd + ox) * C;
  for (int d = threadIdx.x * 4; d < C; d += blockDim.x * 4) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int a = 0; a < ny; ++a) {
      float4 row = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int e = 0; e < nx; ++e) {
        const float4 v = *reinterpret_cast<const float4*>(base + ((size_t)iy[a] * Ws + ix[e]) * C + d);
        row.x = fmaf(wx[e], v.x, row.x); row.y = fmaf(wx[e], v.y, row.y);
        row.z = fmaf(wx[e], v.z, row.z); row.w = fmaf(wx[e], v.w, row.w);
      }
      acc.x = fmaf(wy[a], row.x, acc.x); acc.y = fmaf(wy[a], row.y, acc.y);
      acc.z = fmaf(wy[a], row.z, acc.z); acc.w = fmaf(wy[a], row.w, acc.w);
    }
    *reinterpret_cast<float4*>(out + d) = acc;
  }
}

// ------------------------------------------------------------------------------------------------ host side
template <int VPL>
static int launch_dwconv7_ln(const float* X, const float* wt, const float* wb, const float* scale, const float* bias,
                             float eps, __nv_bfloat16* Y, int n, int H, int W, int C, cudaStream_t st) {
  int TH = 8;
  while (TH > 2 && (size_t)TH * DW_TW * C * sizeof(float) > (size_t)DW_SMEM_MAX) TH /= 2;
  const int tiles_w = (W + DW_TW - 1) / DW_TW;
  while (TH > 1 && (long)n * ((H + TH - 1) / TH) * tiles_w < 2L * sm_count()) TH /= 2;
  const int tiles_h = (H + TH - 1) / TH;
  const int threads = (int)min((long)DW_THREADS_MAX, ((long)TH * C + 31) / 32 * 32);
  const size_t smem = (size_t)TH * DW_TW * C * sizeof(float);
  static const cudaError_t cfg = cudaFuncSetAttribute(dwconv7_ln_kernel<VPL>,
                                                      cudaFuncAttributeMaxDynamicSharedMemorySize, DW_SMEM_MAX);
  (void)cfg;   // a failure shows at the launch
  dwconv7_ln_kernel<VPL><<<(unsigned)((long)n * tiles_h * tiles_w), threads, smem, st>>>(X, wt, wb, scale, bias, Y, H, W,
                                                                                        C, TH, tiles_h, tiles_w, eps);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

static int launch_dwconv7_ln(const float* X, const float* wt, const float* wb, const float* scale, const float* bias,
                             float eps, __nv_bfloat16* Y, int n, int H, int W, int C, cudaStream_t st) {
  switch (C) {     // the widths d3_layernorm_fwd specialises, so that each row takes the same instructions
    case 128: return launch_dwconv7_ln<1>(X, wt, wb, scale, bias, eps, Y, n, H, W, C, st);
    case 256: return launch_dwconv7_ln<2>(X, wt, wb, scale, bias, eps, Y, n, H, W, C, st);
    case 384: return launch_dwconv7_ln<3>(X, wt, wb, scale, bias, eps, Y, n, H, W, C, st);
    case 512: return launch_dwconv7_ln<4>(X, wt, wb, scale, bias, eps, Y, n, H, W, C, st);
    case 768: return launch_dwconv7_ln<6>(X, wt, wb, scale, bias, eps, Y, n, H, W, C, st);
    case 1024: return launch_dwconv7_ln<8>(X, wt, wb, scale, bias, eps, Y, n, H, W, C, st);
    case 1536: return launch_dwconv7_ln<12>(X, wt, wb, scale, bias, eps, Y, n, H, W, C, st);
    default: return launch_dwconv7_ln<0>(X, wt, wb, scale, bias, eps, Y, n, H, W, C, st);
  }
}

template <int VPL>
static int launch_ln_patchify2(const float* X, const float* scale, const float* bias, float eps, __nv_bfloat16* Y, long T,
                               int H, int W, int C, cudaStream_t st) {
  const int blocks = (int)min((T + 7) / 8, (long)sm_count() * 8);
  ln_patchify2_kernel<VPL><<<blocks, 256, 0, st>>>(X, scale, bias, Y, T, H, W, C, eps);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

}  // namespace d3

using namespace d3;

extern "C" {

int d3_dwconv7_layernorm(const float* X, const float* w, const float* wb, const float* scale, const float* bias, float eps,
                         void* Y, int n, int H, int W, int C, void* stream) {
  if (!X || !w || !wb || !scale || !bias || !Y) return set_error(D3_ERR_ARG, "d3_dwconv7_layernorm: null pointer");
  if (n < 0 || H < 1 || W < 1 || C < 8 || C % 8 || C > 1536)
    return set_error(D3_ERR_ARG, "d3_dwconv7_layernorm: need n >= 0, H, W >= 1 and C a multiple of 8 in [8, 1536]");
  if ((long long)n * H * W * C >= (1LL << 40)) return set_error(D3_ERR_ARG, "d3_dwconv7_layernorm: X too large");
  if (((uintptr_t)X | (uintptr_t)scale | (uintptr_t)bias) % 16 || (uintptr_t)w % 4 || (uintptr_t)wb % 4 ||
      (uintptr_t)Y % 16)
    return set_error(D3_ERR_ARG, "d3_dwconv7_layernorm: X, Y, scale and bias must be 16-byte aligned, w and wb 4-byte");
  if (n == 0) return D3_OK;
  cudaStream_t st = STREAM(stream);
  auto* y = reinterpret_cast<__nv_bfloat16*>(Y);
  return launch_dwconv7_ln(X, w, wb, scale, bias, eps, y, n, H, W, C, st);
}

int d3_layernorm_patchify2(const float* X, const float* scale, const float* bias, float eps, void* Y, int n, int H, int W,
                           int C, void* stream) {
  if (!X || !scale || !bias || !Y) return set_error(D3_ERR_ARG, "d3_layernorm_patchify2: null pointer");
  if (n < 0 || H < 2 || W < 2 || H % 2 || W % 2 || C < 4 || C % 4)
    return set_error(D3_ERR_ARG, "d3_layernorm_patchify2: need n >= 0, even H, W >= 2 and C a positive multiple of 4");
  if ((long long)n * H * W * C >= (1LL << 40)) return set_error(D3_ERR_ARG, "d3_layernorm_patchify2: X too large");
  if (((uintptr_t)X | (uintptr_t)scale | (uintptr_t)bias) % 16 || (uintptr_t)Y % 8)
    return set_error(D3_ERR_ARG, "d3_layernorm_patchify2: X, scale and bias must be 16-byte aligned, Y 8-byte");
  if (n == 0) return D3_OK;
  const long T = (long)n * H * W;
  auto* y = reinterpret_cast<__nv_bfloat16*>(Y);
  cudaStream_t st = STREAM(stream);
  switch (C) {
    case 128: return launch_ln_patchify2<1>(X, scale, bias, eps, y, T, H, W, C, st);
    case 256: return launch_ln_patchify2<2>(X, scale, bias, eps, y, T, H, W, C, st);
    case 384: return launch_ln_patchify2<3>(X, scale, bias, eps, y, T, H, W, C, st);
    case 512: return launch_ln_patchify2<4>(X, scale, bias, eps, y, T, H, W, C, st);
    case 768: return launch_ln_patchify2<6>(X, scale, bias, eps, y, T, H, W, C, st);
    case 1024: return launch_ln_patchify2<8>(X, scale, bias, eps, y, T, H, W, C, st);
    case 1536: return launch_ln_patchify2<12>(X, scale, bias, eps, y, T, H, W, C, st);
    default: return launch_ln_patchify2<0>(X, scale, bias, eps, y, T, H, W, C, st);
  }
}

int d3_pool_tokens(const float* X, float* out, int n, int P, int C, int rows, int copy_tokens, void* stream) {
  if (!X || !out) return set_error(D3_ERR_ARG, "d3_pool_tokens: null pointer");
  if (n < 0 || P < 1 || C < 4 || C % 4 || rows < 1 || (copy_tokens && rows != 1 + P))
    return set_error(D3_ERR_ARG, "d3_pool_tokens: need n >= 0, P >= 1, C a positive multiple of 4, rows >= 1 "
                                 "(rows == 1 + P to copy the tokens)");
  if ((long long)n * P * C >= (1LL << 40) || (long long)n * rows * C >= (1LL << 40))
    return set_error(D3_ERR_ARG, "d3_pool_tokens: X too large");
  if (((uintptr_t)X | (uintptr_t)out) % 16) return set_error(D3_ERR_ARG, "d3_pool_tokens: X and out must be 16-byte aligned");
  if (n == 0) return D3_OK;
  const dim3 grid((C / 4 + PT_QUADS - 1) / PT_QUADS, n);
  pool_tokens_kernel<<<grid, PT_GROUPS * PT_QUADS, 0, STREAM(stream)>>>(X, out, P, C, rows, copy_tokens ? 1 : 0);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_resize_tokens_bilinear_aa(const float* src, float* dst, int n, int Hs, int Ws, int Hd, int Wd, int C, int prefix,
                                 void* stream) {
  if (!src || !dst) return set_error(D3_ERR_ARG, "d3_resize_tokens_bilinear_aa: null pointer");
  if (n < 0 || Hs < 1 || Ws < 1 || Hd < 1 || Wd < 1 || C < 4 || C % 4 || prefix < 0)
    return set_error(D3_ERR_ARG, "d3_resize_tokens_bilinear_aa: need positive sizes, C % 4 == 0 and prefix >= 0");
  if ((long long)n * Hs * Ws * C >= (1LL << 40) || (long long)n * (prefix + (long long)Hd * Wd) * C >= (1LL << 40))
    return set_error(D3_ERR_ARG, "d3_resize_tokens_bilinear_aa: map too large");
  if (((uintptr_t)src | (uintptr_t)dst) % 16)
    return set_error(D3_ERR_ARG, "d3_resize_tokens_bilinear_aa: src and dst must be 16-byte aligned");
  // taps per output: at most 2 * scale + 2 (support scale on each side, one more for the rounding of the ends)
  if (2.f * fmaxf((float)Hs / Hd, (float)Ws / Wd) + 2.f > (float)BL_TAPS)
    return set_error(D3_ERR_ARG, "d3_resize_tokens_bilinear_aa: down-scaling factor too large (<= 7)");
  if (n == 0) return D3_OK;
  const int threads = min(256, max(32, ((C / 4 + 31) / 32) * 32));
  resize_bilinear_aa_kernel<<<(unsigned)((long)n * Hd * Wd), threads, 0, STREAM(stream)>>>(src, dst, Hs, Ws, Hd, Wd, C,
                                                                                             prefix);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

}  // extern "C"
