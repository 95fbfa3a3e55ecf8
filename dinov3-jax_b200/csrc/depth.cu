// Linear monocular-depth probe of a frozen backbone: the "linear" bin head's depth per patch cell, the scale-invariant
// log loss of that depth upsampled bilinearly to the ground truth with its gradient to the patch logits, the per-image
// regression metrics of the upsampled prediction, and the crop of a float depth plane.  The head's BatchNorm, GEMMs,
// bias gradient and update are the segmentation probe's (seg.cu, d3_gemm_bf16, d3_colsum_bf16, d3_adamw_ema) and the
// image crop is d3_seg_crop; nothing here multiplies matrices.
//
// Head: bin centres c_k = linspace(min_depth, max_depth, n_bins); per cell q_k = relu(z_k) + 0.1, S = sum_k q_k and
// d = sum_k q_k c_k / S.  Upsampling is torch's bilinear F.interpolate(align_corners = False), with the tile-per-cell
// geometry of bilinear.cuh.  Loss, over the pixels V with min_depth < gt <= max_depth: g = log(d_hat + 1e-3) -
// log(gt + 1e-3), L = sqrt(var(g) + 0.15 mean(g)^2) with the unbiased variance; |V| < 2 gives L = 0 and no gradient.
//
// The gradient of one pixel depends on the batch's mean and variance, so the loss takes four passes:
//   (a) per cell, one warp: S and d;
//   (b) per tile, one thread per pixel: (count, mean, M2) of g by Welford's update in pixel order, merged across the
//       threads and warps in a fixed tree by Chan's formula; one CTA then merges the tiles the same way and writes L.
//       Merging centred moments keeps var(g) accurate when |mean(g)| is large against its spread, which
//       (sum g^2 - N mean^2) / (N - 1) in fp32 does not;
//   (c) per tile: dL/d d_hat = ((g - mean) / (N - 1) + 0.15 mean / N) / L / (d_hat + 1e-3) per pixel, times its four
//       bilinear weights, added in pixel order and a fixed tree into one partial per (tile, corner);
//   (d) per (cell, bin): the cell's (at most four) partials in a fixed order give dL/dd, and
//       dL/dz_k = 1[z_k > 0] (c_k - d) / S dL/dd.
// Deterministic: no atomics, the same bits on every run.
#include "ptx.cuh"
#include "d3_internal.h"
#include "bilinear.cuh"

#include <math.h>
#include <stdio.h>

#include <algorithm>

namespace d3 {

constexpr float DEPTH_EPS = 1e-3f;          // inside the logs of the loss
constexpr float SI_LAMBDA = 0.15f;          // weight of mean(g)^2 in the loss
constexpr float BIN_FLOOR = 0.1f;           // q_k = relu(z_k) + 0.1
constexpr int DC_WARPS = 8;                 // cells per CTA of the cell pass
constexpr int DT_THREADS = 128;             // one CTA per tile, one thread per pixel
constexpr int DT_WARPS = DT_THREADS / 32;
constexpr int N_METRICS = 9;                // count, abs_rel, sq_rel, sq, sq_log, log10, a1, a2, a3

// torch.linspace(lo, hi, n)[k] in fp32: the first half counts up from lo, the second down from hi
__device__ __forceinline__ float bin_centre(int k, int n, float lo, float hi) {
  const float step = (hi - lo) / (float)(n - 1);
  return k < n / 2 ? lo + step * (float)k : hi - step * (float)(n - 1 - k);
}

// ------------------------------------------------------------------------------------------------ (a) cell depth
// One warp per cell: lane-strided sums over the bins, then butterflies (every lane gets the same bits).
__global__ void __launch_bounds__(DC_WARPS * 32) depth_cell_kernel(const float* __restrict__ logits, int ld,
                                                                   long long cells, int nb, float lo, float hi,
                                                                   float* __restrict__ cell_s,
                                                                   float* __restrict__ cell_d) {
  const int lane = threadIdx.x & 31;
  const long long cell = (long long)blockIdx.x * DC_WARPS + (threadIdx.x >> 5);
  if (cell >= cells) return;
  const float* z = logits + cell * ld;
  float s = 0.f, m = 0.f;
  for (int k = lane; k < nb; k += 32) {
    const float q = fmaxf(z[k], 0.f) + BIN_FLOOR;
    s += q;
    m = fmaf(q, bin_centre(k, nb, lo, hi), m);
  }
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    m += __shfl_xor_sync(0xffffffffu, m, o);
  }
  if (lane == 0) {
    cell_s[cell] = s;
    cell_d[cell] = m / s;
  }
}

// ------------------------------------------------------------------------------------------------ per-pixel helpers
// the depths of the tile's four corner cells (00, 01, 10, 11)
__device__ __forceinline__ void depth_corners(const float* __restrict__ cell_d, const SegGeom& g, const SegTile& t,
                                              float (&D)[4]) {
  const long long base = (long long)t.b * g.h;
  D[0] = cell_d[(base + t.ty) * g.w + t.tx];
  D[1] = cell_d[(base + t.ty) * g.w + t.x1];
  D[2] = cell_d[(base + t.y1) * g.w + t.tx];
  D[3] = cell_d[(base + t.y1) * g.w + t.x1];
}

// bilinear depth at pixel (y, x) of tile t, as seg.cu's seg_pixel on one channel, and its four corner weights
__device__ __forceinline__ float depth_pixel(const SegGeom& g, const SegTile& t, int y, int x, const float (&D)[4],
                                             float (&wk)[4]) {
  const float ly = seg_src(y, g.sh) - (float)t.ty, lx = seg_src(x, g.sw) - (float)t.tx;
  const float h0 = 1.f - ly, w0 = 1.f - lx;
  wk[0] = h0 * w0; wk[1] = h0 * lx; wk[2] = ly * w0; wk[3] = ly * lx;
  return h0 * (w0 * D[0] + lx * D[1]) + ly * (w0 * D[2] + lx * D[3]);
}

__device__ __forceinline__ bool depth_valid(float gt, float lo, float hi) { return gt > lo && gt <= hi; }

// fp32 sums of N values per thread -> thread 0: a shfl_down tree in each warp, then the warps in order
template <int N>
__device__ __forceinline__ void block_sum(float (&a)[N], float (*red)[N]) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
#pragma unroll
    for (int k = 0; k < N; ++k) a[k] += __shfl_down_sync(0xffffffffu, a[k], o);
  if (lane == 0)
#pragma unroll
    for (int k = 0; k < N; ++k) red[wid][k] = a[k];
  __syncthreads();
  if (threadIdx.x == 0)
#pragma unroll
    for (int k = 0; k < N; ++k) {
      a[k] = red[0][k];
      for (int w = 1; w < DT_WARPS; ++w) a[k] += red[w][k];
    }
}

// ------------------------------------------------------------------------------------------------ (b) moments of g
struct Moments {
  int n;
  float mean, m2;     // mean and sum of squared deviations from it
};

// Chan et al.'s merge of two sets' centred moments
__device__ __forceinline__ Moments chan(const Moments& a, const Moments& b) {
  if (b.n == 0) return a;
  if (a.n == 0) return b;
  const int n = a.n + b.n;
  const float fb = (float)b.n / (float)n, d = b.mean - a.mean;
  return Moments{n, fmaf(d, fb, a.mean), a.m2 + b.m2 + d * d * ((float)a.n * fb)};
}

__device__ __forceinline__ Moments shfl_down(const Moments& m, int o) {
  return Moments{__shfl_down_sync(0xffffffffu, m.n, o), __shfl_down_sync(0xffffffffu, m.mean, o),
                 __shfl_down_sync(0xffffffffu, m.m2, o)};
}

__global__ void __launch_bounds__(DT_THREADS) depth_moments_kernel(const float* __restrict__ cell_d,
                                                                   const float* __restrict__ gt, SegGeom g, float lo,
                                                                   float hi, Moments* __restrict__ tile_m) {
  __shared__ int range[4];
  __shared__ Moments red[DT_WARPS];
  const SegTile t = seg_tile(g, range);
  float D[4];
  depth_corners(cell_d, g, t, D);
  const int nx = t.x_hi - t.x_lo, np = (t.y_hi - t.y_lo) * nx;
  const float* gp = gt + (size_t)t.b * g.Hl * g.Wl;
  Moments m{0, 0.f, 0.f};
  for (int p = threadIdx.x; p < np; p += DT_THREADS) {
    const int y = t.y_lo + p / nx, x = t.x_lo + p % nx;
    const float v = gp[(size_t)y * g.Wl + x];
    if (!depth_valid(v, lo, hi)) continue;
    float wk[4];
    const float gv = logf(depth_pixel(g, t, y, x, D, wk) + DEPTH_EPS) - logf(v + DEPTH_EPS);
    ++m.n;
    const float dl = gv - m.mean;
    m.mean += dl / (float)m.n;
    m.m2 = fmaf(dl, gv - m.mean, m.m2);
  }
  for (int o = 16; o > 0; o >>= 1) m = chan(m, shfl_down(m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    m = red[0];
    for (int w = 1; w < DT_WARPS; ++w) m = chan(m, red[w]);
    tile_m[blockIdx.x] = m;
  }
}

// One CTA: thread t merges tiles t, t + 1024, ... in order, then a fixed tree over the threads.  Writes the loss, the
// valid count and the coefficients of pass (c): coef = (mean, 1 / ((N - 1) L), 0.15 mean / (N L)), both 0 when N < 2
// or L = 0 (where the square root has no derivative).
constexpr int DL_THREADS = 1024;
__global__ void __launch_bounds__(DL_THREADS) depth_loss_kernel(const Moments* __restrict__ tile_m, long long n_tiles,
                                                                float* __restrict__ loss, int* __restrict__ count,
                                                                float* __restrict__ coef) {
  __shared__ Moments red[DL_THREADS];
  Moments m{0, 0.f, 0.f};
  for (long long i = threadIdx.x; i < n_tiles; i += DL_THREADS) m = chan(m, tile_m[i]);
  red[threadIdx.x] = m;
  __syncthreads();
  for (int o = DL_THREADS / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] = chan(red[threadIdx.x], red[threadIdx.x + o]);
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    m = red[0];
    float L = 0.f, inv = 0.f, c = 0.f;
    if (m.n >= 2) {
      L = sqrtf(m.m2 / (float)(m.n - 1) + SI_LAMBDA * m.mean * m.mean);
      if (L > 0.f) {
        inv = 1.f / ((float)(m.n - 1) * L);
        c = SI_LAMBDA * m.mean / ((float)m.n * L);
      }
    }
    *loss = L;
    *count = m.n;
    coef[0] = m.mean; coef[1] = inv; coef[2] = c;
  }
}

// ------------------------------------------------------------------------------------------------ (c) gradient tiles
// part[tile * 4 + k] = sum over the tile's valid pixels of w_k dL/d d_hat; corners that coincide at the last row /
// column (y1 == y0, x1 == x0) are folded into one, as seg.cu does.
__global__ void __launch_bounds__(DT_THREADS) depth_grad_tile_kernel(const float* __restrict__ cell_d,
                                                                     const float* __restrict__ gt, SegGeom g, float lo,
                                                                     float hi, const float* __restrict__ coef,
                                                                     float* __restrict__ part) {
  __shared__ int range[4];
  __shared__ float red[DT_WARPS][4];
  const SegTile t = seg_tile(g, range);
  float D[4];
  depth_corners(cell_d, g, t, D);
  const float mean = coef[0], inv = coef[1], c = coef[2];
  const int nx = t.x_hi - t.x_lo, np = (t.y_hi - t.y_lo) * nx;
  const float* gp = gt + (size_t)t.b * g.Hl * g.Wl;
  float a[4] = {0.f, 0.f, 0.f, 0.f};
  for (int p = threadIdx.x; p < np; p += DT_THREADS) {
    const int y = t.y_lo + p / nx, x = t.x_lo + p % nx;
    const float v = gp[(size_t)y * g.Wl + x];
    if (!depth_valid(v, lo, hi)) continue;
    float wk[4];
    const float dh = depth_pixel(g, t, y, x, D, wk) + DEPTH_EPS;
    const float gv = logf(dh) - logf(v + DEPTH_EPS);
    const float gd = fmaf(gv - mean, inv, c) / dh;
#pragma unroll
    for (int k = 0; k < 4; ++k) a[k] = fmaf(wk[k], gd, a[k]);
  }
  block_sum<4>(a, red);
  if (threadIdx.x == 0) {
    if (t.x1 == t.tx) { a[0] += a[1]; a[2] += a[3]; a[1] = 0.f; a[3] = 0.f; }
    if (t.y1 == t.ty) { a[0] += a[2]; a[1] += a[3]; a[2] = 0.f; a[3] = 0.f; }
#pragma unroll
    for (int k = 0; k < 4; ++k) part[(size_t)blockIdx.x * 4 + k] = a[k];
  }
}

// ------------------------------------------------------------------------------------------------ (d) dZ
// dL/dd of a cell = part[cell, 00] + part[cell - 1, 01] + part[cell - w, 10] + part[cell - w - 1, 11];
// dZ[cell, k] = 1[z_k > 0] (c_k - d) / S dL/dd for k < nb, 0 for k in [nb, Cp); fp32 and / or bf16
__global__ void depth_dz_kernel(const float* __restrict__ logits, int ld, const float* __restrict__ part,
                                const float* __restrict__ cell_s, const float* __restrict__ cell_d, SegGeom g, int nb,
                                int Cp, float lo, float hi, float* __restrict__ dz_f32,
                                __nv_bfloat16* __restrict__ dz_bf16, int ld_dz) {
  const long long n = (long long)g.B * g.h * g.w * Cp;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long cell = i / Cp;
    const int k = (int)(i - cell * Cp);
    float v = 0.f;
    if (k < nb && logits[cell * ld + k] > 0.f) {
      const int x = (int)(cell % g.w), y = (int)((cell / g.w) % g.h);
      float gdd = part[cell * 4 + 0];
      if (x > 0) gdd += part[(cell - 1) * 4 + 1];
      if (y > 0) gdd += part[(cell - g.w) * 4 + 2];
      if (x > 0 && y > 0) gdd += part[(cell - g.w - 1) * 4 + 3];
      v = gdd * ((bin_centre(k, nb, lo, hi) - cell_d[cell]) / cell_s[cell]);
    }
    if (dz_f32) dz_f32[cell * ld_dz + k] = v;
    if (dz_bf16) dz_bf16[cell * ld_dz + k] = __float2bfloat16(v);
  }
}

// ------------------------------------------------------------------------------------------------ metrics
// Per tile, over the valid pixels inside rows [crop.x, crop.y) and columns [crop.z, crop.w): with p = the upsampled
// depth clamped to [lo, hi] and t = gt, fp32 sums of 1, |p - t| / t, (p - t)^2 / t, (p - t)^2, (ln p - ln t)^2,
// |log10 p - log10 t| and 1[max(p / t, t / p) < 1.25^k] for k = 1, 2, 3.
__global__ void __launch_bounds__(DT_THREADS) depth_metrics_tile_kernel(const float* __restrict__ cell_d,
                                                                        const float* __restrict__ gt, SegGeom g,
                                                                        float lo, float hi, int4 crop,
                                                                        float* __restrict__ tile_sums) {
  __shared__ int range[4];
  __shared__ float red[DT_WARPS][N_METRICS];
  const SegTile t = seg_tile(g, range);
  float D[4];
  depth_corners(cell_d, g, t, D);
  const int nx = t.x_hi - t.x_lo, np = (t.y_hi - t.y_lo) * nx;
  const float* gp = gt + (size_t)t.b * g.Hl * g.Wl;
  float a[N_METRICS];
#pragma unroll
  for (int k = 0; k < N_METRICS; ++k) a[k] = 0.f;
  for (int p = threadIdx.x; p < np; p += DT_THREADS) {
    const int y = t.y_lo + p / nx, x = t.x_lo + p % nx;
    if (y < crop.x || y >= crop.y || x < crop.z || x >= crop.w) continue;
    const float v = gp[(size_t)y * g.Wl + x];
    if (!depth_valid(v, lo, hi)) continue;
    float wk[4];
    const float pr = fminf(fmaxf(depth_pixel(g, t, y, x, D, wk), lo), hi);
    const float df = pr - v, lg = logf(pr) - logf(v), r = fmaxf(pr / v, v / pr);
    a[0] += 1.f;
    a[1] += fabsf(df) / v;
    a[2] += df * df / v;
    a[3] += df * df;
    a[4] += lg * lg;
    a[5] += fabsf(log10f(pr) - log10f(v));
    a[6] += r < 1.25f ? 1.f : 0.f;
    a[7] += r < 1.5625f ? 1.f : 0.f;
    a[8] += r < 1.953125f ? 1.f : 0.f;
  }
  block_sum<N_METRICS>(a, red);
  if (threadIdx.x == 0)
#pragma unroll
    for (int k = 0; k < N_METRICS; ++k) tile_sums[(size_t)blockIdx.x * N_METRICS + k] = a[k];
}

// One CTA per image: thread t adds the image's tiles t, t + 128, ... in order in fp64, then a fixed tree.
constexpr int DM_THREADS = 128;
__global__ void __launch_bounds__(DM_THREADS) depth_metrics_image_kernel(const float* __restrict__ tile_sums,
                                                                         int tiles_per_image,
                                                                         double* __restrict__ sums) {
  __shared__ double red[N_METRICS][DM_THREADS];
  double a[N_METRICS];
#pragma unroll
  for (int k = 0; k < N_METRICS; ++k) a[k] = 0.0;
  const float* ts = tile_sums + (size_t)blockIdx.x * tiles_per_image * N_METRICS;
  for (int i = threadIdx.x; i < tiles_per_image; i += DM_THREADS)
#pragma unroll
    for (int k = 0; k < N_METRICS; ++k) a[k] += (double)ts[(size_t)i * N_METRICS + k];
#pragma unroll
  for (int k = 0; k < N_METRICS; ++k) red[k][threadIdx.x] = a[k];
  __syncthreads();
  for (int o = DM_THREADS / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o)
#pragma unroll
      for (int k = 0; k < N_METRICS; ++k) red[k][threadIdx.x] += red[k][threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x < N_METRICS) sums[(size_t)blockIdx.x * N_METRICS + threadIdx.x] = red[threadIdx.x][0];
}

// ------------------------------------------------------------------------------------------------ depth-plane crop
// The depth plane of d3_seg_crop's box: torch's 'nearest' (src = min(floor(dst * in / out), in - 1), fp32) from the
// float map of image n's size at depth_src + desc offset / 3, mirrored within the part inside the resized image when
// flipped; 0 (invalid) outside it.
__global__ void depth_plane_crop_kernel(const float* __restrict__ src, const long long* __restrict__ desc,
                                        const int* __restrict__ boxes, int out_h, int out_w, float* __restrict__ out) {
  const int n = blockIdx.y;
  const long long off = desc[3 * n] / 3;
  const int H = (int)desc[3 * n + 1], W = (int)desc[3 * n + 2];
  const int* bx = boxes + 6 * n;
  const int rh = bx[0], rw = bx[1], top = bx[2], left = bx[3], flip = bx[4];
  const int vh = min(out_h, rh - top), vw = min(out_w, rw - left);
  const float nsy = (float)H / (float)rh, nsx = (float)W / (float)rw;
  const int total = out_h * out_w;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < total; p += gridDim.x * blockDim.x) {
    const int oy = p / out_w, ox = p % out_w;
    float v = 0.f;
    if (oy < vh && ox < vw) {
      const int sx = flip ? vw - 1 - ox : ox;
      const int ly = min((int)floorf((float)(top + oy) * nsy), H - 1);
      const int lx = min((int)floorf((float)(left + sx) * nsx), W - 1);
      v = src[off + (size_t)ly * W + lx];
    }
    out[(size_t)n * total + p] = v;
  }
}

}  // namespace d3

using namespace d3;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

namespace {

int depth_geom(const char* who, int B, int h, int w, int Hl, int Wl, int nb, int ld, float lo, float hi, SegGeom& g) {
  char msg[200];
  if (h < 1 || w < 1 || Hl < 1 || Wl < 1 || nb < 2 || ld < nb || !(lo >= 0.f) || !(hi > lo)) {
    snprintf(msg, sizeof(msg), "%s: need h, w, Hl, Wl >= 1, n_bins >= 2, ld >= n_bins and 0 <= min_depth < max_depth",
             who);
    return set_error(D3_ERR_ARG, msg);
  }
  if ((long long)B * h * w > 0x7fffffffLL) {
    snprintf(msg, sizeof(msg), "%s: more than 2^31 - 1 patch cells", who);
    return set_error(D3_ERR_ARG, msg);
  }
  g = SegGeom{B, h, w, Hl, Wl, (float)h / (float)Hl, (float)w / (float)Wl};
  return D3_OK;
}

}  // namespace

extern "C" {

int d3_depth_crop(const void* src_u8, const long long* desc, const float* depth_src, const int* boxes, int n, int out_h,
                  int out_w, int max_taps, const float* mean3, const float* std3, void* out, int out_u8,
                  float* depth_out, void* stream) {
  if (n <= 0) return D3_OK;
  if (depth_out && !depth_src) return set_error(D3_ERR_ARG, "d3_depth_crop: depth_out needs depth_src");
  if (int rc = d3_seg_crop(src_u8, desc, nullptr, boxes, n, out_h, out_w, max_taps, mean3, std3, out, out_u8, nullptr,
                           stream))
    return rc;
  if (!depth_out) return D3_OK;
  const int blocks = std::min((out_h * out_w + 255) / 256, 1024);
  depth_plane_crop_kernel<<<dim3(blocks, n), 256, 0, STREAM(stream)>>>(depth_src, desc, boxes, out_h, out_w, depth_out);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_depth_head_fwd_bwd(const float* logits, int ld, const float* gt, int B, int h, int w, int Hl, int Wl,
                          int n_bins, int Cp, float min_depth, float max_depth, float* loss, int* count, float* dz_f32,
                          void* dz_bf16, int ld_dz, void* stream) {
  if (B <= 0) return D3_OK;
  SegGeom g;
  if (int rc = depth_geom("d3_depth_head_fwd_bwd", B, h, w, Hl, Wl, n_bins, ld, min_depth, max_depth, g)) return rc;
  if (!logits || !gt || !loss || !count || Cp < n_bins || ((dz_f32 || dz_bf16) && ld_dz < Cp))
    return set_error(D3_ERR_ARG, "d3_depth_head_fwd_bwd: need Cp >= n_bins, ld_dz >= Cp and non-null buffers");
  cudaStream_t st = STREAM(stream);
  const long long tiles = (long long)B * h * w;
  static_assert(sizeof(Moments) == 3 * sizeof(float), "Moments packs into three floats");
  // cell S, cell d, tile moments, tile partials, coef
  float* ws = slab_workspace((size_t)tiles * (2 + 3 + 4) + 4, st);
  if (!ws) return D3_ERR_CUDA;
  float* cell_s = ws;
  float* cell_d = cell_s + tiles;
  Moments* tile_m = reinterpret_cast<Moments*>(cell_d + tiles);
  float* part = cell_d + tiles + 3 * tiles;
  float* coef = part + 4 * tiles;
  depth_cell_kernel<<<(unsigned)((tiles + DC_WARPS - 1) / DC_WARPS), DC_WARPS * 32, 0, st>>>(
      logits, ld, tiles, n_bins, min_depth, max_depth, cell_s, cell_d);
  cudaError_t e = cudaPeekAtLastError();
  if (e == cudaSuccess) {
    count_launch();
    depth_moments_kernel<<<(unsigned)tiles, DT_THREADS, 0, st>>>(cell_d, gt, g, min_depth, max_depth, tile_m);
    e = cudaPeekAtLastError();
  }
  if (e == cudaSuccess) {
    count_launch();
    depth_loss_kernel<<<1, DL_THREADS, 0, st>>>(tile_m, tiles, loss, count, coef);
    e = cudaPeekAtLastError();
  }
  if (e == cudaSuccess && (dz_f32 || dz_bf16)) {
    count_launch();
    depth_grad_tile_kernel<<<(unsigned)tiles, DT_THREADS, 0, st>>>(cell_d, gt, g, min_depth, max_depth, coef, part);
    e = cudaPeekAtLastError();
    if (e == cudaSuccess) {
      count_launch();
      const long long n = tiles * Cp;
      const int blocks = (int)std::min<long long>((n + 255) / 256, (long long)sm_count() * 16);
      depth_dz_kernel<<<blocks, 256, 0, st>>>(logits, ld, part, cell_s, cell_d, g, n_bins, Cp, min_depth, max_depth,
                                              dz_f32, (__nv_bfloat16*)dz_bf16, ld_dz);
      e = cudaPeekAtLastError();
    }
  }
  int rc = D3_OK;
  if (e != cudaSuccess) rc = set_error(D3_ERR_CUDA, cudaGetErrorString(e)); else count_launch();
  slab_release(ws, st);
  return rc;
}

int d3_depth_predict_metrics(const float* logits, int ld, const float* gt, int B, int h, int w, int Hl, int Wl,
                             int n_bins, float min_depth, float max_depth, int crop_top, int crop_bottom,
                             int crop_left, int crop_right, double* sums, void* stream) {
  if (B <= 0) return D3_OK;
  SegGeom g;
  if (int rc = depth_geom("d3_depth_predict_metrics", B, h, w, Hl, Wl, n_bins, ld, min_depth, max_depth, g)) return rc;
  if (!logits || !gt || !sums) return set_error(D3_ERR_ARG, "d3_depth_predict_metrics: null buffer");
  cudaStream_t st = STREAM(stream);
  const long long tiles = (long long)B * h * w;
  float* ws = slab_workspace((size_t)tiles * (2 + N_METRICS), st);
  if (!ws) return D3_ERR_CUDA;
  float* cell_s = ws;
  float* cell_d = cell_s + tiles;
  float* tile_sums = cell_d + tiles;
  depth_cell_kernel<<<(unsigned)((tiles + DC_WARPS - 1) / DC_WARPS), DC_WARPS * 32, 0, st>>>(
      logits, ld, tiles, n_bins, min_depth, max_depth, cell_s, cell_d);
  cudaError_t e = cudaPeekAtLastError();
  if (e == cudaSuccess) {
    count_launch();
    depth_metrics_tile_kernel<<<(unsigned)tiles, DT_THREADS, 0, st>>>(
        cell_d, gt, g, min_depth, max_depth, make_int4(crop_top, crop_bottom, crop_left, crop_right), tile_sums);
    e = cudaPeekAtLastError();
  }
  if (e == cudaSuccess) {
    count_launch();
    depth_metrics_image_kernel<<<B, DM_THREADS, 0, st>>>(tile_sums, h * w, sums);
    e = cudaPeekAtLastError();
  }
  int rc = D3_OK;
  if (e != cudaSuccess) rc = set_error(D3_ERR_CUDA, cudaGetErrorString(e)); else count_launch();
  slab_release(ws, st);
  return rc;
}

}  // extern "C"
