// Linear semantic-segmentation probe of a frozen backbone: BatchNorm (no affine) statistics and normalisation of the
// patch-feature rows, the per-pixel cross-entropy of bilinearly upsampled patch logits with its gradient, and the
// argmax confusion matrix at the label resolution.  The head's logits and weight gradients are d3_gemm_bf16, the bias
// gradients d3_colsum_bf16, the update d3_adamw_ema and the crops d3_seg_crop (knn.cu); nothing here multiplies
// matrices.
//
// Upsampling is torch's bilinear F.interpolate with align_corners = False at any ratio: output pixel (y, x) of an
// Hl x Wl map reads source position s = max((y + 0.5) * h / Hl - 0.5, 0), cells y0 = floor(s), y1 = min(y0 + 1, h - 1)
// with weights (1 - (s - y0), s - y0), and the same along x.  The pixels whose (y0, x0) is patch cell (i, j) form tile
// (i, j); they read only the four cells (y0 | y1) x (x0 | x1), so a CTA per tile holds those four logit rows in
// registers and never materialises a full-resolution logit or gradient.
//
// Deterministic: no float atomics.  A tile adds its pixels' gradients for its four cells in a fixed order and writes
// them as one partial per (tile, corner); a second pass adds, for each cell, the (at most four) partials of the tiles
// that touch it in a fixed order.  The loss is summed over tiles in a fixed tree; the valid-pixel count and the
// confusion matrix are integer atomics, whose sums do not depend on order.
#include "ptx.cuh"
#include "d3_internal.h"
#include "bilinear.cuh"

#include <math.h>
#include <stdio.h>

#include <algorithm>

namespace d3 {

// ---------------------------------------------------------------------------------------------------- BatchNorm
// Column statistics of a bf16 [M, N] matrix: CTA (cx, s) adds rows [s * BN_ROWS, (s + 1) * BN_ROWS) of columns
// [2 * (cx * BN_THREADS + t), + 2) in row order, shifted by row 0 (so var = E[d^2] - E[d]^2 does not cancel at large
// means), into slab s = (sum d, sum d^2); slab_combine adds the slabs in order.
constexpr int BN_THREADS = 256;
constexpr int BN_ROWS = 64;

__global__ void __launch_bounds__(BN_THREADS) seg_bn_partial_kernel(const __nv_bfloat16* __restrict__ x, int ld, int M,
                                                                    int N, float* __restrict__ ws) {
  const int c = 2 * (blockIdx.x * BN_THREADS + threadIdx.x);
  if (c >= N) return;
  const int r0 = blockIdx.y * BN_ROWS, r1 = min(M, r0 + BN_ROWS);
  const float2 sh = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(x + c));
  float a1 = 0.f, a2 = 0.f, b1 = 0.f, b2 = 0.f;
  for (int r = r0; r < r1; ++r) {
    const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(x + (size_t)r * ld + c));
    const float da = v.x - sh.x, db = v.y - sh.y;
    a1 += da; a2 += da * da;
    b1 += db; b2 += db * db;
  }
  float* s = ws + (size_t)blockIdx.y * 2 * N;
  s[c] = a1; s[c + 1] = b1;
  s[N + c] = a2; s[N + c + 1] = b2;
}

// mean, biased var of the batch; running_mean / running_var (optional) <- (1 - momentum) * running + momentum * batch,
// with the unbiased variance, as torch's BatchNorm in training mode
__global__ void seg_bn_finalize_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ sums, int M, int N,
                                       float* __restrict__ mean, float* __restrict__ var, float* __restrict__ run_mean,
                                       float* __restrict__ run_var, float momentum) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= N) return;
  const float inv_m = 1.f / (float)M;
  const float d = sums[c] * inv_m;
  const float v = fmaxf(sums[N + c] * inv_m - d * d, 0.f);
  const float mu = __bfloat162float(x[c]) + d;
  mean[c] = mu;
  var[c] = v;
  if (run_mean) {
    const float unbiased = M > 1 ? v * ((float)M / (float)(M - 1)) : v;
    run_mean[c] = (1.f - momentum) * run_mean[c] + momentum * mu;
    run_var[c] = (1.f - momentum) * run_var[c] + momentum * unbiased;
  }
}

// out = bf16((x - mean) * rsqrt(var + eps)), two columns per thread
__global__ void seg_bn_apply_kernel(const __nv_bfloat16* __restrict__ x, int ld, long long M, int N,
                                    const float* __restrict__ mean, const float* __restrict__ var, float eps,
                                    __nv_bfloat16* __restrict__ out, int ld_out) {
  const int half = N / 2;
  const long long n = M * half;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / half;
    const int c = 2 * (int)(i - r * half);
    const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(x + r * ld + c));
    const float ya = (v.x - mean[c]) * rsqrtf(var[c] + eps), yb = (v.y - mean[c + 1]) * rsqrtf(var[c + 1] + eps);
    *reinterpret_cast<uint32_t*>(out + r * ld_out + c) = pack_bf16(ya, yb);
  }
}

// --------------------------------------------------------------------------------------------- upsampling geometry
constexpr int SX_WARPS = 4;
constexpr int SX_THREADS = SX_WARPS * 32;
constexpr int SX_MAX_R = 8;                 // classes per lane: C <= 256

// the four corner logit rows (00, 01, 10, 11) of the lane's classes c = lane + 32 r
template <int R>
__device__ __forceinline__ void seg_load_corners(const float* __restrict__ logits, int ld, const SegGeom& g,
                                                 const SegTile& t, int C, float (&L)[4][R]) {
  const int lane = threadIdx.x & 31;
  const long long base = (long long)t.b * g.h;
  const long long rows[4] = {(base + t.ty) * g.w + t.tx, (base + t.ty) * g.w + t.x1, (base + t.y1) * g.w + t.tx,
                             (base + t.y1) * g.w + t.x1};
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int c = lane + 32 * r;
      L[k][r] = c < C ? logits[rows[k] * ld + c] : 0.f;
    }
}

// bilinear value of the lane's classes at pixel (y, x) of tile t: torch's h0 (w0 L00 + w1 L01) + h1 (w0 L10 + w1 L11)
template <int R>
__device__ __forceinline__ void seg_pixel(const SegGeom& g, const SegTile& t, int y, int x, const float (&L)[4][R],
                                          float (&z)[R], float (&wk)[4]) {
  const float ly = seg_src(y, g.sh) - (float)t.ty, lx = seg_src(x, g.sw) - (float)t.tx;
  const float h0 = 1.f - ly, w0 = 1.f - lx;
#pragma unroll
  for (int r = 0; r < R; ++r) z[r] = h0 * (w0 * L[0][r] + lx * L[1][r]) + ly * (w0 * L[2][r] + lx * L[3][r]);
  wk[0] = h0 * w0; wk[1] = h0 * lx; wk[2] = ly * w0; wk[3] = ly * lx;
}

// ---------------------------------------------------------------------------------------------------- cross-entropy
// One CTA per tile, one warp per pixel (pixel p of the tile's rectangle, row-major, goes to warp p % SX_WARPS), the
// lanes over the classes.  Per pixel: the bilinear logits, their max and sum of exp by butterflies (every lane gets
// the same bits), the loss lse - z[label] (lane 0, in pixel order) and g = softmax - onehot, added into the lane's
// four corner accumulators w_k * g in pixel order.  The warps' accumulators are then added in warp order; corners that
// coincide at the last row / column (y1 == y0, x1 == x0) are folded into one.  part[(tile * 4 + k) * C + c] receives
// corner k, tile_loss[tile] the tile's loss sum, *count the number of valid pixels (label < C; 255 is the ignore label).
template <int R>
__global__ void __launch_bounds__(SX_THREADS, 4) seg_xent_tile_kernel(const float* __restrict__ logits, int ld,
                                                                   const uint8_t* __restrict__ labels, SegGeom g, int C,
                                                                   float* __restrict__ part,
                                                                   float* __restrict__ tile_loss, int* __restrict__ count) {
  __shared__ float acc_s[SX_WARPS][4][R * 32];
  __shared__ float loss_s[SX_WARPS];
  __shared__ int cnt_s[SX_WARPS];
  __shared__ int range[4];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const SegTile t = seg_tile(g, range);
  float L[4][R], acc[4][R];
  seg_load_corners<R>(logits, ld, g, t, C, L);
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int r = 0; r < R; ++r) acc[k][r] = 0.f;
  float loss = 0.f;
  int cnt = 0;
  const int nx = t.x_hi - t.x_lo, np = (t.y_hi - t.y_lo) * nx;
  const uint8_t* lab = labels + (size_t)t.b * g.Hl * g.Wl;
  for (int p = wid; p < np; p += SX_WARPS) {
    const int y = t.y_lo + p / nx, x = t.x_lo + p % nx;
    const int label = lab[(size_t)y * g.Wl + x];
    if (label >= C) continue;                                   // warp-uniform
    float z[R], wk[4];
    seg_pixel<R>(g, t, y, x, L, z, wk);
    float m = -INFINITY, zy = 0.f;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      if (lane + 32 * r < C) m = fmaxf(m, z[r]);
      if (r == (label >> 5)) zy = z[r];
    }
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    zy = __shfl_sync(0xffffffffu, zy, label & 31);
    float s = 0.f;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      z[r] = lane + 32 * r < C ? expf(z[r] - m) : 0.f;
      s += z[r];
    }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    // softmax = exp(z - max) / sum and loss = (max - z[y]) + log(sum), as the linear probe's cross-entropy
    loss += (m - zy) + logf(s);
    ++cnt;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const float gr = z[r] / s - (lane + 32 * r == label ? 1.f : 0.f);
#pragma unroll
      for (int k = 0; k < 4; ++k) acc[k][r] = fmaf(wk[k], gr, acc[k][r]);
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int r = 0; r < R; ++r) acc_s[wid][k][lane + 32 * r] = acc[k][r];
  if (lane == 0) { loss_s[wid] = loss; cnt_s[wid] = cnt; }
  __syncthreads();
  const long long tile = blockIdx.x;
  const bool fold_x = t.x1 == t.tx, fold_y = t.y1 == t.ty;
  for (int c = threadIdx.x; c < C; c += SX_THREADS) {
    float a[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      a[k] = acc_s[0][k][c];
      for (int w = 1; w < SX_WARPS; ++w) a[k] += acc_s[w][k][c];
    }
    if (fold_x) { a[0] += a[1]; a[2] += a[3]; a[1] = 0.f; a[3] = 0.f; }
    if (fold_y) { a[0] += a[2]; a[1] += a[3]; a[2] = 0.f; a[3] = 0.f; }
#pragma unroll
    for (int k = 0; k < 4; ++k) part[(tile * 4 + k) * C + c] = a[k];
  }
  if (threadIdx.x == 0) {
    float l = loss_s[0];
    int n = cnt_s[0];
    for (int w = 1; w < SX_WARPS; ++w) { l += loss_s[w]; n += cnt_s[w]; }
    tile_loss[tile] = l;
    if (n) atomicAdd(count, n);
  }
}

// loss = sum of the tile sums / count (0 when no pixel is valid): thread t adds tiles t, t + 1024, ... in order, then
// a fixed tree over the threads
constexpr int SL_THREADS = 1024;
__global__ void __launch_bounds__(SL_THREADS) seg_loss_kernel(const float* __restrict__ tile_loss, long long n_tiles,
                                                              const int* __restrict__ count, float* __restrict__ loss) {
  __shared__ float red[SL_THREADS];
  float s = 0.f;
  for (long long i = threadIdx.x; i < n_tiles; i += SL_THREADS) s += tile_loss[i];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = SL_THREADS / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) *loss = *count > 0 ? red[0] / (float)*count : 0.f;
}

// dZ[cell, c] = (part[cell, corner 00] + part[cell - 1, corner 01] + part[cell - w, corner 10]
//               + part[cell - w - 1, corner 11]) / count for c < C, 0 for c in [C, Cp); fp32 and / or bf16
__global__ void seg_grad_kernel(const float* __restrict__ part, SegGeom g, int C, int Cp, const int* __restrict__ count,
                                float* __restrict__ dz_f32, __nv_bfloat16* __restrict__ dz_bf16, int ld_dz) {
  const long long n = (long long)g.B * g.h * g.w * Cp;
  const int cntv = *count;
  const float cnt = cntv > 0 ? (float)cntv : 0.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long cell = i / Cp;
    const int c = (int)(i - cell * Cp);
    float v = 0.f;
    if (c < C && cntv > 0) {
      const int x = (int)(cell % g.w), y = (int)((cell / g.w) % g.h);
      v = part[(cell * 4 + 0) * C + c];
      if (x > 0) v += part[((cell - 1) * 4 + 1) * C + c];
      if (y > 0) v += part[((cell - g.w) * 4 + 2) * C + c];
      if (x > 0 && y > 0) v += part[((cell - g.w - 1) * 4 + 3) * C + c];
      v = v / cnt;
    }
    if (dz_f32) dz_f32[cell * ld_dz + c] = v;
    if (dz_bf16) dz_bf16[cell * ld_dz + c] = __float2bfloat16(v);
  }
}

// ------------------------------------------------------------------------------------------- prediction, confusion
// The tiles and warps of the cross-entropy; per pixel the argmax of the bilinear logits (ties to the lower class) and,
// for labels < C, conf[label * C + pred] += 1.  Lane 0 of each warp keeps a run of equal (label, pred) pairs and adds
// it with one 64-bit integer atomic when the pair changes.
template <int R>
__global__ void __launch_bounds__(SX_THREADS, 4) seg_predict_kernel(const float* __restrict__ logits, int ld,
                                                                 const uint8_t* __restrict__ labels, SegGeom g, int C,
                                                                 unsigned long long* __restrict__ conf) {
  __shared__ int range[4];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const SegTile t = seg_tile(g, range);
  float L[4][R];
  seg_load_corners<R>(logits, ld, g, t, C, L);
  const int nx = t.x_hi - t.x_lo, np = (t.y_hi - t.y_lo) * nx;
  const uint8_t* lab = labels + (size_t)t.b * g.Hl * g.Wl;
  long long run_key = -1;
  unsigned long long run_n = 0;
  for (int p = wid; p < np; p += SX_WARPS) {
    const int y = t.y_lo + p / nx, x = t.x_lo + p % nx;
    const int label = lab[(size_t)y * g.Wl + x];
    if (label >= C) continue;
    float z[R], wk[4];
    seg_pixel<R>(g, t, y, x, L, z, wk);
    float bv = -INFINITY;
    int bi = 0x7fffffff;
#pragma unroll
    for (int r = 0; r < R; ++r)
      if (lane + 32 * r < C && (z[r] > bv || bi == 0x7fffffff)) { bv = z[r]; bi = lane + 32 * r; }
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi) || (bi == 0x7fffffff && oi != 0x7fffffff)) { bv = ov; bi = oi; }
    }
    if (lane == 0) {
      const long long key = (long long)label * C + bi;
      if (key != run_key) {
        if (run_n) atomicAdd(conf + run_key, run_n);
        run_key = key;
        run_n = 0;
      }
      ++run_n;
    }
  }
  if (lane == 0 && run_n) atomicAdd(conf + run_key, run_n);
}

}  // namespace d3

using namespace d3;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

namespace {

int seg_geom(const char* who, int B, int h, int w, int Hl, int Wl, int C, SegGeom& g) {
  if (h < 1 || w < 1 || Hl < 1 || Wl < 1 || C < 2 || C > 32 * SX_MAX_R) {
    char msg[160];
    snprintf(msg, sizeof(msg), "%s: need h, w, Hl, Wl >= 1 and 2 <= C <= %d", who, 32 * SX_MAX_R);
    return set_error(D3_ERR_ARG, msg);
  }
  if ((long long)B * h * w > 0x7fffffffLL) return set_error(D3_ERR_ARG, "seg: more than 2^31 - 1 patch cells");
  g = SegGeom{B, h, w, Hl, Wl, (float)h / (float)Hl, (float)w / (float)Wl};
  return D3_OK;
}

}  // namespace

#define SEG_DISPATCH(KERNEL, R_, ...)                     \
  switch (R_) {                                           \
    case 1: KERNEL<1><<<__VA_ARGS__; break;               \
    case 2: KERNEL<2><<<__VA_ARGS__; break;               \
    case 3: KERNEL<3><<<__VA_ARGS__; break;               \
    case 4: KERNEL<4><<<__VA_ARGS__; break;               \
    case 5: KERNEL<5><<<__VA_ARGS__; break;               \
    case 6: KERNEL<6><<<__VA_ARGS__; break;               \
    case 7: KERNEL<7><<<__VA_ARGS__; break;               \
    default: KERNEL<8><<<__VA_ARGS__; break;              \
  }

extern "C" {

int d3_seg_bn_stats(const void* x, int ld, int M, int N, float* mean, float* var, float* run_mean, float* run_var,
                    float momentum, void* stream) {
  if (M <= 0) return D3_OK;
  if (!x || !mean || !var || N < 2 || N % 2 || ld < N || ld % 2 || (uintptr_t)x % 4 || (!run_mean != !run_var))
    return set_error(D3_ERR_ARG, "d3_seg_bn_stats: need N even, ld >= N even, x 4-byte aligned, both running buffers "
                                 "or neither");
  cudaStream_t st = STREAM(stream);
  const int slabs = (M + BN_ROWS - 1) / BN_ROWS;
  float* ws = slab_workspace((size_t)(slabs + 1) * 2 * N, st);
  if (!ws) return D3_ERR_CUDA;
  float* sums = ws + (size_t)slabs * 2 * N;                    // zeroed by slab_workspace
  seg_bn_partial_kernel<<<dim3((N / 2 + BN_THREADS - 1) / BN_THREADS, slabs), BN_THREADS, 0, st>>>(
      (const __nv_bfloat16*)x, ld, M, N, ws);
  cudaError_t e = cudaPeekAtLastError();
  int rc = e == cudaSuccess ? D3_OK : set_error(D3_ERR_CUDA, cudaGetErrorString(e));
  if (!rc) { count_launch(); rc = slab_combine(ws, slabs, 2LL * N, 1, 2 * N, sums, 2LL * N, st); }
  if (!rc) {
    seg_bn_finalize_kernel<<<(N + 255) / 256, 256, 0, st>>>((const __nv_bfloat16*)x, sums, M, N, mean, var, run_mean,
                                                             run_var, momentum);
    e = cudaPeekAtLastError();
    if (e != cudaSuccess) rc = set_error(D3_ERR_CUDA, cudaGetErrorString(e)); else count_launch();
  }
  slab_release(ws, st);
  return rc;
}

int d3_seg_bn_apply(const void* x, int ld, long long M, int N, const float* mean, const float* var, float eps, void* out,
                    int ld_out, void* stream) {
  if (M <= 0) return D3_OK;
  if (!x || !out || !mean || !var || N < 2 || N % 2 || ld < N || ld % 2 || ld_out < N || ld_out % 2 ||
      ((uintptr_t)x | (uintptr_t)out) % 4)
    return set_error(D3_ERR_ARG, "d3_seg_bn_apply: need N, ld, ld_out even (ld, ld_out >= N), 4-byte aligned rows");
  const long long n = M * (N / 2);
  const int blocks = (int)std::min<long long>((n + 255) / 256, (long long)sm_count() * 16);
  seg_bn_apply_kernel<<<blocks, 256, 0, STREAM(stream)>>>((const __nv_bfloat16*)x, ld, M, N, mean, var, eps,
                                                           (__nv_bfloat16*)out, ld_out);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_seg_xent_fwd_bwd(const float* logits, int ld, const void* labels_u8, int B, int h, int w, int Hl, int Wl, int C,
                        int Cp, float* loss, int* count, float* dz_f32, void* dz_bf16, int ld_dz, void* stream) {
  if (B <= 0) return D3_OK;
  SegGeom g;
  if (int rc = seg_geom("d3_seg_xent_fwd_bwd", B, h, w, Hl, Wl, C, g)) return rc;
  if (!logits || !labels_u8 || !loss || !count || ld < C || Cp < C || ((dz_f32 || dz_bf16) && ld_dz < Cp))
    return set_error(D3_ERR_ARG, "d3_seg_xent_fwd_bwd: need ld >= C, Cp >= C, ld_dz >= Cp and non-null buffers");
  cudaStream_t st = STREAM(stream);
  const long long tiles = (long long)B * h * w;
  float* ws = slab_workspace((size_t)tiles * (4 * C + 1), st);
  if (!ws) return D3_ERR_CUDA;
  float* tile_loss = ws + (size_t)tiles * 4 * C;
  cudaError_t e = cudaMemsetAsync(count, 0, sizeof(int), st);
  const int R = (C + 31) / 32;
  if (e == cudaSuccess) {
    SEG_DISPATCH(seg_xent_tile_kernel, R, (unsigned)tiles, SX_THREADS, 0, st>>>(logits, ld, (const uint8_t*)labels_u8,
                                                                               g, C, ws, tile_loss, count))
    e = cudaPeekAtLastError();
  }
  if (e == cudaSuccess) {
    count_launch();
    seg_loss_kernel<<<1, SL_THREADS, 0, st>>>(tile_loss, tiles, count, loss);
    e = cudaPeekAtLastError();
  }
  if (e == cudaSuccess && (dz_f32 || dz_bf16)) {
    count_launch();
    const long long n = tiles * Cp;
    const int blocks = (int)std::min<long long>((n + 255) / 256, (long long)sm_count() * 16);
    seg_grad_kernel<<<blocks, 256, 0, st>>>(ws, g, C, Cp, count, dz_f32, (__nv_bfloat16*)dz_bf16, ld_dz);
    e = cudaPeekAtLastError();
  }
  int rc = D3_OK;
  if (e != cudaSuccess) rc = set_error(D3_ERR_CUDA, cudaGetErrorString(e)); else count_launch();
  slab_release(ws, st);
  return rc;
}

int d3_seg_predict_confusion(const float* logits, int ld, const void* labels_u8, int B, int h, int w, int Hl, int Wl,
                             int C, long long* conf, void* stream) {
  if (B <= 0) return D3_OK;
  SegGeom g;
  if (int rc = seg_geom("d3_seg_predict_confusion", B, h, w, Hl, Wl, C, g)) return rc;
  if (!logits || !labels_u8 || !conf || ld < C)
    return set_error(D3_ERR_ARG, "d3_seg_predict_confusion: need ld >= C and non-null buffers");
  const int R = (C + 31) / 32;
  const unsigned tiles = (unsigned)((long long)B * h * w);
  cudaStream_t st = STREAM(stream);
  SEG_DISPATCH(seg_predict_kernel, R, tiles, SX_THREADS, 0, st>>>(logits, ld, (const uint8_t*)labels_u8, g, C,
                                                                  (unsigned long long*)conf))
  D3_CHECK_LAUNCH();
  return D3_OK;
}

}  // extern "C"
