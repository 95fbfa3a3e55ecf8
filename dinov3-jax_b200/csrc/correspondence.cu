// Keypoint correspondence by nearest neighbour over bilinearly upsampled patch features (the SPair-71k style semantic
// correspondence evaluation): the source descriptors at the keypoints, the per-patch Gram of a target map, and the
// exact cosine argmax over every pixel of the upsampled target, without any full-resolution feature map.  The
// patch-level similarities s = Q . F_t^T come from d3_gemm_bf16 (fp32 results); nothing here multiplies matrices.
//
// Upsampling: U(y, x) of an [h, w, D] map at Hs x Ws is torch's bilinear F.interpolate(align_corners = False), the
// geometry of bilinear.cuh: corners A = (y0, x0), B = (y0, x1), C = (y1, x0), D = (y1, x1) with weights
// wA = hy hx, wB = hy lx, wC = ly hx, wD = ly lx (hy = 1 - ly, hx = 1 - lx); at the last row / column the two corners
// are the same cell.
//
// Descriptors: q_k = U_s(y_k, x_k) / ||U_s(y_k, x_k)||, blended in fp32 as torch writes it (hy (hx A + lx B) +
// ly (hx C + lx D)), normalised in fp32 and rounded to bf16; qnorm_k is the norm of the rounded row, so that the
// reported cosine is that of the descriptor the GEMM reads.
//
// Gram: for every patch (i, j) of a target map, in fp32 from the bf16 rows: g0 = <f_ij, f_ij>, g1 = <f_ij, f_i,j+1>
// (right), g2 = <f_ij, f_i+1,j> (lower), g3 = <f_ij, f_i+1,j+1> (lower right), g4 = <f_ij, f_i+1,j-1> (lower left); a
// neighbour outside the map gives 0.  Lane l adds channels [8 l + 256 i, 8 l + 256 i + 8) in i order, then a fixed
// butterfly over the lanes.
//
// Argmax: because the dot product commutes with the blend, <q, U(y, x)> = wA sA + wB sB + wC sC + wD sD with
// s = <q, f> at the four corners, and ||U||^2 = sum_ab w_a w_b <f_a, f_b> over the corner pairs, which the Gram holds
// (a corner pair that coincides at the last row / column reads the coinciding entry).  Where the two rows (columns)
// of corners are the same cell, its two weights are folded into one (ly = 0, lx = 0): the same U, and every pixel of
// such a clamped band computes the same bits, so its equal cosines tie exactly.  The cosine is
// <q, U> / (qnorm sqrt(||U||^2)), 0 where ||U||^2 <= 0.  Each CTA owns one (keypoint, cell) tile of bilinear.cuh's
// seg_tile and writes the tile's best (cosine, pixel index) at patch resolution; a second kernel takes the best of the
// h w tiles per keypoint.  Ties go to the lowest pixel index y Ws + x at every step, so the result does not depend on
// the order of the comparisons: no atomics, the same bits on every run.
#include "ptx.cuh"
#include "d3_internal.h"
#include "bilinear.cuh"

#include <math.h>
#include <stdint.h>

#include <climits>

namespace d3 {

constexpr int CD_WARPS = 4;                 // descriptors: one warp per keypoint
constexpr int CG_WARPS = 8;                 // Gram: one warp per patch
constexpr int CA_THREADS = 128;             // argmax: one CTA per (keypoint, cell) tile
constexpr int CR_WARPS = 4;                 // argmax merge: one warp per keypoint
constexpr int CORR_GRAM = 5;

__device__ __forceinline__ void bf16x8(const uint4& u, float (&v)[8]) {
  const uint32_t p[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = unpack_bf16(p[i]);
    v[2 * i] = f.x;
    v[2 * i + 1] = f.y;
  }
}

// ------------------------------------------------------------------------------------------------ descriptors
__global__ void __launch_bounds__(CD_WARPS * 32) corr_desc_kernel(const __nv_bfloat16* __restrict__ feats, int ld,
                                                                  const int* __restrict__ kp, int K, SegGeom g, int D,
                                                                  __nv_bfloat16* __restrict__ out, int ldo,
                                                                  float* __restrict__ qnorm) {
  const int lane = threadIdx.x & 31;
  const int k = blockIdx.x * CD_WARPS + (threadIdx.x >> 5);
  if (k >= K) return;
  const int m = kp[3 * k], x = kp[3 * k + 1], y = kp[3 * k + 2];
  const float fy = seg_src(y, g.sh), fx = seg_src(x, g.sw);
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = min(y0 + 1, g.h - 1), x1 = min(x0 + 1, g.w - 1);
  const float ly = fy - (float)y0, lx = fx - (float)x0;
  const float hy = 1.f - ly, hx = 1.f - lx;
  const long long base = (long long)m * g.h;
  const __nv_bfloat16* rA = feats + ((base + y0) * g.w + x0) * ld;
  const __nv_bfloat16* rB = feats + ((base + y0) * g.w + x1) * ld;
  const __nv_bfloat16* rC = feats + ((base + y1) * g.w + x0) * ld;
  const __nv_bfloat16* rD = feats + ((base + y1) * g.w + x1) * ld;
  float ss = 0.f;
  for (int pass = 0; pass < 2; ++pass) {
    const float inv = pass == 0 ? 0.f : (ss > 0.f ? 1.f / sqrtf(ss) : 0.f);
    float rs = 0.f;
    for (int c = 8 * lane; c < D; c += 256) {
      float a[8], b[8], cc[8], d[8], u[8];
      bf16x8(*reinterpret_cast<const uint4*>(rA + c), a);
      bf16x8(*reinterpret_cast<const uint4*>(rB + c), b);
      bf16x8(*reinterpret_cast<const uint4*>(rC + c), cc);
      bf16x8(*reinterpret_cast<const uint4*>(rD + c), d);
#pragma unroll
      for (int i = 0; i < 8; ++i) u[i] = hy * (hx * a[i] + lx * b[i]) + ly * (hx * cc[i] + lx * d[i]);
      if (pass == 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i) rs = fmaf(u[i], u[i], rs);
      } else {
        __align__(16) __nv_bfloat16 o[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          o[i] = __float2bfloat16(u[i] * inv);
          const float r = __bfloat162float(o[i]);
          rs = fmaf(r, r, rs);
        }
        *reinterpret_cast<uint4*>(out + (size_t)k * ldo + c) = *reinterpret_cast<const uint4*>(o);
      }
    }
    rs = warp_sum(rs);
    if (pass == 0) ss = rs;
    else if (lane == 0) qnorm[k] = sqrtf(rs);
  }
}

// ------------------------------------------------------------------------------------------------ Gram
__global__ void __launch_bounds__(CG_WARPS * 32) corr_gram_kernel(const __nv_bfloat16* __restrict__ feats, int ld,
                                                                  int n_maps, int h, int w, int D,
                                                                  float* __restrict__ gram) {
  const int lane = threadIdx.x & 31;
  const long long p = (long long)blockIdx.x * CG_WARPS + (threadIdx.x >> 5);
  if (p >= (long long)n_maps * h * w) return;
  const int j = (int)(p % w), i = (int)((p / w) % h);
  const bool right = j + 1 < w, lower = i + 1 < h;
  // neighbour rows; one that does not exist points at the patch itself and its sum is discarded
  const __nv_bfloat16* r0 = feats + p * ld;
  const __nv_bfloat16* nb[4] = {right ? r0 + ld : r0, lower ? r0 + (long long)w * ld : r0,
                                right && lower ? r0 + (long long)(w + 1) * ld : r0,
                                j > 0 && lower ? r0 + (long long)(w - 1) * ld : r0};
  float acc[CORR_GRAM] = {0.f, 0.f, 0.f, 0.f, 0.f};
  for (int c = 8 * lane; c < D; c += 256) {
    float a[8];
    bf16x8(*reinterpret_cast<const uint4*>(r0 + c), a);
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[0] = fmaf(a[e], a[e], acc[0]);
#pragma unroll
    for (int n = 0; n < 4; ++n) {
      float b[8];
      bf16x8(*reinterpret_cast<const uint4*>(nb[n] + c), b);
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[n + 1] = fmaf(a[e], b[e], acc[n + 1]);
    }
  }
#pragma unroll
  for (int n = 0; n < CORR_GRAM; ++n) acc[n] = warp_sum(acc[n]);
  if (lane == 0) {
    float* gp = gram + p * CORR_GRAM;
    gp[0] = acc[0];
    gp[1] = right ? acc[1] : 0.f;
    gp[2] = lower ? acc[2] : 0.f;
    gp[3] = right && lower ? acc[3] : 0.f;
    gp[4] = j > 0 && lower ? acc[4] : 0.f;
  }
}

// ------------------------------------------------------------------------------------------------ argmax
// (v, i) beats (bv, bi): larger cosine, or the same cosine at a lower pixel index
__device__ __forceinline__ bool corr_better(float v, int i, float bv, int bi) {
  return v > bv || (v == bv && i < bi);
}

__device__ __forceinline__ void corr_warp_best(float& bv, int& bi) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float v = __shfl_xor_sync(0xffffffffu, bv, o);
    const int i = __shfl_xor_sync(0xffffffffu, bi, o);
    if (corr_better(v, i, bv, bi)) { bv = v; bi = i; }
  }
}

// Tile b * h w + cell of seg_tile: keypoint b = t.b, its similarity row sim[b * lds + ...] over the target's h w
// patches.  part_v / part_i [K h w] receive the tile's best cosine and pixel index.
__global__ void __launch_bounds__(CA_THREADS) corr_argmax_tile_kernel(const float* __restrict__ sim, int lds,
                                                                      const float* __restrict__ gram,
                                                                      const float* __restrict__ qnorm, SegGeom g,
                                                                      float* __restrict__ part_v,
                                                                      int* __restrict__ part_i) {
  __shared__ int range[4];
  __shared__ float red_v[CA_THREADS / 32];
  __shared__ int red_i[CA_THREADS / 32];
  const SegTile t = seg_tile(g, range);
  const int cA = t.ty * g.w + t.tx, cB = t.ty * g.w + t.x1, cC = t.y1 * g.w + t.tx, cD = t.y1 * g.w + t.x1;
  const float* srow = sim + (size_t)t.b * lds;
  const float sA = srow[cA], sB = srow[cB], sC = srow[cC], sD = srow[cD];
  const float* gA = gram + (size_t)cA * CORR_GRAM;
  const float* gB = gram + (size_t)cB * CORR_GRAM;
  const bool col1 = t.x1 == t.tx, row1 = t.y1 == t.ty;          // the corners coincide along x / along y
  const float AA = gA[0], BB = gB[0], CC = gram[(size_t)cC * CORR_GRAM], DD = gram[(size_t)cD * CORR_GRAM];
  const float AB = col1 ? AA : gA[1];
  const float AC = row1 ? AA : gA[2];
  const float AD = row1 ? AB : (col1 ? AC : gA[3]);
  const float BD = row1 ? BB : gB[2];
  const float CD = col1 ? CC : gram[(size_t)cC * CORR_GRAM + 1];
  const float BC = col1 ? AC : (row1 ? AB : gB[4]);
  const float qn = qnorm[t.b];
  const int tw = t.x_hi - t.x_lo, np = (t.y_hi - t.y_lo) * tw;
  float bv = -INFINITY;
  int bi = INT_MAX;
  for (int i = threadIdx.x; i < np; i += CA_THREADS) {             // increasing pixel index within the thread
    const int y = t.y_lo + i / tw, x = t.x_lo + i % tw;
    const float ly = row1 ? 0.f : seg_src(y, g.sh) - (float)t.ty;
    const float lx = col1 ? 0.f : seg_src(x, g.sw) - (float)t.tx;
    const float hy = 1.f - ly, hx = 1.f - lx;
    const float wA = hy * hx, wB = hy * lx, wC = ly * hx, wD = ly * lx;
    const float num = wA * sA + wB * sB + wC * sC + wD * sD;
    const float sq = wA * wA * AA + wB * wB * BB + wC * wC * CC + wD * wD * DD;
    const float cross = wA * (wB * AB + wC * AC + wD * AD) + wB * (wC * BC + wD * BD) + wC * wD * CD;
    const float n2 = sq + 2.f * cross;
    const float den = qn * sqrtf(fmaxf(n2, 0.f));
    const float v = den > 0.f ? num / den : 0.f;
    const int idx = y * g.Wl + x;
    if (corr_better(v, idx, bv, bi)) { bv = v; bi = idx; }
  }
  corr_warp_best(bv, bi);
  if ((threadIdx.x & 31) == 0) { red_v[threadIdx.x >> 5] = bv; red_i[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int wi = 1; wi < CA_THREADS / 32; ++wi)
      if (corr_better(red_v[wi], red_i[wi], bv, bi)) { bv = red_v[wi]; bi = red_i[wi]; }
    part_v[blockIdx.x] = bv;
    part_i[blockIdx.x] = bi;
  }
}

__global__ void __launch_bounds__(CR_WARPS * 32) corr_argmax_merge_kernel(const float* __restrict__ part_v,
                                                                          const int* __restrict__ part_i, int K,
                                                                          int cells, int Wl, int* __restrict__ xy,
                                                                          float* __restrict__ cosine) {
  const int lane = threadIdx.x & 31;
  const int k = blockIdx.x * CR_WARPS + (threadIdx.x >> 5);
  if (k >= K) return;
  float bv = -INFINITY;
  int bi = INT_MAX;
  for (int c = lane; c < cells; c += 32) {
    const float v = part_v[(size_t)k * cells + c];
    const int i = part_i[(size_t)k * cells + c];
    if (corr_better(v, i, bv, bi)) { bv = v; bi = i; }
  }
  corr_warp_best(bv, bi);
  if (lane == 0) {
    xy[2 * k] = bi % Wl;
    xy[2 * k + 1] = bi / Wl;
    cosine[k] = bv;
  }
}

}  // namespace d3

using namespace d3;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

int d3_corr_descriptors(const void* feats, int ld, int n_maps, int h, int w, int D, int out_h, int out_w,
                        const int* kp, int K, void* out, int ldo, float* qnorm, void* stream) {
  if (K < 0 || h < 1 || w < 1 || n_maps < 1 || out_h < 1 || out_w < 1 || D < 8 || D % 8 || ld < D || ld % 8 ||
      ldo < D || ldo % 8)
    return set_error(D3_ERR_ARG, "d3_corr_descriptors: need K >= 0, h, w, n_maps, out_h, out_w >= 1, D a positive "
                                 "multiple of 8 and ld, ldo >= D multiples of 8");
  if (K == 0) return D3_OK;
  if (!feats || !kp || !out || !qnorm || (uintptr_t)feats % 16 || (uintptr_t)out % 16)
    return set_error(D3_ERR_ARG, "d3_corr_descriptors: need non-null buffers, feats and out 16-byte aligned");
  for (int k = 0; k < K; ++k)
    if (kp[3 * k] < 0 || kp[3 * k] >= n_maps || kp[3 * k + 1] < 0 || kp[3 * k + 1] >= out_w || kp[3 * k + 2] < 0 ||
        kp[3 * k + 2] >= out_h)
      return set_error(D3_ERR_ARG, "d3_corr_descriptors: a keypoint's map is outside [0, n_maps) or its pixel "
                                   "outside [0, out_w) x [0, out_h)");
  cudaStream_t st = STREAM(stream);
  float* ws = slab_workspace((size_t)3 * K, st);
  if (!ws) return D3_ERR_CUDA;
  cudaError_t e = cudaMemcpyAsync(ws, kp, sizeof(int) * 3 * (size_t)K, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) {
    const SegGeom g{1, h, w, out_h, out_w, (float)h / (float)out_h, (float)w / (float)out_w};
    corr_desc_kernel<<<(K + CD_WARPS - 1) / CD_WARPS, CD_WARPS * 32, 0, st>>>(
        (const __nv_bfloat16*)feats, ld, reinterpret_cast<const int*>(ws), K, g, D, (__nv_bfloat16*)out, ldo, qnorm);
    e = cudaPeekAtLastError();
  }
  int rc = D3_OK;
  if (e != cudaSuccess) rc = set_error(D3_ERR_CUDA, cudaGetErrorString(e)); else count_launch();
  slab_release(ws, st);
  return rc;
}

int d3_corr_gram(const void* feats, int ld, int n_maps, int h, int w, int D, float* gram, void* stream) {
  if (n_maps < 0 || h < 1 || w < 1 || D < 8 || D % 8 || ld < D || ld % 8)
    return set_error(D3_ERR_ARG, "d3_corr_gram: need n_maps >= 0, h, w >= 1, D a positive multiple of 8 and ld >= D "
                                 "a multiple of 8");
  if (n_maps == 0) return D3_OK;
  if (!feats || !gram || (uintptr_t)feats % 16)
    return set_error(D3_ERR_ARG, "d3_corr_gram: need non-null buffers, feats 16-byte aligned");
  const long long P = (long long)n_maps * h * w;
  corr_gram_kernel<<<(unsigned)((P + CG_WARPS - 1) / CG_WARPS), CG_WARPS * 32, 0, STREAM(stream)>>>(
      (const __nv_bfloat16*)feats, ld, n_maps, h, w, D, gram);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_corr_argmax(const float* sim, int lds, const float* gram, const float* qnorm, int K, int h, int w, int out_h,
                   int out_w, int* xy, float* cosine, void* stream) {
  if (K < 0 || h < 1 || w < 1 || out_h < 1 || out_w < 1 || lds < h * w || (long long)out_h * out_w > INT_MAX ||
      (long long)K * h * w > INT_MAX)
    return set_error(D3_ERR_ARG, "d3_corr_argmax: need K >= 0, h, w, out_h, out_w >= 1, lds >= h w and fewer than "
                                 "2^31 pixels and tiles");
  if (K == 0) return D3_OK;
  if (!sim || !gram || !qnorm || !xy || !cosine)
    return set_error(D3_ERR_ARG, "d3_corr_argmax: null buffer");
  cudaStream_t st = STREAM(stream);
  const int tiles = K * h * w;
  float* ws = slab_workspace((size_t)2 * tiles, st);
  if (!ws) return D3_ERR_CUDA;
  float* part_v = ws;
  int* part_i = reinterpret_cast<int*>(ws + tiles);
  const SegGeom g{K, h, w, out_h, out_w, (float)h / (float)out_h, (float)w / (float)out_w};
  corr_argmax_tile_kernel<<<tiles, CA_THREADS, 0, st>>>(sim, lds, gram, qnorm, g, part_v, part_i);
  cudaError_t e = cudaPeekAtLastError();
  if (e == cudaSuccess) {
    count_launch();
    corr_argmax_merge_kernel<<<(K + CR_WARPS - 1) / CR_WARPS, CR_WARPS * 32, 0, st>>>(part_v, part_i, K, h * w,
                                                                                       out_w, xy, cosine);
    e = cudaPeekAtLastError();
  }
  int rc = D3_OK;
  if (e != cudaSuccess) rc = set_error(D3_ERR_CUDA, cudaGetErrorString(e)); else count_launch();
  slab_release(ws, st);
  return rc;
}

}  // extern "C"
