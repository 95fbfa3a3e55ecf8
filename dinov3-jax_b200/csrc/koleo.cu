// Top-k KoLeo over gathered rows (loss/koleo_loss.py:39-70, KoLeoLossDistributed), forward and backward in one call.
//
// x [N, D] fp32 holds the rows of every rank in rank order.  A loss group is the row range [g0, g0 + gn); this rank's
// B rows [row0, row0 + B) lie inside it.  For every local row i:
//   xn = x / (||x|| + eps)                                   (every row of the group)
//   nbr(i, 0..k-1) = the k largest fp32 dots xn_i . xn_j over the group's rows j != row0 + i, ties to the lower j
//   L = -1/(B k) sum_{i, s} log(||xn_i - xn_nbr(i,s)|| + eps + eps)
//   metric += w_metric * L;  dx[j] += w_grad * dL/dx_j for every row j of the group (rows outside it are untouched)
// parity unpinned: the reference's own distributed KoLeo does not run (it normalises without keepdims), so these are
// upstream DINOv3's semantics written out.
//
//   koleo_topk_norm_kernel  one CTA per group row: the norm and the normalised row (in scratch).
//   koleo_topk_scan_kernel  grid (column chunks, tiles of KT_RT local rows): each warp takes every KT_NW-th column of
//                           its chunk, forms the KT_RT dots with the tile's rows (held in shared memory) in a fixed
//                           lane order and a butterfly sum, and keeps a sorted top-k per (warp, row); the warps' lists
//                           are merged into the chunk's top-k.
//   koleo_topk_loss_kernel  one CTA per local row: the top-k of the chunks' candidates (k rounds of a block-wide
//                           selection of the best candidate after the previous one, in the (dot desc, index asc) total
//                           order, so the result does not depend on the chunking), the distances, the row's loss
//                           term and each pair's gradient coefficient.
//   koleo_topk_bwd_kernel   one CTA per group row j, a gather: j's own pairs (if j is local), then the (i, slot) pairs
//                           that chose j in (i, slot) order, then the backward through the normalisation.
//   koleo_topk_metric_kernel the row terms summed in a fixed tree into metric.
// No atomics: the same bits on every run.
#include <math_constants.h>
#include "ptx.cuh"
#include "d3_internal.h"

#include <math.h>
#include <stdint.h>

#include <algorithm>

namespace d3 {

constexpr int KT_THREADS = 256;
constexpr int KT_NW = KT_THREADS / 32;
constexpr int KT_RT = 8;                 // local rows per scan CTA
constexpr int KT_KMAX = 16;
constexpr int KT_MIN_CHUNK = 64;         // columns per scan CTA at least
constexpr int KT_MAX_CHUNKS = 512;
constexpr int KT_MAX_D = 6144;           // KT_RT rows of D floats in shared memory

__device__ __forceinline__ float kt_block_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();                      // red may still be read by a previous call
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
  for (int w = 0; w < KT_NW; ++w) t += red[w];
  return t;
}
// (v, j) comes before (bv, bj) in the (dot desc, index asc) order; bj < 0 is an empty slot.  A total order only for
// dots that are not NaN: the scan stores a NaN dot (a non-finite row) as -inf, below every number, so it is never
// preferred and ties by index like any other value.
__device__ __forceinline__ bool kt_better(float v, int j, float bv, int bj) {
  return bj < 0 || v > bv || (v == bv && j < bj);
}

__global__ void __launch_bounds__(KT_THREADS) koleo_topk_norm_kernel(const float4* __restrict__ x,
                                                                      float4* __restrict__ xn, float* __restrict__ nrm,
                                                                      int g0, int D4, float eps) {
  __shared__ float red[KT_NW];
  const long j = g0 + blockIdx.x;
  const float4* xr = x + j * D4;
  float s = 0.f;
  for (int q = threadIdx.x; q < D4; q += KT_THREADS) {
    const float4 v = xr[q];
    s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  const float n = sqrtf(kt_block_sum(s, red));
  if (threadIdx.x == 0) nrm[j] = n;
  const float inv = 1.f / (n + eps);
  for (int q = threadIdx.x; q < D4; q += KT_THREADS) {
    const float4 v = xr[q];
    xn[j * D4 + q] = make_float4(v.x * inv, v.y * inv, v.z * inv, v.w * inv);
  }
}

// cand_v / cand_j [B][C][k]: chunk c's top-k of local row i (j = -1: fewer than k columns in the chunk)
__global__ void __launch_bounds__(KT_THREADS) koleo_topk_scan_kernel(const float4* __restrict__ xn, int D4, int g0,
                                                                      int gn, int row0, int B, int k, int chunk,
                                                                      float* __restrict__ cand_v,
                                                                      int* __restrict__ cand_j) {
  extern __shared__ float4 rows[];                         // [KT_RT][D4]
  __shared__ float lv[KT_NW][KT_RT][KT_KMAX];
  __shared__ int lj[KT_NW][KT_RT][KT_KMAX];
  __shared__ int head[KT_RT][KT_NW];
  const int C = gridDim.x, c = blockIdx.x, i0 = blockIdx.y * KT_RT;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int e = threadIdx.x; e < KT_RT * D4; e += KT_THREADS) {
    const int r = e / D4, q = e - r * D4;
    rows[e] = i0 + r < B ? xn[(long)(row0 + i0 + r) * D4 + q] : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (int e = threadIdx.x; e < KT_NW * KT_RT * KT_KMAX; e += KT_THREADS) {
    (&lv[0][0][0])[e] = -CUDART_INF_F;
    (&lj[0][0][0])[e] = -1;
  }
  __syncthreads();
  const int j_begin = g0 + c * chunk, j_end = min(j_begin + chunk, g0 + gn);
  // lane r keeps the list of tile row r; a column is skipped for the row whose own gathered index it is
  const int my_row = i0 + lane;
  const bool keeps = lane < KT_RT && my_row < B;
  float* Lv = lv[warp][lane < KT_RT ? lane : 0];
  int* Lj = lj[warp][lane < KT_RT ? lane : 0];
  for (int j = j_begin + warp; j < j_end; j += KT_NW) {
    float acc[KT_RT];
#pragma unroll
    for (int r = 0; r < KT_RT; ++r) acc[r] = 0.f;
    const float4* xj = xn + (long)j * D4;
    for (int q = lane; q < D4; q += 32) {
      const float4 b = xj[q];
#pragma unroll
      for (int r = 0; r < KT_RT; ++r) {
        const float4 a = rows[r * D4 + q];
        acc[r] += a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
      }
    }
    float mine = 0.f;
#pragma unroll
    for (int r = 0; r < KT_RT; ++r) {
      const float s = warp_sum(acc[r]);
      if (lane == r) mine = s;
    }
    if (mine != mine) mine = -CUDART_INF_F;
    if (keeps && j != row0 + my_row && kt_better(mine, j, Lv[k - 1], Lj[k - 1])) {
      int p = k - 1;
      while (p > 0 && kt_better(mine, j, Lv[p - 1], Lj[p - 1])) {
        Lv[p] = Lv[p - 1];
        Lj[p] = Lj[p - 1];
        --p;
      }
      Lv[p] = mine;
      Lj[p] = j;
    }
  }
  __syncthreads();
  // merge the warps' sorted lists of row r into the chunk's top-k (thread r)
  const int r = threadIdx.x;
  if (r < KT_RT && i0 + r < B) {
    for (int w = 0; w < KT_NW; ++w) head[r][w] = 0;
    const long out = ((long)(i0 + r) * C + c) * k;
    for (int s = 0; s < k; ++s) {
      int bw = -1;
      float bv = -CUDART_INF_F;
      int bj = -1;
      for (int w = 0; w < KT_NW; ++w) {
        const int h = head[r][w];
        if (h < k && lj[w][r][h] >= 0 && kt_better(lv[w][r][h], lj[w][r][h], bv, bj)) {
          bw = w;
          bv = lv[w][r][h];
          bj = lj[w][r][h];
        }
      }
      if (bw >= 0) ++head[r][bw];
      cand_v[out + s] = bv;
      cand_j[out + s] = bj;
    }
  }
}

__global__ void __launch_bounds__(KT_THREADS) koleo_topk_loss_kernel(const float4* __restrict__ xn, int D4,
                                                                      const float* __restrict__ cand_v,
                                                                      const int* __restrict__ cand_j, int C, int k,
                                                                      int row0, int B, float eps, float w_metric,
                                                                      float w_grad, int* __restrict__ nbr,
                                                                      float* __restrict__ coef,
                                                                      float* __restrict__ row_loss) {
  __shared__ float red[KT_NW];
  __shared__ float wv[KT_NW];
  __shared__ int wj[KT_NW];
  __shared__ float pv;
  __shared__ int pj;
  const int i = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* cv = cand_v + (long)i * C * k;
  const int* cj = cand_j + (long)i * C * k;
  const int n = C * k;
  for (int s = 0; s < k; ++s) {
    float bv = -CUDART_INF_F;
    int bj = -1;
    for (int e = threadIdx.x; e < n; e += KT_THREADS) {
      const float v = cv[e];
      const int j = cj[e];
      // strictly after the previous selection in the total order (every column appears in one chunk at most)
      if (j >= 0 && (s == 0 || kt_better(pv, pj, v, j)) && kt_better(v, j, bv, bj)) { bv = v; bj = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
      if (oj >= 0 && kt_better(ov, oj, bv, bj)) { bv = ov; bj = oj; }
    }
    if (lane == 0) { wv[warp] = bv; wj[warp] = bj; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < KT_NW; ++w)
        if (wj[w] >= 0 && kt_better(wv[w], wj[w], bv, bj)) { bv = wv[w]; bj = wj[w]; }
      // every candidate is a number and gn - 1 >= k columns were scanned, so bj >= 0; the row itself (distance 0,
      // no gradient) stands in if that ever fails, so no index leaves the group
      if (bj < 0) bj = row0 + i;
      pv = bv;
      pj = bj;
      nbr[(long)i * k + s] = bj;
    }
    __syncthreads();
  }
  const float4* xi = xn + (long)(row0 + i) * D4;
  const float scale = 1.f / ((float)B * k);
  float total = 0.f;
  for (int s = 0; s < k; ++s) {
    const float4* xj = xn + (long)nbr[(long)i * k + s] * D4;
    float dd = 0.f;
    for (int q = threadIdx.x; q < D4; q += KT_THREADS) {
      const float4 a = xi[q], b = xj[q];
      const float t0 = a.x - b.x, t1 = a.y - b.y, t2 = a.z - b.z, t3 = a.w - b.w;
      dd += t0 * t0 + t1 * t1 + t2 * t2 + t3 * t3;
    }
    dd = kt_block_sum(dd, red);
    if (threadIdx.x == 0) {
      const float dn = sqrtf(dd);
      const float dist = dn + eps;                        // pairwise_distance(...) + eps
      total += logf(dist + eps);
      // d(-w/(B k) * log(dist + eps))/d(delta) = -w/(B k) / (dist + eps) * delta / ||delta||
      coef[(long)i * k + s] = dn > 0.f ? -w_grad * scale / (dist + eps) / dn : 0.f;
    }
  }
  if (threadIdx.x == 0) row_loss[i] = -w_metric * scale * total;
}

__global__ void __launch_bounds__(KT_THREADS) koleo_topk_bwd_kernel(const float4* __restrict__ x,
                                                                     const float4* __restrict__ xn,
                                                                     const float* __restrict__ nrm,
                                                                     const int* __restrict__ nbr,
                                                                     const float* __restrict__ coef, int D4, int g0,
                                                                     int row0, int B, int k, float eps,
                                                                     float4* __restrict__ dx) {
  extern __shared__ float4 g[];                            // [D4] gradient w.r.t. xn_j (each thread owns its q)
  __shared__ float red[KT_NW];
  __shared__ unsigned char hit[KT_THREADS];
  const long j = g0 + blockIdx.x;
  const float4* xj = xn + j * D4;
  for (int q = threadIdx.x; q < D4; q += KT_THREADS) g[q] = make_float4(0.f, 0.f, 0.f, 0.f);
  bool any = false;
  if (j >= row0 && j < row0 + B) {                         // j's own pairs: + coef * (xn_j - xn_nbr)
    const long i = j - row0;
    for (int s = 0; s < k; ++s) {
      const float cf = coef[i * k + s];
      const float4* xm = xn + (long)nbr[i * k + s] * D4;
      for (int q = threadIdx.x; q < D4; q += KT_THREADS) {
        const float4 a = xj[q], b = xm[q];
        float4 t = g[q];
        t.x += cf * (a.x - b.x); t.y += cf * (a.y - b.y); t.z += cf * (a.z - b.z); t.w += cf * (a.w - b.w);
        g[q] = t;
      }
    }
    any = true;
  }
  const int P = B * k;
  for (int base = 0; base < P; base += KT_THREADS) {       // pairs that chose j: - coef * (xn_i - xn_j)
    const int p = base + threadIdx.x;
    const bool h = p < P && nbr[p] == j;
    hit[threadIdx.x] = h;
    if (!__syncthreads_or(h)) continue;
    any = true;
    const int n = min(KT_THREADS, P - base);
    for (int t = 0; t < n; ++t) {
      if (!hit[t]) continue;
      const int pp = base + t;
      const float cf = coef[pp];
      const float4* xi = xn + (long)(row0 + pp / k) * D4;
      for (int q = threadIdx.x; q < D4; q += KT_THREADS) {
        const float4 a = xi[q], b = xj[q];
        float4 u = g[q];
        u.x -= cf * (a.x - b.x); u.y -= cf * (a.y - b.y); u.z -= cf * (a.z - b.z); u.w -= cf * (a.w - b.w);
        g[q] = u;
      }
    }
    __syncthreads();                                       // hit[] is rewritten by the next round
  }
  if (!any) return;                                        // uniform over the block: nothing reaches this row
  // dx_j += J_norm^T g = g / (n + eps) - x_j (x_j . g) / ((n + eps)^2 n)
  const float4* xr = x + j * D4;
  float dot = 0.f;
  for (int q = threadIdx.x; q < D4; q += KT_THREADS) {
    const float4 a = xr[q], b = g[q];
    dot += a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
  }
  dot = kt_block_sum(dot, red);
  const float n = nrm[j];
  const float inv = 1.f / (n + eps);
  const float c2 = n > 0.f ? dot * inv * inv / n : 0.f;
  for (int q = threadIdx.x; q < D4; q += KT_THREADS) {
    const float4 a = xr[q], b = g[q];
    float4 o = dx[j * D4 + q];
    o.x += b.x * inv - a.x * c2; o.y += b.y * inv - a.y * c2; o.z += b.z * inv - a.z * c2; o.w += b.w * inv - a.w * c2;
    dx[j * D4 + q] = o;
  }
}

__global__ void __launch_bounds__(KT_THREADS) koleo_topk_metric_kernel(const float* __restrict__ row_loss, int B,
                                                                        float* __restrict__ metric) {
  __shared__ float sh[KT_THREADS];
  float s = 0.f;
  for (int i = threadIdx.x; i < B; i += KT_THREADS) s += row_loss[i];
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int w = KT_THREADS / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) sh[threadIdx.x] += sh[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) metric[0] += sh[0];
}

}  // namespace d3

using namespace d3;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

int d3_koleo_topk_rows(const float* x, int N, int D, int g0, int gn, int row0, int B, int topk, float eps,
                       float w_metric, float w_grad, float* scratch, long long scratch_floats, float* metric, float* dx,
                       void* stream) {
  if (N < 2 || D < 4 || D % 4 || D > KT_MAX_D)
    return set_error(D3_ERR_ARG, "d3_koleo_topk_rows: need N >= 2 and D a multiple of 4 in [4, 6144]");
  if (g0 < 0 || gn < 2 || gn > N - g0)
    return set_error(D3_ERR_ARG, "d3_koleo_topk_rows: the group [g0, g0 + gn) must hold >= 2 rows inside [0, N)");
  if (B < 1 || row0 < g0 || B > g0 + gn - row0)
    return set_error(D3_ERR_ARG, "d3_koleo_topk_rows: the local rows [row0, row0 + B) must lie inside the group");
  if (topk < 1 || topk > KT_KMAX || topk > gn - 1)
    return set_error(D3_ERR_ARG, "d3_koleo_topk_rows: need 1 <= topk <= min(16, rows in the group - 1)");
  if (!x || !scratch || !metric || !dx)
    return set_error(D3_ERR_ARG, "d3_koleo_topk_rows: null buffer");
  if (((uintptr_t)x | (uintptr_t)scratch | (uintptr_t)dx) % 16)
    return set_error(D3_ERR_ARG, "d3_koleo_topk_rows: x, scratch and dx must be 16-byte aligned");
  const long long need = (long long)N * D + N + 2LL * B * topk;
  if (scratch_floats < need)
    return set_error(D3_ERR_ARG, "d3_koleo_topk_rows: scratch needs N*D + N + 2*B*topk floats");
  cudaStream_t st = STREAM(stream);
  const int D4 = D / 4;
  float* xn = scratch;
  float* nrm = scratch + (long long)N * D;
  int* nbr = reinterpret_cast<int*>(nrm + N);
  float* coef = nrm + N + (long long)B * topk;
  // column chunks: enough CTAs to fill the GPU, at least KT_MIN_CHUNK columns each
  const int tiles = (B + KT_RT - 1) / KT_RT;
  int C = std::max(1, (2 * sm_count() + tiles - 1) / tiles);
  C = std::min({C, (gn + KT_MIN_CHUNK - 1) / KT_MIN_CHUNK, KT_MAX_CHUNKS});
  C = std::max(C, 1);
  const int chunk = (gn + C - 1) / C;
  C = (gn + chunk - 1) / chunk;
  if (tiles > 65535) return set_error(D3_ERR_ARG, "d3_koleo_topk_rows: B > 524280 local rows");
  const size_t scan_smem = (size_t)KT_RT * D * sizeof(float);
  static const cudaError_t attr = cudaFuncSetAttribute(koleo_topk_scan_kernel,
                                                       cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                       KT_RT * KT_MAX_D * (int)sizeof(float));
  if (attr != cudaSuccess) return set_error(D3_ERR_CUDA, "d3_koleo_topk_rows: shared memory attribute");
  const size_t cand = (size_t)B * C * topk;
  float* ws = slab_workspace(2 * cand + B, st);            // cand_v | cand_j | row_loss
  if (!ws) return D3_ERR_CUDA;
  float* cand_v = ws;
  int* cand_j = reinterpret_cast<int*>(ws + cand);
  float* row_loss = ws + 2 * cand;
  koleo_topk_norm_kernel<<<gn, KT_THREADS, 0, st>>>((const float4*)x, (float4*)xn, nrm, g0, D4, eps);
  koleo_topk_scan_kernel<<<dim3(C, tiles), KT_THREADS, scan_smem, st>>>((const float4*)xn, D4, g0, gn, row0, B, topk,
                                                                        chunk, cand_v, cand_j);
  koleo_topk_loss_kernel<<<B, KT_THREADS, 0, st>>>((const float4*)xn, D4, cand_v, cand_j, C, topk, row0, B, eps,
                                                   w_metric, w_grad, nbr, coef, row_loss);
  koleo_topk_bwd_kernel<<<gn, KT_THREADS, D * sizeof(float), st>>>((const float4*)x, (const float4*)xn, nrm, nbr,
                                                                   coef, D4, g0, row0, B, topk, eps, (float4*)dx);
  koleo_topk_metric_kernel<<<1, KT_THREADS, 0, st>>>(row_loss, B, metric);
  cudaError_t e = cudaPeekAtLastError();
  slab_release(ws, st);
  if (e != cudaSuccess) return set_error(D3_ERR_CUDA, cudaGetErrorString(e));
  count_launch(5);
  return D3_OK;
}

}  // extern "C"
