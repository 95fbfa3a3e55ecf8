// Instance retrieval (revisited Oxford / Paris): the crop-and-resize of queries and database images at each scale,
// the fixed-order sum of the per-scale class tokens, and the exact revisited ranking with junk removal, AP and P@k.
// The similarities s = Q DB^T come from d3_gemm_bf16 (fp32 results) and the descriptors are normalised by
// d3_knn_normalize; nothing here multiplies matrices.
//
// Resize: torch's F.interpolate(mode="bicubic", antialias=True, align_corners=False) on float values, from a uint8 HWC
// image straight to the output size, the source window being the crop box [x0, x1) x [y0, y1).  The taps and the
// normalised weights of each output column and row come from resample.cuh, in fp64; each output pixel sums its rows'
// horizontal sums in fp64 (horizontal first, as torch's separable pass), without clamping, and (v / 255 - mean) / std
// in fp64 is rounded once to bf16, so the result is within one bf16 ulp of torch's float64 resize.  At an identity
// size the weights are exactly (0, 1, 0, 0), so the result is the plain normalisation of the pixel.
//
// Ranking, per query q over the N columns of its similarity row: a column's key is (order-preserving bits of s) << 32
// | ~index (-0 keyed as +0, which it equals), so "larger key" is exactly (s desc, index asc) and no two columns share
// a key.  The rank of a listed image j (easy, hard or junk) is the number of columns with a larger key, an integer
// count:
//   ret_sort_kernel   sorts the query's listed keys (bitonic, in shared memory);
//   ret_count_kernel  gives every column of a chunk the number c of listed keys >= its key (binary search) and counts
//                     the columns per c (integer shared-memory atomics: the counts are exact in any order);
//   ret_ap_kernel     adds the chunks' counts, so rank(sorted position k) = #columns with c <= k, marks each sorted
//                     position with the lists it is in, then per protocol walks the positions in rank order: a junk
//                     image increments the junk count, an ok image takes its rank minus that count (the merge of the
//                     ok and junk rank lists), and AP and P@1/5/10 are summed in fp64 in ascending rank order.
// No float atomics and no order-dependent float sums: the same bits on every run.
#include "ptx.cuh"
#include "d3_internal.h"
#include "resample.cuh"

#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <vector>

namespace d3 {

constexpr int RR_THREADS = 256;
constexpr int RR_TH = 16, RR_TW = 64;           // output rows and columns per resize CTA
constexpr int RR_SMEM_MAX = 200 * 1024;
constexpr int RT_THREADS = 512;
constexpr int RET_MAX_LIST = 8192;              // easy + hard + junk entries per query
constexpr int RET_CHUNK = 32768;                // columns per counting CTA

// ------------------------------------------------------------------------------------------------------ resize
// Taps and normalised weights of output positions [first, first + count) of an axis resized from `in` to `out`.
__device__ void ret_axis_table(int in, int out, int first, int count, int max_taps, int* lo_out, int* n_out,
                               double* w_out) {
  const double scale = (double)in / out;
  const double support = scale >= 1.0 ? 2.0 * scale : 2.0;
  const double inv = scale >= 1.0 ? 1.0 / scale : 1.0;
  const int taps = min(2 * (int)ceil(support) + 1, max_taps);
  for (int c = threadIdx.x; c < count; c += blockDim.x) {
    int lo, hi;
    const double ctr = scale * (first + c + 0.5);
    const double s = aa_window<double>(ctr, support, inv, in, taps, lo, hi);
    lo_out[c] = lo;
    n_out[c] = s != 0.0 ? hi - lo : 0;
    for (int j = 0; j < max_taps; ++j)
      w_out[(size_t)c * max_taps + j] = j < hi - lo && s != 0.0 ? cubic_aa<double>((lo + j - ctr + 0.5) * inv) / s
                                                                : 0.0;
  }
}

// desc[7 n .. 7 n + 6] = (byte offset, H, W, x0, y0, x1, y1) of image n = blockIdx.z; out bf16 [n, out_h, out_w, 3].
// One CTA per RR_TH x RR_TW output tile.
__global__ void __launch_bounds__(RR_THREADS) ret_resize_kernel(const uint8_t* __restrict__ src,
                                                               const long long* __restrict__ desc, int out_h,
                                                               int out_w, int max_taps, float m0, float m1, float m2,
                                                               float s0, float s1, float s2,
                                                               __nv_bfloat16* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char rr_smem[];
  double* w_x = reinterpret_cast<double*>(rr_smem);
  double* w_y = w_x + (size_t)RR_TW * max_taps;
  int* lo_x = reinterpret_cast<int*>(w_y + (size_t)RR_TH * max_taps);
  int* n_x = lo_x + RR_TW;
  int* lo_y = n_x + RR_TW;
  int* n_y = lo_y + RR_TH;
  const int n = blockIdx.z;
  const long long* d = desc + 7 * (size_t)n;
  const int W = (int)d[2], x0 = (int)d[3], y0 = (int)d[4], x1 = (int)d[5], y1 = (int)d[6];
  const int col0 = blockIdx.x * RR_TW, cols = min(RR_TW, out_w - col0);
  const int row0 = blockIdx.y * RR_TH, rows = min(RR_TH, out_h - row0);
  ret_axis_table(x1 - x0, out_w, col0, cols, max_taps, lo_x, n_x, w_x);
  ret_axis_table(y1 - y0, out_h, row0, rows, max_taps, lo_y, n_y, w_y);
  __syncthreads();
  const uint8_t* img = src + d[0] + ((size_t)y0 * W + x0) * 3;
  for (int p = threadIdx.x; p < rows * cols; p += blockDim.x) {
    const int oy = p / cols, ox = p % cols;
    const double* wy = w_y + (size_t)oy * max_taps;
    const double* wx = w_x + (size_t)ox * max_taps;
    const int ty = n_y[oy], tx = n_x[ox];
    const uint8_t* base = img + ((size_t)lo_y[oy] * W + lo_x[ox]) * 3;
    double ar = 0.0, ag = 0.0, ab = 0.0;
    for (int j = 0; j < ty; ++j) {
      const uint8_t* row = base + (size_t)j * W * 3;
      double hr = 0.0, hg = 0.0, hb = 0.0;
      for (int i = 0; i < tx; ++i) {
        const double w = wx[i];
        hr = fma(w, (double)row[3 * i], hr);
        hg = fma(w, (double)row[3 * i + 1], hg);
        hb = fma(w, (double)row[3 * i + 2], hb);
      }
      const double v = wy[j];
      ar = fma(v, hr, ar);
      ag = fma(v, hg, ag);
      ab = fma(v, hb, ab);
    }
    __nv_bfloat16* y = out + (((size_t)n * out_h + row0 + oy) * out_w + col0 + ox) * 3;
    y[0] = __double2bfloat16((ar / 255.0 - (double)m0) / (double)s0);
    y[1] = __double2bfloat16((ag / 255.0 - (double)m1) / (double)s1);
    y[2] = __double2bfloat16((ab / 255.0 - (double)m2) / (double)s2);
  }
}

// ------------------------------------------------------------------------------------------------------ scale sum
// out[i] = x[i] + x[stride + i] + ... + x[(S - 1) stride + i], added in scale order.
__global__ void ret_scale_sum_kernel(const float* __restrict__ x, int S, long long stride, long long count,
                                     float* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < count;
       i += (long long)gridDim.x * blockDim.x) {
    float acc = x[i];
    for (int s = 1; s < S; ++s) acc += x[s * stride + i];
    out[i] = acc;
  }
}

// ------------------------------------------------------------------------------------------------------ ranking
__device__ __forceinline__ uint64_t ret_key(float s, int idx) {
  const uint32_t u = s == 0.f ? 0u : __float_as_uint(s);      // -0 == +0: one key, so they tie as the ranks define
  const uint32_t k = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ((uint64_t)k << 32) | (uint32_t)~(uint32_t)idx;
}

// The query's list entries: lists[3 (Q + 1)] holds the three CSR row pointers (easy, hard, junk), each already offset
// to its place in the concatenated index array idx (easy entries, then hard, then junk).
struct RetLists {
  const int* ptr;     // [3][Q + 1]
  const int* idx;
  int Q;
  __device__ __forceinline__ int begin(int list, int q) const { return ptr[list * (Q + 1) + q]; }
  __device__ __forceinline__ int end(int list, int q) const { return ptr[list * (Q + 1) + q + 1]; }
  __device__ __forceinline__ int count(int q) const {
    return end(0, q) - begin(0, q) + end(1, q) - begin(1, q) + end(2, q) - begin(2, q);
  }
  // the list (0 easy, 1 hard, 2 junk) and the position in idx of the query's e-th entry
  __device__ __forceinline__ int entry(int q, int e, int* list) const {
    for (int l = 0; l < 2; ++l) {
      const int n = end(l, q) - begin(l, q);
      if (e < n) { *list = l; return begin(l, q) + e; }
      e -= n;
    }
    *list = 2;
    return begin(2, q) + e;
  }
};

// keys[q * ld_keys + k], k < count(q): the query's listed keys in descending order
__global__ void __launch_bounds__(RT_THREADS) ret_sort_kernel(const float* __restrict__ sim, long long lds,
                                                             RetLists L, uint64_t* __restrict__ keys, int ld_keys) {
  extern __shared__ __align__(16) uint64_t rs_keys[];
  const int q = blockIdx.x, m = L.count(q);
  if (m == 0) return;
  int P = 1;
  while (P < m) P <<= 1;
  const float* row = sim + (size_t)q * lds;
  for (int e = threadIdx.x; e < P; e += blockDim.x) {
    int list;
    const int j = e < m ? L.idx[L.entry(q, e, &list)] : 0;
    rs_keys[e] = e < m ? ret_key(row[j], j) : 0ull;      // every real key is above 0 (~index has its top bit set)
  }
  __syncthreads();
  for (int size = 2; size <= P; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = threadIdx.x; i < P / 2; i += blockDim.x) {
        const int lo = 2 * stride * (i / stride) + (i % stride), hi = lo + stride;
        const uint64_t a = rs_keys[lo], b = rs_keys[hi];
        if ((a < b) == ((lo & size) == 0)) { rs_keys[lo] = b; rs_keys[hi] = a; }
      }
      __syncthreads();
    }
  }
  for (int k = threadIdx.x; k < m; k += blockDim.x) keys[(size_t)q * ld_keys + k] = rs_keys[k];
}

// counts[((q * chunks) + chunk) * (ld_keys + 1) + c] = #columns of the chunk with exactly c listed keys >= their key
__global__ void __launch_bounds__(RT_THREADS) ret_count_kernel(const float* __restrict__ sim, long long lds, int N,
                                                              RetLists L, const uint64_t* __restrict__ keys,
                                                              int ld_keys, int* __restrict__ counts) {
  extern __shared__ __align__(16) uint64_t rc_keys[];
  const int q = blockIdx.y, m = L.count(q);
  if (m == 0) return;
  int* hist = reinterpret_cast<int*>(rc_keys + m);
  for (int k = threadIdx.x; k < m; k += blockDim.x) rc_keys[k] = keys[(size_t)q * ld_keys + k];
  for (int c = threadIdx.x; c <= m; c += blockDim.x) hist[c] = 0;
  __syncthreads();
  const float* row = sim + (size_t)q * lds;
  const int i0 = blockIdx.x * RET_CHUNK, i1 = min(N, i0 + RET_CHUNK);
  for (int base = i0; base < i1; base += blockDim.x) {         // block-uniform trip count: whole warps in the match
    const int i = base + threadIdx.x;
    int c = -1;
    if (i < i1) {
      const uint64_t key = ret_key(row[i], i);
      int lo = 0, hi = m;                                      // first position whose key is below key
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (rc_keys[mid] >= key) lo = mid + 1; else hi = mid;
      }
      c = lo;
    }
    const unsigned same = __match_any_sync(0xffffffffu, c);
    if (c >= 0 && (threadIdx.x & 31) == __ffs(same) - 1) atomicAdd(&hist[c], __popc(same));
  }
  __syncthreads();
  int* out = counts + ((size_t)q * gridDim.x + blockIdx.x) * (ld_keys + 1);
  for (int c = threadIdx.x; c <= m; c += blockDim.x) out[c] = hist[c];
}

// exclusive block-wide prefix sum of v; *total receives the sum (every thread calls it)
__device__ __forceinline__ int ret_block_scan(int v, int* warp_tot, int* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int inc = v;
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) warp_tot[wid] = inc;
  __syncthreads();
  int before = 0, all = 0;
  for (int w = 0; w < nw; ++w) {
    const int t = warp_tot[w];
    before += w < wid ? t : 0;
    all += t;
  }
  *total = all;
  __syncthreads();
  return before + inc - v;
}

// Per query: ranks[e] for every list entry (in the concatenated idx layout), and for each protocol p (0 Easy,
// 1 Medium, 2 Hard) ap[3 q + p], pk[(3 q + p) * 3 + t] (P@1, P@5, P@10) and n_ok[3 q + p]; NaN AP and P@k for a
// protocol without an ok image.
__global__ void __launch_bounds__(RT_THREADS) ret_ap_kernel(const float* __restrict__ sim, long long lds, RetLists L,
                                                           const uint64_t* __restrict__ keys, int ld_keys,
                                                           const int* __restrict__ counts, int chunks,
                                                           int* __restrict__ ranks, double* __restrict__ ap,
                                                           double* __restrict__ pk, int* __restrict__ n_ok) {
  extern __shared__ __align__(16) uint64_t ra_keys[];
  __shared__ int warp_tot[RT_THREADS / 32];
  const int q = blockIdx.x, m = L.count(q);
  int* rank = reinterpret_cast<int*>(ra_keys + m);
  int* flags = rank + m;
  for (int k = threadIdx.x; k < m; k += blockDim.x) {
    ra_keys[k] = keys[(size_t)q * ld_keys + k];
    flags[k] = 0;
  }
  // rank(k) = sum over c <= k of the columns with c listed keys above-or-equal: a segmented inclusive scan
  const int seg = (m + blockDim.x - 1) / blockDim.x;
  const int k0 = min(m, (int)threadIdx.x * seg), k1 = min(m, k0 + seg);
  int local = 0;
  for (int k = k0; k < k1; ++k) {
    int h = 0;
    for (int ch = 0; ch < chunks; ++ch) h += counts[((size_t)q * chunks + ch) * (ld_keys + 1) + k];
    rank[k] = h;
    local += h;
  }
  int total;
  int run = ret_block_scan(local, warp_tot, &total);
  for (int k = k0; k < k1; ++k) {
    run += rank[k];
    rank[k] = run;
  }
  __syncthreads();
  // each entry marks the first sorted position of its key (duplicates share a key) and reads its rank
  const float* row = sim + (size_t)q * lds;
  for (int e = threadIdx.x; e < m; e += blockDim.x) {
    int list;
    const int pos_e = L.entry(q, e, &list);
    const int j = L.idx[pos_e];
    const uint64_t key = ret_key(row[j], j);
    int lo = 0, hi = m;                                        // first position whose key is <= key
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (ra_keys[mid] > key) lo = mid + 1; else hi = mid;
    }
    atomicOr(&flags[lo], 1 << list);
    ranks[pos_e] = rank[lo];
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    const int p = threadIdx.x;
    // ok / junk list bits per protocol: easy = 1, hard = 2, junk = 4
    const int ok_bits = p == 0 ? 1 : p == 1 ? 3 : 2;
    const int junk_bits = p == 0 ? 6 : p == 1 ? 4 : 5;
    int n_junk = 0, j = 0, last = 0, c1 = 0, c5 = 0, c10 = 0;
    double sum = 0.0;
    for (int k = 0; k < m; ++k) {
      if (k > 0 && ra_keys[k] == ra_keys[k - 1]) continue;
      const int f = flags[k];
      if (f & ok_bits) {
        const int r = rank[k] - n_junk;                        // 0-based, junk removed
        sum += (r == 0 ? 1.0 : (double)j / r) + (double)(j + 1) / (r + 1);
        ++j;
        last = r + 1;
        c1 += last <= 1;
        c5 += last <= 5;
        c10 += last <= 10;
      } else if (f & junk_bits) {
        ++n_junk;
      }
    }
    const int o = 3 * q + p;
    n_ok[o] = j;
    if (j == 0) {
      ap[o] = pk[3 * o] = pk[3 * o + 1] = pk[3 * o + 2] = __longlong_as_double(0x7ff8000000000000LL);
    } else {
      ap[o] = sum / (2.0 * j);
      // kq = min(max rank, k): P = |{rank <= kq}| / kq
      pk[3 * o] = last >= 1 ? c1 / 1.0 : (double)j / last;
      pk[3 * o + 1] = last >= 5 ? c5 / 5.0 : (double)j / last;
      pk[3 * o + 2] = last >= 10 ? c10 / 10.0 : (double)j / last;
    }
  }
}

}  // namespace d3

using namespace d3;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

int d3_ret_resize(const void* src_u8, long long src_bytes, const long long* desc, int n, int out_h, int out_w,
                  const float* mean3, const float* std3, void* out, void* stream) {
  if (n < 0 || out_h < 1 || out_w < 1 || src_bytes < 0 || !mean3 || !std3)
    return set_error(D3_ERR_ARG, "d3_ret_resize: need n >= 0, out_h, out_w >= 1, src_bytes >= 0, mean and std");
  if (n == 0) return D3_OK;
  if (n > 65535 || out_h > (1 << 20) || !src_u8 || !desc || !out || (uintptr_t)out % 2)
    return set_error(D3_ERR_ARG, "d3_ret_resize: need n <= 65535, out_h <= 2^20 and non-null buffers, out 2-byte "
                                 "aligned");
  int max_taps = 1;
  for (int i = 0; i < n; ++i) {
    const long long* d = desc + 7 * (size_t)i;
    const long long off = d[0], H = d[1], W = d[2], x0 = d[3], y0 = d[4], x1 = d[5], y1 = d[6];
    if (off < 0 || H < 1 || W < 1 || H > (1 << 20) || W > (1 << 20) || off + H * W * 3 > src_bytes)
      return set_error(D3_ERR_ARG, "d3_ret_resize: an image (byte offset, H, W) lies outside the source buffer");
    if (x0 < 0 || y0 < 0 || x1 > W || y1 > H || x1 <= x0 || y1 <= y0)
      return set_error(D3_ERR_ARG, "d3_ret_resize: a crop box (x0, y0, x1, y1) is empty or outside its image");
    for (const double sc : {(double)(x1 - x0) / out_w, (double)(y1 - y0) / out_h})
      max_taps = std::max(max_taps, 2 * (int)ceil(sc >= 1.0 ? 2.0 * sc : 2.0) + 1);
  }
  const size_t smem = (size_t)(RR_TW + RR_TH) * (2 * sizeof(int) + (size_t)max_taps * sizeof(double));
  if (smem > RR_SMEM_MAX)
    return set_error(D3_ERR_ARG, "d3_ret_resize: the downscale needs more filter taps than shared memory holds");
  cudaStream_t st = STREAM(stream);
  static const cudaError_t attr =
      cudaFuncSetAttribute(ret_resize_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, RR_SMEM_MAX);
  if (attr != cudaSuccess) return set_error(D3_ERR_CUDA, "d3_ret_resize: shared memory attribute");
  float* ws = slab_workspace(2 * 7 * (size_t)n, st);
  if (!ws) return D3_ERR_CUDA;
  // a copy from pageable memory is staged before the call returns, so desc may be freed afterwards
  cudaError_t e = cudaMemcpyAsync(ws, desc, sizeof(long long) * 7 * n, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) {
    ret_resize_kernel<<<dim3((out_w + RR_TW - 1) / RR_TW, (out_h + RR_TH - 1) / RR_TH, n), RR_THREADS, smem, st>>>(
        (const uint8_t*)src_u8, reinterpret_cast<const long long*>(ws), out_h, out_w, max_taps, mean3[0], mean3[1],
        mean3[2], std3[0], std3[1], std3[2], (__nv_bfloat16*)out);
    e = cudaPeekAtLastError();
  }
  int rc = D3_OK;
  if (e != cudaSuccess) rc = set_error(D3_ERR_CUDA, cudaGetErrorString(e)); else count_launch();
  slab_release(ws, st);
  return rc;
}

int d3_ret_scale_sum(const float* x, int S, long long stride, long long count, float* out, void* stream) {
  if (S < 1 || count < 0 || (S > 1 && stride < count))
    return set_error(D3_ERR_ARG, "d3_ret_scale_sum: need S >= 1, count >= 0 and stride >= count");
  if (count == 0) return D3_OK;
  if (!x || !out) return set_error(D3_ERR_ARG, "d3_ret_scale_sum: null buffer");
  const int blocks = (int)std::min<long long>((count + 255) / 256, (long long)sm_count() * 8);
  ret_scale_sum_kernel<<<blocks, 256, 0, STREAM(stream)>>>(x, S, stride, count, out);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_ret_rank_ap(const float* sim, long long lds, int Q, int N, const int* easy_ptr, const int* easy_idx,
                   const int* hard_ptr, const int* hard_idx, const int* junk_ptr, const int* junk_idx, int* ranks,
                   double* ap, double* pk, int* n_ok, void* stream) {
  if (Q < 0 || Q > 65535 || N < 1 || lds < N)
    return set_error(D3_ERR_ARG, "d3_ret_rank_ap: need 0 <= Q <= 65535, N >= 1 and lds >= N");
  if (Q == 0) return D3_OK;
  const int* ptrs[3] = {easy_ptr, hard_ptr, junk_ptr};
  const int* idxs[3] = {easy_idx, hard_idx, junk_idx};
  if (!sim || !ap || !pk || !n_ok || !easy_ptr || !hard_ptr || !junk_ptr || (uintptr_t)sim % 4)
    return set_error(D3_ERR_ARG, "d3_ret_rank_ap: need non-null buffers and list pointers, sim 4-byte aligned");
  // the lists: row pointers from 0, non-decreasing; indices in [0, N); at most RET_MAX_LIST entries per query
  long long total = 0;
  for (int l = 0; l < 3; ++l) {
    const int* p = ptrs[l];
    if (p[0] != 0) return set_error(D3_ERR_ARG, "d3_ret_rank_ap: a list's row pointers do not start at 0");
    for (int q = 0; q < Q; ++q)
      if (p[q + 1] < p[q]) return set_error(D3_ERR_ARG, "d3_ret_rank_ap: a list's row pointers decrease");
    if (p[Q] > 0 && !idxs[l]) return set_error(D3_ERR_ARG, "d3_ret_rank_ap: a non-empty list without indices");
    for (int e = 0; e < p[Q]; ++e)
      if (idxs[l][e] < 0 || idxs[l][e] >= N)
        return set_error(D3_ERR_ARG, "d3_ret_rank_ap: a list index is outside [0, N)");
    total += p[Q];
  }
  if (total > 0x3fffffffLL) return set_error(D3_ERR_ARG, "d3_ret_rank_ap: too many list entries");
  if (total > 0 && !ranks) return set_error(D3_ERR_ARG, "d3_ret_rank_ap: ranks is null");
  int m_max = 1;
  for (int q = 0; q < Q; ++q) {
    long long m = 0;
    for (int l = 0; l < 3; ++l) m += ptrs[l][q + 1] - ptrs[l][q];
    if (m > RET_MAX_LIST)
      return set_error(D3_ERR_ARG, "d3_ret_rank_ap: a query lists more than 8192 easy, hard and junk entries");
    m_max = std::max(m_max, (int)m);
  }
  // device copies: row pointers offset into the concatenated index array, then the indices
  std::vector<int> meta(3 * (size_t)(Q + 1) + (size_t)total);
  long long base = 0;
  for (int l = 0; l < 3; ++l) {
    for (int q = 0; q <= Q; ++q) meta[l * (size_t)(Q + 1) + q] = (int)(base + ptrs[l][q]);
    std::copy(idxs[l], idxs[l] + ptrs[l][Q], meta.begin() + 3 * (size_t)(Q + 1) + base);
    base += ptrs[l][Q];
  }
  const int chunks = (N + RET_CHUNK - 1) / RET_CHUNK;
  const size_t key_words = 2 * (size_t)Q * m_max;                       // uint64 keys, in 4-byte words
  const size_t count_words = (size_t)Q * chunks * (m_max + 1);
  cudaStream_t st = STREAM(stream);
  static const cudaError_t a0 = cudaFuncSetAttribute(ret_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                     RET_MAX_LIST * 8);
  static const cudaError_t a1 = cudaFuncSetAttribute(ret_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                     RET_MAX_LIST * 12 + 4);
  static const cudaError_t a2 = cudaFuncSetAttribute(ret_ap_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                     RET_MAX_LIST * 16);
  if (a0 != cudaSuccess || a1 != cudaSuccess || a2 != cudaSuccess)
    return set_error(D3_ERR_CUDA, "d3_ret_rank_ap: shared memory attribute");
  float* ws = slab_workspace(key_words + count_words + meta.size(), st);
  if (!ws) return D3_ERR_CUDA;
  uint64_t* keys = reinterpret_cast<uint64_t*>(ws);
  int* counts = reinterpret_cast<int*>(ws + key_words);
  int* dmeta = reinterpret_cast<int*>(ws + key_words + count_words);
  RetLists L{dmeta, dmeta + 3 * (Q + 1), Q};
  int p2 = 1;
  while (p2 < m_max) p2 <<= 1;
  // a copy from pageable memory is staged before the call returns, so meta may go out of scope
  cudaError_t e = cudaMemcpyAsync(dmeta, meta.data(), sizeof(int) * meta.size(), cudaMemcpyHostToDevice, st);
  int launched = 0;
  if (e == cudaSuccess) {
    ret_sort_kernel<<<Q, RT_THREADS, (size_t)p2 * 8, st>>>(sim, lds, L, keys, m_max);
    e = cudaPeekAtLastError();
    launched += e == cudaSuccess;
  }
  if (e == cudaSuccess) {
    ret_count_kernel<<<dim3(chunks, Q), RT_THREADS, (size_t)m_max * 12 + 4, st>>>(sim, lds, N, L, keys, m_max,
                                                                                  counts);
    e = cudaPeekAtLastError();
    launched += e == cudaSuccess;
  }
  if (e == cudaSuccess) {
    ret_ap_kernel<<<Q, RT_THREADS, (size_t)m_max * 16, st>>>(sim, lds, L, keys, m_max, counts, chunks, ranks, ap, pk,
                                                            n_ok);
    e = cudaPeekAtLastError();
    launched += e == cudaSuccess;
  }
  count_launch(launched);
  const int rc = e == cudaSuccess ? D3_OK : set_error(D3_ERR_CUDA, cudaGetErrorString(e));
  slab_release(ws, st);
  return rc;
}

}  // extern "C"
