// k-NN evaluation of a frozen backbone (the DINO / DINOv2 / DINOv3 k-NN protocol): the eval transform of a batch of
// decoded images of any size (and, with the same kernel, the linear probe's RandomResizedCrop + flip train crop), the L2 normalisation of the features, the running top-k merge over chunks of
// similarities, and the softmax-weighted class vote.  The similarities themselves are d3_gemm_bf16 with an fp32
// output (queries . bank_chunk^T); nothing here multiplies matrices.
//
// Every kernel is deterministic: no float atomics, every sum in a fixed order, and the top-k order is the total order
// (similarity descending, bank index ascending), so the neighbour lists do not depend on the chunk size or on how the
// queries are tiled.
#include "ptx.cuh"
#include "d3_internal.h"
#include "resample.cuh"

#include <math.h>
#include <stdio.h>

namespace d3 {

// ---------------------------------------------------------------------------------------------------- eval transform
// torchvision Resize(resize, BICUBIC, antialias=True) of a uint8 image, short side to `resize` and the long side to
// int(resize * long / short), then CenterCrop(crop), with torch's uint8 arithmetic (UpSampleKernel's separable uint8
// path): per axis the normalised fp64 weights become int16 with the largest precision that keeps the axis' largest
// weight below 2^15; the horizontal pass rounds and clamps to uint8, then the vertical pass does the same.  Only the
// crop's pixels are computed.  Out: uint8 NHWC, or bf16 NHWC (u8 / 255 - mean) / std.
constexpr int EV_THREADS = 256;
constexpr int EV_ROWS = 32;          // output rows per CTA (grid.x bands of one image)

struct EvalAxis {
  int out;          // resized length
  int first;        // first crop position in the resized axis
  double scale, support, inv;
  int taps;         // torch's max_interp_size: 2 * ceil(support) + 1
};

__device__ __forceinline__ EvalAxis eval_axis(int in, int out, int first) {
  EvalAxis a;
  a.out = out;
  a.first = first;
  a.scale = (double)in / out;
  a.support = a.scale >= 1.0 ? 2.0 * a.scale : 2.0;
  a.inv = a.scale >= 1.0 ? 1.0 / a.scale : 1.0;
  a.taps = 2 * (int)ceil(a.support) + 1;
  return a;
}

// largest normalised weight over every output position of the axis (block-wide; every thread gets it)
__device__ double eval_axis_wmax(const EvalAxis& a, int in, double* red) {
  double m = 0.0;
  for (int i = threadIdx.x; i < a.out; i += blockDim.x) {
    int lo, hi;
    const double c = a.scale * (i + 0.5);
    const double s = aa_window(c, a.support, a.inv, in, a.taps, lo, hi);
    if (s != 0.0)
      for (int j = lo; j < hi; ++j) m = fmax(m, cubic_aa<double>((j - c + 0.5) * a.inv) / s);
  }
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = 0.0;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) m = fmax(m, red[w]);
  __syncthreads();
  return m;
}

__device__ __forceinline__ int eval_precision(double wmax) {
  int p = 0;
  for (; p < 22; ++p)
    if ((int)(0.5 + wmax * (double)(1 << (p + 1))) >= (1 << 15)) break;
  return p;
}

// int16 weights and first tap of the crop positions [0, crop) of one axis
__device__ void eval_axis_table(const EvalAxis& a, int in, int crop, int prec, int max_taps, int* lo_out,
                                short* w_out) {
  for (int c = threadIdx.x; c < crop; c += blockDim.x) {
    int lo, hi;
    const double ctr = a.scale * (a.first + c + 0.5);
    const double s = aa_window(ctr, a.support, a.inv, in, min(a.taps, max_taps), lo, hi);
    lo_out[c] = lo;
    short* w = w_out + (size_t)c * max_taps;
    for (int j = 0; j < max_taps; ++j) {
      double v = 0.0;
      if (lo + j < hi && s != 0.0) v = cubic_aa<double>((lo + j - ctr + 0.5) * a.inv) / s;
      w[j] = (short)round(v * (double)(1 << prec));
    }
  }
}

// One resampled axis of the window a crop reads: source positions [src0, src0 + axis.in) of the image feed output
// positions [0, crop) of the resized axis from `first` on (mirrored when flip).
struct CropAxis {
  EvalAxis a;
  int in, src0, flip;
};

// The eval transform (boxes == nullptr: Resize(resize) of the whole image + CenterCrop(crop)) and the train crop
// (boxes[5n .. 5n+4] = (top, left, height, width, flip): crop the box, resize it to crop x crop, mirror when flip).
// Both take their int16 weights from eval_axis_wmax / eval_precision / eval_axis_table, so the two share torch's uint8
// arithmetic bit for bit.
template <bool U8>
__global__ void __launch_bounds__(EV_THREADS) eval_resize_crop_kernel(
    const uint8_t* __restrict__ src, const long long* __restrict__ desc, const int* __restrict__ boxes, int resize,
    int crop, int max_taps, float m0, float m1, float m2, float s0, float s1, float s2, void* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char ev_smem[];
  __shared__ double red[EV_THREADS / 32];
  int* lo_x = reinterpret_cast<int*>(ev_smem);
  int* lo_y = lo_x + crop;
  short* w_x = reinterpret_cast<short*>(lo_y + crop);
  short* w_y = w_x + (size_t)crop * max_taps;
  const int n = blockIdx.y;
  const long long off = desc[3 * n];
  const int H = (int)desc[3 * n + 1], W = (int)desc[3 * n + 2];
  CropAxis cx, cy;
  if (boxes) {
    const int* bx = boxes + 5 * n;
    cy = {eval_axis(bx[2], crop, 0), bx[2], bx[0], 0};
    cx = {eval_axis(bx[3], crop, 0), bx[3], bx[1], bx[4]};
  } else {
    // torchvision _compute_resized_output_size and center_crop (offsets rounded half to even, like Python's round)
    const int shorter = min(H, W), longer = max(H, W);
    const int new_long = (int)((double)((long long)resize * longer) / (double)shorter);
    const int oh = W <= H ? new_long : resize, ow = W <= H ? resize : new_long;
    cx = {eval_axis(W, ow, (int)rint((ow - crop) / 2.0)), W, 0, 0};
    cy = {eval_axis(H, oh, (int)rint((oh - crop) / 2.0)), H, 0, 0};
  }
  const EvalAxis& ax = cx.a;
  const EvalAxis& ay = cy.a;
  const int px = eval_precision(eval_axis_wmax(ax, cx.in, red));
  const int py = eval_precision(eval_axis_wmax(ay, cy.in, red));
  eval_axis_table(ax, cx.in, crop, px, max_taps, lo_x, w_x);
  eval_axis_table(ay, cy.in, crop, py, max_taps, lo_y, w_y);
  __syncthreads();
  const int tx = min(ax.taps, max_taps), ty = min(ay.taps, max_taps);
  const uint8_t* img = src + off + ((size_t)cy.src0 * W + cx.src0) * 3;
  const int row0 = blockIdx.x * EV_ROWS, rows = min(EV_ROWS, crop - row0);
  const int hx = px > 0 ? 1 << (px - 1) : 0, hy = py > 0 ? 1 << (py - 1) : 0;
  for (int p = threadIdx.x; p < rows * crop; p += blockDim.x) {
    const int oy = row0 + p / crop, ox = p % crop;
    const int sx = cx.flip ? crop - 1 - ox : ox;
    const short* wy = w_y + (size_t)oy * max_taps;
    const short* wx = w_x + (size_t)sx * max_taps;
    const int y0 = lo_y[oy], x0 = lo_x[sx];
    int ar = hy, ag = hy, ab = hy;
    for (int j = 0; j < ty; ++j) {
      const int wv = wy[j];
      if (wv == 0 || y0 + j >= cy.in) continue;
      const uint8_t* row = img + ((size_t)(y0 + j) * W + x0) * 3;
      int hr = hx, hg = hx, hb = hx;
      for (int i = 0; i < tx && x0 + i < cx.in; ++i) {
        const int w = wx[i];
        hr += w * row[3 * i]; hg += w * row[3 * i + 1]; hb += w * row[3 * i + 2];
      }
      ar += wv * min(max(hr >> px, 0), 255);
      ag += wv * min(max(hg >> px, 0), 255);
      ab += wv * min(max(hb >> px, 0), 255);
    }
    const int r = min(max(ar >> py, 0), 255), g = min(max(ag >> py, 0), 255), b = min(max(ab >> py, 0), 255);
    const size_t o = (((size_t)n * crop + oy) * crop + ox) * 3;
    if constexpr (U8) {
      uint8_t* y = reinterpret_cast<uint8_t*>(out) + o;
      y[0] = (uint8_t)r; y[1] = (uint8_t)g; y[2] = (uint8_t)b;
    } else {
      __nv_bfloat16* y = reinterpret_cast<__nv_bfloat16*>(out) + o;
      y[0] = __float2bfloat16((r / 255.f - m0) / s0);
      y[1] = __float2bfloat16((g / 255.f - m1) / s1);
      y[2] = __float2bfloat16((b / 255.f - m2) / s2);
    }
  }
}

// The segmentation probe's image and label crops (one kernel for both, from the same box).  Image n (desc as above) is
// resized to (rh, rw) = boxes[6n], boxes[6n + 1] with the arithmetic above (the whole image is the source window), and
// the out_h x out_w window at (top, left) = boxes[6n + 2], boxes[6n + 3] of the resized image is written; the part of
// the window inside the resized image (vh x vw) is mirrored within its own width when flip = boxes[6n + 4], and the
// rest (bottom / right) is 0 in the image (after normalisation) and 255 in the labels.  Labels: torch's 'nearest'
// (src = min(floor(dst * in / out), in - 1)) from a uint8 map of the image's size at lab_src + desc offset / 3.
template <bool U8>
__global__ void __launch_bounds__(EV_THREADS) seg_crop_kernel(
    const uint8_t* __restrict__ src, const long long* __restrict__ desc, const uint8_t* __restrict__ lab_src,
    const int* __restrict__ boxes, int out_h, int out_w, int max_taps, float m0, float m1, float m2, float s0, float s1,
    float s2, void* __restrict__ out, uint8_t* __restrict__ lab_out) {
  extern __shared__ __align__(16) unsigned char ev_smem[];
  __shared__ double red[EV_THREADS / 32];
  int* lo_x = reinterpret_cast<int*>(ev_smem);
  int* lo_y = lo_x + out_w;
  short* w_x = reinterpret_cast<short*>(lo_y + out_h);
  short* w_y = w_x + (size_t)out_w * max_taps;
  const int n = blockIdx.y;
  const long long off = desc[3 * n];
  const int H = (int)desc[3 * n + 1], W = (int)desc[3 * n + 2];
  const int* bx = boxes + 6 * n;
  const int rh = bx[0], rw = bx[1], top = bx[2], left = bx[3], flip = bx[4];
  const EvalAxis ax = eval_axis(W, rw, left), ay = eval_axis(H, rh, top);
  const int px = eval_precision(eval_axis_wmax(ax, W, red));
  const int py = eval_precision(eval_axis_wmax(ay, H, red));
  eval_axis_table(ax, W, out_w, px, max_taps, lo_x, w_x);
  eval_axis_table(ay, H, out_h, py, max_taps, lo_y, w_y);
  __syncthreads();
  const int tx = min(ax.taps, max_taps), ty = min(ay.taps, max_taps);
  const int vh = min(out_h, rh - top), vw = min(out_w, rw - left);
  const float nsy = (float)H / (float)rh, nsx = (float)W / (float)rw;
  const uint8_t* img = src + off;
  const int row0 = blockIdx.x * EV_ROWS, rows = min(EV_ROWS, out_h - row0);
  const int hx = px > 0 ? 1 << (px - 1) : 0, hy = py > 0 ? 1 << (py - 1) : 0;
  for (int p = threadIdx.x; p < rows * out_w; p += blockDim.x) {
    const int oy = row0 + p / out_w, ox = p % out_w;
    const size_t o = ((size_t)n * out_h + oy) * out_w + ox;
    const bool inside = oy < vh && ox < vw;
    int r = 0, g = 0, b = 0;
    if (inside) {
      const int sx = flip ? vw - 1 - ox : ox;
      const short* wy = w_y + (size_t)oy * max_taps;
      const short* wx = w_x + (size_t)sx * max_taps;
      const int y0 = lo_y[oy], x0 = lo_x[sx];
      int ar = hy, ag = hy, ab = hy;
      for (int j = 0; j < ty; ++j) {
        const int wv = wy[j];
        if (wv == 0 || y0 + j >= H) continue;
        const uint8_t* row = img + ((size_t)(y0 + j) * W + x0) * 3;
        int hr = hx, hg = hx, hb = hx;
        for (int i = 0; i < tx && x0 + i < W; ++i) {
          const int w = wx[i];
          hr += w * row[3 * i]; hg += w * row[3 * i + 1]; hb += w * row[3 * i + 2];
        }
        ar += wv * min(max(hr >> px, 0), 255);
        ag += wv * min(max(hg >> px, 0), 255);
        ab += wv * min(max(hb >> px, 0), 255);
      }
      r = min(max(ar >> py, 0), 255); g = min(max(ag >> py, 0), 255); b = min(max(ab >> py, 0), 255);
      if (lab_out) {
        const int ly = min((int)floorf((float)(top + oy) * nsy), H - 1);
        const int lx = min((int)floorf((float)(left + sx) * nsx), W - 1);
        lab_out[o] = lab_src[off / 3 + (size_t)ly * W + lx];
      }
    } else if (lab_out) {
      lab_out[o] = 255;
    }
    if constexpr (U8) {
      uint8_t* y = reinterpret_cast<uint8_t*>(out) + 3 * o;
      y[0] = (uint8_t)r; y[1] = (uint8_t)g; y[2] = (uint8_t)b;
    } else {
      __nv_bfloat16* y = reinterpret_cast<__nv_bfloat16*>(out) + 3 * o;
      y[0] = __float2bfloat16(inside ? (r / 255.f - m0) / s0 : 0.f);
      y[1] = __float2bfloat16(inside ? (g / 255.f - m1) / s1 : 0.f);
      y[2] = __float2bfloat16(inside ? (b / 255.f - m2) / s2 : 0.f);
    }
  }
}

// ------------------------------------------------------------------------------------------------- L2 normalisation
// y = x / max(||x||, 1e-12) per row (F.normalize), one warp per row, lanes strided then a butterfly: the same bits on
// every run.  Writes fp32 and / or bf16.
__global__ void knn_normalize_kernel(const float* __restrict__ x, int ldx, int R, int D, float* __restrict__ yf,
                                     __nv_bfloat16* __restrict__ yb, int ldy) {
  const int warps = blockDim.x >> 5, lane = threadIdx.x & 31;
  for (long row = (long)blockIdx.x * warps + (threadIdx.x >> 5); row < R; row += (long)gridDim.x * warps) {
    const float* xr = x + row * ldx;
    float s = 0.f;
    for (int e = lane; e < D; e += 32) s += xr[e] * xr[e];
    s = warp_sum(s);
    const float nrm = fmaxf(sqrtf(s), 1e-12f);
    for (int e = lane; e < D; e += 32) {
      const float v = xr[e] / nrm;
      if (yf) yf[row * ldy + e] = v;
      if (yb) yb[row * ldy + e] = __float2bfloat16(v);
    }
  }
}

// ------------------------------------------------------------------------------------------------------ top-k merge
// One CTA per query row.  Candidates are 64-bit keys (order-preserving uint32 of the similarity) << 32 | ~index, so
// "larger key" is exactly (similarity desc, index asc) and no two candidates are equal; 0 is an empty slot.
// 1. the running list (sorted) is read into shared memory; when it is full, a chunk element can only enter with a
//    similarity key above its k-th (chunk indices are above every running index, so an equal key loses the tie);
// 2. the chunk elements that pass are gathered into shared memory (in any order: they are sorted next);
// 3. if more pass than fit (the first chunk of every row), an 8-bit radix select over the running list and the chunk
//    finds the key T of the k-th best candidate; the chunk is gathered again keeping keys above T, and the first
//    (k - #above) elements equal to T in index order (a block-wide scan keeps them in order);
// 4. the candidates are bitonic-sorted and merged with the running list by rank (binary search), the first k kept.
constexpr int TK_THREADS = 512;
constexpr int TK_MAX_K = 1024;
constexpr int TK_CAP = 2 * TK_MAX_K;

__device__ __forceinline__ uint32_t sim_key(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_sim(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
__device__ __forceinline__ uint64_t cand_of(uint32_t key, int idx) {
  return ((uint64_t)key << 32) | (uint32_t)~(uint32_t)idx;
}

// exclusive block-wide prefix sum of v (every thread of the CTA calls it); *total receives the sum
__device__ __forceinline__ int block_excl_scan(int v, int* warp_tot, int* total) {
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

// gather the chunk elements with key > gt_key, plus (EQ) the first eq_limit elements with key == eq_key in index
// order, into cand[*count ...] (slots past TK_CAP are counted, not written)
template <bool EQ>
__device__ void tk_gather(const float* __restrict__ row, int valid, uint32_t gt_key, uint32_t eq_key, int eq_limit,
                          uint64_t* cand, int* count, int* warp_tot, int offset) {
  const int lane = threadIdx.x & 31;
  int eq_taken = 0;
  for (int base = 0; base < valid; base += 4 * TK_THREADS) {
    const int i0 = base + 4 * threadIdx.x;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (i0 < valid) v = *reinterpret_cast<const float4*>(row + i0);
    const float f[4] = {v.x, v.y, v.z, v.w};
    uint32_t k[4];
    bool gt[4], eq[4];
    int n_eq = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      k[j] = sim_key(f[j]);
      const bool in = i0 + j < valid;
      gt[j] = in && k[j] > gt_key;
      eq[j] = EQ && in && k[j] == eq_key;
      n_eq += eq[j];
    }
    int eq_before = 0;
    if constexpr (EQ) {
      if (eq_taken < eq_limit) {                    // block-uniform
        int tot;
        eq_before = eq_taken + block_excl_scan(n_eq, warp_tot, &tot);
        eq_taken += tot;
      } else {
        eq_before = eq_limit;
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      bool take = gt[j];
      if constexpr (EQ) {
        if (eq[j]) { take = eq_before < eq_limit; ++eq_before; }
      }
      const unsigned m = __ballot_sync(0xffffffffu, take);
      if (m) {
        const int leader = __ffs(m) - 1;
        int pos = 0;
        if (lane == leader) pos = atomicAdd(count, __popc(m));
        pos = __shfl_sync(0xffffffffu, pos, leader) + __popc(m & ((1u << lane) - 1u));
        if (take && pos < TK_CAP) cand[pos] = cand_of(k[j], offset + i0 + j);
      }
    }
  }
}

__global__ void __launch_bounds__(TK_THREADS) topk_merge_kernel(const float* __restrict__ sims, long long lds, int valid,
                                                                 int offset, float* __restrict__ top_sim,
                                                                 int* __restrict__ top_idx, int ldk, int k, int fresh) {
  __shared__ uint64_t run[TK_MAX_K];
  __shared__ uint64_t cand[TK_CAP];
  __shared__ int hist[256];
  __shared__ int warp_tot[TK_THREADS / 32];
  __shared__ int s_count, s_sel[2];
  const int q = blockIdx.x;
  const float* row = sims + (size_t)q * lds;
  float* ts = top_sim + (size_t)q * ldk;
  int* ti = top_idx + (size_t)q * ldk;
  for (int i = threadIdx.x; i < k; i += blockDim.x) {
    const int idx = fresh ? -1 : ti[i];
    run[i] = idx < 0 ? 0ull : cand_of(sim_key(ts[i]), idx);
  }
  if (threadIdx.x == 0) s_count = 0;
  __syncthreads();
  const uint32_t thr = (uint32_t)(run[k - 1] >> 32);       // 0 while the list is not full: every element passes
  tk_gather<false>(row, valid, thr, 0u, 0, cand, &s_count, warp_tot, offset);
  __syncthreads();
  int n = s_count;
  if (n > TK_CAP) {
    // radix select of the k-th largest key over the running list and the chunk elements above thr
    uint32_t prefix = 0, mask = 0;
    int remaining = k;
    for (int shift = 24; shift >= 0; shift -= 8) {
      for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
      __syncthreads();
      for (int i = threadIdx.x; i < k; i += blockDim.x) {
        const uint32_t key = (uint32_t)(run[i] >> 32);
        if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255], 1);
      }
      for (int i = 4 * threadIdx.x; i < valid; i += 4 * TK_THREADS) {
        const float4 v = *reinterpret_cast<const float4*>(row + i);
        const float f[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint32_t key = sim_key(f[j]);
          if (i + j < valid && key > thr && (key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255], 1);
        }
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        int above = 0, d = 255;
        for (; d > 0 && above + hist[d] < remaining; --d) above += hist[d];
        s_sel[0] = d;
        s_sel[1] = remaining - above;
      }
      __syncthreads();
      prefix |= (uint32_t)s_sel[0] << shift;
      mask |= 255u << shift;
      remaining = s_sel[1];
      __syncthreads();
    }
    // prefix = T, the k-th largest key; `remaining` of the candidates equal to T are needed
    if (threadIdx.x == 0) s_count = 0;
    __syncthreads();
    // (T is never below thr; when T == thr, chunk elements equal to it lose the tie to the running list)
    tk_gather<true>(row, valid, prefix, prefix, prefix > thr ? remaining : 0, cand, &s_count, warp_tot, offset);
    __syncthreads();
    n = min(s_count, TK_CAP);
  }
  // bitonic sort of cand[0, P) descending, P = next power of two >= n (padded with empty slots)
  int P = 1;
  while (P < n) P <<= 1;
  for (int i = n + threadIdx.x; i < P; i += blockDim.x) cand[i] = 0ull;
  __syncthreads();
  for (int size = 2; size <= P; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = threadIdx.x; i < P / 2; i += blockDim.x) {
        const int lo = 2 * stride * (i / stride) + (i % stride), hi = lo + stride;
        const uint64_t a = cand[lo], b = cand[hi];
        const bool desc = (lo & size) == 0;
        if ((a < b) == desc) { cand[lo] = b; cand[hi] = a; }
      }
      __syncthreads();
    }
  }
  // merge by rank: position = own rank + number of larger entries in the other sorted list
  for (int i = threadIdx.x; i < k + n; i += blockDim.x) {
    const bool is_run = i < k;
    const uint64_t v = is_run ? run[i] : cand[i - k];
    const uint64_t* other = is_run ? cand : run;
    int lo = 0, hi = is_run ? n : k;                       // count of other[] > v (other sorted descending)
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (other[mid] > v) lo = mid + 1; else hi = mid;
    }
    const int pos = (is_run ? i : i - k) + lo;
    if (pos < k) {
      const uint32_t key = (uint32_t)(v >> 32);
      ts[pos] = v ? key_sim(key) : -INFINITY;
      ti[pos] = v ? (int)~(uint32_t)v : -1;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------- vote
// One CTA per query.  For each k of the list: w = softmax(sims[:k] / T) in fp32 (max subtracted, the sum in a fixed
// warp order), class scores accumulated in shared memory by one thread in neighbour order, then the 5 best classes
// (score desc, class index asc) by five block-wide argmax passes.
constexpr int VOTE_THREADS = 256;
constexpr int VOTE_MAX_NK = 16;
constexpr int VOTE_MAX_CLASSES = 32768;
struct KnnList { int n; int k[VOTE_MAX_NK]; };

__global__ void __launch_bounds__(VOTE_THREADS) knn_vote_kernel(const float* __restrict__ top_sim,
                                                                const int* __restrict__ top_idx, int ldk,
                                                                const int* __restrict__ labels, int n_bank, KnnList ks,
                                                                float temperature, int C, int* __restrict__ preds) {
  extern __shared__ __align__(16) float scores[];
  __shared__ float w[TK_MAX_K];
  __shared__ int lab[TK_MAX_K];
  __shared__ float rv[VOTE_THREADS / 32];
  __shared__ int ri[VOTE_THREADS / 32];
  const int q = blockIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const float* s = top_sim + (size_t)q * ldk;
  const int* ix = top_idx + (size_t)q * ldk;
  int kmax = 0;
  for (int t = 0; t < ks.n; ++t) kmax = max(kmax, ks.k[t]);
  for (int j = threadIdx.x; j < kmax; j += blockDim.x) {
    const int b = ix[j];
    lab[j] = (b >= 0 && b < n_bank) ? labels[b] : -1;
  }
  for (int t = 0; t < ks.n; ++t) {
    const int k = ks.k[t];
    for (int c = threadIdx.x; c < C; c += blockDim.x) scores[c] = 0.f;
    if (wid == 0) {
      float m = -INFINITY;
      for (int j = lane; j < k; j += 32) m = fmaxf(m, s[j] / temperature);
      for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
      float z = 0.f;
      for (int j = lane; j < k; j += 32) {
        const float e = expf(s[j] / temperature - m);
        w[j] = e;
        z += e;
      }
      z = warp_sum(z);
      for (int j = lane; j < k; j += 32) w[j] = w[j] / z;
    }
    __syncthreads();
    if (threadIdx.x == 0)
      for (int j = 0; j < k; ++j)
        if (lab[j] >= 0 && lab[j] < C) scores[lab[j]] += w[j];
    __syncthreads();
    for (int r = 0; r < 5; ++r) {
      float bv = -INFINITY;
      int bi = 0x7fffffff;
      for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const float v = scores[c];
        if (v > bv) { bv = v; bi = c; }                        // classes visited in increasing order: ties keep the lower
      }
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
      }
      if (lane == 0) { rv[wid] = bv; ri[wid] = bi; }
      __syncthreads();
      if (threadIdx.x == 0) {
        for (int u = 1; u < VOTE_THREADS / 32; ++u)
          if (rv[u] > bv || (rv[u] == bv && ri[u] < bi)) { bv = rv[u]; bi = ri[u]; }
        preds[((size_t)q * ks.n + t) * 5 + r] = bi < C ? bi : -1;
        if (bi < C) scores[bi] = -INFINITY;
      }
      __syncthreads();
    }
  }
}

}  // namespace d3

using namespace d3;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

static int crop_error(int code, const char* who, const char* what) {
  char msg[160];
  snprintf(msg, sizeof(msg), "%s: %s", who, what);
  return set_error(code, msg);
}

static int launch_resize_crop(const char* who, const void* src_u8, const long long* desc, const int* boxes, int n,
                              int resize, int crop, int max_taps, const float* mean3, const float* std3, void* out,
                              int out_u8, void* stream) {
  const size_t smem = (size_t)2 * crop * sizeof(int) + (size_t)2 * crop * max_taps * sizeof(short);
  constexpr int SMEM_MAX = 200 * 1024;
  if (smem > SMEM_MAX) return crop_error(D3_ERR_ARG, who, "crop * max_taps too large (downscale > ~100x)");
  if (!out_u8 && (!mean3 || !std3)) return crop_error(D3_ERR_ARG, who, "mean / std needed for bf16 output");
  static const cudaError_t c0 =
      cudaFuncSetAttribute(eval_resize_crop_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_MAX);
  static const cudaError_t c1 =
      cudaFuncSetAttribute(eval_resize_crop_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_MAX);
  if (c0 != cudaSuccess || c1 != cudaSuccess) return crop_error(D3_ERR_CUDA, who, "smem attribute");
  const dim3 grid((crop + EV_ROWS - 1) / EV_ROWS, n);
  const float m[3] = {out_u8 ? 0.f : mean3[0], out_u8 ? 0.f : mean3[1], out_u8 ? 0.f : mean3[2]};
  const float s[3] = {out_u8 ? 1.f : std3[0], out_u8 ? 1.f : std3[1], out_u8 ? 1.f : std3[2]};
  if (out_u8)
    eval_resize_crop_kernel<true><<<grid, EV_THREADS, smem, STREAM(stream)>>>(
        (const uint8_t*)src_u8, desc, boxes, resize, crop, max_taps, m[0], m[1], m[2], s[0], s[1], s[2], out);
  else
    eval_resize_crop_kernel<false><<<grid, EV_THREADS, smem, STREAM(stream)>>>(
        (const uint8_t*)src_u8, desc, boxes, resize, crop, max_taps, m[0], m[1], m[2], s[0], s[1], s[2], out);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_eval_resize_crop(const void* src_u8, const long long* desc, int n, int resize, int crop, int max_taps,
                        const float* mean3, const float* std3, void* out, int out_u8, void* stream) {
  if (n <= 0) return D3_OK;
  if (crop < 1 || resize < crop || max_taps < 1 || !src_u8 || !desc || !out)
    return set_error(D3_ERR_ARG, "d3_eval_resize_crop: need 1 <= crop <= resize, max_taps >= 1");
  return launch_resize_crop("d3_eval_resize_crop", src_u8, desc, nullptr, n, resize, crop, max_taps, mean3, std3, out,
                            out_u8, stream);
}

int d3_train_resized_crop(const void* src_u8, const long long* desc, const int* boxes, int n, int crop, int max_taps,
                          const float* mean3, const float* std3, void* out, int out_u8, void* stream) {
  if (n <= 0) return D3_OK;
  if (crop < 1 || max_taps < 1 || !src_u8 || !desc || !boxes || !out)
    return set_error(D3_ERR_ARG, "d3_train_resized_crop: need crop >= 1, max_taps >= 1 and non-null buffers");
  return launch_resize_crop("d3_train_resized_crop", src_u8, desc, boxes, n, 0, crop, max_taps, mean3, std3, out,
                            out_u8, stream);
}

int d3_seg_crop(const void* src_u8, const long long* desc, const void* labels_u8, const int* boxes, int n, int out_h,
                int out_w, int max_taps, const float* mean3, const float* std3, void* out, int out_u8, void* label_out,
                void* stream) {
  if (n <= 0) return D3_OK;
  if (out_h < 1 || out_w < 1 || max_taps < 1 || !src_u8 || !desc || !boxes || !out || (label_out && !labels_u8))
    return set_error(D3_ERR_ARG, "d3_seg_crop: need out_h, out_w, max_taps >= 1, non-null buffers (labels with label_out)");
  const size_t smem = (size_t)(out_h + out_w) * sizeof(int) + (size_t)(out_h + out_w) * max_taps * sizeof(short);
  constexpr int SMEM_MAX = 200 * 1024;
  if (smem > SMEM_MAX) return set_error(D3_ERR_ARG, "d3_seg_crop: (out_h + out_w) * max_taps too large");
  if (!out_u8 && (!mean3 || !std3)) return set_error(D3_ERR_ARG, "d3_seg_crop: mean / std needed for bf16 output");
  static const cudaError_t c0 =
      cudaFuncSetAttribute(seg_crop_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_MAX);
  static const cudaError_t c1 =
      cudaFuncSetAttribute(seg_crop_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_MAX);
  if (c0 != cudaSuccess || c1 != cudaSuccess) return set_error(D3_ERR_CUDA, "d3_seg_crop: smem attribute");
  const dim3 grid((out_h + EV_ROWS - 1) / EV_ROWS, n);
  const float m[3] = {out_u8 ? 0.f : mean3[0], out_u8 ? 0.f : mean3[1], out_u8 ? 0.f : mean3[2]};
  const float s[3] = {out_u8 ? 1.f : std3[0], out_u8 ? 1.f : std3[1], out_u8 ? 1.f : std3[2]};
  if (out_u8)
    seg_crop_kernel<true><<<grid, EV_THREADS, smem, STREAM(stream)>>>(
        (const uint8_t*)src_u8, desc, (const uint8_t*)labels_u8, boxes, out_h, out_w, max_taps, m[0], m[1], m[2], s[0],
        s[1], s[2], out, (uint8_t*)label_out);
  else
    seg_crop_kernel<false><<<grid, EV_THREADS, smem, STREAM(stream)>>>(
        (const uint8_t*)src_u8, desc, (const uint8_t*)labels_u8, boxes, out_h, out_w, max_taps, m[0], m[1], m[2], s[0],
        s[1], s[2], out, (uint8_t*)label_out);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_knn_normalize(const float* x, int ldx, int R, int D, float* y_f32, void* y_bf16, int ldy, void* stream) {
  if (R <= 0) return D3_OK;
  if (D <= 0 || ldx < D || ldy < D || (!y_f32 && !y_bf16)) return set_error(D3_ERR_ARG, "d3_knn_normalize: bad shape");
  knn_normalize_kernel<<<min((R + 7) / 8, sm_count() * 8), 256, 0, STREAM(stream)>>>(x, ldx, R, D, y_f32,
                                                                                     (__nv_bfloat16*)y_bf16, ldy);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_topk_merge(const float* sims, long long lds, int Q, int valid, int offset, float* top_sim, int* top_idx, int ldk,
                  int k, int fresh, void* stream) {
  if (Q <= 0) return D3_OK;
  if (k < 1 || k > TK_MAX_K || ldk < k || valid < 0 || valid > lds || offset < 0 || (lds % 4) ||
      (reinterpret_cast<uintptr_t>(sims) & 15) || (long long)offset + valid > 0x7fffffffLL)
    return set_error(D3_ERR_ARG, "d3_topk_merge: need 1 <= k <= 1024 <= ..., valid <= lds, lds % 4 == 0, "
                                 "16-byte aligned sims, indices below 2^31");
  topk_merge_kernel<<<Q, TK_THREADS, 0, STREAM(stream)>>>(sims, lds, valid, offset, top_sim, top_idx, ldk, k, fresh);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_knn_vote(const float* top_sim, const int* top_idx, int ldk, int Q, const int* bank_labels, int n_bank,
                const int* nb_knn, int n_k, float temperature, int num_classes, int* preds, void* stream) {
  if (Q <= 0) return D3_OK;
  if (n_k < 1 || n_k > VOTE_MAX_NK || num_classes < 1 || num_classes > VOTE_MAX_CLASSES || !(temperature > 0.f))
    return set_error(D3_ERR_ARG, "d3_knn_vote: need 1 <= len(nb_knn) <= 16, 1 <= classes <= 32768, temperature > 0");
  KnnList ks;
  ks.n = n_k;
  for (int t = 0; t < n_k; ++t) {
    if (nb_knn[t] < 1 || nb_knn[t] > ldk || nb_knn[t] > TK_MAX_K)
      return set_error(D3_ERR_ARG, "d3_knn_vote: every k must be in [1, min(ldk, 1024)]");
    ks.k[t] = nb_knn[t];
  }
  const size_t smem = (size_t)num_classes * sizeof(float);
  static const cudaError_t c0 = cudaFuncSetAttribute(knn_vote_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                     VOTE_MAX_CLASSES * (int)sizeof(float));
  if (c0 != cudaSuccess) return set_error(D3_ERR_CUDA, "d3_knn_vote: smem attribute");
  knn_vote_kernel<<<Q, VOTE_THREADS, smem, STREAM(stream)>>>(top_sim, top_idx, ldk, bank_labels, n_bank, ks, temperature,
                                                            num_classes, preds);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

}  // extern "C"
