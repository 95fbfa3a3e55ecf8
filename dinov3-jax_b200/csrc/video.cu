// Semi-supervised video object segmentation by label propagation (DINO's eval_video_segmentation.py protocol): the frame
// resize, the windowed top-k propagation of soft labels through patch-feature affinities, the upsampled, normalised
// argmax label map at the annotation size, and the integer counts behind the DAVIS J (region IoU) and F (boundary
// F-measure) scores.  The affinities themselves come from d3_gemm_bf16 (fp32 results); nothing here multiplies matrices.
//
// Resize: torch's bilinear F.interpolate(align_corners = False, antialias = False) of the uint8 frame / 255 in fp32
// (scale in / out, source max(scale (d + 0.5) - 0.5, 0), the second tap clamped at the last row / column), then
// (v - mean) / std, rounded to bf16.
//
// Propagation of target patch q (grid h x w, P = h w rows) against n_ctx context frames: the candidates are the context
// patches s with |row(s) - row(q)| <= radius and |col(s) - col(q)| <= radius, enumerated context frame first, then row,
// then column.  With the fp32 similarity x_s = <f_q, f_s>, the k-th largest x over the candidates (with multiplicity) is
// the threshold t (-inf when there are fewer than k); every candidate with x >= t is kept, ties included.  Weights
// w_s = exp((x_s - x_max) / temperature), which are exp(x_s / temperature) up to one factor that the normalisation
// cancels; the soft label of q is sum_s w_s L_s / sum_s w_s over the kept candidates, added in candidate order in fp32.
// One warp per target row: the top-k list lives in the lanes' registers (lane i holds the i-th largest, k <= 32), lane
// c owns channel c (C <= 32).  No atomics: the same bits on every run.
//
// Label map: the soft map [h, w, C] upsampled by the patch size p (bilinear, align_corners = False, scale 1 / p, the
// arithmetic of bilinear.cuh), each channel min-max normalised over the whole upsampled frame when its maximum is > 0
// ((v - min) / (max - min); a constant channel becomes 0), the argmax over channels (lowest index on ties), taken at the
// upsampled pixel torch's nearest-exact picks for each annotation pixel: src = min(floor((d + 0.5) * in / out), in - 1)
// in fp32.  The per-channel min / max come from a first pass over the whole upsampled grid; min and max are exact, so
// any order gives the same bits.  No [C, h p, w p] buffer is allocated.
//
// J and F counts per (frame, object k): with void = (gt == 255), pm = (pred == k) and not void, gm = (gt == k):
// intersection and union of pm and gm outside void; the boundary pixels of each mask (a pixel differs from its right,
// lower or lower-right neighbour; the last row compares with the right one only, the last column with the lower one
// only, the bottom-right pixel is 0); and the boundary pixels of one mask with a boundary pixel of the other within the
// disk dy^2 + dx^2 <= r^2.  One CTA per 32 x 32 tile of a frame holds both label maps and both boundary maps of the tile
// with an r-pixel halo in shared memory.  The counts are integers, added with integer atomics: exact.
#include "ptx.cuh"
#include "d3_internal.h"
#include "bilinear.cuh"

#include <math.h>
#include <stdio.h>

#include <algorithm>

namespace d3 {

constexpr int VR_THREADS = 256;             // resize: one thread per output pixel
constexpr int VP_WARPS = 4;                 // propagation: target rows per CTA
constexpr int VIDEO_MAX_K = 32;
constexpr int VIDEO_MAX_C = 32;
constexpr int VM_THREADS = 256;             // min / max and label map passes
constexpr int VM_ROWS = 8;                  // upsampled rows per CTA of the min / max pass
constexpr int JF_TILE = 32;
constexpr int JF_THREADS = 256;
constexpr int JF_COUNTS = 6;                // intersection, union, pred boundary, gt boundary, pred matched, gt matched

// ------------------------------------------------------------------------------------------------ frame resize
__global__ void __launch_bounds__(VR_THREADS) video_resize_kernel(const uint8_t* __restrict__ src,
                                                                  const long long* __restrict__ desc, int out_h,
                                                                  int out_w, float m0, float m1, float m2, float s0,
                                                                  float s1, float s2,
                                                                  __nv_bfloat16* __restrict__ out) {
  const int n = blockIdx.y;
  const uint8_t* im = src + desc[3 * n];
  const int H = (int)desc[3 * n + 1], W = (int)desc[3 * n + 2];
  const float sy = (float)H / (float)out_h, sx = (float)W / (float)out_w;
  const int total = out_h * out_w;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < total; p += gridDim.x * blockDim.x) {
    const int oy = p / out_w, ox = p % out_w;
    const float fy = seg_src(oy, sy), fx = seg_src(ox, sx);
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + (y0 < H - 1 ? 1 : 0), x1 = x0 + (x0 < W - 1 ? 1 : 0);
    const float ly = fy - (float)y0, lx = fx - (float)x0;
    const float hy = 1.f - ly, hx = 1.f - lx;
    const uint8_t* r0 = im + (size_t)y0 * W * 3;
    const uint8_t* r1 = im + (size_t)y1 * W * 3;
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float a = (float)r0[x0 * 3 + c] / 255.f, b = (float)r0[x1 * 3 + c] / 255.f;
      const float d = (float)r1[x0 * 3 + c] / 255.f, e = (float)r1[x1 * 3 + c] / 255.f;
      v[c] = hy * (hx * a + lx * b) + ly * (hx * d + lx * e);
    }
    __nv_bfloat16* o = out + ((size_t)n * total + p) * 3;
    o[0] = __float2bfloat16((v[0] - m0) / s0);
    o[1] = __float2bfloat16((v[1] - m1) / s1);
    o[2] = __float2bfloat16((v[2] - m2) / s2);
  }
}

// ------------------------------------------------------------------------------------------------ propagation
struct Window {
  int y0, x0, nx, per, total;        // first row / column, columns per row, candidates per frame, in all frames
};

__device__ __forceinline__ float candidate(const float* __restrict__ s0, const float* __restrict__ sr, int P,
                                           int w, const Window& win, int j, const float* __restrict__ lab0,
                                           const float* __restrict__ labr, int C, const float** lab) {
  const int c = j / win.per, rem = j - c * win.per;
  const int s = (win.y0 + rem / win.nx) * w + win.x0 + rem % win.nx;
  if (lab) *lab = c == 0 ? lab0 + (size_t)s * C : labr + ((size_t)(c - 1) * P + s) * C;
  return c == 0 ? s0[s] : sr[(size_t)(c - 1) * P + s];
}

__global__ void __launch_bounds__(VP_WARPS * 32) video_propagate_kernel(
    const float* __restrict__ sim0, int ld0, const float* __restrict__ simr, int ldr, const float* __restrict__ lab0,
    const float* __restrict__ labr, int n_recent, int h, int w, int C, int radius, int k, float inv_temp,
    float* __restrict__ out) {
  const int lane = threadIdx.x & 31, P = h * w;
  const int q = blockIdx.x * VP_WARPS + (threadIdx.x >> 5);
  if (q >= P) return;
  const int qy = q / w, qx = q % w;
  Window win;
  win.y0 = max(qy - radius, 0);
  win.x0 = max(qx - radius, 0);
  win.nx = min(qx + radius, w - 1) + 1 - win.x0;
  win.per = (min(qy + radius, h - 1) + 1 - win.y0) * win.nx;
  win.total = (1 + n_recent) * win.per;
  const float* s0 = sim0 + (size_t)q * ld0;
  const float* sr = simr ? simr + (size_t)q * ldr : nullptr;

  // pass 1: the sorted top-k list, lane i its i-th largest entry; a candidate enters only when it beats the k-th
  float top = -INFINITY;
  for (int base = 0; base < win.total; base += 32) {
    const int j = base + lane;
    const float v = j < win.total ? candidate(s0, sr, P, w, win, j, lab0, labr, C, nullptr) : -INFINITY;
    unsigned m = __ballot_sync(0xffffffffu, v > __shfl_sync(0xffffffffu, top, k - 1));
    while (m) {
      const int src = __ffs(m) - 1;
      m &= m - 1;
      const float u = __shfl_sync(0xffffffffu, v, src);
      if (!(u > __shfl_sync(0xffffffffu, top, k - 1))) continue;
      const int pos = __popc(__ballot_sync(0xffffffffu, lane < k && top >= u));
      const float up = __shfl_up_sync(0xffffffffu, top, 1);
      top = lane == pos ? u : (lane > pos ? up : top);
    }
  }
  const float thr = __shfl_sync(0xffffffffu, top, k - 1), xmax = __shfl_sync(0xffffffffu, top, 0);

  // pass 2: the kept candidates in candidate order; every lane adds the same weights in the same order
  float acc = 0.f, wsum = 0.f;
  for (int base = 0; base < win.total; base += 32) {
    const int j = base + lane;
    const float v = j < win.total ? candidate(s0, sr, P, w, win, j, lab0, labr, C, nullptr) : -INFINITY;
    unsigned m = __ballot_sync(0xffffffffu, j < win.total && v >= thr);
    while (m) {
      const int src = __ffs(m) - 1;
      m &= m - 1;
      const float u = __shfl_sync(0xffffffffu, v, src);
      const float* row;
      candidate(s0, sr, P, w, win, base + src, lab0, labr, C, &row);
      const float wt = expf((u - xmax) * inv_temp);
      wsum += wt;
      if (lane < C) acc = fmaf(wt, row[lane], acc);
    }
  }
  if (lane < C) out[(size_t)q * C + lane] = acc / wsum;
}

// ------------------------------------------------------------------------------------------------ label map
// bilinear value of channel c of the soft map [h, w, C] at upsampled pixel (uy, ux), scale 1 / p
__device__ __forceinline__ float soft_up(const float* __restrict__ soft, int h, int w, int C, float scale, int uy,
                                         int ux, int c) {
  const float fy = seg_src(uy, scale), fx = seg_src(ux, scale);
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = min(y0 + 1, h - 1), x1 = min(x0 + 1, w - 1);
  const float ly = fy - (float)y0, lx = fx - (float)x0;
  const float hy = 1.f - ly, hx = 1.f - lx;
  const float a = soft[((size_t)y0 * w + x0) * C + c], b = soft[((size_t)y0 * w + x1) * C + c];
  const float d = soft[((size_t)y1 * w + x0) * C + c], e = soft[((size_t)y1 * w + x1) * C + c];
  return hy * (hx * a + lx * b) + ly * (hx * d + lx * e);
}

// CTA (row block, channel): min and max of channel c over upsampled rows [VM_ROWS rb, VM_ROWS rb + VM_ROWS)
__global__ void __launch_bounds__(VM_THREADS) video_minmax_kernel(const float* __restrict__ soft, int h, int w, int C,
                                                                  int p, float* __restrict__ part) {
  __shared__ float red[2][VM_THREADS / 32];
  const int c = blockIdx.y, Hu = h * p, Wu = w * p;
  const float scale = 1.f / (float)p;
  const int r0 = blockIdx.x * VM_ROWS, r1 = min(r0 + VM_ROWS, Hu), np = (r1 - r0) * Wu;
  float mn = INFINITY, mx = -INFINITY;
  for (int i = threadIdx.x; i < np; i += VM_THREADS) {
    const float v = soft_up(soft, h, w, C, scale, r0 + i / Wu, i % Wu, c);
    mn = fminf(mn, v);
    mx = fmaxf(mx, v);
  }
  for (int o = 16; o > 0; o >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = mn; red[1][threadIdx.x >> 5] = mx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < VM_THREADS / 32; ++i) { mn = fminf(mn, red[0][i]); mx = fmaxf(mx, red[1][i]); }
    part[((size_t)c * gridDim.x + blockIdx.x) * 2] = mn;
    part[((size_t)c * gridDim.x + blockIdx.x) * 2 + 1] = mx;
  }
}

// one warp per channel: the row blocks' (min, max) -> norm[c] = (max > 0, min, max - min)
__global__ void video_minmax_final_kernel(const float* __restrict__ part, int blocks, int C,
                                          float* __restrict__ norm) {
  const int c = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (c >= C) return;
  float mn = INFINITY, mx = -INFINITY;
  for (int i = lane; i < blocks; i += 32) {
    mn = fminf(mn, part[((size_t)c * blocks + i) * 2]);
    mx = fmaxf(mx, part[((size_t)c * blocks + i) * 2 + 1]);
  }
  for (int o = 16; o > 0; o >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if (lane == 0) {
    const bool on = mx > 0.f;
    norm[3 * c] = on ? 1.f : 0.f;
    norm[3 * c + 1] = mn;
    norm[3 * c + 2] = mx - mn;
  }
}

__device__ __forceinline__ int nearest_exact(int d, float scale, int in) {
  return min((int)floorf(((float)d + 0.5f) * scale), in - 1);
}

__global__ void __launch_bounds__(VM_THREADS) video_label_kernel(const float* __restrict__ soft,
                                                                 const float* __restrict__ norm, int h, int w, int C,
                                                                 int p, int out_h, int out_w,
                                                                 uint8_t* __restrict__ labels) {
  __shared__ float nrm[3 * VIDEO_MAX_C];
  for (int i = threadIdx.x; i < 3 * C; i += VM_THREADS) nrm[i] = norm[i];
  __syncthreads();
  const int Hu = h * p, Wu = w * p;
  const float scale = 1.f / (float)p, ny = (float)Hu / (float)out_h, nx = (float)Wu / (float)out_w;
  const int total = out_h * out_w;
  for (int i = blockIdx.x * VM_THREADS + threadIdx.x; i < total; i += gridDim.x * VM_THREADS) {
    const int uy = nearest_exact(i / out_w, ny, Hu), ux = nearest_exact(i % out_w, nx, Wu);
    int best = 0;
    float bv = -INFINITY;
    for (int c = 0; c < C; ++c) {
      float v = soft_up(soft, h, w, C, scale, uy, ux, c);
      if (nrm[3 * c] != 0.f) v = nrm[3 * c + 2] > 0.f ? (v - nrm[3 * c + 1]) / nrm[3 * c + 2] : 0.f;
      if (v > bv) { bv = v; best = c; }
    }
    labels[i] = (uint8_t)best;
  }
}

// ------------------------------------------------------------------------------------------------ J and F counts
// bit 0: the pred mask of object k, bit 1: the gt mask (void pixels cleared in both)
__device__ __forceinline__ int masks_at(const uint8_t* __restrict__ pl, const uint8_t* __restrict__ gl, int i, int k) {
  const int g = gl[i];
  return (pl[i] == k && g != 255 ? 1 : 0) | (g == k ? 2 : 0);
}

__global__ void __launch_bounds__(JF_THREADS) video_jf_kernel(const uint8_t* __restrict__ pred,
                                                              const uint8_t* __restrict__ gt, int H, int W, int K,
                                                              int r, unsigned long long* __restrict__ counts) {
  extern __shared__ uint8_t smem[];
  const int S = JF_TILE + 2 * r + 1, B = JF_TILE + 2 * r;     // label region (one more row / column), boundary region
  uint8_t* pl = smem;
  uint8_t* gl = pl + S * S;
  uint8_t* bd = gl + S * S;                                    // boundary bits of both masks
  __shared__ int red[JF_THREADS / 32][JF_COUNTS];
  const int f = blockIdx.z, ty0 = blockIdx.y * JF_TILE, tx0 = blockIdx.x * JF_TILE;
  const int oy = ty0 - r, ox = tx0 - r;                       // image position of region element (0, 0)
  const uint8_t* pf = pred + (size_t)f * H * W;
  const uint8_t* gf = gt + (size_t)f * H * W;
  for (int i = threadIdx.x; i < S * S; i += JF_THREADS) {
    const int y = oy + i / S, x = ox + i % S;
    const bool in = y >= 0 && y < H && x >= 0 && x < W;
    pl[i] = in ? pf[(size_t)y * W + x] : 0;
    gl[i] = in ? gf[(size_t)y * W + x] : 0;
  }
  for (int k = 1; k <= K; ++k) {
    __syncthreads();                                            // labels loaded / the previous object's search done
    for (int i = threadIdx.x; i < B * B; i += JF_THREADS) {
      const int ry = i / B, rx = i % B, y = oy + ry, x = ox + rx;
      int b = 0;
      if (y >= 0 && y < H && x >= 0 && x < W && !(y == H - 1 && x == W - 1)) {
        const int li = ry * S + rx;
        const int m = masks_at(pl, gl, li, k);
        if (y == H - 1) b = m ^ masks_at(pl, gl, li + 1, k);
        else if (x == W - 1) b = m ^ masks_at(pl, gl, li + S, k);
        else b = (m ^ masks_at(pl, gl, li + 1, k)) | (m ^ masks_at(pl, gl, li + S, k)) |
                 (m ^ masks_at(pl, gl, li + S + 1, k));
      }
      bd[i] = (uint8_t)b;
    }
    __syncthreads();
    int a[JF_COUNTS] = {0, 0, 0, 0, 0, 0};
    for (int i = threadIdx.x; i < JF_TILE * JF_TILE; i += JF_THREADS) {
      const int y = ty0 + i / JF_TILE, x = tx0 + i % JF_TILE;
      if (y >= H || x >= W) continue;
      const int ry = y - oy, rx = x - ox;
      const int m = masks_at(pl, gl, ry * S + rx, k);
      if (gl[ry * S + rx] != 255) {
        a[0] += m == 3;
        a[1] += m != 0;
      }
      const int b = bd[ry * B + rx];
      for (int side = 0; side < 2; ++side) {
        if (!(b >> side & 1)) continue;
        const int other = 2 - side;                             // search the other mask's boundary bit
        ++a[2 + side];
        bool hit = false;
        for (int dy = -r; dy <= r && !hit; ++dy) {
          int e = (int)sqrtf((float)(r * r - dy * dy));
          while (e * e + dy * dy > r * r) --e;
          while ((e + 1) * (e + 1) + dy * dy <= r * r) ++e;
          const uint8_t* row = bd + (ry + dy) * B + rx;
          for (int dx = -e; dx <= e; ++dx)
            if (row[dx] & other) { hit = true; break; }
        }
        a[4 + side] += hit;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
#pragma unroll
      for (int j = 0; j < JF_COUNTS; ++j) a[j] += __shfl_down_sync(0xffffffffu, a[j], o);
    if ((threadIdx.x & 31) == 0)
#pragma unroll
      for (int j = 0; j < JF_COUNTS; ++j) red[threadIdx.x >> 5][j] = a[j];
    __syncthreads();
    if (threadIdx.x < JF_COUNTS) {
      int s = 0;
      for (int wi = 0; wi < JF_THREADS / 32; ++wi) s += red[wi][threadIdx.x];
      if (s) atomicAdd(counts + ((size_t)f * K + (k - 1)) * JF_COUNTS + threadIdx.x, (unsigned long long)s);
    }
  }
}

}  // namespace d3

using namespace d3;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

int d3_video_resize(const void* src_u8, const long long* desc, int n, int out_h, int out_w, const float* mean3,
                    const float* std3, void* out, void* stream) {
  if (n <= 0) return D3_OK;
  if (out_h < 1 || out_w < 1 || !src_u8 || !desc || !out || !mean3 || !std3)
    return set_error(D3_ERR_ARG, "d3_video_resize: need out_h, out_w >= 1, non-null buffers and mean / std");
  const int blocks = std::min((out_h * out_w + VR_THREADS - 1) / VR_THREADS, 2048);
  video_resize_kernel<<<dim3(blocks, n), VR_THREADS, 0, STREAM(stream)>>>(
      (const uint8_t*)src_u8, desc, out_h, out_w, mean3[0], mean3[1], mean3[2], std3[0], std3[1], std3[2],
      (__nv_bfloat16*)out);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_video_propagate(const float* sim0, int ld0, const float* simr, int ldr, const float* lab0, const float* labr,
                       int n_recent, int h, int w, int C, int radius, int topk, float temperature, float* out,
                       void* stream) {
  if (h < 1 || w < 1 || C < 1 || C > VIDEO_MAX_C || topk < 1 || topk > VIDEO_MAX_K || radius < 0 || n_recent < 0 ||
      !(temperature > 0.f) || ld0 < h * w || !sim0 || !lab0 || !out ||
      (n_recent > 0 && (!simr || !labr || (long long)ldr < (long long)n_recent * h * w)))
    return set_error(D3_ERR_ARG, "d3_video_propagate: need 1 <= C <= 32, 1 <= topk <= 32, radius >= 0, "
                                 "temperature > 0, ld0 >= h w, ldr >= n_recent h w and non-null buffers");
  const int P = h * w;
  video_propagate_kernel<<<(P + VP_WARPS - 1) / VP_WARPS, VP_WARPS * 32, 0, STREAM(stream)>>>(
      sim0, ld0, n_recent > 0 ? simr : nullptr, ldr, lab0, labr, n_recent, h, w, C, radius, topk, 1.f / temperature,
      out);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_video_label_map(const float* soft, int h, int w, int C, int patch, int out_h, int out_w, void* labels_u8,
                       void* stream) {
  if (h < 1 || w < 1 || C < 1 || C > VIDEO_MAX_C || patch < 1 || out_h < 1 || out_w < 1 || !soft || !labels_u8)
    return set_error(D3_ERR_ARG, "d3_video_label_map: need h, w, patch, out_h, out_w >= 1, 1 <= C <= 32");
  cudaStream_t st = STREAM(stream);
  const int blocks = (h * patch + VM_ROWS - 1) / VM_ROWS;
  float* ws = slab_workspace((size_t)C * blocks * 2 + 3 * VIDEO_MAX_C, st);
  if (!ws) return D3_ERR_CUDA;
  float* part = ws;
  float* norm = ws + (size_t)C * blocks * 2;
  video_minmax_kernel<<<dim3(blocks, C), VM_THREADS, 0, st>>>(soft, h, w, C, patch, part);
  cudaError_t e = cudaPeekAtLastError();
  if (e == cudaSuccess) {
    count_launch();
    video_minmax_final_kernel<<<1, 32 * C, 0, st>>>(part, blocks, C, norm);
    e = cudaPeekAtLastError();
  }
  if (e == cudaSuccess) {
    count_launch();
    const int lb = std::min((out_h * out_w + VM_THREADS - 1) / VM_THREADS, sm_count() * 8);
    video_label_kernel<<<lb, VM_THREADS, 0, st>>>(soft, norm, h, w, C, patch, out_h, out_w, (uint8_t*)labels_u8);
    e = cudaPeekAtLastError();
  }
  int rc = D3_OK;
  if (e != cudaSuccess) rc = set_error(D3_ERR_CUDA, cudaGetErrorString(e)); else count_launch();
  slab_release(ws, st);
  return rc;
}

int d3_video_jf_counts(const void* pred_u8, const void* gt_u8, int F, int H, int W, int K, int radius,
                       long long* counts, void* stream) {
  if (F <= 0 || K <= 0) return D3_OK;
  if (H < 1 || W < 1 || K > 254 || radius < 0 || !pred_u8 || !gt_u8 || !counts)
    return set_error(D3_ERR_ARG, "d3_video_jf_counts: need H, W >= 1, K <= 254, radius >= 0 and non-null buffers");
  const int S = JF_TILE + 2 * radius + 1, B = JF_TILE + 2 * radius;
  const size_t smem = (size_t)2 * S * S + (size_t)B * B;
  constexpr int SMEM_MAX = 200 * 1024;
  if (smem > SMEM_MAX) return set_error(D3_ERR_ARG, "d3_video_jf_counts: radius too large for one tile");
  static const cudaError_t c0 =
      cudaFuncSetAttribute(video_jf_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_MAX);
  if (c0 != cudaSuccess) return set_error(D3_ERR_CUDA, "d3_video_jf_counts: smem attribute");
  cudaStream_t st = STREAM(stream);
  cudaError_t e = cudaMemsetAsync(counts, 0, sizeof(long long) * (size_t)F * K * JF_COUNTS, st);
  if (e != cudaSuccess) return set_error(D3_ERR_CUDA, cudaGetErrorString(e));
  const dim3 grid((W + JF_TILE - 1) / JF_TILE, (H + JF_TILE - 1) / JF_TILE, F);
  video_jf_kernel<<<grid, JF_THREADS, smem, st>>>((const uint8_t*)pred_u8, (const uint8_t*)gt_u8, H, W, K, radius,
                                                  (unsigned long long*)counts);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

}  // extern "C"
