// The tile-per-cell geometry of torch's bilinear F.interpolate with align_corners = False, shared by the dense probes'
// upsampling kernels (seg.cu, depth.cu).  Output pixel (y, x) of an Hl x Wl map reads source position
// s = max((y + 0.5) * h / Hl - 0.5, 0), cells y0 = floor(s), y1 = min(y0 + 1, h - 1) with weights (1 - (s - y0), s - y0),
// and the same along x.  The pixels whose (y0, x0) is cell (i, j) form tile (i, j) and read only the four cells
// (y0 | y1) x (x0 | x1), so one CTA per tile needs those four rows and nothing at full resolution.
#pragma once

namespace d3 {

struct SegGeom {
  int B, h, w, Hl, Wl;
  float sh, sw;       // h / Hl, w / Wl (torch's area_pixel_compute_scale in fp32)
};

__device__ __forceinline__ float seg_src(int d, float scale) { return fmaxf(__fmul_rn(d + 0.5f, scale) - 0.5f, 0.f); }

// first output index in [0, n) whose source cell floor(seg_src) is >= t (n if none); seg_src is non-decreasing
__device__ __forceinline__ int seg_first(int t, int n, float scale) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if ((int)seg_src(mid, scale) >= t) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// The tile's pixel rectangle [y_lo, y_hi) x [x_lo, x_hi), its four corner rows of the logits and the corner weights of
// one of its pixels.
struct SegTile {
  int b, ty, tx, y1, x1, y_lo, y_hi, x_lo, x_hi;
};

__device__ __forceinline__ SegTile seg_tile(const SegGeom& g, int* range) {
  SegTile t;
  const int tile = blockIdx.x;
  t.tx = tile % g.w;
  t.ty = (tile / g.w) % g.h;
  t.b = tile / (g.w * g.h);
  t.y1 = min(t.ty + 1, g.h - 1);
  t.x1 = min(t.tx + 1, g.w - 1);
  if (threadIdx.x < 4) {
    const int k = threadIdx.x;
    range[k] = k < 2 ? seg_first(t.ty + k, g.Hl, g.sh) : seg_first(t.tx + k - 2, g.Wl, g.sw);
  }
  __syncthreads();
  t.y_lo = range[0]; t.y_hi = range[1]; t.x_lo = range[2]; t.x_hi = range[3];
  return t;
}

}  // namespace d3
