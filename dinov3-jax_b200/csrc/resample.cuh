// The antialiased bicubic filter of torch's _upsample_bicubic2d_aa (align_corners = False) and the window of taps one
// output position reads.  The training crops (aug_resized_crop_kernel in augment.cu, fp32) and the evaluation
// transform (eval_resize_crop_kernel in knn.cu, fp64 like torch's uint8 path) both take their taps and weight sums
// from here, so the two resizes cannot drift apart.
#pragma once

namespace d3 {

template <typename T>
__device__ __forceinline__ T cubic_aa(T x) {                    // Keys cubic, a = -0.5 (PIL / torch antialias bicubic)
  x = x < (T)0 ? -x : x;
  if (x < (T)1) return (((T)1.5 * x - (T)2.5) * x) * x + (T)1;
  if (x < (T)2) return (((T)-0.5 * x + (T)2.5) * x - (T)4) * x + (T)2;
  return (T)0;
}

// Taps [lo, hi) of the output position whose centre in input coordinates is `center` (= scale * (i + 0.5)), for an
// axis of `in_size` inputs and support = 2 * max(scale, 1); inv = 1 / max(scale, 1).  At most max_taps taps (torch
// clips a window that rounding made one tap too long).  Returns the sum of the unnormalised weights
// cubic_aa((j - center + 0.5) * inv), by which every weight of the window is divided.
template <typename T>
__device__ __forceinline__ T aa_window(T center, T support, T inv, int in_size, int max_taps, int& lo, int& hi) {
  lo = max((int)(center - support + (T)0.5), 0);
  hi = min(min((int)(center + support + (T)0.5), in_size), lo + max_taps);
  T sum = (T)0;
  for (int j = lo; j < hi; ++j) sum += cubic_aa<T>((j - center + (T)0.5) * inv);
  return sum;
}

}  // namespace d3
