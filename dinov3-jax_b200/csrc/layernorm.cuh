// Row statistics and normalisation of the LayerNorm forward (models/vision_transformer.py:40: eps 1e-6, biased
// variance E[x^2]-E[x]^2, fp32 statistics), one warp per row.  Every LayerNorm forward (layernorm_fwd_kernel,
// ln_tokens_out_kernel in elementwise.cu; dwconv7_ln_kernel and ln_patchify2_kernel in convnext.cu) goes through
// ln_row_stats and ln_store4, so a row normalised by any of them gets the same bits.
#pragma once
#include "ptx.cuh"

namespace d3 {

// 4 values stored at columns 4e..4e+3 of the row yr (bf16: round to nearest even)
template <typename OutT>
__device__ __forceinline__ void store4(OutT* yr, int e, float o0, float o1, float o2, float o3) {
  if constexpr (sizeof(OutT) == 2) {
    reinterpret_cast<uint2*>(yr)[e] = make_uint2(pack_bf16(o0, o1), pack_bf16(o2, o3));
  } else {
    reinterpret_cast<float4*>(yr)[e] = make_float4(o0, o1, o2, o3);
  }
}

// columns 4e..4e+3 of the row yr: (v - mean) rstd scale + bias
template <typename OutT>
__device__ __forceinline__ void ln_store4(OutT* yr, int e, const float4& v, const float* scale, const float* bias, float mean,
                                          float rstd) {
  const float4 g = reinterpret_cast<const float4*>(scale)[e];
  const float4 b = reinterpret_cast<const float4*>(bias)[e];
  const float o0 = (v.x - mean) * rstd * g.x + b.x, o1 = (v.y - mean) * rstd * g.y + b.y;
  const float o2 = (v.z - mean) * rstd * g.z + b.z, o3 = (v.w - mean) * rstd * g.w + b.w;
  store4(yr, e, o0, o1, o2, o3);
}

// Mean and rstd of the row xr ([D] fp32, 16-byte aligned), computed by one warp: lane l sums the float4 columns
// l, l + 32, ... in that order, then a butterfly.  VPL > 0: D = 128 * VPL known at compile time; the row is left in v
// (lane l holds float4 columns k * 32 + l), all VPL 16-byte loads of a lane in flight together.  VPL == 0: any
// D % 4 == 0 (`width` is read only then), v unused.
template <int VPL>
__device__ __forceinline__ void ln_row_stats(const float4* __restrict__ xr, int lane, int width, float eps,
                                             float4 (&v)[VPL > 0 ? VPL : 1], float& mean, float& rstd) {
  const int D = VPL > 0 ? VPL * 128 : width;
  float s = 0.f, s2 = 0.f;
  if constexpr (VPL > 0) {
#pragma unroll
    for (int k = 0; k < VPL; ++k) v[k] = xr[k * 32 + lane];
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
      s += v[k].x + v[k].y + v[k].z + v[k].w;
      s2 += v[k].x * v[k].x + v[k].y * v[k].y + v[k].z * v[k].z + v[k].w * v[k].w;
    }
  } else {
    for (int e = lane; e < D / 4; e += 32) {
      const float4 w = xr[e];
      s += w.x + w.y + w.z + w.w;
      s2 += w.x * w.x + w.y * w.y + w.z * w.z + w.w * w.w;
    }
  }
  s = warp_sum(s);
  s2 = warp_sum(s2);
  mean = s * (1.f / D);
  const float var = fmaxf(s2 * (1.f / D) - mean * mean, 0.f);
  rstd = rsqrtf(var + eps);
}

// the whole row xr normalised into yr (one warp; v and mean / rstd from ln_row_stats<VPL>)
template <int VPL, typename OutT>
__device__ __forceinline__ void ln_store_row(OutT* yr, const float4* __restrict__ xr, int lane, int D,
                                             const float4 (&v)[VPL > 0 ? VPL : 1], const float* scale, const float* bias,
                                             float mean, float rstd) {
  if constexpr (VPL > 0) {
#pragma unroll
    for (int k = 0; k < VPL; ++k) ln_store4(yr, k * 32 + lane, v[k], scale, bias, mean, rstd);
  } else {
    for (int e = lane; e < D / 4; e += 32) ln_store4(yr, e, xr[e], scale, bias, mean, rstd);
  }
}

}  // namespace d3
