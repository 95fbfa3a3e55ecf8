// Row-wise e4m3 quantisation of the FP8 block linears' GEMM operands (d3_gemm_e4m3 reads them K-major):
//   quant_rows_kernel     a bf16 [R, C] view (activations, gradients, W [in, out] for the input gradient) per row
//   colmax_kernel, col_scale_kernel, quant_cols_t_kernel
//                         W [in, out] per column, written as W^T [out, in] through a shared-memory tile transpose
// The scale of a row is the power of two 2^e with e the smallest integer such that the row's largest finite magnitude
// is at most 448 * 2^e (1 for a row of zeros), so x / 2^e is exact and within the e4m3 range; the conversion rounds to
// nearest even (cvt.rn.satfinite, torch's .to(torch.float8_e4m3fn)).  A maximum is exact in any order, so the bits do
// not depend on the launch geometry or on the order of the column-maximum atomics.
#include "ptx.cuh"
#include "d3_internal.h"

namespace d3 {

#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

__device__ __forceinline__ float finite_abs(float v) { return isfinite(v) ? fabsf(v) : 0.f; }

// 2^e, e the smallest integer with amax <= 448 * 2^e (448 = 0.875 * 2^9); 1 when amax is 0
__device__ __forceinline__ float e4m3_scale(float amax) {
  if (!(amax > 0.f)) return 1.f;
  int E;
  const float m = frexpf(amax, &E);   // amax = m 2^E, m in [0.5, 1)
  return ldexpf(1.f, m <= 0.875f ? E - 9 : E - 8);
}

// e4m3 bytes of (a / s, b / s): a in the low byte.  A non-finite input becomes the e4m3 NaN (0x7f, sign kept), as
// torch's conversion does; finite quotients never exceed 448, so satfinite never clamps one.
__device__ __forceinline__ uint16_t e4m3x2(float a, float b, float s) {
  const float qa = __fdiv_rn(a, s), qb = __fdiv_rn(b, s);
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(qb), "f"(qa));
  if (!isfinite(qa)) r = (r & 0xff00) | (signbit(qa) ? 0xff : 0x7f);
  if (!isfinite(qb)) r = (r & 0x00ff) | ((signbit(qb) ? 0xff : 0x7f) << 8);
  return r;
}

// one CTA per row: the row's maximum, then the row again (from L1 / L2) converted.  VEC: 8 elements per access
// (C % 8 == 0, 16-byte aligned rows in, 8-byte aligned rows out).
constexpr int QR_THREADS = 128;
template <bool VEC>
__global__ void __launch_bounds__(QR_THREADS)
quant_rows_kernel(const __nv_bfloat16* __restrict__ src, int ld, int C, uint8_t* __restrict__ dst, int ld_dst,
                  float* __restrict__ scale) {
  __shared__ float red[QR_THREADS / 32];
  const __nv_bfloat16* x = src + (size_t)blockIdx.x * ld;
  uint8_t* y = dst + (size_t)blockIdx.x * ld_dst;
  float m = 0.f;
  if constexpr (VEC) {
    for (int c = 8 * threadIdx.x; c < C; c += 8 * QR_THREADS) {
      const uint4 v = *reinterpret_cast<const uint4*>(x + c);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16(w[j]);
        m = fmaxf(m, fmaxf(finite_abs(f.x), finite_abs(f.y)));
      }
    }
  } else {
    for (int c = threadIdx.x; c < C; c += QR_THREADS) m = fmaxf(m, finite_abs(__bfloat162float(x[c])));
  }
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int i = 1; i < QR_THREADS / 32; ++i) m = fmaxf(m, red[i]);
  const float s = e4m3_scale(m);
  if (threadIdx.x == 0) scale[blockIdx.x] = s;
  if constexpr (VEC) {
    for (int c = 8 * threadIdx.x; c < C; c += 8 * QR_THREADS) {
      const uint4 v = *reinterpret_cast<const uint4*>(x + c);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
      uint32_t q[2];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const float2 f0 = unpack_bf16(w[2 * j]), f1 = unpack_bf16(w[2 * j + 1]);
        q[j] = (uint32_t)e4m3x2(f0.x, f0.y, s) | ((uint32_t)e4m3x2(f1.x, f1.y, s) << 16);
      }
      *reinterpret_cast<uint2*>(y + c) = make_uint2(q[0], q[1]);
    }
  } else {
    for (int c = threadIdx.x; c < C; c += QR_THREADS) y[c] = (uint8_t)e4m3x2(__bfloat162float(x[c]), 0.f, s);
  }
}

// column maxima of a [R, C] bf16 matrix: a CTA takes 64 columns x 128 rows; the per-column result is max-ed into amax
// (the zeroed scale vector; a non-negative float orders like its bits as an unsigned integer, so atomicMax on the bits
// is the max)
constexpr int QC_COLS = 64, QC_ROWS = 128;
__global__ void __launch_bounds__(256)
colmax_kernel(const __nv_bfloat16* __restrict__ src, int ld, int R, int C, unsigned* __restrict__ amax) {
  __shared__ float red[4][QC_COLS];
  const int c = blockIdx.x * QC_COLS + (threadIdx.x & 63), ry = threadIdx.x >> 6;
  float m = 0.f;
  if (c < C) {
    const int r1 = min(R, (int)(blockIdx.y + 1) * QC_ROWS);
    for (int r = blockIdx.y * QC_ROWS + ry; r < r1; r += 4) m = fmaxf(m, finite_abs(__bfloat162float(src[(size_t)r * ld + c])));
  }
  red[ry][threadIdx.x & 63] = m;
  __syncthreads();
  if (ry == 0 && c < C) {
    m = fmaxf(fmaxf(red[0][threadIdx.x], red[1][threadIdx.x]), fmaxf(red[2][threadIdx.x], red[3][threadIdx.x]));
    atomicMax(amax + c, __float_as_uint(m));
  }
}

// the column maxima (bits, in place) -> the column scales
__global__ void col_scale_kernel(float* __restrict__ scale, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) scale[c] = e4m3_scale(scale[c]);
}

// a 64 x 64 tile of W [R, C] -> the transposed 64 x 64 tile of dst [C, R], each column by its own scale
constexpr int QT = 64, QT_PITCH = QT + 4;
__global__ void __launch_bounds__(256)
quant_cols_t_kernel(const __nv_bfloat16* __restrict__ src, int ld, int R, int C, const float* __restrict__ scale,
                    uint8_t* __restrict__ dst, int ld_dst) {
  __shared__ __align__(16) uint8_t tile[QT][QT_PITCH];   // [column][row]
  const int r0 = blockIdx.y * QT, c0 = blockIdx.x * QT;
  const int cl = threadIdx.x & 63, c = c0 + cl;
  const float s = c < C ? scale[c] : 1.f;
  for (int rl = threadIdx.x >> 6; rl < QT; rl += 4) {
    const int r = r0 + rl;
    const float v = (r < R && c < C) ? __bfloat162float(src[(size_t)r * ld + c]) : 0.f;
    tile[cl][rl] = (uint8_t)e4m3x2(v, 0.f, s);
  }
  __syncthreads();
  // dst row c0 + (t >> 2), bytes r0 + 16 (t & 3) .. + 15
  const int oc = c0 + (threadIdx.x >> 2), orow = 16 * (threadIdx.x & 3);
  if (oc >= C) return;
  const uint8_t* t = &tile[threadIdx.x >> 2][orow];
  uint8_t* y = dst + (size_t)oc * ld_dst + r0 + orow;
  if (r0 + orow + 16 <= R && ((reinterpret_cast<uintptr_t>(y) & 15) == 0)) {
    const uint32_t* t4 = reinterpret_cast<const uint32_t*>(t);
    *reinterpret_cast<uint4*>(y) = make_uint4(t4[0], t4[1], t4[2], t4[3]);
  } else {
    for (int j = 0; j < 16 && r0 + orow + j < R; ++j) y[j] = t[j];
  }
}

}  // namespace d3

using namespace d3;

extern "C" {

int d3_quant_rows_e4m3(const void* src_bf16, int ld, int R, int C, void* dst_u8, int ld_dst, float* scale,
                       void* stream) {
  if (!src_bf16 || !dst_u8 || !scale) return set_error(D3_ERR_ARG, "d3_quant_rows_e4m3: null pointer");
  if (R <= 0 || C <= 0 || ld < C || ld_dst < C) return set_error(D3_ERR_ARG, "d3_quant_rows_e4m3: bad shape");
  const bool vec = C % 8 == 0 && ld % 8 == 0 && ld_dst % 8 == 0 && (reinterpret_cast<uintptr_t>(src_bf16) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(dst_u8) & 7) == 0;
  const auto* x = static_cast<const __nv_bfloat16*>(src_bf16);
  auto* y = static_cast<uint8_t*>(dst_u8);
  if (vec) quant_rows_kernel<true><<<R, QR_THREADS, 0, STREAM(stream)>>>(x, ld, C, y, ld_dst, scale);
  else quant_rows_kernel<false><<<R, QR_THREADS, 0, STREAM(stream)>>>(x, ld, C, y, ld_dst, scale);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_quant_cols_e4m3_t(const void* src_bf16, int ld, int R, int C, void* dst_u8, int ld_dst, float* scale,
                         void* stream) {
  if (!src_bf16 || !dst_u8 || !scale) return set_error(D3_ERR_ARG, "d3_quant_cols_e4m3_t: null pointer");
  if (R <= 0 || C <= 0 || ld < C || ld_dst < R) return set_error(D3_ERR_ARG, "d3_quant_cols_e4m3_t: bad shape");
  // column maxima into the zeroed scale vector, converted in place, then the transposing quantization: no workspace
  cudaStream_t st = STREAM(stream);
  cudaError_t e = cudaMemsetAsync(scale, 0, (size_t)C * sizeof(float), st);
  if (e != cudaSuccess) return set_error(D3_ERR_CUDA, cudaGetErrorString(e));
  const auto* x = static_cast<const __nv_bfloat16*>(src_bf16);
  colmax_kernel<<<dim3((C + QC_COLS - 1) / QC_COLS, (R + QC_ROWS - 1) / QC_ROWS), 256, 0, st>>>(
      x, ld, R, C, reinterpret_cast<unsigned*>(scale));
  D3_CHECK_LAUNCH();
  col_scale_kernel<<<(C + 255) / 256, 256, 0, st>>>(scale, C);
  D3_CHECK_LAUNCH();
  quant_cols_t_kernel<<<dim3((C + QT - 1) / QT, (R + QT - 1) / QT), 256, 0, st>>>(x, ld, R, C, scale,
                                                                                  static_cast<uint8_t*>(dst_u8), ld_dst);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

}  // extern "C"
