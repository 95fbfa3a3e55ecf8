// Linear-probe evaluation of a frozen backbone (the DINOv2 / DINOv3 linear protocol): the classifiers' input rows and
// the cross-entropy of many linear classifiers trained at once on the same features.  The logits and the weight
// gradients are d3_gemm_bf16, the bias gradients d3_colsum_bf16, the update d3_sgd_momentum (optim.cu) and the patch
// mean d3_pool_tokens; nothing here multiplies matrices.
//
// Deterministic: no float atomics, every sum in a fixed order.
#include "ptx.cuh"
#include "d3_internal.h"

#include <math.h>

namespace d3 {

// ------------------------------------------------------------------------------------------------------ input rows
// out[b, s * D + c] = bf16(src_s[b, c]) for the sources in order: the class tokens of the last n_max blocks and the
// patch mean of the last block make one row [cls_{L-n_max} | ... | cls_{L-1} | mean(patches_{L-1})].  A thread moves
// four channels of one source.
constexpr int LIN_MAX_SRC = 32;
struct LinSources { const float* p[LIN_MAX_SRC]; };

__global__ void linear_inputs_kernel(LinSources srcs, int n_src, int D, __nv_bfloat16* __restrict__ out, int ld_out) {
  const int b = blockIdx.y, q = D / 4;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n_src * q; t += gridDim.x * blockDim.x) {
    const int s = t / q, c = 4 * (t % q);
    const float4 v = *reinterpret_cast<const float4*>(srcs.p[s] + (size_t)b * D + c);
    *reinterpret_cast<uint2*>(out + (size_t)b * ld_out + (size_t)s * D + c) =
        make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
  }
}

// ---------------------------------------------------------------------------------------------------- cross-entropy
// One CTA per (classifier g, row b) of the fp32 logits [B, G * Cp]; the classifier's logits are columns
// [g * Cp, g * Cp + C).  Each thread keeps an online (max, sum of exp) over its columns in increasing order; the
// threads combine by a butterfly within each warp and the warps in order, so (max, sum) have the same bits on every
// run.  dZ = (softmax - onehot(label)) / B in bf16, 0 in the padding columns [C, Cp); the row's loss
// (log-sum-exp - z[label]) / B goes to slab b of the workspace, summed over rows in row order by slab_combine.
constexpr int XE_THREADS = 256;

__device__ __forceinline__ void lse_merge(float& m, float& s, float om, float os) {
  const float mx = fmaxf(m, om);
  if (mx == -INFINITY) return;                               // both empty
  s = s * expf(m - mx) + os * expf(om - mx);
  m = mx;
}

__global__ void __launch_bounds__(XE_THREADS) linear_xent_kernel(const float* __restrict__ logits, int ld,
                                                                 const int* __restrict__ labels, int B, int G, int C,
                                                                 int Cp, float* __restrict__ row_loss,
                                                                 __nv_bfloat16* __restrict__ dz, int ld_dz) {
  __shared__ float wm[XE_THREADS / 32], ws[XE_THREADS / 32];
  const int g = blockIdx.x, b = blockIdx.y, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const float* z = logits + (size_t)b * ld + (size_t)g * Cp;
  float m = -INFINITY, s = 0.f;
  for (int c = threadIdx.x; c < C; c += XE_THREADS) {
    const float v = z[c];
    if (v > m) { s = s * expf(m - v) + 1.f; m = v; } else { s += expf(v - m); }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o), os = __shfl_xor_sync(0xffffffffu, s, o);
    lse_merge(m, s, om, os);
  }
  if (lane == 0) { wm[wid] = m; ws[wid] = s; }
  __syncthreads();
  m = wm[0]; s = ws[0];
  for (int w = 1; w < XE_THREADS / 32; ++w) lse_merge(m, s, wm[w], ws[w]);
  // softmax = exp(z - max) / sum and loss = (max - z[y]) + log(sum): z - max is exact near the max, so a probability
  // close to 1 keeps its last bits (exp(z - lse) would inherit the rounding of lse, up to |z| ulps)
  const int y = labels[b];
  const float inv_b = 1.f / (float)B;
  __nv_bfloat16* d = dz + (size_t)b * ld_dz + (size_t)g * Cp;
  for (int c = threadIdx.x; c < Cp; c += XE_THREADS) {
    float v = 0.f;
    if (c < C) v = (expf(z[c] - m) / s - (c == y ? 1.f : 0.f)) * inv_b;
    d[c] = __float2bfloat16(v);
  }
  if (threadIdx.x == 0)
    row_loss[(size_t)b * G + g] = (y >= 0 && y < C) ? ((m - z[y]) + logf(s)) * inv_b : __int_as_float(0x7fc00000);
}

}  // namespace d3

using namespace d3;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

int d3_linear_inputs(const float* const* srcs, int n_src, int B, int D, void* out, int ld_out, void* stream) {
  if (B <= 0) return D3_OK;
  if (!srcs || !out || n_src < 1 || n_src > LIN_MAX_SRC || D < 4 || D % 4 || ld_out < n_src * D || ld_out % 4 ||
      (uintptr_t)out % 8)
    return set_error(D3_ERR_ARG, "d3_linear_inputs: need 1 <= n_src <= 32, D a positive multiple of 4, "
                                 "ld_out >= n_src * D a multiple of 4, out 8-byte aligned");
  LinSources s{};
  for (int i = 0; i < n_src; ++i) {
    if (!srcs[i] || (uintptr_t)srcs[i] % 16) return set_error(D3_ERR_ARG, "d3_linear_inputs: sources must be 16-byte aligned");
    s.p[i] = srcs[i];
  }
  const int work = n_src * (D / 4);
  const dim3 grid((work + 255) / 256, B);
  linear_inputs_kernel<<<grid, 256, 0, STREAM(stream)>>>(s, n_src, D, (__nv_bfloat16*)out, ld_out);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_linear_xent_fwd_bwd(const float* logits, int ld, const int* labels, int B, int G, int C, int Cp, float* loss,
                           void* dz, int ld_dz, void* stream) {
  if (B <= 0 || G <= 0) return D3_OK;
  if (!logits || !labels || !loss || !dz || C < 2 || C > 32768 || Cp < C || Cp % 8 || ld < G * Cp || ld_dz < G * Cp)
    return set_error(D3_ERR_ARG, "d3_linear_xent_fwd_bwd: need 2 <= C <= 32768, Cp >= C a multiple of 8, "
                                 "ld and ld_dz >= G * Cp");
  cudaStream_t st = STREAM(stream);
  float* ws = slab_workspace((size_t)B * G, st);
  if (!ws) return D3_ERR_CUDA;
  linear_xent_kernel<<<dim3(G, B), XE_THREADS, 0, st>>>(logits, ld, labels, B, G, C, Cp, ws, (__nv_bfloat16*)dz, ld_dz);
  cudaError_t e = cudaPeekAtLastError();
  if (e == cudaSuccess) e = cudaMemsetAsync(loss, 0, (size_t)G * sizeof(float), st);
  int rc = e == cudaSuccess ? D3_OK : set_error(D3_ERR_CUDA, cudaGetErrorString(e));
  if (!rc) { count_launch(); rc = slab_combine(ws, B, G, 1, G, loss, G, st); }
  slab_release(ws, st);
  return rc;
}

}  // extern "C"
