// Optimiser kernels on flat fp32 parameter shards: squared-norm reduction (for the per-submodule clip,
// dinov3_jax/train/train.py:516-541) and a fused clip + AdamW (optax.adamw semantics, train/train.py:95-106,562-563)
// + teacher EMA (train/ssl_meta_arch.py:650-652) + bf16 re-cast of the compute copies; and the SGD-momentum update of
// the linear-probe classifiers.
#include <cmath>
#include "ptx.cuh"
#include "d3_internal.h"

namespace d3 {

// each CTA's share of sum(g^2) goes to ws[blockIdx.x]; the shares are added in CTA order (reproducible clip factor)
__global__ void sumsq_kernel(const float* __restrict__ g, long n, float* __restrict__ ws) {
  __shared__ float sh[32];
  float acc = 0.f;
  const long n4 = n / 4;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
    float4 v = reinterpret_cast<const float4*>(g)[i];
    acc += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  if (blockIdx.x == 0)
    for (long i = n4 * 4 + threadIdx.x; i < n; i += blockDim.x) acc += g[i] * g[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (threadIdx.x == 0) ws[blockIdx.x] = t;
  }
}

// segment table: one entry per parameter tensor inside the flat buffer (starts are multiples of 4 elements)
struct Seg {
  long long start;  // element offset of the tensor in the flat buffer
  float lr_mult, wd_mult;
  int is_last_layer, pad;
};

// p, m, v, teacher: fp32 flat [n].  g: fp32 flat [n] (already averaged over ranks).
// clip scale = min(1, max_norm / (sqrt(sumsq[0]) + 1e-6)) read on device (no host sync).
__global__ void adamw_ema_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                 float* __restrict__ v, float* __restrict__ teacher,
                                 __nv_bfloat16* __restrict__ p_bf16, __nv_bfloat16* __restrict__ t_bf16,
                                 long n_bf16,  // leading elements that have a bf16 compute copy (matrix region)
                                 const Seg* __restrict__ segs, int nseg, long n, const float* __restrict__ sumsq,
                                 float max_norm, float lr, float last_layer_lr, float wd, float b1, float b2, float eps,
                                 float bc1, float bc2, float momentum) {
  const long i4 = (blockIdx.x * (long)blockDim.x + threadIdx.x) * 4;
  if (i4 >= n) return;
  // find segment containing i4 (binary search on starts)
  int lo = 0, hi = nseg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (segs[mid].start <= i4) lo = mid; else hi = mid - 1;
  }
  const Seg sg = segs[lo];
  float scale = 1.f;
  if (max_norm > 0.f) scale = fminf(1.f, max_norm / (sqrtf(*sumsq) + 1e-6f));
  const float lr_eff = sg.lr_mult * (sg.is_last_layer ? last_layer_lr : lr);
  const float wd_eff = sg.wd_mult * wd;
  float pv[4], gv[4], mv[4], vv[4], tv[4];
  *reinterpret_cast<float4*>(pv) = *reinterpret_cast<const float4*>(p + i4);
  *reinterpret_cast<float4*>(gv) = *reinterpret_cast<const float4*>(g + i4);
  *reinterpret_cast<float4*>(mv) = *reinterpret_cast<const float4*>(m + i4);
  *reinterpret_cast<float4*>(vv) = *reinterpret_cast<const float4*>(v + i4);
  *reinterpret_cast<float4*>(tv) = *reinterpret_cast<const float4*>(teacher + i4);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float gg = gv[j] * scale;
    mv[j] = b1 * mv[j] + (1.f - b1) * gg;
    vv[j] = b2 * vv[j] + (1.f - b2) * gg * gg;
    const float mh = mv[j] / bc1, vh = vv[j] / bc2;
    pv[j] = pv[j] - lr_eff * (mh / (sqrtf(vh) + eps) + wd_eff * pv[j]);
    tv[j] = tv[j] * momentum + pv[j] * (1.f - momentum);
  }
  *reinterpret_cast<float4*>(p + i4) = *reinterpret_cast<float4*>(pv);
  *reinterpret_cast<float4*>(m + i4) = *reinterpret_cast<float4*>(mv);
  *reinterpret_cast<float4*>(v + i4) = *reinterpret_cast<float4*>(vv);
  *reinterpret_cast<float4*>(teacher + i4) = *reinterpret_cast<float4*>(tv);
  if (i4 < n_bf16) {
    *reinterpret_cast<uint2*>(p_bf16 + i4) = make_uint2(pack_bf16(pv[0], pv[1]), pack_bf16(pv[2], pv[3]));
    *reinterpret_cast<uint2*>(t_bf16 + i4) = make_uint2(pack_bf16(tv[0], tv[1]), pack_bf16(tv[2], tv[3]));
  }
}

// teacher <- m*teacher + (1-m)*student on a flat shard, with the bf16 re-cast of the teacher's matrix region: the
// stand-alone form of the EMA (train/ssl_meta_arch.py:644-660: `update_ema()` returns fn(ema, params, mom)) for callers
// that keep the reference's two-call step (train_step, then update_ema); the engine's own loop uses the fused kernel.
__global__ void ema_kernel(float* __restrict__ teacher, const float* __restrict__ student,
                           __nv_bfloat16* __restrict__ t_bf16, long n_bf16, long n, float momentum) {
  const long i4 = (blockIdx.x * (long)blockDim.x + threadIdx.x) * 4;
  if (i4 >= n) return;
  float4 t = *reinterpret_cast<const float4*>(teacher + i4);
  const float4 p = *reinterpret_cast<const float4*>(student + i4);
  const float w = 1.f - momentum;
  t.x = t.x * momentum + p.x * w; t.y = t.y * momentum + p.y * w;
  t.z = t.z * momentum + p.z * w; t.w = t.w * momentum + p.w * w;
  *reinterpret_cast<float4*>(teacher + i4) = t;
  if (i4 < n_bf16) *reinterpret_cast<uint2*>(t_bf16 + i4) = make_uint2(pack_bf16(t.x, t.y), pack_bf16(t.z, t.w));
}

// torch.optim.SGD(momentum, dampening = 0, nesterov = False, weight_decay = 0) on a [rows, cols] fp32 matrix whose
// rows come in groups of Cp per classifier: buf = first ? g : momentum * buf + g (torch's mul_ then add_, two
// roundings), p = p - lr * buf with lr = lr_base[(i / cols) / Cp] * lr_scale; the bf16 copy the next forward GEMM reads
// is written alongside.  Four elements per thread (n % 4 == 0).
__global__ void sgd_momentum_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                    __nv_bfloat16* __restrict__ p_bf16, long n, int cols, const float* __restrict__ lr,
                                    int Cp, float lr_scale, float momentum, int first) {
  const long i4 = (blockIdx.x * (long)blockDim.x + threadIdx.x) * 4;
  if (i4 >= n) return;
  float pv[4], gv[4], mv[4];
  *reinterpret_cast<float4*>(pv) = *reinterpret_cast<const float4*>(p + i4);
  *reinterpret_cast<float4*>(gv) = *reinterpret_cast<const float4*>(g + i4);
  if (!first) *reinterpret_cast<float4*>(mv) = *reinterpret_cast<const float4*>(m + i4);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float l = lr[(i4 + j) / cols / Cp] * lr_scale;
    mv[j] = first ? gv[j] : __fadd_rn(__fmul_rn(mv[j], momentum), gv[j]);
    pv[j] = fmaf(-l, mv[j], pv[j]);
  }
  *reinterpret_cast<float4*>(p + i4) = *reinterpret_cast<float4*>(pv);
  *reinterpret_cast<float4*>(m + i4) = *reinterpret_cast<float4*>(mv);
  if (p_bf16) *reinterpret_cast<uint2*>(p_bf16 + i4) = make_uint2(pack_bf16(pv[0], pv[1]), pack_bf16(pv[2], pv[3]));
}

}  // namespace d3

using namespace d3;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

int d3_sumsq(const float* g, long long n, float* out, void* stream) {
  if (n <= 0) return D3_OK;
  if ((uintptr_t)g & 15) return set_error(D3_ERR_ARG, "d3_sumsq: alignment");
  cudaStream_t st = STREAM(stream);
  const int blocks = (int)min((n / 4 + 255) / 256 + 1, (long long)sm_count() * 8);
  float* ws = slab_workspace(blocks, st);
  if (!ws) return D3_ERR_CUDA;
  sumsq_kernel<<<blocks, 256, 0, st>>>(g, n, ws);
  cudaError_t e = cudaPeekAtLastError();
  int rc = e == cudaSuccess ? D3_OK : set_error(D3_ERR_CUDA, cudaGetErrorString(e));
  if (!rc) { count_launch(); rc = slab_combine(ws, blocks, 1, 1, 1, out, 1, st); }
  slab_release(ws, st);
  return rc;
}

int d3_adamw_ema(float* p, const float* g, float* m, float* v, float* teacher, void* p_bf16, void* t_bf16,
                 long long n_bf16, const void* segs, int nseg, long long n, const float* sumsq, float max_norm, float lr,
                 float last_layer_lr, float wd, float b1, float b2, float eps, int step, float momentum, void* stream) {
  if (n <= 0) return D3_OK;
  if (n % 4 || n_bf16 % 4 || nseg <= 0) return set_error(D3_ERR_ARG, "d3_adamw_ema: n, n_bf16 must be multiples of 4");
  const float bc1 = (float)(1.0 - pow((double)b1, (double)step)), bc2 = (float)(1.0 - pow((double)b2, (double)step));
  const long th = n / 4;
  adamw_ema_kernel<<<(int)((th + 255) / 256), 256, 0, STREAM(stream)>>>(
      p, g, m, v, teacher, (__nv_bfloat16*)p_bf16, (__nv_bfloat16*)t_bf16, n_bf16, (const Seg*)segs, nseg, n, sumsq,
      max_norm, lr, last_layer_lr, wd, b1, b2, eps, bc1, bc2, momentum);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_ema(float* teacher, const float* student, void* t_bf16, long long n_bf16, long long n, float momentum,
           void* stream) {
  if (n <= 0) return D3_OK;
  if (n % 4 || n_bf16 % 4) return set_error(D3_ERR_ARG, "d3_ema: n, n_bf16 must be multiples of 4");
  ema_kernel<<<(int)((n / 4 + 255) / 256), 256, 0, STREAM(stream)>>>(teacher, student, (__nv_bfloat16*)t_bf16, n_bf16, n,
                                                                  momentum);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_sgd_momentum(float* p, const float* g, float* m, void* p_bf16, long long rows, int cols, const float* lr, int Cp,
                    float lr_scale, float momentum, int first, void* stream) {
  if (rows <= 0) return D3_OK;
  const long long n = rows * cols;
  if (!p || !g || !m || !lr || cols < 1 || Cp < 1 || n % 4 || ((uintptr_t)p | (uintptr_t)g | (uintptr_t)m) % 16 ||
      (uintptr_t)p_bf16 % 8)
    return set_error(D3_ERR_ARG, "d3_sgd_momentum: need rows * cols % 4 == 0, p, g, m 16-byte and p_bf16 8-byte aligned");
  sgd_momentum_kernel<<<(int)((n / 4 + 255) / 256), 256, 0, STREAM(stream)>>>(
      p, g, m, (__nv_bfloat16*)p_bf16, n, cols, lr, Cp, lr_scale, momentum, first ? 1 : 0);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

}  // extern "C"
