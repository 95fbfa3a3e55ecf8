// Loss-head kernels: Sinkhorn-Knopp teacher normalisation (as diagonal scalings of exp(logits/temp)),
// fused cross-entropy forward+backward over the prototype dimension, KoLeo regulariser forward+backward.
// References: dinov3_jax/loss/dino_clstoken_loss.py:35-89, loss/ibot_patch_loss.py:13-14,45-109,
// loss/koleo_loss.py:16-35, train/ssl_meta_arch.py:463-525.
#include <math_constants.h>
#include "ptx.cuh"
#include "d3_internal.h"

namespace d3 {

// block reductions over 256 threads (8 warps)
__device__ __forceinline__ float block_sum(float v, float* sh) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = (threadIdx.x < (blockDim.x >> 5)) ? sh[threadIdx.x] : 0.f;
  if (threadIdx.x < 32) t = warp_sum(t);
  if (threadIdx.x == 0) sh[0] = t;
  __syncthreads();
  return sh[0];
}
__device__ __forceinline__ float block_max(float v, float* sh) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = (threadIdx.x < (blockDim.x >> 5)) ? sh[threadIdx.x] : -CUDART_INF_F;
  if (threadIdx.x < 32) t = warp_max(t);
  if (threadIdx.x == 0) sh[0] = t;
  __syncthreads();
  return sh[0];
}
// Elements 4g .. 4g+3 of a row of n floats.  VEC: one 128-bit load (the row is 16-byte aligned and n % 4 == 0).
// Otherwise four scalar loads, and an element at or past n reads as `fill`, the neutral value of the reduction it
// enters, so that both instances walk the same four-column groups.
template <bool VEC, class I>
__device__ __forceinline__ float4 load4(const float* __restrict__ row, I g, I n, float fill) {
  if constexpr (VEC) {
    return reinterpret_cast<const float4*>(row)[g];
  } else {
    const I k = 4 * g;
    return make_float4(k < n ? row[k] : fill, k + 1 < n ? row[k + 1] : fill, k + 2 < n ? row[k + 2] : fill,
                       k + 3 < n ? row[k + 3] : fill);
  }
}
// 1/s for a Sinkhorn column sum; a column whose terms all underflowed (s == 0) contributes nothing instead of 0/0
__device__ __forceinline__ float rcp_pos(float s) { return s > 0.f ? __fdividef(1.f, s) : 0.f; }
__device__ __forceinline__ void atomic_max_float(float* addr, float v) {
  // ordered-int trick; *addr must be initialised to -inf
  if (v >= 0.f) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
  else atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}

// ------------------------------------------------------------------------------------------------ Sinkhorn-Knopp
// Q = exp(L/temp)^T; Q/=sum; 3x { Q /= rowsum*K ; Q /= colsum*B } ; Q*=B      (dino_clstoken_loss.py:35-62)
// is a sequence of diagonal scalings:  Q[b,k] = E[b,k] * r[k] * a[b],  E = exp((L[b,k] - cm[k])/temp), with
//   r = 1/(K * E^T a)   and   a = 1/(B * E r)   alternating.  Any per-COLUMN shift cm[k] cancels exactly in E*r (the
// reference has no shift at all, :39); cm[k] = max_b L[b,k] (d3_colmax, all-reduced over ranks) keeps every column's
// largest term at 1, so a prototype far below the batch maximum keeps its Sinkhorn mass 1/K like in the reference
// instead of underflowing to 0/0 (a single global shift loses columns more than ~3.5 below the maximum at temp 0.04).
// The row step's E^T a (K floats) is what the reference psums over "dp" (:53 / ibot :99).
// absmax, colmax, sk_rowsum and the cross-entropy take four columns per thread.  VEC reads them with 128-bit loads,
// used when K % 4 == 0 and the rows are 16-byte aligned (every recipe: K = 65536); otherwise the same walk reads them
// with scalar loads (load4).
// n4 = ceil(n / 4) groups of four elements
template <bool VEC>
__global__ void absmax_kernel(const float* __restrict__ L, long n4, float* __restrict__ out, long n) {
  __shared__ float sh[32];
  float m = -CUDART_INF_F;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
    const float4 v = load4<VEC>(L, i, n, -CUDART_INF_F);
    m = fmaxf(fmaxf(m, fmaxf(v.x, v.y)), fmaxf(v.z, v.w));
  }
  m = block_max(m, sh);
  if (threadIdx.x == 0) atomic_max_float(out, m);
}
// cm[k] = max(cm[k], max_b L[b,k])   (cm pre-set to -inf; atomics across row slabs), four columns per thread
template <bool VEC>
__global__ void colmax_kernel(const float* __restrict__ L, float* __restrict__ cm, int R, int K) {
  const int k = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const int slab = (R + gridDim.y - 1) / gridDim.y;
  const int r0 = blockIdx.y * slab, r1 = min(R, r0 + slab);
  if (k >= K || r0 >= r1) return;
  float4 m = make_float4(-CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F);
#pragma unroll 4
  for (int b = r0; b < r1; ++b) {
    const float4 v = load4<VEC>(L + (long)b * K + k, 0, K - k, -CUDART_INF_F);   // row b from column k on
    m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
  }
  const float mv[4] = {m.x, m.y, m.z, m.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if constexpr (!VEC) if (k + j >= K) break;
    atomic_max_float(&cm[k + j], mv[j]);
  }
}
// Sinkhorn column sums, part[slab][k] = sum over the row slab of E[b,k] * a[b]  (a == nullptr -> a = 1); slab_combine
// then adds the slabs in a fixed order.  Float atomics here would perturb s[k] in the last bit from run to run, which
// flips a few bf16 roundings of the iBOT d(logits) and grows to ~3e-3 in the embedding gradients through the bf16
// backward chain (tools/check_determinism.py); with the slabs the whole dX chain of a step is bit-reproducible.
// VEC: four columns per thread with 128-bit loads (K % 4 == 0, 16-byte aligned L and mx); otherwise one column.
template <bool VEC>
__global__ void sk_colsum_part_kernel(const float* __restrict__ L, const float* __restrict__ mx, float inv_temp,
                                      const float* __restrict__ a, float* __restrict__ part, int R, int K) {
  const int k = (blockIdx.x * blockDim.x + threadIdx.x) * (VEC ? 4 : 1);
  const int slab = (R + gridDim.y - 1) / gridDim.y;
  const int r0 = blockIdx.y * slab, r1 = min(R, r0 + slab);
  if (k >= K) return;
  const float c = inv_temp * 1.4426950408889634f;
  if constexpr (VEC) {
    const float4 m4 = *reinterpret_cast<const float4*>(mx + k);
    const float4 mc = make_float4(m4.x * c, m4.y * c, m4.z * c, m4.w * c);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
    for (int b = r0; b < r1; ++b) {
      const float4 v = *reinterpret_cast<const float4*>(L + (long)b * K + k);
      const float w = a ? a[b] : 1.f;
      acc.x += exp2f(v.x * c - mc.x) * w; acc.y += exp2f(v.y * c - mc.y) * w;
      acc.z += exp2f(v.z * c - mc.z) * w; acc.w += exp2f(v.w * c - mc.w) * w;
    }
    *reinterpret_cast<float4*>(part + (long)blockIdx.y * K + k) = acc;
  } else {
    const float mc = mx[k] * c;
    float acc = 0.f;
#pragma unroll 4
    for (int b = r0; b < r1; ++b) acc += exp2f(L[(long)b * K + k] * c - mc) * (a ? a[b] : 1.f);
    part[(long)blockIdx.y * K + k] = acc;
  }
}
// a[b] = 1 / (Btot * sum_k E[b,k] * r[k]),  r[k] = 1/(K*s[k])
template <bool VEC>
__global__ void sk_rowsum_kernel(const float* __restrict__ L, const float* __restrict__ mx, float inv_temp,
                                 const float* __restrict__ s, const float* __restrict__ btot, float* __restrict__ a,
                                 int R, int K) {
  __shared__ float sh[32];
  const int b = blockIdx.x;
  const float c = inv_temp * 1.4426950408889634f;
  const float* Lb = L + (long)b * K;
  float acc = 0.f;
#pragma unroll 4
  for (int k = threadIdx.x; k < (VEC ? K / 4 : (K + 3) / 4); k += blockDim.x) {
    // past the row E = 2^-inf = 0 and r = rcp_pos(0) = 0
    const float4 v = load4<VEC>(Lb, k, K, -CUDART_INF_F), sv = load4<VEC>(s, k, K, 0.f), mv = load4<VEC>(mx, k, K, 0.f);
    acc += exp2f((v.x - mv.x) * c) * rcp_pos(sv.x) + exp2f((v.y - mv.y) * c) * rcp_pos(sv.y) +
           exp2f((v.z - mv.z) * c) * rcp_pos(sv.z) + exp2f((v.w - mv.w) * c) * rcp_pos(sv.w);
  }
  acc = block_sum(acc, sh) / (float)K;
  if (threadIdx.x == 0) a[b] = acc > 0.f ? 1.f / (*btot * acc) : 0.f;
}
// Q[b,k] for teacher logit t = L[b,k], shift m = mx[k], ct = log2(e) / temp, r = rcp_pos(s[k]) and
// coef = Btot * a[b] / K.  The cross-entropy and sk_probs_kernel both evaluate it here, so the Q a test materialises
// is the Q behind dS.  It takes r rather than s so that the cross-entropy computes r once for both teacher rows.
__device__ __forceinline__ float teacher_prob(float t, float m, float ct, float r, float coef) {
  return coef * exp2f((t - m) * ct) * r;
}
// materialise teacher probabilities (tests / optional consumers)
__global__ void sk_probs_kernel(const float* __restrict__ L, const float* __restrict__ mx, float inv_temp,
                                const float* __restrict__ s, const float* __restrict__ a,
                                const float* __restrict__ btot, float* __restrict__ Q, int R, int K) {
  const long n = (long)R * K;
  const float bt = *btot, ct = inv_temp * 1.4426950408889634f, invK = 1.f / (float)K;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int b = (int)(i / K), k = (int)(i % K);
    Q[i] = teacher_prob(L[i], mx[k], ct, rcp_pos(s[k]), bt * a[b] * invK);
  }
}


// ------------------------------------------------------------------------------------------------ softmax centering
// Optional teacher normalisation (loss/dino_clstoken_loss.py:24-33,91-95; loss/ibot_patch_loss.py:28-36,69-73):
//   center <- m*center + (1-m)*mean_rows(L)  (mean all-reduced over ranks), probs = softmax((L - center)/temp).
// With s[k] = exp((center[k]-cmax)/temp)/K the existing row-sum kernel yields a[b] such that
// Btot*E*a[b]/(K*s[k]) = softmax((L-center)/temp): the cross-entropy kernel is shared with the Sinkhorn path.
// ws[slab][k] = sum over the row slab of L[b, k]   (the slabs are added in order by slab_combine)
__global__ void colsum_f32_kernel(const float* __restrict__ L, float* __restrict__ ws, int R, int K) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const int slab = (R + gridDim.y - 1) / gridDim.y;
  const int r0 = blockIdx.y * slab, r1 = min(R, r0 + slab);
  if (k >= K) return;
  float acc = 0.f;
  for (int b = r0; b < r1; ++b) acc += L[(long)b * K + k];
  ws[(long)blockIdx.y * K + k] = acc;
}
__global__ void center_update_kernel(float* __restrict__ center, const float* __restrict__ colsum,
                                     const float* __restrict__ total_rows, float momentum, float inv_temp,
                                     float* __restrict__ s_out, int K) {
  __shared__ float sh[32];
  const float inv_rows = 1.f / *total_rows;
  float mx = -CUDART_INF_F;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const float c = center[k] * momentum + colsum[k] * inv_rows * (1.f - momentum);
    center[k] = c;
    mx = fmaxf(mx, c);
  }
  mx = block_max(mx, sh);
  for (int k = threadIdx.x; k < K; k += blockDim.x) s_out[k] = __expf((center[k] - mx) * inv_temp) / (float)K;
}

// ------------------------------------------------------------------------------------------------ cross-entropy
// per student row i (logits S[i,:]):  loss_i = - sum_p sum_k Q_p[k] * log_softmax(S[i,:]/ts)[k]   over its teacher
// rows p in {t0[i], t1[i]} (-1 = none), Q_p from the Sinkhorn scalings above.
// row_loss[i] = wm[i] * loss_i (added to metric[slot[i]] by metric_rows_kernel) ;  dS[i,k] = wg[i]/ts * (npairs * softmax[k] - sum_p Q_p[k])   (bf16)
// (dino_clstoken_loss.py:66-89; ibot_patch_loss.py:13-14,55-67; weights per train/ssl_meta_arch.py:480-525)
// The second pass re-reads the student row from L2.
template <bool VEC>
__global__ void __launch_bounds__(512)
ce_fwd_bwd_kernel(const float* __restrict__ S, float inv_ts, const float* __restrict__ Lt,
                  const float* __restrict__ mx, float inv_tt, const float* __restrict__ s_t,
                  const float* __restrict__ a_t, const float* __restrict__ btot, const int* __restrict__ t0,
                  const int* __restrict__ t1, const float* __restrict__ wm, const float* __restrict__ wg,
                  const int* __restrict__ slot, float* __restrict__ row_loss, __nv_bfloat16* __restrict__ dS, int K) {
  __shared__ float sh[32];
  const int i = blockIdx.x;
  const int K4 = VEC ? K >> 2 : (K + 3) >> 2;
  const float LOG2E = 1.4426950408889634f;
  const float* Si = S + (long)i * K;
  const float cs = inv_ts * LOG2E;
  // online max / sum of 2^(cs * s) per thread, one float4 at a time (a column past the row adds 2^-inf = 0)
  float m = -CUDART_INF_F, z = 0.f;
#pragma unroll 2
  for (int k = threadIdx.x; k < K4; k += blockDim.x) {
    const float4 v = load4<VEC>(Si, k, K, -CUDART_INF_F);
    const float m4 = fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)) * cs;
    if (m4 > m) { z *= exp2f(m - m4); m = m4; }
    z += exp2f(v.x * cs - m) + exp2f(v.y * cs - m) + exp2f(v.z * cs - m) + exp2f(v.w * cs - m);
  }
  const float gm = block_max(m, sh);
  z = block_sum(z * exp2f(m - gm), sh);
  const float lse2 = gm + log2f(z);                 // log2-domain logsumexp of the scaled row
  const int p0 = t0[i], p1 = t1[i];
  const float np = (p0 >= 0 ? 1.f : 0.f) + (p1 >= 0 ? 1.f : 0.f);
  const float ct = inv_tt * LOG2E;
  const float bt = s_t ? *btot : 1.f;
  const float invK = 1.f / (float)K;
  const float c0 = (s_t && p0 >= 0) ? bt * a_t[p0] * invK : 0.f;
  const float c1 = (s_t && p1 >= 0) ? bt * a_t[p1] * invK : 0.f;
  const float* L0 = Lt + (long)(p0 >= 0 ? p0 : 0) * K;
  const float* L1 = Lt + (long)(p1 >= 0 ? p1 : 0) * K;
  const float g = wg[i] * inv_ts;
  const float LN2 = 0.6931471805599453f;
  __nv_bfloat16* dSi = dS ? dS + (long)i * K : nullptr;
  float loss = 0.f;
#pragma unroll 2
  for (int k = threadIdx.x; k < K4; k += blockDim.x) {
    const float4 v = load4<VEC>(Si, k, K, -CUDART_INF_F);
    float l2[4] = {v.x * cs - lse2, v.y * cs - lse2, v.z * cs - lse2, v.w * cs - lse2};   // log2 softmax
    float q[4] = {0.f, 0.f, 0.f, 0.f};
    if (s_t) {
      const float4 sv = load4<VEC>(s_t, k, K, 0.f), mv = load4<VEC>(mx, k, K, 0.f);
      const float r[4] = {rcp_pos(sv.x), rcp_pos(sv.y), rcp_pos(sv.z), rcp_pos(sv.w)};
      if (p0 >= 0) {
        const float4 t = load4<VEC>(L0, k, K, 0.f);
        q[0] += teacher_prob(t.x, mv.x, ct, r[0], c0); q[1] += teacher_prob(t.y, mv.y, ct, r[1], c0);
        q[2] += teacher_prob(t.z, mv.z, ct, r[2], c0); q[3] += teacher_prob(t.w, mv.w, ct, r[3], c0);
      }
      if (p1 >= 0) {
        const float4 t = load4<VEC>(L1, k, K, 0.f);
        q[0] += teacher_prob(t.x, mv.x, ct, r[0], c1); q[1] += teacher_prob(t.y, mv.y, ct, r[1], c1);
        q[2] += teacher_prob(t.z, mv.z, ct, r[2], c1); q[3] += teacher_prob(t.w, mv.w, ct, r[3], c1);
      }
    } else {          // teacher rows are already probabilities
      if (p0 >= 0) { const float4 t = load4<VEC>(L0, k, K, 0.f); q[0] += t.x; q[1] += t.y; q[2] += t.z; q[3] += t.w; }
      if (p1 >= 0) { const float4 t = load4<VEC>(L1, k, K, 0.f); q[0] += t.x; q[1] += t.y; q[2] += t.z; q[3] += t.w; }
    }
    if constexpr (!VEC) {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (4 * k + j >= K) { q[j] = 0.f; l2[j] = 0.f; }   // past the row: no loss term (not 0 * -inf), no dS below
    }
    loss -= (q[0] * l2[0] + q[1] * l2[1] + q[2] * l2[2] + q[3] * l2[3]) * LN2;
    if (dSi) {
      const float d[4] = {g * (np * exp2f(l2[0]) - q[0]), g * (np * exp2f(l2[1]) - q[1]),
                          g * (np * exp2f(l2[2]) - q[2]), g * (np * exp2f(l2[3]) - q[3])};
      if constexpr (VEC) {
        reinterpret_cast<uint2*>(dSi)[k] = make_uint2(pack_bf16(d[0], d[1]), pack_bf16(d[2], d[3]));
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (4 * k + j < K) dSi[4 * k + j] = __float2bfloat16(d[j]);
      }
    }
  }
  loss = block_sum(loss, sh);
  if (threadIdx.x == 0) row_loss[i] = wm[i] * loss;
}
// Instantiated here, not implicitly at the end of the file: where a kernel sits in the module changes the code NVVM
// makes of it.  Emitted last, this instance compiles to other loop code (1024 SASS instructions instead of 1064).
template __global__ decltype(ce_fwd_bwd_kernel<true>) ce_fwd_bwd_kernel<true>;

// ------------------------------------------------------------------------------------------------ KoLeo
// loss/koleo_loss.py:16-35:  xn = x/(||x||+eps); nn(i) = argmax_{j!=i} xn_i.xn_j; L = -mean_i log(||xn_i - xn_nn(i)|| + 2 eps)
__global__ void koleo_norm_kernel(const float* __restrict__ x, float* __restrict__ xn, float* __restrict__ nrm, int D,
                                  float eps) {
  __shared__ float sh[32];
  const int i = blockIdx.x;
  float s = 0.f;
  for (int e = threadIdx.x; e < D; e += blockDim.x) { const float v = x[(long)i * D + e]; s += v * v; }
  s = block_sum(s, sh);
  const float n = sqrtf(s);
  if (threadIdx.x == 0) nrm[i] = n;
  const float inv = 1.f / (n + eps);
  for (int e = threadIdx.x; e < D; e += blockDim.x) xn[(long)i * D + e] = x[(long)i * D + e] * inv;
}
// Rows [row0, row0 + nrows) are the "local" rows whose terms enter the loss (mean over nrows); neighbours are searched
// over all B rows.  row0 = 0, nrows = B is the plain KoLeo; a sub-range is KoLeoLossDistributed (loss/koleo_loss.py:39-70:
// local rows against the all-gathered rows of every rank).
__global__ void koleo_nn_kernel(const float* __restrict__ xn, int* __restrict__ nn, float* __restrict__ coef,
                                float* __restrict__ row_loss, int B, int D, float eps, float w_metric, float w_grad,
                                int row0, int nrows) {
  __shared__ float sh[32];
  __shared__ float best_v;
  __shared__ int best_j;
  const int i = blockIdx.x;
  if (i < row0 || i >= row0 + nrows) {      // not a local row: no term, no gradient source
    if (threadIdx.x == 0) { nn[i] = i; coef[i] = 0.f; }
    return;
  }
  if (threadIdx.x == 0) { best_v = -CUDART_INF_F; best_j = 0; }
  __syncthreads();
  for (int j = 0; j < B; ++j) {
    float d = 0.f;
    for (int e = threadIdx.x; e < D; e += blockDim.x) d += xn[(long)i * D + e] * xn[(long)j * D + e];
    d = block_sum(d, sh);
    if (threadIdx.x == 0) {
      if (j == i) d = -1.f;                       // dots.at[diag].set(-1)
      if (d > best_v) { best_v = d; best_j = j; } // first maximum, like jnp.argmax
    }
    __syncthreads();
  }
  const int j = best_j;
  float dd = 0.f;
  for (int e = threadIdx.x; e < D; e += blockDim.x) {
    const float t = xn[(long)i * D + e] - xn[(long)j * D + e];
    dd += t * t;
  }
  dd = block_sum(dd, sh);
  if (threadIdx.x == 0) {
    const float dn = sqrtf(dd);
    const float dist = dn + eps;                  // pairwise_distance(...) + eps
    nn[i] = j;
    row_loss[i] = -w_metric * logf(dist + eps) / nrows;
    // d(-w/nrows * log(dist+eps))/d(delta) = -w/nrows / (dist+eps) * delta/||delta||
    coef[i] = dn > 0.f ? -w_grad / nrows / (dist + eps) / dn : 0.f;
  }
}
// dx_i += J_norm^T ( coef_i * delta_i - sum_{j: nn(j)=i} coef_j * delta_j ),  delta_j = xn_j - xn_nn(j)
__global__ void koleo_bwd_kernel(const float* __restrict__ x, const float* __restrict__ xn,
                                 const float* __restrict__ nrm, const int* __restrict__ nn,
                                 const float* __restrict__ coef, float* __restrict__ dx, int B, int D, float eps) {
  extern __shared__ float gsm[];  // [D] gradient w.r.t. xn_i
  __shared__ float sh[32];
  const int i = blockIdx.x;
  const int ni = nn[i];
  const float ci = coef[i];
  for (int e = threadIdx.x; e < D; e += blockDim.x) gsm[e] = ci * (xn[(long)i * D + e] - xn[(long)ni * D + e]);
  __syncthreads();
  for (int j = 0; j < B; ++j) {
    if (nn[j] != i) continue;
    const float cj = coef[j];
    for (int e = threadIdx.x; e < D; e += blockDim.x) gsm[e] -= cj * (xn[(long)j * D + e] - xn[(long)i * D + e]);
  }
  __syncthreads();
  float dot = 0.f;
  for (int e = threadIdx.x; e < D; e += blockDim.x) dot += x[(long)i * D + e] * gsm[e];
  dot = block_sum(dot, sh);
  const float n = nrm[i];
  const float inv = 1.f / (n + eps);
  const float c2 = n > 0.f ? dot * inv * inv / n : 0.f;
  for (int e = threadIdx.x; e < D; e += blockDim.x) dx[(long)i * D + e] += gsm[e] * inv - x[(long)i * D + e] * c2;
}

// ---- Gram-anchoring loss (loss/gram_loss.py:13-50): elementwise stage between the similarity GEMMs and the backward
// GEMM.  Ss = Xs Xs^T and St = Xt Xt^T are fp32 [n, n] (wgmma GEMMs); per element
//   mode 1 (remove_neg):              s' = max(s, 0), t' = max(t, 0),            ds'/ds = [s > 0]
//   mode 2 (remove_only_teacher_neg): s' = (s < 0 && t < 0) ? 0 : s, t' = max(t, 0), ds'/ds = !(s < 0 && t < 0)
//   mode 0:                           s' = s, t' = t
// ws[CTA] = inv_count * sum over the CTA's elements of (s' - t')^2 (added to loss in CTA order by slab_combine);
// G = (s' - t') * ds'/ds  (bf16: the A operand of dX = (4 w / n^2) G Xs).
// block > 0 (gram.img_level: true, gram_loss.py:24-26): only the diagonal blocks of `block` x `block` tokens (one image each)
// count; everything else contributes nothing and gets G = 0 (the full similarity GEMM is kept: one launch, 128x the
// needed FLOPs at 196 tokens per image, still ~1 ms on the tensor cores).
__global__ void gram_diff_kernel(const float* __restrict__ Ss, const float* __restrict__ St, __nv_bfloat16* __restrict__ G,
                                 long n4, int mode, float inv_count, float* __restrict__ ws, int n, int block) {
  __shared__ float sh[32];
  float acc = 0.f;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
    const float4 s4 = reinterpret_cast<const float4*>(Ss)[i];
    const float4 t4 = reinterpret_cast<const float4*>(St)[i];
    const float sv[4] = {s4.x, s4.y, s4.z, s4.w}, tv[4] = {t4.x, t4.y, t4.z, t4.w};
    float g[4];
    const long e0 = i * 4;
    const int row_blk = block > 0 ? (int)(e0 / n) / block : 0;
    const int col0 = block > 0 ? (int)(e0 % n) : 0;               // n % 4 == 0: the four elements share a row
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float s = sv[j], t = tv[j], d = 1.f;
      if (block > 0 && (col0 + j) / block != row_blk) { g[j] = 0.f; continue; }
      if (mode == 1) { d = s > 0.f ? 1.f : 0.f; s = fmaxf(s, 0.f); t = fmaxf(t, 0.f); }
      else if (mode == 2) { if (s < 0.f && t < 0.f) { s = 0.f; d = 0.f; } t = fmaxf(t, 0.f); }
      const float e = s - t;
      acc = fmaf(e, e, acc);
      g[j] = e * d;
    }
    if (G) reinterpret_cast<uint2*>(G)[i] = make_uint2(pack_bf16(g[0], g[1]), pack_bf16(g[2], g[3]));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (threadIdx.x == 0 && ws) ws[blockIdx.x] = t * inv_count;
  }
}

}  // namespace d3

using namespace d3;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

int d3_absmax(const float* L, long long n, float* out /* pre-set to -inf */, void* stream) {
  if (n <= 0) return D3_OK;
  const long long n4 = (n + 3) / 4;
  const auto kernel = n % 4 == 0 && (uintptr_t)L % 16 == 0 ? absmax_kernel<true> : absmax_kernel<false>;
  kernel<<<(int)min((n4 + 1023) / 1024, (long long)sm_count() * 8), 256, 0, STREAM(stream)>>>(L, n4, out, n);
  D3_CHECK_LAUNCH();
  return D3_OK;
}
int d3_colmax(const float* L, float* cm /* [K] pre-set to -inf */, int R, int K, void* stream) {
  if (R <= 0) return D3_OK;
  const int cx = ((K + 3) / 4 + 127) / 128;
  const dim3 grid(cx, max(1, min(R / 8, max(1, sm_count() * 8 / cx))));
  const auto kernel = K % 4 == 0 && (uintptr_t)L % 16 == 0 ? colmax_kernel<true> : colmax_kernel<false>;
  kernel<<<grid, 128, 0, STREAM(stream)>>>(L, cm, R, K);
  D3_CHECK_LAUNCH();
  return D3_OK;
}
int d3_sinkhorn_colsum(const float* L, const float* mx, float temp, const float* a, float* s /* zeroed, += */, int R,
                       int K, void* stream) {
  if (R <= 0) return D3_OK;
  cudaStream_t st = STREAM(stream);
  const bool vec = K % 4 == 0 && ((uintptr_t)L | (uintptr_t)mx) % 16 == 0;
  // column CTAs of 128 threads x row slabs: aim at ~8 CTAs per SM, at most 16 slabs
  const int cx = ((vec ? K / 4 : K) + 127) / 128;
  const dim3 grid(cx, min(16, max(1, min(R / 8, max(1, sm_count() * 8 / cx)))));
  float* ws = slab_workspace((size_t)grid.y * K, st);
  if (!ws) return D3_ERR_CUDA;
  if (vec) sk_colsum_part_kernel<true><<<grid, 128, 0, st>>>(L, mx, 1.f / temp, a, ws, R, K);
  else sk_colsum_part_kernel<false><<<grid, 128, 0, st>>>(L, mx, 1.f / temp, a, ws, R, K);
  cudaError_t e = cudaPeekAtLastError();
  int rc = e == cudaSuccess ? D3_OK : set_error(D3_ERR_CUDA, cudaGetErrorString(e));
  if (!rc) { count_launch(); rc = slab_combine(ws, grid.y, K, 1, K, s, K, st); }
  slab_release(ws, st);
  return rc;
}
int d3_sinkhorn_rowsum(const float* L, const float* mx, float temp, const float* s, const float* btot, float* a, int R,
                       int K, void* stream) {
  if (R <= 0) return D3_OK;
  const auto kernel = K % 4 == 0 && ((uintptr_t)L | (uintptr_t)s | (uintptr_t)mx) % 16 == 0 ? sk_rowsum_kernel<true>
                                                                                             : sk_rowsum_kernel<false>;
  kernel<<<R, 256, 0, STREAM(stream)>>>(L, mx, 1.f / temp, s, btot, a, R, K);
  D3_CHECK_LAUNCH();
  return D3_OK;
}
int d3_sinkhorn_probs(const float* L, const float* mx, float temp, const float* s, const float* a, const float* btot,
                      float* Q, int R, int K, void* stream) {
  if (R <= 0) return D3_OK;
  long n = (long)R * K;
  sk_probs_kernel<<<(int)min((n + 255) / 256, (long)sm_count() * 16), 256, 0, STREAM(stream)>>>(L, mx, 1.f / temp, s, a,
                                                                                             btot, Q, R, K);
  D3_CHECK_LAUNCH();
  return D3_OK;
}
int d3_colsum_f32(const float* L, float* out /*[K] zeroed, +=*/, int R, int K, void* stream) {
  if (R <= 0) return D3_OK;
  cudaStream_t st = STREAM(stream);
  const dim3 grid((K + 255) / 256, max(1, min(R / 8, 64)));
  float* ws = slab_workspace((size_t)grid.y * K, st);
  if (!ws) return D3_ERR_CUDA;
  colsum_f32_kernel<<<grid, 256, 0, st>>>(L, ws, R, K);
  cudaError_t e = cudaPeekAtLastError();
  int rc = e == cudaSuccess ? D3_OK : set_error(D3_ERR_CUDA, cudaGetErrorString(e));
  if (!rc) { count_launch(); rc = slab_combine(ws, grid.y, K, 1, K, out, K, st); }
  slab_release(ws, st);
  return rc;
}
int d3_center_update(float* center, const float* colsum, const float* total_rows, float momentum, float temp,
                     float* s_out, int K, void* stream) {
  center_update_kernel<<<1, 1024, 0, STREAM(stream)>>>(center, colsum, total_rows, momentum, 1.f / temp, s_out, K);
  D3_CHECK_LAUNCH();
  return D3_OK;
}
}  // extern "C"

namespace d3 {
// metric[slot[i]] += row_loss[i] (slot == nullptr: every row to metric[0]; slots 0..7), rows added in a fixed order
__global__ void __launch_bounds__(256) metric_rows_kernel(const float* __restrict__ row_loss, const int* __restrict__ slot,
                                                          int n, float* __restrict__ metric) {
  __shared__ float sh[8][256];
  __shared__ int used;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  int seen = 0;
  if (threadIdx.x == 0) used = 0;
  for (int i = threadIdx.x; i < n; i += 256) {
    const int sl = slot ? slot[i] : 0;
#pragma unroll
    for (int k = 0; k < 8; ++k)
      if (sl == k) { acc[k] += row_loss[i]; seen |= 1 << k; }
  }
  __syncthreads();
  if (seen) atomicOr(&used, seen);
#pragma unroll
  for (int k = 0; k < 8; ++k) sh[k][threadIdx.x] = acc[k];
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w)
#pragma unroll
      for (int k = 0; k < 8; ++k) sh[k][threadIdx.x] += sh[k][threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x < 8 && (used >> threadIdx.x & 1)) metric[threadIdx.x] += sh[threadIdx.x][0];
}
static int add_row_losses(float* row_loss, const int* slot, int n, float* metric, cudaStream_t st) {
  metric_rows_kernel<<<1, 256, 0, st>>>(row_loss, slot, n, metric);
  cudaError_t e = cudaPeekAtLastError();
  slab_release(row_loss, st);
  if (e != cudaSuccess) return set_error(D3_ERR_CUDA, cudaGetErrorString(e));
  count_launch();
  return D3_OK;
}
}  // namespace d3

extern "C" {

int d3_ce_fwd_bwd(const float* S, float student_temp, const float* Lt, const float* mx, float teacher_temp,
                  const float* s_t, const float* a_t, const float* btot, const int* t0, const int* t1, const float* wm,
                  const float* wg, const int* slot, float* metric, void* dS, int Rs, int K, void* stream) {
  if (Rs <= 0) return D3_OK;
  cudaStream_t st = STREAM(stream);
  float* rows = slab_workspace(Rs, st);
  if (!rows) return D3_ERR_CUDA;
  const auto kernel =
      K % 4 == 0 && ((uintptr_t)S | (uintptr_t)Lt | (uintptr_t)s_t | (uintptr_t)dS | (uintptr_t)mx) % 16 == 0
          ? ce_fwd_bwd_kernel<true> : ce_fwd_bwd_kernel<false>;
  kernel<<<Rs, 512, 0, st>>>(S, 1.f / student_temp, Lt, mx, 1.f / teacher_temp, s_t, a_t, btot, t0, t1, wm, wg, slot,
                             rows, (__nv_bfloat16*)dS, K);
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) { slab_release(rows, st); return set_error(D3_ERR_CUDA, cudaGetErrorString(e)); }
  count_launch();
  return add_row_losses(rows, slot, Rs, metric, st);
}
int d3_koleo_fwd_bwd_rows(const float* x, float* xn_scratch, float* nrm_scratch, int* nn_scratch, float* coef_scratch,
                          float* metric, float* dx, int B, int D, int row0, int nrows, float eps, float w_metric,
                          float w_grad, void* stream) {
  if (B <= 1 || nrows <= 0) return D3_OK;
  if (row0 < 0 || row0 + nrows > B) return set_error(D3_ERR_ARG, "d3_koleo_fwd_bwd_rows: local row range outside [0, B)");
  cudaStream_t st = STREAM(stream);
  float* rows = slab_workspace(B, st);
  if (!rows) return D3_ERR_CUDA;
  koleo_norm_kernel<<<B, 256, 0, st>>>(x, xn_scratch, nrm_scratch, D, eps);
  koleo_nn_kernel<<<B, 256, 0, st>>>(xn_scratch, nn_scratch, coef_scratch, rows, B, D, eps, w_metric, w_grad, row0, nrows);
  koleo_bwd_kernel<<<B, 256, D * sizeof(float), st>>>(x, xn_scratch, nrm_scratch, nn_scratch, coef_scratch, dx, B, D, eps);
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) { slab_release(rows, st); return set_error(D3_ERR_CUDA, cudaGetErrorString(e)); }
  count_launch(3);
  return add_row_losses(rows, nullptr, B, metric, st);
}
int d3_gram_diff(const float* Ss, const float* St, void* G_bf16, long long n_elems, int mode, float inv_count, float* loss,
                 int n, int block, void* stream) {
  if (n_elems <= 0) return D3_OK;
  if (mode < 0 || mode > 2) return set_error(D3_ERR_ARG, "d3_gram_diff: mode 0 | 1 (remove_neg) | 2 (remove_only_teacher_neg)");
  if ((n_elems % 4) || (((uintptr_t)Ss | (uintptr_t)St) % 16) || ((uintptr_t)G_bf16 % 8))
    return set_error(D3_ERR_ARG, "d3_gram_diff: n_elems % 4 == 0 and 16-byte aligned similarity buffers");
  const long n4 = n_elems / 4;
  const int blocks = (int)std::min<long>((n4 + 255) / 256, (long)sm_count() * 8);
  if (block > 0 && (n <= 0 || (n % 4) || (long long)n * n != n_elems || (n % block)))
    return set_error(D3_ERR_ARG, "d3_gram_diff: block-diagonal form needs n % 4 == 0, n % block == 0 and n_elems == n * n");
  cudaStream_t st = STREAM(stream);
  float* ws = nullptr;
  if (loss && !(ws = slab_workspace(blocks, st))) return D3_ERR_CUDA;
  gram_diff_kernel<<<blocks, 256, 0, st>>>(Ss, St, (__nv_bfloat16*)G_bf16, n4, mode, inv_count, ws, n, block);
  cudaError_t e = cudaPeekAtLastError();
  int rc = e == cudaSuccess ? D3_OK : set_error(D3_ERR_CUDA, cudaGetErrorString(e));
  if (!rc) { count_launch(); rc = slab_combine(ws, blocks, 1, 1, 1, loss, 1, st); }
  slab_release(ws, st);
  return rc;
}

}  // extern "C"
