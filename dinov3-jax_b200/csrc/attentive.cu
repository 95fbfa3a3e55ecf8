// Attentive-probe video classification: the probe's single-query cross-attention pooling over a clip's frame tokens,
// folded so that the [N, 2D] keys and values of the tokens are never formed.
//
// With one query q (q = q0 Wq^T + bq) and H heads of width dh = D / H, head h's score of token n is
//   q_h . (Wk y_n)_h / sqrt(dh) = y_n . kt_h,   kt_h = Wk_h^T q_h / sqrt(dh)   (Wk_h: the head's dh rows of Wk),
// with y_n = g1 * uh_n + b1 the LN1 output and uh_n the normalised u_n = x_n + e_{t(n)}.  The part b1 . kt_h is the
// same for every token of a head, so the softmax ignores it: the kernels score s_{n,h} = (uh_n * g1) . kt_h.  The
// values fold out of the sum: sum_n p_{n,h} (Wv y_n + bv)_h = Wv_h ybar_h + bv_h with ybar_h = sum_n p_{n,h} y_n, so
// one pass over the tokens gives ybar [B, H, D] and the rest of the probe runs on [B, D] rows (d3_gemm_bf16).
//
// - d3_atp_query_fwd / d3_atp_query_bwd: q and kt from fp32 q0, Wq, bq, Wk, and their gradients.  They stay in fp32:
//   a score of magnitude 30 moves by 0.06 when the query is rounded to bf16, which changes a sharp softmax by 6 %.
// - d3_atp_pool_fwd: one CTA per (head group, frame, clip) streams the frame's P tokens once: LN1 statistics, H
//   scores per token and an online softmax with sum_n p uh_n per head; the per-frame (max, sum, sum p uh) are merged in
//   frame order.  Every CTA of a frame reads the same tokens, and the head groups of a frame are adjacent in the grid,
//   so the tokens come from HBM once.
// - d3_atp_pool_bwd: the same walk, given dybar = dL/dybar.  Per token, with c_h = ybar_h . dybar_h,
//     p = exp(s - lse), dp_h = y_n . dybar_h, ds_h = p (dp_h - c_h), dy_n = sum_h ds_h kt_h + p_h dybar_h,
//   and the LN1 backward du_n = rstd (g1 dy - mean(g1 dy) - uh mean(g1 dy uh)), whose two means are per-token sums of
//   per-head scalars (g1 . kt_h, g1 . dybar_h, b1 . dybar_h are per clip and head).  Column sums dkt = sum ds y,
//   dg1 = sum dy uh, db1 = sum dy and de_t = sum_{n in t} du go to slabs added in order by slab_combine.
// - d3_atp_gelu_erf_bwd: the exact GELU's derivative for the probe MLP's backward.
//
// Deterministic: no float atomics, every sum in a fixed order.  LayerNorm eps 1e-6.  D <= 1536, a multiple of 8.
#include "ptx.cuh"
#include "d3_internal.h"

#include <math.h>
#include <stdio.h>

#include <algorithm>

namespace d3 {

constexpr int ATP_THREADS = 256;
constexpr int ATP_WARPS = ATP_THREADS / 32;     // one token per warp per tile
constexpr int ATP_MAX_D = 1536;
constexpr float ATP_EPS = 1e-6f;

// Columns per thread CPT = ceil(D / 256): a warp holds a token as CPT 8-element vectors per lane, and a thread of the
// column phase owns CPT columns.  A CTA takes HG heads with HG * CPT <= 32 accumulators per thread (HG <= 4 above
// D = 1024, where the backward would spill otherwise).
template <int CPT>
__host__ __device__ constexpr int atp_hg_max() { return CPT <= 4 ? 8 : 4; }

// Token n of the walk into registers: uh = LayerNorm(x + e_t) without scale or bias (two-pass variance), the lane's
// vectors v = lane + 32 k, columns 8 v .. 8 v + 7.  Returns rstd.
template <int CPT>
__device__ __forceinline__ float atp_load_token(const __nv_bfloat16* __restrict__ xr, const float* __restrict__ et,
                                                int D, int lane, float (&uh)[CPT][8]) {
  const int nv = D / 8;
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < CPT; ++k) {
    const int v = lane + 32 * k;
    if (v < nv) {
      const uint4 raw = *reinterpret_cast<const uint4*>(xr + 8 * v);
      const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = unpack_bf16(w[i]);
        uh[k][2 * i] = f.x + et[8 * v + 2 * i];
        uh[k][2 * i + 1] = f.y + et[8 * v + 2 * i + 1];
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) s += uh[k][i];
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) uh[k][i] = 0.f;
    }
  }
  const float mean = warp_sum(s) / (float)D;
  float q = 0.f;
#pragma unroll
  for (int k = 0; k < CPT; ++k) {
    if (lane + 32 * k < nv) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        uh[k][i] -= mean;
        q += uh[k][i] * uh[k][i];
      }
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / (float)D + ATP_EPS);
#pragma unroll
  for (int k = 0; k < CPT; ++k)
#pragma unroll
    for (int i = 0; i < 8; ++i) uh[k][i] *= rstd;
  return rstd;
}

// uh <- uh * g1 in place (the scores' and dp's left operand), g1 read as float4 pairs
template <int CPT>
__device__ __forceinline__ void atp_scale(float (&uh)[CPT][8], const float* __restrict__ g1, int D, int lane) {
#pragma unroll
  for (int k = 0; k < CPT; ++k) {
    const int v = lane + 32 * k;
    if (v < D / 8) {
      const float4 a = *reinterpret_cast<const float4*>(g1 + 8 * v), b = *reinterpret_cast<const float4*>(g1 + 8 * v + 4);
      uh[k][0] *= a.x; uh[k][1] *= a.y; uh[k][2] *= a.z; uh[k][3] *= a.w;
      uh[k][4] *= b.x; uh[k][5] *= b.y; uh[k][6] *= b.z; uh[k][7] *= b.w;
    }
  }
}

// sum_c ug_c w_c over the warp's token (w in shared memory, read as float4 pairs); every lane gets the result (fixed
// order: lane partials in column order, then the butterfly)
template <int CPT>
__device__ __forceinline__ float atp_dot(const float (&ug)[CPT][8], const float* __restrict__ w, int D, int lane) {
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < CPT; ++k) {
    const int v = lane + 32 * k;
    if (v < D / 8) {
      const float4 a = *reinterpret_cast<const float4*>(w + 8 * v), b = *reinterpret_cast<const float4*>(w + 8 * v + 4);
      s += ug[k][0] * a.x; s += ug[k][1] * a.y; s += ug[k][2] * a.z; s += ug[k][3] * a.w;
      s += ug[k][4] * b.x; s += ug[k][5] * b.y; s += ug[k][6] * b.z; s += ug[k][7] * b.w;
    }
  }
  return warp_sum(s);
}

template <int CPT>
__device__ __forceinline__ void atp_store_row(const float (&uh)[CPT][8], float* __restrict__ row, int D, int lane) {
#pragma unroll
  for (int k = 0; k < CPT; ++k) {
    const int v = lane + 32 * k;
    if (v < D / 8) {
      *reinterpret_cast<float4*>(row + 8 * v) = make_float4(uh[k][0], uh[k][1], uh[k][2], uh[k][3]);
      *reinterpret_cast<float4*>(row + 8 * v + 4) = make_float4(uh[k][4], uh[k][5], uh[k][6], uh[k][7]);
    }
  }
}

// ------------------------------------------------------------------------------------------------------- query
// q[j] = bq[j] + sum_i Wq[j, i] q0[i]: one warp per row
__global__ void atp_q_kernel(const float* __restrict__ q0, const float* __restrict__ Wq, const float* __restrict__ bq,
                             int D, float* __restrict__ q) {
  const int j = blockIdx.x * ATP_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (j >= D) return;
  const float* w = Wq + (size_t)j * D;
  float s = 0.f;
  for (int i = lane; i < D; i += 32) s += w[i] * q0[i];
  s = warp_sum(s);
  if (lane == 0) q[j] = bq[j] + s;
}

// kt[h, c] = scale * sum_{j in head h} Wk[j, c] q[j]
__global__ void atp_kt_kernel(const float* __restrict__ q, const float* __restrict__ Wk, int D, int dh, float scale,
                              float* __restrict__ kt) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x, h = blockIdx.y;
  if (c >= D) return;
  float s = 0.f;
  for (int j = h * dh; j < (h + 1) * dh; ++j) s += Wk[(size_t)j * D + c] * q[j];
  kt[(size_t)h * D + c] = s * scale;
}

// Row j of Wk (head h = j / dh): dq[j] = scale * sum_c Wk[j, c] dkt[h, c] and dWk[j, c] = scale * q[j] dkt[h, c].
// dbq = dq.
__global__ void atp_dq_kernel(const float* __restrict__ Wk, const float* __restrict__ q, const float* __restrict__ dkt,
                              int D, int dh, float scale, float* __restrict__ dWk, float* __restrict__ dq) {
  const int j = blockIdx.x * ATP_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (j >= D) return;
  const float* w = Wk + (size_t)j * D;
  const float* g = dkt + (size_t)(j / dh) * D;
  const float qs = q[j] * scale;
  float s = 0.f;
  for (int c = lane; c < D; c += 32) {
    s += w[c] * g[c];
    dWk[(size_t)j * D + c] = qs * g[c];
  }
  s = warp_sum(s);
  if (lane == 0) dq[j] = s * scale;
}

// Column i of Wq: dWq[j, i] = dq[j] q0[i] for every j, dq0[i] += sum_j Wq[j, i] dq[j] (j in order)
__global__ void atp_dq0_kernel(const float* __restrict__ Wq, const float* __restrict__ q0, const float* __restrict__ dq,
                               int D, float* __restrict__ dWq, float* __restrict__ dq0) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D) return;
  const float x = q0[i];
  float s = 0.f;
  for (int j = 0; j < D; ++j) {
    const float g = dq[j];
    s += Wq[(size_t)j * D + i] * g;
    dWq[(size_t)j * D + i] = g * x;
  }
  dq0[i] += s;
}

// ----------------------------------------------------------------------------------------------- pooling forward
// Shared memory (floats): kt [HG, D] | g1 [D] | e_t [D] | uh tile [8, D] | p [8, HGM] | corr [HGM]
template <int CPT>
__global__ void __launch_bounds__(ATP_THREADS, 2)
atp_fwd_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ e, const float* __restrict__ g1,
               const float* __restrict__ kt, int T, int P, int D, int H, int HG, float* __restrict__ part_ml,
               float* __restrict__ part_acc) {
  constexpr int HGM = atp_hg_max<CPT>();
  extern __shared__ __align__(16) float smem[];
  float* kts = smem;
  float* gs = kts + HG * D;
  float* es = gs + D;
  float* U = es + D;
  float* pw = U + ATP_WARPS * D;
  float* corr = pw + ATP_WARPS * HGM;
  const int h0 = blockIdx.x * HG, t = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  for (int i = tid; i < HG * D; i += ATP_THREADS) kts[i] = kt[(size_t)h0 * D + i];
  for (int c = tid; c < D; c += ATP_THREADS) {
    gs[c] = g1[c];
    es[c] = e[(size_t)t * D + c];
  }
  __syncthreads();
  const __nv_bfloat16* xf = x + ((size_t)b * T + t) * (size_t)P * D;
  float acc[HGM][CPT];
#pragma unroll
  for (int j = 0; j < HGM; ++j)
#pragma unroll
    for (int k = 0; k < CPT; ++k) acc[j][k] = 0.f;
  float m = -INFINITY, l = 0.f;                       // head tid's running (max, sum), threads tid < HG
  for (int n0 = 0; n0 < P; n0 += ATP_WARPS) {
    const int nt = min(ATP_WARPS, P - n0);
    if (w < nt) {
      float uh[CPT][8];
      atp_load_token<CPT>(xf + (size_t)(n0 + w) * D, es, D, lane, uh);
      atp_store_row<CPT>(uh, U + w * D, D, lane);
      atp_scale<CPT>(uh, gs, D, lane);
#pragma unroll
      for (int j = 0; j < HGM; ++j) {
        if (j < HG) {
          const float s = atp_dot<CPT>(uh, kts + j * D, D, lane);
          if (lane == 0) pw[w * HGM + j] = s;
        }
      }
    }
    __syncthreads();
    if (tid < HG) {
      float mx = m;
      for (int n = 0; n < nt; ++n) mx = fmaxf(mx, pw[n * HGM + tid]);
      const float cr = expf(m - mx);
      float sum = 0.f;
      for (int n = 0; n < nt; ++n) {
        const float p = expf(pw[n * HGM + tid] - mx);
        pw[n * HGM + tid] = p;
        sum += p;
      }
      l = l * cr + sum;
      m = mx;
      corr[tid] = cr;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < CPT; ++k) {
      const int c = tid + ATP_THREADS * k;
      if (c < D) {
#pragma unroll
        for (int j = 0; j < HGM; ++j) {
          if (j < HG) {
            float a = acc[j][k] * corr[j];
            for (int n = 0; n < nt; ++n) a += pw[n * HGM + j] * U[n * D + c];
            acc[j][k] = a;
          }
        }
      }
    }
    __syncthreads();
  }
  const size_t slot = ((size_t)b * T + t) * H + h0;
#pragma unroll
  for (int k = 0; k < CPT; ++k) {
    const int c = tid + ATP_THREADS * k;
    if (c < D) {
#pragma unroll
      for (int j = 0; j < HGM; ++j)
        if (j < HG) part_acc[(slot + j) * D + c] = acc[j][k];
    }
  }
  if (tid < HG) {
    part_ml[2 * (slot + tid)] = m;
    part_ml[2 * (slot + tid) + 1] = l;
  }
}

// One CTA per (head, clip): the frames' (max, sum, sum p uh) in frame order -> ybar = g1 * (sum p uh) / L + b1 and
// lse = M + log L.
__global__ void atp_merge_kernel(const float* __restrict__ part_ml, const float* __restrict__ part_acc,
                                 const float* __restrict__ g1, const float* __restrict__ b1, int T, int H, int D,
                                 float* __restrict__ ybar, float* __restrict__ lse) {
  const int h = blockIdx.x, b = blockIdx.y;
  const float* ml = part_ml + 2 * ((size_t)b * T * H + h);
  float M = -INFINITY;
  for (int t = 0; t < T; ++t) M = fmaxf(M, ml[2 * (size_t)t * H]);
  float L = 0.f;
  for (int t = 0; t < T; ++t) L += ml[2 * (size_t)t * H + 1] * expf(ml[2 * (size_t)t * H] - M);
  const float inv = 1.f / L;
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    float s = 0.f;
    for (int t = 0; t < T; ++t)
      s += part_acc[(((size_t)b * T + t) * H + h) * D + c] * expf(ml[2 * (size_t)t * H] - M);
    ybar[((size_t)b * H + h) * D + c] = g1[c] * (s * inv) + b1[c];
  }
  if (threadIdx.x == 0) lse[(size_t)b * H + h] = M + logf(L);
}

// ---------------------------------------------------------------------------------------------- pooling backward
// Shared memory (floats): kt [HG, D] | dybar [HG, D] | g1 [D] | b1 [D] | e_t [D] | uh tile [8, D] |
// p, ds [8, HGM] each | per token (mean(g1 dy), mean(g1 dy uh), rstd) [8] each | per head (c, g1.kt, g1.dybar,
// b1.dybar, lse) [HGM] each
template <int CPT>
__global__ void __launch_bounds__(ATP_THREADS, 2)
atp_bwd_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ e, const float* __restrict__ g1,
               const float* __restrict__ b1, const float* __restrict__ kt, const float* __restrict__ lse,
               const float* __restrict__ ybar, const float* __restrict__ dybar, int T, int P, int D, int H, int HG,
               float* __restrict__ ws_dkt, float* __restrict__ ws_dgb, float* __restrict__ ws_de) {
  constexpr int HGM = atp_hg_max<CPT>();
  extern __shared__ __align__(16) float smem[];
  float* kts = smem;
  float* dys = kts + HG * D;
  float* gs = dys + HG * D;
  float* bs = gs + D;
  float* es = bs + D;
  float* U = es + D;
  float* pw = U + ATP_WARPS * D;
  float* dsw = pw + ATP_WARPS * HGM;
  float* rowA = dsw + ATP_WARPS * HGM;
  float* rowB = rowA + ATP_WARPS;
  float* rowR = rowB + ATP_WARPS;
  float* hc = rowR + ATP_WARPS;
  float* hgk = hc + HGM;
  float* hgd = hgk + HGM;
  float* hbd = hgd + HGM;
  float* hl = hbd + HGM;
  const int g = blockIdx.x, G = gridDim.x, h0 = g * HG, t = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  for (int i = tid; i < HG * D; i += ATP_THREADS) {
    kts[i] = kt[(size_t)h0 * D + i];
    dys[i] = dybar[((size_t)b * H + h0) * D + i];
  }
  for (int c = tid; c < D; c += ATP_THREADS) {
    gs[c] = g1[c];
    bs[c] = b1[c];
    es[c] = e[(size_t)t * D + c];
  }
  __syncthreads();
  for (int j = w; j < HG; j += ATP_WARPS) {             // per head: one warp, columns in lane order
    const float* yb = ybar + ((size_t)b * H + h0 + j) * D;
    float c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f;
    for (int c = lane; c < D; c += 32) {
      const float d = dys[j * D + c];
      c0 += yb[c] * d;
      c1 += gs[c] * kts[j * D + c];
      c2 += gs[c] * d;
      c3 += bs[c] * d;
    }
    c0 = warp_sum(c0); c1 = warp_sum(c1); c2 = warp_sum(c2); c3 = warp_sum(c3);
    if (lane == 0) {
      hc[j] = c0; hgk[j] = c1; hgd[j] = c2; hbd[j] = c3;
      hl[j] = lse[(size_t)b * H + h0 + j];
    }
  }
  __syncthreads();
  const __nv_bfloat16* xf = x + ((size_t)b * T + t) * (size_t)P * D;
  const float invD = 1.f / (float)D;
  float dk[HGM][CPT], dg[CPT], db[CPT], de[CPT];
#pragma unroll
  for (int k = 0; k < CPT; ++k) {
    dg[k] = db[k] = de[k] = 0.f;
#pragma unroll
    for (int j = 0; j < HGM; ++j) dk[j][k] = 0.f;
  }
  for (int n0 = 0; n0 < P; n0 += ATP_WARPS) {
    const int nt = min(ATP_WARPS, P - n0);
    if (w < nt) {
      float uh[CPT][8];
      const float rstd = atp_load_token<CPT>(xf + (size_t)(n0 + w) * D, es, D, lane, uh);
      atp_store_row<CPT>(uh, U + w * D, D, lane);
      atp_scale<CPT>(uh, gs, D, lane);
      float A = 0.f, Bs = 0.f;
#pragma unroll
      for (int j = 0; j < HGM; ++j) {
        if (j < HG) {
          const float s = atp_dot<CPT>(uh, kts + j * D, D, lane);
          const float dp = atp_dot<CPT>(uh, dys + j * D, D, lane) + hbd[j];
          const float p = expf(s - hl[j]);
          const float ds = p * (dp - hc[j]);
          A += ds * hgk[j] + p * hgd[j];
          Bs += ds * s + p * (dp - hbd[j]);
          if (lane == 0) {
            pw[w * HGM + j] = p;
            dsw[w * HGM + j] = ds;
          }
        }
      }
      if (lane == 0) {
        rowA[w] = A * invD;
        rowB[w] = Bs * invD;
        rowR[w] = rstd;
      }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < CPT; ++k) {
      const int c = tid + ATP_THREADS * k;
      if (c < D) {
        const float gc = gs[c], bc = bs[c];
        for (int n = 0; n < nt; ++n) {
          float dy = 0.f;
#pragma unroll
          for (int j = 0; j < HGM; ++j)
            if (j < HG) dy += dsw[n * HGM + j] * kts[j * D + c] + pw[n * HGM + j] * dys[j * D + c];
          const float u = U[n * D + c];
          dg[k] += dy * u;
          db[k] += dy;
          de[k] += rowR[n] * (gc * dy - rowA[n] - u * rowB[n]);
          const float yv = gc * u + bc;
#pragma unroll
          for (int j = 0; j < HGM; ++j)
            if (j < HG) dk[j][k] += dsw[n * HGM + j] * yv;
        }
      }
    }
    __syncthreads();
  }
  // slabs: dkt [(b, t)][H, D]; dg1 / db1 [(b, t, g)][2, D]; de [(b, g)][T, D]
  const size_t s_bt = (size_t)b * T + t;
  const size_t s_btg = s_bt * G + g;
  const size_t s_bg = (size_t)b * G + g;
#pragma unroll
  for (int k = 0; k < CPT; ++k) {
    const int c = tid + ATP_THREADS * k;
    if (c < D) {
#pragma unroll
      for (int j = 0; j < HGM; ++j)
        if (j < HG) ws_dkt[(s_bt * H + h0 + j) * D + c] = dk[j][k];
      ws_dgb[s_btg * 2 * D + c] = dg[k];
      ws_dgb[s_btg * 2 * D + D + c] = db[k];
      ws_de[(s_bg * T + t) * D + c] = de[k];
    }
  }
}

// out[r, c] = bf16(dh[r, c] * GELU'(pre[r, c])), GELU'(u) = Phi(u) + u phi(u)
__global__ void atp_gelu_erf_bwd_kernel(const float* __restrict__ dh, int ld_dh, const __nv_bfloat16* __restrict__ pre,
                                        int ld_pre, int rows, int cols, __nv_bfloat16* __restrict__ out, int ld_out) {
  const long long n = (long long)rows * cols;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols, c = i - r * cols;
    const float u = __bfloat162float(pre[r * ld_pre + c]);
    const float d = 0.5f * (1.f + erff(u * 0.70710678118654752f)) + u * 0.3989422804014327f * expf(-0.5f * u * u);
    out[r * ld_out + c] = __float2bfloat16(dh[r * ld_dh + c] * d);
  }
}

// The head group of a D-wide backbone with H heads: the most heads HG <= hg_max(CPT) that divide H.
template <int CPT>
int atp_groups(int H) {
  int hg = atp_hg_max<CPT>();
  while (H % hg) --hg;
  return hg;
}

template <int CPT>
size_t atp_fwd_smem(int D, int HG) {
  return sizeof(float) * ((size_t)HG * D + 2 * D + ATP_WARPS * D + ATP_WARPS * atp_hg_max<CPT>() + atp_hg_max<CPT>());
}

template <int CPT>
size_t atp_bwd_smem(int D, int HG) {
  constexpr int HGM = atp_hg_max<CPT>();
  return sizeof(float) * ((size_t)2 * HG * D + 3 * D + ATP_WARPS * D + 2 * ATP_WARPS * HGM + 3 * ATP_WARPS + 5 * HGM);
}

template <int CPT>
int atp_fwd_launch(const void* x, const float* e, const float* g1, const float* b1, const float* kt, int B, int T,
                   int P, int D, int H, float* ybar, float* lse, cudaStream_t st) {
  const int HG = atp_groups<CPT>(H);
  const size_t smem = atp_fwd_smem<CPT>(D, HG);
  cudaError_t err = cudaFuncSetAttribute(atp_fwd_kernel<CPT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (err != cudaSuccess) return set_error(D3_ERR_CUDA, cudaGetErrorString(err));
  const size_t slots = (size_t)B * T * H;
  float* ws = nullptr;
  err = cudaMallocAsync(reinterpret_cast<void**>(&ws), sizeof(float) * slots * (D + 2), st);
  if (err != cudaSuccess) return set_error(D3_ERR_CUDA, cudaGetErrorString(err));
  float* part_ml = ws;
  float* part_acc = ws + 2 * slots;
  atp_fwd_kernel<CPT><<<dim3(H / HG, T, B), ATP_THREADS, smem, st>>>(
      (const __nv_bfloat16*)x, e, g1, kt, T, P, D, H, HG, part_ml, part_acc);
  err = cudaPeekAtLastError();
  if (err == cudaSuccess) {
    count_launch();
    atp_merge_kernel<<<dim3(H, B), ATP_THREADS, 0, st>>>(part_ml, part_acc, g1, b1, T, H, D, ybar, lse);
    err = cudaPeekAtLastError();
  }
  cudaFreeAsync(ws, st);
  if (err != cudaSuccess) return set_error(D3_ERR_CUDA, cudaGetErrorString(err));
  count_launch();
  return D3_OK;
}

template <int CPT>
int atp_bwd_launch(const void* x, const float* e, const float* g1, const float* b1, const float* kt, const float* lse,
                   const float* ybar, const float* dybar, int B, int T, int P, int D, int H, float* dkt, float* dg1,
                   float* db1, float* de, cudaStream_t st) {
  const int HG = atp_groups<CPT>(H), G = H / HG;
  const size_t smem = atp_bwd_smem<CPT>(D, HG);
  cudaError_t err = cudaFuncSetAttribute(atp_bwd_kernel<CPT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (err != cudaSuccess) return set_error(D3_ERR_CUDA, cudaGetErrorString(err));
  const size_t n_dkt = (size_t)B * T * H * D, n_dgb = (size_t)B * T * G * 2 * D, n_de = (size_t)B * G * T * D;
  float* ws = slab_workspace(n_dkt + n_dgb + n_de, st);
  if (!ws) return D3_ERR_CUDA;
  float* ws_dkt = ws;
  float* ws_dgb = ws + n_dkt;
  float* ws_de = ws_dgb + n_dgb;
  atp_bwd_kernel<CPT><<<dim3(G, T, B), ATP_THREADS, smem, st>>>((const __nv_bfloat16*)x, e, g1, b1, kt, lse, ybar,
                                                                 dybar, T, P, D, H, HG, ws_dkt, ws_dgb, ws_de);
  err = cudaPeekAtLastError();
  if (err == cudaSuccess) err = cudaMemsetAsync(dkt, 0, sizeof(float) * H * D, st);
  if (err == cudaSuccess) err = cudaMemsetAsync(de, 0, sizeof(float) * T * D, st);
  if (err == cudaSuccess) err = cudaMemsetAsync(dg1, 0, sizeof(float) * D, st);
  if (err == cudaSuccess) err = cudaMemsetAsync(db1, 0, sizeof(float) * D, st);
  int rc = err == cudaSuccess ? D3_OK : set_error(D3_ERR_CUDA, cudaGetErrorString(err));
  if (!rc) { count_launch(); rc = slab_combine(ws_dkt, B * T, (long long)H * D, 1, H * D, dkt, H * D, st); }
  if (!rc) rc = slab_combine(ws_dgb, B * T * G, 2LL * D, 1, D, dg1, D, st);
  if (!rc) rc = slab_combine(ws_dgb + D, B * T * G, 2LL * D, 1, D, db1, D, st);
  if (!rc) rc = slab_combine(ws_de, B * G, (long long)T * D, 1, T * D, de, T * D, st);
  slab_release(ws, st);
  return rc;
}

// host-side checks shared by the two pooling entry points
int atp_check(const char* fn, const void* x, int B, int T, int P, int D, int H) {
  char buf[200];
  if (B < 1 || T < 1 || P < 1 || H < 1 || D < 8 || D % 8 || D > ATP_MAX_D || D % H) {
    snprintf(buf, sizeof(buf), "%s: need B, T, P, H >= 1 and D a multiple of 8 in [8, %d] divisible by H (got B %d, T %d, "
             "P %d, D %d, H %d)", fn, ATP_MAX_D, B, T, P, D, H);
    return set_error(D3_ERR_ARG, buf);
  }
  if ((uintptr_t)x % 16) {
    snprintf(buf, sizeof(buf), "%s: the tokens must be 16-byte aligned", fn);
    return set_error(D3_ERR_ARG, buf);
  }
  return D3_OK;
}

}  // namespace d3

using namespace d3;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

int d3_atp_query_fwd(const float* q0, const float* Wq, const float* bq, const float* Wk, int D, int H, float* q,
                     float* kt, void* stream) {
  if (!q0 || !Wq || !bq || !Wk || !q || !kt || D < 1 || H < 1 || D % H)
    return set_error(D3_ERR_ARG, "d3_atp_query_fwd: need every buffer, D >= 1 and H >= 1 dividing D");
  cudaStream_t st = STREAM(stream);
  const int dh = D / H;
  atp_q_kernel<<<(D + ATP_WARPS - 1) / ATP_WARPS, ATP_THREADS, 0, st>>>(q0, Wq, bq, D, q);
  D3_CHECK_LAUNCH();
  atp_kt_kernel<<<dim3((D + 255) / 256, H), 256, 0, st>>>(q, Wk, D, dh, 1.f / sqrtf((float)dh), kt);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_atp_query_bwd(const float* q0, const float* Wq, const float* Wk, const float* q, const float* dkt, int D, int H,
                     float* dWq, float* dbq, float* dWk, float* dq0, void* stream) {
  if (!q0 || !Wq || !Wk || !q || !dkt || !dWq || !dbq || !dWk || !dq0 || D < 1 || H < 1 || D % H)
    return set_error(D3_ERR_ARG, "d3_atp_query_bwd: need every buffer, D >= 1 and H >= 1 dividing D");
  cudaStream_t st = STREAM(stream);
  const int dh = D / H;
  atp_dq_kernel<<<(D + ATP_WARPS - 1) / ATP_WARPS, ATP_THREADS, 0, st>>>(Wk, q, dkt, D, dh, 1.f / sqrtf((float)dh),
                                                                        dWk, dbq);
  D3_CHECK_LAUNCH();
  atp_dq0_kernel<<<(D + 255) / 256, 256, 0, st>>>(Wq, q0, dbq, D, dWq, dq0);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_atp_pool_fwd(const void* x, const float* e, const float* g1, const float* b1, const float* kt, int B, int T,
                    int P, int D, int H, float* ybar, float* lse, void* stream) {
  if (int rc = atp_check("d3_atp_pool_fwd", x, B, T, P, D, H)) return rc;
  if (!e || !g1 || !b1 || !kt || !ybar || !lse) return set_error(D3_ERR_ARG, "d3_atp_pool_fwd: null buffer");
  cudaStream_t st = STREAM(stream);
  switch ((D + 255) / 256) {
    case 1: return atp_fwd_launch<1>(x, e, g1, b1, kt, B, T, P, D, H, ybar, lse, st);
    case 2: return atp_fwd_launch<2>(x, e, g1, b1, kt, B, T, P, D, H, ybar, lse, st);
    case 3: return atp_fwd_launch<3>(x, e, g1, b1, kt, B, T, P, D, H, ybar, lse, st);
    case 4: return atp_fwd_launch<4>(x, e, g1, b1, kt, B, T, P, D, H, ybar, lse, st);
    case 5: return atp_fwd_launch<5>(x, e, g1, b1, kt, B, T, P, D, H, ybar, lse, st);
    default: return atp_fwd_launch<6>(x, e, g1, b1, kt, B, T, P, D, H, ybar, lse, st);
  }
}

int d3_atp_pool_bwd(const void* x, const float* e, const float* g1, const float* b1, const float* kt, const float* lse,
                    const float* ybar, const float* dybar, int B, int T, int P, int D, int H, float* dkt, float* dg1,
                    float* db1, float* de, void* stream) {
  if (int rc = atp_check("d3_atp_pool_bwd", x, B, T, P, D, H)) return rc;
  if (!e || !g1 || !b1 || !kt || !lse || !ybar || !dybar || !dkt || !dg1 || !db1 || !de)
    return set_error(D3_ERR_ARG, "d3_atp_pool_bwd: null buffer");
  cudaStream_t st = STREAM(stream);
  switch ((D + 255) / 256) {
    case 1: return atp_bwd_launch<1>(x, e, g1, b1, kt, lse, ybar, dybar, B, T, P, D, H, dkt, dg1, db1, de, st);
    case 2: return atp_bwd_launch<2>(x, e, g1, b1, kt, lse, ybar, dybar, B, T, P, D, H, dkt, dg1, db1, de, st);
    case 3: return atp_bwd_launch<3>(x, e, g1, b1, kt, lse, ybar, dybar, B, T, P, D, H, dkt, dg1, db1, de, st);
    case 4: return atp_bwd_launch<4>(x, e, g1, b1, kt, lse, ybar, dybar, B, T, P, D, H, dkt, dg1, db1, de, st);
    case 5: return atp_bwd_launch<5>(x, e, g1, b1, kt, lse, ybar, dybar, B, T, P, D, H, dkt, dg1, db1, de, st);
    default: return atp_bwd_launch<6>(x, e, g1, b1, kt, lse, ybar, dybar, B, T, P, D, H, dkt, dg1, db1, de, st);
  }
}

int d3_atp_gelu_erf_bwd(const float* dh, int ld_dh, const void* pre, int ld_pre, int rows, int cols, void* out,
                        int ld_out, void* stream) {
  if (rows <= 0 || cols <= 0) return D3_OK;
  if (!dh || !pre || !out || ld_dh < cols || ld_pre < cols || ld_out < cols)
    return set_error(D3_ERR_ARG, "d3_atp_gelu_erf_bwd: need every buffer and ld_dh, ld_pre, ld_out >= cols");
  const long long n = (long long)rows * cols;
  const int blocks = (int)std::min<long long>((n + 255) / 256, (long long)sm_count() * 8);
  atp_gelu_erf_bwd_kernel<<<blocks, 256, 0, STREAM(stream)>>>(dh, ld_dh, (const __nv_bfloat16*)pre, ld_pre, rows, cols,
                                                               (__nv_bfloat16*)out, ld_out);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

}  // extern "C"
