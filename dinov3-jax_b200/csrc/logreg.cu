// Multinomial logistic regression on frozen features, a whole grid of regularisation strengths at once (the
// logistic-regression evaluation, dinov3_jax/eval/logreg.py).  Problem g minimises the scaled objective
//   F_g(W, b) = (1/N) sum_i CE(W x_i + b, y_i) + ||W||^2 / (2 c_g N)
// over W [Cp, K] and b [Cp] (Cp = classes padded to a multiple of 8; the padding rows stay 0).  Its parameters are one
// fp32 vector theta_g = [W_g row-major | b_g] of P = Cp K + Cp floats; every [G, P] buffer is indexed by the problem's
// slot g, and a launch covers the Ga problems of a device list act[0 .. Ga) (the active set, compacted by the host).
//
// One evaluation of F and grad F for the active problems:
//   d3_logreg_weights   W of each active problem as bf16 rows [Wh | Wl | Wh] (hi + lo split of fp32) and its bias;
//   per row chunk:      logits = [Xh | Xh | Xl] . [Wh | Wl | Wh]^T (d3_gemm_bf16, fp32 out), the fp32 product to
//                       about 2^-17;
//                       d3_logreg_xent: log-sum-exp, row loss and the residual (softmax - onehot) / N split hi + lo;
//                       grad W += [Rh; Rh; Rl]^T . [Xh; Xl; Xh] (d3_gemm_bf16), grad b += colsums of Rh and Rl;
//   d3_logreg_finish    adds W / (c N) to the gradient and ||W||^2 / (2 c N) to the loss, and reduces per problem the
//                       objective, grad . d, max |grad| and ||grad||^2 for the host's line search.
// The L-BFGS vector work is here too: the trial point theta + alpha_g d_g, the two-loop recursion over each problem's
// history, and the history update.  The host reads one G-sized vector per evaluation and nothing per element.
//
// Deterministic: no float atomics; every reduction runs in a fixed order over fixed slabs (LR_SLABS per problem).
#include "ptx.cuh"
#include "d3_internal.h"

#include <math.h>

namespace d3 {

constexpr int LR_THREADS = 256;
constexpr int LR_SLABS = 96;           // CTAs per problem of every [G, P] reduction: the partials' order is fixed
constexpr int LR_MAX_HISTORY = 64;
constexpr int LR_MAX_Q = 4;

__device__ __forceinline__ void split_bf16(float v, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(v);
  lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}

// Block-wide reduction of Q doubles per thread (sum, or max where bit q of max_mask is set), in a fixed order: a
// butterfly within each warp, then the warps in order.  The result is valid in thread 0.
template <int Q>
__device__ __forceinline__ void block_reduce(double (&v)[Q], unsigned max_mask) {
  __shared__ double red[LR_THREADS / 32][LR_MAX_Q];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < Q; ++q)
    for (int o = 16; o > 0; o >>= 1) {
      const double w = __shfl_xor_sync(0xffffffffu, v[q], o);
      v[q] = (max_mask >> q & 1) ? fmax(v[q], w) : v[q] + w;
    }
  __syncthreads();                                        // red may still be read by an earlier call
  if (lane == 0)
#pragma unroll
    for (int q = 0; q < Q; ++q) red[wid][q] = v[q];
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < LR_THREADS / 32; ++w)
#pragma unroll
      for (int q = 0; q < Q; ++q) v[q] = (max_mask >> q & 1) ? fmax(v[q], red[w][q]) : v[q] + red[w][q];
}

// slab s of P elements: [s * seg, min(P, (s + 1) * seg))
__device__ __forceinline__ void slab_range(long long P, long long& e0, long long& e1) {
  const long long seg = (P + LR_SLABS - 1) / LR_SLABS;
  e0 = blockIdx.x * seg;
  e1 = min(P, e0 + seg);
}

// ------------------------------------------------------------------------------------------------- operands
// Row r of x (fp32 [n, ldx]) into xa [rows, 3K] = [h | h | l] and, when xg is given, into the gradient operand of its
// chunk c = r / chunk, i = r % chunk: xg rows c * 3 chunk + i (h), + chunk + i (l), + 2 chunk + i (h).  Rows in
// [n, rows) are written as zeros.
__global__ void lr_split_x_kernel(const float* __restrict__ x, int ldx, int n, int rows, int K, int chunk,
                                  __nv_bfloat16* __restrict__ xa, __nv_bfloat16* __restrict__ xg) {
  for (int r = blockIdx.y; r < rows; r += gridDim.y) {
    const int c = r / chunk, i = r - c * chunk;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < K; k += gridDim.x * blockDim.x) {
      __nv_bfloat16 h, l;
      split_bf16(r < n ? x[(size_t)r * ldx + k] : 0.f, h, l);
      __nv_bfloat16* a = xa + (size_t)r * 3 * K;
      a[k] = h; a[K + k] = h; a[2 * K + k] = l;
      if (xg) {
        __nv_bfloat16* g = xg + ((size_t)c * 3 * chunk + i) * K;
        g[k] = h; g[(size_t)chunk * K + k] = l; g[(size_t)2 * chunk * K + k] = h;
      }
    }
  }
}

// Row j of active problem a's W (theta[g][j * K ...]) into wcat row a * Cp + j = [h | l | h]; its bias into
// bias[a * Cp + j].
__global__ void lr_weights_kernel(const float* __restrict__ theta, long long P, const int* __restrict__ act, int Cp,
                                  int K, __nv_bfloat16* __restrict__ wcat, float* __restrict__ bias) {
  const int a = blockIdx.z, j = blockIdx.y, g = act[a];
  const float* w = theta + (size_t)g * P + (size_t)j * K;
  __nv_bfloat16* o = wcat + ((size_t)a * Cp + j) * 3 * K;
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < K; k += gridDim.x * blockDim.x) {
    __nv_bfloat16 h, l;
    split_bf16(w[k], h, l);
    o[k] = h; o[K + k] = l; o[2 * K + k] = h;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) bias[(size_t)a * Cp + j] = theta[(size_t)g * P + (size_t)Cp * K + j];
}

// ---------------------------------------------------------------------------------------------- cross-entropy
// One warp per (row i, active problem a) of a chunk of `rows` rows, the first n of them real.  z = logits + bias; each
// lane keeps an online (max, sum of exp) over its classes in increasing order, merged by a butterfly, so (max, sum)
// have the same bits on every run.  The row's loss (max - z_y + log sum) / N goes to row_loss[i, a]; the residual
// (softmax - onehot) / N, split hi + lo, to r rows i (hi), rows + i (hi) and 2 rows + i (lo), columns a Cp + c, and 0
// in the padding columns and the padding rows.
__device__ __forceinline__ void lse_merge(float& m, float& s, float om, float os) {
  const float mx = fmaxf(m, om);
  if (mx == -INFINITY) return;
  s = s * expf(m - mx) + os * expf(om - mx);
  m = mx;
}

__global__ void __launch_bounds__(LR_THREADS) lr_xent_kernel(const float* __restrict__ logits, int ld,
                                                            const float* __restrict__ bias,
                                                            const int* __restrict__ labels, int n, int rows, int C,
                                                            int Cp, float inv_n, float* __restrict__ row_loss, int Ga,
                                                            __nv_bfloat16* __restrict__ r, int ld_r) {
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * (LR_THREADS / 32) + (threadIdx.x >> 5), a = blockIdx.y;
  if (i >= rows) return;
  __nv_bfloat16* rh = r + (size_t)i * ld_r + (size_t)a * Cp;
  __nv_bfloat16* rh2 = rh + (size_t)rows * ld_r;
  __nv_bfloat16* rl = rh2 + (size_t)rows * ld_r;
  if (i >= n) {
    for (int c = lane; c < Cp; c += 32) rh[c] = rh2[c] = rl[c] = __float2bfloat16_rn(0.f);
    if (lane == 0) row_loss[(size_t)i * Ga + a] = 0.f;
    return;
  }
  const float* z = logits + (size_t)i * ld + (size_t)a * Cp;
  const float* b = bias + (size_t)a * Cp;
  float m = -INFINITY, s = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float v = z[c] + b[c];
    if (v > m) { s = s * expf(m - v) + 1.f; m = v; } else { s += expf(v - m); }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o), os = __shfl_xor_sync(0xffffffffu, s, o);
    lse_merge(m, s, om, os);
  }
  const int y = labels[i];
  for (int c = lane; c < Cp; c += 32) {
    float v = 0.f;
    if (c < C) v = (expf(z[c] + b[c] - m) / s - (c == y ? 1.f : 0.f)) * inv_n;
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    rh[c] = h; rh2[c] = h; rl[c] = l;
  }
  if (lane == 0)
    row_loss[(size_t)i * Ga + a] =
        (y >= 0 && y < C) ? ((m - (z[y] + b[y])) + logf(s)) * inv_n : __int_as_float(0x7fc00000);
}

// loss[a] += sum over the rows of row_loss[i, a], in double, in a fixed order (one CTA per problem)
__global__ void __launch_bounds__(LR_THREADS) lr_rows_sum_kernel(const float* __restrict__ row_loss, int rows, int Ga,
                                                                double* __restrict__ loss) {
  const int a = blockIdx.x;
  double v[1] = {0.0};
  for (int i = threadIdx.x; i < rows; i += LR_THREADS) v[0] += (double)row_loss[(size_t)i * Ga + a];
  block_reduce<1>(v, 0u);
  if (threadIdx.x == 0) loss[a] += v[0];
}

// ------------------------------------------------------------------------------------------------- finish
// grad[g] = [gw_a + W_g * icn_g | gb_a]; partials per (problem, slab): ||W||^2, grad . d, max |grad|, ||grad||^2.
__global__ void __launch_bounds__(LR_THREADS) lr_finish_kernel(const float* __restrict__ theta,
                                                              const float* __restrict__ gw,
                                                              const float* __restrict__ gb,
                                                              const float* __restrict__ icn,
                                                              const float* __restrict__ d, const int* __restrict__ act,
                                                              int Cp, int K, long long P, float* __restrict__ grad,
                                                              double* __restrict__ part) {
  const int a = blockIdx.y, g = act[a];
  const long long nw = (long long)Cp * K;
  const float c = icn[g];
  long long e0, e1;
  slab_range(P, e0, e1);
  double v[4] = {0.0, 0.0, 0.0, 0.0};
  for (long long e = e0 + threadIdx.x; e < e1; e += LR_THREADS) {
    float gv;
    if (e < nw) {
      const float w = theta[(size_t)g * P + e];
      gv = gw[(size_t)a * nw + e] + w * c;
      v[0] += (double)w * w;
    } else {
      gv = gb[(size_t)a * Cp + (e - nw)];
    }
    grad[(size_t)g * P + e] = gv;
    if (d) v[1] += (double)gv * d[(size_t)g * P + e];
    v[2] = fmax(v[2], (double)fabsf(gv));
    v[3] += (double)gv * gv;
  }
  block_reduce<4>(v, 1u << 2);
  if (threadIdx.x == 0)
    for (int q = 0; q < 4; ++q) part[((size_t)a * LR_SLABS + blockIdx.x) * 4 + q] = v[q];
}

// out[a, q] = the slabs of part[a, :, q] summed (or max-reduced, bit q of max_mask) in slab order; with `loss`,
// out[a, 0] = loss[a] + icn_g / 2 * (that sum) (the objective from ||W||^2).
__global__ void lr_combine_kernel(const double* __restrict__ part, int Ga, int Q, unsigned max_mask,
                                  const double* __restrict__ loss, const float* __restrict__ icn,
                                  const int* __restrict__ act, double* __restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= Ga * Q) return;
  const int a = t / Q, q = t - a * Q;
  const bool mx = max_mask >> q & 1;
  double v = 0.0;                                        // the max-reduced quantity is |grad| >= 0
  for (int s = 0; s < LR_SLABS; ++s) {
    const double p = part[((size_t)a * LR_SLABS + s) * Q + q];
    v = mx ? fmax(v, p) : v + p;
  }
  if (loss && q == 0) v = loss[a] + 0.5 * (double)icn[act[a]] * v;
  out[t] = v;
}

// ------------------------------------------------------------------------------------------------- L-BFGS
// theta_t[g] = theta[g] + alpha[g] d[g]
__global__ void lr_trial_kernel(const float* __restrict__ theta, const float* __restrict__ d,
                                const float* __restrict__ alpha, const int* __restrict__ act, long long P,
                                float* __restrict__ theta_t) {
  const int g = act[blockIdx.y];
  const float al = alpha[g];
  long long e0, e1;
  slab_range(P, e0, e1);
  for (long long e = e0 + threadIdx.x; e < e1; e += LR_THREADS) {
    const size_t o = (size_t)g * P + e;
    theta_t[o] = theta[o] + al * d[o];
  }
}

// The history of problem g: count[g] pairs, the newest in slot newest[g] of [G, m, P]; pair j (0 = newest) is in slot
// (newest - j) mod m, or absent (-1) when j >= count.
struct LrHist {
  const int* count;
  const int* newest;
  int m;
};
__device__ __forceinline__ int hist_slot(const LrHist& h, int g, int j) {
  return j < h.count[g] ? (h.newest[g] - j + h.m) % h.m : -1;
}

// part[a, slab] = u . q over the slab, u = pair j's row of U [G, m, P] (0 when absent), or with j < 0 the plain vector
// U [G, P]
__global__ void __launch_bounds__(LR_THREADS) lr_dot_kernel(const float* __restrict__ U, const float* __restrict__ q,
                                                           const int* __restrict__ act, LrHist h, int j, long long P,
                                                           double* __restrict__ part) {
  const int a = blockIdx.y, g = act[a];
  double v[1] = {0.0};
  const float* u = U + (size_t)g * P;
  bool on = true;
  if (j >= 0) {
    const int slot = hist_slot(h, g, j);
    on = slot >= 0;
    u = U + ((size_t)g * h.m + (on ? slot : 0)) * P;
  }
  if (on) {
    long long e0, e1;
    slab_range(P, e0, e1);
    for (long long e = e0 + threadIdx.x; e < e1; e += LR_THREADS) v[0] += (double)u[e] * q[(size_t)g * P + e];
  }
  block_reduce<1>(v, 0u);
  if (threadIdx.x == 0) part[(size_t)a * LR_SLABS + blockIdx.x] = v[0];
}

// The update of pair j of the two-loop recursion, from its dot product (part, summed in slab order):
//   phase 1 (newest to oldest): alpha_j = rho_j s_j . q;  q -= alpha_j y_j   (V = Y)
//   phase 2 (oldest to newest): beta = rho_j y_j . q;     q += (alpha_j - beta) s_j   (V = S)
__global__ void __launch_bounds__(LR_THREADS) lr_axpy_kernel(const double* __restrict__ part,
                                                            const float* __restrict__ rho, double* __restrict__ alph,
                                                            const float* __restrict__ V, float* __restrict__ q,
                                                            const int* __restrict__ act, LrHist h, int j, int phase,
                                                            long long P) {
  const int a = blockIdx.y, g = act[a];
  const int slot = hist_slot(h, g, j);
  if (slot < 0) return;
  double dot = 0.0;
  for (int s = 0; s < LR_SLABS; ++s) dot += part[(size_t)a * LR_SLABS + s];
  const double r = (double)rho[(size_t)g * h.m + slot] * dot;
  float coef;
  if (phase == 1) {
    coef = (float)-r;
    if (blockIdx.x == 0 && threadIdx.x == 0) alph[(size_t)a * h.m + j] = r;
  } else {
    coef = (float)(alph[(size_t)a * h.m + j] - r);
  }
  const float* v = V + ((size_t)g * h.m + slot) * P;
  long long e0, e1;
  slab_range(P, e0, e1);
  for (long long e = e0 + threadIdx.x; e < e1; e += LR_THREADS) q[(size_t)g * P + e] += coef * v[e];
}

// q[g] = -grad[g] (mode 0), or q[g] *= gamma[g] where the problem has a history (mode 1)
__global__ void lr_scale_kernel(const float* __restrict__ grad, const float* __restrict__ gamma,
                                const int* __restrict__ act, LrHist h, int mode, long long P, float* __restrict__ q) {
  const int g = act[blockIdx.y];
  if (mode == 1 && h.count[g] == 0) return;
  const float gm = mode == 1 ? gamma[g] : -1.f;
  long long e0, e1;
  slab_range(P, e0, e1);
  for (long long e = e0 + threadIdx.x; e < e1; e += LR_THREADS) {
    const size_t o = (size_t)g * P + e;
    q[o] = (mode == 1 ? q[o] : grad[o]) * gm;
  }
}

// s = theta_t - theta and y = grad_t - grad into slot[g] of S and Y; theta = theta_t, grad = grad_t; partials of
// s . y, y . y and s . s
__global__ void __launch_bounds__(LR_THREADS) lr_accept_kernel(float* __restrict__ theta, float* __restrict__ grad,
                                                              const float* __restrict__ theta_t,
                                                              const float* __restrict__ grad_t, float* __restrict__ S,
                                                              float* __restrict__ Y, const int* __restrict__ slot,
                                                              const int* __restrict__ act, int m, long long P,
                                                              double* __restrict__ part) {
  const int a = blockIdx.y, g = act[a];
  float* sv = S + ((size_t)g * m + slot[g]) * P;
  float* yv = Y + ((size_t)g * m + slot[g]) * P;
  long long e0, e1;
  slab_range(P, e0, e1);
  double v[3] = {0.0, 0.0, 0.0};
  for (long long e = e0 + threadIdx.x; e < e1; e += LR_THREADS) {
    const size_t o = (size_t)g * P + e;
    const float s = theta_t[o] - theta[o], y = grad_t[o] - grad[o];
    sv[e] = s; yv[e] = y;
    theta[o] = theta_t[o];
    grad[o] = grad_t[o];
    v[0] += (double)s * y; v[1] += (double)y * y; v[2] += (double)s * s;
  }
  block_reduce<3>(v, 0u);
  if (threadIdx.x == 0)
    for (int q = 0; q < 3; ++q) part[((size_t)a * LR_SLABS + blockIdx.x) * 3 + q] = v[q];
}

}  // namespace d3

using namespace d3;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

namespace {

double* part_workspace(int Ga, int Q, cudaStream_t st) {
  return reinterpret_cast<double*>(slab_workspace((size_t)Ga * LR_SLABS * Q * 2, st));
}

int combine(double* part, int Ga, int Q, unsigned max_mask, const double* loss, const float* icn, const int* act,
            double* out, cudaStream_t st) {
  lr_combine_kernel<<<(Ga * Q + 127) / 128, 128, 0, st>>>(part, Ga, Q, max_mask, loss, icn, act, out);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int release(double* part, int rc, cudaStream_t st) {
  slab_release(reinterpret_cast<float*>(part), st);
  return rc;
}

}  // namespace

extern "C" {

int d3_logreg_split_x(const float* x, int ldx, int n, int K, int chunk, void* xa, void* xg, void* stream) {
  if (n <= 0) return D3_OK;
  if (!x || !xa || K < 8 || K % 8 || ldx < K || chunk < 64 || chunk % 64)
    return set_error(D3_ERR_ARG, "d3_logreg_split_x: need K a positive multiple of 8, ldx >= K, chunk a positive "
                                 "multiple of 64");
  const int rows = (n + chunk - 1) / chunk * chunk;
  const dim3 grid((K + 255) / 256, rows < 65535 ? rows : 65535);
  lr_split_x_kernel<<<grid, 256, 0, STREAM(stream)>>>(x, ldx, n, rows, K, chunk, (__nv_bfloat16*)xa,
                                                      (__nv_bfloat16*)xg);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_logreg_weights(const float* theta, long long P, const int* act, int Ga, int Cp, int K, void* wcat, float* bias,
                      void* stream) {
  if (Ga <= 0) return D3_OK;
  if (!theta || !act || !wcat || !bias || Cp < 8 || Cp % 8 || K < 8 || K % 8 || P != (long long)Cp * K + Cp)
    return set_error(D3_ERR_ARG, "d3_logreg_weights: need Cp and K positive multiples of 8, P = Cp K + Cp");
  if (Cp > 65535 || Ga > 65535) return set_error(D3_ERR_ARG, "d3_logreg_weights: Cp and Ga must be <= 65535");
  const dim3 grid((K + 255) / 256, Cp, Ga);
  lr_weights_kernel<<<grid, 256, 0, STREAM(stream)>>>(theta, P, act, Cp, K, (__nv_bfloat16*)wcat, bias);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_logreg_xent(const float* logits, int ld, const float* bias, const int* labels, int n, int rows, int Ga, int C,
                   int Cp, float inv_n, double* loss, void* r, int ld_r, void* stream) {
  if (rows <= 0 || Ga <= 0) return D3_OK;
  if (!logits || !bias || !labels || !loss || !r || C < 2 || Cp < C || Cp % 8 || ld < Ga * Cp || ld_r < Ga * Cp ||
      n < 0 || n > rows || Ga > 65535)
    return set_error(D3_ERR_ARG, "d3_logreg_xent: need 2 <= C <= Cp, Cp a multiple of 8, ld and ld_r >= Ga Cp, "
                                 "0 <= n <= rows, Ga <= 65535");
  cudaStream_t st = STREAM(stream);
  float* ws = slab_workspace((size_t)rows * Ga, st);
  if (!ws) return D3_ERR_CUDA;
  const dim3 grid((rows + LR_THREADS / 32 - 1) / (LR_THREADS / 32), Ga);
  lr_xent_kernel<<<grid, LR_THREADS, 0, st>>>(logits, ld, bias, labels, n, rows, C, Cp, inv_n, ws, Ga,
                                              (__nv_bfloat16*)r, ld_r);
  cudaError_t e = cudaPeekAtLastError();
  if (e == cudaSuccess) {
    count_launch();
    lr_rows_sum_kernel<<<Ga, LR_THREADS, 0, st>>>(ws, rows, Ga, loss);
    e = cudaPeekAtLastError();
  }
  int rc = e == cudaSuccess ? D3_OK : set_error(D3_ERR_CUDA, cudaGetErrorString(e));
  if (!rc) count_launch();
  slab_release(ws, st);
  return rc;
}

int d3_logreg_finish(const float* theta, const float* gw, const float* gb, const double* loss, const float* icn,
                     const float* d, const int* act, int Ga, int Cp, int K, float* grad, double* out, void* stream) {
  if (Ga <= 0) return D3_OK;
  if (!theta || !gw || !gb || !loss || !icn || !act || !grad || !out || Cp < 8 || Cp % 8 || K < 8 || Ga > 65535)
    return set_error(D3_ERR_ARG, "d3_logreg_finish: need Cp a positive multiple of 8, K >= 8, Ga <= 65535");
  cudaStream_t st = STREAM(stream);
  const long long P = (long long)Cp * K + Cp;
  double* part = part_workspace(Ga, 4, st);
  if (!part) return D3_ERR_CUDA;
  lr_finish_kernel<<<dim3(LR_SLABS, Ga), LR_THREADS, 0, st>>>(theta, gw, gb, icn, d, act, Cp, K, P, grad, part);
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) return release(part, set_error(D3_ERR_CUDA, cudaGetErrorString(e)), st);
  count_launch();
  return release(part, combine(part, Ga, 4, 1u << 2, loss, icn, act, out, st), st);
}

int d3_logreg_trial(const float* theta, const float* d, const float* alpha, const int* act, int Ga, long long P,
                    float* theta_t, void* stream) {
  if (Ga <= 0) return D3_OK;
  if (!theta || !d || !alpha || !act || !theta_t || P <= 0 || Ga > 65535)
    return set_error(D3_ERR_ARG, "d3_logreg_trial: need P > 0, Ga <= 65535");
  lr_trial_kernel<<<dim3(LR_SLABS, Ga), LR_THREADS, 0, STREAM(stream)>>>(theta, d, alpha, act, P, theta_t);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_logreg_direction(const float* grad, const float* S, const float* Y, const float* rho, const float* gamma,
                        const int* count, const int* newest, const int* act, int Ga, long long P, int m, float* d,
                        double* gd, void* stream) {
  if (Ga <= 0) return D3_OK;
  if (!grad || !S || !Y || !rho || !gamma || !count || !newest || !act || !d || !gd || P <= 0 || m < 1 ||
      m > LR_MAX_HISTORY || Ga > 65535)
    return set_error(D3_ERR_ARG, "d3_logreg_direction: need P > 0, 1 <= m <= 64, Ga <= 65535");
  cudaStream_t st = STREAM(stream);
  double* part = part_workspace(Ga, 1, st);
  double* alph = reinterpret_cast<double*>(slab_workspace((size_t)Ga * m * 2, st));
  if (!part || !alph) {
    slab_release(reinterpret_cast<float*>(alph), st);
    return release(part, D3_ERR_CUDA, st);
  }
  const LrHist h{count, newest, m};
  const dim3 grid(LR_SLABS, Ga);
  int rc = D3_OK;
  cudaError_t e;
#define LR_STEP(launch)                                                               \
  do {                                                                                \
    launch;                                                                           \
    e = cudaPeekAtLastError();                                                        \
    if (e != cudaSuccess) { rc = set_error(D3_ERR_CUDA, cudaGetErrorString(e)); goto done; } \
    count_launch();                                                                   \
  } while (0)
  LR_STEP((lr_scale_kernel<<<grid, LR_THREADS, 0, st>>>(grad, gamma, act, h, 0, P, d)));
  for (int j = 0; j < m; ++j) {
    LR_STEP((lr_dot_kernel<<<grid, LR_THREADS, 0, st>>>(S, d, act, h, j, P, part)));
    LR_STEP((lr_axpy_kernel<<<grid, LR_THREADS, 0, st>>>(part, rho, alph, Y, d, act, h, j, 1, P)));
  }
  LR_STEP((lr_scale_kernel<<<grid, LR_THREADS, 0, st>>>(grad, gamma, act, h, 1, P, d)));
  for (int j = m - 1; j >= 0; --j) {
    LR_STEP((lr_dot_kernel<<<grid, LR_THREADS, 0, st>>>(Y, d, act, h, j, P, part)));
    LR_STEP((lr_axpy_kernel<<<grid, LR_THREADS, 0, st>>>(part, rho, alph, S, d, act, h, j, 2, P)));
  }
  LR_STEP((lr_dot_kernel<<<grid, LR_THREADS, 0, st>>>(grad, d, act, h, -1, P, part)));
#undef LR_STEP
  rc = combine(part, Ga, 1, 0u, nullptr, nullptr, act, gd, st);
done:
  slab_release(reinterpret_cast<float*>(alph), st);
  return release(part, rc, st);
}

int d3_logreg_accept(float* theta, float* grad, const float* theta_t, const float* grad_t, float* S, float* Y,
                     const int* slot, const int* act, int Ga, long long P, int m, double* out, void* stream) {
  if (Ga <= 0) return D3_OK;
  if (!theta || !grad || !theta_t || !grad_t || !S || !Y || !slot || !act || !out || P <= 0 || m < 1 ||
      m > LR_MAX_HISTORY || Ga > 65535)
    return set_error(D3_ERR_ARG, "d3_logreg_accept: need P > 0, 1 <= m <= 64, Ga <= 65535");
  cudaStream_t st = STREAM(stream);
  double* part = part_workspace(Ga, 3, st);
  if (!part) return D3_ERR_CUDA;
  lr_accept_kernel<<<dim3(LR_SLABS, Ga), LR_THREADS, 0, st>>>(theta, grad, theta_t, grad_t, S, Y, slot, act, m, P,
                                                               part);
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) return release(part, set_error(D3_ERR_CUDA, cudaGetErrorString(e)), st);
  count_launch();
  return release(part, combine(part, Ga, 3, 0u, nullptr, nullptr, act, out, st), st);
}

}  // extern "C"
