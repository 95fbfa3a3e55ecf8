// Unsupervised object discovery (TokenCut's normalized cut on the patch-affinity graph): the thresholded graph, its
// normalized-cut eigenvector, and the box of the seed's connected component with its best IoU against the ground
// truth.  A launch covers n images that share one N = h w patch grid; the similarities s = F F^T come from d3_gemm_bf16
// (fp32 results); nothing here multiplies matrices.
//
// Graph: A_ij = 1 if s_ij > tau, else eps (the diagonal included), stored as a bit matrix, N x ceil(N / 32) words per
// image, bit j % 32 of word j / 32 of row i set when s_ij > tau.  The degree d_i = c_i + (N - c_i) eps from the
// integer count c_i of set bits, in fp32.
//
// Eigenvector: the generalized eigenproblem (D - A) x = lambda D x at its second-smallest lambda is the eigenproblem of
// M = D^-1/2 A D^-1/2 at its second-largest eigenvalue theta (x = D^-1/2 y, lambda_2 = 1 - theta).  M's top eigenpair
// is (1, u1 = D^1/2 1 / ||D^1/2 1||), simple because every A_ij > 0.  od_fiedler_kernel runs Lanczos on M in fp32, one
// CTA per image, from a fixed pseudo-random start vector, with classical Gram-Schmidt twice against u1 and every stored
// Lanczos vector (so the Krylov space stays orthogonal to u1 and its largest Ritz value approximates theta).  The
// matvec reads the bit matrix: (A z)_i = (1 - eps) sum_{j: bit ij} z_j + eps sum_j z_j, lane l of the row's warp adding
// column 32 k + l for k in order, then a fixed butterfly.  After step m the largest eigenvalue of the m x m tridiagonal
// T_m is bracketed in fp64 by Sturm-count multisection (every thread one point, six rounds), its vector s by two
// steps of inverse iteration at the bracket's upper end (T - sigma I is then negative definite, so the LDL^T solve
// without pivoting is stable); the iteration stops when the residual bound beta_m |s_m| <= OD_TOL, when the Krylov
// space is exhausted (m = N - 1), or at m = k_max (then the image is flagged unconverged and still gets its Ritz
// vector).  Output x = D^-1/2 Q s with ||Q s|| = 1, so x^T D x = 1; its sign is whatever Lanczos produced.
//
// Box: the candidates are the patches with x_i > mean(x) (fp64 mean); the seed is argmax |x_i|, the lowest index on
// ties; if the seed is not a candidate the complement is taken (TokenCut's sign flip).  The 4-connected component of
// the seed is grown in shared memory as a bit set over the flat grid index, expanded one step per round until nothing
// changes; its grid bounding box [x0, y0, x1, y1] gives the pixel box [x0 p, y0 p, (x1 + 1) p, (y1 + 1) p] clipped to
// W x H.  The IoU with each ground-truth box is computed on continuous areas in fp64 (no + 1); hit = best IoU >= 0.5.
//
// Every reduction runs in a fixed order and nothing uses atomics: the same bits on every run.
#include "ptx.cuh"
#include "d3_internal.h"

#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <vector>

namespace d3 {

constexpr int OD_MAX_N = 4096;                  // patches per image; the bits of one image are at most 2 MB
constexpr int OD_KMAX = 256;                    // Lanczos steps at most
constexpr float OD_TOL = 1e-6f;                 // residual bound beta_m |s_m| (||M|| = 1)
constexpr int OG_WARPS = 8;                     // graph: one warp per row
constexpr int OF_THREADS = 512;                 // fiedler: one CTA per image
constexpr int OF_VPT = OD_MAX_N / OF_THREADS;   // vector elements owned per thread
constexpr int OF_ROUNDS = 6;                    // multisection rounds of 512 points: ~2^-54 of the Gershgorin width
constexpr int OB_THREADS = 256;                 // box: one CTA per image
constexpr int OB_WORDS = OD_MAX_N / 32;

// ------------------------------------------------------------------------------------------------ graph
__global__ void __launch_bounds__(OG_WARPS * 32) od_graph_kernel(const float* __restrict__ sim, int lds, int n, int N,
                                                                 int words, float tau, float eps,
                                                                 uint32_t* __restrict__ bits,
                                                                 float* __restrict__ degree) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * OG_WARPS + (threadIdx.x >> 5);
  if (row >= (long long)n * N) return;
  const float* s = sim + row * lds;                       // image m's rows start at m N lds
  uint32_t* b = bits + row * words;
  int c = 0;
  for (int k = 0; k < words; ++k) {
    const int j = 32 * k + lane;
    const uint32_t m = __ballot_sync(0xffffffffu, j < N && s[j] > tau);
    if (lane == 0) b[k] = m;
    c += __popc(m);
  }
  if (lane == 0) degree[row] = (float)c + (float)(N - c) * eps;
}

// ------------------------------------------------------------------------------------------------ fiedler
struct FiedlerSmem {
  float z[OD_MAX_N];        // D^-1/2 q, read by column in the matvec
  float v[OD_MAX_N];        // the matvec's rows; the vector being orthogonalised
  float h[OD_KMAX + 1];     // Gram-Schmidt coefficients against u1 and the Lanczos vectors
  float red[32];
  double a[OD_KMAX], b[OD_KMAX], b2[OD_KMAX];   // T: diagonal, off-diagonal, off-diagonal squared
  double s[OD_KMAX], l[OD_KMAX], rd[OD_KMAX];   // Ritz vector; LDL^T multipliers and reciprocal pivots
  double theta, resid;
};

// the sum over the CTA, the same bits in every thread
__device__ __forceinline__ float od_block_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();                                        // red is free
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  return warp_sum((threadIdx.x & 31) < (int)(blockDim.x >> 5) ? red[threadIdx.x & 31] : 0.f);
}

__device__ __forceinline__ float od_start(int i) {
  uint32_t x = (uint32_t)i * 2654435761u + 0x9e3779b9u;
  x ^= x >> 16;
  x *= 0x85ebca6bu;
  x ^= x >> 13;
  x *= 0xc2b2ae35u;
  x ^= x >> 16;
  return (float)(x >> 8) * (1.f / 16777216.f) - 0.5f;
}

// w -= Q[0:rows]^T (Q[0:rows] w): one classical Gram-Schmidt pass, Q rows of N floats
__device__ void od_reorth(float (&w)[OF_VPT], const float* __restrict__ Q, int rows, int N, FiedlerSmem& sm) {
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  __syncthreads();                                        // sm.v and sm.h are free
#pragma unroll
  for (int r = 0; r < OF_VPT; ++r)
    if (t + r * OF_THREADS < N) sm.v[t + r * OF_THREADS] = w[r];
  __syncthreads();
  for (int m = warp; m < rows; m += OF_THREADS / 32) {
    const float* qm = Q + (size_t)m * N;
    float acc = 0.f;
    for (int i = lane; i < N; i += 32) acc = fmaf(qm[i], sm.v[i], acc);
    acc = warp_sum(acc);
    if (lane == 0) sm.h[m] = acc;
  }
  __syncthreads();
  for (int m = 0; m < rows; ++m) {
    const float hm = sm.h[m];
    const float* qm = Q + (size_t)m * N;
#pragma unroll
    for (int r = 0; r < OF_VPT; ++r)
      if (t + r * OF_THREADS < N) w[r] = fmaf(-hm, qm[t + r * OF_THREADS], w[r]);
  }
}

// eigenvalues of T_m below x: the negative pivots of the LDL^T of T - x I
__device__ __forceinline__ int od_sturm(const double* __restrict__ a, const double* __restrict__ b2, int m, double x) {
  int c = 0;
  double d = 1.0;
  for (int k = 0; k < m; ++k) {
    d = (a[k] - x) - (k ? b2[k - 1] / d : 0.0);
    if (d == 0.0) d = -1e-300;
    c += d < 0.0;
  }
  return c;
}

// The largest eigenvalue of T_m (sm.a, sm.b) into sm.theta, its unit vector into sm.s and beta_m |s_m| into
// sm.resid; every thread calls it.
__device__ void od_ritz(int m, FiedlerSmem& sm) {
  double lo = 1e300, hi = -1e300;
  for (int k = 0; k < m; ++k) {                           // Gershgorin, in every thread alike
    const double r = (k ? fabs(sm.b[k - 1]) : 0.0) + (k + 1 < m ? fabs(sm.b[k]) : 0.0);
    lo = fmin(lo, sm.a[k] - r);
    hi = fmax(hi, sm.a[k] + r);
  }
  lo -= 1e-12;
  hi += 1e-12;
  for (int round = 0; round < OF_ROUNDS; ++round) {
    const double step = (hi - lo) / (double)(OF_THREADS + 1);
    const double x = lo + step * (double)(threadIdx.x + 1);
    const int below = __syncthreads_count(od_sturm(sm.a, sm.b2, m, x) < m);   // points that leave one eigenvalue above
    const double nlo = below > 0 ? lo + step * (double)below : lo;
    hi = below < OF_THREADS ? lo + step * (double)(below + 1) : hi;
    lo = nlo;
  }
  if (threadIdx.x == 0) {
    const double sigma = hi + 1e-12 * fmax(1.0, fabs(hi));      // above theta: T - sigma I is negative definite
    double d = sm.a[0] - sigma;
    sm.rd[0] = 1.0 / d;
    for (int k = 1; k < m; ++k) {
      sm.l[k] = sm.b[k - 1] * sm.rd[k - 1];
      d = (sm.a[k] - sigma) - sm.l[k] * sm.b[k - 1];
      if (d > -1e-300) d = -1e-300;
      sm.rd[k] = 1.0 / d;
    }
    for (int k = 0; k < m; ++k) sm.s[k] = 1.0;
    for (int it = 0; it < 2; ++it) {
      for (int k = 1; k < m; ++k) sm.s[k] -= sm.l[k] * sm.s[k - 1];
      sm.s[m - 1] *= sm.rd[m - 1];
      for (int k = m - 2; k >= 0; --k) sm.s[k] = (sm.s[k] - sm.b[k] * sm.s[k + 1]) * sm.rd[k];
      double ss = 0.0;
      for (int k = 0; k < m; ++k) ss += sm.s[k] * sm.s[k];
      const double inv = 1.0 / sqrt(ss);
      for (int k = 0; k < m; ++k) sm.s[k] *= inv;
    }
    sm.theta = 0.5 * (lo + hi);
    sm.resid = fabs(sm.b[m - 1] * sm.s[m - 1]);
  }
  __syncthreads();
}

// Q: per image (k_eff + 1) x N floats of workspace: row 0 = u1, row 1 + k = the k-th Lanczos vector
__global__ void __launch_bounds__(OF_THREADS, 1) od_fiedler_kernel(const uint32_t* __restrict__ bits,
                                                                   const float* __restrict__ degree, int N, int words,
                                                                   float eps, int k_eff, float* __restrict__ Qws,
                                                                   float* __restrict__ x, float* __restrict__ lambda2,
                                                                   int* __restrict__ iters,
                                                                   int* __restrict__ converged) {
  __shared__ FiedlerSmem sm;
  const int img = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  bits += (size_t)img * N * words;
  degree += (size_t)img * N;
  float* Q = Qws + (size_t)img * (k_eff + 1) * N;
  float di[OF_VPT], q[OF_VPT], w[OF_VPT];
  float part = 0.f;
#pragma unroll
  for (int r = 0; r < OF_VPT; ++r) {
    const int i = t + r * OF_THREADS;
    const float d = i < N ? degree[i] : 0.f;
    di[r] = i < N ? 1.f / sqrtf(d) : 0.f;
    part += d;
  }
  const float un = 1.f / sqrtf(od_block_sum(part, sm.red));
#pragma unroll
  for (int r = 0; r < OF_VPT; ++r) {
    const int i = t + r * OF_THREADS;
    if (i < N) Q[i] = sqrtf(degree[i]) * un;             // u1
    w[r] = i < N ? od_start(i) : 0.f;
  }
  od_reorth(w, Q, 1, N, sm);
  od_reorth(w, Q, 1, N, sm);
  part = 0.f;
#pragma unroll
  for (int r = 0; r < OF_VPT; ++r) part = fmaf(w[r], w[r], part);
  float inv = 1.f / sqrtf(od_block_sum(part, sm.red));
#pragma unroll
  for (int r = 0; r < OF_VPT; ++r) {
    const int i = t + r * OF_THREADS;
    q[r] = w[r] * inv;
    if (i < N) Q[N + i] = q[r];
  }
  float beta = 0.f;
  int m = 0;
  for (int j = 0; j < k_eff; ++j) {
    // w = M q
    part = 0.f;
#pragma unroll
    for (int r = 0; r < OF_VPT; ++r) {
      const int i = t + r * OF_THREADS;
      const float zi = di[r] * q[r];
      if (i < N) sm.z[i] = zi;
      part += zi;
    }
    const float zsum = od_block_sum(part, sm.red);        // its barriers also publish sm.z
    for (int row = warp; row < N; row += OF_THREADS / 32) {
      const uint32_t* br = bits + (size_t)row * words;
      float acc = 0.f;
      for (int k0 = 0; k0 < words; k0 += 32) {
        const uint32_t mine = k0 + lane < words ? br[k0 + lane] : 0u;
        const int kn = min(32, words - k0);
        for (int k = 0; k < kn; ++k) {
          const uint32_t wd = __shfl_sync(0xffffffffu, mine, k);
          if ((wd >> lane) & 1u) acc += sm.z[32 * (k0 + k) + lane];
        }
      }
      acc = warp_sum(acc);
      if (lane == 0) sm.v[row] = (1.f - eps) * acc + eps * zsum;
    }
    __syncthreads();
    part = 0.f;
#pragma unroll
    for (int r = 0; r < OF_VPT; ++r) {
      const int i = t + r * OF_THREADS;
      w[r] = i < N ? di[r] * sm.v[i] : 0.f;
      part = fmaf(q[r], w[r], part);
    }
    const float alpha = od_block_sum(part, sm.red);
#pragma unroll
    for (int r = 0; r < OF_VPT; ++r) w[r] = fmaf(-alpha, q[r], w[r]);     // beta q_{j-1} goes with the reorthogonalisation
    od_reorth(w, Q, j + 2, N, sm);
    od_reorth(w, Q, j + 2, N, sm);
    part = 0.f;
#pragma unroll
    for (int r = 0; r < OF_VPT; ++r) part = fmaf(w[r], w[r], part);
    beta = sqrtf(od_block_sum(part, sm.red));
    if (t == 0) {
      sm.a[j] = alpha;
      sm.b[j] = beta;
      sm.b2[j] = (double)beta * (double)beta;
    }
    __syncthreads();
    m = j + 1;
    od_ritz(m, sm);
    if (sm.resid <= OD_TOL || m == k_eff) break;
    inv = 1.f / beta;
#pragma unroll
    for (int r = 0; r < OF_VPT; ++r) {
      const int i = t + r * OF_THREADS;
      q[r] = w[r] * inv;
      if (i < N) Q[(size_t)(j + 2) * N + i] = q[r];
    }
  }
  // y = Q s over the Lanczos vectors, x = D^-1/2 y / ||y||
  part = 0.f;
#pragma unroll
  for (int r = 0; r < OF_VPT; ++r) {
    const int i = t + r * OF_THREADS;
    float y = 0.f;
    if (i < N)
      for (int k = 0; k < m; ++k) y = fmaf((float)sm.s[k], Q[(size_t)(k + 1) * N + i], y);
    w[r] = y;
    part = fmaf(y, y, part);
  }
  inv = 1.f / sqrtf(od_block_sum(part, sm.red));
#pragma unroll
  for (int r = 0; r < OF_VPT; ++r) {
    const int i = t + r * OF_THREADS;
    if (i < N) x[(size_t)img * N + i] = di[r] * w[r] * inv;
  }
  if (t == 0) {
    lambda2[img] = (float)(1.0 - sm.theta);
    iters[img] = m;
    converged[img] = sm.resid <= OD_TOL || m == N - 1;
  }
}

// ------------------------------------------------------------------------------------------------ box
// bit c of the result = bit c - s of v (bits below 0 read as 0)
__device__ __forceinline__ uint32_t od_from_lower(const uint32_t* v, int k, int s, int nw) {
  const int q = s >> 5, r = s & 31, k0 = k - q;
  const uint32_t a = k0 >= 0 && k0 < nw ? v[k0] << r : 0u;
  const uint32_t b = r && k0 - 1 >= 0 && k0 - 1 < nw ? v[k0 - 1] >> (32 - r) : 0u;
  return a | b;
}

// bit c of the result = bit c + s of v (bits beyond the words read as 0)
__device__ __forceinline__ uint32_t od_from_higher(const uint32_t* v, int k, int s, int nw) {
  const int q = s >> 5, r = s & 31, k0 = k + q;
  const uint32_t a = k0 < nw ? v[k0] >> r : 0u;
  const uint32_t b = r && k0 + 1 < nw ? v[k0 + 1] << (32 - r) : 0u;
  return a | b;
}

// (v, i) beats (bv, bi): larger value, or the same value at a lower index
__device__ __forceinline__ bool od_better(float v, int i, float bv, int bi) {
  return v > bv || (v == bv && i < bi);
}

// meta (workspace copy of the host arrays) int [n, 3] = (H, W, number of ground-truth boxes)
__global__ void __launch_bounds__(OB_THREADS) od_box_kernel(const float* __restrict__ xs, int N, int h, int w,
                                                            int patch, const int* __restrict__ meta,
                                                            const float* __restrict__ gt, int b_max,
                                                            uint8_t* __restrict__ fg_out, int* __restrict__ box,
                                                            float* __restrict__ best_iou, int* __restrict__ hit) {
  __shared__ uint32_t fg[OB_WORDS], comp[OB_WORDS], nxt[OB_WORDS], first[OB_WORDS], last[OB_WORDS];
  __shared__ double dred[OB_THREADS / 32];
  __shared__ float vred[OB_THREADS / 32];
  __shared__ int ired[4][OB_THREADS / 32];
  const int img = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const float* x = xs + (size_t)img * N;
  const int nw = (N + 31) / 32;
  // the mean (fp64) and the seed
  double sum = 0.0;
  float bv = -1.f;
  int bi = N;
  for (int i = t; i < N; i += OB_THREADS) {
    sum += (double)x[i];
    const float a = fabsf(x[i]);
    if (od_better(a, i, bv, bi)) { bv = a; bi = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float v = __shfl_xor_sync(0xffffffffu, bv, o);
    const int i = __shfl_xor_sync(0xffffffffu, bi, o);
    if (od_better(v, i, bv, bi)) { bv = v; bi = i; }
  }
  if (lane == 0) { dred[warp] = sum; vred[warp] = bv; ired[0][warp] = bi; }
  __syncthreads();
  sum = 0.0;
  bv = -1.f;
  bi = N;
  for (int k = 0; k < OB_THREADS / 32; ++k) {
    sum += dred[k];
    if (od_better(vred[k], ired[0][k], bv, bi)) { bv = vred[k]; bi = ired[0][k]; }
  }
  const double mean = sum / (double)N;
  const int seed = bi;
  const bool flip = !((double)x[seed] > mean);
  // the foreground, the column masks, the seed
  for (int k = t; k < nw; k += OB_THREADS) {
    uint32_t f = 0u, c0 = 0u, c1 = 0u;
    for (int b = 0; b < 32; ++b) {
      const int c = 32 * k + b;
      if (c >= N) break;
      const bool on = ((double)x[c] > mean) != flip;
      fg_out[(size_t)img * N + c] = on;
      f |= (uint32_t)on << b;
      c0 |= (uint32_t)(c % w == 0) << b;
      c1 |= (uint32_t)(c % w == w - 1) << b;
    }
    fg[k] = f;
    first[k] = c0;
    last[k] = c1;
    comp[k] = k == (seed >> 5) ? 1u << (seed & 31) : 0u;
  }
  // grow the seed's 4-connected component to a fixed point
  for (;;) {
    __syncthreads();
    int changed = 0;
    for (int k = t; k < nw; k += OB_THREADS) {
      const uint32_t grown = comp[k] | (od_from_lower(comp, k, 1, nw) & ~first[k]) |
                             (od_from_higher(comp, k, 1, nw) & ~last[k]) | od_from_lower(comp, k, w, nw) |
                             od_from_higher(comp, k, w, nw);
      nxt[k] = grown & fg[k];
      changed |= nxt[k] != comp[k];
    }
    if (!__syncthreads_or(changed)) break;
    for (int k = t; k < nw; k += OB_THREADS) comp[k] = nxt[k];
  }
  // its bounding box on the grid
  int x0 = w, y0 = h, x1 = -1, y1 = -1;
  for (int k = t; k < nw; k += OB_THREADS) {
    uint32_t c = comp[k];
    while (c) {
      const int cell = 32 * k + __ffs(c) - 1;
      c &= c - 1;
      const int cy = cell / w, cx = cell % w;
      x0 = min(x0, cx); x1 = max(x1, cx);
      y0 = min(y0, cy); y1 = max(y1, cy);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    x0 = min(x0, __shfl_xor_sync(0xffffffffu, x0, o));
    y0 = min(y0, __shfl_xor_sync(0xffffffffu, y0, o));
    x1 = max(x1, __shfl_xor_sync(0xffffffffu, x1, o));
    y1 = max(y1, __shfl_xor_sync(0xffffffffu, y1, o));
  }
  if (lane == 0) { ired[0][warp] = x0; ired[1][warp] = y0; ired[2][warp] = x1; ired[3][warp] = y1; }
  __syncthreads();
  if (t == 0) {
    for (int k = 1; k < OB_THREADS / 32; ++k) {
      x0 = min(x0, ired[0][k]); y0 = min(y0, ired[1][k]);
      x1 = max(x1, ired[2][k]); y1 = max(y1, ired[3][k]);
    }
    const int H = meta[3 * img], W = meta[3 * img + 1], nb = meta[3 * img + 2];
    const int bx0 = min(x0 * patch, W), by0 = min(y0 * patch, H);
    const int bx1 = min((x1 + 1) * patch, W), by1 = min((y1 + 1) * patch, H);
    box[4 * img] = bx0;
    box[4 * img + 1] = by0;
    box[4 * img + 2] = bx1;
    box[4 * img + 3] = by1;
    const double area = (double)(bx1 - bx0) * (double)(by1 - by0);
    double best = 0.0;
    for (int g = 0; g < nb; ++g) {
      const float* gb = gt + ((size_t)img * b_max + g) * 4;
      const double gx0 = gb[0], gy0 = gb[1], gx1 = gb[2], gy1 = gb[3];
      const double iw = fmax(0.0, fmin((double)bx1, gx1) - fmax((double)bx0, gx0));
      const double ih = fmax(0.0, fmin((double)by1, gy1) - fmax((double)by0, gy0));
      const double inter = iw * ih;
      const double uni = area + (gx1 - gx0) * (gy1 - gy0) - inter;
      const double iou = uni > 0.0 ? inter / uni : 0.0;
      best = fmax(best, iou);
    }
    best_iou[img] = (float)best;
    hit[img] = best >= 0.5;
  }
}

}  // namespace d3

using namespace d3;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

int d3_od_graph(const float* sim, int lds, int n, int N, float tau, float eps, void* bits, float* degree,
                void* stream) {
  if (n < 0 || N < 2 || N > OD_MAX_N || lds < N || lds % 4 || !(eps > 0.f) || !(eps < 1.f) || tau != tau)
    return set_error(D3_ERR_ARG, "d3_od_graph: need n >= 0, 2 <= N <= 4096 patches, lds >= N a multiple of 4, "
                                 "0 < eps < 1 and a finite tau");
  if (n == 0) return D3_OK;
  if (!sim || !bits || !degree || (uintptr_t)sim % 16 || (uintptr_t)bits % 4 || (uintptr_t)degree % 4)
    return set_error(D3_ERR_ARG, "d3_od_graph: need non-null buffers, sim 16-byte aligned, bits and degree 4-byte "
                                 "aligned");
  const long long rows = (long long)n * N;
  od_graph_kernel<<<(unsigned)((rows + OG_WARPS - 1) / OG_WARPS), OG_WARPS * 32, 0, STREAM(stream)>>>(
      sim, lds, n, N, (N + 31) / 32, tau, eps, (uint32_t*)bits, degree);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_od_fiedler(const void* bits, const float* degree, int n, int N, float eps, int k_max, float* x,
                  float* lambda2, int* iters, int* converged, void* stream) {
  if (n < 0 || N < 2 || N > OD_MAX_N || k_max < 1 || k_max > OD_KMAX || !(eps > 0.f) || !(eps < 1.f))
    return set_error(D3_ERR_ARG, "d3_od_fiedler: need n >= 0, 2 <= N <= 4096 patches, 1 <= k_max <= 256 and "
                                 "0 < eps < 1");
  if (n == 0) return D3_OK;
  if (!bits || !degree || !x || !lambda2 || !iters || !converged || (uintptr_t)bits % 4 || (uintptr_t)degree % 4 ||
      (uintptr_t)x % 4)
    return set_error(D3_ERR_ARG, "d3_od_fiedler: need non-null, 4-byte aligned buffers");
  cudaStream_t st = STREAM(stream);
  const int k_eff = std::min(k_max, N - 1);               // the space orthogonal to u1 has N - 1 dimensions
  float* ws = slab_workspace((size_t)n * (k_eff + 1) * N, st);
  if (!ws) return D3_ERR_CUDA;
  od_fiedler_kernel<<<n, OF_THREADS, 0, st>>>((const uint32_t*)bits, degree, N, (N + 31) / 32, eps, k_eff, ws, x,
                                              lambda2, iters, converged);
  const cudaError_t e = cudaPeekAtLastError();
  int rc = D3_OK;
  if (e != cudaSuccess) rc = set_error(D3_ERR_CUDA, cudaGetErrorString(e)); else count_launch();
  slab_release(ws, st);
  return rc;
}

int d3_od_box(const float* x, int n, int h, int w, int patch, const int* sizes, const int* n_gt, const float* gt,
              int b_max, void* fg_u8, int* box, float* best_iou, int* hit, void* stream) {
  if (n < 0 || h < 1 || w < 1 || (long long)h * w < 2 || (long long)h * w > OD_MAX_N || patch < 1 || b_max < 0)
    return set_error(D3_ERR_ARG, "d3_od_box: need n >= 0, h, w >= 1 with 2 <= h w <= 4096, patch >= 1 and "
                                 "b_max >= 0");
  if (n == 0) return D3_OK;
  if (!x || !sizes || !n_gt || (b_max > 0 && !gt) || !fg_u8 || !box || !best_iou || !hit || (uintptr_t)x % 4 ||
      (uintptr_t)gt % 4)
    return set_error(D3_ERR_ARG, "d3_od_box: need non-null, 4-byte aligned buffers");
  std::vector<int> meta(3 * (size_t)n);
  for (int i = 0; i < n; ++i) {
    const int H = sizes[2 * i], W = sizes[2 * i + 1];
    if (H < 1 || W < 1 || (H + patch - 1) / patch != h || (W + patch - 1) / patch != w)
      return set_error(D3_ERR_ARG, "d3_od_box: an image size (H, W) does not give the h x w grid "
                                   "(ceil(H / patch), ceil(W / patch))");
    if (n_gt[i] < 0 || n_gt[i] > b_max)
      return set_error(D3_ERR_ARG, "d3_od_box: a ground-truth box count is outside [0, b_max]");
    meta[3 * i] = H;
    meta[3 * i + 1] = W;
    meta[3 * i + 2] = n_gt[i];
  }
  cudaStream_t st = STREAM(stream);
  float* ws = slab_workspace(meta.size(), st);
  if (!ws) return D3_ERR_CUDA;
  // a copy from pageable memory is staged before the call returns, so meta may go out of scope
  cudaError_t e = cudaMemcpyAsync(ws, meta.data(), sizeof(int) * meta.size(), cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) {
    od_box_kernel<<<n, OB_THREADS, 0, st>>>(x, h * w, h, w, patch, reinterpret_cast<const int*>(ws), gt, b_max,
                                            (uint8_t*)fg_u8, box, best_iou, hit);
    e = cudaPeekAtLastError();
  }
  int rc = D3_OK;
  if (e != cudaSuccess) rc = set_error(D3_ERR_CUDA, cudaGetErrorString(e)); else count_launch();
  slab_release(ws, st);
  return rc;
}

}  // extern "C"
