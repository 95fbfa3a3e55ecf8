// Multi-head self-attention forward / backward on the Hopper tensor cores (wgmma): replaces flax
// `nn.dot_product_attention(q, k, v)` at dinov3_jax/layers/attention.py:116 (softmax((q / sqrt(head_dim)) k^T) v, no mask,
// no dropout) and its jax.grad, for head_dim 64 and 128 and any crop length up to ATTN_MAX_TOKENS.
//
// Operands come by TMA (SWIZZLE_128B) from the fused qkv buffer [T, 3D] (q | k | v thirds, heads contiguous); every
// product is a warpgroup MMA with fp32 accumulators in registers.  Short crops (N <= 64) are packed G per 128-row tile
// with a block-diagonal mask, so one CTA covers a "crop group" of span = G * N token rows.
//
// Three kernel families; d3_attn_fwd / d3_attn_bwd pick one from D / H and the span:
//   resident, head_dim 64   the DINOv3 crops (N = 197 / 37 / 257 / 50; span <= 448 forward, <= 256 backward):
//                           attn_fwd_kernel and attn_bwd_fused_kernel keep every tile of the crop group in shared memory.
//   streamed, head_dim 64   longer crops, G = 1: attn_fwd_stream_kernel, attn_bwd_dkdv_kernel, attn_bwd_dq_kernel.
//   head_dim 128 (vit_7b)   any span: attn_fwd_hd128_kernel, attn_bwd_dkdv_hd128_kernel, attn_bwd_dq_hd128_kernel.
// The streamed and head_dim 128 kernels share one TileRing: a producer warpgroup streams 128-row K / V (or Q / dO) tiles
// through an mbarrier ring that both consumer warpgroups read, so shared memory does not grow with N.  All three
// families run the same per-tile arithmetic: S = Q K^T, online softmax (forward) or P / dS from the saved LSE (backward),
// with the score fragments handed to the next product straight from registers (RS form).
#include "ptx.cuh"
#include <climits>
#include <cstdlib>
#include "d3_internal.h"

namespace d3 {

constexpr float LOG2E = 1.4426950408889634f;
constexpr int SMEM_ALIGN = 1024;   // dynamic shared memory slack for smem_base_1024 (SWIZZLE_128B tiles are 1 KB aligned)

__device__ __forceinline__ uint8_t* smem_base_1024(uint8_t* raw) {
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~uintptr_t(1023));
}

struct AttnShape {
  int G;         // crops packed per CTA (block-diagonal attention inside one 128-row tile when G*N <= 128)
  int span;      // G*N: token rows owned by one CTA (grid.z = ceil(n_crops / G))
  int n_crops;
  int N;         // tokens per crop
  int nkb;       // 64-key blocks covering the span
  int D;         // embed dim (row stride of o / do); qkv row stride = 3D
  int H;
  float scale;   // head_dim^-0.5
  const float* sin_t;  // backward only: RoPE tables [P, 64] (nullptr = gradients stay in the rotated frame)
  const float* cos_t;
  int prefix;          // tokens before the first patch token (cls + storage tokens)
};

// swizzled (SWIZZLE_128B, K-major) byte offset of element (row, col) in a [rows x 64] bf16 chunk
__device__ __forceinline__ uint32_t sw128_offset(int row, int col) {
  return (uint32_t)(row * 128 + ((((col >> 3) ^ (row & 7)) & 7) << 4) + (col & 7) * 2);
}

// the crop of a token row inside the group and its key range [klo, khi)
struct RowInfo { int g, klo, khi; bool ok; };
__device__ __forceinline__ RowInfo row_info(const AttnShape& sh, int c, int q) {
  RowInfo ri;
  ri.g = min(q / sh.N, sh.G - 1);
  ri.klo = ri.g * sh.N;
  ri.khi = ri.klo + sh.N;
  ri.ok = (q < sh.span) && (c * sh.G + ri.g < sh.n_crops);
  return ri;
}

// Online softmax of one block of 8*NI keys starting at key k0, on the S accumulator fragment (this thread: rows ri[0],
// ri[1], columns k0 + 8i + c2 + {0,1}).  S becomes P; the running max m, sum l and the output accumulator o (NO = head_dim
// / 2 registers) are rescaled.  Keys outside a row's [klo, khi) give exactly 0.
template <int NI, int NO>
__device__ __forceinline__ void online_softmax(float (&s)[4 * NI], float (&o)[NO], float (&m)[2], float (&l)[2],
                                               const RowInfo (&ri)[2], int k0, int c2, float cs) {
  const int kb0 = k0 + c2;
  const bool full = k0 >= max(ri[0].klo, ri[1].klo) && k0 + 8 * NI <= min(ri[0].khi, ri[1].khi);
  float mx[2] = {-3.0e38f, -3.0e38f};
#pragma unroll
  for (int i = 0; i < NI; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int hh = j >> 1, kk = kb0 + 8 * i + (j & 1);
      if (full || (kk >= ri[hh].klo && kk < ri[hh].khi)) mx[hh] = fmaxf(mx[hh], s[4 * i + j]);
    }
  float corr[2], ms[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
    mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
    const float mn = fmaxf(m[hh], mx[hh]);
    corr[hh] = ex2_approx((m[hh] - mn) * cs);
    m[hh] = mn;
    ms[hh] = mn * cs;
    l[hh] *= corr[hh];
  }
#pragma unroll
  for (int i = 0; i < NI; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int hh = j >> 1, kk = kb0 + 8 * i + (j & 1);
      const float p = (full || (kk >= ri[hh].klo && kk < ri[hh].khi)) ? ex2_approx(fmaf(s[4 * i + j], cs, -ms[hh])) : 0.f;
      s[4 * i + j] = p;
      l[hh] += p;
      if (i < NO / 4) o[4 * i + j] *= corr[hh];
    }
}

// O = o / l as bf16 and the natural-log LSE of the scaled scores ([crop, head, token]) for this thread's two rows
// (head_dim = 2 * NO)
template <int NO>
__device__ __forceinline__ void store_o_lse(const float (&o)[NO], float (&l)[2], const float (&m)[2], const RowInfo (&ri)[2],
                                            const AttnShape& sh, int c, int h, int row_base, int wq0, int r_in, int c2,
                                            __nv_bfloat16* O, float* LSE) {
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
    const int q = wq0 + r_in + 8 * hh;
    if (!ri[hh].ok) continue;
    const float inv = 1.f / l[hh];
    __nv_bfloat16* dst = O + (size_t)(row_base + q) * sh.D + h * (2 * NO) + c2;
#pragma unroll
    for (int i = 0; i < NO / 4; ++i)
      *reinterpret_cast<uint32_t*>(dst + 8 * i) = pack_bf16(o[4 * i + 2 * hh] * inv, o[4 * i + 2 * hh + 1] * inv);
    if (LSE && c2 == 0)
      LSE[((size_t)(c * sh.G + ri[hh].g) * sh.H + h) * sh.N + (q - ri[hh].klo)] = m[hh] * sh.scale + logf(l[hh]);
  }
}

// Resident forward: one CTA per (q-tile of 128 rows, head, crop group), two warpgroups of 64 query rows each.  Q and the
// whole key / value range of the group are staged once; each warpgroup walks the keys in blocks of 64: S = Q K^T (SS
// form), online softmax on the accumulator fragment, then O += P V with P handed to the tensor core straight from
// registers (RS form: the accumulator fragment of S is the A-operand fragment of the PV product).
// Shared memory: [Q 128 x 128 B][K nkb x 8 KB][V nkb x 8 KB][barrier].
__host__ __device__ constexpr int fwd_smem(int nkb) { return SMEM_ALIGN + 16384 + 2 * nkb * 8192 + 8; }

__global__ void __launch_bounds__(256)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV,
                __nv_bfloat16* __restrict__ O, float* __restrict__ LSE, const AttnShape sh) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sQ = smem_base_1024(smem_raw);
  uint8_t* sK = sQ + 16384;
  uint8_t* sV = sK + sh.nkb * 8192;
  uint64_t* bar = reinterpret_cast<uint64_t*>(sV + sh.nkb * 8192);

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int qt = blockIdx.x, h = blockIdx.y, c = blockIdx.z;
  const int q0 = qt * 128;
  const int row_base = c * sh.span;  // first token row of this CTA's crop group in [T, ...]
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmKV);
    mbar_init(bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x < 32 && elect_one()) {
    mbar_expect_tx(bar, 16384 + 2 * sh.nkb * 8192);
    tma_load_2d(&tmQ, bar, sQ, h * 64, row_base + q0);
    for (int b = 0; b < sh.nkb; ++b) {
      tma_load_2d(&tmKV, bar, sK + b * 8192, sh.D + h * 64, row_base + b * 64);
      tma_load_2d(&tmKV, bar, sV + b * 8192, 2 * sh.D + h * 64, row_base + b * 64);
    }
  }
  // warpgroups whose 64 query rows all lie beyond the crop group (ragged last tile: 197 = 128 + 69) have nothing to do
  const int wq0 = q0 + wg * 64;
  if (wq0 >= sh.span) return;
  mbar_wait(bar, 0);

  const int r_in = 16 * (t >> 5) + ((t & 31) >> 2), c2 = 2 * (t & 3);
  RowInfo ri[2];
  ri[0] = row_info(sh, c, wq0 + r_in);
  ri[1] = row_info(sh, c, wq0 + r_in + 8);
  // key blocks any row of this warpgroup needs (packed short crops: only the blocks of its own crops)
  const int b_lo = (min(wq0 / sh.N, sh.G - 1) * sh.N) >> 6;
  const int b_hi = min(sh.nkb, ((min(min(wq0 + 63, sh.span - 1) / sh.N, sh.G - 1) + 1) * sh.N + 63) >> 6);
  const float cs = sh.scale * LOG2E;
  float m[2] = {-3.0e38f, -3.0e38f}, l[2] = {0.f, 0.f};
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  const uint64_t qd = gmma_desc_sw128(smem_u32(sQ + wg * 8192), 16, 1024);

#pragma unroll 1
  for (int b = b_lo; b < b_hi; ++b) {
    float s[32];
    const uint64_t kd = gmma_desc_sw128(smem_u32(sK + b * 8192), 16, 1024);
    fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_m64n64k16_ss<0, 0>(s, qd + 2 * k, kd + 2 * k, k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    online_softmax<8>(s, o, m, l, ri, b * 64, c2, cs);
    // ---- O += P V (A = P from registers, B = V block MN-major: 16 keys per k-step = 2048 B)
    uint32_t a[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int e = 0; e < 4; ++e) a[kk][e] = pack_bf16(s[8 * kk + 2 * e], s[8 * kk + 2 * e + 1]);
    const uint64_t vd = gmma_desc_sw128(smem_u32(sV + b * 8192), 8192, 1024);
    fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_m64n64k16_rs<1>(o, a[kk], vd + 128 * kk, 1u);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
  }
  store_o_lse(o, l, m, ri, sh, c, h, row_base, wq0, r_in, c2, O, LSE);
}

// ------------------------------------------------------------------------------------------------ tile ring
// STAGES shared-memory stages of BYTES each, [STAGES x BYTES][full x STAGES][empty x STAGES], filled by TMA from one
// producer thread and read by the consumer warps.  Full barriers count the TMA bytes; empty barriers one arrive per
// consumer warp.  Tile j sits in stage j % STAGES and is that stage's use u = j / STAGES: consumers wait on full parity
// u & 1, the producer waits on empty parity (u - 1) & 1 before every use u >= 1.
template <int STAGES, int BYTES>
struct TileRing {
  static constexpr int SMEM = STAGES * BYTES + 2 * STAGES * 8;   // bytes from the base to end()
  uint8_t* buf;
  uint64_t* full;
  uint64_t* empty;

  __device__ __forceinline__ explicit TileRing(uint8_t* base)
      : buf(base), full(reinterpret_cast<uint64_t*>(base + STAGES * BYTES)), empty(full + STAGES) {}
  __device__ __forceinline__ uint64_t* end() const { return empty + STAGES; }
  // one thread, before the fence_mbar_init / __syncthreads that publish the barriers
  __device__ __forceinline__ void init(int consumer_warps) const {
    for (int st = 0; st < STAGES; ++st) {
      mbar_init(full + st, 1);
      mbar_init(empty + st, consumer_warps);
    }
  }
  // producer thread: tiles 0 .. n-1, load(bar, dst, j) issues the TMA loads of BYTES bytes of tile j into dst
  template <class Load>
  __device__ __forceinline__ void fill(int n, Load load) const {
    for (int j = 0; j < n; ++j) {
      const int st = j % STAGES, u = j / STAGES;
      if (u > 0) mbar_wait(empty + st, (u - 1) & 1);
      mbar_expect_tx(full + st, BYTES);
      load(full + st, buf + st * BYTES, j);
    }
  }
  // consumer: the stage of tile j once it has landed
  __device__ __forceinline__ uint8_t* wait(int j) const {
    mbar_wait(full + j % STAGES, (j / STAGES) & 1);
    return buf + (j % STAGES) * BYTES;
  }
  // consumer warp, converged: it no longer reads the stage of tile j
  __device__ __forceinline__ void release(int j) const {
    if (lane_id() == 0) mbar_arrive(empty + j % STAGES);
  }
};

constexpr int FWD_STAGES = 4, DKDV_STAGES = 3, DQ_STAGES = 4, HD128_STAGES = 2;
constexpr int RING_THREADS = 384;            // two consumer warpgroups + a producer warpgroup (registers: 232 / 40)

// Role split of a ring kernel: warpgroup 2 hands its registers to the consumers and one of its threads runs `produce`
// (the resident loads, then TileRing::fill); true there and in the rest of warpgroup 2, which return.  The consumer
// warpgroups 0 and 1 take 232 registers each and get false.
template <class Produce>
__device__ __forceinline__ bool ring_producer(int wg, Produce produce) {
  if (wg == 2) {
    setmaxnreg_dec<40>();
    if (threadIdx.x < 288 && elect_one()) produce();
    return true;
  }
  setmaxnreg_inc<232>();
  return false;
}

// ------------------------------------------------------------------------------------------------ streamed forward
// One CTA per (128-row query tile, head, crop), G = 1, any N.  The producer loads Q once, then streams every 128-key
// K | V block through the ring (the empty barriers count the consumer warps that have rows in this crop).  Per block each
// consumer warpgroup runs S = Q K^T (m64n128), the resident kernel's online softmax, and O += P V as 8 RS k-steps.
using FwdRing = TileRing<FWD_STAGES, 32768>;                            // K 16 KB | V 16 KB
constexpr int FWD_STREAM_SMEM = SMEM_ALIGN + 16384 + FwdRing::SMEM + 8;   // [Q][ring][q barrier]

__global__ void __launch_bounds__(RING_THREADS, 1)
attn_fwd_stream_kernel(const __grid_constant__ CUtensorMap tmQKV, __nv_bfloat16* __restrict__ O, float* __restrict__ LSE,
                       const AttnShape sh) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sQ = smem_base_1024(smem_raw);
  const FwdRing ring(sQ + 16384);
  uint64_t* bar_q = ring.end();

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int qt = blockIdx.x, h = blockIdx.y, c = blockIdx.z;
  const int q0 = qt * 128, row_base = c * sh.N, nkb = (sh.N + 127) >> 7;
  const int n_wg = (q0 + 64 < sh.N) ? 2 : 1;   // consumer warpgroups with at least one query row of the crop
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQKV);
    ring.init(4 * n_wg);
    mbar_init(bar_q, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (ring_producer(wg, [&] {
        mbar_expect_tx(bar_q, 16384);
        tma_load_2d(&tmQKV, bar_q, sQ, h * 64, row_base + q0);
        ring.fill(nkb, [&](uint64_t* bar, uint8_t* dst, int b) {
          tma_load_2d(&tmQKV, bar, dst, sh.D + h * 64, row_base + b * 128);
          tma_load_2d(&tmQKV, bar, dst + 16384, 2 * sh.D + h * 64, row_base + b * 128);
        });
      }))
    return;
  const int wq0 = q0 + wg * 64;
  if (wq0 >= sh.N) return;                     // not counted by the empty barriers (n_wg)
  mbar_wait(bar_q, 0);

  const int r_in = 16 * (t >> 5) + ((t & 31) >> 2), c2 = 2 * (t & 3);
  RowInfo ri[2];
  ri[0] = row_info(sh, c, wq0 + r_in);
  ri[1] = row_info(sh, c, wq0 + r_in + 8);
  const float cs = sh.scale * LOG2E;
  float m[2] = {-3.0e38f, -3.0e38f}, l[2] = {0.f, 0.f};
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  const uint64_t qd = gmma_desc_sw128(smem_u32(sQ + wg * 8192), 16, 1024);

#pragma unroll 1
  for (int b = 0; b < nkb; ++b) {
    const uint8_t* sK = ring.wait(b);
    float s[64];
    const uint64_t kd = gmma_desc_sw128(smem_u32(sK), 16, 1024);
    fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_m64n128k16_ss<0, 0>(s, qd + 2 * k, kd + 2 * k, k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    online_softmax<16>(s, o, m, l, ri, b * 128, c2, cs);
    uint32_t a[8][4];
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)
#pragma unroll
      for (int e = 0; e < 4; ++e) a[kk][e] = pack_bf16(s[8 * kk + 2 * e], s[8 * kk + 2 * e + 1]);
    const uint64_t vd = gmma_desc_sw128(smem_u32(sK + 16384), 8192, 1024);   // V MN-major: 16 keys per k-step
    fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) wgmma_m64n64k16_rs<1>(o, a[kk], vd + 128 * kk, 1u);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
    ring.release(b);
  }
  store_o_lse(o, l, m, ri, sh, c, h, row_base, wq0, r_in, c2, O, LSE);
}

// Delta[c,h,q] = sum_d dO[q, h, d] * O[q, h, d]    (backward softmax term)
template <int HD>
__global__ void attn_delta_kernel(const __nv_bfloat16* __restrict__ O, const __nv_bfloat16* __restrict__ dO,
                                  float* __restrict__ delta, long T, int N, int D, int H) {
  // HD / 8 threads per (row, head): one 16-byte load of O and of dO each, log2(HD / 8) shuffle steps inside the group
  constexpr int LANES = HD / 8;
  static_assert(LANES == 8 || LANES == 16, "head_dim 64 or 128");
  const long g = blockIdx.x * (long)blockDim.x + threadIdx.x;
  const int per_row = D >> 3;
  const bool ok = g < T * per_row;
  float s = 0.f;
  long row = 0;
  int c8 = 0;
  if (ok) {
    row = g / per_row;
    c8 = (int)(g % per_row);
    const uint4 a = *reinterpret_cast<const uint4*>(O + row * D + c8 * 8);
    const uint4 b = *reinterpret_cast<const uint4*>(dO + row * D + c8 * 8);
    const float2 a0 = unpack_bf16(a.x), a1 = unpack_bf16(a.y), a2 = unpack_bf16(a.z), a3 = unpack_bf16(a.w);
    const float2 b0 = unpack_bf16(b.x), b1 = unpack_bf16(b.y), b2 = unpack_bf16(b.z), b3 = unpack_bf16(b.w);
    s = a0.x * b0.x + a0.y * b0.y + a1.x * b1.x + a1.y * b1.y + a2.x * b2.x + a2.y * b2.y + a3.x * b3.x + a3.y * b3.y;
  }
  if (LANES == 16) s += __shfl_xor_sync(0xffffffffu, s, 8);
  s += __shfl_xor_sync(0xffffffffu, s, 4);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  if (ok && (c8 & (LANES - 1)) == 0) delta[((row / N) * H + (c8 >> (LANES == 16 ? 4 : 3))) * N + (row % N)] = s;
}

// ------------------------------------------------------------------------------------------------ backward
// For a 128-query x 128-key tile pair:
//   S  = Q K^T, dP = dO V^T,  P = exp(S*scale - lse),  dS = P * (dP - Delta) * scale
//   dV += P^T dO, dK += dS^T Q, dQ += dS K
// Crop groups of span <= 256 take attn_bwd_fused_kernel (all of it in one pass); longer crops the streamed pair below,
// which shares the helpers p_ds_tile / stash_p_ds / dkdv_mma / dq_mma.
// inverse RoPE on the gradient: transpose of y = x*cos + rot_half(x)*sin (dinov3_jax/layers/attention.py:14-20); this
// thread holds columns d = 8i + c2 + {0,1} of a row, i.e. both partners (d, d + head_dim / 2) of every rotation pair it
// touches.  head_dim = 2 * NA; the tables are [P, head_dim].
template <int NA>
__device__ __forceinline__ void store_grad_rows(float (&a)[NA], const AttnShape& sh, int c, int row_base, int tile_row0,
                                                int r_in, int c2, int h, int third, bool rope, __nv_bfloat16* dQKV) {
  constexpr int HD = 2 * NA;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int row = tile_row0 + r_in + 8 * hh;
    const RowInfo ri = row_info(sh, c, row);
    if (!ri.ok) continue;
    const int tok = row - ri.klo;
    float v[NA / 2];
#pragma unroll
    for (int i = 0; i < NA / 4; ++i) { v[2 * i] = a[4 * i + 2 * hh]; v[2 * i + 1] = a[4 * i + 2 * hh + 1]; }
    if (rope && sh.sin_t && tok >= sh.prefix) {
      const float* sn = sh.sin_t + (size_t)(tok - sh.prefix) * HD;
      const float* cn = sh.cos_t + (size_t)(tok - sh.prefix) * HD;
#pragma unroll
      for (int i = 0; i < NA / 8; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int d = 8 * i + c2 + j;
          const float lo = v[2 * i + j], hi = v[2 * (i + NA / 8) + j];
          v[2 * i + j] = lo * cn[d] + hi * sn[d];
          v[2 * (i + NA / 8) + j] = hi * cn[d] - lo * sn[d];
        }
    }
    __nv_bfloat16* dst = dQKV + (size_t)(row_base + row) * (3 * sh.D) + third * sh.D + h * HD + c2;
#pragma unroll
    for (int i = 0; i < NA / 4; ++i) *reinterpret_cast<uint32_t*>(dst + 8 * i) = pack_bf16(v[2 * i], v[2 * i + 1]);
  }
}

// lse * log2(e) and Delta of token row q of the crop group (0 for rows outside it)
__device__ __forceinline__ void row_stats(const AttnShape& sh, const float* __restrict__ LSE, const float* __restrict__ Delta,
                                          int c, int h, int q, float& lse2, float& dl) {
  const RowInfo ri = row_info(sh, c, q);
  const size_t stat = ((size_t)(c * sh.G + ri.g) * sh.H + h) * sh.N + (ri.ok ? q - ri.klo : 0);
  lse2 = ri.ok ? LSE[stat] * LOG2E : 0.f;
  dl = ri.ok ? Delta[stat] : 0.f;
}

// S and dP of one warpgroup's 64 query rows (first row q0 of the crop group, tiles sQw / sDOw: 64 rows x 128 B) against
// the 128-key tile kt (sK, sV), turned into P (in s) and dS (in dp).  Keys outside a row's crop and rows outside the group
// give exactly 0.
__device__ __forceinline__ void p_ds_tile(const AttnShape& sh, const float* __restrict__ LSE, const float* __restrict__ Delta,
                                          int c, int h, int q0, int kt, const uint8_t* sQw, const uint8_t* sDOw,
                                          const uint8_t* sK, const uint8_t* sV, int r_in, int c2, float (&s)[64],
                                          float (&dp)[64]) {
  const float cs = sh.scale * LOG2E;
  const uint64_t qd = gmma_desc_sw128(smem_u32(sQw), 16, 1024);
  const uint64_t dod = gmma_desc_sw128(smem_u32(sDOw), 16, 1024);
  const uint64_t kd = gmma_desc_sw128(smem_u32(sK), 16, 1024);
  const uint64_t vd = gmma_desc_sw128(smem_u32(sV), 16, 1024);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k) {   // S and dP are independent accumulator chains: interleave them
    wgmma_m64n128k16_ss<0, 0>(s, qd + 2 * k, kd + 2 * k, k > 0 ? 1u : 0u);
    wgmma_m64n128k16_ss<0, 0>(dp, dod + 2 * k, vd + 2 * k, k > 0 ? 1u : 0u);
  }
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(s);
  fence_regs(dp);
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int q = q0 + r_in + 8 * hh;
    const RowInfo ri = row_info(sh, c, q);
    float lse2, dl;
    row_stats(sh, LSE, Delta, c, h, q, lse2, dl);
    const int lo = ri.ok ? ri.klo - kt * 128 : 0, hi = ri.ok ? ri.khi - kt * 128 : 0;   // valid key columns
#pragma unroll
    for (int i = 0; i < 16; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int e = 4 * i + 2 * hh + j, col = 8 * i + c2 + j;
        const bool ok = col >= lo && col < hi;
        const float p = ok ? ex2_approx(fmaf(s[e], cs, -lse2)) : 0.f;
        dp[e] = ok ? (p * sh.scale) * (dp[e] - dl) : 0.f;
        s[e] = p;
      }
  }
}

// P and dS of this thread's rows `row`, `row + 8` of the 128-row query tile into bf16 SWIZZLE_128B tiles
// [2 chunks of 64 keys][128 q x 128 B] (sP, sDS), read back MN-major by dkdv_mma
__device__ __forceinline__ void stash_p_ds(const float (&s)[64], const float (&dp)[64], uint8_t* sP, uint8_t* sDS, int row,
                                           int c2) {
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const uint32_t off = (i >> 3) * 16384 + sw128_offset(row + 8 * hh, (8 * i + c2) & 63);
      *reinterpret_cast<uint32_t*>(sP + off) = pack_bf16(s[4 * i + 2 * hh], s[4 * i + 2 * hh + 1]);
      *reinterpret_cast<uint32_t*>(sDS + off) = pack_bf16(dp[4 * i + 2 * hh], dp[4 * i + 2 * hh + 1]);
    }
  }
}

// dV[keys, 64] += P^T dO ; dK[keys, 64] += dS^T Q over the 128 query rows of one tile (sDOt, sQt), for this warpgroup's
// 64 keys (A MN-major: 16 query rows per k-step = 2048 B)
__device__ __forceinline__ void dkdv_mma(float (&dk)[32], float (&dv)[32], const uint8_t* sP, const uint8_t* sDS,
                                         const uint8_t* sDOt, const uint8_t* sQt, int wg) {
  const uint64_t pd = gmma_desc_sw128(smem_u32(sP + wg * 16384), 16384, 1024);
  const uint64_t sd = gmma_desc_sw128(smem_u32(sDS + wg * 16384), 16384, 1024);
  const uint64_t dod = gmma_desc_sw128(smem_u32(sDOt), 8192, 1024);
  const uint64_t qd = gmma_desc_sw128(smem_u32(sQt), 8192, 1024);
  fence_regs(dk);
  fence_regs(dv);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    wgmma_m64n64k16_ss<1, 1>(dv, pd + 128 * k, dod + 128 * k, 1u);
    wgmma_m64n64k16_ss<1, 1>(dk, sd + 128 * k, qd + 128 * k, 1u);
  }
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(dk);
  fence_regs(dv);
}

// dQ += dS K over one 128-key tile, dS straight from registers (RS form), K as MN-major B (keys x d)
__device__ __forceinline__ void dq_mma(float (&dq)[32], const float (&dp)[64], const uint8_t* sK) {
  uint32_t a[8][4];
#pragma unroll
  for (int kk = 0; kk < 8; ++kk)
#pragma unroll
    for (int e = 0; e < 4; ++e) a[kk][e] = pack_bf16(dp[8 * kk + 2 * e], dp[8 * kk + 2 * e + 1]);
  const uint64_t kd = gmma_desc_sw128(smem_u32(sK), 8192, 1024);
  fence_regs(dq);
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) wgmma_m64n64k16_rs<1>(dq, a[kk], kd + 128 * kk, 1u);
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(dq);
}

// One CTA per (head, crop group) for span <= 256, two warpgroups.  At most two 128-row tiles: every Q / dO / K / V tile
// stays resident, and one thread issues all their TMA loads at the start (one mbarrier per tile, so the first pair
// starts as soon as it has landed and the rest arrives under it; a producer warpgroup would have nothing left to do).
// dK, dV and dQ come out of one pass over the tile pairs (kt outer, qt inner), keys on the accumulator rows: warpgroup w
// owns keys kt*128 + w*64 .. + 63 and, for each half of 64 query columns,
//   S^T = K Q^T, dP^T = V dO^T                                 (SS, m64n64: registers)
//   P^T = exp(S^T*scale - lse), dS^T = P^T * (dP^T - Delta) * scale   (LSE / Delta per query column, staged in smem)
//   dV += P^T dO, dK += dS^T Q                                  (RS: the fragments of P^T / dS^T are the A operands)
// and stashes its dS^T as bf16 (MN-major for the dQ product).  After a named barrier, warpgroup w computes
//   dQ[qt rows w*64 ..] += dS K over all 128 keys of the tile  (SS, A = the stash read MN-major)
// as one accumulation chain per query tile, no atomics.  The chains run over the key tiles in a fixed order, the one
// the two-phase backward before this kernel used, so that training runs keep their bits: query tile 1 ascending (its
// partial sum after key tile 0 waits in shared memory as fp32), query tile 0 from the last key tile down (the stash of
// pair (0, 0) is kept and its products are issued after those of pair (1, 0)).
// Five tile products per pair and one ex2 per score; 244 registers, no spills.  Shared memory at span 256: K/V 64 KB,
// Q/dO 64 KB, two stashes 64 KB, dQ partial sum 32 KB, LSE / Delta 2 KB (one CTA per SM).

// bytes of dynamic shared memory for n_t 128-row tiles (layout in attn_bwd_fused_kernel)
__host__ __device__ constexpr int bwd_fused_smem(int n_t) {
  return n_t * 32768 * 2 + 32768 + (n_t > 1 ? 2 * 32768 : 0) + n_t * 128 * 8 + 2 * n_t * 8;
}

// descriptor of a tile computed where it is used: loop-invariant descriptors (and their per-k-step offsets) would
// otherwise be hoisted out of the tile loops and held in registers across the whole pass
__device__ __forceinline__ uint64_t desc_here(const void* p, uint32_t lbo, uint32_t sbo) {
  uint32_t a;
  asm volatile("mov.b32 %0, %1;" : "=r"(a) : "r"(smem_u32(p)));
  return gmma_desc_sw128(a, lbo, sbo);
}

// registers of the RS A fragments stay untouched until the wgmma reading them has completed
template <int R>
__device__ __forceinline__ void fence_frag(uint32_t (&a)[R][4]) {
#pragma unroll
  for (int i = 0; i < R; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) asm volatile("" : "+r"(a[i][e])::"memory");
}

__global__ void __launch_bounds__(256, 1)
attn_bwd_fused_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmDO,
                      const float* __restrict__ LSE, const float* __restrict__ Delta, __nv_bfloat16* __restrict__ dQKV,
                      const AttnShape sh) {
  // no round-up of the base as in the other kernels: span 256 leaves under 1 KB of the 227 KB opt-in, so the window's
  // own 1 KB alignment (requested here) is what the SWIZZLE_128B tiles rely on
  extern __shared__ __align__(1024) uint8_t smem_al[];
  const int nT = (sh.span + 127) / 128;
  uint8_t* sKV = smem_al;                       // [nT][K 16 KB | V 16 KB]
  uint8_t* sQDO = sKV + nT * 32768;             // [nT][Q 16 KB | dO 16 KB]
  uint8_t* sDS = sQDO + nT * 32768;             // dS^T of one tile pair: [2 chunks of 64 q][128 keys x 128 B]
  uint8_t* sDS0 = sDS + 32768;                  // nT = 2: dS^T of pair (0, 0), kept until pair (1, 0)
  float* sDQ = reinterpret_cast<float*>(sDS0 + 32768);   // nT = 2: dQ of query tile 1 after key tile 0, [2 wg][8][128][4]
  float* sLSE = reinterpret_cast<float*>(sDS + (nT > 1 ? 3 * 32768 : 32768));   // [nT * 128] lse * log2(e) per query row
  float* sDel = sLSE + nT * 128;                 // [nT * 128]
  uint64_t* bar_kv = reinterpret_cast<uint64_t*>(sDel + nT * 128);
  uint64_t* bar_q = bar_kv + nT;

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int r_in = 16 * (t >> 5) + ((t & 31) >> 2), c2 = 2 * (t & 3);
  const int h = blockIdx.x, c = blockIdx.y;
  const int row_base = c * sh.span;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQKV);
    tma_prefetch_desc(&tmDO);
    for (int i = 0; i < 2 * nT; ++i) mbar_init(bar_kv + i, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x < 32 && elect_one()) {
    for (int i = 0; i < nT; ++i) {             // K/V 0, Q/dO 0, then the second tiles: the first pair starts early
      mbar_expect_tx(bar_kv + i, 32768);
      tma_load_2d(&tmQKV, bar_kv + i, sKV + i * 32768, sh.D + h * 64, row_base + i * 128);
      tma_load_2d(&tmQKV, bar_kv + i, sKV + i * 32768 + 16384, 2 * sh.D + h * 64, row_base + i * 128);
      mbar_expect_tx(bar_q + i, 32768);
      tma_load_2d(&tmQKV, bar_q + i, sQDO + i * 32768, h * 64, row_base + i * 128);
      tma_load_2d(&tmDO, bar_q + i, sQDO + i * 32768 + 16384, h * 64, row_base + i * 128);
    }
  }
  for (int q = threadIdx.x; q < nT * 128; q += 256) {   // row_stats without its clamp of the index of rows outside the group
    const RowInfo ri = row_info(sh, c, q);
    const size_t stat = ((size_t)(c * sh.G + ri.g) * sh.H + h) * sh.N + (q - ri.klo);
    sLSE[q] = ri.ok ? LSE[stat] * LOG2E : 0.f;
    sDel[q] = ri.ok ? Delta[stat] : 0.f;
  }
  __syncthreads();

  const float cs = sh.scale * LOG2E;
  int pair = 0;
#pragma unroll 1
  for (int kt = 0; kt < nT; ++kt) {
    mbar_wait(bar_kv + kt, 0);
    const uint8_t* sK = sKV + kt * 32768;
    const uint8_t* sV = sK + 16384;
    // valid query columns of this thread's two key rows: the key's own crop (none for keys outside the group)
    int lo[2], hi[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const RowInfo ri = row_info(sh, c, kt * 128 + wg * 64 + r_in + 8 * hh);
      lo[hh] = ri.ok ? ri.klo : 0;
      hi[hh] = ri.ok ? ri.khi : 0;
    }
    float dk[32], dv[32];
#pragma unroll 1
    for (int qt = 0; qt < nT; ++qt, ++pair) {
      mbar_wait(bar_q + qt, 0);
      const uint8_t* sQt = sQDO + qt * 32768;
      const uint8_t* sDOt = sQt + 16384;
      const bool defer = nT == 2 && kt == 0 && qt == 0;   // dQ of query tile 0 starts with key tile 1
      uint8_t* stash = defer ? sDS0 : sDS;
      // the 128 query columns in two halves of 64: S^T / dP^T of one half (64 registers) at a time, so that the
      // accumulators, the fragments of the half still being read by its RS products and the scores fit without spills
      uint32_t pa[2][4][4], da[2][4][4];   // bf16 A fragments of P^T / dS^T (k-step kk: query columns 16 kk ..)
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        float s[32], dp[32];
        {
          const uint64_t kd = desc_here(sK + wg * 8192, 16, 1024);
          const uint64_t vd = desc_here(sV + wg * 8192, 16, 1024);
          const uint64_t qd = desc_here(sQt + hf * 8192, 16, 1024);
          const uint64_t dod = desc_here(sDOt + hf * 8192, 16, 1024);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            wgmma_m64n64k16_ss<0, 0>(s, kd + 2 * k, qd + 2 * k, k > 0 ? 1u : 0u);
            wgmma_m64n64k16_ss<0, 0>(dp, vd + 2 * k, dod + 2 * k, k > 0 ? 1u : 0u);
          }
          wgmma_commit();
          wgmma_wait<0>();        // also retires the first half's RS products
          fence_regs(s);
          fence_regs(dp);
          if (hf == 1) { fence_frag(pa[0]); fence_frag(da[0]); }
        }
        const float* lse2 = sLSE + qt * 128 + hf * 64;
        const float* del = sDel + qt * 128 + hf * 64;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int col = 8 * i + c2;
          const float2 l2 = *reinterpret_cast<const float2*>(lse2 + col);
          const float2 dl = *reinterpret_cast<const float2*>(del + col);
          const int q = qt * 128 + hf * 64 + col;
          float pv[4], dv4[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int hh = j >> 1, qq = q + (j & 1);
            const bool ok = qq >= lo[hh] && qq < hi[hh];
            const float p = ok ? ex2_approx(fmaf(s[4 * i + j], cs, -((j & 1) ? l2.y : l2.x))) : 0.f;
            dv4[j] = ok ? (p * sh.scale) * (dp[4 * i + j] - ((j & 1) ? dl.y : dl.x)) : 0.f;
            pv[j] = p;
          }
          pa[hf][i >> 1][2 * (i & 1)] = pack_bf16(pv[0], pv[1]);
          pa[hf][i >> 1][2 * (i & 1) + 1] = pack_bf16(pv[2], pv[3]);
          da[hf][i >> 1][2 * (i & 1)] = pack_bf16(dv4[0], dv4[1]);
          da[hf][i >> 1][2 * (i & 1) + 1] = pack_bf16(dv4[2], dv4[3]);
        }
        // the dQ products of the previous pair (both warpgroups) have finished reading the stash (pairs 0 and 1 of
        // nT = 2 write different stashes)
        if (hf == 0 && pair > 1) named_bar_sync(1, 256);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
          for (int i = 0; i < 8; ++i) {   // chunk hf of the stash holds query columns hf * 64 ..
            const uint32_t off = hf * 16384 + sw128_offset(wg * 64 + r_in + 8 * hh, 8 * i + c2);
            *reinterpret_cast<uint32_t*>(stash + off) = da[hf][i >> 1][2 * (i & 1) + hh];
          }
        {
          const uint64_t dod = desc_here(sDOt, 8192, 1024);   // B MN-major: 16 query rows per k-step
          const uint64_t qd = desc_here(sQt, 8192, 1024);
          const uint32_t acc_on = (qt > 0 || hf > 0) ? 1u : 0u;
          if (acc_on) { fence_regs(dk); fence_regs(dv); }
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            const int ks = 4 * hf + kk;
            wgmma_m64n64k16_rs<1>(dv, pa[hf][kk], dod + 128 * ks, (acc_on || kk > 0) ? 1u : 0u);
            wgmma_m64n64k16_rs<1>(dk, da[hf][kk], qd + 128 * ks, (acc_on || kk > 0) ? 1u : 0u);
          }
          wgmma_commit();
        }
      }
      fence_proxy_async_smem();   // generic-proxy smem writes (the stash) -> visible to the tensor core (async proxy)
      if (defer) {                // pair (1, 0) reads this stash; only the RS products remain to retire
        wgmma_wait<0>();
        fence_regs(dk);
        fence_regs(dv);
        fence_frag(pa[1]);
        fence_frag(da[1]);
        continue;
      }
      named_bar_sync(2, 256);     // both halves of dS^T are in the stash
      const bool from_partial = nT == 2 && kt == 1 && qt == 1;
      float dq[32];
      float4* part = reinterpret_cast<float4*>(sDQ) + wg * 8 * 128 + t;
      if (from_partial) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float4 v = part[j * 128];
          dq[4 * j] = v.x; dq[4 * j + 1] = v.y; dq[4 * j + 2] = v.z; dq[4 * j + 3] = v.w;
        }
      }
      {
        const uint64_t sd = desc_here(sDS + wg * 16384, 16384, 1024);   // A MN-major: 16 keys per k-step
        const uint64_t kbd = desc_here(sK, 8192, 1024);                 // B MN-major
        fence_regs(dq);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 8; ++kk)
          wgmma_m64n64k16_ss<1, 1>(dq, sd + 128 * kk, kbd + 128 * kk, (from_partial || kk > 0) ? 1u : 0u);
        if (nT == 2 && kt == 1 && qt == 0) {   // then key tile 0, from the kept stash of pair (0, 0)
          const uint64_t sd0 = desc_here(sDS0 + wg * 16384, 16384, 1024);
          const uint64_t k0d = desc_here(sKV, 8192, 1024);
#pragma unroll
          for (int kk = 0; kk < 8; ++kk) wgmma_m64n64k16_ss<1, 1>(dq, sd0 + 128 * kk, k0d + 128 * kk, 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(dq);
        fence_regs(dk);
        fence_regs(dv);
        fence_frag(pa[1]);
        fence_frag(da[1]);
      }
      if (nT == 2 && kt == 0) {
#pragma unroll
        for (int j = 0; j < 8; ++j) part[j * 128] = make_float4(dq[4 * j], dq[4 * j + 1], dq[4 * j + 2], dq[4 * j + 3]);
      } else {
        store_grad_rows(dq, sh, c, row_base, qt * 128 + wg * 64, r_in, c2, h, 0, true, dQKV);
      }
    }
    store_grad_rows(dk, sh, c, row_base, kt * 128 + wg * 64, r_in, c2, h, 1, true, dQKV);
    store_grad_rows(dv, sh, c, row_base, kt * 128 + wg * 64, r_in, c2, h, 2, false, dQKV);
  }
}

// ------------------------------------------------------------------------------------------------ streamed backward
// Any N, G = 1, as two grids that each write their outputs once, with every sum in ascending tile order (no atomics):
//   dK / dV: one CTA per (128-key tile, head, crop).  K / V stay resident; the query tiles' Q / dO stream through a ring
//            of DKDV_STAGES stages.  Per query tile: p_ds_tile, P and dS staged in shared memory, dkdv_mma (the resident
//            kernel's phase 1).
//   dQ:      one CTA per (128-row query tile, head, crop).  Q / dO stay resident; K / V stream through a ring of DQ_STAGES
//            stages.  Per key tile: p_ds_tile, dq_mma (the resident kernel's phase 2).
// Warpgroup 2 is the producer of the TileRing.
using DkdvRing = TileRing<DKDV_STAGES, 32768>;                                  // Q 16 KB | dO 16 KB
constexpr int DKDV_SMEM = SMEM_ALIGN + 2 * 16384 + 2 * 32768 + DkdvRing::SMEM + 8;   // [K][V][P][dS][ring][kv barrier]
using DqRing = TileRing<DQ_STAGES, 32768>;                                      // K 16 KB | V 16 KB
constexpr int DQ_SMEM = SMEM_ALIGN + 2 * 16384 + DqRing::SMEM + 8;                 // [Q][dO][ring][q barrier]

__global__ void __launch_bounds__(RING_THREADS, 1)
attn_bwd_dkdv_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmDO,
                     const float* __restrict__ LSE, const float* __restrict__ Delta, __nv_bfloat16* __restrict__ dQKV,
                     const AttnShape sh) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sK = smem_base_1024(smem_raw);      // 16 KB
  uint8_t* sV = sK + 16384;                    // 16 KB
  uint8_t* sP = sV + 16384;                    // 32 KB
  uint8_t* sDS = sP + 32768;                   // 32 KB
  const DkdvRing ring(sDS + 32768);
  uint64_t* bar_kv = ring.end();

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int r_in = 16 * (t >> 5) + ((t & 31) >> 2), c2 = 2 * (t & 3);
  const int kt = blockIdx.x, h = blockIdx.y, c = blockIdx.z;
  const int row_base = c * sh.N, nq = (sh.N + 127) >> 7;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQKV);
    tma_prefetch_desc(&tmDO);
    ring.init(8);                              // both consumer warpgroups read every query tile
    mbar_init(bar_kv, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (ring_producer(wg, [&] {
        mbar_expect_tx(bar_kv, 32768);
        tma_load_2d(&tmQKV, bar_kv, sK, sh.D + h * 64, row_base + kt * 128);
        tma_load_2d(&tmQKV, bar_kv, sV, 2 * sh.D + h * 64, row_base + kt * 128);
        ring.fill(nq, [&](uint64_t* bar, uint8_t* dst, int qt) {
          tma_load_2d(&tmQKV, bar, dst, h * 64, row_base + qt * 128);
          tma_load_2d(&tmDO, bar, dst + 16384, h * 64, row_base + qt * 128);
        });
      }))
    return;
  mbar_wait(bar_kv, 0);
  float dk[32], dv[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) { dk[i] = 0.f; dv[i] = 0.f; }
#pragma unroll 1
  for (int qt = 0; qt < nq; ++qt) {
    const uint8_t* sQt = ring.wait(qt);
    const uint8_t* sDOt = sQt + 16384;
    float s[64], dp[64];
    p_ds_tile(sh, LSE, Delta, c, h, qt * 128 + wg * 64, kt, sQt + wg * 8192, sDOt + wg * 8192, sK, sV, r_in, c2, s, dp);
    stash_p_ds(s, dp, sP, sDS, wg * 64 + r_in, c2);
    fence_proxy_async_smem();
    named_bar_sync(1, 256);                    // the consumer warpgroups only: P / dS of all 128 query rows are staged
    dkdv_mma(dk, dv, sP, sDS, sDOt, sQt, wg);
    ring.release(qt);
    named_bar_sync(1, 256);                    // both are done reading sP / sDS before the next tile rewrites them
  }
  store_grad_rows(dk, sh, c, row_base, kt * 128 + wg * 64, r_in, c2, h, 1, true, dQKV);
  store_grad_rows(dv, sh, c, row_base, kt * 128 + wg * 64, r_in, c2, h, 2, false, dQKV);
}

__global__ void __launch_bounds__(RING_THREADS, 1)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmDO,
                   const float* __restrict__ LSE, const float* __restrict__ Delta, __nv_bfloat16* __restrict__ dQKV,
                   const AttnShape sh) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sQ = smem_base_1024(smem_raw);      // 16 KB
  uint8_t* sDO = sQ + 16384;                   // 16 KB
  const DqRing ring(sDO + 16384);
  uint64_t* bar_q = ring.end();

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int r_in = 16 * (t >> 5) + ((t & 31) >> 2), c2 = 2 * (t & 3);
  const int qt = blockIdx.x, h = blockIdx.y, c = blockIdx.z;
  const int q0 = qt * 128, row_base = c * sh.N, nk = (sh.N + 127) >> 7;
  const int n_wg = (q0 + 64 < sh.N) ? 2 : 1;   // consumer warpgroups with at least one query row of the crop
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQKV);
    tma_prefetch_desc(&tmDO);
    ring.init(4 * n_wg);
    mbar_init(bar_q, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (ring_producer(wg, [&] {
        mbar_expect_tx(bar_q, 32768);
        tma_load_2d(&tmQKV, bar_q, sQ, h * 64, row_base + q0);
        tma_load_2d(&tmDO, bar_q, sDO, h * 64, row_base + q0);
        ring.fill(nk, [&](uint64_t* bar, uint8_t* dst, int kt) {
          tma_load_2d(&tmQKV, bar, dst, sh.D + h * 64, row_base + kt * 128);
          tma_load_2d(&tmQKV, bar, dst + 16384, 2 * sh.D + h * 64, row_base + kt * 128);
        });
      }))
    return;
  const int wq0 = q0 + wg * 64;
  if (wq0 >= sh.N) return;                     // not counted by the empty barriers (n_wg)
  mbar_wait(bar_q, 0);
  float dq[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dq[i] = 0.f;
#pragma unroll 1
  for (int kt = 0; kt < nk; ++kt) {
    const uint8_t* sK = ring.wait(kt);
    float s[64], dp[64];
    p_ds_tile(sh, LSE, Delta, c, h, wq0, kt, sQ + wg * 8192, sDO + wg * 8192, sK, sK + 16384, r_in, c2, s, dp);
    dq_mma(dq, dp, sK);
    ring.release(kt);
  }
  store_grad_rows(dq, sh, c, row_base, wq0, r_in, c2, h, 0, true, dQKV);
}

// ------------------------------------------------------------------------------------------------ head_dim 128
// ViT-7B (embed 4096, 32 heads).  A 128-row x 128-column bf16 tile is two 64-column SWIZZLE_128B chunks of 16 KB (one TMA
// box each, chunk j at +16 KB): K-major operands walk 8 k16 steps, 4 per chunk; the MN-major B operands of the P V,
// P^T dO, dS^T Q and dS K products span both chunks with N = 128 (LBO = 16 KB).  Three kernels serve every N up to
// ATTN_MAX_TOKENS and every packing of attn_shape: one CTA owns a crop group of span = G * N rows, short crops keep the
// block-diagonal mask of row_info.  Each has the streamed kernels' producer warpgroup and TileRing, with HD128_STAGES
// stages of two 32 KB tiles (K | V or Q | dO):
//   forward  one CTA per (128-row query tile, head, crop group), Q resident.  Per 128-key tile and consumer warpgroup:
//            S = Q K^T (m64n128), online softmax, O += P V (RS m64n128, 8 k-steps).  Scores and O: 64 + 64 registers.
//   dK / dV  one CTA per (128-key tile, head, crop group), K / V resident, Q / dO stream.  Keys on the accumulator rows
//            as in attn_bwd_fused_kernel; per 32 query columns: S^T = K Q^T and dP^T = V dO^T (m64n32), then
//            dV += P^T dO and dK += dS^T Q (RS m64n128).  dK + dV take 128 registers, the scores 32.
//   dQ       one CTA per (128-row query tile, head, crop group), Q / dO resident, K / V stream.  Per half of 64 keys:
//            S and dP (m64n64), dQ += dS K (RS m64n128).
// Every output row is written once by one CTA and every sum runs over the tiles in ascending order: no atomics, the
// same bits on every run.  Shared memory: 32 KB (forward) or 64 KB (backward) resident, the ring, its barrier.
using Hd128Ring = TileRing<HD128_STAGES, 65536>;
constexpr int HD128_FWD_SMEM = SMEM_ALIGN + 32768 + Hd128Ring::SMEM + 8;
constexpr int HD128_BWD_SMEM = SMEM_ALIGN + 65536 + Hd128Ring::SMEM + 8;

// K-major descriptor of k16 step k (0..7) of a 128-column tile whose first chunk (at the operand's first row) is p
__device__ __forceinline__ uint64_t kdesc128(const uint8_t* p, int k) {
  return gmma_desc_sw128(smem_u32(p + (k >> 2) * 16384), 16, 1024) + 2 * (k & 3);
}

// 128 rows x 128 columns starting at column `col`: two 64-column boxes
__device__ __forceinline__ void tma_load_tile128(const CUtensorMap* m, uint64_t* bar, uint8_t* dst, int col, int row) {
  tma_load_2d(m, bar, dst, col, row);
  tma_load_2d(m, bar, dst + 16384, col + 64, row);
}

__global__ void __launch_bounds__(RING_THREADS, 1)
attn_fwd_hd128_kernel(const __grid_constant__ CUtensorMap tmQKV, __nv_bfloat16* __restrict__ O, float* __restrict__ LSE,
                      const AttnShape sh) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sQ = smem_base_1024(smem_raw);      // [Q 32 KB][ring][q barrier]
  const Hd128Ring ring(sQ + 32768);
  uint64_t* bar_q = ring.end();

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int qt = blockIdx.x, h = blockIdx.y, c = blockIdx.z;
  const int q0 = qt * 128, row_base = c * sh.span, nkb = (sh.span + 127) >> 7;
  const int n_wg = (q0 + 64 < sh.span) ? 2 : 1;   // consumer warpgroups with at least one query row in the group
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQKV);
    ring.init(4 * n_wg);
    mbar_init(bar_q, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (ring_producer(wg, [&] {
        mbar_expect_tx(bar_q, 32768);
        tma_load_tile128(&tmQKV, bar_q, sQ, h * 128, row_base + q0);
        ring.fill(nkb, [&](uint64_t* bar, uint8_t* dst, int b) {
          tma_load_tile128(&tmQKV, bar, dst, sh.D + h * 128, row_base + b * 128);
          tma_load_tile128(&tmQKV, bar, dst + 32768, 2 * sh.D + h * 128, row_base + b * 128);
        });
      }))
    return;
  const int wq0 = q0 + wg * 64;
  if (wq0 >= sh.span) return;                  // not counted by the empty barriers (n_wg)
  mbar_wait(bar_q, 0);

  const int r_in = 16 * (t >> 5) + ((t & 31) >> 2), c2 = 2 * (t & 3);
  RowInfo ri[2];
  ri[0] = row_info(sh, c, wq0 + r_in);
  ri[1] = row_info(sh, c, wq0 + r_in + 8);
  const float cs = sh.scale * LOG2E;
  float m[2] = {-3.0e38f, -3.0e38f}, l[2] = {0.f, 0.f};
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;

#pragma unroll 1
  for (int b = 0; b < nkb; ++b) {
    const uint8_t* sK = ring.wait(b);
    float s[64];
    fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 8; ++k)
      wgmma_m64n128k16_ss<0, 0>(s, kdesc128(sQ + wg * 8192, k), kdesc128(sK, k), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    online_softmax<16>(s, o, m, l, ri, b * 128, c2, cs);
    uint32_t a[8][4];
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)
#pragma unroll
      for (int e = 0; e < 4; ++e) a[kk][e] = pack_bf16(s[8 * kk + 2 * e], s[8 * kk + 2 * e + 1]);
    const uint64_t vd = desc_here(sK + 32768, 16384, 1024);   // V MN-major: 16 keys per k-step, d chunks 16 KB apart
    fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) wgmma_m64n128k16_rs<1>(o, a[kk], vd + 128 * kk, 1u);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
    ring.release(b);
  }
  store_o_lse(o, l, m, ri, sh, c, h, row_base, wq0, r_in, c2, O, LSE);
}

__global__ void __launch_bounds__(RING_THREADS, 1)
attn_bwd_dkdv_hd128_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmDO,
                           const float* __restrict__ LSE, const float* __restrict__ Delta, __nv_bfloat16* __restrict__ dQKV,
                           const AttnShape sh) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sK = smem_base_1024(smem_raw);      // [K 32 KB][V 32 KB][ring][kv barrier]
  uint8_t* sV = sK + 32768;
  const Hd128Ring ring(sK + 65536);
  uint64_t* bar_kv = ring.end();

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int r_in = 16 * (t >> 5) + ((t & 31) >> 2), c2 = 2 * (t & 3);
  const int kt = blockIdx.x, h = blockIdx.y, c = blockIdx.z;
  const int row_base = c * sh.span, nq = (sh.span + 127) >> 7;
  const int n_wg = (kt * 128 + 64 < sh.span) ? 2 : 1;   // consumer warpgroups with at least one key row in the group
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQKV);
    tma_prefetch_desc(&tmDO);
    ring.init(4 * n_wg);
    mbar_init(bar_kv, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (ring_producer(wg, [&] {
        mbar_expect_tx(bar_kv, 65536);
        tma_load_tile128(&tmQKV, bar_kv, sK, sh.D + h * 128, row_base + kt * 128);
        tma_load_tile128(&tmQKV, bar_kv, sV, 2 * sh.D + h * 128, row_base + kt * 128);
        ring.fill(nq, [&](uint64_t* bar, uint8_t* dst, int qt) {
          tma_load_tile128(&tmQKV, bar, dst, h * 128, row_base + qt * 128);
          tma_load_tile128(&tmDO, bar, dst + 32768, h * 128, row_base + qt * 128);
        });
      }))
    return;
  const int wk0 = kt * 128 + wg * 64;
  if (wk0 >= sh.span) return;                  // not counted by the empty barriers (n_wg)
  mbar_wait(bar_kv, 0);
  // valid query columns of this thread's two key rows: the key's own crop (none for keys outside the group)
  int lo[2], hi[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const RowInfo ri = row_info(sh, c, wk0 + r_in + 8 * hh);
    lo[hh] = ri.ok ? ri.klo : 0;
    hi[hh] = ri.ok ? ri.khi : 0;
  }
  const float cs = sh.scale * LOG2E;
  float dk[64], dv[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) { dk[i] = 0.f; dv[i] = 0.f; }
#pragma unroll 1
  for (int qt = 0; qt < nq; ++qt) {
    const uint8_t* sQt = ring.wait(qt);
    const uint8_t* sDOt = sQt + 32768;
#pragma unroll 1
    for (int qc = 0; qc < 4; ++qc) {   // 32 query columns at a time: with dK + dV resident, 64 would spill
      float s[16], dp[16];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 8; ++k) {   // S^T and dP^T are independent accumulator chains: interleave them
        wgmma_m64n32k16_ss<0, 0>(s, kdesc128(sK + wg * 8192, k), kdesc128(sQt + qc * 4096, k), k > 0 ? 1u : 0u);
        wgmma_m64n32k16_ss<0, 0>(dp, kdesc128(sV + wg * 8192, k), kdesc128(sDOt + qc * 4096, k), k > 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(s);
      fence_regs(dp);
      uint32_t pa[2][4], da[2][4];    // bf16 A fragments of P^T / dS^T (k-step kk: query columns 16 kk ..)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int q = qt * 128 + qc * 32 + 8 * i + c2;
        float l2[2], dl[2];
        row_stats(sh, LSE, Delta, c, h, q, l2[0], dl[0]);
        row_stats(sh, LSE, Delta, c, h, q + 1, l2[1], dl[1]);
        float pv[4], dv4[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int hh = j >> 1, qq = q + (j & 1);
          const bool ok = qq >= lo[hh] && qq < hi[hh];
          const float p = ok ? ex2_approx(fmaf(s[4 * i + j], cs, -l2[j & 1])) : 0.f;
          dv4[j] = ok ? (p * sh.scale) * (dp[4 * i + j] - dl[j & 1]) : 0.f;
          pv[j] = p;
        }
        pa[i >> 1][2 * (i & 1)] = pack_bf16(pv[0], pv[1]);
        pa[i >> 1][2 * (i & 1) + 1] = pack_bf16(pv[2], pv[3]);
        da[i >> 1][2 * (i & 1)] = pack_bf16(dv4[0], dv4[1]);
        da[i >> 1][2 * (i & 1) + 1] = pack_bf16(dv4[2], dv4[3]);
      }
      const uint64_t dod = desc_here(sDOt + qc * 4096, 16384, 1024);   // B MN-major: 16 query rows per k-step
      const uint64_t qd = desc_here(sQt + qc * 4096, 16384, 1024);
      fence_regs(dk);
      fence_regs(dv);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
        wgmma_m64n128k16_rs<1>(dv, pa[kk], dod + 128 * kk, 1u);
        wgmma_m64n128k16_rs<1>(dk, da[kk], qd + 128 * kk, 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(dk);
      fence_regs(dv);
      fence_frag(pa);
      fence_frag(da);
    }
    ring.release(qt);
  }
  store_grad_rows(dk, sh, c, row_base, wk0, r_in, c2, h, 1, true, dQKV);
  store_grad_rows(dv, sh, c, row_base, wk0, r_in, c2, h, 2, false, dQKV);
}

__global__ void __launch_bounds__(RING_THREADS, 1)
attn_bwd_dq_hd128_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmDO,
                         const float* __restrict__ LSE, const float* __restrict__ Delta, __nv_bfloat16* __restrict__ dQKV,
                         const AttnShape sh) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sQ = smem_base_1024(smem_raw);      // [Q 32 KB][dO 32 KB][ring][q barrier]
  uint8_t* sDO = sQ + 32768;
  const Hd128Ring ring(sQ + 65536);
  uint64_t* bar_q = ring.end();

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int r_in = 16 * (t >> 5) + ((t & 31) >> 2), c2 = 2 * (t & 3);
  const int qt = blockIdx.x, h = blockIdx.y, c = blockIdx.z;
  const int q0 = qt * 128, row_base = c * sh.span, nk = (sh.span + 127) >> 7;
  const int n_wg = (q0 + 64 < sh.span) ? 2 : 1;   // consumer warpgroups with at least one query row in the group
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQKV);
    tma_prefetch_desc(&tmDO);
    ring.init(4 * n_wg);
    mbar_init(bar_q, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (ring_producer(wg, [&] {
        mbar_expect_tx(bar_q, 65536);
        tma_load_tile128(&tmQKV, bar_q, sQ, h * 128, row_base + q0);
        tma_load_tile128(&tmDO, bar_q, sDO, h * 128, row_base + q0);
        ring.fill(nk, [&](uint64_t* bar, uint8_t* dst, int kt) {
          tma_load_tile128(&tmQKV, bar, dst, sh.D + h * 128, row_base + kt * 128);
          tma_load_tile128(&tmQKV, bar, dst + 32768, 2 * sh.D + h * 128, row_base + kt * 128);
        });
      }))
    return;
  const int wq0 = q0 + wg * 64;
  if (wq0 >= sh.span) return;                  // not counted by the empty barriers (n_wg)
  mbar_wait(bar_q, 0);
  float lse2[2], dl[2];
  int lo[2], hi[2];                            // valid key columns of this thread's two query rows
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const RowInfo ri = row_info(sh, c, wq0 + r_in + 8 * hh);
    row_stats(sh, LSE, Delta, c, h, wq0 + r_in + 8 * hh, lse2[hh], dl[hh]);
    lo[hh] = ri.ok ? ri.klo : 0;
    hi[hh] = ri.ok ? ri.khi : 0;
  }
  const float cs = sh.scale * LOG2E;
  float dq[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) dq[i] = 0.f;
#pragma unroll 1
  for (int kt = 0; kt < nk; ++kt) {
    const uint8_t* sK = ring.wait(kt);
    const uint8_t* sV = sK + 32768;
#pragma unroll 1
    for (int hf = 0; hf < 2; ++hf) {
      float s[32], dp[32];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        wgmma_m64n64k16_ss<0, 0>(s, kdesc128(sQ + wg * 8192, k), kdesc128(sK + hf * 8192, k), k > 0 ? 1u : 0u);
        wgmma_m64n64k16_ss<0, 0>(dp, kdesc128(sDO + wg * 8192, k), kdesc128(sV + hf * 8192, k), k > 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(s);
      fence_regs(dp);
      uint32_t da[4][4];              // bf16 A fragments of dS (k-step kk: keys 16 kk ..)
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int key = kt * 128 + hf * 64 + 8 * i + c2;
        float d4[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int hh = j >> 1, kk = key + (j & 1);
          const bool ok = kk >= lo[hh] && kk < hi[hh];
          const float p = ok ? ex2_approx(fmaf(s[4 * i + j], cs, -lse2[hh])) : 0.f;
          d4[j] = ok ? (p * sh.scale) * (dp[4 * i + j] - dl[hh]) : 0.f;
        }
        da[i >> 1][2 * (i & 1)] = pack_bf16(d4[0], d4[1]);
        da[i >> 1][2 * (i & 1) + 1] = pack_bf16(d4[2], d4[3]);
      }
      const uint64_t kd = desc_here(sK + hf * 8192, 16384, 1024);   // B MN-major: 16 keys per k-step
      fence_regs(dq);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_m64n128k16_rs<1>(dq, da[kk], kd + 128 * kk, 1u);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(dq);
      fence_frag(da);
    }
    ring.release(kt);
  }
  store_grad_rows(dq, sh, c, row_base, wq0, r_in, c2, h, 0, true, dQKV);
}

static int make_map(CUtensorMap* map, const void* ptr, long rows, int cols, int ld, int box_rows) {
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  return encode_tensor_map_2d_bf16(map, ptr, dims, strides, box, estr);
}

// Largest crop the attention entry points take.  The streamed kernels need no resource that grows with N; the bound keeps
// every token coordinate (crop * N + token, TMA row coordinates and kernel offsets are 32-bit) and the grid inside what
// is checked below.  It covers a 2 880^2 crop at patch 16 with 5 prefix tokens (32 405 tokens).
constexpr int ATTN_MAX_TOKENS = 32768;
constexpr int ATTN_FWD_RESIDENT_SPAN = 448;   // attn_fwd_kernel: Q and all of K / V of a crop group in shared memory
constexpr int ATTN_BWD_RESIDENT_SPAN = 256;   // attn_bwd_fused_kernel: all Q / dO / K / V tiles of a crop group resident

static int attn_shape(AttnShape* s, int n_crops, int N, int D, int H) {
  if (D != H * 64 && D != H * 128) return set_error(D3_ERR_ARG, "attention: head_dim must be 64 or 128");
  if (N <= 0 || n_crops <= 0) return set_error(D3_ERR_ARG, "attention: empty problem");
  if (N > ATTN_MAX_TOKENS) return set_error(D3_ERR_ARG, "attention: N > 32768 tokens per crop");
  if ((long)n_crops * N > INT_MAX) return set_error(D3_ERR_ARG, "attention: n_crops * N must be below 2^31 token rows");
  s->N = N; s->D = D; s->H = H; s->n_crops = n_crops;
  s->scale = (D == H * 64) ? 0.125f : 0.08838834764831845f;   // head_dim^-0.5
  s->sin_t = nullptr; s->cos_t = nullptr; s->prefix = 0;
  s->G = (N <= 64) ? (128 / N) : 1;                 // short crops: several per 128-row tile, block-diagonal mask
  if (s->G > n_crops) s->G = n_crops;
  s->span = s->G * N;
  s->nkb = (s->span + 63) / 64;
  return D3_OK;
}

// grid of every kernel that owns 128-row tiles of a crop group: (tiles of the span, head, crop group)
static int tile_grid(const AttnShape& s, dim3* grid) {
  const int groups = (s.n_crops + s.G - 1) / s.G;
  if (s.H > 65535 || groups > 65535) return set_error(D3_ERR_ARG, "attention: H and crop groups must be <= 65535");
  *grid = dim3((s.span + 127) / 128, s.H, groups);
  return D3_OK;
}

// Launches `kernel` with `smem` bytes of dynamic shared memory.  The first launch of a kernel in the process raises its
// opt-in limit to `smem_max`, the most any of its launches asks for.
template <auto kernel, class... Args>
static int launch(dim3 grid, int threads, int smem, int smem_max, cudaStream_t st, const Args&... args) {
  static const cudaError_t cfg = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max);
  (void)cfg;   // a failure shows at the launch
  kernel<<<grid, threads, smem, st>>>(args...);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

}  // namespace d3

using namespace d3;

extern "C" {

int d3_attn_fwd(const void* qkv, void* o, float* lse, int n_crops, int N, int D, int H, void* stream) {
  AttnShape s;
  int rc = attn_shape(&s, n_crops, N, D, H);
  if (rc) return rc;
  dim3 grid;
  if ((rc = tile_grid(s, &grid))) return rc;
  const long T = (long)n_crops * N;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  __nv_bfloat16* out = (__nv_bfloat16*)o;
  CUtensorMap tqkv;
  if ((rc = make_map(&tqkv, qkv, T, 3 * D, 3 * D, 128))) return rc;
  if (D == H * 128)
    return launch<attn_fwd_hd128_kernel>(grid, RING_THREADS, HD128_FWD_SMEM, HD128_FWD_SMEM, st, tqkv, out, lse, s);
  if (s.span > ATTN_FWD_RESIDENT_SPAN)
    return launch<attn_fwd_stream_kernel>(grid, RING_THREADS, FWD_STREAM_SMEM, FWD_STREAM_SMEM, st, tqkv, out, lse, s);
  CUtensorMap tkv;
  if ((rc = make_map(&tkv, qkv, T, 3 * D, 3 * D, 64))) return rc;
  return launch<attn_fwd_kernel>(grid, 256, fwd_smem(s.nkb), fwd_smem((ATTN_FWD_RESIDENT_SPAN + 63) / 64), st, tqkv, tkv,
                                 out, lse, s);
}

int d3_attn_bwd(const void* qkv, const void* o, const void* d_o, const float* lse, float* delta_scratch, void* dqkv,
                int n_crops, int N, int D, int H, const float* rope_sin, const float* rope_cos, int rope_prefix,
                void* stream) {
  AttnShape s;
  int rc = attn_shape(&s, n_crops, N, D, H);
  if (rc) return rc;
  if ((rope_sin == nullptr) != (rope_cos == nullptr)) return set_error(D3_ERR_ARG, "d3_attn_bwd: sin/cos tables");
  if (!delta_scratch) return set_error(D3_ERR_ARG, "d3_attn_bwd: delta scratch buffer");
  const bool hd128 = D == H * 128;
  const bool streamed = s.span > ATTN_BWD_RESIDENT_SPAN;
  dim3 grid;   // ring kernels; key tiles and query tiles of a crop group are both (span + 127) / 128
  if ((hd128 || streamed) && (rc = tile_grid(s, &grid))) return rc;
  s.sin_t = rope_sin; s.cos_t = rope_cos; s.prefix = rope_prefix;
  const long T = (long)n_crops * N;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long threads = T * (D / 8);
  if (hd128)
    attn_delta_kernel<128><<<(int)((threads + 255) / 256), 256, 0, st>>>((const __nv_bfloat16*)o, (const __nv_bfloat16*)d_o,
                                                                       delta_scratch, T, N, D, H);
  else
    attn_delta_kernel<64><<<(int)((threads + 255) / 256), 256, 0, st>>>((const __nv_bfloat16*)o, (const __nv_bfloat16*)d_o,
                                                                      delta_scratch, T, N, D, H);
  D3_CHECK_LAUNCH();
  CUtensorMap tqkv, tdo;
  if ((rc = make_map(&tqkv, qkv, T, 3 * D, 3 * D, 128))) return rc;
  if ((rc = make_map(&tdo, d_o, T, D, D, 128))) return rc;
  __nv_bfloat16* dq = (__nv_bfloat16*)dqkv;
  if (hd128) {
    if ((rc = launch<attn_bwd_dkdv_hd128_kernel>(grid, RING_THREADS, HD128_BWD_SMEM, HD128_BWD_SMEM, st, tqkv, tdo, lse,
                                                 delta_scratch, dq, s)))
      return rc;
    return launch<attn_bwd_dq_hd128_kernel>(grid, RING_THREADS, HD128_BWD_SMEM, HD128_BWD_SMEM, st, tqkv, tdo, lse,
                                            delta_scratch, dq, s);
  }
  if (streamed) {
    if ((rc = launch<attn_bwd_dkdv_kernel>(grid, RING_THREADS, DKDV_SMEM, DKDV_SMEM, st, tqkv, tdo, lse, delta_scratch, dq,
                                           s)))
      return rc;
    return launch<attn_bwd_dq_kernel>(grid, RING_THREADS, DQ_SMEM, DQ_SMEM, st, tqkv, tdo, lse, delta_scratch, dq, s);
  }
  return launch<attn_bwd_fused_kernel>(dim3(H, (n_crops + s.G - 1) / s.G), 256, bwd_fused_smem((s.span + 127) / 128),
                                       bwd_fused_smem(ATTN_BWD_RESIDENT_SPAN / 128), st, tqkv, tdo, lse, delta_scratch,
                                       dq, s);
}

}  // extern "C"
