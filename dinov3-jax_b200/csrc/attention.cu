// Multi-head self-attention forward / backward on the Hopper tensor cores (wgmma) for the short ViT sequences of the
// DINOv3 crops (N = 197 / 37 / 257 / 50 tokens, head_dim = 64): replaces flax `nn.dot_product_attention(q, k, v)` at
// dinov3_jax/layers/attention.py:116 (softmax((q / sqrt(64)) k^T) v, no mask, no dropout) and its jax.grad.
//
// Short crops (N <= 64) are packed G per 128-row tile with a block-diagonal mask, so one CTA covers a "crop group" of
// span = G * N token rows.  Operands come by TMA (SWIZZLE_128B) from the fused qkv buffer [T, 3D] (q | k | v thirds,
// heads contiguous); every product is a warpgroup MMA with fp32 accumulators in registers.
//
// Forward: one CTA per (q-tile of 128 rows, head, crop group), two warpgroups of 64 query rows each.  Q and the whole
// key / value range of the group are staged once; each warpgroup walks the keys in blocks of 64: S = Q K^T (SS form),
// online softmax on the accumulator fragment, then O += P V with P handed to the tensor core straight from registers
// (RS form: the accumulator fragment of S is the A-operand fragment of the PV product).
#include "ptx.cuh"
#include <cstdlib>
#include "d3_internal.h"

namespace d3 {

constexpr float LOG2E = 1.4426950408889634f;

__device__ long long* g_attn_dbg = nullptr;   // optional clock64() trace of CTA (0,0) (tools/attn_trace.py)
__device__ __forceinline__ void dbg_mark(int slot) {
  if (g_attn_dbg && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && (threadIdx.x == 0 || threadIdx.x == 200))
    g_attn_dbg[slot * 2 + (threadIdx.x == 0 ? 0 : 1)] = clock64();
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

__global__ void __launch_bounds__(256)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV,
                __nv_bfloat16* __restrict__ O, float* __restrict__ LSE, const AttnShape sh) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // layout: [Q 128 x 128 B][K nkb x 8 KB][V nkb x 8 KB][barrier]
  uint8_t* sQ = smem;
  uint8_t* sK = smem + 16384;
  uint8_t* sV = sK + sh.nkb * 8192;
  uint64_t* bar = reinterpret_cast<uint64_t*>(sV + sh.nkb * 8192);

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int qt = blockIdx.x, h = blockIdx.y, c = blockIdx.z;
  const int q0 = qt * 128;
  const int row_base = c * sh.span;  // first token row of this CTA's crop group in [T, ...]
  dbg_mark(0);
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
    // ---- online softmax of the two rows this thread holds (columns 8i + c2 + {0,1})
    const int kb0 = b * 64 + c2;
    const bool full = kb0 - c2 >= max(ri[0].klo, ri[1].klo) && kb0 - c2 + 64 <= min(ri[0].khi, ri[1].khi);
    float mx[2] = {-3.0e38f, -3.0e38f};
#pragma unroll
    for (int i = 0; i < 8; ++i)
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
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int hh = j >> 1, kk = kb0 + 8 * i + (j & 1);
        const float p = (full || (kk >= ri[hh].klo && kk < ri[hh].khi)) ? ex2_approx(fmaf(s[4 * i + j], cs, -ms[hh])) : 0.f;
        s[4 * i + j] = p;
        l[hh] += p;
        o[4 * i + j] *= corr[hh];
      }
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
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
    const int q = wq0 + r_in + 8 * hh;
    if (!ri[hh].ok) continue;
    const float inv = 1.f / l[hh];
    __nv_bfloat16* dst = O + (size_t)(row_base + q) * sh.D + h * 64 + c2;
#pragma unroll
    for (int i = 0; i < 8; ++i)
      *reinterpret_cast<uint32_t*>(dst + 8 * i) = pack_bf16(o[4 * i + 2 * hh] * inv, o[4 * i + 2 * hh + 1] * inv);
    if (LSE && c2 == 0)   // natural-log LSE of the scaled scores, indexed [crop, head, token]
      LSE[((size_t)(c * sh.G + ri[hh].g) * sh.H + h) * sh.N + (q - ri[hh].klo)] = m[hh] * sh.scale + logf(l[hh]);
  }
  dbg_mark(1);
}

// Delta[c,h,q] = sum_d dO[q, h, d] * O[q, h, d]    (backward softmax term)
__global__ void attn_delta_kernel(const __nv_bfloat16* __restrict__ O, const __nv_bfloat16* __restrict__ dO,
                                  float* __restrict__ delta, long T, int N, int D, int H) {
  // 8 threads per (row, head): one 16-byte load of O and of dO each, 3 shuffle steps inside the 8-lane group
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
  s += __shfl_xor_sync(0xffffffffu, s, 4);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  if (ok && (c8 & 7) == 0) delta[((row / N) * H + (c8 >> 3)) * N + (row % N)] = s;
}

// ------------------------------------------------------------------------------------------------ backward
// One CTA per (head, crop group); span <= 384 (up to 3 query tiles x 3 key tiles of 128), two warpgroups of 64 rows.
// Q and dO tiles stay resident; K / V come one 128-key tile at a time.  For a tile pair (kt, qt):
//   S  = Q K^T, dP = dO V^T                                    (registers)
//   P  = exp(S*scale - lse), dS = P * (dP - Delta) * scale
// Phase 1 (kt outer, qt inner): P and dS go to shared memory as bf16 SWIZZLE_128B tiles [128 q x 128 keys], then
//   dV[kt] += P^T dO, dK[kt] += dS^T Q      (A = P / dS read MN-major: each warpgroup owns 64 keys)
// Phase 2 (qt outer, kt inner): S and dP are recomputed and dQ[qt] += dS K with dS straight from registers (RS form).
// The recomputation costs two small products per tile pair and keeps every accumulator in registers.
// inverse RoPE on the gradient: transpose of y = x*cos + rot_half(x)*sin (dinov3_jax/layers/attention.py:14-20); this
// thread holds columns d = 8i + c2 + {0,1} of a row, i.e. both partners (d, d + 32) of every rotation pair it touches.
__device__ __forceinline__ void store_grad_rows(float (&a)[32], const AttnShape& sh, int c, int row_base, int tile_row0,
                                                int r_in, int c2, int h, int third, bool rope, __nv_bfloat16* dQKV) {
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int row = tile_row0 + r_in + 8 * hh;
    const RowInfo ri = row_info(sh, c, row);
    if (!ri.ok) continue;
    const int tok = row - ri.klo;
    float v[16];
#pragma unroll
    for (int i = 0; i < 8; ++i) { v[2 * i] = a[4 * i + 2 * hh]; v[2 * i + 1] = a[4 * i + 2 * hh + 1]; }
    if (rope && sh.sin_t && tok >= sh.prefix) {
      const float* sn = sh.sin_t + (size_t)(tok - sh.prefix) * 64;
      const float* cn = sh.cos_t + (size_t)(tok - sh.prefix) * 64;
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int d = 8 * i + c2 + j;
          const float lo = v[2 * i + j], hi = v[2 * (i + 4) + j];
          v[2 * i + j] = lo * cn[d] + hi * sn[d];
          v[2 * (i + 4) + j] = hi * cn[d] - lo * sn[d];
        }
    }
    __nv_bfloat16* dst = dQKV + (size_t)(row_base + row) * (3 * sh.D) + third * sh.D + h * 64 + c2;
#pragma unroll
    for (int i = 0; i < 8; ++i) *reinterpret_cast<uint32_t*>(dst + 8 * i) = pack_bf16(v[2 * i], v[2 * i + 1]);
  }
}

__global__ void __launch_bounds__(256)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmDO,
                const float* __restrict__ LSE, const float* __restrict__ Delta, __nv_bfloat16* __restrict__ dQKV,
                const AttnShape sh) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int nQ = (sh.span + 127) / 128, nK = nQ;
  uint8_t* sQ = smem;                          // [nQ][128 x 64]
  uint8_t* sDO = sQ + nQ * 16384;              // [nQ][128 x 64]
  uint8_t* sK = sDO + nQ * 16384;              // 16 KB (current key tile)
  uint8_t* sV = sK + 16384;                    // 16 KB
  uint8_t* sP = sV + 16384;                    // [2 chunks of 64 keys][128 q x 128 B] 32 KB
  uint8_t* sDS = sP + 32768;                   // 32 KB
  uint64_t* bars = reinterpret_cast<uint64_t*>(sDS + 32768);
  uint64_t* bar_q = bars;
  uint64_t* bar_kv = bars + 1;

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int r_in = 16 * (t >> 5) + ((t & 31) >> 2), c2 = 2 * (t & 3);
  const int h = blockIdx.x, c = blockIdx.y;
  const int row_base = c * sh.span;
  const float cs = sh.scale * LOG2E;
  dbg_mark(0);
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQKV);
    tma_prefetch_desc(&tmDO);
    mbar_init(bar_q, 1);
    mbar_init(bar_kv, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x < 32 && elect_one()) {
    mbar_expect_tx(bar_q, nQ * 2 * 16384);
    for (int qt = 0; qt < nQ; ++qt) {
      tma_load_2d(&tmQKV, bar_q, sQ + qt * 16384, h * 64, row_base + qt * 128);
      tma_load_2d(&tmDO, bar_q, sDO + qt * 16384, h * 64, row_base + qt * 128);
    }
  }
  uint32_t kv_phase = 0;
  int kv_loaded = -1;
  auto load_kv = [&](int kt) {       // every thread: K / V tile kt resident (the previous tile's readers are done)
    if (kv_loaded == kt) return;
    __syncthreads();
    if (threadIdx.x < 32 && elect_one()) {
      mbar_expect_tx(bar_kv, 2 * 16384);
      tma_load_2d(&tmQKV, bar_kv, sK, sh.D + h * 64, row_base + kt * 128);
      tma_load_2d(&tmQKV, bar_kv, sV, 2 * sh.D + h * 64, row_base + kt * 128);
    }
    mbar_wait(bar_kv, kv_phase);
    kv_phase ^= 1;
    kv_loaded = kt;
  };
  // S and dP of this warpgroup's 64 query rows of tile qt against key tile kt, turned into P (in s) and dS (in dp)
  auto p_ds = [&](int qt, int kt, float (&s)[64], float (&dp)[64]) {
    const uint64_t qd = gmma_desc_sw128(smem_u32(sQ + qt * 16384 + wg * 8192), 16, 1024);
    const uint64_t dod = gmma_desc_sw128(smem_u32(sDO + qt * 16384 + wg * 8192), 16, 1024);
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
      const int q = qt * 128 + wg * 64 + r_in + 8 * hh;
      const RowInfo ri = row_info(sh, c, q);
      const size_t stat = ((size_t)(c * sh.G + ri.g) * sh.H + h) * sh.N + (ri.ok ? q - ri.klo : 0);
      const float lse2 = ri.ok ? LSE[stat] * LOG2E : 0.f;
      const float dl = ri.ok ? Delta[stat] : 0.f;
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
  };

  mbar_wait(bar_q, 0);
  // ---- phase 1: dK, dV of key tile kt (this warpgroup: keys kt*128 + wg*64 ..)
#pragma unroll 1
  for (int kt = 0; kt < nK; ++kt) {
    load_kv(kt);
    float dk[32], dv[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) { dk[i] = 0.f; dv[i] = 0.f; }
#pragma unroll 1
    for (int qt = 0; qt < nQ; ++qt) {
      float s[64], dp[64];
      p_ds(qt, kt, s, dp);
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int row = wg * 64 + r_in + 8 * hh;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const uint32_t off = (i >> 3) * 16384 + sw128_offset(row, (8 * i + c2) & 63);
          *reinterpret_cast<uint32_t*>(sP + off) = pack_bf16(s[4 * i + 2 * hh], s[4 * i + 2 * hh + 1]);
          *reinterpret_cast<uint32_t*>(sDS + off) = pack_bf16(dp[4 * i + 2 * hh], dp[4 * i + 2 * hh + 1]);
        }
      }
      fence_proxy_async_smem();   // generic-proxy smem writes -> visible to the tensor core (async proxy)
      __syncthreads();
      // dV[keys, 64] += P^T dO ; dK[keys, 64] += dS^T Q   (A MN-major: 16 query rows per k-step = 2048 B)
      const uint64_t pd = gmma_desc_sw128(smem_u32(sP + wg * 16384), 16384, 1024);
      const uint64_t sd = gmma_desc_sw128(smem_u32(sDS + wg * 16384), 16384, 1024);
      const uint64_t dod = gmma_desc_sw128(smem_u32(sDO + qt * 16384), 8192, 1024);
      const uint64_t qd = gmma_desc_sw128(smem_u32(sQ + qt * 16384), 8192, 1024);
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
      __syncthreads();            // both warpgroups are done reading sP / sDS before the next tile pair rewrites them
    }
    store_grad_rows(dk, sh, c, row_base, kt * 128 + wg * 64, r_in, c2, h, 1, true, dQKV);
    store_grad_rows(dv, sh, c, row_base, kt * 128 + wg * 64, r_in, c2, h, 2, false, dQKV);
  }
  // ---- phase 2: dQ of query tile qt (this warpgroup: rows qt*128 + wg*64 ..); the key tiles are walked in alternating
  // directions so that each walk starts with the tile that is still resident
#pragma unroll 1
  for (int qt = 0; qt < nQ; ++qt) {
    float dq[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) dq[i] = 0.f;
#pragma unroll 1
    for (int j = 0; j < nK; ++j) {
      const int kt = (qt & 1) ? j : nK - 1 - j;
      load_kv(kt);
      float s[64], dp[64];
      p_ds(qt, kt, s, dp);
      uint32_t a[8][4];
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)
#pragma unroll
        for (int e = 0; e < 4; ++e) a[kk][e] = pack_bf16(dp[8 * kk + 2 * e], dp[8 * kk + 2 * e + 1]);
      const uint64_t kd = gmma_desc_sw128(smem_u32(sK), 8192, 1024);   // K as MN-major B (keys x d)
      fence_regs(dq);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) wgmma_m64n64k16_rs<1>(dq, a[kk], kd + 128 * kk, 1u);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(dq);
    }
    store_grad_rows(dq, sh, c, row_base, qt * 128 + wg * 64, r_in, c2, h, 0, true, dQKV);
  }
  dbg_mark(1);
}

static int make_map(CUtensorMap* map, const void* ptr, long rows, int cols, int ld, int box_rows) {
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  return encode_tensor_map_2d_bf16(map, ptr, dims, strides, box, estr);
}

static int attn_shape(AttnShape* s, int n_crops, int N, int D, int H) {
  if (D != H * 64) return set_error(D3_ERR_ARG, "attention: head_dim must be 64");
  if (N <= 0 || n_crops <= 0) return set_error(D3_ERR_ARG, "attention: empty problem");
  s->N = N; s->D = D; s->H = H; s->scale = 0.125f; s->n_crops = n_crops;
  s->sin_t = nullptr; s->cos_t = nullptr; s->prefix = 0;
  s->G = (N <= 64) ? (128 / N) : 1;                 // short crops: several per 128-row tile, block-diagonal mask
  if (s->G > n_crops) s->G = n_crops;
  s->span = s->G * N;
  s->nkb = (s->span + 63) / 64;
  if (s->span > 448) return set_error(D3_ERR_ARG, "attention: N > 448 tokens per crop not supported by the single-pass kernel");
  return D3_OK;
}

}  // namespace d3

using namespace d3;

extern "C" {

int d3_debug_attn_trace(long long* buf /*device [64] or NULL*/) {
  cudaError_t e = cudaMemcpyToSymbol(g_attn_dbg, &buf, sizeof(buf));
  return e == cudaSuccess ? D3_OK : set_error(D3_ERR_CUDA, cudaGetErrorString(e));
}

int d3_attn_fwd(const void* qkv, void* o, float* lse, int n_crops, int N, int D, int H, void* stream) {
  AttnShape s;
  int rc = attn_shape(&s, n_crops, N, D, H);
  if (rc) return rc;
  const long T = (long)n_crops * N;
  CUtensorMap tq, tkv;
  if ((rc = make_map(&tq, qkv, T, 3 * D, 3 * D, 128))) return rc;
  if ((rc = make_map(&tkv, qkv, T, 3 * D, 3 * D, 64))) return rc;
  const int smem = 16384 + 2 * s.nkb * 8192 + 64 + 1024;
  static bool cfg = false;
  if (!cfg) { cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); cfg = true; }
  dim3 grid((s.span + 127) / 128, H, (n_crops + s.G - 1) / s.G);
  attn_fwd_kernel<<<grid, 256, smem, reinterpret_cast<cudaStream_t>(stream)>>>(tq, tkv, (__nv_bfloat16*)o, lse, s);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_attn_bwd(const void* qkv, const void* o, const void* d_o, const float* lse, float* delta_scratch, void* dqkv,
                int n_crops, int N, int D, int H, const float* rope_sin, const float* rope_cos, int rope_prefix,
                void* stream) {
  AttnShape s;
  int rc = attn_shape(&s, n_crops, N, D, H);
  if (rc) return rc;
  if (N > 384) return set_error(D3_ERR_ARG, "d3_attn_bwd: N > 384 tokens per crop not supported (3 query tiles of 128)");
  if ((rope_sin == nullptr) != (rope_cos == nullptr)) return set_error(D3_ERR_ARG, "d3_attn_bwd: sin/cos tables");
  if (!delta_scratch) return set_error(D3_ERR_ARG, "d3_attn_bwd: delta scratch buffer");
  s.sin_t = rope_sin; s.cos_t = rope_cos; s.prefix = rope_prefix;
  const long T = (long)n_crops * N;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long threads = T * (D / 8);
  attn_delta_kernel<<<(int)((threads + 255) / 256), 256, 0, st>>>((const __nv_bfloat16*)o, (const __nv_bfloat16*)d_o,
                                                                delta_scratch, T, N, D, H);
  D3_CHECK_LAUNCH();
  CUtensorMap tqkv, tdo;
  if ((rc = make_map(&tqkv, qkv, T, 3 * D, 3 * D, 128))) return rc;
  if ((rc = make_map(&tdo, d_o, T, D, D, 128))) return rc;
  static bool cfg = false;
  if (!cfg) { cudaFuncSetAttribute(attn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024); cfg = true; }
  const int nq = (s.span + 127) / 128;
  const int smem = 2 * nq * 16384 + 32768 + 65536 + 64 + 1024;
  dim3 grid(H, (n_crops + s.G - 1) / s.G);
  attn_bwd_kernel<<<grid, 256, smem, st>>>(tqkv, tdo, lse, delta_scratch, (__nv_bfloat16*)dqkv, s);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

}  // extern "C"
