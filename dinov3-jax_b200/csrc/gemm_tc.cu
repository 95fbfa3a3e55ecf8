// Persistent, warp-specialised bf16 GEMM on the Hopper tensor cores (wgmma, register accumulators, TMA operand
// staging through an mbarrier ring).  One kernel family covers every dense contraction on the DINOv3 training path:
//   forward  Y = X W        (A K-major, B MN-major: reference kernels are stored [in,out])
//   dgrad    dX = dY W^T    (A K-major, B K-major)
//   wgrad    dW = X^T dY    (A MN-major, B MN-major, fp32 output, split-K reduced in a fixed order)
// replacing nn.Dense / nn.Conv(stride=kernel) call sites of the reference:
//   dinov3_jax/layers/attention.py:63-65,94,101   dinov3_jax/layers/ffn_layers.py:36-47
//   dinov3_jax/layers/patch_embed.py:38-51        dinov3_jax/layers/dino_head.py:20-43,65-85
// The epilogue fuses bias, tanh-GELU, GELU', LayerScale (gamma) and the residual add
// (dinov3_jax/layers/block.py:198-199, dinov3_jax/layers/layer_scale.py:17-21), and the exact (erf) GELU of the
// ConvNeXt block's first pointwise layer (dinov3_jax/models/convnext.py:70-72).
//
// One kernel, 128 x {64,128} output tiles, 384 threads, launched in clusters of 2 CTAs that compute the tiles (m0, n0)
// and (m0, n0 + BN) of a pair side by side, over the same k-blocks (128 x 256 tiles: see below):
//   warpgroup 0      TMA producer (one elected thread): A and B k-blocks of 64, tile after tile of this CTA's work
//                    list, into one shared-memory ring.  A is shared by the pair: each CTA loads one 64-row half and
//                    multicasts it into both CTAs' ring, so a CTA reads 3/4 (BN = 128) or 2/3 (BN = 64) of the
//                    operand bytes it consumes from L2.  A ring stage is written by both producers, so it is refilled
//                    only after the consumers of both CTAs released it (empty barriers count 2 arrivals: one local,
//                    one from the peer through its cluster address);
//   warpgroups 1, 2  consumers in ping-pong: the CTA's tiles alternate between them, so one warpgroup's epilogue
//                    runs under the other's main loop.  A tile is two m64nBNk16 wgmma chains (rows 0-63 / 64-127)
//                    over SWIZZLE_128B operands, K-major or MN-major through the descriptor transpose bits.
// Both consumers walk the whole ring in fill order, stepping over the other's k-blocks.  The main loops take turns: a
// consumer starts its main loop only after the other has passed its last full-barrier wait (named barriers 1 / 2), so
// every fill of a stage is waited on by exactly one consumer, in order, and no wait can be two phases ahead (which the
// phase parity could not tell apart).  The main loop of one tile so has the whole ring in flight.
//
// 128 x 256 tiles (BN = 256, only when forced by tile_n): both consumers share every tile, warpgroup 1 rows 0-63 and
// warpgroup 2 rows 64-127, each one m64n256k16 chain; both wait on every full barrier and release every stage, locally
// and on the peer (empty barriers count 4).  The cluster pairs tiles (m0, n0) and (m0 + 128, n0): each CTA loads its own
// A and multicasts one 128-column half of B.  Each element keeps the k-blocks, k16 steps and split-K slices of BN = 128,
// so the bits are the same.  The epilogue is not hidden under another main loop.
//
// The epilogue's arithmetic is one function, epi_value (one element, accumulator to stored value), under two tile
// walkers.  The epilogue flags are a template parameter.  The flag sets one training step issues are compiled with
// their flags fixed (dispatch() lists them) and run epilogue_tile: bias and gamma are staged in shared memory by
// cp.async during the main loop, each thread issues all loads of a 64 x 64 chunk before its first store, and the
// results go through a shared-memory staging area to TMA stores (all but the weight gradients', which store from
// registers).  Every other call (fused reduce-scatter, misaligned operands, odd N, other flag sets) runs the same
// kernel with the flags read at run time (EPI_RUNTIME) and epilogue_tile_runtime, which loads per column pair.
#include <cstdlib>
#include <cstring>
#include "ptx.cuh"
#include "d3_internal.h"

namespace d3 {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int GEMM_THREADS = 384;

// ---------------------------------------------------------------------------------------------------------------
// Epilogue.  epi_value takes one element from the fp32 accumulator to the value stored; the two tile walkers below
// load its operands and store its results, and repeat none of its steps.  Every step is rounded on its own
// (__fmul_rn / __fadd_rn, GELU' spelled out in gelu_grad_epi), so no FMA contraction depends on the code around it and
// a fixed flag set gives the bits of the run-time flags.
constexpr int EPI_RUNTIME = -1;
constexpr int EPI_FLAGS = EP_BIAS | EP_GELU | EP_STORE_PRE | EP_MUL_DGELU | EP_GAMMA | EP_RESID | EP_OUT_F32 | EP_ACCUM |
                          EP_SLABS | EP_GELU_ERF;

// The epilogue stores through shared memory: every fixed flag set but the weight gradients' (split-K slabs, ACCUM),
// whose main loop runs over all tokens and so hides a register-store epilogue, and which keep the deeper ring.
template <int EF>
constexpr bool kStaged = EF != EPI_RUNTIME && (EF & (EP_SLABS | EP_ACCUM)) == 0;

// flag f: a compile-time constant for a fixed flag set EF, read from ep.flags for EPI_RUNTIME
template <int EF>
__device__ __forceinline__ bool epi_has(const GemmEpilogue& ep, int f) {
  return EF == EPI_RUNTIME ? (ep.flags & f) != 0 : (EF & f) != 0;
}

// gelu_tanh_grad_fast with every rounding step written out.  Its last add has a product on both sides, and which one
// the compiler contracts into an FMA depends on the surrounding code; fixing it to fma(0.5u (1 - t^2), dz, 0.5 (1 + t))
// makes the result independent of the code it is inlined into.
__device__ __forceinline__ float gelu_grad_epi(float u) {
  const float u2 = __fmul_rn(u, u);
  const float t = tanh_approx(__fmul_rn(u, fmaf(0.0356774081363001f, u2, 0.7978845608028654f)));
  const float dz = fmaf(0.1070322244089003f, u2, 0.7978845608028654f);
  return fmaf(__fmul_rn(__fmul_rn(0.5f, u), fmaf(-t, t, 1.0f)), dz, __fmul_rn(0.5f, __fadd_rn(1.0f, t)));
}

// the exact GELU 0.5 u (1 + erf(u / sqrt 2)) (torch nn.GELU(), the ConvNeXt block), each step rounded on its own
__device__ __forceinline__ float gelu_erf_epi(float u) {
  return __fmul_rn(__fmul_rn(0.5f, u), __fadd_rn(1.0f, erff(__fmul_rn(u, 0.70710678118654752f))));
}

// alpha, bias, GELU (tanh or erf), GELU' (of the bf16 pre-activation u), gamma, residual, accumulate (old: the fp32
// `out`), in this order; the operands of flags that are not set are ignored.  `pre` receives the value before the
// activation (EP_STORE_PRE).  The tanh-GELU and GELU' use the hardware tanh (rel. error 2^-11, below the bf16 rounding
// of the GEMM operands).
template <int EF>
__device__ __forceinline__ float epi_value(const GemmEpilogue& ep, float acc, float bias, float u, float gamma,
                                           float resid, float old, float& pre) {
  float v = __fmul_rn(acc, ep.alpha);
  if (epi_has<EF>(ep, EP_BIAS)) v = __fadd_rn(v, bias);
  pre = v;
  if (epi_has<EF>(ep, EP_GELU)) v = gelu_tanh_fast(v);
  if (epi_has<EF>(ep, EP_GELU_ERF)) v = gelu_erf_epi(v);
  if (epi_has<EF>(ep, EP_MUL_DGELU)) v = __fmul_rn(v, gelu_grad_epi(u));
  if (epi_has<EF>(ep, EP_GAMMA)) v = __fmul_rn(v, gamma);
  if (epi_has<EF>(ep, EP_RESID)) v = __fadd_rn(v, resid);
  if (epi_has<EF>(ep, EP_ACCUM)) v = __fadd_rn(v, old);
  return v;
}

// Columns (n, n + 1) of one row: one access of the pair when `vec`, else scalar accesses of the columns in range
// (`two`: n + 1 < N).
__device__ __forceinline__ float2 ld_pair(const float* p, bool vec, bool two) {
  if (vec) return *reinterpret_cast<const float2*>(p);
  return make_float2(p[0], two ? p[1] : 0.f);
}
__device__ __forceinline__ float2 ld_pair(const __nv_bfloat16* p, bool vec, bool two) {
  if (vec) return unpack_bf16(*reinterpret_cast<const uint32_t*>(p));
  return make_float2(__bfloat162float(p[0]), two ? __bfloat162float(p[1]) : 0.f);
}
__device__ __forceinline__ void st_pair(float* p, float a, float b, bool vec, bool two) {
  if (vec) {
    *reinterpret_cast<float2*>(p) = make_float2(a, b);
  } else {
    p[0] = a;
    if (two) p[1] = b;
  }
}
__device__ __forceinline__ void st_pair(__nv_bfloat16* p, float a, float b, bool vec, bool two) {
  if (vec) {
    *reinterpret_cast<uint32_t*>(p) = pack_bf16(a, b);
  } else {
    p[0] = __float2bfloat16(a);
    if (two) p[1] = __float2bfloat16(b);
  }
}

// Run-time flags (EPI_RUNTIME): the fused reduce-scatter, operands that fail gemm_bf16's alignment checks, odd N and
// flag sets not compiled fixed.  Each column pair loads its own operands (prefetching a row's under run-time flags
// would cost registers), with vector accesses unless EP_SLOW is set or N cuts the pair.
template <int BN>
__device__ __forceinline__ void epilogue_tile_runtime(const GemmEpilogue& ep, float (&acc)[2][BN / 2], int m0, int n0,
                                                      int M, int N, size_t slab_row0, int r_in, int c_in) {
  float* const out_f = reinterpret_cast<float*>(ep.out);
  __nv_bfloat16* const out_h = reinterpret_cast<__nv_bfloat16*>(ep.out);
  const bool aligned = (ep.flags & EP_SLOW) == 0;
#pragma unroll
  for (int mh = 0; mh < 2; ++mh)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const size_t row = (size_t)(m0 + mh * 64 + r_in + 8 * h);
      if (row >= (size_t)M) continue;
      const size_t orow = slab_row0 + row;
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        const int n = n0 + 8 * i + c_in;
        if (n >= N) break;
        const bool two = n + 1 < N, vec = aligned && two;
        float2 b{}, u{}, g{}, x{}, o{};
        if (epi_has<EPI_RUNTIME>(ep, EP_BIAS)) b = ld_pair(ep.bias + n, vec, two);
        if (epi_has<EPI_RUNTIME>(ep, EP_MUL_DGELU)) u = ld_pair(ep.aux_in + row * ep.ld_aux + n, vec, two);
        if (epi_has<EPI_RUNTIME>(ep, EP_GAMMA)) g = ld_pair(ep.gamma + n, vec, two);
        if (epi_has<EPI_RUNTIME>(ep, EP_RESID)) x = ld_pair(ep.resid + row * ep.ld_resid + n, vec, two);
        if (epi_has<EPI_RUNTIME>(ep, EP_ACCUM)) o = ld_pair(out_f + orow * ep.ld_out + n, vec, two);
        float p0, p1;
        const float v0 = epi_value<EPI_RUNTIME>(ep, acc[mh][4 * i + 2 * h], b.x, u.x, g.x, x.x, o.x, p0);
        const float v1 = epi_value<EPI_RUNTIME>(ep, acc[mh][4 * i + 2 * h + 1], b.y, u.y, g.y, x.y, o.y, p1);
        if (epi_has<EPI_RUNTIME>(ep, EP_SCATTER)) {   // add into the owning rank's shard slice (NVLink peer mapping)
          const unsigned long long g_idx = (unsigned long long)ep.sc_off + orow * ep.ld_out + n;
          const unsigned long long shard = (unsigned long long)ep.sc_shard;
          const unsigned r = (unsigned)(g_idx / shard);   // a pair never straddles two owners (shard % 4 == 0)
          float* const dst = ep.sc_peer[r] + (g_idx - r * shard);
          if (!two) atomicAdd(dst, v0);
          else atomicAdd(reinterpret_cast<float2*>(dst), make_float2(v0, v1));
          continue;
        }
        if (epi_has<EPI_RUNTIME>(ep, EP_STORE_PRE)) st_pair(ep.aux_out + row * ep.ld_aux + n, p0, p1, vec, two);
        if (epi_has<EPI_RUNTIME>(ep, EP_OUT_F32)) st_pair(out_f + orow * ep.ld_out + n, v0, v1, vec, two);
        else st_pair(out_h + orow * ep.ld_out + n, v0, v1, vec, two);
      }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Fixed flag sets EF, for a call that passed gemm_bf16's alignment checks and has an even N (a column pair is in range
// as a whole, and every access is a vector one).  The tile is walked in 64 x 64 chunks (a 64-row half by 64 columns);
// a thread issues every load of a chunk (`resid`, GELU' input, ACCUM `out`) before the chunk's first store, so it waits
// on memory once per chunk.  `resid` may alias `out`: each element is read before it is written, by the same thread.
// Two store back ends:
//   staged (kStaged<EF>): a chunk's outputs go to shared memory as 64-row boxes of 128 B rows (64 bf16 or 32 fp32
//     columns) in SWIZZLE_128B layout, so the fragment's st.shared of 8 consecutive rows hit 8 different 16-byte bank
//     groups, and leave by TMA in whole lines (from the fragment, a warp's store covers 8 rows x 16 B).  The
//     consumer's staging area holds NBUF chunks in a ring; thread 0 of the consumer commits one bulk group per chunk
//     and, after the chunk's loads are issued and before the chunk is written, waits until the group that last read
//     its buffer is done.  TMA clips rows >= M and columns >= N.
//   registers (the weight gradients): st.global from the fragment; split-K slab s at rows [s*M, s*M + M) of `out`.
constexpr int STG_BOX = 64 * 128;
constexpr int STG_BYTES = 3 * STG_BOX;    // per consumer
__device__ __forceinline__ uint32_t sw128(int r, int byte) {
  return r * 128 + ((((byte >> 4) ^ r) & 7) << 4) + (byte & 15);
}

// `acc` holds MH 64-row halves of BN columns: a whole 128-row tile (MH = 2) or, at BN = 256, the consumer's 64 rows
// starting at m0 (MH = 1).
template <int MH, int BN, int EF>
__device__ __forceinline__ void epilogue_tile(const GemmEpilogue& ep, const CUtensorMap* tm_out,
                                              const CUtensorMap* tm_pre, float (&acc)[MH][BN / 2], const float* s_bias,
                                              const float* s_gamma, uint8_t* stg, int& seq, int bar, int t, int m0,
                                              int n0, int M, int N, size_t slab_row0, int r_in, int c_in) {
  constexpr bool STAGED = kStaged<EF>;
  constexpr bool F32 = (EF & EP_OUT_F32) != 0;
  constexpr int OUT_BOXES = F32 ? 2 : 1;
  constexpr int CHUNK = (OUT_BOXES + ((EF & EP_STORE_PRE) ? 1 : 0)) * STG_BOX;
  constexpr int NBUF = STG_BYTES / CHUNK;
  static_assert(NBUF >= 1, "a chunk must fit the staging area");
  float* const out_f = reinterpret_cast<float*>(ep.out);
  __nv_bfloat16* const out_h = reinterpret_cast<__nv_bfloat16*>(ep.out);
#pragma unroll
  for (int mh = 0; mh < MH; ++mh)
#pragma unroll
    for (int cb = 0; cb < BN / 64; ++cb) {
      const int row0 = m0 + mh * 64, col0 = n0 + cb * 64;
      if (row0 >= M || col0 >= N) continue;   // uniform over the warpgroup
      float2 xr[2][8], xo[2][8];
      uint32_t xu[2][8];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const size_t row = (size_t)row0 + r_in + 8 * h;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int n = col0 + 8 * i + c_in;
          if (row < (size_t)M && n < N) {
            if (epi_has<EF>(ep, EP_RESID))
              xr[h][i] = *reinterpret_cast<const float2*>(ep.resid + row * ep.ld_resid + n);
            if (epi_has<EF>(ep, EP_MUL_DGELU))
              xu[h][i] = *reinterpret_cast<const uint32_t*>(ep.aux_in + row * ep.ld_aux + n);
            if (epi_has<EF>(ep, EP_ACCUM))
              xo[h][i] = *reinterpret_cast<const float2*>(out_f + (slab_row0 + row) * ep.ld_out + n);
          }
        }
      }
      uint8_t* const buf = stg + (seq % NBUF) * CHUNK;
      if constexpr (STAGED) {
        if (t == 0) tma_store_wait_read<NBUF - 1>();   // the group that last read `buf` is done
        named_bar_sync(bar, 128);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r_in + 8 * h;
        const size_t row = (size_t)row0 + r;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int cl = cb * 64 + 8 * i + c_in;   // column within the tile
          const int n = n0 + cl;
          const float2 b = epi_has<EF>(ep, EP_BIAS) ? *reinterpret_cast<const float2*>(s_bias + cl) : float2{};
          const float2 g = epi_has<EF>(ep, EP_GAMMA) ? *reinterpret_cast<const float2*>(s_gamma + cl) : float2{};
          const float2 u = epi_has<EF>(ep, EP_MUL_DGELU) ? unpack_bf16(xu[h][i]) : float2{};
          float p0, p1;
          const float v0 = epi_value<EF>(ep, acc[mh][4 * (cl >> 3) + 2 * h], b.x, u.x, g.x, xr[h][i].x, xo[h][i].x, p0);
          const float v1 = epi_value<EF>(ep, acc[mh][4 * (cl >> 3) + 2 * h + 1], b.y, u.y, g.y, xr[h][i].y, xo[h][i].y,
                                         p1);
          if constexpr (STAGED) {
            if (epi_has<EF>(ep, EP_STORE_PRE))
              *reinterpret_cast<uint32_t*>(buf + OUT_BOXES * STG_BOX + sw128(r, 16 * i + 2 * c_in)) = pack_bf16(p0, p1);
            if constexpr (F32) {
              *reinterpret_cast<float2*>(buf + (i >> 2) * STG_BOX + sw128(r, 32 * (i & 3) + 4 * c_in)) =
                  make_float2(v0, v1);
            } else {
              *reinterpret_cast<uint32_t*>(buf + sw128(r, 16 * i + 2 * c_in)) = pack_bf16(v0, v1);
            }
          } else if (row < (size_t)M && n < N) {
            if (epi_has<EF>(ep, EP_STORE_PRE)) st_pair(ep.aux_out + row * ep.ld_aux + n, p0, p1, true, true);
            if constexpr (F32) st_pair(out_f + (slab_row0 + row) * ep.ld_out + n, v0, v1, true, true);
            else st_pair(out_h + (slab_row0 + row) * ep.ld_out + n, v0, v1, true, true);
          }
        }
      }
      if constexpr (STAGED) {
        fence_proxy_async_smem();                // the writes above are visible to the TMA (async proxy)
        named_bar_sync(bar, 128);
        if (t == 0) {
          tma_store_2d(tm_out, buf, col0, row0);
          if (F32 && col0 + 32 < N) tma_store_2d(tm_out, buf + STG_BOX, col0 + 32, row0);
          if constexpr ((EF & EP_STORE_PRE) != 0) tma_store_2d(tm_pre, buf + OUT_BOXES * STG_BOX, col0, row0);
          tma_store_commit();
        }
        ++seq;
      }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// STAGED: the epilogue stores through shared memory, which takes one ring stage's worth of space (227 KB in all)
// WIDE (BN = 256): both consumers share each tile, so bias and gamma are staged once per tile
template <int BN, bool STAGED>
struct Cfg {
  static constexpr bool WIDE = BN == 256;
  static constexpr int STAGES = (BN == 256 ? 4 : BN == 128 ? 6 : 8) - (STAGED ? 1 : 0);
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int BAR_BYTES = 256;                       // full and empty mbarriers
  static constexpr int VEC_BYTES = (WIDE ? 1 : 2) * 2 * BN * 4;   // bias and gamma of a tile (fp32), per consumer
  static constexpr int VEC_END = STAGES * STAGE_BYTES + BAR_BYTES + VEC_BYTES;
  static constexpr int STG_OFF = (VEC_END + 1023) / 1024 * 1024;   // SWIZZLE_128B staging: 1024-byte aligned
  static constexpr int SMEM_BYTES = (STAGED ? STG_OFF + 2 * STG_BYTES : VEC_END) + 1024;
  static_assert(SMEM_BYTES <= 227 * 1024, "over the opt-in shared-memory limit");
};

// work item = (tile pair, split), walked by both CTAs of a cluster, k-blocks [kb0, kb1).  BN = 64 / 128: the pair is
// (m tile, pair of N tiles) and CTA `rank` takes N tile 2 * pair + rank; BN = 256: the pair is (pair of M tiles, N tile)
// and CTA `rank` takes M tile 2 * pair + rank.  The second tile of a ragged pair lies wholly beyond N or M.
// `num_n`: N positions of the list (pairs of N tiles, or N tiles at BN = 256); `num_tiles`: tile pairs per split.
struct WorkRange { int m0, n0, kb0, kb1, sp; };
// Tiles are rasterised N-fastest: the CTAs resident at any moment cover a few M row-panels times all N tiles, so the
// large activation operand streams from HBM once while the (small) weight operand stays L2-resident.  Splits are the
// slowest index: the items resident at once read the same k-range of both operands, which L2 holds for all of them
// (split-fastest, every resident slice read its own k-range, and the weight gradients split over the tokens streamed
// each from HBM).  The order items run in does not change their sums or the slab order.
template <int BN>
__device__ __forceinline__ WorkRange work_item(int w, int rank, int num_n, int num_tiles, int num_k, int splits) {
  const int tile = w % num_tiles, sp = w / num_tiles;
  const int per = (num_k + splits - 1) / splits;
  WorkRange r;
  if constexpr (BN == 256) {
    r.n0 = (tile % num_n) * BN;
    r.m0 = (2 * (tile / num_n) + rank) * BM;
  } else {
    r.n0 = (2 * (tile % num_n) + rank) * BN;
    r.m0 = (tile / num_n) * BM;
  }
  r.kb0 = sp * per;
  r.kb1 = min(num_k, r.kb0 + per);
  r.sp = sp;
  return r;
}

// MH 64-row halves of A starting at `sa` (A rows 64-127 start 8 KB into the stage in both layouts: 64 rows x 128 B, or
// the second 64-row box) times all BN columns of B, one wgmma chain per half
template <int MH, int BN, int A_MN, int B_MN>
__device__ __forceinline__ void mma_kblock(float (&acc)[MH][BN / 2], uint32_t sa, uint32_t sb, bool first) {
  const uint64_t bd = B_MN ? gmma_desc_sw128(sb, 8192, 1024) : gmma_desc_sw128(sb, 16, 1024);
  constexpr uint64_t a_adv = A_MN ? (2048 >> 4) : (32 >> 4);
  constexpr uint64_t b_adv = B_MN ? (2048 >> 4) : (32 >> 4);
#pragma unroll
  for (int k = 0; k < BK / 16; ++k) {
    const uint32_t sc = (first && k == 0) ? 0u : 1u;
#pragma unroll
    for (int mh = 0; mh < MH; ++mh) {
      const uint64_t ad = A_MN ? gmma_desc_sw128(sa + mh * 8192, 8192, 1024) : gmma_desc_sw128(sa + mh * 8192, 16, 1024);
      if constexpr (BN == 256) wgmma_m64n256k16_ss<A_MN, B_MN>(acc[mh], ad + k * a_adv, bd + k * b_adv, sc);
      else if constexpr (BN == 128) wgmma_m64n128k16_ss<A_MN, B_MN>(acc[mh], ad + k * a_adv, bd + k * b_adv, sc);
      else wgmma_m64n64k16_ss<A_MN, B_MN>(acc[mh], ad + k * a_adv, bd + k * b_adv, sc);
    }
  }
}

// E4M3 (both operands K-major): a 128-element k-block of 128-byte rows has the same SWIZZLE_128B layout as a bf16
// k-block of 64; a k32 step advances 32 bytes.  This is half of it, k32 steps 2 h and 2 h + 1, chained from zero: the
// caller promotes the sum into the fp32 accumulator.
template <int MH, int BN>
__device__ __forceinline__ void mma_khalf_e4m3(float (&acc)[MH][BN / 2], uint32_t sa, uint32_t sb, int h) {
  static_assert(BN == 64, "the e4m3 GEMM runs 128 x 64 tiles");
  const uint64_t bd = gmma_desc_sw128(sb, 16, 1024);
#pragma unroll
  for (int k = 0; k < 2; ++k) {
#pragma unroll
    for (int mh = 0; mh < MH; ++mh) {
      const uint64_t ad = gmma_desc_sw128(sa + mh * 8192, 16, 1024);
      wgmma_m64n64k32_e4m3(acc[mh], ad + (2 * h + k) * (32 >> 4), bd + (2 * h + k) * (32 >> 4), k == 0 ? 0u : 1u);
    }
  }
}

template <int MH, int BN>
__device__ __forceinline__ void add_acc(float (&acc)[MH][BN / 2], const float (&part)[MH][BN / 2]) {
#pragma unroll
  for (int mh = 0; mh < MH; ++mh)
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[mh][i] = __fadd_rn(acc[mh][i], part[mh][i]);
}

// E4M3 = true: A [M, K] and B [N, K] are e4m3 bytes (K-major), sa [M] / sb [N] their power-of-two row scales.  Every 64
// k-elements (half a k-block) the tensor core's sum goes into a zeroed temporary that is added to the fp32 accumulator
// once it completes (two-level FP8 accumulation: the tensor core's FP8 sums keep fewer bits than fp32; promoting every
// 128 left 6.8e-4 relative error at K = 4096 on all-positive operands).  The add waits for the wgmma: a second
// temporary to overlap them would take the consumer past the 168 registers a thread of a 384-thread CTA is compiled
// for, and reading one while the other is in flight serializes the wgmma (C7514).
// The accumulator is multiplied by sa[m] sb[n] (exact: powers of two) before the epilogue.
template <int BN, int A_MN, int B_MN, int EF, bool E4M3 = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
            const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmP, const GemmEpilogue ep,
            int M, int N, int K, int splits, const float* scale_a, const float* scale_b) {
  static_assert(!E4M3 || (BN == 64 && !A_MN && !B_MN), "e4m3: 128 x 64 tiles, both operands K-major");
  constexpr int KB = E4M3 ? 128 : BK;    // elements per k-block (128 bytes per row either way)
  constexpr bool staged = kStaged<EF>;   // tmO / tmP (out, pre-activation stash) are used only then
  using C = Cfg<BN, staged>;
  constexpr bool WIDE = C::WIDE;
  constexpr int MH = WIDE ? 1 : 2;       // 64-row halves of a tile one consumer computes
  static_assert(!WIDE || EF != EPI_RUNTIME, "run-time flags run on the 128-wide tile");
  static_assert(2 * C::STAGES * 8 <= C::BAR_BYTES, "mbarriers overflow their slot");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + C::STAGES * C::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + C::STAGES;
  float* vecs = reinterpret_cast<float*>(smem + C::STAGES * C::STAGE_BYTES + C::BAR_BYTES);

  const int wg = threadIdx.x >> 7;
  const int rank = blockIdx.x & 1;                  // CTA within the cluster (cluster dims {2, 1, 1})
  const int cluster = blockIdx.x >> 1, num_clusters = gridDim.x >> 1;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if constexpr (staged) {
      tma_prefetch_desc(&tmO);
      if constexpr ((EF & EP_STORE_PRE) != 0) tma_prefetch_desc(&tmP);
    }
    // a stage is released by every consumer that reads it, in both CTAs
    for (int s = 0; s < C::STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], WIDE ? 4 : 2); }
    fence_mbar_init();
  }
  cluster_sync();   // both CTAs' barriers are initialised before either multicasts into or arrives on the other's

  const int num_m = (M + BM - 1) / BM;
  const int num_n = WIDE ? (N + BN - 1) / BN : ((N + BN - 1) / BN + 1) / 2;
  const int num_k = (K + KB - 1) / KB;
  const int num_tiles = (WIDE ? (num_m + 1) / 2 : num_m) * num_n;
  const int num_work = num_tiles * splits;

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (threadIdx.x < 32 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int w = cluster; w < num_work; w += num_clusters) {
        const WorkRange wr = work_item<BN>(w, rank, num_n, num_tiles, num_k, splits);
        for (int kb = wr.kb0; kb < wr.kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * C::STAGE_BYTES;
          uint8_t* sb = sa + C::A_BYTES;
          // the shared operand: this CTA's half goes to both CTAs, the peer's half completes the stage's bytes
          mbar_expect_tx(&full_bar[stage], C::STAGE_BYTES);
          if constexpr (WIDE) {            // own 128 rows of A (two 64-row boxes), 128-column half of B to both
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              if (A_MN) tma_load_2d(&tmA, &full_bar[stage], sa + i * 8192, wr.m0 + i * 64, kb * KB);
              else tma_load_2d(&tmA, &full_bar[stage], sa + i * 8192, kb * KB, wr.m0 + i * 64);
            }
            if (B_MN) {
#pragma unroll
              for (int i = 2 * rank; i < 2 * rank + 2; ++i)
                tma_load_2d_multicast(&tmB, &full_bar[stage], sb + i * 8192, wr.n0 + i * 64, kb * KB, 0b11);
            } else {
              tma_load_2d_multicast(&tmB, &full_bar[stage], sb + rank * 16384, kb * KB, wr.n0 + rank * 128, 0b11);
            }
          } else {                         // 64-row half of A to both, own B
            if (A_MN) {
              tma_load_2d_multicast(&tmA, &full_bar[stage], sa + rank * 8192, wr.m0 + rank * 64, kb * KB, 0b11);
            } else {
              tma_load_2d_multicast(&tmA, &full_bar[stage], sa + rank * 8192, kb * KB, wr.m0 + rank * 64, 0b11);
            }
            if (B_MN) {
#pragma unroll
              for (int i = 0; i < BN / 64; ++i) tma_load_2d(&tmB, &full_bar[stage], sb + i * 8192, wr.n0 + i * 64, kb * KB);
            } else {
              tma_load_2d(&tmB, &full_bar[stage], sb, kb * KB, wr.n0);
            }
          }
          if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    // consumer warpgroup: in ping-pong, tiles j of this CTA with j % 2 == cw; WIDE, rows 64 cw .. 64 cw + 63 of every
    // tile
    const int cw = wg - 1;
    const int t = threadIdx.x & 127;
    const int r_in = 16 * (t >> 5) + ((t & 31) >> 2);
    const int c_in = 2 * (t & 3);
    float* const s_bias = vecs + (WIDE ? 0 : cw * 2 * BN);
    float* const s_gamma = s_bias + BN;
    constexpr bool stage_vecs = EF != EPI_RUNTIME && (EF & (EP_BIAS | EP_GAMMA)) != 0;
    constexpr int VEC_THREADS = WIDE ? 256 : 128;   // the consumers that read s_bias / s_gamma
    const int vt = WIDE ? threadIdx.x - 128 : t;
    uint8_t* const stg = smem + C::STG_OFF + cw * STG_BYTES;   // output staging (staged epilogues only)
    const uint32_t peer_empty = mapa_shared(smem_u32(empty_bar), rank ^ 1);   // the peer's empty barriers
    int stg_seq = 0;                           // chunks this consumer has staged
    int stage = 0;                             // position in the ring, counting the other consumer's k-blocks too
    uint32_t phase = 0;
    int j = 0;
    for (int w = cluster; w < num_work; w += num_clusters, ++j) {
      const WorkRange wr = work_item<BN>(w, rank, num_n, num_tiles, num_k, splits);
      const int nkb = wr.kb1 > wr.kb0 ? wr.kb1 - wr.kb0 : 0;
      if (!WIDE && (j & 1) != cw) {            // the other consumer's tile: step over its fills
        stage += nkb;
        phase ^= (stage / C::STAGES) & 1;
        stage %= C::STAGES;
        continue;
      }
      if constexpr (stage_vecs) {
        named_bar_sync(3 + cw * !WIDE, VEC_THREADS);   // the previous epilogue has read bias / gamma
        if (vt < BN && wr.n0 + vt < N) {
          if constexpr ((EF & EP_BIAS) != 0) cp_async_4(s_bias + vt, ep.bias + wr.n0 + vt);
          if constexpr ((EF & EP_GAMMA) != 0) cp_async_4(s_gamma + vt, ep.gamma + wr.n0 + vt);
        }
      }
      if (!WIDE && j > 0) named_bar_sync(1 + cw, 256);   // tile j-1's main loop has passed its last full-barrier wait
      float acc[MH][BN / 2];
#pragma unroll
      for (int mh = 0; mh < MH; ++mh)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[mh][i] = 0.f;
      if constexpr (E4M3) {
        float part[MH][BN / 2];
        for (int kb = wr.kb0; kb < wr.kb1; ++kb) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t sa = smem_u32(smem + stage * C::STAGE_BYTES);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int mh = 0; mh < MH; ++mh) fence_regs(part[mh]);
            wgmma_fence();
            mma_khalf_e4m3<MH, BN>(part, sa, sa + C::A_BYTES, h);
            wgmma_commit();
            wgmma_wait<0>();
#pragma unroll
            for (int mh = 0; mh < MH; ++mh) fence_regs(part[mh]);
            if (h == 1 && t == 0) { mbar_arrive(&empty_bar[stage]); mbar_arrive_cluster(peer_empty + 8 * stage); }
            add_acc<MH, BN>(acc, part);
          }
          if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
        }
        if (!WIDE && w + num_clusters < num_work) named_bar_arrive(1 + (cw ^ 1), 256);   // tile j+1 may start its main loop
        // dequantise: rows r_in, r_in + 8 of each 64-row half, columns 8 i + c_in, + 1
#pragma unroll
        for (int mh = 0; mh < MH; ++mh)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = wr.m0 + mh * 64 + r_in + 8 * h;
            const float s_row = row < M ? scale_a[row] : 0.f;
#pragma unroll
            for (int i = 0; i < BN / 8; ++i) {
              const int n = wr.n0 + 8 * i + c_in;
              const float s0 = n < N ? scale_b[n] : 0.f, s1 = n + 1 < N ? scale_b[n + 1] : 0.f;
              acc[mh][4 * i + 2 * h] = __fmul_rn(__fmul_rn(acc[mh][4 * i + 2 * h], s_row), s0);
              acc[mh][4 * i + 2 * h + 1] = __fmul_rn(__fmul_rn(acc[mh][4 * i + 2 * h + 1], s_row), s1);
            }
          }
      } else {
        int prev = -1;
        for (int kb = wr.kb0; kb < wr.kb1; ++kb) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t sa = smem_u32(smem + stage * C::STAGE_BYTES);
#pragma unroll
          for (int mh = 0; mh < MH; ++mh) fence_regs(acc[mh]);
          wgmma_fence();
          mma_kblock<MH, BN, A_MN, B_MN>(acc, sa + (WIDE ? cw * 8192 : 0), sa + C::A_BYTES, kb == wr.kb0);
          wgmma_commit();
#pragma unroll
          for (int mh = 0; mh < MH; ++mh) fence_regs(acc[mh]);
          if (prev >= 0) {                       // the k-block before this one has been consumed: release its stage
            wgmma_wait<1>();
            if (t == 0) { mbar_arrive(&empty_bar[prev]); mbar_arrive_cluster(peer_empty + 8 * prev); }
          }
          prev = stage;
          if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
        }
        if (!WIDE && w + num_clusters < num_work) named_bar_arrive(1 + (cw ^ 1), 256);   // tile j+1 may start its main loop
        wgmma_wait<0>();
#pragma unroll
        for (int mh = 0; mh < MH; ++mh) fence_regs(acc[mh]);
        if (prev >= 0 && t == 0) { mbar_arrive(&empty_bar[prev]); mbar_arrive_cluster(peer_empty + 8 * prev); }
      }
      if constexpr (stage_vecs) {
        cp_async_wait_all();
        named_bar_sync(3 + cw * !WIDE, VEC_THREADS);   // bias / gamma of this tile are in shared memory
      }
      if (nkb <= 0) continue;                  // empty split-K slice: nothing to add
      const size_t slab_row0 = epi_has<EF>(ep, EP_SLABS) ? (size_t)wr.sp * M : 0;
      if constexpr (EF == EPI_RUNTIME) {
        epilogue_tile_runtime<BN>(ep, acc, wr.m0, wr.n0, M, N, slab_row0, r_in, c_in);
      } else {
        epilogue_tile<MH, BN, EF>(ep, &tmO, &tmP, acc, s_bias, s_gamma, stg, stg_seq, 5 + cw, t,
                                  wr.m0 + (WIDE ? cw * 64 : 0), wr.n0, M, N, slab_row0, r_in, c_in);
      }
    }
    if (staged && t == 0) tma_store_wait_all();   // shared memory stays valid until the last store has read it
  }
  cluster_sync();   // neither CTA exits while the peer may still arrive on its barriers
}

// ------------------------------------------------------------------------------------------------ host side
static int make_operand_map(CUtensorMap* map, const void* ptr, int mn, int k, int ld, int is_mn_major, int box_mn) {
  // K-major : memory [mn][k], row stride ld   -> dims {k, mn}, box {64, box_mn}
  // MN-major: memory [k][mn], row stride ld   -> dims {mn, k}, box {64, 64}
  cuuint64_t dims[2], strides[1];
  cuuint32_t box[2], estr[2] = {1, 1};
  if (is_mn_major) {
    dims[0] = (cuuint64_t)mn; dims[1] = (cuuint64_t)k; box[0] = 64; box[1] = 64;
  } else {
    dims[0] = (cuuint64_t)k; dims[1] = (cuuint64_t)mn; box[0] = 64; box[1] = (cuuint32_t)box_mn;
  }
  strides[0] = (cuuint64_t)ld * 2;
  return encode_tensor_map_2d_bf16(map, ptr, dims, strides, box, estr);
}

template <int BN, int A_MN, int B_MN, int EF, bool E4M3 = false>
static int launch(const CUtensorMap& ta, const CUtensorMap& tb, const GemmEpilogue& ep, int M, int N, int K,
                  int splits, cudaStream_t stream, const float* scale_a = nullptr, const float* scale_b = nullptr) {
  using C = Cfg<BN, kStaged<EF>>;
  auto kern = gemm_kernel<BN, A_MN, B_MN, EF, E4M3>;
  cudaLaunchAttribute attr{};
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = 2;
  attr.val.clusterDim.y = 1;
  attr.val.clusterDim.z = 1;
  cudaLaunchConfig_t cfg{};
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = C::SMEM_BYTES;
  cfg.stream = stream;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  // persistent grid: as many clusters as can be resident at once (GPCs need not hold an even number of free SMs)
  static int max_clusters = 0;
  if (max_clusters == 0) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    if (e != cudaSuccess) return set_error(D3_ERR_CUDA, cudaGetErrorString(e));
    cfg.gridDim = dim3(2 * sm_count());
    e = cudaOccupancyMaxActiveClusters(&max_clusters, kern, &cfg);
    if (e != cudaSuccess) return set_error(D3_ERR_CUDA, cudaGetErrorString(e));
    if (max_clusters < 1) return set_error(D3_ERR_CUDA, "gemm: no 2-CTA cluster fits on the device");
  }
  // output maps of the staged epilogue: the logical [M, N] with the real leading dimension, so TMA clips ragged rows
  // and columns (gemm_bf16's alignment checks already meet TMA's 16-byte address and stride rules)
  CUtensorMap to{}, tp{};
  if constexpr (kStaged<EF>) {
    const int elt = (EF & EP_OUT_F32) ? 4 : 2;
    int rc = encode_tensor_map_2d(&to, ep.out, elt, N, M, (cuuint64_t)ep.ld_out * elt, 128 / elt, 64, 128);
    if (rc) return rc;
    if constexpr ((EF & EP_STORE_PRE) != 0) {
      rc = encode_tensor_map_2d(&tp, ep.aux_out, 2, N, M, (cuuint64_t)ep.ld_aux * 2, 64, 64, 128);
      if (rc) return rc;
    }
  }
  const int num_m = (M + BM - 1) / BM, num_n = (N + BN - 1) / BN;
  const int work = (BN == 256 ? (num_m + 1) / 2 * num_n : num_m * ((num_n + 1) / 2)) * splits;   // tile pairs
  cfg.gridDim = dim3(2 * (work < max_clusters ? work : max_clusters));
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, ta, tb, to, tp, ep, M, N, K, splits, scale_a, scale_b);
  if (e == cudaSuccess) e = cudaPeekAtLastError();
  if (e != cudaSuccess) return set_error(D3_ERR_CUDA, cudaGetErrorString(e));
  count_launch();
  return D3_OK;
}

template <int BN>
static int dispatch(int a_mn, int b_mn, const CUtensorMap& ta, const CUtensorMap& tb, const GemmEpilogue& ep, int M,
                    int N, int K, int splits, cudaStream_t s) {
  // (A layout, B layout, flags) of the calls in one training step, compiled with their epilogue fixed
  if (!(ep.flags & (EP_SLOW | EP_SCATTER)) && N % 2 == 0) {
    const int f = ep.flags & EPI_FLAGS;
#define D3_EPI(A, B, F) \
    if (a_mn == A && b_mn == B && f == (F)) return launch<BN, A, B, (F)>(ta, tb, ep, M, N, K, splits, s);
    // forward: qkv, patch embedding and head layers, fc1, proj, fc2, prototype logits; qkv without a bias (vit_7b)
    D3_EPI(0, 1, 0)
    D3_EPI(0, 1, EP_BIAS)
    D3_EPI(0, 1, EP_BIAS | EP_OUT_F32)
    D3_EPI(0, 1, EP_BIAS | EP_GELU)
    D3_EPI(0, 1, EP_BIAS | EP_GELU | EP_STORE_PRE)
    D3_EPI(0, 1, EP_BIAS | EP_GAMMA | EP_RESID | EP_OUT_F32)
    D3_EPI(0, 1, EP_BIAS | EP_STORE_PRE | EP_GAMMA | EP_RESID | EP_OUT_F32)
    D3_EPI(0, 1, EP_BIAS | EP_GELU | EP_GAMMA | EP_RESID | EP_OUT_F32)
    D3_EPI(0, 1, EP_BIAS | EP_GELU | EP_STORE_PRE | EP_GAMMA | EP_RESID | EP_OUT_F32)
    D3_EPI(0, 1, EP_OUT_F32)
    // ConvNeXt pwconv1 (the exact GELU); its pwconv2 is the bias + gamma + residual instance above
    D3_EPI(0, 1, EP_BIAS | EP_GELU_ERF)
    // input gradients
    D3_EPI(0, 0, 0)
    D3_EPI(0, 0, EP_MUL_DGELU)
    D3_EPI(0, 0, EP_OUT_F32)
    // weight gradients: split-K slabs, or accumulated in place
    D3_EPI(1, 1, EP_OUT_F32 | EP_SLABS)
    D3_EPI(1, 1, EP_OUT_F32 | EP_ACCUM)
#undef D3_EPI
  }
  // Every other call (run-time flags: D3_EP_SCATTER, misaligned operands, odd N, other flag sets) runs on a 64- or
  // 128-wide tile: the run-time-flag epilogue is not compiled at BN = 256, whose operand maps are those of BN = 128.
  if constexpr (BN == 256) {
    return dispatch<128>(a_mn, b_mn, ta, tb, ep, M, N, K, splits, s);
  } else {
    if (!a_mn && !b_mn) return launch<BN, 0, 0, EPI_RUNTIME>(ta, tb, ep, M, N, K, splits, s);
    if (!a_mn && b_mn) return launch<BN, 0, 1, EPI_RUNTIME>(ta, tb, ep, M, N, K, splits, s);
    if (a_mn && !b_mn) return launch<BN, 1, 0, EPI_RUNTIME>(ta, tb, ep, M, N, K, splits, s);
    return launch<BN, 1, 1, EPI_RUNTIME>(ta, tb, ep, M, N, K, splits, s);
  }
}

// tile_n: 0 = auto (256 for weight gradients, else 64 or 128); 64 / 128 / 256 force that tile width; 512 is taken as
// 256, the widest tile.
// split_k: 0 = auto (only when the epilogue is a plain fp32 accumulate-able output), >= 1 forced.
int gemm_bf16(const void* A, int lda, int a_mn, const void* B, int ldb, int b_mn, int M, int N, int K,
              GemmEpilogue ep, int tile_n, int split_k, cudaStream_t stream) {
  if (M <= 0 || N <= 0 || K <= 0) return set_error(D3_ERR_ARG, "gemm: empty problem");
  if ((lda % 8) || (ldb % 8) || (reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(B) & 15))
    return set_error(D3_ERR_ARG, "gemm: operands must be 16-byte aligned with ld % 8 == 0");
  const int sms = sm_count();
  const int num_k = (K + BK - 1) / BK;
  // ---- tile choice: fewest waves of (tile width + fixed per-tile cost) over the SMs.  BN = 256 is not a candidate
  //      here: at every forward and input-gradient shape of a ViT-L step it measured slower than 128 (DESIGN.md
  //      section 4); the weight gradients take it below, after their split count
  int bn = tile_n >= 256 ? 256 : tile_n;
  if (tile_n == 0) {
    const int cand[2] = {128, 64};
    long best = -1;
    for (int i = 0; i < 2; ++i) {
      const long tiles = (long)((M + BM - 1) / BM) * ((N + cand[i] - 1) / cand[i]);
      const long waves = (tiles + sms - 1) / sms;
      const long cost = waves * (cand[i] + 24);
      if (best < 0 || cost < best) { best = cost; bn = cand[i]; }
    }
  }
  // ---- split-K: only for plain fp32 outputs (weight gradients) accumulated into (EP_ACCUM); every slice stores its
  //      partial tile into a workspace and the slices are added to out in slice order (reproducible bit for bit)
  const bool plain_f32 = (ep.flags & EP_OUT_F32) && !(ep.flags & (EP_BIAS | EP_GELU | EP_STORE_PRE | EP_MUL_DGELU |
                                                                  EP_GAMMA | EP_RESID | EP_GELU_ERF));
  int splits = 1;
  if (split_k >= 1) {
    splits = split_k;
  } else if (plain_f32 && (ep.flags & EP_ACCUM)) {
    const int unit_n = bn < 128 ? bn : 128;   // the tile widths before BN = 256 (its split counts and bits)
    const long units = (long)((M + BM - 1) / BM) * ((N + unit_n - 1) / unit_n);
    if (units <= sms && num_k >= 16) {
      // fill the SMs; and keep every accumulation chain within 64 k-blocks: the tensor core's fp32 accumulation drifts
      // measurably (> 1e-5 relative) over longer chains, the fp32 reduction of the slices does not
      splits = units * 2 <= sms ? (int)(sms / units) : 1;
      if (splits < (num_k + 63) / 64) splits = (num_k + 63) / 64;
      if (splits > num_k / 4) splits = num_k / 4;
      if (splits < 1) splits = 1;
    }
  }
  // weight gradients (both operands MN-major) run on the 128 x 256 tile: its M-paired clusters read a third fewer
  // operand bytes from L2 per FLOP, and their main loops run over the tokens, so the epilogue it does not hide is a
  // small part of a tile's time.  The split count above stays that of the narrower tile, and so do the bits.
  if (tile_n == 0 && a_mn && b_mn) bn = 256;
  if (ep.flags & EP_SCATTER) {
    if (!plain_f32) return set_error(D3_ERR_ARG, "gemm: SCATTER needs a plain fp32 output");
    if (ep.sc_world < 1 || ep.sc_world > 8 || ep.sc_shard <= 0 || (ep.sc_shard % 4) || (ep.sc_off % 4) || (ep.ld_out % 4))
      return set_error(D3_ERR_ARG, "gemm: SCATTER needs 1..8 ranks and 4-element aligned shard / offset / ld_out");
    if ((unsigned long long)ep.sc_off + (unsigned long long)(M - 1) * ep.ld_out + N > (unsigned long long)ep.sc_shard * ep.sc_world)
      return set_error(D3_ERR_ARG, "gemm: SCATTER output exceeds the sharded range");
  }
  if (splits > 1) {
    if (!plain_f32) return set_error(D3_ERR_ARG, "gemm: split-K needs a plain fp32 output");
    if (!(ep.flags & EP_ACCUM)) return set_error(D3_ERR_ARG, "gemm: split-K accumulates into out (set ACCUM, zero it first)");
    if (splits > num_k) splits = num_k;
  }
  // every SCATTER contribution is an atomic add into the owners' shards (other ranks add into the same slice): `out`
  // is neither read nor written
  if (ep.flags & EP_SCATTER) ep.flags &= ~EP_ACCUM;
  // ---- epilogue fast-path eligibility
  const int out_elt = (ep.flags & EP_OUT_F32) ? 4 : 2;
  bool aligned = ((uintptr_t)ep.out % 16 == 0) && ((ep.ld_out * out_elt) % 16 == 0);
  if (ep.flags & EP_BIAS) aligned = aligned && ((uintptr_t)ep.bias % 16 == 0);
  if (ep.flags & EP_GAMMA) aligned = aligned && ((uintptr_t)ep.gamma % 16 == 0);
  if (ep.flags & EP_RESID) aligned = aligned && ((uintptr_t)ep.resid % 16 == 0) && (ep.ld_resid % 4 == 0);
  if (ep.flags & EP_STORE_PRE) aligned = aligned && ((uintptr_t)ep.aux_out % 16 == 0) && (ep.ld_aux % 8 == 0);
  if (ep.flags & EP_MUL_DGELU) aligned = aligned && ((uintptr_t)ep.aux_in % 16 == 0) && (ep.ld_aux % 8 == 0);
  if (!aligned) ep.flags |= EP_SLOW;

  CUtensorMap ta, tb;
  int rc = make_operand_map(&ta, A, M, K, lda, a_mn, 64);   // A arrives as two 64-row halves, one per cluster CTA
  if (rc) return rc;
  rc = make_operand_map(&tb, B, N, K, ldb, b_mn, bn < 128 ? bn : 128);   // BN = 256: one 128-row half per cluster CTA
  if (rc) return rc;
  float* ws = nullptr;
  GemmEpilogue out_ep = ep;
  if (splits > 1 && !(ep.flags & EP_SCATTER)) {   // slices -> [splits * M, N] workspace, then the ordered reduction
    ws = slab_workspace((size_t)splits * M * N, stream);
    if (!ws) return D3_ERR_CUDA;
    ep.out = ws;
    ep.ld_out = N;
    ep.flags = (ep.flags & ~(EP_ACCUM | EP_SLOW)) | EP_SLABS | (N % 4 ? EP_SLOW : 0);
  }
  switch (bn) {
    case 256: rc = dispatch<256>(a_mn, b_mn, ta, tb, ep, M, N, K, splits, stream); break;
    case 128: rc = dispatch<128>(a_mn, b_mn, ta, tb, ep, M, N, K, splits, stream); break;
    case 64: rc = dispatch<64>(a_mn, b_mn, ta, tb, ep, M, N, K, splits, stream); break;
    default: rc = set_error(D3_ERR_ARG, "gemm: bad tile N");
  }
  if (ws) {
    if (!rc) rc = slab_combine(ws, splits, (long long)M * N, M, N, reinterpret_cast<float*>(out_ep.out), out_ep.ld_out, stream);
    slab_release(ws, stream);
  }
  return rc;
}

// ---------------------------------------------------------------------------------------------------------------
// E4M3: out = epilogue(alpha * (A B^T) * sa[m] * sb[n]), A [M, K] and B [N, K] e4m3 bytes, K-major (FP8 wgmma has no
// transpose bits), on 128 x 64 tiles: two m64n64 chains and their two promotion temporaries fit a consumer's registers,
// two m64n128 chains would not.  No split-K and no scatter: the block linears' forward and input-gradient GEMMs.
static int dispatch_e4m3(const CUtensorMap& ta, const CUtensorMap& tb, const GemmEpilogue& ep, int M, int N, int K,
                         const float* sa, const float* sb, cudaStream_t s) {
  if (!(ep.flags & EP_SLOW) && N % 2 == 0) {
    const int f = ep.flags & EPI_FLAGS;
#define D3_EPI(F) \
    if (f == (F)) return launch<64, 0, 0, (F), true>(ta, tb, ep, M, N, K, 1, s, sa, sb);
    // forward: qkv (with and without a bias), fc1 / w1 / w2, proj, fc2 / w3 (with and without the stash)
    D3_EPI(0)
    D3_EPI(EP_BIAS)
    D3_EPI(EP_BIAS | EP_GELU)
    D3_EPI(EP_BIAS | EP_GELU | EP_STORE_PRE)
    D3_EPI(EP_BIAS | EP_GAMMA | EP_RESID | EP_OUT_F32)
    D3_EPI(EP_BIAS | EP_STORE_PRE | EP_GAMMA | EP_RESID | EP_OUT_F32)
    D3_EPI(EP_BIAS | EP_GELU | EP_GAMMA | EP_RESID | EP_OUT_F32)
    D3_EPI(EP_BIAS | EP_GELU | EP_STORE_PRE | EP_GAMMA | EP_RESID | EP_OUT_F32)
    // input gradients: dQKV / dP Wᵀ, fc2's through GELU', swiglu's fp32 dz = dx1 W1ᵀ + dx2 W2ᵀ
    D3_EPI(EP_MUL_DGELU)
    D3_EPI(EP_OUT_F32)
    D3_EPI(EP_OUT_F32 | EP_ACCUM)
#undef D3_EPI
  }
  return launch<64, 0, 0, EPI_RUNTIME, true>(ta, tb, ep, M, N, K, 1, s, sa, sb);
}

int gemm_e4m3(const void* A, int lda, const float* sa, const void* B, int ldb, const float* sb, int M, int N, int K,
              GemmEpilogue ep, cudaStream_t stream) {
  if (M <= 0 || N <= 0 || K <= 0) return set_error(D3_ERR_ARG, "gemm_e4m3: empty problem");
  if (K % 16) return set_error(D3_ERR_ARG, "gemm_e4m3: K must be a multiple of 16");
  if ((lda % 16) || (ldb % 16) || (reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(B) & 15))
    return set_error(D3_ERR_ARG, "gemm_e4m3: operands must be 16-byte aligned with ld % 16 == 0");
  if (ep.flags & (EP_SCATTER | EP_GELU_ERF)) return set_error(D3_ERR_ARG, "gemm_e4m3: SCATTER / GELU_ERF not supported");
  const int out_elt = (ep.flags & EP_OUT_F32) ? 4 : 2;
  bool aligned = ((uintptr_t)ep.out % 16 == 0) && ((ep.ld_out * out_elt) % 16 == 0);
  if (ep.flags & EP_BIAS) aligned = aligned && ((uintptr_t)ep.bias % 16 == 0);
  if (ep.flags & EP_GAMMA) aligned = aligned && ((uintptr_t)ep.gamma % 16 == 0);
  if (ep.flags & EP_RESID) aligned = aligned && ((uintptr_t)ep.resid % 16 == 0) && (ep.ld_resid % 4 == 0);
  if (ep.flags & EP_STORE_PRE) aligned = aligned && ((uintptr_t)ep.aux_out % 16 == 0) && (ep.ld_aux % 8 == 0);
  if (ep.flags & EP_MUL_DGELU) aligned = aligned && ((uintptr_t)ep.aux_in % 16 == 0) && (ep.ld_aux % 8 == 0);
  if (!aligned) ep.flags |= EP_SLOW;
  CUtensorMap ta, tb;
  int rc = encode_tensor_map_2d_u8(&ta, A, K, M, lda, 128, 64);   // A: one 64-row half per cluster CTA
  if (rc) return rc;
  rc = encode_tensor_map_2d_u8(&tb, B, K, N, ldb, 128, 64);
  if (rc) return rc;
  return dispatch_e4m3(ta, tb, ep, M, N, K, sa, sb, stream);
}

}  // namespace d3
