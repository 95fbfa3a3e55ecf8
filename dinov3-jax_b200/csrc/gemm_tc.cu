// Persistent, warp-specialised bf16 GEMM on the Hopper tensor cores (wgmma, register accumulators, TMA operand
// staging through an mbarrier ring).  One kernel family covers every dense contraction on the DINOv3 training path:
//   forward  Y = X W        (A K-major, B MN-major: reference kernels are stored [in,out])
//   dgrad    dX = dY W^T    (A K-major, B K-major)
//   wgrad    dW = X^T dY    (A MN-major, B MN-major, fp32 output, split-K reduced in a fixed order)
// replacing nn.Dense / nn.Conv(stride=kernel) call sites of the reference:
//   dinov3_jax/layers/attention.py:63-65,94,101   dinov3_jax/layers/ffn_layers.py:36-47
//   dinov3_jax/layers/patch_embed.py:38-51        dinov3_jax/layers/dino_head.py:20-43,65-85
// The epilogue fuses bias, tanh-GELU, GELU', LayerScale (gamma) and the residual add
// (dinov3_jax/layers/block.py:198-199, dinov3_jax/layers/layer_scale.py:17-21).
//
// One kernel, 128 x {64,128} output tiles, 384 threads:
//   warpgroup 0      TMA producer (one elected thread): A and B k-blocks of 64, tile after tile of this CTA's work
//                    list, into the shared-memory ring of the consumer that owns the tile;
//   warpgroups 1, 2  consumers in ping-pong: the CTA's tiles alternate between them, so one warpgroup's epilogue
//                    (straight from its accumulator registers) runs under the other's main loop.  A tile is two
//                    m64nBNk16 wgmma chains (rows 0-63 / 64-127) over SWIZZLE_128B operands, K-major or MN-major through
//                    the descriptor transpose bits.
// Each consumer has its own ring (half of the stages) and waits on every fill of it in order: with one shared ring the
// consumer of tile j+1 would wait on fills two barrier phases ahead, which the phase parity cannot tell apart.
#include <cstdlib>
#include <cstring>
#include "ptx.cuh"
#include "d3_internal.h"

namespace d3 {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int GEMM_THREADS = 384;

// ---------------------------------------------------------------------------------------------------------------
// epilogue for two adjacent columns (n, n+1) of one row; `vec`: both columns in range and every operand 16-byte
// aligned with even leading dimensions (vector loads / stores of pairs)
__device__ __forceinline__ void epilogue_pair(const GemmEpilogue& ep, size_t row, int n, int N, float v0, float v1,
                                              bool vec) {
  v0 *= ep.alpha;
  v1 *= ep.alpha;
  if (ep.flags & EP_SCATTER) {  // fused reduce-scatter: add into the owning rank's shard slice (NVLink peer mapping)
    const unsigned long long g = (unsigned long long)ep.sc_off + row * ep.ld_out + n;
    const unsigned long long shard = (unsigned long long)ep.sc_shard;
    if (n + 1 < N) {                                         // a pair never straddles two owners (shard % 4 == 0)
      const unsigned r = (unsigned)(g / shard);
      float* dst = ep.sc_peer[r] + (g - r * shard);
      if (ep.sc_sys) {
        atomicAdd_system(dst, v0); atomicAdd_system(dst + 1, v1);
      } else {
        atomicAdd(reinterpret_cast<float2*>(dst), make_float2(v0, v1));
      }
    } else if (n < N) {
      const unsigned r = (unsigned)(g / shard);
      atomicAdd(ep.sc_peer[r] + (g - r * shard), v0);
    }
    return;
  }
  const bool fast_act = (ep.flags & EP_FAST_ACT) != 0;
  if (vec) {
    if (ep.flags & EP_BIAS) {
      const float2 b = *reinterpret_cast<const float2*>(ep.bias + n);
      v0 += b.x; v1 += b.y;
    }
    if (ep.flags & EP_STORE_PRE) *reinterpret_cast<uint32_t*>(ep.aux_out + row * ep.ld_aux + n) = pack_bf16(v0, v1);
    if (ep.flags & EP_GELU) {
      v0 = fast_act ? gelu_tanh_fast(v0) : gelu_tanh(v0);
      v1 = fast_act ? gelu_tanh_fast(v1) : gelu_tanh(v1);
    }
    if (ep.flags & EP_MUL_DGELU) {
      const float2 u = unpack_bf16(*reinterpret_cast<const uint32_t*>(ep.aux_in + row * ep.ld_aux + n));
      v0 *= fast_act ? gelu_tanh_grad_fast(u.x) : gelu_tanh_grad(u.x);
      v1 *= fast_act ? gelu_tanh_grad_fast(u.y) : gelu_tanh_grad(u.y);
    }
    if (ep.flags & EP_GAMMA) {
      const float2 g = *reinterpret_cast<const float2*>(ep.gamma + n);
      v0 *= g.x; v1 *= g.y;
    }
    if (ep.flags & EP_RESID) {
      const float2 x = *reinterpret_cast<const float2*>(ep.resid + row * ep.ld_resid + n);
      v0 += x.x; v1 += x.y;
    }
    if (ep.flags & EP_OUT_F32) {
      float2* dst = reinterpret_cast<float2*>(reinterpret_cast<float*>(ep.out) + row * ep.ld_out + n);
      if (ep.flags & EP_ACCUM) {
        const float2 x = *dst;
        v0 += x.x; v1 += x.y;
      }
      *dst = make_float2(v0, v1);
    } else {
      *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(ep.out) + row * ep.ld_out + n) = pack_bf16(v0, v1);
    }
    return;
  }
  // ragged / unaligned edge: scalar path with bounds checks
#pragma unroll 1
  for (int j = 0; j < 2; ++j) {
    const int c = n + j;
    if (c >= N) break;
    float x = j ? v1 : v0;
    if (ep.flags & EP_BIAS) x += ep.bias[c];
    if (ep.flags & EP_STORE_PRE) ep.aux_out[row * ep.ld_aux + c] = __float2bfloat16(x);
    if (ep.flags & EP_GELU) x = fast_act ? gelu_tanh_fast(x) : gelu_tanh(x);
    if (ep.flags & EP_MUL_DGELU) {
      const float u = __bfloat162float(ep.aux_in[row * ep.ld_aux + c]);
      x *= fast_act ? gelu_tanh_grad_fast(u) : gelu_tanh_grad(u);
    }
    if (ep.flags & EP_GAMMA) x *= ep.gamma[c];
    if (ep.flags & EP_RESID) x += ep.resid[row * ep.ld_resid + c];
    if (ep.flags & EP_OUT_F32) {
      float* o = reinterpret_cast<float*>(ep.out) + row * ep.ld_out + c;
      if (ep.flags & EP_ACCUM) x += *o;
      *o = x;
    } else {
      reinterpret_cast<__nv_bfloat16*>(ep.out)[row * ep.ld_out + c] = __float2bfloat16(x);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
template <int BN>
struct Cfg {
  static constexpr int STAGES = BN == 128 ? 6 : 8;   // two rings of STAGES / 2
  static constexpr int RS = STAGES / 2;
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;
};

// work item = (tile, split): k-blocks [kb0, kb1)
struct WorkRange { int m0, n0, kb0, kb1; };
// Tiles are rasterised N-fastest: the CTAs resident at any moment cover a few M row-panels times all N tiles, so the
// large activation operand streams from HBM once while the (small) weight operand stays L2-resident.
__device__ __forceinline__ WorkRange work_item(int w, int num_n, int num_k, int splits, int tile_n) {
  const int tile = w / splits, sp = w % splits;
  const int per = (num_k + splits - 1) / splits;
  WorkRange r;
  r.n0 = (tile % num_n) * tile_n;
  r.m0 = (tile / num_n) * BM;
  r.kb0 = sp * per;
  r.kb1 = min(num_k, r.kb0 + per);
  return r;
}

template <int BN, int A_MN, int B_MN>
__device__ __forceinline__ void mma_kblock(float (&acc)[2][BN / 2], uint32_t sa, uint32_t sb, bool first) {
  // A rows 64-127 start 8 KB into the stage in both layouts (64 rows x 128 B, or the second 64-row box)
  const uint64_t bd = B_MN ? gmma_desc_sw128(sb, 8192, 1024) : gmma_desc_sw128(sb, 16, 1024);
  constexpr uint64_t a_adv = A_MN ? (2048 >> 4) : (32 >> 4);
  constexpr uint64_t b_adv = B_MN ? (2048 >> 4) : (32 >> 4);
#pragma unroll
  for (int k = 0; k < BK / 16; ++k) {
    const uint32_t sc = (first && k == 0) ? 0u : 1u;
#pragma unroll
    for (int mh = 0; mh < 2; ++mh) {
      const uint64_t ad = A_MN ? gmma_desc_sw128(sa + mh * 8192, 8192, 1024) : gmma_desc_sw128(sa + mh * 8192, 16, 1024);
      if constexpr (BN == 128) wgmma_m64n128k16_ss<A_MN, B_MN>(acc[mh], ad + k * a_adv, bd + k * b_adv, sc);
      else wgmma_m64n64k16_ss<A_MN, B_MN>(acc[mh], ad + k * a_adv, bd + k * b_adv, sc);
    }
  }
}

template <int BN, int A_MN, int B_MN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmEpilogue ep,
            int M, int N, int K, int splits) {
  using C = Cfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + C::STAGES * C::STAGE_BYTES);   // [ring * RS + stage]
  uint64_t* empty_bar = full_bar + C::STAGES;

  const int wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < C::STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 1); }
    fence_mbar_init();
  }
  __syncthreads();

  const int num_m = (M + BM - 1) / BM;
  const int num_n = (N + BN - 1) / BN;
  const int num_k = (K + BK - 1) / BK;
  const int num_work = num_m * num_n * splits;

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (threadIdx.x < 32 && elect_one()) {
      int stage[2] = {0, 0};
      uint32_t phase[2] = {0, 0};
      int j = 0;
      for (int w = blockIdx.x; w < num_work; w += gridDim.x, ++j) {
        const WorkRange wr = work_item(w, num_n, num_k, splits, BN);
        const int r = j & 1;                   // the ring of the consumer that owns tile j
        for (int kb = wr.kb0; kb < wr.kb1; ++kb) {
          const int slot = r * C::RS + stage[r];
          mbar_wait(&empty_bar[slot], phase[r] ^ 1);
          uint8_t* sa = smem + slot * C::STAGE_BYTES;
          uint8_t* sb = sa + C::A_BYTES;
          mbar_expect_tx(&full_bar[slot], C::STAGE_BYTES);
          if (A_MN) {
#pragma unroll
            for (int i = 0; i < BM / 64; ++i) tma_load_2d(&tmA, &full_bar[slot], sa + i * 8192, wr.m0 + i * 64, kb * BK);
          } else {
            tma_load_2d(&tmA, &full_bar[slot], sa, kb * BK, wr.m0);
          }
          if (B_MN) {
#pragma unroll
            for (int i = 0; i < BN / 64; ++i) tma_load_2d(&tmB, &full_bar[slot], sb + i * 8192, wr.n0 + i * 64, kb * BK);
          } else {
            tma_load_2d(&tmB, &full_bar[slot], sb, kb * BK, wr.n0);
          }
          if (++stage[r] == C::RS) { stage[r] = 0; phase[r] ^= 1; }
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    const int cw = wg - 1;                     // consumer warpgroup: tiles j of this CTA with j % 2 == cw
    const int t = threadIdx.x & 127;
    const int r_in = 16 * (t >> 5) + ((t & 31) >> 2);
    const int c_in = 2 * (t & 3);
    const bool fast = (ep.flags & EP_SLOW) == 0;
    int stage = 0;                             // position in this consumer's ring
    uint32_t phase = 0;
    for (int w = blockIdx.x + cw * gridDim.x; w < num_work; w += 2 * gridDim.x) {
      const WorkRange wr = work_item(w, num_n, num_k, splits, BN);
      const int nkb = wr.kb1 - wr.kb0;
      float acc[2][BN / 2];
#pragma unroll
      for (int mh = 0; mh < 2; ++mh)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[mh][i] = 0.f;
      int prev = -1;
      for (int kb = wr.kb0; kb < wr.kb1; ++kb) {
        const int slot = cw * C::RS + stage;
        mbar_wait(&full_bar[slot], phase);
        const uint32_t sa = smem_u32(smem + slot * C::STAGE_BYTES);
        fence_regs(acc[0]);
        fence_regs(acc[1]);
        wgmma_fence();
        mma_kblock<BN, A_MN, B_MN>(acc, sa, sa + C::A_BYTES, kb == wr.kb0);
        wgmma_commit();
        fence_regs(acc[0]);
        fence_regs(acc[1]);
        if (prev >= 0) {                       // the k-block before this one has been consumed: release its stage
          wgmma_wait<1>();
          if (t == 0) mbar_arrive(&empty_bar[prev]);
        }
        prev = slot;
        if (++stage == C::RS) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      fence_regs(acc[0]);
      fence_regs(acc[1]);
      if (prev >= 0 && t == 0) mbar_arrive(&empty_bar[prev]);
      if (nkb <= 0) continue;                  // empty split-K slice: nothing to add
#pragma unroll
      for (int mh = 0; mh < 2; ++mh)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = wr.m0 + mh * 64 + r_in + 8 * h;
          if (row >= M) continue;
          const size_t orow = (ep.flags & EP_SLABS) ? (size_t)(w % splits) * M + row : (size_t)row;
#pragma unroll
          for (int i = 0; i < BN / 8; ++i) {
            const int n = wr.n0 + 8 * i + c_in;
            if (n >= N) break;
            epilogue_pair(ep, orow, n, N, acc[mh][4 * i + 2 * h], acc[mh][4 * i + 2 * h + 1], fast && n + 1 < N);
          }
        }
    }
  }
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

template <int BN, int A_MN, int B_MN>
static int launch(const CUtensorMap& ta, const CUtensorMap& tb, const GemmEpilogue& ep, int M, int N, int K,
                  int splits, cudaStream_t stream) {
  using C = Cfg<BN>;
  auto kern = gemm_kernel<BN, A_MN, B_MN>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    if (e != cudaSuccess) return set_error(D3_ERR_CUDA, cudaGetErrorString(e));
    configured = true;
  }
  const int work = ((M + BM - 1) / BM) * ((N + BN - 1) / BN) * splits;
  const int grid = work < sm_count() ? work : sm_count();
  kern<<<grid, GEMM_THREADS, C::SMEM_BYTES, stream>>>(ta, tb, ep, M, N, K, splits);
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) return set_error(D3_ERR_CUDA, cudaGetErrorString(e));
  count_launch();
  return D3_OK;
}

template <int BN>
static int dispatch(int a_mn, int b_mn, const CUtensorMap& ta, const CUtensorMap& tb, const GemmEpilogue& ep, int M,
                    int N, int K, int splits, cudaStream_t s) {
  if (!a_mn && !b_mn) return launch<BN, 0, 0>(ta, tb, ep, M, N, K, splits, s);
  if (!a_mn && b_mn) return launch<BN, 0, 1>(ta, tb, ep, M, N, K, splits, s);
  if (a_mn && !b_mn) return launch<BN, 1, 0>(ta, tb, ep, M, N, K, splits, s);
  return launch<BN, 1, 1>(ta, tb, ep, M, N, K, splits, s);
}

// tile_n: 0 = auto; 64/128 force that tile width; 256 and 512 (wider tiles) are taken as 128.
// split_k: 0 = auto (only when the epilogue is a plain fp32 accumulate-able output), >= 1 forced.
int gemm_bf16(const void* A, int lda, int a_mn, const void* B, int ldb, int b_mn, int M, int N, int K,
              GemmEpilogue ep, int tile_n, int split_k, cudaStream_t stream) {
  if (M <= 0 || N <= 0 || K <= 0) return set_error(D3_ERR_ARG, "gemm: empty problem");
  if ((lda % 8) || (ldb % 8) || (reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(B) & 15))
    return set_error(D3_ERR_ARG, "gemm: operands must be 16-byte aligned with ld % 8 == 0");
  const int sms = sm_count();
  const int num_k = (K + BK - 1) / BK;
  // ---- tile choice: fewest waves of (tile width + fixed per-tile cost) over the SMs
  int bn = tile_n >= 256 ? 128 : tile_n;
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
                                                                  EP_GAMMA | EP_RESID));
  int splits = 1;
  if (split_k >= 1) {
    splits = split_k;
  } else if (plain_f32 && (ep.flags & EP_ACCUM)) {
    const long units = (long)((M + BM - 1) / BM) * ((N + bn - 1) / bn);
    if (units <= sms && num_k >= 16) {
      // fill the SMs; and keep every accumulation chain within 64 k-blocks: the tensor core's fp32 accumulation drifts
      // measurably (> 1e-5 relative) over longer chains, the fp32 reduction of the slices does not
      splits = units * 2 <= sms ? (int)(sms / units) : 1;
      if (splits < (num_k + 63) / 64) splits = (num_k + 63) / 64;
      if (splits > num_k / 4) splits = num_k / 4;
      if (splits < 1) splits = 1;
    }
  }
  if (ep.flags & EP_SCATTER) {
    if (!plain_f32) return set_error(D3_ERR_ARG, "gemm: SCATTER needs a plain fp32 output");
    if (ep.sc_world < 1 || ep.sc_world > 8 || ep.sc_shard <= 0 || (ep.sc_shard % 4) || (ep.sc_off % 4) || (ep.ld_out % 4))
      return set_error(D3_ERR_ARG, "gemm: SCATTER needs 1..8 ranks and 4-element aligned shard / offset / ld_out");
    if ((unsigned long long)ep.sc_off + (unsigned long long)(M - 1) * ep.ld_out + N > (unsigned long long)ep.sc_shard * ep.sc_world)
      return set_error(D3_ERR_ARG, "gemm: SCATTER output exceeds the sharded range");
    ep.flags |= EP_ATOMIC;       // every contribution is an atomic add (other ranks add into the same slice)
  }
  if (splits > 1) {
    if (!plain_f32) return set_error(D3_ERR_ARG, "gemm: split-K needs a plain fp32 output");
    if (!(ep.flags & EP_ACCUM)) return set_error(D3_ERR_ARG, "gemm: split-K accumulates into out (set ACCUM, zero it first)");
    if (splits > num_k) splits = num_k;
  }
  // ---- epilogue fast-path eligibility
  const int out_elt = (ep.flags & EP_OUT_F32) ? 4 : 2;
  bool aligned = ((uintptr_t)ep.out % 16 == 0) && ((ep.ld_out * out_elt) % 16 == 0);
  if (ep.flags & EP_BIAS) aligned = aligned && ((uintptr_t)ep.bias % 16 == 0);
  if (ep.flags & EP_GAMMA) aligned = aligned && ((uintptr_t)ep.gamma % 16 == 0);
  if (ep.flags & EP_RESID) aligned = aligned && ((uintptr_t)ep.resid % 16 == 0) && (ep.ld_resid % 4 == 0);
  if (ep.flags & EP_STORE_PRE) aligned = aligned && ((uintptr_t)ep.aux_out % 16 == 0) && (ep.ld_aux % 8 == 0);
  if (ep.flags & EP_MUL_DGELU) aligned = aligned && ((uintptr_t)ep.aux_in % 16 == 0) && (ep.ld_aux % 8 == 0);
  if (!aligned) ep.flags |= EP_SLOW;
  ep.flags |= EP_FAST_ACT;   // hardware tanh (rel. error 2^-11, below the bf16 rounding of the GEMM operands feeding it)

  CUtensorMap ta, tb;
  int rc = make_operand_map(&ta, A, M, K, lda, a_mn, BM);
  if (rc) return rc;
  rc = make_operand_map(&tb, B, N, K, ldb, b_mn, bn);
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

}  // namespace d3
