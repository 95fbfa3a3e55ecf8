// HBM-bound kernels of the ViT forward/backward: im2col, token assembly, LayerNorm fwd/bwd, RoPE, row
// gather/scatter, L2-normalise, LayerScale/GELU backward, column sums.  All use 128-bit loads where the layout
// allows, warp-shuffle reductions, fp32 statistics.
#include "ptx.cuh"
#include "d3_internal.h"
#include "layernorm.cuh"

namespace d3 {

// ------------------------------------------------------------------------------------------------ im2col
// layers/patch_embed.py:38-51: conv with kernel == stride == p is a GEMM over flattened patches.
// img bf16 [n, H, W, 3] -> out bf16 [n*Hp*Wp, p*p*3], k = (a*p + b)*3 + c  (kernel layout [p,p,3,D]).
__global__ void im2col_kernel(const __nv_bfloat16* __restrict__ img, __nv_bfloat16* __restrict__ out, int n, int H,
                              int W, int p, int ld) {
  const int Hp = H / p, Wp = W / p;
  const int rowlen = p * 3;              // contiguous run in the image per (patch row a)
  const long total = (long)n * Hp * Wp * p;   // one work item = one contiguous run
  for (long w = blockIdx.x * (long)blockDim.x / 32 + threadIdx.x / 32; w < total; w += (long)gridDim.x * blockDim.x / 32) {
    const int a = (int)(w % p);
    long r = w / p;                      // patch row index in out
    const int j = (int)(r % Wp);
    const int i = (int)((r / Wp) % Hp);
    const long c = r / ((long)Wp * Hp);
    const __nv_bfloat16* src = img + ((c * H + (long)i * p + a) * W + (long)j * p) * 3;
    __nv_bfloat16* dst = out + r * (long)ld + (long)a * rowlen;
    for (int e = threadIdx.x & 31; e < rowlen; e += 32) dst[e] = src[e];
    if (a == p - 1)   // zero the alignment padding of the row (ld may exceed p*p*3)
      for (int e = p * rowlen + (threadIdx.x & 31); e < ld; e += 32) out[r * (long)ld + e] = __float2bfloat16(0.f);
  }
}

// ------------------------------------------------------------------------------------------------ tokens
// models/vision_transformer.py:173-203: where(mask, mask_token, x); prepend cls (+0*mask_token) and the R storage
// (register) tokens.  tok fp32 [n*P, D] -> X fp32 [n, 1+R+P, D]
__global__ void assemble_tokens_kernel(const float* __restrict__ tok, const float* __restrict__ cls,
                                       const float* __restrict__ storage, const float* __restrict__ mask_token,
                                       const uint8_t* __restrict__ masks, float* __restrict__ X, int n, int P, int R,
                                       int D) {
  const int N = P + 1 + R;
  const long rows = (long)n * N;
  const int D4 = D / 4;
  for (long r = blockIdx.x; r < rows; r += gridDim.x) {
    const long c = r / N;
    const int t = (int)(r % N);
    const float4* src;
    if (t == 0) src = reinterpret_cast<const float4*>(cls);
    else if (t <= R) src = reinterpret_cast<const float4*>(storage + (long)(t - 1) * D);
    else if (masks && masks[c * P + (t - 1 - R)]) src = reinterpret_cast<const float4*>(mask_token);
    else src = reinterpret_cast<const float4*>(tok + (c * P + (t - 1 - R)) * (long)D);
    float4* dst = reinterpret_cast<float4*>(X + r * (long)D);
    for (int e = threadIdx.x; e < D4; e += blockDim.x) dst[e] = src[e];
  }
}
// backward: dX fp32 [n,1+R+P,D] -> dTok bf16 [n*P, D] (0 where masked); the crop slab's sums of dX[c,0] (cls),
// of the masked rows (mask token) and of dX[c,1..R] (storage tokens) go to its workspace slab [cls D | mask D | R*D]
__global__ void assemble_tokens_bwd_kernel(const float* __restrict__ dX, const uint8_t* __restrict__ masks,
                                           __nv_bfloat16* __restrict__ dTok, float* __restrict__ ws, int n, int P, int R,
                                           int D) {
  // grid.x = column chunks of 128 floats (threads 128: one column each), grid.y = slabs of whole crops
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  const int N = P + 1 + R;
  const long slab = ((long)n + gridDim.y - 1) / gridDim.y;
  const long c0 = blockIdx.y * slab, c1 = min((long)n, c0 + slab);
  if (col >= D) return;
  float acc_cls = 0.f, acc_mask = 0.f;
  float* slab_ws = ws + (long)blockIdx.y * (2 + R) * D;
  for (int t = 1; t <= R; ++t) {
    float acc = 0.f;
    for (long c = c0; c < c1; ++c) acc += dX[c * N * (long)D + (long)t * D + col];
    slab_ws[(long)(1 + t) * D + col] = acc;
  }
  for (long c = c0; c < c1; ++c) {
    const float* row = dX + c * N * (long)D + col;
    acc_cls += row[0];
    for (int t = 0; t < P; ++t) {
      const float g = row[(long)(1 + R + t) * D];
      const bool m = masks && masks[c * P + t];
      if (m) acc_mask += g;
      dTok[(c * P + t) * (long)D + col] = __float2bfloat16(m ? 0.f : g);
    }
  }
  slab_ws[col] = acc_cls;
  slab_ws[D + col] = acc_mask;
}

// ------------------------------------------------------------------------------------------------ LayerNorm
// models/vision_transformer.py:40 (flax nn.LayerNorm, eps 1e-6, biased variance E[x^2]-E[x]^2, fp32 stats).
// One warp per row; x fp32 [T, D]; y bf16 or fp32.  The row statistics and normalisation are layernorm.cuh's.

// VPL > 0: the row stays in registers between the statistics and the normalisation (one read of x).  VPL == 0: x read
// twice.
template <int VPL, typename OutT>
__global__ void __launch_bounds__(256)
layernorm_fwd_kernel(const float* __restrict__ x, const float* __restrict__ scale, const float* __restrict__ bias,
                     OutT* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out, int T, float eps,
                     int width) {
  const int D = VPL > 0 ? VPL * 128 : width;
  const int warps = blockDim.x >> 5, lane = threadIdx.x & 31;
  for (long row = (long)blockIdx.x * warps + (threadIdx.x >> 5); row < T; row += (long)gridDim.x * warps) {
    const float4* xr = reinterpret_cast<const float4*>(x + row * (long)D);
    float4 v[VPL > 0 ? VPL : 1];
    float mean, rstd;
    ln_row_stats<VPL>(xr, lane, D, eps, v, mean, rstd);
    if (lane == 0 && mean_out) { mean_out[row] = mean; rstd_out[row] = rstd; }
    ln_store_row<VPL>(y + row * (long)D, xr, lane, D, v, scale, bias, mean, rstd);
  }
}

// ------------------------------------------------------------------------------------------------ block output -> features
// models/vision_transformer.py:280-313 (get_intermediate_layers): one block output X [n, N = 1 + R + P, D] fp32 ->
// cls [n, D], storage [n, R, D] and the patches, channels-last [n, P, D] or channels-first [n, D, Hp, Wp], each row
// LayerNorm-ed with (pre_scale, pre_bias) for the 1 + R prefix rows and (scale, bias) for the patch rows, or only
// converted when scale is null.
struct TokensOut {
  const float *X, *scale, *bias, *pre_scale, *pre_bias;
  void *cls, *storage, *patches;
  int n, N, R, P, D;
  float eps;
  int tp;                // channels-first: patch rows per tile (8 or 16 .. 64)
  int tiles_per_img;     // ceil(P / tp)
  int vec_bytes;         // channels-first: bytes per store along a channel plane (16, 8, 4 or 2)
};

constexpr int TOK_WARPS = 8;
constexpr int TOK_PAD = 4;       // elements after each staged row: keeps rows 16-byte aligned, spreads the column reads

// row t of image b (one warp) -> its output row, LayerNorm-ed or converted
template <int VPL, typename OutT>
__device__ __forceinline__ void tokens_out_row(const TokensOut& a, int b, int t, OutT* dst, int lane) {
  const int D = a.D;
  const float4* xr = reinterpret_cast<const float4*>(a.X + ((long)b * a.N + t) * D);
  const bool prefix = t <= a.R;
  const float* g = prefix ? a.pre_scale : a.scale;
  const float* bb = prefix ? a.pre_bias : a.bias;
  if (g) {
    float4 v[VPL > 0 ? VPL : 1];
    float mean, rstd;
    ln_row_stats<VPL>(xr, lane, D, a.eps, v, mean, rstd);
    ln_store_row<VPL>(dst, xr, lane, D, v, g, bb, mean, rstd);
  } else {
    for (int e = lane; e < D / 4; e += 32) {
      const float4 w = xr[e];
      store4(dst, e, w.x, w.y, w.z, w.w);
    }
  }
}

template <typename OutT>
__device__ __forceinline__ OutT* tokens_out_dst(const TokensOut& a, int b, int t) {
  const long D = a.D;
  if (t == 0) return (OutT*)a.cls + b * D;
  if (t <= a.R) return (OutT*)a.storage + ((long)b * a.R + t - 1) * D;
  return (OutT*)a.patches + ((long)b * a.P + t - 1 - a.R) * D;
}

// `vb` bytes of channel plane `dst` from the staged column src[0], src[ld], ... (vb / sizeof(OutT) rows)
template <typename OutT>
__device__ __forceinline__ void store_column_run(OutT* dst, const OutT* src, int ld, int vb) {
  if constexpr (sizeof(OutT) == 4) {
    if (vb == 16) *reinterpret_cast<float4*>(dst) = make_float4(src[0], src[ld], src[2 * ld], src[3 * ld]);
    else if (vb == 8) *reinterpret_cast<float2*>(dst) = make_float2(src[0], src[ld]);
    else *dst = src[0];
  } else {
    const unsigned short* s = reinterpret_cast<const unsigned short*>(src);
    auto pair = [&](int i) { return (uint32_t)s[i * ld] | ((uint32_t)s[(i + 1) * ld] << 16); };
    if (vb == 16) *reinterpret_cast<uint4*>(dst) = make_uint4(pair(0), pair(2), pair(4), pair(6));
    else if (vb == 8) *reinterpret_cast<uint2*>(dst) = make_uint2(pair(0), pair(2));
    else if (vb == 4) *reinterpret_cast<uint32_t*>(dst) = pair(0);
    else *reinterpret_cast<unsigned short*>(dst) = s[0];
  }
}

// CF = false: one warp per row of all n * N rows (grid-stride).
// CF = true: CTAs [0, n * tiles_per_img) each take tp patch rows of one image: every warp normalises whole rows into a
// shared-memory tile [tp][D + TOK_PAD] (x read once), then the CTA writes the tile out channel by channel, a run of
// vec_bytes along Hp*Wp per thread, consecutive threads on consecutive runs of the same plane.  The CTAs after them take
// the n * (1 + R) prefix rows, one warp per row.
template <int VPL, typename OutT, bool CF>
__global__ void __launch_bounds__(32 * TOK_WARPS, 2)
ln_tokens_out_kernel(const TokensOut a) {
  extern __shared__ __align__(16) unsigned char tok_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tiles = CF ? a.n * a.tiles_per_img : 0;
  if (CF && (int)blockIdx.x < n_tiles) {
    OutT* tile = reinterpret_cast<OutT*>(tok_smem);
    const int ld = a.D + TOK_PAD;
    const int b = blockIdx.x / a.tiles_per_img, p0 = blockIdx.x % a.tiles_per_img * a.tp;
    const int rows = min(a.tp, a.P - p0);
    for (int r = warp; r < rows; r += TOK_WARPS) tokens_out_row<VPL>(a, b, 1 + a.R + p0 + r, tile + (long)r * ld, lane);
    __syncthreads();
    const int w = a.vec_bytes / (int)sizeof(OutT), runs = a.tp / w;
    OutT* plane0 = (OutT*)a.patches + (long)b * a.D * a.P + p0;
    for (int i = threadIdx.x; i < a.D * runs; i += blockDim.x) {
      const int c = i / runs, p = i % runs * w;
      if (p < rows) store_column_run(plane0 + (long)c * a.P + p, tile + (long)p * ld + c, ld, a.vec_bytes);
    }
    return;
  }
  const int per_img = CF ? 1 + a.R : a.N;
  const long total = (long)a.n * per_img;
  for (long r = (long)(blockIdx.x - n_tiles) * TOK_WARPS + warp; r < total; r += (long)(gridDim.x - n_tiles) * TOK_WARPS) {
    const int b = (int)(r / per_img), t = (int)(r % per_img);
    tokens_out_row<VPL>(a, b, t, tokens_out_dst<OutT>(a, b, t), lane);
  }
}

// The per-element steps of the LayerNorm backward and of the LayerScale/GELU tail.  ln_bwd_ls_kernel and
// ls_act_bwd_kernel call these helpers; ln_bwd_ring_kernel spells out the same expressions inline, because calling
// them changes its register allocation and instruction order.

// 4 consecutive elements as fp32 (p: 8-byte aligned bf16 or 16-byte aligned fp32)
template <typename T>
__device__ __forceinline__ void load4(const T* p, float (&v)[4]) {
  if constexpr (sizeof(T) == 2) {
    const uint2 u = *reinterpret_cast<const uint2*>(p);
    const float2 v0 = unpack_bf16(u.x), v1 = unpack_bf16(u.y);
    v[0] = v0.x; v[1] = v0.y; v[2] = v1.x; v[3] = v1.y;
  } else {
    const float4 f = *reinterpret_cast<const float4*>(p);
    v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
  }
}

// LayerNorm input gradient of 4 columns of a row with rstd rs, from gs = dy * scale and xh = x̂, with a = mean(gs),
// b = mean(gs x̂):  o = rs (gs - a - x̂ b)  (+ the residual-stream gradient at `add`, 16-byte aligned, if `has_add`)
__device__ __forceinline__ void ln_dx4(float (&o)[4], const float (&gs)[4], const float (&xh)[4], float a, float b,
                                       float rs, bool has_add, const float* add) {
#pragma unroll
  for (int j = 0; j < 4; ++j) o[j] = rs * (gs[j] - a - xh[j] * b);
  if (has_add) {
    const float4 r4 = *reinterpret_cast<const float4*>(add);
    o[0] += r4.x; o[1] += r4.y; o[2] += r4.z; o[3] += r4.w;
  }
}

// LayerScale / activation backward of 4 columns of x_out = x_in + gamma * act(u), given o = dx_out: returns the packed
// du = bf16(o gamma act'(u)), adds o act(u) to the dgamma partials `dg` and the rounded du, the values the weight-
// gradient GEMM sees, to the dbias partials `db`.  act = tanh-GELU with the hardware tanh (the forward's GEMM epilogue
// computed act(u) with it) if `gelu`, else identity.  u: 4 bf16 (8-byte aligned), read only if `has_u`; without it
// act = identity and `dg` is untouched.
__device__ __forceinline__ uint2 ls_tail4(const float (&o)[4], const float (&gm)[4], bool has_u,
                                          const __nv_bfloat16* u, bool gelu, float (&dg)[4], float (&db)[4]) {
  float d[4];
  if (has_u) {
    float uv[4];
    load4(u, uv);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float act = gelu ? gelu_tanh_fast(uv[j]) : uv[j];
      const float dact = gelu ? gelu_tanh_grad_fast(uv[j]) : 1.f;
      d[j] = o[j] * gm[j] * dact;
      dg[j] += o[j] * act;
    }
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) d[j] = o[j] * gm[j];
  }
  const uint32_t p0 = pack_bf16(d[0], d[1]), p1 = pack_bf16(d[2], d[3]);
  const float2 r0 = unpack_bf16(p0), r1 = unpack_bf16(p1);
  db[0] += r0.x; db[1] += r0.y; db[2] += r1.x; db[3] += r1.y;
  return make_uint2(p0, p1);
}

// LayerNorm backward fused with the LayerScale/GELU backward of the branch that *feeds on* its result.
// The row gradient dx (fp32 residual-stream gradient) produced here is exactly the dX the next branch upstream
// needs (block.py:198-199: x_out = x_in + gamma * act(u)), so the same pass also writes
//     du = bf16(dx * gamma * act'(u)),   dgamma += colsum(dx * act(u)),   dbias += colsum(du)
// and the separate ls_act_bwd pass (one more read of dx and u, one more launch) disappears.
//   ls_u == nullptr : act = identity and dgamma is not produced here (it is recovered from the weight gradient:
//                     dgamma_j = (sum_i W_ij dW_ij + b_j db_j) / gamma_j, see ls_gamma_from_wgrad_kernel)
// Layout: a row is owned by 128 threads (4 warps, float4 chunks, NC = ceil(D / 512) chunks per thread), two rows in
// flight per CTA; every thread keeps its columns' parameter-gradient partial sums in registers over all its rows.
template <int NC, typename InT>
__global__ void __launch_bounds__(256)
ln_bwd_ls_kernel(const InT* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ mean,
                 const float* __restrict__ rstd, const float* __restrict__ scale, const float* __restrict__ dx_add,
                 float* __restrict__ dx, float* __restrict__ dscale, float* __restrict__ dbias, int T, int D,
                 const float* __restrict__ ls_gamma, const __nv_bfloat16* __restrict__ ls_u, int ls_gelu,
                 __nv_bfloat16* __restrict__ ls_du, float* __restrict__ ls_dgamma, float* __restrict__ ls_dbias,
                 float* __restrict__ ws) {
  extern __shared__ float part[];                 // [4][D] cross-group reduction of the column sums
  __shared__ float red[2][2][4][2];               // [group][parity][warp][a | b]
  const int grp = threadIdx.x >> 7, t = threadIdx.x & 127, wig = t >> 5, lane = threadIdx.x & 31;
  const float invD = 1.f / (float)D;
  const bool tail = ls_gamma != nullptr;
  float sc[NC][4], gm[NC][4];
  float ads[NC][4], adb[NC][4], tdg[NC][4], tdb[NC][4];
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    const int col = (c * 128 + t) * 4;
    const bool ok = col < D;
    const float4 s4 = ok ? *reinterpret_cast<const float4*>(scale + col) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 g4 = (ok && tail) ? *reinterpret_cast<const float4*>(ls_gamma + col) : make_float4(0.f, 0.f, 0.f, 0.f);
    sc[c][0] = s4.x; sc[c][1] = s4.y; sc[c][2] = s4.z; sc[c][3] = s4.w;
    gm[c][0] = g4.x; gm[c][1] = g4.y; gm[c][2] = g4.z; gm[c][3] = g4.w;
#pragma unroll
    for (int j = 0; j < 4; ++j) { ads[c][j] = 0.f; adb[c][j] = 0.f; tdg[c][j] = 0.f; tdb[c][j] = 0.f; }
  }
  int parity = 0;
  for (long row = (long)blockIdx.x * 2 + grp; row < T; row += (long)gridDim.x * 2, parity ^= 1) {
    const float mu = mean[row], rs = rstd[row];
    float xh[NC][4], gs[NC][4];
    float a = 0.f, b = 0.f;
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const int col = (c * 128 + t) * 4;
      if (col < D) {
        float xs[4], g[4];
        load4(x + row * (long)D + col, xs);
        load4(dy + row * (long)D + col, g);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          xh[c][j] = (xs[j] - mu) * rs;
          gs[c][j] = g[j] * sc[c][j];
          a += gs[c][j];
          b += gs[c][j] * xh[c][j];
          ads[c][j] += g[j] * xh[c][j];
          adb[c][j] += g[j];
        }
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) { xh[c][j] = 0.f; gs[c][j] = 0.f; }
      }
    }
    a = warp_sum(a);
    b = warp_sum(b);
    if (lane == 0) { red[grp][parity][wig][0] = a; red[grp][parity][wig][1] = b; }
    asm volatile("bar.sync %0, 128;" ::"r"(grp + 1) : "memory");
    a = (red[grp][parity][0][0] + red[grp][parity][1][0] + red[grp][parity][2][0] + red[grp][parity][3][0]) * invD;
    b = (red[grp][parity][0][1] + red[grp][parity][1][1] + red[grp][parity][2][1] + red[grp][parity][3][1]) * invD;
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const int col = (c * 128 + t) * 4;
      if (col < D) {
        const long off = row * (long)D + col;
        float o[4];
        ln_dx4(o, gs[c], xh[c], a, b, rs, dx_add != nullptr, dx_add ? dx_add + off : nullptr);
        *reinterpret_cast<float4*>(dx + off) = make_float4(o[0], o[1], o[2], o[3]);
        if (tail)
          *reinterpret_cast<uint2*>(ls_du + off) =
              ls_tail4(o, gm[c], ls_u != nullptr, ls_u ? ls_u + off : nullptr, ls_gelu, tdg[c], tdb[c]);
      }
    }
  }
  // ---- column sums: group 1 -> shared, group 0 adds its own and stores the CTA's partial into its workspace slab
  const bool want_ln = dscale != nullptr;
  if (!want_ln && !tail) return;
  if (grp == 1) {
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const int col = (c * 128 + t) * 4;
      if (col < D) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          part[col + j] = ads[c][j]; part[D + col + j] = adb[c][j];
          part[2 * D + col + j] = tdg[c][j]; part[3 * D + col + j] = tdb[c][j];
        }
      }
    }
  }
  __syncthreads();
  if (grp == 0) {
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const int col = (c * 128 + t) * 4;
      if (col < D) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float* slab_ws = ws + (long)blockIdx.x * 4 * D + col + j;   // [dscale | dbias | ls_dgamma | ls_dbias]
          if (want_ln) {
            slab_ws[0] = ads[c][j] + part[col + j];
            slab_ws[D] = adb[c][j] + part[D + col + j];
          }
          if (tail) {
            if (ls_dgamma && ls_u) slab_ws[2 * D] = tdg[c][j] + part[2 * D + col + j];
            if (ls_dbias) slab_ws[3 * D] = tdb[c][j] + part[3 * D + col + j];
          }
        }
      }
    }
  }
}


// ---- the same fused pass as ln_bwd_ls_kernel, organised for HBM throughput (D = 128 * VPL, VPL <= 8) -----------------
// One persistent CTA per SM.  A producer warp streams whole rows (x | dx_add | dy | u) into a shared-memory ring with
// 1-D bulk copies (cp.async.bulk + mbarrier complete_tx), so the bytes in flight are set by the ring (up to ~200 KB
// per SM) and not by registers; seven consumer warps each take a row, make the two LayerNorm passes out of shared
// memory, store dx / du straight to global with 512-byte warp stores and keep the four column-sum vectors
// (dscale, dbias, ls_dgamma, ls_dbias) for their columns in registers until the end.
constexpr int LNR_MAX_STAGES = 16;
constexpr int LNR_CONSUMERS = 7;     // + 1 producer warp = 8 warps: two per SM sub-partition, so 255 registers stay available
constexpr int LNR_SMEM_BUDGET = 200 * 1024;   // dynamic shared memory: barriers, scale | gamma, the ring

__device__ __forceinline__ void bulk_load_1d(void* dst_smem, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst_smem)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

template <int VPL, typename InT>
__global__ void __launch_bounds__(32 * (LNR_CONSUMERS + 1), 1)
ln_bwd_ring_kernel(const InT* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ mean,
                   const float* __restrict__ rstd, const float* __restrict__ scale, const float* __restrict__ dx_add,
                   float* __restrict__ dx, float* __restrict__ dscale, float* __restrict__ dbias, int T, int stages,
                   const float* __restrict__ ls_gamma, const __nv_bfloat16* __restrict__ ls_u, int ls_gelu,
                   __nv_bfloat16* __restrict__ ls_du, float* __restrict__ ls_dgamma, float* __restrict__ ls_dbias,
                   float* __restrict__ ws) {
  constexpr int D = VPL * 128;
  extern __shared__ __align__(128) uint8_t lnr_smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(lnr_smem);
  uint64_t* empty = full + LNR_MAX_STAGES;
  float* s_scale = reinterpret_cast<float*>(lnr_smem + 256);
  float* s_gamma = s_scale + D;
  uint8_t* ring = lnr_smem + 256 + 2 * D * sizeof(float);
  const bool tail = ls_gamma != nullptr;
  const uint32_t xB = D * 4, aB = dx_add ? D * 4 : 0, gB = D * sizeof(InT), uB = (tail && ls_u) ? D * 2 : 0;
  const uint32_t stageB = xB + aB + gB + uB;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < stages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 1); }
    fence_mbar_init();
  }
  for (int e = threadIdx.x; e < D; e += blockDim.x) { s_scale[e] = scale[e]; s_gamma[e] = tail ? ls_gamma[e] : 0.f; }
  __syncthreads();
  const long nrows = blockIdx.x < T ? ((long)T - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

  if (warp == LNR_CONSUMERS) {
    if (elect_one()) {      // elected lane of the converged producer warp: plain UBLKCP, no per-instruction ELECT loop
      for (long k = 0; k < nrows; ++k) {
        const int st = (int)(k % stages);
        const long use = k / stages;
        if (use > 0) mbar_wait(&empty[st], (uint32_t)((use - 1) & 1));
        const long row = blockIdx.x + k * (long)gridDim.x;
        uint8_t* dst = ring + (size_t)st * stageB;
        mbar_expect_tx(&full[st], stageB);
        bulk_load_1d(dst, x + row * (long)D, xB, &full[st]);
        if (aB) bulk_load_1d(dst + xB, dx_add + row * (long)D, aB, &full[st]);
        bulk_load_1d(dst + xB + aB, dy + row * (long)D, gB, &full[st]);
        if (uB) bulk_load_1d(dst + xB + aB + gB, ls_u + row * (long)D, uB, &full[st]);
      }
    }
    return;      // the producer warp takes no part in the consumers' named barriers below
  }

  float ads[VPL][4], adb[VPL][4], tdg[VPL][4], tdb[VPL][4];
#pragma unroll
  for (int k = 0; k < VPL; ++k)
#pragma unroll
    for (int j = 0; j < 4; ++j) { ads[k][j] = 0.f; adb[k][j] = 0.f; tdg[k][j] = 0.f; tdb[k][j] = 0.f; }

  for (long k = warp; k < nrows; k += LNR_CONSUMERS) {
    const int st = (int)(k % stages);
    const long row = blockIdx.x + k * (long)gridDim.x;
    const float mu = mean[row], rs = rstd[row];
    mbar_wait(&full[st], (uint32_t)((k / stages) & 1));
    const uint8_t* base = ring + (size_t)st * stageB;
    const float* sx = reinterpret_cast<const float*>(base);
    const float* sa = reinterpret_cast<const float*>(base + xB);
    const InT* sg = reinterpret_cast<const InT*>(base + xB + aB);
    const __nv_bfloat16* su = reinterpret_cast<const __nv_bfloat16*>(base + xB + aB + gB);
    float a = 0.f, b = 0.f;
#pragma unroll
    for (int c = 0; c < VPL; ++c) {
      const int e = (c * 32 + lane) * 4;
      const float4 xv = *reinterpret_cast<const float4*>(sx + e);
      const float4 sc = *reinterpret_cast<const float4*>(s_scale + e);
      float g[4];
      if constexpr (sizeof(InT) == 2) {
        const uint2 u2 = *reinterpret_cast<const uint2*>(sg + e);
        const float2 g0 = unpack_bf16(u2.x), g1 = unpack_bf16(u2.y);
        g[0] = g0.x; g[1] = g0.y; g[2] = g1.x; g[3] = g1.y;
      } else {
        const float4 gv = *reinterpret_cast<const float4*>(sg + e);
        g[0] = gv.x; g[1] = gv.y; g[2] = gv.z; g[3] = gv.w;
      }
      const float xs[4] = {xv.x, xv.y, xv.z, xv.w}, scs[4] = {sc.x, sc.y, sc.z, sc.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float xh = (xs[j] - mu) * rs, gsv = g[j] * scs[j];
        a += gsv;
        b += gsv * xh;
        ads[c][j] += g[j] * xh;
        adb[c][j] += g[j];
      }
    }
    a = warp_sum(a) * (1.f / D);
    b = warp_sum(b) * (1.f / D);
#pragma unroll
    for (int c = 0; c < VPL; ++c) {
      const int e = (c * 32 + lane) * 4;
      const float4 xv = *reinterpret_cast<const float4*>(sx + e);
      const float4 sc = *reinterpret_cast<const float4*>(s_scale + e);
      float g[4];
      if constexpr (sizeof(InT) == 2) {
        const uint2 u2 = *reinterpret_cast<const uint2*>(sg + e);
        const float2 g0 = unpack_bf16(u2.x), g1 = unpack_bf16(u2.y);
        g[0] = g0.x; g[1] = g0.y; g[2] = g1.x; g[3] = g1.y;
      } else {
        const float4 gv = *reinterpret_cast<const float4*>(sg + e);
        g[0] = gv.x; g[1] = gv.y; g[2] = gv.z; g[3] = gv.w;
      }
      const float xs[4] = {xv.x, xv.y, xv.z, xv.w}, scs[4] = {sc.x, sc.y, sc.z, sc.w};
      float o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) o[j] = rs * (g[j] * scs[j] - a - (xs[j] - mu) * rs * b);
      if (aB) {
        const float4 r4 = *reinterpret_cast<const float4*>(sa + e);
        o[0] += r4.x; o[1] += r4.y; o[2] += r4.z; o[3] += r4.w;
      }
      *reinterpret_cast<float4*>(dx + row * (long)D + e) = make_float4(o[0], o[1], o[2], o[3]);
      if (tail) {
        const float4 gm = *reinterpret_cast<const float4*>(s_gamma + e);
        const float gms[4] = {gm.x, gm.y, gm.z, gm.w};
        float d[4];
        if (uB) {
          const uint2 uu = *reinterpret_cast<const uint2*>(su + e);
          const float2 u0 = unpack_bf16(uu.x), u1 = unpack_bf16(uu.y);
          const float uv[4] = {u0.x, u0.y, u1.x, u1.y};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float act = ls_gelu ? gelu_tanh_fast(uv[j]) : uv[j];
            const float dact = ls_gelu ? gelu_tanh_grad_fast(uv[j]) : 1.f;
            d[j] = o[j] * gms[j] * dact;
            tdg[c][j] += o[j] * act;
          }
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j) d[j] = o[j] * gms[j];
        }
        const uint32_t p0 = pack_bf16(d[0], d[1]), p1 = pack_bf16(d[2], d[3]);
        const float2 r0 = unpack_bf16(p0), r1 = unpack_bf16(p1);
        tdb[c][0] += r0.x; tdb[c][1] += r0.y; tdb[c][2] += r1.x; tdb[c][3] += r1.y;
        *reinterpret_cast<uint2*>(ls_du + row * (long)D + e) = make_uint2(p0, p1);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[st]);
  }

  // ---- column sums: every consumer warp has drained its rows; reuse the ring as [8 warps][D] slabs, one quantity at a
  // time; the CTA's totals go to its workspace slab [dscale | dbias | ls_dgamma | ls_dbias]
  float* slab = reinterpret_cast<float*>(ring);
  const int ct = threadIdx.x;                 // consumer threads only
#define LNR_REDUCE(ACC, DST, Q)                                                                      \
  {                                                                                                  \
    float* dst__ = (DST);                                                                            \
    asm volatile("bar.sync 1, %0;" ::"n"(32 * LNR_CONSUMERS) : "memory");                           \
    if (dst__) {                                                                                     \
      _Pragma("unroll") for (int c = 0; c < VPL; ++c)                                                \
        *reinterpret_cast<float4*>(slab + warp * D + (c * 32 + lane) * 4) =                          \
            make_float4(ACC[c][0], ACC[c][1], ACC[c][2], ACC[c][3]);                                 \
    }                                                                                                \
    asm volatile("bar.sync 1, %0;" ::"n"(32 * LNR_CONSUMERS) : "memory");                           \
    if (dst__) {                                                                                     \
      for (int e = ct; e < D; e += 32 * LNR_CONSUMERS) {                                             \
        float tot = 0.f;                                                                             \
        _Pragma("unroll") for (int w = 0; w < LNR_CONSUMERS; ++w) tot += slab[w * D + e];            \
        ws[((long)blockIdx.x * 4 + (Q)) * D + e] = tot;                                              \
      }                                                                                              \
    }                                                                                                \
  }
  LNR_REDUCE(ads, dscale, 0)
  LNR_REDUCE(adb, dscale ? dbias : nullptr, 1)
  LNR_REDUCE(tdg, (tail && uB) ? ls_dgamma : nullptr, 2)
  LNR_REDUCE(tdb, tail ? ls_dbias : nullptr, 3)
#undef LNR_REDUCE
}

// LayerScale gradient of a linear branch x + gamma * (a W + b) recovered from the weight gradient
// (dW = a^T (dx * gamma), db = colsum(dx * gamma)):   dgamma_j += (sum_i W_ij dW_ij + b_j db_j) / gamma_j.
// W bf16 [K, N] (the compute copy the forward used), dW fp32 [K, N]; one CTA per 32 columns.
__global__ void ls_gamma_from_wgrad_kernel(const __nv_bfloat16* __restrict__ W, const float* __restrict__ dW,
                                           const float* __restrict__ bias, const float* __restrict__ dbias,
                                           const float* __restrict__ gamma, float* __restrict__ ws, int K, int N) {
  // grid (N / 64, K-slabs): a thread owns two adjacent columns of a slab of rows; the 8 warps of the CTA interleave rows
  __shared__ float acc[8][64];
  const int lane = threadIdx.x & 31, wy = threadIdx.x >> 5;
  const int col = blockIdx.x * 64 + lane * 2;
  const int slab = (K + gridDim.y - 1) / gridDim.y;
  const int r0 = blockIdx.y * slab, r1 = min(K, r0 + slab);
  float s0 = 0.f, s1 = 0.f;
  if (col < N) {   // N is even
    for (int i = r0 + wy; i < r1; i += 8) {
      const float2 w = unpack_bf16(*reinterpret_cast<const uint32_t*>(W + (long)i * N + col));
      const float2 g = *reinterpret_cast<const float2*>(dW + (long)i * N + col);
      s0 += w.x * g.x; s1 += w.y * g.y;
    }
  }
  acc[wy][lane * 2] = s0; acc[wy][lane * 2 + 1] = s1;
  __syncthreads();
  if (threadIdx.x < 64) {
    const int c = blockIdx.x * 64 + threadIdx.x;
    if (c < N) {
      float tot = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) tot += acc[k][threadIdx.x];
      if (blockIdx.y == 0) tot += bias[c] * dbias[c];
      const float g = gamma[c];
      if (g != 0.f) ws[(long)blockIdx.y * N + c] = tot / g;   // this K-slab's share of dgamma[c]
    }
  }
}

// ------------------------------------------------------------------------------------------------ RoPE
// layers/attention.py:14-20,69-90 + layers/rope_position_encoding.py:117-123.  In place on the q and k thirds of
// qkv bf16 [T, 3D]; token t of each crop (N tokens) is rotated iff t >= prefix; math in fp32.
// sincos fp32 [P, hd] each.  inverse=1 applies the transpose rotation (backward).
__global__ void rope_kernel(__nv_bfloat16* __restrict__ qkv, const float* __restrict__ sin_t,
                            const float* __restrict__ cos_t, long T, int Ntok, int prefix, int D, int hd, int inverse) {
  // one thread = 8 rotation pairs: elements [i0, i0+8) and [i0+half, i0+half+8) of one head of q or k (16-byte accesses;
  // the 4 threads of a head touch one full 128-byte line).  The tables repeat their first half (angles are tiled x2).
  const int half = hd / 2;
  const int groups = half / 8;
  const int H = D / hd;
  const int items_per_row = 2 * H * groups;
  const long total = T * (long)items_per_row;
  for (long w = blockIdx.x * (long)blockDim.x + threadIdx.x; w < total; w += (long)gridDim.x * blockDim.x) {
    const long row = w / items_per_row;
    int r = (int)(w % items_per_row);
    const int t = (int)(row % Ntok);
    if (t < prefix) continue;
    const int which = r / (H * groups);
    r -= which * H * groups;
    const int head = r / groups, i0 = (r % groups) * 8;
    const float* sp = sin_t + (long)(t - prefix) * hd + i0;
    const float* cp = cos_t + (long)(t - prefix) * hd + i0;
    float sn[8], cs[8];
    *reinterpret_cast<float4*>(sn) = *reinterpret_cast<const float4*>(sp);
    *reinterpret_cast<float4*>(sn + 4) = *reinterpret_cast<const float4*>(sp + 4);
    *reinterpret_cast<float4*>(cs) = *reinterpret_cast<const float4*>(cp);
    *reinterpret_cast<float4*>(cs + 4) = *reinterpret_cast<const float4*>(cp + 4);
    __nv_bfloat16* base = qkv + row * (long)(3 * D) + which * D + head * hd + i0;
    const uint4 lo = *reinterpret_cast<const uint4*>(base);
    const uint4 hi = *reinterpret_cast<const uint4*>(base + half);
    const uint32_t lw[4] = {lo.x, lo.y, lo.z, lo.w}, hw[4] = {hi.x, hi.y, hi.z, hi.w};
    uint32_t ol[4], oh[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 a = unpack_bf16(lw[j]), b = unpack_bf16(hw[j]);
      float y1a, y1b, y2a, y2b;
      if (!inverse) {   // y = x*cos + rot_half(x)*sin, rot_half([x1,x2]) = [-x2, x1]
        y1a = a.x * cs[2 * j] - b.x * sn[2 * j];          y2a = b.x * cs[2 * j] + a.x * sn[2 * j];
        y1b = a.y * cs[2 * j + 1] - b.y * sn[2 * j + 1];  y2b = b.y * cs[2 * j + 1] + a.y * sn[2 * j + 1];
      } else {          // transpose rotation (backward)
        y1a = a.x * cs[2 * j] + b.x * sn[2 * j];          y2a = b.x * cs[2 * j] - a.x * sn[2 * j];
        y1b = a.y * cs[2 * j + 1] + b.y * sn[2 * j + 1];  y2b = b.y * cs[2 * j + 1] - a.y * sn[2 * j + 1];
      }
      ol[j] = pack_bf16(y1a, y1b);
      oh[j] = pack_bf16(y2a, y2b);
    }
    *reinterpret_cast<uint4*>(base) = make_uint4(ol[0], ol[1], ol[2], ol[3]);
    *reinterpret_cast<uint4*>(base + half) = make_uint4(oh[0], oh[1], oh[2], oh[3]);
  }
}

// ------------------------------------------------------------------------------------------------ gather / scatter
// train/ssl_meta_arch.py:377,432: patch.reshape(-1, D)[mask_indices_list]; cls rows = token 0 of each crop.
// mode 0: rows[i] = idx[i]/P*(P+1) + 1 + idx[i]%P (masked patch i -> token row); mode 1: rows[i] = i*(P+1) (cls)
__global__ void token_rows_kernel(const long long* __restrict__ idx, int* __restrict__ rows, int count, int P, int prefix,
                                  int mode) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  if (mode == 0) {
    const long long m = idx[i];
    rows[i] = (int)(m / P * (P + prefix) + prefix + m % P);
  } else {
    rows[i] = i * (P + prefix);
  }
}
__global__ void gather_rows_kernel(const float* __restrict__ src, const int* __restrict__ rows,
                                   __nv_bfloat16* __restrict__ dst_bf16, float* __restrict__ dst_f32, int R, int D) {
  for (int r = blockIdx.x; r < R; r += gridDim.x) {
    const float* s = src + (long)rows[r] * D;
    for (int e = threadIdx.x; e < D; e += blockDim.x) {
      const float v = s[e];
      if (dst_bf16) dst_bf16[(long)r * D + e] = __float2bfloat16(v);
      if (dst_f32) dst_f32[(long)r * D + e] = v;
    }
  }
}
// dst[rows[r]] += src[r]  (rows unique within a call)
template <typename InT>
__global__ void scatter_add_rows_kernel(const InT* __restrict__ src, const int* __restrict__ rows,
                                        float* __restrict__ dst, int R, int D) {
  for (int r = blockIdx.x; r < R; r += gridDim.x) {
    float* d = dst + (long)rows[r] * D;
    for (int e = threadIdx.x; e < D; e += blockDim.x) {
      float v;
      if constexpr (sizeof(InT) == 2) v = __bfloat162float(src[(long)r * D + e]); else v = src[(long)r * D + e];
      d[e] += v;
    }
  }
}

// ------------------------------------------------------------------------------------------------ L2 normalise
// layers/dino_head.py:80-82: x / (||x||_2 + 1e-12).  u fp32 [R, C] -> y bf16 [R, C]; one warp per row.
__global__ void l2norm_fwd_kernel(const float* __restrict__ u, __nv_bfloat16* __restrict__ y, float* __restrict__ nrm,
                                  int R, int C, float eps) {
  const int warps = blockDim.x >> 5, lane = threadIdx.x & 31;
  for (long row = (long)blockIdx.x * warps + (threadIdx.x >> 5); row < R; row += (long)gridDim.x * warps) {
    const float* ur = u + row * C;
    float s = 0.f;
    for (int e = lane; e < C; e += 32) s += ur[e] * ur[e];
    s = warp_sum(s);
    const float n = sqrtf(s);
    const float inv = 1.f / (n + eps);
    if (lane == 0) nrm[row] = n;
    for (int e = lane; e < C; e += 32) y[row * C + e] = __float2bfloat16(ur[e] * inv);
  }
}
// du = g/(n+eps) - u * (u.g) / (n (n+eps)^2);  g bf16 [R,C] (dgrad of the prototype layer), du bf16 out
__global__ void l2norm_bwd_kernel(const __nv_bfloat16* __restrict__ g, const float* __restrict__ u,
                                  const float* __restrict__ nrm, __nv_bfloat16* __restrict__ du, int R, int C, float eps) {
  const int warps = blockDim.x >> 5, lane = threadIdx.x & 31;
  for (long row = (long)blockIdx.x * warps + (threadIdx.x >> 5); row < R; row += (long)gridDim.x * warps) {
    const float* ur = u + row * C;
    const __nv_bfloat16* gr = g + row * C;
    float dot = 0.f;
    for (int e = lane; e < C; e += 32) dot += ur[e] * __bfloat162float(gr[e]);
    dot = warp_sum(dot);
    const float n = nrm[row];
    const float inv = 1.f / (n + eps);
    const float coef = (n > 0.f) ? dot * inv * inv / n : 0.f;
    for (int e = lane; e < C; e += 32)
      du[row * C + e] = __float2bfloat16(__bfloat162float(gr[e]) * inv - ur[e] * coef);
  }
}

// ------------------------------------------------------------------------------------------------ LayerScale / GELU bwd
// block output x_out = x_in + gamma * act(u),  act = tanh-GELU (use_gelu) or identity   (layers/block.py:198-199)
// given dX fp32 [T,D] and the bf16 stash u: du bf16 = dX*gamma*act'(u); dgamma += colsum(dX*act(u)); dbias += colsum(du).
// The same ls_tail4 as the LayerNorm backward's fused tail, on 4 columns per thread; grid.y = row slabs.
__global__ void ls_act_bwd_kernel(const float* __restrict__ dX, const __nv_bfloat16* __restrict__ u,
                                  const float* __restrict__ gamma, __nv_bfloat16* __restrict__ du,
                                  float* __restrict__ ws, int T, int D, int use_gelu) {
  const int col = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const long slab = ((long)T + gridDim.y - 1) / gridDim.y;
  const long r0 = blockIdx.y * slab, r1 = min((long)T, r0 + slab);
  if (col >= D) return;
  float gm[4], ag[4] = {0.f, 0.f, 0.f, 0.f}, ab[4] = {0.f, 0.f, 0.f, 0.f};
  load4(gamma + col, gm);
  for (long r = r0; r < r1; ++r) {
    float o[4];
    load4(dX + r * D + col, o);
    *reinterpret_cast<uint2*>(du + r * D + col) = ls_tail4(o, gm, true, u + r * D + col, use_gelu, ag, ab);
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    ws[(long)blockIdx.y * 2 * D + col + j] = ag[j];        // row slab's share of [dgamma | dbias]
    ws[(long)blockIdx.y * 2 * D + D + col + j] = ab[j];
  }
}

// ws[slab][n] = sum over the row slab of x[t, n]   (bias gradients; the slabs are added in order).  x bf16 [T, N], row
// stride ld.  blockDim = (32, 8): a thread owns 8 adjacent columns and one of 8 row phases, reduced in shared memory.
// VEC: 16-byte loads (N % 8 == 0, ld % 8 == 0, x 16-byte aligned); otherwise scalar loads of the columns < N, over the
// same walk, so the sums do not depend on the layout.
template <bool VEC>
__global__ void __launch_bounds__(256)
colsum_bf16_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ ws, long T, int N, int ld) {
  __shared__ float red[8][32][9];
  const int col = (blockIdx.x * 32 + threadIdx.x) * 8;
  const long slab = (T + gridDim.y - 1) / gridDim.y;
  const long r0 = blockIdx.y * slab, r1 = min(T, r0 + slab);
  float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (col < N) {
#pragma unroll 4
    for (long r = r0 + threadIdx.y; r < r1; r += 8) {
      if constexpr (VEC) {
        const uint4 v = *reinterpret_cast<const uint4*>(x + r * ld + col);
        const float2 f0 = unpack_bf16(v.x), f1 = unpack_bf16(v.y), f2 = unpack_bf16(v.z), f3 = unpack_bf16(v.w);
        a[0] += f0.x; a[1] += f0.y; a[2] += f1.x; a[3] += f1.y; a[4] += f2.x; a[5] += f2.y; a[6] += f3.x; a[7] += f3.y;
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (col + j < N) a[j] += __bfloat162float(x[r * ld + col + j]);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[threadIdx.y][threadIdx.x][j] = a[j];
  __syncthreads();
  // 256 threads -> 256 columns of this CTA
  const int t = threadIdx.y * 32 + threadIdx.x;
  const int lc = t >> 3, j = t & 7;
  const int c = (blockIdx.x * 32 + lc) * 8 + j;
  if (c < N) {
    float tot = 0.f;
#pragma unroll
    for (int y = 0; y < 8; ++y) tot += red[y][lc][j];
    ws[(long)blockIdx.y * N + c] = tot;
  }
}

// dst bf16 <- src fp32 (compute copy of weight matrices)
__global__ void cast_f32_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long n) {
  const long i4 = (blockIdx.x * (long)blockDim.x + threadIdx.x) * 4;
  if (i4 + 3 < n) {
    float4 v = *reinterpret_cast<const float4*>(src + i4);
    *reinterpret_cast<uint2*>(dst + i4) = make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
  } else {
    for (long i = i4; i < n; ++i) dst[i] = __float2bfloat16(src[i]);
  }
}


// ------------------------------------------------------------------------------------------------ SwiGLU gate
// SwiGLUFFN (dinov3_jax/layers/ffn_layers.py:71-76): h = silu(x1) * x2 with x1 | x2 the two halves of one [T, 2*Hs]
// bf16 buffer (the w1 / w2 projections write the halves), and its backward
//   dx1 = dh * x2 * silu'(x1),  dx2 = dh * silu(x1),   silu'(x) = s * (1 + x * (1 - s)),  s = sigmoid(x).
// 8 elements (16 bytes) per thread; Hs is a multiple of 8.
__device__ __forceinline__ float sigmoid_fast(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }

__global__ void swiglu_fwd_kernel(const __nv_bfloat16* __restrict__ x12, __nv_bfloat16* __restrict__ h, long T, int Hs) {
  const int per_row = Hs >> 3;
  const long g = blockIdx.x * (long)blockDim.x + threadIdx.x;
  if (g >= T * per_row) return;
  const long row = g / per_row;
  const int c = (int)(g - row * per_row) * 8;
  const uint4 a = *reinterpret_cast<const uint4*>(x12 + row * 2 * Hs + c);
  const uint4 b = *reinterpret_cast<const uint4*>(x12 + row * 2 * Hs + Hs + c);
  const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
  uint32_t o[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 x1 = unpack_bf16(aw[i]), x2 = unpack_bf16(bw[i]);
    o[i] = pack_bf16(x1.x * sigmoid_fast(x1.x) * x2.x, x1.y * sigmoid_fast(x1.y) * x2.y);
  }
  *reinterpret_cast<uint4*>(h + row * Hs + c) = make_uint4(o[0], o[1], o[2], o[3]);
}

__global__ void swiglu_bwd_kernel(const __nv_bfloat16* __restrict__ x12, const __nv_bfloat16* __restrict__ dh,
                                  __nv_bfloat16* __restrict__ dx12, long T, int Hs) {
  const int per_row = Hs >> 3;
  const long g = blockIdx.x * (long)blockDim.x + threadIdx.x;
  if (g >= T * per_row) return;
  const long row = g / per_row;
  const int c = (int)(g - row * per_row) * 8;
  const uint4 a = *reinterpret_cast<const uint4*>(x12 + row * 2 * Hs + c);
  const uint4 b = *reinterpret_cast<const uint4*>(x12 + row * 2 * Hs + Hs + c);
  const uint4 d = *reinterpret_cast<const uint4*>(dh + row * Hs + c);
  const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w}, dw[4] = {d.x, d.y, d.z, d.w};
  uint32_t o1[4], o2[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 x1 = unpack_bf16(aw[i]), x2 = unpack_bf16(bw[i]), g2 = unpack_bf16(dw[i]);
    const float s0 = sigmoid_fast(x1.x), s1 = sigmoid_fast(x1.y);
    o1[i] = pack_bf16(g2.x * x2.x * s0 * (1.f + x1.x * (1.f - s0)), g2.y * x2.y * s1 * (1.f + x1.y * (1.f - s1)));
    o2[i] = pack_bf16(g2.x * x1.x * s0, g2.y * x1.y * s1);
  }
  *reinterpret_cast<uint4*>(dx12 + row * 2 * Hs + c) = make_uint4(o1[0], o1[1], o1[2], o1[3]);
  *reinterpret_cast<uint4*>(dx12 + row * 2 * Hs + Hs + c) = make_uint4(o2[0], o2[1], o2[2], o2[3]);
}

// ------------------------------------------------------------------------------------------------ peer reduce-scatter
// Push-style reduce-scatter of a flat fp32 gradient range over NVLink peer mappings (replaces psum_scatter / pmean,
// fsdp/utils.py:61-64,108): element g of src (g = off + i) is added, scaled by alpha, into rank g / shard's slice.
struct PeerPtrs { float* p[8]; };
__global__ void scatter_add_peers_kernel(const float* __restrict__ src, long n4, PeerPtrs peers, unsigned long long off,
                                         unsigned shard, float alpha) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(src)[i];
    const unsigned long long g = off + (unsigned long long)i * 4;
    const unsigned r = (unsigned)(g / shard);
    float* dst = peers.p[r] + (g - (unsigned long long)r * shard);
    atomicAdd(reinterpret_cast<float4*>(dst), make_float4(v.x * alpha, v.y * alpha, v.z * alpha, v.w * alpha));
  }
}

// Bicubic resize of token feature maps [n, Hs, Ws, D] -> [n, Hd, Wd, D] (fp32): the gram teacher's patch tokens, computed
// at crops.gram_teacher_crops_size, brought to the student's patch grid (gram.global_teacher_resize_method: bicubic,
// gram.global_teacher_resize_antialias; upstream DINOv3 get_gram_teacher_output -> F.interpolate).  Definitions follow
// torch: antialias = 0 is upsample_bicubic2d (align_corners false: 4 taps, Keys a = -0.75, indices clamped to the edge),
// antialias = 1 is _upsample_bicubic2d_aa (a = -0.5, support 2 * max(scale, 1), normalised taps clipped to the map).
__device__ __forceinline__ float cubic_keys(float x, float a) {
  x = fabsf(x);
  if (x <= 1.f) return ((a + 2.f) * x - (a + 3.f)) * x * x + 1.f;
  if (x < 2.f) return ((a * x - 5.f * a) * x + 8.f * a) * x - 4.f * a;
  return 0.f;
}
constexpr int RS_TAPS = 16;
__device__ __forceinline__ int resize_taps(int o, int in, int out, int aa, int* idx, float* w) {
  const float scale = (float)in / (float)out;
  if (!aa) {
    const float real = scale * (o + 0.5f) - 0.5f;
    const float fl = floorf(real);
    const float t = real - fl;
    const int i0 = (int)fl;
    for (int k = 0; k < 4; ++k) {
      idx[k] = min(max(i0 - 1 + k, 0), in - 1);
      w[k] = cubic_keys(t + 1.f - k, -0.75f);
    }
    return 4;
  }
  const float sup = 2.f * fmaxf(scale, 1.f), inv = 1.f / fmaxf(scale, 1.f);
  const float c = scale * (o + 0.5f);
  const int lo = max((int)(c - sup + 0.5f), 0), hi = min((int)(c + sup + 0.5f), in);
  int n = 0;
  float tot = 0.f;
  for (int x = lo; x < hi && n < RS_TAPS; ++x, ++n) {
    idx[n] = x;
    w[n] = cubic_keys((x - c + 0.5f) * inv, -0.5f);
    tot += w[n];
  }
  for (int k = 0; k < n; ++k) w[k] /= tot;
  return n;
}
__global__ void resize_tokens_kernel(const float* __restrict__ src, float* __restrict__ dst, int Hs, int Ws, int Hd, int Wd,
                                     int D, int aa) {
  const int ox = blockIdx.x % Wd, oy = (blockIdx.x / Wd) % Hd, n = blockIdx.x / (Wd * Hd);
  int ix[RS_TAPS], iy[RS_TAPS];
  float wx[RS_TAPS], wy[RS_TAPS];
  const int nx = resize_taps(ox, Ws, Wd, aa, ix, wx), ny = resize_taps(oy, Hs, Hd, aa, iy, wy);
  const float* base = src + (size_t)n * Hs * Ws * D;
  float* out = dst + (((size_t)n * Hd + oy) * Wd + ox) * D;
  for (int d = threadIdx.x * 4; d < D; d += blockDim.x * 4) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int a = 0; a < ny; ++a) {
      float4 row = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int b = 0; b < nx; ++b) {
        const float4 v = *reinterpret_cast<const float4*>(base + ((size_t)iy[a] * Ws + ix[b]) * D + d);
        row.x = fmaf(wx[b], v.x, row.x); row.y = fmaf(wx[b], v.y, row.y);
        row.z = fmaf(wx[b], v.z, row.z); row.w = fmaf(wx[b], v.w, row.w);
      }
      acc.x = fmaf(wy[a], row.x, acc.x); acc.y = fmaf(wy[a], row.y, acc.y);
      acc.z = fmaf(wy[a], row.z, acc.z); acc.w = fmaf(wy[a], row.w, acc.w);
    }
    *reinterpret_cast<float4*>(out + d) = acc;
  }
}

// Small all-reduce over NVLink peer mappings (jax.lax.psum / pmax of the loss heads' K-vectors and scalars:
// loss/dino_clstoken_loss.py:53, loss/ibot_patch_loss.py:99, train/train.py:516-541): every rank reads all ranks'
// staged inputs and reduces them in rank order, so all ranks obtain bit-identical results.  One pull of world x n
// floats (n = 2K + 4 = 512 KB at K = 65536) replaces an NCCL ring whose cost at this size is pure latency.  The loads
// bypass the (non-coherent) L1: the same staging addresses are re-read every other call.
struct PeerCPtrs { const float* p[8]; };
template <int OP>
__global__ void allreduce_peers_kernel(PeerCPtrs peers, int world, float* __restrict__ out, long n4, long n) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
    float4 acc = __ldcv(reinterpret_cast<const float4*>(peers.p[0]) + i);
    for (int r = 1; r < world; ++r) {
      const float4 v = __ldcv(reinterpret_cast<const float4*>(peers.p[r]) + i);
      if (OP == 0) { acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w; }
      else { acc.x = fmaxf(acc.x, v.x); acc.y = fmaxf(acc.y, v.y); acc.z = fmaxf(acc.z, v.z); acc.w = fmaxf(acc.w, v.w); }
    }
    reinterpret_cast<float4*>(out)[i] = acc;
  }
  if (blockIdx.x == 0)
    for (long i = n4 * 4 + threadIdx.x; i < n; i += blockDim.x) {
      float acc = __ldcv(peers.p[0] + i);
      for (int r = 1; r < world; ++r) {
        const float v = __ldcv(peers.p[r] + i);
        acc = OP == 0 ? acc + v : fmaxf(acc, v);
      }
      out[i] = acc;
    }
}

}  // namespace d3

using namespace d3;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

// d3_layernorm_bwd_ls's operands
struct LnBwd {
  const void* dy;
  const float *x, *mean, *rstd, *scale, *dx_add;
  float *dx, *dscale, *dbias;
  int T, D;
  const float* ls_gamma;
  const void* ls_u;
  int ls_gelu;
  void* ls_du;
  float *ls_dgamma, *ls_dbias;
};

// Launches a LayerNorm backward kernel instance (dy of type InT) over `grid` CTAs, each writing one
// [dscale | dbias | ls_dgamma | ls_dbias] workspace slab, and adds the slabs to the outputs (nullptr: skipped; a
// quantity the kernel did not compute adds zeros).  `arg` is the kernel's int after T: D (ln_bwd_ls_kernel) or the
// ring's stage count (ln_bwd_ring_kernel).
template <typename InT, typename Kernel>
static int launch_ln_bwd(Kernel kernel, const LnBwd& a, int grid, int threads, size_t smem, int arg, cudaStream_t st) {
  float* ws = slab_workspace((size_t)grid * 4 * a.D, st);
  if (!ws) return D3_ERR_CUDA;
  kernel<<<grid, threads, smem, st>>>((const InT*)a.dy, a.x, a.mean, a.rstd, a.scale, a.dx_add, a.dx, a.dscale, a.dbias, a.T,
                                      arg, a.ls_gamma, (const __nv_bfloat16*)a.ls_u, a.ls_gelu, (__nv_bfloat16*)a.ls_du,
                                      a.ls_dgamma, a.ls_dbias, ws);
  cudaError_t e = cudaPeekAtLastError();
  int rc = e == cudaSuccess ? D3_OK : set_error(D3_ERR_CUDA, cudaGetErrorString(e));
  if (!rc) count_launch();
  float* dst[4] = {a.dscale, a.dbias, a.ls_dgamma, a.ls_dbias};
  for (int q = 0; q < 4 && !rc; ++q) rc = slab_combine(ws + (long)q * a.D, grid, 4LL * a.D, 1, a.D, dst[q], a.D, st);
  slab_release(ws, st);
  return rc;
}

template <int NC, typename InT>
static int launch_ln_bwd_ls(const LnBwd& a, cudaStream_t st) {
  const size_t smem = (size_t)4 * a.D * sizeof(float);
  static int occ = 0;
  if (!occ) {
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, ln_bwd_ls_kernel<NC, InT>, 256, smem);
    occ = max(occ, 1);
  }
  const int blocks = min((a.T + 1) / 2, sm_count() * occ);
  return launch_ln_bwd<InT>(ln_bwd_ls_kernel<NC, InT>, a, blocks, 256, smem, a.D, st);
}

template <int VPL, typename InT>
static int launch_ln_bwd_ring(const LnBwd& a, cudaStream_t st) {
  constexpr int D = VPL * 128;
  constexpr size_t fixed = 256 + 2 * D * sizeof(float);
  constexpr size_t max_stageB = (size_t)D * (4 + 4 + 4 + 2);      // x | dx_add | fp32 dy | u
  static_assert((LNR_SMEM_BUDGET - fixed) / max_stageB >= LNR_CONSUMERS, "the ring holds a stage per consumer warp");
  const size_t stageB = (size_t)D * 4 + (a.dx_add ? D * 4 : 0) + (size_t)D * sizeof(InT) + ((a.ls_gamma && a.ls_u) ? D * 2 : 0);
  int stages = (int)min((size_t)LNR_MAX_STAGES, (LNR_SMEM_BUDGET - fixed) / stageB);
  // A multiple of the consumer count: then every use of a ring stage is handled by the same consumer warp, in order, so
  // a warp can never start waiting for use u of a stage before use u-1 has completed (an mbarrier parity wait that is
  // two phases ahead would return immediately).
  stages = stages / LNR_CONSUMERS * LNR_CONSUMERS;
  const size_t need = max(stageB * stages, (size_t)LNR_CONSUMERS * D * sizeof(float));    // ring doubles as the reduction slabs
  static const cudaError_t cfg = cudaFuncSetAttribute(ln_bwd_ring_kernel<VPL, InT>,
                                                      cudaFuncAttributeMaxDynamicSharedMemorySize, LNR_SMEM_BUDGET);
  (void)cfg;   // a failure shows at the launch
  return launch_ln_bwd<InT>(ln_bwd_ring_kernel<VPL, InT>, a, min(a.T, sm_count()), 32 * (LNR_CONSUMERS + 1), fixed + need,
                            stages, st);
}

// the ring for the widths it is instantiated for, ln_bwd_ls_kernel for every other
template <typename InT>
static int launch_ln_bwd(const LnBwd& a, cudaStream_t st) {
  switch (a.D) {
    case 128: return launch_ln_bwd_ring<1, InT>(a, st);
    case 256: return launch_ln_bwd_ring<2, InT>(a, st);
    case 384: return launch_ln_bwd_ring<3, InT>(a, st);
    case 512: return launch_ln_bwd_ring<4, InT>(a, st);
    case 768: return launch_ln_bwd_ring<6, InT>(a, st);
    case 1024: return launch_ln_bwd_ring<8, InT>(a, st);
    default: break;
  }
  const int nc = (a.D + 511) / 512;
  return nc == 1 ? launch_ln_bwd_ls<1, InT>(a, st) : nc == 2 ? launch_ln_bwd_ls<2, InT>(a, st) : launch_ln_bwd_ls<3, InT>(a, st);
}

template <int VPL>
static int launch_ln_fwd(const float* x, const float* scale, const float* bias, void* y, int y_is_f32, float* mean,
                         float* rstd, int T, int D, float eps, cudaStream_t st) {
  const int blocks = min((T + 7) / 8, sm_count() * 8);
  if (y_is_f32)
    layernorm_fwd_kernel<VPL, float><<<blocks, 256, 0, st>>>(x, scale, bias, (float*)y, mean, rstd, T, eps, D);
  else
    layernorm_fwd_kernel<VPL, __nv_bfloat16><<<blocks, 256, 0, st>>>(x, scale, bias, (__nv_bfloat16*)y, mean, rstd, T, eps, D);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

constexpr size_t TOK_SMEM_MAX = 227 * 1024;
constexpr size_t TOK_SMEM_TARGET = 113 * 1024;       // two tiles per SM

template <int VPL, typename OutT>
static int launch_tokens_out(TokensOut a, int channels_first, cudaStream_t st) {
  if (!channels_first) {
    const long rows = (long)a.n * a.N;
    const int blocks = (int)min((rows + TOK_WARPS - 1) / TOK_WARPS, (long)sm_count() * 8);
    ln_tokens_out_kernel<VPL, OutT, false><<<blocks, 32 * TOK_WARPS, 0, st>>>(a);
    D3_CHECK_LAUNCH();
    return D3_OK;
  }
  const size_t row_bytes = (size_t)(a.D + TOK_PAD) * sizeof(OutT);
  // at least 32 bytes (one DRAM sector) of a channel plane per tile, 64 rows where two tiles fit on an SM
  a.tp = 64;
  while (a.tp > 32 / (int)sizeof(OutT) && a.tp * row_bytes > TOK_SMEM_TARGET) a.tp /= 2;
  const size_t smem = a.tp * row_bytes;
  if (smem > TOK_SMEM_MAX) return set_error(D3_ERR_ARG, "d3_layernorm_tokens_out: D too large for the channels-first tile");
  a.tiles_per_img = (a.P + a.tp - 1) / a.tp;
  static const cudaError_t cfg = cudaFuncSetAttribute(ln_tokens_out_kernel<VPL, OutT, true>,
                                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TOK_SMEM_MAX);
  (void)cfg;   // a failure shows at the launch
  const long prefix_rows = (long)a.n * (1 + a.R);
  const long blocks = (long)a.n * a.tiles_per_img + (prefix_rows + TOK_WARPS - 1) / TOK_WARPS;
  ln_tokens_out_kernel<VPL, OutT, true><<<(unsigned)blocks, 32 * TOK_WARPS, smem, st>>>(a);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

template <typename OutT>
static int launch_tokens_out(const TokensOut& a, int channels_first, cudaStream_t st) {
  if (!a.scale) return launch_tokens_out<0, OutT>(a, channels_first, st);    // no statistics: plain copy / conversion
  switch (a.D) {      // the widths d3_layernorm_fwd specialises, so that each row takes the same instructions
    case 128: return launch_tokens_out<1, OutT>(a, channels_first, st);
    case 256: return launch_tokens_out<2, OutT>(a, channels_first, st);
    case 384: return launch_tokens_out<3, OutT>(a, channels_first, st);
    case 512: return launch_tokens_out<4, OutT>(a, channels_first, st);
    case 768: return launch_tokens_out<6, OutT>(a, channels_first, st);
    case 1024: return launch_tokens_out<8, OutT>(a, channels_first, st);
    case 1536: return launch_tokens_out<12, OutT>(a, channels_first, st);
    default: return launch_tokens_out<0, OutT>(a, channels_first, st);
  }
}


extern "C" {

int d3_im2col(const void* img, void* out, int ld_out, int n, int H, int W, int p, void* stream) {
  if (!img || !out || H % p || W % p) return set_error(D3_ERR_ARG, "d3_im2col: bad args (H, W must divide by p)");
  if (ld_out < p * p * 3) return set_error(D3_ERR_ARG, "d3_im2col: ld_out < p*p*3");
  long runs = (long)n * (H / p) * (W / p) * p;
  int blocks = (int)min((runs + 7) / 8, (long)sm_count() * 16);
  im2col_kernel<<<blocks, 256, 0, STREAM(stream)>>>((const __nv_bfloat16*)img, (__nv_bfloat16*)out, n, H, W, p, ld_out);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_assemble_tokens(const float* tok, const float* cls, const float* storage, const float* mask_token,
                       const unsigned char* masks, float* X, int n, int P, int R, int D, void* stream) {
  if (D % 4) return set_error(D3_ERR_ARG, "d3_assemble_tokens: D % 4");
  if (R < 0 || (R > 0 && !storage)) return set_error(D3_ERR_ARG, "d3_assemble_tokens: storage tokens pointer");
  long rows = (long)n * (P + 1 + R);
  assemble_tokens_kernel<<<(int)min(rows, (long)sm_count() * 16), 128, 0, STREAM(stream)>>>(tok, cls, storage, mask_token,
                                                                                           masks, X, n, P, R, D);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_assemble_tokens_bwd(const float* dX, const unsigned char* masks, void* dTok, float* dcls, float* dstorage,
                           float* dmask, int n, int P, int R, int D, void* stream) {
  if (R < 0 || (R > 0 && !dstorage)) return set_error(D3_ERR_ARG, "d3_assemble_tokens_bwd: storage gradient pointer");
  dim3 grid((D + 127) / 128, max(1, min(n, 128)));
  cudaStream_t st = STREAM(stream);
  const long long stride = (long long)(2 + R) * D;        // per crop slab: [cls D | mask token D | storage R*D]
  float* ws = slab_workspace((size_t)grid.y * stride, st);
  if (!ws) return D3_ERR_CUDA;
  assemble_tokens_bwd_kernel<<<grid, 128, 0, st>>>(dX, masks, (__nv_bfloat16*)dTok, ws, n, P, R, D);
  cudaError_t e = cudaPeekAtLastError();
  int rc = e == cudaSuccess ? D3_OK : set_error(D3_ERR_CUDA, cudaGetErrorString(e));
  if (!rc) {
    count_launch();
    rc = slab_combine(ws, grid.y, stride, 1, D, dcls, D, st);
    if (!rc && masks) rc = slab_combine(ws + D, grid.y, stride, 1, D, dmask, D, st);
    if (!rc && R > 0) rc = slab_combine(ws + 2 * D, grid.y, stride, 1, R * D, dstorage, R * D, st);
  }
  slab_release(ws, st);
  return rc;
}

int d3_layernorm_fwd(const float* x, const float* scale, const float* bias, void* y, int y_is_f32, float* mean,
                     float* rstd, int T, int D, float eps, void* stream) {
  if (D % 4) return set_error(D3_ERR_ARG, "d3_layernorm_fwd: D % 4");
  if (((uintptr_t)x | (uintptr_t)scale | (uintptr_t)bias) % 16 || (uintptr_t)y % (y_is_f32 ? 16 : 8))
    return set_error(D3_ERR_ARG, "d3_layernorm_fwd: x, scale, bias and fp32 y must be 16-byte aligned, bf16 y 8-byte");
  cudaStream_t st = STREAM(stream);
  switch (D) {
    case 128: return launch_ln_fwd<1>(x, scale, bias, y, y_is_f32, mean, rstd, T, D, eps, st);
    case 256: return launch_ln_fwd<2>(x, scale, bias, y, y_is_f32, mean, rstd, T, D, eps, st);
    case 384: return launch_ln_fwd<3>(x, scale, bias, y, y_is_f32, mean, rstd, T, D, eps, st);
    case 512: return launch_ln_fwd<4>(x, scale, bias, y, y_is_f32, mean, rstd, T, D, eps, st);
    case 768: return launch_ln_fwd<6>(x, scale, bias, y, y_is_f32, mean, rstd, T, D, eps, st);
    case 1024: return launch_ln_fwd<8>(x, scale, bias, y, y_is_f32, mean, rstd, T, D, eps, st);
    case 1536: return launch_ln_fwd<12>(x, scale, bias, y, y_is_f32, mean, rstd, T, D, eps, st);
    default: return launch_ln_fwd<0>(x, scale, bias, y, y_is_f32, mean, rstd, T, D, eps, st);
  }
}

int d3_layernorm_tokens_out(const float* X, const float* scale, const float* bias, const float* pre_scale,
                            const float* pre_bias, float eps, int n, int N, int R, int Hp, int Wp, int D, void* cls,
                            void* storage, void* patches, int out_f32, int channels_first, void* stream) {
  if (!X || !cls || !patches || (R > 0 && !storage)) return set_error(D3_ERR_ARG, "d3_layernorm_tokens_out: null pointer");
  if (!scale != !bias || !pre_scale != !pre_bias || !scale != !pre_scale)
    return set_error(D3_ERR_ARG, "d3_layernorm_tokens_out: scale, bias, pre_scale and pre_bias are all given (norm) or all null");
  if (n < 0 || R < 0 || Hp < 1 || Wp < 1 || D < 4 || D % 4)
    return set_error(D3_ERR_ARG, "d3_layernorm_tokens_out: need n >= 0, R >= 0, Hp, Wp >= 1, D a positive multiple of 4");
  if ((long long)N != 1LL + R + (long long)Hp * Wp) return set_error(D3_ERR_ARG, "d3_layernorm_tokens_out: N != 1 + R + Hp*Wp");
  if ((long long)n * N * D >= (1LL << 40)) return set_error(D3_ERR_ARG, "d3_layernorm_tokens_out: X too large");
  const uintptr_t out_align = out_f32 ? 16 : 8;
  if (((uintptr_t)X | (uintptr_t)scale | (uintptr_t)bias | (uintptr_t)pre_scale | (uintptr_t)pre_bias) % 16 ||
      ((uintptr_t)cls | (uintptr_t)storage | (channels_first ? 0 : (uintptr_t)patches)) % out_align ||
      (uintptr_t)patches % (out_f32 ? 4 : 2))
    return set_error(D3_ERR_ARG, "d3_layernorm_tokens_out: X and the norm vectors must be 16-byte aligned, cls, storage and "
                                 "channels-last patches 16-byte (fp32) / 8-byte (bf16), channels-first patches element-aligned");
  if (n == 0) return D3_OK;
  TokensOut a{X, scale, bias, pre_scale, pre_bias, cls, storage, patches, n, N, R, Hp * Wp, D, eps, 0, 0, 0};
  // widest store whose size divides both a channel plane's byte stride and the plane base (odd grids: narrower)
  const int es = out_f32 ? 4 : 2;
  a.vec_bytes = 16;
  while (a.vec_bytes > es && (((long)a.P * es) % a.vec_bytes || (uintptr_t)patches % a.vec_bytes)) a.vec_bytes /= 2;
  cudaStream_t st = STREAM(stream);
  return out_f32 ? launch_tokens_out<float>(a, channels_first, st) : launch_tokens_out<__nv_bfloat16>(a, channels_first, st);
}

int d3_layernorm_bwd_ls(const void* dy, int dy_is_f32, const float* x, const float* mean, const float* rstd,
                        const float* scale, const float* dx_add, float* dx, float* dscale, float* dbias, int T, int D,
                        const float* ls_gamma, const void* ls_u, int ls_gelu, void* ls_du, float* ls_dgamma,
                        float* ls_dbias, void* stream) {
  if (T <= 0) return D3_OK;
  if (D % 4 != 0 || D > 1536) return set_error(D3_ERR_ARG, "d3_layernorm_bwd_ls: D must be a multiple of 4 and <= 1536");
  if (ls_gamma && !ls_du) return set_error(D3_ERR_ARG, "d3_layernorm_bwd_ls: ls_du required with ls_gamma");
  // 16-byte loads of every row operand and parameter vector, and the ring's bulk copies of whole rows
  if (((uintptr_t)dy | (uintptr_t)x | (uintptr_t)dx | (uintptr_t)scale | (uintptr_t)dx_add | (uintptr_t)ls_gamma |
       (uintptr_t)ls_u | (uintptr_t)ls_du) % 16 != 0)
    return set_error(D3_ERR_ARG, "d3_layernorm_bwd_ls: misaligned buffer (all must be 16-byte aligned)");
  const LnBwd a{dy, x, mean, rstd, scale, dx_add, dx, dscale, dbias, T, D, ls_gamma, ls_u, ls_gelu, ls_du, ls_dgamma, ls_dbias};
  return dy_is_f32 ? launch_ln_bwd<float>(a, STREAM(stream)) : launch_ln_bwd<__nv_bfloat16>(a, STREAM(stream));
}

int d3_ls_gamma_from_wgrad(const void* W, const float* dW, const float* bias, const float* dbias, const float* gamma,
                           float* dgamma, int K, int N, void* stream) {
  if (K <= 0 || N <= 0) return D3_OK;
  if (N % 2) return set_error(D3_ERR_ARG, "d3_ls_gamma_from_wgrad: N must be even");
  dim3 grid((N + 63) / 64, max(1, min(32, K / 32)));
  cudaStream_t st = STREAM(stream);
  float* ws = slab_workspace((size_t)grid.y * N, st);
  if (!ws) return D3_ERR_CUDA;
  ls_gamma_from_wgrad_kernel<<<grid, 256, 0, st>>>((const __nv_bfloat16*)W, dW, bias, dbias, gamma, ws, K, N);
  cudaError_t e = cudaPeekAtLastError();
  int rc = e == cudaSuccess ? D3_OK : set_error(D3_ERR_CUDA, cudaGetErrorString(e));
  if (!rc) { count_launch(); rc = slab_combine(ws, grid.y, N, 1, N, dgamma, N, st); }
  slab_release(ws, st);
  return rc;
}

int d3_scatter_add_peers(const float* src, long long n, float* const* peers /*host array [world]*/, int world,
                         long long off, int shard, float alpha, void* stream) {
  if (n <= 0) return D3_OK;
  if (world < 1 || world > 8 || shard <= 0 || (shard % 4) || (off % 4) || (n % 4) || ((uintptr_t)src % 16))
    return set_error(D3_ERR_ARG, "d3_scatter_add_peers: 1..8 ranks, 4-element aligned range");
  if ((unsigned long long)off + n > (unsigned long long)shard * world) return set_error(D3_ERR_ARG, "d3_scatter_add_peers: range exceeds shards");
  PeerPtrs pp;
  for (int i = 0; i < 8; ++i) pp.p[i] = i < world ? peers[i] : nullptr;
  const long n4 = n / 4;
  const int blocks = (int)min((n4 + 255) / 256, (long)sm_count() * 4);
  scatter_add_peers_kernel<<<blocks, 256, 0, STREAM(stream)>>>(src, n4, pp, (unsigned long long)off, (unsigned)shard, alpha);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_resize_tokens_bicubic(const float* src, float* dst, int n, int Hs, int Ws, int Hd, int Wd, int D, int antialias,
                             void* stream) {
  if (n <= 0) return D3_OK;
  if (Hs <= 0 || Ws <= 0 || Hd <= 0 || Wd <= 0 || D <= 0 || (D % 4) || (((uintptr_t)src | (uintptr_t)dst) % 16))
    return set_error(D3_ERR_ARG, "d3_resize_tokens_bicubic: D % 4 == 0, 16-byte aligned maps");
  if (antialias && (2.f * 2.f * fmaxf((float)Hs / Hd, (float)Ws / Wd) + 1.f > (float)RS_TAPS))
    return set_error(D3_ERR_ARG, "d3_resize_tokens_bicubic: antialiased down-scaling factor too large (<= 3.75)");
  const int threads = min(256, max(32, ((D / 4 + 31) / 32) * 32));
  resize_tokens_kernel<<<n * Hd * Wd, threads, 0, STREAM(stream)>>>(src, dst, Hs, Ws, Hd, Wd, D, antialias ? 1 : 0);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_allreduce_peers(const float* const* peers /*host array [world]*/, int world, float* out, long long n, int op,
                       void* stream) {
  if (n <= 0) return D3_OK;
  if (world < 1 || world > 8 || (op != 0 && op != 1)) return set_error(D3_ERR_ARG, "d3_allreduce_peers: 1..8 ranks, op 0 (sum) | 1 (max)");
  PeerCPtrs pp;
  long al = (long)(uintptr_t)out;
  for (int i = 0; i < 8; ++i) {
    pp.p[i] = i < world ? peers[i] : nullptr;
    if (i < world) al |= (long)(uintptr_t)peers[i];
  }
  const long n4 = (al % 16 == 0) ? n / 4 : 0;      // unaligned buffers: scalar path for everything
  const int blocks = (int)max(1L, min((n4 + 255) / 256, (long)sm_count() * 2));
  if (op == 0) allreduce_peers_kernel<0><<<blocks, 256, 0, STREAM(stream)>>>(pp, world, out, n4, n);
  else allreduce_peers_kernel<1><<<blocks, 256, 0, STREAM(stream)>>>(pp, world, out, n4, n);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_rope(void* qkv, const float* sin_t, const float* cos_t, long long T, int Ntok, int prefix, int D, int head_dim,
            int inverse, void* stream) {
  if (head_dim % 16 || D % head_dim) return set_error(D3_ERR_ARG, "d3_rope: head_dim must be a multiple of 16");
  long total = T * (long)(2 * (D / head_dim) * (head_dim / 16));
  int blocks = (int)min((total + 255) / 256, (long)sm_count() * 32);
  rope_kernel<<<blocks, 256, 0, STREAM(stream)>>>((__nv_bfloat16*)qkv, sin_t, cos_t, T, Ntok, prefix, D, head_dim,
                                                 inverse);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_token_rows(const long long* idx, int* rows, int count, int P, int prefix, int mode, void* stream) {
  if (count <= 0) return D3_OK;
  if (prefix < 1) return set_error(D3_ERR_ARG, "d3_token_rows: prefix >= 1 (cls token)");
  token_rows_kernel<<<(count + 255) / 256, 256, 0, STREAM(stream)>>>(idx, rows, count, P, prefix, mode);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_gather_rows(const float* src, const int* rows, void* dst_bf16, float* dst_f32, int R, int D, void* stream) {
  if (R <= 0) return D3_OK;
  gather_rows_kernel<<<min(R, sm_count() * 16), 128, 0, STREAM(stream)>>>(src, rows, (__nv_bfloat16*)dst_bf16, dst_f32,
                                                                          R, D);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_scatter_add_rows(const void* src, int src_is_f32, const int* rows, float* dst, int R, int D, void* stream) {
  if (R <= 0) return D3_OK;
  if (src_is_f32)
    scatter_add_rows_kernel<float><<<min(R, sm_count() * 16), 128, 0, STREAM(stream)>>>((const float*)src, rows, dst, R, D);
  else
    scatter_add_rows_kernel<__nv_bfloat16><<<min(R, sm_count() * 16), 128, 0, STREAM(stream)>>>(
        (const __nv_bfloat16*)src, rows, dst, R, D);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_l2norm_fwd(const float* u, void* y, float* nrm, int R, int C, float eps, void* stream) {
  if (R <= 0) return D3_OK;
  l2norm_fwd_kernel<<<min((R + 7) / 8, sm_count() * 8), 256, 0, STREAM(stream)>>>(u, (__nv_bfloat16*)y, nrm, R, C, eps);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_l2norm_bwd(const void* g, const float* u, const float* nrm, void* du, int R, int C, float eps, void* stream) {
  if (R <= 0) return D3_OK;
  l2norm_bwd_kernel<<<min((R + 7) / 8, sm_count() * 8), 256, 0, STREAM(stream)>>>((const __nv_bfloat16*)g, u, nrm,
                                                                                  (__nv_bfloat16*)du, R, C, eps);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_ls_act_bwd(const float* dX, const void* u, const float* gamma, void* du, float* dgamma, float* dbias, int T,
                  int D, int use_gelu, void* stream) {
  if (D % 4 || ((uintptr_t)dX | (uintptr_t)gamma) % 16 || ((uintptr_t)u | (uintptr_t)du) % 8)
    return set_error(D3_ERR_ARG, "d3_ls_act_bwd: D % 4, dX and gamma 16-byte aligned, u and du 8-byte aligned");
  dim3 grid((D / 4 + 127) / 128, min(256, max(1, T / 64)));
  cudaStream_t st = STREAM(stream);
  float* ws = slab_workspace((size_t)grid.y * 2 * D, st);
  if (!ws) return D3_ERR_CUDA;
  ls_act_bwd_kernel<<<grid, 128, 0, st>>>(dX, (const __nv_bfloat16*)u, gamma, (__nv_bfloat16*)du, ws, T, D, use_gelu);
  cudaError_t e = cudaPeekAtLastError();
  int rc = e == cudaSuccess ? D3_OK : set_error(D3_ERR_CUDA, cudaGetErrorString(e));
  if (!rc) {
    count_launch();
    rc = slab_combine(ws, grid.y, 2LL * D, 1, D, dgamma, D, st);
    if (!rc) rc = slab_combine(ws + D, grid.y, 2LL * D, 1, D, dbias, D, st);
  }
  slab_release(ws, st);
  return rc;
}

int d3_colsum_bf16(const void* x, float* out, long long T, int N, int ld, void* stream) {
  if (T <= 0) return D3_OK;
  cudaStream_t st = STREAM(stream);
  dim3 grid((N + 255) / 256);
  grid.y = (int)max(1LL, min(T / 32, (long long)(sm_count() * 8 + grid.x - 1) / grid.x));
  float* ws = slab_workspace((size_t)grid.y * N, st);
  if (!ws) return D3_ERR_CUDA;
  if (N % 8 == 0 && ld % 8 == 0 && (uintptr_t)x % 16 == 0)
    colsum_bf16_kernel<true><<<grid, dim3(32, 8), 0, st>>>((const __nv_bfloat16*)x, ws, T, N, ld);
  else
    colsum_bf16_kernel<false><<<grid, dim3(32, 8), 0, st>>>((const __nv_bfloat16*)x, ws, T, N, ld);
  cudaError_t e = cudaPeekAtLastError();
  int rc = e == cudaSuccess ? D3_OK : set_error(D3_ERR_CUDA, cudaGetErrorString(e));
  if (!rc) { count_launch(); rc = slab_combine(ws, grid.y, N, 1, N, out, N, st); }
  slab_release(ws, st);
  return rc;
}

int d3_cast_f32_bf16(const float* src, void* dst, long long n, void* stream) {
  if (n <= 0) return D3_OK;
  if (((uintptr_t)src & 15) || ((uintptr_t)dst & 7)) return set_error(D3_ERR_ARG, "d3_cast_f32_bf16: alignment");
  long th = (n + 3) / 4;
  cast_f32_bf16_kernel<<<(int)((th + 255) / 256), 256, 0, STREAM(stream)>>>(src, (__nv_bfloat16*)dst, n);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_swiglu_fwd(const void* x12, void* h, long long T, int Hs, void* stream) {
  if (T <= 0) return D3_OK;
  if (Hs % 8 || ((uintptr_t)x12 & 15) || ((uintptr_t)h & 15)) return set_error(D3_ERR_ARG, "d3_swiglu_fwd: Hs % 8, 16-byte alignment");
  const long th = T * (Hs / 8);
  swiglu_fwd_kernel<<<(int)((th + 255) / 256), 256, 0, STREAM(stream)>>>((const __nv_bfloat16*)x12, (__nv_bfloat16*)h, T, Hs);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

int d3_swiglu_bwd(const void* x12, const void* dh, void* dx12, long long T, int Hs, void* stream) {
  if (T <= 0) return D3_OK;
  if (Hs % 8 || (((uintptr_t)x12 | (uintptr_t)dh | (uintptr_t)dx12) & 15)) return set_error(D3_ERR_ARG, "d3_swiglu_bwd: Hs % 8, 16-byte alignment");
  const long th = T * (Hs / 8);
  swiglu_bwd_kernel<<<(int)((th + 255) / 256), 256, 0, STREAM(stream)>>>((const __nv_bfloat16*)x12, (const __nv_bfloat16*)dh,
                                                                      (__nv_bfloat16*)dx12, T, Hs);
  D3_CHECK_LAUNCH();
  return D3_OK;
}

}  // extern "C"
