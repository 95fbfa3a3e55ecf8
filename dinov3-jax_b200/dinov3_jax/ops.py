"""Thin Python wrappers over the C ABI (one function per exported kernel family).

Tensors are containers only: every function validates dtype / contiguity, passes raw device pointers and the
current CUDA stream, and raises NativeError on a non-zero status.  No function here computes anything in PyTorch.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from . import _native as N

bf16 = torch.bfloat16
f32 = torch.float32

# optional per-launch timing hook (bench.py roofline leg): a list that receives (kind, flops, start_evt, end_evt)
PROFILE: list | None = None


def _ld(t: torch.Tensor) -> int:
    assert t.dim() == 2 and t.stride(1) == 1, "expect 2-D row-major (unit inner stride)"
    return t.stride(0)


def _epilogue(out, Nn, bias, gelu, gelu_erf, store_pre, dgelu_of, gamma, resid, accum, alpha, scatter):
    """The d3_gemm_epilogue of a call writing `out` [M, Nn], with the flags its arguments select."""
    flags = 0
    ep = N.GemmEpilogue()
    ep.out = out.data_ptr(); ep.ld_out = _ld(out)
    if out.dtype == f32:
        flags |= N.EP_OUT_F32
    if bias is not None:
        assert bias.dtype == f32 and bias.numel() == Nn
        flags |= N.EP_BIAS; ep.bias = bias.data_ptr()
    if gelu:
        flags |= N.EP_GELU
    if gelu_erf:
        flags |= N.EP_GELU_ERF
    if store_pre is not None:
        assert store_pre.dtype == bf16 and store_pre.shape == out.shape
        flags |= N.EP_STORE_PRE; ep.aux_out = store_pre.data_ptr(); ep.ld_aux = _ld(store_pre)
    if dgelu_of is not None:
        assert dgelu_of.dtype == bf16 and dgelu_of.shape == out.shape and store_pre is None
        flags |= N.EP_MUL_DGELU; ep.aux_in = dgelu_of.data_ptr(); ep.ld_aux = _ld(dgelu_of)
    if gamma is not None:
        assert gamma.dtype == f32 and gamma.numel() == Nn
        flags |= N.EP_GAMMA; ep.gamma = gamma.data_ptr()
    if resid is not None:
        assert resid.dtype == f32 and resid.shape == out.shape
        flags |= N.EP_RESID; ep.resid = resid.data_ptr(); ep.ld_resid = _ld(resid)
    if accum:
        assert out.dtype == f32
        flags |= N.EP_ACCUM
    if scatter is not None:
        # fused reduce-scatter: (peer_ptrs, offset of out[0,0] in the sharded range, shard_len); `out` gives the geometry
        peers, sc_off, sc_shard = scatter
        assert out.dtype == f32 and out.is_contiguous() and 1 <= len(peers) <= 8
        flags |= N.EP_SCATTER
        for i, ptr in enumerate(peers):
            ep.sc_peer[i] = ptr
        ep.sc_off, ep.sc_shard, ep.sc_world = int(sc_off), int(sc_shard), len(peers)
    ep.flags = flags
    ep.alpha = float(alpha)
    return ep


def gemm(A: torch.Tensor, B: torch.Tensor, out: torch.Tensor, *, a_mn: bool = False, b_mn: bool = False,
         bias: torch.Tensor | None = None, gelu: bool = False, gelu_erf: bool = False,
         store_pre: torch.Tensor | None = None,
         dgelu_of: torch.Tensor | None = None, gamma: torch.Tensor | None = None,
         resid: torch.Tensor | None = None, accum: bool = False, alpha: float = 1.0, tile_n: int = 0,
         split_k: int = 0, scatter=None) -> torch.Tensor:
    """out[M,N] = epilogue(alpha * A.B) on the wgmma tensor cores (d3_gemm_bf16).

    A is [M,K] (a_mn=False) or stored transposed [K,M] (a_mn=True); B is [N,K] (b_mn=False) or [K,N] (b_mn=True).
    gelu: the tanh-GELU of the ViT MLP; gelu_erf: the exact GELU (torch nn.GELU()) of the ConvNeXt block.
    """
    l = N.init()
    assert A.dtype == bf16 and B.dtype == bf16
    M, K = (A.shape[1], A.shape[0]) if a_mn else (A.shape[0], A.shape[1])
    Nn, Kb = (B.shape[1], B.shape[0]) if b_mn else (B.shape[0], B.shape[1])
    assert K == Kb, f"contraction mismatch {K} vs {Kb}"
    assert out.shape[0] == M and out.shape[1] == Nn and out.dtype in (bf16, f32)
    ep = _epilogue(out, Nn, bias, gelu, gelu_erf, store_pre, dgelu_of, gamma, resid, accum, alpha, scatter)
    if PROFILE is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    N.check(l.d3_gemm_bf16(N.ptr(A), _ld(A), int(a_mn), N.ptr(B), _ld(B), int(b_mn), M, Nn, K, C.byref(ep),
                           int(tile_n), int(split_k), N.stream_ptr()), "d3_gemm_bf16")
    if PROFILE is not None:
        e1.record()
        PROFILE.append(("gemm", 2.0 * M * Nn * K, e0, e1, (M, Nn, K, int(a_mn), int(b_mn))))
    return out


def quant_rows(x: torch.Tensor, q: torch.Tensor, scale: torch.Tensor):
    """q[r] = e4m3(x[r] / scale[r]) (d3_quant_rows_e4m3): x a bf16 [R, C] view with unit inner stride, q uint8 [R, >= C]
    (its first C columns written), scale fp32 [R] receives each row's power-of-two scale."""
    l = N.init()
    R, Cc = x.shape
    assert x.dtype == bf16 and q.dtype == torch.uint8 and scale.dtype == f32 and scale.is_contiguous()
    assert q.shape[0] == R and q.shape[1] >= Cc and scale.numel() == R
    N.check(l.d3_quant_rows_e4m3(N.ptr(x), _ld(x), R, Cc, N.ptr(q), _ld(q), N.ptr(scale), N.stream_ptr()),
            "d3_quant_rows_e4m3")
    return q, scale


def quant_cols_t(W: torch.Tensor, qt: torch.Tensor, scale: torch.Tensor):
    """qt[c] = e4m3(W[:, c] / scale[c]) (d3_quant_cols_e4m3_t): W a bf16 [R, C] view, qt uint8 [C, >= R] (W^T, per
    column of W), scale fp32 [C]."""
    l = N.init()
    R, Cc = W.shape
    assert W.dtype == bf16 and qt.dtype == torch.uint8 and scale.dtype == f32 and scale.is_contiguous()
    assert qt.shape[0] == Cc and qt.shape[1] >= R and scale.numel() == Cc
    N.check(l.d3_quant_cols_e4m3_t(N.ptr(W), _ld(W), R, Cc, N.ptr(qt), _ld(qt), N.ptr(scale), N.stream_ptr()),
            "d3_quant_cols_e4m3_t")
    return qt, scale


def gemm_e4m3(A: torch.Tensor, sa: torch.Tensor, B: torch.Tensor, sb: torch.Tensor, out: torch.Tensor, *,
              bias: torch.Tensor | None = None, gelu: bool = False, store_pre: torch.Tensor | None = None,
              dgelu_of: torch.Tensor | None = None, gamma: torch.Tensor | None = None,
              resid: torch.Tensor | None = None, accum: bool = False, alpha: float = 1.0) -> torch.Tensor:
    """out[M,N] = epilogue(alpha * (A B^T) * sa[m] * sb[n]) on the FP8 tensor cores (d3_gemm_e4m3).

    A uint8 e4m3 [M, K] and B uint8 e4m3 [N, K] (both K-major: quant_rows / quant_cols_t outputs), sa / sb their fp32
    row scales; the epilogue arguments are those of `gemm`.
    """
    l = N.init()
    assert A.dtype == torch.uint8 and B.dtype == torch.uint8 and sa.dtype == f32 and sb.dtype == f32
    M, K = A.shape
    Nn, Kb = B.shape
    assert K == Kb, f"contraction mismatch {K} vs {Kb}"
    assert sa.numel() == M and sb.numel() == Nn and sa.is_contiguous() and sb.is_contiguous()
    assert out.shape[0] == M and out.shape[1] == Nn and out.dtype in (bf16, f32)
    ep = _epilogue(out, Nn, bias, gelu, False, store_pre, dgelu_of, gamma, resid, accum, alpha, None)
    if PROFILE is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    N.check(l.d3_gemm_e4m3(N.ptr(A), _ld(A), N.ptr(sa), N.ptr(B), _ld(B), N.ptr(sb), M, Nn, K, C.byref(ep),
                           N.stream_ptr()), "d3_gemm_e4m3")
    if PROFILE is not None:
        e1.record()
        PROFILE.append(("gemm_e4m3", 2.0 * M * Nn * K, e0, e1, (M, Nn, K, 0, 0)))
    return out


# --------------------------------------------------------------------------------------------------------------------
def _p(t):
    return None if t is None else t.data_ptr()


def _s():
    return torch.cuda.current_stream().cuda_stream


def im2col(img: torch.Tensor, out: torch.Tensor, patch: int) -> torch.Tensor:
    n, H, W, c = img.shape
    assert c == 3 and img.dtype == bf16 and img.is_contiguous() and out.dtype == bf16 and out.stride(1) == 1
    N.check(N.init().d3_im2col(_p(img), _p(out), out.stride(0), n, H, W, patch, _s()), "d3_im2col")
    return out


def assemble_tokens(tok, cls, mask_token, masks_u8, X, n, P, D, storage=None):
    """X [n, 1+R+P, D] = [cls | R storage tokens | patches (mask_token where masked)]; storage fp32 [R*D] or None."""
    assert tok.dtype == f32 and X.dtype == f32 and (masks_u8 is None or masks_u8.dtype == torch.uint8)
    R = 0 if storage is None else storage.numel() // D
    N.check(N.init().d3_assemble_tokens(_p(tok), _p(cls), _p(storage), _p(mask_token), _p(masks_u8), _p(X), n, P, R, D, _s()),
            "d3_assemble_tokens")
    return X


def assemble_tokens_bwd(dX, masks_u8, dTok, dcls, dmask, n, P, D, dstorage=None):
    assert dX.dtype == f32 and dTok.dtype == bf16 and dcls.dtype == f32
    R = 0 if dstorage is None else dstorage.numel() // D
    N.check(N.init().d3_assemble_tokens_bwd(_p(dX), _p(masks_u8), _p(dTok), _p(dcls), _p(dstorage), _p(dmask), n, P, R, D,
                                            _s()), "d3_assemble_tokens_bwd")


def layernorm_fwd(x, scale, bias, y, mean=None, rstd=None, eps=1e-6):
    T, D = x.shape
    assert x.dtype == f32 and x.is_contiguous() and y.shape == x.shape and y.is_contiguous()
    N.check(N.init().d3_layernorm_fwd(_p(x), _p(scale), _p(bias), _p(y), int(y.dtype == f32), _p(mean), _p(rstd), T, D,
                                      eps, _s()), "d3_layernorm_fwd")
    return y


def layernorm_tokens_out(X, cls, storage, patches, Hp, Wp, norm=None, pre_norm=None, eps=1e-6, channels_first=False):
    """One block output X [n, 1+R+Hp*Wp, D] fp32 -> cls [n, D], storage [n, R, D] (None when R == 0) and patches
    ([n, Hp*Wp, D], or [n, D, Hp, Wp] with channels_first), all fp32 or all bf16 (d3_layernorm_tokens_out).
    norm / pre_norm: (scale, bias) for the patch rows / the 1+R prefix rows (pre_norm None: the same norm); norm None:
    copied / converted only."""
    n, Ntok, D = X.shape
    R = Ntok - 1 - Hp * Wp
    out_dtype = cls.dtype
    assert X.dtype == f32 and X.is_contiguous() and out_dtype in (f32, bf16)
    assert cls.shape == (n, D) and patches.shape == ((n, D, Hp, Wp) if channels_first else (n, Hp * Wp, D))
    assert storage is None if R == 0 else storage.shape == (n, R, D)
    for t in (cls, storage, patches):
        assert t is None or (t.dtype == out_dtype and t.is_contiguous())
    pre_norm = norm if pre_norm is None else pre_norm
    sc, bi = norm if norm is not None else (None, None)
    psc, pbi = pre_norm if norm is not None else (None, None)
    N.check(N.init().d3_layernorm_tokens_out(_p(X), _p(sc), _p(bi), _p(psc), _p(pbi), float(eps), n, Ntok, R, Hp, Wp, D,
                                             _p(cls), _p(storage), _p(patches), int(out_dtype == f32), int(channels_first),
                                             _s()), "d3_layernorm_tokens_out")
    return cls, storage, patches


def layernorm_bwd_ls(dy, x, mean, rstd, scale, dx, dx_add=None, dscale=None, dbias=None, *, ls_gamma=None, ls_u=None,
                     ls_gelu=False, ls_du=None, ls_dgamma=None, ls_dbias=None):
    """LayerNorm backward + the LayerScale/activation backward of the branch upstream (d3_layernorm_bwd_ls)."""
    T, D = x.shape
    assert x.dtype == f32 and dx.dtype == f32 and (ls_du is None or ls_du.dtype == bf16)
    N.check(N.init().d3_layernorm_bwd_ls(_p(dy), int(dy.dtype == f32), _p(x), _p(mean), _p(rstd), _p(scale), _p(dx_add),
                                         _p(dx), _p(dscale), _p(dbias), T, D, _p(ls_gamma), _p(ls_u), int(ls_gelu),
                                         _p(ls_du), _p(ls_dgamma), _p(ls_dbias), _s()), "d3_layernorm_bwd_ls")


def scatter_add_peers(src, peers, off, shard, alpha):
    """alpha * src (flat fp32) added into the owners' shard slices over peer mappings (d3_scatter_add_peers)."""
    assert src.dtype == f32 and src.is_contiguous()
    arr = (C.c_void_p * len(peers))(*peers)
    N.check(N.init().d3_scatter_add_peers(_p(src), src.numel(), arr, len(peers), int(off), int(shard), float(alpha), _s()),
            "d3_scatter_add_peers")


GRAM_MODES = {(False, False): 0, (True, False): 1, (False, True): 2}      # (remove_neg, remove_only_teacher_neg)


def gram_diff(Ss, St, G, mode: int, inv_count: float, loss, block: int = 0):
    """Elementwise stage of the Gram loss (d3_gram_diff): loss += inv_count * sum (s' - t')^2, G = (s' - t') ds'/ds (bf16);
    block > 0 restricts both to the diagonal blocks of block x block tokens (per-image Gram matrices)."""
    assert Ss.dtype == f32 and St.dtype == f32 and Ss.is_contiguous() and St.is_contiguous() and Ss.numel() == St.numel()
    assert G is None or (G.dtype == bf16 and G.is_contiguous() and G.numel() == Ss.numel())
    N.check(N.init().d3_gram_diff(_p(Ss), _p(St), _p(G), Ss.numel(), int(mode), float(inv_count), _p(loss), int(Ss.shape[0]),
                                  int(block), _s()), "d3_gram_diff")


def resize_tokens_bicubic(src, dst, n, Hs, Ws, Hd, Wd, D, antialias: bool):
    """fp32 token maps [n,Hs,Ws,D] -> [n,Hd,Wd,D] (d3_resize_tokens_bicubic; torch bicubic / antialiased-bicubic arithmetic)."""
    assert src.dtype == f32 and dst.dtype == f32 and src.is_contiguous() and dst.is_contiguous()
    assert src.numel() == n * Hs * Ws * D and dst.numel() == n * Hd * Wd * D
    N.check(N.init().d3_resize_tokens_bicubic(_p(src), _p(dst), n, Hs, Ws, Hd, Wd, D, int(bool(antialias)), _s()),
            "d3_resize_tokens_bicubic")


def dwconv7_layernorm(X, w, wb, scale, bias, Y, eps=1e-6):
    """ConvNeXt block head: Y bf16 [n*H*W, C] = LayerNorm(dwconv7x7(X) + wb) per pixel; X fp32 [n, H, W, C], w fp32
    [49, C] (tap-major), zero padding 3 (d3_dwconv7_layernorm)."""
    n, H, W, Cc = X.shape
    assert X.dtype == f32 and X.is_contiguous() and Y.dtype == bf16 and Y.is_contiguous() and Y.shape == (n * H * W, Cc)
    assert w.dtype == f32 and w.is_contiguous() and w.shape == (49, Cc)
    N.check(N.init().d3_dwconv7_layernorm(_p(X), _p(w), _p(wb), _p(scale), _p(bias), float(eps), _p(Y), n, H, W, Cc, _s()),
            "d3_dwconv7_layernorm")
    return Y


def layernorm_patchify2(X, scale, bias, Y, eps=1e-6):
    """ConvNeXt downsampling: Y bf16 [n*H/2*W/2, 4C], column (kh*2 + kw)*C + c = LayerNorm(X[b, 2i+kh, 2j+kw])[c]
    (d3_layernorm_patchify2), the operand of the 2x2 stride-2 conv GEMM."""
    n, H, W, Cc = X.shape
    assert X.dtype == f32 and X.is_contiguous() and Y.dtype == bf16 and Y.is_contiguous()
    assert Y.shape == (n * (H // 2) * (W // 2), 4 * Cc)
    N.check(N.init().d3_layernorm_patchify2(_p(X), _p(scale), _p(bias), float(eps), _p(Y), n, H, W, Cc, _s()),
            "d3_layernorm_patchify2")
    return Y


def pool_tokens(X, out, copy_tokens: bool = True):
    """out fp32 [n, rows, C]: row 0 = mean over the P rows of X [n, P, C] (fixed summation order); copy_tokens (rows ==
    1 + P): rows 1..P = X (d3_pool_tokens)."""
    n, P, Cc = X.shape
    assert X.dtype == f32 and X.is_contiguous() and out.dtype == f32 and out.is_contiguous()
    assert out.dim() == 3 and out.shape[0] == n and out.shape[2] == Cc
    N.check(N.init().d3_pool_tokens(_p(X), _p(out), n, P, Cc, out.shape[1], int(bool(copy_tokens)), _s()), "d3_pool_tokens")
    return out


def resize_tokens_bilinear_aa(src, dst, Hd, Wd, prefix: int = 0):
    """fp32 maps src [n, Hs, Ws, C] -> rows prefix .. prefix + Hd*Wd - 1 of dst [n, prefix + Hd*Wd, C]: torch's
    F.interpolate(mode="bilinear", antialias=True) (d3_resize_tokens_bilinear_aa)."""
    n, Hs, Ws, Cc = src.shape
    assert src.dtype == f32 and dst.dtype == f32 and src.is_contiguous() and dst.is_contiguous()
    assert dst.shape == (n, prefix + Hd * Wd, Cc)
    N.check(N.init().d3_resize_tokens_bilinear_aa(_p(src), _p(dst), n, Hs, Ws, Hd, Wd, Cc, int(prefix), _s()),
            "d3_resize_tokens_bilinear_aa")
    return dst


def allreduce_peers(peers, out, n, op="sum"):
    """out[:n] = reduce over ranks (rank order) of the float buffers at the peer-mapped addresses `peers` (d3_allreduce_peers)."""
    assert out.dtype == f32 and out.is_contiguous() and out.numel() >= n
    arr = (C.c_void_p * len(peers))(*peers)
    N.check(N.init().d3_allreduce_peers(arr, len(peers), _p(out), int(n), {"sum": 0, "max": 1}[op], _s()), "d3_allreduce_peers")


def ls_gamma_from_wgrad(W, dW, bias, dbias, gamma, dgamma):
    K, Nn = W.shape
    assert W.dtype == bf16 and dW.dtype == f32 and W.is_contiguous() and dW.is_contiguous()
    N.check(N.init().d3_ls_gamma_from_wgrad(_p(W), _p(dW), _p(bias), _p(dbias), _p(gamma), _p(dgamma), K, Nn, _s()),
            "d3_ls_gamma_from_wgrad")


def rope(qkv, sin_t, cos_t, tokens_per_crop, prefix, D, head_dim, inverse=False):
    T = qkv.shape[0]
    assert qkv.dtype == bf16 and qkv.shape[1] == 3 * D and qkv.is_contiguous() and sin_t.dtype == f32
    N.check(N.init().d3_rope(_p(qkv), _p(sin_t), _p(cos_t), T, tokens_per_crop, prefix, D, head_dim, int(inverse),
                             _s()), "d3_rope")
    return qkv


def attn_fwd(qkv, o, lse, n_crops, Ntok, D, H):
    assert qkv.dtype == bf16 and o.dtype == bf16 and qkv.is_contiguous() and o.is_contiguous()
    N.check(N.init().d3_attn_fwd(_p(qkv), _p(o), _p(lse), n_crops, Ntok, D, H, _s()), "d3_attn_fwd")
    return o


def attn_bwd(qkv, o, do, lse, delta, dqkv, n_crops, Ntok, D, H, rope_sin=None, rope_cos=None, rope_prefix=0):
    assert all(t.dtype == bf16 and t.is_contiguous() for t in (qkv, o, do, dqkv))
    N.check(N.init().d3_attn_bwd(_p(qkv), _p(o), _p(do), _p(lse), _p(delta), _p(dqkv), n_crops, Ntok, D, H,
                                 _p(rope_sin), _p(rope_cos), rope_prefix, _s()), "d3_attn_bwd")
    return dqkv


def token_rows(mask_indices, rows, count, P, mode, prefix=1):
    assert rows.dtype == torch.int32 and (mask_indices is None or mask_indices.dtype == torch.int64)
    N.check(N.init().d3_token_rows(_p(mask_indices), _p(rows), count, P, prefix, mode, _s()), "d3_token_rows")
    return rows


def gather_rows(src, rows, R, D, dst_bf16=None, dst_f32=None):
    assert src.dtype == f32 and rows.dtype == torch.int32
    N.check(N.init().d3_gather_rows(_p(src), _p(rows), _p(dst_bf16), _p(dst_f32), R, D, _s()), "d3_gather_rows")


def scatter_add_rows(src, rows, dst, R, D):
    assert dst.dtype == f32
    N.check(N.init().d3_scatter_add_rows(_p(src), int(src.dtype == f32), _p(rows), _p(dst), R, D, _s()),
            "d3_scatter_add_rows")


def l2norm_fwd(u, y, nrm, eps=1e-12):
    R, Cc = u.shape
    assert u.dtype == f32 and y.dtype == bf16
    N.check(N.init().d3_l2norm_fwd(_p(u), _p(y), _p(nrm), R, Cc, eps, _s()), "d3_l2norm_fwd")
    return y


def l2norm_bwd(g, u, nrm, du, eps=1e-12):
    R, Cc = u.shape
    assert g.dtype == bf16 and du.dtype == bf16
    N.check(N.init().d3_l2norm_bwd(_p(g), _p(u), _p(nrm), _p(du), R, Cc, eps, _s()), "d3_l2norm_bwd")
    return du


def ls_act_bwd(dX, u, gamma, du, dgamma, dbias, use_gelu: bool):
    T, D = dX.shape
    assert dX.dtype == f32 and u.dtype == bf16 and du.dtype == bf16
    N.check(N.init().d3_ls_act_bwd(_p(dX), _p(u), _p(gamma), _p(du), _p(dgamma), _p(dbias), T, D, int(use_gelu), _s()),
            "d3_ls_act_bwd")


def colsum_bf16(x, out):
    T, Nn = x.shape
    assert x.dtype == bf16 and out.dtype == f32
    N.check(N.init().d3_colsum_bf16(_p(x), _p(out), T, Nn, x.stride(0), _s()), "d3_colsum_bf16")


def cast_f32_bf16(src, dst):
    assert src.dtype == f32 and dst.dtype == bf16 and src.numel() == dst.numel()
    N.check(N.init().d3_cast_f32_bf16(_p(src), _p(dst), src.numel(), _s()), "d3_cast_f32_bf16")


def absmax(L, out):
    N.check(N.init().d3_absmax(_p(L), L.numel(), _p(out), _s()), "d3_absmax")


def colmax(L, cm):
    """cm[k] = max(cm[k], max_b L[b,k]); cm pre-set to -inf ([K] fp32)."""
    R, K = L.shape
    N.check(N.init().d3_colmax(_p(L), _p(cm), R, K, _s()), "d3_colmax")


def sinkhorn_colsum(L, mx, temp, a, s):
    R, K = L.shape
    N.check(N.init().d3_sinkhorn_colsum(_p(L), _p(mx), temp, _p(a), _p(s), R, K, _s()), "d3_sinkhorn_colsum")


def sinkhorn_rowsum(L, mx, temp, s, btot, a):
    R, K = L.shape
    N.check(N.init().d3_sinkhorn_rowsum(_p(L), _p(mx), temp, _p(s), _p(btot), _p(a), R, K, _s()), "d3_sinkhorn_rowsum")


def sinkhorn_probs(L, mx, temp, s, a, btot, Q):
    R, K = L.shape
    N.check(N.init().d3_sinkhorn_probs(_p(L), _p(mx), temp, _p(s), _p(a), _p(btot), _p(Q), R, K, _s()),
            "d3_sinkhorn_probs")


def colsum_f32(L, out):
    R, K = L.shape
    N.check(N.init().d3_colsum_f32(_p(L), _p(out), R, K, _s()), "d3_colsum_f32")


def center_update(center, colsum, total_rows, momentum, temp, s_out):
    N.check(N.init().d3_center_update(_p(center), _p(colsum), _p(total_rows), momentum, temp, _p(s_out), center.numel(), _s()),
            "d3_center_update")


def ce_fwd_bwd(S, student_temp, Lt, mx, teacher_temp, s_t, a_t, btot, t0, t1, wm, wg, slot, metric, dS):
    Rs, K = S.shape
    assert S.dtype == f32 and Lt.dtype == f32 and (dS is None or dS.dtype == bf16) and t0.dtype == torch.int32
    N.check(N.init().d3_ce_fwd_bwd(_p(S), student_temp, _p(Lt), _p(mx), teacher_temp, _p(s_t), _p(a_t), _p(btot),
                                   _p(t0), _p(t1), _p(wm), _p(wg), _p(slot), _p(metric), _p(dS), Rs, K, _s()),
            "d3_ce_fwd_bwd")


def koleo_fwd_bwd(x, xn, nrm, nn, coef, metric, dx, w_metric, w_grad, eps=1e-8, row0=0, nrows=None):
    """KoLeo over the rows of x, with the loss terms restricted to rows [row0, row0+nrows) (default: all rows)."""
    B, D = x.shape
    assert x.dtype == f32 and nn.dtype == torch.int32
    nrows = B if nrows is None else nrows
    N.check(N.init().d3_koleo_fwd_bwd_rows(_p(x), _p(xn), _p(nrm), _p(nn), _p(coef), _p(metric), _p(dx), B, D, int(row0),
                                           int(nrows), eps, w_metric, w_grad, _s()), "d3_koleo_fwd_bwd_rows")


def koleo_topk_scratch(N, D, B, topk, device):
    """fp32 scratch for koleo_topk: the normalised rows, their norms and the chosen pairs."""
    return torch.empty(N * D + N + 2 * B * topk, dtype=f32, device=device)


def koleo_topk(x, group, row0, B, topk, scratch, metric, dx, w_metric, w_grad, eps=1e-8):
    """Top-k KoLeo of the gathered rows x [N, D]: local rows [row0, row0 + B) against the other rows of the loss group
    `group` = (g0, gn).  metric += w_metric * loss; dx [N, D] += w_grad * this rank's gradient for every row."""
    R, D = x.shape
    assert x.dtype == f32 and dx.dtype == f32 and dx.shape == x.shape and x.is_contiguous() and dx.is_contiguous()
    assert scratch.dtype == f32 and metric.dtype == f32
    g0, gn = group
    N.check(N.init().d3_koleo_topk_rows(_p(x), R, D, int(g0), int(gn), int(row0), int(B), int(topk), eps, w_metric,
                                        w_grad, _p(scratch), scratch.numel(), _p(metric), _p(dx), _s()),
            "d3_koleo_topk_rows")


def swiglu_fwd(x12, h):
    """h[T,Hs] = silu(x12[:, :Hs]) * x12[:, Hs:] (bf16)."""
    T, Hs = h.shape
    assert x12.dtype == bf16 and h.dtype == bf16 and x12.shape == (T, 2 * Hs) and x12.is_contiguous() and h.is_contiguous()
    N.check(N.init().d3_swiglu_fwd(_p(x12), _p(h), T, Hs, _s()), "d3_swiglu_fwd")


def swiglu_bwd(x12, dh, dx12):
    T, Hs = dh.shape
    assert x12.shape == (T, 2 * Hs) and dx12.shape == x12.shape and dh.is_contiguous() and dx12.is_contiguous()
    N.check(N.init().d3_swiglu_bwd(_p(x12), _p(dh), _p(dx12), T, Hs, _s()), "d3_swiglu_bwd")


def sumsq(g, out):
    N.check(N.init().d3_sumsq(_p(g), g.numel(), _p(out), _s()), "d3_sumsq")


def ema(teacher, student, t_bf16, n_bf16, momentum):
    """teacher <- momentum*teacher + (1-momentum)*student (flat fp32 shards) + bf16 re-cast of the matrix region."""
    N.check(N.init().d3_ema(_p(teacher), _p(student), _p(t_bf16), n_bf16, teacher.numel(), momentum, _s()), "d3_ema")


def adamw_ema(p, g, m, v, teacher, p_bf16, t_bf16, n_bf16, segs, nseg, sumsq_t, max_norm, lr, last_layer_lr, wd, step,
              momentum, b1=0.9, b2=0.999, eps=1e-8):
    n = p.numel()
    N.check(N.init().d3_adamw_ema(_p(p), _p(g), _p(m), _p(v), _p(teacher), _p(p_bf16), _p(t_bf16), n_bf16, _p(segs),
                                  nseg, n, _p(sumsq_t), max_norm, lr, last_layer_lr, wd, b1, b2, eps, step, momentum,
                                  _s()), "d3_adamw_ema")


# ------------------------------------------------------------------------------------------------------ k-NN evaluation
def eval_max_taps(sizes, resize: int) -> int:
    """The filter taps of the widest window d3_eval_resize_crop meets over images of (H, W) `sizes`: torch's
    2 * ceil(support) + 1 with support = 2 * max(input / resized, 1), over both axes of every image."""
    taps = 5
    for H, W in sizes:
        short, long = min(H, W), max(H, W)
        new_long = int(resize * long / short)
        for i, o in ((short, resize), (long, new_long)):
            s = i / o
            taps = max(taps, 2 * int(math.ceil(2.0 * s if s >= 1.0 else 2.0)) + 1)
    return taps


def eval_resize_crop(src: torch.Tensor, desc: torch.Tensor, out: torch.Tensor, *, resize: int, max_taps: int,
                     mean=None, std=None) -> torch.Tensor:
    """Resize(resize, bicubic, antialias) + CenterCrop of n packed uint8 HWC images (d3_eval_resize_crop).

    src uint8 (flat), desc int64 [n, 3] = (byte offset, H, W) on the device, out [n, crop, crop, 3]: bf16 normalised
    with mean / std (3 floats each), or uint8 (the crop itself, mean / std not used)."""
    n, S = out.shape[0], out.shape[1]
    assert src.dtype == torch.uint8 and src.is_contiguous() and desc.dtype == torch.int64 and desc.is_contiguous()
    assert desc.shape == (n, 3) and out.shape == (n, S, S, 3) and out.is_contiguous() and out.dtype in (bf16, torch.uint8)
    u8 = out.dtype == torch.uint8
    m = (C.c_float * 3)(*([0.0] * 3 if u8 else [float(v) for v in mean]))
    s = (C.c_float * 3)(*([1.0] * 3 if u8 else [float(v) for v in std]))
    N.check(N.init().d3_eval_resize_crop(_p(src), _p(desc), n, int(resize), S, int(max_taps), m, s, _p(out), int(u8),
                                         _s()), "d3_eval_resize_crop")
    return out


def knn_normalize(x: torch.Tensor, y_f32: torch.Tensor | None = None, y_bf16: torch.Tensor | None = None):
    """Rows of x (fp32 [R, D], unit inner stride) / max(||row||, 1e-12) into y_f32 and / or y_bf16 ([>= R, ld >= D],
    the same row stride when both are given) (d3_knn_normalize)."""
    R, D = x.shape
    assert x.dtype == f32 and (y_f32 is not None or y_bf16 is not None)
    assert y_f32 is None or (y_f32.dtype == f32 and y_f32.shape[0] >= R and y_f32.shape[1] >= D)
    assert y_bf16 is None or (y_bf16.dtype == bf16 and y_bf16.shape[0] >= R and y_bf16.shape[1] >= D)
    lds = {_ld(t) for t in (y_f32, y_bf16) if t is not None}
    assert len(lds) == 1, "y_f32 and y_bf16 need the same row stride"
    N.check(N.init().d3_knn_normalize(_p(x), _ld(x), R, D, _p(y_f32), _p(y_bf16), lds.pop(), _s()), "d3_knn_normalize")


def topk_merge(sims: torch.Tensor, top_sim: torch.Tensor, top_idx: torch.Tensor, *, offset: int, valid: int | None = None,
               fresh: bool = False):
    """Merge the similarity chunk sims (fp32 [Q, >= valid], bank indices offset + column) into the running sorted top-k
    top_sim fp32 / top_idx int32 [Q, k] (d3_topk_merge).  fresh: the running lists start empty."""
    Q = sims.shape[0]
    valid = sims.shape[1] if valid is None else int(valid)
    assert sims.dtype == f32 and top_sim.dtype == f32 and top_idx.dtype == torch.int32
    assert top_sim.shape == top_idx.shape and top_sim.shape[0] == Q and _ld(top_sim) == _ld(top_idx)
    N.check(N.init().d3_topk_merge(_p(sims), _ld(sims), Q, valid, int(offset), _p(top_sim), _p(top_idx), _ld(top_sim),
                                   top_sim.shape[1], int(bool(fresh)), _s()), "d3_topk_merge")


def knn_vote(top_sim: torch.Tensor, top_idx: torch.Tensor, labels: torch.Tensor, nb_knn, temperature: float,
             num_classes: int, preds: torch.Tensor) -> torch.Tensor:
    """preds int32 [Q, len(nb_knn), 5]: the 5 best classes of the softmax(sims[:k] / T)-weighted vote of each query's k
    first neighbours, for every k of nb_knn (d3_knn_vote)."""
    Q = top_sim.shape[0]
    nk = len(nb_knn)
    assert top_sim.dtype == f32 and top_idx.dtype == torch.int32 and labels.dtype == torch.int32 and labels.is_contiguous()
    assert preds.dtype == torch.int32 and preds.shape == (Q, nk, 5) and preds.is_contiguous()
    ks = (C.c_int * nk)(*[int(k) for k in nb_knn])
    N.check(N.init().d3_knn_vote(_p(top_sim), _p(top_idx), _ld(top_sim), Q, _p(labels), labels.numel(), ks, nk,
                                 float(temperature), int(num_classes), _p(preds), _s()), "d3_knn_vote")
    return preds


# ------------------------------------------------------------------------------------------------- linear probe
def train_max_taps(boxes, crop: int) -> int:
    """The filter taps of the widest window d3_train_resized_crop meets for crop boxes (top, left, height, width, ...)
    resized to crop x crop: torch's 2 * ceil(support) + 1 with support = 2 * max(box / crop, 1), over both axes."""
    taps = 5
    for b in boxes:
        for length in (int(b[2]), int(b[3])):
            s = length / crop
            taps = max(taps, 2 * int(math.ceil(2.0 * s if s >= 1.0 else 2.0)) + 1)
    return taps


def train_resized_crop(src: torch.Tensor, desc: torch.Tensor, boxes: torch.Tensor, out: torch.Tensor, *, max_taps: int,
                       mean=None, std=None) -> torch.Tensor:
    """torchvision resized_crop(top, left, height, width -> crop x crop, bicubic, antialias) + hflip of n packed uint8
    HWC images (d3_train_resized_crop).

    src uint8 (flat), desc int64 [n, 3] = (byte offset, H, W) and boxes int32 [n, 5] = (top, left, height, width, flip)
    on the device; out [n, crop, crop, 3]: bf16 normalised with mean / std, or uint8."""
    n, S = out.shape[0], out.shape[1]
    assert src.dtype == torch.uint8 and src.is_contiguous() and desc.dtype == torch.int64 and desc.is_contiguous()
    assert boxes.dtype == torch.int32 and boxes.is_contiguous() and boxes.shape == (n, 5) and desc.shape == (n, 3)
    assert out.shape == (n, S, S, 3) and out.is_contiguous() and out.dtype in (bf16, torch.uint8)
    u8 = out.dtype == torch.uint8
    m = (C.c_float * 3)(*([0.0] * 3 if u8 else [float(v) for v in mean]))
    s = (C.c_float * 3)(*([1.0] * 3 if u8 else [float(v) for v in std]))
    N.check(N.init().d3_train_resized_crop(_p(src), _p(desc), _p(boxes), n, S, int(max_taps), m, s, _p(out), int(u8),
                                           _s()), "d3_train_resized_crop")
    return out


def linear_inputs(srcs, out: torch.Tensor) -> torch.Tensor:
    """out[:, s*D:(s+1)*D] = bf16(srcs[s]) for fp32 [B, D] contiguous sources, in one launch (d3_linear_inputs).  out:
    bf16 [>= B, >= len(srcs) * D] with unit inner stride."""
    B, D = srcs[0].shape
    for t in srcs:
        assert t.dtype == f32 and t.is_contiguous() and t.shape == (B, D)
    assert out.dtype == bf16 and out.shape[0] >= B and out.shape[1] >= len(srcs) * D
    ptrs = (C.c_void_p * len(srcs))(*[t.data_ptr() for t in srcs])
    N.check(N.init().d3_linear_inputs(ptrs, len(srcs), B, D, _p(out), _ld(out), _s()), "d3_linear_inputs")
    return out


def linear_xent_fwd_bwd(logits: torch.Tensor, labels: torch.Tensor, num_classes: int, Cp: int, loss: torch.Tensor,
                        dz: torch.Tensor):
    """Cross-entropy of G = loss.numel() classifiers against hard labels (d3_linear_xent_fwd_bwd): logits fp32 [B, >=
    G * Cp] (classifier g in columns g*Cp .. g*Cp + num_classes), labels int32 [B]; loss fp32 [G] = batch means, dz
    bf16 [>= B, >= G * Cp] = (softmax - onehot) / B with zero padding columns."""
    B = logits.shape[0]
    G = loss.numel()
    assert logits.dtype == f32 and labels.dtype == torch.int32 and labels.is_contiguous() and labels.numel() == B
    assert loss.dtype == f32 and loss.is_contiguous() and dz.dtype == bf16 and dz.shape[0] >= B
    N.check(N.init().d3_linear_xent_fwd_bwd(_p(logits), _ld(logits), _p(labels), B, G, int(num_classes), int(Cp), _p(loss),
                                            _p(dz), _ld(dz), _s()), "d3_linear_xent_fwd_bwd")


def sgd_momentum(p: torch.Tensor, g: torch.Tensor, m: torch.Tensor, p_bf16: torch.Tensor | None, lr: torch.Tensor, Cp: int,
                 *, lr_scale: float = 1.0, momentum: float = 0.9, first: bool = False):
    """torch SGD(momentum) on fp32 [rows, cols] (or [rows]) p / g / m with lr[row // Cp] * lr_scale per row, the bf16
    copy of p into p_bf16 (d3_sgd_momentum).  first: the momentum buffer starts as the gradient."""
    rows, cols = (p.shape[0], 1) if p.dim() == 1 else tuple(p.shape)
    for t in (p, g, m):
        assert t.dtype == f32 and t.is_contiguous() and t.shape == p.shape
    assert lr.dtype == f32 and lr.is_contiguous() and lr.numel() * Cp >= rows
    assert p_bf16 is None or (p_bf16.dtype == bf16 and p_bf16.is_contiguous() and p_bf16.shape == p.shape)
    N.check(N.init().d3_sgd_momentum(_p(p), _p(g), _p(m), _p(p_bf16), rows, cols, _p(lr), int(Cp), float(lr_scale),
                                     float(momentum), int(bool(first)), _s()), "d3_sgd_momentum")


# --------------------------------------------------------------------------------------- logistic regression
def _i32(t):
    assert t.dtype == torch.int32 and t.is_contiguous()
    return _p(t)


def logreg_split_x(x: torch.Tensor, chunk: int, xa: torch.Tensor, xg: torch.Tensor | None = None):
    """xa bf16 [rows, 3K] = [Xh | Xh | Xl] of the fp32 rows x [n, K] and, with xg bf16 [3 rows, K], chunk c of xg =
    [Xh; Xl; Xh] of its rows (d3_logreg_split_x); rows = n rounded up to whole chunks, padding rows zero."""
    n, K = x.shape
    rows = -(-n // chunk) * chunk
    assert x.dtype == f32 and xa.dtype == bf16 and xa.is_contiguous() and tuple(xa.shape) == (rows, 3 * K)
    assert xg is None or (xg.dtype == bf16 and xg.is_contiguous() and tuple(xg.shape) == (3 * rows, K))
    N.check(N.init().d3_logreg_split_x(_p(x), _ld(x), n, K, int(chunk), _p(xa), _p(xg), _s()), "d3_logreg_split_x")


def logreg_weights(theta: torch.Tensor, act: torch.Tensor, Cp: int, K: int, wcat: torch.Tensor, bias: torch.Tensor):
    """wcat bf16 [Ga Cp, 3K] = [Wh | Wl | Wh] and bias fp32 [Ga Cp] of the problems in act (d3_logreg_weights)."""
    Ga = act.numel()
    assert theta.dtype == f32 and theta.is_contiguous() and theta.shape[1] == Cp * K + Cp
    assert wcat.dtype == bf16 and wcat.is_contiguous() and wcat.shape[0] >= Ga * Cp and wcat.shape[1] == 3 * K
    assert bias.dtype == f32 and bias.is_contiguous() and bias.numel() >= Ga * Cp
    N.check(N.init().d3_logreg_weights(_p(theta), theta.shape[1], _i32(act), Ga, Cp, K, _p(wcat), _p(bias), _s()),
            "d3_logreg_weights")


def logreg_xent(logits: torch.Tensor, bias: torch.Tensor, labels: torch.Tensor, n: int, Ga: int, C: int, Cp: int,
                inv_n: float, loss: torch.Tensor, r: torch.Tensor):
    """One row chunk of the cross-entropy (d3_logreg_xent): logits fp32 [rows, >= Ga Cp], labels int32 [>= n]; loss
    float64 [Ga] += the chunk's loss / N, r bf16 [3 rows, >= Ga Cp] the split residual."""
    rows = logits.shape[0]
    assert logits.dtype == f32 and bias.dtype == f32 and labels.numel() >= n and loss.dtype == torch.float64
    assert r.dtype == bf16 and r.shape[0] == 3 * rows and loss.is_contiguous() and loss.numel() >= Ga
    N.check(N.init().d3_logreg_xent(_p(logits), _ld(logits), _p(bias), _i32(labels), int(n), rows, int(Ga), int(C),
                                    int(Cp), float(inv_n), _p(loss), _p(r), _ld(r), _s()), "d3_logreg_xent")


def logreg_finish(theta, gw, gb, loss, icn, d, act, Cp: int, K: int, grad, out):
    """grad[g] = [gw_a + W_g icn_g | gb_a]; out float64 [Ga, 4] = (objective, grad . d, max |grad|, ||grad||^2)
    (d3_logreg_finish)."""
    Ga = act.numel()
    for t in (theta, gw, gb, icn, grad) + (() if d is None else (d,)):
        assert t.dtype == f32 and t.is_contiguous()
    assert loss.dtype == torch.float64 and out.dtype == torch.float64 and out.numel() >= 4 * Ga
    N.check(N.init().d3_logreg_finish(_p(theta), _p(gw), _p(gb), _p(loss), _p(icn), _p(d), _i32(act), Ga, int(Cp),
                                      int(K), _p(grad), _p(out), _s()), "d3_logreg_finish")


def logreg_trial(theta, d, alpha, act, theta_t):
    """theta_t[g] = theta[g] + alpha[g] d[g] for the slots in act (d3_logreg_trial)."""
    for t in (theta, d, alpha, theta_t):
        assert t.dtype == f32 and t.is_contiguous()
    N.check(N.init().d3_logreg_trial(_p(theta), _p(d), _p(alpha), _i32(act), act.numel(), theta.shape[1],
                                     _p(theta_t), _s()), "d3_logreg_trial")


def logreg_direction(grad, S, Y, rho, gamma, count, newest, act, d, gd):
    """d[g] = -H_g grad[g], the L-BFGS two-loop recursion over each slot's history; gd float64 [Ga] = grad . d
    (d3_logreg_direction)."""
    G, m, P = S.shape
    for t in (grad, S, Y, rho, gamma, d):
        assert t.dtype == f32 and t.is_contiguous()
    assert gd.dtype == torch.float64 and gd.numel() >= act.numel()
    N.check(N.init().d3_logreg_direction(_p(grad), _p(S), _p(Y), _p(rho), _p(gamma), _i32(count), _i32(newest),
                                         _i32(act), act.numel(), P, m, _p(d), _p(gd), _s()), "d3_logreg_direction")


def logreg_accept(theta, grad, theta_t, grad_t, S, Y, slot, act, out):
    """Pair (theta_t - theta, grad_t - grad) into slot[g] of S / Y, theta = theta_t, grad = grad_t; out float64
    [Ga, 3] = (s.y, y.y, s.s) (d3_logreg_accept)."""
    G, m, P = S.shape
    for t in (theta, grad, theta_t, grad_t, S, Y):
        assert t.dtype == f32 and t.is_contiguous()
    assert out.dtype == torch.float64 and out.numel() >= 3 * act.numel()
    N.check(N.init().d3_logreg_accept(_p(theta), _p(grad), _p(theta_t), _p(grad_t), _p(S), _p(Y), _i32(slot),
                                      _i32(act), act.numel(), P, m, _p(out), _s()), "d3_logreg_accept")


# --------------------------------------------------------------------------------------------- attentive probe
def _f32c(*ts):
    for t in ts:
        assert t.dtype == f32 and t.is_contiguous(), "expect contiguous fp32"


def atp_query_fwd(q0, Wq, bq, Wk, H: int, q, kt):
    """q = Wq q0 + bq (fp32 [D]) and the folded keys kt fp32 [H, D] = Wk_h^T q_h / sqrt(D / H) (d3_atp_query_fwd)."""
    D = q0.numel()
    _f32c(q0, Wq, bq, Wk, q, kt)
    assert Wq.shape == (D, D) and Wk.shape == (D, D) and bq.numel() == D and q.numel() == D and kt.shape == (H, D)
    N.check(N.init().d3_atp_query_fwd(_p(q0), _p(Wq), _p(bq), _p(Wk), D, int(H), _p(q), _p(kt), _s()),
            "d3_atp_query_fwd")


def atp_query_bwd(q0, Wq, Wk, q, dkt, dWq, dbq, dWk, dq0):
    """From dkt [H, D]: dWk, dWq [D, D] and dbq [D] written, dq0 [D] += Wq^T dq (d3_atp_query_bwd)."""
    H, D = dkt.shape
    _f32c(q0, Wq, Wk, q, dkt, dWq, dbq, dWk, dq0)
    assert dWq.shape == (D, D) and dWk.shape == (D, D) and dbq.numel() == D and dq0.numel() == D
    N.check(N.init().d3_atp_query_bwd(_p(q0), _p(Wq), _p(Wk), _p(q), _p(dkt), D, H, _p(dWq), _p(dbq), _p(dWk), _p(dq0),
                                      _s()), "d3_atp_query_bwd")


def atp_pool_fwd(x: torch.Tensor, T: int, e, g1, b1, kt, ybar, lse):
    """The folded pooling (d3_atp_pool_fwd): x bf16 [B, T * P, D] -> ybar fp32 [B, H, D] = sum_n p_{n,h} LN1(x_n + e_t),
    lse fp32 [B, H]."""
    B, NT, D = x.shape
    H = kt.shape[0]
    assert x.dtype == bf16 and x.is_contiguous() and NT % int(T) == 0
    _f32c(e, g1, b1, kt, ybar, lse)
    assert e.shape == (T, D) and g1.numel() == D and b1.numel() == D and ybar.shape == (B, H, D) and lse.shape == (B, H)
    N.check(N.init().d3_atp_pool_fwd(_p(x), _p(e), _p(g1), _p(b1), _p(kt), B, int(T), NT // int(T), D, H, _p(ybar),
                                     _p(lse), _s()), "d3_atp_pool_fwd")


def atp_pool_bwd(x: torch.Tensor, T: int, e, g1, b1, kt, lse, ybar, dybar, dkt, dg1, db1, de):
    """The pooling's backward (d3_atp_pool_bwd): from dybar fp32 [B, H, D], dkt [H, D], dg1, db1 [D] and de [T, D]
    written (summed over the clips)."""
    B, NT, D = x.shape
    H = kt.shape[0]
    assert x.dtype == bf16 and x.is_contiguous() and NT % int(T) == 0
    _f32c(e, g1, b1, kt, lse, ybar, dybar, dkt, dg1, db1, de)
    assert ybar.shape == (B, H, D) and dybar.shape == (B, H, D) and lse.shape == (B, H) and dkt.shape == (H, D)
    assert e.shape == (T, D) and de.shape == (T, D) and dg1.numel() == D and db1.numel() == D
    N.check(N.init().d3_atp_pool_bwd(_p(x), _p(e), _p(g1), _p(b1), _p(kt), _p(lse), _p(ybar), _p(dybar), B, int(T),
                                     NT // int(T), D, H, _p(dkt), _p(dg1), _p(db1), _p(de), _s()), "d3_atp_pool_bwd")


def atp_gelu_erf_bwd(dh: torch.Tensor, pre: torch.Tensor, out: torch.Tensor):
    """out bf16 [rows, cols] = dh fp32 * GELU_erf'(pre bf16) (d3_atp_gelu_erf_bwd); row-major views."""
    rows, cols = dh.shape
    assert dh.dtype == f32 and pre.dtype == bf16 and out.dtype == bf16
    assert pre.shape == (rows, cols) and out.shape == (rows, cols)
    N.check(N.init().d3_atp_gelu_erf_bwd(_p(dh), _ld(dh), _p(pre), _ld(pre), rows, cols, _p(out), _ld(out), _s()),
            "d3_atp_gelu_erf_bwd")


# ------------------------------------------------------------------------------------------ segmentation probe
def seg_max_taps(sizes, resized) -> int:
    """The filter taps of the widest window d3_seg_crop meets for images of (H, W) `sizes` resized to (rh, rw)
    `resized`: torch's 2 * ceil(support) + 1 with support = 2 * max(input / resized, 1), over both axes."""
    taps = 5
    for (H, W), (rh, rw) in zip(sizes, resized):
        for i, o in ((int(H), int(rh)), (int(W), int(rw))):
            s = i / o
            taps = max(taps, 2 * int(math.ceil(2.0 * s if s >= 1.0 else 2.0)) + 1)
    return taps


def seg_crop(src: torch.Tensor, desc: torch.Tensor, boxes: torch.Tensor, out: torch.Tensor, *, max_taps: int,
             labels: torch.Tensor | None = None, label_out: torch.Tensor | None = None, mean=None, std=None):
    """Resize + crop + flip of n packed uint8 HWC images and their label maps (d3_seg_crop).

    src uint8 (flat), desc int64 [n, 3] = (byte offset, H, W), boxes int32 [n, 6] = (rh, rw, top, left, flip, 0) on the
    device; out [n, out_h, out_w, 3]: bf16 normalised with mean / std, or uint8.  labels: uint8 (flat, image n's map at
    offset desc[n, 0] / 3) and label_out uint8 [n, out_h, out_w], or both None."""
    n, Ho, Wo = out.shape[0], out.shape[1], out.shape[2]
    assert src.dtype == torch.uint8 and src.is_contiguous() and desc.dtype == torch.int64 and desc.is_contiguous()
    assert boxes.dtype == torch.int32 and boxes.is_contiguous() and boxes.shape == (n, 6) and desc.shape == (n, 3)
    assert out.shape == (n, Ho, Wo, 3) and out.is_contiguous() and out.dtype in (bf16, torch.uint8)
    assert (labels is None) == (label_out is None)
    if label_out is not None:
        assert labels.dtype == torch.uint8 and labels.is_contiguous()
        assert label_out.dtype == torch.uint8 and label_out.is_contiguous() and label_out.shape == (n, Ho, Wo)
    u8 = out.dtype == torch.uint8
    m = (C.c_float * 3)(*([0.0] * 3 if u8 else [float(v) for v in mean]))
    s = (C.c_float * 3)(*([1.0] * 3 if u8 else [float(v) for v in std]))
    N.check(N.init().d3_seg_crop(_p(src), _p(desc), _p(labels), _p(boxes), n, Ho, Wo, int(max_taps), m, s, _p(out),
                                 int(u8), _p(label_out), _s()), "d3_seg_crop")
    return out


def seg_bn_stats(x: torch.Tensor, mean: torch.Tensor, var: torch.Tensor, running_mean: torch.Tensor | None = None,
                 running_var: torch.Tensor | None = None, momentum: float = 0.1):
    """Column mean and biased variance of bf16 x [M, N] into fp32 [N] mean / var; the running statistics (both or
    neither) are updated as torch's BatchNorm in training mode does (d3_seg_bn_stats)."""
    M, Nn = x.shape
    assert x.dtype == bf16
    for t in (mean, var, running_mean, running_var):
        assert t is None or (t.dtype == f32 and t.is_contiguous() and t.numel() == Nn)
    N.check(N.init().d3_seg_bn_stats(_p(x), _ld(x), M, Nn, _p(mean), _p(var), _p(running_mean), _p(running_var),
                                     float(momentum), _s()), "d3_seg_bn_stats")


def seg_bn_apply(x: torch.Tensor, mean: torch.Tensor, var: torch.Tensor, out: torch.Tensor, eps: float = 1e-5):
    """out = bf16((x - mean) / sqrt(var + eps)) per column of bf16 x [M, N] (d3_seg_bn_apply)."""
    M, Nn = x.shape
    assert x.dtype == bf16 and out.dtype == bf16 and out.shape[0] >= M and out.shape[1] >= Nn
    assert mean.dtype == f32 and var.dtype == f32 and mean.numel() == Nn and var.numel() == Nn
    N.check(N.init().d3_seg_bn_apply(_p(x), _ld(x), M, Nn, _p(mean), _p(var), float(eps), _p(out), _ld(out), _s()),
            "d3_seg_bn_apply")
    return out


def seg_xent_fwd_bwd(logits: torch.Tensor, labels: torch.Tensor, hw, num_classes: int, loss: torch.Tensor,
                     count: torch.Tensor, dz_f32: torch.Tensor | None = None, dz_bf16: torch.Tensor | None = None,
                     Cp: int | None = None):
    """Mean cross-entropy over the valid pixels (label < num_classes; 255 is the ignore label) of the patch logits
    upsampled bilinearly (align_corners=False) to the label size, and its gradient to the patch logits
    (d3_seg_xent_fwd_bwd).  logits fp32 [B * h * w, >= num_classes] (ld any), labels uint8 [B, Hl, Wl], hw = (h, w);
    loss fp32 [1], count int32 [1]; dz_f32 / dz_bf16 [>= B * h * w, >= Cp] (columns [num_classes, Cp) zeroed)."""
    B, Hl, Wl = labels.shape
    h, w = int(hw[0]), int(hw[1])
    Cp = int(num_classes) if Cp is None else int(Cp)
    assert logits.dtype == f32 and logits.shape[0] >= B * h * w and labels.dtype == torch.uint8 and labels.is_contiguous()
    assert loss.dtype == f32 and count.dtype == torch.int32
    ld = None
    for t, dt in ((dz_f32, f32), (dz_bf16, bf16)):
        if t is not None:
            assert t.dtype == dt and t.shape[0] >= B * h * w and t.shape[1] >= Cp
            assert ld is None or ld == _ld(t), "dz_f32 and dz_bf16 share one row stride"
            ld = _ld(t)
    N.check(N.init().d3_seg_xent_fwd_bwd(_p(logits), _ld(logits), _p(labels), B, h, w, Hl, Wl, int(num_classes), Cp,
                                         _p(loss), _p(count), _p(dz_f32), _p(dz_bf16), ld or Cp, _s()),
            "d3_seg_xent_fwd_bwd")


def seg_predict_confusion(logits: torch.Tensor, labels: torch.Tensor, hw, num_classes: int, conf: torch.Tensor):
    """conf int64 [C, C] += counts of (label, argmax of the upsampled logits) over the pixels with label < C
    (d3_seg_predict_confusion); shapes as seg_xent_fwd_bwd."""
    B, Hl, Wl = labels.shape
    h, w = int(hw[0]), int(hw[1])
    C_ = int(num_classes)
    assert logits.dtype == f32 and logits.shape[0] >= B * h * w and labels.dtype == torch.uint8 and labels.is_contiguous()
    assert conf.dtype == torch.int64 and conf.is_contiguous() and conf.shape == (C_, C_)
    N.check(N.init().d3_seg_predict_confusion(_p(logits), _ld(logits), _p(labels), B, h, w, Hl, Wl, C_, _p(conf), _s()),
            "d3_seg_predict_confusion")
    return conf


# ------------------------------------------------------------------------------------------ depth probe
def depth_crop(src: torch.Tensor, desc: torch.Tensor, boxes: torch.Tensor, out: torch.Tensor, *, max_taps: int,
               depths: torch.Tensor | None = None, depth_out: torch.Tensor | None = None, mean=None, std=None):
    """seg_crop's image (the same bits) and, optionally, the fp32 depth planes cropped from the same boxes by torch's
    'nearest', 0 outside the resized image (d3_depth_crop).  depths: fp32 (flat, image n's plane at element
    desc[n, 0] / 3) and depth_out fp32 [n, out_h, out_w], or both None; the rest as seg_crop."""
    n, Ho, Wo = out.shape[0], out.shape[1], out.shape[2]
    assert src.dtype == torch.uint8 and src.is_contiguous() and desc.dtype == torch.int64 and desc.is_contiguous()
    assert boxes.dtype == torch.int32 and boxes.is_contiguous() and boxes.shape == (n, 6) and desc.shape == (n, 3)
    assert out.shape == (n, Ho, Wo, 3) and out.is_contiguous() and out.dtype in (bf16, torch.uint8)
    assert (depths is None) == (depth_out is None)
    if depth_out is not None:
        assert depths.dtype == f32 and depths.is_contiguous()
        assert depth_out.dtype == f32 and depth_out.is_contiguous() and depth_out.shape == (n, Ho, Wo)
    u8 = out.dtype == torch.uint8
    m = (C.c_float * 3)(*([0.0] * 3 if u8 else [float(v) for v in mean]))
    s = (C.c_float * 3)(*([1.0] * 3 if u8 else [float(v) for v in std]))
    N.check(N.init().d3_depth_crop(_p(src), _p(desc), _p(depths), _p(boxes), n, Ho, Wo, int(max_taps), m, s, _p(out),
                                   int(u8), _p(depth_out), _s()), "d3_depth_crop")
    return out


def depth_head_fwd_bwd(logits: torch.Tensor, gt: torch.Tensor, hw, n_bins: int, min_depth: float, max_depth: float,
                       loss: torch.Tensor, count: torch.Tensor, dz_f32: torch.Tensor | None = None,
                       dz_bf16: torch.Tensor | None = None, Cp: int | None = None):
    """The scale-invariant log loss of the "linear" bin head's depth, upsampled bilinearly (align_corners=False) to the
    ground truth, over its valid pixels (min_depth < gt <= max_depth), and its gradient to the bin logits
    (d3_depth_head_fwd_bwd).  logits fp32 [B * h * w, >= n_bins] (ld any), gt fp32 [B, Hl, Wl], hw = (h, w); loss fp32
    [1], count int32 [1]; dz_f32 / dz_bf16 [>= B * h * w, >= Cp] (columns [n_bins, Cp) zeroed)."""
    B, Hl, Wl = gt.shape
    h, w = int(hw[0]), int(hw[1])
    Cp = int(n_bins) if Cp is None else int(Cp)
    assert logits.dtype == f32 and logits.shape[0] >= B * h * w and gt.dtype == f32 and gt.is_contiguous()
    assert loss.dtype == f32 and count.dtype == torch.int32
    ld = None
    for t, dt in ((dz_f32, f32), (dz_bf16, bf16)):
        if t is not None:
            assert t.dtype == dt and t.shape[0] >= B * h * w and t.shape[1] >= Cp
            assert ld is None or ld == _ld(t), "dz_f32 and dz_bf16 share one row stride"
            ld = _ld(t)
    N.check(N.init().d3_depth_head_fwd_bwd(_p(logits), _ld(logits), _p(gt), B, h, w, Hl, Wl, int(n_bins), Cp,
                                           float(min_depth), float(max_depth), _p(loss), _p(count), _p(dz_f32),
                                           _p(dz_bf16), ld or Cp, _s()), "d3_depth_head_fwd_bwd")


def depth_predict_metrics(logits: torch.Tensor, gt: torch.Tensor, hw, n_bins: int, min_depth: float, max_depth: float,
                          sums: torch.Tensor, crop=None):
    """sums fp64 [B, 9] = per image, over the valid pixels inside crop = (top, bottom, left, right) (None: all): the
    count and the sums of abs_rel, sq_rel, squared error, squared log error, |log10 error| and the a1, a2, a3 hits of
    the upsampled depth clamped to [min_depth, max_depth] (d3_depth_predict_metrics); shapes as depth_head_fwd_bwd."""
    B, Hl, Wl = gt.shape
    h, w = int(hw[0]), int(hw[1])
    assert logits.dtype == f32 and logits.shape[0] >= B * h * w and gt.dtype == f32 and gt.is_contiguous()
    assert sums.dtype == torch.float64 and sums.is_contiguous() and sums.shape == (B, 9)
    top, bottom, left, right = (0, Hl, 0, Wl) if crop is None else (int(v) for v in crop)
    N.check(N.init().d3_depth_predict_metrics(_p(logits), _ld(logits), _p(gt), B, h, w, Hl, Wl, int(n_bins),
                                              float(min_depth), float(max_depth), top, bottom, left, right, _p(sums),
                                              _s()), "d3_depth_predict_metrics")
    return sums


# ------------------------------------------------------------------------------------------ video segmentation
def video_resize(src: torch.Tensor, desc: torch.Tensor, out: torch.Tensor, *, mean, std) -> torch.Tensor:
    """torch bilinear (align_corners=False, antialias=False) of n packed uint8 HWC frames / 255 to out bf16 [n, H, W, 3],
    normalised with mean / std (d3_video_resize).  src uint8 (flat), desc int64 [n, 3] = (byte offset, H, W)."""
    n, Ho, Wo = out.shape[0], out.shape[1], out.shape[2]
    assert src.dtype == torch.uint8 and src.is_contiguous() and desc.dtype == torch.int64 and desc.is_contiguous()
    assert desc.shape == (n, 3) and out.shape == (n, Ho, Wo, 3) and out.is_contiguous() and out.dtype == bf16
    m = (C.c_float * 3)(*[float(v) for v in mean])
    s = (C.c_float * 3)(*[float(v) for v in std])
    N.check(N.init().d3_video_resize(_p(src), _p(desc), n, Ho, Wo, m, s, _p(out), _s()), "d3_video_resize")
    return out


def video_propagate(sim0: torch.Tensor, simr: torch.Tensor | None, lab0: torch.Tensor, labr: torch.Tensor | None,
                    hw, radius: int, topk: int, temperature: float, out: torch.Tensor) -> torch.Tensor:
    """out fp32 [h * w, C] = the soft labels of one target frame propagated from frame 0 (sim0 fp32 [h * w, >= h * w]
    similarities, lab0 fp32 [h * w, C] labels) and the recent frames (simr fp32 [h * w, >= n * h * w], frame c at
    columns [c h w, (c + 1) h w), labr fp32 [n * h * w, C]; both None when there are none) (d3_video_propagate)."""
    h, w = int(hw[0]), int(hw[1])
    P, Cc = h * w, lab0.shape[1]
    assert sim0.dtype == f32 and sim0.shape[0] == P and sim0.shape[1] >= P
    assert lab0.dtype == f32 and lab0.is_contiguous() and lab0.shape == (P, Cc)
    assert out.dtype == f32 and out.is_contiguous() and out.shape == (P, Cc)
    assert (simr is None) == (labr is None)
    n = 0
    if labr is not None:
        assert labr.dtype == f32 and labr.is_contiguous() and labr.shape[1] == Cc and labr.shape[0] % P == 0
        n = labr.shape[0] // P
        assert simr.dtype == f32 and simr.shape[0] == P and simr.shape[1] >= n * P
    N.check(N.init().d3_video_propagate(_p(sim0), _ld(sim0), _p(simr), _ld(simr) if simr is not None else 0, _p(lab0),
                                        _p(labr), n, h, w, Cc, int(radius), int(topk), float(temperature), _p(out),
                                        _s()), "d3_video_propagate")
    return out


def video_label_map(soft: torch.Tensor, hw, patch: int, out: torch.Tensor) -> torch.Tensor:
    """out uint8 [H, W] = the argmax label map of the soft labels fp32 [h * w, C] upsampled by `patch` (bilinear),
    min-max normalised per channel and sampled by nearest-exact at H x W (d3_video_label_map)."""
    h, w = int(hw[0]), int(hw[1])
    assert soft.dtype == f32 and soft.is_contiguous() and soft.dim() == 2 and soft.shape[0] == h * w
    assert out.dtype == torch.uint8 and out.is_contiguous() and out.dim() == 2
    N.check(N.init().d3_video_label_map(_p(soft), h, w, soft.shape[1], int(patch), out.shape[0], out.shape[1], _p(out),
                                        _s()), "d3_video_label_map")
    return out


def video_jf_counts(pred: torch.Tensor, gt: torch.Tensor, num_objects: int, radius: int,
                    counts: torch.Tensor) -> torch.Tensor:
    """counts int64 [F, K, 6] = per frame and object 1..K: intersection, union (void = gt 255 excluded), pred and gt
    boundary pixels, pred and gt boundary pixels matched within the disk of `radius` (d3_video_jf_counts).  pred, gt
    uint8 [F, H, W]."""
    F_, H, W = gt.shape
    K = int(num_objects)
    assert pred.dtype == torch.uint8 and gt.dtype == torch.uint8 and pred.shape == gt.shape
    assert pred.is_contiguous() and gt.is_contiguous()
    assert counts.dtype == torch.int64 and counts.is_contiguous() and counts.shape == (F_, K, 6)
    N.check(N.init().d3_video_jf_counts(_p(pred), _p(gt), F_, H, W, K, int(radius), _p(counts), _s()),
            "d3_video_jf_counts")
    return counts


# ------------------------------------------------------------------------------------------ keypoint correspondence
def corr_descriptors(feats: torch.Tensor, n_maps: int, hw, out_hw, kp, out: torch.Tensor,
                     qnorm: torch.Tensor) -> torch.Tensor:
    """out bf16 [K, D] row k = the bilinear upsampling (align_corners=False) of patch map kp[k, 0] (feats bf16
    [n_maps * h * w, D] rows) to out_hw sampled at pixel (x, y) = kp[k, 1:], L2-normalised; qnorm fp32 [K] the norms of
    the rounded rows (d3_corr_descriptors).  kp: host integers [K, 3] = (map, x, y), checked before any launch."""
    h, w = int(hw[0]), int(hw[1])
    rows = [[int(v) for v in r] for r in kp]
    assert all(len(r) == 3 for r in rows), "kp: (map, x, y) per keypoint"
    K, D = len(rows), feats.shape[1]
    kp_host = (C.c_int * (3 * K))(*[v for r in rows for v in r])
    assert feats.dtype == bf16 and feats.shape[0] >= int(n_maps) * h * w
    assert out.dtype == bf16 and out.shape[0] == K and out.shape[1] == D
    assert qnorm.dtype == f32 and qnorm.is_contiguous() and qnorm.shape == (K,)
    N.check(N.init().d3_corr_descriptors(_p(feats), _ld(feats), int(n_maps), h, w, D, int(out_hw[0]), int(out_hw[1]),
                                         kp_host, K, _p(out), _ld(out), _p(qnorm), _s()), "d3_corr_descriptors")
    return out


def corr_gram(feats: torch.Tensor, n_maps: int, hw, gram: torch.Tensor) -> torch.Tensor:
    """gram fp32 [n_maps * h * w, 5] = per patch its squared norm and its dot products with the right, lower,
    lower-right and lower-left neighbours (0 where there is none) (d3_corr_gram)."""
    h, w = int(hw[0]), int(hw[1])
    assert feats.dtype == bf16 and feats.shape[0] >= int(n_maps) * h * w
    assert gram.dtype == f32 and gram.is_contiguous() and gram.shape == (int(n_maps) * h * w, 5)
    N.check(N.init().d3_corr_gram(_p(feats), _ld(feats), int(n_maps), h, w, feats.shape[1], _p(gram), _s()),
            "d3_corr_gram")
    return gram


def corr_argmax(sim: torch.Tensor, gram: torch.Tensor, qnorm: torch.Tensor, hw, out_hw, xy: torch.Tensor,
                cosine: torch.Tensor):
    """For each of K keypoints, the pixel xy int32 [K, 2] = (x, y) of the out_hw bilinear upsampling of one target map
    with the largest cosine to the descriptor, and that cosine fp32 [K] (d3_corr_argmax).  sim fp32 [K, >= h * w]: the
    descriptors' dot products with the target's patches; gram fp32 [h * w, 5] the target's (corr_gram); qnorm fp32 [K]
    the descriptors' norms (corr_descriptors).  Ties go to the lowest y * out_w + x."""
    h, w = int(hw[0]), int(hw[1])
    K = sim.shape[0]
    assert sim.dtype == f32 and sim.shape[1] >= h * w
    assert gram.dtype == f32 and gram.is_contiguous() and gram.shape == (h * w, 5)
    assert qnorm.dtype == f32 and qnorm.is_contiguous() and qnorm.shape == (K,)
    assert xy.dtype == torch.int32 and xy.is_contiguous() and xy.shape == (K, 2)
    assert cosine.dtype == f32 and cosine.is_contiguous() and cosine.shape == (K,)
    N.check(N.init().d3_corr_argmax(_p(sim), _ld(sim), _p(gram), _p(qnorm), K, h, w, int(out_hw[0]), int(out_hw[1]),
                                    _p(xy), _p(cosine), _s()), "d3_corr_argmax")
    return xy, cosine



# ------------------------------------------------------------------------------------------ object discovery
def od_graph(sim: torch.Tensor, tau: float, eps: float, bits: torch.Tensor, degree: torch.Tensor):
    """The thresholded patch graph of n images of P patches (d3_od_graph): bits int32 [n, P, ceil(P / 32)] (bit j % 32
    of word j / 32 of row i set when sim[m, i, j] > tau) and degree fp32 [n, P] = c_i + (P - c_i) eps.  sim fp32
    [n, P, P], a view with unit inner stride of a buffer whose rows hold a multiple of 4 floats."""
    n, P = sim.shape[0], sim.shape[1]
    assert sim.dtype == f32 and sim.dim() == 3 and sim.shape[2] == P and sim.stride(2) == 1
    assert sim.stride(0) == P * sim.stride(1), "the images' rows must follow one another"
    assert bits.dtype == torch.int32 and bits.is_contiguous() and bits.shape == (n, P, -(-P // 32))
    assert degree.dtype == f32 and degree.is_contiguous() and degree.shape == (n, P)
    N.check(N.init().d3_od_graph(_p(sim), sim.stride(1), n, P, float(tau), float(eps), _p(bits), _p(degree), _s()),
            "d3_od_graph")
    return bits, degree


def od_fiedler(bits: torch.Tensor, degree: torch.Tensor, eps: float, x: torch.Tensor, lambda2: torch.Tensor,
               iters: torch.Tensor, converged: torch.Tensor, k_max: int = 256):
    """The normalized-cut eigenvector of each image's graph (d3_od_fiedler): x fp32 [n, P] solves (D - A) x = lambda D x
    at the second-smallest lambda (lambda2 fp32 [n]), x^T D x = 1; iters int32 [n] the Lanczos steps, converged int32
    [n] 0 where k_max steps did not reach the residual bound.  bits, degree: od_graph's, with the same eps."""
    n, P = degree.shape
    assert bits.dtype == torch.int32 and bits.is_contiguous() and bits.shape == (n, P, -(-P // 32))
    assert degree.dtype == f32 and degree.is_contiguous()
    assert x.dtype == f32 and x.is_contiguous() and x.shape == (n, P)
    for t, dt in ((lambda2, f32), (iters, torch.int32), (converged, torch.int32)):
        assert t.dtype == dt and t.is_contiguous() and t.shape == (n,)
    N.check(N.init().d3_od_fiedler(_p(bits), _p(degree), n, P, float(eps), int(k_max), _p(x), _p(lambda2),
                                   _p(iters), _p(converged), _s()), "d3_od_fiedler")
    return x, lambda2, iters, converged


def od_box(x: torch.Tensor, grid, patch: int, sizes, n_gt, gt: torch.Tensor, fg: torch.Tensor, box: torch.Tensor,
           best_iou: torch.Tensor, hit: torch.Tensor):
    """TokenCut's box per image (d3_od_box): fg uint8 [n, h * w] the bipartition after the sign flip, box int32 [n, 4]
    the pixel box (x0, y0, x1, y1) of the seed's 4-connected component, best_iou fp32 [n] against the image's
    ground-truth boxes and hit int32 [n] = best_iou >= 0.5.  x fp32 [n, h * w] (od_fiedler); sizes host ints [n, 2] =
    (H, W); n_gt host ints [n]; gt fp32 [n, b_max, 4] (x1 y1 x2 y2).  sizes and n_gt are checked before any launch."""
    h, w = int(grid[0]), int(grid[1])
    n = x.shape[0]
    hw_ = [[int(v) for v in r] for r in sizes]
    counts = [int(v) for v in n_gt]
    assert len(hw_) == n and all(len(r) == 2 for r in hw_) and len(counts) == n
    assert x.dtype == f32 and x.is_contiguous() and x.shape == (n, h * w)
    assert gt.dtype == f32 and gt.is_contiguous() and gt.dim() == 3 and gt.shape[0] == n and gt.shape[2] == 4
    assert fg.dtype == torch.uint8 and fg.is_contiguous() and fg.shape == (n, h * w)
    assert box.dtype == torch.int32 and box.is_contiguous() and box.shape == (n, 4)
    assert best_iou.dtype == f32 and best_iou.is_contiguous() and best_iou.shape == (n,)
    assert hit.dtype == torch.int32 and hit.is_contiguous() and hit.shape == (n,)
    sz = (C.c_int * max(2 * n, 1))(*[v for r in hw_ for v in r])
    cnt = (C.c_int * max(n, 1))(*counts)
    N.check(N.init().d3_od_box(_p(x), n, h, w, int(patch), sz, cnt, _p(gt), gt.shape[1], _p(fg), _p(box),
                               _p(best_iou), _p(hit), _s()), "d3_od_box")
    return box, best_iou, hit


# ------------------------------------------------------------------------------------------------ instance retrieval
def ret_resize(src: torch.Tensor, desc, out: torch.Tensor, *, mean, std) -> torch.Tensor:
    """torch's F.interpolate(bicubic, antialias=True, align_corners=False) of the crop box of each of n packed uint8
    HWC images to out bf16 [n, h, w, 3], on float values, then (v / 255 - mean) / std (d3_ret_resize).  src uint8
    (flat, on the device); desc host ints [n, 7] = (byte offset, H, W, x0, y0, x1, y1), the box [x0, x1) x [y0, y1);
    checked before any launch."""
    n, h, w = out.shape[0], out.shape[1], out.shape[2]
    rows = [[int(v) for v in r] for r in desc]
    assert src.dtype == torch.uint8 and src.is_contiguous()
    assert out.dtype == bf16 and out.is_contiguous() and out.shape == (n, h, w, 3)
    assert len(rows) == n and all(len(r) == 7 for r in rows)
    d = (C.c_longlong * max(7 * n, 1))(*[v for r in rows for v in r])
    m = (C.c_float * 3)(*[float(v) for v in mean])
    s = (C.c_float * 3)(*[float(v) for v in std])
    N.check(N.init().d3_ret_resize(_p(src), src.numel(), d, n, h, w, m, s, _p(out), _s()), "d3_ret_resize")
    return out


def ret_scale_sum(x: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out fp32 [n, D] = x[0] + x[1] + ... + x[S - 1], added in that order, of x fp32 [S, n, D] (d3_ret_scale_sum)."""
    S = x.shape[0]
    assert x.dtype == f32 and x.is_contiguous() and x.dim() == 3
    assert out.dtype == f32 and out.is_contiguous() and out.shape == x.shape[1:]
    N.check(N.init().d3_ret_scale_sum(_p(x), S, out.numel(), out.numel(), _p(out), _s()), "d3_ret_scale_sum")
    return out


def _csr(ptr, idx):
    """A host CSR pair as int32 arrays (kept alive by the caller while the C call reads them)."""
    p, i = (np.ascontiguousarray(np.asarray(v).reshape(-1), dtype=np.int32) for v in (ptr, idx))
    return p, i


def ret_rank_ap(sim: torch.Tensor, n_cols: int, easy, hard, junk, ranks: torch.Tensor, ap: torch.Tensor,
                pk: torch.Tensor, n_ok: torch.Tensor):
    """The revisited ranking of the first n_cols columns of sim fp32 [Q, >= n_cols] (d3_ret_rank_ap): ranks int32
    [n_easy + n_hard + n_junk] the exact 0-based rank of every list entry (easy, then hard, then junk entries), ap fp64
    [Q, 3] and pk fp64 [Q, 3, 3] (P@1, P@5, P@10) for the Easy, Medium and Hard protocols, n_ok int32 [Q, 3].  easy,
    hard, junk: host CSR pairs (ptr [Q + 1], idx), checked before any launch."""
    Q = sim.shape[0]
    assert sim.dtype == f32 and sim.dim() == 2 and sim.stride(1) == 1
    lists = [_csr(*l) for l in (easy, hard, junk)]
    assert all(l[0].size == Q + 1 for l in lists), "every list needs Q + 1 row pointers"
    total = sum(l[1].size for l in lists)
    assert ranks.dtype == torch.int32 and ranks.is_contiguous() and ranks.numel() == total
    assert ap.dtype == torch.float64 and ap.is_contiguous() and ap.shape == (Q, 3)
    assert pk.dtype == torch.float64 and pk.is_contiguous() and pk.shape == (Q, 3, 3)
    assert n_ok.dtype == torch.int32 and n_ok.is_contiguous() and n_ok.shape == (Q, 3)
    args = [a.ctypes.data_as(C.POINTER(C.c_int)) for l in lists for a in l]
    N.check(N.init().d3_ret_rank_ap(_p(sim), sim.stride(0), Q, int(n_cols), *args, _p(ranks), _p(ap), _p(pk),
                                    _p(n_ok), _s()), "d3_ret_rank_ap")
    return ranks, ap, pk, n_ok
