"""Thin Python wrappers over the C ABI (one function per exported kernel family).

Tensors are containers only: every function validates dtype / contiguity, passes raw device pointers and the
current CUDA stream, and raises NativeError on a non-zero status.  No function here computes anything in PyTorch.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _native as N

bf16 = torch.bfloat16
f32 = torch.float32

# optional per-launch timing hook (bench.py roofline leg): a list that receives (kind, flops, start_evt, end_evt)
PROFILE: list | None = None


def _ld(t: torch.Tensor) -> int:
    assert t.dim() == 2 and t.stride(1) == 1, "expect 2-D row-major (unit inner stride)"
    return t.stride(0)


def gemm(A: torch.Tensor, B: torch.Tensor, out: torch.Tensor, *, a_mn: bool = False, b_mn: bool = False,
         bias: torch.Tensor | None = None, gelu: bool = False, store_pre: torch.Tensor | None = None,
         dgelu_of: torch.Tensor | None = None, gamma: torch.Tensor | None = None,
         resid: torch.Tensor | None = None, accum: bool = False, alpha: float = 1.0, tile_n: int = 0,
         split_k: int = 0, scatter=None) -> torch.Tensor:
    """out[M,N] = epilogue(alpha * A.B) on the wgmma tensor cores (d3_gemm_bf16).

    A is [M,K] (a_mn=False) or stored transposed [K,M] (a_mn=True); B is [N,K] (b_mn=False) or [K,N] (b_mn=True).
    """
    l = N.init()
    assert A.dtype == bf16 and B.dtype == bf16
    M, K = (A.shape[1], A.shape[0]) if a_mn else (A.shape[0], A.shape[1])
    Nn, Kb = (B.shape[1], B.shape[0]) if b_mn else (B.shape[0], B.shape[1])
    assert K == Kb, f"contraction mismatch {K} vs {Kb}"
    assert out.shape[0] == M and out.shape[1] == Nn and out.dtype in (bf16, f32)
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
    if PROFILE is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    N.check(l.d3_gemm_bf16(N.ptr(A), _ld(A), int(a_mn), N.ptr(B), _ld(B), int(b_mn), M, Nn, K, C.byref(ep),
                           int(tile_n), int(split_k), N.stream_ptr()), "d3_gemm_bf16")
    if PROFILE is not None:
        e1.record()
        PROFILE.append(("gemm", 2.0 * M * Nn * K, e0, e1, (M, Nn, K, int(a_mn), int(b_mn))))
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


def koleo_fwd_bwd(x, xn, nrm, nn, coef, metric, dx, w_metric, w_grad, eps=1e-8):
    B, D = x.shape
    assert x.dtype == f32 and nn.dtype == torch.int32
    N.check(N.init().d3_koleo_fwd_bwd(_p(x), _p(xn), _p(nrm), _p(nn), _p(coef), _p(metric), _p(dx), B, D, eps,
                                      w_metric, w_grad, _s()), "d3_koleo_fwd_bwd")


def koleo_fwd_bwd_rows(x, xn, nrm, nn, coef, metric, dx, row0, nrows, w_metric, w_grad, eps=1e-8):
    """KoLeo with the loss terms restricted to rows [row0, row0+nrows) of the (all-gathered) matrix x."""
    B, D = x.shape
    assert x.dtype == f32 and nn.dtype == torch.int32
    N.check(N.init().d3_koleo_fwd_bwd_rows(_p(x), _p(xn), _p(nrm), _p(nn), _p(coef), _p(metric), _p(dx), B, D, int(row0),
                                           int(nrows), eps, w_metric, w_grad, _s()), "d3_koleo_fwd_bwd_rows")


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
