"""-m gpu: every CUDA kernel behind the C ABI against plain PyTorch fp32 on the same inputs (tolerances are the
bf16 storage rounding of the kernel's output; integer / indexing work is checked bit-exactly)."""
import math

import numpy as np
import pytest
import torch

from attention_helpers import attn_ref, bwd, fwd

pytestmark = pytest.mark.gpu

BF16_TOL = 6e-3      # norm-wise relative error of a bf16-stored result (2^-9 per element)


def rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-30)).item()


@pytest.fixture(autouse=True)
def _seed(native):
    torch.manual_seed(0)


# --------------------------------------------------------------------------------------------------- GEMM
@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (0, 1), (1, 0), (1, 1)])
@pytest.mark.parametrize("shape", [(128, 64, 64), (384, 320, 192), (296, 200, 136), (1000, 1152, 384), (4096, 1024, 1024)])
@pytest.mark.parametrize("bn", [0, 64, 128, 256, 512])
def test_gemm_matches_fp32_matmul(a_mn, b_mn, shape, bn):
    from dinov3_jax import ops
    M, N, K = shape
    A = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    B = torch.randn(K, N, device="cuda").to(torch.bfloat16)
    ref = A.float() @ B.float()
    out = torch.full((M, N), float("nan"), device="cuda")
    ops.gemm(A.t().contiguous() if a_mn else A, B if b_mn else B.t().contiguous(), out, a_mn=bool(a_mn), b_mn=bool(b_mn), tile_n=bn)
    assert rel(out, ref) < 1e-5      # fp32 accumulation of exact bf16 products


def test_gemm_epilogues():
    from dinov3_jax import ops
    M, N, K = 500, 384, 256
    A = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    B = (torch.randn(K, N, device="cuda") * 0.1).to(torch.bfloat16)
    bias, gamma, resid = torch.randn(N, device="cuda"), torch.randn(N, device="cuda"), torch.randn(M, N, device="cuda")
    acc = A.float() @ B.float()
    u = acc + bias
    out = torch.empty(M, N, device="cuda"); pre = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    ops.gemm(A, B, out, b_mn=True, bias=bias, gelu=True, store_pre=pre, gamma=gamma, resid=resid)
    assert rel(out, resid + gamma * torch.nn.functional.gelu(u, approximate="tanh")) < 5e-4   # hardware tanh (2^-11)
    assert rel(pre, u) < BF16_TOL
    ub = torch.randn(M, N, device="cuda").to(torch.bfloat16)
    uf = ub.float().requires_grad_(True)
    torch.nn.functional.gelu(uf, approximate="tanh").sum().backward()
    out2 = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    ops.gemm(A, B, out2, b_mn=True, dgelu_of=ub)
    assert rel(out2, acc * uf.grad) < BF16_TOL
    out3 = torch.ones(M, N, device="cuda")
    ops.gemm(A, B, out3, b_mn=True, accum=True, alpha=0.5)
    assert rel(out3, 1 + 0.5 * acc) < 1e-5


@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (0, 1), (1, 1)])
@pytest.mark.parametrize("shape", [(1000, 512, 256), (776, 1024, 320)])
def test_gemm_pair_kernel_tma_epilogue(a_mn, b_mn, shape):
    """Every epilogue combination the engine uses, in each operand layout (fixed-flag kernels in the engine's layouts,
    run-time flags in the others), at a ragged M, against PyTorch fp32."""
    from dinov3_jax import ops
    M, N, K = shape
    A = torch.randn(M, K, device="cuda").to(torch.bfloat16); B = (torch.randn(K, N, device="cuda") * 0.1).to(torch.bfloat16)
    A_st = A.t().contiguous() if a_mn else A
    B_st = B if b_mn else B.t().contiguous()
    kw = dict(a_mn=bool(a_mn), b_mn=bool(b_mn), tile_n=128)
    bias, gamma, resid = torch.randn(N, device="cuda"), torch.randn(N, device="cuda"), torch.randn(M, N, device="cuda")
    acc = A.float() @ B.float(); u = acc + bias
    gel = torch.nn.functional.gelu(u, approximate="tanh")
    nanb = lambda: torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)
    nanf = lambda: torch.full((M, N), float("nan"), device="cuda")
    o = nanb(); ops.gemm(A_st, B_st, o, bias=bias, **kw); assert rel(o, u) < BF16_TOL
    o, pre = nanb(), nanb(); ops.gemm(A_st, B_st, o, bias=bias, gelu=True, store_pre=pre, **kw)
    assert rel(o, gel) < BF16_TOL and rel(pre, u) < BF16_TOL
    o, pre = nanf(), nanb(); ops.gemm(A_st, B_st, o, bias=bias, store_pre=pre, gamma=gamma, resid=resid, **kw)
    assert rel(o, resid + gamma * u) < 1e-5 and rel(pre, u) < BF16_TOL
    o = nanf(); ops.gemm(A_st, B_st, o, bias=bias, gelu=True, store_pre=pre, gamma=gamma, resid=resid, **kw)
    assert rel(o, resid + gamma * gel) < 5e-4
    ub = torch.randn(M, N, device="cuda").to(torch.bfloat16); uf = ub.float().requires_grad_(True)
    torch.nn.functional.gelu(uf, approximate="tanh").sum().backward()
    o = nanb(); ops.gemm(A_st, B_st, o, dgelu_of=ub, **kw); assert rel(o, acc * uf.grad) < BF16_TOL
    o = nanf(); ops.gemm(A_st, B_st, o, **kw); assert rel(o, acc) < 1e-5


@pytest.mark.parametrize("M,N,K,bn,sk", [(256, 256, 4096, 512, 8), (1024, 1024, 8192, 512, 4), (384, 320, 2048, 128, 5), (1024, 1024, 12032, 0, 0)])
def test_gemm_split_k_accumulates(M, N, K, bn, sk):
    from dinov3_jax import ops
    A = torch.randn(K, M, device="cuda").to(torch.bfloat16); B = torch.randn(K, N, device="cuda").to(torch.bfloat16)
    out = torch.ones(M, N, device="cuda")
    ops.gemm(A, B, out, a_mn=True, b_mn=True, accum=True, tile_n=bn, split_k=sk)
    assert rel(out, 1 + A.float().t() @ B.float()) < 1e-5
    again = torch.ones(M, N, device="cuda")
    ops.gemm(A, B, again, a_mn=True, b_mn=True, accum=True, tile_n=bn, split_k=sk)
    assert torch.equal(out, again)                   # the slices are reduced in a fixed order


def test_gemm_rejects_bad_arguments():
    from dinov3_jax import ops, _native
    A = torch.randn(64, 60, device="cuda").to(torch.bfloat16)     # ld = 60 is not a multiple of 8
    B = torch.randn(64, 60, device="cuda").to(torch.bfloat16)
    with pytest.raises(_native.NativeError):
        ops.gemm(A, B, torch.empty(64, 64, device="cuda"))


# --------------------------------------------------------------------------------------------------- attention
@pytest.mark.parametrize("n,N,H", [(3, 197, 2), (5, 37, 2), (2, 128, 1), (2, 257, 1), (4, 50, 3), (1, 1, 1), (2, 17, 6),
                                   (2, 256, 1), (3, 200, 1), (7, 64, 1), (4, 65, 2), (3, 129, 1),
                                   (40, 197, 16), (130, 37, 16), (9, 201, 8)])
def test_attention_forward(n, N, H):
    qkv = torch.randn(n * N, 3 * 64 * H, device="cuda").to(torch.bfloat16)
    o, lse = fwd(qkv, n, N, H)
    ro, rl = attn_ref(qkv, n, N, H)
    assert rel(o, ro) < BF16_TOL and rel(lse, rl) < 1e-5


@pytest.mark.parametrize("n,N,H", [(2, 128, 1), (3, 197, 2), (5, 37, 2), (4, 50, 3), (2, 256, 1), (2, 17, 6), (2, 257, 2), (1, 384, 1), (3, 300, 1)])
def test_attention_backward(n, N, H):
    D = 64 * H
    qkv = torch.randn(n * N, 3 * D, device="cuda").to(torch.bfloat16)
    do = torch.randn(n * N, D, device="cuda").to(torch.bfloat16)
    x = qkv.float().requires_grad_(True)
    attn_ref(x, n, N, H)[0].backward(do.float())
    o, lse = fwd(qkv, n, N, H)
    dqkv = bwd(qkv, o, do, lse, n, N, H)
    for j in range(3):
        assert rel(dqkv[:, j * D:(j + 1) * D], x.grad[:, j * D:(j + 1) * D]) < 1e-2


def test_attention_backward_fused_inverse_rope():
    """dqkv with rope tables == separate inverse-RoPE of the plain backward (tokens < prefix untouched, v untouched)."""
    from dinov3_jax import ops
    from oracle.model import rope_sincos
    n, Hp, H = 3, 6, 2
    N, D = Hp * Hp + 1, 64 * H
    sin, cos = [t.cuda().contiguous() for t in rope_sincos(Hp, Hp, 64, 100.0, torch.float32)]
    qkv = torch.randn(n * N, 3 * D, device="cuda").to(torch.bfloat16)
    do = torch.randn(n * N, D, device="cuda").to(torch.bfloat16)
    o, lse = fwd(qkv, n, N, H)
    d1 = bwd(qkv, o, do, lse, n, N, H)
    ops.rope(d1, sin, cos, N, 1, D, 64, inverse=True)
    d2 = bwd(qkv, o, do, lse, n, N, H, rope_sin=sin, rope_cos=cos, rope_prefix=1)
    assert rel(d2, d1) < BF16_TOL          # d1 is rounded to bf16 twice, d2 once
    assert torch.equal(d2[:, 2 * D:], d1[:, 2 * D:])


# --------------------------------------------------------------------------------------------------- integer / layout work
def test_im2col_and_tokens_bit_exact():
    from dinov3_jax import ops
    n, Hh, p, D = 3, 64, 16, 128
    img = torch.randn(n, Hh, Hh, 3, device="cuda").to(torch.bfloat16)
    P = (Hh // p) ** 2
    out = torch.empty(n * P, p * p * 3, device="cuda", dtype=torch.bfloat16)
    ops.im2col(img, out, p)
    ref = img.reshape(n, Hh // p, p, Hh // p, p, 3).permute(0, 1, 3, 2, 4, 5).reshape(out.shape)
    assert torch.equal(out, ref)
    tok, cls, mt = torch.randn(n * P, D, device="cuda"), torch.randn(D, device="cuda"), torch.randn(D, device="cuda")
    masks = torch.rand(n, P, device="cuda") < 0.3
    X = torch.empty(n, P + 1, D, device="cuda")
    ops.assemble_tokens(tok, cls, mt, masks.to(torch.uint8), X, n, P, D)
    assert torch.equal(X, torch.cat([cls.expand(n, 1, D), torch.where(masks[..., None], mt, tok.reshape(n, P, D))], 1))
    X2 = torch.empty(n, P + 1, D, device="cuda")
    ops.assemble_tokens(tok, cls, mt, None, X2, n, P, D)
    assert torch.equal(X2[:, 1:], tok.reshape(n, P, D))
    dX = torch.randn(n, P + 1, D, device="cuda"); dTok = torch.empty(n * P, D, device="cuda", dtype=torch.bfloat16)
    dcls, dm = torch.zeros(D, device="cuda"), torch.zeros(D, device="cuda")
    ops.assemble_tokens_bwd(dX, masks.to(torch.uint8), dTok, dcls, dm, n, P, D)
    assert torch.equal(dTok, torch.where(masks[..., None], torch.zeros_like(dX[:, 1:]), dX[:, 1:]).reshape(n * P, D).to(torch.bfloat16))
    assert rel(dcls, dX[:, 0].sum(0)) < 1e-5 and rel(dm, (dX[:, 1:] * masks[..., None]).sum((0, 1))) < 1e-5


def test_token_rows_gather_scatter_bit_exact():
    from dinov3_jax import ops
    P, n, D = 16, 4, 128
    src = torch.randn(n * (P + 1), D, device="cuda")
    midx = torch.tensor([0, 3, 17, 18, 40, 63], device="cuda", dtype=torch.int64)
    rows = torch.empty(6, dtype=torch.int32, device="cuda")
    ops.token_rows(midx, rows, 6, P, 0)
    want = (midx // P * (P + 1) + 1 + midx % P)
    assert torch.equal(rows.long(), want)
    crow = torch.empty(n, dtype=torch.int32, device="cuda")
    ops.token_rows(None, crow, n, P, 1)
    assert torch.equal(crow.long(), torch.arange(n, device="cuda") * (P + 1))
    gb, gf = torch.empty(6, D, device="cuda", dtype=torch.bfloat16), torch.empty(6, D, device="cuda")
    ops.gather_rows(src, rows, 6, D, gb, gf)
    assert torch.equal(gf, src[want]) and torch.equal(gb, src[want].to(torch.bfloat16))
    dst = torch.zeros_like(src)
    ops.scatter_add_rows(gf, rows, dst, 6, D)
    ref = torch.zeros_like(src); ref[want] += gf
    assert torch.equal(dst, ref)
    ops.gather_rows(src, rows, 0, D, gb, gf)      # empty gather is a no-op


@pytest.mark.parametrize("n", [100003 * 4, 100003 * 4 + 3])
def test_cast_f32_bf16_bit_exact(n):
    """d3_cast_f32_bf16 (the bf16 compute copy of the weights) rounds as torch does, in the 4-wide body and the tail."""
    from dinov3_jax import ops
    src = torch.randn(n, device="cuda")
    dst = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    ops.cast_f32_bf16(src, dst)
    assert torch.equal(dst, src.to(torch.bfloat16))


# --------------------------------------------------------------------------------------------------- normalisation / rope
@pytest.mark.parametrize("T,D", [(1000, 384), (333, 1024), (7, 128), (2051, 768), (100, 256), (300, 1536), (64, 192)])
def test_layernorm_forward_and_plain_backward(T, D):
    """d3_layernorm_fwd and d3_layernorm_bwd_ls without a LayerScale tail (the plain LayerNorm backward), fp32 dy."""
    from dinov3_jax import ops
    from oracle.model import layer_norm
    x = torch.randn(T, D, device="cuda") * 2 + 0.5
    sc, bi = torch.randn(D, device="cuda"), torch.randn(D, device="cuda")
    y, yf = torch.empty(T, D, device="cuda", dtype=torch.bfloat16), torch.empty(T, D, device="cuda")
    mean, rstd = torch.empty(T, device="cuda"), torch.empty(T, device="cuda")
    ops.layernorm_fwd(x, sc, bi, y, mean, rstd); ops.layernorm_fwd(x, sc, bi, yf)
    xr, scr, bir = x.clone().requires_grad_(True), sc.clone().requires_grad_(True), bi.clone().requires_grad_(True)
    ref = layer_norm(xr, scr, bir, 1e-6)
    assert rel(y, ref) < BF16_TOL and rel(yf, ref) < 1e-5
    dy, add = torch.randn(T, D, device="cuda"), torch.randn(T, D, device="cuda")
    ref.backward(dy)
    dx, ds, db = torch.empty(T, D, device="cuda"), torch.zeros(D, device="cuda"), torch.zeros(D, device="cuda")
    ops.layernorm_bwd_ls(dy, x, mean, rstd, sc, dx, dx_add=add, dscale=ds, dbias=db)
    assert rel(dx, xr.grad + add) < 1e-4 and rel(ds, scr.grad) < 1e-4 and rel(db, bir.grad) < 1e-4


@pytest.mark.parametrize("T,D", [(1000, 384), (333, 1024), (7, 128), (2051, 768), (301, 1536), (64, 192), (1, 1024)])
@pytest.mark.parametrize("mode", ["plain", "linear_tail", "gelu_tail", "identity_tail_with_stash"])
def test_layernorm_backward_with_layerscale_tail(T, D, mode):
    """d3_layernorm_bwd_ls: LN backward + (optionally) du = dx*gamma*act'(u), dgamma, dbias of the upstream branch."""
    from dinov3_jax import ops
    from oracle.model import layer_norm
    x = torch.randn(T, D, device="cuda") * 2 + 0.5
    sc, bi = torch.randn(D, device="cuda"), torch.randn(D, device="cuda")
    y = torch.empty(T, D, device="cuda", dtype=torch.bfloat16)
    mean, rstd = torch.empty(T, device="cuda"), torch.empty(T, device="cuda")
    ops.layernorm_fwd(x, sc, bi, y, mean, rstd)
    xr, scr, bir = x.clone().requires_grad_(True), sc.clone().requires_grad_(True), bi.clone().requires_grad_(True)
    dy = torch.randn(T, D, device="cuda").to(torch.bfloat16)
    add = torch.randn(T, D, device="cuda")
    layer_norm(xr, scr, bir, 1e-6).backward(dy.float())
    dx_ref = xr.grad + add
    dx, ds, db = torch.empty(T, D, device="cuda"), torch.zeros(D, device="cuda"), torch.zeros(D, device="cuda")
    gam = torch.randn(D, device="cuda")
    ub = torch.randn(T, D, device="cuda").to(torch.bfloat16)
    du = torch.empty(T, D, device="cuda", dtype=torch.bfloat16)
    dg, dbl = torch.zeros(D, device="cuda"), torch.zeros(D, device="cuda")
    kw = {}
    if mode == "linear_tail":
        kw = dict(ls_gamma=gam, ls_du=du, ls_dbias=dbl)
    elif mode == "gelu_tail":
        kw = dict(ls_gamma=gam, ls_u=ub, ls_gelu=True, ls_du=du, ls_dgamma=dg, ls_dbias=dbl)
    elif mode == "identity_tail_with_stash":
        kw = dict(ls_gamma=gam, ls_u=ub, ls_gelu=False, ls_du=du, ls_dgamma=dg, ls_dbias=dbl)
    ops.layernorm_bwd_ls(dy, x, mean, rstd, sc, dx, dx_add=add, dscale=ds, dbias=db, **kw)
    assert rel(dx, dx_ref) < 1e-4 and rel(ds, scr.grad) < 1e-4 and rel(db, bir.grad) < 1e-4
    if mode == "plain":
        return
    uu = ub.float()
    if mode == "gelu_tail":
        ur = uu.clone().requires_grad_(True)
        act = torch.nn.functional.gelu(ur, approximate="tanh")
        act.sum().backward()
        dact, act = ur.grad, act.detach()
    else:
        dact, act = torch.ones_like(uu), uu
    du_ref = dx_ref * gam * dact
    assert rel(du, du_ref) < BF16_TOL
    assert rel(dbl, du.float().sum(0)) < 1e-4          # bias gradient = column sum of the rounded du the wgrad GEMM sees
    if mode != "linear_tail":
        assert rel(dg, (dx_ref * act).sum(0)) < 1e-4


@pytest.mark.parametrize("D", [1024, 1152, 1536])
@pytest.mark.parametrize("gelu", [True, False])
def test_fused_layerscale_tail_matches_ls_act_bwd(D, gelu):
    """The tail fused into d3_layernorm_bwd_ls (the ring kernel at D = 1024, ln_bwd_ls_kernel at 1152 and 1536) and
    d3_ls_act_bwd on the dx it produced give the same du bits and the same parameter gradients."""
    from dinov3_jax import ops
    T = 999
    x = torch.randn(T, D, device="cuda") * 2 + 0.5
    sc, bi = torch.randn(D, device="cuda"), torch.randn(D, device="cuda")
    y = torch.empty(T, D, device="cuda", dtype=torch.bfloat16)
    mean, rstd = torch.empty(T, device="cuda"), torch.empty(T, device="cuda")
    ops.layernorm_fwd(x, sc, bi, y, mean, rstd)
    dy = torch.randn(T, D, device="cuda").to(torch.bfloat16)
    add = torch.randn(T, D, device="cuda")
    gam = torch.randn(D, device="cuda")
    ub = torch.randn(T, D, device="cuda").to(torch.bfloat16)
    dx, ds, db = torch.empty(T, D, device="cuda"), torch.zeros(D, device="cuda"), torch.zeros(D, device="cuda")
    du, dg, dbl = torch.empty(T, D, device="cuda", dtype=torch.bfloat16), torch.zeros(D, device="cuda"), torch.zeros(D, device="cuda")
    ops.layernorm_bwd_ls(dy, x, mean, rstd, sc, dx, dx_add=add, dscale=ds, dbias=db, ls_gamma=gam, ls_u=ub, ls_gelu=gelu,
                         ls_du=du, ls_dgamma=dg, ls_dbias=dbl)
    du2, dg2, dbl2 = torch.empty_like(du), torch.zeros(D, device="cuda"), torch.zeros(D, device="cuda")
    ops.ls_act_bwd(dx, ub, gam, du2, dg2, dbl2, gelu)
    assert torch.equal(du, du2)
    assert rel(dbl2, dbl) < 1e-5 and rel(dg2, dg) < 1e-5
    assert rel(dbl2, du.float().sum(0)) < 1e-5


@pytest.mark.parametrize("N", [1152, 1001, 3072])
@pytest.mark.parametrize("T", [37, 1001])
def test_colsum_bf16_does_not_depend_on_layout(T, N):
    """d3_colsum_bf16 of an aligned buffer (16-byte loads) and of a copy stored 2 elements past a 16-byte boundary
    (scalar loads) walk the same rows and columns in the same order: bit-identical sums."""
    from dinov3_jax import ops
    xb = torch.randn(T, N, device="cuda").to(torch.bfloat16)
    a = torch.zeros(N, device="cuda")
    ops.colsum_bf16(xb, a)
    buf = torch.empty(T * N + 8, device="cuda", dtype=torch.bfloat16)
    shifted = buf[2:2 + T * N].view(T, N)
    shifted.copy_(xb)
    b = torch.zeros(N, device="cuda")
    ops.colsum_bf16(shifted, b)
    assert torch.equal(a, b)
    assert rel(a, xb.float().sum(0)) < 1e-5


def test_layerscale_gamma_from_weight_gradient():
    """dgamma of x + gamma*(a W + b) recovered from dW, db (d3_ls_gamma_from_wgrad) equals the direct column sum."""
    from dinov3_jax import ops
    T, K, N = 900, 320, 200
    a = torch.randn(T, K, device="cuda").to(torch.bfloat16)
    W = (torch.randn(K, N, device="cuda") / K ** 0.5).to(torch.bfloat16)
    b, gam = torch.randn(N, device="cuda") * 0.1, torch.randn(N, device="cuda") * 1e-3
    dx = torch.randn(T, N, device="cuda")
    du = dx * gam
    dW = a.float().t() @ du
    dbias = du.sum(0)
    want = (dx * (a.float() @ W.float() + b)).sum(0)
    got = torch.zeros(N, device="cuda")
    ops.ls_gamma_from_wgrad(W, dW.contiguous(), b, dbias, gam, got)
    assert rel(got, want) < 1e-4


def test_rope_forward_and_adjoint():
    from dinov3_jax import ops
    from oracle.model import rope_apply, rope_sincos
    n, Hp, H = 3, 6, 2
    N, D = Hp * Hp + 1, 64 * H
    sin, cos = [t.cuda().contiguous() for t in rope_sincos(Hp, Hp, 64, 100.0, torch.float32)]
    qkv = torch.randn(n * N, 3 * D, device="cuda").to(torch.bfloat16)
    ref = qkv.float().reshape(n, N, 3, H, 64).clone()
    for w in (0, 1):
        ref[:, 1:, w] = rope_apply(ref[:, 1:, w].transpose(1, 2), sin, cos).transpose(1, 2)
    q2 = qkv.clone()
    ops.rope(q2, sin, cos, N, 1, D, 64)
    assert rel(q2, ref.reshape(n * N, 3 * D)) < BF16_TOL
    assert torch.equal(q2.reshape(n, N, 3 * D)[:, 0], qkv.reshape(n, N, 3 * D)[:, 0])       # cls token untouched
    assert torch.equal(q2[:, 2 * D:], qkv[:, 2 * D:])                                     # v untouched
    g = torch.randn(n * N, 3 * D, device="cuda").to(torch.bfloat16); gi = g.clone()
    ops.rope(gi, sin, cos, N, 1, D, 64, inverse=True)
    lhs, rhs = (ref.reshape(n * N, 3 * D) * g.float()).sum().item(), (qkv.float() * gi.float()).sum().item()
    assert abs(lhs - rhs) < 2e-2 * abs(lhs) + 0.5


def test_l2norm_and_layerscale_backward_rounded_bias():
    """d3_l2norm_fwd / _bwd, and d3_ls_act_bwd, whose bias gradient is the column sum of the bf16 du it stores (the
    values the weight-gradient GEMM sees), as in the LayerScale tail of d3_layernorm_bwd_ls."""
    from dinov3_jax import ops
    R, C = 300, 256
    u = torch.randn(R, C, device="cuda"); y = torch.empty(R, C, device="cuda", dtype=torch.bfloat16); nr = torch.empty(R, device="cuda")
    ops.l2norm_fwd(u, y, nr)
    ur = u.clone().requires_grad_(True); yr = ur / (ur.norm(dim=-1, keepdim=True) + 1e-12)
    assert rel(y, yr) < BF16_TOL
    g = torch.randn(R, C, device="cuda").to(torch.bfloat16); yr.backward(g.float())
    du = torch.empty(R, C, device="cuda", dtype=torch.bfloat16); ops.l2norm_bwd(g, u, nr, du)
    assert rel(du, ur.grad) < BF16_TOL
    T, D = 777, 384
    dX = torch.randn(T, D, device="cuda"); ub = torch.randn(T, D, device="cuda").to(torch.bfloat16); gam = torch.randn(D, device="cuda")
    for use_gelu in (True, False):
        uu, gg = ub.float().requires_grad_(True), gam.clone().requires_grad_(True)
        act = torch.nn.functional.gelu(uu, approximate="tanh") if use_gelu else uu
        (gg * act * dX).sum().backward()
        du = torch.empty(T, D, device="cuda", dtype=torch.bfloat16); dg, db = torch.zeros(D, device="cuda"), torch.zeros(D, device="cuda")
        ops.ls_act_bwd(dX, ub, gam, du, dg, db, use_gelu)
        assert rel(du, uu.grad) < BF16_TOL and rel(dg, gg.grad) < 1e-4
        assert rel(db, du.float().sum(0)) < 1e-5     # the column sum of the rounded du the weight-gradient GEMM sees
    xb = torch.randn(1001, 1152, device="cuda").to(torch.bfloat16); cs = torch.zeros(1152, device="cuda")
    ops.colsum_bf16(xb, cs)
    assert rel(cs, xb.float().sum(0)) < 1e-5


# --------------------------------------------------------------------------------------------------- losses
def test_sinkhorn_ce_koleo_match_oracle():
    _sinkhorn_ce_koleo_vs_oracle(4096)


def test_sinkhorn_ce_koleo_match_oracle_with_k_not_a_multiple_of_4():
    """K % 4 != 0: the scalar Sinkhorn column-sum, row-sum, colmax and cross-entropy paths."""
    _sinkhorn_ce_koleo_vs_oracle(1001)


def _sinkhorn_ce_koleo_vs_oracle(K):
    from dinov3_jax import ops
    from oracle.losses import dino_loss, ibot_loss_masked, koleo_loss, sinkhorn_knopp
    R, temp = 24, 0.05
    L = torch.randn(R, K, device="cuda") * 0.3
    gmx = torch.full((1,), float("-inf"), device="cuda"); ops.absmax(L, gmx)
    assert gmx.item() == L.max().item()
    mx = torch.full((K,), float("-inf"), device="cuda"); ops.colmax(L, mx)
    assert torch.equal(mx, L.max(0).values)
    btot = torch.tensor([float(R)], device="cuda")
    a, s, av = None, torch.zeros(K, device="cuda"), torch.empty(R, device="cuda")
    for _ in range(3):
        s.zero_(); ops.sinkhorn_colsum(L, mx, temp, a, s); ops.sinkhorn_rowsum(L, mx, temp, s, btot, av); a = av
    Q = torch.empty(R, K, device="cuda"); ops.sinkhorn_probs(L, mx, temp, s, a, btot, Q)
    Qr = sinkhorn_knopp(L.double(), temp, R)
    assert rel(Q, Qr) < 1e-4
    B = R // 2
    S = torch.randn(10 * B, K, device="cuda") * 0.5
    Sr = S.double().requires_grad_(True)
    Ll = dino_loss(Sr[2 * B:].reshape(8, B, K), Qr.reshape(2, B, K), 0.1, False)
    Lg = dino_loss(Sr[:2 * B].reshape(2, B, K), Qr.reshape(2, B, K), 0.1, True)
    (16 / 18 * Ll + 2 / 18 * Lg).backward()
    t0 = torch.empty(10 * B, dtype=torch.int32); t1 = torch.full((10 * B,), -1, dtype=torch.int32)
    wm, wg, slot = torch.empty(10 * B), torch.empty(10 * B), torch.empty(10 * B, dtype=torch.int32)
    for i in range(10 * B):
        sidx, b = divmod(i, B)
        if sidx < 2:
            t0[i] = (1 - sidx) * B + b; wm[i] = 1 / (2 * B); wg[i] = 2 / 18 / (2 * B); slot[i] = 1
        else:
            t0[i] = b; t1[i] = B + b; wm[i] = 1 / (16 * B); wg[i] = 16 / 18 / (16 * B); slot[i] = 0
    metric = torch.zeros(4, device="cuda"); dS = torch.empty(10 * B, K, device="cuda", dtype=torch.bfloat16)
    ops.ce_fwd_bwd(S, 0.1, L, mx, temp, s, a, btot, t0.cuda(), t1.cuda(), wm.cuda(), wg.cuda(), slot.cuda(), metric, dS)
    assert abs(metric[0].item() - Ll.item()) < 1e-4 * abs(Ll.item()) and abs(metric[1].item() - Lg.item()) < 1e-4 * abs(Lg.item())
    assert rel(dS, Sr.grad) < BF16_TOL
    Bk, D = 64, 384
    x = torch.randn(Bk, D, device="cuda")
    xr = x.double().requires_grad_(True); lk = koleo_loss(xr); (0.1 * lk).backward()
    xn, nr = torch.empty(Bk, D, device="cuda"), torch.empty(Bk, device="cuda")
    nn, cf = torch.empty(Bk, dtype=torch.int32, device="cuda"), torch.empty(Bk, device="cuda")
    met, dx = torch.zeros(1, device="cuda"), torch.zeros(Bk, D, device="cuda")
    ops.koleo_fwd_bwd(x, xn, nr, nn, cf, met, dx, 1.0, 0.1)
    assert abs(met.item() - lk.item()) < 1e-5 and rel(dx, xr.grad) < 1e-4


def _off16(t):
    """A copy of t stored one float (4 bytes) past a 16-byte boundary."""
    e = 4 // t.element_size()
    buf = torch.empty(t.numel() + e, dtype=t.dtype, device=t.device)
    assert buf.data_ptr() % 16 == 0
    out = buf[e:].view(t.shape)
    out.copy_(t)
    return out


def test_sinkhorn_ce_misaligned_rows_match_aligned():
    """Buffers one float past a 16-byte boundary take the scalar-load instances of absmax, colmax, the Sinkhorn sums
    and the cross-entropy.  At K = 4096 they walk the same four-column groups as the 128-bit instances with the same
    arithmetic, so they must agree with the aligned run."""
    from dinov3_jax import ops
    R, K, temp = 24, 4096, 0.05
    L0 = torch.randn(R, K, device="cuda") * 0.3
    S0 = torch.randn(R, K, device="cuda") * 0.5
    t0 = torch.arange(R, dtype=torch.int32, device="cuda")
    t1 = torch.where(t0 % 3 == 0, -1, (t0 + 5) % R).to(torch.int32)      # one or two teacher rows per student row
    wm, wg = torch.rand(R, device="cuda"), torch.rand(R, device="cuda")
    slot = (t0 % 2).to(torch.int32)
    btot = torch.tensor([float(R)], device="cuda")

    def run(place):
        L, S = place(L0), place(S0)
        gmx = place(torch.full((1,), float("-inf"), device="cuda")); ops.absmax(L, gmx)
        mx = place(torch.full((K,), float("-inf"), device="cuda")); ops.colmax(L, mx)
        s, a, av = place(torch.zeros(K, device="cuda")), None, place(torch.empty(R, device="cuda"))
        for _ in range(3):
            s.zero_(); ops.sinkhorn_colsum(L, mx, temp, a, s); ops.sinkhorn_rowsum(L, mx, temp, s, btot, av); a = av
        Q = place(torch.empty(R, K, device="cuda")); ops.sinkhorn_probs(L, mx, temp, s, a, btot, Q)
        metric = torch.zeros(2, device="cuda"); dS = place(torch.empty(R, K, device="cuda", dtype=torch.bfloat16))
        ops.ce_fwd_bwd(S, 0.1, L, mx, temp, s, a, btot, t0, t1, wm, wg, slot, metric, dS)
        # teacher rows that are already probabilities (s_t == NULL)
        metric_p = torch.zeros(2, device="cuda"); dS_p = place(torch.empty(R, K, device="cuda", dtype=torch.bfloat16))
        ops.ce_fwd_bwd(S, 0.1, Q, None, 1.0, None, None, None, t0, t1, wm, wg, slot, metric_p, dS_p)
        return dict(absmax=gmx, colmax=mx, s=s, a=a, Q=Q, metric=metric, dS=dS, metric_p=metric_p, dS_p=dS_p)

    ref = run(lambda t: t.clone())
    mis = run(_off16)
    assert ref["dS"].data_ptr() % 16 == 0 and mis["dS"].data_ptr() % 16 == 4
    differ = {k: rel(mis[k], ref[k]) for k in ref if not torch.equal(ref[k], mis[k])}
    assert not differ, differ


def test_adamw_ema_clip_matches_optax_formula():
    from dinov3_jax import ops
    n = 4096 * 3 + 64
    p, g = torch.randn(n, device="cuda"), torch.randn(n, device="cuda") * 0.01
    m, v, t = torch.randn(n, device="cuda") * 1e-3, torch.rand(n, device="cuda") * 1e-4, torch.randn(n, device="cuda")
    ss = torch.zeros(1, device="cuda"); ops.sumsq(g, ss)
    assert rel(ss, (g.double() ** 2).sum().reshape(1)) < 1e-5
    segs_np = np.zeros(3, dtype=[("start", "<i8"), ("lr", "<f4"), ("wd", "<f4"), ("last", "<i4"), ("pad", "<i4")])
    segs_np["start"] = [0, 4096, 8256]; segs_np["lr"] = [1.0, 0.5, 0.2]; segs_np["wd"] = [1.0, 0.0, 1.0]; segs_np["last"] = [0, 0, 1]
    segs = torch.from_numpy(segs_np.view(np.uint8)).cuda()
    lr, llr, wd, mom, step, maxn = 1e-3, 5e-4, 0.04, 0.99, 3, 0.5
    P0, M0, V0, T0 = p.double(), m.double(), v.double(), t.double()
    G = g.double() * min(1.0, maxn / (math.sqrt(ss.item()) + 1e-6))
    idx = torch.arange(n, device="cuda")
    lrm = torch.where(idx < 4096, 1.0, torch.where(idx < 8256, 0.5, 0.2)).double()
    wdm = torch.where(idx < 4096, 1.0, torch.where(idx < 8256, 0.0, 1.0)).double()
    base = torch.where(idx < 8256, lr, llr).double()
    M1 = 0.9 * M0 + 0.1 * G; V1 = 0.999 * V0 + 0.001 * G * G
    upd = (M1 / (1 - 0.9 ** step)) / ((V1 / (1 - 0.999 ** step)).sqrt() + 1e-8) + wd * wdm * P0
    P1 = P0 - base * lrm * upd; T1 = T0 * mom + P1 * (1 - mom)
    pb, tb = torch.zeros(8192, device="cuda", dtype=torch.bfloat16), torch.zeros(8192, device="cuda", dtype=torch.bfloat16)
    ops.adamw_ema(p, g, m, v, t, pb, tb, 8192, segs, 3, ss, maxn, lr, llr, wd, step, mom)
    assert rel(p, P1) < 1e-6 and rel(m, M1) < 1e-6 and rel(v, V1) < 1e-6 and rel(t, T1) < 1e-6
    assert torch.equal(pb, p[:8192].to(torch.bfloat16)) and torch.equal(tb, t[:8192].to(torch.bfloat16))


def _gram_ref(Ss, St, mode, block):
    """float64 sum of (s' - t')^2 over the counted elements (d3_gram_diff's modes and block-diagonal form)."""
    s, t = Ss.double(), St.double()
    if mode == 1:
        s = s.clamp(min=0)
    elif mode == 2:
        s = torch.where((s < 0) & (t < 0), torch.zeros_like(s), s)
    if mode:
        t = t.clamp(min=0)
    d2 = (s - t) ** 2
    if block:
        i = torch.arange(s.shape[0], device=s.device) // block
        d2 = d2 * (i[:, None] == i[None, :])
    return d2.sum()


@pytest.mark.parametrize("case", ["sinkhorn_colsum", "sinkhorn_colsum_k1001", "colsum_f32", "gram_diff", "gram_diff_blocks"])
def test_sums_are_bit_reproducible(case):
    """Column sums and the Gram loss add their slab partials in a fixed order: two calls on the same input give the same
    bits; the result matches a float64 sum."""
    from dinov3_jax import ops
    if case.startswith("sinkhorn"):
        R, K, temp = 3771, (65536 if case == "sinkhorn_colsum" else 1001), 0.05
        L = torch.randn(R, K, device="cuda") * 0.3
        mx = L.max(0).values
        a = torch.rand(R, device="cuda") + 0.5

        def run():
            s = torch.zeros(K, device="cuda")
            ops.sinkhorn_colsum(L, mx, temp, a, s)
            return s
        ref = (torch.exp((L.double() - mx.double()) / temp) * a.double()[:, None]).sum(0)
    elif case == "colsum_f32":
        L = torch.randn(3771, 65536, device="cuda")

        def run():
            out = torch.zeros(L.shape[1], device="cuda")
            ops.colsum_f32(L, out)
            return out
        ref = L.double().sum(0)
    else:
        n, block, mode = (1024, 0, 1) if case == "gram_diff" else (980, 196, 2)
        Ss, St = torch.rand(n, n, device="cuda") * 2 - 1, torch.rand(n, n, device="cuda") * 2 - 1
        inv = 1.0 / (n * n)

        def run():
            loss = torch.full((1,), 0.5, device="cuda")          # the loss is accumulated into
            ops.gram_diff(Ss, St, None, mode, inv, loss, block=block)
            return loss
        ref = (0.5 + inv * _gram_ref(Ss, St, mode, block)).reshape(1)
    first, second = run(), run()
    assert torch.equal(first, second)
    assert rel(first, ref) < 1e-5


# --------------------------------------------------------------------------------------------------- fused reduce-scatter
@pytest.mark.parametrize("M,N,K,world", [(512, 768, 4096, 2), (1024, 1024, 8192, 4), (296, 264, 2048, 8)])
def test_gemm_scatter_epilogue_and_peer_push(M, N, K, world):
    """D3_EP_SCATTER: the weight-gradient tile is added into the slice owner's buffer (here `world` local buffers stand
    in for the peers' NVLink mappings); d3_scatter_add_peers does the same for a flat range.  Two "ranks" contribute."""
    from dinov3_jax import ops
    total = ((M * N + 8 * world - 1) // (8 * world)) * 8 * world + 64 * world     # tensor sits at offset 64 in the range
    shard = total // world
    shards = [torch.zeros(shard, device="cuda") for _ in range(world)]
    peers = [t.data_ptr() for t in shards]
    ref = torch.zeros(total, device="cuda")
    for seed in (0, 1):
        g = torch.Generator(device="cuda").manual_seed(seed)
        a = torch.randn(K, M, device="cuda", generator=g).to(torch.bfloat16)       # a^T b with a stored [K, M]
        b = torch.randn(K, N, device="cuda", generator=g).to(torch.bfloat16)
        geom = torch.empty(M, N, device="cuda")
        ops.gemm(a, b, geom, a_mn=True, b_mn=True, accum=True, scatter=(peers, 64, shard), alpha=0.5)
        ref[64:64 + M * N] += 0.5 * (a.float().t() @ b.float()).reshape(-1)
    got = torch.cat(shards)
    assert rel(got, ref) < 2e-3
    # flat push of a vector range at an offset
    src = torch.randn(8 * world * 5, device="cuda")
    ops.scatter_add_peers(src, peers, 8 * world, shard, 0.25)
    ref[8 * world: 8 * world + src.numel()] += 0.25 * src
    assert rel(torch.cat(shards), ref) < 2e-3


def test_token_assembly_with_storage_tokens_bit_exact():
    from dinov3_jax import ops
    n, P, R, D = 3, 16, 4, 128
    tok = torch.randn(n * P, D, device="cuda"); cls = torch.randn(D, device="cuda"); st = torch.randn(R * D, device="cuda")
    mt = torch.randn(D, device="cuda"); masks = (torch.rand(n, P, device="cuda") < 0.4)
    X = torch.empty(n, 1 + R + P, D, device="cuda")
    ops.assemble_tokens(tok, cls, mt, masks.to(torch.uint8).contiguous(), X, n, P, D, storage=st)
    ref = torch.cat([cls.expand(n, 1, D), st.view(1, R, D).expand(n, R, D),
                     torch.where(masks[..., None], mt.view(1, 1, D), tok.view(n, P, D))], dim=1)
    assert torch.equal(X, ref)
    dX = torch.randn(n, 1 + R + P, D, device="cuda")
    dTok = torch.empty(n * P, D, device="cuda", dtype=torch.bfloat16)
    dcls, dst, dm = torch.zeros(D, device="cuda"), torch.zeros(R * D, device="cuda"), torch.zeros(D, device="cuda")
    ops.assemble_tokens_bwd(dX, masks.to(torch.uint8).contiguous(), dTok, dcls, dm, n, P, D, dstorage=dst)
    assert rel(dcls, dX[:, 0].sum(0)) < 1e-6 and rel(dst.view(R, D), dX[:, 1:1 + R].sum(0)) < 1e-6
    dp = dX[:, 1 + R:]
    assert rel(dm, (dp * masks[..., None]).sum((0, 1))) < 1e-6
    assert torch.equal(dTok.view(n, P, D), torch.where(masks[..., None], torch.zeros_like(dp), dp).to(torch.bfloat16))
    idx = masks.flatten().nonzero().flatten()
    rows = torch.empty(idx.numel(), dtype=torch.int32, device="cuda")
    ops.token_rows(idx, rows, idx.numel(), P, 0, prefix=1 + R)
    assert torch.equal(X.view(-1, D)[rows.long()], mt.expand(idx.numel(), D))        # masked rows hold the mask token


def test_swiglu_gate_forward_backward():
    from dinov3_jax import ops
    T, Hs = 1000, 344
    x12 = (torch.randn(T, 2 * Hs, device="cuda") * 1.5).to(torch.bfloat16)
    dh = torch.randn(T, Hs, device="cuda").to(torch.bfloat16)
    h = torch.empty(T, Hs, device="cuda", dtype=torch.bfloat16)
    dx12 = torch.empty(T, 2 * Hs, device="cuda", dtype=torch.bfloat16)
    ops.swiglu_fwd(x12, h)
    ops.swiglu_bwd(x12, dh, dx12)
    x = x12.float().requires_grad_(True)
    ref = torch.nn.functional.silu(x[:, :Hs]) * x[:, Hs:]
    ref.backward(dh.float())
    assert rel(h, ref) < BF16_TOL and rel(dx12, x.grad) < BF16_TOL


@pytest.mark.parametrize("n,world,op", [(2 * 65536 + 4, 8, "sum"), (2 * 65536, 2, "max"), (3, 4, "sum"), (1031, 3, "max")])
def test_allreduce_peers_matches_rank_ordered_reduction(n, world, op):
    """d3_allreduce_peers: `world` local buffers stand in for the ranks' symmetric staging buffers; the result is the
    reduction in rank order (bit-exact against the same order in torch), also for unaligned views and n % 4 != 0."""
    from dinov3_jax import ops
    g = torch.Generator(device="cuda").manual_seed(n + world)
    base = [torch.randn(n + 4, device="cuda", generator=g) for _ in range(world)]
    for shift in (0, 1):                                  # shift 1: 4-byte aligned only -> scalar path
        ins = [b[shift:shift + n] for b in base]
        out = torch.full((n,), float("nan"), device="cuda")
        ops.allreduce_peers([t.data_ptr() for t in ins], out, n, op)
        ref = ins[0].clone()
        for t in ins[1:]:
            ref = ref + t if op == "sum" else torch.maximum(ref, t)
        assert torch.equal(out, ref)


# --------------------------------------------------------------------------------------------------- Gram loss (8f.2)
def _gram_gpu(fs, ft, mode, weight=1.0, n_valid=None):
    """Loss and d(weight * loss)/d(fs) of loss/gram_loss.py through the library: l2norm -> two similarity GEMMs ->
    d3_gram_diff -> backward GEMM -> l2norm backward.  fs, ft: fp32 [n, D] on the GPU (n % 8 == 0, D % 8 == 0)."""
    from dinov3_jax import ops
    n, D = fs.shape
    nv = n if n_valid is None else n_valid
    bf, f32 = torch.bfloat16, torch.float32
    xs, xt = torch.empty(n, D, dtype=bf, device="cuda"), torch.empty(n, D, dtype=bf, device="cuda")
    ns, nt = torch.empty(n, device="cuda"), torch.empty(n, device="cuda")
    ops.l2norm_fwd(fs, xs, ns, 1e-12)
    ops.l2norm_fwd(ft, xt, nt, 1e-12)
    Ss, St = torch.empty(n, n, device="cuda"), torch.empty(n, n, device="cuda")
    ops.gemm(xt, xt, St)
    ops.gemm(xs, xs, Ss)
    G = torch.empty(n, n, dtype=bf, device="cuda")
    loss = torch.zeros(1, device="cuda")
    inv = 1.0 / (nv * nv)
    ops.gram_diff(Ss, St, G, mode, inv, loss)
    dX = torch.empty(n, D, dtype=bf, device="cuda")
    ops.gemm(G, xs, dX, b_mn=True, alpha=4.0 * weight * inv)
    dF = torch.empty(n, D, dtype=bf, device="cuda")
    ops.l2norm_bwd(dX, fs, ns, dF)
    return float(loss.item()), dF.float()


@pytest.mark.parametrize("remove_neg,only_teacher", [(True, False), (False, True), (False, False)])
def test_gram_loss_forward_backward_match_oracle(remove_neg, only_teacher):
    """SURVEY 8f.2: the Gram-anchoring loss over a batch of patch tokens (img_level false) and its gradient w.r.t. the
    student features, against oracle.losses.gram_loss (pinned to the reference's GramLoss) under autograd."""
    from dinov3_jax import ops
    from oracle.losses import gram_loss
    n, D = 384, 128
    g = torch.Generator().manual_seed(5)
    base = torch.randn(n, D, generator=g)
    fs = (base + 0.5 * torch.randn(n, D, generator=g)).requires_grad_(True)
    ft = base + 0.5 * torch.randn(n, D, generator=g)
    ref = gram_loss(fs[None].double(), ft[None].double(), img_level=False, remove_neg=remove_neg, remove_only_teacher_neg=only_teacher)
    (gref,) = torch.autograd.grad(ref, fs)
    loss, dF = _gram_gpu(fs.detach().cuda(), ft.cuda(), ops.GRAM_MODES[(remove_neg, only_teacher)])
    ref_v = float(ref.detach())
    assert abs(loss - ref_v) < 2e-2 * ref_v                      # bf16 operands of the similarity GEMMs
    err = float((dF.cpu() - gref.float()).norm() / gref.float().norm())
    assert err < 3e-2, err


def test_gram_loss_reference_golden_value():
    """The batch-level value the reference's own GramLoss produced for the committed fixture (tests/golden/make_golden.py:
    27 tokens x 16 channels, zero-padded here to the kernels' 8-element granularity; zero rows add nothing to the sum)."""
    import numpy as np
    import os
    from conftest import reference_vectors
    G = reference_vectors()
    s, t = torch.from_numpy(G["gram_s"]).float().reshape(-1, 16), torch.from_numpy(G["gram_t"]).float().reshape(-1, 16)
    n = s.shape[0]
    pad = lambda x: torch.nn.functional.pad(x, (0, 64 - 16, 0, 32 - n)).contiguous().cuda()
    loss, _ = _gram_gpu(pad(s), pad(t), 1, n_valid=n)
    assert abs(loss - float(G["gram_batch"])) < 2e-2 * float(G["gram_batch"])


@pytest.mark.parametrize("Hs,Hd,aa", [(20, 14, False), (20, 14, True), (6, 4, False), (4, 7, False), (32, 14, True), (5, 5, False)])
def test_resize_tokens_bicubic_matches_torch_interpolate(Hs, Hd, aa):
    """d3_resize_tokens_bicubic (gram teacher features -> student patch grid) against torch.nn.functional.interpolate,
    mode bicubic, align_corners False, with and without antialias."""
    from dinov3_jax import ops
    n, D = 3, 72
    g = torch.Generator().manual_seed(Hs * 100 + Hd)
    x = torch.randn(n, Hs, Hs + 1, D, generator=g)                       # non-square source: Ws = Hs + 1
    ref = torch.nn.functional.interpolate(x.permute(0, 3, 1, 2), size=(Hd, Hd + 2), mode="bicubic", align_corners=False,
                                          antialias=aa).permute(0, 2, 3, 1).contiguous()
    out = torch.empty(n, Hd, Hd + 2, D, device="cuda")
    ops.resize_tokens_bicubic(x.cuda().contiguous(), out, n, Hs, Hs + 1, Hd, Hd + 2, D, aa)
    assert float((out.cpu() - ref).abs().max()) < 2e-5 * max(1.0, float(ref.abs().max()))


def test_gram_loss_class_against_the_reference_fixture():
    """dinov3_jax.loss.GramLoss (the reference's class name and call signature, loss/gram_loss.py:13-50) on the values the
    reference's own class produced for the committed fixture: per image and over the batch; and the block-diagonal
    (single-GEMM) form of the per-image loss against the oracle on aligned sizes."""
    import numpy as np
    import os
    from dinov3_jax.loss import GramLoss
    from oracle.losses import gram_loss
    from conftest import reference_vectors
    G = reference_vectors()
    s, t = torch.from_numpy(G["gram_s"]).float().cuda(), torch.from_numpy(G["gram_t"]).float().cuda()
    gl = GramLoss()
    assert abs(float(gl(s, t, img_level=True)) - float(G["gram_img"])) < 2e-2 * float(G["gram_img"])
    assert abs(float(gl(s, t, img_level=False)) - float(G["gram_batch"])) < 2e-2 * float(G["gram_batch"])
    g = torch.Generator().manual_seed(1)
    s2, t2 = torch.randn(4, 16, 64, generator=g), torch.randn(4, 16, 64, generator=g)
    for kw in (dict(remove_neg=True, remove_only_teacher_neg=False), dict(remove_neg=False, remove_only_teacher_neg=True)):
        ref = float(gram_loss(s2.double(), t2.double(), img_level=True, **kw))
        got = float(GramLoss(**kw)(s2.cuda(), t2.cuda(), img_level=True))
        assert abs(got - ref) < 2e-2 * ref, (kw, got, ref)
