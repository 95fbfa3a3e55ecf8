"""Helpers of the GEMM epilogue tests (test_gemm_epilogue_variants_gpu.py, test_gemm_staged_epilogue_gpu.py): operands,
the fp32 reference, and a GEMM into an output view inside a buffer of sentinels.  An output view one element off 16-byte
alignment selects the epilogue that reads its flags at run time, on the same data as the fixed-flag one."""
import torch

BF16_TOL = 6e-3          # norm-wise relative error of a bf16-stored result
SENTINEL = 12345.0
bf16, f32 = torch.bfloat16, torch.float32


def rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-30)).item()


def _transposed(X):
    """X^T as a column slice of a buffer whose rows are padded to a multiple of 8 elements (TMA's 16-byte stride)."""
    r = X.shape[0]
    buf = torch.zeros(X.shape[1], (r + 7) // 8 * 8, device="cuda", dtype=X.dtype)
    buf[:, :r] = X.t()
    return buf[:, :r]


def inputs(layout, feats, m, k, n, b_scale):
    """Operands of an [m, n] GEMM with epilogue `feats`, stored in `layout` (A MN-major, B MN-major)."""
    a_mn, b_mn = layout
    A = torch.randn(m, k, device="cuda").to(bf16)
    B = (torch.randn(k, n, device="cuda") * b_scale).to(bf16)
    return dict(
        feats=feats, m=m, n=n, A=A, B=B, a_mn=bool(a_mn), b_mn=bool(b_mn),
        A_st=_transposed(A) if a_mn else A, B_st=B if b_mn else B.t().contiguous(),
        bias=torch.randn(n, device="cuda") if "bias" in feats else None,
        gamma=torch.randn(n, device="cuda") if "gamma" in feats else None,
        resid=torch.randn(m, n, device="cuda") if "resid" in feats else None,
        ub=torch.randn(m, n, device="cuda").to(bf16) if "dgelu" in feats else None,
        init=torch.randn(m, n, device="cuda") if "accum" in feats else float("nan"))


def reference(x, alpha):
    """(pre-activation, output) in fp32."""
    feats = x["feats"]
    acc = alpha * (x["A"].float() @ x["B"].float())
    u = acc + x["bias"] if "bias" in feats else acc
    y = torch.nn.functional.gelu(u, approximate="tanh") if "gelu" in feats else u
    if "dgelu" in feats:
        uf = x["ub"].float().requires_grad_(True)
        torch.nn.functional.gelu(uf, approximate="tanh").sum().backward()
        y = y * uf.grad
    if "gamma" in feats:
        y = y * x["gamma"]
    if "resid" in feats:
        y = y + x["resid"]
    if "accum" in feats:
        y = y + x["init"]
    return u, y


def run(x, bn, offset, pad=(0, 0), in_place=False, alpha=1.0, split_k=1):
    """The GEMM into an [m, n] view that starts `offset` elements into a buffer of sentinels with `pad` extra rows and
    columns; the view holds `init` (NaN unless accumulated) or, in place, the residual, and the stash is NaN-prefilled.
    Checks that nothing outside the view was written.  Returns (out, stash)."""
    from dinov3_jax import ops
    m, n, feats = x["m"], x["n"], x["feats"]
    ld = n + pad[1]
    flat = torch.full(((m + pad[0]) * ld + offset,), SENTINEL, device="cuda", dtype=f32 if "f32" in feats else bf16)
    out = flat[offset: offset + m * ld].view(m, ld)[:, :n]
    out.copy_(x["resid"] if in_place else x["init"])
    outside = torch.ones_like(flat, dtype=torch.bool)
    outside[offset: offset + m * ld].view(m, ld)[:, :n] = False
    pre = torch.full((m, n), float("nan"), device="cuda", dtype=bf16) if "pre" in feats else None
    resid = out if in_place else (x["resid"].clone() if x["resid"] is not None else None)
    ops.gemm(x["A_st"], x["B_st"], out, a_mn=x["a_mn"], b_mn=x["b_mn"], bias=x["bias"], gelu="gelu" in feats,
             store_pre=pre, dgelu_of=x["ub"], gamma=x["gamma"], resid=resid, accum="accum" in feats, alpha=alpha,
             tile_n=bn, split_k=split_k)
    torch.cuda.synchronize()
    assert bool((flat[outside] == SENTINEL).all()), "padding columns, rows past M or the bytes before the view were written"
    return out.contiguous(), pre


def fixed_and_runtime(x, bn, pad=(0, 0), alpha=1.0):
    """The fixed-flag result, checked complete and bit-identical to the run-time-flag one (output and stash)."""
    fixed, pre = run(x, bn, 0, pad, alpha=alpha)
    runtime, pre_rt = run(x, bn, 1, pad, alpha=alpha)
    assert not torch.isnan(fixed).any()
    assert torch.equal(fixed.view(torch.int8), runtime.view(torch.int8))
    if pre is not None:
        assert not torch.isnan(pre).any()
        assert torch.equal(pre.view(torch.int8), pre_rt.view(torch.int8))
    return fixed, pre
