"""-m gpu: the GEMM epilogues compiled with their flags fixed (one per flag set a training step issues), at ragged M and
N, into column-slice views, in place, accumulated and split-K.  Each result is checked against PyTorch fp32 and, bit for
bit, against the epilogue that reads its flags at run time: an output view one element off 16-byte alignment selects
that path on the same data."""
import pytest
import torch

pytestmark = pytest.mark.gpu

BF16_TOL = 6e-3          # norm-wise relative error of a bf16-stored result
M, N, K = 3771, 200, 320
PAD_R, PAD_C = 5, 24     # the output is a [M, N] view into a [M + PAD_R, N + PAD_C] buffer
SENTINEL = 12345.0
bf16, f32 = torch.bfloat16, torch.float32

# (A MN-major, B MN-major), epilogue features
VARIANTS = [
    ((0, 1), ("bias",)),
    ((0, 1), ("bias", "f32")),
    ((0, 1), ("bias", "gelu")),
    ((0, 1), ("bias", "gelu", "pre")),
    ((0, 1), ("bias", "gamma", "resid", "f32")),
    ((0, 1), ("bias", "pre", "gamma", "resid", "f32")),
    ((0, 1), ("bias", "gelu", "gamma", "resid", "f32")),
    ((0, 1), ("bias", "gelu", "pre", "gamma", "resid", "f32")),
    ((0, 1), ("f32",)),
    ((0, 0), ()),
    ((0, 0), ("dgelu",)),
    ((0, 0), ("f32",)),
    ((1, 1), ("f32", "accum")),
]


def rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-30)).item()


@pytest.fixture(autouse=True)
def _seed(native):
    torch.manual_seed(0)


def _transposed(X):
    """X^T as a column slice of a buffer whose rows are padded to a multiple of 8 elements (TMA's 16-byte stride)."""
    r = X.shape[0]
    buf = torch.zeros(X.shape[1], (r + 7) // 8 * 8, device="cuda", dtype=X.dtype)
    buf[:, :r] = X.t()
    return buf[:, :r]


def _operands(a_mn, b_mn, k=K, n=N):
    A = torch.randn(M, k, device="cuda").to(bf16)
    B = (torch.randn(k, n, device="cuda") * 0.1).to(bf16)
    return A, B, (_transposed(A) if a_mn else A), (B if b_mn else B.t().contiguous())


def _padded(dtype, fill, offset):
    """A [M, N] view holding `fill` in a buffer of sentinels; the view starts `offset` elements into the buffer."""
    ld = N + PAD_C
    flat = torch.full(((M + PAD_R) * ld + offset,), SENTINEL, device="cuda", dtype=dtype)
    view = flat[offset: offset + M * ld].view(M, ld)[:, :N]
    view.copy_(fill)
    outside = torch.ones_like(flat, dtype=torch.bool)
    outside[offset: offset + M * ld].view(M, ld)[:, :N] = False
    return flat, view, outside


def _reference(acc, feats, bias, gamma, resid, ub, init):
    u = acc + bias if "bias" in feats else acc
    y = torch.nn.functional.gelu(u, approximate="tanh") if "gelu" in feats else u
    if "dgelu" in feats:
        uf = ub.float().requires_grad_(True)
        torch.nn.functional.gelu(uf, approximate="tanh").sum().backward()
        y = y * uf.grad
    if "gamma" in feats:
        y = y * gamma
    if "resid" in feats:
        y = y + resid
    if "accum" in feats:
        y = y + init
    return u, y


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("layout,feats", VARIANTS)
def test_fixed_epilogue_matches_fp32_and_runtime_path(layout, feats, bn):
    from dinov3_jax import ops
    a_mn, b_mn = layout
    A, B, A_st, B_st = _operands(a_mn, b_mn)
    acc = A.float() @ B.float()
    odt = f32 if "f32" in feats else bf16
    bias = torch.randn(N, device="cuda") if "bias" in feats else None
    gamma = torch.randn(N, device="cuda") if "gamma" in feats else None
    resid = torch.randn(M, N, device="cuda") if "resid" in feats else None
    ub = torch.randn(M, N, device="cuda").to(bf16) if "dgelu" in feats else None
    init = torch.randn(M, N, device="cuda") if "accum" in feats else float("nan")
    u, ref = _reference(acc, feats, bias, gamma, resid, ub, init)

    def run(offset, in_place=False):
        flat, out, outside = _padded(odt, resid if in_place else init, offset)
        pre = torch.full((M, N), float("nan"), device="cuda", dtype=bf16) if "pre" in feats else None
        r = out if in_place else (resid.clone() if resid is not None else None)
        ops.gemm(A_st, B_st, out, a_mn=bool(a_mn), b_mn=bool(b_mn), bias=bias, gelu="gelu" in feats, store_pre=pre,
                 dgelu_of=ub, gamma=gamma, resid=r, accum="accum" in feats, tile_n=bn, split_k=1)
        torch.cuda.synchronize()
        assert bool((flat[outside] == SENTINEL).all()), "padding columns or rows past M were written"
        return out.contiguous(), pre

    fixed, pre = run(0)
    runtime, pre_rt = run(1)
    tol = BF16_TOL if odt == bf16 else (5e-4 if "gelu" in feats else 1e-5)
    assert not torch.isnan(fixed).any()
    assert rel(fixed, ref) < tol
    assert torch.equal(fixed.view(torch.int8), runtime.view(torch.int8))
    if pre is not None:
        assert rel(pre, u) < BF16_TOL
        assert torch.equal(pre.view(torch.int8), pre_rt.view(torch.int8))
    if resid is not None:                     # resid is out: every element is read before it is overwritten
        assert torch.equal(run(0, in_place=True)[0].view(torch.int8), fixed.view(torch.int8))
        assert torch.equal(run(1, in_place=True)[0].view(torch.int8), fixed.view(torch.int8))


@pytest.mark.parametrize("bn", [64, 128])
def test_split_k_slabs_match_fp32_and_runtime_path(bn):
    """Weight-gradient layout, split-K: the slabs of N = 200 (fixed epilogue) against those of N = 198 (N % 4 != 0
    runs the run-time epilogue), which compute the same first 198 columns from the same operands."""
    from dinov3_jax import ops
    k = 1024
    A, B, A_st, B_st = _operands(1, 1, k=k)
    init = torch.randn(M, N, device="cuda")
    flat, out, outside = _padded(f32, init, 0)
    ops.gemm(A_st, B_st, out, a_mn=True, b_mn=True, accum=True, tile_n=bn, split_k=3)
    torch.cuda.synchronize()
    assert bool((flat[outside] == SENTINEL).all())
    assert rel(out, init + A.float() @ B.float()) < 1e-5
    narrow = init[:, :198].contiguous()
    ops.gemm(A_st, B_st[:, :198], narrow, a_mn=True, b_mn=True, accum=True, tile_n=bn, split_k=3)
    assert torch.equal(out[:, :198].contiguous().view(torch.int8), narrow.view(torch.int8))
