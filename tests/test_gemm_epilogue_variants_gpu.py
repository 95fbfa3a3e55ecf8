"""-m gpu: the GEMM epilogues compiled with their flags fixed (one per flag set a training step issues), at ragged M and
N, into column-slice views, in place, accumulated, with alpha = 1 and alpha != 1, and split-K.  Each result is checked
against PyTorch fp32 and, bit for bit, against the epilogue that reads its flags at run time: an output view one element
off 16-byte alignment selects that path on the same data."""
import pytest
import torch

from gemm_epilogue_helpers import BF16_TOL, fixed_and_runtime, inputs, reference, rel, run

pytestmark = pytest.mark.gpu

M, N, K = 3771, 200, 320
PAD = (5, 24)            # the output is a [M, N] view into a [M + 5, N + 24] buffer

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


@pytest.fixture(autouse=True)
def _seed(native):
    torch.manual_seed(0)


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("layout,feats", VARIANTS)
def test_fixed_epilogue_matches_fp32_and_runtime_path(layout, feats, bn):
    """alpha = 0.37 pins that both paths round alpha * acc on its own before the next step (alpha = 1 is exact)."""
    x = inputs(layout, feats, M, K, N, 0.1)
    for alpha in (1.0, 0.37):
        u, ref = reference(x, alpha)
        fixed, pre = fixed_and_runtime(x, bn, PAD, alpha)
        tol = BF16_TOL if "f32" not in feats else (5e-4 if "gelu" in feats else 1e-5)   # GELU: hardware tanh (2^-11)
        assert rel(fixed, ref) < tol
        if pre is not None:
            assert rel(pre, u) < BF16_TOL
        if x["resid"] is not None:            # resid is out: every element is read before it is overwritten
            for offset in (0, 1):
                in_place, _ = run(x, bn, offset, PAD, in_place=True, alpha=alpha)
                assert torch.equal(in_place.view(torch.int8), fixed.view(torch.int8))


@pytest.mark.parametrize("bn", [64, 128])
def test_split_k_slabs_match_fp32_and_runtime_path(bn):
    """Weight-gradient layout, split-K: the slabs of N = 200 (fixed epilogue) against those of N = 198 (N % 4 != 0
    runs the run-time epilogue), which compute the same first 198 columns from the same operands."""
    from dinov3_jax import ops
    x = inputs((1, 1), ("f32", "accum"), M, 1024, N, 0.1)
    out, _ = run(x, bn, 0, PAD, split_k=3)
    assert rel(out, x["init"] + x["A"].float() @ x["B"].float()) < 1e-5
    narrow = x["init"][:, :198].contiguous()
    ops.gemm(x["A_st"], x["B_st"][:, :198], narrow, a_mn=True, b_mn=True, accum=True, tile_n=bn, split_k=3)
    assert torch.equal(out[:, :198].contiguous().view(torch.int8), narrow.view(torch.int8))
