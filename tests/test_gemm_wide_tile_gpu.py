"""-m gpu: the GEMM's 128 x 256 tile (tile_n = 256), which both consumer warpgroups share, in 2-CTA clusters paired
along M that multicast the weight operand.  Every output element keeps its accumulation chain (the same k-blocks,
k16 steps and split-K slices in the same order), so each result is checked against PyTorch fp32 and, bit for bit,
against tile_n = 128 on the same inputs.  Shapes: N not a multiple of 256, an odd number of M tiles (the last M pair's
second tile lies past M), K not a multiple of 64, work lists shorter than the grid, and split-K weight gradients."""
import pytest
import torch

from gemm_epilogue_helpers import BF16_TOL, inputs, reference, rel, run

pytestmark = pytest.mark.gpu

M, K = 600, 200          # 5 M tiles, the last one 88 rows; 4 k-blocks, the last one 8 deep
PAD = (5, 24)            # the output is an [M, N] view into an [M + 5, N + 24] buffer
OFFSET = 64              # elements of sentinels before the view (keeps it 16-byte aligned: the fixed-flag path)

# (A MN-major, B MN-major), epilogue features: every flag set compiled fixed
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


def same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int8), b.contiguous().view(torch.int8))


def wide_equals_narrow(x, pad=PAD, alpha=1.0, split_k=1):
    """tile_n = 256 into a view with sentinels before it, around it and past M, bit for bit against tile_n = 128."""
    wide, pre = run(x, 256, OFFSET, pad, alpha=alpha, split_k=split_k)
    narrow, pre_n = run(x, 128, 0, pad, alpha=alpha, split_k=split_k)
    assert not torch.isnan(wide).any()
    assert same_bits(wide, narrow)
    if pre is not None:
        assert not torch.isnan(pre).any()
        assert same_bits(pre, pre_n)
    return wide, pre


@pytest.mark.parametrize("n", [1000, 3072 + 64])
@pytest.mark.parametrize("layout,feats", VARIANTS)
def test_wide_tile_matches_fp32_and_tile_128(layout, feats, n):
    x = inputs(layout, feats, M, K, n, 0.1)
    for alpha in (1.0, 0.37):
        u, ref = reference(x, alpha)
        wide, pre = wide_equals_narrow(x, alpha=alpha)
        tol = BF16_TOL if "f32" not in feats else (5e-4 if "gelu" in feats else 1e-5)   # GELU: hardware tanh (2^-11)
        assert rel(wide, ref) < tol
        if pre is not None:
            assert rel(pre, u) < BF16_TOL
        if x["resid"] is not None:            # resid is out: every element is read before it is overwritten
            in_place, _ = run(x, 256, 0, PAD, in_place=True, alpha=alpha)
            assert same_bits(in_place, wide)


@pytest.mark.parametrize("m,n", [(128, 256), (100, 64), (300, 512), (77, 640)])
@pytest.mark.parametrize("layout,feats", [((0, 1), ("bias", "gelu", "pre")),
                                          ((0, 0), ("dgelu",)),
                                          ((1, 1), ("f32", "accum"))])
def test_wide_tile_work_list_shorter_than_grid(layout, feats, m, n):
    """One or a few tile pairs: the second M tile of a pair lies wholly or partly past M, N may be below 256."""
    x = inputs(layout, feats, m, 256, n, 256 ** -0.5)
    wide, _ = wide_equals_narrow(x, pad=(3, 128))
    assert rel(wide, reference(x, 1.0)[1]) < (BF16_TOL if "f32" not in feats else 1e-5)


def test_wide_tile_forced_split_k_at_ragged_m():
    """M = 1000 leaves every slab's last row tile ragged and its M pair incomplete; N = 320 is one full and one
    ragged N tile."""
    x = inputs((1, 1), ("f32", "accum"), 1000, 1024, 320, 0.1)
    wide, _ = wide_equals_narrow(x, pad=(5, 192), split_k=3)
    assert rel(wide, x["init"] + x["A"].float() @ x["B"].float()) < 1e-5


@pytest.mark.parametrize("m,n", [(1024, 3072), (1024, 1024), (4096, 1024)])
def test_wide_tile_auto_split_at_step_shapes(m, n):
    """The weight gradients of qkv, proj and fc2 over the student tokens of one step, at the automatic split-K count:
    the split count (and so the slab order) is that of tile_n = 128.  The automatic tile choice (the wide tile for
    this layout) gives the same bits."""
    x = inputs((1, 1), ("f32", "accum"), m, 44160, n, 44160 ** -0.5)
    wide, _ = wide_equals_narrow(x, pad=(0, 0), split_k=0)
    auto, _ = run(x, 0, 0, (0, 0), split_k=0)
    assert same_bits(auto, wide)
