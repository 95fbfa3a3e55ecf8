"""-m gpu: the GEMM's 2-CTA clusters, where the pair of N tiles a cluster computes is incomplete or the work list is
short.  The second tile of a pair lies wholly beyond N when the N-tile count is odd: that CTA still loads and multicasts
its half of A but must store nothing (its columns are checked against the sentinels of a padded output view).  A work
list shorter than the grid, split-K slabs at a ragged M and the fused reduce-scatter (D3_EP_SCATTER) also go through a
pair.  Each result is checked against PyTorch fp32 and, bit for bit, against the epilogue that reads its flags at run
time (an output view one element off 16-byte alignment selects that path on the same data)."""
import pytest
import torch

from gemm_epilogue_helpers import BF16_TOL, fixed_and_runtime, inputs, reference, rel, run

pytestmark = pytest.mark.gpu

# (A MN-major, B MN-major), epilogue features: a staged forward, a staged input gradient, a weight gradient
LAYOUTS = [((0, 1), ("bias", "gelu", "pre")),
           ((0, 0), ("dgelu",)),
           ((1, 1), ("f32", "accum"))]


@pytest.fixture(autouse=True)
def _seed(native):
    torch.manual_seed(0)


def check(x, bn, pad):
    u, ref = reference(x, 1.0)
    out, pre = fixed_and_runtime(x, bn, pad)
    assert rel(out, ref) < (BF16_TOL if "f32" not in x["feats"] else 1e-5)
    if pre is not None:
        assert rel(pre, u) < BF16_TOL


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("layout,feats", LAYOUTS)
def test_ragged_pair_stores_nothing_past_n(layout, feats, bn):
    """N = 320 is 5 tiles of 64 or 3 of 128: the last pair's second tile starts at or past N.  The view's 192 padding
    columns cover that tile's columns."""
    check(inputs(layout, feats, 1000, 384, 320, 384 ** -0.5), bn, pad=(5, 192))


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("m,n", [(128, 64), (100, 128), (77, 640)])
@pytest.mark.parametrize("layout,feats", LAYOUTS)
def test_work_list_shorter_than_grid(layout, feats, m, n, bn):
    """One tile (one pair, half of it or all of it live), and M < 128 (A's second 64-row half lies past M)."""
    check(inputs(layout, feats, m, 256, n, 256 ** -0.5), bn, pad=(3, 128))


@pytest.mark.parametrize("bn", [64, 128])
def test_split_k_pairs_at_ragged_m(bn):
    """M = 1000 leaves every slab's last row tile ragged, N = 320 leaves the last pair ragged.  The slabs of N = 320
    (fixed epilogue) against those of N = 316 (N % 4 != 0 runs the run-time epilogue) over the same first columns."""
    from dinov3_jax import ops
    x = inputs((1, 1), ("f32", "accum"), 1000, 1024, 320, 0.1)
    out, _ = run(x, bn, 0, (5, 192), split_k=3)
    assert rel(out, x["init"] + x["A"].float() @ x["B"].float()) < 1e-5
    narrow = x["init"][:, :316].contiguous()
    ops.gemm(x["A_st"], x["B_st"][:, :316], narrow, a_mn=True, b_mn=True, accum=True, tile_n=bn, split_k=3)
    assert torch.equal(out[:, :316].contiguous().view(torch.int8), narrow.view(torch.int8))


@pytest.mark.parametrize("bn", [64, 128])
def test_scatter_through_a_ragged_pair(bn):
    """D3_EP_SCATTER with one rank: every output element is added once into a zeroed shard at an offset, which gives
    the bits of the fixed-flag accumulate into zeros; the shard's elements around the output stay zero."""
    from dinov3_jax import ops
    m, n, off = 1000, 320, 8
    x = inputs((1, 1), ("f32", "accum"), m, 512, n, 0.1)
    x["init"] = torch.zeros(m, n, device="cuda")
    fixed, _ = fixed_and_runtime(x, bn)
    shard = torch.zeros(off + m * n + 8, device="cuda")
    geometry = torch.empty(m, n, device="cuda")
    ops.gemm(x["A_st"], x["B_st"], geometry, a_mn=True, b_mn=True, tile_n=bn, split_k=1,
             scatter=([shard.data_ptr()], off, shard.numel()))
    torch.cuda.synchronize()
    assert not shard[:off].any() and not shard[off + m * n:].any()
    scattered = shard[off: off + m * n].view(m, n)
    assert rel(scattered, x["A"].float() @ x["B"].float()) < 1e-5
    assert torch.equal(scattered.view(torch.int8), fixed.view(torch.int8))
