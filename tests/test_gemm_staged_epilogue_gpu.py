"""-m gpu: the GEMM epilogues that store through shared memory with TMA, at the shapes of a ViT-L/16 student block
(M = 44 160 tokens) and at the edges TMA clips (M < 128, N a multiple of 64 but not of 128).  Each staged result is
checked bit for bit against the epilogue that reads its flags at run time: an output view one element off 16-byte
alignment selects that path on the same data.  Also: split-K slabs at a ragged M, whose partial tiles must stay inside
their own slab."""
import pytest
import torch

from gemm_epilogue_helpers import bf16, fixed_and_runtime, inputs, run

pytestmark = pytest.mark.gpu

T = 44160                # tokens of the student stream at B = 64
D, HD = 1024, 4096

# (A MN-major, B MN-major), epilogue features, K, N: the call each staged variant serves in a training step
STUDENT = [
    ((0, 1), ("bias",), D, 3 * D),                                   # qkv
    ((0, 1), ("bias", "gelu", "pre"), D, HD),                        # fc1
    ((0, 1), ("bias", "gelu"), D, HD),                               # fc1, teacher
    ((0, 1), ("bias", "pre", "gamma", "resid", "f32"), D, D),        # proj
    ((0, 1), ("bias", "gamma", "resid", "f32"), D, D),               # proj, teacher
    ((0, 1), ("bias", "gelu", "pre", "gamma", "resid", "f32"), HD, D),
    ((0, 1), ("bias", "gelu", "gamma", "resid", "f32"), HD, D),
    ((0, 1), ("bias", "f32"), D, D),
    ((0, 1), ("f32",), D, D),
    ((0, 0), (), HD, D),                                             # dgrad fc1
    ((0, 0), ("dgelu",), D, HD),                                     # dgrad fc2
    ((0, 0), ("f32",), D, D),
]


@pytest.fixture(autouse=True)
def _seed(native):
    torch.manual_seed(0)


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("layout,feats,k,n", STUDENT)
def test_staged_epilogue_matches_runtime_path_at_student_shapes(layout, feats, k, n, bn):
    fixed_and_runtime(inputs(layout, feats, T, k, n, k ** -0.5), bn)


@pytest.mark.parametrize("bn", [64, 128])
def test_staged_epilogue_in_place_residual_at_full_size(bn):
    x = inputs((0, 1), ("bias", "pre", "gamma", "resid", "f32"), T, D, D, D ** -0.5)
    staged, _ = fixed_and_runtime(x, bn)
    in_place, _ = run(x, bn, 0, in_place=True)
    assert torch.equal(in_place.view(torch.int8), staged.view(torch.int8))


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("m,n", [(100, 256), (3771, 192), (77, 192), (100, 224)])
@pytest.mark.parametrize("layout,feats", [((0, 1), ("bias", "gelu", "pre")),
                                          ((0, 1), ("bias", "pre", "gamma", "resid", "f32")),
                                          ((0, 0), ("dgelu",))])
def test_staged_epilogue_clips_ragged_rows_and_columns(layout, feats, m, n, bn):
    fixed_and_runtime(inputs(layout, feats, m, 320, n, 320 ** -0.5), bn)


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("splits", [3, 5])
def test_split_k_slabs_stay_in_their_slab_at_ragged_m(splits, bn):
    """M = 1000 output rows leave the last row tile of every slab ragged; a partial tile stored past its slab's M rows
    would land in the next slab's first rows and change the sum."""
    from dinov3_jax import ops
    m, tokens, n = 1000, 2048, 256
    At = torch.zeros(tokens, 1008, device="cuda", dtype=bf16)[:, :m]    # A stored [tokens, m], rows 16-byte strided
    At.copy_(torch.randn(tokens, m, device="cuda"))
    B = (torch.randn(tokens, n, device="cuda") * tokens ** -0.5).to(bf16)
    init = torch.randn(m, n, device="cuda")
    out = init.clone()
    # weight-gradient layout: out[m, n] += At^T B, contraction over the tokens
    ops.gemm(At, B, out, a_mn=True, b_mn=True, accum=True, tile_n=bn, split_k=splits)
    torch.cuda.synchronize()
    ref = init.double() + At.double().t() @ B.double()
    assert ((out.double() - ref).norm() / ref.norm()).item() < 1e-5
