"""-m gpu: the GEMM epilogues that store through shared memory with TMA, at the shapes of a ViT-L/16 student block
(M = 44 160 tokens) and at the edges TMA clips (M < 128, N a multiple of 64 but not of 128).  Each staged result is
checked bit for bit against the epilogue that reads its flags at run time and stores from registers: an output view one
element off 16-byte alignment selects that path on the same data.  Also: split-K slabs at a ragged M, whose partial
tiles must stay inside their own slab."""
import pytest
import torch

pytestmark = pytest.mark.gpu

T = 44160                # tokens of the student stream at B = 64
D, HD = 1024, 4096
bf16, f32 = torch.bfloat16, torch.float32

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


def _inputs(layout, feats, m, k, n):
    a_mn, b_mn = layout
    A = torch.randn(m, k, device="cuda").to(bf16)
    B = (torch.randn(k, n, device="cuda") * k ** -0.5).to(bf16)
    if not b_mn:
        B = B.t().contiguous()
    x = dict(A=A, B=B, a_mn=bool(a_mn), b_mn=bool(b_mn), gelu="gelu" in feats)
    x["bias"] = torch.randn(n, device="cuda") if "bias" in feats else None
    x["gamma"] = torch.randn(n, device="cuda") if "gamma" in feats else None
    x["resid"] = torch.randn(m, n, device="cuda") if "resid" in feats else None
    x["dgelu_of"] = torch.randn(m, n, device="cuda").to(bf16) if "dgelu" in feats else None
    return x


def _run(x, feats, m, n, bn, offset, in_place=False):
    """The GEMM into an [m, n] output that starts `offset` elements into its buffer (NaN-prefilled)."""
    from dinov3_jax import ops
    odt = f32 if "f32" in feats else bf16
    flat = torch.full((m * n + offset,), float("nan"), device="cuda", dtype=odt)
    out = flat[offset:].view(m, n)
    pre = torch.full((m, n), float("nan"), device="cuda", dtype=bf16) if "pre" in feats else None
    resid = x["resid"]
    if in_place:
        out.copy_(resid)
        resid = out
    elif resid is not None:
        resid = resid.clone()
    ops.gemm(x["A"], x["B"], out, a_mn=x["a_mn"], b_mn=x["b_mn"], bias=x["bias"], gelu=x["gelu"], store_pre=pre,
             dgelu_of=x["dgelu_of"], gamma=x["gamma"], resid=resid, tile_n=bn, split_k=1)
    torch.cuda.synchronize()
    return out.clone(), pre


def _check_against_runtime(layout, feats, m, k, n, bn):
    x = _inputs(layout, feats, m, k, n)
    staged, pre = _run(x, feats, m, n, bn, 0)
    runtime, pre_rt = _run(x, feats, m, n, bn, 1)
    assert not torch.isnan(staged).any()
    assert torch.equal(staged.view(torch.int8), runtime.view(torch.int8))
    if pre is not None:
        assert not torch.isnan(pre).any()
        assert torch.equal(pre.view(torch.int8), pre_rt.view(torch.int8))
    return x, staged


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("layout,feats,k,n", STUDENT)
def test_staged_epilogue_matches_runtime_path_at_student_shapes(layout, feats, k, n, bn):
    _check_against_runtime(layout, feats, T, k, n, bn)


@pytest.mark.parametrize("bn", [64, 128])
def test_staged_epilogue_in_place_residual_at_full_size(bn):
    feats = ("bias", "pre", "gamma", "resid", "f32")
    x, staged = _check_against_runtime((0, 1), feats, T, D, D, bn)
    in_place, _ = _run(x, feats, T, D, bn, 0, in_place=True)
    assert torch.equal(in_place.view(torch.int8), staged.view(torch.int8))


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("m,n", [(100, 256), (3771, 192), (77, 192), (100, 224)])
@pytest.mark.parametrize("layout,feats", [((0, 1), ("bias", "gelu", "pre")),
                                          ((0, 1), ("bias", "pre", "gamma", "resid", "f32")),
                                          ((0, 0), ("dgelu",))])
def test_staged_epilogue_clips_ragged_rows_and_columns(layout, feats, m, n, bn):
    _check_against_runtime(layout, feats, m, 320, n, bn)


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
