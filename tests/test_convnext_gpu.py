"""-m gpu: the ConvNeXt backbone.  Each new kernel against torch (float64 where it computes, bit for bit where it only
moves or reuses the LayerNorm arithmetic), the erf-GELU GEMM instance against the run-time-flag epilogue, and
ConvNeXt.forward_features / get_intermediate_layers against the float64 restatement of upstream DINOv3
(tests/convnext_helpers.py)."""
import pytest
import torch
import torch.nn.functional as F

from convnext_helpers import forward_features, intermediate_layers, upstream_state_dict

pytestmark = pytest.mark.gpu
f32, bf16, f64 = torch.float32, torch.bfloat16, torch.float64


def rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


def bf16_ulp(x):
    """Spacing of bf16 numbers at |x| (8 significant bits)."""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -120)))
    return torch.exp2(e - 7)


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("C", [96, 128, 192, 384, 768, 1024, 1536])
def test_dwconv7_layernorm_within_one_bf16_ulp(native, C):
    from dinov3_jax import ops
    g = torch.Generator(device="cuda").manual_seed(C)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)
    w, wb = (rnd(49, C) / 7).contiguous(), 0.1 * rnd(C)
    sc, bi = 1 + 0.2 * rnd(C), 0.2 * rnd(C)
    for H, W in ((3, 5), (7, 7), (14, 14), (56, 56)):
        for n in (1, 3):
            X = (rnd(n, H, W, C) + 0.3).contiguous()
            Y = torch.empty(n * H * W, C, dtype=bf16, device="cuda")
            ops.dwconv7_layernorm(X, w, wb, sc, bi, Y)
            k = w.double().t().reshape(C, 1, 7, 7)
            conv = F.conv2d(X.double().permute(0, 3, 1, 2), k, wb.double(), padding=3, groups=C).permute(0, 2, 3, 1)
            conv = conv.reshape(-1, C)
            xhat = (conv - conv.mean(1, keepdim=True)) / torch.sqrt(conv.var(1, unbiased=False, keepdim=True) + 1e-6)
            want = xhat * sc.double() + bi.double()
            # the ulp at the size of the terms of the last add: where xhat * scale and bias cancel, the fp32 rounding
            # of those terms (not of the small result) sets the error
            mag = (xhat * sc.double()).abs() + bi.double().abs()
            err = (Y.double() - want).abs()
            assert bool((err <= bf16_ulp(mag)).all()), (C, H, W, n, (err / bf16_ulp(mag)).max().item())
    torch.cuda.synchronize()


def test_gelu_erf_epilogue_matches_runtime_flags_and_float64(native):
    """The fixed (0, 1, BIAS | GELU_ERF) instance against the run-time-flag epilogue (forced by a misaligned output),
    bit for bit, and against float64."""
    from dinov3_jax import ops
    g = torch.Generator(device="cuda").manual_seed(0)
    for M, K, N in ((3136, 96, 384), (784, 768, 3072), (200, 1536, 6144)):
        A = torch.randn(M, K, device="cuda", generator=g).to(bf16)
        B = (torch.randn(K, N, device="cuda", generator=g) * K ** -0.5).to(bf16)
        bias = 0.3 * torch.randn(N, device="cuda", generator=g)
        fast = torch.empty(M, N, dtype=bf16, device="cuda")
        ops.gemm(A, B, fast, b_mn=True, bias=bias, gelu_erf=True)
        wide = torch.zeros(M, N + 8, dtype=bf16, device="cuda")
        slow = wide[:, 1:N + 1]                                   # 2-byte offset: the run-time-flag path
        ops.gemm(A, B, slow, b_mn=True, bias=bias, gelu_erf=True)
        assert torch.equal(fast, slow), (M, K, N)
        want = F.gelu(A.double() @ B.double() + bias.double())
        assert (fast.double() - want).abs().max().item() <= 2e-2 * want.abs().max().item(), (M, K, N)
        assert rel(fast, want) < 4e-3, (M, K, N)


@pytest.mark.parametrize("C", [96, 192, 384, 768])
def test_layernorm_patchify2_is_layernorm_fwd_permuted(native, C):
    from dinov3_jax import ops
    g = torch.Generator(device="cuda").manual_seed(C)
    sc, bi = 1 + 0.2 * torch.randn(C, device="cuda", generator=g), 0.2 * torch.randn(C, device="cuda", generator=g)
    for n, H, W in ((1, 56, 56), (3, 14, 28), (2, 2, 6)):
        X = torch.randn(n, H, W, C, device="cuda", generator=g).contiguous()
        Y = torch.empty(n * (H // 2) * (W // 2), 4 * C, dtype=bf16, device="cuda")
        ops.layernorm_patchify2(X, sc, bi, Y)
        ln = torch.empty(n * H * W, C, dtype=bf16, device="cuda")
        ops.layernorm_fwd(X.view(-1, C), sc, bi, ln)
        want = ln.view(n, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, 4 * C)
        assert torch.equal(Y, want), (C, n, H, W)


def test_pool_tokens(native):
    from dinov3_jax import ops
    g = torch.Generator(device="cuda").manual_seed(1)
    for n, P, C in ((1, 49, 768), (3, 3136, 96), (2, 196, 1536), (16, 256, 1024)):
        X = (torch.randn(n, P, C, device="cuda", generator=g) + 1.0).contiguous()
        out = torch.full((n, 1 + P, C), float("nan"), device="cuda")
        ops.pool_tokens(X, out)
        assert torch.equal(out[:, 1:], X)
        assert rel(out[:, 0], X.double().mean(dim=1)) < 1e-6
        again = torch.full_like(out, float("nan"))
        ops.pool_tokens(X, again)
        assert torch.equal(again, out)
        only = torch.full((n, 5, C), 7.0, device="cuda")
        ops.pool_tokens(X, only, copy_tokens=False)
        assert torch.equal(only[:, 0], out[:, 0]) and bool((only[:, 1:] == 7.0).all())


@pytest.mark.parametrize("src,dst", [((56, 56), (14, 14)), ((28, 28), (14, 14)), ((14, 14), (14, 14)), ((7, 7), (14, 14)),
                                     ((20, 13), (14, 9)), ((16, 32), (32, 32))])
def test_resize_bilinear_aa_matches_torch(native, src, dst):
    """x4, x2, x1, x0.5 (up-scaling), non-integer factors, and a map scaled differently along H and W."""
    from dinov3_jax import ops
    g = torch.Generator(device="cuda").manual_seed(2)
    n, C = 3, 192
    X = torch.randn(n, *src, C, device="cuda", generator=g).contiguous()
    out = torch.full((n, 1 + dst[0] * dst[1], C), float("nan"), device="cuda")
    out[:, 0] = 5.0
    ops.resize_tokens_bilinear_aa(X, out, *dst, prefix=1)
    want = F.interpolate(X.double().permute(0, 3, 1, 2), size=dst, mode="bilinear", antialias=True)
    want = want.permute(0, 2, 3, 1).reshape(n, -1, C)
    assert bool((out[:, 0] == 5.0).all())
    assert (out[:, 1:].double() - want).abs().max().item() < 1e-5


# ------------------------------------------------------------------------------------------------ the model
def _model(size, seed, patch_size=None):
    from dinov3_jax.checkpointer import convert_convnext_torch_hub_state_dict
    from dinov3_jax.models import ConvNeXt, convnext_sizes
    arch = convnext_sizes[size] if isinstance(size, str) else size
    tree = convert_convnext_torch_hub_state_dict(upstream_state_dict(arch["depths"], arch["dims"], seed, dtype=f32))
    ref_tree = {k: v for k, v in tree.items()}
    return ConvNeXt(tree, **arch, patch_size=patch_size), ref_tree


def _tree_to(tree, device, dtype):
    return {k: (_tree_to(v, device, dtype) if isinstance(v, dict) else v.to(device, dtype)) for k, v in tree.items()}


@pytest.mark.parametrize("size,res", [("tiny", 224), ("base", 224), ("large", 224), ("base", 512)])
def test_forward_features_matches_restatement(native, size, res):
    model, tree = _model(size, seed=7)
    x = torch.randn(2, res, res, 3, generator=torch.Generator().manual_seed(res))
    got = model.forward_features(x.cuda())
    want = forward_features(_tree_to(tree, "cuda", f64), x.cuda().double())
    for key in ("x_norm_clstoken", "x_norm_patchtokens", "x_prenorm"):
        assert got[key].shape == want[key].shape, key
        assert rel(got[key], want[key]) < 2e-2, (key, rel(got[key], want[key]))
    assert got["x_storage_tokens"].shape == (2, 0, model.embed_dim) and got["masks"] is None
    assert torch.equal(model(x.cuda()), got["x_norm_clstoken"])


def test_intermediate_layers_bitwise_and_reproducible(native):
    """n=1, norm=True, no resize: the same bits as forward_features' normalised tokens; two calls, the same bits."""
    model, _ = _model("tiny", seed=8)
    x = torch.randn(2, 224, 224, 3, generator=torch.Generator().manual_seed(1)).cuda()
    ff = model.forward_features(x)
    (patches, cls), = model.get_intermediate_layers(x, n=1, return_class_token=True)
    assert torch.equal(patches, ff["x_norm_patchtokens"]) and torch.equal(cls, ff["x_norm_clstoken"])
    (shaped,) = model.get_intermediate_layers(x, n=1, reshape=True)
    assert torch.equal(shaped.flatten(2).transpose(1, 2), patches)
    a = model.get_intermediate_layers(x, n=[0, 1, 2, 3], return_class_token=True)
    b = model.get_intermediate_layers(x, n=[0, 1, 2, 3], return_class_token=True)
    for (pa, ca), (pb, cb) in zip(a, b):
        assert torch.equal(pa, pb) and torch.equal(ca, cb)
    ff2 = model.forward_features(x)
    assert torch.equal(ff2["x_norm_patchtokens"], ff["x_norm_patchtokens"])


@pytest.mark.parametrize("patch_size", [None, 16])
def test_intermediate_layers_match_restatement(native, patch_size):
    model, tree = _model("tiny", seed=9, patch_size=patch_size)
    x = torch.randn(2, 256, 192, 3, generator=torch.Generator().manual_seed(2))
    ref_tree = _tree_to(tree, "cuda", f64)
    for n in (4, [0, 2], 1):
        for norm in (True, False):
            for reshape in (False, True):
                got = model.get_intermediate_layers(x.cuda(), n=n, reshape=reshape, return_class_token=True, norm=norm)
                want = intermediate_layers(ref_tree, x.cuda().double(), n, patch_size=patch_size, reshape=reshape,
                                           return_class_token=True, norm=norm)
                assert len(got) == len(want)
                for (gp, gc), (wp, wc) in zip(got, want):
                    assert gp.shape == wp.shape and gc.shape == wc.shape, (n, norm, reshape)
                    assert rel(gp, wp) < 2e-2 and rel(gc, wc) < 2e-2, (n, norm, reshape, rel(gp, wp), rel(gc, wc))
    (p16,) = model.get_intermediate_layers(x.cuda(), n=[0], out_dtype=bf16)
    (p32,) = model.get_intermediate_layers(x.cuda(), n=[0])
    assert p16.dtype == bf16 and torch.equal(p16, p32.to(bf16))
